"""The recurrent and linear policy kernels (csrc/rexsim_agent.cu gru_policy_kernel, linear_policy_kernel) and the sampler all
four policy kernels share (head_outputs) at rounding level, against agent_restate.py's restatement of their own arithmetic.
test_gpu_recurrent_agent.py holds the cells to the fp64 oracle at 2e-4; this file asks what each kernel computes:

* Gate readouts.  Saturating a gate turns the cell's GEMMs into something the new state shows (state_dict()["hidden"] reads
  it, load_state_dict sets it): sigmoidf is exactly 1 at pre-activations >= 24 and exactly 0 at <= -96 (asserted on the
  CPU), and the saturating biases are powers of two past those limits by more than any |dot product| the inputs allow.
    carry      u = 1:                 h' = h, over several steps; the head sum is restated bit for bit, the mean within tanhf's
                                      2 ulp of tanh(s)
    candidate  r = 1, u = 0:          h' = tanhf(c), c restated bit for bit from the fmaf chain over [a1, h]
    reset      r = 0, u = 0:          the same with the h rows contributing exactly +-0
    u gate     w_c = 0, r = 1, h = 1: h' = sigmoidf(pre_u) within sigmoid_bound, pre_u restated bit for bit
    r gate     u = 0, w_c = [0; I], h = 1: h' = tanhf(sigmoidf(pre_r)) within the composed bound
    blend      the u readout with w_ru's h rows of u zero, the candidate readout, then both at once: h' equals
                                      fmaf(U, h, (1 - U) T) bit for bit, U and T the two readouts' device values
  Each on realistic weights (test_gpu_recurrent_agent._weights: the restated chains catch any reordering) and on exact
  networks (dyadic inputs, weights and states, every partial sum exact in fp32, asserted on the arrays: blind to order,
  they catch a wrong row, column or tile; non-zeros in the first and last row of every 16-row chunk, at k = H1 - 1 and H1
  and in the whole last chunk, in every column).  Every batch size of test_gpu_recurrent_agent.batch_sizes(), random begin
  masks, and the state rows n .. num_envs - 1 bit-unchanged.
* The full cell on realistic weights over 64 steps, free of trajectory divergence: each step is restated from the state
  the device held before it and held to agent_restate.gru_step_bound (its docstring derives it).
* The linear kernel: the head sum restated bit for bit (mean within tanhf's 2 ulp) on every row of every batch size, and
  exact networks at every LIN_ROWS shape with the 128-env tile edges.
* The sampler on the fp32, tensor-core, recurrent and linear cells: u1, u2 restated bit for bit
  ((k + 1/2) 2^-23, exact in fp32), z, the action and the log-prob within agent_restate's bounds, at the draws where
  logf is near 0 and at its largest argument range and where cospif is at its extremes and zeros, found by a vectorised
  search over the generator and run through env_offset; and the draw whose 24-bit uniform used to round to 1.0.
"""
import math

import numpy as np
import pytest
import torch

import agent_restate as R
from oracle import agent_oracle as AO
from oracle import recurrent_oracle as RO
from test_gpu_recurrent_agent import (LIN_ROWS, ROWS as AGENT_ROWS, SEED, _filters, _net, _probes, _sm, _weights,
                                      batch_sizes, row_id)

F32 = np.float32
KC = 16                                     # gru_gemm's rows per streamed chunk (RNN_KC)
ROWS = AGENT_ROWS + [  # (O, A, H1, G, value layers): the chunk geometry the agent rows miss
    (4, 2, 4, 4, (64, 12)),               # K = 8: one partial chunk; 16 of the block's 128 threads compute cell columns
    (4, 2, 20, 4, (64, 12)),              # K = 24: a short last chunk of 8 with the a1 -> h switch inside it
    (4, 2, 252, 8, (64, 12)),             # K = 260: 17 chunks, a last chunk of 4, the switch inside chunk 15
    (32, 8, 256, 128, (64, 12)),          # the largest shared-memory tile (174 KB)
]
READOUTS = ("carry", "candidate", "reset", "u_gate", "r_gate")
CELLS = ("fp32", "tensor_cores", "gru", "linear")
ONE_DRAW = (99, 1872961, 0, 0)              # (seed, global env, step, action) whose top 24 bits are all ones


# ---- networks ---------------------------------------------------------------------------------------------------------
def special_rows(H1, G):
    """The first and last row of every 16-row chunk, k = H1 - 1 and H1, and every row of the last chunk."""
    K = H1 + G
    nch = -(-K // KC)
    rows = {H1 - 1, H1} | set(range((nch - 1) * KC, K))
    for c in range(nch):
        rows.update((c * KC, min(c * KC + KC, K) - 1))
    return sorted(rows)


def _sparse(rng, shape, values, density, rows):
    x = np.where(rng.random(shape) < density, rng.choice(values, shape), 0.0)
    x[rows] = rng.choice(values, (len(rows), shape[1]))
    return x.astype(F32)


def exact_gru_network(O, A, H1, G, n, vl, seed=0):
    """(weights, observ mean, observations [n][O], states [n][G]) on dyadic grids, with filter count 0 (inv = 1): observations
    and means on 1/4 (a tenth beyond the clip), W1 in +-{1/16, 1/8}, b1 on 1/8, w_ru and w_c sparse in +-{1/32, 1/16, 1/8}
    with every special_rows row non-zero in every column, states on 1/8 in [-1, 1], W3 on 1/8 with rows 0 and G - 1
    non-zero, b3 non-zero.  The value network is _weights' (not read out here)."""
    rng = np.random.default_rng(seed + 1000 * O + 100 * A + H1 + G)
    K, rows = H1 + G, special_rows(H1, G)
    q = np.array([1, 2, 4]) / 32.0
    w = {k: v for k, v in _weights(rng, O, A, H1, G, vl).items() if k[0] == "v"}
    w.update(pW1=rng.choice([-0.125, -0.0625, 0.0625, 0.125], (O, H1)).astype(F32), pb1=(rng.integers(-8, 9, H1) / 8).astype(F32),
             w_ru=_sparse(rng, (K, 2 * G), np.r_[-q, q], 0.05, rows), b_ru=(rng.integers(-16, 17, 2 * G) / 8).astype(F32),
             w_c=_sparse(rng, (K, G), np.r_[-q, q], 0.05, rows), b_c=(rng.integers(-8, 9, G) / 8).astype(F32),
             pW3=_sparse(rng, (G, A), [-0.25, -0.125, 0.125, 0.25], 0.1, [0, G - 1]),
             pb3=rng.choice([-0.375, -0.125, 0.125, 0.375], A).astype(F32), logstd=np.zeros(A, F32))
    mean = (rng.integers(-4, 5, O) / 4).astype(F32)
    obs = (rng.integers(-12, 13, (n, O)) / 4).astype(F32)
    wide = rng.random((n, O)) < 0.1
    obs[wide] = (np.sign(rng.standard_normal(wide.sum())) * rng.integers(24, 33, wide.sum()) / 4).astype(F32)
    h = (rng.integers(-8, 9, (n, G)) / 8).astype(F32)
    return w, mean, obs, h


def saturating_bias(inp, W):
    """A power of two B with B - |inp . W| >= 96 for every row and column: +B saturates sigmoidf to 1, -B to 0."""
    m = float((np.abs(inp.astype(np.float64)) @ np.abs(W.astype(np.float64))).max())
    return 2.0 ** math.ceil(math.log2(-R.SIGMOID_ZERO + m))


def readout_weights(w, kind, a1, h0, rng):
    """w with the readout's biases and weights (module docstring); a1, h0: every input row it will see."""
    G, H1 = h0.shape[1], a1.shape[1]
    w = dict(w)
    b = np.array(w["b_ru"], F32)
    B = saturating_bias(np.concatenate([a1, h0], 1), w["w_ru"])
    spread = (rng.integers(-80, 81, 2 * G) / 8).astype(F32)       # gate pre-activations over about +-12
    if kind == "carry":
        b[G:] = B
    elif kind == "candidate":
        b[:G], b[G:] = B, -B
    elif kind == "reset":
        b[:] = -B
    elif kind in ("u_gate", "u_only"):
        b[:G], b[G:] = B, spread[G:]
        w["w_c"], w["b_c"] = np.zeros_like(w["w_c"]), np.zeros_like(w["b_c"])
        if kind == "u_only":                                      # pre_u from a1 alone: the blend readout's u
            w["w_ru"] = np.array(w["w_ru"]); w["w_ru"][H1:, G:] = 0
    elif kind == "r_gate":
        b[:G], b[G:] = spread[:G], -B
        w["w_c"] = np.concatenate([np.zeros((H1, G), F32), np.eye(G, dtype=F32)])
        w["b_c"] = np.zeros(G, F32)
    w["b_ru"] = b
    return w


def readout_expected(w, kind, a1, h0, exact=False):
    """(expected h' in fp64, bound) of a readout for rows a1, h0 (begin rows already zero), with the saturation each readout
    relies on asserted on the restated pre-activations (bit for bit the kernel's).  exact: also assert that every chain is
    exact in fp32 and that the restated chain equals the exact sum."""
    G = h0.shape[1]
    xin = np.concatenate([a1, h0], 1)
    pre = R.gru_gate_sums(a1, h0, w).astype(np.float64)
    if exact:
        np.testing.assert_array_equal(pre, R.assert_exact_dot(xin, w["w_ru"], w["b_ru"], "gates"))
    pr, pu = pre[:, :G], pre[:, G:]
    h64 = h0.astype(np.float64)
    if kind == "carry":
        assert pu.min() >= R.SIGMOID_ONE
        return h64, np.zeros_like(h64)
    if kind in ("candidate", "reset"):
        assert pu.max() <= R.SIGMOID_ZERO
        assert pr.min() >= R.SIGMOID_ONE if kind == "candidate" else pr.max() <= R.SIGMOID_ZERO
        rh = h0 if kind == "candidate" else np.zeros_like(h0)
        c = R.fma_chain(np.concatenate([a1, rh], 1), w["w_c"], w["b_c"]).astype(np.float64)
        if exact:
            np.testing.assert_array_equal(c, R.assert_exact_dot(np.concatenate([a1, rh], 1), w["w_c"], w["b_c"], "candidate"))
        t = np.tanh(c)
        return t, R.TANHF_ULP * R.ulp32(t)
    if kind in ("u_gate", "u_only"):
        assert pr.min() >= R.SIGMOID_ONE
        return R.sigmoid(pu) * h64, R.sigmoid_bound(pu) * np.abs(h64)
    assert kind == "r_gate" and pu.max() <= R.SIGMOID_ZERO
    c = R.sigmoid(pr) * h64
    return np.tanh(c), R.tanh_bound(c, R.sigmoid_bound(pr) * np.abs(h64))


def assert_exact_inputs(w, x, h):
    """The dense layer and the head of an exact network are exact in fp32; returns the dense activations."""
    a1 = np.maximum(R.assert_exact_dot(x, w["pW1"], w["pb1"], "dense"), 0)
    np.testing.assert_array_equal(a1, R.layer1(x, w["pW1"], w["pb1"]))
    np.testing.assert_array_equal(R.fma_chain(h, w["pW3"], w["pb3"]), R.assert_exact_dot(h, w["pW3"], w["pb3"], "head"))
    return a1.astype(F32)


# ---- the sampler's draws ------------------------------------------------------------------------------------------------
def rand_u32(seed, env, counter, slot):
    """rexsim_kernel.cuh rand_u32 over an array of envs (uint64 arithmetic wraps like the kernel's)."""
    M = np.uint64
    z = M(seed) + M(0x9E3779B97F4A7C15) * (np.asarray(env).astype(M) + M(1))
    z ^= (M(counter) << M(32)) | M(slot)
    z += M(0x9E3779B97F4A7C15)
    z = (z ^ (z >> M(30))) * M(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> M(27))) * M(0x94D049BB133111EB)
    z ^= z >> M(31)
    return (z >> M(32)).astype(np.uint32)


def extreme_envs(seed, step, A, span=1 << 23, chunk=1 << 21):
    """Global envs in [0, span) whose draws of some action reach the sampler's extremes: the largest and smallest k of u1
    (logf nearest 0, z largest) and u2 nearest 0, 1/4, 1/2, 3/4 and 1 (cospif at +-1 and at its zeros)."""
    best = {}
    targets = [("u1 max", lambda k1, k2: -k1.astype(np.int64)), ("u1 min", lambda k1, k2: k1.astype(np.int64))]
    for f in (0, 0.25, 0.5, 0.75, 1.0):
        targets.append(("u2 %.2f" % f, lambda k1, k2, f=f: np.abs(k2.astype(np.float64) + 0.5 - f * 2.0 ** 23)))
    for e0 in range(0, span, chunk):
        env = np.arange(e0, e0 + chunk, dtype=np.uint64)
        for a in range(A):
            k1 = rand_u32(seed, env, step, 2 * a) >> np.uint32(9)
            k2 = rand_u32(seed, env, step, 2 * a + 1) >> np.uint32(9)
            for name, key in targets:
                v = key(k1, k2)
                i = int(np.argmin(v))
                if (a, name) not in best or v[i] < best[a, name][0]:
                    best[a, name] = (v[i], e0 + i)
    return {k: g for k, (_, g) in best.items()}


def sampler_expected(seed, genv, step, logstd, mean):
    """(action, bound on it, log-prob, bound on it) for global envs genv [n] given the kernel's means [n][A]."""
    A = len(logstd)
    u = [[R.uniforms(rand_u32(seed, genv, step, 2 * a + i)) for a in range(A)] for i in (0, 1)]
    u1, u2 = np.stack(u[0], 1), np.stack(u[1], 1)
    z, dz = R.normal_bound(u1, u2)
    act, da = R.action_bound(z, dz, np.asarray(logstd, F32)[None, :], mean)
    lp, dl = R.logprob_bound(z, dz, np.asarray(logstd, F32)[None, :])
    return act, da, lp, dl


def _cell(kind, n, O=4, A=2):
    from rex_gym_b200.agents import ForwardGaussianPolicy, LinearGaussianPolicy, RecurrentGaussianPolicy
    if kind in ("fp32", "tensor_cores"):
        net = ForwardGaussianPolicy(O, A, seed=2, tensor_cores=kind == "tensor_cores")
    elif kind == "gru":
        net = RecurrentGaussianPolicy(O, A, seed=2, num_envs=n)
    else:
        net = LinearGaussianPolicy(O, A, seed=2, num_envs=n)
    w = net.get_weights()
    w["logstd"] = np.array([-0.5, 0.25][:A], F32)              # exp(ls) below and above 1
    net.set_weights(w)
    return net, w["logstd"]


# ---- CPU -----------------------------------------------------------------------------------------------------------------
def test_saturation_constants():
    """sigmoidf(x) = 1 / (1 + expf(-x)) is exactly 1 for x >= 24: even with expf's 2 ulp, E <= expf(-24) < 2^-25 and 1 + E
    rounds to 1.  It is exactly 0 for x <= -96: exp(96) exceeds FLT_MAX by far more than 2 ulp, so expf overflows to inf
    and 1 / inf = 0.  sigmoid_bound covers both limits and the distance of the fp32 results to the exact sigmoid."""
    E = math.exp(-R.SIGMOID_ONE) * (1 + R.EXPF_ULP * 2.0 ** -23)
    assert E < 2.0 ** -25 and F32(1) + F32(E) == F32(1)
    assert math.exp(-R.SIGMOID_ZERO) > R.FLT_MAX * (1 + 2.0 ** -10)
    x = np.array([24.0, 30.0, 1e4, -96.0, -100.0, -1e4])
    want = np.where(x > 0, 1.0, 0.0)
    assert np.all(np.abs(want - R.sigmoid(x)) <= R.sigmoid_bound(x))
    v = np.linspace(-85, 20, 10001)                    # below about -88.7 expf(-x) overflows and sigmoidf is 0
    s, b = R.sigmoid(v), R.sigmoid_bound(v)
    assert np.all(b > 0) and np.all(b <= 8 * R.ulp32(s) + 2.0 ** -149)         # a few ulp, not a loose bound


def test_uniform_law_is_exact_for_every_k():
    """All 2^23 values of k = r >> 9: ((float)k + 0.5f) * 2^-23 in fp32 equals the oracle's (k + 0.5) / 2^23 in fp64, and
    lies strictly inside (0, 1).  The former law, ((r >> 8) + 0.5f) * 2^-24, was inexact for half of its 2^24 k (every
    k >= 2^23, where k + 0.5 needs 25 bits) and gave exactly 1.0 at k = 2^24 - 1."""
    k = np.arange(1 << 23, dtype=np.uint32)
    u = R.uniforms(k << np.uint32(9))
    assert np.array_equal(u.astype(np.float64), (k.astype(np.float64) + 0.5) / 2.0 ** 23)
    assert u.min() == 2.0 ** -24 and u.max() == 1 - 2.0 ** -24
    k = np.arange(1 << 24, dtype=np.uint32)
    old = (k.astype(F32) + F32(0.5)) * F32(2.0 ** -24)
    assert old[-1] == 1.0 and np.mean(old.astype(np.float64) != (k + 0.5) / 2.0 ** 24) == 0.5


def test_sampler_restatement_against_the_oracle():
    """The vectorised generator equals agent_oracle.rand_u32; the restated uniforms equal agent_oracle.uniform_pair; z from
    them equals normal_noise, and its bound stays at a few ulp.  The ONE_DRAW key has all 24 top bits set."""
    rng = np.random.default_rng(0)
    env = rng.integers(0, 2 ** 32, 300).astype(np.uint64)
    for seed, step, a in ((99, 0, 0), (2 ** 63 + 5, 2 ** 32 - 1, 7), (0, 3, 1)):
        r1 = rand_u32(seed, env, step, 2 * a)
        assert [int(v) for v in r1] == [AO.rand_u32(seed, int(e), step, 2 * a) for e in env]
        u1, u2 = R.uniforms(r1), R.uniforms(rand_u32(seed, env, step, 2 * a + 1))
        assert [(float(p), float(q)) for p, q in zip(u1, u2)] == [AO.uniform_pair(seed, int(e), step, a) for e in env]
        z, dz = R.normal_bound(u1, u2)
        np.testing.assert_allclose(z, [AO.normal_noise(seed, int(e), step, a) for e in env], rtol=1e-13, atol=1e-15)
        assert np.all(dz <= 8 * R.ulp32(np.abs(z)) + 2.0 ** -40)
    seed, g, step, a = ONE_DRAW
    assert AO.rand_u32(seed, g, step, 2 * a) >> 8 == 2 ** 24 - 1
    assert (F32(2 ** 24 - 1) + F32(0.5)) * F32(2.0 ** -24) == 1.0


def test_extreme_draw_search():
    ex = extreme_envs(SEED, 5, 2, span=1 << 20, chunk=1 << 18)
    for (a, name), g in ex.items():
        k1 = AO.rand_u32(SEED, g, 5, 2 * a) >> 9
        k2 = AO.rand_u32(SEED, g, 5, 2 * a + 1) >> 9
        if name == "u1 max":
            assert k1 > 2 ** 23 - 40
        elif name == "u1 min":
            assert k1 < 40
        else:
            assert abs(k2 + 0.5 - float(name.split()[1]) * 2 ** 23) < 40


@pytest.mark.parametrize("row", ROWS[:2] + ROWS[-3:], ids=row_id)
def test_restatements_against_the_fp64_oracle(row):
    """The GRU step (gru_step_bound) and the linear head (fma_chain) against recurrent_oracle in fp64: the new state and the
    mean at fp32 distance, and inside the step bound, which stays far below the 2e-4 of test_gpu_recurrent_agent."""
    O, A, H1, G, vl = row
    rng = np.random.default_rng(O + H1 + G)
    w, f = _weights(rng, O, A, H1, G, vl), _filters(rng, O)
    obs = rng.normal(0.3, 3.0, (64, O)).astype(F32)
    h = rng.uniform(-0.9, 0.9, (64, G)).astype(F32)
    x = R.normalise(obs, *R.normaliser(f.count, f.mean, f.var_sum))
    hp, dh, s, es = R.gru_step_bound(w, R.layer1(x, w["pW1"], w["pb1"]), h)
    _, mean, _, _, h2 = RO.perform(w, f, obs, False, state=h)
    assert np.abs(hp - h2).max() < 1e-5 and np.abs(np.tanh(s) - mean).max() < 1e-5
    assert np.all(np.abs(hp - h2) <= dh + 1e-6) and dh.max() < 2e-5, float(dh.max())
    w.update(pW=(rng.standard_normal((O, A)) / math.sqrt(O)).astype(F32), pb=rng.normal(0, 0.1, A).astype(F32))
    sl = R.fma_chain(x, w["pW"], w["pb"])
    want, _, _ = RO.linear_gaussian_policy(w, f.transform(obs))
    np.testing.assert_allclose(np.tanh(sl.astype(np.float64)), want, atol=2e-5)


@pytest.mark.parametrize("row", ROWS, ids=row_id)
def test_constructed_networks_are_exact(row):
    """Every exact network (at the largest batch of a 132-SM H100) and its readouts: the chains exact in fp32, the
    saturations in force, the special rows non-zero in every column, the u and r pre-activations spread over +-8."""
    O, A, H1, G, vl = row
    n = 128 * 131 + 1
    w, mean, obs, h = exact_gru_network(O, A, H1, G, n, vl)
    x = R.normalise(obs, mean, np.ones(O, F32))
    assert np.array_equal(x, np.clip(obs.astype(np.float64) - mean, -5, 5))
    idx = np.random.default_rng(1).choice(n, 300, replace=False)
    a1 = assert_exact_inputs(w, x[idx], h[idx])
    for k in ("w_ru", "w_c"):
        assert np.all(w[k][special_rows(H1, G)] != 0)
    rng = np.random.default_rng(2)
    for kind in READOUTS + ("u_only",):
        h0 = np.ones_like(h[idx]) if kind in ("u_gate", "r_gate", "u_only") else h[idx]
        wr = readout_weights(w, kind, a1, h0, rng)
        readout_expected(wr, kind, a1, h0, exact=True)
        if kind in ("u_gate", "r_gate"):
            pre = R.gru_gate_sums(a1, h0, wr)[:, (0 if kind == "r_gate" else G):][:, :G]
            assert np.mean(np.abs(pre) < 8) > 0.3, kind


@pytest.mark.parametrize("row", ROWS[-4:], ids=row_id)
def test_new_rows_are_accepted(row):
    import ctypes as C
    from rex_gym_b200 import _capi
    O, A, H1, G, vl = row
    a, r = _capi.RexAgentConfig(O, A, vl[0], vl[1], 5.0, 10.0), _capi.RexRnnConfig(_capi.REXRNN_GRU, H1, G, 1)
    assert _capi.load().rexrnn_check(C.byref(a), C.byref(r)) == 0


# ---- GPU -----------------------------------------------------------------------------------------------------------------
def _rnet(row, n, w, count, mean, var_sum):
    from rex_gym_b200.agents import RecurrentGaussianPolicy
    O, A, H1, G, vl = row
    net = RecurrentGaussianPolicy(O, A, (H1, 100), vl, seed=1, num_envs=n, cell_size=G)
    net.set_weights(w)
    net.set_filters(count, mean, var_sum, 0, 0.0, 0.0)
    return net


def _hidden(net):
    return net.state_dict()["hidden"].cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["realistic", "exact"])
@pytest.mark.parametrize("row", ROWS, ids=row_id)
def test_gate_readouts(row, kind):
    O, A, H1, G, vl = row
    sizes = batch_sizes()
    N = max(sizes)
    rng = np.random.default_rng(10 * O + A + H1 + G)
    if kind == "realistic":
        w, f = _weights(rng, O, A, H1, G, vl), _filters(rng, O)
        filt = (f.count, f.mean, f.var_sum)
        obs = rng.normal(0.3, 3.0, (N, O)).astype(F32)
        obs[rng.random(N) < 0.01] = 100.0
        hs = rng.uniform(-0.9, 0.9, (N, G)).astype(F32)
    else:
        w, mean, obs, hs = exact_gru_network(O, A, H1, G, N, vl)
        filt = (0, mean, np.zeros(O, F32))
    begin = rng.random(N) < 0.05
    probes = {n: _probes(n) for n in sizes}
    rows = np.unique(np.concatenate(list(probes.values())))
    where = {e: i for i, e in enumerate(rows)}
    x = R.normalise(obs[rows], *R.normaliser(*filt))
    a1 = assert_exact_inputs(w, x, hs[rows]) if kind == "exact" else R.layer1(x, w["pW1"], w["pb1"])
    net = _rnet(row, N, w, *filt)
    xd, bd = torch.from_numpy(obs).cuda(), torch.from_numpy(begin.astype(np.uint8)).cuda()
    sd = net.state_dict()
    ones = np.ones((N, G), F32)
    device = {}

    def run(wr, state, n, steps=1, use_begin=True):
        net.set_weights(wr)
        net.load_state_dict(dict(sd, hidden=torch.from_numpy(state).cuda()))
        outs = [net.perform(xd[:n], training=False, begin=bd[:n] if use_begin and t == 0 else None) for t in range(steps)]
        hid = _hidden(net)
        assert np.array_equal(hid[n:].view(np.uint32), state[n:].view(np.uint32)), n
        return hid, outs[-1]["mean"].cpu().numpy()

    for rk in READOUTS:
        state = ones if rk in ("u_gate", "r_gate") else hs
        h0 = np.where(begin[rows, None], F32(0), state[rows])
        wr = readout_weights(w, rk, a1, h0, rng)
        want, bound = readout_expected(wr, rk, a1, h0, exact=kind == "exact")
        s = R.fma_chain(h0, wr["pW3"], wr["pb3"]) if rk == "carry" else None
        for n in sizes:
            p = probes[n]
            k = np.array([where[e] for e in p])
            hid, mean = run(wr, state, n, steps=4 if rk == "carry" else 1)
            err = np.abs(hid[p].astype(np.float64) - want[k])
            assert np.all(err <= bound[k]), (rk, n, float((err - bound[k]).max()), np.unravel_index((err - bound[k]).argmax(), err.shape))
            if rk == "carry":
                ratio = R.within_tanhf(mean[p], s[k])
                assert ratio.max() <= 1, (n, float(ratio.max()))
    # blend: U = sigmoidf(pre_u) with pre_u from a1 alone (read through the u readout at h = 1), T = tanhf(c) (read through
    # the candidate readout at the state h), then both at once: h' = fmaf(U, h, (1 - U) * T) bit for bit
    wu = readout_weights(w, "u_only", a1, ones[rows], rng)
    want, bound = readout_expected(wu, "u_only", a1, ones[rows], exact=kind == "exact")
    wc = readout_weights(w, "candidate", a1, hs[rows], rng)
    wb = dict(wc, w_ru=wu["w_ru"], b_ru=np.r_[wc["b_ru"][:G], wu["b_ru"][G:]])
    assert R.gru_gate_sums(a1, hs[rows], wb)[:, :G].min() >= R.SIGMOID_ONE
    for n in sizes[::3] + sizes[-1:]:
        U, _ = run(wu, ones, n, use_begin=False)
        assert np.all(np.abs(U[rows[rows < n]] - want[rows < n]) <= bound[rows < n]), n
        T, _ = run(wc, hs, n, use_begin=False)
        hb, _ = run(wb, hs, n, use_begin=False)
        np.testing.assert_array_equal(hb[:n], R.gru_blend(U[:n], hs[:n], T[:n]), err_msg=str(n))
    assert np.mean((U > 0.01) & (U < 0.99)) > 0.1                # u away from 0 and 1: neither blend product vanishes
    net.close()


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROWS, ids=row_id)
def test_full_cell_within_the_one_step_bound(row, capsys):
    """_weights over 64 steps with fresh observations and 5 % episode starts at 64 x SMs + 1 envs: before each step the
    device's state of the probe rows is read; every step is restated from it (agent_restate.gru_step_bound) and the new
    state and the mean held to the bound.  Prints the largest error / bound ratios and the largest bounds."""
    O, A, H1, G, vl = row
    rng = np.random.default_rng(1000 + O + A + H1 + G)
    w, f = _weights(rng, O, A, H1, G, vl), _filters(rng, O)
    n = 64 * _sm() + 1
    net = _net(row, n, w, f)
    idx = _probes(n)
    idt = torch.from_numpy(idx).cuda()
    rec = {k: [] for k in ("obs", "h0", "h1", "mean")}
    for t in range(64):
        obs = rng.normal(0.3, 3.0, (n, O)).astype(F32)
        obs[rng.random(n) < 0.01] = 100.0
        begin = rng.random(n) < 0.05
        before = net.state_dict()["hidden"][idt].cpu().numpy()
        g = net.perform(torch.from_numpy(obs).cuda(), training=False, begin=torch.from_numpy(begin.astype(np.uint8)).cuda())
        rec["obs"].append(obs[idx]); rec["h0"].append(np.where(begin[idx, None], F32(0), before))
        rec["h1"].append(net.state_dict()["hidden"][idt].cpu().numpy()); rec["mean"].append(g["mean"][idt].cpu().numpy())
    net.close()
    obs, h0, h1, mean = (np.concatenate(rec[k]) for k in ("obs", "h0", "h1", "mean"))
    x = R.normalise(obs, *R.normaliser(f.count, f.mean, f.var_sum))
    hp, dh, s, es = R.gru_step_bound(w, R.layer1(x, w["pW1"], w["pb1"]), h0)
    s = s.astype(np.float64)
    bm = R.tanh_bound(s, es)
    rh = np.abs(h1 - hp) / dh
    rm = np.abs(mean - np.tanh(s)) / bm
    with capsys.disabled():
        print("\n%s: full cell, largest error / bound: state %.3f, mean %.3f (bounds up to %.2e / %.2e)" % (
            row_id(row), rh.max(), rm.max(), dh.max(), bm.max()))
    assert rh.max() <= 1 and rm.max() <= 1, (float(rh.max()), float(rm.max()))
    assert dh.max() < 2e-5 and bm.max() < 2e-5


@pytest.mark.gpu
@pytest.mark.parametrize("row", LIN_ROWS, ids=lambda r: "O%d-A%d" % r[:2])
def test_linear_policy_head_and_exact_networks(row):
    """Realistic weights: on every row of every batch size the mean within tanhf's 2 ulp of tanh(fma_chain(x, pW, pb)), the
    deterministic action equal to it.  Exact networks (x on 1/4 with filter count 0, pW on +-{1/8, 1/4, 1/2}, pb on 1/8): the
    same against the exact sum, at every size including both edges of each 128-env tile."""
    from rex_gym_b200.agents import LinearGaussianPolicy
    O, A, vl = row
    rng = np.random.default_rng(3 * O + A)
    f = _filters(rng, O)
    sizes = [1, 127, 128, 129, 255, 256, 257, 65536 + 37]
    N = max(sizes)
    w = _weights(rng, O, A, 4, 4, vl)
    w.update(pW=(rng.standard_normal((O, A)) / math.sqrt(O)).astype(F32), pb=rng.normal(0, 0.1, A).astype(F32))
    obs = rng.normal(0.3, 3.0, (N, O)).astype(F32)
    obs[rng.random(N) < 0.01] = 100.0
    s_real = R.fma_chain(R.normalise(obs, *R.normaliser(f.count, f.mean, f.var_sum)), w["pW"], w["pb"])
    we = dict(w, pW=rng.choice([-0.5, -0.25, -0.125, 0.125, 0.25, 0.5], (O, A)).astype(F32),
              pb=rng.choice([-0.375, -0.125, 0.125, 0.375], A).astype(F32))
    me = (rng.integers(-4, 5, O) / 4).astype(F32)
    oe = (rng.integers(-28, 29, (N, O)) / 4).astype(F32)
    s_exact = R.assert_exact_dot(R.normalise(oe, me, np.ones(O, F32)), we["pW"], we["pb"], "linear")
    np.testing.assert_array_equal(R.fma_chain(R.normalise(oe, me, np.ones(O, F32)), we["pW"], we["pb"]), s_exact)
    net = LinearGaussianPolicy(O, A, value_layers=vl, num_envs=N)
    for ww, filt, ob, s in ((w, (f.count, f.mean, f.var_sum), obs, s_real), (we, (0, me, np.zeros(O, F32)), oe, s_exact)):
        net.set_weights(ww)
        net.set_filters(*filt, 0, 0.0, 0.0)
        xd = torch.from_numpy(ob).cuda()
        for n in sizes:
            g = {k: v.cpu().numpy() for k, v in net.perform(xd[:n], training=False).items()}
            ratio = R.within_tanhf(g["mean"], s[:n])
            assert ratio.max() <= 1, (n, float(ratio.max()), np.unravel_index(ratio.argmax(), ratio.shape))
            assert np.array_equal(g["action"], g["mean"]), n
    net.close()


@pytest.mark.gpu
@pytest.mark.parametrize("cell", CELLS)
def test_sampler_at_its_extreme_draws(cell, capsys):
    """For each extreme draw of extreme_envs (both actions) a 64-env batch through env_offset that puts it at row 17: every
    row's action and log-prob within agent_restate's bounds of the restated draw, given the kernel's own mean."""
    step, n = 5, 64
    ex = extreme_envs(SEED, step, 2)
    net, logstd = _cell(cell, n)
    x = torch.from_numpy(np.random.default_rng(4).normal(0, 2, (n, 4)).astype(F32)).cuda()
    worst = [0.0, 0.0]
    for (a, name), g in sorted(ex.items()):
        off = max(g - 17, 0)
        out = {k: v.cpu().numpy() for k, v in net.perform(x, training=True, seed=SEED, step=step, env_offset=off).items()}
        act, da, lp, dl = sampler_expected(SEED, np.arange(off, off + n, dtype=np.uint64), step, logstd, out["mean"])
        ra, rl = np.abs(out["action"] - act) / da, np.abs(out["logprob"] - lp) / dl
        assert ra.max() <= 1 and rl.max() <= 1, (a, name, g, float(ra.max()), float(rl.max()))
        worst = [max(worst[0], float(ra.max())), max(worst[1], float(rl.max()))]
    net.close()
    with capsys.disabled():
        print("\n%s sampler: largest error / bound: action %.3f, log-prob %.3f" % (cell, worst[0], worst[1]))


@pytest.mark.gpu
@pytest.mark.parametrize("cell", CELLS)
def test_the_top_draw_is_not_one(cell):
    """ONE_DRAW's first uniform is 1 - 2^-24 (the 24-bit law rounded it to 1.0, so z = 0 and the action equalled the mean):
    the action differs from the mean and is within the bound of the restated draw."""
    seed, g, step, a = ONE_DRAW
    net, logstd = _cell(cell, 1)
    x = torch.zeros((1, 4), device="cuda")
    out = {k: v.cpu().numpy() for k, v in net.perform(x, training=True, seed=seed, step=step, env_offset=g).items()}
    net.close()
    act, da, _, _ = sampler_expected(seed, np.array([g], np.uint64), step, logstd, out["mean"])
    assert out["action"][0, a] != out["mean"][0, a]
    assert np.all(np.abs(out["action"] - act) <= da), (out["action"], act, da)

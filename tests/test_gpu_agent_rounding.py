"""The agent's perform kernels (csrc/rexsim_agent.cu) at rounding level, against agent_restate.py's restatement of their own
arithmetic.  test_gpu_agent.py and test_gpu_agent_shapes.py hold them to the fp64 network (5e-3 for the tensor-core form);
this file asks what each kernel computes, exactly:

* Exact networks (every row of test_gpu_agent_shapes.ROWS, both kernels on the tf32 rows, every batch size): inputs and
  weights on coarse dyadic grids, so every operand is tf32-representable and every partial sum, in any order, is exact in
  fp32 (both asserted on the arrays).  The value equals the exact value bit for bit, the mean is within tanhf's error of
  the fp64 tanh of the exact argument, the deterministic action equals the mean.  These checks are blind to accumulation
  order, so an operand layout, descriptor, K-step, column-chunk, padding-column, epilogue lane, shuffle or tile-position
  mistake fails with no tolerance.
* A rounding probe on the tensor cores: layer-1 activations and W2 entries with bits below tf32 precision (exact ties, just
  below and above a half, a round-up into the next binade, negative entries) in the first and last K-step, read out
  through a value head that is one-hot on a column, in the first, last and padded 16-column chunks.  The exact sum of the
  rna-rounded operands is again exact in fp32, so the value must match it bit for bit: rounding mode and rounded operands
  become visible.
* Realistic weights: the fp32 kernel's value bit for bit and its mean within tanhf's error of tanh(restated argument); the
  tensor-core kernel within a per-output bound propagated from the accumulation model of agent_restate.head_tf32, and that
  model measured on the H100 through the one-hot readout, which shows the accumulator d itself.
* The reward transform bit for bit, and a tensor-core rollout captured in a CUDA graph equal to the step-by-step loop.
"""
import ctypes as C
import ctypes.util

import numpy as np
import pytest
import torch

import agent_restate as R
from oracle import agent_oracle as AO
from test_gpu_agent_shapes import ROWS, _half, _setup, _weights, batch_sizes, probe_envs, row_id, tiling

F32 = np.float32
TF32_ROWS = [r for r in ROWS if r[4] == "tf32"]


# ---- the networks -----------------------------------------------------------------------------------------------------
def _grid(rng, shape, values, nnz_per_col=None):
    """Entries drawn from `values` (dyadic), sparse: nnz_per_col non-zeros per column at random rows."""
    x = rng.choice(np.asarray(values, np.float64), size=shape)
    if nnz_per_col is not None and nnz_per_col < shape[0]:
        keep = np.zeros(shape, bool)
        for j in range(shape[1]):
            keep[rng.choice(shape[0], nnz_per_col, replace=False), j] = True
        x = np.where(keep, x, 0.0)
    return x.astype(F32)


def exact_network(O, A, H1, H2, n, seed=0):
    """(weights, observ mean, observations [n][O]) on dyadic grids, filter count 0 (inv = 1 exactly): observations and means
    on a 1/4 grid, a tenth of the inputs beyond the +-5 clip; W1 in +-{1/8, 1/4}, b1 on 1/8; W2 and W3 sparse in
    +-{1/8 .. 1/2}, W2 with a non-zero in the first and the last K-step of every column; biases on 1/8, b3 non-zero."""
    rng = np.random.default_rng(seed + 1000 * O + 100 * A + H1 + H2)
    q = np.arange(1, 5) / 8.0
    w = {}
    for p, AO_ in (("p", A), ("v", 1)):
        w[p + "W1"] = _grid(rng, (O, H1), [-0.25, -0.125, 0.125, 0.25])
        w[p + "b1"] = _grid(rng, (H1,), np.arange(-8, 9) / 8.0)
        W2 = _grid(rng, (H1, H2), np.r_[-q, q], nnz_per_col=min(H1, 8))
        first, last = rng.integers(0, min(8, H1), H2), H1 - 1 - rng.integers(0, min(8, H1), H2)
        W2[first, np.arange(H2)] = _grid(rng, (H2,), np.r_[-q, q])
        W2[last, np.arange(H2)] = _grid(rng, (H2,), np.r_[-q, q])
        w[p + "W2"] = W2
        w[p + "b2"] = _grid(rng, (H2,), np.arange(-8, 9) / 8.0)
        w[p + "W3"] = _grid(rng, (H2, AO_), [-0.25, -0.125, 0.125, 0.25], nnz_per_col=min(H2, 6))
        w[p + "b3"] = _grid(rng, (AO_,), [-0.5, -0.375, -0.25, -0.125, 0.125, 0.25, 0.375, 0.5])
    w["logstd"] = np.zeros(A, F32)
    mean = (rng.integers(-4, 5, O) / 4.0).astype(F32)
    obs = (rng.integers(-12, 13, (n, O)) / 4.0).astype(F32)
    wide = rng.random((n, O)) < 0.1
    obs[wide] = (np.sign(rng.standard_normal(wide.sum())) * rng.integers(24, 33, wide.sum()) / 4.0).astype(F32)
    return w, mean, obs


def exact_outputs(w, mean, obs):
    """The exact pre-tanh sums [n][A] and values [n], with every exactness condition asserted on the arrays: the
    normalised inputs, h1 and W2 carry at most 11 significant bits (tf32 keeps them), every dot product stays below 2^24
    units of its grid (exact in fp32 in any order)."""
    x = R.normalise(obs, mean, np.ones_like(mean))
    assert R.significant_bits(x) <= 11
    assert np.array_equal(x, np.clip(obs.astype(np.float64) - mean, -5, 5))
    out = []
    for net in (0, 1):
        W1, b1, W2, b2, W3, b3 = R.net_params(w, net)
        h1 = np.maximum(R.assert_exact_dot(x, W1, b1, "layer 1"), 0)
        assert R.significant_bits(h1) <= 11 and R.significant_bits(W2) <= 11, (R.significant_bits(h1), R.significant_bits(W2))
        h2 = np.maximum(R.assert_exact_dot(h1, W2, b2, "layer 2"), 0)
        out.append(R.assert_exact_dot(h2, W3, b3, "head"))
    return out[0], out[1][:, 0]


def _from_bits(bits):
    return np.asarray(bits, np.uint32).view(F32)


# rounding probe: (activation, W2 entry) as float32 bit patterns; each crosses tf32 precision in one operand or both
ONE, TIE, BELOW, ABOVE, CARRY = 0x3F800000, 0x3F801000, 0x3F800FFF, 0x3F801001, 0x3FFFF000
NEG = 0x80000000
PROBE_CASES = [
    (TIE, ONE), (BELOW, ONE), (ABOVE, ONE), (CARRY, ONE),                          # the activation only
    (ONE, TIE), (ONE, NEG | TIE), (ONE, NEG | BELOW), (ONE, CARRY), (ONE, NEG | CARRY),   # the weight only
    (TIE, TIE), (ABOVE, NEG | TIE), (CARRY, NEG | ABOVE), (TIE + (3 << 23), 0x3E801000),  # both; 8 (1 + 2^-11) x 0.25 (..)
]
PROBE_OFFSET = 8.0                         # b2 of the probed column: keeps relu(d + b2) = d + b2 with negative products


def probe_columns(H2):
    return sorted({0, min(15, H2 - 1), min(16, H2 - 1), H2 - 1})


def probe_ks(H1):
    """One activation in the first K-step and one in the last (both inside the single step when H1 = 8)."""
    return (1, 6) if H1 == 8 else (2, H1 - 3)


def probe_network(O, A, H1, H2, col, case):
    """Layer 1 is its bias (W1 = 0): h1 = b1 = the probe activation at the two probe ks, zero elsewhere; W2 non-zero only
    in column col at those ks; the value head one-hot on col, b3 = 0, so value = relu(d_col + 8) = d_col + 8.  The policy
    network is all zeros."""
    a, b = (_from_bits(v) for v in case)
    w = {k: np.zeros(s, F32) for k, s in dict(pW1=(O, H1), pb1=(H1,), pW2=(H1, H2), pb2=(H2,), pW3=(H2, A), pb3=(A,),
                                                 logstd=(A,), vW1=(O, H1), vb1=(H1,), vW2=(H1, H2), vb2=(H2,), vW3=(H2, 1),
                                                 vb3=(1,)).items()}
    for k in probe_ks(H1):
        w["vb1"][k] = a
        w["vW2"][k, col] = b
    w["vb2"][col] = PROBE_OFFSET
    w["vW3"][col, 0] = 1.0
    return w


def probe_value(w, col):
    """The value of the probe network with both operands rna-rounded, asserted exact in fp32."""
    a = R.tf32_rna(w["vb1"])[None, :]
    b = R.tf32_rna(w["vW2"][:, col:col + 1])
    assert R.significant_bits(a) <= 11 and R.significant_bits(b) <= 11
    v = R.assert_exact_dot(a, b, w["vb2"][col:col + 1], "probe")[0, 0]
    assert v > 0
    return F32(v)


# ---- CPU: the restatement's arithmetic ---------------------------------------------------------------------------------
def _libm_fmaf():
    libm = C.CDLL(ctypes.util.find_library("m"))
    f = libm.fmaf
    f.argtypes, f.restype = [C.c_float] * 3, C.c_float
    return lambda a, b, c: np.array([f(x, y, z) for x, y, z in zip(a.tolist(), b.tolist(), c.tolist())], F32)


def test_fmaf32_equals_the_c_library_fmaf():
    """Random triples over 80 binades, near-cancelling triples (c close to -a b) and triples whose fp64 sum lands exactly
    on a float32 midpoint while the exact sum lies just beside it, or exactly on it (ties to even)."""
    rng = np.random.default_rng(11)
    fmaf = _libm_fmaf()
    n = 200000

    def rnd(k, span):
        return (rng.standard_normal(k) * np.ldexp(1.0, rng.integers(-span, span, k))).astype(F32)
    a, b, c = rnd(n, 20), rnd(n, 20), rnd(n, 40)
    ca, cb = rnd(n, 20), rnd(n, 20)
    cc = (-(ca.astype(np.float64) * cb) * (1 + rng.standard_normal(n) * 2.0 ** -rng.integers(10, 30, n))).astype(F32)
    # midpoints: c = q (random float32), a b = +-(ulp(q) / 2) (1 + i 2^-23)(1 + j 2^-23) with i, j in {-1, 0, 1}
    m = 60000
    q = rnd(m, 30)
    h = R.ulp32(q.astype(np.float64)) / 2
    e1 = rng.integers(-10, 10, m)
    i, j = rng.integers(-1, 2, m), rng.integers(-1, 2, m)
    ma = (np.ldexp(1.0, e1) * (1 + i * 2.0 ** -23) * rng.choice([-1, 1], m)).astype(F32)
    mb = (h / np.ldexp(1.0, e1) * (1 + j * 2.0 ** -23)).astype(F32)
    mid = (ma.astype(np.float64) * mb + q)
    assert np.mean(np.abs(mid - q) > 0) > 0.9
    A_, B_, C_ = np.r_[a, ca, ma], np.r_[b, cb, mb], np.r_[c, cc, q]
    want, got = fmaf(A_, B_, C_), R.fmaf32(A_, B_, C_)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))[:5]
    # the midpoint cases are the ones a plain fp64 sum rounded to float32 gets wrong
    naive = (ma.astype(np.float64) * mb + q).astype(F32)
    assert (naive != want[2 * n:]).sum() > 1000


def test_tf32_rna_on_constructed_cases():
    cases = [  # input bits, cvt.rna.tf32.f32 bits
        (0x3F801000, 0x3F802000), (0x3F800FFF, 0x3F800000), (0x3F801001, 0x3F802000),      # tie away from zero, below, above
        (0x3F803000, 0x3F804000), (0x3F802000, 0x3F802000),                                 # tie from an odd kept bit; exact
        (0x3FFFF000, 0x40000000), (0x3FFFFFFF, 0x40000000), (0x7F7FF000, 0x7F800000),       # carry into the exponent
        (0xBF801000, 0xBF802000), (0xBF800FFF, 0xBF800000), (0xBFFFF000, 0xC0000000),       # the sign is kept
        (0x00000000, 0x00000000), (0x80000000, 0x80000000), (0x00001000, 0x00002000),       # zeros, a subnormal tie
    ]
    x = np.array([c[0] for c in cases], np.uint32).view(F32)
    np.testing.assert_array_equal(R.tf32_rna(x).view(np.uint32), np.array([c[1] for c in cases], np.uint32))
    rng = np.random.default_rng(3)
    v = (rng.standard_normal(100000) * np.ldexp(1.0, rng.integers(-30, 30, 100000))).astype(F32)
    t = R.tf32_rna(v)
    assert R.significant_bits(t) <= 11 and np.array_equal(R.tf32_rna(t), t)
    assert np.all(np.abs(t.astype(np.float64) - v) <= np.abs(v) * 2.0 ** -11)


def test_grid_and_significant_bits():
    x = np.array([0.375, -1.5, 96.0, 0.0])
    assert R.grid_exponent(x) == 3 and R.significant_bits(x) == 2
    assert R.significant_bits(np.array([1 + 2.0 ** -10])) == 11 and R.grid_exponent(np.array([2.0 ** -20])) == 20
    with pytest.raises(AssertionError):
        R.assert_exact_dot(np.full((1, 3), 2.0 ** 22), np.ones((3, 1)), np.array([2.0 ** -2]), "too wide")


@pytest.mark.parametrize("row", ROWS[:2] + TF32_ROWS[2:4], ids=row_id)
def test_restatement_matches_the_fp64_oracle(row):
    """Both restatements against AO.forward_gaussian_policy at fp32 / tf32 distance, on _weights and a fitted filter."""
    O, A, H1, H2, _ = row
    rng = np.random.default_rng(5)
    w = _weights(rng, O, A, H1, H2)
    f = AO.StreamingNormalize((O,), True, True, 5)
    f.update(rng.normal(0.3, 1.7, (5000, O)))
    obs = rng.normal(0.3, 3.0, (300, O)).astype(F32)
    obs[0] = 100.0
    want_mean, _, want_value = AO.forward_gaussian_policy(w, f.transform(obs))
    x = R.normalise(obs, *R.normaliser(f.count, f.mean, f.var_sum))
    np.testing.assert_allclose(x, f.transform(obs), rtol=2e-6, atol=2e-6)
    zp = R.head_sums_fp32(x, *R.net_params(w, 0))
    zv = R.head_sums_fp32(x, *R.net_params(w, 1))
    np.testing.assert_allclose(np.tanh(zp), want_mean, atol=2e-5)
    np.testing.assert_allclose(zv[:, 0], want_value, atol=5e-5)
    for net, want in ((0, want_mean), (1, want_value[:, None])):
        W1, b1, W2, b2, W3, b3 = R.net_params(w, net)
        D, S = R.layer2_tf32(R.layer1(x, W1, b1), W2)
        z, bound = R.head_tf32(D, S, b2, W3, b3, H1)
        got = np.tanh(z) if net == 0 else z
        assert np.abs(got - want).max() < 5e-3 and 0 < bound.max() < 1e-3, (net, np.abs(got - want).max(), bound.max())


@pytest.mark.parametrize("row", ROWS, ids=row_id)
def test_exact_networks_are_exact(row):
    """The exactness conditions of the exact network of every row (at the largest batch of a 132-SM H100) and of every
    rounding probe, asserted on the arrays; the tanh arguments stay O(1), so the mean check is not saturated."""
    O, A, H1, H2, prec = row
    n = max(batch_sizes(66))
    w, mean, obs = exact_network(O, A, H1, H2, n)
    z, v = exact_outputs(w, mean, obs)
    assert np.mean(np.abs(z) < 2) > 0.5 and np.all(w["pb3"] != 0) and np.all(w["vb3"] != 0)
    assert np.mean(np.abs(np.clip(obs - mean, -5, 5)) == 5) > 0.05
    if prec == "tf32":
        for col in probe_columns(H2):
            for case in PROBE_CASES:
                probe_value(probe_network(O, A, H1, H2, col, case), col)


# ---- GPU ----------------------------------------------------------------------------------------------------------------
def _net(O, A, H1, H2, tensor_cores):
    from rex_gym_b200.agents import ForwardGaussianPolicy
    return ForwardGaussianPolicy(O, A, (H1, H2), (H1, H2), tensor_cores=tensor_cores)


def _numpy(out):
    return {k: t.cpu().numpy() for k, t in out.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROWS, ids=row_id)
def test_exact_networks_bit_for_bit(row):
    O, A, H1, H2, prec = row
    sizes = batch_sizes(_half())
    w, mean, obs = exact_network(O, A, H1, H2, max(sizes))
    z, v = exact_outputs(w, mean, obs)
    x_all = torch.from_numpy(obs).cuda()
    for tc in ((False, True) if prec == "tf32" else (False,)):
        net = _net(O, A, H1, H2, tc)
        net.set_weights(w)
        net.set_filters(0, mean, np.zeros(O, F32), 0, 0.0, 0.0)
        for n in sizes:
            g = _numpy(net.perform(x_all[:n], training=False))
            bad = np.flatnonzero(g["value"] != v[:n].astype(F32))
            assert bad.size == 0, (tc, n, bad[:5], g["value"][bad[:5]], v[bad[:5]])
            ratio = R.within_tanhf(g["mean"], z[:n])
            assert ratio.max() <= 1, (tc, n, float(ratio.max()), np.unravel_index(ratio.argmax(), ratio.shape))
            assert np.array_equal(g["action"], g["mean"]), (tc, n)
        net.close()


@pytest.mark.gpu
@pytest.mark.parametrize("row", TF32_ROWS, ids=row_id)
def test_tensor_core_rounding_probe(row):
    """Every PROBE_CASES pair at the first and last K-step, read out of the first, last and padded 16-column chunks: the
    value equals the fp32-exact sum of the rna-rounded operands bit for bit, in both tiles of a 129-env batch."""
    O, A, H1, H2, _ = row
    n = 129
    rng = np.random.default_rng(O + A + H1 + H2)
    x = torch.from_numpy(rng.normal(0, 2, (n, O)).astype(F32)).cuda()
    net = _net(O, A, H1, H2, True)
    net.set_filters(0, np.zeros(O, F32), np.zeros(O, F32), 0, 0.0, 0.0)
    fails = []
    for col in probe_columns(H2):
        for case in PROBE_CASES:
            w = probe_network(O, A, H1, H2, col, case)
            want = probe_value(w, col)
            net.set_weights(w)
            got = net.perform(x, training=False)["value"].cpu().numpy()
            if not np.all(got == want):
                fails.append((col, "%08x x %08x" % case, float(want), sorted(set(got.tolist()))[:3]))
    net.close()
    assert not fails, fails


def _restate_rows(w, f, obs):
    """Normalised inputs and layer-1 activations of the policy and value networks, restated for the rows of obs."""
    x = R.normalise(obs, *R.normaliser(f.count, f.mean, f.var_sum))
    return x, [R.layer1(x, *R.net_params(w, net)[:2]) for net in (0, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("row", TF32_ROWS, ids=row_id)
def test_tensor_core_accumulation_model(row, capsys):
    """_weights, with the value head replaced by a one-hot readout of column c (b2[c] = 0, b3 = 0), so value =
    max(d_c, 0) exactly: d_c itself wherever it is positive.  Against D_c of the rna-rounded operands, every column:
    |d_c - D_c| <= (ceil(H1 / 8) + 1) 2^-23 S_c (agent_restate.accumulation_bound).  Prints the largest ratio."""
    O, A, H1, H2, _ = row
    n = 1024
    w, f, obs, nets = _setup(row, n)
    for nt in nets[:-1]:
        nt.close()
    net = nets[-1]
    _, (_, h1v) = _restate_rows(w, f, obs)
    D, S = R.layer2_tf32(h1v, w["vW2"])
    E = R.accumulation_bound(S, H1)
    x = torch.from_numpy(obs).cuda()
    worst, seen = 0.0, 0
    for c in range(H2):
        r = dict(w)
        r["vb2"] = w["vb2"].copy(); r["vb2"][c] = 0
        r["vW3"] = np.zeros_like(w["vW3"]); r["vW3"][c, 0] = 1
        r["vb3"] = np.zeros(1, F32)
        net.set_weights(r)
        got = net.perform(x, training=False)["value"].cpu().numpy().astype(np.float64)
        pos = got > 0
        seen += int(pos.sum())
        assert np.all(got >= 0) and np.all(D[~pos, c] <= E[~pos, c]), c
        ratio = np.abs(got[pos] - D[pos, c]) / E[pos, c]
        worst = max(worst, float(ratio.max(initial=0)))
    net.close()
    with capsys.disabled():
        print("\n%s: accumulation |d - D| / ((ceil(H1/8) + 1) 2^-23 S): largest %.3f over %d accumulators" % (row_id(row), worst, seen))
    assert seen > n * H2 // 4 and worst <= 1, worst


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROWS, ids=row_id)
def test_perform_against_the_restatement(row, capsys):
    """_weights and a fitted filter at every batch size, at the probe envs of test_gpu_agent_shapes and a linspace.  fp32
    kernel (every row): value bit for bit, mean within tanhf's error of tanh(restated argument), deterministic action = mean.
    Tensor-core kernel (the tf32 rows): mean and value within the bound agent_restate.head_tf32 propagates from the
    accumulation model; prints the largest error / bound ratio."""
    O, A, H1, H2, prec = row
    half = _half()
    sizes = batch_sizes(half)
    w, f, obs, nets = _setup(row, max(sizes))
    idx = {}
    for n in sizes:
        for p in set(["fp32", prec]):
            idx[n, p] = np.unique(np.r_[probe_envs(n, *tiling(n, half, p)), np.linspace(0, n - 1, 16).astype(int)])
    rows = np.unique(np.concatenate(list(idx.values())))
    x, h1 = _restate_rows(w, f, obs[rows])
    zp = R.head_sums_fp32(x, *R.net_params(w, 0))
    zv = R.head_sums_fp32(x, *R.net_params(w, 1))[:, 0]
    where = {e: i for i, e in enumerate(rows)}
    x_all = torch.from_numpy(obs).cuda()
    worst = [0.0, 0.0]
    for n in sizes:
        k = np.array([where[e] for e in idx[n, "fp32"]])
        g = _numpy(nets[0].perform(x_all[:n], training=False))
        e = idx[n, "fp32"]
        bad = np.flatnonzero(g["value"][e] != zv[k])
        assert bad.size == 0, (n, e[bad[:5]], g["value"][e[bad[:5]]], zv[k[bad[:5]]])
        ratio = R.within_tanhf(g["mean"][e], zp[k])
        assert ratio.max() <= 1, (n, float(ratio.max()))
        assert np.array_equal(g["action"], g["mean"]), n
    if prec == "tf32":
        heads = []
        for net in (0, 1):
            W1, b1, W2, b2, W3, b3 = R.net_params(w, net)
            D, S = R.layer2_tf32(h1[net], W2)
            heads.append(R.head_tf32(D, S, b2, W3, b3, H1))
        (zt, bz), (vt, bv) = heads
        mb = R.tanh_bound(zt, bz)
        for n in sizes:
            k = np.array([where[e] for e in idx[n, "tf32"]])
            e = idx[n, "tf32"]
            g = _numpy(nets[1].perform(x_all[:n], training=False))
            rm = np.abs(g["mean"][e] - np.tanh(zt[k])) / mb[k]
            rv = np.abs(g["value"][e] - vt[k, 0]) / bv[k, 0]
            worst = [max(worst[0], float(rm.max())), max(worst[1], float(rv.max()))]
            assert rm.max() <= 1 and rv.max() <= 1, (n, float(rm.max()), float(rv.max()))
            assert np.array_equal(g["action"], g["mean"]), n
        with capsys.disabled():
            print("\n%s: tensor cores, largest error / bound: mean %.3f, value %.3f (bounds up to %.2e / %.2e)" % (
                row_id(row), worst[0], worst[1], float(mb.max()), float(bv.max())))
    for nt in nets:
        nt.close()


@pytest.mark.gpu
@pytest.mark.parametrize("count", [0, 1, 2, 5000, 2**32 + 5])
def test_transform_reward_bit_for_bit(count):
    """fminf(fmaxf(r * inv, -10), 10) in float32 with inv from filter_inv_std: +-1e6, exactly +-10, zero, and the rewards
    that land just inside, on and just beyond the clip after scaling."""
    from rex_gym_b200.agents import ForwardGaussianPolicy
    rng = np.random.default_rng(count % 1000)
    vs = F32(0.37 * max(count - 1, 0))
    inv = R.normaliser(count, np.zeros(1), np.array([vs]))[1][0]
    edge = F32(10) / inv
    near = np.array([np.nextafter(edge, F32(0)), edge, np.nextafter(edge, F32(np.inf))], F32)
    rr = np.r_[rng.normal(0, 20, 3000), 1e6, -1e6, 10.0, -10.0, 0.0, near, -near].astype(F32)
    net = ForwardGaussianPolicy(4, 2)
    net.set_filters(0, np.zeros(4), np.zeros(4), count, 0.3, float(vs))
    got = net.transform_reward(torch.from_numpy(rr).cuda()).cpu().numpy()
    net.close()
    want = R.transform_reward(rr, count, vs)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.flatnonzero(got != want)[:5]
    assert (np.abs(want) == 10).sum() > 100 and (np.abs(want) < 10).sum() > 100


@pytest.mark.gpu
def test_tensor_core_rollout_graph_equals_the_step_by_step_loop():
    """test_gpu_agent.py's graph-vs-loop rollout check with the networks' layer 2 on the tensor cores."""
    from test_gpu_agent import rollout_graph_equals_the_step_by_step_loop
    rollout_graph_equals_the_step_by_step_loop(tensor_cores=True)

"""The agent kernels (csrc/rexsim_agent.cu) at every network shape and batch size they accept, against the fp64 numpy oracle
(oracle/agent_oracle.py).

`rexagent_perform` has two forms.  The fp32 kernel runs `perform_kernel<TM>` on 64-env tiles while ceil(n / 128) is below half
the SM count and on 128-env tiles above it, on a grid of min(tiles, SMs / 2) persistent CTAs per network; its block has
16 * H2 / 4 threads, rounded up to TM.  The tf32 kernel (`perform_tc_kernel<O, A>`, eight instances) always uses 128-env tiles.
ROWS lists one network configuration per code path (shapes, widths, block sizes, tensor-core instances); every row runs at the
batch sizes around each tiling switch of the device it runs on.  The filter update, the reward transform and the scans are
checked at the lengths where their loops change shape, and the filter counts across 2^31 and 2^32.

The CPU tests check the table itself against the acceptance rule of `rexagent_create`, which validates a configuration before
its first CUDA call."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import agent_oracle as AO

# ---- the acceptance rule of rexagent_create / rexagent_set_precision (rexsim_agent.cu) --------------------------------
MAX_O, MAX_A, MAX_H1, MAX_H2 = 32, 8, 256, 128
SMEM = 227 * 1024
OK, ERR_INVALID, ERR_CUDA, ERR_UNSUPPORTED = 0, -1, -3, -4


def _pad4(n):
    return (n + 3) & ~3


def policy_floats(O, A, H1, H2):
    return _pad4(O * H1 + H1 + H1 * H2 + H2 + H2 * A + A + A)


def value_floats(O, A, H1, H2):
    return _pad4(O * H1 + H1 + H1 * H2 + H2 + H2 + 1)


def fp32_smem_bytes(O, A, H1, H2, tm=128):
    """perform_smem_bytes: the larger weight block, xs [MAX_O][TM], h1 [H1][TM], the normaliser constants."""
    return (max(policy_floats(O, A, H1, H2), value_floats(O, A, H1, H2)) + MAX_O * tm + H1 * tm + 2 * MAX_O) * 4


def tf32_smem_bytes(O, A, H1, H2):
    """perform_tc_smem_bytes: the A and B operands, the small layers, xs and the normaliser constants."""
    npad = (H2 + 15) & ~15
    small = (O * H1 + H1 + H2 + H2 * MAX_A + 2 * MAX_A + O * 128 + 2 * MAX_O) * 4
    return 128 * H1 * 4 + npad * H1 * 4 + small + 64


def create_code(O, A, H1, H2):
    """What rexagent_create returns before it touches the device: 0 for an accepted configuration."""
    if not (1 <= O <= MAX_O and 1 <= A <= MAX_A):
        return ERR_INVALID
    if not (0 < H1 <= MAX_H1 and 0 < H2 <= MAX_H2 and H1 % 4 == 0 and H2 % 4 == 0):
        return ERR_UNSUPPORTED
    if fp32_smem_bytes(O, A, H1, H2) > SMEM:
        return ERR_UNSUPPORTED
    if A * (H2 // 4) > H1:
        return ERR_UNSUPPORTED
    return OK


def tf32_accepted(O, A, H1, H2):
    return H1 % 8 == 0 and O <= 16 and tf32_smem_bytes(O, A, H1, H2) <= SMEM


def tc_instance(O, A):
    """perform_tc_pick: the (OT, AT) template arguments, 0 = generic."""
    if O == 4:
        return (4, A) if A in (1, 2, 8) else (4, 0)
    if O == 16:
        return (16, A) if A in (2, 4) else (16, 0)
    return (0, 0)


# (O, A, H1, H2, precision).  The block of the fp32 kernel has 16 * H2 / 4 threads, rounded up to the tile's TM.
ROWS = [
    (4, 2, 200, 100, "fp32"),      # walk / turn / standup / poses policies
    (16, 4, 200, 100, "fp32"),     # gallop policies
    (1, 1, 64, 12, "fp32"),        # 48 threads: rounded up to TM on both tile sizes
    (32, 8, 64, 4, "fp32"),        # widest input and head, 16 threads, A * H2 / 4 = 8
    (32, 3, 200, 100, "fp32"),     # O = 32 with the shipped hidden sizes: 227 072 of 232 448 bytes of shared memory
    (4, 2, 256, 64, "fp32"),       # the largest hidden1
    (4, 1, 200, 128, "fp32"),      # 512 threads, the launch bound
    (4, 2, 64, 100, "fp32"),
    (32, 1, 8, 12, "fp32"),        # hidden1 = 8
    (4, 2, 100, 36, "fp32"),       # hidden1 = 4 mod 8, 144 threads
    (4, 2, 200, 100, "tf32"),      # perform_tc_kernel<4, 2>
    (4, 1, 200, 128, "tf32"),      # <4, 1>; H2 = 128: all eight 16-column chunks
    (4, 8, 8, 4, "tf32"),          # <4, 8>; hidden1 = 8: a single K-step; H2 = 4 padded to 16
    (4, 5, 64, 12, "tf32"),        # <4, 0>
    (16, 2, 200, 100, "tf32"),     # <16, 2>
    (16, 4, 200, 100, "tf32"),     # <16, 4>
    (16, 3, 128, 100, "tf32"),     # <16, 0>
    (1, 3, 64, 12, "tf32"),        # <0, 0>
]


def row_id(r):
    return "O%d-A%d-%dx%d-%s" % r


def _lib():
    from rex_gym_b200 import _capi
    return _capi, _capi.load()


def _create(O, A, H1, H2):
    """rexagent_create's return code; an agent it creates (on a machine with a GPU) is destroyed again."""
    _capi, L = _lib()
    cfg = _capi.RexAgentConfig(O, A, H1, H2, 5.0, 10.0)
    h = C.c_void_p()
    rc = L.rexagent_create(C.byref(cfg), C.byref(h))
    if rc == OK:
        L.rexagent_destroy(h)
    return rc


def _assert_create_follows_the_rule(O, A, H1, H2):
    want, rc = create_code(O, A, H1, H2), _create(O, A, H1, H2)
    if want == OK:
        assert rc in (OK, ERR_CUDA), ((O, A, H1, H2), rc)        # accepted: fails only at its first CUDA call without a GPU
    else:
        assert rc == want, ((O, A, H1, H2), rc, want)


# ---- CPU: the table against the rule ----------------------------------------------------------------------------------
def test_every_table_row_is_accepted_and_the_table_covers_every_path():
    for O, A, H1, H2, prec in ROWS:
        assert create_code(O, A, H1, H2) == OK, (O, A, H1, H2)
        _assert_create_follows_the_rule(O, A, H1, H2)
        if prec == "tf32":
            assert tf32_accepted(O, A, H1, H2), (O, A, H1, H2)
    fp32 = [r for r in ROWS if r[4] == "fp32"]
    tf32 = [r for r in ROWS if r[4] == "tf32"]
    assert {r[:2] for r in ROWS} >= {(4, 2), (16, 4)}
    assert {r[0] for r in fp32} >= {1, 32} and {r[1] for r in ROWS} >= {1, 8}
    assert {r[3] for r in ROWS} >= {4, 12, 100, 128} and {r[2] for r in ROWS} >= {8, 64, 200, 256}
    assert any(16 * r[3] // 4 == 512 for r in fp32)                                 # the launch bound
    assert any(16 * r[3] // 4 < 64 for r in fp32)                                   # block rounded up on 64-env tiles
    assert any(r[2] == MAX_H1 for r in fp32)                                        # the largest hidden1
    assert {tc_instance(r[0], r[1]) for r in tf32} == {(4, 1), (4, 2), (4, 8), (4, 0), (16, 2), (16, 4), (16, 0), (0, 0)}
    assert any(r[3] == 128 for r in tf32) and any(r[2] == 8 for r in tf32)
    assert all(r[0] <= 16 for r in tf32)


def test_create_refuses_exactly_past_each_limit():
    cases = [  # (O, A, H1, H2), the code rexagent_create must return
        ((0, 2, 64, 12), ERR_INVALID), ((1, 2, 64, 12), OK), ((32, 2, 64, 12), OK), ((33, 2, 64, 12), ERR_INVALID),
        ((4, 0, 64, 12), ERR_INVALID), ((4, 1, 64, 12), OK), ((4, 8, 64, 12), OK), ((4, 9, 64, 12), ERR_INVALID),
        ((4, 1, 3, 4), ERR_UNSUPPORTED), ((4, 1, 4, 4), OK), ((4, 1, 256, 4), OK), ((4, 1, 260, 4), ERR_UNSUPPORTED),
        ((4, 1, 64, 3), ERR_UNSUPPORTED), ((4, 1, 64, 4), OK), ((4, 1, 200, 128), OK), ((4, 1, 200, 132), ERR_UNSUPPORTED),
        ((4, 1, 66, 12), ERR_UNSUPPORTED), ((4, 1, 64, 14), ERR_UNSUPPORTED),                    # not multiples of 4
        ((4, 8, 64, 32), OK), ((4, 8, 64, 36), ERR_UNSUPPORTED),                                  # A * H2 / 4 <= H1
    ]
    # the first hidden1 whose fp32 kernel does not fit in shared memory, at hidden2 = 128 and at the widest input
    for O, A, H2 in ((4, 2, 128), (32, 1, 100)):
        h1 = next(h for h in range(4, MAX_H1 + 1, 4) if fp32_smem_bytes(O, A, h, H2) > SMEM)
        assert fp32_smem_bytes(O, A, h1 - 4, H2) <= SMEM < fp32_smem_bytes(O, A, h1, H2)
        cases += [((O, A, h1 - 4, H2), OK), ((O, A, h1, H2), ERR_UNSUPPORTED)]
    for cfg, want in cases:
        assert create_code(*cfg) == want, cfg
        _assert_create_follows_the_rule(*cfg)


def test_parameter_block_sizes_match_the_oracle_packing():
    _capi, L = _lib()
    for O, A, H1, H2, _ in ROWS + [(33, 9, 300, 132, "")]:
        cfg = _capi.RexAgentConfig(O, A, H1, H2, 5.0, 10.0)
        shapes = dict(pW1=(O, H1), pb1=(H1,), pW2=(H1, H2), pb2=(H2,), pW3=(H2, A), pb3=(A,), logstd=(A,),
                      vW1=(O, H1), vb1=(H1,), vW2=(H1, H2), vb2=(H2,), vW3=(H2, 1), vb3=(1,))
        block = AO.pack_params({k: np.zeros(s, np.float32) for k, s in shapes.items()}, O, A, H1, H2)
        npol, nval = L.rexagent_policy_floats(C.byref(cfg)), L.rexagent_value_floats(C.byref(cfg))
        assert (npol, nval) == (policy_floats(O, A, H1, H2), value_floats(O, A, H1, H2))
        assert npol + nval == block.size and npol % 4 == 0 and nval % 4 == 0
        w = {k: np.arange(np.prod(s), dtype=np.float32).reshape(s) + i for i, (k, s) in enumerate(shapes.items())}
        back = AO.unpack_params(AO.pack_params(w, O, A, H1, H2), O, A, H1, H2)
        for k in shapes:
            np.testing.assert_array_equal(back[k], w[k])


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _half():
    return max(torch.cuda.get_device_properties(0).multi_processor_count // 2, 1)


def batch_sizes(half):
    """The sizes around every tiling switch of the fp32 kernel on a device with 2 * half SMs."""
    return [1, 63, 64, 65, 129, 64 * half, 64 * half + 1,       # 64 * half + 1: a second 64-env tile on CTA 0
            128 * (half - 1), 128 * (half - 1) + 1,              # the last size on 64-env tiles, the first on 128-env tiles
            128 * half + 1, 65536 + 37]


def tiling(n, half, prec):
    if prec == "tf32":
        tm = 128
    else:
        tm = 128 if (n + 127) // 128 >= half else 64
    ntiles = (n + tm - 1) // tm
    return tm, ntiles, min(ntiles, half)


def probe_envs(n, tm, ntiles, grid):
    """First and last env of every CTA's second and last tile, and the last env of the batch."""
    s = {0, n - 1}
    for b in range(grid):
        tiles = list(range(b, ntiles, grid))
        for t in set(tiles[1:2] + tiles[-1:]):
            s.update((t * tm, min((t + 1) * tm, n) - 1))
    return np.array(sorted(s))


def _weights(rng, O, A, H1, H2):
    """Per-layer scale 1 / sqrt(fan_in) (sqrt(2 / fan_in) after a ReLU) keeps every pre-activation O(1) at every width."""
    def dense(i, o, gain):
        return (rng.standard_normal((i, o)) * gain / math.sqrt(i)).astype(np.float32)

    def bias(k):
        return rng.normal(0, 0.1, k).astype(np.float32)
    return dict(pW1=dense(O, H1, 0.7), pb1=bias(H1), pW2=dense(H1, H2, math.sqrt(2)), pb2=bias(H2), pW3=dense(H2, A, 1.0),
                pb3=bias(A), logstd=rng.uniform(-1.2, -0.5, A).astype(np.float32),
                vW1=dense(O, H1, 0.7), vb1=bias(H1), vW2=dense(H1, H2, math.sqrt(2)), vb2=bias(H2), vW3=dense(H2, 1, 1.0), vb3=bias(1))


def _noise(seed, step, genv, A):
    return np.array([[AO.normal_noise(seed, int(g), step, a) for a in range(A)] for g in genv])


def _setup(row, n_max):
    from rex_gym_b200.agents import ForwardGaussianPolicy
    O, A, H1, H2, prec = row
    rng = np.random.default_rng(1000 * O + 100 * A + H1 + H2 + (7 if prec == "tf32" else 0))
    w = _weights(rng, O, A, H1, H2)
    f = AO.StreamingNormalize((O,), True, True, 5)
    f.update(rng.normal(0.3, 1.7, (5000, O)))
    obs = rng.normal(0.3, 3.0, (n_max, O)).astype(np.float32)
    obs[0], obs[n_max // 3] = 100.0, -100.0                             # clipped at +-5 after normalisation
    nets = []
    for tc in ((False, True) if prec == "tf32" else (False,)):
        net = ForwardGaussianPolicy(O, A, (H1, H2), (H1, H2), seed=1, tensor_cores=tc)
        net.set_weights(w)
        net.set_filters(f.count, f.mean, f.var_sum, 0, 0.0, 0.0)
        nets.append(net)
    return w, f, obs, nets


SEED, STEP, OFFSET = 99, 5, 1000


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROWS, ids=row_id)
def test_perform_matches_the_oracle_at_every_batch_size(row):
    """fp32: mean 2e-5, value 5e-5, sampled action 5e-5, log-prob 2e-4 (the bounds of test_gpu_agent.py).  tf32: mean and
    value 5e-3 against the oracle and against the fp32 kernel (a K <= 256 dot product of O(1) terms at 2^-11 relative operand
    error); the sampled action adds the noise term, which does not pass through the tensor cores, so it gets the tf32 mean
    bound plus the fp32 action bound, 5e-3 + 5e-5; log-prob 2e-4 as in fp32.  Every output alone equals the all-outputs run
    bit for bit, and observ_copy equals the input."""
    O, A, H1, H2, prec = row
    half = _half()
    sizes = batch_sizes(half)
    w, f, obs, nets = _setup(row, max(sizes))
    net = nets[-1]
    want_mean, logstd, want_value = AO.forward_gaussian_policy(w, f.transform(obs))
    x_all = torch.from_numpy(obs).cuda()
    tol = dict(mean=2e-5, value=5e-5, action=5e-5) if prec == "fp32" else dict(mean=5e-3, value=5e-3, action=5e-3 + 5e-5)
    for n in sizes:
        x = x_all[:n]
        det = {k: t.cpu().numpy() for k, t in net.perform(x, training=False).items()}
        cp = torch.full_like(x, float("nan"))
        out = net.perform(x, training=True, seed=SEED, step=STEP, env_offset=OFFSET, observ_copy=cp)
        g = {k: t.cpu().numpy() for k, t in out.items()}
        assert torch.equal(cp, x), n
        em, ev = np.abs(det["mean"] - want_mean[:n]).max(), np.abs(det["value"] - want_value[:n]).max()
        assert em < tol["mean"] and ev < tol["value"], (n, em, ev)
        assert np.array_equal(det["action"], det["mean"]) and np.array_equal(g["mean"], det["mean"]), n
        assert np.array_equal(g["value"], det["value"]), n
        idx = np.unique(np.r_[probe_envs(n, *tiling(n, half, prec)), np.linspace(0, n - 1, 16).astype(int)])
        z = _noise(SEED, STEP, OFFSET + idx, A)
        want_a = want_mean[idx] + np.exp(logstd)[None, :] * z
        want_lp = (-0.5 * z * z - logstd[None, :] - 0.5 * math.log(2 * math.pi)).sum(1)
        ea, elp = np.abs(g["action"][idx] - want_a).max(), np.abs(g["logprob"][idx] - want_lp).max()
        assert ea < tol["action"] and elp < 2e-4, (n, ea, elp)
        for k in ("action", "mean", "logprob", "value"):                  # one output at a time
            one = {k: torch.full_like(out[k], float("nan"))}
            net.perform(x, training=True, seed=SEED, step=STEP, env_offset=OFFSET, out=one)
            assert torch.equal(one[k], out[k]), (n, k)
        boot = {"value": torch.full_like(out["value"], float("nan"))}   # Rollout's bootstrap call
        net.perform(x, training=False, out=boot)
        assert np.array_equal(boot["value"].cpu().numpy(), det["value"]), n
        if prec == "tf32":                                               # the same inputs through the fp32 kernel
            r = {k: t.cpu().numpy() for k, t in nets[0].perform(x, training=True, seed=SEED, step=STEP, env_offset=OFFSET).items()}
            assert np.abs(g["mean"] - r["mean"]).max() < 5e-3 and np.abs(g["value"] - r["value"]).max() < 5e-3, n
            assert np.abs((g["action"] - g["mean"]) - (r["action"] - r["mean"])).max() < 1e-5, n
    for nt in nets:
        nt.close()


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROWS, ids=row_id)
def test_perform_does_not_depend_on_the_env_position(row, capsys):
    """Every sum of perform_kernel runs in an order fixed by the code, whatever TM and the env's place in its tile: an env's
    mean, value and noise-free action are bit-identical inside a batch of n, inside a batch of 128 * (half - 1) + 1 (128-env
    tiles) and alone in a batch of 1; so are its sampled action and log-prob when the lone run carries env_offset = env.
    The tensor-core form is held to 1e-6 and reports whether it is bit-identical too."""
    O, A, H1, H2, prec = row
    half = _half()
    n_big = 128 * (half - 1) + 1
    sizes = [64 * half + 1, 128 * (half - 1), 65536 + 37]
    _, _, obs, nets = _setup(row, max(sizes))
    net = nets[-1]
    x_all = torch.from_numpy(obs).cuda()
    worst = 0.0
    for n in sizes:
        tm, ntiles, grid = tiling(n, half, prec)
        envs = np.unique(np.r_[probe_envs(n, tm, ntiles, grid)[:6], probe_envs(n, tm, ntiles, grid)[-6:], n // 2, 1])
        x = x_all[:n]
        det = {k: t.cpu().numpy() for k, t in net.perform(x, training=False).items()}
        smp = {k: t.cpu().numpy() for k, t in net.perform(x, training=True, seed=SEED, step=STEP).items()}
        pos = np.linspace(0, n_big - 1, len(envs)).astype(int)            # distinct places in the 128-env-tile batch
        xb = x_all[:n_big].clone()
        xb[torch.from_numpy(pos).cuda()] = x[torch.from_numpy(envs).cuda()]
        big = {k: t.cpu().numpy() for k, t in net.perform(xb, training=False).items()}
        got = [(det, envs, big, pos, ("action", "mean", "value"))]
        for e in envs:
            one = {k: t.cpu().numpy() for k, t in net.perform(x[e:e + 1], training=True, seed=SEED, step=STEP, env_offset=int(e)).items()}
            got.append((smp, np.array([e]), one, np.array([0]), ("action", "mean", "logprob", "value")))
            lone = {k: t.cpu().numpy() for k, t in net.perform(x[e:e + 1], training=False).items()}
            got.append((det, np.array([e]), lone, np.array([0]), ("action", "mean", "value")))
        for ref, ri, other, oi, keys in got:
            for k in keys:
                d = np.abs(ref[k][ri] - other[k][oi]).max()
                worst = max(worst, float(d))
                if prec == "fp32":
                    assert d == 0, (n, k, ri[:4], d)
                else:
                    assert d <= 1e-6, (n, k, ri[:4], d)
    with capsys.disabled():
        print("\n%s: largest difference across batch positions %.3g (%s)" % (row_id(row), worst,
                                                                              "bit-identical" if worst == 0 else "not bit-identical"))
    for nt in nets:
        nt.close()


def _filters_match(g, fo, fr):
    assert g["observ_count"] == fo.count and g["reward_count"] == fr.count, (g["observ_count"], fo.count)
    np.testing.assert_allclose(g["observ_mean"], fo.mean, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(g["observ_var_sum"], fo.var_sum, rtol=5e-5, atol=1e-5)
    np.testing.assert_allclose(g["reward_mean"], fr.mean, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(g["reward_var_sum"], fr.var_sum, rtol=5e-5, atol=1e-5)


def _experience_split(net, x, r):
    """The env-sharded form on one rank: partial sums of the whole batch, then finalize."""
    from rex_gym_b200 import _capi
    sums = torch.zeros((net.O + 1, 2), dtype=torch.float32, device="cuda")
    st = net._stream()
    _capi.check(net._L.rexagent_experience_partial(net._h, x.data_ptr(), r.data_ptr(), x.shape[0], sums.data_ptr(), st))
    _capi.check(net._L.rexagent_experience_finalize(net._h, sums.data_ptr(), x.shape[0], x.data_ptr(), r.data_ptr(), st))


@pytest.mark.gpu
@pytest.mark.parametrize("O", [1, 4, 32])
def test_experience_at_every_reduction_shape(O):
    """One block per 256 envs up to RED_BLOCKS = 256 blocks (65 536 envs), then strided rows; the first call has n = 1 (the
    count <= 1 branch: the mean becomes the first row).  The single call and partial + finalize both follow the oracle."""
    from rex_gym_b200.agents import ForwardGaussianPolicy
    rng = np.random.default_rng(40 + O)
    a, b = ForwardGaussianPolicy(O, 1, (64, 12), (64, 12)), ForwardGaussianPolicy(O, 1, (64, 12), (64, 12))
    fo, fr = AO.StreamingNormalize((O,), True, True, 5), AO.StreamingNormalize((), False, True, 10)
    for n in (1, 2, 255, 256, 257, 65535, 65536, 65537, 1048576):
        obs = rng.normal(0.5, 2.0, (n, O)).astype(np.float32)
        rew = rng.normal(0.1, 0.3, n).astype(np.float32)
        x, r = torch.from_numpy(obs).cuda(), torch.from_numpy(rew).cuda()
        a.experience(x, r)
        _experience_split(b, x, r)
        fo.update(obs); fr.update(rew)
        for net in (a, b):
            _filters_match(net.get_filters(), fo, fr)
        if n == 1:
            np.testing.assert_array_equal(a.get_filters()["observ_mean"], obs[0])
    assert int(a._cnt[2]) == int(b._cnt[2]) == 9 and int(a._cnt[3]) == int(b._cnt[3]) == 0
    rr = rng.normal(0, 5, 5000).astype(np.float32)
    for net in (a, b):
        got = net.transform_reward(torch.from_numpy(rr).cuda()).cpu().numpy()
        np.testing.assert_allclose(got, fr.transform(rr), rtol=1e-5, atol=1e-6)
    a.close(); b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("count", [0, 1, 2, 5000])
def test_transform_reward_scales_and_clips(count):
    """count <= 1: no scaling, only the clip at +-10; count >= 2: divided by sqrt(var_sum / (count - 1) + 1e-4) + 1e-8."""
    from rex_gym_b200.agents import ForwardGaussianPolicy
    rng = np.random.default_rng(count)
    net = ForwardGaussianPolicy(4, 2)
    fr = AO.StreamingNormalize((), False, True, 10)
    fr.count, fr.mean, fr.var_sum = count, np.float64(np.float32(0.3)), np.float64(np.float32(0.5 * max(count - 1, 0)))
    net.set_filters(0, np.zeros(4), np.zeros(4), count, 0.3, float(fr.var_sum))
    rr = np.r_[rng.normal(0, 20, 3000), 1e6, -1e6, 10.0, -10.0, 0.0].astype(np.float32)
    got = net.transform_reward(torch.from_numpy(rr).cuda()).cpu().numpy()
    want = fr.transform(rr)
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-6)
    assert got.max() == 10.0 and got.min() == -10.0 and (np.abs(got) == 10.0).sum() > 100
    net.close()


@pytest.mark.gpu
@pytest.mark.parametrize("split", [False, True], ids=["experience", "partial_finalize"])
@pytest.mark.parametrize("start", [2**31 - 1000, 2**32 + 5])
def test_filter_counts_go_past_two_to_the_31(start, split):
    """At 65 536 envs the observation count passes 2^31 after 32 768 control steps.  Counts are 64-bit: they match the
    oracle's integers exactly across 2^31, mean and var_sum follow it, and the next perform and reward transform still scale.
    The batches sit 1000 above the running means, so each update moves mean and var_sum by at least ten times the tolerance
    of the comparison (asserted on the oracle): a count that reached the division wrapped or in 32 bits would show."""
    from rex_gym_b200.agents import ForwardGaussianPolicy
    O, A, n = 4, 2, 4096
    rng = np.random.default_rng(start % 1000 + split)
    net = ForwardGaussianPolicy(O, A, seed=2)
    w = net.get_weights()
    fo, fr = AO.StreamingNormalize((O,), True, True, 5), AO.StreamingNormalize((), False, True, 10)
    m0 = rng.normal(0.3, 0.3, O).astype(np.float32)
    v0 = ((start - 1) * rng.uniform(1.0, 3.0, O)).astype(np.float32)
    rm0, rv0 = np.float32(0.1), np.float32((start - 1) * 0.09)
    net.set_filters(start, m0, v0, start, float(rm0), float(rv0))
    fo.count, fo.mean, fo.var_sum = start, m0.astype(np.float64), v0.astype(np.float64)
    fr.count, fr.mean, fr.var_sum = start, np.float64(rm0), np.float64(rv0)
    _filters_match(net.get_filters(), fo, fr)
    def moved(new, old, rtol, atol):               # the update is at least ten times what _filters_match tolerates
        return np.all(np.abs(np.asarray(new) - old) > 10 * (rtol * np.abs(new) + atol))

    for _ in range(3):
        obs = rng.normal(fo.mean + 1000.0, 1.5, (n, O)).astype(np.float32)
        rew = rng.normal(fr.mean + 1000.0, 0.3, n).astype(np.float32)
        x, r = torch.from_numpy(obs).cuda(), torch.from_numpy(rew).cuda()
        if split:
            _experience_split(net, x, r)
        else:
            net.experience(x, r)
        before = (fo.mean, fo.var_sum, fr.mean, fr.var_sum)
        fo.update(obs); fr.update(rew)
        assert moved(fo.mean, before[0], 2e-5, 2e-6) and moved(fo.var_sum, before[1], 5e-5, 1e-5)
        assert moved(fr.mean, before[2], 2e-5, 2e-6) and moved(fr.var_sum, before[3], 5e-5, 1e-5)
        _filters_match(net.get_filters(), fo, fr)
    assert fo.count == start + 3 * n and int(net._cnt[0]) == int(net._cnt[1]) == fo.count and int(net._cnt[2]) == 3
    obs = rng.normal(fo.mean, 1.5 * np.sqrt(fo.var_sum / (fo.count - 1)), (n, O)).astype(np.float32)    # around the filter
    x = torch.from_numpy(obs).cuda()
    out = net.perform(x, training=False)
    _, m, _, v = AO.perform(w, fo, obs, False)
    np.testing.assert_allclose(out["mean"].cpu().numpy(), m, atol=2e-5)
    np.testing.assert_allclose(out["value"].cpu().numpy(), v, atol=5e-5)
    rr = rng.normal(0, 2, 3000).astype(np.float32)
    np.testing.assert_allclose(net.transform_reward(torch.from_numpy(rr).cuda()).cpu().numpy(), fr.transform(rr), rtol=1e-5, atol=1e-6)
    net.close()


# ---- scans ------------------------------------------------------------------------------------------------------------
def _scan_atol(L, want, *inputs, base=1e-4):
    """Rounding of a length-L recurrence agg_t = cur_t + g * agg_{t+1} (g <= 1): every step adds at most u * (|g agg| + |agg_t|)
    for its two roundings and 9 u M for the (at most three) roundings of cur_t, u = 2^-24, M = the largest input; earlier
    errors are multiplied by g <= 1.  So |error| <= L u (2 max|agg| + 9 M); the GAE advantage rounds g * lambda * nd * adv as
    well, counted by doubling the first term.  The floor is the 1e-4 (2e-4 for advantages) of test_gpu_agent.py; at L = 1000
    with discount 1 the sums reach |agg| ~ 100 and the bound is ~3e-2."""
    M = max(float(np.abs(i).max()) for i in inputs)
    return max(base, L * 2.0**-24 * (4 * float(np.abs(want).max()) + 9 * M))


SCAN_LENGTHS = [1, 7, 8, 9, 1000]


@pytest.mark.gpu
@pytest.mark.parametrize("discount", [0.0, 0.985, 1.0])
@pytest.mark.parametrize("L", SCAN_LENGTHS)
def test_row_scans_at_every_length(L, discount):
    """discounted_return / lambda_advantage with lengths 0, L and in between, contiguous rows and rows of a wider buffer
    (stride_e = L + 5).  The kernels load SCAN_U = 8 steps ahead: lengths below, at and above 8 and one far above."""
    from rex_gym_b200.agents import utility
    rng = np.random.default_rng(L * 10 + int(discount * 1000))
    E = 300
    g = float(np.float32(discount))                                      # the kernels receive the discount as a float
    wide_r = rng.normal(size=(E, L + 5)).astype(np.float32)
    wide_v = rng.normal(size=(E, L + 5)).astype(np.float32)
    r, v = wide_r[:, :L], wide_v[:, :L]
    length = rng.integers(0, L + 1, E).astype(np.int32)
    length[:3] = (0, L, min(1, L))
    want_r, want_a = AO.discounted_return(r, length, g), AO.lambda_advantage(r, v, length, g)
    tol_r, tol_a = _scan_atol(L, want_r, r), _scan_atol(L, want_a, r, v, base=2e-4)
    lt = torch.from_numpy(length).cuda()
    wr_t, wv_t = torch.from_numpy(wide_r).cuda(), torch.from_numpy(wide_v).cuda()
    views = [(torch.from_numpy(np.ascontiguousarray(r)).cuda(), torch.from_numpy(np.ascontiguousarray(v)).cuda()),
             (wr_t[:, :L], wv_t[:, :L])]
    assert views[1][0].stride() == (L + 5, 1)
    for rt, vt in views:
        got_r = utility.discounted_return(rt, lt, discount).cpu().numpy()
        got_a = utility.lambda_advantage(rt, vt, lt, discount).cpu().numpy()
        np.testing.assert_allclose(got_r, want_r, rtol=1e-4, atol=tol_r)
        np.testing.assert_allclose(got_a, want_a, rtol=1e-4, atol=tol_a)
        assert np.all(got_r[length == 0] == 0) and np.all(got_a[length == 0] == 0)
    if discount == 0:
        mask = np.arange(L)[None, :] < length[:, None]
        np.testing.assert_array_equal(got_r, np.where(mask, r, 0))
    # the strided rows written into a wide output buffer: the row view equals the result above, the padding columns keep
    # their NaN
    from rex_gym_b200 import _capi
    lib, st = _capi.load(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for which, want in (("return", got_r), ("advantage", got_a)):
        wide_out = torch.full((E, L + 5), float("nan"), device="cuda")
        if which == "return":
            _capi.check(lib.rexagent_discounted_return(wr_t.data_ptr(), lt.data_ptr(), E, L, L + 5, 1, discount, wide_out.data_ptr(), st))
        else:
            _capi.check(lib.rexagent_lambda_advantage(wr_t.data_ptr(), wv_t.data_ptr(), lt.data_ptr(), E, L, L + 5, 1, discount,
                                                      wide_out.data_ptr(), st))
        wo = wide_out.cpu().numpy()
        np.testing.assert_array_equal(wo[:, :L], want)
        assert np.isnan(wo[:, L:]).all(), which


@pytest.mark.gpu
@pytest.mark.parametrize("lam", [0.0, 0.95, 1.0])
@pytest.mark.parametrize("discount", [0.0, 0.985, 1.0])
@pytest.mark.parametrize("T", SCAN_LENGTHS)
def test_gae_segments_at_every_length(T, discount, lam):
    """Columns with done nowhere, on t = 0, on t = T - 1, everywhere and at random.  Either output may be NULL: the other is
    bit-identical to the both-outputs call."""
    from rex_gym_b200 import _capi
    from rex_gym_b200.agents import utility
    rng = np.random.default_rng(T * 100 + int(discount * 10) + int(lam * 1000))
    k = 61
    n = 5 * k
    r = rng.normal(size=(T, n)).astype(np.float32)
    v = rng.normal(size=(T + 1, n)).astype(np.float32)
    done = np.zeros((T, n), bool)
    done[0, k:2 * k] = True
    done[T - 1, 2 * k:3 * k] = True
    done[:, 3 * k:4 * k] = True
    done[:, 4 * k:] = rng.random((T, k)) < 0.05
    g, lm = float(np.float32(discount)), float(np.float32(lam))
    want_r, want_a = AO.gae_segments(r, v, done, g, lm)
    rt, vt, dt = torch.from_numpy(r).cuda(), torch.from_numpy(v).cuda(), torch.from_numpy(done).cuda()
    got_r, got_a = utility.gae_segments(rt, vt, dt, discount, lam)
    np.testing.assert_allclose(got_r.cpu().numpy(), want_r, rtol=1e-4, atol=_scan_atol(T, want_r, r, v))
    np.testing.assert_allclose(got_a.cpu().numpy(), want_a, rtol=1e-4, atol=_scan_atol(T, want_a, r, v, base=2e-4))
    L = _capi.load()
    d8 = dt.view(torch.uint8)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for keep in ("return", "advantage"):
        only = torch.full_like(rt, float("nan"))
        ptrs = (only.data_ptr(), None) if keep == "return" else (None, only.data_ptr())
        _capi.check(L.rexagent_gae_segments(rt.data_ptr(), vt.data_ptr(), d8.data_ptr(), T, n, float(discount), float(lam), *ptrs, st))
        assert torch.equal(only, got_r if keep == "return" else got_a), keep

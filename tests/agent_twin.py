"""A policy network on the device and its fp64 oracle, as the agent-kernel tests build, feed and compare them.

Not collected by pytest (like twin.py): the agent-kernel tests and tools/dev_ab_outputs.py import what they share from here.
Every helper draws from the generator it is handed, in a fixed order, so a test's inputs depend only on its seed and its calls.
"""
import math

import numpy as np
import torch

from oracle import agent_oracle as AO
from rex_gym_b200 import BatchedRexEnv
from rex_gym_b200.agents import ForwardGaussianPolicy, LinearGaussianPolicy, RecurrentGaussianPolicy, Rollout

SEED, STEP, OFFSET = 99, 5, 1000        # the sampled runs' noise key: seed, step, env_offset

# (O, A, H1, H2, precision).  The block of the fp32 kernel has 16 * H2 / 4 threads, rounded up to the tile's TM.
FF_ROWS = [
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

GRU_ROWS = [  # (O, A, H1, G, value layers)
    (4, 2, 200, 100, (200, 100)),     # walk / turn / standup / poses with the shipped sizes
    (16, 4, 200, 100, (200, 100)),    # gallop
    (1, 1, 64, 12, (64, 12)),         # O = 1; 48 of the block's 128 threads compute cell columns
    (32, 3, 64, 32, (64, 12)),        # O = 32
    (4, 8, 64, 16, (64, 12)),         # A = 8
    (4, 2, 36, 8, (64, 12)),          # small G, H1 = 4 mod 8: K = 44, a 12-row tail chunk
    (4, 2, 256, 128, (64, 12)),       # the largest H1 and G: 512 threads, 24 chunks
]

LIN_ROWS = [(4, 2, (200, 100)), (16, 4, (200, 100)), (32, 8, (64, 12)), (1, 1, (64, 12))]    # (O, A, value layers)


def ff_id(r):
    return "O%d-A%d-%dx%d-%s" % r


def gru_id(r):
    return "O%d-A%d-%dx%d" % r[:4]


def lin_id(r):
    return "O%d-A%d" % r[:2]


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def half_sm():
    """The fp32 perform kernel's largest grid: SMs / 2 persistent CTAs per network."""
    return max(sm_count() // 2, 1)


def ff_batch_sizes(half):
    """The sizes around every tiling switch of the fp32 kernel on a device with 2 * half SMs."""
    return [1, 63, 64, 65, 129, 64 * half, 64 * half + 1,       # 64 * half + 1: a second 64-env tile on CTA 0
            128 * (half - 1), 128 * (half - 1) + 1,              # the last size on 64-env tiles, the first on 128-env tiles
            128 * half + 1, 65536 + 37]


def gru_batch_sizes():
    """The sizes around the 64-env tiles of gru_policy_kernel on min(tiles, SMs) CTAs and its value network's tile switch."""
    sm = sm_count()
    return [1, 63, 64, 65, 64 * sm, 64 * sm + 1, 128 * (sm - 1), 128 * (sm - 1) + 1]


def tiling(n, half, prec):
    """(TM, tiles, CTAs) of a perform call on n envs: the tf32 kernel always takes 128-env tiles."""
    tm = 128 if prec == "tf32" or (n + 127) // 128 >= half else 64
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


def tile_probes(n, tm=64):
    """First and last env of the first, second and last tiles, a spread, and the last env."""
    s = {0, n - 1}
    for t in {0, 1, (n - 1) // tm}:
        s.update((min(t * tm, n - 1), min((t + 1) * tm, n) - 1))
    s.update(np.linspace(0, n - 1, 24).astype(int).tolist())
    return np.array(sorted(s))


def param_shapes(O, A, H1, H2):
    """The feed-forward parameter set, in TF variable order."""
    return dict(pW1=(O, H1), pb1=(H1,), pW2=(H1, H2), pb2=(H2,), pW3=(H2, A), pb3=(A,), logstd=(A,),
                vW1=(O, H1), vb1=(H1,), vW2=(H1, H2), vb2=(H2,), vW3=(H2, 1), vb3=(1,))


def _dense(rng, i, o, gain):
    return (rng.standard_normal((i, o)) * gain / math.sqrt(i)).astype(np.float32)


def _bias(rng, k, m=0.0):
    return (m + rng.normal(0, 0.1, k)).astype(np.float32)


def _value_block(rng, O, H1, H2):
    return dict(vW1=_dense(rng, O, H1, 0.7), vb1=_bias(rng, H1), vW2=_dense(rng, H1, H2, math.sqrt(2)), vb2=_bias(rng, H2),
                vW3=_dense(rng, H2, 1, 1.0), vb3=_bias(rng, 1))


def ff_weights(rng, O, A, H1, H2):
    """Per-layer scale 1 / sqrt(fan_in) (sqrt(2 / fan_in) after a ReLU) keeps every pre-activation O(1) at every width."""
    w = dict(pW1=_dense(rng, O, H1, 0.7), pb1=_bias(rng, H1), pW2=_dense(rng, H1, H2, math.sqrt(2)), pb2=_bias(rng, H2),
             pW3=_dense(rng, H2, A, 1.0), pb3=_bias(rng, A), logstd=rng.uniform(-1.2, -0.5, A).astype(np.float32))
    w.update(_value_block(rng, O, H1, H2))
    return w


def gru_weights(rng, O, A, H1, G, vl):
    """ff_weights' law for the dense layer, the head and the value network (layers vl); the gate biases around 1."""
    w = dict(pW1=_dense(rng, O, H1, 0.7), pb1=_bias(rng, H1), w_ru=_dense(rng, H1 + G, 2 * G, 1.0), b_ru=_bias(rng, 2 * G, 1.0),
             w_c=_dense(rng, H1 + G, G, 1.0), b_c=_bias(rng, G), pW3=_dense(rng, G, A, 1.0), pb3=_bias(rng, A),
             logstd=rng.uniform(-1.2, -0.5, A).astype(np.float32))
    w.update(_value_block(rng, O, *vl))
    return w


def lin_head(rng, O, A):
    """The linear policy's pW, pb."""
    return dict(pW=(rng.standard_normal((O, A)) / math.sqrt(O)).astype(np.float32), pb=rng.normal(0, 0.1, A).astype(np.float32))


def lin_weights(rng, O, A, vl):
    """gru_weights at H1 = G = 4 (the linear network reads its value block and logstd), then lin_head."""
    w = gru_weights(rng, O, A, 4, 4, vl)
    w.update(lin_head(rng, O, A))
    return w


def flat_weights(rng, O, A, H1=200, H2=100):
    """Every parameter N(0, 0.15), logstd as ff_weights'."""
    w = {k: rng.normal(0, 0.15, s).astype(np.float32) for k, s in param_shapes(O, A, H1, H2).items()}
    w["logstd"] = rng.uniform(-1.2, -0.5, A).astype(np.float32)
    return w


def fitted_filter(rng, O):
    """The oracle's observation filter after 5000 rows of N(0.3, 1.7)."""
    f = AO.StreamingNormalize((O,), True, True, 5)
    f.update(rng.normal(0.3, 1.7, (5000, O)))
    return f


def observations(rng, n, O, outliers=0.0):
    """n rows of N(0.3, 3.0); then, if `outliers`, that fraction of the rows set to 100, which the filter clips at +5."""
    obs = rng.normal(0.3, 3.0, (n, O)).astype(np.float32)
    if outliers:
        obs[rng.random(n) < outliers] = 100.0
    return obs


def load(net, w=None, f=None):
    """Weights w and observation filter f (the oracle's StreamingNormalize or a (count, mean, var_sum) triple; the reward
    filter empty) into net."""
    if w is not None:
        net.set_weights(w)
    if f is not None:
        count, mean, var_sum = (f.count, f.mean, f.var_sum) if isinstance(f, AO.StreamingNormalize) else f
        net.set_filters(count, mean, var_sum, 0, 0.0, 0.0)
    return net


def ff_net(O, A, H1, H2, w=None, f=None, tensor_cores=False, seed=0):
    return load(ForwardGaussianPolicy(O, A, (H1, H2), (H1, H2), seed=seed, tensor_cores=tensor_cores), w, f)


def gru_net(row, n, w, f):
    O, A, H1, G, vl = row
    return load(RecurrentGaussianPolicy(O, A, (H1, 100), vl, seed=1, num_envs=n, cell_size=G), w, f)


def lin_net(O, A, vl, n, w=None, f=None):
    return load(LinearGaussianPolicy(O, A, value_layers=vl, num_envs=n), w, f)


def ff_value_twin(O, A, vl, w, f, policy=None):
    """A feed-forward network with layers vl carrying w's value block (and `policy`'s entries): its value is the one the
    recurrent and linear networks compute, on the same kernel."""
    ff = ForwardGaussianPolicy(O, A, vl, vl, seed=1)
    ffw = ff.get_weights()
    ffw.update({k: w[k] for k in ("vW1", "vb1", "vW2", "vb2", "vW3", "vb3")})
    ffw.update(policy or {})
    return load(ff, ffw, f)


def ff_setup(row, n_max):
    """ff_weights, a fitted filter and n_max observations (rows 0 and n_max // 3 at +-100) drawn from the row's seed; the
    fp32 network and, on a tf32 row, the tensor-core network after it, both loaded with them."""
    O, A, H1, H2, prec = row
    rng = np.random.default_rng(1000 * O + 100 * A + H1 + H2 + (7 if prec == "tf32" else 0))
    w = ff_weights(rng, O, A, H1, H2)
    f = fitted_filter(rng, O)
    obs = observations(rng, n_max, O)
    obs[0], obs[n_max // 3] = 100.0, -100.0                             # clipped at +-5 after normalisation
    nets = [ff_net(O, A, H1, H2, w, f, tensor_cores=tc, seed=1) for tc in ((False, True) if prec == "tf32" else (False,))]
    return w, f, obs, nets


def to_numpy(out):
    return {k: t.cpu().numpy() for k, t in out.items()}


def filters_match(g, fo, fr):
    """A network's filters g (get_filters()) against the oracle's observation and reward filters."""
    assert g["observ_count"] == fo.count and g["reward_count"] == fr.count, (g["observ_count"], fo.count)
    np.testing.assert_allclose(g["observ_mean"], fo.mean, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(g["observ_var_sum"], fo.var_sum, rtol=5e-5, atol=1e-5)
    np.testing.assert_allclose(g["reward_mean"], fr.mean, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(g["reward_var_sum"], fr.var_sum, rtol=5e-5, atol=1e-5)


def experience_split(net, x, r):
    """The env-sharded form of experience on one rank: partial sums of the whole batch, then finalize."""
    from rex_gym_b200 import _capi
    sums = torch.zeros((net.O + 1, 2), dtype=torch.float32, device="cuda")
    st = net._stream()
    _capi.check(net._L.rexagent_experience_partial(net._h, x.data_ptr(), r.data_ptr(), x.shape[0], sums.data_ptr(), st))
    _capi.check(net._L.rexagent_experience_finalize(net._h, sums.data_ptr(), x.shape[0], x.data_ptr(), r.data_ptr(), st))


SCAN_LENGTHS = [1, 7, 8, 9, 1000]       # the scans load SCAN_U = 8 steps ahead: below, at and above 8, and far above


def noise(seed, step, genv, A):
    """The oracle's N(0, 1) draws [len(genv)][A] of global envs genv."""
    return np.array([[AO.normal_noise(seed, int(g), step, a) for a in range(A)] for g in genv])


def sampled(mean, logstd, z):
    """The oracle's sampled action mean + exp(logstd) z and its log-density sum(-z^2 / 2 - logstd - log(2 pi) / 2)."""
    logstd = np.asarray(logstd, np.float64)
    return mean + np.exp(logstd) * z, (-0.5 * z * z - logstd - 0.5 * math.log(2 * math.pi)).sum(1)


def rollout_graph_equals_the_step_by_step_loop(tensor_cores):
    """simulate(): T control steps of perform -> env.step -> experience captured as one CUDA graph; same buffers as the
    unrolled loop on twin environments, and consistent with stepping the env by hand with the recorded actions.  With
    tensor_cores=True the networks run perform_tc_kernel."""
    n, T = 512, 16
    kw = dict(task="walk", num_envs=n, signal_type="ik", normalize=True, auto_reset=True, max_episode_steps=25, target_position=2.0, backwards=False)
    outs = []
    for use_graph in (False, True):
        env = BatchedRexEnv(**kw)
        net = ForwardGaussianPolicy(env.obs_dim, env.action_dim, seed=3, tensor_cores=tensor_cores)
        ro = Rollout(env, net, T, seed=17, training=True, use_graph=use_graph)
        a = {k: v.clone() for k, v in ro.collect().items()}
        b = {k: v.clone() for k, v in ro.collect().items()}               # second window: continues the episodes
        outs.append((a, b, net.get_filters(), net.launch_count + env.launch_count))
        if use_graph:
            hand = BatchedRexEnv(**kw)
            o = torch.from_numpy(hand.reset()).cuda()
            for t in range(T):
                np.testing.assert_allclose(a["observ"][t].cpu().numpy(), o.cpu().numpy(), atol=1e-6)
                o2, r2, d2, _ = hand.step(a["action"][t])
                np.testing.assert_allclose(a["reward"][t].cpu().numpy(), r2.cpu().numpy(), atol=1e-6)
                np.testing.assert_array_equal(a["done"][t].cpu().numpy(), d2.cpu().numpy())
                o = o2.clone()
            hand.close()
        ret, adv = ro.returns_and_advantages(0.985, 0.95)
        wr, wa = AO.gae_segments(b["reward"].cpu().numpy(), b["value"].cpu().numpy(), b["done"].cpu().numpy(), 0.985, 0.95)
        np.testing.assert_allclose(ret.cpu().numpy(), wr, rtol=1e-4, atol=1e-4)
        np.testing.assert_allclose(adv.cpu().numpy(), wa, rtol=1e-4, atol=2e-4)
        env.close(); net.close()
    (a0, b0, f0, _), (a1, b1, f1, _) = outs
    for k in a0:
        np.testing.assert_array_equal(a0[k].cpu().numpy(), a1[k].cpu().numpy(), err_msg=k)
        np.testing.assert_array_equal(b0[k].cpu().numpy(), b1[k].cpu().numpy(), err_msg=k)
    assert f0["observ_count"] == f1["observ_count"] == 2 * T * n
    np.testing.assert_array_equal(f0["observ_var_sum"], f1["observ_var_sum"])
    assert b0["done"].any()                                              # LimitDuration(25) fired inside the second window
    assert np.abs((a0["action"] - a0["mean"]).cpu().numpy()).max() > 1e-3   # training: sampled actions

"""On-device episode statistics (BatchedRexEnv(episode_statistics=True), RexSimConfig.episode_stats): simulate()'s score and
length bookkeeping, its StreamingMean totals and RexGymEnv's objectives, kept by the step kernel.

CPU: the entry points are declared and exported, create validates the switch before any CUDA call, and the objectives restated
from the fp64 oracle's state make the reward its step returned.
GPU: with the switch on, every output of every step-kernel instance is bit-identical to the switch off; the bookkeeping equals a
host restatement from the returned rewards and dones, bit for bit, under auto-reset and under explicit resets; the summary is
independent of rebalancing, repeatable, resumable from a checkpoint and additive over shards; the objectives match the fp32
restatement of the kernel's state, the returned reward and the fp64 oracle; a graph-captured rollout keeps the same books.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest
import task_outputs as T
from twin import BUILDS, INSTANCES, NOISE, bound, force_build, instance_config, launched, make_env, make_oracle, row_id, sync

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("rexsim_episode_buffers", "rexsim_episode_summary")
OBJECTIVE_ROWS = [r for r in INSTANCES if r[0] in ("walk", "gallop")]
F32 = np.float32


# ---- CPU -----------------------------------------------------------------------------------------------------------------
def test_entry_points_are_declared_and_exported():
    from rex_gym_b200 import _capi
    L = _capi.load()
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rexsim.h")).read(), flags=re.S)
    for name in NEW:
        assert name in _capi.SIGNATURES and name in _capi.EXPORTS
        assert re.search(r"\b%s\s*\(" % name, header), name
        assert hasattr(L, name)
    assert [f for f, _ in _capi.RexSimConfig._fields_][-1] == "episode_stats"


def test_create_validates_the_switch_without_the_gpu():
    from rex_gym_b200 import _capi
    L = _capi.load()
    cfg = _capi.RexSimConfig()
    cfg.num_envs, cfg.num_motors, cfg.task, cfg.action_repeat, cfg.solver_iterations, cfg.sim_dt_d, cfg.toe_npts = 8, 12, 0, 5, 60, 0.001, 27
    cfg.gait_clock_scale = 1.0
    h = C.c_void_p()
    tb = np.zeros(952, np.float32)
    cfg.episode_stats = 1                 # accepted: the model table's size is checked next, still before any CUDA call
    assert L.rexsim_create(C.byref(cfg), tb.ctypes.data, 951, C.byref(h)) == -2
    cfg.episode_stats = 2
    assert L.rexsim_create(C.byref(cfg), tb.ctypes.data, 952, C.byref(h)) == -1
    assert b"episode_stats" in L.rexsim_last_error()
    # a null handle is refused by both entry points
    p = [C.c_void_p() for _ in range(5)] + [C.c_int64()]
    assert L.rexsim_episode_buffers(None, *(C.byref(x) for x in p)) == -1
    assert L.rexsim_episode_summary(None, 1, None) == -1


def _oracle_objectives(ora, cfg):
    """The fp64 oracle's objectives of the step it just took: RexGymEnv._reward's four terms before the weights, restated by
    task_outputs from the oracle's own post-step state (observed torques and sensor history included) -> [N][4]."""
    unit = T.types.SimpleNamespace(**{**vars(cfg), "w": (1.0, 1.0, 1.0, 1.0)})
    r = T.restate(unit, T.oracle_words(ora), T.oracle_ring(ora) if cfg.sensor else None)
    return np.stack([r.terms[k] for k in ("fwd", "energy", "drift", "shake")], 1), r


@pytest.mark.parametrize("task,sig,kw", [("walk", "ik", {}), ("gallop", "ol", dict(motor_kp_range=(0.8, 1.2))),
                                         ("walk", "ol", dict(mark="arm", control_latency=0.0125, observation_noise_stdev=NOISE))])
def test_oracle_objectives_make_its_reward(task, sig, kw):
    """The objectives the GPU tests take as the oracle's, weighted by the task's weights, sum to the reward the oracle's step
    returned (to its float32 rounding)."""
    n = 6
    ora = make_oracle(task, n, signal_type=sig, seed=3, **kw)
    cfg = T.cfg_of(ora)
    ora.reset()
    rng = np.random.default_rng(4)
    for _ in range(12):
        _, rew, _ = ora.step(rng.uniform(-bound(task, sig), bound(task, sig), size=(n, ora.A)).astype(np.float32))
        obj, _ = _oracle_objectives(ora, cfg)
        assert np.isfinite(obj).all()
        np.testing.assert_allclose(obj @ np.array(cfg.w), rew, rtol=1e-6, atol=1e-7)


# ---- GPU: helpers ----------------------------------------------------------------------------------------------------------
def _outputs(env):
    out = dict(state_f=env._state_f.cpu().numpy(), state_i=env._state_i.cpu().numpy(), cmd=env.last_command().cpu().numpy())
    if env._ring is not None:
        out["ring"] = env._ring.cpu().numpy()
    return out


def _totals(env, clear=False):
    return env.episode_totals(clear).cpu().numpy().copy()


class _Books:
    """simulate()'s bookkeeping restated on the host from what the steps returned: float32 score, int length, fp64 sums."""

    def __init__(self, n):
        self.score, self.length = np.zeros(n, F32), np.zeros(n, np.int64)
        self.count, self.sum_score, self.sum_length = 0, 0.0, 0

    def step(self, reward, done):
        self.score = (self.score + np.asarray(reward, F32)).astype(F32)
        self.length += 1
        d = np.asarray(done, bool)
        self.count += int(d.sum())
        self.sum_score += float(self.score[d].astype(np.float64).sum())
        self.sum_length += int(self.length[d].sum())
        self.score[d], self.length[d] = 0, 0

    def reset(self, idx):
        self.score[idx], self.length[idx] = 0, 0

    def check(self, env, label):
        np.testing.assert_array_equal(env.episode_score().cpu().numpy(), self.score, err_msg=f"score {label}")
        np.testing.assert_array_equal(env.episode_length().cpu().numpy(), self.length, err_msg=f"length {label}")

    def check_totals(self, t):
        assert t[0] == self.count and t[1] == 0 and t[3] == self.sum_length, (t, self.count, self.sum_length)
        assert abs(t[2] - self.sum_score) <= 1e-12 * max(1.0, abs(self.sum_score)), (t[2], self.sum_score)


# ---- GPU: the switch changes nothing else ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("row", INSTANCES, ids=[row_id(r) for r in INSTANCES])
def test_switch_leaves_every_output_bit_identical(row, monkeypatch):
    """60 auto-resetting steps of 15-step episodes, switch off and on: obs, reward, done, the whole SoA state, the sensor ring
    and the motor commands bit for bit, the state layout unchanged, and the switched-on books hold episodes."""
    task, sig, arm, terrain, build = row
    force_build(monkeypatch, build)
    n = 37
    kw = dict(instance_config(row), auto_reset=True)
    envs = [make_env(task, n, episode_statistics=s, **kw) for s in (False, True)]
    assert envs[0]._state_f.shape == envs[1]._state_f.shape and envs[0]._state_i.shape == envs[1]._state_i.shape
    assert set(envs[1].state_dict()) - set(envs[0].state_dict()) == {"episode_statistics"}
    for e in envs:
        e.reset()
    rng = np.random.default_rng(11)
    for k in range(60):
        a = rng.uniform(-bound(task, sig), bound(task, sig), size=(n, envs[0].action_dim)).astype(np.float32)
        res = [e.step(a)[:3] for e in envs]
        assert launched(envs[0]) == launched(envs[1]) == BUILDS[build]
        for x, y, what in zip(res[0], res[1], ("obs", "reward", "done")):
            np.testing.assert_array_equal(x, y, err_msg=f"{what}, step {k}")
    o0, o1 = _outputs(envs[0]), _outputs(envs[1])
    for key in o0:
        np.testing.assert_array_equal(o0[key], o1[key], err_msg=key)
    assert _totals(envs[1])[0] >= n
    for e in envs:
        e.close()


# ---- GPU: exact bookkeeping --------------------------------------------------------------------------------------------------
BOOK_CONFIGS = {
    "walk-ik": ("walk", dict(signal_type="ik")),
    "gallop-ol-gains": ("gallop", dict(signal_type="ol", motor_kp_range=(0.8, 1.2), motor_kd_range=(0.01, 0.03))),
    "standup-arm": ("standup", dict(signal_type="ol", mark="arm")),
    "turn-ik-heightfield-sensor": ("turn", dict(signal_type="ik", terrain_type="random", num_fields=4, control_latency=0.0125,
                                                observation_noise_stdev=NOISE)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("auto_reset", [True, False], ids=["auto-reset", "explicit-reset"])
@pytest.mark.parametrize("name", list(BOOK_CONFIGS))
def test_books_match_the_host_restatement(name, auto_reset):
    """300 steps of 96 envs with 25-step episodes, de-synchronised by resetting random envs over the first 25 steps (and, without
    auto-reset, resetting the done envs after every step as simulate() does).  After every step score and length equal the host's
    float32 restatement from the returned rewards and dones, bit for bit; a reset zeroes the listed envs only and submits nothing;
    the totals count every done, their length sum exactly and their score sum within 1e-12."""
    task, kw = BOOK_CONFIGS[name]
    n = 96
    env = make_env(task, n, seed=17, max_episode_steps=25, auto_reset=auto_reset, episode_statistics=True, **kw)
    env.reset()
    books = _Books(n)
    books.check(env, "after reset")
    rng = np.random.default_rng(5)
    b = 1.5 * bound(task, kw["signal_type"])
    dones = 0
    for k in range(300):
        if k < 25:
            idx = rng.choice(n, size=4, replace=False)
            before = _totals(env)
            env.reset(idx)
            books.reset(idx)
            np.testing.assert_array_equal(_totals(env), before)           # a reset submits nothing
        _, r, d, _ = env.step(rng.uniform(-b, b, size=(n, env.action_dim)).astype(np.float32))
        books.step(r, d)
        dones += int(d.sum())
        books.check(env, f"step {k}")
        if not auto_reset and d.any():
            env.reset(np.nonzero(d)[0])
            books.reset(np.nonzero(d)[0])
            books.check(env, f"reset after step {k}")
    assert dones == books.count and dones >= n
    books.check_totals(_totals(env))
    s = env.episode_summary()
    assert s["count"] == dones and s["nonfinite"] == 0
    assert s["mean_length"] == books.sum_length / dones
    assert abs(s["mean_score"] - books.sum_score / dones) <= 1e-12 * max(1.0, abs(books.sum_score / dones))
    assert env.episode_summary() == dict(count=0, nonfinite=0, mean_score=None, mean_length=None)     # cleared
    assert (env.check_errors() & 1) == 0
    env.close()


# ---- GPU: edge cases -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_non_finite_episode_is_counted_apart():
    """An inf injected through set_state (as in test_gpu_parity's error test): the env's episode ends non-finite -- counted in
    `nonfinite`, not submitted -- and its score and length restart."""
    import torch
    n = 8
    env = make_env("walk", n, signal_type="ik", target_position=2.0, backwards=False, auto_reset=True, episode_statistics=True)
    env.reset()
    a = torch.zeros((n, 2), device="cuda")
    env.step(a)
    st = env.get_state()
    bad = st["pos"].copy(); bad[3, 2] = np.inf
    env.set_state(bad, st["quat"], st["linvel"], st["angvel"], st["q"], st["qd"])
    _, r, d, _ = env.step(a)
    assert bool(d[3])
    with pytest.raises(ValueError):
        env.check_errors()
    s = env.episode_summary()
    assert s["nonfinite"] == 1 and s["count"] == int(d.sum()) - 1
    assert float(env.episode_score()[3]) == 0 and int(env.episode_length()[3]) == 0
    env.close()


def _walk_run(n, steps, seed=9, **kw):
    import torch
    env = make_env("walk", n, signal_type="ik", seed=seed, max_episode_steps=40, auto_reset=True, normalize=True,
                   episode_statistics=True, **kw)
    env.reset()
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    acts = torch.rand((steps, n, 2), device="cuda", generator=g) * 2 - 1
    return env, acts


@pytest.mark.gpu
def test_summary_is_independent_of_rebalance_and_repeatable():
    """8192 envs (where the warps are re-grouped), 120 steps: the totals, scores and lengths with re-grouping every step, twice, and
    without it -- bit for bit."""
    runs = []
    for every in (1, 1, 0):
        env, acts = _walk_run(8192, 120, rebalance_every=every)
        assert env._rebalance_every == every
        for k in range(120):
            env.step(acts[k])
        runs.append((_totals(env), env.episode_score().cpu().numpy(), env.episode_length().cpu().numpy()))
        env.close()
    assert runs[0][0][0] > 0
    for r in runs[1:]:
        for x, y in zip(runs[0], r):
            np.testing.assert_array_equal(x, y)


@pytest.mark.gpu
def test_state_dict_resumes_the_books():
    """A checkpoint after 30 steps, 30 more steps, the checkpoint loaded back and the same 30 steps again: score, length and the
    totals bit for bit."""
    env, acts = _walk_run(64, 60)
    for k in range(30):
        env.step(acts[k])
    sd = env.state_dict()
    assert sd["episode_statistics"].numel() == 64 * 32

    def finish():
        for k in range(30, 60):
            env.step(acts[k])
        return _totals(env), env.episode_score().cpu().numpy(), env.episode_length().cpu().numpy()
    first = finish()
    env.load_state_dict(sd)
    second = finish()
    assert first[0][0] > 0
    for x, y in zip(first, second):
        np.testing.assert_array_equal(x, y)
    env.close()


@pytest.mark.gpu
def test_shard_totals_add_up_to_the_batch():
    """Two handles with env_offset 0 and N/2 step the two halves of one batch's actions: their totals add up to the whole
    batch's (counts and lengths exactly, the score sum within 1e-12), and sharding.episode_summary without a process group is
    the handle's own summary."""
    from rex_gym_b200 import sharding
    n = 128
    whole, acts = _walk_run(n, 100)
    halves = [make_env("walk", n // 2, signal_type="ik", seed=9, max_episode_steps=40, auto_reset=True, normalize=True,
                       episode_statistics=True, env_offset=o) for o in (0, n // 2)]
    for h in halves:
        h.reset()
    for k in range(100):
        whole.step(acts[k])
        for j, h in enumerate(halves):
            h.step(acts[k, j * n // 2:(j + 1) * n // 2].contiguous())
    t = _totals(whole)
    parts = [_totals(h) for h in halves]
    s = parts[0] + parts[1]
    assert t[0] > 0 and t[0] == s[0] and t[1] == s[1] == 0 and t[3] == s[3]
    assert abs(t[2] - s[2]) <= 1e-12 * max(1.0, abs(t[2]))
    assert sharding.episode_summary(halves[0], clear=False) == halves[0].episode_summary(clear=False)
    for e in [whole] + halves:
        e.close()


# ---- GPU: objectives -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("row", OBJECTIVE_ROWS, ids=[row_id(r) for r in OBJECTIVE_ROWS])
def test_objectives_restate_and_make_the_reward(row, monkeypatch):
    """60 steps of 37 envs: the objectives equal task_outputs.restate at unit weights from the kernel's own words (energy where
    the sensor ring holds the observed torques), envs within 1e-5 of a reward threshold excused; weighted by
    objective_weights they sum to the returned reward at rounding level."""
    task, sig, arm, terrain, build = row
    force_build(monkeypatch, build)
    n = 37
    kw = instance_config(row)
    env, ora = make_env(task, n, episode_statistics=True, **kw), make_oracle(task, n, **kw)
    cfg = T.cfg_of(ora)
    unit = T.types.SimpleNamespace(**{**vars(cfg), "w": (1.0, 1.0, 1.0, 1.0)})
    w = np.array(env.objective_weights, np.float64)
    np.testing.assert_array_equal(w, np.array(cfg.w, F32))
    env.reset()
    rng = np.random.default_rng(13)
    for k in range(60):
        _, rg, _, _ = env.step(rng.uniform(-bound(task, sig), bound(task, sig), size=(n, env.action_dim)).astype(np.float32))
        assert launched(env) == BUILDS[build]
        ob = env.objectives().cpu().numpy().astype(np.float64)
        assert ob.shape == (n, 4)
        r = T.restate(unit, T.kernel_words(env), T.kernel_ring(env))
        ok = r.rew_margin >= 1e-5
        for j, key in enumerate(("fwd", "energy", "drift", "shake")):
            if r.terms[key] is None:
                continue
            tol = 2e-6 + (1e-5 if key == "energy" else 1e-6) * np.abs(r.terms[key])
            bad = (np.abs(ob[:, j] - r.terms[key]) > tol) & ok
            assert not bad.any(), f"{key}, step {k}, env {np.argmax(bad)}: {ob[bad, j][:3]} vs {r.terms[key][bad][:3]}"
        mag = np.abs(ob * w).sum(1)
        assert (np.abs(ob @ w - rg) <= 4e-7 * mag + np.spacing(np.abs(rg).astype(F32))).all(), f"reward, step {k}"
    assert ok.mean() > 0.9
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("row", OBJECTIVE_ROWS, ids=[row_id(r) for r in OBJECTIVE_ROWS])
def test_objectives_match_the_oracle(row, monkeypatch):
    """50 steps of 16 envs from the oracle's settled state (no auto-reset): each weighted objective within the 5e-3 test_gpu_parity
    holds rewards to, envs near a jump of the forward objective excused."""
    task, sig, arm, terrain, build = row
    force_build(monkeypatch, build)
    n = 16
    kw = dict(instance_config(row), max_episode_steps=0)
    env, ora = make_env(task, n, episode_statistics=True, **kw), make_oracle(task, n, **kw)
    cfg = T.cfg_of(ora)
    env.reset(); ora.reset()
    sync(env, ora)
    w = np.array(cfg.w)
    rng = np.random.default_rng(21)
    worst = 0.0
    for k in range(50):
        a = rng.uniform(-bound(task, sig), bound(task, sig), size=(n, env.action_dim)).astype(np.float32)
        env.step(a); ora.step(a)
        obj, r = _oracle_objectives(ora, cfg)
        ok = r.rew_margin >= 1e-2
        d = np.abs(env.objectives().cpu().numpy() - obj) * w
        worst = max(worst, float(d[ok].max(initial=0.0)))
        assert (d[ok] < 5e-3).all(), f"step {k}: {d[ok].max(0)}"
    print(f"{row_id(row)}: worst weighted objective difference {worst:.2e}")
    env.close()


@pytest.mark.gpu
def test_tasks_without_objectives_refuse():
    for task, sig in (("turn", "ik"), ("standup", "ol"), ("poses", "ik")):
        env = make_env(task, 4, signal_type=sig, episode_statistics=True)
        with pytest.raises(ValueError):
            env.objectives()
        assert env.episode_score().shape == (4,)
        env.close()
    env = make_env("walk", 4)
    for f in (env.objectives, env.episode_score, env.episode_length, env.episode_summary):
        with pytest.raises(ValueError):
            f()
    assert "episode_statistics" not in env.state_dict()
    env.close()


# ---- GPU: the rollout ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rollout_summary_in_and_out_of_the_graph():
    """Three 16-step collects of a graph-captured Rollout and of the plain loop on twin envs: the same summary, and the summary is
    the host restatement from rollout.reward and rollout.done."""
    from rex_gym_b200.agents import ForwardGaussianPolicy, Rollout
    n, T_ = 64, 16
    out = []
    for graph in (True, False):
        env = make_env("walk", n, signal_type="ik", seed=2, normalize=True, auto_reset=True, max_episode_steps=12,
                       episode_statistics=True)
        net = ForwardGaussianPolicy(env.obs_dim, env.action_dim, seed=1)
        ro = Rollout(env, net, T_, seed=2, training=True, use_graph=graph)
        books = _Books(n)
        for _ in range(3):
            b = ro.collect()
            for t in range(T_):
                books.step(b["reward"][t].cpu().numpy(), b["done"][t].cpu().numpy())
            books.check(env, f"graph={graph}")
        books.check_totals(_totals(env))
        out.append(ro.summary())
        assert out[-1]["count"] == books.count > 0
        env.close(); net.close()
    assert out[0] == out[1]

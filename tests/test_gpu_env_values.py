"""Per-env constructor values on the GPU: a batch whose envs were given different task keywords and gains runs each env
exactly as a batch built with that env's keywords as scalars would (the reference's BatchEnv over separately constructed
envs), in every step-kernel instance; the reset hold at each env's gains against the fp64 oracle; curricula, checkpoints
and sharding."""
import numpy as np
import pytest
import torch

from twin import BUILDS, INSTANCES, LAYOUT, TOL_P, TOL_Q, bound, force_build, instance_config, launched, make_env, make_oracle, row_id

pytestmark = pytest.mark.gpu

GAINS = [(1.0, 0.02), (1.3, 0.03), (0.8, 0.015)]          # the default pair, and two others


def value_table(task):
    """Small table of constructor-keyword tuples per task: fixed or drawn values, every direction, every pose coordinate."""
    if task == "walk":
        return [dict(target_position=t, backwards=b) for t in (None, 2.0) for b in (None, False, True)]
    if task == "gallop":
        return [dict(target_position=t) for t in (None, 1.5)]
    if task == "turn":
        return [dict(init_orient=i, target_orient=o) for i in (None, 1.0) for o in (None, 4.0)]
    if task == "poses":
        return [dict(base_y=0.005), dict(base_z=-0.02), dict(base_roll=0.3), dict(base_pitch=-0.2), dict(base_yaw=0.5), dict()]
    return [dict()]


def tuples_for(task, gains=True):
    """Full per-env tuples (keywords + motor_kp / motor_kd): the value table zipped cyclically with the three gain pairs."""
    vals = value_table(task)
    if not gains:
        return [dict(v) for v in vals]
    return [dict(vals[j % len(vals)], motor_kp=GAINS[j % 3][0], motor_kd=GAINS[j % 3][1]) for j in range(max(len(vals), 3))]


def mixed_keywords(tuples, n):
    """Env i takes tuple i % len(tuples): one list per keyword that any tuple names (None where a tuple leaves it out)."""
    names = sorted({k for t in tuples for k in t})
    default = dict(motor_kp=1.0, motor_kd=0.02)
    return {k: [tuples[i % len(tuples)].get(k, default.get(k)) for i in range(n)] for k in names}


def _bits(t):
    t = torch.as_tensor(t).contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _assert_rows_equal(a, b, rows, what):
    if len(rows) == 0:
        return
    a, b = _bits(a), _bits(b)
    bad = (a[rows] != b[rows]).reshape(len(rows), -1).any(1)
    assert not bad.any(), "%s differs in envs %s" % (what, torch.as_tensor(rows).cpu()[bad.cpu()].tolist())


def _assert_envs_equal(mixed, twin, envs, what, skip_i=()):
    """Raw state words (float and int, by name from the kernel's header) of `envs`, bit for bit."""
    sel = torch.as_tensor(envs, device="cuda")
    f1, f2 = mixed._state_f[:, sel], twin._state_f[:, sel]
    i1, i2 = mixed._state_i[:, sel], twin._state_i[:, sel]
    for w in range(LAYOUT.NF):
        assert torch.equal(_bits(f1[w]), _bits(f2[w])), "%s: float word %d of envs %s" % (what, w, envs)
    for w in range(LAYOUT.NI):
        if w not in skip_i:
            assert torch.equal(i1[w], i2[w]), "%s: int word %d of envs %s" % (what, w, envs)


def run_against_twins(task, n, cfg, tuples, steps=36, reset_at=17, extra=None):
    """A batch of n envs cycling through `tuples` and one scalar twin per tuple, stepped on the same actions with auto-reset
    and one explicit reset of some envs mid-run: every env's outputs and state words equal its twin's, bit for bit.
    extra(mixed, twin, envs, step) adds comparisons."""
    mixed = make_env(task, n, auto_reset=True, **cfg, **mixed_keywords(tuples, n))
    twins = [make_env(task, n, auto_reset=True, **cfg, **t) for t in tuples]
    groups = [np.arange(j, n, len(tuples)) for j in range(len(tuples))]
    idx = [torch.as_tensor(g, device="cuda") for g in groups]
    o = mixed.reset(torch.arange(n, dtype=torch.int32, device="cuda"))
    for t, g in zip(twins, idx):
        _assert_rows_equal(o, t.reset(torch.arange(n, dtype=torch.int32, device="cuda")), g, "reset obs")
    gen = torch.Generator(device="cuda"); gen.manual_seed(3)
    b = bound(task, cfg.get("signal_type", "ik"))
    mid = torch.tensor([1, n // 2, n - 2], dtype=torch.int32, device="cuda")
    for k in range(steps):
        a = (torch.rand((n, mixed.action_dim), device="cuda", generator=gen) * 2 - 1) * b
        om, rm, dm, _ = mixed.step(a)
        om, rm, dm = om.clone(), rm.clone(), dm.clone()
        for j, (t, g) in enumerate(zip(twins, idx)):
            ot, rt, dt, _ = t.step(a)
            _assert_rows_equal(om, ot, g, "obs, step %d, tuple %d" % (k, j))
            _assert_rows_equal(rm, rt, g, "reward, step %d, tuple %d" % (k, j))
            _assert_rows_equal(dm, dt, g, "done, step %d, tuple %d" % (k, j))
            _assert_envs_equal(mixed, t, groups[j], "step %d, tuple %d" % (k, j))
            if extra:
                extra(mixed, t, g, k)
        if k == reset_at:
            r = mixed.reset(mid)
            for t, g in zip(twins, idx):
                sel = torch.isin(mid.long(), g)
                _assert_rows_equal(r, t.reset(mid), torch.nonzero(sel).reshape(-1), "explicit reset obs")
    assert mixed.check_errors() == 0
    return mixed, twins


@pytest.mark.parametrize("row", INSTANCES, ids=row_id)
def test_mixed_batch_matches_scalar_twins_in_every_instance(row, monkeypatch):
    task, sig, arm, terrain, build = row
    force_build(monkeypatch, build)
    cfg = instance_config(row)
    ranges = "motor_kp_range" in cfg                       # per-env gains and drawn gains exclude each other
    tuples = tuples_for(task, gains=not ranges)
    mixed, twins = run_against_twins(task, 4 * len(tuples), cfg, tuples)
    assert launched(mixed) == BUILDS[build]
    if mixed._values is not None and not ranges:
        assert mixed._values["gains"].shape[0] == 3
    for e in [mixed] + twins:
        e.close()


@pytest.mark.parametrize("task,kw", [
    ("walk", dict(target_position=2.0, backwards=True, motor_kp=1.2, motor_kd=0.025)),
    ("turn", dict(init_orient=1.0, target_orient=4.0, terrain_type="random", num_fields=4, control_latency=0.0125)),
    ("poses", dict(base_z=-0.02, motor_kp=0.9)),
])
def test_all_equal_arrays_equal_the_scalar_construction(task, kw):
    n = 16
    arrays = {k: (v if k in ("terrain_type", "num_fields", "control_latency") else [v] * n) for k, v in kw.items()}
    mixed = make_env(task, n, auto_reset=True, seed=21, max_episode_steps=12, **arrays)
    twin = make_env(task, n, auto_reset=True, seed=21, max_episode_steps=12, **kw)
    assert mixed._values is not None
    everyone = torch.arange(n, device="cuda")
    _assert_rows_equal(mixed.reset(everyone), twin.reset(everyone), everyone, "reset obs")
    gen = torch.Generator(device="cuda"); gen.manual_seed(4)
    for k in range(30):
        a = (torch.rand((n, mixed.action_dim), device="cuda", generator=gen) * 2 - 1) * bound(task, "ik")
        om, rm, dm, _ = mixed.step(a)
        om, rm, dm = om.clone(), rm.clone(), dm.clone()
        ot, rt, dt, _ = twin.step(a)
        for x, y, what in ((om, ot, "obs"), (rm, rt, "reward"), (dm, dt, "done")):
            _assert_rows_equal(x, y, everyone, "%s, step %d" % (what, k))
        _assert_envs_equal(mixed, twin, np.arange(n), "step %d" % k)
    if twin._ring is not None:
        assert torch.equal(mixed._ring, twin._ring)
    mixed.close(); twin.close()


@pytest.mark.parametrize("terrain", ["plane", "random"])
def test_reset_hold_at_each_envs_gains_matches_the_oracle(terrain):
    """Rex.Reset's hold runs at the env's own gains (rex.py:314-323 -> ApplyAction -> self._kp): every pair's settled state
    against the fp64 oracle built with those gains, within the reset-hold tolerances of the parity tests."""
    n = 12
    kw = dict(signal_type="ik", seed=77, target_position=2.0, backwards=False)
    if terrain == "random":
        kw.update(terrain_type="random", num_fields=4)
    pair = np.arange(n) % 3
    env = make_env("walk", n, motor_kp=[GAINS[p][0] for p in pair], motor_kd=[GAINS[p][1] for p in pair], **kw)
    og = env.reset()
    sg = env.get_state()
    # flat: the north-star bound.  At gains other than the default the base is still moving when the hold ends, so its end
    # state is as sensitive to rounding as the arm's (measured on an H100: 1.6e-4 rad, 6.6e-5 m); bumps: toes creep on the
    # 45-degree block edges (measured: 4.8e-4 rad, 5.4e-5 m)
    tq, tp = (TOL_Q, TOL_P) if terrain == "plane" else (5e-3, 5e-3)
    spread = []
    for p, (kp, kd) in enumerate(GAINS):
        ora = make_oracle("walk", n, motor_kp=kp, motor_kd=kd, **kw)
        oc = ora.reset()
        so = ora.states()
        e = pair == p
        assert np.abs(sg["q"][e] - so["q"][e]).max() < tq and np.abs(sg["pos"][e] - so["pos"][e]).max() < tp
        assert np.abs(sg["quat"][e] - so["quat"][e]).max() < tq
        np.testing.assert_allclose(og[e][:, :2], oc[e][:, :2], atol=10 * tq)
        sf = env._state_f.cpu().numpy()
        np.testing.assert_array_equal(sf[LAYOUT.F_KP][e], np.float32(kp))
        np.testing.assert_array_equal(sf[LAYOUT.F_KD][e], np.float32(kd))
        spread.append(sg["q"][e][0])
    # the gains do change the settled pose: the hold is not the default pair's for every env
    assert np.abs(spread[1] - spread[0]).max() > 1e-3 or terrain == "random"
    assert env.check_errors() == 0
    env.close()


def test_composes_with_episode_statistics_final_observation_and_frame_history():
    cfg = dict(signal_type="ik", seed=13, max_episode_steps=15, episode_statistics=True, final_observation=True,
               frame_history=[0, 1, 3], frame_delta=True)

    def extra(mixed, twin, g, k):
        _assert_rows_equal(mixed.final_observation(), twin.final_observation(), g, "final obs, step %d" % k)
        _assert_rows_equal(mixed.limit_bytes(), twin.limit_bytes(), g, "limit byte, step %d" % k)
        for name in ("score", "length"):
            _assert_rows_equal(mixed._episode[name], twin._episode[name], g, "%s, step %d" % (name, k))
        _assert_rows_equal(mixed.objectives(), twin.objectives(), g, "objectives, step %d" % k)
        for key in mixed._frames:
            n = mixed.num_envs
            _assert_rows_equal(mixed._frames[key].view(-1, n).t(), twin._frames[key].view(-1, n).t(), g, key)
    mixed, twins = run_against_twins("walk", 24, cfg, tuples_for("walk"), extra=extra)
    for e in [mixed] + twins:
        e.close()


def test_set_task_values_between_graph_replays_takes_effect_at_the_next_reset():
    from rex_gym_b200.agents import ForwardGaussianPolicy, Rollout
    n = 32
    cfg = dict(normalize=True, auto_reset=True, max_episode_steps=20, seed=8)
    env = make_env("walk", n, target_position=[None] * n, backwards=[-1, 0, 1, 0] * (n // 4), **cfg)
    net = ForwardGaussianPolicy(env.obs_dim, env.action_dim, seed=1)
    ro = Rollout(env, net, 8, seed=2, training=False)
    env.reset()
    ro.collect()
    before = {k: v.clone() for k, v in env.task_values().items()}
    moved = torch.tensor([0, 5, 9, 30], dtype=torch.int32, device="cuda")
    env.set_task_values(moved, target_position=2.5, backwards=torch.ones(4, device="cuda"))
    after = env.task_values()
    assert torch.equal(after["episode_backwards"], before["episode_backwards"])      # running episodes keep their direction
    assert (after["target_position"][moved.long()] == 2.5).all() and (after["backwards"][moved.long()] == 1).all()
    rest = torch.ones(n, dtype=torch.bool, device="cuda"); rest[moved.long()] = False
    assert torch.equal(after["backwards"][rest], before["backwards"][rest])
    ro.collect()                                            # replay of the captured graph
    obs = env.reset(torch.arange(n, dtype=torch.int32, device="cuda"))
    twin = make_env("walk", n, target_position=2.5, backwards=True, **cfg)
    ot = twin.reset(torch.arange(n, dtype=torch.int32, device="cuda"))
    g = moved.long()
    _assert_rows_equal(obs, ot, g, "reset obs")
    assert (env.task_values()["episode_backwards"][g] == 1).all()
    # the reset counts differ (the batch has lived longer); every other word is the twin's, and so is the next step
    _assert_envs_equal(env, twin, moved.cpu().numpy(), "after reset", skip_i=(LAYOUT.I_RESETCNT,))
    a = torch.rand((n, env.action_dim), device="cuda") * 2 - 1
    om, rm, _, _ = env.step(a)
    om, rm = om.clone(), rm.clone()
    ot, rt, _, _ = twin.step(a)
    _assert_rows_equal(om, ot, g, "obs after a step")
    _assert_rows_equal(rm, rt, g, "reward after a step (flipped by the new direction)")
    env.close(); twin.close(); net.close()


def test_state_dict_round_trip():
    n = 24
    tuples = tuples_for("walk")
    kw = dict(auto_reset=True, max_episode_steps=15, seed=5, **mixed_keywords(tuples, n))
    a_env = make_env("walk", n, **kw)
    a_env.reset()
    gen = torch.Generator(device="cuda"); gen.manual_seed(6)
    acts = [(torch.rand((n, 2), device="cuda", generator=gen) * 2 - 1) * 0.4 for _ in range(20)]
    for a in acts[:10]:
        a_env.step(a)
    a_env.set_task_values([2, 3], target_position=[1.5, 2.5])
    sd = a_env.state_dict()
    ref = []
    for a in acts[10:]:
        o, r, d, _ = a_env.step(a)
        ref.append((o.clone(), r.clone(), d.clone()))
    b_env = make_env("walk", n, **kw)
    b_env.load_state_dict(sd)
    everyone = torch.arange(n, device="cuda")
    for (o, r, d), a in zip(ref, acts[10:]):
        ob, rb, db, _ = b_env.step(a)
        for x, y, what in ((o, ob, "obs"), (r, rb, "reward"), (d, db, "done")):
            _assert_rows_equal(x, y, everyone, what)
    _assert_envs_equal(a_env, b_env, np.arange(n), "after resume")
    other = dict(kw, motor_kp=[1.0] * n, motor_kd=[0.02] * n)
    with pytest.raises(ValueError):
        make_env("walk", n, **other).load_state_dict(sd)
    with pytest.raises(ValueError):
        make_env("walk", n, auto_reset=True, max_episode_steps=15, seed=5).load_state_dict(sd)
    a_env.close(); b_env.close()


def test_two_env_offset_shards_reproduce_the_single_batch():
    from rex_gym_b200.sharding import make_sharded_env
    n = 24
    kw = dict(task="walk", auto_reset=True, max_episode_steps=15, seed=5, **mixed_keywords(tuples_for("walk"), n))
    import rex_gym_b200 as R
    whole = R.BatchedRexEnv(num_envs=n, **kw)
    shards = [make_sharded_env(n, r, 2, **kw) for r in range(2)]
    everyone = torch.arange(n, device="cuda")
    o = whole.reset()
    os_ = np.concatenate([s.reset() for s in shards])
    np.testing.assert_array_equal(o.view(np.int32), os_.view(np.int32))
    gen = torch.Generator(device="cuda"); gen.manual_seed(9)
    for k in range(30):
        a = (torch.rand((n, 2), device="cuda", generator=gen) * 2 - 1) * 0.4
        ow, rw, dw, _ = whole.step(a)
        parts = [s.step(a[r * 12:(r + 1) * 12].contiguous()) for r, s in enumerate(shards)]
        for x, i, what in ((ow, 0, "obs"), (rw, 1, "reward"), (dw, 2, "done")):
            _assert_rows_equal(x, torch.cat([p[i] for p in parts]), everyone, "%s, step %d" % (what, k))
    whole.close()
    for s in shards:
        s.close()

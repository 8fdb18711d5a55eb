"""Per-env sensor latencies on the GPU: a batch whose envs were given different control_latency and pd_latency runs each env
exactly as a batch built with that env's latencies as scalars would (the reference's BatchEnv over envs that differ only in
latency), in every sensor step-kernel instance; the reset hold at each (kp, kd, pd_latency) setting against the fp64 oracle;
composition with the frame wrappers, final observations, episode statistics, the warp re-grouping and a captured Rollout;
checkpoints and sharding."""
import numpy as np
import pytest
import torch

from twin import BUILDS, HOLD_THRESHOLDS, INSTANCES, LAYOUT, NOISE, TOL_P, TOL_Q, bound, force_build, instance_config, \
    launched, make_env, make_oracle, row_id

pytestmark = pytest.mark.gpu

CTL = (0.0, 0.0105, 0.02)           # none, a blend of rows 10 and 11, exactly row 20
PD = (0.0, 0.0005, 0.001)           # none, half a sub-step, one sub-step
GAINS = [(1.0, 0.02), (1.3, 0.03), (0.8, 0.015)]
SENSOR_ROWS = [r for r in INSTANCES if r[4] == "sensor"]


def value_table(task):
    """A few constructor-keyword tuples per task, mixed in with the latencies."""
    if task == "walk":
        return [dict(target_position=t, backwards=b) for t in (None, 2.0) for b in (None, True)]
    if task == "gallop":
        return [dict(target_position=t) for t in (None, 1.5)]
    if task == "turn":
        return [dict(init_orient=i, target_orient=4.0) for i in (None, 1.0)]
    if task == "poses":
        return [dict(base_z=-0.02), dict(base_roll=0.3), dict()]
    return [dict()]


def latency_tuples(task, gains=True):
    """The 9 (control_latency, pd_latency) tuples, each with a task-value tuple and (gains=True) a gain pair."""
    vals = value_table(task)
    out = []
    for j, (c, p) in enumerate((c, p) for c in CTL for p in PD):
        t = dict(vals[j % len(vals)], control_latency=c, pd_latency=p)
        if gains:
            g = GAINS[(j // 3 + j) % 3]                      # every gain pair at every pd latency: 9 hold settings
            t.update(motor_kp=g[0], motor_kd=g[1])
        out.append(t)
    return out


def mixed_keywords(tuples, n):
    """Env i takes tuple i % len(tuples): one list per keyword that any tuple names."""
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


def _assert_envs_equal(mixed, twin, envs, what):
    """Every raw state word (float and int, by name from the kernel's header) of `envs`, bit for bit."""
    sel = torch.as_tensor(envs, device="cuda")
    f1, f2 = mixed._state_f[:, sel], twin._state_f[:, sel]
    i1, i2 = mixed._state_i[:, sel], twin._state_i[:, sel]
    for w in range(LAYOUT.NF):
        assert torch.equal(_bits(f1[w]), _bits(f2[w])), "%s: float word %d of envs %s" % (what, w, envs)
    for w in range(LAYOUT.NI):
        assert torch.equal(i1[w], i2[w]), "%s: int word %d of envs %s" % (what, w, envs)


def run_against_twins(task, n, cfg, tuples, steps=36, reset_at=17, extra=None, rebalance_at=None):
    """A batch of n envs cycling through `tuples` and one scalar twin per tuple, stepped on the same actions with auto-reset
    and one explicit reset of some envs mid-run: every env's outputs and state words equal its twin's, bit for bit."""
    mixed = make_env(task, n, auto_reset=True, **cfg, **mixed_keywords(tuples, n))
    twins = [make_env(task, n, auto_reset=True, **cfg, **t) for t in tuples]
    groups = [np.arange(j, n, len(tuples)) for j in range(len(tuples))]
    idx = [torch.as_tensor(g, device="cuda") for g in groups]
    everyone = torch.arange(n, dtype=torch.int32, device="cuda")
    o = mixed.reset(everyone)
    for t, g in zip(twins, idx):
        _assert_rows_equal(o, t.reset(everyone), g, "reset obs")
    gen = torch.Generator(device="cuda"); gen.manual_seed(3)
    b = bound(task, cfg.get("signal_type", "ik"))
    mid = torch.tensor([1, n // 2, n - 2], dtype=torch.int32, device="cuda")
    for k in range(steps):
        if k == rebalance_at:
            mixed._call(mixed._L.rexsim_rebalance, mixed._h)       # slots permuted: per-env terms are read by env
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


@pytest.mark.parametrize("row", SENSOR_ROWS, ids=row_id)
def test_mixed_latencies_match_scalar_twins_in_every_sensor_instance(row, monkeypatch):
    task, sig, arm, terrain, build = row
    force_build(monkeypatch, build)
    cfg = instance_config(row)
    cfg.pop("control_latency")                               # the tuples' latencies replace the row's scalar one
    ranges = "motor_kp_range" in cfg                         # per-env gains and drawn gains exclude each other
    tuples = latency_tuples(task, gains=not ranges)
    mixed, twins = run_against_twins(task, 2 * len(tuples), cfg, tuples)
    assert launched(mixed) == BUILDS[build]
    assert launched(twins[0]) != BUILDS["sensor"]            # the zero-latency twin runs the build without the sensor model
    assert mixed._ring.numel() == 22 * (61 if arm else 43) * mixed.num_envs     # the deepest env's rows: n = 20, + 2
    if not ranges:
        assert mixed._values["gains"].shape[0] == 9        # (kp, kd, pd_latency) settings: 3 gain pairs x 3 pd latencies
    for e in [mixed] + twins:
        e.close()


@pytest.mark.parametrize("task,kw", [
    ("walk", dict(control_latency=0.0125, pd_latency=0.001, motor_kp=1.2, motor_kd=0.025)),
    ("turn", dict(control_latency=0.0105, init_orient=1.0, target_orient=4.0, terrain_type="random", num_fields=4,
                  observation_noise_stdev=NOISE)),
    ("walk", dict(control_latency=0.0, pd_latency=0.0, observation_noise_stdev=NOISE)),
])
def test_all_equal_arrays_equal_the_scalar_construction(task, kw):
    n = 16
    per_env = ("control_latency", "pd_latency", "motor_kp", "motor_kd")
    arrays = {k: ([v] * n if k in per_env else v) for k, v in kw.items()}
    mixed = make_env(task, n, auto_reset=True, seed=21, max_episode_steps=12, **arrays)
    twin = make_env(task, n, auto_reset=True, seed=21, max_episode_steps=12, **kw)
    assert mixed._latency is not None and twin._latency is None
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
    assert launched(mixed) == launched(twin)
    assert torch.equal(mixed._ring, twin._ring)             # same depth, same rows
    mixed.close(); twin.close()


@pytest.mark.parametrize("terrain", ["plane", "random"])
def test_reset_hold_at_each_setting_matches_the_oracle(terrain):
    """Rex.Reset clears the history and holds through ApplyAction (rex.py:303-323), which reads the PD observation
    pd_latency ago: every (kp, kd, pd_latency) setting's settled state, and the first observation (read control_latency ago),
    against the fp64 oracle built with those values, within the reset-hold tolerances of the gain test.  The CUDA result is
    held to the range the oracle's fp64 and fp32 builds over HOLD_THRESHOLDS span, widened by those tolerances.  On the
    heightfield the default gains at 1 ms are left out: there the oracles themselves end up to 0.063 rad apart, and the
    CUDA hold landed 1.5e-3 rad beyond that band widened by 5e-3 (H100, seed 77); 0.5 ms and the other pairs at 1 ms stay."""
    pd1 = 0.001 if terrain == "plane" else 0.0005
    settings = [(1.0, 0.02, 0.0), (1.0, 0.02, pd1), (1.3, 0.03, 0.0005), (0.8, 0.015, 0.001)]
    ctl = (0.0, 0.0105, 0.02)
    n = 24
    kw = dict(signal_type="ik", seed=77, target_position=2.0, backwards=False)
    if terrain == "random":
        kw.update(terrain_type="random", num_fields=4)
    which = np.arange(n) % len(settings)
    lat = np.array([ctl[i % 3] for i in range(n)])
    env = make_env("walk", n, motor_kp=[settings[s][0] for s in which], motor_kd=[settings[s][1] for s in which],
                   pd_latency=[settings[s][2] for s in which], control_latency=lat, **kw)
    assert env._values["gains"].shape[0] == len(settings)
    og = env.reset()
    sg = env.get_state()
    tq, tp = (TOL_Q, TOL_P) if terrain == "plane" else (5e-3, 5e-3)

    def inside(x, band, tol, what):
        lo, hi = band.min(0) - tol, band.max(0) + tol
        assert ((x >= lo) & (x <= hi)).all(), "%s: %.3g outside the oracles' band" % (what, np.maximum(lo - x, x - hi).max())
    settled = []
    for s, (kp, kd, pd) in enumerate(settings):
        for c in ctl:
            e = (which == s) & (lat == c)
            oras = [make_oracle("walk", n, motor_kp=kp, motor_kd=kd, pd_latency=pd, control_latency=c, residual_threshold=t,
                                f32=f, **kw) for t in HOLD_THRESHOLDS for f in (False, True)]
            oc = np.array([o.reset() for o in oras])[:, e]
            so = [o.states() for o in oras]
            what = "setting %d, control latency %g" % (s, c)
            for k, tol in (("q", tq), ("pos", tp), ("quat", tq)):
                inside(sg[k][e], np.array([x[k][e] for x in so]), tol, "%s, %s" % (k, what))
            inside(og[e][:, :2], oc[:, :, :2], 10 * tq, "first observation, " + what)
        settled.append(sg["q"][which == s][0])
    # the PD latency does change the settled pose: (1.0, 0.02) at 0 and at 1 ms (0.5 ms on the heightfield)
    assert np.abs(settled[1] - settled[0]).max() > 1e-6
    assert env.check_errors() == 0
    env.close()


def test_composes_with_frame_history_final_observation_episode_statistics_and_rebalance():
    cfg = dict(signal_type="ik", seed=13, max_episode_steps=15, episode_statistics=True, final_observation=True,
               frame_history=[0, 1, 3], frame_delta=True)

    def extra(mixed, twin, g, k):
        # the final observation is delayed by the ending env's own control latency
        _assert_rows_equal(mixed.final_observation(), twin.final_observation(), g, "final obs, step %d" % k)
        _assert_rows_equal(mixed.limit_bytes(), twin.limit_bytes(), g, "limit byte, step %d" % k)
        for name in ("score", "length"):
            _assert_rows_equal(mixed._episode[name], twin._episode[name], g, "%s, step %d" % (name, k))
        _assert_rows_equal(mixed.objectives(), twin.objectives(), g, "objectives, step %d" % k)
        for key in mixed._frames:
            n = mixed.num_envs
            _assert_rows_equal(mixed._frames[key].view(-1, n).t(), twin._frames[key].view(-1, n).t(), g, key)
    mixed, twins = run_against_twins("walk", 27, cfg, latency_tuples("walk"), extra=extra, rebalance_at=5)
    for e in [mixed] + twins:
        e.close()


def test_captured_rollout_matches_scalar_twins():
    from rex_gym_b200.agents import ForwardGaussianPolicy, Rollout
    tuples = [dict(control_latency=c, pd_latency=p) for c, p in ((0.0, 0.0), (0.0105, 0.0005), (0.02, 0.001), (0.0, 0.001))]
    n = 16
    cfg = dict(normalize=True, auto_reset=True, max_episode_steps=20, seed=8, target_position=2.0, backwards=False)
    mixed = make_env("walk", n, **cfg, **mixed_keywords(tuples, n))
    twins = [make_env("walk", n, **cfg, **t) for t in tuples]
    net = ForwardGaussianPolicy(mixed.obs_dim, mixed.action_dim, seed=1)
    runs = []
    for e in [mixed] + twins:
        ro = Rollout(e, net, 8, seed=2, training=False)
        ro.collect()
        b = ro.collect()                                     # a replay of the captured graph
        runs.append({k: b[k].clone() for k in ("observ", "reward", "done")})
    for j, r in enumerate(runs[1:]):
        g = torch.arange(j, n, len(tuples), device="cuda")
        for k in ("observ", "reward", "done"):
            _assert_rows_equal(runs[0][k].transpose(0, 1), r[k].transpose(0, 1), g, "%s, tuple %d" % (k, j))
    for e in [mixed] + twins:
        e.close()
    net.close()


def test_state_dict_round_trip():
    n = 18
    tuples = latency_tuples("walk")
    kw = dict(auto_reset=True, max_episode_steps=15, seed=5, **mixed_keywords(tuples, n))
    a_env = make_env("walk", n, **kw)
    a_env.reset()
    gen = torch.Generator(device="cuda"); gen.manual_seed(6)
    acts = [(torch.rand((n, 2), device="cuda", generator=gen) * 2 - 1) * 0.4 for _ in range(20)]
    for a in acts[:10]:
        a_env.step(a)
    sd = a_env.state_dict()
    assert sd["env_latency"].dtype == torch.float64 and sd["env_latency"].shape == (2, n)
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
    assert torch.equal(a_env._ring, b_env._ring)
    other = dict(kw, control_latency=list(reversed(kw["control_latency"])))
    with pytest.raises(ValueError, match="latencies"):
        make_env("walk", n, **other).load_state_dict(sd)
    scalar = {k: v for k, v in kw.items() if k not in ("control_latency", "pd_latency")}
    with pytest.raises(ValueError, match="latencies"):
        make_env("walk", n, control_latency=0.02, **scalar).load_state_dict(sd)
    a_env.close(); b_env.close()


def test_two_env_offset_shards_reproduce_the_single_batch():
    from rex_gym_b200.sharding import make_sharded_env
    import rex_gym_b200 as R
    n = 24
    # the shards' deepest rows differ (the first has no 20 ms env): the ring depth does not change what an env reads
    ctl = [0.0, 0.0105, 0.0, 0.0105] * 3 + [0.02, 0.0, 0.0105, 0.0] * 3
    kw = dict(task="walk", auto_reset=True, max_episode_steps=15, seed=5, control_latency=ctl,
              pd_latency=[0.0, 0.0005, 0.001] * 8, motor_kp=[1.0, 1.3] * 12)
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


def test_the_entry_point_is_refused_twice_and_after_the_first_step():
    n = 8
    env = make_env("walk", n, control_latency=[0.0, 0.01] * 4)
    lat = np.zeros(n)
    assert env._L.rexsim_set_env_latencies(env._h, lat.ctypes.data, None) == -1          # a second call
    env.close()
    env = make_env("walk", n)
    env.reset()
    assert env._L.rexsim_set_env_latencies(env._h, lat.ctypes.data, None) == -1          # after the first reset
    env.close()
    env = make_env("walk", n)
    bad = np.array([0.0, -1e-3] * 4)
    assert env._L.rexsim_set_env_latencies(env._h, None, bad.ctypes.data) == -1          # negative
    bad[1] = np.nan
    assert env._L.rexsim_set_env_latencies(env._h, bad.ctypes.data, None) == -1          # NaN
    env.close()

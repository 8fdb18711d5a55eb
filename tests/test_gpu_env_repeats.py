"""Per-env control rates on the GPU: a batch whose envs share the simulation time step but differ in control_time_step and
action_repeat (and so in the PGS cap int(300 / action_repeat)) runs each env exactly as the batch built with that env's rate as
the scalars would (the reference's BatchEnv over envs that differ only in those keywords), in every step-kernel build, each
(terrain, rate) group stepped as its own slot range; all-equal arrays against the scalar construction; the reset hold of every
(setting, iteration count, terrain, field); the rebalance partition at 16 groups; composition with the sensor model, the frame
wrappers, final observations, episode statistics, per-env task values, a captured Rollout and the renderer; checkpoints,
shards and the ABI's refusals."""
import ctypes

import numpy as np
import pytest
import torch

from mixed_twin import assert_envs_equal, assert_rows_equal, label_groups, run_twins
from twin import BUILDS, INSTANCES, LAYOUT, NOISE, force_build, instance_config, launched, make_env, solver_cost

pytestmark = pytest.mark.gpu

RATES = [(0.005, 5), (0.006, 6), (0.010, 10)]          # 1 ms sub-steps: 60, 50 and 30 PGS iterations
TERRAIN_IDS = {"plane": 0, "random": 1}
# (task, signal, arm, build) of every step_kernel instance; the terrain alternates from row to row
ROWS = list(dict.fromkeys((t, s, arm, b) for t, s, arm, _, b in INSTANCES))


def rid(row):
    task, sig, arm, build = row
    return "-".join([task, sig] + (["arm"] if arm else []) + [build])


def rate_kw(rates):
    """The keywords of one rate per env."""
    return dict(control_time_step=[c for c, _ in rates], action_repeat=[r for _, r in rates])


def uneven(n, choices):
    """Entry (i + i // k) % k of the k choices for env i: every choice on about n / k envs (n >= k), interleaved, the order
    shifting every k envs."""
    k = len(choices)
    return [choices[(i + i // k) % k] for i in range(n)]


def groups_of(env):
    """[(terrain, action_repeat, solver_iterations, first, count, (CTA size, CTAs per SM, sensor))] (rexsim_launch_group)."""
    out = []
    for g in range(env._L.rexsim_launch_groups(env._h)):
        info = np.zeros(8, np.int32)
        assert env._L.rexsim_launch_group(env._h, g, info.ctypes.data) == 0
        out.append(tuple(int(x) for x in info[:5]) + (tuple(int(x) for x in info[5:]),))
    return out


def slots(env):
    """-> (perm [N] slot -> env, or None: the identity; group byte [N] of each env, or None: one group)."""
    p, q = ctypes.c_void_p(), ctypes.c_void_p()
    assert env._L.rexsim_slot_buffers(env._h, ctypes.byref(p), ctypes.byref(q)) == 0
    from rex_gym_b200 import _capi
    n = env.num_envs
    perm = torch.as_tensor(_capi.DevArray(p.value, (n,), "<i4", env), device="cuda").cpu().numpy() if p.value else None
    grp = torch.as_tensor(_capi.DevArray(q.value, (n,), "|u1", env), device="cuda").cpu().numpy() if q.value else None
    return perm, grp


def close(*envs):
    for e in envs:
        for x in (e.values() if isinstance(e, dict) else [e]):
            x.close()


@pytest.mark.parametrize("row", ROWS, ids=rid)
def test_mixed_rates_match_the_scalar_twins_in_every_build(row, monkeypatch):
    task, sig, arm, build = row
    force_build(monkeypatch, build)
    terrain = ("plane", "random")[ROWS.index(row) % 2]
    cfg = instance_config((task, sig, arm, terrain, build))
    n = 27
    rates = uneven(n, RATES)
    twin_kw = {r: dict(cfg, control_time_step=r[0], action_repeat=r[1]) for r in RATES}
    mixed, twins, groups = run_twins(task, n, dict(cfg, **rate_kw(rates)), twin_kw, rates)
    assert mixed.control_time_step == tuple(c for c, _ in rates) and mixed._action_repeat == tuple(r for _, r in rates)
    gs = groups_of(mixed)
    assert [g[1:3] for g in gs] == [(r, 300 // r) for _, r in dict.fromkeys(rates)]      # in order of first appearance
    for t, r, it, first, count, b in gs:
        assert t == TERRAIN_IDS[terrain] and count == len(groups[next(x for x in RATES if x[1] == r)])
        assert b == BUILDS[build] == launched(twins[next(x for x in RATES if x[1] == r)]), (r, b)
    assert launched(mixed) == gs[-1][5]
    close(mixed, twins)


@pytest.mark.parametrize("task,rates", [("walk", RATES), ("turn", [(0.005, 5), (0.010, 10), (0.001, 1)])],
                         ids=["walk-ik", "turn-ik"])
def test_terrains_and_rates_match_their_six_twins(task, rates):
    n = 40
    labels = uneven(n, [(t, r) for t in TERRAIN_IDS for r in rates])
    cfg = dict(signal_type="ik", seed=13, max_episode_steps=15, num_fields=4)
    mixed_kw = dict(cfg, terrain_type=[t for t, _ in labels], **rate_kw([r for _, r in labels]))
    twin_kw = {(t, r): dict(cfg, terrain_type=t, control_time_step=r[0], action_repeat=r[1]) for t in TERRAIN_IDS for r in rates}
    mixed, twins, groups = run_twins(task, n, mixed_kw, twin_kw, labels)
    gs = groups_of(mixed)
    assert len(gs) == 6 and [g[0] for g in gs] == [0, 0, 0, 1, 1, 1]        # terrain-major, plane first
    assert sum(g[4] for g in gs) == n and [g[3] for g in gs] == [sum(h[4] for h in gs[:i]) for i in range(6)]
    for t, r, it, first, count, b in gs:
        label = next(l for l in groups if TERRAIN_IDS[l[0]] == t and l[1][1] == r)
        assert count == len(groups[label]) and it == int(300 / r) and b == launched(twins[label])
    close(mixed, twins)


def test_all_equal_arrays_build_the_scalar_construction():
    n, task = 16, "gallop"
    kw = dict(auto_reset=True, seed=21, max_episode_steps=12)
    mixed = make_env(task, n, control_time_step=np.full(n, 0.004), action_repeat=[4] * n, **kw)
    twin = make_env(task, n, control_time_step=0.004, action_repeat=4, **kw)
    assert mixed._repeats is None and mixed.control_time_step == 0.004 and mixed._action_repeat == 4
    p = ctypes.c_void_p()
    assert mixed._L.rexsim_env_repeat_buffers(mixed._h, ctypes.byref(p)) == -1           # the feature is off
    assert groups_of(mixed) == groups_of(twin) == [(0, 4, 75, 0, n, (0, 0, 0))]
    assert mixed.launch_count == twin.launch_count
    everyone = torch.arange(n, device="cuda")
    assert_rows_equal(mixed.reset(everyone), twin.reset(everyone), everyone, "reset obs")
    gen = torch.Generator(device="cuda"); gen.manual_seed(4)
    for k in range(30):
        a = torch.rand((n, mixed.action_dim), device="cuda", generator=gen) * 0.4
        om, rm, dm, _ = mixed.step(a)
        om, rm, dm = om.clone(), rm.clone(), dm.clone()
        ot, rt, dt, _ = twin.step(a)
        for x, y, what in ((om, ot, "obs"), (rm, rt, "reward"), (dm, dt, "done")):
            assert_rows_equal(x, y, everyone, "%s, step %d" % (what, k))
        assert_envs_equal(mixed, twin, np.arange(n), "step %d" % k)
    assert mixed.launch_count == twin.launch_count
    assert slots(mixed) == (None, None)
    close(mixed, twin)


def test_reset_hold_of_every_setting_count_terrain_and_field_equals_the_twins():
    """Per-env gains, pd_latency, terrains and rates: after each of four resets every env has been reset from the (setting,
    terrain, field) snapshot its twin resets from, settled at its own iteration count, bit for bit."""
    n = 48
    gains = [(1.0, 0.02), (1.3, 0.03), (0.8, 0.015)]
    i = np.arange(n)
    rates = [RATES[0] if (e // 6) % 2 else RATES[2] for e in i]                        # 60 and 30 iterations
    terrain = ["plane" if (e // 12) % 2 else "random" for e in i]
    kw = dict(signal_type="ik", seed=77, num_fields=4, target_position=2.0, backwards=False,
              motor_kp=[gains[e % 3][0] for e in i], motor_kd=[gains[e % 3][1] for e in i],
              pd_latency=[(0.0, 0.0005)[(e // 3) % 2] for e in i], control_latency=0.0105)
    labels = list(zip(terrain, rates))
    mixed = make_env("walk", n, terrain_type=terrain, **rate_kw(rates), **kw)
    twins = {l: make_env("walk", n, terrain_type=l[0], control_time_step=l[1][0], action_repeat=l[1][1], **kw)
             for l in dict.fromkeys(labels)}
    assert mixed._values["gains"].shape[0] == 12                        # 3 gain pairs x 2 pd latencies x 2 iteration counts
    pair = mixed._values["pair"].cpu().numpy()
    assert (pair[[e for e in i if rates[e] == RATES[2]]] < 6).all()      # each count's settings contiguous, first seen first
    groups = label_groups(labels)
    seen = set()
    for r in range(4):
        o = torch.as_tensor(mixed.reset())
        for l, tw in twins.items():
            assert_rows_equal(o, torch.as_tensor(tw.reset()), groups[l], "reset %d obs, %s" % (r, l))
            assert_envs_equal(mixed, tw, groups[l], "reset %d, %s" % (r, l))
        field = mixed._state_i[LAYOUT.I_FIELD].cpu().numpy()
        seen |= {(int(pair[e]), terrain[e], int(field[e])) for e in range(n)}
    assert seen == {(s, "plane", 0) for s in range(12)} | {(s, "random", f) for s in range(12) for f in range(4)}
    assert mixed.check_errors() == 0
    close(mixed, twins)


def test_rebalance_keeps_sixteen_groups_in_their_ranges():
    """2 terrains x 8 rates (r ms, r sub-steps for r = 1..8): 4096 rebalance bins, the wide scan.  After rexsim_rebalance every
    group's slot range holds exactly its envs, most expensive first, and the step goes on matching the group's twin."""
    n = 200
    rates = [(r / 1000, r) for r in range(1, 9)]
    labels = uneven(n, [(t, r) for t in TERRAIN_IDS for r in rates])
    mixed = make_env("walk", n, terrain_type=[t for t, _ in labels], **rate_kw([r for _, r in labels]), num_fields=4,
                     auto_reset=True, max_episode_steps=10, seed=3)
    mixed.reset()
    gen = torch.Generator(device="cuda"); gen.manual_seed(2)
    for k in range(12):
        mixed.step(torch.rand((n, 2), device="cuda", generator=gen) * 0.8 - 0.4)
        if k in (3, 11):
            mixed._call(mixed._L.rexsim_rebalance, mixed._h)
            torch.cuda.synchronize()
            perm, grp = slots(mixed)
            cost = solver_cost(mixed)
            gs = groups_of(mixed)
            assert len(gs) == 16
            for g, (t, r, it, first, count, _) in enumerate(gs):
                envs = [e for e, (lt, lr) in enumerate(labels) if TERRAIN_IDS[lt] == t and lr[1] == r]
                assert sorted(perm[first:first + count].tolist()) == envs, g
                assert (grp[envs] == g).all()
                bins = 255 - np.minimum(cost[perm[first:first + count]] >> 1, 255)
                assert (np.diff(bins) >= 0).all(), g
    assert mixed.check_errors() == 0
    mixed.close()


def test_composes_with_sensor_noise_frames_final_observation_statistics_and_task_values():
    n = 25
    cfg = dict(signal_type="ik", seed=13, max_episode_steps=15, episode_statistics=True, final_observation=True,
               frame_history=[0, 1, 3], frame_delta=True, observation_noise_stdev=NOISE, control_latency=0.0105,
               target_position=[(1.5, 2.0, None)[e % 3] for e in range(n)], backwards=[(None, True)[e % 2] for e in range(n)])
    rates = uneven(n, RATES)

    def extra(mixed, twin, g, k):
        assert_rows_equal(mixed.final_observation(), twin.final_observation(), g, "final obs, step %d" % k)
        assert_rows_equal(mixed.limit_bytes(), twin.limit_bytes(), g, "limit byte, step %d" % k)
        for name in ("score", "length"):
            assert_rows_equal(mixed._episode[name], twin._episode[name], g, "%s, step %d" % (name, k))
        assert_rows_equal(mixed.objectives(), twin.objectives(), g, "objectives, step %d" % k)
        for key in mixed._frames:
            assert_rows_equal(mixed._frames[key].view(-1, n).t(), twin._frames[key].view(-1, n).t(), g, key)
        assert_rows_equal(mixed._values["values"].t(), twin._values["values"].t(), g, "task values")

    twin_kw = {r: dict(cfg, control_time_step=r[0], action_repeat=r[1]) for r in RATES}
    mixed, twins, groups = run_twins("walk", n, dict(cfg, **rate_kw(rates)), twin_kw, rates, extra=extra)
    assert mixed.episode_summary(clear=False)["count"] > 0
    close(mixed, twins)


def test_captured_rollout_launches_every_group_and_matches_the_twins():
    from rex_gym_b200.agents import ForwardGaussianPolicy, Rollout
    n = 21
    rates = uneven(n, RATES)
    cfg = dict(normalize=True, auto_reset=True, max_episode_steps=20, seed=8, target_position=2.0, backwards=False)
    mixed = make_env("walk", n, **rate_kw(rates), **cfg)
    twins = {r: make_env("walk", n, control_time_step=r[0], action_repeat=r[1], **cfg) for r in RATES}
    net = ForwardGaussianPolicy(mixed.obs_dim, mixed.action_dim, seed=1)
    runs, launches = {}, {}
    for name, e in [("mixed", mixed)] + list(twins.items()):
        ro = Rollout(e, net, 8, seed=2, training=False)
        before = e.launch_count
        ro.collect()
        launches[name] = e.launch_count - before
        b = ro.collect()                                     # a replay of the captured graph
        runs[name] = {k: b[k].clone() for k in ("observ", "reward", "done")}
    # warm-up and capture: every control step is three step launches in the mixed batch, one in each twin
    assert all(launches["mixed"] == 3 * launches[r] for r in RATES) and launches["mixed"] == 3 * 2 * 8
    for r, g in label_groups(rates).items():
        for k in ("observ", "reward", "done"):
            assert_rows_equal(runs["mixed"][k].transpose(0, 1), runs[r][k].transpose(0, 1), g, "%s, %s" % (k, r))
    close(mixed, twins)
    net.close()


def test_render_batch_draws_each_env_as_its_twin():
    n = 12
    rates = uneven(n, RATES)
    cfg = dict(signal_type="ik", seed=2, target_position=2.0, backwards=False)
    mixed = make_env("turn", n, **rate_kw(rates), **cfg)
    twins = {r: make_env("turn", n, control_time_step=r[0], action_repeat=r[1], **cfg) for r in RATES}
    gen = torch.Generator(device="cuda"); gen.manual_seed(1)
    for e in [mixed] + list(twins.values()):
        e.reset()
    for k in range(20):
        a = (torch.rand((n, mixed.action_dim), device="cuda", generator=gen) * 2 - 1) * 0.01
        for e in [mixed] + list(twins.values()):
            e.step(a)
    frames = mixed.render_batch(list(range(n)), width=96, height=72, pitch=-45.0)
    for r, g in label_groups(rates).items():
        assert_envs_equal(mixed, twins[r], g, "before render, %s" % (r,))
        assert torch.equal(frames[torch.as_tensor(g, device="cuda")], twins[r].render_batch(list(g), width=96, height=72, pitch=-45.0))
    close(mixed, twins)


def test_state_dict_round_trip_and_refusal():
    n = 19
    rates = uneven(n, RATES)
    kw = dict(auto_reset=True, max_episode_steps=15, seed=5)
    a_env = make_env("walk", n, **rate_kw(rates), **kw)
    a_env.reset()
    gen = torch.Generator(device="cuda"); gen.manual_seed(6)
    acts = [(torch.rand((n, 2), device="cuda", generator=gen) * 2 - 1) * 0.4 for _ in range(20)]
    for a in acts[:10]:
        a_env.step(a)
    sd = a_env.state_dict()
    assert sd["env_repeats"].dtype == torch.int32
    assert sd["env_repeats"].cpu().tolist() == [[r for _, r in rates], [300 // r for _, r in rates]]
    ref = []
    for a in acts[10:]:
        o, r, d, _ = a_env.step(a)
        ref.append((o.clone(), r.clone(), d.clone()))
    b_env = make_env("walk", n, **rate_kw(rates), **kw)
    b_env.load_state_dict(sd)
    everyone = torch.arange(n, device="cuda")
    for (o, r, d), a in zip(ref, acts[10:]):
        ob, rb, db, _ = b_env.step(a)
        for x, y, what in ((o, ob, "obs"), (r, rb, "reward"), (d, db, "done")):
            assert_rows_equal(x, y, everyone, what)
    assert_envs_equal(a_env, b_env, np.arange(n), "after resume")
    for other in (make_env("walk", n, **rate_kw(list(reversed(rates))), **kw),
                  make_env("walk", n, **rate_kw(rates), solver_iterations=40, **kw),
                  make_env("walk", n, **kw)):
        with pytest.raises(ValueError, match="control rates"):
            other.load_state_dict(sd)
        other.close()
    close(a_env, b_env)


def test_two_env_offset_shards_reproduce_the_single_batch():
    from rex_gym_b200.sharding import make_sharded_env
    import rex_gym_b200 as R
    n = 24
    rates = [RATES[0]] * 3 + [RATES[2]] * 9 + [RATES[1], RATES[0]] * 6
    kw = dict(task="walk", auto_reset=True, max_episode_steps=15, seed=5, **rate_kw(rates))
    whole = R.BatchedRexEnv(num_envs=n, **kw)
    shards = [make_sharded_env(n, r, 2, **kw) for r in range(2)]
    assert [s._action_repeat for s in shards] == [tuple(r for _, r in rates[:12]), tuple(r for _, r in rates[12:])]
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
            assert_rows_equal(x, torch.cat([p[i] for p in parts]), everyone, "%s, step %d" % (what, k))
    close(whole, *shards)


def test_the_entry_point_refusals():
    n = 9
    rep = np.array([5, 10, 6] * 3, np.int32)
    it = np.array([60, 30, 50] * 3, np.int32)
    env = make_env("walk", n, **rate_kw([RATES[e % 3] for e in range(n)]))
    assert env._L.rexsim_set_env_repeats(env._h, rep.ctypes.data, it.ctypes.data) == -1         # a second call
    env.close()
    env = make_env("walk", n)
    env.reset()
    env.step(torch.zeros((n, 2), device="cuda"))
    assert env._L.rexsim_set_env_repeats(env._h, rep.ctypes.data, it.ctypes.data) == -1         # after the first step
    env.close()
    env = make_env("walk", n)
    for bad in (np.array([5, 0, 6] * 3, np.int32), np.array([5, -1, 6] * 3, np.int32)):
        assert env._L.rexsim_set_env_repeats(env._h, bad.ctypes.data, it.ctypes.data) == -1    # an entry <= 0
        assert env._L.rexsim_set_env_repeats(env._h, rep.ctypes.data, bad.ctypes.data) == -1
    many = np.arange(1, 10, dtype=np.int32)                                                      # nine pairs
    assert env._L.rexsim_set_env_repeats(env._h, many.ctypes.data, None) == -1
    assert env._L.rexsim_launch_groups(env._h) == 1
    assert env._L.rexsim_set_env_repeats(env._h, rep.ctypes.data, it.ctypes.data) == 0          # the refusals left it unset
    assert [g[1:5] for g in groups_of(env)] == [(5, 60, 0, 3), (10, 30, 3, 3), (6, 50, 6, 3)]
    info = np.zeros(8, np.int32)
    assert env._L.rexsim_launch_group(env._h, 3, info.ctypes.data) == -1
    env.close()

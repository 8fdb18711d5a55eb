"""Per-env tasks and signals on the GPU: a batch whose envs differ in task and signal_type but share their spaces runs each env
exactly as the batch built with that env's pair as the scalars would (the reference's BatchEnv over such envs), in every
step-kernel build, each (terrain, step unit, rate) group stepped as its own slot range; all-equal arrays against the scalar
construction; the groups and slot ranges through rexsim_rebalance; composition with terrains and rates up to the 16-group
cap, latencies with noise, per-env task values, the frame wrappers, final observations, episode statistics, a captured
Rollout and the renderer; checkpoints, shards and the ABI's refusals."""
import ctypes

import numpy as np
import pytest
import torch

from mixed_twin import assert_envs_equal, assert_rows_equal, label_groups
from twin import BUILDS, NOISE, force_build, launched, make_env

pytestmark = pytest.mark.gpu

TASK_IDS = {"walk": 0, "gallop": 1, "turn": 2, "standup": 3, "poses": 4}
SIGNAL_IDS = {"ik": 0, "ol": 1}
# the mixes whose spaces agree: (pairs, normalize, action bound of the test's actions)
WALK_TURN = ([("walk", "ik"), ("turn", "ik"), ("turn", "ol")], True, 0.5)
TURN = ([("turn", "ik"), ("turn", "ol")], False, 0.01)
STAND_POSES = ([("standup", "ol"), ("poses", "ik"), ("standup", "ik")], False, 0.1)     # at each task's default rate
MIXES = {"walk-turn-normalized": WALK_TURN, "turn-raw": TURN, "standup-poses-raw": STAND_POSES}
CASES = [(m, arm, b) for m in MIXES for arm in (False, True) for b in ("small", "big", "sensor")
         if not (arm and (b == "big" or m == "turn-raw"))]


def uneven(n, choices):
    """Entry (i + i // k) % k of the k choices for env i: every choice on about n / k envs, interleaved."""
    k = len(choices)
    return [choices[(i + i // k) % k] for i in range(n)]


def tasks_of(pairs):
    return [t for t, _ in pairs]


def signals_of(pairs):
    return [s for _, s in pairs]


def unit(task, sig):
    """The step unit of a pair (unit_of in rexsim_kernel.cuh): standup and poses ignore the signal."""
    return task if task in ("standup", "poses") else (task, sig)


def groups_of(env):
    """[(terrain, task, signal, action_repeat, solver_iterations, first, count, build)] (rexsim_launch_group and
    rexsim_launch_group_task)."""
    out = []
    for g in range(env._L.rexsim_launch_groups(env._h)):
        info = np.zeros(8, np.int32)
        assert env._L.rexsim_launch_group(env._h, g, info.ctypes.data) == 0
        t, s = ctypes.c_int32(), ctypes.c_int32()
        assert env._L.rexsim_launch_group_task(env._h, g, ctypes.byref(t), ctypes.byref(s)) == 0
        out.append((int(info[0]), t.value, s.value) + tuple(int(x) for x in info[1:5]) + (tuple(int(x) for x in info[5:]),))
    return out


def slots(env):
    """-> (perm [N] slot -> env, or None: the identity; group byte [N] of each env, or None: one group)."""
    from rex_gym_b200 import _capi
    p, q = ctypes.c_void_p(), ctypes.c_void_p()
    assert env._L.rexsim_slot_buffers(env._h, ctypes.byref(p), ctypes.byref(q)) == 0
    n = env.num_envs
    perm = torch.as_tensor(_capi.DevArray(p.value, (n,), "<i4", env), device="cuda").cpu().numpy() if p.value else None
    grp = torch.as_tensor(_capi.DevArray(q.value, (n,), "|u1", env), device="cuda").cpu().numpy() if q.value else None
    return perm, grp


def run_task_twins(n, mixed_kw, twin_kw, labels, action_bound, steps=36, reset_at=17, rebalance_at=9, extra=None):
    """mixed_twin.run_twins with each batch's task in its keywords: a mixed batch of n envs (make_env(mixed_kw['task'], n,
    auto_reset=True, ...)) and one twin per group label (make_env(twin_kw[label]['task'], n, auto_reset=True, ...)), stepped on
    the same actions, uniform in +-action_bound, with auto-reset, one explicit reset whose indices span every group, and a
    re-grouping (rexsim_rebalance) mid-run: every env's outputs and state words equal its group's twin's, bit for bit.
    extra(mixed, twin, envs, step) adds checks after each step.  -> (mixed, {label: twin}, {label: env indices})."""
    def build(kw):
        kw = dict(kw)
        return make_env(kw.pop("task"), n, auto_reset=True, **kw)
    groups = label_groups(labels)
    mixed = build(mixed_kw)
    twins = {g: build(twin_kw[g]) for g in groups}
    everyone = torch.arange(n, dtype=torch.int32, device="cuda")
    o = mixed.reset(everyone)
    for g, tw in twins.items():
        assert_rows_equal(o, tw.reset(everyone), groups[g], "reset obs, %s" % (g,))
        assert_envs_equal(mixed, tw, groups[g], "after reset, %s" % (g,))
    gen = torch.Generator(device="cuda"); gen.manual_seed(3)
    mid = torch.tensor(sorted({int(e[len(e) // 2]) for e in groups.values()} | {n - 1}), dtype=torch.int32, device="cuda")
    for k in range(steps):
        if k == rebalance_at:
            mixed._call(mixed._L.rexsim_rebalance, mixed._h)       # slots re-sorted within each group's range
        a = (torch.rand((n, mixed.action_dim), device="cuda", generator=gen) * 2 - 1) * action_bound
        om, rm, dm, _ = mixed.step(a)
        om, rm, dm = om.clone(), rm.clone(), dm.clone()
        for g, tw in twins.items():
            ot, rt, dt, _ = tw.step(a)
            assert_rows_equal(om, ot, groups[g], "obs, step %d, %s" % (k, g))
            assert_rows_equal(rm, rt, groups[g], "reward, step %d, %s" % (k, g))
            assert_rows_equal(dm, dt, groups[g], "done, step %d, %s" % (k, g))
            assert_envs_equal(mixed, tw, groups[g], "step %d, %s" % (k, g))
            if extra:
                extra(mixed, tw, groups[g], k)
        if k == reset_at:
            r = mixed.reset(mid)
            for g, tw in twins.items():
                sel = np.nonzero(np.isin(mid.cpu().numpy(), groups[g]))[0]
                assert_rows_equal(r, tw.reset(mid), sel, "explicit reset obs, %s" % (g,))
    assert mixed.check_errors() == 0
    return mixed, twins, groups


def close(*envs):
    for e in envs:
        for x in (e.values() if isinstance(e, dict) else [e]):
            x.close()


@pytest.mark.parametrize("mix,arm,build", CASES, ids=["-".join([m] + (["arm"] if a else []) + [b]) for m, a, b in CASES])
def test_mixed_tasks_match_the_scalar_twins_in_every_build(mix, arm, build, monkeypatch):
    pairs, normalize, b = MIXES[mix]
    force_build(monkeypatch, build)
    terrain = ("plane", "random")[CASES.index((mix, arm, build)) % 2]
    cfg = dict(seed=13, max_episode_steps=15, normalize=normalize, terrain_type=terrain, num_fields=4)
    if arm:
        cfg["mark"] = "arm"
    if build == "sensor":
        cfg["control_latency"] = 0.0125
    n = 27
    labels = uneven(n, pairs)
    twin_kw = {p: dict(cfg, task=p[0], signal_type=p[1]) for p in pairs}
    mixed_kw = dict(cfg, task=tasks_of(labels), signal_type=signals_of(labels))
    mixed, twins, groups = run_task_twins(n, mixed_kw, twin_kw, labels, action_bound=b)
    assert mixed.task == tuple(t for t, _ in labels) and mixed.signal_type == tuple(s for _, s in labels)
    assert mixed._tasks.cpu().tolist() == [[TASK_IDS[t] for t, _ in labels], [SIGNAL_IDS[s] for _, s in labels]]
    gs = groups_of(mixed)
    units = list(dict.fromkeys(unit(*p) for p in labels))
    assert [unit(*next(p for p in pairs if (TASK_IDS[p[0]], SIGNAL_IDS[p[1]]) == g[1:3])) for g in gs] == units
    for t, task, sig, r, it, first, count, built in gs:
        mine = [p for p in pairs if unit(*p) == unit(*next(q for q in pairs if (TASK_IDS[q[0]], SIGNAL_IDS[q[1]]) == (task, sig)))]
        assert count == sum(len(groups[p]) for p in mine)
        assert r == twins[mine[0]]._action_repeat and built == launched(twins[mine[0]]), (task, sig, built)
        if build != "sensor":
            assert built == BUILDS["small" if arm else build]
    close(mixed, twins)


def test_all_equal_arrays_build_the_scalar_construction():
    n = 16
    kw = dict(auto_reset=True, seed=21, max_episode_steps=12)
    mixed = make_env(["turn"] * n, n, signal_type=np.array(["ol"] * n), **kw)
    twin = make_env("turn", n, signal_type="ol", **kw)
    assert mixed._tasks is None and mixed.task == "turn" and mixed.signal_type == "ol"
    p = ctypes.c_void_p()
    assert mixed._L.rexsim_env_task_buffers(mixed._h, ctypes.byref(p)) == -1             # the feature is off
    assert groups_of(mixed) == groups_of(twin) == [(0, 2, 1, 5, 60, 0, n, (0, 0, 0))]
    everyone = torch.arange(n, device="cuda")
    assert_rows_equal(mixed.reset(everyone), twin.reset(everyone), everyone, "reset obs")
    gen = torch.Generator(device="cuda"); gen.manual_seed(4)
    for k in range(30):
        a = (torch.rand((n, 2), device="cuda", generator=gen) * 2 - 1) * 0.01
        om, rm, dm, _ = mixed.step(a)
        om, rm, dm = om.clone(), rm.clone(), dm.clone()
        ot, rt, dt, _ = twin.step(a)
        for x, y, what in ((om, ot, "obs"), (rm, rt, "reward"), (dm, dt, "done")):
            assert_rows_equal(x, y, everyone, "%s, step %d" % (what, k))
        assert_envs_equal(mixed, twin, np.arange(n), "step %d" % k)
    assert mixed.launch_count == twin.launch_count
    assert slots(mixed) == (None, None)
    close(mixed, twin)


def test_groups_and_slot_ranges_hold_only_their_envs_through_rebalance():
    n = 96
    pairs = [("turn", "ol"), ("walk", "ik"), ("turn", "ik")]
    labels = uneven(n, pairs)
    mixed = make_env(tasks_of(labels), n, signal_type=signals_of(labels), normalize=True, auto_reset=True, max_episode_steps=10,
                     seed=3)
    gs = groups_of(mixed)
    assert [g[1:3] for g in gs] == [(2, 1), (0, 0), (2, 0)]                     # in order of first appearance
    assert [g[5] for g in gs] == [0, 32, 64] and [g[6] for g in gs] == [32] * 3

    def check(rebalanced):
        perm, grp = slots(mixed)
        for g, (t, task, sig, r, it, first, count, _) in enumerate(gs):
            envs = [e for e, p in enumerate(labels) if (TASK_IDS[p[0]], SIGNAL_IDS[p[1]]) == (task, sig)]
            got = perm[first:first + count].tolist()
            assert (sorted(got) if rebalanced else got) == envs, g
            assert (grp[envs] == g).all()
    check(False)
    mixed.reset()
    gen = torch.Generator(device="cuda"); gen.manual_seed(2)
    for k in range(12):
        mixed.step(torch.rand((n, 2), device="cuda", generator=gen) * 2 - 1)
        if k in (3, 11):
            mixed._call(mixed._L.rexsim_rebalance, mixed._h)
            torch.cuda.synchronize()
            check(True)
    assert mixed.check_errors() == 0
    mixed.close()


def test_terrains_and_rates_up_to_sixteen_groups_match_their_twins():
    """2 terrains x 2 step units (turn ik, turn ol) x 4 rates: the 16 groups of the cap, each against its twin; a fifth rate
    is refused."""
    n = 48
    rates = [(0.005, 5), (0.010, 10), (0.001, 1), (0.003, 3)]
    combos = [(t, s, r) for t in ("plane", "random") for s in ("ik", "ol") for r in rates]
    labels = uneven(n, combos)
    cfg = dict(seed=13, max_episode_steps=15, num_fields=4)
    mixed_kw = dict(cfg, terrain_type=[t for t, _, _ in labels], signal_type=[s for _, s, _ in labels],
                    control_time_step=[r[0] for _, _, r in labels], action_repeat=[r[1] for _, _, r in labels])
    twin_kw = {l: dict(cfg, terrain_type=l[0], signal_type=l[1], control_time_step=l[2][0], action_repeat=l[2][1]) for l in combos}
    mixed, twins, groups = run_task_twins(n, dict(mixed_kw, task="turn"), {l: dict(kw, task="turn") for l, kw in twin_kw.items()},
                                          labels, action_bound=0.01, steps=24)
    gs = groups_of(mixed)
    assert len(gs) == 16 and [g[0] for g in gs] == [0] * 8 + [1] * 8
    for t, task, sig, r, it, first, count, built in gs:
        label = next(l for l in combos if (l[0] == ("plane", "random")[t] and SIGNAL_IDS[l[1]] == sig and l[2][1] == r))
        assert count == len(groups[label]) and built == launched(twins[label])
    close(mixed, twins)
    more = uneven(n, [(t, s, r) for t in ("plane", "random") for s in ("ik", "ol") for r in rates + [(0.002, 2)]])
    with pytest.raises(ValueError, match="more than 16 launch groups"):
        make_env("turn", n, terrain_type=[t for t, _, _ in more], signal_type=[s for _, s, _ in more],
                 control_time_step=[r[0] for _, _, r in more], action_repeat=[r[1] for _, _, r in more], num_fields=4)


def test_composes_with_latencies_noise_values_frames_final_observation_and_statistics():
    n = 27
    pairs = WALK_TURN[0]
    labels = uneven(n, pairs)
    walk = [e for e, p in enumerate(labels) if p[0] == "walk"]
    cfg = dict(seed=13, max_episode_steps=15, normalize=True, episode_statistics=True, final_observation=True,
               frame_history=[0, 1, 3], frame_delta=True, observation_noise_stdev=NOISE,
               control_latency=[(0.0, 0.0105, 0.02)[e % 3] for e in range(n)], pd_latency=[(0.0, 0.0005)[e % 2] for e in range(n)],
               target_position=[(1.5, 2.0, None)[e % 3] for e in range(n)], target_orient=[(0.5, None, 2.5)[e % 3] for e in range(n)],
               backwards=[(None, True)[e % 2] for e in range(n)])

    def extra(mixed, twin, g, k):
        assert_rows_equal(mixed.final_observation(), twin.final_observation(), g, "final obs, step %d" % k)
        assert_rows_equal(mixed.limit_bytes(), twin.limit_bytes(), g, "limit byte, step %d" % k)
        for name in ("score", "length"):
            assert_rows_equal(mixed._episode[name], twin._episode[name], g, "%s, step %d" % (name, k))
        if twin.task == "walk":
            assert_rows_equal(mixed.objectives(), twin.objectives(), g, "objectives, step %d" % k)
        else:
            assert twin._episode["objectives"] is None
            assert torch.isnan(mixed.objectives()[torch.as_tensor(g, device="cuda")]).all()
        for key in mixed._frames:
            assert_rows_equal(mixed._frames[key].view(-1, n).t(), twin._frames[key].view(-1, n).t(), g, key)
        assert_rows_equal(mixed._values["values"].t(), twin._values["values"].t(), g, "task values")

    twin_kw = {p: dict(cfg, task=p[0], signal_type=p[1]) for p in pairs}
    mixed_kw = dict(cfg, task=tasks_of(labels), signal_type=signals_of(labels))
    mixed, twins, groups = run_task_twins(n, mixed_kw, twin_kw, labels, action_bound=0.5, extra=extra)
    assert mixed.episode_summary(clear=False)["count"] > 0
    assert mixed._latency is not None and mixed._ring is not None and len(walk) == 9
    close(mixed, twins)


def test_captured_rollout_launches_every_group_and_matches_the_twins():
    from rex_gym_b200.agents import ForwardGaussianPolicy, Rollout
    n = 21
    pairs = WALK_TURN[0]
    labels = uneven(n, pairs)
    cfg = dict(normalize=True, auto_reset=True, max_episode_steps=20, seed=8, target_position=2.0, backwards=False)
    mixed = make_env(tasks_of(labels), n, signal_type=signals_of(labels), **cfg)
    twins = {p: make_env(p[0], n, signal_type=p[1], **cfg) for p in pairs}
    net = ForwardGaussianPolicy(mixed.obs_dim, mixed.action_dim, seed=1)
    runs, launches = {}, {}
    for name, e in [("mixed", mixed)] + list(twins.items()):
        ro = Rollout(e, net, 8, seed=2, training=False)
        before = e.launch_count
        ro.collect()
        launches[name] = e.launch_count - before
        b = ro.collect()                                     # a replay of the captured graph
        runs[name] = {k: b[k].clone() for k in ("observ", "reward", "done")}
    assert all(launches["mixed"] == 3 * launches[p] for p in pairs) and launches["mixed"] == 3 * 2 * 8
    for p, g in label_groups(labels).items():
        for k in ("observ", "reward", "done"):
            assert_rows_equal(runs["mixed"][k].transpose(0, 1), runs[p][k].transpose(0, 1), g, "%s, %s" % (k, p))
    close(mixed, twins)
    net.close()


def test_render_batch_draws_each_env_as_its_twin():
    n = 12
    pairs = STAND_POSES[0]
    labels = uneven(n, pairs)
    cfg = dict(seed=2)
    mixed = make_env(tasks_of(labels), n, signal_type=signals_of(labels), **cfg)
    twins = {p: make_env(p[0], n, signal_type=p[1], **cfg) for p in pairs}
    gen = torch.Generator(device="cuda"); gen.manual_seed(1)
    for e in [mixed] + list(twins.values()):
        e.reset()
    for k in range(20):
        a = (torch.rand((n, 1), device="cuda", generator=gen) * 2 - 1) * 0.1
        for e in [mixed] + list(twins.values()):
            e.step(a)
    frames = mixed.render_batch(list(range(n)), width=96, height=72, pitch=-45.0)
    for p, g in label_groups(labels).items():
        assert_envs_equal(mixed, twins[p], g, "before render, %s" % (p,))
        assert torch.equal(frames[torch.as_tensor(g, device="cuda")], twins[p].render_batch(list(g), width=96, height=72, pitch=-45.0))
    close(mixed, twins)


def test_state_dict_round_trip_and_refusal():
    n = 19
    labels = uneven(n, TURN[0])
    kw = dict(auto_reset=True, max_episode_steps=15, seed=5)
    a_env = make_env("turn", n, signal_type=signals_of(labels), **kw)
    a_env.reset()
    gen = torch.Generator(device="cuda"); gen.manual_seed(6)
    acts = [(torch.rand((n, 2), device="cuda", generator=gen) * 2 - 1) * 0.01 for _ in range(20)]
    for a in acts[:10]:
        a_env.step(a)
    sd = a_env.state_dict()
    assert sd["env_tasks"].dtype == torch.uint8
    assert sd["env_tasks"].cpu().tolist() == [[2] * n, [SIGNAL_IDS[s] for _, s in labels]]
    ref = []
    for a in acts[10:]:
        o, r, d, _ = a_env.step(a)
        ref.append((o.clone(), r.clone(), d.clone()))
    b_env = make_env("turn", n, signal_type=signals_of(labels), **kw)
    b_env.load_state_dict(sd)
    everyone = torch.arange(n, device="cuda")
    for (o, r, d), a in zip(ref, acts[10:]):
        ob, rb, db, _ = b_env.step(a)
        for x, y, what in ((o, ob, "obs"), (r, rb, "reward"), (d, db, "done")):
            assert_rows_equal(x, y, everyone, what)
    assert_envs_equal(a_env, b_env, np.arange(n), "after resume")
    for other in (make_env("turn", n, signal_type=signals_of(reversed(labels)), **kw), make_env("turn", n, **kw)):
        with pytest.raises(ValueError, match="per-env tasks"):
            other.load_state_dict(sd)
        other.close()
    close(a_env, b_env)


def test_two_env_offset_shards_reproduce_the_single_batch():
    from rex_gym_b200.sharding import make_sharded_env
    import rex_gym_b200 as R
    n = 24
    labels = [("walk", "ik")] * 3 + [("turn", "ol")] * 9 + [("turn", "ik"), ("walk", "ik")] * 6
    kw = dict(normalize=True, auto_reset=True, max_episode_steps=15, seed=5, task=tasks_of(labels), signal_type=signals_of(labels))
    whole = R.BatchedRexEnv(num_envs=n, **kw)
    shards = [make_sharded_env(n, r, 2, **kw) for r in range(2)]
    assert [s.task for s in shards] == [tuple(t for t, _ in labels[:12]), tuple(t for t, _ in labels[12:])]
    everyone = torch.arange(n, device="cuda")
    o = whole.reset()
    os_ = np.concatenate([s.reset() for s in shards])
    np.testing.assert_array_equal(o.view(np.int32), os_.view(np.int32))
    gen = torch.Generator(device="cuda"); gen.manual_seed(9)
    for k in range(30):
        a = (torch.rand((n, 2), device="cuda", generator=gen) * 2 - 1) * 0.5
        ow, rw, dw, _ = whole.step(a)
        parts = [s.step(a[r * 12:(r + 1) * 12].contiguous()) for r, s in enumerate(shards)]
        for x, i, what in ((ow, 0, "obs"), (rw, 1, "reward"), (dw, 2, "done")):
            assert_rows_equal(x, torch.cat([p[i] for p in parts]), everyone, "%s, step %d" % (what, k))
    close(whole, *shards)


def test_the_entry_point_refusals():
    n = 8
    ik, ol = np.zeros(n, np.int32), np.ones(n, np.int32)
    turn, walk = np.full(n, 2, np.int32), np.array([0, 2] * 4, np.int32)
    mix = np.array([0, 1] * 4, np.int32)
    env = make_env("turn", n, signal_type=["ik", "ol"] * 4)
    assert env._L.rexsim_set_env_tasks(env._h, turn.ctypes.data, mix.ctypes.data) == -1          # a second call
    env.close()
    env = make_env("turn", n)
    env.reset()
    env.step(torch.zeros((n, 2), device="cuda"))
    assert env._L.rexsim_set_env_tasks(env._h, turn.ctypes.data, mix.ctypes.data) == -1          # after the first step
    env.close()
    env = make_env("turn", n)
    for t, s in ((np.array([2, 5] * 4, np.int32), ik), (turn, np.array([0, 2] * 4, np.int32)),   # no such task, signal
                 (np.array([2, -1] * 4, np.int32), ik),
                 (walk, ik),                                         # raw walk ik: the action bound differs
                 (np.array([2, 0] * 4, np.int32), ol),               # walk ol: 8 actions
                 (np.array([2, 1] * 4, np.int32), ik),               # gallop: 16 observations
                 (np.array([2, 3] * 4, np.int32), ik)):              # standup: 1 action
        assert env._L.rexsim_set_env_tasks(env._h, t.ctypes.data, s.ctypes.data) == -1
    assert env._L.rexsim_launch_groups(env._h) == 1
    assert env._L.rexsim_set_env_tasks(env._h, turn.ctypes.data, mix.ctypes.data) == 0          # the refusals left it unset
    assert [g[1:3] + g[5:7] for g in groups_of(env)] == [(2, 0, 0, 4), (2, 1, 4, 4)]
    t, s = ctypes.c_int32(), ctypes.c_int32()
    assert env._L.rexsim_launch_group_task(env._h, 2, ctypes.byref(t), ctypes.byref(s)) == -1
    env.close()
    env = make_env("turn", n, mark="arm")
    gallop = np.array([2, 1] * 4, np.int32)
    assert env._L.rexsim_set_env_tasks(env._h, gallop.ctypes.data, ik.ctypes.data) == -1         # gallop with the arm
    env.close()
    env = make_env("walk", n, normalize=True)
    assert env._L.rexsim_set_env_tasks(env._h, walk.ctypes.data, ik.ctypes.data) == 0            # normalized: accepted
    env.close()
    # a rate setter after the tasks refuses a batch past the group cap: 2 units x 2 terrains x 5 rates
    env = make_env("turn", n * 4, terrain_type=["plane", "random"] * (2 * n), signal_type=["ik", "ik", "ol", "ol"] * n,
                   num_fields=4)
    assert env._L.rexsim_launch_groups(env._h) == 4
    rep = np.array([(1, 2, 3, 4, 5)[(e // 4) % 5] for e in range(4 * n)], np.int32)
    assert env._L.rexsim_set_env_repeats(env._h, rep.ctypes.data, None) == -1
    assert env._L.rexsim_launch_groups(env._h) == 4
    env.close()

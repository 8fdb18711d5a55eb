"""Per-env marks on the GPU: a batch whose envs differ in mark runs each env exactly as the batch built with that env's mark as
the scalar would (the reference's BatchEnv over RexWalkEnv(mark='base') and RexWalkEnv(mark='arm')), in every step-kernel
build, each (terrain, mark, unit, rate) group stepped as its own slot range: outputs, every state word, the command columns and
the sensor-history words each mark owns; the reset hold of every (mark, setting, terrain, field); the groups through
rexsim_rebalance up to the 16-group cap; composition with latencies, noise, task values, gains, gain ranges, the frame
wrappers, final observations, episode statistics, a captured Rollout and the renderer; checkpoints, shards, the ABI's
refusals and all-equal arrays."""
import ctypes

import numpy as np
import pytest
import torch

from mixed_twin import assert_rows_equal, bits, label_groups
from twin import BUILDS, LAYOUT, NOISE, bound, force_build, launched

pytestmark = pytest.mark.gpu

MOTORS = {"base": 12, "arm": 18}
HW_WORDS = {"base": 43, "arm": 61}         # sensor-history words of one ring row (rexsim_kernel.cuh HW_WORDS / HW_WORDS_ARM)
PAIRS = [("walk", "ik"), ("walk", "ol"), ("turn", "ik"), ("turn", "ol"), ("standup", "ol"), ("poses", "ik")]
CASES = [(t, s, b) for t, s in PAIRS for b in ("small", "big", "sensor")]


def interleaved(n):
    """'base' and 'arm' alternating by env, a 50/50 mix."""
    return ["base", "arm"] * (n // 2) + ["base"] * (n % 2)


def build(n, **kw):
    import rex_gym_b200 as R
    return R.BatchedRexEnv(num_envs=n, **kw)


def groups_of(env):
    """[(terrain, motors, action_repeat, first, count, build)] of rexsim_launch_group and rexsim_launch_group_mark."""
    out = []
    for g in range(env._L.rexsim_launch_groups(env._h)):
        info = np.zeros(8, np.int32)
        assert env._L.rexsim_launch_group(env._h, g, info.ctypes.data) == 0
        m = ctypes.c_int32()
        assert env._L.rexsim_launch_group_mark(env._h, g, ctypes.byref(m)) == 0
        out.append((int(info[0]), m.value, int(info[1]), int(info[3]), int(info[4]), tuple(int(x) for x in info[5:])))
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


def assert_marked_envs_equal(mixed, twin, envs, mark, what):
    """Every raw state word of `envs`, bit for bit, their command columns (a base env's rows 12..17 of the mixed batch's 18 are
    NaN) and the sensor-history words their mark owns: a base env's column of the mixed batch's 61-word ring holds its
    [depth][43] rows in its first depth * 43 words, the rest of the column is never written."""
    sel = torch.as_tensor(np.asarray(envs), device="cuda").long()
    for w in range(LAYOUT.NF):
        assert torch.equal(bits(mixed._state_f[w, sel]), bits(twin._state_f[w, sel])), "%s: float word %d" % (what, w)
    for w in range(LAYOUT.NI):
        assert torch.equal(mixed._state_i[w, sel], twin._state_i[w, sel]), "%s: int word %d" % (what, w)
    nm = MOTORS[mark]
    cm, ct = mixed.last_command()[:, sel], twin.last_command()[:, sel]
    assert torch.equal(bits(cm[:nm]), bits(ct)), "%s: command" % what
    if nm < mixed.num_motors:
        assert torch.isnan(cm[nm:]).all(), "%s: a base env's arm command columns are NaN" % what
    assert (mixed._ring is None) == (twin._ring is None)
    if mixed._ring is not None:
        n = mixed.num_envs
        col, tcol = mixed._ring.view(-1, n)[:, sel], twin._ring.view(-1, n)[:, sel]
        own, full = tcol.shape[0], col.shape[0]
        assert own == (full if mixed._marks is None else full * HW_WORDS[mark] // HW_WORDS["arm"])
        assert torch.equal(bits(col[:own]), bits(tcol)), "%s: sensor history" % what
        assert (col[own:] == 0).all(), "%s: ring words past the base's are untouched" % what


def run_mark_twins(n, kw, marks, action_bound, steps=36, reset_at=17, rebalance_at=9, extra=None):
    """A batch of n envs built with kw and mark=marks, and one twin per mark built with kw and that mark as the scalar, stepped
    on the same actions, uniform in +-action_bound, with auto-reset, one explicit reset whose indices span both marks, and a
    re-grouping (rexsim_rebalance) mid-run: every env equals its mark's twin (assert_marked_envs_equal, obs, reward, done),
    bit for bit.  extra(mixed, twin, envs, mark, step) adds checks after each step.  -> (mixed, {mark: twin}, {mark: envs})."""
    groups = label_groups(marks)
    kw = dict(kw, auto_reset=True)
    mixed = build(n, mark=list(marks), **kw)
    twins = {m: build(n, mark=m, **kw) for m in groups}
    everyone = torch.arange(n, dtype=torch.int32, device="cuda")
    o = mixed.reset(everyone)
    for m, tw in twins.items():
        assert_rows_equal(o, tw.reset(everyone), groups[m], "reset obs, %s" % m)
        assert_marked_envs_equal(mixed, tw, groups[m], m, "after reset, %s" % m)
    gen = torch.Generator(device="cuda"); gen.manual_seed(3)
    mid = torch.tensor(sorted({int(e[len(e) // 2]) for e in groups.values()} | {n - 1}), dtype=torch.int32, device="cuda")
    for k in range(steps):
        if k == rebalance_at:
            mixed._call(mixed._L.rexsim_rebalance, mixed._h)       # slots re-sorted within each group's range
        a = (torch.rand((n, mixed.action_dim), device="cuda", generator=gen) * 2 - 1) * action_bound
        om, rm, dm, info = mixed.step(a)
        om, rm, dm = om.clone(), rm.clone(), dm.clone()
        info.materialize()
        for m, tw in twins.items():
            ot, rt, dt, tinfo = tw.step(a)
            assert_rows_equal(om, ot, groups[m], "obs, step %d, %s" % (k, m))
            assert_rows_equal(rm, rt, groups[m], "reward, step %d, %s" % (k, m))
            assert_rows_equal(dm, dt, groups[m], "done, step %d, %s" % (k, m))
            assert_marked_envs_equal(mixed, tw, groups[m], m, "step %d, %s" % (k, m))
            e = int(groups[m][0])
            assert len(info[e]["action"]) == MOTORS[m]
            np.testing.assert_array_equal(info[e]["action"].view(np.int32), tinfo[e]["action"].view(np.int32))
            if extra:
                extra(mixed, tw, groups[m], m, k)
        if k == reset_at:
            r = mixed.reset(mid)
            for m, tw in twins.items():
                sel = np.nonzero(np.isin(mid.cpu().numpy(), groups[m]))[0]
                assert_rows_equal(r, tw.reset(mid), sel, "explicit reset obs, %s" % m)
                assert_marked_envs_equal(mixed, tw, groups[m], m, "after the explicit reset, %s" % m)
    assert mixed.check_errors() == 0
    return mixed, twins, groups


def close(*envs):
    for e in envs:
        for x in (e.values() if isinstance(e, dict) else [e]):
            x.close()


@pytest.mark.parametrize("task,sig,build_name", CASES, ids=["%s-%s-%s" % c for c in CASES])
def test_mixed_marks_match_the_scalar_twins_in_every_build(task, sig, build_name, monkeypatch):
    force_build(monkeypatch, build_name)
    terrain = ("plane", "random")[CASES.index((task, sig, build_name)) % 2]
    kw = dict(task=task, signal_type=sig, seed=13, max_episode_steps=15, terrain_type=terrain, num_fields=4)
    if build_name == "sensor":
        kw["control_latency"] = 0.0125
    n = 27
    marks = interleaved(n)
    mixed, twins, groups = run_mark_twins(n, kw, marks, bound(task, sig))
    assert mixed.mark == tuple(marks) and mixed.num_motors == 18
    assert mixed._marks.cpu().tolist() == [int(m == "arm") for m in marks]
    gs = groups_of(mixed)
    assert [g[1] for g in gs] == [12, 18]                                # in order of first appearance
    for t, nm, r, first, count, built in gs:
        m = "base" if nm == 12 else "arm"
        assert count == len(groups[m]) and built == launched(twins[m]), (m, built)
        assert built == BUILDS["sensor" if build_name == "sensor" else "small" if m == "arm" else build_name]
    close(mixed, twins)


def test_every_reset_hold_matches_its_twin():
    """(mark, gain pair, pd latency, terrain, field): explicit resets only, enough of them to pass every field of the bank."""
    n = 32
    marks = [("base", "arm")[(e // 2) % 2] for e in range(n)]
    kw = dict(task="walk", seed=4, terrain_type=[("plane", "random")[e % 2] for e in range(n)], num_fields=3,
              motor_kp=[(1.0, 1.3)[(e // 4) % 2] for e in range(n)], motor_kd=0.02,
              pd_latency=[(0.0, 0.003)[(e // 8) % 2] for e in range(n)], observation_noise_stdev=NOISE)
    groups = label_groups(marks)
    mixed = build(n, mark=marks, **kw)
    twins = {m: build(n, mark=m, **kw) for m in groups}
    everyone = torch.arange(n, dtype=torch.int32, device="cuda")
    for k in range(4):
        o = mixed.reset(everyone)
        for m, tw in twins.items():
            assert_rows_equal(o, tw.reset(everyone), groups[m], "reset %d obs, %s" % (k, m))
            assert_marked_envs_equal(mixed, tw, groups[m], m, "reset %d, %s" % (k, m))
    fields = mixed._state_i[LAYOUT.I_FIELD].cpu().numpy()
    assert len(set(fields[1::2].tolist())) > 1
    assert mixed._values["gains"].shape[0] == 2 * 2 * 2                   # (mark, kp, pd_latency) settings
    assert mixed.check_errors() == 0
    close(mixed, twins)


def test_groups_and_slot_ranges_hold_only_their_envs_through_rebalance_up_to_sixteen():
    """2 terrains x 2 marks x 2 rates x 2 step units (turn ik, turn ol): the 16 groups of the cap, each env against its mark's
    twin, the slot ranges through two rebalances; a third rate is refused."""
    n = 64
    combos = [(t, m, r, s) for t in ("plane", "random") for m in ("base", "arm") for r in ((0.005, 5), (0.010, 10))
              for s in ("ik", "ol")]
    labels = [combos[(i + i // 16) % 16] for i in range(n)]
    kw = dict(task="turn", seed=13, max_episode_steps=15, num_fields=4, terrain_type=[l[0] for l in labels],
              control_time_step=[l[2][0] for l in labels], action_repeat=[l[2][1] for l in labels],
              signal_type=[l[3] for l in labels])
    marks = [l[1] for l in labels]
    mixed, twins, groups = run_mark_twins(n, kw, marks, 0.01, steps=20, rebalance_at=5)
    gs = groups_of(mixed)
    assert len(gs) == 16 and [g[0] for g in gs] == [0] * 8 + [1] * 8
    perm, grp = slots(mixed)
    for g, (t, nm, r, first, count, built) in enumerate(gs):
        envs = np.nonzero(grp == g)[0]
        assert sorted(perm[first:first + count].tolist()) == envs.tolist() and count == len(envs)
        assert all(labels[e][0] == ("plane", "random")[t] and MOTORS[labels[e][1]] == nm and labels[e][2][1] == r for e in envs)
    close(mixed, twins)
    more = [(t, m, r) for t in ("plane", "random") for m in ("base", "arm") for r in ((0.005, 5), (0.010, 10), (0.001, 1))]
    more = [more[i % len(more)] for i in range(n)]                  # 12 (terrain, mark, rate) x 2 signals: 24 groups
    with pytest.raises(ValueError, match="more than 16 launch groups"):
        build(n, task="turn", terrain_type=[l[0] for l in more], mark=[l[1] for l in more],
              control_time_step=[l[2][0] for l in more], action_repeat=[l[2][1] for l in more],
              signal_type=[("ik", "ol")[(i // 12) % 2] for i in range(n)], num_fields=4)


def test_composes_with_latencies_noise_values_gains_frames_final_observation_and_statistics():
    n = 27
    marks = [("base", "arm", "arm")[e % 3] for e in range(n)]
    kw = dict(task="walk", seed=13, max_episode_steps=15, normalize=True, episode_statistics=True, final_observation=True,
              frame_history=[0, 1, 3], frame_delta=True, observation_noise_stdev=NOISE,
              control_latency=[(0.0, 0.0105, 0.02)[e % 2] for e in range(n)], pd_latency=[(0.0, 0.0005)[(e // 2) % 2] for e in range(n)],
              target_position=[(1.5, 2.0, None)[(e // 3) % 3] for e in range(n)], backwards=[(None, True)[(e // 5) % 2] for e in range(n)],
              motor_kp=[(1.0, 1.2)[(e // 4) % 2] for e in range(n)], motor_kd=[(0.02, 0.03)[(e // 4) % 2] for e in range(n)])

    def extra(mixed, twin, g, m, k):
        assert_rows_equal(mixed.final_observation(), twin.final_observation(), g, "final obs, step %d" % k)
        assert_rows_equal(mixed.limit_bytes(), twin.limit_bytes(), g, "limit byte, step %d" % k)
        for name in ("score", "length"):
            assert_rows_equal(mixed._episode[name], twin._episode[name], g, "%s, step %d" % (name, k))
        assert_rows_equal(mixed.objectives(), twin.objectives(), g, "objectives, step %d" % k)
        for key in mixed._frames:
            assert_rows_equal(mixed._frames[key].view(-1, n).t(), twin._frames[key].view(-1, n).t(), g, key)
        assert_rows_equal(mixed._values["values"].t(), twin._values["values"].t(), g, "task values")

    mixed, twins, groups = run_mark_twins(n, kw, marks, 0.5, extra=extra)
    assert mixed.episode_summary(clear=False)["count"] > 0
    assert mixed._latency is not None and mixed._ring is not None
    close(mixed, twins)


def test_composes_with_a_gain_range():
    n = 20
    kw = dict(task="turn", signal_type="ol", seed=7, max_episode_steps=12, motor_kp_range=(0.8, 1.4), motor_kd_range=(0.01, 0.04),
              terrain_type="random", num_fields=4)
    mixed, twins, _ = run_mark_twins(n, kw, interleaved(n), 0.01, steps=28)
    close(mixed, twins)


def test_captured_rollout_launches_every_group_and_matches_the_twins():
    from rex_gym_b200.agents import ForwardGaussianPolicy, Rollout
    n = 21
    marks = interleaved(n)
    kw = dict(task="walk", normalize=True, auto_reset=True, max_episode_steps=20, seed=8, target_position=2.0, backwards=False)
    mixed = build(n, mark=marks, **kw)
    twins = {m: build(n, mark=m, **kw) for m in ("base", "arm")}
    net = ForwardGaussianPolicy(mixed.obs_dim, mixed.action_dim, seed=1)
    runs, launches = {}, {}
    for name, e in [("mixed", mixed)] + list(twins.items()):
        ro = Rollout(e, net, 8, seed=2, training=False)
        before = e.launch_count
        ro.collect()
        launches[name] = e.launch_count - before
        b = ro.collect()                                     # a replay of the captured graph
        runs[name] = {k: b[k].clone() for k in ("observ", "reward", "done")}
    assert launches["mixed"] == 2 * launches["base"] == 2 * launches["arm"]
    for m, g in label_groups(marks).items():
        for k in ("observ", "reward", "done"):
            assert_rows_equal(runs["mixed"][k].transpose(0, 1), runs[m][k].transpose(0, 1), g, "%s, %s" % (k, m))
    close(mixed, twins)
    net.close()


@pytest.mark.parametrize("terrain", ["plane", "random"])
def test_render_batch_draws_each_env_as_its_twin(terrain):
    n = 12
    marks = interleaved(n)
    kw = dict(task="standup", signal_type="ol", seed=2, terrain_type=terrain, num_fields=4)
    mixed = build(n, mark=marks, **kw)
    twins = {m: build(n, mark=m, **kw) for m in ("base", "arm")}
    gen = torch.Generator(device="cuda"); gen.manual_seed(1)
    for e in [mixed] + list(twins.values()):
        e.reset()
    for k in range(20):
        a = (torch.rand((n, 1), device="cuda", generator=gen) * 2 - 1) * 0.1
        for e in [mixed] + list(twins.values()):
            e.step(a)
    frames = mixed.render_batch(list(range(n)), width=96, height=72, pitch=-45.0)
    for m, g in label_groups(marks).items():
        assert_marked_envs_equal(mixed, twins[m], g, m, "before render, %s" % m)
        assert torch.equal(frames[torch.as_tensor(g, device="cuda")], twins[m].render_batch(list(g), width=96, height=72, pitch=-45.0))
    close(mixed, twins)


def test_state_dict_round_trip_and_refusal():
    n = 19
    marks = interleaved(n)
    kw = dict(task="turn", auto_reset=True, max_episode_steps=15, seed=5, control_latency=0.01)
    a_env = build(n, mark=marks, **kw)
    a_env.reset()
    gen = torch.Generator(device="cuda"); gen.manual_seed(6)
    acts = [(torch.rand((n, 2), device="cuda", generator=gen) * 2 - 1) * 0.01 for _ in range(20)]
    for a in acts[:10]:
        a_env.step(a)
    sd = a_env.state_dict()
    assert sd["env_marks"].dtype == torch.uint8 and sd["env_marks"].cpu().tolist() == [int(m == "arm") for m in marks]
    ref = []
    for a in acts[10:]:
        o, r, d, _ = a_env.step(a)
        ref.append((o.clone(), r.clone(), d.clone()))
    b_env = build(n, mark=marks, **kw)
    b_env.load_state_dict(sd)
    everyone = torch.arange(n, device="cuda")
    for (o, r, d), a in zip(ref, acts[10:]):
        ob, rb, db, _ = b_env.step(a)
        for x, y, what in ((o, ob, "obs"), (r, rb, "reward"), (d, db, "done")):
            assert_rows_equal(x, y, everyone, what)
    assert torch.equal(bits(a_env._state_f), bits(b_env._state_f)) and torch.equal(a_env._state_i, b_env._state_i)
    assert torch.equal(bits(a_env._ring), bits(b_env._ring))
    for other in (build(n, mark=marks[1:] + marks[:1], **kw), build(n, mark="arm", **kw)):
        with pytest.raises(ValueError, match="per-env marks"):
            other.load_state_dict(sd)
        other.close()
    close(a_env, b_env)


def test_two_env_offset_shards_reproduce_the_single_batch():
    from rex_gym_b200.sharding import make_sharded_env
    n = 24
    marks = ["base"] * 3 + ["arm"] * 9 + ["arm", "base"] * 6
    kw = dict(task="walk", normalize=True, auto_reset=True, max_episode_steps=15, seed=5, mark=marks)
    whole = build(n, **kw)
    shards = [make_sharded_env(n, r, 2, **kw) for r in range(2)]
    assert [s.mark for s in shards] == [tuple(marks[:12]), tuple(marks[12:])]
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
    mix = np.array([12, 18] * 4, np.int32)
    env = build(n, task="walk", mark=interleaved(n))
    assert env._L.rexsim_set_env_marks(env._h, mix.ctypes.data) == -1              # a second call
    env.close()
    env = build(n, task="walk", mark="arm")
    env.reset()
    env.step(torch.zeros((n, 2), device="cuda"))
    assert env._L.rexsim_set_env_marks(env._h, mix.ctypes.data) == -1              # after the first step
    env.close()
    env = build(n, task="walk", mark="base")
    assert env._L.rexsim_set_env_marks(env._h, mix.ctypes.data) == -1              # a base handle cannot serve the arm
    env.close()
    env = build(n, task="walk", mark="arm")
    for bad in (np.array([12, 16] * 4, np.int32), np.array([12, 0] * 4, np.int32), np.array([-18] * n, np.int32)):
        assert env._L.rexsim_set_env_marks(env._h, bad.ctypes.data) == -1
    assert env._L.rexsim_launch_groups(env._h) == 1
    p = ctypes.c_void_p()
    assert env._L.rexsim_env_mark_buffers(env._h, ctypes.byref(p)) == -1            # the refusals left it unset
    assert env._L.rexsim_set_env_marks(env._h, mix.ctypes.data) == 0
    assert [(g[1], g[3], g[4]) for g in groups_of(env)] == [(12, 0, 4), (18, 4, 4)]
    m = ctypes.c_int32()
    assert env._L.rexsim_launch_group_mark(env._h, 2, ctypes.byref(m)) == -1
    env.close()
    # the marks after the rates refuse a batch past the group cap: 2 terrains x 4 rates x 2 marks
    env = build(4 * n, task="walk", mark="arm", terrain_type=["plane", "random"] * (2 * n), num_fields=4,
                control_time_step=[(0.005, 0.01, 0.001, 0.003)[(e // 2) % 4] for e in range(4 * n)],
                action_repeat=[(5, 10, 1, 3)[(e // 2) % 4] for e in range(4 * n)])
    assert env._L.rexsim_launch_groups(env._h) == 8
    wide = np.array([(12, 18)[(e // 8) % 2] for e in range(4 * n)], np.int32)
    assert env._L.rexsim_set_env_marks(env._h, wide.ctypes.data) == 0                 # 16 groups: at the cap
    env.close()
    env = build(4 * n, task="walk", mark="arm", terrain_type=["plane", "random"] * (2 * n), num_fields=4,
                control_time_step=[(0.005, 0.01, 0.001, 0.003, 0.002)[(e // 2) % 5] for e in range(4 * n)],
                action_repeat=[(5, 10, 1, 3, 2)[(e // 2) % 5] for e in range(4 * n)])
    assert env._L.rexsim_launch_groups(env._h) == 10
    assert env._L.rexsim_set_env_marks(env._h, wide.ctypes.data) == -1                # 20 groups
    assert env._L.rexsim_launch_groups(env._h) == 10
    env.close()
    # more than 64 hold settings: 40 gain pairs x 2 marks
    n2 = 80
    env = build(n2, task="walk", mark="arm", motor_kp=[1.0 + 0.01 * (e % 40) for e in range(n2)])
    both = np.array([(12, 18)[e // 40] for e in range(n2)], np.int32)
    assert env._L.rexsim_set_env_marks(env._h, both.ctypes.data) == -1
    env.close()


def test_all_equal_arrays_build_the_scalar_construction():
    n = 16
    kw = dict(task="walk", auto_reset=True, seed=21, max_episode_steps=12, control_latency=0.01)
    for m in ("base", "arm"):
        mixed = build(n, mark=[m] * n, **kw)
        twin = build(n, mark=m, **kw)
        assert mixed._marks is None and mixed.mark == m and mixed.num_motors == MOTORS[m]
        p = ctypes.c_void_p()
        assert mixed._L.rexsim_env_mark_buffers(mixed._h, ctypes.byref(p)) == -1           # the feature is off
        assert groups_of(mixed) == groups_of(twin) == [(0, MOTORS[m], 5, 0, n, (0, 0, 0))]
        everyone = torch.arange(n, device="cuda")
        assert_rows_equal(mixed.reset(everyone), twin.reset(everyone), everyone, "reset obs")
        gen = torch.Generator(device="cuda"); gen.manual_seed(4)
        for k in range(20):
            a = (torch.rand((n, 2), device="cuda", generator=gen) * 2 - 1) * 0.4
            om, rm, dm, _ = mixed.step(a)
            om, rm, dm = om.clone(), rm.clone(), dm.clone()
            ot, rt, dt, _ = twin.step(a)
            for x, y, what in ((om, ot, "obs"), (rm, rt, "reward"), (dm, dt, "done")):
                assert_rows_equal(x, y, everyone, "%s, step %d" % (what, k))
            assert_marked_envs_equal(mixed, twin, np.arange(n), m, "step %d" % k)
        assert mixed.launch_count == twin.launch_count
        assert slots(mixed) == (None, None)
        close(mixed, twin)

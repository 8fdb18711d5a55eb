"""Per-env terrains on the GPU: a batch whose envs stand on the plane and on the heightfield runs each env exactly as the batch
built with that env's terrain as the scalar would (the reference's BatchEnv over envs that differ only in terrain_type), in
every step-kernel build, with the two terrains stepped as two slot ranges of one batch; all-equal arrays against the scalar
construction; the reset hold of every (setting, terrain, field) against the twins; composition with the sensor model, the
frame wrappers, final observations, episode statistics, per-env task values, a captured Rollout and the renderer;
checkpoints, shards and the ABI's refusals."""
import ctypes

import numpy as np
import pytest
import torch

from twin import BUILDS, INSTANCES, LAYOUT, NOISE, bound, force_build, instance_config, launched, make_env

pytestmark = pytest.mark.gpu

TERRAIN_IDS = {"plane": 0, "random": 1}
# (task, signal, arm, build) of every step_kernel instance: the terrain axis is the batch's own here
ROWS = list(dict.fromkeys((t, s, arm, b) for t, s, arm, _, b in INSTANCES))


def rid(row):
    task, sig, arm, build = row
    return "-".join([task, sig] + (["arm"] if arm else []) + [build])


def uneven(n):
    """Env i on the plane when i % 3 == 1: a third of the batch, both ranges ending in partial warps for odd n."""
    return ["plane" if i % 3 == 1 else "random" for i in range(n)]


def terrain_build(env, terrain):
    """(CTA size, CTAs per SM, sensor) of the last step launch over `terrain`'s envs (rexsim_last_terrain_build)."""
    v = [ctypes.c_int32() for _ in range(3)]
    assert env._L.rexsim_last_terrain_build(env._h, TERRAIN_IDS[terrain], *[ctypes.byref(x) for x in v]) == 0
    return tuple(x.value for x in v)


def _bits(t):
    t = torch.as_tensor(t).contiguous()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _assert_rows_equal(a, b, rows, what):
    rows = torch.as_tensor(rows, device=torch.as_tensor(a).device).long()
    if rows.numel() == 0:
        return
    a, b = _bits(a), _bits(b)
    bad = (a[rows] != b[rows]).reshape(len(rows), -1).any(1)
    assert not bad.any(), "%s differs in envs %s" % (what, rows.cpu()[bad.cpu()].tolist())


def _assert_envs_equal(mixed, twin, envs, what):
    """Every raw state word (float and int, by name from the kernel's header) of `envs`, bit for bit, and the envs' columns
    of the sensor history ring."""
    sel = torch.as_tensor(envs, device="cuda").long()
    f1, f2 = mixed._state_f[:, sel], twin._state_f[:, sel]
    i1, i2 = mixed._state_i[:, sel], twin._state_i[:, sel]
    for w in range(LAYOUT.NF):
        assert torch.equal(_bits(f1[w]), _bits(f2[w])), "%s: float word %d of envs %s" % (what, w, list(envs))
    for w in range(LAYOUT.NI):
        assert torch.equal(i1[w], i2[w]), "%s: int word %d of envs %s" % (what, w, list(envs))
    assert (mixed._ring is None) == (twin._ring is None)
    if mixed._ring is not None:
        n = mixed.num_envs
        assert torch.equal(_bits(mixed._ring.view(-1, n)[:, sel]), _bits(twin._ring.view(-1, n)[:, sel])), "%s: ring" % what


def _accumulators(env):
    """The per-env episode accumulators of env's block: sum_score f64 | sum_length i64 | score f32 | length i32 | count i32 |
    nonfinite i32, [N] each."""
    n, b = env.num_envs, env._episode["block"]
    return dict(sum_score=b[:8 * n].view(torch.float64), sum_length=b[8 * n:16 * n].view(torch.int64),
                count=b[24 * n:28 * n].view(torch.int32), nonfinite=b[28 * n:32 * n].view(torch.int32))


def run_against_twins(task, n, cfg, terrain, steps=36, reset_at=17, rebalance_at=9, extra=None):
    """A batch of n envs on `terrain` (one entry per env) and its plane and heightfield twins, stepped on the same actions with
    auto-reset, one explicit reset spanning both terrains and a re-grouping mid-run: every env's outputs and state words
    equal its twin's, bit for bit.  -> (mixed, {terrain: twin}, {terrain: env indices})."""
    mixed = make_env(task, n, auto_reset=True, terrain_type=list(terrain), **cfg)
    twins = {t: make_env(task, n, auto_reset=True, terrain_type=t, **cfg) for t in TERRAIN_IDS}
    groups = {t: np.nonzero(np.array(terrain) == t)[0] for t in TERRAIN_IDS}
    assert all(len(g) for g in groups.values())
    everyone = torch.arange(n, dtype=torch.int32, device="cuda")
    o = mixed.reset(everyone)
    for t, tw in twins.items():
        _assert_rows_equal(o, tw.reset(everyone), groups[t], "reset obs, %s" % t)
        _assert_envs_equal(mixed, tw, groups[t], "after reset, %s" % t)
    gen = torch.Generator(device="cuda"); gen.manual_seed(3)
    b = bound(task, cfg.get("signal_type", "ik"))
    mid = torch.tensor([1, 12, n - 1], dtype=torch.int32, device="cuda")   # plane, heightfield, heightfield
    for k in range(steps):
        if k == rebalance_at:
            mixed._call(mixed._L.rexsim_rebalance, mixed._h)       # slots re-sorted within each terrain's range
        a = (torch.rand((n, mixed.action_dim), device="cuda", generator=gen) * 2 - 1) * b
        om, rm, dm, _ = mixed.step(a)
        om, rm, dm = om.clone(), rm.clone(), dm.clone()
        for t, tw in twins.items():
            ot, rt, dt, _ = tw.step(a)
            _assert_rows_equal(om, ot, groups[t], "obs, step %d, %s" % (k, t))
            _assert_rows_equal(rm, rt, groups[t], "reward, step %d, %s" % (k, t))
            _assert_rows_equal(dm, dt, groups[t], "done, step %d, %s" % (k, t))
            _assert_envs_equal(mixed, tw, groups[t], "step %d, %s" % (k, t))
            if extra:
                extra(mixed, tw, groups[t], k)
        if k == reset_at:
            r = mixed.reset(mid)
            for t, tw in twins.items():
                sel = np.nonzero(np.isin(mid.cpu().numpy(), groups[t]))[0]
                _assert_rows_equal(r, tw.reset(mid), sel, "explicit reset obs, %s" % t)
    assert mixed.check_errors() == 0
    return mixed, twins, groups


@pytest.mark.parametrize("row", ROWS, ids=rid)
def test_mixed_terrains_match_the_scalar_twins_in_every_build(row, monkeypatch):
    task, sig, arm, build = row
    force_build(monkeypatch, build)
    cfg = instance_config((task, sig, arm, "random", build))
    cfg.pop("terrain_type")
    n = 27
    mixed, twins, groups = run_against_twins(task, n, cfg, uneven(n))
    # the plane envs always run the plane build, the heightfield envs the heightfield build, each the row's build
    for t, tw in twins.items():
        assert terrain_build(mixed, t) == BUILDS[build] == terrain_build(tw, t), t
    assert launched(mixed) == terrain_build(mixed, "random")            # a mixed step's last launch: the heightfield range
    sf = mixed._state_i[LAYOUT.I_FIELD].cpu().numpy()
    assert (sf[groups["plane"]] == 0).all()
    for e in [mixed] + list(twins.values()):
        e.close()


@pytest.mark.parametrize("terrain", ["plane", "random"])
def test_all_equal_arrays_build_the_scalar_construction(terrain):
    n, task = 16, "walk"
    kw = dict(auto_reset=True, seed=21, max_episode_steps=12, num_fields=4)
    mixed = make_env(task, n, terrain_type=np.array([terrain] * n), **kw)
    twin = make_env(task, n, terrain_type=terrain, **kw)
    assert mixed._terrain is None and mixed.terrain_type == terrain
    assert (mixed._fields is None) == (twin._fields is None) == (terrain == "plane")
    assert mixed.launch_count == twin.launch_count
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
    assert mixed.launch_count == twin.launch_count
    assert terrain_build(mixed, terrain) == terrain_build(twin, terrain) != (0, 0, 0)
    mixed.close(); twin.close()


def test_reset_hold_of_every_setting_terrain_and_field_equals_the_twins():
    """Per-env gains and per-env pd_latency mixed with both terrains: after each of four resets every env has been reset from
    the (setting, terrain, field) snapshot its twin resets from, and its state and history rows are the twin's, bit for bit.
    Four resets take every env through the four fields (field = (env + reset count) mod 4)."""
    n = 36
    gains = [(1.0, 0.02), (1.3, 0.03), (0.8, 0.015)]
    i = np.arange(n)
    terrain = ["plane" if (e // 6) % 2 else "random" for e in i]          # every (setting, terrain) pair, on several envs
    kw = dict(signal_type="ik", seed=77, num_fields=4, target_position=2.0, backwards=False,
              motor_kp=[gains[e % 3][0] for e in i], motor_kd=[gains[e % 3][1] for e in i],
              pd_latency=[(0.0, 0.0005)[(e // 3) % 2] for e in i], control_latency=0.0105)
    mixed = make_env("walk", n, terrain_type=terrain, **kw)
    twins = {t: make_env("walk", n, terrain_type=t, **kw) for t in TERRAIN_IDS}
    assert mixed._values["gains"].shape[0] == 6                         # 3 gain pairs x 2 pd latencies
    groups = {t: np.nonzero(np.array(terrain) == t)[0] for t in TERRAIN_IDS}
    seen = set()
    for r in range(4):
        o = mixed.reset()
        for t, tw in twins.items():
            _assert_rows_equal(torch.as_tensor(o), torch.as_tensor(tw.reset()), groups[t], "reset %d obs, %s" % (r, t))
            _assert_envs_equal(mixed, tw, groups[t], "reset %d, %s" % (r, t))
        field = mixed._state_i[LAYOUT.I_FIELD].cpu().numpy()
        pair = mixed._values["pair"].cpu().numpy()
        seen |= {(int(pair[e]), terrain[e], int(field[e])) for e in range(n)}
    assert seen == {(s, "plane", 0) for s in range(6)} | {(s, "random", f) for s in range(6) for f in range(4)}
    assert mixed.check_errors() == 0
    for e in [mixed] + list(twins.values()):
        e.close()


def test_composes_with_sensor_noise_frames_final_observation_statistics_and_task_values():
    n = 25
    cfg = dict(signal_type="ik", seed=13, max_episode_steps=15, episode_statistics=True, final_observation=True,
               frame_history=[0, 1, 3], frame_delta=True, num_fields=4, observation_noise_stdev=NOISE, control_latency=0.0105,
               target_position=[(1.5, 2.0, None)[e % 3] for e in range(n)], backwards=[(None, True)[e % 2] for e in range(n)])

    def extra(mixed, twin, g, k):
        _assert_rows_equal(mixed.final_observation(), twin.final_observation(), g, "final obs, step %d" % k)
        _assert_rows_equal(mixed.limit_bytes(), twin.limit_bytes(), g, "limit byte, step %d" % k)
        for name in ("score", "length"):
            _assert_rows_equal(mixed._episode[name], twin._episode[name], g, "%s, step %d" % (name, k))
        _assert_rows_equal(mixed.objectives(), twin.objectives(), g, "objectives, step %d" % k)
        for key in mixed._frames:
            _assert_rows_equal(mixed._frames[key].view(-1, n).t(), twin._frames[key].view(-1, n).t(), g, key)
        _assert_rows_equal(mixed._values["values"].t(), twin._values["values"].t(), g, "task values")

    mixed, twins, groups = run_against_twins("walk", n, cfg, uneven(n), extra=extra)
    acc = {k: _accumulators(e) for k, e in [("mixed", mixed)] + list(twins.items())}
    for t in TERRAIN_IDS:
        for name in ("sum_score", "sum_length", "count", "nonfinite"):
            _assert_rows_equal(acc["mixed"][name], acc[t][name], groups[t], "%s, %s" % (name, t))
    # the batch's summary is its envs' submissions, each the twin's
    count = sum(int(acc[t]["count"][torch.as_tensor(groups[t], device="cuda")].sum()) for t in TERRAIN_IDS)
    assert mixed.episode_summary(clear=False)["count"] == count > 0
    for e in [mixed] + list(twins.values()):
        e.close()


def test_captured_rollout_launches_both_ranges_and_matches_the_twins():
    from rex_gym_b200.agents import ForwardGaussianPolicy, Rollout
    n = 21
    terrain = uneven(n)
    cfg = dict(normalize=True, auto_reset=True, max_episode_steps=20, seed=8, target_position=2.0, backwards=False, num_fields=4)
    mixed = make_env("walk", n, terrain_type=terrain, **cfg)
    twins = {t: make_env("walk", n, terrain_type=t, **cfg) for t in TERRAIN_IDS}
    net = ForwardGaussianPolicy(mixed.obs_dim, mixed.action_dim, seed=1)
    runs, launches = {}, {}
    for name, e in [("mixed", mixed)] + list(twins.items()):
        ro = Rollout(e, net, 8, seed=2, training=False)
        before = e.launch_count
        ro.collect()
        launches[name] = e.launch_count - before
        b = ro.collect()                                     # a replay of the captured graph
        runs[name] = {k: b[k].clone() for k in ("observ", "reward", "done")}
    # warm-up and capture: every control step is two step launches in the mixed batch, one in each twin
    assert launches["mixed"] == 2 * launches["plane"] == 2 * launches["random"] == 2 * 2 * 8
    for t in TERRAIN_IDS:
        g = np.nonzero(np.array(terrain) == t)[0]
        for k in ("observ", "reward", "done"):
            _assert_rows_equal(runs["mixed"][k].transpose(0, 1), runs[t][k].transpose(0, 1), g, "%s, %s" % (k, t))
    for e in [mixed] + list(twins.values()):
        e.close()
    net.close()


def test_render_batch_draws_each_envs_own_ground():
    n = 12
    terrain = uneven(n)
    cfg = dict(signal_type="ik", seed=2, num_fields=4, target_position=2.0, backwards=False)
    mixed = make_env("turn", n, terrain_type=terrain, **cfg)
    twins = {t: make_env("turn", n, terrain_type=t, **cfg) for t in TERRAIN_IDS}
    gen = torch.Generator(device="cuda"); gen.manual_seed(1)
    for e in [mixed] + list(twins.values()):
        e.reset()
    for k in range(40):
        a = (torch.rand((n, mixed.action_dim), device="cuda", generator=gen) * 2 - 1) * 0.01
        for e in [mixed] + list(twins.values()):
            e.step(a)
    frames = mixed.render_batch(list(range(n)), width=96, height=72, pitch=-45.0)
    for t, tw in twins.items():
        g = np.nonzero(np.array(terrain) == t)[0]
        _assert_envs_equal(mixed, tw, g, "before render, %s" % t)
        ft = tw.render_batch(list(g), width=96, height=72, pitch=-45.0)
        assert torch.equal(frames[torch.as_tensor(g, device="cuda")], ft), t
    # the two grounds do differ: a plane env's frame is not its heightfield twin's
    p = int(np.nonzero(np.array(terrain) == "plane")[0][0])
    assert not torch.equal(frames[p], twins["random"].render_batch([p], width=96, height=72, pitch=-45.0)[0])
    for e in [mixed] + list(twins.values()):
        e.close()


def test_state_dict_round_trip_and_refusal():
    n = 19
    terrain = uneven(n)
    kw = dict(auto_reset=True, max_episode_steps=15, seed=5, num_fields=4)
    a_env = make_env("walk", n, terrain_type=terrain, **kw)
    a_env.reset()
    gen = torch.Generator(device="cuda"); gen.manual_seed(6)
    acts = [(torch.rand((n, 2), device="cuda", generator=gen) * 2 - 1) * 0.4 for _ in range(20)]
    for a in acts[:10]:
        a_env.step(a)
    sd = a_env.state_dict()
    assert sd["env_terrain"].dtype == torch.uint8 and sd["env_terrain"].cpu().tolist() == [TERRAIN_IDS[t] for t in terrain]
    ref = []
    for a in acts[10:]:
        o, r, d, _ = a_env.step(a)
        ref.append((o.clone(), r.clone(), d.clone()))
    b_env = make_env("walk", n, terrain_type=terrain, **kw)
    b_env.load_state_dict(sd)
    everyone = torch.arange(n, device="cuda")
    for (o, r, d), a in zip(ref, acts[10:]):
        ob, rb, db, _ = b_env.step(a)
        for x, y, what in ((o, ob, "obs"), (r, rb, "reward"), (d, db, "done")):
            _assert_rows_equal(x, y, everyone, what)
    _assert_envs_equal(a_env, b_env, np.arange(n), "after resume")
    with pytest.raises(ValueError, match="terrains"):
        make_env("walk", n, terrain_type=list(reversed(terrain)), **kw).load_state_dict(sd)
    with pytest.raises(ValueError, match="terrains"):
        make_env("walk", n, terrain_type="random", **kw).load_state_dict(sd)
    a_env.close(); b_env.close()


def test_two_env_offset_shards_reproduce_the_single_batch():
    from rex_gym_b200.sharding import make_sharded_env
    import rex_gym_b200 as R
    n = 24
    terrain = ["plane"] * 3 + ["random"] * 9 + ["random", "plane"] * 6       # the first shard's plane range is short
    kw = dict(task="walk", auto_reset=True, max_episode_steps=15, seed=5, num_fields=4, terrain_type=terrain)
    whole = R.BatchedRexEnv(num_envs=n, **kw)
    shards = [make_sharded_env(n, r, 2, **kw) for r in range(2)]
    assert [s.terrain_type for s in shards] == [tuple(terrain[:12]), tuple(terrain[12:])]
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


def test_the_entry_point_refusals():
    n = 8
    t = np.array([0, 1] * 4, np.int32)
    env = make_env("walk", n, terrain_type=["plane", "random"] * 4, num_fields=4)
    assert env._L.rexsim_set_env_terrains(env._h, t.ctypes.data, 0.5) == -1             # a second call
    env.close()
    env = make_env("walk", n, terrain_type="random", num_fields=4)
    env.reset()
    assert env._L.rexsim_set_env_terrains(env._h, t.ctypes.data, 0.5) == -1             # after the first reset
    env.close()
    env = make_env("walk", n, terrain_type="random", num_fields=4)
    bad = np.array([0, 1, 2, 0, 1, 0, 1, 0], np.int32)
    assert env._L.rexsim_set_env_terrains(env._h, bad.ctypes.data, 0.5) == -1           # not a terrain
    assert env._L.rexsim_set_env_terrains(env._h, t.ctypes.data, -1.0) == -1            # negative friction
    assert env._L.rexsim_set_env_terrains(env._h, t.ctypes.data, 0.5) == 0              # the refusals left it unset
    env.close()
    env = make_env("walk", n)                                                            # created on the plane: no bank
    assert env._L.rexsim_set_env_terrains(env._h, t.ctypes.data, 0.5) == -1
    p, q = ctypes.c_void_p(), ctypes.c_int32()
    assert env._L.rexsim_env_terrain_buffers(env._h, ctypes.byref(p), ctypes.byref(q)) == -1
    env.close()

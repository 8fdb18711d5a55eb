"""The 18-DOF arm (mark='arm') on every task but gallop: walk with either signal, turn with either signal, standup and poses.

The arm is a fifth limb on lane 0 of each env (rex_gym_b200/csrc/rexsim_arm.cuh) and holds ARM_POSES['rest'] whatever the task
(rex_gym_env.py:363-367): the 12 leg commands come from the task, the 6 arm commands are the rest pose.  Gallop stays refused:
the reference's gallop observes all 18 motor angles, and the step and reset kernels fix the observation at the 12 legs.

ARM_INSTANCES is the arm half of the step kernel's dispatch image: 6 (task, signal) units x 2 terrains x the small and sensor
builds (arm batches never take the 128-register build) = 24 rows.  The 8 rows of walk-ik and standup are run by
test_gpu_builds::test_instance_against_the_oracle; test_arm_instance_against_the_oracle runs the other 16 here.
"""
import json
import os

import numpy as np
import pytest
import torch
from twin import (BUILDS, LAYOUT, STATE_KEYS, IterationBand, assert_draws, bound, force_build, launched, make_env, make_oracle,
                  oracle_protection, protection, state_errors, sync)

HERE = os.path.dirname(os.path.abspath(__file__))
ARM_REST = np.array(json.load(open(os.path.join(HERE, "golden", "constants_golden.json")))["arm_poses"]["rest"], np.float32)
UNITS = [("walk", "ik"), ("walk", "ol"), ("gallop", "ik"), ("gallop", "ol"), ("turn", "ik"), ("turn", "ol"), ("standup", "ol"), ("poses", "ik")]
ALL_GROUPS = 0x7FFF                   # contact groups 0-8 of the legged robot and 9-14 of the arm links
BUILDS_TEST = "test_gpu_builds::test_instance_against_the_oracle"

#  task      signal terrain   build     run by
ARM_INSTANCES = [
    ("walk",    "ik", "plane",  "small",  BUILDS_TEST),
    ("walk",    "ik", "plane",  "sensor", BUILDS_TEST),
    ("walk",    "ik", "random", "small",  BUILDS_TEST),
    ("walk",    "ik", "random", "sensor", BUILDS_TEST),
    ("walk",    "ol", "plane",  "small",  None),
    ("walk",    "ol", "plane",  "sensor", None),
    ("walk",    "ol", "random", "small",  None),
    ("walk",    "ol", "random", "sensor", None),
    ("turn",    "ik", "plane",  "small",  None),
    ("turn",    "ik", "plane",  "sensor", None),
    ("turn",    "ik", "random", "small",  None),
    ("turn",    "ik", "random", "sensor", None),
    ("turn",    "ol", "plane",  "small",  None),
    ("turn",    "ol", "plane",  "sensor", None),
    ("turn",    "ol", "random", "small",  None),
    ("turn",    "ol", "random", "sensor", None),
    ("standup", "ol", "plane",  "small",  BUILDS_TEST),
    ("standup", "ol", "plane",  "sensor", BUILDS_TEST),
    ("standup", "ol", "random", "small",  BUILDS_TEST),
    ("standup", "ol", "random", "sensor", BUILDS_TEST),
    ("poses",   "ik", "plane",  "small",  None),
    ("poses",   "ik", "plane",  "sensor", None),
    ("poses",   "ik", "random", "small",  None),
    ("poses",   "ik", "random", "sensor", None),
]
NEW = [r[:4] for r in ARM_INSTANCES if r[4] is None]
NEW_PAIRS = [("walk", "ol"), ("turn", "ik"), ("turn", "ol"), ("poses", "ik")]


def _row_id(row):
    task, sig, terrain, build = row[:4]
    return "-".join([task, sig, "arm", terrain, build])


def _create_status(task, sig):
    """rexsim_create's status for an 18-motor config of (task, sig) handed a base-sized (952-float) model table: -2 once the
    config is accepted (the table size is checked after validation and before any CUDA call), -4 when the arm is refused."""
    import ctypes as C
    from rex_gym_b200 import _capi
    from rex_gym_b200.envs.batched_env import SIGNALS, TASKS
    L = _capi.load()
    cfg = _capi.RexSimConfig()
    cfg.num_envs, cfg.task, cfg.signal, cfg.num_motors = 8, TASKS[task], SIGNALS[sig], 18
    cfg.action_repeat, cfg.solver_iterations, cfg.sim_dt_d, cfg.toe_npts, cfg.gait_clock_scale = 5, 60, 0.001, 27, 1.0
    h = C.c_void_p()
    tb = np.zeros(952, np.float32)
    return L.rexsim_create(C.byref(cfg), tb.ctypes.data, 952, C.byref(h)), L.rexsim_last_error()


@pytest.mark.parametrize("task,sig", [u for u in UNITS if u[0] != "gallop"] + [("standup", "ik"), ("poses", "ol")])
def test_create_accepts_the_arm_for_every_task_but_gallop(task, sig):
    """CPU: an 18-motor config of any task but gallop passes validation (it fails on the model table size, -2)."""
    rc, msg = _create_status(task, sig)
    assert rc == -2 and b"model table" in msg, (rc, msg)


@pytest.mark.parametrize("sig", ["ik", "ol"])
def test_create_still_refuses_gallop_with_the_arm(sig):
    """CPU: gallop with the arm is refused before any CUDA call, with the arm and gallop named in the message."""
    rc, msg = _create_status("gallop", sig)
    assert rc == -4 and b"arm" in msg and b"gallop" in msg, (rc, msg)


def test_arm_instance_table_is_the_arm_half_of_the_dispatch_image():
    """CPU: the table above lists each arm instance once, for exactly the units the library accepts the arm for, on both
    terrains and in the small and sensor builds; the rows this file does not run name an existing test."""
    arm_units = [(t, s) for t, s in UNITS if _create_status(t, s)[0] == -2]
    want = {(t, s, ter, b) for t, s in arm_units for ter in ("plane", "random") for b in ("small", "sensor")}
    got = [r[:4] for r in ARM_INSTANCES]
    assert len(got) == len(set(got)) == len(want) == 24
    assert set(got) == want
    assert len(NEW) == 16 and {(t, s) for t, s, _, _ in NEW} == set(NEW_PAIRS)
    for row in ARM_INSTANCES:
        if row[4] is not None:
            mod, name = row[4].split("::")
            assert ("def %s(" % name) in open(os.path.join(HERE, mod + ".py")).read(), row


def _config(task, sig, terrain, build):
    kw = dict(signal_type=sig, seed=13, max_episode_steps=15, mark="arm")    # short episodes: two in-kernel resets per env
    if terrain == "random":
        kw.update(terrain_type="random", num_fields=4)
    if build == "sensor":
        kw["control_latency"] = 0.0125                                      # a blend of two history rows, 12 sub-steps back
    return kw


def _masks(ora):
    return np.array([ora.env(i).contact_mask & ALL_GROUPS for i in range(ora.N)])


@pytest.mark.gpu
@pytest.mark.parametrize("row", NEW, ids=[_row_id(r) for r in NEW])
def test_arm_instance_against_the_oracle(monkeypatch, row):
    """One new arm instance, forced by force_build (the sensor build by its config; rexsim_last_step_build confirms which one ran
    every step), against the oracle: 37 envs, 40 control steps of random actions inside the task's bound, auto-reset after 15
    steps.  Done, draws and counters bit for bit after every step.  The state starts from the oracle's settled state and is
    re-synchronised at each reset; between resets it stays within the bounds the walk-ik and standup arm rows meet
    (5e-3 rad / 2e-3 m at the 90th percentile of the envs, none beyond 5e-2 / 5e-3), and every auto-reset lands within
    test_reset_settle_and_draws' loosest bounds.  Every step's command block has 18 rows, the last six ARM_POSES['rest']; on flat
    ground the 12 leg commands are within 5e-4 of the oracle's and the rewards within 5e-3.  Roll / pitch observations and the
    contact masks of all 15 groups (arm links included) as in test_instance_against_the_oracle."""
    task, sig, terrain, build = row
    force_build(monkeypatch, build)
    n, steps = 37, 40
    kw = _config(task, sig, terrain, build)
    env, ora = make_env(task, n, auto_reset=True, **kw), make_oracle(task, n, **kw)
    env.reset(); ora.reset()
    rough = terrain == "random"
    sync(env, ora)
    rng = np.random.default_rng(11)
    b = bound(task, sig)
    err_rp, contact_total, contact_bad = [], 0, 0
    for k in range(steps):
        a = rng.uniform(-b, b, size=(n, env.action_dim)).astype(np.float32)
        og, rg, dg, info = env.step(a)
        assert launched(env) == BUILDS[build], launched(env)
        assert info[n - 1]["action"].shape == (18,)
        np.testing.assert_array_equal(info[n - 1]["action"][12:], ARM_REST)
        oc, rc, dc = ora.step(a)
        np.testing.assert_array_equal(dg, dc, err_msg=f"done, step {k}")
        cmd = env.last_command().cpu().numpy().T
        np.testing.assert_array_equal(cmd[:, 12:], np.broadcast_to(ARM_REST, (n, 6)))
        ocmd = np.array([np.array(ora.env(i).cmd[:12]) for i in range(n)])
        idx = np.nonzero(dc)[0]
        if len(idx):
            oc[idx] = ora.reset(idx)                      # the oracle has no auto-reset: the same semantics by hand
        sg, so = env.get_state(), ora.states()
        assert_draws(env, ora, task)
        fresh = np.zeros(n, bool)
        fresh[idx] = True
        eq, ep = state_errors(env, ora)
        if not rough:
            ep = np.maximum(ep, np.abs(sg["quat"] - so["quat"]).max(axis=1))
        if len(idx):
            # the in-kernel reset restarts from the CUDA settle: test_reset_settle_and_draws' loosest bounds (standup with the arm)
            assert eq[idx].max() < 3e-2 and ep[idx].max() < 2e-3, f"reset, step {k}: {eq[idx].max():.2e} {ep[idx].max():.2e}"
        eq, ep = eq[~fresh], ep[~fresh]
        if len(eq):
            assert np.percentile(eq, 90) < 5e-3 and np.percentile(ep, 90) < 2e-3, f"step {k}: {eq.max():.2e} {ep.max():.2e}"
            assert eq.max() < 5e-2 and ep.max() < 5e-3, f"step {k}: {eq.max():.2e} {ep.max():.2e}"
            # a re-synchronised sensor build reads its own settle's history rows for the first 3 control steps of an episode
            ocmp = ~fresh & (sg["env_step_counter"] >= 3) if build == "sensor" else ~fresh
            err_rp.append(np.abs(og[ocmp, :2] - oc[ocmp, :2]).max(axis=1))
        if not rough:
            assert np.abs(cmd[:, :12] - ocmd).max() < 5e-4, f"cmd step {k}"     # the controller half: fp32 IK / Bezier vs fp64
            np.testing.assert_allclose(rg, rc, atol=5e-3, err_msg=f"reward, step {k}")
        # the mask of contacts in the last sub-step: after a reset the CUDA path reports none yet, the oracle its settle's last
        contact_total += (~fresh).sum()
        contact_bad += ((_masks(ora) != (sg["contact_mask"] & ALL_GROUPS)) & ~fresh).sum()
        if len(idx):
            sync(env, ora, idx)
    err_rp = np.concatenate(err_rp)
    assert np.percentile(err_rp, 90) < 1e-3 and err_rp.max() < (2e-2 if rough else 5e-3), (np.percentile(err_rp, 90), err_rp.max())
    assert contact_bad <= 0.02 * max(contact_total, 1), (contact_bad, contact_total)
    assert env.check_errors() == 0
    env.close()


RESET_CASES = [(t, s, "plane") for t, s in NEW_PAIRS] + [("turn", "ik", "random")]


@pytest.mark.gpu
@pytest.mark.parametrize("task,sig,terrain", RESET_CASES)
def test_arm_reset_settle_and_draws(task, sig, terrain):
    """Rex.Reset with the arm on the GPU against the oracle, 16 envs: draws and motor-enabled bits bit for bit.
    On flat ground the settled state is within the walk-ik arm bounds (2e-4 rad / 2e-5 m) and the base rates at the end of the
    hold within 2e-3 rad/s of the range the oracle spans over its early-out thresholds (the arm's limit rows keep the base
    rocking, see test_gpu_parity::test_reset_settle_and_draws).  On the bank two of the four fields leave the robot creeping down
    a slope with the arm's limit rows pressed when the hold ends: joint angles within 2e-2 rad (H100: 8.3e-3 on a foot joint,
    5.5e-3 on the first arm joint), base rates within 0.1 rad/s of the oracle's range (H100: 7.5e-2; rates on heightfield
    contact are chaotic at that level, see test_gpu_parity::test_batches_that_do_not_fill_their_last_warp) and the overheat
    counters of those fields within 12 counts; the other fields settle within the flat-ground bound, counters bit for bit.
    Turn re-poses the base after the settle (at the origin, 0.21 m up, yawed to the drawn initial orientation); the joints, the
    arm's included, keep the settled state of the walk with the same signal bit for bit.  Poses skips both holding phases: the
    arm starts at rest, at rest."""
    n = 16
    kw = dict(signal_type=sig, seed=77, mark="arm")
    if terrain == "random":
        kw.update(terrain_type="random", num_fields=4)
    env, ora = make_env(task, n, **kw), make_oracle(task, n, **kw)
    og, oc = env.reset(), ora.reset()
    sg, so = env.get_state(), ora.states()
    tq, tp = (2e-2, 2e-3) if terrain == "random" else (2e-4, 2e-5)
    eq, ep = state_errors(env, ora)
    assert eq.max() < tq and ep.max() < tp, (eq.max(), ep.max())
    assert np.abs(sg["quat"] - so["quat"]).max() < tq
    np.testing.assert_allclose(og[:, :2], oc[:, :2], atol=10 * tq)
    runs = [o.reset()[:, 2:4] for o in IterationBand(lambda **b: make_oracle(task, n, **kw, **b)).oracles]
    lo, hi = np.min(runs, 0), np.max(runs, 0)
    rate_tol = 0.1 if terrain == "random" else 2e-3
    bad = (og[:, 2:4] < lo - rate_tol) | (og[:, 2:4] > hi + rate_tol)
    assert not bad.any(), ("outside the oracle's band", og[:, 2:4][bad], lo[bad], hi[bad])
    assert_draws(env, ora, task)
    cnt, en = protection(env)
    ocnt, oen = oracle_protection(ora)
    np.testing.assert_array_equal(en, oen)
    assert en.all()
    # overheat counters bit for bit wherever the hold settles alike; where it diverges, a motor near the 2.45 N m threshold
    # crosses it some sub-steps apart (H100: up to 8 of the hold's 600 sub-steps, on the bank's two creeping fields)
    alike = eq < 2e-4
    assert alike.all() if terrain == "plane" else alike.sum() >= n // 2, eq
    np.testing.assert_array_equal(cnt[alike], ocnt[alike])
    assert np.abs(cnt - ocnt).max() <= 12
    if task == "turn":
        io = env._state_f[LAYOUT.F_IORIENT].cpu().numpy()
        np.testing.assert_array_equal(sg["pos"], np.broadcast_to(np.float32([0, 0, 0.21]), (n, 3)))
        np.testing.assert_array_equal(sg["quat"][:, :2], 0)
        np.testing.assert_allclose(sg["quat"][:, 2:], np.stack([np.sin(io / 2), np.cos(io / 2)], 1), atol=1e-6)
        walk = make_env("walk", n, **kw)
        walk.reset()
        sw = walk.get_state()
        for k in ("q", "qd"):
            np.testing.assert_array_equal(sg[k], sw[k])
        walk.close()
    if task == "poses":
        np.testing.assert_array_equal(sg["q"][:, 12:], np.broadcast_to(ARM_REST, (n, 6)))
        np.testing.assert_array_equal(sg["qd"], 0)
        assert (sg["step_counter"] == 0).all()
    assert env.check_errors() == 0
    env.close()


@pytest.mark.gpu
def test_turn_ik_arm_heightfield_batch_against_the_oracle():
    """The C4 configuration with the arm at its per-GPU size (turn-ik, 64 fields, 16 384 envs): a window of 48 consecutive envs
    from the middle of the batch is re-simulated by the fp64 oracle with the same global env ids, from the oracle's settled
    state, over 40 control steps.  Reset draws bit for bit.  At every step the 90th percentile of the window's state errors stays
    within the arm rows' bounds (5e-3 rad / 2e-3 m) and the roll / pitch observations within the C4 bounds (90th percentile of all
    samples below 1e-3 rad).  At most one env may leave the per-env bounds (5e-2 rad, 5e-3 m, 2e-2 rad observed): a toe handing
    over across a crease of the field a sub-step apart in fp32 and fp64 (H100: one env from step 16 on, to 0.11 rad on a foot
    joint, 6.9e-3 m and 5.3e-2 rad observed).  That env is held to 0.2 rad / 1e-2 m / 0.1 rad, and done is bit for bit on every
    other env and on that one until it leaves."""
    n, nw, steps = 16384, 48, 40
    w0 = n // 2 + 37
    kw = dict(signal_type="ik", terrain_type="random", num_fields=64, mark="arm", normalize=True, seed=11)
    env, ora = make_env("turn", n, **kw), make_oracle("turn", nw, env_offset=w0, **kw)
    og = env.reset()[w0:w0 + nw]
    oc = ora.reset()
    np.testing.assert_allclose(og[:, :2], oc[:, :2], atol=2e-4)          # RangeNormalize'd roll / pitch
    assert_draws(env, ora, "turn", window=w0)
    st, so = env.get_state(), ora.states()
    for k in STATE_KEYS:
        st[k][w0:w0 + nw] = so[k]
    env.set_state(*(st[k] for k in STATE_KEYS))
    g = torch.Generator(device="cuda"); g.manual_seed(5)
    acts = torch.rand((steps, n, env.action_dim), device="cuda", generator=g) * 2 - 1
    err, left = [], np.zeros(nw, bool)
    for k in range(steps):
        o, r, d, _ = env.step(acts[k])
        assert launched(env) == BUILDS["small"], launched(env)
        oc, rc, dc = ora.step(acts[k, w0:w0 + nw].cpu().numpy())
        eo = np.abs(o[w0:w0 + nw, :2].cpu().numpy() - oc[:, :2]).max(axis=1) * (2 * np.pi + 0.01)     # RangeNormalize'd -> radians
        eq, ep = state_errors(env, ora, window=w0)
        left |= (eq >= 5e-2) | (ep >= 5e-3) | (eo >= 2e-2)
        np.testing.assert_array_equal(d[w0:w0 + nw].cpu().numpy()[~left], dc[~left], err_msg=f"done, step {k}")
        assert np.percentile(eq, 90) < 5e-3 and np.percentile(ep, 90) < 2e-3, f"step {k}: {np.percentile(eq, 90):.2e} {np.percentile(ep, 90):.2e}"
        assert eq.max() < 0.2 and ep.max() < 1e-2 and eo.max() < 0.1, f"step {k}: {eq.max():.2e} {ep.max():.2e} {eo.max():.2e}"
        err.append(eo)
    assert left.sum() <= 1, np.nonzero(left)[0]
    assert np.percentile(np.concatenate(err), 90) < 1e-3
    assert (env.check_errors() & 1) == 0
    env.close()


@pytest.mark.gpu
def test_turn_ik_with_the_arm_on_the_heightfield_renders_as_the_oracle():
    """render_batch of two turn-ik arm envs on the heightfield bank, stepped 50 times, against tests/render_oracle.py under the
    bounds of test_gpu_render.py: at most 0.5 % of the pixels differ by more than 2/255 in a channel, each within 1 px of a
    change of surface patch in the oracle's id image.  The arm is in the picture."""
    import render_oracle as RO
    from rex_gym_b200.envs.batched_env import RexTurnBatchEnv
    env = RexTurnBatchEnv(num_envs=2, signal_type="ik", terrain_type="random", num_fields=4, mark="arm", seed=2)
    env.reset()
    rng = np.random.default_rng(2)
    for _ in range(50):
        env.step(rng.uniform(-0.01, 0.01, size=(2, env.action_dim)).astype(np.float32))
    img = env.render_batch([0, 1]).cpu().numpy()
    st = env.get_state()
    field = env.state_dict()["state_i"][LAYOUT.I_FIELD].cpu().numpy()
    for i in range(2):
        heights = env._fields[int(field[i])].cpu().numpy().reshape(256, 256)
        ref, ids = RO.render("arm", st["pos"][i].astype(np.float64), st["quat"][i].astype(np.float64),
                             st["q"][i].astype(np.float64), 480, 360, 1.0, 0.0, -30.0, "random", heights)
        bad = (np.abs(img[i].astype(np.int16) - ref.astype(np.int16)) > 2).any(-1)
        assert bad.mean() <= 0.005, "env %d: %.3f %% of pixels differ" % (i, 100 * bad.mean())
        pad = np.pad(ids, 1, mode="edge")
        edge = np.zeros(ids.shape, bool)
        for dy in (0, 1, 2):
            for dx in (0, 1, 2):
                edge |= pad[dy:dy + ids.shape[0], dx:dx + ids.shape[1]] != ids
        assert not (bad & ~edge).any(), "env %d: pixels differ away from any patch edge" % i
        shapes = set((ids[(ids >= 0) & (ids < RO.GROUND_ID)] // 1000 - 1).tolist())
        assert any(s >= 19 for s in shapes)                 # shapes 19 on are the arm's
    env.close()


SURFACE = [("RexTurn-v0", "turn", dict()), ("RexWalk-v0", "walk", dict(signal_type="ol")), ("RexPoses-v0", "poses", dict())]


@pytest.mark.gpu
@pytest.mark.parametrize("env_id,task,kw", SURFACE, ids=[s[0] for s in SURFACE])
def test_public_surface_with_the_arm(env_id, task, kw):
    """make(env_id, mark='arm') and the single-env facade take the arm with no new keyword.  The spaces, obs_dim and action_dim
    are the base mark's; info['action'] and last_command() carry 18 motors; get_state / set_state round-trip 18 joints;
    state_dict / load_state_dict resume bit for bit; render and render_batch give frames; a shard created with env_offset
    reproduces its block of the whole batch bit for bit, auto-resets included."""
    import rex_gym_b200 as R
    from rex_gym_b200.envs import single_env
    n = 8
    arm = R.make(env_id, num_envs=n, mark="arm", auto_reset=True, max_episode_steps=6, seed=3, **kw)
    base = R.make(env_id, num_envs=n, **kw)
    assert arm.num_motors == 18 and base.num_motors == 12
    assert (arm.obs_dim, arm.action_dim) == (base.obs_dim, base.action_dim) and arm.obs_dim == 4
    for sa, sb in ((arm.action_space, base.action_space), (arm.observation_space, base.observation_space)):
        np.testing.assert_array_equal(sa.low, sb.low)
        np.testing.assert_array_equal(sa.high, sb.high)
    base.close()
    shard = R.make(env_id, num_envs=n // 2, env_offset=n // 2, mark="arm", auto_reset=True, max_episode_steps=6, seed=3, **kw)
    o, os_ = arm.reset(), shard.reset()
    assert o.shape == (n, 4)
    np.testing.assert_array_equal(o[n // 2:], os_)
    b = bound(task, kw.get("signal_type", "ik"))
    rng = np.random.default_rng(4)
    acts = rng.uniform(-b, b, size=(14, n, arm.action_dim)).astype(np.float32)
    for k in range(14):
        o, r, d, info = arm.step(acts[k])
        os_, rs, ds, _ = shard.step(acts[k, n // 2:])
        assert len(info) == n and info[2]["action"].shape == (18,)
        np.testing.assert_array_equal(info[2]["action"][12:], ARM_REST)
        for x, y in ((o[n // 2:], os_), (r[n // 2:], rs), (d[n // 2:], ds)):
            np.testing.assert_array_equal(x, y)
    assert arm.get_state()["env_step_counter"].max() < 6             # the batch went through auto-resets
    assert tuple(arm.last_command().shape) == (18, n)
    st = arm.get_state()
    assert st["q"].shape == (n, 18) and st["qd"].shape == (n, 18)
    st["q"][:, 12:] += 0.01
    arm.set_state(*(st[k] for k in STATE_KEYS))
    st2 = arm.get_state()
    for k in STATE_KEYS:
        np.testing.assert_array_equal(st2[k], st[k])
    sd = arm.state_dict()
    o1 = arm.step(acts[0])[0].copy()
    arm.load_state_dict(sd)
    np.testing.assert_array_equal(arm.step(acts[0])[0], o1)
    f = arm.render()
    assert f.shape == (360, 480, 3) and f.dtype == np.uint8
    assert np.array_equal(arm[3].render(), arm.render_batch([3])[0].cpu().numpy())
    assert arm.check_errors() == 0 and shard.check_errors() == 0
    arm.close(); shard.close()
    cls = {"turn": single_env.RexTurnEnv, "walk": single_env.RexWalkEnv, "poses": single_env.RexPosesEnv}[task]
    e = cls(mark="arm", **kw)
    assert e.num_motors == 18 and e.reset().shape == (4,)
    o, r, d, info = e.step(np.zeros(e.action_space.shape, np.float32))
    assert o.shape == (4,) and isinstance(r, float) and isinstance(d, bool) and info["action"].shape == (18,)
    assert e.render().shape == (360, 480, 3) and len(e.rex.GetMotorAngles()) == 18
    e.close()


@pytest.mark.gpu
def test_gallop_with_the_arm_still_raises():
    import rex_gym_b200 as R
    with pytest.raises(ValueError, match="arm"):
        R.make("RexGalloping-v0", mark="arm")

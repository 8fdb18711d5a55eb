"""GPU: every build of the step kernel the dispatcher can launch, against the fp64 oracle (called through the C ABI).

`step_kernel<TASK, SIGNAL, TERRAIN, OCC, ARM, SENSOR, BLOCK>` (rex_gym_b200/csrc/rexsim_kernel.cu) exists in three builds for each
(task, signal, terrain, arm); `launch_step_tsta` picks one on every step launch:

  sensor  any control / PD latency or observation noise > 0        255 registers, 128-thread CTAs
  big     no sensor model, no arm, and ceil(N / 32) > 2 x SMs on    128 registers (REXSIM_OCC_BIG), 256-thread CTAs
          flat ground, > 4 x SMs on heightfields                    (REXSIM_BLOCK_BIG); on heightfields its 64 tiles per CTA
          (H100 SXM, 132 SMs: N > 8448 / N > 16 896)                take 78 KB of shared memory through the opt-in
  small   everything else                                           255 registers, 128-thread CTAs

twin.force_build(monkeypatch, "big" | "small") replaces the size rule (arm batches stay on the small build); the forced build is
read on every step launch and does not touch the reset or settle kernels.

twin.INSTANCES is the dispatch rule's whole image: 8 (task, signal) units x 2 terrains x 3 builds, plus the 6 arm units (every
task but gallop) x 2 terrains x the small and sensor builds = 72 rows.  test_instance_against_the_oracle[<row id>] runs every row;
ALSO names the other tests of the suite that launch the same instance.
"""
import os

import numpy as np
import pytest
import torch
from twin import (ARM_REST, ARM_UNITS, BUILDS, BUILDS_OF, INSTANCES, TOL_P, TOL_Q, UNITS, assert_draws, bound, create_status,
                  force_build, instance_config, launched, make_env, make_oracle, one_step_is_tight, row_id, state_errors, sync,
                  toe_masks, window_twin)

FR, HF, SA = "test_gpu_parity::test_free_running_rollout", "test_gpu_parity::test_heightfield_contact_parity", "test_gpu_parity::test_sensor_latency_and_noise"
BL, WARP = "test_gpu_parity::test_baseline_size_batches_against_the_oracle", "test_gpu_parity::test_batches_that_do_not_fill_their_last_warp"
REGROUP, HOST = ("test_gpu_parity::test_warp_regrouping_does_not_change_any_result_on_the_128_register_build",
                 "test_gpu_parity::test_numpy_and_device_paths_agree_beyond_the_zero_copy_limit")
NATURAL, SWITCH = "test_gpu_builds::test_heightfield_big_build_at_its_natural_size", "test_gpu_builds::test_the_dispatcher_switches_builds_at_its_thresholds"

# the other tests of the suite that launch an instance
ALSO = {
    "walk-ik-plane-small": (FR,), "walk-ik-plane-big": (BL + "[C2]", REGROUP, HOST, SWITCH), "walk-ik-plane-sensor": (SA,),
    "walk-ik-random-small": (WARP,), "walk-ik-random-sensor": (SA,),
    "walk-ol-plane-small": (FR,),
    "gallop-ik-plane-small": (FR,),
    "gallop-ol-plane-small": (FR,), "gallop-ol-plane-big": (BL + "[C3]",), "gallop-ol-plane-sensor": (SA,),
    "turn-ik-plane-small": (FR,), "turn-ik-plane-sensor": (SA,), "turn-ik-random-small": (HF, BL + "[C4]"),
    "turn-ik-random-big": (NATURAL, SWITCH),
    "turn-ol-plane-small": (FR,),
    "standup-ol-plane-small": (FR,),
    "poses-ik-plane-small": (FR,), "poses-ik-plane-sensor": (SA,),
    "walk-ik-arm-plane-small": (FR,),
    "standup-ol-arm-plane-small": (FR, BL + "[C5]"), "standup-ol-arm-plane-sensor": (SA,),
}


def test_instance_table_lists_every_reachable_instance():
    """CPU: the dispatch image lists each instance once; its arm half covers exactly the units the library accepts the arm for
    (rexsim_create, before any CUDA call); every row's build is one of its mark's; every test ALSO names exists."""
    assert len(INSTANCES) == len(set(INSTANCES)) == 72
    assert {(t, s) for t, s, arm, _, _ in INSTANCES if arm} == {u for u in UNITS if create_status(*u)[0] == -2} == set(ARM_UNITS)
    assert all(b in BUILDS_OF["arm" if arm else "base"] for _, _, arm, _, b in INSTANCES)
    ids = {row_id(r) for r in INSTANCES}
    here = os.path.dirname(os.path.abspath(__file__))
    for rid, refs in ALSO.items():
        assert rid in ids, rid
        for ref in refs:
            mod, name = ref.split("[")[0].split("::")
            assert ("def %s(" % name) in open(os.path.join(here, mod + ".py")).read(), ref


@pytest.mark.gpu
@pytest.mark.parametrize("row", INSTANCES, ids=[row_id(r) for r in INSTANCES])
def test_instance_against_the_oracle(monkeypatch, row):
    """One instance, forced by force_build (the sensor build by its config; rexsim_last_step_build confirms which one ran
    every step), against the oracle: 37 envs (padding lanes in
    both CTA sizes), 40 control steps of random actions inside the task's bound, auto-reset after 15 steps.  Integer results bit
    for bit after every step; continuous ones within the bounds the small build meets elsewhere in the suite:
      flat-ground locomotion  test_free_running_rollout's strict window (90th percentile of the envs within 1e-3 rad / 1e-3 m,
                              none beyond 5e-2 / 5e-3; motor commands 5e-4, rewards 5e-3);
      standup, arm            its standup bounds (5e-3 / 2e-3 at the 90th percentile), from the oracle's settled state;
      heightfields            test_heightfield_contact_parity's (1e-3 / 1e-3 at the 90th percentile, none beyond 2e-2 / 5e-3), from
                              the oracle's settled state (toes creep on block edges while settling);
    roll / pitch observations as in test_baseline_size_batches_against_the_oracle, contact masks (the 9 groups of the legged
    robot, all 15 with the arm) in 98 % of the samples that are not the first of an episode.
    Where the state starts from the oracle's, every auto-reset lands within the settle bounds and is re-synchronised.
    With the arm, every step's command block has 18 rows, the last six ARM_POSES['rest'] (rex_gym_env.py:363-367), and so
    has info['action']."""
    task, sig, arm, terrain, build = row
    force_build(monkeypatch, build)
    n, steps = 37, 40
    kw = instance_config(row)
    env, ora = make_env(task, n, auto_reset=True, **kw), make_oracle(task, n, **kw)
    env.reset(); ora.reset()
    rough, standup = terrain == "random", task == "standup" or arm
    resync = rough or standup
    tol_q, tol_p = (5e-3, 2e-3) if standup else (TOL_Q, TOL_P)                     # test_free_running_rollout
    max_q, max_p = (2e-2, 5e-3) if rough and not standup else (5e-2, 5e-3)
    ta = 5e-3 if (rough or standup) else 1e-3                                      # roll / pitch observations
    groups = 0x7FFF if arm else 0x1FF                                              # contact groups 0-8, 9-14 the arm links
    if resync:
        sync(env, ora)
    rng = np.random.default_rng(11)
    b = bound(task, sig)
    err_rp, contact_total, contact_bad = [], 0, 0
    for k in range(steps):
        a = rng.uniform(-b, b, size=(n, env.action_dim)).astype(np.float32)
        og, rg, dg, info = env.step(a)
        assert launched(env) == BUILDS[build], launched(env)
        oc, rc, dc = ora.step(a)
        np.testing.assert_array_equal(dg, dc, err_msg=f"done, step {k}")
        cmd = env.last_command().cpu().numpy().T
        if arm:
            assert info[n - 1]["action"].shape == (18,)
            np.testing.assert_array_equal(info[n - 1]["action"][12:], ARM_REST)
            np.testing.assert_array_equal(cmd[:, 12:], np.broadcast_to(ARM_REST, (n, 6)))
        ocmd = np.array([np.array(ora.env(i).cmd[:12]) for i in range(n)])
        idx = np.nonzero(dc)[0]
        if len(idx):
            oc[idx] = ora.reset(idx)                      # the oracle has no auto-reset: the same semantics by hand
        sg, so = env.get_state(), ora.states()
        assert_draws(env, ora, task)
        fresh = np.zeros(n, bool)
        fresh[idx] = True
        cmp = ~fresh if resync else np.ones(n, bool)
        eq, ep = state_errors(env, ora)
        if not rough:
            ep = np.maximum(ep, np.abs(sg["quat"] - so["quat"]).max(axis=1))
        if resync and len(idx):
            # the in-kernel reset restarts from the CUDA settle: test_reset_settle_and_draws' loosest bounds (standup with the arm)
            assert eq[idx].max() < 3e-2 and ep[idx].max() < 2e-3, f"reset, step {k}: {eq[idx].max():.2e} {ep[idx].max():.2e}"
        eq, ep = eq[cmp], ep[cmp]
        if len(eq):
            assert np.percentile(eq, 90) < tol_q and np.percentile(ep, 90) < tol_p, f"step {k}: {eq.max():.2e} {ep.max():.2e}"
            assert eq.max() < max_q and ep.max() < max_p, f"step {k}: {eq.max():.2e} {ep.max():.2e}"
            # a re-synchronised sensor build reads its own settle's history rows for the first 3 control steps of an episode
            ocmp = cmp & (sg["env_step_counter"] >= 3) if (resync and build == "sensor") else cmp
            err_rp.append(np.abs(og[ocmp, :2] - oc[ocmp, :2]).max(axis=1))
        if not rough:
            assert np.abs(cmd[:, :12] - ocmd).max() < 5e-4, f"cmd step {k}"     # the controller half: fp32 IK / Bezier vs fp64
            rcmp = np.ones(n, bool)
            if task == "standup":      # the standup reward jumps by 1 where the base crosses z = 0.21 or the L1 distance 0.1
                l1 = np.abs(so["pos"][:, 0]) + np.abs(so["pos"][:, 1]) + np.abs(0.21 - so["pos"][:, 2])
                rcmp &= (np.abs(so["pos"][:, 2] - 0.21) > 2e-3) & (np.abs(l1 - 0.1) > 2e-3) & ~fresh
            np.testing.assert_allclose(rg[rcmp], rc[rcmp], atol=5e-3, err_msg=f"reward, step {k}")
        # the mask of contacts in the last sub-step: after a reset the CUDA path reports none yet, the oracle its settle's last
        omask = np.array([ora.env(i).contact_mask for i in range(n)]) & groups
        contact_total += (~fresh).sum(); contact_bad += ((omask != sg["contact_mask"]) & ~fresh).sum()
        if resync and len(idx):
            sync(env, ora, idx)
    err_rp = np.concatenate(err_rp)
    assert np.percentile(err_rp, 90) < ta / 5 and err_rp.max() < (2e-2 if rough else ta), (np.percentile(err_rp, 90), err_rp.max())
    assert contact_bad <= 0.02 * max(contact_total, 1), (contact_bad, contact_total)
    assert env.check_errors() == 0
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("build", ["small", "big"])
@pytest.mark.parametrize("task,sig,kw,bound", [("walk", "ik", dict(target_position=2.0, backwards=False), 0.4),
                                               ("standup", "ol", dict(), 0.1)], ids=["walk-ik", "standup-ol"])
def test_one_step_is_tight_in_both_builds(monkeypatch, build, task, sig, kw, bound):
    """test_one_step_is_tight (30 single control steps from an oracle-synchronised state) with the build forced: the big build
    meets the same rounding-level bounds as the small one."""
    force_build(monkeypatch, build)
    one_step_is_tight(task, sig, kw, bound)


@pytest.mark.gpu
def test_heightfield_big_build_at_its_natural_size():
    """test_baseline_size_batches_against_the_oracle's window on a heightfield batch large enough for the dispatcher to pick the big
    build by itself (turn-ik, 64 fields, 32 768 envs: ceil(N / 32) = 1024 > 4 x SMs), so the 78 KB shared-memory opt-in and the
    64-tile-per-CTA indexing run as a user's batch runs them.  48 consecutive envs from the middle of the batch are re-simulated by
    the fp64 oracle (same global env ids): draws and done bit for bit; the window starts from the oracle's settled state, and its
    base position and joint angles stay within test_heightfield_contact_parity's bounds, its roll / pitch observations within the
    C4 bounds, over 40 control steps."""
    n, w0, nw, steps = 32768, 32768 // 2 + 37, 48, 40
    assert -(-n // 32) > 4 * torch.cuda.get_device_properties(0).multi_processor_count       # really above the switch
    env, ora, _, _, acts = window_twin("turn", n, w0, nw, steps, settled=True, signal_type="ik", terrain_type="random",
                                       num_fields=64, normalize=True, seed=11)
    err, bad = [], 0
    for k in range(steps):
        o, r, d, _ = env.step(acts[k])
        oc, rc, dc = ora.step(acts[k, w0:w0 + nw].cpu().numpy())
        np.testing.assert_array_equal(d[w0:w0 + nw].cpu().numpy(), dc)
        err.append(np.abs(o[w0:w0 + nw, :2].cpu().numpy() - oc[:, :2]).max(axis=1))
        eq, ep = state_errors(env, ora, window=w0)
        assert np.percentile(eq, 90) < TOL_Q and np.percentile(ep, 90) < TOL_P and eq.max() < 2e-2 and ep.max() < 5e-3, \
            f"step {k}: {np.percentile(eq, 90):.2e} {np.percentile(ep, 90):.2e} {eq.max():.2e} {ep.max():.2e}"
        bad += (toe_masks(ora) != env.get_state()["contact_mask"][w0:w0 + nw]).sum()
    err = np.concatenate(err) * (2 * np.pi + 0.01)                      # RangeNormalize'd -> radians
    assert np.percentile(err, 90) < 1e-3 and err.max() < 2e-2, (np.percentile(err, 90), err.max())
    assert bad <= 0.02 * steps * nw
    assert (env.check_errors() & 1) == 0
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("terrain,per_sm", [("plane", 2), ("random", 4)])
def test_the_dispatcher_switches_builds_at_its_thresholds(monkeypatch, terrain, per_sm):
    """The size rule pinned where it switches: ceil(N / 32) > 2 x SMs on flat ground, > 4 x SMs on heightfields.  At the threshold
    the unforced batch launches the same kernel as one forced onto the small build and is bit-identical to it over 12 steps (with
    auto-resets); one env above it, the same holds with the big build.  The forced batches launch different instances (128-thread
    CTAs at 1 CTA per SM, 256-thread CTAs at 4), so neither identity holds by accident: the two builds can agree bit for bit
    (walk-ik and turn-ik do on an H100)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    threshold = 32 * per_sm * sms                     # the largest N that stays on the small build
    task = "walk" if terrain == "plane" else "turn"
    kw = dict(signal_type="ik", auto_reset=True, max_episode_steps=10, normalize=True, seed=7)
    if terrain == "random":
        kw.update(terrain_type="random", num_fields=4)
    for n, picked in ((threshold, "small"), (threshold + 1, "big")):
        envs = {b: make_env(task, n, **kw) for b in ("auto", "small", "big")}
        for e in envs.values():
            e.reset()
        g = torch.Generator(device="cuda"); g.manual_seed(9)
        ran = {}
        for k in range(12):
            act = torch.rand((n, 2), device="cuda", generator=g) * 2 - 1
            out = {}
            for b, e in envs.items():
                force_build(monkeypatch, None if b == "auto" else b)
                out[b] = [t.clone() for t in e.step(act)[:3]]
                ran.setdefault(b, set()).add(launched(e))
            assert all(torch.equal(x, y) for x, y in zip(out["auto"], out[picked])), (n, k)
        assert ran["small"] == {(128, 1, 0)} and ran["big"] == {(256, 4, 0)} and ran["auto"] == ran[picked], (n, ran)
        assert torch.equal(envs["auto"]._state_f, envs[picked]._state_f) and torch.equal(envs["auto"]._state_i, envs[picked]._state_i)
        for e in envs.values():
            assert (e.check_errors() & 1) == 0
            e.close()

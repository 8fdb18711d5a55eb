"""Motor overheat protection (Rex.ApplyAction, rex.py:601-608) in the step kernel against the fp64 oracle.

Every sub-step, a motor whose applied torque exceeds 2.45 N m counts up, any other motor resets its count to 0, and a motor whose
count passes floor(1 / sim_dt) is switched off until the next reset.  apply_action_and_step (rex_gym_b200/csrc/rexsim_kernel.cu)
keeps the counts in 10-bit saturating fields, three per word (I_OVH: 4 words for the legs, I_OVHA: 2 for the arm), and the
enabled bits in bits 8-19 (legs) and 20-25 (arm) of I_FLAGS; store_lane and store_arm merge them into the flags word, and a reset
copies them from the settled snapshot.  The oracle counts in an int32, so counters are compared as min(oracle, 1023).

No task reaches a shutdown by itself within an episode, so the scenarios seed counters near the limit on motors the oracle shows
to be hot, in both implementations at once (only integer state is written: no sensor ring goes stale).
test_scenarios_switch_motors_off (CPU) pins what each scenario reaches, so the GPU tests cannot go vacuous.  The GPU tests run
37 envs, seeded envs mixed with unseeded ones in every warp (the last env, which the padding lanes replicate, is seeded), in
{small, big, sensor} x {plane, random} for the leg scenarios and {small, sensor} x {plane, random} for the arm.
"""
import ctypes

import numpy as np
import pytest

from twin import (BUILDS, BUILDS_OF, NOISE, SUB, bound, force_build, launched, make_env, make_oracle, oracle_protection,
                  protection, state_errors, sync)

N = 37
SEEDED = np.array([i % 3 != 1 for i in range(N)])              # envs 0, 2, 3, 5, ..., 36 seeded; 1, 4, ..., 34 not
FEET = [2, 5, 8, 11]
EDGE = dict(control_time_step=0.00489, action_repeat=5)        # 1 / dt = 1022.49: the largest floor(1 / dt) the counters serve

# scenario: (task, signal, mark, control steps of random actions before the seeding, extra kwargs)
SCENARIOS = {
    "standup": ("standup", "ol", "base", 0, dict()),
    "gallop": ("gallop", "ol", "base", 20, dict(motor_kp_range=(0.8, 1.2), motor_kd_range=(0.01, 0.03))),
    "walk": ("walk", "ik", "base", 40, dict(target_position=2.0, backwards=False)),
    "turn": ("turn", "ik", "base", 40, dict()),
    "arm-standup": ("standup", "ol", "arm", 0, dict()),
    "arm-walk": ("walk", "ik", "arm", 0, dict(target_position=2.0, backwards=False)),
}
LEG_SCENARIOS = ["standup", "gallop", "walk", "turn"]
ARM_SCENARIOS = ["arm-standup", "arm-walk"]
ARM_DISPLACEMENT = 0.4          # rad added to every arm joint of a seeded env: the arm's counters are 0 after the hold


def _okw(name, terrain, **extra):
    task, sig, mark, _, kw = SCENARIOS[name]
    kw = dict(kw, signal_type=sig, seed=31, **extra)
    if mark == "arm":
        kw["mark"] = "arm"
    if terrain == "random":
        kw.update(terrain_type="random", num_fields=4)
    return task, kw


def _seed(ora, name, values):
    """Seed the oracle: counters `values[i]` (None: env untouched) on every motor of the scenario; the arm scenarios also displace
    the arm's joints."""
    mark = SCENARIOS[name][2]
    motors = range(12, 18) if mark == "arm" else range(12)
    for i, v in enumerate(values):
        if v is None:
            continue
        e = ora.env(i)
        for m in motors:
            e.overheat[m] = v
        if mark == "arm":
            for j in range(12, 18):
                e.q[j] += ARM_DISPLACEMENT


def _prepare(name, terrain, env=None, **extra):
    """Oracle (and, if given, the GPU env) reset and stepped to the seeding point on the same actions; the oracle seeded on the
    SEEDED envs.  -> (oracle, rng for the actions that follow)."""
    task, kw = _okw(name, terrain, **extra)
    ora = make_oracle(task, N, **kw)
    ora.reset()
    if env is not None:
        env.reset()
    rng = np.random.default_rng(5)
    b = bound(task, SCENARIOS[name][1])
    for k in range(SCENARIOS[name][3]):
        a = rng.uniform(-b, b, size=(N, ora.A)).astype(np.float32)
        ora.step(a)
        if env is not None:
            env.step(a)
    v = 1000 if SCENARIOS[name][2] == "arm" else 996           # the arm scenarios seed only the arm
    _seed(ora, name, [v if s else None for s in SEEDED])
    return ora, rng


def _gpu_env(name, terrain, build, monkeypatch, **extra):
    force_build(monkeypatch, build)
    if build == "sensor":                                      # the sensor build, with zero latencies
        extra.setdefault("observation_noise_stdev", NOISE)
    task, kw = _okw(name, terrain, **extra)
    return make_env(task, N, **kw), extra


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("terrain", ["plane", "random"])
def test_scenarios_switch_motors_off(terrain):
    """CPU: over the control steps the GPU tests run after the seeding (15), every one of the 18 motors switches off in at least
    one env of some scenario (shoulders in standup, legs in gallop, feet in every leg scenario), all four feet in every seeded
    standup env on flat ground, and nothing in an unseeded env."""
    off_any = np.zeros(18, bool)
    per_joint = {0: set(), 1: set(), 2: set()}
    for name in LEG_SCENARIOS + ARM_SCENARIOS:
        ora, rng = _prepare(name, terrain)
        task, sig = SCENARIOS[name][:2]
        b = bound(task, sig)
        for k in range(15):
            ora.step(rng.uniform(-b, b, size=(N, ora.A)).astype(np.float32))
        _, en = oracle_protection(ora)
        off = ~en
        assert not off[~SEEDED].any(), (name, np.nonzero(off[~SEEDED]))
        assert off.any(), name
        off_any[:ora.nm] |= off.any(0)
        for m in range(12):
            if off[:, m].any():
                per_joint[m % 3].add(name)
        if name == "standup" and terrain == "plane":
            assert off[SEEDED][:, FEET].all(), name                         # all four feet in every seeded env
    assert off_any.all(), np.nonzero(~off_any)
    assert all(per_joint.values()), per_joint


def test_create_refuses_time_steps_the_counters_cannot_count():
    """A motor switches off once its count c > floor(1 / sim_dt), and c saturates at 1023: rexsim_create refuses
    floor(1 / sim_dt) >= 1023 (REXSIM_ERR_UNSUPPORTED, -4) before it touches the GPU, and names the counter."""
    from rex_gym_b200 import _capi
    L = _capi.load()
    h = ctypes.c_void_p()
    tb = np.zeros(952, np.float32)
    # action_repeat 10 at the default 5 ms control step (2000 counts), 1 / dt = 1023.3, and 1 / dt = 1023 exactly
    for dt in (0.005 / 10, 0.004886 / 5, 1.0 / 1023):
        cfg = _capi.RexSimConfig()
        cfg.num_envs, cfg.num_motors, cfg.task, cfg.solver_iterations, cfg.toe_npts, cfg.gait_clock_scale = 8, 12, 0, 60, 27, 1.0
        cfg.action_repeat, cfg.sim_dt_d = 5, dt
        assert L.rexsim_create(ctypes.byref(cfg), tb.ctypes.data, 952, ctypes.byref(h)) == -4, dt
        assert b"overheat" in L.rexsim_last_error()
    assert int(1.0 / (EDGE["control_time_step"] / EDGE["action_repeat"])) == 1022       # accepted: the edge tests run it


def test_oracle_switches_off_on_count_1023_at_the_largest_accepted_rate():
    """CPU: at 1 / dt = 1022.49 the oracle switches a motor off on its 1023rd consecutive hot sub-step -- the top value of the
    kernel's 10-bit field -- and standup's hold leaves 511 on the feet (it holds them hot for its last 0.5 s)."""
    ora = make_oracle("standup", 4, signal_type="ol", **EDGE)
    ora.reset()
    cnt, en = oracle_protection(ora)
    assert (cnt[:, FEET] == 511).all() and en.all()
    for i, v in enumerate((1018, 1017, 1016, None)):           # 5 hot sub-steps per control step
        for m in FEET:
            if v is not None:
                ora.env(i).overheat[m] = v
    ora.step(np.zeros((4, 1), np.float32))
    cnt, en = oracle_protection(ora)
    assert (cnt[:, FEET] == [[1023], [1022], [1021], [516]]).all(), cnt[:, FEET]
    np.testing.assert_array_equal(en[:, FEET].all(1), [False, True, True, True])
    ora.step(np.zeros((4, 1), np.float32))
    cnt, en = oracle_protection(ora)
    np.testing.assert_array_equal(en[:, FEET].any(1), [False, False, False, True])


# ---------------------------------------------------------------------------------------------------------------- GPU
LEG_CONFIGS = [(s, t, b) for s in LEG_SCENARIOS for t in ("plane", "random") for b in BUILDS_OF["base"]]
ARM_CONFIGS = [(s, t, b) for s in ARM_SCENARIOS for t in ("plane", "random") for b in BUILDS_OF["arm"]]
CONFIGS = LEG_CONFIGS + ARM_CONFIGS
IDS = ["-".join(c) for c in CONFIGS]
TIES = 2
EXACT_CONFIGS = [c for c in CONFIGS if c[0] in ("standup", "arm-standup")]
EXACT_IDS = ["-".join(c) for c in EXACT_CONFIGS]


def _assert_protection(env, ora, what, budget=0):
    """Enabled bits equal the oracle's; at most `budget` counters differ.  -> (counters, enabled, differing counters)."""
    cnt, en = protection(env)
    ocnt, oen = oracle_protection(ora)
    np.testing.assert_array_equal(en, oen, err_msg=f"enabled bits, {what}")
    bad = int((cnt != ocnt).sum())
    assert bad <= budget, (what, bad, np.argwhere(cnt != ocnt)[:8], cnt[cnt != ocnt][:8], ocnt[cnt != ocnt][:8])
    return cnt, en, bad


@pytest.mark.gpu
@pytest.mark.parametrize("name,terrain,build", EXACT_CONFIGS, ids=EXACT_IDS)
def test_shutdown_on_the_exact_substep(monkeypatch, name, terrain, build):
    """One control step = one physics sub-step (control_time_step 1 ms, action_repeat 1; limit floor(1 / dt) = 1000): seeded
    envs start their counters at 1000 - s, s = 0 ... 4, so their motors switch off on sub-steps 1 ... 5.  After every one of 8
    sub-steps, run from the oracle's physical state (the protection words are never re-synchronised), the enabled bits and the
    counters equal the oracle's, and q / pos keep test_one_step_is_tight's rounding-level bounds (a motor cut one sub-step early
    or late moves its joint far more).  Measured on an H100 over the 296 samples of a configuration (the builds of a terrain agree
    bit for bit): q p90 2.0e-7 / max 3.7e-7 rad on flat ground, 1.9e-6 / 4.3e-6 on the heightfield; pos max 1.1e-8 m; 117-200
    motors off after the fifth sub-step."""
    env, extra = _gpu_env(name, terrain, build, monkeypatch, **SUB)
    task, sig = SCENARIOS[name][:2]
    ora, rng = _prepare(name, terrain, env, **extra)
    mark = SCENARIOS[name][2]
    motors = range(12, 18) if mark == "arm" else range(12)
    for i in np.nonzero(SEEDED)[0]:
        for m in motors:
            ora.env(i).overheat[m] = 1000 - (i % 5)
    sync(env, ora, protection=True)
    b = bound(task, sig)
    eq, ep, offs = [], [], []
    for k in range(8):
        sync(env, ora)
        a = rng.uniform(-b, b, size=(N, env.action_dim)).astype(np.float32)
        env.step(a)
        assert launched(env) == BUILDS[build], launched(env)
        ora.step(a)
        _, en, _ = _assert_protection(env, ora, f"sub-step {k}")
        offs.append((~en).sum())
        q, p = state_errors(env, ora)
        eq.append(q); ep.append(p)
    eq, ep = np.concatenate(eq), np.concatenate(ep)
    print("exact sub-step: motors off after each sub-step", offs, "q (p90, max)", np.percentile(eq, 90), eq.max(),
          "pos (p90, max)", np.percentile(ep, 90), ep.max())
    assert offs[0] > 0 and offs[-1] > offs[0]                  # shutdowns on the first and on later sub-steps
    t90 = 2e-3 if mark == "arm" else 2e-5
    assert np.percentile(eq, 90) < t90 and eq.max() < 3e-3, (np.percentile(eq, 90), eq.max())
    assert np.percentile(ep, 90) < (2e-4 if mark == "arm" else 2e-6), np.percentile(ep, 90)
    assert env.check_errors() == 0
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,terrain,build", CONFIGS, ids=IDS)
def test_shutdowns_in_the_task_configuration(monkeypatch, name, terrain, build):
    """The task configuration (5 or 6 sub-steps per control step), 15 control steps of random actions after the seeding, each from
    the oracle's physical state and protection words: after every step the enabled bits and the counters equal the oracle's.  Over
    the run the switched-off motors are relieved (counter back to 0, motor still off) or stay hot until their counter saturates at
    1023; on the arm, the arm's enabled bits survive store_lane's write of the flags word.
    The motor model's torque curve passes through 2.45 N m at 30 A, so a motor whose current crosses 30 A can sit on the threshold
    within the fp32 / fp64 difference: measured on an H100, one (env, motor, step) sample of the 6660 of a gallop configuration
    (|torque| 2.4499974 N m in the oracle, counted hot by the kernel), none in any other configuration.  Counters may differ in
    TIES samples per run; enabled bits never."""
    env, extra = _gpu_env(name, terrain, build, monkeypatch)
    task, sig = SCENARIOS[name][:2]
    ora, rng = _prepare(name, terrain, env, **extra)
    b = bound(task, sig)
    saturated = relieved = ties = 0
    for k in range(15):
        sync(env, ora, protection=True)
        a = rng.uniform(-b, b, size=(N, env.action_dim)).astype(np.float32)
        _, _, dg, _ = env.step(a)
        assert launched(env) == BUILDS[build], launched(env)
        _, _, dc = ora.step(a)
        np.testing.assert_array_equal(dg, dc, err_msg=f"done, step {k}")
        cnt, en, bad = _assert_protection(env, ora, f"step {k}", TIES - ties)
        ties += bad
        saturated += ((cnt == 1023) & ~en).sum()
        relieved += ((cnt == 0) & ~en).sum()
        if dc.any():                                           # a fallen robot ends its episode: restart both sides' envs
            ora.reset(np.nonzero(dc)[0])
            env.reset(np.nonzero(dc)[0])
    print(f"{name}: (env, motor, step) samples switched off and saturated {saturated}, switched off and relieved {relieved}, "
          f"counters on a threshold tie {ties}")
    assert saturated > 0 or relieved > 0
    assert (env.check_errors() & 1) == 0
    env.close()


@pytest.mark.gpu
def test_batched_env_refuses_time_steps_the_counters_cannot_count():
    import rex_gym_b200 as R
    with pytest.raises(ValueError, match="overheat"):
        R.BatchedRexEnv(task="walk", num_envs=2, action_repeat=10)
    with pytest.raises(ValueError, match="overheat"):
        R.BatchedRexEnv(task="walk", num_envs=2, control_time_step=0.004886, action_repeat=5)
    R.BatchedRexEnv(task="walk", num_envs=2, **EDGE).close()


@pytest.mark.gpu
@pytest.mark.parametrize("build", ["small", "big", "sensor"])
def test_edge_rate_switches_off_on_count_1023(monkeypatch, build):
    """At 1 / dt = 1022.49 (floor 1022) the hold leaves 511 on standup's feet on both sides.  Feet seeded at 1018 reach 1023 -- the
    top of the 10-bit field -- on the last sub-step of the first control step and switch off there; feet seeded at 1017 / 1016 one
    and two sub-steps into the second.  After every step the GPU's enabled bits and counters equal the oracle's."""
    env, extra = _gpu_env("standup", "plane", build, monkeypatch, **EDGE)
    ora = make_oracle("standup", N, **_okw("standup", "plane", **extra)[1])
    env.reset(); ora.reset()
    _assert_protection(env, ora, "reset")
    assert (protection(env)[0][:, FEET] == 511).all()
    for i in range(N):
        if i % 4 != 3:                                         # every fourth env unseeded
            for m in FEET:
                ora.env(i).overheat[m] = 1016 + i % 3
    sync(env, ora, protection=True)
    rng = np.random.default_rng(3)
    offs = []
    for k in range(4):
        a = rng.uniform(-0.1, 0.1, size=(N, 1)).astype(np.float32)
        env.step(a)
        assert launched(env) == BUILDS[build], launched(env)
        ora.step(a)
        _, en, _ = _assert_protection(env, ora, f"step {k}")
        offs.append(int((~en[:, FEET]).any(1).sum()))
        sync(env, ora, protection=True)                        # the next step from the oracle's state (protection words included)
    seeded = sum(i % 4 != 3 for i in range(N))
    assert offs == [sum(i % 4 != 3 and i % 3 == 2 for i in range(N))] + [seeded] * 3, offs
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("build", ["small", "sensor"])
def test_reset_restores_the_snapshot_protection(monkeypatch, build):
    """After shutdowns (standup seeded at 996 on every motor, 3 control steps), rexsim_reset(idx) on half the envs restores the
    snapshot's words (500 on the feet, 0 elsewhere, every motor on) bit for bit against the oracle's reset, the other half keep
    theirs; those auto-reset through max_episode_steps 6 and get the snapshot's words as well; the next 5 steps track the oracle."""
    env, extra = _gpu_env("standup", "plane", build, monkeypatch, max_episode_steps=6, auto_reset=True)
    extra.pop("auto_reset")
    ora, rng = _prepare("standup", "plane", env, **extra)
    b = bound("standup", "ol")
    half = np.arange(0, N, 2)
    for k in range(11):
        if k == 0:
            sync(env, ora, protection=True)
        if k == 3:
            before = protection(env)
            assert (~before[1]).any()
            env.reset(half); ora.reset(half)
            cnt, en, _ = _assert_protection(env, ora, "rexsim_reset")
            assert (cnt[half][:, FEET] == 500).all() and (np.delete(cnt[half], FEET, 1) == 0).all() and en[half].all()
            keep = np.setdiff1d(np.arange(N), half)
            np.testing.assert_array_equal(cnt[keep], before[0][keep]); np.testing.assert_array_equal(en[keep], before[1][keep])
            sync(env, ora)                                   # the reset envs restart from the oracle's settle (chaotic fold-down)
        a = rng.uniform(-b, b, size=(N, 1)).astype(np.float32)
        _, _, dg, _ = env.step(a)
        _, _, dc = ora.step(a)
        np.testing.assert_array_equal(dg, dc, err_msg=f"done, step {k}")
        idx = np.nonzero(dc)[0]
        if len(idx):
            ora.reset(idx)
            if k == 5:
                assert set(idx) >= set(np.setdiff1d(np.arange(N), half))       # the auto-reset half
            cnt, en, _ = _assert_protection(env, ora, f"auto-reset, step {k}")
            assert en[idx].all() and (cnt[idx][:, FEET] == 500).all()
            sync(env, ora)
        else:
            _assert_protection(env, ora, f"step {k}")
    assert (env.check_errors() & 1) == 0
    env.close()


NATURAL = [("turn", "ik", dict()), ("walk", "ik", dict(target_position=2.0, backwards=False)), ("standup", "ol", dict()),
           ("gallop", "ol", dict(motor_kp_range=(0.8, 1.2), motor_kd_range=(0.01, 0.03)))]


@pytest.mark.gpu
@pytest.mark.parametrize("task,sig,kw", NATURAL, ids=[t + "-" + s for t, s, _ in NATURAL])
def test_natural_counting(task, sig, kw):
    """Unseeded counting: 30 control steps of random actions, each from the oracle's physical state and protection words; after
    each step the counters and enabled bits equal the oracle's, except (env, motor, step) samples where the applied torque sits on
    the 2.45 N m threshold within the fp32 / fp64 difference (budgeted like contact masks at 0.1 %).  Measured on an H100: no sample
    of the 13 320 per task differs; turn-ik, standup-ol and gallop-ol have 580, 3010 and 2610 hot samples, walk-ik none."""
    env, ora = make_env(task, N, signal_type=sig, seed=7, **kw), make_oracle(task, N, signal_type=sig, seed=7, **kw)
    env.reset(); ora.reset()
    rng = np.random.default_rng(8)
    b = bound(task, sig)
    bad = total = hot = 0
    for k in range(30):
        sync(env, ora, protection=True)
        a = rng.uniform(-b, b, size=(N, env.action_dim)).astype(np.float32)
        env.step(a); ora.step(a)
        cnt, en = protection(env)
        ocnt, oen = oracle_protection(ora)
        np.testing.assert_array_equal(en, oen)
        bad += int((cnt != ocnt).sum()); total += cnt.size; hot += int((ocnt > 0).sum())
    print(f"natural counting {task}-{sig}: {bad} of {total} samples differ, {hot} hot")
    assert (hot > 0 or task == "walk") and bad <= 0.001 * total, (bad, total, hot)
    env.close()


@pytest.mark.gpu
def test_standup_shutdown_with_pd_latency():
    """The sensor build with pd_latency 0.5 ms: the PD loop -- and with it the hot / not-hot decision -- reads a blend of the two
    newest history rows.  Standup at reset, feet seeded at 996: 10 control steps, each from the oracle's physical state and
    protection words (the history ring is each side's own), enabled bits and counters equal the oracle's after every step, and
    every seeded foot is off at the end.  Measured on an H100: q p90 5.2e-7, max 2.1e-6 rad; bounded here at 2e-5."""
    kw = dict(signal_type="ol", seed=31, pd_latency=0.0005)
    env, ora = make_env("standup", N, **kw), make_oracle("standup", N, **kw)
    env.reset(); ora.reset()
    _seed(ora, "standup", [996 if s else None for s in SEEDED])
    rng = np.random.default_rng(4)
    eq = []
    for k in range(10):
        sync(env, ora, protection=True)
        a = rng.uniform(-0.1, 0.1, size=(N, 1)).astype(np.float32)
        env.step(a)
        assert launched(env) == BUILDS["sensor"]
        ora.step(a)
        _assert_protection(env, ora, f"step {k}")
        eq.append(state_errors(env, ora)[0])
    eq = np.concatenate(eq)
    print("pd latency: q (p90, max)", np.percentile(eq, 90), eq.max())
    assert eq.max() < 2e-5, eq.max()
    assert (~protection(env)[1][SEEDED][:, FEET]).all()
    env.close()

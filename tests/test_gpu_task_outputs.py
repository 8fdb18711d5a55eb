"""The step kernel's task outputs -- reward term by term, termination, observation, motor command -- at rounding level.

GPU-vs-oracle trajectories diverge through contact chaos, so the suite's trajectory tests bound rewards at 5e-3 and commands at
5e-4: looser than the energy and shake terms of the reward (1e-5 to 1e-3 weighted).  Every output of a step is a pure function
of the state the step leaves behind, and the kernel stores that state: task_outputs.restate() restates the outputs in fp64 from
the kernel's own SoA words and sensor-history ring, so no divergence enters the comparison.

CPU: the restatement reproduces what the fp64 oracle's step returned (and its reward_done_obs), from the oracle's own state, for
every task and signal, both marks, normalize on and off, and the sensor configurations of test_gpu_parity.
GPU: every step-kernel instance the dispatcher can launch (twin.INSTANCES), 300
control steps of 37 envs without auto-reset, each output against the restatement of the kernel's words after every step, and
every motor command against the oracle's controller fed the kernel's pre-step task words.
"""
import math

import numpy as np
import pytest
import task_outputs as T
import twin
from twin import ARM_UNITS, BUILDS, INSTANCES, LAYOUT, NOISE, UNITS, bound, force_build, launched, make_env, make_oracle, row_id

EPS32 = float(np.finfo(np.float32).eps)
MARGIN = 1e-5          # envs this close to a threshold of their termination or a jump of their reward: counted, not compared


def _f32_tol(v):
    """Half an fp32 ulp of each value, and a floor: what rounding the oracle's fp64 outputs to float32 may move them."""
    return np.spacing(np.abs(np.asarray(v, np.float32))).astype(np.float64) + 1e-12


def _check_against_oracle_outputs(cfg, ora, rew, done, obs, label):
    r = T.restate(cfg, T.oracle_words(ora), T.oracle_ring(ora) if cfg.sensor else None)
    np.testing.assert_array_equal(r.done, done, err_msg=f"done {label}")
    bad = np.abs(r.reward - rew) > _f32_tol(rew)
    assert not bad.any(), f"reward {label}: env {np.argmax(bad)} {r.reward[bad][:3]} vs {rew[bad][:3]}, terms " \
        f"{ {k: v[np.argmax(bad)] for k, v in r.terms.items()} }"
    bad = np.abs(r.obs - obs) > _f32_tol(obs)
    assert not bad.any(), f"obs {label}: {np.argwhere(bad)[:4]} {r.obs[bad][:4]} vs {obs[bad][:4]}"
    return r


def _check_reward_done_obs(cfg, ora, label):
    """The oracle's reward_done_obs (the state's outputs, noise keyed on the current count, raw observation) in fp64."""
    raw = T.types.SimpleNamespace(**{**vars(cfg), "normalize": False})
    r = T.restate(raw, T.oracle_words(ora), T.oracle_ring(ora) if cfg.sensor else None, after_step=False)
    for i in range(ora.N):
        rr, dd, oo = ora.reward_done_obs(i)
        assert abs(r.reward[i] - rr) < 1e-12 * max(1.0, abs(rr)) and r.done[i] == dd, (label, i, r.reward[i], rr, r.done[i], dd)
        np.testing.assert_allclose(r.obs[i], oo, rtol=1e-12, atol=1e-12, err_msg=f"{label} env {i}")


def _cpu_run(task, sig, n, steps, seed, kw, act_scale=1.0):
    ora = make_oracle(task, n, seed=seed, **kw)
    cfg = T.cfg_of(ora)
    obs0 = ora.reset()
    r0 = T.restate(cfg, T.oracle_words(ora), T.oracle_ring(ora) if cfg.sensor else None, after_step=False)
    assert (np.abs(r0.obs - obs0) <= _f32_tol(obs0)).all(), "reset observation"
    rng = np.random.default_rng(seed)
    b = bound(task, sig)
    for k in range(steps):
        lim = 1.5 if kw.get("normalize") else b * act_scale
        a = rng.uniform(-lim, lim, size=(n, ora.A)).astype(np.float32)
        obs, rew, done = ora.step(a)
        _check_against_oracle_outputs(cfg, ora, rew, done, obs, f"step {k}")
        if k % 10 == 0:
            _check_reward_done_obs(cfg, ora, f"step {k}")
        idx = np.nonzero(done)[0]
        if kw.get("auto_reset") and len(idx):
            o = ora.reset(idx)
            r = T.restate(cfg, T.oracle_words(ora), T.oracle_ring(ora) if cfg.sensor else None, after_step=False)
            assert (np.abs(r.obs[idx] - o) <= _f32_tol(o)).all(), f"reset observation, step {k}"
    return ora


CPU_CASES = [(t, s, "base") for t, s in UNITS] + [(t, s, "arm") for t, s in ARM_UNITS]


@pytest.mark.parametrize("normalize", [False, True], ids=["raw", "normalize"])
@pytest.mark.parametrize("task,sig,mark", CPU_CASES, ids=["-".join(c) for c in CPU_CASES])
def test_restatement_reproduces_the_oracle_step(task, sig, mark, normalize):
    """CPU: 8 envs, 50 control steps of random actions (beyond +-1 when normalised), LimitDuration after 40: every reward,
    done and observation the oracle's step returned, restated from its post-step state within fp32 output rounding; every 10th
    step the oracle's reward_done_obs at 1e-12.  Walk runs with the constructor's backwards drawn and set."""
    kw = dict(signal_type=sig, mark=mark, normalize=normalize, max_episode_steps=40)
    if task == "walk":
        kw["backwards"] = True if normalize else None
    if (task, sig) == ("gallop", "ol"):
        kw.update(motor_kp_range=(0.8, 1.2), motor_kd_range=(0.01, 0.03))
    _cpu_run(task, sig, 8, 50, 3, kw, act_scale=2.0)


def _sensor_cases():
    from test_gpu_parity import SENSOR_CASES
    return SENSOR_CASES


@pytest.mark.parametrize("case", range(6))
def test_restatement_reproduces_the_oracle_with_the_sensor_model(case):
    """CPU: test_gpu_parity's SENSOR_CASES (control latencies 10.5-105 sub-steps back, PD latency, noise on every group, the
    arm, a heightfield with auto-reset): the history ring rebuilt from the oracle's deque in the kernel's layout, the noise keyed
    as the oracle keys it; 40 steps, every output within fp32 output rounding, the reset observations of auto-reset envs too."""
    task, sig, n, kw = _sensor_cases()[case]
    _cpu_run(task, sig, min(n, 8), 40, 5, dict(kw, signal_type=sig))


# ---- GPU sweep ---------------------------------------------------------------------------------------------------------------
SWEEP = [r + (k % 2 == 1,) for k, r in enumerate(INSTANCES)]        # every other row: normalize=True, actions beyond +-1


def _row_id(row):
    return row_id(row[:5]) + ("-norm" if row[5] else "")


def _sweep_config(task, sig, arm, terrain, build, norm):
    kw = dict(signal_type=sig, seed=17, max_episode_steps=250, normalize=norm)
    if arm:
        kw["mark"] = "arm"
    if (task, sig) == ("gallop", "ol"):
        kw.update(motor_kp_range=(0.8, 1.2), motor_kd_range=(0.01, 0.03))
    if task == "walk" and norm:
        kw["backwards"] = True                 # the forward objective flipped by the constructor
    if terrain == "random":
        kw.update(terrain_type="random", num_fields=4)
    if build == "sensor":
        kw.update(control_latency=0.0125, observation_noise_stdev=NOISE)
    else:
        kw["energy_weight"] = 0.0              # the observed torques are not state words: test_energy_term_* covers the term
    return kw


class _Counts:
    def __init__(self):
        self.margin = self.branch = self.samples = 0


def _obs_tolerance(cfg, r, sensor):
    """Per element: the fp32 rounding the kernel's observation may carry."""
    n = r.obs.shape[0]
    cond = 1.0 / np.sqrt(np.maximum(1.0 - r.pitch_arg ** 2, 1e-12))       # d asin / d x (roll's atan2 shares the cos(pitch))
    raw = np.zeros_like(r.obs)
    hi = np.array([T.TWO_PI + T.OBS_EPS] * 2 + [T.TWO_PI / cfg.dt + T.OBS_EPS] * 2 + [T.TWO_PI + T.OBS_EPS] * (r.obs.shape[1] - 4))
    v = (r.obs + 1) * hi - hi if cfg.normalize else r.obs
    raw[:, :2] = 8 * EPS32 * cond[:, None] + (8 * EPS32 * (np.abs(v[:, :2]) + 1) if sensor else 0)
    raw[:, 2:4] = 8 * EPS32 * (np.abs(v[:, 2:4]) + 1) if sensor else 0.0
    if r.obs.shape[1] > 4:
        raw[:, 4:] = np.spacing(np.float32(np.pi)) + abs(T.TWO_PI - float(np.float32(T.TWO_PI))) + \
            (8 * EPS32 * (np.abs(v[:, 4:]) + 1) if sensor else 0)
    if cfg.normalize:
        return raw / hi + 2 * EPS32
    return raw + np.zeros((n, 1))


def _compare_outputs(cfg, r, og, rg, dg, sensor, label, counts, rows=None):
    """Kernel outputs (og, rg, dg) against the restatement r of its words, on envs `rows` (default all)."""
    rows = np.ones(len(rg), bool) if rows is None else rows
    tol = _obs_tolerance(cfg, r, sensor)
    # the pitch branch of getEulerFromQuaternion: an env whose fp32 and fp64 sin arguments can straddle +-0.99999 is excused
    straddle = np.abs(np.abs(r.pitch_arg) - 0.99999) < 4e-7
    counts.branch += (straddle & rows).sum()
    ok_obs = rows & ~straddle
    if not sensor and not cfg.normalize:
        np.testing.assert_array_equal(og[ok_obs, 2:4], r.obs[ok_obs, 2:4], err_msg=f"base rates {label}")
    bad = (np.abs(og - r.obs) > tol) & ok_obs[:, None]
    assert not bad.any(), f"obs {label}: (env, column) {np.argwhere(bad)[:4].tolist()} kernel {og[bad][:4]} restated {r.obs[bad][:4]}"
    near = r.margin < MARGIN
    counts.margin += (near & rows).sum()
    counts.samples += rows.sum()
    cmp = rows & ~near
    d = dg != r.done
    assert not (d & cmp).any(), f"done {label}: envs {np.nonzero(d & cmp)[0]} kernel {dg[d & cmp]}"
    nterms = sum(t is not None for t in r.terms.values())
    bad = (np.abs(rg - r.reward) > 2e-6 * nterms) & cmp
    if bad.any():
        i = int(np.argmax(bad))
        raise AssertionError(f"reward {label}, env {i}: kernel {rg[i]:.9g} restated {r.reward[i]:.9g}; terms "
                             + ", ".join(f"{k} {v[i]:.3e}" for k, v in r.terms.items() if v is not None))


def _env_action(a, task, sig):
    """ClipAction + RangeNormalize._denormalize_action (wrappers.py:232-236,262-265) in float32, as the wrappers compute it on
    the float32 Box (gallop's inverted: low = +b, high = -b).  Clipped actions land exactly on the bound, where the controller's
    windows (t <= 0.8 + a, phi >= 0.99) compare against it: the env sees the float32 bound, not the decimal one."""
    b = np.float32(-bound(task, sig) if task == "gallop" else bound(task, sig))
    v = np.clip(np.asarray(a, np.float32), np.float32(-1), np.float32(1))
    return (v + np.float32(1)) / np.float32(2) * (np.float32(2) * b) + (-b)


def _oracle_command(ora, cfg, pre_f, pre_i, a, i):
    """The oracle's <task>._transform_action_to_motor_command for env i, on the kernel's pre-step task words."""
    L, e, dt = LAYOUT, ora.env(i), cfg.dt
    fl = int(pre_i[L.I_FLAGS, i])
    e.step_counter = int(pre_i[L.I_STEP, i])
    e.end_time = int(pre_i[L.I_ENDSTEP, i]) * dt
    e.gp_last_time = int(pre_i[L.I_GPLAST, i]) * dt * ora.cfg.gait_clock_scale
    e.gp_phi = float(np.array([pre_i[L.I_PHI_LO, i], pre_i[L.I_PHI_HI, i]], np.int32).view(np.float64)[0])
    e.gp_alpha = float(pre_f[L.F_ALPHA, i])
    e.target_position = e.target_value = float(pre_f[L.F_TARGET, i])
    e.target_orient = float(pre_f[L.F_TORIENT, i])
    e.goal_reached, e.is_terminating, e.stay_still = bool(fl & L.FL_GOAL), bool(fl & L.FL_TERMINATING), bool(fl & L.FL_STILL)
    e.backwards, e.clockwise, e.env_goal_reached = bool(fl & L.FL_BACKWARDS), bool(fl & L.FL_CLOCKWISE), bool(fl & L.FL_ENVGOAL)
    e.next_pose = (fl >> L.FL_POSE_SHIFT) & 7
    for k in range(3):
        e.pos[k] = float(pre_f[L.F_POS + k, i])
    for k in range(4):
        e.quat[k] = float(pre_f[L.F_QUAT + k, i])
    return ora.transform_action(a, i)


@pytest.mark.gpu
@pytest.mark.parametrize("row", SWEEP, ids=[_row_id(r) for r in SWEEP])
def test_task_outputs_restate_the_kernel_state(monkeypatch, row):
    """One step-kernel instance (forced as in test_gpu_builds, confirmed by rexsim_last_step_build every step): 37 envs, no
    auto-reset, 300 control steps of random actions (robots fall and keep stepping; LimitDuration from step 250).  After every
    step, against the restatement of the kernel's own words and ring: base rates equal to the F_ANGVEL words (1 ulp after
    normalisation), roll / pitch within a few fp32 ulps of the conditioning of asin, gallop's motor angles within an ulp, each
    reward term within 2e-6 (energy: sensor rows), done bit for bit -- envs within 1e-5 of a threshold counted, at most 1 %.
    Before every step the oracle's controller is fed the kernel's task words: all motor commands within 1e-5 rad (the sensed
    turn goal check reads the oracle's own history, so turn on the sensor build is left to test_gpu_builds)."""
    task, sig, arm, terrain, build, norm = row
    force_build(monkeypatch, build)
    n, steps = 37, 300
    kw = _sweep_config(*row)
    env, ora = make_env(task, n, **kw), make_oracle(task, n, **kw)
    cora = make_oracle(task, n, **dict(kw, normalize=False))       # the controller, handed the env's float32 action
    cfg = T.cfg_of(ora)
    sensor = build == "sensor"
    env.reset()
    rng = np.random.default_rng(23)
    lim = 1.5 if norm else bound(task, sig)
    counts, cmd_err = _Counts(), 0.0
    check_cmd = not (sensor and task == "turn")
    for k in range(steps):
        a = rng.uniform(-lim, lim, size=(n, env.action_dim)).astype(np.float32)
        pre_f, pre_i = env._state_f.cpu().numpy(), env._state_i.cpu().numpy()
        og, rg, dg, _ = env.step(a)
        assert launched(env) == BUILDS[build], launched(env)
        r = T.restate(cfg, T.kernel_words(env), T.kernel_ring(env))
        _compare_outputs(cfg, r, og, rg, dg, sensor, f"step {k}", counts)
        if check_cmd:
            cmd = env.last_command().cpu().numpy()
            ea = _env_action(a, task, sig) if norm else a
            oc = np.stack([_oracle_command(cora, cfg, pre_f, pre_i, ea[i], i) for i in range(n)], 1)
            cmd_err = max(cmd_err, float(np.abs(cmd - oc).max()))
            assert np.abs(cmd - oc).max() < 1e-5, f"command step {k}: {np.abs(cmd - oc).max():.2e} env {np.argmax(np.abs(cmd - oc).max(0))}"
    print(f"{_row_id(row)}: {counts.margin} env-steps within {MARGIN} of a threshold, {counts.branch} at the pitch branch, "
          f"of {counts.samples}; max command error {cmd_err:.2e}; done at the end {int(dg.sum())}")
    assert counts.margin <= 0.01 * counts.samples and counts.branch <= 0.01 * counts.samples
    assert (env.check_errors() & 1) == 0
    env.close()


AUTO_UNITS = UNITS + [("walk", "ik", "arm")]


@pytest.mark.gpu
@pytest.mark.parametrize("unit", AUTO_UNITS, ids=["-".join(u) for u in AUTO_UNITS])
def test_auto_reset_observation_restates_the_reset_words(unit):
    """Auto-reset on the sensor build (noise on every group, the snapshot's history ring copied in): 37 envs, episodes of 15
    steps, 60 steps.  The observation of an env the step finished is the first of its new episode: equal to the restatement of
    the post-reset words and ring (noise keyed on control step 0); the other envs' outputs as in the sweep."""
    task, sig = unit[:2]
    kw = dict(signal_type=sig, seed=19, max_episode_steps=15, auto_reset=True, control_latency=0.0125, observation_noise_stdev=NOISE)
    if len(unit) > 2:
        kw["mark"] = "arm"
    n = 37
    env, ora = make_env(task, n, **kw), make_oracle(task, n, **kw)
    cfg = T.cfg_of(ora)
    env.reset()
    rng = np.random.default_rng(29)
    counts, resets = _Counts(), 0
    for k in range(60):
        a = rng.uniform(-bound(task, sig), bound(task, sig), size=(n, env.action_dim)).astype(np.float32)
        og, rg, dg, _ = env.step(a)
        assert launched(env) == BUILDS["sensor"]
        w = T.kernel_words(env)
        r = T.restate(cfg, w, T.kernel_ring(env))
        np.testing.assert_array_equal(w["env_step"][dg], 0)
        resets += dg.sum()
        tol = _obs_tolerance(cfg, r, True)
        assert (np.abs(og - r.obs) <= tol)[dg].all(), f"reset observation, step {k}"
        _compare_outputs(cfg, r, og, rg, dg, True, f"step {k}", counts, rows=~dg)
    assert resets >= 2 * n
    assert (env.check_errors() & 1) == 0
    env.close()


# ---- placements on the branches -----------------------------------------------------------------------------------------------
# Each placement puts the 40 envs of a batch (right after the reset, from the oracle's settled state) at and either side of one
# threshold or branch of the outputs, through the physical state and the task words F_TARGET, I_FLAGS, I_ENDSTEP, I_ENVSTEP.
PLACE_N = 40
PITCH_SWITCH = math.pi / 2 - math.asin(0.99999)         # getEulerFromQuaternion's +-0.99999 branch, as a distance from +-pi/2
PLACEMENTS = [
    ("forward-0", "walk", "ik", dict(backwards=False)),          # the four forward branches and their edges
    ("forward-1", "walk", "ik", dict(backwards=True)),
    ("forward-drawn", "walk", "ik", dict()),
    ("up", "walk", "ik", dict(target_position=2.0)),             # up = 0.85 +- 1e-3
    ("up", "turn", "ik", dict()),
    ("roll-pitch-y", "gallop", "ol", dict(target_position=2.0)),  # roll 0.3, pitch 0.5, y 0.3, each +- 1e-3
    ("standup", "standup", "ol", dict()),                        # |pr| = 0.1 and z = 0.21
    ("turn-delay", "turn", "ik", dict()),                        # the stay-still timer crossing 1 s inside the step
    ("limit", "walk", "ik", dict(target_position=2.0, max_episode_steps=50)),  # I_ENVSTEP = max - 1
    ("pitch-branch", "walk", "ik", dict(target_position=2.0)),   # pitch +-(pi/2 - eps) across the branch
]


def _place(name, ora, task):
    """Put the oracle's (settled, just reset) envs at the placement `name`: state via set_state, task words via the structs."""
    n = ora.N
    d = np.linspace(-1e-3, 1e-3, n)
    for i in range(n):
        st, e = ora.state(i), ora.env(i)
        st["linvel"][:], st["angvel"][:] = 0, 0
        if name.startswith("forward"):
            tp = 1.0 + 0.5 * (i % 2)
            e.target_position = -tp if i % 4 >= 2 else tp                     # |target| is what the reward reads
            cx = [tp + 0.4, tp + 0.07, 0.02, 0.5 * tp, tp + 0.15 + d[i], 0.05 + d[i]][i % 6]
            sign = -1.0 if ora.cfg.backwards != 1 else 1.0                    # x = -cx, flipped by the constructor's backwards
            st["pos"][0] = sign * cx
            st["pos"][1] = 0.1 * d[i] * 1e3
        elif name == "up":
            st["quat"][:] = twin.quat(math.acos(0.85 + d[i]) * (1 if i % 2 else -1), 0.0, 0.3)
        elif name == "roll-pitch-y":
            k = i % 3
            st["quat"][:] = twin.quat(0.3 + d[i] if k == 0 else 0.0, (0.5 + d[i]) * (1 if i % 2 else -1) if k == 1 else 0.0, 0.0)
            if k == 2:
                st["pos"][1] = 0.3 + d[i]
        elif name == "standup":
            if i % 2:
                st["pos"][2] = 0.21 + d[i]
            else:
                st["pos"][:] = [0.05 * (1 if i % 4 else -1), 0.02 + d[i], 0.21 - 0.03]      # l1 = 0.1 + d
        elif name == "turn-delay":
            e.stay_still, e.goal_reached, e.is_terminating = 1, 1, 1
            e.step_counter = 2000
            e.end_time = (2000 - 1000 + 4 - i % 10) * ora.cfg.sim_dt           # t - end_time = 0.996 .. 1.005 s
        elif name == "limit":
            e.env_step_counter = e.limit_step = ora.cfg.max_episode_steps - 1 - i % 2
        elif name == "pitch-branch":
            eps = PITCH_SWITCH * (1 + np.linspace(-0.02, 0.02, n)[i])
            st["quat"][:] = twin.quat(0.2, (math.pi / 2 - eps) * (1 if i % 2 else -1), 0.1)
        if name in ("up", "roll-pitch-y", "pitch-branch"):
            st["pos"][2] = 0.5              # in the air: no contact turns the placed orientation during the step
        ora.set_state(i, st)


def _words_to_kernel(env, ora):
    """The oracle's placed state and task words into the batch: set_state, then raw edits of F_TARGET, I_FLAGS (enabled bits
    kept), I_STEP, I_ENDSTEP and I_ENVSTEP."""
    import torch
    L = LAYOUT
    twin.sync(env, ora)
    sf, si = env._state_f.cpu().numpy(), env._state_i.cpu().numpy()
    for i in range(ora.N):
        e = ora.env(i)
        sf[L.F_TARGET, i] = e.target_position
        si[L.I_FLAGS, i] = (si[L.I_FLAGS, i] & ~0xFF) | T.oracle_flags(e)
        si[L.I_STEP, i] = e.step_counter
        si[L.I_ENDSTEP, i] = int(round(e.end_time / ora.cfg.sim_dt))
        si[L.I_ENVSTEP, i] = e.env_step_counter
    env._state_f.copy_(torch.from_numpy(sf)); env._state_i.copy_(torch.from_numpy(si))


@pytest.mark.parametrize("name,task,sig,kw", PLACEMENTS, ids=[f"{p[0]}-{p[1]}" for p in PLACEMENTS])
def test_placements_restate_the_oracle(name, task, sig, kw):
    """CPU: every placement, one control step of the oracle: its outputs restated from its state within fp32 rounding."""
    ora = make_oracle(task, PLACE_N, signal_type=sig, seed=31, **kw)
    cfg = T.cfg_of(ora)
    ora.reset()
    _place(name, ora, task)
    a = np.random.default_rng(3).uniform(-1, 1, size=(PLACE_N, ora.A)).astype(np.float32) * 0.3 * bound(task, sig)
    obs, rew, done = ora.step(a)
    r = _check_against_oracle_outputs(cfg, ora, rew, done, obs, name)
    if name in ("up", "roll-pitch-y", "turn-delay", "limit"):
        assert 0 < r.done.sum() < PLACE_N                     # both sides of the threshold


@pytest.mark.gpu
@pytest.mark.parametrize("build", ["small", "big"])
@pytest.mark.parametrize("name,task,sig,kw", PLACEMENTS, ids=[f"{p[0]}-{p[1]}" for p in PLACEMENTS])
def test_placements_against_the_restatement_and_the_oracle(monkeypatch, build, name, task, sig, kw):
    """Every placement in the batch, one control step: the kernel's outputs against the restatement of its own words (as in
    the sweep; at the pitch branch only envs whose fp32 and fp64 sin arguments straddle +-0.99999 are excused), and against the
    oracle stepped from the same state and task words: rewards within 1e-4, done bit for bit on envs 1e-5 or more away from
    every threshold."""
    force_build(monkeypatch, build)
    env = make_env(task, PLACE_N, signal_type=sig, seed=31, energy_weight=0.0, **kw)      # as the sweep's non-sensor rows
    ora = make_oracle(task, PLACE_N, signal_type=sig, seed=31, energy_weight=0.0, **kw)
    cfg = T.cfg_of(ora)
    env.reset(); ora.reset()
    _place(name, ora, task)
    _words_to_kernel(env, ora)
    twin.sync(env, ora, protection=True)
    a = np.random.default_rng(3).uniform(-1, 1, size=(PLACE_N, env.action_dim)).astype(np.float32) * 0.3 * bound(task, sig)
    og, rg, dg, _ = env.step(a)
    assert launched(env) == BUILDS[build]
    oc, rc, dc = ora.step(a)
    r = T.restate(cfg, T.kernel_words(env), None)
    counts = _Counts()
    _compare_outputs(cfg, r, og, rg, dg, False, name, counts)
    far = r.margin > MARGIN
    np.testing.assert_array_equal(dg[far], dc[far], err_msg=f"done vs the oracle, {name}")
    np.testing.assert_allclose(rg, rc, atol=1e-4, err_msg=f"reward vs the oracle, {name}")
    print(f"{name} {task}: {int(dg.sum())} done, {counts.margin} within {MARGIN}, {counts.branch} at the pitch branch")
    assert counts.margin <= PLACE_N // 4
    env.close()


# ---- the energy term -----------------------------------------------------------------------------------------------------------
ENERGY_CASES = [("walk-ik", "walk", "ik", dict(target_position=2.0, backwards=False)),
                ("gallop-ol", "gallop", "ol", dict(target_position=2.0, motor_kp_range=(0.8, 1.2), motor_kd_range=(0.01, 0.03))),
                ("turn-ik-random", "turn", "ik", dict(terrain_type="random", num_fields=4)),
                ("standup", "standup", "ol", dict()),
                ("walk-ik-arm", "walk", "ik", dict(target_position=2.0, backwards=False, mark="arm"))]
ENERGY_ROWS = [(c, b) for c in ENERGY_CASES for b in ("small", "big") if not (b == "big" and "mark" in c[3])]


@pytest.mark.gpu
@pytest.mark.parametrize("case,build", ENERGY_ROWS, ids=[f"{c[0]}-{b}" for c, b in ENERGY_ROWS])
def test_energy_term_is_the_oracle_s(monkeypatch, case, build):
    """The energy term (rex_gym_env.py:535-537, -|tau_obs . qdot| dt, the arm's six motors included) where the observed torques
    are not state words: two batches that differ only in energy_weight (0 and 1) keep bit-identical state words after every
    step, so E = r1 - r0 is the kernel's term.  Against the oracle's after each of 20 control steps of one sub-step (twin.SUB)
    from the oracle's state (overheat protection synchronised): the 90th percentile of |E - E_oracle| / |E_oracle| within 1e-3 over the envs whose
    contact masks agree.  Turn and standup rewards have no energy term: E = 0 exactly.  The arm case displaces the arm 0.4 rad
    so its motors work."""
    import torch
    name, task, sig, kw = case
    force_build(monkeypatch, build)
    n = 37
    kw = dict(kw, **twin.SUB)          # one sub-step per control step: the physics agrees at rounding level after it
    envs = [make_env(task, n, signal_type=sig, energy_weight=wt, seed=37, **kw) for wt in (0.0, 1.0)]
    ora = make_oracle(task, n, signal_type=sig, seed=37, **kw)
    for e in envs:
        e.reset()
    ora.reset()
    if kw.get("mark") == "arm":
        for i in range(n):
            st = ora.state(i)
            st["q"][12:] += 0.4
            ora.set_state(i, st)
    md = [ora.model.motor_dof[m] for m in range(ora.nm)]
    rng = np.random.default_rng(41)
    rel, arm_share = [], []
    for k in range(20):
        for e in envs:
            twin.sync(e, ora, protection=True)
        a = rng.uniform(-bound(task, sig), bound(task, sig), size=(n, envs[0].action_dim)).astype(np.float32)
        r0, r1 = (e.step(a)[1] for e in envs)
        for e in envs:
            assert launched(e) == BUILDS[build]
        assert torch.equal(envs[0]._state_f, envs[1]._state_f) and torch.equal(envs[0]._state_i, envs[1]._state_i), k
        ora.step(a)
        E = r1.astype(np.float64) - r0
        if task in ("turn", "standup"):
            np.testing.assert_array_equal(r1, r0)
            continue
        tau = np.array([ora.env(i).tau_obs[:ora.nm] for i in range(n)])
        qd = np.array([[ora.env(i).qd[j] for j in md] for i in range(n)])
        Eo = -np.abs((tau * qd).sum(1)) * ora.cfg.sim_dt
        if ora.nm == 18:
            arm_share.append(np.abs((tau * qd)[:, 12:].sum(1)) / np.maximum(np.abs((tau * qd).sum(1)), 1e-12))
        same = envs[0].get_state()["contact_mask"] == np.array([ora.env(i).contact_mask for i in range(n)]) & \
            (0x7FFF if ora.nm == 18 else 0x1FF)
        rel.append((np.abs(E - Eo) / np.maximum(np.abs(Eo), 1e-6))[same])
    if rel:
        rel = np.concatenate(rel)
        print(f"{name} {build}: energy term relative error p90 {np.percentile(rel, 90):.2e} max {rel.max():.2e} over {len(rel)}")
        assert len(rel) > 0.8 * 20 * n and np.percentile(rel, 90) < 1e-3
    if arm_share:
        assert np.median(np.concatenate(arm_share)) > 0.01          # the arm's motors really enter the sum
    for e in envs:
        e.close()

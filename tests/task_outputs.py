"""The step kernel's task outputs restated in fp64 from the post-step state: reward term by term, termination, observation.

Not collected by pytest (like twin.py).  Every output of a control step (rex_gym_env.py:369-414) is a pure function of the state
the step leaves behind: the base pose and rates, the joint state, the task words (target, flags, control-step count) and, with
the sensor model on, the observation history the sub-steps pushed.  restate() reads that state as `words` and `ring`, taken from
the kernel's SoA buffers (kernel_words / kernel_ring) or from the oracle's env structs (oracle_words / oracle_ring), so a
comparison against it carries no trajectory divergence: it holds at fp32 rounding over any horizon.
"""
import math
import os
import re
import types

import numpy as np
from twin import LAYOUT

TASKS = ("walk", "gallop", "turn", "standup", "poses")
SIGNALS = ("ik", "ol")
OBS_EPS = 0.01                         # rex_gym_env.py:19 OBSERVATION_EPS
TWO_PI = 2 * math.pi


def _read_history_layout():
    """HW_* word indices of a sensor-history row and HIST_MAXLEN (the deque's maxlen), from the step kernel's header."""
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "rex_gym_b200", "csrc", "rexsim_kernel.cuh")
    src = re.sub(r"//[^\n]*|/\*.*?\*/", "", open(path).read(), flags=re.S)
    return types.SimpleNamespace(**{k: int(v) for k, v in re.findall(r"\b(HW_\w+|HIST_MAXLEN)\s*=\s*(\d+)", src)})


HW = _read_history_layout()


def q_word(m):
    """History-row word of motor m's angle; +3 / +6 (legs) or +6 / +12 (arm) are its rate and observed torque."""
    return 9 * (m // 3) + m % 3 if m < 12 else HW.HW_ARM + (m - 12)


def qd_word(m):
    return q_word(m) + (3 if m < 12 else 6)


def tau_word(m):
    return q_word(m) + (6 if m < 12 else 12)


# ---- configuration and state ---------------------------------------------------------------------------------------------
def cfg_of(ora):
    """The restatement's configuration, read from an oracle built with the same keywords as the batch (twin.make_oracle)."""
    c = ora.cfg
    tk = {v: k for k, v in zip(TASKS, range(5))}
    return types.SimpleNamespace(
        task=tk[c.task], sig=SIGNALS[c.signal], nm=ora.nm, dt=c.sim_dt, backwards=c.backwards,
        w=(c.w_distance, c.w_energy, c.w_drift, c.w_shake), normalize=bool(c.normalize), max_steps=c.max_episode_steps,
        seed=c.seed, env_offset=c.env_offset, latency=c.control_latency, sd=np.array(c.noise_stdev[:5]),
        sensor=c.control_latency > 0 or c.pd_latency > 0 or max(c.noise_stdev[:5]) > 0)


def kernel_words(env):
    """The state words restate() reads, from the kernel's SoA buffers (fp32 / int32 as stored); no observed torques (the kernel
    keeps them in the sensor history only)."""
    L, nm = LAYOUT, env.num_motors
    sf = env._state_f.cpu().numpy().astype(np.float64)
    si = env._state_i.cpu().numpy().astype(np.int64)
    jq = list(range(L.F_Q, L.F_Q + 12)) + list(range(L.F_AQ, L.F_AQ + nm - 12))
    jqd = list(range(L.F_QD, L.F_QD + 12)) + list(range(L.F_AQD, L.F_AQD + nm - 12))
    n = env.num_envs
    return dict(pos=sf[L.F_POS:L.F_POS + 3].T, quat=sf[L.F_QUAT:L.F_QUAT + 4].T, angvel=sf[L.F_ANGVEL:L.F_ANGVEL + 3].T,
                q=sf[jq].T, qd=sf[jqd].T, tau=None, target=sf[L.F_TARGET], flags=si[L.I_FLAGS] & 0xFFFFFFFF,
                env_step=si[L.I_ENVSTEP], reset_count=si[L.I_RESETCNT] & 0xFFFFFFFF,
                genv=np.arange(n) + env._cfg.env_offset)


def kernel_ring(env):
    """-> (ring [depth][words][N], push [N]) of the kernel's sensor history, or None with the sensor model off."""
    if env._ring is None:
        return None
    n = env.num_envs
    words = HW.HW_WORDS_ARM if env.num_motors == 18 else HW.HW_WORDS
    r = env._ring.cpu().numpy().astype(np.float64)
    return r.reshape(-1, words, n), env._state_i[LAYOUT.I_HPUSH].cpu().numpy().astype(np.int64)


def oracle_flags(e):
    L = LAYOUT
    return ((L.FL_GOAL if e.goal_reached else 0) | (L.FL_TERMINATING if e.is_terminating else 0) |
            (L.FL_STILL if e.stay_still else 0) | (L.FL_BACKWARDS if e.backwards else 0) |
            (L.FL_CLOCKWISE if e.clockwise else 0) | (L.FL_ENVGOAL if e.env_goal_reached else 0))


def oracle_words(ora):
    """The same words from the oracle's env structs (fp64), observed torques included."""
    E = [ora.env(i) for i in range(ora.N)]
    md = [ora.model.motor_dof[m] for m in range(ora.nm)]
    return dict(pos=np.array([e.pos[:] for e in E]), quat=np.array([e.quat[:] for e in E]),
                angvel=np.array([e.angvel[:] for e in E]), q=np.array([[e.q[j] for j in md] for e in E]),
                qd=np.array([[e.qd[j] for j in md] for e in E]), tau=np.array([e.tau_obs[:ora.nm] for e in E]),
                target=np.array([e.target_position for e in E]), flags=np.array([oracle_flags(e) for e in E]),
                env_step=np.array([e.env_step_counter for e in E]), reset_count=np.array([e.reset_count for e in E]),
                genv=np.arange(ora.N) + ora.cfg.env_offset)


def oracle_ring(ora):
    """The oracle's observation histories in the kernel's ring layout: [HIST_MAXLEN][words][N], push = the deque's length."""
    nm, n = ora.nm, ora.N
    ring = np.zeros((HW.HIST_MAXLEN, HW.HW_WORDS_ARM if nm == 18 else HW.HW_WORDS, n))
    push = np.zeros(n, np.int64)
    for i in range(n):
        h = ora.sensor_history(i)               # oracle row: q[nm], qd[nm], tau[nm], quat[4], rpy rate[3]
        push[i] = len(h)
        for k, row in enumerate(h):
            slot = len(h) - 1 - k
            for m in range(nm):
                ring[slot, q_word(m), i], ring[slot, qd_word(m), i], ring[slot, tau_word(m), i] = row[m], row[nm + m], row[2 * nm + m]
            ring[slot, HW.HW_BASE:HW.HW_BASE + 7, i] = row[3 * nm:3 * nm + 7]
    return ring, push


# ---- the reference's formulas, vectorised over envs -------------------------------------------------------------------------
def noise_unit(seed, genv, rc, step, site, comp):
    """Counter-based N(0, 1) of the sensor noise (rexsim_kernel.cuh noise_unit, oracle rexo_noise) in fp64, per env."""
    M = np.uint64(0xFFFFFFFFFFFFFFFF)
    g = np.uint64(0x9E3779B97F4A7C15)
    genv, rc, step = (np.asarray(x).astype(np.uint64) for x in (genv, rc, step))
    slot = (np.uint64(1024) + ((((step * np.uint64(8) + np.uint64(site)) * np.uint64(32) + np.uint64(comp)) << np.uint64(1))
                               & np.uint64(0xFFFFFFFF))) & np.uint64(0xFFFFFFFF)

    def draw(s):
        with np.errstate(over="ignore"):
            z = (np.uint64(seed) + g * (genv + np.uint64(1))) & M
            z ^= (rc << np.uint64(32)) | s
            z = z + g
            z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
            z = z ^ (z >> np.uint64(31))
        return (z >> np.uint64(32)) >> np.uint64(8)
    u1 = (draw(slot).astype(np.float64) + 1.0) / 16777216.0
    u2 = draw(slot + np.uint64(1)).astype(np.float64) / 16777216.0
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(TWO_PI * u2)


def euler(q):
    """pybullet.getEulerFromQuaternion (rex.py:426,439), its +-0.99999 branch included: -> roll, pitch, yaw, sin argument."""
    x, y, z, w = q.T
    sarg = -2.0 * (x * z - w * y)
    lo, hi = sarg <= -0.99999, sarg >= 0.99999
    roll = np.where(lo | hi, 0.0, np.arctan2(2 * (y * z + w * x), w * w - x * x - y * y + z * z))
    pitch = np.where(lo, -0.5 * math.pi, np.where(hi, 0.5 * math.pi, np.arcsin(np.clip(sarg, -1, 1))))
    yaw = np.where(lo, 2 * np.arctan2(x, -y), np.where(hi, 2 * np.arctan2(-x, y),
                                                       np.arctan2(2 * (x * y + w * z), w * w + x * x - y * y - z * z)))
    return roll, pitch, yaw, sarg


def quat_from_euler(r, p, y):
    """pybullet.getQuaternionFromEuler (rex.py:536 GetBaseOrientation)."""
    cr, sr, cp, sp, cy, sy = np.cos(r / 2), np.sin(r / 2), np.cos(p / 2), np.sin(p / 2), np.cos(y / 2), np.sin(y / 2)
    return np.stack([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy], 1)


def bottom_row(q):
    """Row 2 of pybullet.getMatrixFromQuaternion (rot_matrix[6:9]) for an unnormalised quaternion, as btMatrix3x3::setRotation."""
    x, y, z, w = q.T
    s = 2.0 / (x * x + y * y + z * z + w * w)
    return x * z * s - w * y * s, y * z * s + w * x * s, 1.0 - (x * x * s + y * y * s)


def map_pi(a):
    """MapToMinusPiToPi (rex.py:26-41)."""
    r = np.fmod(a, TWO_PI)
    return np.where(r >= math.pi, r - TWO_PI, np.where(r < -math.pi, r + TWO_PI, r))


class _Sensor:
    """Rex._GetDelayedObservation (rex.py:735-753) on a history ring and Rex._AddSensorNoise (rex.py:763-769)."""

    def __init__(self, cfg, w, ring):
        self.cfg, self.w = cfg, w
        self.ring, self.push = ring
        self.depth = self.ring.shape[0]
        self.n = int(cfg.latency / cfg.dt)
        self.a = (cfg.latency - self.n * cfg.dt) / cfg.dt
        self.cols = np.arange(self.ring.shape[2])

    def at(self, k, word):            # history[k]: slot (push - 1 - k) mod depth
        return self.ring[(self.push - 1 - k) % self.depth, word, self.cols]

    def delayed(self, word):
        ln = np.minimum(self.push, HW.HIST_MAXLEN)
        if self.cfg.latency <= 0:
            return self.at(0, word)
        n, a = self.n, self.a
        out = (1.0 - a) * self.at(np.minimum(n, ln - 1), word) + a * self.at(np.minimum(n + 1, ln - 1), word)
        out = np.where(n + 1 >= ln, self.at(ln - 1, word), out)
        return np.where(ln == 1, self.at(0, word), out)

    def noise(self, group, step, site, comp):
        sd = self.cfg.sd[group]
        if sd <= 0:
            return 0.0
        return sd * noise_unit(self.cfg.seed, self.w["genv"], self.w["reset_count"], step, site, comp)

    def quat(self, step, site):
        """Rex.GetBaseOrientation (rex.py:530-537): quaternion of the delayed orientation's Euler angles + noise."""
        r, p, y, _ = euler(np.stack([self.delayed(HW.HW_BASE + a) for a in range(4)], 1))
        return quat_from_euler(*(v + self.noise(3, step, site, a) for a, v in enumerate((r, p, y))))


def restate(cfg, w, ring=None, after_step=True):
    """The outputs of a control step from the state it left behind, in fp64.

    w: the words (kernel_words / oracle_words); ring: (history ring, push) with the sensor model on.  after_step: the outputs of
    RexGymEnv.step -- reward and termination keyed on the control step before its count went up, LimitDuration applied;
    False: the state's outputs as the oracle's reward_done_obs computes them (all keyed on the current count, no time limit).
    -> namespace: terms {name: weighted term [N]} (energy None without observed torques), reward (their sum), done [N],
       obs [N][O], margin [N] (distance of the env's state to the nearest threshold of its termination or discontinuity
       of its reward), pitch_arg [N] (getEulerFromQuaternion's sin argument of the observed orientation)."""
    task, n = cfg.task, len(w["pos"])
    S = _Sensor(cfg, w, ring) if cfg.sensor else None
    k_obs = w["env_step"]
    k_rew = w["env_step"] - 1 if after_step else w["env_step"]
    x, y, z = w["pos"].T
    inf = np.full(n, np.inf)
    rew_margin, done_margin = inf, inf
    terms = {}
    # ---- reward ----
    if task == "poses":
        terms["pose"] = np.ones(n)                                                       # poses_env.py:256-258
    elif task == "turn":
        terms["turn"] = 0.035 - np.abs(x) - np.abs(y)                                    # turn_env.py:362-367
    elif task == "standup":                                                              # standup_env.py:151-167
        l1 = np.abs(0.0 - x) + np.abs(0.0 - y) + np.abs(0.21 - z)
        pr = np.where(np.abs(l1) < 0.1, 1.0 - l1, -l1)
        terms["standup"] = np.where(z > 0.21, -1.0 - pr, pr)
        rew_margin = np.minimum(np.abs(l1 - 0.1), np.abs(z - 0.21))
    else:                                                                                # rex_gym_env.py:501-542
        wd, we, wdr, ws = cfg.w
        cx = -x
        if cfg.backwards == 1:           # `self._backwards`: the constructor's argument, not the direction drawn at reset
            cx = -cx
        tp = np.abs(w["target"])
        fwd = np.where(cx > tp + 0.15, tp - cx, np.where((tp <= cx) & (cx <= tp + 0.15), 1.0, np.where(cx <= 0.05, 0.0, cx / tp)))
        rew_margin = np.minimum(np.abs(cx - (tp + 0.15)), np.abs(cx - 0.05))
        if S is not None:
            r6, r7, _ = bottom_row(S.quat(k_rew, 3))
            dot = sum((S.delayed(tau_word(m)) + S.noise(2, k_rew, 4, m)) * (S.delayed(qd_word(m)) + S.noise(1, k_rew, 5, m))
                      for m in range(cfg.nm))
        else:
            r6, r7, _ = bottom_row(w["quat"])
            dot = None if w["tau"] is None else (w["tau"] * w["qd"]).sum(1)
        terms["fwd"] = fwd * wd
        terms["energy"] = None if dot is None else -np.abs(dot) * cfg.dt * we
        terms["drift"] = -np.abs(y) * wdr
        terms["shake"] = -np.abs(1 * r6 + 1 * r7) * ws
    reward = sum(t for t in terms.values() if t is not None)
    # ---- termination ----
    envgoal = (w["flags"] & LAYOUT.FL_ENVGOAL) != 0
    if task in ("walk", "turn"):                                                         # rex_gym_env.py:485-495
        up = bottom_row(S.quat(k_rew, 6) if S is not None else w["quat"])[2]
        done = (up < 0.85) | envgoal
        done_margin = np.abs(up - 0.85)
    elif task == "poses":
        done = np.zeros(n, bool)                                                         # poses_env.py:259-265
    else:                                                                                # gallop_env.py:315-329, standup_env.py:136-149
        roll, pitch, _, _ = euler(w["quat"])
        fallen = (np.abs(roll) > 0.3) | (np.abs(pitch) > 0.5)
        done_margin = np.minimum(np.abs(np.abs(roll) - 0.3), np.abs(np.abs(pitch) - 0.5))
        if task == "standup":
            done = fallen
        else:
            done = fallen | envgoal | (y > 0.3)
            done_margin = np.minimum(done_margin, np.abs(y - 0.3))
    if after_step and cfg.max_steps > 0:                                                 # LimitDuration (wrappers.py:141-166)
        done = done | (w["env_step"] >= cfg.max_steps)
    # ---- observation (walk_env.py:356-362, gallop_env.py:349-356) ----
    if S is not None:
        roll, pitch, _, sarg = euler(np.stack([S.delayed(HW.HW_BASE + a) for a in range(4)], 1))
        roll, pitch = roll + S.noise(3, k_obs, 0, 0), pitch + S.noise(3, k_obs, 0, 1)
        rates = [S.delayed(HW.HW_BASE + 4) + S.noise(4, k_obs, 1, 0), S.delayed(HW.HW_BASE + 5) + S.noise(4, k_obs, 1, 1)]
    else:
        roll, pitch, _, sarg = euler(w["quat"])
        rates = [w["angvel"][:, 0], w["angvel"][:, 1]]
    cols = [roll, pitch] + rates
    hi = [TWO_PI + OBS_EPS] * 2 + [TWO_PI / cfg.dt + OBS_EPS] * 2
    if task == "gallop":
        for m in range(12):
            a = S.delayed(q_word(m)) + S.noise(0, k_obs, 2, m) if S is not None else w["q"][:, m]
            cols.append(map_pi(a))
            hi.append(TWO_PI + OBS_EPS)
    obs = np.stack(cols, 1)
    if cfg.normalize:                                      # RangeNormalize._normalize_observ (wrappers.py:238-242), Box +-hi
        hi = np.array(hi)
        obs = 2 * (obs + hi) / (2 * hi) - 1
    return types.SimpleNamespace(terms=terms, reward=reward, done=done, obs=obs, margin=np.minimum(rew_margin, done_margin),
                                 rew_margin=rew_margin, done_margin=done_margin, pitch_arg=sarg)

"""A GPU batch and its fp64 oracle twin, as the GPU-vs-oracle tests build, synchronise and compare them.

Not collected by pytest (like render_oracle.py): the tests import what they need from here, and each keeps its own scenario,
its own bounds and its own asserts.
"""
import json
import math
import os
import re
import types

import numpy as np

TOL_Q, TOL_P = 1e-3, 1e-3             # north star: joint angles 1e-3 rad, base pose 1e-3 m
SUB = dict(control_time_step=0.001, action_repeat=1, solver_iterations=60)    # one control step = one physics sub-step
NOISE = (0.01, 0.05, 0.1, 0.02, 0.1)  # motor angle, velocity, torque, base rpy, rpy rate (SENSOR_NOISE_STDDEV order)
FOLDED = np.array([-0.42, -1.51, 2.70, 0.42, -1.51, 2.70, -0.44, -1.49, 2.69, 0.44, -1.49, 2.69])   # standup's settled legs
HERE = os.path.dirname(os.path.abspath(__file__))
ARM_REST = np.array(json.load(open(os.path.join(HERE, "golden", "constants_golden.json")))["arm_poses"]["rest"], np.float32)

# oracle contact groups, the same bits in the kernel's contact mask: 0 base / chassis; per leg 1 + 2l shoulder and leg boxes,
# 2 + 2l foot box and toe hull; 9-14 the arm links
TOES, UPPER, ARM_BITS = (2, 4, 6, 8), (1, 3, 5, 7), tuple(range(9, 15))
TOE_BITS, UPPER_BITS, ARM_MASK = (sum(1 << b for b in g) for g in (TOES, UPPER, ARM_BITS))
BODY_BITS = 1 | UPPER_BITS

# Early-out thresholds of the oracle's PGS around its 1e-7: where a result depends on which iteration first meets the early-out,
# the CUDA path is held to the range the oracle spans over these thresholds in its fp64 and fp32 builds.
HOLD_THRESHOLDS = (0.8e-7, 0.9e-7, 1e-7, 1.1e-7, 1.2e-7)

STATE_KEYS = ("pos", "quat", "linvel", "angvel", "q", "qd")       # what BatchedRexEnv.set_state carries

# step_kernel instance (CTA size, CTAs per SM, sensor) of each build the dispatcher can launch
BUILDS = {"small": (128, 1, 0), "big": (256, 4, 0), "sensor": (128, 1, 1)}
BUILDS_OF = {"base": ("small", "big", "sensor"), "arm": ("small", "sensor")}     # arm batches never take the big build

# ---- the step kernel's dispatch image --------------------------------------------------------------------------------
# (task, signal) of each compilation unit, in the order of c_units in rex_gym_b200/csrc/rexsim_kernel.cu
UNITS = [("walk", "ik"), ("walk", "ol"), ("gallop", "ik"), ("gallop", "ol"), ("turn", "ik"), ("turn", "ol"), ("standup", "ol"), ("poses", "ik")]
ARM_UNITS = [u for u in UNITS if u[0] != "gallop"]              # launch_step_ts: HAS_ARM
# every step_kernel instance the dispatcher can launch: (task, signal, arm, terrain, build), 8 x 2 x 3 + 6 x 2 x 2 = 72 rows
INSTANCES = [(t, s, arm, ter, b) for arm, mark, units in ((False, "base", UNITS), (True, "arm", ARM_UNITS)) for t, s in units
             for ter in ("plane", "random") for b in BUILDS_OF[mark]]


def row_id(row):
    """walk-ik-plane-small, standup-ol-arm-random-sensor."""
    task, sig, arm, terrain, build = row
    return "-".join([task, sig] + (["arm"] if arm else []) + [terrain, build])


def instance_config(row):
    """BatchedRexEnv / oracle keywords that reach the instance `row` (with force_build for the small and big builds)."""
    task, sig, arm, terrain, build = row
    kw = dict(signal_type=sig, seed=13, max_episode_steps=15)         # short episodes: every env runs the in-kernel reset twice
    if arm:
        kw["mark"] = "arm"
    if (task, sig) == ("gallop", "ol"):
        kw.update(motor_kp_range=(0.8, 1.2), motor_kd_range=(0.01, 0.03))
    if terrain == "random":
        kw.update(terrain_type="random", num_fields=4)
    if build == "sensor":
        kw["control_latency"] = 0.0125                                # a blend of two history rows, 12 sub-steps back
    return kw


def create_status(task, sig):
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


def _read_layout():
    """The SoA state word indices and flag bits (F_*, I_*, FL_*, NF, NI) of the step kernel's header."""
    path = os.path.join(HERE, "..", "rex_gym_b200", "csrc", "rexsim_kernel.cuh")
    src = re.sub(r"//[^\n]*|/\*.*?\*/", "", open(path).read(), flags=re.S)
    words = {k: int(v) for block in re.findall(r"\benum\s*\{(.*?)\}", src, re.S)
             for k, v in re.findall(r"\b((?:F|I|FL)_\w+|NF|NI)\s*=\s*(\d+)", block)}
    return types.SimpleNamespace(**words)          # a name the header lost raises AttributeError where it is read


LAYOUT = _read_layout()


# ---- the twin ------------------------------------------------------------------------------------------------------
def make_env(task, n, **kw):
    import rex_gym_b200 as R
    return R.BatchedRexEnv(task=task, num_envs=n, **kw)


def make_oracle(task, n, **kw):
    """The fp64 oracle of make_env(task, n, **kw), in BatchedRexEnv's keyword vocabulary (auto_reset has no oracle side: a test
    resets the oracle's done envs itself).  Oracle-only keywords pass through: fields, env_offset, residual_threshold, f32."""
    from oracle.oracle import OracleSim
    kw = dict(kw)
    sig = kw.pop("signal_type", "ik")
    ter = kw.pop("terrain_type", "plane")
    nf = kw.pop("num_fields", 0)
    kr, dr = kw.pop("motor_kp_range", None), kw.pop("motor_kd_range", None)
    kw.pop("auto_reset", None)
    return OracleSim(n, task, sig, terrain=ter, nfields=nf, kp_range=kr, kd_range=dr, **kw)


def bound(task, sig):
    """The task's action bound (RangeNormalize's Box)."""
    from rex_gym_b200.envs.batched_env import ACTION_BOUND
    return ACTION_BOUND[(task, sig)]


def force_build(monkeypatch, build):
    """Make the step launches that follow run `build` ("small" or "big"); None or "sensor": the dispatcher chooses (the sensor
    build is chosen by a sensor config, which the caller adds)."""
    if build in (None, "sensor"):
        monkeypatch.delenv("REXSIM_FORCE_BUILD", raising=False)
    else:
        monkeypatch.setenv("REXSIM_FORCE_BUILD", build)


def launched(env):
    """(CTA size, CTAs per SM, sensor) of the step_kernel instance env's last step launched (rexsim_last_step_build)."""
    import ctypes
    v = [ctypes.c_int32() for _ in range(3)]
    assert env._L.rexsim_last_step_build(env._h, *[ctypes.byref(x) for x in v]) == 0
    return tuple(x.value for x in v)


def solver_cost(env):
    """-> int32 [N]: the last step's solver cost per env, 64 per sub-step on the generic path + the PGS iterations."""
    import ctypes
    import torch
    from rex_gym_b200.envs.batched_env import _DevArray
    p = ctypes.c_void_p()
    assert env._L.rexsim_solver_cost(env._h, ctypes.byref(p)) == 0
    return torch.as_tensor(_DevArray(p.value, (env.num_envs,), "<i4", env), device="cuda").cpu().numpy().copy()


def sync(env, ora, idx=None, protection=False, window=None):
    """Set the physical state of envs `idx` (default: all) to the oracle's; the rest of the batch is written back unchanged.
    With `window`, oracle env i is batch env window + i (and `idx` counts oracle envs).  protection=True (whole batches only)
    also copies every env's overheat counters and motor-enabled bits, which set_state does not carry: a counter one sub-step
    off re-fires its event."""
    so = ora.states()
    if idx is not None or window is not None:
        idx = np.arange(ora.N) if idx is None else np.asarray(idx)
        st = env.get_state()
        for k in STATE_KEYS:
            st[k][idx + (window or 0)] = so[k][idx]
        so = st
    env.set_state(*(so[k] for k in STATE_KEYS))
    if protection:
        _sync_protection(env, ora)


def window_twin(task, n, w0, nw, steps, settled=False, **kw):
    """A batch of n envs and the oracle of its nw envs from w0 on (same global env ids: env_offset keys every reset draw), both
    reset, the window's draws checked bit for bit; settled=True starts the window from the oracle's settled state.
    -> (env, oracle, the window's reset observations from the batch and from the oracle, [steps][n][action_dim] seeded
        uniform actions in [-1, 1) on the device)."""
    import torch
    env, ora = make_env(task, n, **kw), make_oracle(task, nw, env_offset=w0, **kw)
    og, oc = env.reset()[w0:w0 + nw], ora.reset()
    assert_draws(env, ora, task, window=w0)
    if settled:
        sync(env, ora, window=w0)
    g = torch.Generator(device="cuda"); g.manual_seed(5)
    return env, ora, og, oc, torch.rand((steps, n, env.action_dim), device="cuda", generator=g) * 2 - 1


# ---- state words --------------------------------------------------------------------------------------------------------
# Packed overheat protection (rex.py:601-608): motor m's 10-bit saturating counter is field m % 3 of word I_OVH + m // 3 for the
# legs (m < 12) and of word I_OVHA + (m - 12) // 3 for the arm; its enabled bit is bit FL_ENABLED_SHIFT + m of I_FLAGS (legs
# 8-19, arm 20-25).  The oracle counts in an int32 that goes on past 1023 while a switched-off motor stays hot.
def _protection_word(m):
    return (LAYOUT.I_OVH + m // 3) if m < 12 else (LAYOUT.I_OVHA + (m - 12) // 3)


def _sync_protection(env, ora):
    si = env._state_i
    host = si.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    nm = ora.nm
    mask = (1 << (LAYOUT.FL_ENABLED_SHIFT + nm)) - (1 << LAYOUT.FL_ENABLED_SHIFT)
    for i in range(ora.N):
        e = ora.env(i)
        en, words = 0, {}
        for m in range(nm):
            w = _protection_word(m)
            words[w] = words.get(w, 0) | (min(int(e.overheat[m]), 1023) << (10 * (m % 3)))
            en |= (1 if e.enabled[m] else 0) << (LAYOUT.FL_ENABLED_SHIFT + m)
        for w, v in words.items():
            host[w, i] = v
        host[LAYOUT.I_FLAGS, i] = (host[LAYOUT.I_FLAGS, i] & ~mask) | en
    import torch
    si.copy_(torch.from_numpy(host.astype(np.uint32).view(np.int32)).to(si.device))


def protection(env):
    """-> (counters [N][nm], enabled [N][nm] bool) read back from the raw SoA state."""
    si = env._state_i.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    nm = env.num_motors
    cnt = np.stack([(si[_protection_word(m)] >> (10 * (m % 3))) & 1023 for m in range(nm)], 1)
    en = np.stack([(si[LAYOUT.I_FLAGS] >> (LAYOUT.FL_ENABLED_SHIFT + m)) & 1 for m in range(nm)], 1).astype(bool)
    return cnt, en


def oracle_protection(ora):
    """-> the oracle's (min(counter, 1023) [N][nm], enabled [N][nm] bool): what the kernel's saturating fields must hold."""
    cnt = np.array([[min(int(ora.env(i).overheat[m]), 1023) for m in range(ora.nm)] for i in range(ora.N)])
    en = np.array([[bool(ora.env(i).enabled[m]) for m in range(ora.nm)] for i in range(ora.N)])
    return cnt, en


def assert_draws(env, ora, task, window=None):
    """The integer bookkeeping after a step or a reset, bit for bit: step counters, reset count, field id, the draws of every
    reset (target, target and initial orientation, kp, kd, backwards, clockwise, the poses task's staged coordinate).  With
    `window`, oracle env i is batch env window + i."""
    L, E = LAYOUT, [ora.env(i) for i in range(ora.N)]
    w = slice(None) if window is None else slice(window, window + ora.N)
    sf, si = env._state_f.cpu().numpy()[:, w], env._state_i.cpu().numpy()[:, w]
    sg = env.get_state()
    eq = np.testing.assert_array_equal
    eq(sg["step_counter"][w], [e.step_counter for e in E])
    eq(sg["env_step_counter"][w], [e.env_step_counter for e in E])
    eq(si[L.I_RESETCNT], [e.reset_count for e in E])
    eq(si[L.I_FIELD], [e.field_id for e in E])
    eq(sf[L.F_TARGET], np.array([e.target_value if task == "poses" else e.target_position for e in E], np.float32))
    eq(sf[L.F_TORIENT], np.array([e.target_orient for e in E], np.float32))
    eq(sf[L.F_IORIENT], np.array([e.init_orient for e in E], np.float32))
    eq(sf[L.F_KP], np.array([e.kp for e in E], np.float32))
    eq(sf[L.F_KD], np.array([e.kd for e in E], np.float32))
    eq((si[L.I_FLAGS] & L.FL_BACKWARDS) != 0, [bool(e.backwards) for e in E])
    eq((si[L.I_FLAGS] & L.FL_CLOCKWISE) != 0, [bool(e.clockwise) for e in E])
    if task == "poses":
        eq((si[L.I_FLAGS] >> L.FL_POSE_SHIFT) & 7, [e.next_pose for e in E])


def state_errors(env, ora, window=None):
    """-> per oracle env, max |q - q_oracle| and max |pos - pos_oracle|.  With `window`, oracle env i is batch env window + i."""
    sg, so = env.get_state(), ora.states()
    w = slice(None) if window is None else slice(window, window + ora.N)
    return np.abs(sg["q"][w] - so["q"]).max(1), np.abs(sg["pos"][w] - so["pos"]).max(1)


def toe_masks(ora):
    """The oracle's contact masks over the 9 groups of the legged robot (same bit layout as the kernel's)."""
    return np.array([ora.env(i).contact_mask & 0x1FF for i in range(ora.N)])


# ---- quaternions (x, y, z, w) ------------------------------------------------------------------------------------------
def quat(r, p, y):
    cr, sr, cp, sp, cy, sy = (f(0.5 * a) for a in (r, p, y) for f in (math.cos, math.sin))
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy])


def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz])


def rot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


# ---- the generic solver path ---------------------------------------------------------------------------------------------
def limits(mark):
    """-> (lower, upper) joint limits of the model, [ndof] each."""
    from oracle.oracle import load_model
    m, _ = load_model(mark)
    return np.array([m.lower[j + 1] for j in range(m.ndof)]), np.array([m.upper[j + 1] for j in range(m.ndof)])


def violated(q, mark):
    """Violated joint limits per env as the fp32 kernel sees them: [N][ndof] bool."""
    lo, hi = limits(mark)
    q = np.asarray(q, np.float32)
    return (q - lo.astype(np.float32) <= 0) | (hi.astype(np.float32) - q <= 0)


def generic_path(mask, viol):
    """The generic-path predicate: a body or arm contact, two or more limits in one leg, more than three arm limits."""
    body = (mask & (BODY_BITS | ARM_MASK)) != 0
    legs = viol[:, :12].reshape(-1, 4, 3).sum(2).max(1) >= 2
    arm = viol[:, 12:].sum(1) > 3 if viol.shape[1] > 12 else np.zeros(len(viol), bool)
    return body | legs | arm


class IterationBand:
    """The oracles over HOLD_THRESHOLDS x {fp64, fp32}: factory(residual_threshold=, f32=) builds one of them."""

    def __init__(self, factory):
        self.oracles = [factory(residual_threshold=t, f32=f) for t in HOLD_THRESHOLDS for f in (False, True)]

    def reset(self):
        for o in self.oracles:
            o.reset()

    def start(self, states):
        for o in self.oracles:
            for i in range(o.N):
                o.set_state(i, {k: v[i] for k, v in states.items()})

    def step(self, a):
        """-> (lo, hi) per env: the range of the oracles' PGS iteration counts in this step."""
        its = []
        for o in self.oracles:
            o.step(a)
            its.append([o.env(i).solver_iters for i in range(o.N)])
        return np.min(its, 0), np.max(its, 0)


def compare_substeps(env, ora, band, start, build, labels, exception=None, steps=30):
    """`steps` single sub-steps (SUB) of random actions inside walk-ik's bound, the oracle and the band started at `start` and the
    CUDA state re-synchronised to the oracle before each.  Asserted per sub-step: the launched build; every contact group equals
    the oracle's, except where exception(oracle state, env, differing groups) accepts the difference; on the envs whose masks
    agree, the solver path (solver_cost // 64) is the oracle's generic_path predicate.
    -> (q errors, pos errors, PGS iteration counts outside the band on envs whose masks agree, generic-path samples, excused
        mask differences, error flags [steps][N])."""
    n = ora.N
    for i in range(n):
        ora.set_state(i, {k: v[i] for k, v in start.items()})
    full = 0x7FFF if env.mark == "arm" else 0x1FF
    rng = np.random.default_rng(7)
    eq, ep, flags, off_band, generic_steps, excused = [], [], [], 0, 0, 0
    for k in range(steps):
        sync(env, ora)
        so = ora.states()
        band.start(so)
        viol = violated(so["q"], env.mark)
        a = rng.uniform(-0.4, 0.4, size=(n, env.action_dim)).astype(np.float32)
        env.step(a)
        assert launched(env) == BUILDS[build], launched(env)
        ora.step(a)
        lo, hi = band.step(a)
        cost, gm = solver_cost(env), env.get_state()["contact_mask"] & full
        flags.append(env.error_flags().cpu().numpy())
        mask = np.array([ora.env(i).contact_mask for i in range(n)]) & full
        same = gm == mask
        for i in np.nonzero(~same)[0]:
            groups = [g for g in range(15) if ((gm[i] ^ mask[i]) >> g) & 1]
            assert exception is not None and exception(so, i, groups), \
                f"contact mask, sub-step {k}, env {i} {labels[i]}: {bin(gm[i])} vs {bin(mask[i])}"
            excused += 1
        gen = generic_path(mask, viol)
        np.testing.assert_array_equal((cost >= 64)[same], gen[same], err_msg=f"solver path, sub-step {k}")
        generic_steps += gen.sum()
        off_band += (((cost % 64 < lo) | (cost % 64 > hi)) & same).sum()
        q, p = state_errors(env, ora)
        eq.append(q); ep.append(p)
    return np.concatenate(eq), np.concatenate(ep), off_band, generic_steps, excused, np.array(flags)


def compare_control_steps(env, ora, start, build, labels, q90, p90, qmax, pmax, steps=20, every=5):
    """`steps` control steps of random actions inside walk-ik's bound from the oracle started at `start`, the CUDA state
    re-synchronised to the oracle every `every`.  Asserted per step: the launched build, finite outputs and state, the 90th
    percentile of the envs' q / pos errors below q90 / p90 and none above qmax / pmax.
    -> (q errors, pos errors, error flags [steps][N])."""
    n = ora.N
    for i in range(n):
        ora.set_state(i, {k: v[i] for k, v in start.items()})
    rng = np.random.default_rng(9)
    eqs, eps_, flags = [], [], []
    for k in range(steps):
        if k % every == 0:
            sync(env, ora)
        a = rng.uniform(-0.4, 0.4, size=(n, env.action_dim)).astype(np.float32)
        og, rg, _, _ = env.step(a)
        assert launched(env) == BUILDS[build], launched(env)
        ora.step(a)
        assert np.isfinite(og).all() and np.isfinite(rg).all()
        flags.append(env.error_flags().cpu().numpy())
        assert all(np.isfinite(v).all() for v in env.get_state().values())
        eq, ep = state_errors(env, ora)
        eqs.append(eq); eps_.append(ep)
        assert np.percentile(eq, 90) < q90 and np.percentile(ep, 90) < p90, f"step {k}: {np.percentile(eq, 90):.2e} {np.percentile(ep, 90):.2e}"
        assert eq.max() < qmax and ep.max() < pmax, f"step {k}: {eq.max():.2e} {ep.max():.2e} in {labels[int(np.argmax(eq))]}"
    return np.concatenate(eqs), np.concatenate(eps_), np.array(flags)


# ---- one control step from a synchronised state ------------------------------------------------------------------------------
def one_step_is_tight(task, sig, kw, bound):
    """30 single control steps of random actions inside +-bound, each from the oracle's state: rounding-level agreement."""
    n = 32
    env, ora = make_env(task, n, signal_type=sig, **kw), make_oracle(task, n, signal_type=sig, **kw)
    env.reset(); ora.reset()
    rng = np.random.default_rng(2)
    bad = 0
    for k in range(30):
        a = rng.uniform(-bound, bound, size=(n, env.action_dim)).astype(np.float32)
        sync(env, ora)
        env.step(a); ora.step(a)
        dq, dp = state_errors(env, ora)
        # 5 sub-steps from identical states: rounding level, except envs where a discrete event (a contact or limit row
        # switching on one sub-step apart) falls inside the step
        # the arm's three limit rows sit exactly on their activation boundary (q hovers at the limit under the PD
        # pull), so whether a row exists in a given sub-step is itself rounding-sensitive: 2e-3 there
        t90 = 2e-3 if kw.get("mark") == "arm" else 2e-5
        assert np.percentile(dq, 90) < t90 and dq.max() < 3e-3, (np.percentile(dq, 90), dq.max())
        assert np.percentile(dp, 90) < (2e-4 if kw.get("mark") == "arm" else 2e-6)
        bad += (env.get_state()["contact_mask"] != toe_masks(ora)).sum()
    assert bad <= 0.01 * 30 * n
    env.close()

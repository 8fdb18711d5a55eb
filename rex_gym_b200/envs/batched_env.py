"""BatchedRexEnv -- host-side mirror of the reference's env/BatchEnv surface over the CUDA library.

Reference interface mirrored (same names, argument meaning, error behaviour):
  * BatchEnv.step / reset / __len__ / __getitem__ / close   rex_gym/agents/tools/batch_env.py:18-115
  * RexWalkEnv / RexReactiveEnv / RexTurnEnv constructor kwargs rex_gym/envs/gym/walk_env.py:31-50,
    gallop_env.py:43-63, turn_env.py:30-49 (+ num_envs, device, and the fused training wrappers)
  * gym ids RexWalk-v0 ... rex_gym/playground/__init__.py:17-57 via make()
One call = one kernel launch for all N environments; there is no CPU fallback.
"""
import collections
import ctypes as C
import functools
import math
import numbers

import numpy as np
import torch

from .. import _capi
from ..model_tables import (pack_model_tables, pack_render_tables, contact_breaking_distance, TOE_MARGIN, LINK_DAMPING,
                            MAX_COORDINATE_VELOCITY)
from ..terrain import make_random_fields
from .spaces import Box

TASKS = {"walk": 0, "gallop": 1, "turn": 2, "standup": 3, "poses": 4}
SIGNALS = {"ik": 0, "ol": 1}
TERRAINS = {"plane": 0, "random": 1}
MARKS = {"base": 12, "arm": 18}     # mark -> motors the robot carries (mark_constants.py:1; the arm adds six)
DEFAULT_URDF_VERSION = "default"
OBSERVATION_EPS = 0.01          # rex_gym/envs/rex_gym_env.py:19
ACTION_BOUND = {("walk", "ik"): 0.4, ("walk", "ol"): 0.01, ("gallop", "ik"): 0.4, ("gallop", "ol"): 0.3,
                ("turn", "ik"): 0.01, ("turn", "ol"): 0.01, ("standup", "ol"): 0.1, ("standup", "ik"): 0.1,
                ("poses", "ik"): 0.1, ("poses", "ol"): 0.1}
# action width per signal (ik, ol) and whether the observation carries the motor angles (the library's task_shape, which
# rexsim_action_dim / rexsim_obs_dim report; the constructor checks the two agree)
ACTION_DIM = {"walk": (2, 8), "gallop": (2, 4), "turn": (2, 2), "standup": (1, 1), "poses": (1, 1)}
OBSERVES_ANGLES = {"gallop"}

ERR_NONFINITE, ERR_JOINT_LIMIT, ERR_BODY_CONTACT, ERR_TILE_MISS, ERR_BAD_INDEX = 1, 2, 4, 8, 16
SENSOR_NOISE_STDDEV = (0.0, 0.0, 0.0, 0.0, 0.0)      # rex_gym/model/rex.py:22, default of rex_gym_env.py:61


_DevArray = _capi.DevArray       # the name tests/twin.py wraps the solver-cost buffer with


def _host_block_views(block, N, O):
    """numpy views of the block rexsim_step_host fills (include/rexsim.h): obs [N][O] f32 | reward [N] f32 | done [N] u8 | pad to
    4 bytes | int32 OR of the step's error bits | 8 scratch bytes."""
    views, at = [], 0
    for count, dtype in ((N * O, np.float32), (N, np.float32), (N, np.bool_), (1, np.int32)):
        at = (at + 3) & ~3
        nbytes = count * np.dtype(dtype).itemsize
        views.append(block[at:at + nbytes].view(dtype))
        at += nbytes
    assert at + 8 == block.size, "host block layout differs from rexsim_host_out_bytes()"
    return views[0].reshape(N, O), views[1], views[2], views[3]


def summarize_episodes(totals):
    """Episode totals [4] (BatchedRexEnv.episode_totals, or their sum over shards) -> the summary simulate() logs (one copy to
    the host).  The reference writes no summary when no episode ended (simulate.py:101-106): the means are None then."""
    count, nonfinite, score, length = totals.cpu().tolist()
    count = int(count)
    return dict(count=count, nonfinite=int(nonfinite), mean_score=score / count if count else None,
                mean_length=length / count if count else None)


MAX_FRAME_INDICES, MAX_FRAME_INDEX = 16, 64      # FRAMES_MAX_INDICES / FRAMES_MAX_CAPACITY of the step kernel


def check_frame_history(past_indices):
    """frame_history keyword -> list of ints (empty: off), refused as FrameHistory.__init__ refuses it (wrappers.py:108-109:
    KeyError without 0) and beyond what the kernels keep (ValueError), before any CUDA call."""
    if past_indices is None:
        return []
    idx = [int(i) for i in past_indices]
    if any(i != j for i, j in zip(idx, past_indices)):
        raise ValueError("frame_history takes integer past indices")
    if 0 not in idx:
        raise KeyError('Past indices should include 0 for the current frame.')
    if min(idx) < 0:
        raise ValueError("frame_history: past indices must be non-negative, got %r" % (idx,))
    if max(idx) == 0:
        raise ValueError("frame_history: the largest past index is the ring's capacity and must be positive")
    if len(idx) > MAX_FRAME_INDICES or max(idx) > MAX_FRAME_INDEX:
        raise ValueError("frame_history: at most %d past indices, each at most %d" % (MAX_FRAME_INDICES, MAX_FRAME_INDEX))
    return idx


def frame_space(low, high, past_indices, delta):
    """(low, high) of the observation Box through FrameDelta (wrappers.py:163-168: low - high, high - low) and FrameHistory
    (:116-125: the box repeated once per past index, flattened), in the Box's float32."""
    low, high = np.asarray(low, np.float32), np.asarray(high, np.float32)
    if delta:
        low, high = low - high, high - low
    if past_indices:
        low, high = np.tile(low, len(past_indices)), np.tile(high, len(past_indices))
    return low, high


# constructor keywords that also take one value per env (BatchEnv over separately built envs, batch_env.py:21-42); the block's
# row of each is the library's (rexsim_value_row)
TASK_VALUE_KEYWORDS = ("target_position", "backwards", "target_orient", "init_orient",
                       "base_y", "base_z", "base_roll", "base_pitch", "base_yaw")
MAX_GAIN_PAIRS = 64              # REXSIM_MAX_GAIN_PAIRS: the reset hold is settled once per distinct (motor_kp, motor_kd, pd_latency)
LATENCY_KEYWORDS = ("control_latency", "pd_latency")     # sensor latencies that also take one value per env
RATE_KEYWORDS = ("control_time_step", "action_repeat")   # the control rate, one value per env over one simulation time step
MAX_REPEAT_PAIRS = 8             # REXSIM_MAX_REPEAT_PAIRS: distinct (action_repeat, solver_iterations) pairs, one launch each
# every constructor keyword that takes one value per env
PER_ENV_KEYWORDS = (TASK_VALUE_KEYWORDS + ("motor_kp", "motor_kd") + LATENCY_KEYWORDS + RATE_KEYWORDS +
                    ("terrain_type", "task", "signal_type", "mark"))


def is_per_env(value):
    """A keyword value given per env: a list, tuple, numpy array or tensor with at least one dimension."""
    if isinstance(value, (np.ndarray, torch.Tensor)):
        return value.ndim > 0
    return isinstance(value, (list, tuple))


def task_value(name, value):
    """What the scalar keyword `name` means to the kernels (RexSimConfig): NaN = draw per reset, backwards -1 / 0 / 1."""
    if name == "target_position":            # `if not self._target_position` (walk_env.py:144, gallop_env.py:150)
        return float("nan") if not value else float(value)
    if name == "backwards":
        return -1 if value is None else int(bool(value))
    return float("nan") if value is None else float(value)


def env_entries(name, value, n, numeric=False, names=None):
    """The value of keyword `name`, a scalar or one entry per env (is_per_env) -> its n entries: the scalar repeated, or the
    per-env value with its shape checked.  numeric: float64 [n] on the host, None entries as NaN; otherwise a list, str
    entries as Python str.  A tensor is read on the host, unless the entries are names (`names`: what they are, for the
    refusal)."""
    if not is_per_env(value):
        return np.full(n, float(value)) if numeric else [value] * n
    if isinstance(value, torch.Tensor):
        if names:
            raise ValueError("%s: per-env entries are %s, not a tensor" % (name, names))
        value = value.detach().cpu().numpy()
    if numeric:
        a = np.asarray([np.nan if v is None else v for v in value] if isinstance(value, (list, tuple)) else value, np.float64)
    else:
        a = np.asarray(list(value) if isinstance(value, (list, tuple)) else value, dtype=object)
    if a.shape != (n,):
        raise ValueError("%s: expected one %s per env (%d), got shape %s" % (name, "value" if numeric else "entry", n, a.shape))
    return a if numeric else [str(v) if isinstance(v, str) else v for v in a]


def task_value_entries(name, value, n):
    """Per-env values of keyword `name` -> float32 [n], each entry meaning what the scalar means: NaN (or None) draws per reset
    (target_position 0 too, as the scalar), backwards entries are -1 (draw), 0 or 1."""
    a = env_entries(name, value, n, numeric=True)
    if name == "target_position":
        a = np.where(a == 0, np.nan, a)
    elif name == "backwards":
        a = np.where(np.isnan(a), -1.0, a)
        if not np.isin(a, (-1.0, 0.0, 1.0)).all():
            raise ValueError("backwards: per-env entries must be -1 (draw), 0 or 1")
    return a.astype(np.float32)


def check_env_values(num_envs, values, motor_kp, motor_kd, motor_kp_range=None, motor_kd_range=None):
    """The per-env constructor keywords, checked before any CUDA call.
    values: {keyword of TASK_VALUE_KEYWORDS: scalar or per-env}.  -> (None, None) when every keyword is a scalar; otherwise
    ({keyword: float32 [num_envs]} for all nine keywords (scalars repeated) or None, (kp, kd) float32 [num_envs] each or None)."""
    n = int(num_envs)
    per_env = {k: task_value_entries(k, v, n) for k, v in values.items() if is_per_env(v)}
    rows = None
    if per_env:
        rows = {k: per_env[k] if k in per_env else np.full(n, task_value(k, values.get(k)), np.float32) for k in TASK_VALUE_KEYWORDS}
    gains = None
    if is_per_env(motor_kp) or is_per_env(motor_kd):
        if motor_kp_range is not None or motor_kd_range is not None:
            raise ValueError("per-env motor_kp / motor_kd cannot be combined with motor_kp_range / motor_kd_range")
        kp, kd = (env_entries(k, v, n, numeric=True) for k, v in (("motor_kp", motor_kp), ("motor_kd", motor_kd)))
        kp, kd = kp.astype(np.float32), kd.astype(np.float32)
        if not (np.isfinite(kp).all() and np.isfinite(kd).all() and (kp >= 0).all() and (kd >= 0).all()):
            raise ValueError("motor_kp / motor_kd: per-env gains must be finite and non-negative")
        pairs = len(set(zip(kp.tolist(), kd.tolist())))
        if pairs > MAX_GAIN_PAIRS:
            raise ValueError("motor_kp / motor_kd: %d distinct (kp, kd) pairs, at most %d (the reset hold is settled once per "
                             "pair; motor_kp_range / motor_kd_range draw continuous gains)" % (pairs, MAX_GAIN_PAIRS))
        gains = (np.ascontiguousarray(kp), np.ascontiguousarray(kd))
    if gains is not None and rows is None:
        rows = {k: np.full(n, task_value(k, values.get(k)), np.float32) for k in TASK_VALUE_KEYWORDS}
    return rows, gains


def check_env_latencies(num_envs, control_latency, pd_latency, motor_kp=1.0, motor_kd=0.02, gains=None):
    """The per-env latency keywords, checked before any CUDA call.  gains: check_env_values' per-env (kp, kd) or None.
    -> None when both latencies are scalars; otherwise (control, pd) float64 [num_envs] each (a scalar repeated), the values
    rexsim_set_env_latencies takes (fp64, as the config's scalars: every env's terms are the scalar construction's)."""
    n = int(num_envs)
    if not (is_per_env(control_latency) or is_per_env(pd_latency)):
        return None
    lat = []
    for name, v in (("control_latency", control_latency), ("pd_latency", pd_latency)):
        a = env_entries(name, v, n, numeric=True)
        if not (np.isfinite(a).all() and (a >= 0).all()):
            raise ValueError("%s: per-env latencies must be finite and non-negative" % name)
        lat.append(np.ascontiguousarray(a, np.float64))
    kp, kd = gains if gains is not None else (np.full(n, motor_kp, np.float32), np.full(n, motor_kd, np.float32))
    settings = len(set(zip(kp.tolist(), kd.tolist(), lat[1].tolist())))
    if settings > MAX_GAIN_PAIRS:
        raise ValueError("pd_latency: %d distinct reset-hold settings (motor_kp, motor_kd, pd_latency), at most %d (the reset "
                         "hold reads the PD observation and is settled once per setting)" % (settings, MAX_GAIN_PAIRS))
    return tuple(lat)


def check_terrain(terrain_type):
    """One terrain_type value, refused before any CUDA call unless it is a built terrain."""
    if not isinstance(terrain_type, str) or terrain_type not in TERRAINS:
        raise ValueError("terrain_type %r: only 'plane' and 'random' are built (csv/png assets live in the "
                         "pybullet_data pip package)" % (terrain_type,))


def check_env_terrains(num_envs, terrain_type):
    """The terrain_type keyword, checked before any CUDA call: a scalar, or one entry per env (a list, tuple or ndarray), each
    'plane' or 'random'.  -> (scalar, None) for a scalar or an array whose entries are all equal (the scalar construction);
    (None, int32 [num_envs] of TERRAINS ids) for a batch of both terrains."""
    entries = env_entries("terrain_type", terrain_type, int(num_envs), names="the strings 'plane' / 'random'")
    for t in entries:
        check_terrain(t)
    if len(set(entries)) == 1:
        return entries[0], None
    return None, np.ascontiguousarray([TERRAINS[t] for t in entries], np.int32)


def check_env_repeats(num_envs, task, control_time_step, action_repeat, solver_iterations=None):
    """The control-rate keywords, checked before any CUDA call.  task: the task name, or one per env.  control_time_step and
    action_repeat: a scalar (None: each env's task's default, 6 ms / 6 for gallop and poses, 5 ms / 5 otherwise) or one entry
    per env (a list, tuple or ndarray).  Env e is built as if (control_time_step[e],
    action_repeat[e]) were the scalars, so every control_time_step[e] / action_repeat[e], in fp64 as rex_gym_env.py:173
    computes it, must be the one simulation time step: the observation space's rate bounds are 2 pi / time step, and the
    reference's BatchEnv refuses envs whose spaces differ.  solver_iterations: None (each env int(300 / action_repeat[e]),
    rex_gym_env.py:184) or a scalar for every env.
    -> (control_time_step, action_repeat, time step, None) for a scalar construction (all-equal arrays are one), else
    (control_time_step tuple, action_repeat tuple, time step, (action_repeat, solver_iterations) int32 [num_envs] each)."""
    n = int(num_envs)
    if is_per_env(solver_iterations):
        raise ValueError("solver_iterations takes one value for the batch (None: int(300 / action_repeat) per env)")
    long_step = [t in ("gallop", "poses") for t in (list(task) if is_per_env(task) else [task] * n)]

    def default(v, long, short):                 # a scalar None (or 0) takes each env's task's default
        if is_per_env(v) or v:
            return v
        return long if all(long_step) else short if not any(long_step) else [long if ls else short for ls in long_step]
    cts = env_entries("control_time_step", default(control_time_step, 0.006, 0.005), n)
    for v in cts:
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, numbers.Real) or not (math.isfinite(v) and v > 0):
            raise ValueError("control_time_step: %r is not a positive finite number of seconds" % (v,))
    rep = env_entries("action_repeat", default(action_repeat, 6, 5), n)
    for v in rep:
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, numbers.Integral) or v <= 0:
            raise ValueError("action_repeat: %r is not a positive integer" % (v,))
    cts, rep = [float(v) for v in cts], [int(v) for v in rep]
    steps = sorted({c / r for c, r in zip(cts, rep)})
    if len(steps) > 1:
        raise ValueError("control_time_step / action_repeat: the envs' simulation time steps differ (%s s); the observation "
                         "space's rate bounds are 2 pi / time step, so the spaces differ and the reference's BatchEnv refuses "
                         "the mix" % ", ".join(repr(t) for t in steps[:4]))
    if len(set(zip(cts, rep))) == 1:
        return cts[0], rep[0], steps[0], None
    iters = [solver_iterations or int(300 / r) for r in rep]                     # rex_gym_env.py:25,184
    pairs = len(set(zip(rep, iters)))
    if pairs > MAX_REPEAT_PAIRS:
        raise ValueError("action_repeat: %d distinct (action_repeat, solver_iterations) pairs, at most %d (each is one step "
                         "launch)" % (pairs, MAX_REPEAT_PAIRS))
    return tuple(cts), tuple(rep), steps[0], (np.ascontiguousarray(rep, np.int32), np.ascontiguousarray(iters, np.int32))


def task_spaces(task, signal_type, normalize, time_step, frames=None, frame_delta=False, num_motors=12):
    """(action_space, observation_space) of one (task, signal_type) env: the raw task spaces, or the wrapper-visible ones when
    the training wrappers are fused in, through the frame wrappers."""
    A = ACTION_DIM[task][SIGNALS[signal_type]]
    O = 4 + (num_motors if task in OBSERVES_ANGLES else 0)
    if normalize:
        action_space = Box(-np.inf * np.ones(A, np.float32), np.inf * np.ones(A, np.float32))   # ClipAction wrappers.py:257-260
        lo, hi = -np.ones(O, np.float32), np.ones(O, np.float32)                               # RangeNormalize :204-209
    else:
        ha = np.full(A, ACTION_BOUND[(task, signal_type)], np.float32)
        action_space = Box(ha, -ha) if task == "gallop" else Box(-ha, ha)                         # gallop_env.py:128-130
        ub = np.full(O, 2 * math.pi, np.float32)
        ub[2:4] = 2 * math.pi / time_step
        lo, hi = -(ub + OBSERVATION_EPS), ub + OBSERVATION_EPS
    return action_space, Box(*frame_space(lo, hi, frames, frame_delta))


def _same_box(a, b):
    """Exactly the same Box: shapes first (Box.__eq__ compares bounds by broadcasting only), then every bound."""
    return a.low.shape == b.low.shape and np.array_equal(a.low, b.low) and np.array_equal(a.high, b.high)


def _name_entries(name, value, names, n):
    """A task / signal_type keyword, scalar or per env -> a list of n names, each one of `names`."""
    entries = env_entries(name, value, n, names="names")
    for v in entries:
        if not isinstance(v, str) or v not in names:
            raise ValueError("unknown %s %r (have %s)" % (name, v, sorted(names)))
    return entries


def check_env_marks(num_envs, mark):
    """The mark keyword, checked before any CUDA call: a scalar, or one entry per env (a list, tuple or ndarray), each 'base'
    or 'arm'.  -> (scalar, None) for a scalar or an array whose entries are all equal (the scalar construction); (None,
    int32 [num_envs] of each env's motor count, 12 or 18) for a batch of both marks."""
    entries = env_entries("mark", mark, int(num_envs), names="the strings 'base' / 'arm'")
    if any(not isinstance(m, str) or m not in MARKS for m in entries):
        raise ValueError("mark must be 'base' or 'arm'")          # mark_constants.py:1
    if len(set(entries)) == 1:
        return entries[0], None
    return None, np.ascontiguousarray([MARKS[m] for m in entries], np.int32)


def check_env_tasks(num_envs, task, signal_type, time_step=0.001, normalize=False, frames=None, frame_delta=False, mark="base"):
    """The task and signal_type keywords, checked before any CUDA call: each a scalar or one entry per env (a list, tuple or
    ndarray).  Envs of several (task, signal_type) pairs, or of both marks (`mark`: a scalar or one entry per env), are one
    batch only when their spaces (task_spaces, at each env's own motor count) are the same, as the reference's BatchEnv
    requires (batch_env.py:36-43): e.g. turn ik with turn ol, standup with poses, under normalize walk ik with turn, and any
    task but gallop with and without the arm.  A gallop env with the arm in a batch of both marks is refused with the
    library's message.  -> (task, signal_type, None) for a scalar construction of the pair (all-equal pairs are one), else
    (tasks tuple, signals tuple, (task ids, signal ids) int32 [num_envs] each)."""
    n = int(num_envs)
    tasks = _name_entries("task", task, TASKS, n)
    signals = _name_entries("signal_type", signal_type, SIGNALS, n)
    marks = list(mark) if is_per_env(mark) else [mark] * n
    pairs = list(dict.fromkeys(zip(tasks, signals)))
    envs = list(dict.fromkeys(zip(tasks, signals, marks)))         # the distinct (task, signal_type, mark) of the batch
    if len(set(marks)) > 1 and any(t == "gallop" and m == "arm" for t, _, m in envs):
        raise ValueError("mark='arm' is built for every task but gallop (its observation would carry the 18 motor angles)")
    spaces = {p: task_spaces(p[0], p[1], normalize, time_step, frames, frame_delta, MARKS[p[2]]) for p in envs}
    name = lambda p: "/".join(p if len(set(marks)) > 1 else p[:2])
    a0, o0 = spaces[envs[0]]
    for p in envs[1:]:
        a, o = spaces[p]
        if not (_same_box(o, o0) and _same_box(a, a0)):
            raise ValueError("All environments must use the same observation space. (%s: action %s, observation %s; %s: "
                             "action %s, observation %s%s)" % (name(envs[0]), a0, o0, name(p), a, o, "" if normalize else
                                                              "; normalize=True gives every task the same bounds"))
    if len(pairs) == 1:
        return pairs[0][0], pairs[0][1], None
    ids = (np.ascontiguousarray([TASKS[t] for t in tasks], np.int32), np.ascontiguousarray([SIGNALS[g] for g in signals], np.int32))
    return tuple(tasks), tuple(signals), ids


# The optional per-env device blocks besides the values block: the attribute that views it, its state_dict key, the noun and
# the entries named when a checkpoint's differ, the library call that hands it out (`depth`: it also reports an int32) and
# the view's rows and element type.  Checkpoints compare them in this order.
_EnvBlock = collections.namedtuple("_EnvBlock", "attr key noun entries call depth rows typestr")
_ENV_BLOCKS = (
    _EnvBlock("_marks", "env_marks", "marks", "marks", "rexsim_env_mark_buffers", False, 1, "|u1"),
    _EnvBlock("_tasks", "env_tasks", "tasks", "tasks or signals", "rexsim_env_task_buffers", False, 2, "|u1"),
    _EnvBlock("_repeats", "env_repeats", "control rates", "action repeats or solver iterations", "rexsim_env_repeat_buffers",
              False, 2, "<i4"),
    _EnvBlock("_terrain", "env_terrain", "terrains", "terrains", "rexsim_env_terrain_buffers", True, 1, "|u1"),
    _EnvBlock("_latency", "env_latency", "latencies", "latencies", "rexsim_env_latency_buffers", True, 2, "<f8"),
)


class _Info(object):
    """Stand-in for BatchEnv's `tuple(infos)`: info[i] == {'action': motor command of env i} of THE STEP THAT RETURNED IT
    (rex_gym_env.py:414).  The command block lives on the device and is overwritten by the next step, so the host copy is taken
    on first access; an access after the batch has stepped again raises instead of handing out the later step's commands.
    With final_observation=True, info[i] also carries gym TimeLimit's 'TimeLimit.truncated' on the steps where env i reached
    max_episode_steps, valued `not done` of the task (gym 0.17.1 wrappers/time_limit.py); its limit byte is copied with the
    commands."""

    def __init__(self, env):
        self._env, self._cmd, self._limit, self._at = env, None, None, env._nsteps

    def __len__(self):
        return len(self._env)

    def materialize(self):
        """Take the host copy now (one device sync + D2H copy of [N][num_motors] floats)."""
        if self._cmd is None:
            if self._env._nsteps != self._at:
                raise RuntimeError("info of step %d read after the batch advanced to step %d: call info.materialize() (or read "
                                   "info[i]) before the next step()" % (self._at, self._env._nsteps))
            self._cmd = self._env.last_command().t().contiguous().cpu().numpy()
            if self._env._final is not None:
                lim = self._env.limit_bytes()
                self._limit = lim.cpu().numpy() if isinstance(lim, torch.Tensor) else lim.copy()
        return self

    def __getitem__(self, i):
        cmd = self.materialize()._cmd[i]
        motors = getattr(self._env, "_env_motors", None)       # [N] motors of each env, per-env marks only
        info = {"action": cmd if motors is None else cmd[:motors[i]]}      # a base env of a batch of both marks: its 12
        if self._limit is not None and self._limit[i] & 1:
            info["TimeLimit.truncated"] = not bool(self._limit[i] & 2)
        return info


class _EnvView(object):
    """What BatchEnv.__getitem__ returns: a handle on one environment of the batch."""

    def __init__(self, batch, index):
        self._b, self.index = batch, index
        self.observation_space, self.action_space = batch.observation_space, batch.action_space

    @property
    def env_step_counter(self):
        return int(self._b.get_state()["env_step_counter"][self.index])

    def render(self, mode="rgb_array", close=False):
        """This env's frame (RexGymEnv.render, rex_gym_env.py:416-439)."""
        if mode != "rgb_array":
            return np.array([])
        return self._b.render_batch([self.index])[0].cpu().numpy()


class BatchedRexEnv(object):
    metadata = {"render.modes": ["rgb_array"], "video.frames_per_second": 66}

    def __init__(self, task="walk", num_envs=1, device="cuda:0", debug=False, urdf_version=None,
                 control_time_step=None, action_repeat=None, control_latency=0.0, pd_latency=0.0, on_rack=False,
                 motor_kp=1.0, motor_kd=0.02, render=False, num_steps_to_log=2000, env_randomizer=None,
                 log_path=None, target_position=None, backwards=None, target_orient=None, init_orient=None,
                 energy_weight=None, signal_type="ik", terrain_type="plane", terrain_id=None, mark="base",
                 normalize=False, max_episode_steps=0, auto_reset=False, seed=1234,
                 motor_kp_range=None, motor_kd_range=None, num_fields=64, solver_iterations=None, env_offset=0,
                 base_y=None, base_z=None, base_roll=None, base_pitch=None, base_yaw=None, gait_clock_scale=1.0,
                 rebalance_every=8, observation_noise_stdev=SENSOR_NOISE_STDDEV, episode_statistics=False,
                 frame_history=None, frame_delta=False, final_observation=False):
        """The reference's task-env keywords, plus the batch's own and the training wrappers fused into the kernels:
        normalize (RangeNormalize + ClipAction), max_episode_steps (LimitDuration), auto_reset, episode_statistics, and

        frame_history: None, or FrameHistory's past_indices (wrappers.py:93-151, flatten=True): a list of 1 to 16 indices in
          0..64 that includes 0.  Each observation row becomes the frames t - i for each index i in list order, concatenated
          ([N, len(frame_history) * O]; `.view(N, K, O)` gives the stacked form).  The ring holds max(frame_history) frames and
          is filled with the first observation at every reset.  As in the reference, an index equal to that maximum reads the
          current slot, so [0, 1, 2] returns frames t, t - 1 and t.  Duplicates and any order are allowed.
        frame_delta: FrameDelta (wrappers.py:154-180) inside the history: a step returns obs - last obs in fp32, a reset (and
          so an auto-reset step) the observation itself.
        Both are off by default; with both off nothing is allocated.
        final_observation: every step also keeps, for each env whose step returned done, the observation the step produced
          before the auto-reset replaced it (final_observation(), [N, O] like the observation rows), and every env's time-limit
          byte (truncated(), info[i]['TimeLimit.truncated'] as gym's TimeLimit adds it).  Off by default: no extra buffer, and
          info[i] is {'action': ...}.

        The keywords of PER_ENV_KEYWORDS take a scalar or one entry per env (a list, tuple or ndarray of num_envs entries).
        Entry e builds env e exactly as the batch built with that entry as the scalar would, and entries that are all equal
        build the scalar construction.  Each step launches every (terrain, mark, step-kernel unit, rate) group of envs as one
        slot range of the batch with its own values and kernel build, at most 16 groups; the reset hold is settled once per
        distinct hold setting, at most 64.
        target_position ... base_yaw: the task values, which set_task_values changes later.
        motor_kp, motor_kd: the gains; not with motor_kp_range / motor_kd_range.
        control_latency, pd_latency: the sensor latencies.
        terrain_type: 'plane' or 'random': the env's ground, friction and field sequence from the one num_fields bank.
        control_time_step, action_repeat: every control_time_step[e] / action_repeat[e] must be the one simulation time step,
          which the observation space depends on; each PGS solve is capped at solver_iterations (None: int(300 /
          action_repeat[e])); at most 8 distinct rates.
        task, signal_type: the env's defaults included (a control rate of 6 ms / 6 for gallop and poses, 5 ms / 5 otherwise).
          The envs' spaces must be the same, as the reference's BatchEnv requires: turn ik with turn ol, standup with poses,
          and under normalize walk ik with turn.
        mark: 'base' or 'arm': the env's robot, reset hold and sensor history; every task but gallop, which the arm is not
          built for.  A batch of both is built on the arm's tables, which serve the base envs too: num_motors is 18, the
          width of last_command(), a base env's rows 12..17 are NaN, and its info[i]['action'] has its own 12 entries."""
        if urdf_version is not None and urdf_version != DEFAULT_URDF_VERSION:
            raise ValueError("%s is not a supported urdf_version." % urdf_version)     # rex_gym_env.py:317-318
        n_envs = int(num_envs)
        # per-env marks: a batch of both is created with the arm, then told which envs are base
        mark_scalar, env_marks = check_env_marks(num_envs, mark)
        task_list = _name_entries("task", task, TASKS, n_envs)
        _name_entries("signal_type", signal_type, SIGNALS, n_envs)
        # per-env terrains: a batch of both is created on the heightfield (its bank), then told which envs are on the plane
        terrain_scalar, env_terrain = check_env_terrains(num_envs, terrain_type)
        if render or on_rack:
            raise ValueError("render / on_rack are GUI debugging modes of the reference; not part of the batched path")
        scalar_lat = [0.0 if is_per_env(v) else v for v in (control_latency, pd_latency)]
        if min(scalar_lat) < 0 or len(observation_noise_stdev) != 5 or min(observation_noise_stdev) < 0:
            raise ValueError("control_latency / pd_latency must be >= 0 and observation_noise_stdev five values >= 0")
        if env_randomizer:
            raise ValueError("env_randomizer hooks are Python callbacks; use motor_kp_range / motor_kd_range")
        frames = check_frame_history(frame_history)
        ctor_values = dict(target_position=target_position, backwards=backwards, target_orient=target_orient,
                           init_orient=init_orient, base_y=base_y, base_z=base_z, base_roll=base_roll, base_pitch=base_pitch,
                           base_yaw=base_yaw)
        env_values, env_gains = check_env_values(num_envs, ctor_values, motor_kp, motor_kd, motor_kp_range, motor_kd_range)
        if env_gains is not None:            # the handle's own gains only settle the snapshot rexsim_set_env_values replaces
            motor_kp, motor_kd = float(env_gains[0][0]), float(env_gains[1][0])
        # per-env latencies: the scalar gains of a motor_kp / motor_kd range hold the reset at each distinct pd_latency
        env_latency = check_env_latencies(num_envs, control_latency, pd_latency, motor_kp, motor_kd, env_gains)
        cts, rep, time_step, env_repeats = check_env_repeats(num_envs, task_list, control_time_step, action_repeat, solver_iterations)
        marks = mark_scalar if env_marks is None else tuple(str(m) for m in mark)
        task, signal_type, env_tasks = check_env_tasks(num_envs, task, signal_type, time_step, normalize, frames, frame_delta, marks)
        # env 0's task and signal in the config, as its rate; rexsim_set_env_tasks gives every env its own
        task0, signal0 = (task, signal_type) if env_tasks is None else (task[0], signal_type[0])
        if not torch.cuda.is_available():
            raise RuntimeError("rex_gym_b200 needs a CUDA device: there is no CPU fallback")
        self._L = _capi.load()
        self._debug = bool(debug)
        # the scalars for a scalar construction (an array of equal pairs is one), else the N entries
        self.task, self.signal_type, self.mark = task, signal_type, marks
        # the scalar for a scalar construction (an array of equal entries is one), else the N entries
        self.terrain_type = terrain_scalar if env_terrain is None else tuple(str(t) for t in terrain_type)
        self.device = torch.device(device)
        self.num_envs = int(num_envs)
        # the command block's width: the scalar mark's motors, 18 for a batch of both marks
        self.num_motors = MARKS[mark_scalar or "arm"]
        # the scalars for a scalar construction, else the N entries; the simulation time step is the batch's
        self.control_time_step, self._action_repeat = cts, rep
        self._time_step = time_step
        table_mark = mark_scalar or "arm"
        tables, toe_npts = pack_model_tables(table_mark)
        c = _capi.RexSimConfig()
        c.num_envs, c.task, c.signal = self.num_envs, TASKS[task0], SIGNALS[signal0]
        c.terrain = TERRAINS[terrain_scalar or "random"]
        if env_repeats is None:
            c.num_motors, c.action_repeat = self.num_motors, rep
            c.solver_iterations = solver_iterations or int(300 / rep)                  # rex_gym_env.py:25,184
        else:                                # env 0's rate in the config; rexsim_set_env_repeats gives every env its own
            c.num_motors, c.action_repeat, c.solver_iterations = self.num_motors, int(env_repeats[0][0]), int(env_repeats[1][0])
        c.sim_dt, c.sim_dt_d = self._time_step, self._time_step
        c.motor_kp, c.motor_kd = motor_kp, motor_kd
        c.kp_lo, c.kp_hi = motor_kp_range or (motor_kp, motor_kp)
        c.kd_lo, c.kd_hi = motor_kd_range or (motor_kd, motor_kd)
        # per-env keywords leave the scalar "draw" in the config: the kernels read the value block instead
        scalar = {k: (None if is_per_env(v) else v) for k, v in ctor_values.items()}
        c.target_position = task_value("target_position", scalar["target_position"])
        c.backwards = task_value("backwards", scalar["backwards"])
        c.target_orient = task_value("target_orient", scalar["target_orient"])
        c.init_orient = task_value("init_orient", scalar["init_orient"])
        c.w_distance, c.w_drift, c.w_shake = 1.0, 2.0, 0.005                            # rex_gym_env.py:56-59
        c.w_energy = energy_weight if energy_weight is not None else (0.005 if task0 == "gallop" else 0.0005)
        c.normalize, c.max_episode_steps, c.auto_reset, c.seed = int(normalize), int(max_episode_steps), int(auto_reset), seed
        c.gait_clock_scale = float(gait_clock_scale)     # GaitPlanner clock / simulation clock (the reference reads the wall clock)
        for k, name in enumerate(("base_y", "base_z", "base_roll", "base_pitch", "base_yaw")):   # poses_env.py:49-53 (None = rotate)
            c.pose_values[k] = task_value(name, scalar[name])
        # sensor model (rex_gym_env.py:61,70-71 -> Rex(control_latency, pd_latency, observation_noise_stdev), rex.py:726-769)
        # (per-env latencies leave 0 in the config: rexsim_set_env_latencies gives every env its own)
        c.control_latency, c.pd_latency = (float(v) for v in scalar_lat)
        for k, v in enumerate(observation_noise_stdev):
            c.noise_stdev[k] = float(v)
        c.episode_stats = int(bool(episode_statistics))       # simulate()'s score / length bookkeeping on the device
        self._fields = None
        friction = {"random": 0.5 * 0.5,      # URDF link default 0.5 x createMultiBody default 0.5
                    "plane": 0.5 * 1.0}       # x plane.urdf lateral_friction 1
        with torch.cuda.device(self.device):
            if c.terrain == TERRAINS["random"]:
                self._fields = torch.from_numpy(make_random_fields(num_fields)).to(self.device).contiguous()
                c.nfields, c.fields = num_fields, self._fields.data_ptr()
                c.friction = friction["random"]
            else:
                c.nfields, c.fields = 0, None
                c.friction = friction["plane"]
            c.residual_threshold, c.erp_contact, c.erp_joint = 1e-7, 0.08, 0.2
            c.toe_npts, c.toe_margin = toe_npts, TOE_MARGIN
            c.contact_breaking = contact_breaking_distance(table_mark)
            c.link_damping, c.max_coordinate_velocity = LINK_DAMPING, MAX_COORDINATE_VELOCITY
            c.env_offset = int(env_offset)
            self._cfg = c
            h = C.c_void_p()
            tb = np.ascontiguousarray(tables)
            _capi.check(self._L.rexsim_create(C.byref(c), tb.ctypes.data, tb.size, C.byref(h)))
        self._h = h
        self._dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        # every library call: on this env's device and torch's current stream there, a non-zero status raised (_capi.call)
        self._call = functools.partial(_capi.call, self._dev_index)
        rt = np.ascontiguousarray(pack_render_tables(table_mark))
        self._call(self._L.rexsim_set_render_tables, self._h, rt.ctypes.data, rt.size, stream=False)
        env_obs_dim = self._L.rexsim_obs_dim(c.task, c.num_motors)
        if frames or frame_delta:
            fi = np.ascontiguousarray(frames or [0], np.int32)
            self._call(self._L.rexsim_set_frames, self._h, fi.ctypes.data, len(frames), int(bool(frame_delta)), stream=False)
        self.frame_history, self.frame_delta = (list(frames) if frames else None), bool(frame_delta)
        if env_terrain is not None:
            self._call(self._L.rexsim_set_env_terrains, self._h, env_terrain.ctypes.data, friction["plane"], stream=False)
        if env_repeats is not None:
            self._call(self._L.rexsim_set_env_repeats, self._h, env_repeats[0].ctypes.data, env_repeats[1].ctypes.data,
                       stream=False)
        if env_tasks is not None:
            self._call(self._L.rexsim_set_env_tasks, self._h, env_tasks[0].ctypes.data, env_tasks[1].ctypes.data, stream=False)
        if env_marks is not None:
            self._call(self._L.rexsim_set_env_marks, self._h, env_marks.ctypes.data, stream=False)
        self._env_motors = env_marks         # [N] motors of each env on the host (per-env marks only): info[i]['action'] width
        self._values = None
        if env_values is not None:
            block = np.full((len(TASK_VALUE_KEYWORDS), self.num_envs), np.nan, np.float32)
            for k, v in env_values.items():
                block[self._L.rexsim_value_row(k.encode())] = v
            kp, kd = env_gains if env_gains is not None else (None, None)
            self._call(self._L.rexsim_set_env_values, self._h, block.ctypes.data, None if kp is None else kp.ctypes.data,
                       None if kd is None else kd.ctypes.data, stream=False)
        if env_latency is not None:
            self._call(self._L.rexsim_set_env_latencies, self._h, env_latency[0].ctypes.data, env_latency[1].ctypes.data,
                       stream=False)
        self.obs_dim = self._L.rexsim_out_dim(self._h)           # env_obs_dim x len(frame_history)
        self.action_dim = self._L.rexsim_action_dim(c.task, c.signal)
        N, O, A = self.num_envs, self.obs_dim, self.action_dim
        dev = self.device
        # device path: obs | reward | done of the last step (torch views; `done` is a bool view of the u8 the kernel writes)
        self._obs = torch.zeros((N, O), dtype=torch.float32, device=dev)
        self._reward = torch.zeros((N,), dtype=torch.float32, device=dev)
        self._done_u8 = torch.zeros((N,), dtype=torch.uint8, device=dev)
        self._done = self._done_u8.view(torch.bool)
        # host path (numpy in / numpy out): ONE pinned block each way, filled by rexsim_step_host in one C call
        self._h_act = torch.zeros((N, A), dtype=torch.float32).pin_memory()
        self._h_out = torch.zeros((int(self._L.rexsim_host_out_bytes(self._h)),), dtype=torch.uint8).pin_memory()
        self._h_act_np = self._h_act.numpy()
        self._h_act_ptr, self._h_out_ptr = self._h_act.data_ptr(), self._h_out.data_ptr()
        self._h_obs, self._h_reward, self._h_done, self._h_err = _host_block_views(self._h_out.numpy(), N, O)

        def view(p, shape, typestr):
            return _capi.device_view(p.value, shape, typestr, self, dev)
        p, q = C.c_void_p(), C.c_void_p()
        _capi.check(self._L.rexsim_error_flags(self._h, C.byref(p)))
        self._err = view(p, (N + 1,), "<i4")
        _capi.check(self._L.rexsim_last_command(self._h, C.byref(p)))
        self._cmd = view(p, (self.num_motors, N), "<f4")
        nf, ni = C.c_int32(), C.c_int32()
        _capi.check(self._L.rexsim_state_words(C.byref(c), C.byref(nf), C.byref(ni)))
        _capi.check(self._L.rexsim_state_buffers(self._h, C.byref(p), C.byref(q)))
        self._state_f, self._state_i = view(p, (nf.value, N), "<f4"), view(q, (ni.value, N), "<i4")
        nr = C.c_int64()
        _capi.check(self._L.rexsim_history_buffer(self._h, C.byref(p), C.byref(nr)))           # sensor history ring (None: model off)
        self._ring = view(p, (nr.value,), "<f4") if nr.value else None
        nl = C.c_int64()
        _capi.check(self._L.rexsim_frame_buffers(self._h, C.byref(p), C.byref(nr), C.byref(q), C.byref(nl)))
        self._frames = {k: view(ptr, (n.value,), "<f4") for k, ptr, n in (("frame_history", p, nr), ("frame_delta", q, nl)) if n.value}
        if env_values is not None:
            g, npairs = C.c_void_p(), C.c_int32()
            _capi.check(self._L.rexsim_env_value_buffers(self._h, C.byref(p), C.byref(q), C.byref(g), C.byref(npairs)))
            self._values = dict(values=view(p, (len(TASK_VALUE_KEYWORDS) + 1, N), "<f4"), pair=view(q, (N,), "<i4"),
                                gains=view(g, (npairs.value, 2), "<f4"))
        # _marks [N] u8: 1 for each arm env, 0 for each base env; _tasks [2][N] u8: each env's TASKS and SIGNALS id; _repeats
        # [2][N] i32: each env's action_repeat, solver_iterations; _terrain [N] u8: each env's TERRAINS id; _latency [2][N]
        # f64: each env's control_latency, pd_latency.  None when the keyword is not per env.
        given = dict(_marks=env_marks, _tasks=env_tasks, _repeats=env_repeats, _terrain=env_terrain, _latency=env_latency)
        for b in _ENV_BLOCKS:
            setattr(self, b.attr, None)
            if given[b.attr] is not None:
                _capi.check(getattr(self._L, b.call)(self._h, C.byref(p), *((C.byref(C.c_int32()),) if b.depth else ())))
                setattr(self, b.attr, view(p, (N,) if b.rows == 1 else (b.rows, N), b.typestr))
        self._episode = None
        if episode_statistics:
            o, sm, blk, nb = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_int64()
            _capi.check(self._L.rexsim_episode_buffers(self._h, *(C.byref(x) for x in (p, q, o, sm, blk, nb))))
            self._episode = dict(score=view(p, (N,), "<f4"), length=view(q, (N,), "<i4"), summary=view(sm, (4,), "<f8"),
                                 block=view(blk, (nb.value,), "|u1"),
                                 objectives=view(o, (4, N), "<f4") if o.value else None)
        # spaces: raw task spaces, or the wrapper-visible ones when the training wrappers are fused in (every env's are these)
        self.action_space, self.observation_space = task_spaces(task0, signal0, normalize, self._time_step, frames, frame_delta,
                                                                self.num_motors)
        assert self.observation_space.shape == (O,) and self.action_space.shape == (A,) and env_obs_dim * max(len(frames), 1) == O
        # every `rebalance_every` steps the envs are re-grouped over the warps by solver cost (rexsim_rebalance): a scheduling
        # hint only -- results are bit-identical with 0 (off).  It pays off once the batch is several waves deep (+17-19 % at
        # 16 384 / 65 536 envs); a batch that fits one wave (4096 envs = 128 CTAs on 132 SMs) is bound by its slowest env anyway
        self._rebalance_every = int(rebalance_every) if self.num_envs >= 8192 else 0
        # final observation and time-limit byte of the last step: device buffers for the device path, one pinned block
        # (final obs [N][O] f32 | limit [N] u8, rexsim_host_final_bytes) for the numpy path
        self._final = self._limit = self._h_final = None
        self._last_on_device = True
        if final_observation:
            self._final = torch.zeros((N, O), dtype=torch.float32, device=dev)
            self._limit = torch.zeros((N,), dtype=torch.uint8, device=dev)
            self._h_final = torch.zeros((int(self._L.rexsim_host_final_bytes(self._h)),), dtype=torch.uint8).pin_memory()
            hf = self._h_final.numpy()
            self._h_final_obs, self._h_limit = hf[:N * O * 4].view(np.float32).reshape(N, O), hf[N * O * 4:]
        self._nsteps = 0
        self._closed = False

    # ---- BatchEnv surface ------------------------------------------------------------------------
    def __len__(self):
        return self.num_envs

    def __getitem__(self, index):
        if not -self.num_envs <= index < self.num_envs:
            raise IndexError(index)
        return _EnvView(self, index % self.num_envs)

    def _maybe_rebalance(self):
        self._nsteps += 1
        if self._rebalance_every and self._nsteps % self._rebalance_every == 0:
            self._call(self._L.rexsim_rebalance, self._h)

    def step(self, action):
        """BatchEnv.step (batch_env.py:63-90).  numpy in -> numpy out (host buffers: one rexsim_step_host call = H2D copy,
        kernel, D2H copy, wait);  CUDA tensor in -> CUDA tensors out (one asynchronous kernel launch, no host traffic)."""
        N, A = self.num_envs, self.action_dim
        if isinstance(action, torch.Tensor) and action.is_cuda:
            if tuple(action.shape) != (N, A):
                raise ValueError("Invalid action shape %s, expected %s" % (tuple(action.shape), (N, A)))
            if action.dtype != torch.float32 or not action.is_contiguous():
                action = action.to(torch.float32).contiguous()
            if self._final is None:
                self._call(self._L.rexsim_step, self._h, action.data_ptr(), self._obs.data_ptr(), self._reward.data_ptr(),
                           self._done_u8.data_ptr())
            else:
                self._call(self._L.rexsim_step_final, self._h, action.data_ptr(), self._obs.data_ptr(), self._reward.data_ptr(),
                           self._done_u8.data_ptr(), self._final.data_ptr(), self._limit.data_ptr())
            self._last_on_device = True
            self._maybe_rebalance()
            return self._obs, self._reward, self._done, _Info(self)
        a = np.asarray(action, dtype=np.float32)
        if a.shape != (N, A):
            raise ValueError("Invalid action shape %s, expected %s" % (a.shape, (N, A)))
        if not np.isfinite(a).all():
            raise ValueError("Invalid action: non-finite values")
        np.copyto(self._h_act_np, a)
        if self._final is None:
            self._call(self._L.rexsim_step_host, self._h, self._h_act_ptr, self._h_out_ptr)
        else:
            self._call(self._L.rexsim_step_host_final, self._h, self._h_act_ptr, self._h_out_ptr, self._h_final.data_ptr())
        self._last_on_device = False
        self._maybe_rebalance()
        if self._h_err[0] & ERR_NONFINITE:        # the aggregate word is per step on this path (rexsim_step_host clears it)
            raise ValueError("Infinite observation encountered.")          # ConvertTo32Bit wrappers.py:522-523,542-543
        return self._h_obs.copy(), self._h_reward.copy(), self._h_done.copy(), _Info(self)

    def step_into(self, action, obs, reward, done_u8, final_obs=None, limit=None):
        """Raw device form of step(): CUDA float32 action [N][A] in; obs [N][O], reward [N] (float32) and done [N] (uint8) are
        written into the caller's contiguous CUDA buffers (e.g. slices of a rollout).  One asynchronous kernel launch.
        final_obs [N][O] float32 / limit [N] uint8 (either may be None; any env, whatever its final_observation switch): the
        rows of the envs that returned done get their final observation, the others are left untouched; every env gets its
        time-limit byte (bit 0 max_episode_steps reached, bit 1 the episode also ended otherwise; truncated = limit == 1)."""
        if final_obs is None and limit is None:
            self._call(self._L.rexsim_step, self._h, action.data_ptr(), obs.data_ptr(), reward.data_ptr(), done_u8.data_ptr())
        else:
            ptr = lambda t: None if t is None else t.data_ptr()
            self._call(self._L.rexsim_step_final, self._h, action.data_ptr(), obs.data_ptr(), reward.data_ptr(), done_u8.data_ptr(),
                       ptr(final_obs), ptr(limit))
        self._maybe_rebalance()

    def _indices(self, indices, what):
        """Host or device indices -> int32 CUDA tensor [k].  Host indices outside the batch raise IndexError here.  Device indices
        are not inspected on the host: the kernels skip any index outside [0, N) and raise REXSIM_FLAG_BAD_INDEX in the aggregate
        error word (check_errors() -> IndexError)."""
        if isinstance(indices, torch.Tensor):
            return indices.to(device=self.device, dtype=torch.int32).reshape(-1).contiguous()
        ia = np.asarray(indices, dtype=np.int64).reshape(-1)
        if ia.size and (ia.min() < 0 or ia.max() >= self.num_envs):
            raise IndexError("%s index out of range" % what)
        return torch.from_numpy(ia.astype(np.int32)).to(self.device)

    def reset(self, indices=None):
        """BatchEnv.reset (batch_env.py:92-109): observations of the reset environments."""
        if indices is None:
            k, idx_ptr = self.num_envs, None
        else:
            idx = self._indices(indices, "reset")
            if self._debug and idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= self.num_envs):
                raise IndexError("reset index out of range")       # debug=True inspects device indices too (one sync)
            k, idx_ptr = int(idx.numel()), idx.data_ptr()
        out = torch.zeros((k, self.obs_dim), dtype=torch.float32, device=self.device)
        if k > 0:
            self._call(self._L.rexsim_reset, self._h, idx_ptr, k, out.data_ptr())
        if isinstance(indices, torch.Tensor):
            return out
        return out.cpu().numpy()

    def close(self):
        if not self._closed:
            self._closed = True
            torch.cuda.synchronize(self.device)
            self._L.rexsim_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- extras ------------------------------------------------------------------------------------
    def get_state(self):
        """Physical state of every env (pybullet getBasePositionAndOrientation/getBaseVelocity/getJointState)."""
        N, nm = self.num_envs, self.num_motors
        f = torch.zeros((13 + 2 * nm, N), dtype=torch.float32, device=self.device)
        i = torch.zeros((4, N), dtype=torch.int32, device=self.device)
        self._call(self._L.rexsim_get_state, self._h, f.data_ptr(), i.data_ptr())
        f, i = f.cpu().numpy(), i.cpu().numpy()
        return dict(pos=f[0:3].T.copy(), quat=f[3:7].T.copy(), linvel=f[7:10].T.copy(), angvel=f[10:13].T.copy(),
                    q=f[13:13 + nm].T.copy(), qd=f[13 + nm:13 + 2 * nm].T.copy(),
                    step_counter=i[0].copy(), env_step_counter=i[1].copy(), flags=i[2].copy(), contact_mask=i[3].copy())

    def set_state(self, pos, quat, linvel, angvel, q, qd):
        N, nm = self.num_envs, self.num_motors
        f = np.concatenate([np.asarray(x, np.float32).reshape(N, -1).T for x in (pos, quat, linvel, angvel, q, qd)], axis=0)
        t = torch.from_numpy(np.ascontiguousarray(f)).to(self.device)
        self._call(self._L.rexsim_set_state, self._h, t.data_ptr())
        torch.cuda.current_stream(self.device).synchronize()

    def _final_buffers(self):
        if self._final is None:
            raise ValueError("final observations are off: create the env with final_observation=True")
        return (self._final, self._limit) if self._last_on_device else (self._h_final_obs, self._h_limit)

    def final_observation(self):
        """[N, O] observations of the last step before the auto-reset replaced them (what `obs` holds with auto_reset=False):
        valid in the rows where that step returned done; the other rows keep older values.  A CUDA view after a step with a
        CUDA action, a numpy copy after a numpy step; both are overwritten by the next step."""
        f = self._final_buffers()[0]
        return f if self._last_on_device else f.copy()

    def limit_bytes(self):
        """[N] uint8 time-limit bytes of the last step: bit 0 max_episode_steps was reached, bit 1 the episode also ended by the
        task's termination or a non-finite observation (CUDA view or numpy view, as final_observation())."""
        return self._final_buffers()[1]

    def truncated(self):
        """[N] bool: the last step ended the episode by the time limit alone (gym's info['TimeLimit.truncated'] is True)."""
        return self.limit_bytes() == 1

    def last_command(self):
        """[num_motors, N] motor commands of the last step (info['action'], rex_gym_env.py:414).  In a batch of both marks
        num_motors is 18 and a base env's rows 12..17 are NaN."""
        return self._cmd

    def error_flags(self):
        return self._err[:self.num_envs]

    def check_errors(self):
        """Read AND clear the aggregate error word (every bit raised since the last call; one device sync).  Raises like the
        reference would have for the offending step: ValueError for a non-finite observation (ConvertTo32Bit), IndexError for a
        reset index outside the batch; returns the remaining (informational) bits."""
        e = int(self._err[self.num_envs].item())
        if e:
            self._call(self._L.rexsim_clear_errors, self._h)
        if e & ERR_NONFINITE:
            raise ValueError("Infinite observation encountered.")
        if e & ERR_BAD_INDEX:
            raise IndexError("reset index out of range")
        return e

    def state_dict(self):
        """Exact checkpoint of the whole batch (the reference never checkpoints env state)."""
        sd = {"state_f": self._state_f.clone(), "state_i": self._state_i.clone()}
        if self._ring is not None:
            sd["sensor_history"] = self._ring.clone()
        if self._episode is not None:
            sd["episode_statistics"] = self._episode["block"].clone()
        for k, v in self._frames.items():
            sd[k] = v.clone()
        if self._values is not None:
            sd.update(("env_" + k, v.clone()) for k, v in self._values.items())
        for b in _ENV_BLOCKS:
            if getattr(self, b.attr) is not None:
                sd[b.key] = getattr(self, b.attr).clone()
        return sd

    def load_state_dict(self, sd):
        def present(noun, block, key):
            if (block is None) != (key not in sd):
                raise ValueError("per-env %s: the checkpoint %s them, this batch %s" %
                                 ((noun,) + (("has", "does not") if block is None else ("lacks", "has"))))
        for b in _ENV_BLOCKS:
            block = getattr(self, b.attr)
            present(b.noun, block, b.key)
            if block is not None and not torch.equal(block, sd[b.key].to(block.device)):
                raise ValueError("per-env %s: the checkpoint's %s differ from this batch's" % (b.noun, b.entries))
        present("values", self._values, "env_values")
        if self._values is not None:
            for k in ("gains", "pair"):       # the settled snapshots belong to this handle's pairs
                if not torch.equal(self._values[k], sd["env_" + k].to(self._values[k].device)):
                    raise ValueError("per-env gains: the checkpoint's gain pairs differ from this batch's")
            self._values["values"].copy_(sd["env_values"])
        self._state_f.copy_(sd["state_f"])
        self._state_i.copy_(sd["state_i"])
        if self._ring is not None:
            self._ring.copy_(sd["sensor_history"])
        if self._episode is not None:
            self._episode["block"].copy_(sd["episode_statistics"])
        for k, v in self._frames.items():
            v.copy_(sd[k])

    # ---- per-env task values ------------------------------------------------------------------------------
    def set_task_values(self, indices=None, **values):
        """Give the envs `indices` (default: all) new constructor values, e.g. set_task_values([0, 3], target_position=2.5)
        or a curriculum between Rollout.collect() calls.  Keywords: those of TASK_VALUE_KEYWORDS (the gains, latencies, control
        rates and terrains are fixed at construction), each a scalar or one value per index, meaning what it means to the
        constructor.
        Each env starts using them at its next reset, explicit or automatic.  Enqueued on the current stream without a host sync; host values are
        checked here, device tensors are not inspected.  Needs a batch built with per-env values (any of these keywords, or
        motor_kp / motor_kd, given one value per env)."""
        bad = sorted(set(values) - set(TASK_VALUE_KEYWORDS))
        if bad:
            fixed = tuple(k for k in PER_ENV_KEYWORDS if k not in TASK_VALUE_KEYWORDS)
            raise ValueError("set_task_values takes %s; not %s (the gains, latencies, tasks, marks, control rates and terrains "
                             "are fixed at construction: %s)" % (TASK_VALUE_KEYWORDS, bad, fixed))
        if self._values is None:
            raise ValueError("per-env values are off: build the batch with one value per env for a task keyword")
        idx = None if indices is None else self._indices(indices, "set_task_values")
        k = self.num_envs if idx is None else int(idx.numel())
        if k == 0 or not values:
            return
        block = torch.empty((len(TASK_VALUE_KEYWORDS), k), dtype=torch.float32, device=self.device)
        rows = 0
        for name, v in values.items():
            r = self._L.rexsim_value_row(name.encode())
            rows |= 1 << r
            if isinstance(v, torch.Tensor) and v.is_cuda:
                t = v.to(device=self.device, dtype=torch.float32).reshape(-1).expand(k)
                if name == "target_position":
                    t = torch.where(t == 0, torch.full_like(t, float("nan")), t)
                elif name == "backwards":
                    t = torch.where(torch.isnan(t), torch.full_like(t, -1.0), t)
                block[r] = t
            else:
                a = task_value_entries(name, v, k) if is_per_env(v) else np.full(k, task_value(name, v), np.float32)
                block[r] = torch.from_numpy(a).to(self.device, non_blocking=False)
        self._call(self._L.rexsim_set_task_values, self._h, None if idx is None else idx.data_ptr(), k, block.data_ptr(), rows)

    def task_values(self):
        """{keyword: CUDA view [N]} of every env's constructor values (what its next reset uses), plus 'episode_backwards'
        (the direction its running episode started with); None when the batch has no per-env values."""
        if self._values is None:
            return None
        v = self._values["values"]
        out = {k: v[self._L.rexsim_value_row(k.encode())] for k in TASK_VALUE_KEYWORDS}
        out["episode_backwards"] = v[len(TASK_VALUE_KEYWORDS)]
        return out

    # ---- episode statistics (episode_statistics=True) ------------------------------------------------
    def _episode_buffer(self, name):
        if self._episode is None:
            raise ValueError("episode statistics are off: create the env with episode_statistics=True")
        return self._episode[name]

    @property
    def objective_weights(self):
        """RexGymEnv.objective_weights (rex_gym_env.py:547-556): weights of forward, energy, drift and shake in the reward."""
        c = self._cfg
        return (c.w_distance, c.w_energy, c.w_drift, c.w_shake)

    def objectives(self):
        """RexGymEnv.get_objectives of the last step for every env: CUDA view [N, 4] of forward, energy, drift, shake before
        the weights, overwritten by the next step.  Walk and gallop only: the other tasks' rewards have no objectives (in a
        batch of several tasks with a walking env, their rows are NaN)."""
        o = self._episode_buffer("objectives")
        if o is None:
            raise ValueError("the %s task records no objectives (its _reward replaces RexGymEnv's)" % (self.task,))
        return o.t()

    def episode_score(self):
        """simulate()'s `score`: CUDA view [N] of the reward summed over each env's running episode."""
        return self._episode_buffer("score")

    def episode_length(self):
        """simulate()'s `length`: CUDA view [N] (int32) of the control steps of each env's running episode."""
        return self._episode_buffer("length")

    def episode_totals(self, clear=True):
        """Enqueue the batch's episode totals on the current stream (no sync): CUDA view [4] float64 of episodes submitted,
        episodes ended non-finite, their score sum and length sum.  The next call overwrites it.  clear=True starts the next
        totals from zero (StreamingMean.clear); running episodes go on."""
        self._episode_buffer("summary")
        self._call(self._L.rexsim_episode_summary, self._h, int(bool(clear)))
        return self._episode["summary"]

    def episode_summary(self, clear=True):
        """What simulate() logs (simulate.py:95-106): {'count', 'nonfinite', 'mean_score', 'mean_length'} over the episodes
        that ended since the last clear; the means are None when none did.  One device sync."""
        return summarize_episodes(self.episode_totals(clear))

    @property
    def launch_count(self):
        return int(self._L.rexsim_launch_count(self._h))

    def seed(self, seed=None):
        return [seed]

    def render(self, mode="rgb_array", close=False):
        """RexGymEnv.render as BatchEnv forwards it (batch_env.py:52-61: to env 0): a (360, 480, 3) uint8 frame of env 0 through
        the reference's follow camera for mode 'rgb_array', an empty array for any other mode (rex_gym_env.py:416-418)."""
        if mode != "rgb_array":
            return np.array([])
        return self.render_batch([0])[0].cpu().numpy()

    def render_batch(self, indices, width=480, height=360, distance=1.0, yaw=0.0, pitch=-30.0):
        """Frames of the envs `indices` as a CUDA uint8 tensor [k, height, width, 3] (row 0 at the top), ray-cast from the
        device state on the current stream without synchronising.  The camera follows each env's base the way the reference's
        does (rex_gym_env.py:214-216,420-436): distance [m], yaw and pitch [deg].  What is drawn is the collision geometry.
        Host indices outside the batch raise IndexError; device indices are not inspected (an out-of-range one gives a sky
        image and check_errors() raises IndexError), as in reset()."""
        if not (1 <= int(width) <= 4096 and 1 <= int(height) <= 4096):
            raise ValueError("image sides must be 1..4096")
        idx = self._indices(indices, "render")
        k = int(idx.numel())
        out = torch.empty((k, int(height), int(width), 3), dtype=torch.uint8, device=self.device)
        if k > 0:
            self._call(self._L.rexsim_render, self._h, idx.data_ptr(), k, int(width), int(height), float(distance), float(yaw),
                       float(pitch), out.data_ptr())
        return out


class RexWalkBatchEnv(BatchedRexEnv):
    """rex_gym/envs/gym/walk_env.py:16 RexWalkEnv, batched."""

    def __init__(self, num_envs=1, **kw):
        kw.setdefault("control_time_step", 0.005); kw.setdefault("action_repeat", 5)
        super().__init__(task="walk", num_envs=num_envs, **kw)


class RexGallopBatchEnv(BatchedRexEnv):
    """rex_gym/envs/gym/gallop_env.py:28 RexReactiveEnv, batched."""

    def __init__(self, num_envs=1, **kw):
        kw.setdefault("control_time_step", 0.006); kw.setdefault("action_repeat", 6)
        kw.setdefault("energy_weight", 0.005)
        super().__init__(task="gallop", num_envs=num_envs, **kw)


class RexTurnBatchEnv(BatchedRexEnv):
    """rex_gym/envs/gym/turn_env.py:20 RexTurnEnv, batched."""

    def __init__(self, num_envs=1, **kw):
        kw.setdefault("control_time_step", 0.005); kw.setdefault("action_repeat", 5)
        super().__init__(task="turn", num_envs=num_envs, **kw)


class RexPosesBatchEnv(BatchedRexEnv):
    """rex_gym/envs/gym/poses_env.py:21 RexPosesEnv, batched (no settle at reset; reward 1, never 'fallen')."""

    def __init__(self, num_envs=1, **kw):
        kw.setdefault("control_time_step", 0.006); kw.setdefault("action_repeat", 6)
        super().__init__(task="poses", num_envs=num_envs, **kw)


class RexStandupBatchEnv(BatchedRexEnv):
    """rex_gym/envs/gym/standup_env.py:17 RexStandupEnv, batched (starts from INIT_POSES['rest_position'])."""

    def __init__(self, num_envs=1, **kw):
        kw.setdefault("control_time_step", 0.005); kw.setdefault("action_repeat", 5)
        kw.setdefault("signal_type", "ol")
        super().__init__(task="standup", num_envs=num_envs, **kw)


# gym ids of rex_gym/playground/__init__.py:17-57 -> batched classes
ENV_IDS = {"RexWalk-v0": RexWalkBatchEnv, "RexGalloping-v0": RexGallopBatchEnv, "RexTurn-v0": RexTurnBatchEnv,
           "RexStandup-v0": RexStandupBatchEnv, "RexPoses-v0": RexPosesBatchEnv}


# max_episode_steps of the reference's registrations (playground/__init__.py:17-57): gym.make wraps the env in a TimeLimit
REGISTERED_MAX_EPISODE_STEPS = {"RexWalk-v0": 2500, "RexGalloping-v0": 1000, "RexTurn-v0": 1000, "RexStandup-v0": 400,
                                "RexPoses-v0": 400}


def make(env_id, num_envs=1, **kwargs):
    """gym.make(id, **args) equivalent (rex_gym/playground/trainer.py:47) returning a whole batch; the registered
    max_episode_steps (gym's TimeLimit) is fused into the kernel unless the caller overrides it."""
    if env_id not in ENV_IDS:
        raise ValueError("env id %r not built (have %s)" % (env_id, sorted(ENV_IDS)))
    kwargs.setdefault("max_episode_steps", REGISTERED_MAX_EPISODE_STEPS[env_id])
    return ENV_IDS[env_id](num_envs=num_envs, **kwargs)

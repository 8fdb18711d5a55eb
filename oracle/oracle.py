"""ctypes front-end of the CPU ORACLE (test infrastructure, NOT the product path).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module (see oracle/rexsim_oracle.h).
"""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
MODEL_DIR = os.environ.get("REXO_MODEL_DIR") or os.path.join(HERE, "..", "rex_gym_b200", "model")

MAXB, MAXDOF, MAXSHAPE, MAXPTS = 20, 18, 40, 1024
TASKS = {"walk": 0, "gallop": 1, "turn": 2, "standup": 3, "poses": 4}
SIGNALS = {"ik": 0, "ol": 1}
TERRAINS = {"plane": 0, "random": 1}


class RexoModel(C.Structure):
    _fields_ = [
        ("nb", C.c_int32), ("ndof", C.c_int32), ("parent", C.c_int32 * MAXB),
        ("jpos", (C.c_double * 3) * MAXB), ("jrot", (C.c_double * 9) * MAXB), ("axis", (C.c_double * 3) * MAXB),
        ("lower", C.c_double * MAXB), ("upper", C.c_double * MAXB), ("mass", C.c_double * MAXB),
        ("com", (C.c_double * 3) * MAXB), ("inertia", (C.c_double * 9) * MAXB),
        ("root_mass", C.c_double), ("root_inertia", C.c_double * 3),
        ("nshape", C.c_int32), ("shape_start", C.c_int32 * MAXSHAPE), ("shape_npts", C.c_int32 * MAXSHAPE),
        ("shape_enabled", C.c_int32 * MAXSHAPE), ("pt_body", C.c_int32 * MAXPTS), ("pt_margin", C.c_double * MAXPTS),
        ("pt_terrain", C.c_int32 * MAXPTS),
        ("pts", (C.c_double * 3) * MAXPTS),
        ("nmotor", C.c_int32), ("motor_dof", C.c_int32 * MAXDOF),
    ]


class RexoConfig(C.Structure):
    _fields_ = [
        ("num_envs", C.c_int32), ("task", C.c_int32), ("signal", C.c_int32), ("terrain", C.c_int32),
        ("action_repeat", C.c_int32), ("solver_iterations", C.c_int32), ("sim_dt", C.c_double),
        ("motor_kp", C.c_double), ("motor_kd", C.c_double),
        ("kp_lo", C.c_double), ("kp_hi", C.c_double), ("kd_lo", C.c_double), ("kd_hi", C.c_double),
        ("target_position", C.c_double), ("backwards", C.c_int32),
        ("target_orient", C.c_double), ("init_orient", C.c_double),
        ("w_distance", C.c_double), ("w_energy", C.c_double), ("w_drift", C.c_double), ("w_shake", C.c_double),
        ("normalize", C.c_int32), ("max_episode_steps", C.c_int32), ("seed", C.c_uint64),
        ("nfields", C.c_int32), ("fields", C.POINTER(C.c_float)), ("friction", C.c_double),
        ("residual_threshold", C.c_double), ("erp_contact", C.c_double), ("erp_joint", C.c_double),
        ("settle_on_reset", C.c_int32), ("env_offset", C.c_int32), ("gait_clock_scale", C.c_double),
        ("link_damping", C.c_double), ("contact_breaking", C.c_double),
        ("max_coordinate_velocity", C.c_double),
        ("control_latency", C.c_double), ("pd_latency", C.c_double), ("noise_stdev", C.c_double * 5),
        ("pose_values", C.c_double * 5),
    ]


class RexoEnv(C.Structure):
    _fields_ = [
        ("pos", C.c_double * 3), ("quat", C.c_double * 4), ("linvel", C.c_double * 3), ("angvel", C.c_double * 3),
        ("q", C.c_double * MAXDOF), ("qd", C.c_double * MAXDOF), ("tau_obs", C.c_double * MAXDOF),
        ("cmd", C.c_double * MAXDOF), ("overheat", C.c_int32 * MAXDOF), ("enabled", C.c_int32 * MAXDOF),
        ("step_counter", C.c_int32), ("env_step_counter", C.c_int32), ("limit_step", C.c_int32),
        ("gp_phi", C.c_double), ("gp_last_time", C.c_double), ("gp_alpha", C.c_double),
        ("goal_reached", C.c_int32), ("is_terminating", C.c_int32), ("stay_still", C.c_int32),
        ("backwards", C.c_int32), ("clockwise", C.c_int32), ("env_goal_reached", C.c_int32),
        ("end_time", C.c_double), ("target_position", C.c_double), ("target_orient", C.c_double),
        ("init_orient", C.c_double), ("kp", C.c_double), ("kd", C.c_double),
        ("reset_count", C.c_uint32), ("field_id", C.c_int32),
        ("contact_mask", C.c_int32), ("contact_vertex", C.c_int32 * MAXSHAPE),
        ("solver_iters", C.c_int32), ("limit_rows", C.c_int32),
        ("next_pose", C.c_int32), ("target_value", C.c_double),
    ]


def build(force=False):
    """Compile the oracle shared libraries with the committed Makefile."""
    so = os.path.join(HERE, "librexsim_oracle.so")
    src = os.path.join(HERE, "rexsim_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", HERE, "-s"], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    return so


_LIBS = {}


def lib(f32=False):
    if f32 not in _LIBS:
        build()
        L = C.CDLL(os.path.join(HERE, "librexsim_oracle_f32.so" if f32 else "librexsim_oracle.so"))
        L.rexo_create.restype = C.c_void_p
        L.rexo_create.argtypes = [C.POINTER(RexoModel), C.POINTER(RexoConfig)]
        L.rexo_destroy.argtypes = [C.c_void_p]
        L.rexo_obs_dim.argtypes = [C.c_void_p]
        L.rexo_action_dim.argtypes = [C.c_void_p]
        L.rexo_env.restype = C.POINTER(RexoEnv)
        L.rexo_env.argtypes = [C.c_void_p, C.c_int]
        L.rexo_reset.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.rexo_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.rexo_substep.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.rexo_physics_only.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.rexo_rand_u32.restype = C.c_uint32
        L.rexo_rand_u32.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32]
        L.rexo_sensor_clear.argtypes = [C.c_void_p, C.c_int]
        L.rexo_sensor_push.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.rexo_sensor_delayed.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_void_p]
        L.rexo_sensor_row.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.rexo_noise.restype = C.c_double
        L.rexo_noise.argtypes = [C.c_uint64] + [C.c_uint32] * 5
        L.rexo_mass_matrix.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.rexo_aba.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.rexo_kinetic_momentum.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 4
        _LIBS[f32] = L
    return _LIBS[f32]


def _rpy_to_mat(rpy):
    r, p, y = rpy
    cr, sr, cp, sp, cy, sy = math.cos(r), math.sin(r), math.cos(p), math.sin(p), math.cos(y), math.sin(y)
    rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    return rz @ ry @ rx


# Collision margin added to the toe hull's reach.  Bullet's URDF importer sets a 1 mm margin on convex hulls, but the PyBullet
# trajectories recovered from the reference's checkpoints (tests/golden/pybullet_memory/) put the touchdown of a
# robot dropped from z = 0.21 where the EXACT hull without margin reaches the ground (1 mm of margin lands one control step
# early in all 12 episodes; tools/dev_pybullet_replay.py), so the restatement uses 0.
TOE_MARGIN = float(os.environ.get("REXO_TOE_MARGIN", -0.00025))     # rex_gym_b200/model_tables.py TOE_MARGIN (same constant, same reason)


def load_model(mark="base", toes_only=False, terrain_full_toe=False):
    """Model tables (tools/compile_urdf.py output) -> RexoModel."""
    with open(os.path.join(MODEL_DIR, f"rex_{mark}.json")) as f:
        j = json.load(f)
    m = RexoModel()
    bodies = j["bodies"]
    m.nb, m.ndof = len(bodies), len(bodies) - 1
    for i, b in enumerate(bodies):
        m.parent[i] = b["parent"]
        R = _rpy_to_mat(b.get("joint_rpy", [0, 0, 0]))
        for a in range(3):
            m.jpos[i][a] = b.get("joint_xyz", [0, 0, 0])[a]
            m.axis[i][a] = b.get("axis", [1, 0, 0])[a]
            m.com[i][a] = b["com"][a]
        for a in range(9):
            m.jrot[i][a] = R.flat[a]
            m.inertia[i][a] = np.asarray(b["inertia"]).flat[a]
        m.lower[i], m.upper[i] = b.get("lower", 0.0), b.get("upper", 0.0)
        m.mass[i] = b["mass"]
    # contact groups (one contact per group): base; per leg {shoulder+leg boxes}, {foot box + toe hull}; arm bodies
    groups = [[0]] + [g for l in range(4) for g in ([1 + 3 * l, 2 + 3 * l], [3 + 3 * l])] + [[i] for i in range(13, len(bodies))]
    npts = 0
    for gi, gb in enumerate(groups):
        m.shape_start[gi] = npts
        is_foot = gi >= 1 and gi <= 8 and gi % 2 == 0
        m.shape_enabled[gi] = 1 if (is_foot or not toes_only) else 0
        for bi in gb:
            for sh in bodies[bi]["shapes"]:
                is_toe = sh["kind"] == "hull"
                if toes_only and not is_toe:
                    continue
                nprof = len(sh["points"]) // 2 if is_toe else 0      # prism toe: profile on the y_lo side, then the y_hi side
                for k, p in enumerate(sh["points"]):
                    for a in range(3):
                        m.pts[npts][a] = p[a]
                    m.pt_body[npts] = bi
                    m.pt_margin[npts] = TOE_MARGIN if is_toe else 0.0
                    # heightfield terrain samples every 4th profile vertex (+ the last one) on both sides of the prism
                    m.pt_terrain[npts] = 1 if (not is_toe or terrain_full_toe or (k % nprof) % 4 == 0 or (k % nprof) == nprof - 1) else 0
                    npts += 1
        m.shape_npts[gi] = npts - m.shape_start[gi]
    m.nshape = len(groups)
    m.root_mass = j["root_mass"]
    for a in range(3):
        m.root_inertia[a] = j["root_inertia"][a]
    m.nmotor = len(j["motor_bodies"])
    for i, bidx in enumerate(j["motor_bodies"]):
        m.motor_dof[i] = bidx - 1
    return m, j


def make_fields(nfields, seed=10):
    """Heightfield bank: field k = k-th 256x256 draw of the reference's own stream
    (rex_gym/model/terrain.py:26,36-44: random.seed(10); 2x2 blocks of U(0, 0.05))."""
    import random
    rnd = random.Random(seed)
    out = np.zeros((nfields, 256, 256), dtype=np.float32)
    for k in range(nfields):
        flat = out[k].reshape(-1)
        rows = 256
        for jj in range(128):
            for ii in range(128):
                h = rnd.uniform(0, 0.05)
                flat[2 * ii + 2 * jj * rows] = h
                flat[2 * ii + 1 + 2 * jj * rows] = h
                flat[2 * ii + (2 * jj + 1) * rows] = h
                flat[2 * ii + 1 + (2 * jj + 1) * rows] = h
    return out


class OracleSim:
    def __init__(self, num_envs=1, task="walk", signal="ik", terrain="plane", mark="base", f32=False,
                 action_repeat=None, control_time_step=None, motor_kp=1.0, motor_kd=0.02,
                 kp_range=None, kd_range=None, target_position=None, backwards=None,
                 target_orient=None, init_orient=None, energy_weight=None, normalize=False,
                 max_episode_steps=0, seed=1234, nfields=0, fields=None, toes_only=False, settle=True,
                 solver_iterations=None, residual_threshold=1e-7, env_offset=0,
                 base_y=None, base_z=None, base_roll=None, base_pitch=None, base_yaw=None, terrain_full_toe=False,
                 gait_clock_scale=1.0, max_coordinate_velocity=100.0,
                 link_damping=0.04, contact_breaking=None, control_latency=0.0, pd_latency=0.0, observation_noise_stdev=None):
        self.L = lib(f32)
        self.model, self.model_json = load_model(mark, toes_only=toes_only, terrain_full_toe=terrain_full_toe)
        c = RexoConfig()
        c.num_envs = num_envs
        c.task, c.signal, c.terrain = TASKS[task], SIGNALS[signal], TERRAINS[terrain]
        rep = action_repeat or (6 if task in ("gallop", "poses") else 5)
        cts = control_time_step or (0.006 if task in ("gallop", "poses") else 0.005)
        c.action_repeat = rep
        c.sim_dt = cts / rep
        c.solver_iterations = solver_iterations or int(300 / rep)
        c.motor_kp, c.motor_kd = motor_kp, motor_kd
        # randomisation bounds travel through the C ABI as float32: round them the same way here
        c.kp_lo, c.kp_hi = [float(np.float32(x)) for x in kp_range] if kp_range else (motor_kp, motor_kp)
        c.kd_lo, c.kd_hi = [float(np.float32(x)) for x in kd_range] if kd_range else (motor_kd, motor_kd)
        c.target_position = float("nan") if target_position is None else target_position
        c.backwards = -1 if backwards is None else int(bool(backwards))
        c.target_orient = float("nan") if target_orient is None else target_orient
        c.init_orient = float("nan") if init_orient is None else init_orient
        c.w_distance, c.w_drift, c.w_shake = 1.0, 2.0, 0.005
        c.w_energy = energy_weight if energy_weight is not None else (0.005 if task == "gallop" else 0.0005)
        c.normalize, c.max_episode_steps, c.seed = int(normalize), max_episode_steps, seed
        self.fields = None
        if terrain == "random":
            self.fields = np.ascontiguousarray(fields if fields is not None else make_fields(nfields or 4))
            c.nfields = self.fields.shape[0]
            c.fields = self.fields.ctypes.data_as(C.POINTER(C.c_float))
            c.friction = 0.5 * 0.5      # link default 0.5 x createMultiBody default 0.5
        else:
            c.nfields = 0
            c.friction = 0.5 * 1.0      # link default 0.5 x plane.urdf lateral_friction 1
        c.residual_threshold = residual_threshold
        c.erp_contact, c.erp_joint = 0.08, 0.2
        c.settle_on_reset = int(settle)
        c.env_offset = int(env_offset)
        c.gait_clock_scale = float(gait_clock_scale)
        c.max_coordinate_velocity = float(max_coordinate_velocity)
        c.link_damping = float(link_damping)
        c.control_latency, c.pd_latency = float(control_latency), float(pd_latency)
        for k, v in enumerate(observation_noise_stdev or (0.0,) * 5):      # SENSOR_NOISE_STDDEV rex.py:22
            c.noise_stdev[k] = float(v)
        if contact_breaking is None:       # the Bullet-derived manifold threshold of the toe shape (0.81 mm)
            from rex_gym_b200.model_tables import contact_breaking_distance
            contact_breaking = contact_breaking_distance(mark)
        c.contact_breaking = float(os.environ.get("REXO_BREAKING", contact_breaking))
        for k, v in enumerate((base_y, base_z, base_roll, base_pitch, base_yaw)):
            c.pose_values[k] = float("nan") if v is None else float(v)
        self.cfg = c
        self.h = self.L.rexo_create(C.byref(self.model), C.byref(c))
        self.N = num_envs
        self.O = self.L.rexo_obs_dim(self.h)
        self.A = self.L.rexo_action_dim(self.h)
        self.nm = self.model.nmotor

    def __del__(self):
        try:
            self.L.rexo_destroy(self.h)
        except Exception:
            pass

    def env(self, i):
        return self.L.rexo_env(self.h, i).contents

    def reset(self, indices=None):
        if indices is None:
            obs = np.zeros((self.N, self.O), np.float32)
            self.L.rexo_reset(self.h, None, self.N, obs.ctypes.data)
        else:
            idx = np.ascontiguousarray(indices, np.int32)
            obs = np.zeros((len(idx), self.O), np.float32)
            self.L.rexo_reset(self.h, idx.ctypes.data, len(idx), obs.ctypes.data)
        return obs

    def step(self, actions, nthreads=1):
        a = np.ascontiguousarray(actions, np.float32).reshape(self.N, self.A)
        obs = np.zeros((self.N, self.O), np.float32)
        rew = np.zeros(self.N, np.float32)
        done = np.zeros(self.N, np.uint8)
        self.L.rexo_step(self.h, a.ctypes.data, obs.ctypes.data, rew.ctypes.data, done.ctypes.data, nthreads)
        return obs, rew, done.astype(bool)

    def transform_action(self, action, i=0):
        a = np.zeros(8)
        a[:len(action)] = action
        cmd = np.zeros(MAXDOF)
        self.L.rexo_transform_action(C.c_void_p(self.h), i, a.ctypes.data_as(C.c_void_p), cmd.ctypes.data_as(C.c_void_p))
        return cmd[:self.nm]

    def apply_action(self, i, cmd):
        c = np.zeros(MAXDOF); c[:self.nm] = cmd
        tau = np.zeros(MAXDOF)
        self.L.rexo_apply_action(C.c_void_p(self.h), i, c.ctypes.data_as(C.c_void_p), tau.ctypes.data_as(C.c_void_p))
        return tau[:self.nm]

    def wrap_action(self, action):
        a = np.zeros(8); a[:self.A] = action
        out = np.zeros(8)
        self.L.rexo_wrap_action(C.c_void_p(self.h), a.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
        return out[:self.A]

    def wrap_observation(self, raw):
        r = np.zeros(4 + MAXDOF); r[:self.O] = raw
        out = np.zeros(4 + MAXDOF, np.float32)
        self.L.rexo_wrap_observation(C.c_void_p(self.h), r.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
        return out[:self.O]

    def reward_done_obs(self, i=0):
        r, d = C.c_double(), C.c_int()
        obs = np.zeros(4 + MAXDOF)
        self.L.rexo_reward_done_obs(C.c_void_p(self.h), i, C.byref(r), C.byref(d), obs.ctypes.data_as(C.c_void_p))
        return r.value, bool(d.value), obs[:self.O]

    def sensor_history(self, i):
        """-> [len][3 nm + 7] env i's observation history, newest row first (rex.py:726-733 deque; q, qd, torque, quat, rpy rate)."""
        w = 3 * self.nm + 7
        row = np.zeros(w)
        n = self.L.rexo_sensor_row(self.h, i, 0, row.ctypes.data)
        out = np.zeros((n, w))
        for k in range(n):
            self.L.rexo_sensor_row(self.h, i, k, out[k].ctypes.data)
        return out

    def substep(self, i, cmd):
        c = np.ascontiguousarray(cmd, np.float64)
        self.L.rexo_substep(self.h, i, c.ctypes.data)

    def physics_only(self, i, tau):
        t = np.ascontiguousarray(tau, np.float64)
        self.L.rexo_physics_only(self.h, i, t.ctypes.data)

    def state(self, i=0):
        e = self.env(i)
        nd = self.model.ndof
        return dict(pos=np.array(e.pos), quat=np.array(e.quat), linvel=np.array(e.linvel), angvel=np.array(e.angvel),
                    q=np.array(e.q[:nd]), qd=np.array(e.qd[:nd]))

    def states(self):
        """state() of every env, batched: {key: [N][...]}."""
        st = [self.state(i) for i in range(self.N)]
        return {k: np.stack([s[k] for s in st]) for k in st[0]}

    def set_state(self, i, st):
        """Write a physical state (the keys of state()) into env i."""
        e = self.env(i)
        for k in ("pos", "quat", "linvel", "angvel", "q", "qd"):
            getattr(e, k)[:len(st[k])] = [float(x) for x in st[k]]

    def mass_matrix_inv(self, i=0):
        nd = 6 + self.model.ndof
        M = np.zeros((nd, nd))
        self.L.rexo_mass_matrix(self.h, i, M.ctypes.data)
        return M

    def aba(self, tau, i=0):
        nd = 6 + self.model.ndof
        out = np.zeros(nd)
        t = np.ascontiguousarray(tau, np.float64)
        self.L.rexo_aba(self.h, i, t.ctypes.data, out.ctypes.data)
        return out

    def momentum(self, i=0):
        ke = C.c_double()
        lin, ang, com = np.zeros(3), np.zeros(3), np.zeros(3)
        self.L.rexo_kinetic_momentum(self.h, i, C.byref(ke), lin.ctypes.data, ang.ctypes.data, com.ctypes.data)
        return ke.value, lin, ang, com


# unit-level controller entry points ---------------------------------------------------------
def motor_torque(cmd, q, qd, qd_true, kp, kd):
    L = lib()
    n = len(cmd)
    arrs = [np.ascontiguousarray(np.broadcast_to(x, (n,)), np.float64) for x in (cmd, q, qd, qd_true, kp, kd)]
    ta, to = np.zeros(n), np.zeros(n)
    L.rexo_motor_torque(n, *[a.ctypes.data_as(C.c_void_p) for a in arrs], ta.ctypes.data_as(C.c_void_p), to.ctypes.data_as(C.c_void_p))
    return ta, to


def ik_solve(rpy, pos, frames):
    L = lib()
    r, p, f = (np.ascontiguousarray(x, np.float64) for x in (rpy, pos, frames))
    out = np.zeros((4, 3))
    L.rexo_ik_solve(r.ctypes.data_as(C.c_void_p), p.ctypes.data_as(C.c_void_p), f.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    return out


class GaitState:
    def __init__(self, mode="walk"):
        self.phi, self.last_time, self.alpha = C.c_double(0), C.c_double(0), C.c_double(0)
        self.gallop = int(mode != "walk")

    def loop(self, now, v, angle, w_rot, T, direction, frames=None):
        L = lib()
        L.rexo_gait_loop.argtypes = [C.c_void_p] * 3 + [C.c_int] + [C.c_double] * 6 + [C.c_void_p] * 2
        out = np.zeros((4, 3))
        fp = None
        if frames is not None:
            fr = np.ascontiguousarray(frames, np.float64)
            fp = fr.ctypes.data_as(C.c_void_p)
        L.rexo_gait_loop(C.byref(self.phi), C.byref(self.last_time), C.byref(self.alpha), self.gallop,
                         float(now), float(v), float(angle), float(w_rot), float(T), float(direction), fp,
                         out.ctypes.data_as(C.c_void_p))
        return out


def bezier_swing(phi, v, angle, direction):
    L = lib()
    L.rexo_bezier_swing.argtypes = [C.c_double] * 4 + [C.c_void_p]
    out = np.zeros(3)
    L.rexo_bezier_swing(phi, v, angle, direction, out.ctypes.data_as(C.c_void_p))
    return out


def stance(phi, v, angle):
    L = lib()
    L.rexo_stance.argtypes = [C.c_double] * 3 + [C.c_void_p]
    out = np.zeros(3)
    L.rexo_stance(phi, v, angle, out.ctypes.data_as(C.c_void_p))
    return out

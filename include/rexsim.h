/* rexsim.h -- C ABI of the H100-native batched Rex simulator (librexsim.so).
 *
 * Drop-in boundary for rex-gym's per-step hot path.  The reference has no FFI of its own for this
 * path: its native boundary is pybullet's C-API reached through BulletClient.__getattr__
 * (rex_gym/util/bullet_client.py:40-54), crossed ~265 times per env-step
 * (rex_gym/model/rex.py:158-163,326-330,451,477,545).  Each entry point below replaces a whole
 * group of those crossings for N environments at once:
 *
 *   rexsim_create   <- RexGymEnv.__init__ world setup: resetSimulation / setPhysicsEngineParameter /
 *                      setTimeStep / loadURDF / setGravity      (rex_gym/envs/rex_gym_env.py:304-339)
 *   rexsim_reset    <- BatchEnv.reset(indices) -> <task>.reset -> Rex.Reset (settle) + task draws
 *                      (rex_gym/agents/tools/batch_env.py:92-109; rex_gym/model/rex.py:255-324;
 *                       rex_gym/envs/gym/walk_env.py:125-154)
 *   rexsim_step     <- BatchEnv.step(actions) -> RexGymEnv.step: signal -> Rex.Step x action_repeat
 *                      (ApplyAction + stepSimulation + ReceiveObservation) -> reward/termination/obs
 *                      (rex_gym/agents/tools/batch_env.py:63-90; rex_gym/envs/rex_gym_env.py:369-414)
 *   rexsim_get_state / rexsim_set_state
 *                   <- getBasePositionAndOrientation / getBaseVelocity / getJointState /
 *                      resetBasePositionAndOrientation / resetJointState (rex_gym/model/rex.py:297-299,
 *                      360-372,416,451,545) -- used for golden comparison and checkpoint/resume
 *   rexsim_destroy  <- RexGymEnv.close (rex_gym/envs/rex_gym_env.py:287-291)
 *
 * Conventions: plain C, no exceptions; every function returns 0 or a negative RexSimStatus.
 * All array arguments marked "dev" are DEVICE pointers owned by the caller; the library borrows them
 * for the duration of the enqueue.  All work is enqueued on the cudaStream_t passed as `void* stream`
 * (NULL = legacy default stream); nothing synchronises the host except rexsim_create.
 * A handle is not re-entrant (one stream at a time).
 */
#ifndef REXSIM_H
#define REXSIM_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    REXSIM_OK = 0,
    REXSIM_ERR_INVALID = -1,      /* bad argument / unsupported configuration */
    REXSIM_ERR_MODEL = -2,        /* model tables do not have the Rex leg structure the kernels assume */
    REXSIM_ERR_CUDA = -3,         /* CUDA runtime error (see rexsim_last_error) */
    REXSIM_ERR_UNSUPPORTED = -4,  /* valid reference configuration not built yet */
} RexSimStatus;

enum { REXSIM_TASK_WALK = 0, REXSIM_TASK_GALLOP = 1, REXSIM_TASK_TURN = 2, REXSIM_TASK_STANDUP = 3,
       REXSIM_TASK_POSES = 4 /* RexPosesEnv, rex_gym/envs/gym/poses_env.py:21 */ };
enum { REXSIM_SIGNAL_IK = 0, REXSIM_SIGNAL_OL = 1 };
enum { REXSIM_TERRAIN_PLANE = 0, REXSIM_TERRAIN_RANDOM = 1 };

/* per-env device error bits (rexsim_step ORs them into err_flags[env]) */
enum {
    REXSIM_FLAG_NONFINITE = 1,        /* non-finite state/obs/reward (ConvertTo32Bit raises, wrappers.py:522,542) */
    REXSIM_FLAG_JOINT_LIMIT = 2,      /* reserved (every violated joint limit has its own row since round 2) */
    REXSIM_FLAG_BODY_CONTACT = 4,     /* reserved (body contacts are solved since the generic row path exists) */
    REXSIM_FLAG_TILE_MISS = 8,        /* a contact query fell outside the 0.8 m heightfield window staged in shared memory */
    REXSIM_FLAG_BAD_INDEX = 16,       /* rexsim_reset saw an index outside [0, N): skipped (aggregate word only) */
};

#define REXSIM_MAX_TOE_PTS 96
/* float offsets inside the model table (see rex_gym_b200/model_tables.py for the packer) */
#define REXSIM_MT_BASE 0            /* mass, com[3], inertia[6](xx,yy,zz,xy,xz,yz), root_mass, root_inertia[3], diag flag, toe half width */
#define REXSIM_MT_LEG 16            /* [4 legs][3 bodies][16]: jpos[3], mass, com[3], lower, inertia[6], upper, diag flag */
#define REXSIM_MT_TOE (16 + 192)    /* 384 floats: [toe_npts <= REXSIM_MAX_TOE_PTS][2] (x, z) profile of the toe prism in the foot-body frame
                                     * (the hull of stl/foot.stl is this profile extruded over y in [-w, w]; identical on the 4 feet) */
#define REXSIM_MT_BOX (16 + 192 + 384)         /* [4 legs][3 bodies][8 corners][3] collision box corners, body frame */
#define REXSIM_MT_BASEBOX (16 + 192 + 384 + 288) /* [3 boxes][8][3] base + chassis boxes */
#define REXSIM_MT_FLOATS (16 + 192 + 384 + 288 + 72)
#define REXSIM_MT_ARM REXSIM_MT_FLOATS  /* mark 'arm' only: [6 bodies][32]: jpos[3], jrot[9] (child->parent, row-major), axis[3],
                                         * mass, com[3], inertia[6], lower, upper, pad[5] */
#define REXSIM_MT_FLOATS_ARM (REXSIM_MT_FLOATS + 192)

typedef struct {
    int32_t num_envs;
    int32_t task, signal, terrain;
    int32_t num_motors;               /* 12 (mark 'base') or 18 (mark 'arm': model table has REXSIM_MT_FLOATS_ARM floats) */
    int32_t action_repeat;
    int32_t solver_iterations;        /* int(300 / action_repeat) (rex_gym_env.py:25,184) */
    float sim_dt;                     /* control_time_step / action_repeat (unused: sim_dt_d is authoritative) */
    double sim_dt_d;
    float motor_kp, motor_kd;
    float kp_lo, kp_hi, kd_lo, kd_hi; /* per-env gains drawn at reset when lo != hi */
    float target_position;            /* NaN: random per reset */
    int32_t backwards;                /* -1 random, 0, 1 */
    float target_orient, init_orient; /* NaN: random per reset */
    float w_distance, w_energy, w_drift, w_shake;
    int32_t normalize;                /* ClipAction + RangeNormalize fused (wrappers.py:183-265) */
    int32_t max_episode_steps;        /* LimitDuration (wrappers.py:268-291), 0 = off */
    int32_t auto_reset;               /* 1: done envs are reset at the end of rexsim_step; obs = reset obs */
    uint64_t seed;
    int32_t nfields;                  /* heightfield bank (terrain RANDOM) */
    const float* fields;              /* dev [nfields][256*256], heights in metres (terrain.py:36-53) */
    float friction;                   /* combined link x ground lateral friction */
    float residual_threshold;         /* solver early-out (pybullet default 1e-7) */
    float erp_contact, erp_joint;
    int32_t toe_npts;                 /* profile vertices of the toe prism in the model table */
    float toe_margin;                 /* added to the toe hull's reach [m]; -0.25 mm: identified on the recorded PyBullet touchdown (DESIGN.md 3) */
    float contact_breaking;           /* manifold breaking distance: a contact row exists while the distance is below it (0.81 mm) */
    float link_damping;               /* btMultiBody m_linearDamping = m_angularDamping (0.04), applied to every link */
    float max_coordinate_velocity;    /* btMultiBody m_maxCoordinateVelocity (100): clamp on all generalised velocities */
    int32_t env_offset;               /* global id of env 0 of this shard (multi-GPU): reset draws key on the global id */
    double gait_clock_scale;          /* GaitPlanner clock = simulation time x this.  1 = the deterministic simulation clock (DESIGN.md
                                       * section 2).  The reference reads the WALL clock (gait_planner.py:108-110); the walk-ik episodes stored
                                       * in its shipped checkpoint ran at about 9 (tests/test_pybullet_goldens.py) */
    float pose_values[5];             /* poses task: base_y, base_z, base_roll, base_pitch, base_yaw constructor arguments
                                       * (poses_env.py:49-53); all NaN = None: the pose rotates per reset, target drawn in range */
    /* sensor model (rex_gym/model/rex.py:122,726-769; constructor arguments rex_gym_env.py:61,70-71).  All zero = the reference
     * default: no history is kept and the kernels read the true state.  Otherwise every sub-step pushes the true observation
     * [q, qd, observed torque, base quaternion, base angular velocity] into a per-env ring of the deque's depth (<= 100 rows);
     * the PD loop reads it pd_latency ago, the controller / reward / termination / observation control_latency ago (linear
     * blend of the two neighbouring rows), plus Gaussian noise.  np.random.normal (unseeded upstream) is replaced by a
     * counter-based N(0,1) keyed on (seed, global env, reset count, control step, call site, component): include/rexsim.h
     * rexsim_noise is the same generator host-side. */
    double control_latency, pd_latency;   /* seconds */
    double noise_stdev[5];                /* SENSOR_NOISE_STDDEV order (rex.py:22): motor angle, velocity, torque, base rpy, rpy rate */
} RexSimConfig;

typedef struct RexSim RexSim;

/* observation / action widths for a task (no handle needed) */
int rexsim_obs_dim(int32_t task, int32_t num_motors);
int rexsim_action_dim(int32_t task, int32_t signal);
/* words per env of the SoA state: float words, int words */
int rexsim_state_words(const RexSimConfig* cfg, int32_t* n_float, int32_t* n_int);

/* model_tables: HOST pointer to REXSIM_MT_FLOATS (12 motors) or REXSIM_MT_FLOATS_ARM (18 motors) floats.  Allocates device state, computes the settled
 * reset snapshot(s) (600 physics sub-steps, rex.py:314-323) and synchronises. */
int rexsim_create(const RexSimConfig* cfg, const float* model_tables, int32_t n_model_floats, RexSim** out);
void rexsim_destroy(RexSim* sim);

/* actions dev [N][A] f32; obs dev [N][O] f32; reward dev [N] f32; done dev [N] u8 */
int rexsim_step(RexSim* sim, const float* actions, float* obs, float* reward, uint8_t* done, void* stream);
/* Host-buffer form of rexsim_step -- BatchEnv.step with numpy arrays (batch_env.py:63-90): h_actions HOST [N][A] f32,
 * h_out HOST block of rexsim_host_out_bytes() bytes laid out as obs [N][O] f32 | reward [N] f32 | done [N] u8 | pad to 4 |
 * int32 OR of all error flags | 8 scratch bytes (the kernel's flag bytes on the zero-copy path).  One call = H2D copy of the actions, the step kernel, one D2H copy of the results (+4 bytes of
 * flags) on `stream`, then a wait for that stream.  Pinned (page-locked) host memory gives the full copy speed; with pinned buffers
 * and N <= 16384 the kernel addresses the host block directly (zero-copy) and the two bulk copies disappear. */
int64_t rexsim_host_out_bytes(const RexSim* sim);
int rexsim_step_host(RexSim* sim, const float* h_actions, void* h_out, void* stream);
/* Re-group the environments over the warps by the solver cost of their last control step (counting sort on the device, three
 * small launches).  The step kernel's cost per env is dominated by its PGS iteration count, and a warp of 8 envs runs as long
 * as its slowest one; in a de-synchronised batch (auto-reset) grouping envs of similar cost recovers most of that loss.
 * Purely a scheduling hint: every env's results are bit-identical with and without it.  Call every few steps (the
 * Python mirror does it every 8 for batches of >= 8192 envs; a batch that fits one wave gains nothing). */
int rexsim_rebalance(RexSim* sim, void* stream);
/* idx dev [k] int32 (NULL: all envs, k ignored); obs_out dev [k][O] or NULL */
int rexsim_reset(RexSim* sim, const int32_t* idx, int32_t k, float* obs_out, void* stream);

/* Physical state of every env, SoA on device: out_f dev [13 + 2*nm][N] =
 *   pos[3], quat[4] (x,y,z,w), linvel[3], angvel[3], q[nm], qd[nm];  out_i dev [4][N] =
 *   step_counter, env_step_counter, flags, last-substep contact mask (bit 0: base group, bit 1+2l: shoulder/leg
 *   boxes of leg l, bit 2+2l: foot box + toe hull of leg l) */
int rexsim_get_state(RexSim* sim, float* out_f, int32_t* out_i, void* stream);
int rexsim_set_state(RexSim* sim, const float* in_f, void* stream);
/* raw SoA state for checkpoint/resume: [n_float][N] f32 and [n_int][N] i32 device buffers */
int rexsim_state_buffers(RexSim* sim, float** state_f, int32_t** state_i);
/* sensor history ring (sensor model on): dev [depth][words][N] f32, words = 43 (61 with the arm); n_floats = 0 and ring = NULL when
 * the model is off.  Part of an exact checkpoint together with the state buffers. */
int rexsim_history_buffer(RexSim* sim, float** ring, int64_t* n_floats);
/* dev [N + 1] int32: word e = error bits of env e's most recent step (cleared by a reset of that env); word N = OR of every
 * bit raised since it was last cleared.  rexsim_step_host clears the aggregate after copying it out (per-step semantics, like
 * ConvertTo32Bit raising for the offending step only, wrappers.py:522-543); device-path callers use rexsim_clear_errors. */
int rexsim_error_flags(RexSim* sim, int32_t** err_flags);
int rexsim_clear_errors(RexSim* sim, void* stream);          /* zeroes the aggregate word (enqueued on stream) */
/* last motor command of every env (info['action'], rex_gym_env.py:414): dev [nm][N] */
int rexsim_last_command(RexSim* sim, float** cmd);
/* solver cost of every env's last control step (what rexsim_rebalance sorts by): dev [N] int32, the PGS iterations of its sub-steps
 * plus 64 per sub-step on the generic path */
int rexsim_solver_cost(RexSim* sim, int32_t** cost);
/* kernels launched by this handle since create (the bench reports it) */
int64_t rexsim_launch_count(const RexSim* sim);
/* which build of the step kernel the last rexsim_step / rexsim_step_host launched (all 0 before the first step): CTA size,
 * resident CTAs per SM it is compiled for (1: 255 registers, 4: 128 registers), 1 if the sensor model is compiled in */
int rexsim_last_step_build(const RexSim* sim, int32_t* cta_threads, int32_t* ctas_per_sm, int32_t* sensor);
/* the counter-based generator behind every reset draw (replaces Python's unseeded `random`,
 * walk_env.py:133-147, gallop_env.py:151, turn_env.py:138,147); host-callable so tests can pin it */
uint32_t rexsim_rand_u32(uint64_t seed, uint32_t global_env, uint32_t reset_count, uint32_t slot);
/* the N(0,1) draw behind the sensor noise (replaces the unseeded np.random.normal of Rex._AddSensorNoise, rex.py:763-769):
 * Box-Muller on two draws of the generator above, slots 1024 + 2*((step*8 + site)*32 + comp) and +1.  Sites: 0 observation rpy,
 * 1 observation rpy rate, 2 observation motor angles, 3 reward orientation, 4 reward torques, 5 reward velocities,
 * 6 termination orientation, 7 turn goal-check orientation.  (float arithmetic, as on the device) */
float rexsim_noise(uint64_t seed, uint32_t global_env, uint32_t reset_count, uint32_t control_step, uint32_t site, uint32_t comp);
/* rows per env of the sensor history ring this configuration keeps (0: sensor model off) */
int rexsim_history_depth(const RexSimConfig* cfg);
const char* rexsim_last_error(void);

#ifdef __cplusplus
}
#endif
#endif

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
 *   rexsim_step_final
 *                   <- the same, plus the terminal observation BatchEnv.step returns and gym TimeLimit's
 *                      info['TimeLimit.truncated'] (in_graph_batch_env.py:71-92; gym 0.17.1 wrappers/time_limit.py)
 *   rexsim_get_state / rexsim_set_state
 *                   <- getBasePositionAndOrientation / getBaseVelocity / getJointState /
 *                      resetBasePositionAndOrientation / resetJointState (rex_gym/model/rex.py:297-299,
 *                      360-372,416,451,545) -- used for golden comparison and checkpoint/resume
 *   rexsim_episode_summary
 *                   <- simulate()'s score / length bookkeeping and its StreamingMeans (rex_gym/agents/tools/simulate.py:57-113,
 *                      streaming_mean.py), RexGymEnv.get_objectives (rex_gym_env.py:538-547); kept by rexsim_step when
 *                      RexSimConfig.episode_stats is set
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
                                         * mass, com[3], inertia[6], lower, upper, npts, start, reach (largest point
                                         * distance from the body origin), pad[2] */
#define REXSIM_MT_ARMPTS (REXSIM_MT_FLOATS + 192)   /* mark 'arm' only: [104][3] collision points of the six arm bodies, body frame
                                                     * (16 per cylinder, 8 box corners), body by body; [start, start + npts) above */
#define REXSIM_MT_ARMPTS_N 104
#define REXSIM_MT_FLOATS_ARM (REXSIM_MT_ARMPTS + 3 * REXSIM_MT_ARMPTS_N)

/* float offsets inside the render table (rex_gym_b200/model_tables.py pack_render_tables): everything visual */
#define REXSIM_RT_NSHAPES 26        /* 3 base boxes, 12 leg boxes (leg-major: shoulder, leg, foot), 4 toes, 6 arm cylinders, arm box */
#define REXSIM_RT_LIGHT 0           /* unit direction towards the light [3], ambient, diffuse weight (Lambert + ambient) */
#define REXSIM_RT_SKY 5             /* rgb of misses and of hits outside [near, far] */
#define REXSIM_RT_CHECK 8           /* ground checker: two rgb tones, square size [m] */
#define REXSIM_RT_CAM 15            /* vertical field of view [deg], near, far */
#define REXSIM_RT_COLOR 18          /* [REXSIM_RT_NSHAPES][3] rgb: URDF visual material of each shape's link */
#define REXSIM_RT_TOE 96            /* [toe_npts <= REXSIM_MAX_TOE_PTS][3] edge planes (nx, nz, d) of the toe profile, foot frame */
#define REXSIM_RT_TOESPH 384        /* bounding sphere of the toe prism in the foot frame: centre x, centre z, radius, pad */
#define REXSIM_RT_CYL 388           /* mark 'arm': [6 arm bodies][8] cylinder centre[3], axis[3], radius, half length, body frame */
#define REXSIM_RT_ARMBOX 436        /* mark 'arm': arm body index of the box, then its [8][3] corners in that body's frame */
#define REXSIM_RT_FLOATS 464

typedef struct {
    int32_t num_envs;
    int32_t task, signal, terrain;
    int32_t num_motors;               /* 12 (mark 'base') or 18 (mark 'arm': model table has REXSIM_MT_FLOATS_ARM floats; every
                                         task but gallop, whose observation would carry the 18 motor angles) */
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
    /* 1: keep simulate()'s episode bookkeeping on the device (rex_gym/agents/tools/simulate.py:57-113): every step adds its
     * reward to the env's score and counts its length; a step that returns done submits the episode to per-env accumulators
     * (episode count, score sum, length sum) and restarts both, with or without auto_reset.  An episode ending on a step that
     * raises REXSIM_FLAG_NONFINITE is counted apart and not submitted.  Walk and gallop also record the unweighted objectives
     * [forward, energy, drift, shake] of every step (RexGymEnv._reward, rex_gym_env.py:501-555).  See rexsim_episode_buffers /
     * rexsim_episode_summary.  0: nothing is allocated and every output is what it is without the switch. */
    int32_t episode_stats;
} RexSimConfig;

typedef struct RexSim RexSim;

/* observation / action widths for a task (no handle needed) */
int rexsim_obs_dim(int32_t task, int32_t num_motors);
int rexsim_action_dim(int32_t task, int32_t signal);
/* words per env of the SoA state: float words, int words */
int rexsim_state_words(const RexSimConfig* cfg, int32_t* n_float, int32_t* n_int);

/* model_tables: HOST pointer to REXSIM_MT_FLOATS (12 motors) or REXSIM_MT_FLOATS_ARM (18 motors) floats.  Allocates device state, computes the settled
 * reset snapshot(s) (600 physics sub-steps, rex.py:314-323; one launch, one snapshot per field) and synchronises.
 * Returns REXSIM_ERR_UNSUPPORTED when floor(1 / sim_dt_d) >= 1023: the overheat protection (rex.py:601-608) switches a motor off
 * once it has been hot for more than floor(1 / sim_dt) sub-steps, and its per-motor counter is a 10-bit field that stops at 1023.
 * Time steps of 1/1023 s and below are refused; every configuration of the reference (1 ms) is accepted. */
int rexsim_create(const RexSimConfig* cfg, const float* model_tables, int32_t n_model_floats, RexSim** out);
void rexsim_destroy(RexSim* sim);

/* actions dev [N][A] f32; obs dev [N][O] f32 (O = rexsim_out_dim); reward dev [N] f32; done dev [N] u8 */
int rexsim_step(RexSim* sim, const float* actions, float* obs, float* reward, uint8_t* done, void* stream);
/* Host-buffer form of rexsim_step -- BatchEnv.step with numpy arrays (batch_env.py:63-90): h_actions HOST [N][A] f32,
 * h_out HOST block of rexsim_host_out_bytes() bytes laid out as obs [N][O] f32 | reward [N] f32 | done [N] u8 | pad to 4 |
 * int32 OR of all error flags | 8 scratch bytes (the kernel's flag bytes on the zero-copy path).  One call = H2D copy of the actions, the step kernel, one D2H copy of the results (+4 bytes of
 * flags) on `stream`, then a wait for that stream.  Pinned (page-locked) host memory gives the full copy speed; with pinned buffers
 * and N <= 16384 the kernel addresses the host block directly (zero-copy) and the two bulk copies disappear. */
int64_t rexsim_host_out_bytes(const RexSim* sim);
int rexsim_step_host(RexSim* sim, const float* h_actions, void* h_out, void* stream);
/* rexsim_step plus the two outputs an auto-resetting step would otherwise lose (the reference's BatchEnv.step returns the
 * terminal observation and resets at the top of the next iteration, simulate.py:67-75, in_graph_batch_env.py:71-113; gym's
 * TimeLimit tells a time-limit cut from a termination, gym 0.17.1 wrappers/time_limit.py).  Either may be NULL:
 *   final_obs dev [N][O] f32 (O = rexsim_out_dim): for every env whose step returned done, the observation `obs` would hold with
 *     auto_reset = 0 (RangeNormalize, the sensor model's delayed noisy reads and the frame wrappers included); rows of the other
 *     envs are left untouched.
 *   limit dev [N] u8, written for every env: bit 0 = max_episode_steps was reached at this step; bit 1 = the episode also ended
 *     for another reason (the task's termination or the non-finite guard).  TimeLimit's info['TimeLimit.truncated'] is present
 *     iff bit 0 is set, with the value !(bit 1).
 * rexsim_step launches exactly what it launched before this entry point existed. */
int rexsim_step_final(RexSim* sim, const float* actions, float* obs, float* reward, uint8_t* done, float* final_obs,
                      uint8_t* limit, void* stream);
/* Host-buffer form of rexsim_step_final: h_out as in rexsim_step_host, h_final HOST block of rexsim_host_final_bytes() bytes laid out
 * as final obs [N][O] f32 | limit [N] u8.  Zero-copy when all three buffers are pinned and N <= 16384; otherwise the kernel writes
 * a device staging block that is copied out whole, so the rows of envs that did not end hold what that path last wrote there.
 * Either way a caller that keeps one block and one path gets the bytes rexsim_step_final writes into a device block. */
int64_t rexsim_host_final_bytes(const RexSim* sim);
int rexsim_step_host_final(RexSim* sim, const float* h_actions, void* h_out, void* h_final, void* stream);
/* Re-group the environments over the warps by the solver cost of their last control step (counting sort on the device, three
 * small launches).  The step kernel's cost per env is dominated by its PGS iteration count, and a warp of 8 envs runs as long
 * as its slowest one; in a de-synchronised batch (auto-reset) grouping envs of similar cost recovers most of that loss.
 * Purely a scheduling hint: every env's results are bit-identical with and without it.  Call every few steps (the
 * Python mirror does it every 8 for batches of >= 8192 envs; a batch that fits one wave gains nothing). */
int rexsim_rebalance(RexSim* sim, void* stream);
/* idx dev [k] int32 (NULL: all envs, k ignored); obs_out dev [k][O] (O = rexsim_out_dim) or NULL */
int rexsim_reset(RexSim* sim, const int32_t* idx, int32_t k, float* obs_out, void* stream);

/* Physical state of every env, SoA on device: out_f dev [13 + 2*nm][N] =
 *   pos[3], quat[4] (x,y,z,w), linvel[3], angvel[3], q[nm], qd[nm];  out_i dev [4][N] =
 *   step_counter, env_step_counter, flags, last-substep contact mask (bit 0: base group, bit 1+2l: shoulder/leg
 *   boxes of leg l, bit 2+2l: foot box + toe hull of leg l, bits 9..14: arm bodies 0..5 of mark 'arm') */
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
/* Render table (REXSIM_RT_FLOATS floats, HOST pointer): copied into the buffer rexsim_create allocated for it; synchronous.
 * Kept out of RexSimConfig so that the configuration the step kernels receive stays as it is. */
int rexsim_set_render_tables(RexSim* sim, const float* render_tables, int32_t n_floats);
/* RexGymEnv.render(mode="rgb_array") (rex_gym_env.py:416-439) for k envs at once: idx dev [k] int32, rgb dev [k][height][width][3]
 * uint8, row 0 at the top.  Ray-casts the collision geometry of each env from its state through the reference's follow camera
 * (target = base position; distance [m], yaw and pitch [deg]; the lens of the render table).  Reads the state only.  Sizes
 * 1..4096 per side, k >= 0.  An index outside [0, N) gives a sky image and sets REXSIM_FLAG_BAD_INDEX in the aggregate word. */
int rexsim_render(RexSim* sim, const int32_t* idx, int32_t k, int32_t width, int32_t height, float distance, float yaw_deg,
                  float pitch_deg, uint8_t* rgb, void* stream);
/* Episode statistics (RexSimConfig.episode_stats = 1), device pointers owned by the handle:
 *   score dev [N] f32, length dev [N] int32: the running episode of every env (rexsim_reset zeroes those of the envs it resets
 *     and submits nothing, as simulate(reset=True) does);
 *   objectives dev [4][N] f32: forward, energy, drift, shake of every env's last step, before the task's weights (walk and
 *     gallop; NULL for turn, standup and poses, whose reward has no objectives);
 *   summary dev [4] f64: count, nonfinite, sum of scores, sum of lengths, written by rexsim_episode_summary;
 *   block / block_bytes: the one allocation behind score and length and the per-env accumulators, indexed by env:
 *     sum_score f64 [N] | sum_length i64 [N] | score f32 [N] | length i32 [N] | count i32 [N] | nonfinite i32 [N].
 *     Part of an exact checkpoint together with the state buffers.
 * REXSIM_ERR_INVALID when the switch is off. */
int rexsim_episode_buffers(RexSim* sim, float** score, int32_t** length, float** objectives, double** summary, void** block,
                           int64_t* block_bytes);
/* StreamingMean.submit's totals (simulate.py:90-106, streaming_mean.py:45-60) over the whole batch into the summary block: episodes submitted, episodes
 * ended non-finite, score sum, length sum (sums, not means, so that shards can add them).  The reduction order is fixed (one CTA,
 * thread t sums envs t, t + 1024, ... in order, then a fixed tree): repeated runs give bit-identical sums whatever the device,
 * the rebalancing or the launch history.  clear != 0 also zeroes the accumulators (StreamingMean.clear); running episodes go
 * on.  One launch on `stream`; REXSIM_ERR_INVALID when the switch is off. */
int rexsim_episode_summary(RexSim* sim, int32_t clear, void* stream);
/* Frame wrappers (rex_gym/agents/tools/wrappers.py:93-181), fused into rexsim_step and rexsim_reset as
 *   ConvertTo32Bit(FrameHistory(FrameDelta(ClipAction(RangeNormalize(LimitDuration(env))))))
 * (RangeNormalize and ClipAction only with RexSimConfig.normalize).  Off by default; accepted only before the handle's first
 * rexsim_reset / rexsim_step / rexsim_step_host and only once, REXSIM_ERR_INVALID otherwise.
 *   delta = 1 (FrameDelta): a reset returns the observation itself and keeps it as `last`; a step returns obs - last (fp32
 *     subtraction) and keeps obs.  An auto-reset step therefore returns the new episode's first observation.
 *   count > 0 (FrameHistory, flatten=True): past_indices HOST [count], 1..16 values in 0..64 that include 0, capacity C = their
 *     maximum (> 0).  A reset fills all C slots with the (delta) observation; step t (LimitDuration's counter, 1 after the first
 *     step of an episode) writes slot t % C and returns the slots (t - i) mod C for each index i in order, concatenated, so the
 *     observation row widens to count x obs_dim.  Duplicates and any order are allowed; an index equal to C reads slot t % C,
 *     the current frame, as the reference's ring does.
 * REXSIM_FLAG_NONFINITE keeps its meaning: the observation the step produced (before the wrappers) is non-finite. */
int rexsim_set_frames(RexSim* sim, const int32_t* past_indices, int32_t count, int32_t delta);
/* words per env of the observation rows rexsim_step, rexsim_step_host and rexsim_reset write: rexsim_obs_dim, times the number of
 * past indices when FrameHistory is on */
int rexsim_out_dim(const RexSim* sim);
/* the frame wrappers' device buffers, part of an exact checkpoint together with the state buffers: ring dev [C][obs_dim][N] f32
 * (FrameHistory, NULL and 0 floats when off), last dev [obs_dim][N] f32 (FrameDelta, NULL and 0 floats when off) */
int rexsim_frame_buffers(RexSim* sim, float** ring, int64_t* ring_floats, float** last, int64_t* last_floats);
/* Per-env task-constructor values: what BatchEnv([ctor_0, ctor_1, ...]) gives the reference, each env built with its own
 * keywords (rex_gym/agents/tools/batch_env.py:21-42).  The value block is [REXSIM_VALUE_BLOCK_ROWS][N] f32; row r of env e
 * means for e exactly what the RexSimConfig field of the same name means for the batch (NaN = draw per reset; backwards -1, 0
 * or 1; the five pose values follow pose_values' rule env by env).  The last row is the kernels' own: the backwards value the
 * env's running episode started with (walk's reward flips on it, rex_gym_env.py:506). */
enum {
    REXSIM_VALUE_TARGET_POSITION = 0, REXSIM_VALUE_BACKWARDS = 1, REXSIM_VALUE_TARGET_ORIENT = 2, REXSIM_VALUE_INIT_ORIENT = 3,
    REXSIM_VALUE_POSE = 4,            /* 5 rows: base_y, base_z, base_roll, base_pitch, base_yaw */
    REXSIM_VALUE_ROWS = 9,            /* rows a caller writes */
    REXSIM_VALUE_EPISODE_BACKWARDS = 9,
    REXSIM_VALUE_BLOCK_ROWS = 10,
    REXSIM_MAX_GAIN_PAIRS = 64,       /* distinct hold settings (motor_kp, motor_kd, pd_latency, solver_iterations): the settle
                                         runs once per setting and field */
    REXSIM_MAX_REPEAT_PAIRS = 8,      /* distinct (action_repeat, solver_iterations) pairs of rexsim_set_env_repeats */
    REXSIM_GROUP_WORDS = 8,           /* int32 words rexsim_launch_group writes */
    REXSIM_MAX_LAUNCH_GROUPS = 16     /* launch groups of one batch: rexsim_rebalance sorts on (group, 256 cost bins) in one
                                         block of its scan, 4096 bins at most */
};
/* row of the value block that the constructor keyword `keyword` fills ("target_position", "backwards", "target_orient",
 * "init_orient", "base_y", "base_z", "base_roll", "base_pitch", "base_yaw"); -1 for any other name */
int rexsim_value_row(const char* keyword);
/* Switch the per-env values on.  values HOST [REXSIM_VALUE_ROWS][N]; kp, kd HOST [N] each, or both NULL (every env takes
 * RexSimConfig.motor_kp / motor_kd).  Per-env gains are refused with a motor_kp / motor_kd range, when negative or non-finite,
 * and beyond REXSIM_MAX_GAIN_PAIRS distinct pairs; with them the reset hold is settled again, once per (pair, field), each env
 * resetting from its own pair's snapshot (Rex.Reset holds at the env's gains, rex.py:314-323).  Accepted only before the
 * handle's first reset or step and only once (REXSIM_ERR_INVALID otherwise); synchronous.  Off: nothing is allocated and
 * every launch is what it is without it. */
int rexsim_set_env_values(RexSim* sim, const float* values, const float* kp, const float* kd);
/* Scatter new values into rows of the block: idx dev [k] int32 (NULL: every env, k ignored), values dev [REXSIM_VALUE_ROWS][k]
 * f32 of which only the rows whose bit is set in `rows` are read.  Each env takes them at its next reset, explicit or
 * automatic.  One launch on `stream`, no host synchronisation; an index outside [0, N) is skipped and sets
 * REXSIM_FLAG_BAD_INDEX in the aggregate word.  REXSIM_ERR_INVALID when the per-env values are off. */
int rexsim_set_task_values(RexSim* sim, const int32_t* idx, int32_t k, const float* values, uint32_t rows, void* stream);
/* the per-env values' device buffers, part of an exact checkpoint together with the state buffers: values dev
 * [REXSIM_VALUE_BLOCK_ROWS][N] f32, pair dev [N] int32 (each env's gain pair; its hold setting with per-env latencies), gains
 * dev [npairs][2] f32 (kp, kd of each pair or setting).
 * REXSIM_ERR_INVALID when the per-env values are off. */
int rexsim_env_value_buffers(RexSim* sim, float** values, int32_t** pair, float** gains, int32_t* npairs);
/* Per-env sensor latencies: the control_latency and pd_latency keywords of BatchEnv([ctor_0, ctor_1, ...]) (the latencies do
 * not change the spaces, batch_env.py:36-43).  control_latency, pd_latency HOST [N] seconds each in fp64, as the config's
 * scalars are, NULL: every env takes the RexSimConfig scalar.  Env e then runs as a batch built with (control_latency[e], pd_latency[e]) as scalars: the PD loop
 * reads q, qd pd_latency[e] ago, reward, termination, observation and the turn goal check read the row control_latency[e]
 * ago; an env whose latencies are both 0 in a batch without noise reads the true state, as the scalar build does.  The ring
 * keeps the batch's deepest history; a non-zero latency switches the sensor model on.  The reset hold reads the PD
 * observation (rex.py:303-323), so it is settled again once per hold setting (motor_kp, motor_kd, pd_latency) and field,
 * at most REXSIM_MAX_GAIN_PAIRS settings, each env resetting from its own setting's snapshot; with a motor_kp / motor_kd
 * range the settings hold at the config's gains.  Refused (REXSIM_ERR_INVALID) for a negative or non-finite latency, more
 * settings than the cap, after the handle's first reset or step, and on a second call.  Composes with
 * rexsim_set_env_values in either order; synchronous.  Off: nothing is allocated and every launch is what it is without it. */
int rexsim_set_env_latencies(RexSim* sim, const double* control_latency, const double* pd_latency);
/* the per-env latencies' device buffer, part of an exact checkpoint: latency dev [2][N] f64 (row 0 control_latency, row 1
 * pd_latency), and the rows per env of the history ring.  With per-env values the hold settings are rexsim_env_value_buffers'
 * pair index and gains table, one row per setting.  REXSIM_ERR_INVALID when the per-env latencies are off. */
int rexsim_env_latency_buffers(RexSim* sim, double** latency, int32_t* depth);
/* Per-env terrains: the terrain_type keyword of BatchEnv([ctor_0, ctor_1, ...]) (the terrain does not change the spaces,
 * batch_env.py:36-43), so that one batch holds envs on the plane and envs on the heightfield.  terrain HOST [N] int32, each
 * REXSIM_TERRAIN_PLANE or REXSIM_TERRAIN_RANDOM.  The handle must have been created with terrain RANDOM (the heightfield bank
 * and the heightfield's friction); plane_friction is the friction of the plane envs.  Env e then runs exactly as env e of a
 * batch created with terrain[e] as its terrain and that terrain's friction: a heightfield env resets on field
 * (global env + reset count) mod nfields of the one bank, a plane env on the plane with field word 0.
 * Each step launches the step kernel's build for each terrain that has envs, over that terrain's slots (plane envs in slots
 * [0, nplane), heightfield envs after them; rexsim_rebalance keeps the partition), each launch choosing its build from its
 * own size; both launches are on the stream.  The reset hold is settled once per hold setting on the plane and once per
 * setting and field on the heightfield, each terrain's snapshots by one launch of its own build at its own friction.
 * Refused (REXSIM_ERR_INVALID) for an entry that is neither terrain, a negative or non-finite friction, a handle created on
 * the plane, after the handle's first reset or step, and on a second call.  Composes with rexsim_set_env_values and
 * rexsim_set_env_latencies in any order; synchronous.  Off: nothing is allocated and every launch is what it is without it. */
int rexsim_set_env_terrains(RexSim* sim, const int32_t* terrain, float plane_friction);
/* the per-env terrains' device buffer, part of a checkpoint's identity: terrain dev [N] u8 (REXSIM_TERRAIN_* of each env),
 * and the number of envs on the plane.  REXSIM_ERR_INVALID when the per-env terrains are off. */
int rexsim_env_terrain_buffers(RexSim* sim, uint8_t** terrain, int32_t* nplane);
/* Per-env control rates: the control_time_step and action_repeat keywords of BatchEnv([ctor_0, ctor_1, ...]) over envs that
 * share the simulation time step control_time_step / action_repeat (rex_gym_env.py:170-173), which the observation space
 * depends on; the action space depends on neither (batch_env.py:36-43).  action_repeat, solver_iterations HOST [N] int32
 * each, NULL: every env takes the RexSimConfig scalar.  Env e then runs exactly as a batch created with action_repeat[e] and
 * solver_iterations[e] as its scalars: action_repeat[e] physics sub-steps per control step, each PGS solve capped at
 * solver_iterations[e] iterations, and its reset hold settled at that cap.  Everything derived from sim_dt (sensor delays,
 * overheat limit, gait clock, hold length, rate bounds, energy) stays the batch's.
 * The batch's envs fall into launch groups (terrain, action_repeat, solver_iterations), terrain-major (plane first) and in
 * order of first appearance; group g owns a contiguous slot range of the permutation (rexsim_rebalance keeps the
 * partition), and each step launches the step kernel once per group over its range with the group's values, each launch
 * choosing its build from its own size, all on the stream.  The hold settings become (motor_kp, motor_kd, pd_latency,
 * solver_iterations), each count's settings contiguous, settled once per (terrain, count).
 * Refused (REXSIM_ERR_INVALID) for an entry <= 0, more than REXSIM_MAX_REPEAT_PAIRS distinct (action_repeat,
 * solver_iterations) pairs, more hold settings than REXSIM_MAX_GAIN_PAIRS, after the handle's first reset or step, and on a
 * second call.  Composes with rexsim_set_env_values, rexsim_set_env_latencies and rexsim_set_env_terrains in any order;
 * synchronous.  Off: nothing is allocated and every launch is what it is without it. */
int rexsim_set_env_repeats(RexSim* sim, const int32_t* action_repeat, const int32_t* solver_iterations);
/* the per-env control rates' device buffer, part of a checkpoint's identity: repeats dev [2][N] int32 (row 0 action_repeat,
 * row 1 solver_iterations).  REXSIM_ERR_INVALID when the per-env repeats are off. */
int rexsim_env_repeat_buffers(RexSim* sim, int32_t** repeats);
/* Per-env tasks and signals: the task and signal_type of BatchEnv([ctor_0, ctor_1, ...]) over envs whose spaces agree
 * (batch_env.py:36-43), e.g. turn ik with turn ol, standup with poses, or with RexSimConfig.normalize walk ik with turn.
 * task, signal HOST [N] int32 each (REXSIM_TASK_*, REXSIM_SIGNAL_*).  Env e then runs exactly as a batch created with
 * (task[e], signal[e]) as its scalars: its reset draws, its reset hold, its step kernel, reward and termination.
 * The step kernel's compile unit (standup and poses ignore the signal) becomes one more key of the launch groups, which are
 * (terrain, unit, action_repeat, solver_iterations), terrain-major, then in order of first appearance.  The hold settings
 * become (start, motor_kp, motor_kd, pd_latency, solver_iterations), the start being the pose the hold ends in: the IK stand,
 * the open-loop stand, standup's fold, or none (poses skips the hold); each (count, start)'s settings are contiguous and
 * settled once per terrain.  With episode statistics the objectives are kept when any env is walk or gallop; the columns of
 * the other envs are NaN.
 * Refused (REXSIM_ERR_INVALID) for an entry that is no task or signal, an env whose rexsim_action_dim or rexsim_obs_dim
 * differs from the handle's, with normalize = 0 an env whose raw action bound differs from the handle's, gallop with the
 * 18-motor arm, more than REXSIM_MAX_LAUNCH_GROUPS launch groups or REXSIM_MAX_GAIN_PAIRS hold settings, after the handle's
 * first reset or step, and on a second call.  Composes with the other per-env setters in any order (each refuses a batch
 * past the group cap); synchronous.  Off: nothing is allocated and every launch is what it is without it. */
int rexsim_set_env_tasks(RexSim* sim, const int32_t* task, const int32_t* signal);
/* the per-env tasks' device buffer, part of a checkpoint's identity: task dev [2][N] u8 (row 0 REXSIM_TASK_*, row 1
 * REXSIM_SIGNAL_*, as given).  REXSIM_ERR_INVALID when the per-env tasks are off. */
int rexsim_env_task_buffers(RexSim* sim, uint8_t** task);
/* the task and signal of launch group g's step launches: its first env's (the config's for a batch of one group).
 * REXSIM_ERR_INVALID for g outside [0, rexsim_launch_groups). */
int rexsim_launch_group_task(const RexSim* sim, int32_t g, int32_t* task, int32_t* signal);
/* Per-env marks: the mark of BatchEnv([ctor_0, ctor_1, ...]) over envs with and without the arm, whose spaces agree for every
 * task but gallop.  num_motors HOST [N] int32, 12 (base) or 18 (arm).  The handle must have been created with 18 motors: the
 * arm's model table starts with the base's REXSIM_MT_FLOATS floats, its render table draws the base's shapes, and each row of
 * its sensor history ring holds the base's HW_WORDS words first, so the arm's buffers serve both marks.  Env e then runs
 * exactly as a batch created with num_motors[e]: its reset hold, its step kernel build, its sensor history (a base env uses
 * the first 43 words of each 61-word ring row, the rest stay untouched), its renderer shapes.  The mark becomes one more key
 * of the launch groups, which are (terrain, mark, unit, action_repeat, solver_iterations), terrain-major, then in order of
 * first appearance, and of the hold settings, (mark, start, motor_kp, motor_kd, pd_latency, solver_iterations), each
 * (count, start, mark)'s settings contiguous and settled once per terrain.  The command block stays [18][N]: rows 12..17 of
 * a base env's column are NaN.
 * Refused (REXSIM_ERR_INVALID) for a handle created with 12 motors, an entry other than 12 or 18, 18 for a gallop env (the
 * config's task or its per-env task), more than REXSIM_MAX_LAUNCH_GROUPS launch groups or REXSIM_MAX_GAIN_PAIRS hold
 * settings, after the handle's first reset or step, and on a second call.  Composes with the other per-env setters in any
 * order; synchronous.  Off: nothing is allocated and every launch is what it is without it. */
int rexsim_set_env_marks(RexSim* sim, const int32_t* num_motors);
/* the per-env marks' device buffer, part of a checkpoint's identity: mark dev [N] u8, 1 for the arm, 0 for the base.
 * REXSIM_ERR_INVALID when the per-env marks are off. */
int rexsim_env_mark_buffers(RexSim* sim, uint8_t** mark);
/* the motor count (12 or 18) of launch group g's step launches (the config's for a batch of one group).
 * REXSIM_ERR_INVALID for g outside [0, rexsim_launch_groups). */
int rexsim_launch_group_mark(const RexSim* sim, int32_t g, int32_t* num_motors);
/* launch groups of the batch: 1 unless per-env terrains, repeats, tasks or marks split it (0 for a null handle) */
int rexsim_launch_groups(const RexSim* sim);
/* launch group g: info[REXSIM_GROUP_WORDS] = terrain, action_repeat, solver_iterations, first slot, slot count, and the
 * build its last step launch used (CTA size, CTAs per SM, sensor; all 0 before the first step).  A batch of one group
 * reports the config's values over slots [0, N).  REXSIM_ERR_INVALID for g outside [0, rexsim_launch_groups). */
int rexsim_launch_group(const RexSim* sim, int32_t g, int32_t* info);
/* the permutation the step launches read and each env's launch group: perm dev [N] int32 (slot -> env; group g's envs in
 * slots [first_g, first_g + count_g) of rexsim_launch_group), NULL until rexsim_rebalance or a per-env setter that splits
 * the batch (the identity); group dev [N] u8, NULL for a batch of one launch group */
int rexsim_slot_buffers(RexSim* sim, int32_t** perm, uint8_t** group);
/* kernels launched by this handle since create (the bench reports it); a step counts one launch per launch group */
int64_t rexsim_launch_count(const RexSim* sim);
/* which build of the step kernel the last rexsim_step / rexsim_step_host launched (all 0 before the first step): CTA size,
 * resident CTAs per SM it is compiled for (1: 255 registers, 4: 128 registers), 1 if the sensor model is compiled in.
 * With several launch groups: the build of that step's last launch (rexsim_launch_group has each group's) */
int rexsim_last_step_build(const RexSim* sim, int32_t* cta_threads, int32_t* ctas_per_sm, int32_t* sensor);
/* the same for the last launch over the envs on `terrain`: the last launch group on that terrain; all 0 when the batch has no
 * env on it */
int rexsim_last_terrain_build(const RexSim* sim, int32_t terrain, int32_t* cta_threads, int32_t* ctas_per_sm, int32_t* sensor);
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
/* rexagent_gae_segments (rexsim_agent.h) that bootstraps episodes cut by the time limit instead of treating their last step as terminal (the
 * reference's PPO never does: it has no final observation).  truncated dev [T][N] u8 (non-zero: truncated), final_value dev
 * [T][N] f32 (the value of the step's final observation, rexsim_step_final; read only where done and truncated are both set).
 * At such a step: delta_t = r_t + discount * final_value_t - v_t, adv_t = delta_t, return_t = r_t + discount * final_value_t.
 * Every other step is computed as rexagent_gae_segments computes it, in the same fp32 order: with truncated all zero the
 * outputs are bit-identical to it.  Declared here, not in rexsim_agent.h, whose entry-point list is held fixed (the agent ABI
 * tests pin its 20 functions, so that bindings generated from it stay complete); like rexagent_gae_segments it takes no handle. */
int rexsim_gae_segments_bootstrap(const float* reward, const float* value, const uint8_t* done, const uint8_t* truncated,
                                  const float* final_value, int32_t T, int32_t n, float discount, float lambda,
                                  float* out_return, float* out_advantage, void* stream);
const char* rexsim_last_error(void);

#ifdef __cplusplus
}
#endif
#endif

// rexsim_kernel.cuh -- fused sm_90a step kernel of the batched Rex simulator.
//
// Mapping: FOUR LANES PER ENVIRONMENT, lane = leg (FL, FR, RL, RR in motor order,
// rex_gym/model/mark_constants.py:3-8); 8 environments per warp, everything register-resident for the
// whole control step (state read once / written once).  The 4 legs are the only real parallelism of
// one Rex (three serial joints each); cross-leg coupling goes through the floating base and is done
// with width-4 warp shuffles (articulated-inertia reduction, impulse responses, Gauss-Seidel hand-off).
//
// One launch = one RexGymEnv.step for every env (rex_gym/envs/rex_gym_env.py:369-414):
//   task signal (Bezier gait + 3-DOF leg IK or open loop)      envs/gym/*_env.py, model/gait_planner.py, model/kinematics.py
//   action_repeat x { motor model (model/motor.py:76-143, model/rex.py:568-641), optionally on the PD-delayed observation
//                     + stepSimulation: ABA forward dynamics in a world-aligned common frame, contact candidates (toe hull,
//                       collision boxes) against the plane or the staged heightfield tile, joint-limit rows, PGS, integrate
//                     + ReceiveObservation: push the sensor-history row (sensor model only, model/rex.py:726-733) }
//   reward / termination / observation (+ fused ClipAction/RangeNormalize/LimitDuration, auto-reset)
//
// The physics is algebraically the same algorithm as oracle/rexsim_oracle.c (Bullet btMultiBody pipeline) but formulated
// differently on purpose: common-frame ABA instead of link frames; impulse-space PGS on the Delassus matrix of the foot
// contacts, leg joint limits and arm joint limits (the fast path) or a matrix-free base / limb split (body contacts) instead of
// generalized-velocity space.  Identical iterates in exact arithmetic.  The warps of a CTA re-align at every sub-step: the
// straight-line code of one sub-step (150 KB) outruns the instruction caches otherwise (DESIGN.md section 5).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "../../include/rexsim.h"

namespace rexsim {

// ----- SoA state word indices ---------------------------------------------------------------------
enum {
    F_POS = 0, F_QUAT = 3, F_LINVEL = 7, F_ANGVEL = 10, F_Q = 13, F_QD = 25,
    F_ALPHA = 37, F_TARGET = 38, F_TORIENT = 39, F_IORIENT = 40, F_KP = 41, F_KD = 42,
    F_AQ = 43, F_AQD = 49, NF = 55      // arm joint angles / rates (mark='arm'; unused words otherwise)
};
enum {
    I_STEP = 0, I_ENVSTEP = 1, I_FLAGS = 2, I_RESETCNT = 3, I_FIELD = 4, I_ENDSTEP = 5, I_GPLAST = 6,
    I_PHI_LO = 7, I_PHI_HI = 8, I_OVH = 9 /*4 words, 3x10-bit counters per leg*/, I_CONTACT = 13,
    I_OVHA = 14 /*2 words, 3x10-bit counters of the arm motors*/,
    I_HPUSH = 16 /*observations pushed into the sensor history since Rex.Reset cleared it (sensor model only)*/, NI = 17
};
// sensor history ring (rex_gym/model/rex.py:122,726-753): one row per ReceiveObservation = per sub-step, words per env:
//   [9*leg + 0..2] q, [+3..5] qd, [+6..8] observed torque of leg `leg`; [36..39] base quaternion, [40..42] base angular velocity;
//   mark 'arm': [43..48] arm q, [49..54] arm qd, [55..60] arm observed torque.   Layout ring[slot][word][env].
enum { HW_BASE = 36, HW_ARM = 43, HW_WORDS = 43, HW_WORDS_ARM = 61, HIST_MAXLEN = 100 };
enum {
    FL_GOAL = 1, FL_TERMINATING = 2, FL_STILL = 4, FL_BACKWARDS = 8, FL_CLOCKWISE = 16, FL_ENVGOAL = 32,
    FL_ENABLED_SHIFT = 8,  // 12 leg motor-enabled bits
    FL_ARM_ENABLED_SHIFT = 20,  // 6 arm motor-enabled bits
    FL_POSE_SHIFT = 26          // 3 bits: poses task, which base coordinate is staged (0 base_y, 1 base_z, 2 roll, 3 pitch, 4 yaw)
};

// ----- per-task action width [ik, ol signal], motor angles in the observation, RangeNormalize action bound [ik, ol] -----
struct TaskShape { int act[2]; bool angles; float bound[2]; };
__host__ __device__ constexpr TaskShape task_shape(int task) {
    return task == REXSIM_TASK_WALK   ? TaskShape{{2, 8}, false, {0.4f, 0.01f}}       // walk_env.py:108-113
         : task == REXSIM_TASK_GALLOP ? TaskShape{{2, 4}, true, {-0.4f, -0.3f}}       // gallop_env.py:123-127; inverted Box: low=+b, high=-b
         : task == REXSIM_TASK_TURN   ? TaskShape{{2, 2}, false, {0.01f, 0.01f}}      // turn_env.py:104-108
         : TaskShape{{1, 1}, false, {0.1f, 0.1f}};                                   // standup_env.py:99, poses_env.py:118
}
// the step-kernel compile unit (rexsim_kernel.cu c_units) of a (task, signal) pair: walk, gallop and turn per signal, then
// standup and poses, which ignore the signal; an unknown task takes unit 6
__host__ __device__ constexpr int unit_of(int task, int signal) {
    return task == REXSIM_TASK_POSES ? 7 : (task >= 0 && task < REXSIM_TASK_STANDUP) ? 2 * task + (signal != REXSIM_SIGNAL_IK) : 6;
}
// observation width: base roll, pitch and their rates, then (gallop) the motor angles
__host__ __device__ constexpr int obs_dim(int task, int num_motors) { return 4 + (task_shape(task).angles ? num_motors : 0); }
// width of the rows the kernels write: obs_dim, repeated once per past index when FrameHistory is on (rexsim_out_dim)
__host__ __device__ constexpr int out_dim(int task, int num_motors, int history_count) {
    return obs_dim(task, num_motors) * (history_count > 0 ? history_count : 1);
}

// Episode statistics (RexSimConfig.episode_stats; every pointer is null when it is off): simulate()'s per-env score and length
// (rex_gym/agents/tools/simulate.py:57-105) and what its StreamingMeans were handed by the episodes that ended, per env (not per
// slot, so rexsim_rebalance cannot move them).  score, length and the four accumulators live in one allocation, `block`.
struct EpisodeStats {
    double* __restrict__ sum_score;    // [N] scores of the submitted episodes, summed
    int64_t* __restrict__ sum_length;  // [N] their lengths, summed
    float* __restrict__ score;         // [N] reward summed since the env's episode began
    int32_t* __restrict__ length;      // [N] control steps since the env's episode began
    int32_t* __restrict__ count;       // [N] episodes submitted
    int32_t* __restrict__ nonfinite;   // [N] episodes that ended on a step raising REXSIM_FLAG_NONFINITE (never submitted)
    float* __restrict__ objectives;    // [4][N] forward, energy, drift, shake of the last step, unweighted (walk and gallop only)
};
// bytes of the per-env block behind EpisodeStats: sum_score | sum_length | score | length | count | nonfinite
__host__ __device__ constexpr size_t episode_block_bytes(size_t n) { return n * (2 * sizeof(double) + 4 * sizeof(int32_t)); }

// Frame wrappers (rexsim_set_frames; both pointers null when off): the reference's FrameHistory(FrameDelta(observation))
// (rex_gym/agents/tools/wrappers.py:93-181) in the step and reset kernels' epilogues.  Each lane keeps the words of the
// observation it writes itself (lane 0 the four base terms, every lane its three gallop angles), so no lane reads another's.
enum { FRAMES_MAX_INDICES = 16, FRAMES_MAX_CAPACITY = 64 };
struct Frames {
    float* ring;                       // [capacity][O][N] FrameHistory's buffer, O = obs_dim; null: no history
    float* last;                       // [O][N] FrameDelta's last observation; null: no delta
    const int32_t* index;              // [count] the past indices in the caller's order (duplicates allowed; capacity reads the current slot)
    int32_t capacity;                  // max(past_indices)
    int32_t count;                     // number of past indices
};

// Per-env task-constructor values (rexsim_set_env_values; every pointer null when off).  The reset reads the env's values and
// gain pair instead of the config's scalars; the step reads the backwards value its episode started with.
struct EnvValues {
    float* values;                     // [REXSIM_VALUE_BLOCK_ROWS][N]
    const int32_t* pair;               // [N] gain pair of each env: it resets from snapshot pair * fields + field
    const float* gains;                // [npairs][2] motor_kp, motor_kd
};
// One latency of Rex._GetDelayedObservation (rex.py:735-753): the latency (only its sign is used on the device), n = int(latency
// / dt) and the blend weight a = (latency - n dt) / dt of the older row, computed on the host in fp64 (delay_terms)
struct Delay { float lat; int32_t n; float a; };
// Per-env sensor latencies (rexsim_set_env_latencies; both pointers null when off).  Each env reads its own terms, by env
// (not by slot: rexsim_rebalance permutes the slots); the settle reads the PD term of its hold setting.
struct EnvDelay { Delay ctl, pd; int32_t sensed; int32_t pad; };   // sensed: latency or noise; 0 reads the true state
struct EnvLatencies {
    const EnvDelay* __restrict__ env;  // [N]
    const Delay* __restrict__ hold;    // [settings] PD term of each hold setting (EnvValues.pair indexes it)
};
// Settled reset snapshots of one hold setting on one terrain: one per field of the heightfield bank, one on the plane
__host__ __device__ __forceinline__ int terrain_snapshots(int terrain, int nfields) {
    return terrain == REXSIM_TERRAIN_RANDOM ? nfields : 1;
}
// The snapshot layout, its one owner (the settle writes it, reset_from_snapshot and the auto-reset read it): hold setting h
// owns snapshots [h * per_setting, (h + 1) * per_setting), the plane's first when the batch has plane envs, then one per
// field from `field0` on when it has heightfield envs.  A single-terrain batch: per_setting = terrain_snapshots, field0 0
// on the heightfield (1 on the plane, where it is never read).
struct SnapLayout { int32_t per_setting, field0; };
__host__ __device__ __forceinline__ SnapLayout snap_layout(bool plane, bool random, int nfields) {
    return SnapLayout{(plane ? 1 : 0) + (random ? nfields : 0), plane ? 1 : 0};
}
__host__ __device__ __forceinline__ int snapshot_index(const SnapLayout& s, int setting, int terrain, int field) {
    return setting * s.per_setting + (terrain == REXSIM_TERRAIN_RANDOM ? s.field0 + field : 0);
}

struct Params {
    RexSimConfig cfg;
    EpisodeStats ep;
    Frames fr;
    EnvValues ev;
    EnvLatencies el;
    int32_t out_dim;                   // words per env of the observation rows the step and reset kernels write (rexsim_out_dim)
    const float* __restrict__ model;   // REXSIM_MT_FLOATS floats, 16-byte aligned
    float* __restrict__ sf;            // [NF][N]
    int32_t* __restrict__ si;          // [NI][N]
    const float* __restrict__ snap_f;  // [settings * snaps.per_setting][NF] settled reset snapshots, setting-major
    const int32_t* __restrict__ snap_i;// [settings * snaps.per_setting][NI]
    SnapLayout snaps;
    // per-env terrains (rexsim_set_env_terrains; null: every env on cfg.terrain): [N] REXSIM_TERRAIN_* by env.  The step
    // kernel never reads it: each of its launches covers one launch group's slots, with the group's terrain in cfg.terrain.
    const uint8_t* __restrict__ env_terrain;
    const float* __restrict__ field_zoff; // [nfields]
    int32_t* __restrict__ err;         // [N] per-env bits of the most recent step, [N] = OR of all since last cleared
    uint8_t* err_host;                 // host-buffer step with zero-copy buffers: 8 flag bytes in the caller's block, byte b = 1 when an
                                       // env raised error bit b this step (idempotent stores, no atomics across PCIe); else null
    float* __restrict__ cmd_out;       // [num_motors][N]
    const float* __restrict__ actions; // [N][A]
    float* __restrict__ obs;           // [N][O]
    float* __restrict__ reward;        // [N]
    uint8_t* __restrict__ done;        // [N]
    // step kernel, both nullable (rexsim_step_final): the observation of every env whose step returned done, before the
    // auto-reset overwrites its obs row ([N][out_dim]; other rows untouched), and every env's time-limit byte ([N]: bit 0 the
    // fused max_episode_steps was reached at this step, bit 1 the episode also ended by the task's termination or the
    // non-finite guard)
    float* final_obs;
    uint8_t* limit;
    const int32_t* __restrict__ reset_idx; // reset kernel: [k] or null
    int32_t reset_k;
    int32_t N;                         // envs: the stride of every per-env array
    int32_t nslots;                    // step kernel: slots it covers, perm[0, nslots) (N, or one launch group's range)
    int32_t sm_count;                  // SMs of the device (kernel variant choice)
    int32_t* launched;                 // host: {BLOCK, OCC, SENSOR} of the step_kernel instance the last step launched (never read on the device)
    const int32_t* __restrict__ perm;  // [nslots] slot -> env (null: identity); see rexsim_rebalance
    int32_t* __restrict__ cost;        // [N] solver iterations of the last control step
    // sensor model (control / PD latency, observation noise: rex.py:735-769); all unused when sensor_on == 0
    int32_t sensor_on;
    int32_t ring_depth;                // D rows kept per env: the batch's largest n + 2 (100 = the deque's maxlen when a latency reaches it)
    // [D][HW_WORDS(_ARM)][N]; NOT __restrict__: lanes of an env read what lane 0 wrote.  In a batch of both marks it is
    // [D][HW_WORDS_ARM][N] words and a base env's column holds its [D][HW_WORDS] rows in its first D * HW_WORDS words: only
    // launches of the env's own mark address it
    float* ring;
    float* snap_ring;                  // [npairs * fields][D][HW_WORDS(_ARM)] history the reset hold leaves behind, per snapshot
                                       // (a batch of both marks: one ring per mark, the launch's)
    Delay ctl, pd;                     // the config's control and PD latency (per env: EnvLatencies)
    float noise_sd[5];                 // SENSOR_NOISE_STDDEV order: motor angle, motor velocity, motor torque, base rpy, base rpy rate
    // per-env tasks (rexsim_set_env_tasks; null: every env runs cfg.task): [2][N] REXSIM_TASK_* row, REXSIM_SIGNAL_* row, by
    // env.  Only the reset kernel reads it: each step launch covers one launch group, with the group's task in cfg.task.
    const uint8_t* __restrict__ env_task;
    // per-env marks (rexsim_set_env_marks; null: every env carries cfg.num_motors): [N] by env, 1 for the arm, 0 for the base.
    // The reset kernel (one launch per mark, each skipping the other mark's envs) and the renderer read it; each step and
    // settle launch covers one mark, the launch group's cfg.num_motors.
    const uint8_t* __restrict__ env_mark;
};

// ----- tiny vector algebra ---------------------------------------------------------------------------
struct V3 { float x, y, z; };
__device__ __forceinline__ V3 mk(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ V3 operator+(V3 a, V3 b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ V3 operator-(V3 a, V3 b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ V3 operator*(float s, V3 a) { return mk(s * a.x, s * a.y, s * a.z); }
__device__ __forceinline__ float dot(V3 a, V3 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, a.z * b.z)); }
__device__ __forceinline__ V3 cross(V3 a, V3 b) {
    return mk(fmaf(a.y, b.z, -a.z * b.y), fmaf(a.z, b.x, -a.x * b.z), fmaf(a.x, b.y, -a.y * b.x));
}
__device__ __forceinline__ V3 fma3(float s, V3 a, V3 b) { return mk(fmaf(s, a.x, b.x), fmaf(s, a.y, b.y), fmaf(s, a.z, b.z)); }
struct M3 { V3 c0, c1, c2; };   // columns
__device__ __forceinline__ V3 mul(const M3& R, V3 v) { return fma3(v.x, R.c0, fma3(v.y, R.c1, v.z * R.c2)); }
struct SV { V3 a, l; };         // spatial vector: angular, linear
__device__ __forceinline__ SV operator+(SV p, SV q) { SV r; r.a = p.a + q.a; r.l = p.l + q.l; return r; }
__device__ __forceinline__ SV operator-(SV p, SV q) { SV r; r.a = p.a - q.a; r.l = p.l - q.l; return r; }
__device__ __forceinline__ SV operator*(float s, SV p) { SV r; r.a = s * p.a; r.l = s * p.l; return r; }
__device__ __forceinline__ float sdot(SV p, SV q) { return dot(p.a, q.a) + dot(p.l, q.l); }
__device__ __forceinline__ SV sfma(float s, SV p, SV q) { SV r; r.a = fma3(s, p.a, q.a); r.l = fma3(s, p.l, q.l); return r; }
// symmetric 3x3
struct S3 { float xx, yy, zz, xy, xz, yz; };
__device__ __forceinline__ V3 mul(const S3& S, V3 v) {
    return mk(fmaf(S.xx, v.x, fmaf(S.xy, v.y, S.xz * v.z)), fmaf(S.xy, v.x, fmaf(S.yy, v.y, S.yz * v.z)),
              fmaf(S.xz, v.x, fmaf(S.yz, v.y, S.zz * v.z)));
}
// symmetric 6x6 articulated inertia  [[A, B],[B^T, D]]  (A, D symmetric; B general, rows b0,b1,b2)
struct AI { S3 A; V3 b0, b1, b2; S3 D; };
__device__ __forceinline__ SV mul(const AI& I, SV s) {
    SV r;
    V3 Aa = mul(I.A, s.a);
    r.a = mk(Aa.x + dot(I.b0, s.l), Aa.y + dot(I.b1, s.l), Aa.z + dot(I.b2, s.l));
    V3 Dl = mul(I.D, s.l);
    r.l = fma3(s.a.x, I.b0, fma3(s.a.y, I.b1, fma3(s.a.z, I.b2, Dl)));
    return r;
}
// I -= U U^T * k
__device__ __forceinline__ void rank1_sub(AI& I, SV U, float k) {
    V3 ka = k * U.a, kl = k * U.l;
    I.A.xx = fmaf(-ka.x, U.a.x, I.A.xx); I.A.yy = fmaf(-ka.y, U.a.y, I.A.yy); I.A.zz = fmaf(-ka.z, U.a.z, I.A.zz);
    I.A.xy = fmaf(-ka.x, U.a.y, I.A.xy); I.A.xz = fmaf(-ka.x, U.a.z, I.A.xz); I.A.yz = fmaf(-ka.y, U.a.z, I.A.yz);
    I.D.xx = fmaf(-kl.x, U.l.x, I.D.xx); I.D.yy = fmaf(-kl.y, U.l.y, I.D.yy); I.D.zz = fmaf(-kl.z, U.l.z, I.D.zz);
    I.D.xy = fmaf(-kl.x, U.l.y, I.D.xy); I.D.xz = fmaf(-kl.x, U.l.z, I.D.xz); I.D.yz = fmaf(-kl.y, U.l.z, I.D.yz);
    I.b0 = fma3(-ka.x, U.l, I.b0); I.b1 = fma3(-ka.y, U.l, I.b1); I.b2 = fma3(-ka.z, U.l, I.b2);
}
__device__ __forceinline__ void add(AI& I, const AI& J) {
    I.A.xx += J.A.xx; I.A.yy += J.A.yy; I.A.zz += J.A.zz; I.A.xy += J.A.xy; I.A.xz += J.A.xz; I.A.yz += J.A.yz;
    I.D.xx += J.D.xx; I.D.yy += J.D.yy; I.D.zz += J.D.zz; I.D.xy += J.D.xy; I.D.xz += J.D.xz; I.D.yz += J.D.yz;
    I.b0 = I.b0 + J.b0; I.b1 = I.b1 + J.b1; I.b2 = I.b2 + J.b2;
}
// rigid-body spatial inertia about the frame origin: mass m, COM c (from origin), rotational inertia Iw about COM
__device__ __forceinline__ AI rigid_inertia(float m, V3 c, const S3& Iw) {
    AI I;
    float cc = dot(c, c);
    I.A.xx = Iw.xx + m * (cc - c.x * c.x); I.A.yy = Iw.yy + m * (cc - c.y * c.y); I.A.zz = Iw.zz + m * (cc - c.z * c.z);
    I.A.xy = Iw.xy - m * c.x * c.y; I.A.xz = Iw.xz - m * c.x * c.z; I.A.yz = Iw.yz - m * c.y * c.z;
    I.b0 = mk(0.f, -m * c.z, m * c.y); I.b1 = mk(m * c.z, 0.f, -m * c.x); I.b2 = mk(-m * c.y, m * c.x, 0.f);
    I.D.xx = m; I.D.yy = m; I.D.zz = m; I.D.xy = 0.f; I.D.xz = 0.f; I.D.yz = 0.f;
    return I;
}
// R * diag-ish symmetric * R^T
__device__ __forceinline__ S3 rotate_inertia(const M3& R, const S3& I) {
    // columns of R*I
    V3 r0 = mk(R.c0.x, R.c1.x, R.c2.x), r1 = mk(R.c0.y, R.c1.y, R.c2.y), r2 = mk(R.c0.z, R.c1.z, R.c2.z);  // rows of R
    V3 i0 = mul(I, r0), i1 = mul(I, r1), i2 = mul(I, r2);   // I * row_k(R)^T
    S3 o;
    o.xx = dot(r0, i0); o.yy = dot(r1, i1); o.zz = dot(r2, i2);
    o.xy = dot(r0, i1); o.xz = dot(r0, i2); o.yz = dot(r1, i2);
    return o;
}
// R * diag(d) * R^T for a body whose inertia tensor is diagonal in its own frame (every Rex box link)
__device__ __forceinline__ S3 rotate_inertia_diag(const M3& R, float dx, float dy, float dz) {
    V3 a = dx * R.c0, b = dy * R.c1, c = dz * R.c2;
    S3 o;
    o.xx = fmaf(a.x, R.c0.x, fmaf(b.x, R.c1.x, c.x * R.c2.x));
    o.yy = fmaf(a.y, R.c0.y, fmaf(b.y, R.c1.y, c.y * R.c2.y));
    o.zz = fmaf(a.z, R.c0.z, fmaf(b.z, R.c1.z, c.z * R.c2.z));
    o.xy = fmaf(a.x, R.c0.y, fmaf(b.x, R.c1.y, c.x * R.c2.y));
    o.xz = fmaf(a.x, R.c0.z, fmaf(b.x, R.c1.z, c.x * R.c2.z));
    o.yz = fmaf(a.y, R.c0.z, fmaf(b.y, R.c1.z, c.y * R.c2.z));
    return o;
}
// spatial cross products
__device__ __forceinline__ SV crm(SV v, SV m) { SV r; r.a = cross(v.a, m.a); r.l = cross(v.a, m.l) + cross(v.l, m.a); return r; }
__device__ __forceinline__ SV crf(SV v, SV f) { SV r; r.a = cross(v.a, f.a) + cross(v.l, f.l); r.l = cross(v.a, f.l); return r; }

// ----- body geometry and per-link terms, in the world-aligned frame with origin at the base position ----------------------
__device__ __forceinline__ M3 quat_to_mat(float x, float y, float z, float w) {   // btMatrix3x3::setRotation
    float d = x * x + y * y + z * z + w * w;
    float s = 2.0f / d;
    float xs = x * s, ys = y * s, zs = z * s;
    float wx = w * xs, wy = w * ys, wz = w * zs, xx = x * xs, xy = x * ys, xz = x * zs, yy = y * ys, yz = y * zs, zz = z * zs;
    M3 R;
    R.c0 = mk(1.f - (yy + zz), xy + wz, xz - wy);
    R.c1 = mk(xy - wz, 1.f - (xx + zz), yz + wx);
    R.c2 = mk(xz + wy, yz - wx, 1.f - (xx + yy));
    return R;
}
// frames of a leg's three bodies and their origins relative to the base position, from the base frame R0, the leg's model
// table LB (REXSIM_MT_LEG) and its joint angles q: shoulder about x, leg and foot about y, unrotated joint frames
__device__ __forceinline__ void leg_frames(const M3& R0, const float* LB, const float* q, M3& R1, M3& R2, M3& R3, V3& p1, V3& p2,
                                           V3& p3) {
    float s1, c1, s2, c2, s3, c3;
    sincosf(q[0], &s1, &c1); sincosf(q[1], &s2, &c2); sincosf(q[2], &s3, &c3);
    R1.c0 = R0.c0; R1.c1 = fma3(c1, R0.c1, s1 * R0.c2); R1.c2 = fma3(-s1, R0.c1, c1 * R0.c2);
    R2.c0 = fma3(c2, R1.c0, -s2 * R1.c2); R2.c1 = R1.c1; R2.c2 = fma3(s2, R1.c0, c2 * R1.c2);
    R3.c0 = fma3(c3, R2.c0, -s3 * R2.c2); R3.c1 = R2.c1; R3.c2 = fma3(s3, R2.c0, c3 * R2.c2);
    p1 = mul(R0, mk(LB[0], LB[1], LB[2]));
    p2 = p1 + mul(R1, mk(LB[16], LB[17], LB[18]));
    p3 = p2 + mul(R2, mk(LB[32], LB[33], LB[34]));
}
// world inertia R I R^T of a body whose model table holds I = (xx, yy, zz, xy, xz, yz) and a flag that I is diagonal
__device__ __forceinline__ S3 world_inertia(const M3& R, const float* I, float diag) {
    const S3 Ib = {I[0], I[1], I[2], I[3], I[4], I[5]};
    return diag != 0.f ? rotate_inertia_diag(R, Ib.xx, Ib.yy, Ib.zz) : rotate_inertia(R, Ib);
}
// gravity on mass m with its centre of mass at c, as a bias force (setGravity(0,0,-10) rex_gym_env.py:314)
__device__ __forceinline__ void gravity_bias(float m, V3 c, SV& pA) {
    const float gz = -10.0f;
    pA.a = pA.a - mk(c.y * m * gz, -c.x * m * gz, 0.f); pA.l.z -= m * gz;
}
// btMultiBody::computeAccelerationsArticulatedBodyAlgorithmMultiDof adds the damping term of the base to EVERY link too
// (m_linearDamping = m_angularDamping = 0.04, K1 = K2): torque I w (k + k|w|) about the link origin and force
// m v_o (k + k|v_o|) at it, v_o = velocity of the link origin.  Expressed about the common-frame origin (the base position).
__device__ __forceinline__ void link_damping(float k, float m, const S3& Iw, V3 p, const SV& v, SV& pA) {
    V3 vo = v.l + cross(v.a, p);
    float wn = sqrtf(dot(v.a, v.a)), vn = sqrtf(dot(vo, vo));
    V3 f = (m * fmaf(k, vn, k)) * vo;
    V3 n = fmaf(k, wn, k) * mul(Iw, v.a);
    pA.a = pA.a + n + cross(p, f);
    pA.l = pA.l + f;
}
// ABA pass 1 for one link of a limb (origin p, velocity v, mass m, centre of mass cw, world inertia Iw): its spatial inertia and
// its bias force (velocity product, gravity, link damping k)
__device__ __forceinline__ void link_terms(float m, V3 cw, const S3& Iw, V3 p, const SV& v, float k, AI& IA, SV& pA) {
    IA = rigid_inertia(m, cw, Iw);
    pA = crf(v, mul(IA, v));
    gravity_bias(m, cw, pA);
    link_damping(k, m, Iw, p, v, pA);
}

// ----- width-4 (one env) shuffles -------------------------------------------------------------------
// The member mask names only the 4 lanes of the env: different envs of a warp may diverge (stay-still
// early-outs, auto-reset, converged solvers) without deadlocking each other's shuffles.
__device__ __forceinline__ unsigned env_mask() { return 0xFu << ((threadIdx.x & 31u) & ~3u); }
__device__ __forceinline__ float bcast4(float v, int src) { return __shfl_sync(env_mask(), v, src, 4); }
__device__ __forceinline__ float sum4(float v) {
    const unsigned m = env_mask();
    v += __shfl_xor_sync(m, v, 1, 4);
    v += __shfl_xor_sync(m, v, 2, 4);
    return v;
}
__device__ __forceinline__ float max4(float v) {
    const unsigned m = env_mask();
    v = fmaxf(v, __shfl_xor_sync(m, v, 1, 4));
    v = fmaxf(v, __shfl_xor_sync(m, v, 2, 4));
    return v;
}
__device__ __forceinline__ unsigned or4(unsigned v) {
    const unsigned m = env_mask();
    v |= __shfl_xor_sync(m, v, 1, 4);
    v |= __shfl_xor_sync(m, v, 2, 4);
    return v;
}
__device__ __forceinline__ V3 sum4(V3 v) { return mk(sum4(v.x), sum4(v.y), sum4(v.z)); }
__device__ __forceinline__ SV sum4(SV v) { SV r; r.a = sum4(v.a); r.l = sum4(v.l); return r; }
__device__ __forceinline__ SV bcast4(SV v, int src) {
    SV r; r.a = mk(bcast4(v.a.x, src), bcast4(v.a.y, src), bcast4(v.a.z, src));
    r.l = mk(bcast4(v.l.x, src), bcast4(v.l.y, src), bcast4(v.l.z, src)); return r;
}

// ----- counter-based RNG, bit-identical to oracle rexo_rand_u32 ---------------------------------------
__host__ __device__ __forceinline__ uint32_t rand_u32(uint64_t seed, uint32_t env, uint32_t reset_count, uint32_t slot) {
    uint64_t z = seed + 0x9E3779B97F4A7C15ull * ((uint64_t)env + 1);
    z ^= ((uint64_t)reset_count << 32) | (uint64_t)slot;
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    return (uint32_t)(z >> 32);
}
// counter-based N(0,1): Box-Muller on two draws of the reset generator (oracle rexo_noise in fp64; include/rexsim.h rexsim_noise is this function)
__host__ __device__ __forceinline__ float noise_unit(uint64_t seed, uint32_t genv, uint32_t rc, uint32_t step, uint32_t site, uint32_t comp) {
    const uint32_t slot = 1024u + (((step * 8u + site) * 32u + comp) << 1);
    const float u1 = ((float)(rand_u32(seed, genv, rc, slot) >> 8) + 1.0f) * (1.0f / 16777216.0f);
    const float u2 = (float)(rand_u32(seed, genv, rc, slot + 1u) >> 8) * (1.0f / 16777216.0f);
    return sqrtf(-2.0f * logf(u1)) * cosf(6.283185307179586f * u2);
}
__device__ __forceinline__ double rand_uniform(uint64_t seed, uint32_t env, uint32_t rc, uint32_t slot, double a, double b) {
    double u = (double)(rand_u32(seed, env, rc, slot) >> 8) * (1.0 / 16777216.0);
    return a + (b - a) * u;
}

// ----- 1-D TMA bulk copy global -> shared, completion on an mbarrier ------------------------------------------
// thread 0 initialises the barrier for one arrival; the CTA syncs before any thread waits on it
__device__ __forceinline__ void mbar_init(uint64_t* bar) {
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
}
// thread 0 arms the barrier with `bytes` and issues the copy; every thread waits for the phase with `parity` to complete
__device__ __forceinline__ void tma_bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint32_t parity) {
    const uint32_t bar_a = (uint32_t)__cvta_generic_to_shared(bar);
    const uint32_t dst_a = (uint32_t)__cvta_generic_to_shared(smem_dst);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(dst_a), "l"(gsrc), "r"(bytes), "r"(bar_a) : "memory");
    }
    uint32_t ok = 0;
    while (!ok) {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(bar_a), "r"(parity) : "memory");
    }
}

}  // namespace rexsim

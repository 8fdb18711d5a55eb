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
// observation width: base roll, pitch and their rates, then (gallop) the motor angles
__host__ __device__ constexpr int obs_dim(int task, int num_motors) { return 4 + (task_shape(task).angles ? num_motors : 0); }

struct Params {
    RexSimConfig cfg;
    const float* __restrict__ model;   // REXSIM_MT_FLOATS floats, 16-byte aligned
    float* __restrict__ sf;            // [NF][N]
    int32_t* __restrict__ si;          // [NI][N]
    const float* __restrict__ snap_f;  // [nsnap][NF] settled reset snapshots
    const int32_t* __restrict__ snap_i;// [nsnap][NI]
    const float* __restrict__ field_zoff; // [nfields]
    int32_t* __restrict__ err;         // [N] per-env bits of the most recent step, [N] = OR of all since last cleared
    uint8_t* err_host;                 // host-buffer step with zero-copy buffers: 8 flag bytes in the caller's block, byte b = 1 when an
                                       // env raised error bit b this step (idempotent stores, no atomics across PCIe); else null
    float* __restrict__ cmd_out;       // [num_motors][N]
    const float* __restrict__ actions; // [N][A]
    float* __restrict__ obs;           // [N][O]
    float* __restrict__ reward;        // [N]
    uint8_t* __restrict__ done;        // [N]
    const int32_t* __restrict__ reset_idx; // reset kernel: [k] or null
    int32_t reset_k;
    int32_t settle_snapshot;           // settle kernel: which snapshot this launch produces
    int32_t N;
    int32_t sm_count;                  // SMs of the device (kernel variant choice)
    int32_t* launched;                 // host: {BLOCK, OCC, SENSOR} of the step_kernel instance the last step launched (never read on the device)
    const int32_t* __restrict__ perm;  // [N] slot -> env (null: identity); see rexsim_rebalance
    int32_t* __restrict__ cost;        // [N] solver iterations of the last control step
    // sensor model (control / PD latency, observation noise: rex.py:735-769); all unused when sensor_on == 0
    int32_t sensor_on;
    int32_t ring_depth;                // D rows kept per env: max(n_ctl, n_pd) + 2 (100 = the deque's maxlen when a latency reaches it)
    float* ring;                       // [D][HW_WORDS(_ARM)][N]; NOT __restrict__: lanes of an env read what lane 0 wrote
    float* snap_ring;                  // [nsnap][D][HW_WORDS(_ARM)] history the reset hold leaves behind, per field
    int32_t n_ctl, n_pd;               // int(latency / dt)
    float a_ctl, a_pd;                 // blend weight (latency - n dt) / dt of the older sample
    float lat_ctl, lat_pd;             // the latencies themselves (only their sign is used on the device)
    float noise_sd[5];                 // SENSOR_NOISE_STDDEV order: motor angle, motor velocity, motor torque, base rpy, base rpy rate
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

}  // namespace rexsim

// rexsim_kernel.cu -- sm_90a kernels: fused env step, reset, settle.  See rexsim_kernel.cuh for the design.
#include "rexsim_kernel.cuh"
#include "rexsim_arm.cuh"
#include <math.h>
#include <type_traits>
#include <stdlib.h>

namespace rexsim {

// threads per CTA: small-batch (255-register) build / large-batch (128-register) build.  The warps of a CTA re-align at every
// sub-step, so a larger CTA shares more of the instruction stream -- see REXSIM_SYNC_SUBSTEP below
#ifndef REXSIM_BLOCK
#define REXSIM_BLOCK 128
#endif
#ifndef REXSIM_BLOCK_BIG
#define REXSIM_BLOCK_BIG 256
#endif
// resident CTAs per SM of the large-batch build (register cap 65536 / (128 * REXSIM_OCC_BIG))
#ifndef REXSIM_OCC_BIG
#define REXSIM_OCC_BIG 4
#endif
// 1: the warps of a CTA re-align at every sub-step (__syncthreads) so that the ~200 KB of straight-line per-sub-step code is
// fetched once per CTA instead of once per warp (the kernel is instruction-fetch bound: ncu no_instruction stalls)
#ifndef REXSIM_SYNC_SUBSTEP
#define REXSIM_SYNC_SUBSTEP 1
#endif
// 1: the 255-register builds on flat ground without the arm solve the 12 foot-contact rows replicated on the 4 lanes of an env
// (one exchange per sub-step, no lane-to-lane traffic inside the PGS loop); 0: every build keeps the shuffle solver.
// Bit-identical either way.
#ifndef REXSIM_PGS_REPLICATED
#define REXSIM_PGS_REPLICATED 1
#endif
// the replicated loop doubles the solver's instructions to cut its serial chain: worth it where each scheduler holds one or two
// warps (the 255-register builds), not in the issue-bound 128-register build.  On heightfields the per-sub-step exchange and the
// spills around the loop cost more than the shorter chain saves (C4 turn-ik, 4096 envs: 3.7 % slower on an H100 SXM)
__host__ __device__ constexpr bool pgs_replicated(int occ, bool arm, int terrain) {
    return REXSIM_PGS_REPLICATED && occ == 1 && !arm && terrain == REXSIM_TERRAIN_PLANE;
}
// per env, in dynamic shared memory after the heightfield tiles: the 12 pre-scaled Delassus rows (row-major), their running sums
// and their denominators -- one exchange per sub-step
#define PGS_ENV_FLOATS (12 * 12 + 12 + 12)
#define PI_F 3.14159265358979323846f
#define PI_D 3.14159265358979323846

// -------------------------------------------------------------------------------------------------
// model tables: one 1-D TMA bulk copy global -> shared per CTA (cp.async.bulk + mbarrier)
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_tables(float* smem_dst, const float* gsrc, uint32_t bytes, uint64_t* bar) {
    uint32_t bar_a = (uint32_t)__cvta_generic_to_shared(bar);
    uint32_t dst_a = (uint32_t)__cvta_generic_to_shared(smem_dst);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(dst_a), "l"(gsrc), "r"(bytes), "r"(bar_a) : "memory");
    }
    uint32_t ok = 0;
    while (!ok) {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(bar_a), "r"(0u) : "memory");
    }
}

// -------------------------------------------------------------------------------------------------
// per-lane (leg) working set
// -------------------------------------------------------------------------------------------------
struct Lane {
    // base (replicated on the 4 lanes of an env)
    V3 pos; float qx, qy, qz, qw; V3 vl, w;
    // own leg
    float q[3], qd[3];
    float tau_obs[3];
    uint32_t ovh;          // 3 x 10-bit overheat counters
    uint32_t enabled;      // 3 bits
    int contact;           // own toe in contact during the last sub-step
    int err;
    int cost;              // solver iterations spent this control step (drives the warp re-grouping, rexsim_rebalance)
};

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
__device__ __forceinline__ void quat_to_euler(float x, float y, float z, float w, float* rpy) {   // pybullet getEulerFromQuaternion
    float sqx = x * x, sqy = y * y, sqz = z * z, squ = w * w;
    float sarg = -2.f * (x * z - w * y);
    if (sarg <= -0.99999f) { rpy[0] = 0; rpy[1] = -0.5f * PI_F; rpy[2] = 2 * atan2f(x, -y); }
    else if (sarg >= 0.99999f) { rpy[0] = 0; rpy[1] = 0.5f * PI_F; rpy[2] = 2 * atan2f(-x, y); }
    else {
        rpy[0] = atan2f(2 * (y * z + w * x), squ - sqx - sqy + sqz);
        rpy[1] = asinf(sarg);
        rpy[2] = atan2f(2 * (x * y + w * z), squ + sqx - sqy - sqz);
    }
}

__device__ __forceinline__ void euler_to_quat(const float* rpy, float* q) {                        // pybullet getQuaternionFromEuler
    float sr, cr, sp, cp, sy, cy;
    sincosf(rpy[0] * 0.5f, &sr, &cr); sincosf(rpy[1] * 0.5f, &sp, &cp); sincosf(rpy[2] * 0.5f, &sy, &cy);
    q[0] = sr * cp * cy - cr * sp * sy;
    q[1] = cr * sp * cy + sr * cp * sy;
    q[2] = cr * cp * sy - sr * sp * cy;
    q[3] = cr * cp * cy + sr * sp * sy;
}

// -------------------------------------------------------------------------------------------------
// sensor model: observation history, latency, noise (rex_gym/model/rex.py:122,726-769)
// -------------------------------------------------------------------------------------------------
// One row per ReceiveObservation (= per sub-step) in a ring of P.ring_depth rows, ring[slot][word][env]; `push` counts the rows
// since Rex.Reset cleared the deque (I_HPUSH), so history[k] (k = 0 newest) sits in slot (push - 1 - k) mod depth and the
// deque's length is min(push, 100).  Every lane writes / reads the 9 words of its own leg; lane 0 writes the 7 base words
// (and the arm's 18), which the other lanes read after a __syncwarp over the env's 4 lanes.
struct Sensor { float* ring; int N, env, depth, words, push; uint32_t genv, rc; };
template <bool ARM>
__device__ __forceinline__ Sensor make_sensor(const Params& P, float* ring, int N, int env, uint32_t genv) {   // no rows pushed yet
    return Sensor{ring, N, env, P.ring_depth, ARM ? HW_WORDS_ARM : HW_WORDS, 0, genv, 0u};
}

template <bool ARM>
__device__ __forceinline__ void sensor_push(Sensor& S, int leg, const Lane& L, const Arm& AR, bool valid) {
    if (valid) {
        float* r = S.ring + ((size_t)(S.push % S.depth) * S.words) * S.N + S.env;
        const size_t N = (size_t)S.N;
#pragma unroll
        for (int j = 0; j < 3; j++) {
            r[(9 * leg + j) * N] = L.q[j]; r[(9 * leg + 3 + j) * N] = L.qd[j]; r[(9 * leg + 6 + j) * N] = L.tau_obs[j];
        }
        if (leg == 0) {
            r[(HW_BASE + 0) * N] = L.qx; r[(HW_BASE + 1) * N] = L.qy; r[(HW_BASE + 2) * N] = L.qz; r[(HW_BASE + 3) * N] = L.qw;
            r[(HW_BASE + 4) * N] = L.w.x; r[(HW_BASE + 5) * N] = L.w.y; r[(HW_BASE + 6) * N] = L.w.z;
            if (ARM) {
#pragma unroll
                for (int j = 0; j < ARM_NJ; j++) {
                    r[(HW_ARM + j) * N] = AR.q[j]; r[(HW_ARM + 6 + j) * N] = AR.qd[j]; r[(HW_ARM + 12 + j) * N] = AR.tau_obs[j];
                }
            }
        }
    }
    S.push++;
    __syncwarp(env_mask());          // the base words of lane 0 are visible to the env's other lanes from here on
}
// Rex._GetDelayedObservation (rex.py:735-753) for one word of the row: n = int(latency / dt), a = (latency - n dt) / dt
__device__ __forceinline__ float sensor_delayed(const Sensor& S, float latency, int n, float a, int word) {
    const int len = min(S.push, (int)HIST_MAXLEN);
    const float* base = S.ring + (size_t)word * S.N + S.env;
    const size_t row = (size_t)S.words * S.N;
    auto at = [&](int k) { return base[(size_t)((S.push - 1 - k) % S.depth) * row]; };
    if (latency <= 0.f || len == 1) return at(0);
    if (n + 1 >= len) return at(len - 1);
    return (1.0f - a) * at(n) + a * at(n + 1);
}
__device__ __forceinline__ float sensor_noise(const Params& P, const Sensor& S, uint32_t step, int group, uint32_t site, uint32_t comp) {
    const float sd = P.noise_sd[group];
    if (sd <= 0.f) return 0.f;
    return sd * noise_unit(P.cfg.seed, S.genv, S.rc, step, site, comp);
}
// Rex.GetBaseOrientation (rex.py:530-537): quaternion of (Euler angles of the DELAYED orientation + noise)
__device__ __forceinline__ void sensed_quat(const Params& P, const Sensor& S, uint32_t step, uint32_t site, float* q4) {
    float d4[4], rpy[3];
#pragma unroll
    for (int a = 0; a < 4; a++) d4[a] = sensor_delayed(S, P.lat_ctl, P.n_ctl, P.a_ctl, HW_BASE + a);
    quat_to_euler(d4[0], d4[1], d4[2], d4[3], rpy);
#pragma unroll
    for (int a = 0; a < 3; a++) rpy[a] += sensor_noise(P, S, step, 3, site, a);
    euler_to_quat(rpy, q4);
}

// 6x6 SPD inverse (symmetric storage m[i][j], i>=j used) via Cholesky, fully unrolled in registers
struct Sym6 { float m[21]; };   // packed lower: idx(i,j) = i*(i+1)/2 + j
__device__ __forceinline__ constexpr int ix(int i, int j) { return i >= j ? i * (i + 1) / 2 + j : j * (j + 1) / 2 + i; }
__device__ __forceinline__ Sym6 pack(const AI& I) {
    Sym6 s;
    s.m[ix(0, 0)] = I.A.xx; s.m[ix(1, 0)] = I.A.xy; s.m[ix(1, 1)] = I.A.yy; s.m[ix(2, 0)] = I.A.xz; s.m[ix(2, 1)] = I.A.yz; s.m[ix(2, 2)] = I.A.zz;
    // lower-left block = B^T : element (3+j, i) = B[i][j]
    s.m[ix(3, 0)] = I.b0.x; s.m[ix(3, 1)] = I.b1.x; s.m[ix(3, 2)] = I.b2.x;
    s.m[ix(4, 0)] = I.b0.y; s.m[ix(4, 1)] = I.b1.y; s.m[ix(4, 2)] = I.b2.y;
    s.m[ix(5, 0)] = I.b0.z; s.m[ix(5, 1)] = I.b1.z; s.m[ix(5, 2)] = I.b2.z;
    s.m[ix(3, 3)] = I.D.xx; s.m[ix(4, 3)] = I.D.xy; s.m[ix(4, 4)] = I.D.yy; s.m[ix(5, 3)] = I.D.xz; s.m[ix(5, 4)] = I.D.yz; s.m[ix(5, 5)] = I.D.zz;
    return s;
}
__device__ __forceinline__ Sym6 spd_inverse(const Sym6& A) {
    float L[21], invd[6];      // invd[j] = 1 / L[j][j]: every division of the factorisation becomes a multiply
#pragma unroll
    for (int j = 0; j < 6; j++) {
        float s = A.m[ix(j, j)];
#pragma unroll
        for (int k = 0; k < j; k++) s = fmaf(-L[ix(j, k)], L[ix(j, k)], s);
        float inv = rsqrtf(s);
        // one Newton step keeps the factor at full fp32 accuracy
        inv = inv * (1.5f - 0.5f * s * inv * inv);
        L[ix(j, j)] = s * inv;
        invd[j] = inv;
#pragma unroll
        for (int i = j + 1; i < 6; i++) {
            float t = A.m[ix(i, j)];
#pragma unroll
            for (int k = 0; k < j; k++) t = fmaf(-L[ix(i, k)], L[ix(j, k)], t);
            L[ix(i, j)] = t * inv;
        }
    }
    // Linv (lower)
    float Li[21];
#pragma unroll
    for (int j = 0; j < 6; j++) {
        Li[ix(j, j)] = invd[j];
#pragma unroll
        for (int i = j + 1; i < 6; i++) {
            float t = 0.f;
#pragma unroll
            for (int k = j; k < i; k++) t = fmaf(-L[ix(i, k)], Li[ix(k, j)], t);
            Li[ix(i, j)] = t * invd[i];
        }
    }
    Sym6 R;   // A^-1 = Li^T Li
#pragma unroll
    for (int i = 0; i < 6; i++)
#pragma unroll
        for (int j = 0; j <= i; j++) {
            float t = 0.f;
#pragma unroll
            for (int k = i; k < 6; k++) t = fmaf(Li[ix(k, i)], Li[ix(k, j)], t);
            R.m[ix(i, j)] = t;
        }
    return R;
}
__device__ __forceinline__ SV neg_mul(const Sym6& M, SV p) {   // -(M p)
    float v[6] = {p.a.x, p.a.y, p.a.z, p.l.x, p.l.y, p.l.z}, o[6];
#pragma unroll
    for (int i = 0; i < 6; i++) {
        float t = 0.f;
#pragma unroll
        for (int j = 0; j < 6; j++) t = fmaf(M.m[ix(i, j)], v[j], t);
        o[i] = -t;
    }
    SV r; r.a = mk(o[0], o[1], o[2]); r.l = mk(o[3], o[4], o[5]);
    return r;
}

// ground query --------------------------------------------------------------------------------------
// Random terrain (rex_gym/model/terrain.py:32-53): every env stages a 16x16-cell (0.8 m x 0.8 m) window of its
// heightfield, centred on the base, in shared memory once per control step; all contact queries of the step's
// sub-steps read that tile (4 heights per query) instead of the 256x256 field in L2.
#define TILE_CELLS 16
#define TILE_V (TILE_CELLS + 1)          // vertices per side
#define TILE_STRIDE (TILE_V + 1)         // padded row
#define TILE_FLOATS (TILE_V * TILE_STRIDE)
struct Ground { const float* tile; int ix0, iy0; float zoff; int miss; };

template <int TERRAIN>
__device__ __forceinline__ void load_tile(const Params& P, int field, V3 pos, float* tile, Ground& G, int leg) {
    G.tile = tile; G.ix0 = 0; G.iy0 = 0; G.zoff = 0.f; G.miss = 0;
    if (TERRAIN != REXSIM_TERRAIN_RANDOM) return;
    const float* h = P.cfg.fields + (size_t)field * 65536;
    int cx = (int)floorf(pos.x * 20.0f + 127.5f), cy = (int)floorf(pos.y * 20.0f + 127.5f);
    G.ix0 = min(max(cx - TILE_CELLS / 2, 0), 255 - TILE_CELLS);
    G.iy0 = min(max(cy - TILE_CELLS / 2, 0), 255 - TILE_CELLS);
    G.zoff = P.field_zoff[field];
    // the 4 lanes of the env copy rows leg, leg+4, ... (17 consecutive floats per row)
    for (int r = leg; r < TILE_V; r += 4) {
        const float* src = h + (G.iy0 + r) * 256 + G.ix0;
#pragma unroll
        for (int c = 0; c < TILE_V; c++) tile[r * TILE_STRIDE + c] = __ldg(src + c);
    }
    __syncwarp(env_mask());
}
template <int TERRAIN>
__device__ __forceinline__ void ground_query(Ground& G, V3 wp, float& dist, V3& n) {
    if (TERRAIN == REXSIM_TERRAIN_PLANE) { dist = wp.z; n = mk(0.f, 0.f, 1.f); return; }
    const float inv_cell = 20.0f;   // 1/0.05
    float fx = fminf(fmaxf(wp.x * inv_cell + 127.5f, 0.f), 254.999f);
    float fy = fminf(fmaxf(wp.y * inv_cell + 127.5f, 0.f), 254.999f);
    int ixx = (int)floorf(fx), iyy = (int)floorf(fy);
    float u = fx - ixx, v = fy - iyy;
    int lx = ixx - G.ix0, ly = iyy - G.iy0;
    if (lx < 0 || lx >= TILE_CELLS || ly < 0 || ly >= TILE_CELLS) {      // outside the staged window: flag, clamp
        G.miss = 1; lx = min(max(lx, 0), TILE_CELLS - 1); ly = min(max(ly, 0), TILE_CELLS - 1);
    }
    const float* t = G.tile + ly * TILE_STRIDE + lx;
    float h00 = t[0], h10 = t[1], h01 = t[TILE_STRIDE], h11 = t[TILE_STRIDE + 1];
    float hx, hy;
    if (v >= u) { hx = h11 - h01; hy = h01 - h00; } else { hx = h10 - h00; hy = h11 - h10; }
    float hh = h00 + hx * u + hy * v - G.zoff;
    float nx = -hx * inv_cell, ny = -hy * inv_cell;
    float inv = rsqrtf(nx * nx + ny * ny + 1.f);
    n = mk(nx * inv, ny * inv, inv);
    dist = (wp.z - hh) * n.z;
}
__device__ __forceinline__ void plane_space(V3 n, V3& p, V3& q) {   // btPlaneSpace1
    if (fabsf(n.z) > 0.70710678118654752440f) {
        float a = n.y * n.y + n.z * n.z, k = rsqrtf(a);
        p = mk(0.f, -n.z * k, n.y * k);
        q = mk(a * k, -n.x * p.z, n.x * p.y);
    } else {
        float a = n.x * n.x + n.y * n.y, k = rsqrtf(a);
        p = mk(-n.y * k, n.x * k, 0.f);
        q = mk(-n.z * p.y, n.z * p.x, a * k);
    }
}

// generic-path Gauss-Seidel order after the limit rows (rows 0..2 of a lane = its three joint limits): normals (base, then per leg upper, foot), then frictions
static __constant__ int c_seq_owner[27] = {0, 0, 0, 1, 1, 2, 2, 3, 3, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3};
static __constant__ int c_seq_row[27] = {3, 6, 9, 6, 9, 6, 9, 6, 9, 4, 5, 7, 8, 10, 11, 7, 8, 10, 11, 7, 8, 10, 11, 7, 8, 10, 11};

// motor model + overheat (rex_gym/model/motor.py:76-143, rex_gym/model/rex.py:601-623) for one joint
// q, qd: what the PD loop sees (pd_latency ago, rex.py:755-759); qd_true: the motor's actual rate (back-EMF, motor.py:131)
__device__ __forceinline__ float motor_torque(float cmd, float q, float qd, float qd_true, float kp, float kd, float& tau_obs) {
    const float V = 32.0f, R = 0.186f, Kt = 0.0954f;
    float pwm = -1.f * kp * (q - cmd) - kd * qd;
    pwm = fminf(fmaxf(pwm, -1.f), 1.f);
    const float VoR = V / R, invR = 1.0f / R;     // compile-time constants: the per-motor divisions become multiplies
    tau_obs = fminf(fmaxf(Kt * (pwm * VoR), -5.7f), 5.7f);
    float vnet = fminf(fmaxf(pwm * V - Kt * qd_true, -50.f), 50.f);
    float cur = vnet * invR;
    float mag = fabsf(cur), t;
    // np.interp over [0,10,...,60] -> [0,1,1.9,2.45,3.0,3.25,3.5]
    if (mag >= 60.f) t = 3.5f;
    else if (mag >= 50.f) t = 0.025f * (mag - 50.f) + 3.25f;
    else if (mag >= 40.f) t = 0.025f * (mag - 40.f) + 3.0f;
    else if (mag >= 30.f) t = 0.055f * (mag - 30.f) + 2.45f;
    else if (mag >= 20.f) t = 0.055f * (mag - 20.f) + 1.9f;
    else if (mag >= 10.f) t = 0.09f * (mag - 10.f) + 1.0f;
    else t = 0.1f * mag;
    return copysignf(t, cur) * (cur != 0.f ? 1.f : 0.f);
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
__device__ __forceinline__ float clampv(float v, float lim) { return fminf(fmaxf(v, -lim), lim); }

// -------------------------------------------------------------------------------------------------
// one pybullet.stepSimulation for the 4 lanes of an env (call site rex_gym/model/rex.py:161)
// -------------------------------------------------------------------------------------------------
// REPL: the 12-row fast path runs the replicated PGS loop (REXSIM_PGS_REPLICATED) instead of the shuffle loop, exchanging the
// rows through the env's PGS_ENV_FLOATS floats of shared memory at `pgs`
template <int TERRAIN, bool ARM, bool REPL>
__device__ __forceinline__ void physics_substep(const Params& P, const float* __restrict__ sm, Lane& L, int leg,
                                                const float* tau, Ground& G, Arm& AR, const float* tauA, float* pgs) {
    const float dt = (float)P.cfg.sim_dt_d;
    const float inv_dt = 1.0f / dt;
    const float* LB = sm + REXSIM_MT_LEG + leg * 48;
    // ---- forward kinematics, world-aligned frame with origin at the base position -------------------
    M3 R0 = quat_to_mat(L.qx, L.qy, L.qz, L.qw);
    float s1, c1, s2, c2, s3, c3;
    sincosf(L.q[0], &s1, &c1); sincosf(L.q[1], &s2, &c2); sincosf(L.q[2], &s3, &c3);
    M3 R1; R1.c0 = R0.c0; R1.c1 = fma3(c1, R0.c1, s1 * R0.c2); R1.c2 = fma3(-s1, R0.c1, c1 * R0.c2);
    M3 R2; R2.c0 = fma3(c2, R1.c0, -s2 * R1.c2); R2.c1 = R1.c1; R2.c2 = fma3(s2, R1.c0, c2 * R1.c2);
    M3 R3; R3.c0 = fma3(c3, R2.c0, -s3 * R2.c2); R3.c1 = R2.c1; R3.c2 = fma3(s3, R2.c0, c3 * R2.c2);
    V3 p1 = mul(R0, mk(LB[0], LB[1], LB[2]));
    V3 p2 = p1 + mul(R1, mk(LB[16], LB[17], LB[18]));
    V3 p3 = p2 + mul(R2, mk(LB[32], LB[33], LB[34]));
    SV S1, S2, S3v;
    S1.a = R0.c0; S1.l = cross(p1, S1.a);
    S2.a = R1.c1; S2.l = cross(p2, S2.a);
    S3v.a = R2.c1; S3v.l = cross(p3, S3v.a);
    // ---- velocities and bias terms ------------------------------------------------------------------
    SV v0; v0.a = L.w; v0.l = L.vl;
    SV vj1 = L.qd[0] * S1, vj2 = L.qd[1] * S2, vj3 = L.qd[2] * S3v;
    SV v1 = v0 + vj1, v2 = v1 + vj2, v3 = v2 + vj3;
    SV cJ1 = crm(v1, vj1), cJ2 = crm(v2, vj2), cJ3 = crm(v3, vj3);
    const float gz = -10.0f;   // setGravity(0,0,-10) rex_gym_env.py:314
    AI IA1, IA2, IA3; SV pA1, pA2, pA3;
    {
        float m = LB[3]; V3 cw = p1 + mul(R1, mk(LB[4], LB[5], LB[6]));
        S3 Ib = {LB[8], LB[9], LB[10], LB[11], LB[12], LB[13]};
        const S3 Iw = (LB[15] != 0.f ? rotate_inertia_diag(R1, Ib.xx, Ib.yy, Ib.zz) : rotate_inertia(R1, Ib));
        IA1 = rigid_inertia(m, cw, Iw);
        pA1 = crf(v1, mul(IA1, v1));
        pA1.a = pA1.a - mk(cw.y * m * gz, -cw.x * m * gz, 0.f); pA1.l.z -= m * gz;
        link_damping(P.cfg.link_damping, m, Iw, p1, v1, pA1);
    }
    {
        float m = LB[16 + 3]; V3 cw = p2 + mul(R2, mk(LB[16 + 4], LB[16 + 5], LB[16 + 6]));
        S3 Ib = {LB[16 + 8], LB[16 + 9], LB[16 + 10], LB[16 + 11], LB[16 + 12], LB[16 + 13]};
        const S3 Iw = (LB[16 + 15] != 0.f ? rotate_inertia_diag(R2, Ib.xx, Ib.yy, Ib.zz) : rotate_inertia(R2, Ib));
        IA2 = rigid_inertia(m, cw, Iw);
        pA2 = crf(v2, mul(IA2, v2));
        pA2.a = pA2.a - mk(cw.y * m * gz, -cw.x * m * gz, 0.f); pA2.l.z -= m * gz;
        link_damping(P.cfg.link_damping, m, Iw, p2, v2, pA2);
    }
    {
        float m = LB[32 + 3]; V3 cw = p3 + mul(R3, mk(LB[32 + 4], LB[32 + 5], LB[32 + 6]));
        S3 Ib = {LB[32 + 8], LB[32 + 9], LB[32 + 10], LB[32 + 11], LB[32 + 12], LB[32 + 13]};
        const S3 Iw = (LB[32 + 15] != 0.f ? rotate_inertia_diag(R3, Ib.xx, Ib.yy, Ib.zz) : rotate_inertia(R3, Ib));
        IA3 = rigid_inertia(m, cw, Iw);
        pA3 = crf(v3, mul(IA3, v3));
        pA3.a = pA3.a - mk(cw.y * m * gz, -cw.x * m * gz, 0.f); pA3.l.z -= m * gz;
        link_damping(P.cfg.link_damping, m, Iw, p3, v3, pA3);
    }
    // ---- ABA inward pass over the own leg ------------------------------------------------------------
    SV U3 = mul(IA3, S3v); float k3 = 1.0f / sdot(S3v, U3); float u3 = tau[2] - sdot(S3v, pA3);
    rank1_sub(IA3, U3, k3);
    pA3 = sfma(u3 * k3, U3, pA3 + mul(IA3, cJ3));
    add(IA2, IA3); pA2 = pA2 + pA3;
    SV U2 = mul(IA2, S2); float k2 = 1.0f / sdot(S2, U2); float u2 = tau[1] - sdot(S2, pA2);
    rank1_sub(IA2, U2, k2);
    pA2 = sfma(u2 * k2, U2, pA2 + mul(IA2, cJ2));
    add(IA1, IA2); pA1 = pA1 + pA2;
    SV U1 = mul(IA1, S1); float k1 = 1.0f / sdot(S1, U1); float u1 = tau[0] - sdot(S1, pA1);
    rank1_sub(IA1, U1, k1);
    pA1 = sfma(u1 * k1, U1, pA1 + mul(IA1, cJ1));
    if (ARM && leg == 0) {   // the arm is a fifth limb of lane 0: fold its articulated inertia into this lane's sum
        AI Ia; SV pa; SV vb; vb.a = L.w; vb.l = L.vl;
        arm_inward(sm + REXSIM_MT_ARM, R0, vb, AR, tauA, Ia, pa, P.cfg.link_damping);
        add(IA1, Ia); pA1 = pA1 + pa;
    }
    // ---- base: reduce the 4 legs, add the base body, invert ------------------------------------------
    AI IA0; SV pA0;
    {
        const float* B = sm + REXSIM_MT_BASE;
        float m = B[0]; V3 cw = mul(R0, mk(B[1], B[2], B[3]));
        S3 Ib = {B[4], B[5], B[6], B[7], B[8], B[9]};
        IA0 = rigid_inertia(m, cw, B[14] != 0.f ? rotate_inertia_diag(R0, Ib.xx, Ib.yy, Ib.zz) : rotate_inertia(R0, Ib));
        pA0 = crf(v0, mul(IA0, v0));
        pA0.a = pA0.a - mk(cw.y * m * gz, -cw.x * m * gz, 0.f); pA0.l.z -= m * gz;
        // Bullet default base damping 0.04 (K1 = K2) with the un-merged root link's mass / inertia
        const float kd = 0.04f;
        V3 wb = mk(dot(R0.c0, L.w), dot(R0.c1, L.w), dot(R0.c2, L.w));
        float wn = sqrtf(dot(wb, wb)), vn = sqrtf(dot(L.vl, L.vl));
        V3 tb = mk(B[11] * wb.x, B[12] * wb.y, B[13] * wb.z);
        pA0.a = fma3(kd + kd * wn, mul(R0, tb), pA0.a);
        pA0.l = fma3(B[10] * (kd + kd * vn), L.vl, pA0.l);
        AI Is;
        Is.A.xx = sum4(IA1.A.xx); Is.A.yy = sum4(IA1.A.yy); Is.A.zz = sum4(IA1.A.zz);
        Is.A.xy = sum4(IA1.A.xy); Is.A.xz = sum4(IA1.A.xz); Is.A.yz = sum4(IA1.A.yz);
        Is.D.xx = sum4(IA1.D.xx); Is.D.yy = sum4(IA1.D.yy); Is.D.zz = sum4(IA1.D.zz);
        Is.D.xy = sum4(IA1.D.xy); Is.D.xz = sum4(IA1.D.xz); Is.D.yz = sum4(IA1.D.yz);
        Is.b0 = sum4(IA1.b0); Is.b1 = sum4(IA1.b1); Is.b2 = sum4(IA1.b2);
        add(IA0, Is);
        pA0 = pA0 + sum4(pA1);
    }
    Sym6 Minv = spd_inverse(pack(IA0));
    SV a0 = neg_mul(Minv, pA0);
    // ---- ABA outward pass ------------------------------------------------------------------------------
    SV a1 = a0 + cJ1; float qdd1 = (u1 - sdot(U1, a1)) * k1; a1 = sfma(qdd1, S1, a1);
    SV a2 = a1 + cJ2; float qdd2 = (u2 - sdot(U2, a2)) * k2; a2 = sfma(qdd2, S2, a2);
    SV a3 = a2 + cJ3; float qdd3 = (u3 - sdot(U3, a3)) * k3;
    // unconstrained velocities (btMultiBodyDynamicsWorld::solveConstraints: v += a*dt)
    SV vs; vs.a = fma3(dt, a0.a, L.w); vs.l = fma3(dt, a0.l + cross(L.w, L.vl), L.vl);
    float qs1 = fmaf(dt, qdd1, L.qd[0]), qs2 = fmaf(dt, qdd2, L.qd[1]), qs3 = fmaf(dt, qdd3, L.qd[2]);
    // btMultiBody::applyDeltaVeeMultiDof clamps all 6+n generalised velocities to +-m_maxCoordinateVelocity (100)
    const float vmax = P.cfg.max_coordinate_velocity;
    vs.a = mk(clampv(vs.a.x, vmax), clampv(vs.a.y, vmax), clampv(vs.a.z, vmax));
    vs.l = mk(clampv(vs.l.x, vmax), clampv(vs.l.y, vmax), clampv(vs.l.z, vmax));
    qs1 = clampv(qs1, vmax); qs2 = clampv(qs2, vmax); qs3 = clampv(qs3, vmax);
    if (ARM && leg == 0) arm_outward(AR, a0, dt, vmax);

    // ---- contact candidates: ONE contact per group = its deepest sample point (same groups/order as the oracle) ----
    //   foot group  (own lane): foot box corners, then the toe hull (exact prism support, toe_margin = 0)
    //   upper group (own lane): shoulder box corners, then leg box corners
    //   base group  (owned by lane 0): base + chassis box corners, searched 6 per lane
    float best = 1e30f; V3 rc = mk(0.f, 0.f, 0.f), nrm = mk(0.f, 0.f, 1.f);
    float bestU = 1e30f; V3 rcU = mk(0.f, 0.f, 0.f), nrmU = mk(0.f, 0.f, 1.f); int kU = 1;
    float bestB = 1e30f; V3 rcB = mk(0.f, 0.f, 0.f), nrmB = mk(0.f, 0.f, 1.f);
    const float* BXl = sm + REXSIM_MT_BOX + leg * 72;
    const float* TPl = sm + REXSIM_MT_TOE;          // [npts][2] (x, z) profile of the toe prism, foot frame
    const float toe_w = sm[REXSIM_MT_BASE + 15];     // prism half width along y
    const float* BBl = sm + REXSIM_MT_BASEBOX;
    const int npts = P.cfg.toe_npts;
    int jb = 0;
    if (TERRAIN == REXSIM_TERRAIN_PLANE) {
        // flat ground: the distance is the world z, so the scan needs one row of the rotation (3 FMA per point);
        // the winning point is reconstructed once afterwards
        int jf = 0, ju = 0;
        const V3 z3 = mk(R3.c0.z, R3.c1.z, R3.c2.z), z2 = mk(R2.c0.z, R2.c1.z, R2.c2.z), z1 = mk(R1.c0.z, R1.c1.z, R1.c2.z), z0 = mk(R0.c0.z, R0.c1.z, R0.c2.z);
        // conservative reach bounds (largest corner distance from the body origin, from the URDF boxes): a group whose
        // body origin is higher than its reach cannot touch z = 0, so its scan is skipped (standing / walking: all three)
        const float zf = p3.z + L.pos.z, zs = p1.z + L.pos.z, zl = p2.z + L.pos.z;
        if (zf < 0.115f) {
#pragma unroll 4
            for (int j = 0; j < 8; j++) {
                float d = dot(z3, mk(BXl[48 + 3 * j], BXl[48 + 3 * j + 1], BXl[48 + 3 * j + 2]));
                if (d < best) { best = d; jf = j; }
            }
        }
        {
            // toe prism: the deepest hull vertex is the profile vertex minimising z3.x*x + z3.z*z on the y face that
            // minimises z3.y*y (exact support function of the hull: 2 FMA per profile vertex)
            // The profile is an ordered arc of a convex polygon, so d(j) = z3.x*x_j + z3.z*z_j has at most one interior
            // minimum along it: sample every 8th vertex (+ the last), then the 7 neighbours either side of the best sample --
            // 9 + 15 evaluations instead of 68, same argmin as the full scan (ties aside).
            float bc = 1e30f; int jc = 0;
#pragma unroll 3
            for (int j = 0; j < npts; j += 8) {
                float d = fmaf(z3.x, TPl[2 * j], z3.z * TPl[2 * j + 1]);
                if (d < bc) { bc = d; jc = j; }
            }
            {
                const int j = npts - 1;
                float d = fmaf(z3.x, TPl[2 * j], z3.z * TPl[2 * j + 1]);
                if (d < bc) { bc = d; jc = j; }
            }
            float bt = bc; int jt = jc;
            const int jlo = max(jc - 7, 0), jhi = min(jc + 7, npts - 1);
#pragma unroll 3
            for (int j = jlo; j <= jhi; j++) {
                float d = fmaf(z3.x, TPl[2 * j], z3.z * TPl[2 * j + 1]);
                if (d < bt || (d == bt && j < jt)) { bt = d; jt = j; }
            }
            bt -= fabsf(z3.y) * toe_w + P.cfg.toe_margin;
            if (bt < best) { best = bt; jf = 8 + jt; }
        }
        {
            const V3 q = jf < 8 ? mk(BXl[48 + 3 * jf], BXl[48 + 3 * jf + 1], BXl[48 + 3 * jf + 2])
                                : mk(TPl[2 * (jf - 8)], z3.y > 0.f ? -toe_w : (z3.y < 0.f ? toe_w : -toe_w), TPl[2 * (jf - 8) + 1]);
            rc = p3 + mul(R3, q);
            best += p3.z + L.pos.z;
        }
        if (zs < 0.05f || zl < 0.12f) {
#pragma unroll 4
            for (int j = 0; j < 16; j++) {
                const bool sh = j < 8;
                float d = dot(sh ? z1 : z2, mk(BXl[3 * j], BXl[3 * j + 1], BXl[3 * j + 2])) + (sh ? p1.z : p2.z);
                if (d < bestU) { bestU = d; ju = j; }
            }
            kU = ju < 8 ? 1 : 2;
            V3 c = mk(BXl[3 * ju], BXl[3 * ju + 1], BXl[3 * ju + 2]);
            rcU = kU == 1 ? p1 + mul(R1, c) : p2 + mul(R2, c);
            bestU += L.pos.z;
        }
        if (L.pos.z < 0.19f) {          // env-uniform: the base pose is replicated on the 4 lanes
#pragma unroll
            for (int jj = 0; jj < 6; jj++) {
                const int j = 6 * leg + jj;
                float d = dot(z0, mk(BBl[3 * j], BBl[3 * j + 1], BBl[3 * j + 2]));
                if (d < bestB) { bestB = d; jb = j; }
            }
            const unsigned m4 = env_mask();
#pragma unroll
            for (int o = 1; o < 4; o <<= 1) {
                float od = __shfl_xor_sync(m4, bestB, o, 4); int oj = __shfl_xor_sync(m4, jb, o, 4);
                if (od < bestB || (od == bestB && oj < jb)) { bestB = od; jb = oj; }
            }
            rcB = mul(R0, mk(BBl[3 * jb], BBl[3 * jb + 1], BBl[3 * jb + 2]));
            bestB += L.pos.z;
        }
    } else {
#pragma unroll 1
        for (int j = 0; j < 8; j++) {
            V3 r = p3 + mul(R3, mk(BXl[48 + 3 * j], BXl[48 + 3 * j + 1], BXl[48 + 3 * j + 2]));
            float d; V3 n;
            if (r.z + L.pos.z > 0.06f) continue;
            ground_query<TERRAIN>(G, mk(r.x + L.pos.x, r.y + L.pos.y, r.z + L.pos.z), d, n);
            if (d < best) { best = d; rc = r; nrm = n; }
        }
        // heightfield: every 4th profile vertex (+ the last one) on both faces of the prism, same subset as the oracle
#pragma unroll 1
        for (int side = 0; side < 2; side++) {
#pragma unroll 1
            for (int j = 0; j < npts; j = (j + 4 < npts || j == npts - 1) ? j + 4 : npts - 1) {
                V3 r = p3 + mul(R3, mk(TPl[2 * j], side ? toe_w : -toe_w, TPl[2 * j + 1]));
                float d; V3 n;
                if (r.z + L.pos.z <= 0.06f) {
                    ground_query<TERRAIN>(G, mk(r.x + L.pos.x, r.y + L.pos.y, r.z + L.pos.z), d, n);
                    d -= P.cfg.toe_margin;
                    if (d < best) { best = d; rc = r; nrm = n; }
                }
            }
        }
#pragma unroll 1
        for (int j = 0; j < 16; j++) {
            const bool sh = j < 8;
            V3 c = mk(BXl[3 * j], BXl[3 * j + 1], BXl[3 * j + 2]);
            V3 r = sh ? p1 + mul(R1, c) : p2 + mul(R2, c);
            float d; V3 n;
            if (r.z + L.pos.z > 0.06f) continue;
            ground_query<TERRAIN>(G, mk(r.x + L.pos.x, r.y + L.pos.y, r.z + L.pos.z), d, n);
            if (d < bestU) { bestU = d; rcU = r; nrmU = n; kU = sh ? 1 : 2; }
        }
#pragma unroll 1
        for (int jj = 0; jj < 6; jj++) {
            const int j = 6 * leg + jj;
            V3 r = mul(R0, mk(BBl[3 * j], BBl[3 * j + 1], BBl[3 * j + 2]));
            float d; V3 n;
            if (r.z + L.pos.z > 0.06f) continue;
            ground_query<TERRAIN>(G, mk(r.x + L.pos.x, r.y + L.pos.y, r.z + L.pos.z), d, n);
            if (d < bestB) { bestB = d; rcB = r; nrmB = n; jb = j; }
        }
        // argmin over the 4 lanes; ties resolve to the lowest point index like the oracle's sequential scan
        const unsigned m4 = env_mask();
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {
            float od = __shfl_xor_sync(m4, bestB, o, 4); int oj = __shfl_xor_sync(m4, jb, o, 4);
            V3 orc = mk(__shfl_xor_sync(m4, rcB.x, o, 4), __shfl_xor_sync(m4, rcB.y, o, 4), __shfl_xor_sync(m4, rcB.z, o, 4));
            V3 onr = mk(__shfl_xor_sync(m4, nrmB.x, o, 4), __shfl_xor_sync(m4, nrmB.y, o, 4), __shfl_xor_sync(m4, nrmB.z, o, 4));
            if (od < bestB || (od == bestB && oj < jb)) { bestB = od; jb = oj; rcB = orc; nrmB = onr; }
        }
    }
    // contact while the distance is below the manifold's breaking threshold (btCollisionDispatcher::getNewManifold, relative
    // threshold: getAngularMotionDisc() * 0.02 of the toe link's shape = 0.81 mm; model_tables.contact_breaking_distance)
    const float brk = P.cfg.contact_breaking;
    const bool active = best <= brk;
    const bool activeU = bestU <= brk;
    const bool activeB = (leg == 0) && (bestB <= brk);
    // joint limits (btMultiBodyJointLimitConstraint: a row only while the limit is violated).  One violated limit in the leg
    // rides in the fast solver path (limJ / limSg / limPen); two or three go to the generic path, one row per joint.
    int limJ = -1; float limSg = 0.f, limPen = 0.f; int nviolL = 0;
    float limSgJ[3], limPenJ[3];
    {
#pragma unroll
        for (int j = 2; j >= 0; j--) {
            const float lo = LB[16 * j + 7], hi = LB[16 * j + 14];
            limSgJ[j] = 0.f; limPenJ[j] = 0.f;
            if (hi - L.q[j] <= 0.f) { limJ = j; limSg = -1.f; limPen = hi - L.q[j]; nviolL++; limSgJ[j] = -1.f; limPenJ[j] = limPen; }
            if (L.q[j] - lo <= 0.f) { limJ = j; limSg = 1.f; limPen = L.q[j] - lo; nviolL++; limSgJ[j] = 1.f; limPenJ[j] = limPen; }
        }
    }
    L.contact = (active ? 1 : 0) | (activeU ? 2 : 0) | (activeB ? 4 : 0);
    // arm joint limits (lane 0): bit j set when joint j is outside [lower, upper]; sign +1 lower / -1 upper
    unsigned armLim = 0u; float armSg[ARM_NJ], armPen[ARM_NJ];
    if (ARM) {
#pragma unroll
        for (int j = 0; j < ARM_NJ; j++) { armSg[j] = 0.f; armPen[j] = 0.f; }
        if (leg == 0) {
#pragma unroll
            for (int j = 0; j < ARM_NJ; j++) {
                const float lo = sm[REXSIM_MT_ARM + ARM_STRIDE * j + 25], hi = sm[REXSIM_MT_ARM + ARM_STRIDE * j + 26];
                if (AR.q[j] - lo <= 0.f) { armLim |= 1u << j; armSg[j] = 1.f; armPen[j] = AR.q[j] - lo; }
                else if (hi - AR.q[j] <= 0.f) { armLim |= 1u << j; armSg[j] = -1.f; armPen[j] = hi - AR.q[j]; }
            }
        }
    }
    // bit 0: a foot contact; bit 1: rows only the generic path solves (body contacts, two violated limits in one leg, more than
    // ARM_KA arm limits); bit 2: arm joint limits, bit 3: a leg joint limit -- both ride along in the fast path
    const int nArmLim = ARM ? __popc(armLim) : 0;
    const unsigned envf = or4((active ? 1u : 0u) | ((activeU || activeB || nviolL > 1 || nArmLim > ARM_KA) ? 2u : 0u) |
                              (nArmLim ? 4u : 0u) | (limJ >= 0 ? 8u : 0u));
    float dqA[ARM_NJ];
    if (ARM) {
#pragma unroll
        for (int j = 0; j < ARM_NJ; j++) dqA[j] = 0.f;
    }
    float dq1 = 0.f, dq2 = 0.f, dq3 = 0.f; SV dv0; dv0.a = mk(0, 0, 0); dv0.l = mk(0, 0, 0);
    const float mu = P.cfg.friction, thr = P.cfg.residual_threshold;
    const int iters = P.cfg.solver_iterations;
    // ================= fast path: foot contacts (+ one joint-limit row per leg, + up to ARM_KA arm limit rows) ===========
    // Compiled twice: LIM = false is the lean form every walking / galloping sub-step takes (12 rows); LIM = true adds the
    // leg's joint-limit row as a fourth row of each lane (standing up from the folded rest pose: every such sub-step).
    auto fast_path = [&](auto lim_tag) {
        constexpr bool LIM = decltype(lim_tag)::value;
        constexpr int CL = 12;                                  // first leg-limit column
        constexpr int CA = 12 + (LIM ? 4 : 0);                  // first arm-limit column
        constexpr int NC = CA + (ARM ? ARM_KA : 0);
        constexpr int NR = LIM ? 4 : 3;                         // own rows: n, t1, t2 (, limit)
        // ---- constraint rows of the own contact: n, t1, t2 ----------------------------------------------
        V3 t1, t2;
        if (TERRAIN == REXSIM_TERRAIN_PLANE) { t1 = mk(0.f, -1.f, 0.f); t2 = mk(1.f, 0.f, 0.f); }
        else plane_space(nrm, t1, t2);
        SV F[3];
        F[0].a = cross(rc, nrm); F[0].l = nrm;
        F[1].a = cross(rc, t1); F[1].l = t1;
        F[2].a = cross(rc, t2); F[2].l = t2;
        SV v3s = sfma(qs3, S3v, sfma(qs2, S2, sfma(qs1, S1, vs)));   // foot spatial velocity after the free update
        float relv[3] = {sdot(F[0], v3s), sdot(F[1], v3s), sdot(F[2], v3s)};
        // unit impulse responses of the own rows: inward along the leg gives the base bias g_d, then the base solve
        float uD1[NR], uD2[NR], uD3[NR]; SV g[NR], dvb[NR];
        float Dd[3][3];                // own-leg response with the base held fixed: Dd[r][d] = F_r . w_d
        float eeF[LIM ? 3 : 1];        // joint-rate response of the LIMITED joint to each foot row (fixed base): the limit row's own terms
#pragma unroll
        for (int d = 0; d < 3; d++) {
            SV pD; pD.a = mk(-F[d].a.x, -F[d].a.y, -F[d].a.z); pD.l = mk(-F[d].l.x, -F[d].l.y, -F[d].l.z);
            uD3[d] = -sdot(S3v, pD); pD = sfma(uD3[d] * k3, U3, pD);
            uD2[d] = -sdot(S2, pD); pD = sfma(uD2[d] * k2, U2, pD);
            uD1[d] = -sdot(S1, pD); pD = sfma(uD1[d] * k1, U1, pD);
            g[d] = pD;
            dvb[d] = neg_mul(Minv, pD);
            const float e1 = uD1[d] * k1;
            SV w = e1 * S1;
            const float e2 = (uD2[d] - sdot(U2, w)) * k2; w = sfma(e2, S2, w);
            const float e3 = (uD3[d] - sdot(U3, w)) * k3; w = sfma(e3, S3v, w);
            Dd[0][d] = sdot(F[0], w); Dd[1][d] = sdot(F[1], w); Dd[2][d] = sdot(F[2], w);
            if (LIM) eeF[d] = limJ == 0 ? e1 : (limJ == 1 ? e2 : e3);
        }
        // the own joint-limit row (btMultiBodyJointLimitConstraint): unit generalized force limSg on joint limJ
        float denL = 1.f, rhsL = 0.f, ownLL = 0.f;
        const bool hasL = LIM && limJ >= 0;
        if (LIM) {
            const float j0 = limJ == 0 ? limSg : 0.f, j1 = limJ == 1 ? limSg : 0.f, j2 = limJ == 2 ? limSg : 0.f;
            const float u3 = j2; SV pD = (u3 * k3) * U3;
            const float u2 = j1 - sdot(S2, pD); pD = sfma(u2 * k2, U2, pD);
            const float u1 = j0 - sdot(S1, pD); pD = sfma(u1 * k1, U1, pD);
            uD1[3] = u1; uD2[3] = u2; uD3[3] = u3;
            g[3] = pD; dvb[3] = neg_mul(Minv, pD);
            const float e1 = u1 * k1; SV w = e1 * S1;
            const float e2 = (u2 - sdot(U2, w)) * k2; w = sfma(e2, S2, w);
            const float e3 = (u3 - sdot(U3, w)) * k3;
            ownLL = j0 * e1 + j1 * e2 + j2 * e3;
            denL = hasL ? ownLL - sdot(g[3], dvb[3]) : 1.f;
            const float relL = j0 * qs1 + j1 * qs2 + j2 * qs3;
            // m_splitImpulse: beyond the -0.04 threshold the positional term goes to m_rhsPenetration, which is never applied
            rhsL = hasL ? ((limPen > -0.04f) ? (-limPen * P.cfg.erp_joint * inv_dt - relL) : -relL) / denL : 0.f;
        }
        // ARM builds: up to ARM_KA violated arm joint limits ride along as extra rows owned by lane 0 (slot a = a-th violated
        // joint, ascending); the rest pose of the arm keeps three of them active all the time (rexsim_arm.cuh)
        float A[NR][NC];
        float Aarm[ARM ? ARM_KA : 1][NC];          // rows of the arm slots (meaningful on lane 0, zero elsewhere)
        SV gA[ARM ? ARM_KA : 1];
        if (ARM) {
#pragma unroll
            for (int a = 0; a < ARM_KA; a++) { gA[a].a = mk(0.f, 0.f, 0.f); gA[a].l = mk(0.f, 0.f, 0.f); }
        }
        float rhsA[ARM ? ARM_KA : 1], denA[ARM ? ARM_KA : 1], dinvA[ARM ? ARM_KA : 1], sgA[ARM ? ARM_KA : 1];
        float uuA[ARM ? ARM_KA : 1][ARM_NJ];       // inward joint terms of each slot (lane 0; applied at the end)
        SV bbA[ARM ? ARM_KA : 1];
        bool actA[ARM ? ARM_KA : 1];
        if (ARM) {
            float eeA[ARM_KA][ARM_NJ]; int jA[ARM_KA];
            unsigned rem = armLim;
#pragma unroll
            for (int a = 0; a < ARM_KA; a++) {
                actA[a] = rem != 0u;
                const int j = actA[a] ? __ffs(rem) - 1 : 0;
                rem &= rem - 1u;
                jA[a] = j; sgA[a] = 0.f; rhsA[a] = 0.f; denA[a] = 1.f; dinvA[a] = 0.f;
                bbA[a].a = mk(0.f, 0.f, 0.f); bbA[a].l = mk(0.f, 0.f, 0.f);
#pragma unroll
                for (int cc = 0; cc < ARM_NJ; cc++) { eeA[a][cc] = 0.f; uuA[a][cc] = 0.f; }
                if (actA[a]) {               // lane 0 only (armLim is zero on the other lanes)
                    const float sg = armSg[j];
                    arm_row(AR, j, sg, gA[a], eeA[a], uuA[a]);
                    bbA[a] = neg_mul(Minv, gA[a]);
                    sgA[a] = sg;
                    denA[a] = -sdot(gA[a], bbA[a]) + sg * eeA[a][j];
                    dinvA[a] = 1.0f / denA[a];
                    const float relvA = sg * AR.qs[j];
                    rhsA[a] = (armPen[j] > -0.04f) ? (-armPen[j] * P.cfg.erp_joint * inv_dt - relvA) * dinvA[a] : -relvA * dinvA[a];
                }
            }
            // arm x arm block: velocity of slot a's joint per unit impulse of slot c = sg_a * ee_c[j_a] - g_a . b_c
#pragma unroll
            for (int a = 0; a < ARM_KA; a++)
#pragma unroll
                for (int cc = 0; cc < ARM_KA; cc++)
                    Aarm[a][CA + cc] = (actA[a] && actA[cc]) ? sgA[a] * eeA[cc][jA[a]] - sdot(gA[a], bbA[cc]) : 0.f;
            // every lane needs the arm slots' base responses for its own rows' arm columns, and the slots' status
#pragma unroll
            for (int a = 0; a < ARM_KA; a++) {
                bbA[a] = bcast4(bbA[a], 0);
                actA[a] = __shfl_sync(env_mask(), actA[a] ? 1 : 0, 0, 4) != 0;
                denA[a] = bcast4(denA[a], 0);
#pragma unroll
                for (int r = 0; r < NR; r++) A[r][CA + a] = -sdot(g[r], bbA[a]);
            }
        }
        // Delassus rows A[r][c] = J_r M^-1 J_c^T.  The response of the own foot to a base velocity change b is T b with
        // T = prod(I - S_i k_i U_i^T), and T^T F_r = -g_r is already known from the inward pass, so a foreign column costs one
        // 6-dot; own columns add the fixed-base term (Dd between foot rows; the limited joint's rate eeF between foot and limit row).
#pragma unroll
        for (int s = 0; s < 4; s++) {
            const bool own = (s == leg);
#pragma unroll
            for (int d = 0; d < 3; d++) {
                SV b = bcast4(dvb[d], s);
#pragma unroll
                for (int r = 0; r < 3; r++) A[r][3 * s + d] = (own ? Dd[r][d] : 0.f) - sdot(g[r], b);
                if (LIM) A[3][3 * s + d] = (own ? limSg * eeF[d] : 0.f) - sdot(g[3], b);
                if (ARM) {
#pragma unroll
                    for (int a = 0; a < ARM_KA; a++) Aarm[a][3 * s + d] = -sdot(gA[a], b);
                }
            }
            if (LIM) {
                SV b = bcast4(dvb[3], s);           // zero response when lane s has no violated limit
                const bool sl = __shfl_sync(env_mask(), hasL ? 1 : 0, s, 4) != 0;
#pragma unroll
                for (int r = 0; r < 3; r++) A[r][CL + s] = sl ? (own ? limSg * eeF[r] : 0.f) - sdot(g[r], b) : 0.f;
                A[3][CL + s] = sl ? (own ? ownLL : 0.f) - sdot(g[3], b) : 0.f;
                if (ARM) {
#pragma unroll
                    for (int a = 0; a < ARM_KA; a++) Aarm[a][CL + s] = sl ? -sdot(gA[a], b) : 0.f;
                }
            }
        }
        // right-hand sides (btMultiBodyConstraintSolver::setupMultiBodyContactConstraint)
        float den[NR], dinv[NR], rhs[NR];
#pragma unroll
        for (int d = 0; d < 3; d++) { den[d] = Dd[d][d] - sdot(g[d], dvb[d]); dinv[d] = 1.0f / den[d]; }
        {
            const float slop = 1e-5f;
            float pen = best + slop;
            float poserr = 0.f, velerr = -relv[0];
            if (pen > 0.f) velerr -= pen * inv_dt; else poserr = -pen * P.cfg.erp_contact * inv_dt;
            rhs[0] = (pen > -0.04f) ? (poserr + velerr) * dinv[0] : velerr * dinv[0];
            rhs[1] = -relv[1] * dinv[1];
            rhs[2] = -relv[2] * dinv[2];
        }
        if (LIM) { den[3] = denL; dinv[3] = 1.0f / denL; rhs[3] = rhsL; }
        // ---- PGS in impulse space, Bullet row order: joint-limit rows (legs, arm), normals 0..3, then (t1,t2) of contacts 0..3 ----
        // Each lane keeps only its own impulses and the PRE-SCALED running row sums t[d] = rhs[d] - dinv[d] * sum_j A[d][j] lambda_j:
        // t[d] IS the next impulse change of row d, so the serial chain per row is clamp -> shuffle -> one FMA.  The owner of a
        // row broadcasts its impulse CHANGE and every lane folds it into its sums.  Every lane sees every change, so with the row
        // denominators replicated once per sub-step each lane evaluates the iteration's residual itself: no reduction (two
        // dependent shuffles) at the end of every iteration.  Same max, same early-out decision on all lanes of the env.
        float lam[NR];
        float t[NR];
#pragma unroll
        for (int r = 0; r < NR; r++) {
            lam[r] = 0.f; t[r] = rhs[r];
#pragma unroll
            for (int cc = 0; cc < NC; cc++) A[r][cc] *= -dinv[r];
        }
        bool running = true;             // env-uniform: the 4 lanes of an env leave the loop together
        const bool mine = active;
        float tA[ARM ? ARM_KA : 1], lamA[ARM ? ARM_KA : 1];
        if (ARM) {
#pragma unroll
            for (int a = 0; a < ARM_KA; a++) {
                tA[a] = rhsA[a]; lamA[a] = 0.f;
#pragma unroll
                for (int cc = 0; cc < NC; cc++) Aarm[a][cc] *= -dinvA[a];
            }
        }
        if constexpr (REPL && !LIM && !ARM) {
            // ---- replicated form: every lane of the env sweeps all 12 rows itself ------------------------------------
            // A single warp per scheduler cannot hide the shuffle that hands each impulse change to the next row's owner, and
            // that shuffle sits on the serial chain 8 times per iteration.  So exchange once per sub-step, through shared memory
            // (a shuffle in this env-divergent branch is a collective of ~10 instructions): lane s publishes rows 3s..3s+2 (matrix
            // row, running sum, denominator), every lane loads all 12 into registers, and each row then sees exactly the fmaf
            // sequence lane s performs in the shuffle form below -- bit-identical impulses.  The normal row of a contact that does
            // not touch is published as zeros (matrix row and sum), so its change is fmaxf(0, -0) = 0 with no select, and
            // lam[n] > 0 alone gates its friction.
            // The normal clamp (lam + dI < 0 ? -lam : dI) is fmaxf(dI, -lam): a rounded sum has the sign of the exact sum, so
            // the two differ at most in the sign of a zero change, which leaves lam and the residual unchanged.
            constexpr int NF = 12;
            __syncwarp(env_mask());                     // the env's lanes are done reading the previous sub-step's rows
#pragma unroll
            for (int d = 0; d < 3; d++) {
                const bool keep = mine || d > 0;
                float4* row = reinterpret_cast<float4*>(pgs + (3 * leg + d) * NF);
#pragma unroll
                for (int q = 0; q < NF / 4; q++)
                    row[q] = keep ? make_float4(A[d][4 * q], A[d][4 * q + 1], A[d][4 * q + 2], A[d][4 * q + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
                pgs[NF * NF + 3 * leg + d] = keep ? t[d] : 0.f;
                pgs[NF * NF + NF + 3 * leg + d] = den[d];
            }
            __syncwarp(env_mask());
            float Af[NF][NF], T[NF], lamF[NF], denF[NF];
            const float4* E = reinterpret_cast<const float4*>(pgs);
#pragma unroll
            for (int j = 0; j < NF; j++) {
#pragma unroll
                for (int q = 0; q < NF / 4; q++) {
                    const float4 v = E[j * (NF / 4) + q];
                    Af[j][4 * q] = v.x; Af[j][4 * q + 1] = v.y; Af[j][4 * q + 2] = v.z; Af[j][4 * q + 3] = v.w;
                }
            }
#pragma unroll
            for (int q = 0; q < NF / 4; q++) {
                const float4 v = E[NF * NF / 4 + q], w = E[NF * NF / 4 + NF / 4 + q];
                T[4 * q] = v.x; T[4 * q + 1] = v.y; T[4 * q + 2] = v.z; T[4 * q + 3] = v.w;
                denF[4 * q] = w.x; denF[4 * q + 1] = w.y; denF[4 * q + 2] = w.z; denF[4 * q + 3] = w.w;
            }
#pragma unroll
            for (int j = 0; j < NF; j++) lamF[j] = 0.f;
            for (int it = 0; it < iters && running; it++) {
                L.cost++;
                float resid = 0.f;
#pragma unroll
                for (int s = 0; s < 4; s++) {
                    const int n = 3 * s;
                    const float dI = fmaxf(T[n], -lamF[n]);
                    lamF[n] += dI;
                    const float rr = dI * denF[n]; resid = fmaxf(resid, rr * rr);
#pragma unroll
                    for (int j = 0; j < NF; j++) T[j] = fmaf(Af[j][n], dI, T[j]);
                }
#pragma unroll
                for (int s = 0; s < 4; s++) {
                    // the clamp bounds and the zero of a frozen pair are known before the row's sum: the chain is add, compare, 2 selects
                    const int n = 3 * s, f1 = n + 1, f2 = n + 2;
                    const float lim = mu * lamF[n];
                    const bool upd = lamF[n] > 0.f;
                    const float lo1 = upd ? -lim - lamF[f1] : 0.f, hi1 = upd ? lim - lamF[f1] : 0.f;
                    const float sum1 = lamF[f1] + T[f1];
                    const float dI1 = sum1 < -lim ? lo1 : (sum1 > lim ? hi1 : (upd ? T[f1] : 0.f));
                    lamF[f1] += dI1;
                    const float t2 = fmaf(Af[f2][f1], dI1, T[f2]);
                    const float lo2 = upd ? -lim - lamF[f2] : 0.f, hi2 = upd ? lim - lamF[f2] : 0.f;
                    const float sum2 = lamF[f2] + t2;
                    const float dI2 = sum2 < -lim ? lo2 : (sum2 > lim ? hi2 : (upd ? t2 : 0.f));
                    lamF[f2] += dI2;
                    const float r1 = dI1 * denF[f1], r2 = dI2 * denF[f2];
                    resid = fmaxf(resid, fmaxf(r1 * r1, r2 * r2));
#pragma unroll
                    for (int j = 0; j < NF; j++) T[j] = fmaf(Af[j][f2], dI2, fmaf(Af[j][f1], dI1, T[j]));
                }
                if (resid <= thr) running = false;
            }
#pragma unroll
            for (int d = 0; d < 3; d++)
                lam[d] = leg == 0 ? lamF[d] : (leg == 1 ? lamF[3 + d] : (leg == 2 ? lamF[6 + d] : lamF[9 + d]));
        } else {
            float denAll[4][NR];
#pragma unroll
            for (int s = 0; s < 4; s++)
#pragma unroll
                for (int d = 0; d < NR; d++) denAll[s][d] = bcast4(den[d], s);
            for (int it = 0; it < iters && running; it++) {
                L.cost++;
                float resid = 0.f;
                // joint-limit rows first, in joint order (4 legs, then the arm), the direction alternating per iteration
                // (btMultiBodyConstraintSolver::solveSingleIteration): even iterations descending, odd ascending
                auto arm_round = [&](const int a) {
                    float dI = tA[a];
                    if (lamA[a] + dI < 0.f) dI = -lamA[a];
                    dI = (actA[a] && leg == 0) ? dI : 0.f;
                    lamA[a] += dI;
                    const float dl = bcast4(dI, 0);
                    const float rr = dl * denA[a]; resid = fmaxf(resid, rr * rr);
#pragma unroll
                    for (int r = 0; r < NR; r++) t[r] = fmaf(A[r][CA + a], dl, t[r]);
#pragma unroll
                    for (int c2 = 0; c2 < ARM_KA; c2++) tA[c2] = fmaf(Aarm[c2][CA + a], dl, tA[c2]);
                };
                auto leg_round = [&](const int s) {
                    float dI = t[NR - 1];
                    if (lam[NR - 1] + dI < 0.f) dI = -lam[NR - 1];
                    dI = (hasL && leg == s) ? dI : 0.f;
                    lam[NR - 1] += dI;
                    const float dl = bcast4(dI, s);
                    const float rr = dl * denAll[s][NR - 1]; resid = fmaxf(resid, rr * rr);
#pragma unroll
                    for (int r = 0; r < NR; r++) t[r] = fmaf(A[r][CL + s], dl, t[r]);
                    if (ARM) {
#pragma unroll
                        for (int a = 0; a < ARM_KA; a++) tA[a] = fmaf(Aarm[a][CL + s], dl, tA[a]);
                    }
                };
                if (it & 1) {
                    if (LIM) { leg_round(0); leg_round(1); leg_round(2); leg_round(3); }
                    if (ARM) { arm_round(0); arm_round(1); arm_round(2); }
                } else {
                    if (ARM) { arm_round(2); arm_round(1); arm_round(0); }
                    if (LIM) { leg_round(3); leg_round(2); leg_round(1); leg_round(0); }
                }
#pragma unroll
                for (int s = 0; s < 4; s++) {
                    float dI = t[0];
                    if (lam[0] + dI < 0.f) dI = -lam[0];
                    const bool upd = mine && (leg == s);
                    dI = upd ? dI : 0.f;
                    lam[0] += dI;
                    const float dl = bcast4(dI, s);
                    const float rr = dl * denAll[s][0]; resid = fmaxf(resid, rr * rr);
#pragma unroll
                    for (int r = 0; r < NR; r++) t[r] = fmaf(A[r][3 * s], dl, t[r]);
                    if (ARM) {
#pragma unroll
                        for (int a = 0; a < ARM_KA; a++) tA[a] = fmaf(Aarm[a][3 * s], dl, tA[a]);
                    }
                }
#pragma unroll
                for (int s = 0; s < 4; s++) {
                    // both friction rows of contact s belong to lane s: update t1, fold its change into the own t2 sum
                    // locally, update t2, then broadcast the two changes together (one communication round per contact)
                    const float lim = mu * lam[0];
                    const bool upd = mine && (leg == s) && (lam[0] > 0.f);
                    float dI1 = t[1];
                    const float sum1 = lam[1] + dI1;
                    if (sum1 < -lim) dI1 = -lim - lam[1]; else if (sum1 > lim) dI1 = lim - lam[1];
                    dI1 = upd ? dI1 : 0.f;
                    lam[1] += dI1;
                    float dI2 = fmaf(A[2][3 * s + 1], dI1, t[2]);            // own lane: column 3*leg+1 == 3*s+1 when upd
                    const float sum2 = lam[2] + dI2;
                    if (sum2 < -lim) dI2 = -lim - lam[2]; else if (sum2 > lim) dI2 = lim - lam[2];
                    dI2 = upd ? dI2 : 0.f;
                    lam[2] += dI2;
                    const float dl1 = bcast4(dI1, s), dl2 = bcast4(dI2, s);
                    const float r1 = dl1 * denAll[s][1], r2 = dl2 * denAll[s][2];
                    resid = fmaxf(resid, fmaxf(r1 * r1, r2 * r2));
#pragma unroll
                    for (int r = 0; r < NR; r++) t[r] = fmaf(A[r][3 * s + 2], dl2, fmaf(A[r][3 * s + 1], dl1, t[r]));
                    if (ARM) {
#pragma unroll
                        for (int a = 0; a < ARM_KA; a++) tA[a] = fmaf(Aarm[a][3 * s + 2], dl2, fmaf(Aarm[a][3 * s + 1], dl1, tA[a]));
                    }
                }
                if (resid <= thr) running = false;
            }
        }
        // ---- apply the net impulse: one more response pass ---------------------------------------------------
        float e1 = 0.f, e2 = 0.f, e3 = 0.f;
        SV own_b; own_b.a = mk(0.f, 0.f, 0.f); own_b.l = mk(0.f, 0.f, 0.f);
#pragma unroll
        for (int r = 0; r < NR; r++) {
            e1 = fmaf(lam[r], uD1[r], e1); e2 = fmaf(lam[r], uD2[r], e2); e3 = fmaf(lam[r], uD3[r], e3);
            own_b = sfma(lam[r], dvb[r], own_b);
        }
        float usA[ARM_NJ];
        if (ARM) {
#pragma unroll
            for (int cc = 0; cc < ARM_NJ; cc++) usA[cc] = 0.f;
            if (leg == 0) {
#pragma unroll
                for (int a = 0; a < ARM_KA; a++) {
                    own_b = sfma(lamA[a], bbA[a], own_b);          // lamA is zero for inactive slots
#pragma unroll
                    for (int cc = 0; cc < ARM_NJ; cc++) usA[cc] = fmaf(lamA[a], uuA[a][cc], usA[cc]);
                }
            }
        }
        dv0 = sum4(own_b);
        SV b = dv0;
        dq1 = (e1 - sdot(U1, b)) * k1; b = sfma(dq1, S1, b);
        dq2 = (e2 - sdot(U2, b)) * k2; b = sfma(dq2, S2, b);
        dq3 = (e3 - sdot(U3, b)) * k3;
        if (ARM && leg == 0) arm_apply(AR, dv0, usA, dqA);
    };
    if (envf != 0u && !(envf & 2u)) {
        if (envf & 8u) fast_path(std::true_type{});
        else fast_path(std::false_type{});
    }
    else if (envf & 2u) {
        L.cost += 64;      // the generic path is several times the fast path: such envs sort together (rexsim_rebalance)
        // ================= generic path: body contacts and/or a joint limit ====================================
        // M^-1 of a star-shaped tree = per-leg block + a rank-6 coupling through the base, so no Delassus matrix is
        // needed: a row's velocity is  J_r dV = -g_r . beta + Jq_r . eps  with beta = base velocity change (replicated
        // on the 4 lanes) and eps = own-leg joint-rate change at fixed base.  Rows live in local memory (rare path).
        // rows: 0..2 = joint limits of the own joints | 3..5 base contact (lane 0) | 6..8 upper contact | 9..11 foot contact  (n, t1, t2)
        constexpr int NR = 12;
        float g_[NR][6], b_[NR][6], Jq_[NR][3], ee_[NR][3], uu_[NR][3], rhs_[NR], dinv_[NR], den_[NR], lam_[NR];
#pragma unroll 1
        for (int r = 0; r < NR; r++) {
#pragma unroll
            for (int c = 0; c < 6; c++) { g_[r][c] = 0.f; b_[r][c] = 0.f; }
#pragma unroll
            for (int c = 0; c < 3; c++) { Jq_[r][c] = 0.f; ee_[r][c] = 0.f; uu_[r][c] = 0.f; }
            rhs_[r] = 0.f; dinv_[r] = 0.f; den_[r] = 0.f; lam_[r] = 0.f;
        }
        unsigned actbits = 0u;
        auto setup_row = [&](int ri, SV Jb, float j0, float j1, float j2) -> float {
            float relv = sdot(Jb, vs) + j0 * qs1 + j1 * qs2 + j2 * qs3;
            float u3 = j2; SV pD = (u3 * k3) * U3;
            float u2 = j1 - sdot(S2, pD); pD = sfma(u2 * k2, U2, pD);
            float u1 = j0 - sdot(S1, pD); pD = sfma(u1 * k1, U1, pD);
            SV gg = pD - Jb; SV bb = neg_mul(Minv, gg);
            float e1 = u1 * k1; SV w = e1 * S1;
            float e2 = (u2 - sdot(U2, w)) * k2; w = sfma(e2, S2, w);
            float e3 = (u3 - sdot(U3, w)) * k3;
            float dn = -sdot(gg, bb) + j0 * e1 + j1 * e2 + j2 * e3;
            g_[ri][0] = gg.a.x; g_[ri][1] = gg.a.y; g_[ri][2] = gg.a.z; g_[ri][3] = gg.l.x; g_[ri][4] = gg.l.y; g_[ri][5] = gg.l.z;
            b_[ri][0] = bb.a.x; b_[ri][1] = bb.a.y; b_[ri][2] = bb.a.z; b_[ri][3] = bb.l.x; b_[ri][4] = bb.l.y; b_[ri][5] = bb.l.z;
            Jq_[ri][0] = j0; Jq_[ri][1] = j1; Jq_[ri][2] = j2;
            ee_[ri][0] = e1; ee_[ri][1] = e2; ee_[ri][2] = e3;
            uu_[ri][0] = u1; uu_[ri][1] = u2; uu_[ri][2] = u3;
            den_[ri] = dn; dinv_[ri] = 1.0f / dn;
            actbits |= 1u << ri;
            return relv;
        };
        auto setup_contact = [&](int r0, V3 r, V3 n, int kb, float dist) {
            V3 t1, t2;
            if (TERRAIN == REXSIM_TERRAIN_PLANE) { t1 = mk(0.f, -1.f, 0.f); t2 = mk(1.f, 0.f, 0.f); }
            else plane_space(n, t1, t2);
#pragma unroll 1
            for (int d = 0; d < 3; d++) {
                V3 dir = d == 0 ? n : (d == 1 ? t1 : t2);
                SV F; F.a = cross(r, dir); F.l = dir;
                float j0 = kb >= 1 ? sdot(S1, F) : 0.f, j1 = kb >= 2 ? sdot(S2, F) : 0.f, j2 = kb >= 3 ? sdot(S3v, F) : 0.f;
                float relv = setup_row(r0 + d, F, j0, j1, j2);
                if (d == 0) {
                    float pen = dist + 1e-5f;
                    float poserr = 0.f, velerr = -relv;
                    if (pen > 0.f) velerr -= pen * inv_dt; else poserr = -pen * P.cfg.erp_contact * inv_dt;
                    rhs_[r0] = (pen > -0.04f) ? (poserr + velerr) * dinv_[r0] : velerr * dinv_[r0];
                } else rhs_[r0 + d] = -relv * dinv_[r0 + d];
            }
        };
#pragma unroll 1
        for (int j = 0; j < 3; j++) {
            const float sg = j == 0 ? limSgJ[0] : (j == 1 ? limSgJ[1] : limSgJ[2]);
            if (sg == 0.f) continue;
            const float pen = j == 0 ? limPenJ[0] : (j == 1 ? limPenJ[1] : limPenJ[2]);
            SV z; z.a = mk(0, 0, 0); z.l = mk(0, 0, 0);
            float relv = setup_row(j, z, j == 0 ? sg : 0.f, j == 1 ? sg : 0.f, j == 2 ? sg : 0.f);
            // btMultiBodyJointLimitConstraint with m_splitImpulse: beyond the -0.04 threshold the positional term goes to
            // m_rhsPenetration, which the multibody solver never applies (the row only stops further motion)
            rhs_[j] = (pen > -0.04f) ? (-pen * P.cfg.erp_joint * inv_dt - relv) * dinv_[j] : -relv * dinv_[j];
        }
        if (activeB) setup_contact(3, rcB, nrmB, 0, bestB);
        if (activeU) setup_contact(6, rcU, nrmU, kU, bestU);
        if (active) setup_contact(9, rc, nrm, 3, best);
        // arm joint-limit rows (lane 0)
        float gA_[ARM ? ARM_NJ : 1][6], bA_[ARM ? ARM_NJ : 1][6], eeA_[ARM ? ARM_NJ : 1][ARM_NJ], uuA_[ARM ? ARM_NJ : 1][ARM_NJ];
        float rhsA_[ARM_NJ], dinvA_[ARM_NJ], denA_[ARM_NJ], lamA_[ARM_NJ], epsA[ARM_NJ], usA[ARM_NJ];
        if (ARM) {
#pragma unroll 1
            for (int j = 0; j < ARM_NJ; j++) {
                rhsA_[j] = 0.f; dinvA_[j] = 0.f; denA_[j] = 0.f; lamA_[j] = 0.f; epsA[j] = 0.f; usA[j] = 0.f;
#pragma unroll
                for (int c = 0; c < 6; c++) { gA_[j][c] = 0.f; bA_[j][c] = 0.f; eeA_[j][c] = 0.f; uuA_[j][c] = 0.f; }
                if (!((armLim >> j) & 1u)) continue;
                SV gg; arm_row(AR, j, armSg[j], gg, eeA_[j], uuA_[j]);
                SV bb = neg_mul(Minv, gg);
                st6(gA_[j], gg); st6(bA_[j], bb);
                float dn = -sdot(gg, bb) + armSg[j] * eeA_[j][j];
                denA_[j] = dn; dinvA_[j] = 1.0f / dn;
                float relv = armSg[j] * AR.qs[j];
                rhsA_[j] = (armPen[j] > -0.04f) ? (-armPen[j] * P.cfg.erp_joint * inv_dt - relv) * dinvA_[j] : -relv * dinvA_[j];
            }
        }
        SV beta; beta.a = mk(0, 0, 0); beta.l = mk(0, 0, 0);
        float eps0 = 0.f, eps1 = 0.f, eps2 = 0.f, us0 = 0.f, us1 = 0.f, us2 = 0.f;
        // compact the Gauss-Seidel sequence to the rows that exist in this env (env-uniform: built from shuffled bits)
        constexpr int NLIM = ARM ? 12 + ARM_NJ : 12;     // limit rows in joint order: 3 per leg (lane), then the arm
        unsigned char llist[NLIM], clist[27];
        int nl = 0, nc = 0;
        {
            unsigned actAll[4];
#pragma unroll
            for (int o = 0; o < 4; o++) actAll[o] = __shfl_sync(env_mask(), actbits, o, 4);
            const unsigned armAll = ARM ? __shfl_sync(env_mask(), armLim, 0, 4) : 0u;
#pragma unroll
            for (int idx = 0; idx < NLIM; idx++) {
                const bool a = idx < 12 ? ((actAll[idx < 12 ? idx / 3 : 0] >> (idx % 3)) & 1u) : ((armAll >> (idx - 12)) & 1u);
                if (a) llist[nl++] = (unsigned char)idx;
            }
#pragma unroll 1
            for (int t = 0; t < 27; t++) {
                const int o = c_seq_owner[t], ri = c_seq_row[t];
                const unsigned a = o == 0 ? actAll[0] : (o == 1 ? actAll[1] : (o == 2 ? actAll[2] : actAll[3]));
                if ((a >> ri) & 1u) clist[nc++] = (unsigned char)t;
            }
        }
        bool running = true;
        for (int it = 0; it < iters && running; it++) {
            L.cost++;
            float resid = 0.f;
#pragma unroll 1
            for (int tt = 0; tt < nl + nc; tt++) {
                int o, ri;
                if (tt < nl) {                                      // limit rows: direction alternates per iteration
                    const int idx = llist[(it & 1) ? tt : nl - 1 - tt];
                    if (ARM && idx >= 12) {                         // an arm joint-limit row, owned by lane 0
                        const int j = idx - 12;
                        float rsumA = armSg[j] * epsA[j] - (gA_[j][0] * beta.a.x + gA_[j][1] * beta.a.y + gA_[j][2] * beta.a.z + gA_[j][3] * beta.l.x + gA_[j][4] * beta.l.y + gA_[j][5] * beta.l.z);
                        float dIA = rhsA_[j] - rsumA * dinvA_[j];
                        if (lamA_[j] + dIA < 0.f) dIA = -lamA_[j];
                        dIA = (((armLim >> j) & 1u) && leg == 0) ? dIA : 0.f;
                        lamA_[j] += dIA;
                        float rrA = dIA * denA_[j]; resid = fmaxf(resid, rrA * rrA);
#pragma unroll
                        for (int c = 0; c < ARM_NJ; c++) { epsA[c] = fmaf(dIA, eeA_[j][c], epsA[c]); usA[c] = fmaf(dIA, uuA_[j][c], usA[c]); }
                        SV dBA; dBA.a = mk(dIA * bA_[j][0], dIA * bA_[j][1], dIA * bA_[j][2]); dBA.l = mk(dIA * bA_[j][3], dIA * bA_[j][4], dIA * bA_[j][5]);
                        beta = beta + bcast4(dBA, 0);
                        continue;
                    }
                    o = idx / 3; ri = idx % 3;
                }
                else { const int t = clist[tt - nl]; o = c_seq_owner[t]; ri = c_seq_row[t]; }
                const int ph = (ri < 3) ? 0 : ri % 3;                   // 0: unilateral row (limit / normal), 1/2: friction row
                float rsum = Jq_[ri][0] * eps0 + Jq_[ri][1] * eps1 + Jq_[ri][2] * eps2
                           - (g_[ri][0] * beta.a.x + g_[ri][1] * beta.a.y + g_[ri][2] * beta.a.z + g_[ri][3] * beta.l.x + g_[ri][4] * beta.l.y + g_[ri][5] * beta.l.z);
                float dI = rhs_[ri] - rsum * dinv_[ri];
                const float lr = lam_[ri];
                bool ok = ((actbits >> ri) & 1u) && (leg == o);
                if (ph == 0) { if (lr + dI < 0.f) dI = -lr; }
                else {
                    const float ln = lam_[ri - ph], lim = mu * ln, sum = lr + dI;
                    if (sum < -lim) dI = -lim - lr; else if (sum > lim) dI = lim - lr;
                    ok = ok && (ln > 0.f);
                }
                dI = ok ? dI : 0.f;
                lam_[ri] = lr + dI;
                float rr = dI * den_[ri]; resid = fmaxf(resid, rr * rr);
                eps0 = fmaf(dI, ee_[ri][0], eps0); eps1 = fmaf(dI, ee_[ri][1], eps1); eps2 = fmaf(dI, ee_[ri][2], eps2);
                us0 = fmaf(dI, uu_[ri][0], us0); us1 = fmaf(dI, uu_[ri][1], us1); us2 = fmaf(dI, uu_[ri][2], us2);
                SV dB; dB.a = mk(dI * b_[ri][0], dI * b_[ri][1], dI * b_[ri][2]); dB.l = mk(dI * b_[ri][3], dI * b_[ri][4], dI * b_[ri][5]);
                beta = beta + bcast4(dB, o);
            }
            resid = max4(resid);
            if (resid <= thr) running = false;
        }
        dv0 = beta;
        SV b = dv0;
        dq1 = (us0 - sdot(U1, b)) * k1; b = sfma(dq1, S1, b);
        dq2 = (us1 - sdot(U2, b)) * k2; b = sfma(dq2, S2, b);
        dq3 = (us2 - sdot(U3, b)) * k3;
        if (ARM && leg == 0) arm_apply(AR, dv0, usA, dqA);
    }
    // ---- integrate (btMultiBody::stepPositionsMultiDof) --------------------------------------------------
    L.w = vs.a + dv0.a; L.vl = vs.l + dv0.l;
    L.w = mk(clampv(L.w.x, vmax), clampv(L.w.y, vmax), clampv(L.w.z, vmax));          // processDeltaVeeMultiDof2 -> applyDeltaVee
    L.vl = mk(clampv(L.vl.x, vmax), clampv(L.vl.y, vmax), clampv(L.vl.z, vmax));
    L.qd[0] = clampv(qs1 + dq1, vmax); L.qd[1] = clampv(qs2 + dq2, vmax); L.qd[2] = clampv(qs3 + dq3, vmax);
    L.pos = fma3(dt, L.vl, L.pos);
    L.q[0] = fmaf(dt, L.qd[0], L.q[0]); L.q[1] = fmaf(dt, L.qd[1], L.q[1]); L.q[2] = fmaf(dt, L.qd[2], L.q[2]);
    if (ARM && leg == 0) {
#pragma unroll
        for (int j = 0; j < ARM_NJ; j++) { AR.qd[j] = clampv(AR.qs[j] + dqA[j], vmax); AR.q[j] = fmaf(dt, AR.qd[j], AR.q[j]); }
    }
    {
        float fa = sqrtf(dot(L.w, L.w));
        if (fa * dt > 0.7853981633974483f) fa = 0.5f * 1.5707963267948966f / dt;
        float sc;
        if (fa < 0.001f) sc = 0.5f * dt - dt * dt * dt * 0.020833333333f * fa * fa;
        else sc = sinf(0.5f * fa * dt) / fa;
        float ax = L.w.x * sc, ay = L.w.y * sc, az = L.w.z * sc, aw = cosf(fa * dt * 0.5f);
        float nw = aw * L.qw - ax * L.qx - ay * L.qy - az * L.qz;
        float nx = aw * L.qx + ax * L.qw + ay * L.qz - az * L.qy;
        float ny = aw * L.qy - ax * L.qz + ay * L.qw + az * L.qx;
        float nz = aw * L.qz + ax * L.qy - ay * L.qx + az * L.qw;
        float inv = rsqrtf(nx * nx + ny * ny + nz * nz + nw * nw);
        L.qx = nx * inv; L.qy = ny * inv; L.qz = nz * inv; L.qw = nw * inv;
    }
}

// Rex.ApplyAction + stepSimulation (rex_gym/model/rex.py:158-163,568-641) for the own leg's three motors
static __constant__ float c_arm_rest[6] = {-1.6f, -1.6f, 0.f, 0.f, 1.6f, 0.f};   // ARM_POSES['rest'] rex_constants.py:3-8

template <int TERRAIN, bool ARM, bool SENSOR, bool REPL>
__device__ __forceinline__ void apply_action_and_step(const Params& P, const float* sm, Lane& L, int leg,
                                                      const float* cmd, float kp, float kd, Ground& G, Arm& AR,
                                                      Sensor& S, bool valid, float* pgs) {
    float tau[3];
    float tauA[ARM_NJ];
    const bool pd_delayed = SENSOR && P.lat_pd > 0.f;        // _GetPDObservation (rex.py:755-759): q, qd as they were pd_latency ago
    if (ARM) {
#pragma unroll
        for (int j = 0; j < ARM_NJ; j++) tauA[j] = 0.f;
        if (leg == 0) {
            const uint32_t limitA = (uint32_t)(1.0 / P.cfg.sim_dt_d);
#pragma unroll
            for (int j = 0; j < ARM_NJ; j++) {
                float to;
                float qo = AR.q[j], qdo = AR.qd[j];
                if (pd_delayed) {
                    qo = sensor_delayed(S, P.lat_pd, P.n_pd, P.a_pd, HW_ARM + j);
                    qdo = sensor_delayed(S, P.lat_pd, P.n_pd, P.a_pd, HW_ARM + 6 + j);
                }
                float ta = motor_torque(c_arm_rest[j], qo, qdo, AR.qd[j], kp, kd, to);
                uint32_t w = AR.ovh[j / 3], c = (w >> (10 * (j % 3))) & 1023u;
                c = (fabsf(ta) > 2.45f) ? min(c + 1u, 1023u) : 0u;
                if (c > limitA) AR.enabled &= ~(1u << j);
                AR.ovh[j / 3] = (w & ~(1023u << (10 * (j % 3)))) | (c << (10 * (j % 3)));
                AR.tau_obs[j] = to;
                tauA[j] = ((AR.enabled >> j) & 1u) ? ta : 0.f;
            }
        }
    }
    const uint32_t limit = (uint32_t)(1.0 / P.cfg.sim_dt_d);   // OVERHEAT_SHUTDOWN_TIME / time_step
#pragma unroll
    for (int j = 0; j < 3; j++) {
        float to;
        float qo = L.q[j], qdo = L.qd[j];
        if (pd_delayed) {
            qo = sensor_delayed(S, P.lat_pd, P.n_pd, P.a_pd, 9 * leg + j);
            qdo = sensor_delayed(S, P.lat_pd, P.n_pd, P.a_pd, 9 * leg + 3 + j);
        }
        float ta = motor_torque(cmd[j], qo, qdo, L.qd[j], kp, kd, to);
        uint32_t c = (L.ovh >> (10 * j)) & 1023u;
        c = (fabsf(ta) > 2.45f) ? min(c + 1u, 1023u) : 0u;
        if (c > limit) L.enabled &= ~(1u << j);
        L.ovh = (L.ovh & ~(1023u << (10 * j))) | (c << (10 * j));
        L.tau_obs[j] = to;
        tau[j] = ((L.enabled >> j) & 1u) ? ta : 0.f;
    }
    physics_substep<TERRAIN, ARM, REPL>(P, sm, L, leg, tau, G, AR, tauA, pgs);
    if (SENSOR) sensor_push<ARM>(S, leg, L, AR, valid);         // Rex.ReceiveObservation (rex.py:162,726-733)
}

// -------------------------------------------------------------------------------------------------
// gait planner + IK for the own leg (model/gait_planner.py:31-134, model/kinematics.py:80-142)
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void bezier_sums(float phi, float& SX, float& SZ) {   // sum_k C(11,k) phi^k (1-phi)^(11-k) P_k, k<10
    const float BX[10] = {-0.04f, -0.056f, -0.06f, -0.06f, -0.06f, 0.f, 0.f, 0.f, 0.06f, 0.06f};
    const float BZ[10] = {0.f, 0.f, 0.0405f, 0.0405f, 0.0405f, 0.0405f, 0.0405f, 0.0495f, 0.0495f, 0.0495f};
    const float BIN[10] = {1.f, 11.f, 55.f, 165.f, 330.f, 462.f, 462.f, 330.f, 165.f, 55.f};
    float om = 1.f - phi;
    float pw[12], qw[12];
    pw[0] = 1.f; qw[0] = 1.f;
#pragma unroll
    for (int k = 1; k < 12; k++) { pw[k] = pw[k - 1] * phi; qw[k] = qw[k - 1] * om; }
    SX = 0.f; SZ = 0.f;
#pragma unroll
    for (int k = 0; k < 10; k++) { float b = BIN[k] * pw[k] * qw[11 - k]; SX = fmaf(BX[k], b, SX); SZ = fmaf(BZ[k], b, SZ); }
}
// step contribution (long or rot) given phase data; angle in degrees
__device__ __forceinline__ V3 step_part(bool stance, float phase, float SX, float SZ, float v, float angle_deg, float direction) {
    float s, c; sincosf(angle_deg * (PI_F / 180.0f), &s, &c);
    float av = fabsf(v);
    if (stance) {
        float p = 0.05f * (1.f - 2.f * phase);
        return mk(c * p * av, -s * p * av, -0.001f * cosf(PI_F / (2.f * 0.05f) * p));
    }
    float X = av * c * direction;           // X_i = |v| c BX_i dir
    return mk(X * SX, av * s * (-X) * SX, av * SZ);
}
__device__ __forceinline__ void solve_ik_leg(V3 c, bool right, float* ang) {
    const float hip = 0.055f, leg = 0.10652f, foot = 0.145f;
    float dom = (c.y * c.y + c.z * c.z - hip * hip + c.x * c.x - leg * leg - foot * foot) / (2.f * foot * leg);
    if (dom > 1.f || dom < -1.f) dom = dom > 1.f ? 0.99f : -0.99f;
    float gamma = atan2f(-sqrtf(1.f - dom * dom), dom);
    float sq = c.y * c.y + c.z * c.z - hip * hip;
    if (sq < 0.f) sq = 0.f;
    float sg, cg; sincosf(gamma, &sg, &cg);
    float alpha = atan2f(-c.x, sqrtf(sq)) - atan2f(foot * sg, leg + foot * cg);
    float hv = right ? -hip : hip;
    float theta = -atan2f(c.z, c.y) - atan2f(sqrtf(sq), hv);
    ang[0] = theta; ang[1] = -alpha; ang[2] = -gamma;
}

// Kinematics.transform (kinematics.py:49-78): R(rpy) * (v + pos), R = Rx*Ry*Rz (identity when rpy == 0)
__device__ __forceinline__ V3 ik_transform(V3 v, V3 rpy, V3 pos) {
    V3 t = v + pos;
    if (rpy.x != 0.f || rpy.y != 0.f || rpy.z != 0.f) {
        float sx, cx, sy, cy, sz, cz;
        sincosf(rpy.x, &sx, &cx); sincosf(rpy.y, &sy, &cy); sincosf(rpy.z, &sz, &cz);
        V3 a = mk(cz * t.x - sz * t.y, sz * t.x + cz * t.y, t.z);
        V3 b = mk(cy * a.x + sy * a.z, a.y, -sy * a.x + cy * a.z);
        t = mk(b.x, cx * b.y - sx * b.z, sx * b.y + cx * b.z);
    }
    return t;
}
// Kinematics.solve for the own leg with a general base pose (kinematics.py:104-142); il = IK leg index (FR,FL,RR,RL)
__device__ __forceinline__ void solve_ik_pose(V3 rpy, V3 pos, V3 frame, int il, float* ang) {
    V3 hip = mk((il < 2) ? 0.115f : -0.115f, (il & 1) ? 0.0375f : -0.0375f, 0.f);
    V3 hv = ik_transform(hip, rpy, pos);
    V3 c = frame - hv;
    V3 tc = ik_transform(c, mk(-rpy.x, -rpy.y, -rpy.z), mk(-pos.x, -pos.y, -pos.z));
    solve_ik_leg(tc, (il & 1) == 0, ang);
}

struct GaitState { double phi; int last_step; float alpha; };

// GaitPlanner.loop + Kinematics.solve for the own leg; il = IK leg index (FR,FL,RR,RL) = lane ^ 1
template <bool ROT>
__device__ __forceinline__ void ik_signal(GaitState& G, bool gallop, int step_counter, double dtd, double clk, int leg,
                                          float base_x, float base_z, float v, float w_rot, double T, float direction, float* cmd) {
    const int il = leg ^ 1;
    // fp64 timing must round exactly like the reference's Python floats: no FMA contraction (a - b*c is NOT fused)
    // clk = gait_clock_scale: (step * dt) * clk in exactly the oracle's operation order; x * 1.0 is exact
    double now = __dmul_rn(__dmul_rn((double)step_counter, dtd), clk);
    if (T <= 0.01) T = 0.01;
    if (G.phi >= 0.99) G.last_step = step_counter;
    G.phi = __ddiv_rn(__dsub_rn(now, __dmul_rn(__dmul_rn((double)G.last_step, dtd), clk)), T);
    double off = gallop ? ((il >= 2) ? 0.8 : 0.0) : ((il == 1 || il == 2) ? 0.5 : 0.0);
    double ph = __dadd_rn(G.phi, off);
    if (ph >= 1) ph = __dsub_rn(ph, 1.);
    const bool stance = ph <= 0.5;
    float phase = stance ? (float)(ph / 0.5) : (float)((ph - 0.5) / (1 - 0.5));
    float SX = 0.f, SZ = 0.f;
    if (!stance) bezier_sums(phase, SX, SZ);
    const float fx = (il < 2) ? 0.115f : -0.115f, fy = (il & 1) ? 0.0925f : -0.0925f, fz = -0.2f;
    V3 lg = step_part(stance, phase, SX, SZ, v, 0.f, direction);
    V3 rt;
    if (ROT) {
        // legs update the shared alpha serially in IK order FR, FL, RR, RL (gait_planner.py:66-89)
        const float r = sqrtf(fx * fx + fy * fy);
        const float foot_angle = atan2f(fy, fx);
        float alpha = G.alpha;
        rt = mk(0, 0, 0);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            float circle = (w_rot >= 0.f ? 90.f : 270.f) - (foot_angle - alpha) * (180.0f / PI_F);
            V3 cand = step_part(stance, phase, SX, SZ, w_rot, circle, direction);
            float mag = atan2f(sqrtf(cand.x * cand.x + cand.y * cand.y), r);
            float na = (fy > 0.f) ? ((cand.x < 0.f) ? -mag : mag) : ((cand.x < 0.f) ? mag : -mag);
            if (il == k) rt = cand;
            alpha = bcast4(na, k ^ 1);
        }
        G.alpha = alpha;
    } else {
        rt = mk(0.f, 0.f, stance ? -0.001f * cosf(PI_F / (2.f * 0.05f) * (0.05f * (1.f - 2.f * phase))) : 0.f);
    }
    // Kinematics.solve with zero orientation: hip = HIP + pos; coord = foot - hip; t = coord - pos
    V3 frame = mk(fx + lg.x + rt.x, fy + lg.y + rt.y, fz + lg.z + rt.z);
    V3 hipv = mk(((il < 2) ? 0.115f : -0.115f) + base_x, ((il & 1) ? 0.0375f : -0.0375f), 0.f + base_z);
    V3 c = frame - hipv;
    V3 tc = mk(c.x - base_x, c.y, c.z - base_z);
    solve_ik_leg(tc, (il & 1) == 0, cmd);
}

static __constant__ float c_pose_stand[3] = {0.f, -0.88643435f, 1.30197369f};
static __constant__ float c_pose_stand_ol[3] = {0.15192765f, -0.90412283f, 1.48156545f};   // sign of [0] alternates per leg

__device__ __forceinline__ void init_pose(int signal, int leg, float* p) {
    if (signal == REXSIM_SIGNAL_OL) { p[0] = (leg & 1) ? -c_pose_stand_ol[0] : c_pose_stand_ol[0]; p[1] = c_pose_stand_ol[1]; p[2] = c_pose_stand_ol[2]; }
    else { p[0] = c_pose_stand[0]; p[1] = c_pose_stand[1]; p[2] = c_pose_stand[2]; }
}

// per-env task bookkeeping (replicated on the 4 lanes)
struct Task {
    int step_counter, env_step, flags, end_step;
    float target, torient, iorient;
    GaitState G;
};

// <task>._transform_action_to_motor_command for the own leg
template <int TASK, int SIGNAL>
__device__ __forceinline__ void task_command(const Params& P, Task& K, const Lane& L, int leg, const float* act, float* cmd,
                                             const float* sq = nullptr /* sensed base quaternion (sensor model on), else the true one */) {
    const double dtd = P.cfg.sim_dt_d;
    const double t = __dmul_rn((double)K.step_counter, dtd);     // products via __dmul_rn: never contracted into FMAs
    float ip[3]; init_pose(SIGNAL, leg, ip);
    if (TASK == REXSIM_TASK_WALK) {                                   // envs/gym/walk_env.py:207-324
        if (K.flags & FL_STILL) { cmd[0] = ip[0]; cmd[1] = ip[1]; cmd[2] = ip[2]; return; }
        if (K.target != 0.f) {
            if (fabsf(L.pos.x) >= fabsf(K.target) - 0.15f) {
                K.flags |= FL_GOAL;
                if (!(K.flags & FL_TERMINATING)) { K.end_step = K.step_counter; K.flags |= FL_TERMINATING; }
            }
        }
        const double end_t = __dmul_rn((double)K.end_step, dtd);
        if (SIGNAL == REXSIM_SIGNAL_IK) {
            double p = 0.8 + (double)act[0];
            double gait = (0.0 <= t && t <= p) ? t : 1.0;
            double step = 0.6, period = 0.65; float base_x = 0.01f;
            if (K.flags & FL_BACKWARDS) { step = -.3; period = .5; base_x = 0.f; }
            double sl = step * gait;
            if (K.flags & FL_GOAL) {
                double pb = 0.8 + (double)act[1];
                double brakes = (end_t <= t && t <= pb + end_t) ? 1 - (t - end_t) : 0.0;
                sl *= brakes;
                if (brakes == 0.0) K.flags |= FL_STILL;
            }
            float direction = sl < 0 ? -1.f : 1.f;
            ik_signal<false>(K.G, false, K.step_counter, dtd, P.cfg.gait_clock_scale, leg, base_x, 0.f, (float)sl, 0.f, period, direction, cmd);
        } else {
            double l_a = 0.1, f_a = 0.2;
            if (K.flags & FL_GOAL) {
                double coeff = (end_t <= t && t <= 0.8 + end_t) ? 1 - (t - end_t) : 0.0;
                l_a *= coeff; f_a *= coeff;
                if (coeff == 0.0) K.flags |= FL_STILL;
            }
            double start = (0.0 <= t && t <= 0.8) ? t : 1.0;
            l_a *= start; f_a *= start;
            double cs = cos(2 * PI_D / (1.0 / 8) * t);
            float l_ext = (float)(l_a * cs), f_ext = (float)(f_a * cs);
            const bool diag = (leg == 0 || leg == 3);     // FL and RR extend, FR and RL swing
            cmd[0] = ip[0];
            cmd[1] = ip[1] + ((diag ? l_ext : -l_ext) + act[2 * leg]);
            cmd[2] = ip[2] + ((diag ? f_ext : -f_ext) + act[2 * leg + 1]);
        }
    } else if (TASK == REXSIM_TASK_GALLOP) {                          // envs/gym/gallop_env.py:212-313
        if (K.flags & FL_STILL) { cmd[0] = c_pose_stand[0]; cmd[1] = c_pose_stand[1]; cmd[2] = c_pose_stand[2]; return; }
        if (K.target != 0.f) {
            if (fabsf(L.pos.x) >= fabsf(K.target)) {
                K.flags |= FL_GOAL;
                if (!(K.flags & FL_TERMINATING)) { K.end_step = K.step_counter; K.flags |= FL_TERMINATING; }
            }
        }
        const double end_t = __dmul_rn((double)K.end_step, dtd);
        if (SIGNAL == REXSIM_SIGNAL_IK) {
            double p = 1. + (double)act[1];
            double gait = (0.0 <= t && t <= p) ? t : 1.0;
            double sl = 1.3 * gait;
            if (K.flags & FL_GOAL) {
                double pb = 1. + (double)act[0];
                double brakes = (end_t <= t && t <= pb + end_t) ? 1 - (t - end_t) : 0.0;
                sl *= brakes;
            }
            ik_signal<false>(K.G, true, K.step_counter, dtd, P.cfg.gait_clock_scale, leg, 0.01f, -0.007f, (float)sl, 0.f, 0.3, 1.f, cmd);
        } else {
            float a0 = act[(leg < 2) ? 0 : 2], a1 = act[(leg < 2) ? 1 : 3];
            if (K.flags & FL_GOAL) {
                double coeff = (end_t <= t && t <= 1. + end_t) ? 1 - (t - end_t) : 0.0;
                a0 = (float)((double)a0 * coeff); a1 = (float)((double)a1 * coeff);
                if (coeff == 0.0) K.flags |= FL_STILL;
            }
            cmd[0] = ip[0]; cmd[1] = ip[1] + a0; cmd[2] = ip[2] + a1;
        }
    } else if (TASK == REXSIM_TASK_TURN) {                            // envs/gym/turn_env.py:230-346
        if (K.flags & FL_STILL) {
            if (__dsub_rn(t, __dmul_rn((double)K.end_step, dtd)) >= 1.) K.flags |= FL_ENVGOAL;
            cmd[0] = ip[0]; cmd[1] = ip[1]; cmd[2] = ip[2];
            return;
        }
        {
            float rpy[3];
            if (sq) quat_to_euler(sq[0], sq[1], sq[2], sq[3], rpy);            // rex.GetBaseOrientation() turn_env.py:325
            else quat_to_euler(L.qx, L.qy, L.qz, L.qw, rpy);
            float cz = rpy[2];
            if (cz < 0.f) cz += 6.28f;
            if (fabsf(K.torient - cz) <= 0.01f) {
                K.flags |= FL_GOAL;
                if (!(K.flags & FL_TERMINATING)) { K.end_step = K.step_counter; K.flags |= FL_TERMINATING; }
            }
        }
        if (SIGNAL == REXSIM_SIGNAL_IK) {
            double gait = (0.0 <= t && t <= .8) ? t : 1.0;
            double dirv = __dmul_rn(-0.5, gait);
            if (K.flags & FL_CLOCKWISE) dirv *= -1;
            float step_rotation = (float)(dirv + (double)act[0]);
            double step_period = 0.75 + (double)act[1];
            if (K.flags & FL_GOAL) K.flags |= FL_STILL;
            ik_signal<true>(K.G, false, K.step_counter, dtd, P.cfg.gait_clock_scale, leg, 0.009f, 0.f, 0.02f, step_rotation, step_period, 1.f, cmd);
        } else {
            if (K.flags & FL_GOAL) K.flags |= FL_STILL;
            const float extension = 0.1f, swing = 0.03f + act[0], swipe = 0.05f + act[1];
            int ith = ((int)(t / (1.0 / 10.0))) % 2;
            const bool cw = (K.flags & FL_CLOCKWISE) != 0;
            // pose tables of turn_env.py:281-298, row = leg
            const float sgn = ((leg == 0 || leg == 3) ? 1.f : -1.f) * (cw ? 1.f : -1.f);
            float o0, o1, o2;
            if (!ith) { o0 = (leg & 1) ? -swipe : swipe; o1 = (leg < 2) ? extension : -extension; o2 = sgn * swing; }
            else { o0 = (leg & 1) ? swipe : -swipe; o1 = 0.f; o2 = -sgn * swing; }
            float so[3]; init_pose(REXSIM_SIGNAL_OL, leg, so);
            cmd[0] = so[0] + o0; cmd[1] = so[1] + o1; cmd[2] = so[2] + o2;
        }
    } else if (TASK == REXSIM_TASK_POSES) {                           // envs/gym/poses_env.py:178-225
        const double p = 0.8 + (double)act[0];
        const double coeff = (0.0 <= t && t <= p) ? t : 1.0;
        const float staged = (float)((double)K.target * coeff);
        const int pose = (K.flags >> FL_POSE_SHIFT) & 7;
        V3 pos = mk(0.01f, pose == 0 ? staged : 0.f, pose == 1 ? staged : 0.f);
        V3 rpy = mk(pose == 2 ? staged : 0.f, pose == 3 ? staged : 0.f, pose == 4 ? staged : 0.f);
        const int il = leg ^ 1;
        solve_ik_pose(rpy, pos, mk((il < 2) ? 0.115f : -0.115f, (il & 1) ? 0.0925f : -0.0925f, -0.2f), il, cmd);
    } else {                                                          // envs/gym/standup_env.py:113-134
        if (t > 0.1) { cmd[0] = c_pose_stand[0]; cmd[1] = c_pose_stand[1]; cmd[2] = c_pose_stand[2]; return; }
        double tt = t + 1;
        float sc = (float)((.1 + (double)act[0]) / tt + 1.5);
        cmd[0] = c_pose_stand[0] * sc; cmd[1] = c_pose_stand[1] * sc; cmd[2] = c_pose_stand[2] * sc;
    }
}

// -------------------------------------------------------------------------------------------------
// state load / store (SoA, coalesced across envs)
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void load_lane(const float* sf, const int32_t* si, int N, int env, int leg, Lane& L) {
    L.pos = mk(sf[(F_POS + 0) * (size_t)N + env], sf[(F_POS + 1) * (size_t)N + env], sf[(F_POS + 2) * (size_t)N + env]);
    L.qx = sf[(F_QUAT + 0) * (size_t)N + env]; L.qy = sf[(F_QUAT + 1) * (size_t)N + env];
    L.qz = sf[(F_QUAT + 2) * (size_t)N + env]; L.qw = sf[(F_QUAT + 3) * (size_t)N + env];
    L.vl = mk(sf[(F_LINVEL + 0) * (size_t)N + env], sf[(F_LINVEL + 1) * (size_t)N + env], sf[(F_LINVEL + 2) * (size_t)N + env]);
    L.w = mk(sf[(F_ANGVEL + 0) * (size_t)N + env], sf[(F_ANGVEL + 1) * (size_t)N + env], sf[(F_ANGVEL + 2) * (size_t)N + env]);
#pragma unroll
    for (int j = 0; j < 3; j++) {
        L.q[j] = sf[(F_Q + 3 * leg + j) * (size_t)N + env];
        L.qd[j] = sf[(F_QD + 3 * leg + j) * (size_t)N + env];
        L.tau_obs[j] = 0.f;
    }
    L.ovh = (uint32_t)si[(I_OVH + leg) * (size_t)N + env];
    L.enabled = ((uint32_t)si[I_FLAGS * (size_t)N + env] >> (FL_ENABLED_SHIFT + 3 * leg)) & 7u;
    L.contact = 0; L.err = 0; L.cost = 0;
}
__device__ __forceinline__ void load_task(const float* sf, const int32_t* si, int N, int env, Task& K) {
    K.step_counter = si[I_STEP * (size_t)N + env];
    K.env_step = si[I_ENVSTEP * (size_t)N + env];
    K.flags = si[I_FLAGS * (size_t)N + env];
    K.end_step = si[I_ENDSTEP * (size_t)N + env];
    K.G.last_step = si[I_GPLAST * (size_t)N + env];
    K.G.phi = __hiloint2double(si[I_PHI_HI * (size_t)N + env], si[I_PHI_LO * (size_t)N + env]);
    K.G.alpha = sf[F_ALPHA * (size_t)N + env];
    K.target = sf[F_TARGET * (size_t)N + env];
    K.torient = sf[F_TORIENT * (size_t)N + env];
    K.iorient = sf[F_IORIENT * (size_t)N + env];
}
__device__ __forceinline__ void store_lane(float* sf, int32_t* si, int N, int env, int leg, const Lane& L, const Task& K, bool valid) {
    // shuffles first (all lanes participate), stores predicated on `valid`
    uint32_t en = or4(L.enabled << (3 * leg));
    // contact mask in the oracle's group numbering: bit 0 base, bit 1+2l upper group of leg l, bit 2+2l foot group
    uint32_t ct = or4((((uint32_t)L.contact & 1u) << (2 + 2 * leg)) | ((((uint32_t)L.contact >> 1) & 1u) << (1 + 2 * leg)) | (((uint32_t)L.contact >> 2) & 1u));
    if (!valid) return;
#pragma unroll
    for (int j = 0; j < 3; j++) {
        sf[(F_Q + 3 * leg + j) * (size_t)N + env] = L.q[j];
        sf[(F_QD + 3 * leg + j) * (size_t)N + env] = L.qd[j];
    }
    si[(I_OVH + leg) * (size_t)N + env] = (int32_t)L.ovh;
    if (leg == 0) {
        sf[(F_POS + 0) * (size_t)N + env] = L.pos.x; sf[(F_POS + 1) * (size_t)N + env] = L.pos.y; sf[(F_POS + 2) * (size_t)N + env] = L.pos.z;
        sf[(F_QUAT + 0) * (size_t)N + env] = L.qx; sf[(F_QUAT + 1) * (size_t)N + env] = L.qy;
        sf[(F_QUAT + 2) * (size_t)N + env] = L.qz; sf[(F_QUAT + 3) * (size_t)N + env] = L.qw;
        sf[(F_LINVEL + 0) * (size_t)N + env] = L.vl.x; sf[(F_LINVEL + 1) * (size_t)N + env] = L.vl.y; sf[(F_LINVEL + 2) * (size_t)N + env] = L.vl.z;
        sf[(F_ANGVEL + 0) * (size_t)N + env] = L.w.x; sf[(F_ANGVEL + 1) * (size_t)N + env] = L.w.y; sf[(F_ANGVEL + 2) * (size_t)N + env] = L.w.z;
        sf[F_ALPHA * (size_t)N + env] = K.G.alpha;
        sf[F_TARGET * (size_t)N + env] = K.target;
        si[I_STEP * (size_t)N + env] = K.step_counter;
        si[I_ENVSTEP * (size_t)N + env] = K.env_step;
        si[I_FLAGS * (size_t)N + env] = (K.flags & (((1 << FL_ENABLED_SHIFT) - 1) | (7 << FL_POSE_SHIFT))) | (int32_t)(en << FL_ENABLED_SHIFT);
        si[I_ENDSTEP * (size_t)N + env] = K.end_step;
        si[I_GPLAST * (size_t)N + env] = K.G.last_step;
        si[I_PHI_HI * (size_t)N + env] = __double2hiint(K.G.phi);
        si[I_PHI_LO * (size_t)N + env] = __double2loint(K.G.phi);
        si[I_CONTACT * (size_t)N + env] = (int32_t)ct;
    }
}

// arm state (lane 0 of the env): 6 joint angles / rates, overheat counters, enabled bits
__device__ __forceinline__ void load_arm(const float* sf, const int32_t* si, int N, int env, Arm& A) {
#pragma unroll
    for (int j = 0; j < ARM_NJ; j++) {
        A.q[j] = sf[(F_AQ + j) * (size_t)N + env]; A.qd[j] = sf[(F_AQD + j) * (size_t)N + env]; A.tau_obs[j] = 0.f;
    }
    A.ovh[0] = (uint32_t)si[(I_OVHA + 0) * (size_t)N + env]; A.ovh[1] = (uint32_t)si[(I_OVHA + 1) * (size_t)N + env];
    A.enabled = ((uint32_t)si[I_FLAGS * (size_t)N + env] >> FL_ARM_ENABLED_SHIFT) & 63u;
}
__device__ __forceinline__ void store_arm(float* sf, int32_t* si, int N, int env, const Arm& A) {
#pragma unroll
    for (int j = 0; j < ARM_NJ; j++) { sf[(F_AQ + j) * (size_t)N + env] = A.q[j]; sf[(F_AQD + j) * (size_t)N + env] = A.qd[j]; }
    si[(I_OVHA + 0) * (size_t)N + env] = (int32_t)A.ovh[0]; si[(I_OVHA + 1) * (size_t)N + env] = (int32_t)A.ovh[1];
    // store_lane (which runs first) wrote the flags word without the arm bits
    si[I_FLAGS * (size_t)N + env] = (si[I_FLAGS * (size_t)N + env] & ~(63 << FL_ARM_ENABLED_SHIFT)) | (int32_t)(A.enabled << FL_ARM_ENABLED_SHIFT);
}

// reset one env from the settled snapshot + task draws (BatchEnv.reset -> <task>.reset; rex.py:255-324)
template <bool ARM>
// `valid` is false on the padding lanes that replicate the last env to keep warps whole: they compute, but never write
// (a replica that re-read the counter after the real lane's write would otherwise bump it twice)
__device__ __forceinline__ void reset_from_snapshot(const Params& P, int env, int leg, Lane& L, Task& K, float& kp, float& kd, int& field, Arm& AR, bool valid,
                                                    Sensor& S) {
    const RexSimConfig& c = P.cfg;
    const int N = P.N;
    uint32_t rc = (uint32_t)P.si[I_RESETCNT * (size_t)N + env] + 1u;
    const uint32_t genv = (uint32_t)env + (uint32_t)c.env_offset;   // global env id: draws do not depend on the sharding
    field = (c.terrain == REXSIM_TERRAIN_RANDOM) ? (int)((genv + rc) % (uint32_t)c.nfields) : 0;
    const float* sf = P.snap_f + (size_t)field * NF;
    const int32_t* si = P.snap_i + (size_t)field * NI;
    load_lane(sf, si, 1, 0, leg, L);
    load_task(sf, si, 1, 0, K);
    if (ARM && leg == 0) load_arm(sf, si, 1, 0, AR);
    K.step_counter = 0; K.env_step = 0; K.end_step = 0;
    K.flags = K.flags & ~((1 << FL_ENABLED_SHIFT) - 1);
    K.G.phi = 0.0; K.G.last_step = 0; K.G.alpha = 0.f;
    K.target = 0.f; K.torient = 0.f; K.iorient = 0.f;
    kp = (c.kp_lo == c.kp_hi) ? c.motor_kp : (float)rand_uniform(c.seed, genv, rc,4, c.kp_lo, c.kp_hi);
    kd = (c.kd_lo == c.kd_hi) ? c.motor_kd : (float)rand_uniform(c.seed, genv, rc,5, c.kd_lo, c.kd_hi);
    if (c.task == REXSIM_TASK_WALK) {
        int bw = (c.backwards < 0) ? (int)(rand_u32(c.seed, genv, rc,0) >> 31) : c.backwards;
        if (bw) K.flags |= FL_BACKWARDS;
        if (isnan(c.target_position)) K.target = (float)rand_uniform(c.seed, genv, rc,1, bw ? -2.0 : 1.0, bw ? -3.0 : 3.0);
        else K.target = c.target_position;
    } else if (c.task == REXSIM_TASK_GALLOP) {
        K.target = isnan(c.target_position) ? (float)rand_uniform(c.seed, genv, rc,1, 1.0, 3.0) : c.target_position;
    } else if (c.task == REXSIM_TASK_TURN) {
        double to = isnan(c.target_orient) ? rand_uniform(c.seed, genv, rc,2, 0.2, 6.0) : (double)c.target_orient;
        double io = isnan(c.init_orient) ? rand_uniform(c.seed, genv, rc,3, 0.2, 6.0) : (double)c.init_orient;
        K.torient = (float)to; K.iorient = (float)io;
        double diff = fabs(io - to);
        bool cw = false;
        if (io < to) { if (diff > 3.14) cw = true; } else { if (diff < 3.14) cw = true; }
        if (cw) K.flags |= FL_CLOCKWISE;
        L.pos = mk(0.f, 0.f, 0.21f);
        float hy = (float)(io * 0.5);
        L.qx = 0.f; L.qy = 0.f; L.qz = sinf(hy); L.qw = cosf(hy);
    } else if (c.task == REXSIM_TASK_POSES) {                         // poses_env.py:148-176
        bool any = false;
#pragma unroll
        for (int k = 0; k < 5; k++) any = any || !isnan(c.pose_values[k]);
        int pose;
        if (any) {                      // fill_next_pose_and_target (a None argument counts as 0.0)
            pose = 4;
#pragma unroll
            for (int k = 3; k >= 0; k--) if (!isnan(c.pose_values[k]) && c.pose_values[k] != 0.f) pose = k;
            float v = c.pose_values[pose];
            K.target = isnan(v) ? 0.f : v;
        } else {                        // deque rotation; the constructor's own reset() consumed 'base_y'
            pose = (int)(rc % 5u);
            const double lo = pose == 0 ? -0.007 : pose == 1 ? -0.048 : -PI_D / 4, hi = pose == 0 ? 0.007 : pose == 1 ? 0.021 : PI_D / 4;
            K.target = (float)rand_uniform(c.seed, genv, rc, 6, lo, hi);
        }
        K.flags = (K.flags & ~(7 << FL_POSE_SHIFT)) | (pose << FL_POSE_SHIFT);
    }
    if (P.sensor_on) {
        // the history the reset hold left behind only depends on the field, like the settled state: copy the snapshot's rows
        // (same slots: the push count is copied with them).  Written by the env's own 4 lanes, read after the __syncwarp.
        const int words = S.words, depth = S.depth;
        S.push = si[I_HPUSH]; S.rc = rc;
        if (valid) {
            const float* src = P.snap_ring + (size_t)field * depth * words;
            for (int t = leg; t < depth * words; t += 4) S.ring[(size_t)t * N + env] = src[t];
        }
        __syncwarp(env_mask());
    }
    if (valid && leg == 0) {
        P.si[I_RESETCNT * (size_t)N + env] = (int32_t)rc;
        P.si[I_FIELD * (size_t)N + env] = field;
        if (P.sensor_on) P.si[I_HPUSH * (size_t)N + env] = S.push;
        P.sf[F_KP * (size_t)N + env] = kp; P.sf[F_KD * (size_t)N + env] = kd;
        P.sf[F_TORIENT * (size_t)N + env] = K.torient; P.sf[F_IORIENT * (size_t)N + env] = K.iorient;
    }
}

__device__ __forceinline__ float map_pi(float a) {   // MapToMinusPiToPi rex.py:26-41
    const float TWO_PI = 6.283185307179586f;
    float r = fmodf(a, TWO_PI);
    if (r >= PI_F) r -= TWO_PI; else if (r < -PI_F) r += TWO_PI;
    return r;
}
// _get_observation (+ RangeNormalize) for the env; lane 0 writes the 4 base terms, every lane its 3 angles (gallop).
// Sensor model on: GetBaseRollPitchYaw / GetBaseRollPitchYawRate / GetMotorAngles = delayed row + noise (rex.py:429-442,548-558,457-468)
template <int TASK, bool SENSOR>
__device__ __forceinline__ bool write_obs(const Params& P, int env, int leg, const Lane& L, float* obs_row,
                                          const Sensor& S, uint32_t step) {
    float rpy[3];
    float wx = L.w.x, wy = L.w.y;
    float qa[3] = {L.q[0], L.q[1], L.q[2]};
    if (SENSOR) {
        float d4[4];
#pragma unroll
        for (int a = 0; a < 4; a++) d4[a] = sensor_delayed(S, P.lat_ctl, P.n_ctl, P.a_ctl, HW_BASE + a);
        quat_to_euler(d4[0], d4[1], d4[2], d4[3], rpy);
        rpy[0] += sensor_noise(P, S, step, 3, 0, 0); rpy[1] += sensor_noise(P, S, step, 3, 0, 1);
        wx = sensor_delayed(S, P.lat_ctl, P.n_ctl, P.a_ctl, HW_BASE + 4) + sensor_noise(P, S, step, 4, 1, 0);
        wy = sensor_delayed(S, P.lat_ctl, P.n_ctl, P.a_ctl, HW_BASE + 5) + sensor_noise(P, S, step, 4, 1, 1);
        if (TASK == REXSIM_TASK_GALLOP) {
#pragma unroll
            for (int j = 0; j < 3; j++)
                qa[j] = sensor_delayed(S, P.lat_ctl, P.n_ctl, P.a_ctl, 9 * leg + j) + sensor_noise(P, S, step, 0, 2, 3 * leg + j);
        }
    } else quat_to_euler(L.qx, L.qy, L.qz, L.qw, rpy);
    const float two_pi = 6.283185307179586f;
    const float ub_ang = two_pi + 0.01f, ub_rate = (float)(2.0 * PI_D / P.cfg.sim_dt_d) + 0.01f;
    float o[4] = {rpy[0], rpy[1], wx, wy};
    bool finite = true;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        float v = o[j];
        finite = finite && isfinite(v);
        if (P.cfg.normalize) { float hi = (j < 2) ? ub_ang : ub_rate; v = 2.f * (v + hi) / (2.f * hi) - 1.f; }
        o[j] = v;
    }
    if (leg == 0) { obs_row[0] = o[0]; obs_row[1] = o[1]; obs_row[2] = o[2]; obs_row[3] = o[3]; }
    if (TASK == REXSIM_TASK_GALLOP) {
#pragma unroll
        for (int j = 0; j < 3; j++) {
            float v = map_pi(qa[j]);
            finite = finite && isfinite(v);
            if (P.cfg.normalize) v = 2.f * (v + ub_ang) / (2.f * ub_ang) - 1.f;
            obs_row[4 + 3 * leg + j] = v;
        }
    }
    return finite;
}

// -------------------------------------------------------------------------------------------------
// the fused step kernel
// -------------------------------------------------------------------------------------------------
// OCC = resident CTAs per SM the variant is compiled for: 1 -> 255 registers (lowest latency, small batches),
// 4 -> 128 registers (16 warps/SM hide the serial PGS / ABA chains, large batches)
// SENSOR: the observation-history / latency / noise model of Rex (rex.py:726-769) is compiled in (any latency or noise > 0);
// the default build reads the true state and keeps no history.
// heightfield tiles, (BLOCK / 4) x TILE_FLOATS floats (random terrain only), then (BLOCK / 4) x PGS_ENV_FLOATS (replicated PGS only)
extern __shared__ __align__(16) float dyn_smem[];
template <int TASK, int SIGNAL, int TERRAIN, int OCC, bool ARM, bool SENSOR, int BLOCK>
__global__ void __launch_bounds__(BLOCK, (OCC * 128) / BLOCK) step_kernel(const Params P) {
    __shared__ __align__(16) float sm[ARM ? REXSIM_MT_FLOATS_ARM : REXSIM_MT_FLOATS];
    __shared__ __align__(8) uint64_t bar;
    float* tiles = dyn_smem;
    float* pgs = dyn_smem + (TERRAIN == REXSIM_TERRAIN_RANDOM ? (BLOCK / 4) * TILE_FLOATS : 0) + (threadIdx.x >> 2) * PGS_ENV_FLOATS;
    tma_load_tables(sm, P.model, (ARM ? REXSIM_MT_FLOATS_ARM : REXSIM_MT_FLOATS) * 4, &bar);

    const int N = P.N;
    const int gid = blockIdx.x * blockDim.x + threadIdx.x;
    int slot = gid >> 2;
    const int leg = gid & 3;
    const bool valid = slot < N;
    if (!valid) slot = N - 1;         // keep the warp converged for the shuffles; stores are masked
    // Warp re-grouping: slot -> env through a permutation sorted by last step's solver cost (rexsim_rebalance), so the 8
    // envs of a warp need about the same number of PGS iterations.  Every env's arithmetic is independent of the
    // permutation (bit-identical results); the scattered state accesses stay in L2.
    const int env = P.perm ? P.perm[slot] : slot;
    const RexSimConfig& c = P.cfg;
    constexpr int A = task_shape(TASK).act[SIGNAL == REXSIM_SIGNAL_IK ? 0 : 1];
    constexpr float bound = task_shape(TASK).bound[SIGNAL == REXSIM_SIGNAL_IK ? 0 : 1];
    constexpr int O = obs_dim(TASK, 12);
    constexpr bool REPL = pgs_replicated(OCC, ARM, TERRAIN);

    Lane L; Task K; Arm AR;
    load_lane(P.sf, P.si, N, env, leg, L);
    load_task(P.sf, P.si, N, env, K);
    if (ARM && leg == 0) load_arm(P.sf, P.si, N, env, AR);
    float kp = P.sf[F_KP * (size_t)N + env], kd = P.sf[F_KD * (size_t)N + env];
    int field = P.si[I_FIELD * (size_t)N + env];
    Sensor S = make_sensor<ARM>(P, P.ring, N, env, (uint32_t)env + (uint32_t)c.env_offset);
    if (SENSOR) { S.push = P.si[I_HPUSH * (size_t)N + env]; S.rc = (uint32_t)P.si[I_RESETCNT * (size_t)N + env]; }
    Ground G;
    load_tile<TERRAIN>(P, field, L.pos, tiles + (TERRAIN == REXSIM_TERRAIN_RANDOM ? (threadIdx.x >> 2) * TILE_FLOATS : 0), G, leg);

    // action: ClipAction + RangeNormalize._denormalize_action (wrappers.py:218-236,262-265)
    float act[A];
#pragma unroll
    for (int j = 0; j < A; j++) {
        float v = P.actions[(size_t)env * A + j];
        if (c.normalize) {
            v = fminf(fmaxf(v, -1.f), 1.f);
            v = (v + 1.f) / 2.f * (2.f * bound) + (-bound);
        }
        act[j] = v;
    }
    float cmd[3];
    if (SENSOR && TASK == REXSIM_TASK_TURN) {
        float sq[4]; sensed_quat(P, S, (uint32_t)K.env_step, 7, sq);
        task_command<TASK, SIGNAL>(P, K, L, leg, act, cmd, sq);
    } else task_command<TASK, SIGNAL>(P, K, L, leg, act, cmd);
    if (valid) {
#pragma unroll
        for (int j = 0; j < 3; j++) P.cmd_out[(size_t)(3 * leg + j) * N + env] = cmd[j];
        if (ARM && leg == 0) {            // the arm holds ARM_POSES['rest'] (rex_gym_env.py:363-367): info['action'] has all 18
#pragma unroll
            for (int j = 0; j < ARM_NJ; j++) P.cmd_out[(size_t)(12 + j) * N + env] = c_arm_rest[j];
        }
    }
    // Rex.Step (rex.py:158-163)
    for (int r = 0; r < c.action_repeat; r++) {
#if REXSIM_SYNC_SUBSTEP
        __syncthreads();
#endif
        apply_action_and_step<TERRAIN, ARM, SENSOR, REPL>(P, sm, L, leg, cmd, kp, kd, G, AR, S, valid, pgs);
        K.step_counter += 1;
    }
    if (G.miss) L.err |= REXSIM_FLAG_TILE_MISS;
    // ---- reward (rex_gym_env.py:501-542; turn_env.py:362-367; standup_env.py:151-167) -----------------------
    float reward;
    M3 R = quat_to_mat(L.qx, L.qy, L.qz, L.qw);
    const uint32_t ctl_step = (uint32_t)K.env_step;      // noise key of this step's reward / termination draws
    if (TASK == REXSIM_TASK_TURN) reward = 0.035f - fabsf(L.pos.x) - fabsf(L.pos.y);
    else if (TASK == REXSIM_TASK_POSES) reward = 1.0f;                // poses_env.py:256-258
    else if (TASK == REXSIM_TASK_STANDUP) {
        float pr = fabsf(L.pos.x) + fabsf(L.pos.y) + fabsf(0.21f - L.pos.z);
        pr = (fabsf(pr) < 0.1f) ? 1.0f - pr : -pr;
        if (L.pos.z > 0.21f) pr = -1.0f - pr;
        reward = pr;
    } else {
        float cx = -L.pos.x;
        // the reference flips on the CONSTRUCTOR argument only (rex_gym_env.py:269,506 `self._backwards`): a direction drawn
        // at reset (walk_env.py:133-136, `self.backwards`) leaves the forward objective unflipped -- restated as is
        if (c.backwards == 1) cx = -cx;
        K.target = fabsf(K.target);
        float tp = K.target, fwd;
        if (cx > tp + 0.15f) fwd = tp - cx;
        else if (tp <= cx && cx <= tp + 0.15f) fwd = 1.0f;
        else if (cx <= 0.05f) fwd = 0.0f;
        else fwd = cx / tp;
        float drift = -fabsf(L.pos.y);
        float shake, e;
        if (SENSOR) {
            // rex.GetBaseOrientation() / GetMotorTorques() . GetMotorVelocities() (rex_gym_env.py:530-537): delayed row + noise
            float sq[4]; sensed_quat(P, S, ctl_step, 3, sq);
            M3 Rs = quat_to_mat(sq[0], sq[1], sq[2], sq[3]);
            shake = -fabsf(Rs.c0.z + Rs.c1.z);
            e = 0.f;
#pragma unroll
            for (int j = 0; j < 3; j++) {
                const float to = sensor_delayed(S, P.lat_ctl, P.n_ctl, P.a_ctl, 9 * leg + 6 + j) + sensor_noise(P, S, ctl_step, 2, 4, 3 * leg + j);
                const float vo = sensor_delayed(S, P.lat_ctl, P.n_ctl, P.a_ctl, 9 * leg + 3 + j) + sensor_noise(P, S, ctl_step, 1, 5, 3 * leg + j);
                e = fmaf(to, vo, e);
            }
            if (ARM && leg == 0) {
#pragma unroll
                for (int j = 0; j < ARM_NJ; j++) {
                    const float to = sensor_delayed(S, P.lat_ctl, P.n_ctl, P.a_ctl, HW_ARM + 12 + j) + sensor_noise(P, S, ctl_step, 2, 4, 12 + j);
                    const float vo = sensor_delayed(S, P.lat_ctl, P.n_ctl, P.a_ctl, HW_ARM + 6 + j) + sensor_noise(P, S, ctl_step, 1, 5, 12 + j);
                    e = fmaf(to, vo, e);
                }
            }
        } else {
            shake = -fabsf(R.c0.z + R.c1.z);          // rot_matrix[6] + rot_matrix[7]
            e = L.tau_obs[0] * L.qd[0] + L.tau_obs[1] * L.qd[1] + L.tau_obs[2] * L.qd[2];
            if (ARM && leg == 0) {
#pragma unroll
                for (int j = 0; j < ARM_NJ; j++) e = fmaf(AR.tau_obs[j], AR.qd[j], e);
            }
        }
        float energy = -fabsf(sum4(e)) * (float)c.sim_dt_d;
        reward = fwd * c.w_distance + energy * c.w_energy + drift * c.w_drift + shake * c.w_shake;
    }
    // ---- termination ----------------------------------------------------------------------------------------
    bool done;
    if (TASK == REXSIM_TASK_WALK || TASK == REXSIM_TASK_TURN) {
        float up = R.c2.z;
        if (SENSOR) {                                   // is_fallen reads rex.GetBaseOrientation(): delayed + noisy (rex_gym_env.py:485-488)
            float sq[4]; sensed_quat(P, S, ctl_step, 6, sq);
            up = quat_to_mat(sq[0], sq[1], sq[2], sq[3]).c2.z;
        }
        done = (up < 0.85f) || (K.flags & FL_ENVGOAL);
    }
    else if (TASK == REXSIM_TASK_POSES) done = false;                 // is_fallen() returns False (poses_env.py:247-254)
    else {
        float rpy[3]; quat_to_euler(L.qx, L.qy, L.qz, L.qw, rpy);
        bool fallen = fabsf(rpy[0]) > 0.3f || fabsf(rpy[1]) > 0.5f;
        done = (TASK == REXSIM_TASK_STANDUP) ? fallen : (fallen || (K.flags & FL_ENVGOAL) || (L.pos.y > 0.3f));
    }
    K.env_step += 1;
    if (c.max_episode_steps > 0 && K.env_step >= c.max_episode_steps) done = true;   // LimitDuration
    // ---- non-finite guard (ConvertTo32Bit raises; here: flag + force done) ----------------------------------
    bool finite = isfinite(reward) && isfinite(L.pos.x) && isfinite(L.pos.y) && isfinite(L.pos.z) &&
                  isfinite(L.q[0]) && isfinite(L.q[1]) && isfinite(L.q[2]) && isfinite(L.qd[0]) && isfinite(L.qd[1]) && isfinite(L.qd[2]);
    float* obs_row = P.obs + (size_t)env * O;
    if (valid) finite = write_obs<TASK, SENSOR>(P, env, leg, L, obs_row, S, (uint32_t)K.env_step) && finite;
    finite = (sum4(finite ? 0.f : 1.f) == 0.f);
    if (!finite) { L.err |= REXSIM_FLAG_NONFINITE; done = true; }
    int err = (int)or4((unsigned)L.err);
    if (valid && leg == 0) {
        if (P.cost) P.cost[env] = L.cost;
        P.reward[env] = reward;
        P.done[env] = done ? 1 : 0;
        // per-env word = the error bits of this env's most recent step (ConvertTo32Bit raises for the offending step only,
        // wrappers.py:522-523,542-543); the aggregate word [N] accumulates until the host reads and clears it
        P.err[env] = err;
        if (err) {
            atomicOr(&P.err[N], err);
            if (P.err_host) {
#pragma unroll
                for (int b = 0; b < 8; b++) if ((err >> b) & 1) P.err_host[b] = 1;
            }
        }
    }
    // ---- auto reset: done envs restart from the settled snapshot; obs = first observation of the new episode --
    if (c.auto_reset && done) {
        reset_from_snapshot<ARM>(P, env, leg, L, K, kp, kd, field, AR, valid, S);
        if (valid) write_obs<TASK, SENSOR>(P, env, leg, L, obs_row, S, 0u);
    }
    store_lane(P.sf, P.si, N, env, leg, L, K, valid);
    if (ARM && valid && leg == 0) store_arm(P.sf, P.si, N, env, AR);
    if (SENSOR && valid && leg == 0) P.si[I_HPUSH * (size_t)N + env] = S.push;
}

// -------------------------------------------------------------------------------------------------
// reset kernel: BatchEnv.reset(indices)
// -------------------------------------------------------------------------------------------------
template <int TASK, bool ARM>
__global__ void __launch_bounds__(128) reset_kernel(const Params P, float* obs_out) {
    const int gid = blockIdx.x * blockDim.x + threadIdx.x;
    int j = gid >> 2;
    const int leg = gid & 3;
    const int k = P.reset_idx ? P.reset_k : P.N;
    const bool valid = j < k;
    if (!valid) j = k - 1;
    int env = P.reset_idx ? P.reset_idx[j] : j;
    // an index outside [0, N) never touches state: the lane is parked on env 0 with its stores masked, the aggregate
    // error word gets REXSIM_FLAG_BAD_INDEX (the Python mirror raises IndexError like BatchEnv.reset would)
    const bool inrange = env >= 0 && env < P.N;
    if (!inrange) { if (valid && leg == 0) atomicOr(&P.err[P.N], REXSIM_FLAG_BAD_INDEX); env = 0; }
    const bool wr = valid && inrange;
    constexpr int O = obs_dim(TASK, 12);
    Lane L; Task K; Arm AR; float kp, kd; int field;
    Sensor S = make_sensor<ARM>(P, P.ring, P.N, env, (uint32_t)env + (uint32_t)P.cfg.env_offset);
    reset_from_snapshot<ARM>(P, env, leg, L, K, kp, kd, field, AR, wr, S);
    if (wr && obs_out) {
        if (P.sensor_on) write_obs<TASK, true>(P, env, leg, L, obs_out + (size_t)j * O, S, 0u);
        else write_obs<TASK, false>(P, env, leg, L, obs_out + (size_t)j * O, S, 0u);
    }
    if (wr && leg == 0) P.err[env] = 0;
    store_lane(P.sf, P.si, P.N, env, leg, L, K, wr);
    if (ARM && wr && leg == 0) store_arm(P.sf, P.si, P.N, env, AR);
}

// -------------------------------------------------------------------------------------------------
// settle kernel: Rex.Reset (rex.py:296-324) for one snapshot, 4 lanes: 100 sub-steps holding 'stand'
// then reset_time/dt holding the task's init pose; writes the snapshot row
// -------------------------------------------------------------------------------------------------
template <int TERRAIN, bool ARM, bool SENSOR>
__global__ void __launch_bounds__(32) settle_kernel(const Params P, float* snap_f, int32_t* snap_i, int signal, int task) {
    __shared__ __align__(16) float sm[ARM ? REXSIM_MT_FLOATS_ARM : REXSIM_MT_FLOATS];
    __shared__ __align__(8) uint64_t bar;
    __shared__ float tiles[TERRAIN == REXSIM_TERRAIN_RANDOM ? 8 * TILE_FLOATS : 1];
    tma_load_tables(sm, P.model, (ARM ? REXSIM_MT_FLOATS_ARM : REXSIM_MT_FLOATS) * 4, &bar);
    const int leg = threadIdx.x & 3;
    const int field = P.settle_snapshot;
    Lane L; Task K;
    L.pos = mk(0.f, 0.f, 0.21f); L.qx = 0.f; L.qy = 0.f; L.qz = 0.f; L.qw = 1.f;
    L.vl = mk(0, 0, 0); L.w = mk(0, 0, 0);
    for (int j = 0; j < 3; j++) { L.q[j] = c_pose_stand[j]; L.qd[j] = 0.f; L.tau_obs[j] = 0.f; }
    L.ovh = 0u; L.enabled = 7u; L.contact = 0; L.err = 0; L.cost = 0;
    Arm AR;
    if (ARM) {
#pragma unroll
        for (int j = 0; j < ARM_NJ; j++) { AR.q[j] = c_arm_rest[j]; AR.qd[j] = 0.f; AR.tau_obs[j] = 0.f; }
        AR.ovh[0] = 0u; AR.ovh[1] = 0u; AR.enabled = 63u;
    }
    K.step_counter = 0; K.env_step = 0; K.flags = 0; K.end_step = 0; K.target = 0; K.torient = 0; K.iorient = 0;
    K.G.phi = 0.0; K.G.last_step = 0; K.G.alpha = 0.f;
    Ground G;
    load_tile<TERRAIN>(P, field, L.pos, tiles + (TERRAIN == REXSIM_TERRAIN_RANDOM ? (threadIdx.x >> 2) * TILE_FLOATS : 0), G, leg);
    float stand[3] = {c_pose_stand[0], c_pose_stand[1], c_pose_stand[2]};
    float ip[3];
    if (task == REXSIM_TASK_STANDUP) { ip[0] = (leg & 1) ? 0.4f : -0.4f; ip[1] = -1.5f; ip[2] = 6.f; }
    else init_pose(signal, leg, ip);
    // RexPosesEnv.reset -> RexGymEnv.reset(initial_motor_angles=None): Rex.Reset skips both holding phases (rex.py:307)
    // sensor history of the reset hold: _observation_history.clear() (rex.py:303), one ReceiveObservation before the hold
    // (:313), one per sub-step, one after it (:324).  The 8 replicas of the warp write identical rows to the same addresses.
    Sensor S = make_sensor<ARM>(P, nullptr, 1, 0, 0u);
    if (SENSOR) S.ring = P.snap_ring + (size_t)field * S.depth * S.words;
    const int n1 = (task == REXSIM_TASK_POSES) ? 0 : 100;
    if (SENSOR && n1) sensor_push<ARM>(S, leg, L, AR, true);
    for (int it = 0; it < n1; it++) apply_action_and_step<TERRAIN, ARM, SENSOR, false>(P, sm, L, leg, stand, P.cfg.motor_kp, P.cfg.motor_kd, G, AR, S, true, nullptr);
    const int n2 = (task == REXSIM_TASK_POSES) ? 0 : (int)(0.5 / P.cfg.sim_dt_d);
    for (int it = 0; it < n2; it++) apply_action_and_step<TERRAIN, ARM, SENSOR, false>(P, sm, L, leg, ip, P.cfg.motor_kp, P.cfg.motor_kd, G, AR, S, true, nullptr);
    if (SENSOR) sensor_push<ARM>(S, leg, L, AR, true);
    {
        float* qf = snap_f + (size_t)field * NF; int32_t* qi = snap_i + (size_t)field * NI;
        // snapshot rows are [NF] / [NI] with N = 1; the 8 replicas computed the same thing, the first one stores
        store_lane(qf, qi, 1, 0, leg, L, K, threadIdx.x < 4);
        if (ARM && threadIdx.x == 0) store_arm(qf, qi, 1, 0, AR);
        int err = (int)or4((unsigned)L.err);
        if (threadIdx.x == 0) {
            qf[F_KP] = P.cfg.motor_kp; qf[F_KD] = P.cfg.motor_kd; qf[F_TORIENT] = 0.f; qf[F_IORIENT] = 0.f;
            qi[I_RESETCNT] = 0; qi[I_FIELD] = field; qi[I_HPUSH] = S.push;
            if (err) { P.err[0] |= err; atomicOr(&P.err[P.N], err); }
        }
    }
}

// -------------------------------------------------------------------------------------------------
// host-side launchers (called from rexsim_capi.cu)
//
// Compile units: the file is compiled once per (task, signal) pair with -DREXSIM_UNIT=<k> (k = 0..7, only that
// pair's step kernels are instantiated) and once with -DREXSIM_UNIT=100 (reset / settle / get / set kernels and the
// dispatcher); rex_gym_b200/build.py runs the units in parallel.  Without REXSIM_UNIT everything is one unit.
// -------------------------------------------------------------------------------------------------
// unit k holds the step kernels of the (task, signal) pair c_units[k]: walk, gallop, turn with either signal, then standup, poses
struct StepUnit { int task, signal; };
constexpr StepUnit c_units[8] = {{REXSIM_TASK_WALK, REXSIM_SIGNAL_IK}, {REXSIM_TASK_WALK, REXSIM_SIGNAL_OL},
                                 {REXSIM_TASK_GALLOP, REXSIM_SIGNAL_IK}, {REXSIM_TASK_GALLOP, REXSIM_SIGNAL_OL},
                                 {REXSIM_TASK_TURN, REXSIM_SIGNAL_IK}, {REXSIM_TASK_TURN, REXSIM_SIGNAL_OL},
                                 {REXSIM_TASK_STANDUP, REXSIM_SIGNAL_OL}, {REXSIM_TASK_POSES, REXSIM_SIGNAL_IK}};
// the unit launch_step takes for a (task, signal) pair; standup and poses ignore the signal, an unknown task takes unit 6
constexpr int unit_of(int task, int signal) {
    return task == REXSIM_TASK_POSES ? 7 : (task >= 0 && task < REXSIM_TASK_STANDUP) ? 2 * task + (signal != REXSIM_SIGNAL_IK) : 6;
}
constexpr bool unit_of_inverts_c_units(int u = 0) {
    return u == 8 || (unit_of(c_units[u].task, c_units[u].signal) == u && unit_of_inverts_c_units(u + 1));
}
static_assert(unit_of_inverts_c_units(), "unit_of must map every (task, signal) of c_units to its own unit");
template <int U> cudaError_t launch_step_unit(const Params& P, cudaStream_t st);
#if !defined(REXSIM_UNIT) || REXSIM_UNIT < 100
template <int TASK, int SIGNAL, int TERRAIN, int OCC, bool ARM, bool SENSOR, int BLOCK>
static cudaError_t launch_step_variant(const Params& P, cudaStream_t st) {
    auto kern = step_kernel<TASK, SIGNAL, TERRAIN, OCC, ARM, SENSOR, BLOCK>;
    const int blocks = (P.N * 4 + BLOCK - 1) / BLOCK;
    const size_t smem = ((TERRAIN == REXSIM_TERRAIN_RANDOM ? (size_t)(BLOCK / 4) * TILE_FLOATS : 0) +
                         (pgs_replicated(OCC, ARM, TERRAIN) ? (size_t)(BLOCK / 4) * PGS_ENV_FLOATS : 0)) * sizeof(float);
    if (smem > 48 * 1024) {        // opt in once per kernel (the attribute is sticky)
        static bool done = false;
        if (!done) {
            cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return e;
            done = true;
        }
    }
    kern<<<blocks, BLOCK, smem, st>>>(P);
    if (P.launched) { P.launched[0] = BLOCK; P.launched[1] = OCC; P.launched[2] = SENSOR; }
    return cudaGetLastError();
}
template <int TASK, int SIGNAL, int TERRAIN, bool ARM>
static cudaError_t launch_step_tsta(const Params& P, cudaStream_t st) {
    // sensor model compiled in: one (255-register) build per terrain
    if (P.sensor_on) return launch_step_variant<TASK, SIGNAL, TERRAIN, 1, ARM, true, REXSIM_BLOCK>(P, st);
    // Beyond one wave of 2-CTA/SM residency (128-thread CTAs; two waves on heightfields): the 128-register build (16 warps/SM
    // hide the serial ABA / PGS chains) in larger CTAs; below that the 255-register build, lowest single-wave latency
    // (DESIGN.md section 5).  Arm batches stay on the 255-register build: at 128 registers the arm's working set spills 4 KB.
    bool big = !ARM && (P.N * 4 + 127) / 128 > (TERRAIN == REXSIM_TERRAIN_PLANE ? 2 : 4) * P.sm_count;
    if (const char* f = getenv("REXSIM_FORCE_BUILD")) big = !ARM && f[0] == 'b';      // developer A/B: "big" / "small"
    if (big) return launch_step_variant<TASK, SIGNAL, TERRAIN, ARM ? 1 : REXSIM_OCC_BIG, ARM, false, ARM ? REXSIM_BLOCK : REXSIM_BLOCK_BIG>(P, st);
    return launch_step_variant<TASK, SIGNAL, TERRAIN, 1, ARM, false, REXSIM_BLOCK>(P, st);
}
template <int TASK, int SIGNAL, bool ARM>
static cudaError_t launch_step_tsa(const Params& P, cudaStream_t st) {
    if (P.cfg.terrain == REXSIM_TERRAIN_PLANE) return launch_step_tsta<TASK, SIGNAL, REXSIM_TERRAIN_PLANE, ARM>(P, st);
    return launch_step_tsta<TASK, SIGNAL, REXSIM_TERRAIN_RANDOM, ARM>(P, st);
}
template <int TASK, int SIGNAL>
static cudaError_t launch_step_ts(const Params& P, cudaStream_t st) {
    // the arm (mark='arm') is built for the standup task (BASELINE config 5) and the walk-ik task
    constexpr bool HAS_ARM = (TASK == REXSIM_TASK_STANDUP || (TASK == REXSIM_TASK_WALK && SIGNAL == REXSIM_SIGNAL_IK));
    if (P.cfg.num_motors == 18) {
        if (HAS_ARM) return launch_step_tsa<TASK, SIGNAL, HAS_ARM>(P, st);
        return cudaErrorNotSupported;
    }
    return launch_step_tsa<TASK, SIGNAL, false>(P, st);
}
template <int U>
cudaError_t launch_step_unit(const Params& P, cudaStream_t st) { return launch_step_ts<c_units[U].task, c_units[U].signal>(P, st); }
#ifdef REXSIM_UNIT
template cudaError_t launch_step_unit<REXSIM_UNIT>(const Params&, cudaStream_t);
#endif
#endif

#if !defined(REXSIM_UNIT) || REXSIM_UNIT == 100
// -------------------------------------------------------------------------------------------------
// get / set physical state
// -------------------------------------------------------------------------------------------------
__global__ void get_state_kernel(const Params P, float* out_f, int32_t* out_i) {
    int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= P.N) return;
    const size_t N = P.N;
    const int nm = P.cfg.num_motors;
    for (int w = 0; w < 13; w++) out_f[w * N + env] = P.sf[w * N + env];
    for (int j = 0; j < nm; j++) {
        out_f[(13 + j) * N + env] = P.sf[(j < 12 ? F_Q + j : F_AQ + j - 12) * N + env];
        out_f[(13 + nm + j) * N + env] = P.sf[(j < 12 ? F_QD + j : F_AQD + j - 12) * N + env];
    }
    out_i[0 * N + env] = P.si[I_STEP * N + env];
    out_i[1 * N + env] = P.si[I_ENVSTEP * N + env];
    out_i[2 * N + env] = P.si[I_FLAGS * N + env];
    out_i[3 * N + env] = P.si[I_CONTACT * N + env];
}
__global__ void set_state_kernel(const Params P, const float* in_f) {
    int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= P.N) return;
    const size_t N = P.N;
    const int nm = P.cfg.num_motors;
    for (int w = 0; w < 13; w++) P.sf[w * N + env] = in_f[w * N + env];
    for (int j = 0; j < nm; j++) {
        P.sf[(j < 12 ? F_Q + j : F_AQ + j - 12) * N + env] = in_f[(13 + j) * N + env];
        P.sf[(j < 12 ? F_QD + j : F_AQD + j - 12) * N + env] = in_f[(13 + nm + j) * N + env];
    }
}

// ---- warp re-grouping: counting sort of the envs by solver cost, most expensive first (they start first: LPT order) ----
__global__ void rebalance_hist_kernel(const int32_t* __restrict__ cost, int n, int32_t* __restrict__ hist) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n) atomicAdd(&hist[255 - min(cost[e] >> 1, 255)], 1);
}
__global__ void rebalance_scan_kernel(int32_t* hist) {          // 1 block, 256 threads: exclusive prefix sum in place
    __shared__ int32_t s[256];
    const int t = threadIdx.x;
    s[t] = hist[t];
    __syncthreads();
    for (int o = 1; o < 256; o <<= 1) { int v = t >= o ? s[t - o] : 0; __syncthreads(); s[t] += v; __syncthreads(); }
    hist[t] = s[t] - hist[t];
}
__global__ void rebalance_scatter_kernel(const int32_t* __restrict__ cost, int n, int32_t* __restrict__ offs, int32_t* __restrict__ perm) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n) perm[atomicAdd(&offs[255 - min(cost[e] >> 1, 255)], 1)] = e;
}
cudaError_t launch_rebalance(const int32_t* cost, int n, int32_t* hist, int32_t* perm, cudaStream_t st) {
    cudaError_t e = cudaMemsetAsync(hist, 0, 256 * sizeof(int32_t), st);
    if (e != cudaSuccess) return e;
    rebalance_hist_kernel<<<(n + 255) / 256, 256, 0, st>>>(cost, n, hist);
    rebalance_scan_kernel<<<1, 256, 0, st>>>(hist);
    rebalance_scatter_kernel<<<(n + 255) / 256, 256, 0, st>>>(cost, n, hist, perm);
    return cudaGetLastError();
}

cudaError_t launch_step(const Params& P, cudaStream_t st) {
    static constexpr cudaError_t (*units[])(const Params&, cudaStream_t) = {
        launch_step_unit<0>, launch_step_unit<1>, launch_step_unit<2>, launch_step_unit<3>,
        launch_step_unit<4>, launch_step_unit<5>, launch_step_unit<6>, launch_step_unit<7>};
    return units[unit_of(P.cfg.task, P.cfg.signal)](P, st);
}
cudaError_t launch_reset(const Params& P, float* obs_out, cudaStream_t st) {
    int k = P.reset_idx ? P.reset_k : P.N;
    if (k <= 0) return cudaSuccess;
    int threads = 128, blocks = (k * 4 + threads - 1) / threads;
    const bool arm = P.cfg.num_motors == 18;
    if (P.cfg.task == REXSIM_TASK_GALLOP) reset_kernel<REXSIM_TASK_GALLOP, false><<<blocks, threads, 0, st>>>(P, obs_out);
    else if (arm) reset_kernel<REXSIM_TASK_WALK, true><<<blocks, threads, 0, st>>>(P, obs_out);
    else reset_kernel<REXSIM_TASK_WALK, false><<<blocks, threads, 0, st>>>(P, obs_out);
    return cudaGetLastError();
}
template <int TERRAIN, bool ARM>
static void launch_settle_ta(const Params& P, float* snap_f, int32_t* snap_i, cudaStream_t st) {
    if (P.sensor_on) settle_kernel<TERRAIN, ARM, true><<<1, 32, 0, st>>>(P, snap_f, snap_i, P.cfg.signal, P.cfg.task);
    else settle_kernel<TERRAIN, ARM, false><<<1, 32, 0, st>>>(P, snap_f, snap_i, P.cfg.signal, P.cfg.task);
}
cudaError_t launch_settle(const Params& P, float* snap_f, int32_t* snap_i, cudaStream_t st) {
    const bool arm = P.cfg.num_motors == 18;
    if (P.cfg.terrain == REXSIM_TERRAIN_PLANE) {
        if (arm) launch_settle_ta<REXSIM_TERRAIN_PLANE, true>(P, snap_f, snap_i, st);
        else launch_settle_ta<REXSIM_TERRAIN_PLANE, false>(P, snap_f, snap_i, st);
    } else {
        if (arm) launch_settle_ta<REXSIM_TERRAIN_RANDOM, true>(P, snap_f, snap_i, st);
        else launch_settle_ta<REXSIM_TERRAIN_RANDOM, false>(P, snap_f, snap_i, st);
    }
    return cudaGetLastError();
}
cudaError_t launch_get_state(const Params& P, float* out_f, int32_t* out_i, cudaStream_t st) {
    get_state_kernel<<<(P.N + 127) / 128, 128, 0, st>>>(P, out_f, out_i);
    return cudaGetLastError();
}
cudaError_t launch_set_state(const Params& P, const float* in_f, cudaStream_t st) {
    set_state_kernel<<<(P.N + 127) / 128, 128, 0, st>>>(P, in_f);
    return cudaGetLastError();
}

#endif  // unit 100

}  // namespace rexsim

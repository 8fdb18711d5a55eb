// rexsim_arm.cuh -- the 6-joint arm of mark='arm' (rex_gym/util/pybullet_data/assets/urdf/rex_arm.urdf:611-790,
// rex_gym/model/mark_constants.py:9-12): a fifth limb hanging off the base, owned by lane 0 of the env.
//
// The arm is one serial chain with general joint frames (URDF rpy rotations, +-z axes), so unlike the legs it is
// written as loops over joints with its working set in local memory.  It joins the 4-lane scheme exactly like a
// leg: its articulated inertia / bias reduce onto the base before the base solve, its joints are driven by the
// motor model holding ARM_POSES['rest'] (rex_gym/model/rex_constants.py:3-8, rex_gym/envs/rex_gym_env.py:363-367),
// and its joint-limit rows (rest = -1.6 / 1.6 rad lies outside the +-1.5 rad URDF limits, so three of them are
// active all the time) enter the Gauss-Seidel sweep of the generic solver path.
#pragma once
#include "rexsim_kernel.cuh"

namespace rexsim {

#define ARM_NJ 6
#define ARM_KA 3          // arm joint-limit rows the fast solver path carries (the rest pose violates exactly three: joints 0, 1, 4)
// model-table layout of one arm body (REXSIM_MT_ARM + 32*j): jpos[3] jrot[9] axis[3] mass com[3] inertia[6] lower upper
// npts start reach: its collision points are [start, start + npts) of the point block at REXSIM_MT_ARMPTS, at most reach from
// the body origin
#define ARM_STRIDE 32

struct Arm {
    float q[ARM_NJ], qd[ARM_NJ], tau_obs[ARM_NJ];
    uint32_t ovh[2];          // 6 x 10-bit overheat counters
    uint32_t enabled;         // 6 bits
    // per sub-step working set
    float S[ARM_NJ][6], U[ARM_NJ][6], cJ[ARM_NJ][6], k[ARM_NJ], u[ARM_NJ], qs[ARM_NJ];
    float R[ARM_NJ][9], p[ARM_NJ][3];     // body orientation (columns) and origin relative to the base position
};

__device__ __forceinline__ SV ld6(const float* p) { SV r; r.a = mk(p[0], p[1], p[2]); r.l = mk(p[3], p[4], p[5]); return r; }
__device__ __forceinline__ void st6(float* p, SV v) { p[0] = v.a.x; p[1] = v.a.y; p[2] = v.a.z; p[3] = v.l.x; p[4] = v.l.y; p[5] = v.l.z; }
__device__ __forceinline__ M3 mulM(const M3& A, const M3& B) { M3 r; r.c0 = mul(A, B.c0); r.c1 = mul(A, B.c1); r.c2 = mul(A, B.c2); return r; }
__device__ __forceinline__ M3 axis_angle(V3 a, float q) {   // Rodrigues, columns
    float s, c; sincosf(q, &s, &c); float t = 1.f - c;
    M3 R;
    R.c0 = mk(t * a.x * a.x + c, t * a.x * a.y + s * a.z, t * a.x * a.z - s * a.y);
    R.c1 = mk(t * a.x * a.y - s * a.z, t * a.y * a.y + c, t * a.y * a.z + s * a.x);
    R.c2 = mk(t * a.x * a.z + s * a.y, t * a.y * a.z - s * a.x, t * a.z * a.z + c);
    return R;
}

// ABA passes 1 and 2 over the arm: kinematics, bias terms, inward reduction.  Returns the arm's articulated inertia and
// bias force as seen by the base (to be added to the base sums), fills A.S/U/k/u/cJ.
static __device__ __noinline__ void arm_inward(const float* __restrict__ AT, const M3& R0, SV v0, Arm& A, const float* tauA,
                                        AI& IaOut, SV& paOut, float kdamp) {
    AI IAb[ARM_NJ]; SV pAb[ARM_NJ];
    M3 Rp = R0; V3 pp = mk(0.f, 0.f, 0.f); SV vp = v0;
    const float gz = -10.0f;
#pragma unroll 1
    for (int j = 0; j < ARM_NJ; j++) {
        const float* T = AT + ARM_STRIDE * j;
        M3 Jr; Jr.c0 = mk(T[3], T[6], T[9]); Jr.c1 = mk(T[4], T[7], T[10]); Jr.c2 = mk(T[5], T[8], T[11]);   // row-major -> columns
        V3 ax = mk(T[12], T[13], T[14]);
        M3 Rj = mulM(mulM(Rp, Jr), axis_angle(ax, A.q[j]));
        V3 pj = pp + mul(Rp, mk(T[0], T[1], T[2]));
        SV S; S.a = mul(Rj, ax); S.l = cross(pj, S.a);
        SV vj = A.qd[j] * S;
        SV v = vp + vj;
        SV cJ = crm(v, vj);
        float m = T[15]; V3 cw = pj + mul(Rj, mk(T[16], T[17], T[18]));
        S3 Ib = {T[19], T[20], T[21], T[22], T[23], T[24]};
        const S3 Iw = rotate_inertia(Rj, Ib);
        AI I = rigid_inertia(m, cw, Iw);
        SV pA = crf(v, mul(I, v));
        pA.a = pA.a - mk(cw.y * m * gz, -cw.x * m * gz, 0.f); pA.l.z -= m * gz;
        {   // link damping (same term as the legs: rexsim_kernel.cu link_damping)
            V3 vo = v.l + cross(v.a, pj);
            float wn = sqrtf(dot(v.a, v.a)), vn = sqrtf(dot(vo, vo));
            V3 f = (m * fmaf(kdamp, vn, kdamp)) * vo;
            pA.a = pA.a + fmaf(kdamp, wn, kdamp) * mul(Iw, v.a) + cross(pj, f);
            pA.l = pA.l + f;
        }
        IAb[j] = I; pAb[j] = pA;
        st6(A.S[j], S); st6(A.cJ[j], cJ);
        A.R[j][0] = Rj.c0.x; A.R[j][1] = Rj.c0.y; A.R[j][2] = Rj.c0.z; A.R[j][3] = Rj.c1.x; A.R[j][4] = Rj.c1.y;
        A.R[j][5] = Rj.c1.z; A.R[j][6] = Rj.c2.x; A.R[j][7] = Rj.c2.y; A.R[j][8] = Rj.c2.z;
        A.p[j][0] = pj.x; A.p[j][1] = pj.y; A.p[j][2] = pj.z;
        Rp = Rj; pp = pj; vp = v;
    }
#pragma unroll 1
    for (int j = ARM_NJ - 1; j >= 0; j--) {
        SV S = ld6(A.S[j]);
        AI I = IAb[j]; SV pA = pAb[j];
        SV U = mul(I, S); float k = 1.0f / sdot(S, U); float u = tauA[j] - sdot(S, pA);
        rank1_sub(I, U, k);
        pA = sfma(u * k, U, pA + mul(I, ld6(A.cJ[j])));
        st6(A.U[j], U); A.k[j] = k; A.u[j] = u;
        if (j > 0) { add(IAb[j - 1], I); pAb[j - 1] = pAb[j - 1] + pA; }
        else { IaOut = I; paOut = pA; }
    }
}
// ABA pass 3: joint accelerations -> unconstrained joint rates A.qs
static __device__ __noinline__ void arm_outward(Arm& A, SV a0, float dt, float vmax) {
    SV a = a0;
#pragma unroll 1
    for (int j = 0; j < ARM_NJ; j++) {
        a = a + ld6(A.cJ[j]);
        float qdd = (A.u[j] - sdot(ld6(A.U[j]), a)) * A.k[j];
        a = sfma(qdd, ld6(A.S[j]), a);
        A.qs[j] = fminf(fmaxf(fmaf(dt, qdd, A.qd[j]), -vmax), vmax);
    }
}
// response of the arm joints to a base velocity change b plus accumulated joint impulses us[] (fixed-base part)
static __device__ __noinline__ void arm_apply(Arm& A, SV b, const float* us, float* dq) {
#pragma unroll 1
    for (int j = 0; j < ARM_NJ; j++) {
        dq[j] = (us[j] - sdot(ld6(A.U[j]), b)) * A.k[j];
        b = sfma(dq[j], ld6(A.S[j]), b);
    }
}
// one joint-limit row of the arm (unit generalized force sg on joint jl): base bias g, fixed-base joint response ee[],
// inward joint terms uu[]
static __device__ __noinline__ void arm_row(const Arm& A, int jl, float sg, SV& g, float* ee, float* uu) {
    SV pD; pD.a = mk(0, 0, 0); pD.l = mk(0, 0, 0);
#pragma unroll 1
    for (int j = ARM_NJ - 1; j >= 0; j--) {
        float ud = (j == jl ? sg : 0.f) - ((j < jl) ? sdot(ld6(A.S[j]), pD) : 0.f);
        if (j > jl) ud = 0.f;
        uu[j] = ud;
        if (j <= jl) pD = sfma(ud * A.k[j], ld6(A.U[j]), pD);
    }
    g = pD;
    SV w; w.a = mk(0, 0, 0); w.l = mk(0, 0, 0);
#pragma unroll 1
    for (int j = 0; j < ARM_NJ; j++) {
        float e = (uu[j] - sdot(ld6(A.U[j]), w)) * A.k[j];
        ee[j] = e;
        w = sfma(e, ld6(A.S[j]), w);
    }
}
// one contact row on arm body jb (unit spatial force F about the base position): joint Jacobian jq[] (S_j . F for the joints
// j <= jb that carry the body, 0 beyond), base bias g, fixed-base joint response ee[], inward joint terms uu[]
static __device__ __noinline__ void arm_force_row(const Arm& A, int jb, SV F, SV& g, float* jq, float* ee, float* uu) {
    SV pD; pD.a = mk(0, 0, 0); pD.l = mk(0, 0, 0);
#pragma unroll 1
    for (int j = ARM_NJ - 1; j >= 0; j--) {
        const SV S = ld6(A.S[j]);
        jq[j] = j <= jb ? sdot(S, F) : 0.f;
        float ud = j <= jb ? jq[j] - sdot(S, pD) : 0.f;
        uu[j] = ud;
        if (j <= jb) pD = sfma(ud * A.k[j], ld6(A.U[j]), pD);
    }
    g = pD - F;
    SV w; w.a = mk(0, 0, 0); w.l = mk(0, 0, 0);
#pragma unroll 1
    for (int j = 0; j < ARM_NJ; j++) {
        float e = (uu[j] - sdot(ld6(A.U[j]), w)) * A.k[j];
        ee[j] = e;
        w = sfma(e, ld6(A.S[j]), w);
    }
}

}  // namespace rexsim

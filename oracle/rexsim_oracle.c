/* rexsim_oracle.c -- CPU ORACLE (test infrastructure, NOT the product path).  See rexsim_oracle.h.
 *
 * Every function cites the reference file:line it restates (paths relative to the reference
 * repository root).  Physics follows Bullet's btMultiBody pipeline as *called by* the reference
 * (pybullet==2.8.3 is a pip dependency, requirements.txt:2, source not vendored): parity there is
 * UNPINNED and anchored on the reference's call sites (rex_gym/model/rex.py:161,326-330;
 * rex_gym/envs/rex_gym_env.py:234,306-314).
 */
#include "rexsim_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>

#define PI 3.14159265358979323846

/* ------------------------------------------------------------------------------------------- */
/* small linear algebra                                                                         */
/* ------------------------------------------------------------------------------------------- */
static void v3cross(const real* a, const real* b, real* o) {
    real x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
    o[0] = x; o[1] = y; o[2] = z;
}
static real v3dot(const real* a, const real* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static void m3v(const real* M, const real* v, real* o) {
    real x = M[0] * v[0] + M[1] * v[1] + M[2] * v[2];
    real y = M[3] * v[0] + M[4] * v[1] + M[5] * v[2];
    real z = M[6] * v[0] + M[7] * v[1] + M[8] * v[2];
    o[0] = x; o[1] = y; o[2] = z;
}
static void m3tv(const real* M, const real* v, real* o) {
    real x = M[0] * v[0] + M[3] * v[1] + M[6] * v[2];
    real y = M[1] * v[0] + M[4] * v[1] + M[7] * v[2];
    real z = M[2] * v[0] + M[5] * v[1] + M[8] * v[2];
    o[0] = x; o[1] = y; o[2] = z;
}
static void m3m(const real* A, const real* B, real* O) {
    real T[9];
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++)
        T[3 * i + j] = A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
    memcpy(O, T, sizeof(T));
}
static void m3t(const real* A, real* O) {
    real T[9] = {A[0], A[3], A[6], A[1], A[4], A[7], A[2], A[5], A[8]};
    memcpy(O, T, sizeof(T));
}
static void skew(const real* r, real* S) {
    S[0] = 0; S[1] = -r[2]; S[2] = r[1];
    S[3] = r[2]; S[4] = 0; S[5] = -r[0];
    S[6] = -r[1]; S[7] = r[0]; S[8] = 0;
}
/* rotation about unit axis a by angle q (Rodrigues), maps child coords -> parent coords */
static void axis_angle(const real* a, real q, real* R) {
    real c = cos(q), s = sin(q), t = 1 - c;
    R[0] = t * a[0] * a[0] + c;        R[1] = t * a[0] * a[1] - s * a[2]; R[2] = t * a[0] * a[2] + s * a[1];
    R[3] = t * a[0] * a[1] + s * a[2]; R[4] = t * a[1] * a[1] + c;        R[5] = t * a[1] * a[2] - s * a[0];
    R[6] = t * a[0] * a[2] - s * a[1]; R[7] = t * a[1] * a[2] + s * a[0]; R[8] = t * a[2] * a[2] + c;
}
/* quaternion (x,y,z,w) -> rotation matrix; btMatrix3x3::setRotation (pybullet.getMatrixFromQuaternion,
 * call sites rex_gym/envs/rex_gym_env.py:486,531) */
static void quat_to_mat(const real* q, real* R) {
    real d = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    real s = 2.0 / d;
    real xs = q[0] * s, ys = q[1] * s, zs = q[2] * s;
    real wx = q[3] * xs, wy = q[3] * ys, wz = q[3] * zs;
    real xx = q[0] * xs, xy = q[0] * ys, xz = q[0] * zs;
    real yy = q[1] * ys, yz = q[1] * zs, zz = q[2] * zs;
    R[0] = 1 - (yy + zz); R[1] = xy - wz;       R[2] = xz + wy;
    R[3] = xy + wz;       R[4] = 1 - (xx + zz); R[5] = yz - wx;
    R[6] = xz - wy;       R[7] = yz + wx;       R[8] = 1 - (xx + yy);
}
/* pybullet.getEulerFromQuaternion (ZYX), call sites rex_gym/model/rex.py:426,439 */
static void quat_to_euler(const real* q, real* rpy) {
    real sqx = q[0] * q[0], sqy = q[1] * q[1], sqz = q[2] * q[2], squ = q[3] * q[3];
    real sarg = -2.0 * (q[0] * q[2] - q[3] * q[1]);
    if (sarg <= -0.99999) { rpy[0] = 0; rpy[1] = -0.5 * PI; rpy[2] = 2 * atan2(q[0], -q[1]); }
    else if (sarg >= 0.99999) { rpy[0] = 0; rpy[1] = 0.5 * PI; rpy[2] = 2 * atan2(-q[0], q[1]); }
    else {
        rpy[0] = atan2(2 * (q[1] * q[2] + q[3] * q[0]), squ - sqx - sqy + sqz);
        rpy[1] = asin(sarg);
        rpy[2] = atan2(2 * (q[0] * q[1] + q[3] * q[2]), squ + sqx - sqy - sqz);
    }
}
/* pybullet.getQuaternionFromEuler (rex_gym/envs/gym/turn_env.py:158) */
static void euler_to_quat(const real* rpy, real* q) {
    real hr = rpy[0] * 0.5, hp = rpy[1] * 0.5, hy = rpy[2] * 0.5;
    real cr = cos(hr), sr = sin(hr), cp = cos(hp), sp = sin(hp), cy = cos(hy), sy = sin(hy);
    q[0] = sr * cp * cy - cr * sp * sy;
    q[1] = cr * sp * cy + sr * cp * sy;
    q[2] = cr * cp * sy - sr * sp * cy;
    q[3] = cr * cp * cy + sr * sp * sy;
}

/* 6-vectors: [angular(3); linear(3)];  6x6 row-major */
static void m6v(const real* M, const real* v, real* o) {
    real t[6];
    for (int i = 0; i < 6; i++) { real s = 0; for (int j = 0; j < 6; j++) s += M[6 * i + j] * v[j]; t[i] = s; }
    memcpy(o, t, sizeof(t));
}
static void m6tv(const real* M, const real* v, real* o) {
    real t[6];
    for (int i = 0; i < 6; i++) { real s = 0; for (int j = 0; j < 6; j++) s += M[6 * j + i] * v[j]; t[i] = s; }
    memcpy(o, t, sizeof(t));
}
static real v6dot(const real* a, const real* b) { real s = 0; for (int i = 0; i < 6; i++) s += a[i] * b[i]; return s; }
/* spatial motion cross product  v x m */
static void crm(const real* v, const real* m, real* o) {
    real a[3], b[3], c[3];
    v3cross(v, m, a); v3cross(v, m + 3, b); v3cross(v + 3, m, c);
    o[0] = a[0]; o[1] = a[1]; o[2] = a[2];
    o[3] = b[0] + c[0]; o[4] = b[1] + c[1]; o[5] = b[2] + c[2];
}
/* spatial force cross product  v x* f */
static void crf(const real* v, const real* f, real* o) {
    real a[3], b[3], c[3];
    v3cross(v, f, a); v3cross(v + 3, f + 3, b); v3cross(v, f + 3, c);
    o[0] = a[0] + b[0]; o[1] = a[1] + b[1]; o[2] = a[2] + b[2];
    o[3] = c[0]; o[4] = c[1]; o[5] = c[2];
}
/* Pluecker motion transform parent->child: X = [E 0; -E rx, E] */
static void make_X(const real* E, const real* r, real* X) {
    real rx[9], Erx[9];
    skew(r, rx); m3m(E, rx, Erx);
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
        X[6 * i + j] = E[3 * i + j]; X[6 * i + 3 + j] = 0;
        X[6 * (i + 3) + j] = -Erx[3 * i + j]; X[6 * (i + 3) + 3 + j] = E[3 * i + j];
    }
}
/* O += X^T A X */
static void add_XtAX(const real* X, const real* A, real* O) {
    real T[36];
    for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) {
        real s = 0; for (int k = 0; k < 6; k++) s += A[6 * i + k] * X[6 * k + j]; T[6 * i + j] = s;
    }
    for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) {
        real s = 0; for (int k = 0; k < 6; k++) s += X[6 * k + i] * T[6 * k + j]; O[6 * i + j] += s;
    }
}
/* solve A x = b for SPD 6x6 (Gaussian elimination with partial pivoting on a copy) */
static void solve6(const real* A, const real* b, real* x) {
    real M[6][7];
    for (int i = 0; i < 6; i++) { for (int j = 0; j < 6; j++) M[i][j] = A[6 * i + j]; M[i][6] = b[i]; }
    for (int c = 0; c < 6; c++) {
        int p = c; for (int r = c + 1; r < 6; r++) if (fabs(M[r][c]) > fabs(M[p][c])) p = r;
        if (p != c) for (int j = 0; j < 7; j++) { real t = M[c][j]; M[c][j] = M[p][j]; M[p][j] = t; }
        for (int r = c + 1; r < 6; r++) { real f = M[r][c] / M[c][c]; for (int j = c; j < 7; j++) M[r][j] -= f * M[c][j]; }
    }
    for (int i = 5; i >= 0; i--) { real s = M[i][6]; for (int j = i + 1; j < 6; j++) s -= M[i][j] * x[j]; x[i] = s / M[i][i]; }
}

/* ------------------------------------------------------------------------------------------- */
/* simulator object                                                                             */
/* ------------------------------------------------------------------------------------------- */
struct Hist;
struct RexoSim {
    RexoModel m;
    RexoConfig c;
    RexoEnv* env;
    RexoEnv* snapshot;      /* settled state per field (or 1 for plane) */
    int nsnap;
    int obs_dim, act_dim;
    double init_pose[REXO_MAXDOF];   /* task init pose incl. arm rest */
    double stand_pose[REXO_MAXDOF];  /* Rex.initial_pose = INIT_POSES['stand'] (+arm rest) */
    double* field_zoff;              /* [nfields]: (hmin+hmax)/2 per field */
    /* sensor history: one ring per env, then one per reset snapshot; ctrl = the control observation of the last ReceiveObservation */
    struct Hist* hist;
    double (*ctrl)[REXO_OBSW];
    int sensor_on;                    /* any latency or noise configured */
};
typedef struct Hist { int len, head; double buf[REXO_HIST][REXO_OBSW]; } Hist;

/* per-sub-step scratch (kinematics + ABA caches) */
typedef struct {
    real Rw[REXO_MAXB][9];     /* body->world rotation */
    real pw[REXO_MAXB][3];     /* body origin in world */
    real Xup[REXO_MAXB][36];   /* parent->child motion transform */
    real S[REXO_MAXB][6];
    real v[REXO_MAXB][6], cJ[REXO_MAXB][6];
    real IA[REXO_MAXB][36], pA[REXO_MAXB][6];
    real U[REXO_MAXB][6], d[REXO_MAXB], u[REXO_MAXB];
    real a[REXO_MAXB][6];
} Scratch;

/* rex_gym/model/rex_constants.py:3-47 (values are data, restated) */
static const double POSE_STAND[12] = {0., -0.88643435, 1.30197369, 0., -0.88643435, 1.30197369,
                                      0., -0.88643435, 1.30197369, 0., -0.88643435, 1.30197369};
static const double POSE_STAND_OL[12] = {0.15192765, -0.90412283, 1.48156545, -0.15192765, -0.90412283, 1.48156545,
                                         0.15192765, -0.90412283, 1.48156545, -0.15192765, -0.90412283, 1.48156545};
static const double POSE_REST[12] = {-0.4, -1.5, 6, 0.4, -1.5, 6, -0.4, -1.5, 6, 0.4, -1.5, 6};
static const double ARM_REST[6] = {-1.6, -1.6, 0., 0., 1.6, 0.};

/* ------------------------------------------------------------------------------------------- */
/* counter-based RNG shared bit-exactly with the CUDA path (replaces Python's unseeded `random`  */
/* in walk_env.py:133-147, gallop_env.py:151, turn_env.py:138,147)                               */
/* ------------------------------------------------------------------------------------------- */
uint32_t rexo_rand_u32(uint64_t seed, uint32_t env, uint32_t reset_count, uint32_t slot) {
    uint64_t z = seed + 0x9E3779B97F4A7C15ull * ((uint64_t)env + 1);
    z ^= ((uint64_t)reset_count << 32) | (uint64_t)slot;
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z = z ^ (z >> 31);
    return (uint32_t)(z >> 32);
}
static double rand_uniform(const RexoSim* s, int env, uint32_t rc, uint32_t slot, double a, double b) {
    double u = (double)(rexo_rand_u32(s->c.seed, (uint32_t)env + (uint32_t)s->c.env_offset, rc, slot) >> 8) * (1.0 / 16777216.0);
    return a + (b - a) * u;   /* random.uniform(a,b) = a + (b-a)*random() */
}

/* ------------------------------------------------------------------------------------------- */
/* motor model: rex_gym/model/motor.py:76-143                                                   */
/* ------------------------------------------------------------------------------------------- */
static const double CUR_TAB[7] = {0, 10, 20, 30, 40, 50, 60};
static const double TRQ_TAB[7] = {0, 1, 1.9, 2.45, 3.0, 3.25, 3.5};
static double np_interp(double x) {
    if (x <= CUR_TAB[0]) return TRQ_TAB[0];
    if (x >= CUR_TAB[6]) return TRQ_TAB[6];
    int j = 0; while (j < 5 && x >= CUR_TAB[j + 1]) j++;
    double slope = (TRQ_TAB[j + 1] - TRQ_TAB[j]) / (CUR_TAB[j + 1] - CUR_TAB[j]);
    return slope * (x - CUR_TAB[j]) + TRQ_TAB[j];
}
static double clipd(double x, double lo, double hi) { return x < lo ? lo : (x > hi ? hi : x); }
void rexo_motor_torque(int n, const double* cmd, const double* q, const double* qd, const double* qd_true,
                       const double* kp, const double* kd, double* tau_act, double* tau_obs) {
    const double V = 32.0, R = 0.186, Kt = 0.0954, visc = 0.0;    /* motor.py:6-13 */
    for (int i = 0; i < n; i++) {
        double pwm = -1 * kp[i] * (q[i] - cmd[i]) - kd[i] * qd[i];           /* motor.py:111 */
        pwm = clipd(pwm, -1.0, 1.0);                                         /* motor.py:113 */
        tau_obs[i] = clipd(Kt * (pwm * V / R), -5.7, 5.7);                   /* motor.py:127-129 */
        double vnet = clipd(pwm * V - (Kt + visc) * qd_true[i], -50.0, 50.0);/* motor.py:132-135 */
        double cur = vnet / R;
        double sgn = (cur > 0) - (cur < 0);
        tau_act[i] = sgn * np_interp(fabs(cur)) * 1.0;                       /* motor.py:137-142 */
    }
}

/* ------------------------------------------------------------------------------------------- */
/* gait planner: rex_gym/model/gait_planner.py:22-134                                           */
/* ------------------------------------------------------------------------------------------- */
static double bin_factor(int n, int k) {   /* gait_planner.py:22-24 */
    double f[13]; f[0] = 1; for (int i = 1; i <= 12; i++) f[i] = f[i - 1] * i;
    return f[n] / (f[k] * f[n - k]);
}
void rexo_stance(double phi_st, double v, double angle, double* o) {   /* gait_planner.py:31-40 */
    double c = cos(angle * (PI / 180.0)), s = sin(angle * (PI / 180.0));
    double A = 0.001, half_l = 0.05;
    double p = half_l * (1 - 2 * phi_st);
    o[0] = c * p * fabs(v);
    o[1] = -s * p * fabs(v);
    o[2] = -A * cos(PI / (2 * half_l) * p);
}
void rexo_bezier_swing(double phi, double v, double angle, double direction, double* o) {  /* gait_planner.py:42-58 */
    static const double BX[12] = {-0.04, -0.056, -0.06, -0.06, -0.06, 0., 0., 0., 0.06, 0.06, 0.056, 0.04};
    static const double BZ[12] = {0., 0., 0.0405, 0.0405, 0.0405, 0.0405, 0.0405, 0.0495, 0.0495, 0.0495, 0., 0.};
    double c = cos(angle * (PI / 180.0)), s = sin(angle * (PI / 180.0));
    double sx = 0, sy = 0, sz = 0;
    for (int i = 0; i < 10; i++) {           /* only 10 of the 12 control points (gait_planner.py:53-57) */
        double X = fabs(v) * c * BX[i] * direction;
        double Y = fabs(v) * s * (-X);
        double Z = fabs(v) * BZ[i];
        double b = bin_factor(11, i);
        double tk = pow(phi, (double)i), t1 = pow(1 - phi, (double)(11 - i));
        sx = sx + X * b * tk * t1;
        sy = sy + Y * b * tk * t1;
        sz = sz + Z * b * tk * t1;
    }
    o[0] = sx; o[1] = sy; o[2] = sz;
}
static void step_trajectory(double* alpha, double phi, double v, double angle, double w_rot,
                            const double* c2f, double direction, double* coord) {   /* gait_planner.py:60-94 */
    const double step_offset = 0.5;
    if (phi >= 1) phi = phi - 1.;
    double r = sqrt(c2f[0] * c2f[0] + c2f[1] * c2f[1]);
    double foot_angle = atan2(c2f[1], c2f[0]);
    double circle;
    if (w_rot >= 0.) circle = 90. - (foot_angle - *alpha) * (180.0 / PI);
    else circle = 270. - (foot_angle - *alpha) * (180.0 / PI);
    double L[3], Rr[3];
    if (phi <= step_offset) {
        double ps = phi / step_offset;
        rexo_stance(ps, v, angle, L);
        rexo_stance(ps, w_rot, circle, Rr);
    } else {
        double psw = (phi - step_offset) / (1 - step_offset);
        rexo_bezier_swing(psw, v, angle, direction, L);
        rexo_bezier_swing(psw, w_rot, circle, direction, Rr);
    }
    double mag = atan2(sqrt(Rr[0] * Rr[0] + Rr[1] * Rr[1]), r);
    if (c2f[1] > 0) *alpha = (Rr[0] < 0) ? -mag : mag;
    else *alpha = (Rr[0] < 0) ? mag : -mag;
    coord[0] = L[0] + Rr[0]; coord[1] = L[1] + Rr[1]; coord[2] = L[2] + Rr[2];
}
static const double DEFAULT_FRAMES[12] = {0.115, -0.0925, -0.2, 0.115, 0.0925, -0.2,
                                          -0.115, -0.0925, -0.2, -0.115, 0.0925, -0.2}; /* kinematics.py:10-26 */
/* `now` replaces time.time() (gait_planner.py:108-110): deterministic sim clock, see DESIGN.md F1 */
void rexo_gait_loop(double* phi, double* last_time, double* alpha, int gallop, double now,
                    double v, double angle, double w_rot, double T, double direction,
                    const double* frames_in, double* out) {   /* gait_planner.py:96-134 */
    static const double OFF_WALK[4] = {0., 0.5, 0.5, 0.}, OFF_GALLOP[4] = {0., 0., 0.8, 0.8};
    const double* off = gallop ? OFF_GALLOP : OFF_WALK;
    const double* fr = frames_in ? frames_in : DEFAULT_FRAMES;
    if (T <= 0.01) T = 0.01;
    if (*phi >= 0.99) *last_time = now;
    *phi = (now - *last_time) / T;
    for (int l = 0; l < 4; l++) {   /* FR, FL, RR, RL share alpha serially */
        double c[3];
        step_trajectory(alpha, *phi + off[l], v, angle, w_rot, fr + 3 * l, direction, c);
        out[3 * l] = fr[3 * l] + c[0]; out[3 * l + 1] = fr[3 * l + 1] + c[1]; out[3 * l + 2] = fr[3 * l + 2] + c[2];
    }
}

/* ------------------------------------------------------------------------------------------- */
/* leg IK: rex_gym/model/kinematics.py:49-142                                                   */
/* ------------------------------------------------------------------------------------------- */
static void ik_transform(const double* coord, const double* rpy, const double* pos, double* o) {  /* kinematics.py:49-78 */
    double t[3] = {coord[0] + pos[0], coord[1] + pos[1], coord[2] + pos[2]};   /* translation applied first */
    if (rpy[0] != 0 || rpy[1] != 0 || rpy[2] != 0) {
        double cx = cos(rpy[0]), sx = sin(rpy[0]), cy = cos(rpy[1]), sy = sin(rpy[1]), cz = cos(rpy[2]), sz = sin(rpy[2]);
        /* R = Rx*Ry*Rz */
        double a[3] = {cz * t[0] - sz * t[1], sz * t[0] + cz * t[1], t[2]};          /* Rz */
        double b[3] = {cy * a[0] + sy * a[2], a[1], -sy * a[0] + cy * a[2]};         /* Ry */
        o[0] = b[0]; o[1] = cx * b[1] - sx * b[2]; o[2] = sx * b[1] + cx * b[2];     /* Rx */
    } else { o[0] = t[0]; o[1] = t[1]; o[2] = t[2]; }
}
static void solve_ik_leg(const double* c, int right, double* ang) {   /* kinematics.py:89-102 */
    const double hip = 0.055, leg = 0.10652, foot = 0.145;
    double dom = (c[1] * c[1] + (-c[2]) * (-c[2]) - hip * hip + (-c[0]) * (-c[0]) - leg * leg - foot * foot) / (2 * foot * leg);
    if (dom > 1 || dom < -1) dom = dom > 1 ? 0.99 : -0.99;        /* check_domain :80-87 */
    double gamma = atan2(-sqrt(1 - dom * dom), dom);
    double sq = c[1] * c[1] + (-c[2]) * (-c[2]) - hip * hip;
    if (sq < 0.0) sq = 0.0;
    double alpha = atan2(-c[0], sqrt(sq)) - atan2(foot * sin(gamma), leg + foot * cos(gamma));
    double hv = right ? -hip : hip;
    double theta = -atan2(c[2], c[1]) - atan2(sqrt(sq), hv);
    ang[0] = theta; ang[1] = -alpha; ang[2] = -gamma;
}
void rexo_ik_solve(const double* rpy, const double* pos, const double* frames, double* angles) {  /* kinematics.py:104-142 */
    static const double HIP[12] = {0.115, -0.0375, 0, 0.115, 0.0375, 0, -0.115, -0.0375, 0, -0.115, 0.0375, 0};
    double nrpy[3] = {-rpy[0], -rpy[1], -rpy[2]}, npos[3] = {-pos[0], -pos[1], -pos[2]};
    for (int l = 0; l < 4; l++) {
        double hv[3], c[3], tc[3];
        ik_transform(HIP + 3 * l, rpy, pos, hv);
        for (int k = 0; k < 3; k++) c[k] = frames[3 * l + k] - hv[k];
        ik_transform(c, nrpy, npos, tc);                 /* "inverse" = same map with negated args (:122-127) */
        solve_ik_leg(tc, (l % 2) == 0, angles + 3 * l);  /* FR, RR are right side */
    }
}

/* ------------------------------------------------------------------------------------------- */
/* kinematics + ABA (Featherstone, link frames; Bullet computeAccelerationsArticulatedBody...)  */
/* ------------------------------------------------------------------------------------------- */
static void kinematics(const RexoSim* s, const RexoEnv* e, Scratch* k) {
    const RexoModel* m = &s->m;
    real q0[4] = {e->quat[0], e->quat[1], e->quat[2], e->quat[3]};
    quat_to_mat(q0, k->Rw[0]);
    for (int a = 0; a < 3; a++) k->pw[0][a] = e->pos[a];
    for (int i = 1; i < m->nb; i++) {
        int p = m->parent[i];
        real ax[3] = {m->axis[i][0], m->axis[i][1], m->axis[i][2]};
        real Rj[9], jr[9], Rc2p[9], E[9], r[3];
        axis_angle(ax, e->q[i - 1], Rj);
        for (int a = 0; a < 9; a++) jr[a] = m->jrot[i][a];
        m3m(jr, Rj, Rc2p);                 /* child -> parent */
        m3t(Rc2p, E);                      /* parent -> child */
        for (int a = 0; a < 3; a++) r[a] = m->jpos[i][a];
        make_X(E, r, k->Xup[i]);
        m3m(k->Rw[p], Rc2p, k->Rw[i]);
        real t[3]; m3v(k->Rw[p], r, t);
        for (int a = 0; a < 3; a++) k->pw[i][a] = k->pw[p][a] + t[a];
        for (int a = 0; a < 3; a++) { k->S[i][a] = ax[a]; k->S[i][3 + a] = 0; }
    }
}
static void body_inertia6(const RexoModel* m, int i, real* I6) {
    real c[3] = {m->com[i][0], m->com[i][1], m->com[i][2]}, cx[9], cxT[9], Ic[9], t[9];
    real ms = m->mass[i];
    skew(c, cx); m3t(cx, cxT);
    for (int a = 0; a < 9; a++) Ic[a] = m->inertia[i][a];
    m3m(cx, cxT, t);
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) {
        I6[6 * a + b] = Ic[3 * a + b] + ms * t[3 * a + b];
        I6[6 * a + 3 + b] = ms * cx[3 * a + b];
        I6[6 * (a + 3) + b] = ms * cxT[3 * a + b];
        I6[6 * (a + 3) + 3 + b] = (a == b) ? ms : 0;
    }
}
/* forward dynamics: fills k (articulated inertias etc.), returns generalized accelerations
 * acc[0..2]=world omega-dot, acc[3..5]=world linear accel of base origin, acc[6+j]=joint accel */
static void aba(const RexoSim* s, const RexoEnv* e, Scratch* k, const real* tau, real* acc) {
    const RexoModel* m = &s->m;
    const real g[3] = {0, 0, -10.0};                         /* setGravity(0,0,-10) rex_gym_env.py:314 */
    /* base spatial velocity in base coordinates */
    real ww[3] = {e->angvel[0], e->angvel[1], e->angvel[2]}, vw[3] = {e->linvel[0], e->linvel[1], e->linvel[2]};
    m3tv(k->Rw[0], ww, k->v[0]); m3tv(k->Rw[0], vw, k->v[0] + 3);
    for (int i = 0; i < m->nb; i++) {
        if (i > 0) {
            int p = m->parent[i];
            real vp[6]; m6v(k->Xup[i], k->v[p], vp);
            real vj[6]; for (int a = 0; a < 6; a++) { vj[a] = k->S[i][a] * e->qd[i - 1]; k->v[i][a] = vp[a] + vj[a]; }
            crm(k->v[i], vj, k->cJ[i]);
        }
        body_inertia6(m, i, k->IA[i]);
        real Iv[6]; m6v(k->IA[i], k->v[i], Iv);
        crf(k->v[i], Iv, k->pA[i]);
        /* gravity as an external force at the COM, body coordinates */
        real gb[3], fg[3], ng[3], c[3] = {m->com[i][0], m->com[i][1], m->com[i][2]};
        m3tv(k->Rw[i], g, gb);
        for (int a = 0; a < 3; a++) fg[a] = m->mass[i] * gb[a];
        v3cross(c, fg, ng);
        for (int a = 0; a < 3; a++) { k->pA[i][a] -= ng[a]; k->pA[i][3 + a] -= fg[a]; }
        /* btMultiBody::computeAccelerationsArticulatedBodyAlgorithmMultiDof adds the same damping term to EVERY link
         * (m_linearDamping = m_angularDamping = 0.04, K1 = K2): I w (k + k|w|), m v (k + k|v|) in the link frame.  Fixed
         * children are merged here, so the merged body's mass / inertia at its origin stand in for the separate links.
         * The recorded PyBullet episodes select it: 0.04 on the links lowers the 300-step replay error by 13 %, 0.2 raises it. */
        if (i > 0 && s->c.link_damping > 0) {
            const real kl = s->c.link_damping;
            real* vi = k->v[i];
            real wn = sqrt(v3dot(vi, vi)), vn = sqrt(v3dot(vi + 3, vi + 3));
            real Ib[9], Iw[3]; for (int a = 0; a < 9; a++) Ib[a] = m->inertia[i][a];
            m3v(Ib, vi, Iw);
            for (int a = 0; a < 3; a++) {
                k->pA[i][a] += Iw[a] * (kl + kl * wn);
                k->pA[i][3 + a] += m->mass[i] * vi[3 + a] * (kl + kl * vn);
            }
        }
    }
    /* the base link (un-merged root mass / inertia) */
    {
        const real kd = 0.04;
        real* v0 = k->v[0];
        real wn = sqrt(v3dot(v0, v0)), vn = sqrt(v3dot(v0 + 3, v0 + 3));
        for (int a = 0; a < 3; a++) {
            k->pA[0][a] += s->m.root_inertia[a] * v0[a] * (kd + kd * wn);
            k->pA[0][3 + a] += s->m.root_mass * v0[3 + a] * (kd + kd * vn);
        }
    }
    for (int i = m->nb - 1; i >= 1; i--) {
        int p = m->parent[i];
        m6v(k->IA[i], k->S[i], k->U[i]);
        k->d[i] = v6dot(k->S[i], k->U[i]);
        k->u[i] = tau[i - 1] - v6dot(k->S[i], k->pA[i]);
        real Ia[36], pa[6], Iac[6];
        for (int a = 0; a < 6; a++) for (int b = 0; b < 6; b++) Ia[6 * a + b] = k->IA[i][6 * a + b] - k->U[i][a] * k->U[i][b] / k->d[i];
        m6v(Ia, k->cJ[i], Iac);
        for (int a = 0; a < 6; a++) pa[a] = k->pA[i][a] + Iac[a] + k->U[i][a] * k->u[i] / k->d[i];
        add_XtAX(k->Xup[i], Ia, k->IA[p]);
        real t[6]; m6tv(k->Xup[i], pa, t);
        for (int a = 0; a < 6; a++) k->pA[p][a] += t[a];
    }
    real np[6]; for (int a = 0; a < 6; a++) np[a] = -k->pA[0][a];
    solve6(k->IA[0], np, k->a[0]);
    for (int i = 1; i < m->nb; i++) {
        int p = m->parent[i];
        real ap[6]; m6v(k->Xup[i], k->a[p], ap);
        for (int a = 0; a < 6; a++) ap[a] += k->cJ[i][a];
        real qdd = (k->u[i] - v6dot(k->U[i], ap)) / k->d[i];
        acc[6 + i - 1] = qdd;
        for (int a = 0; a < 6; a++) k->a[i][a] = ap[a] + k->S[i][a] * qdd;
    }
    /* back to world: classical linear acceleration = spatial + omega x v */
    real wxv[3], lin[3];
    v3cross(k->v[0], k->v[0] + 3, wxv);
    for (int a = 0; a < 3; a++) lin[a] = k->a[0][3 + a] + wxv[a];
    m3v(k->Rw[0], k->a[0], acc); m3v(k->Rw[0], lin, acc + 3);
}
/* velocity response to a generalized impulse f (Bullet calcAccelerationDeltasMultiDof) */
static void delta_response(const RexoSim* s, const Scratch* k, const real* f, real* dv) {
    const RexoModel* m = &s->m;
    real pD[REXO_MAXB][6], uD[REXO_MAXB], aD[REXO_MAXB][6];
    memset(pD, 0, sizeof(pD));
    for (int i = m->nb - 1; i >= 1; i--) {
        int p = m->parent[i];
        uD[i] = f[6 + i - 1] - v6dot(k->S[i], pD[i]);
        real pa[6], t[6];
        for (int a = 0; a < 6; a++) pa[a] = pD[i][a] + k->U[i][a] * uD[i] / k->d[i];
        m6tv(k->Xup[i], pa, t);
        for (int a = 0; a < 6; a++) pD[p][a] += t[a];
    }
    real fb[6]; m3tv(k->Rw[0], f, fb); m3tv(k->Rw[0], f + 3, fb + 3);
    real np[6]; for (int a = 0; a < 6; a++) np[a] = -(pD[0][a] - fb[a]);
    solve6(k->IA[0], np, aD[0]);
    for (int i = 1; i < m->nb; i++) {
        int p = m->parent[i];
        real ap[6]; m6v(k->Xup[i], aD[p], ap);
        real dq = (uD[i] - v6dot(k->U[i], ap)) / k->d[i];
        dv[6 + i - 1] = dq;
        for (int a = 0; a < 6; a++) aD[i][a] = ap[a] + k->S[i][a] * dq;
    }
    m3v(k->Rw[0], aD[0], dv); m3v(k->Rw[0], aD[0] + 3, dv + 3);
}
/* generalized Jacobian row of a unit force along n at world point p on body b */
static void contact_jacobian(const RexoSim* s, const Scratch* k, int b, const real* p, const real* n, real* J) {
    const RexoModel* m = &s->m;
    int nd = 6 + m->ndof;
    for (int a = 0; a < nd; a++) J[a] = 0;
    real r[3] = {p[0] - k->pw[0][0], p[1] - k->pw[0][1], p[2] - k->pw[0][2]}, t[3];
    v3cross(r, n, t);
    J[0] = t[0]; J[1] = t[1]; J[2] = t[2]; J[3] = n[0]; J[4] = n[1]; J[5] = n[2];
    for (int i = b; i >= 1; i = m->parent[i]) {
        real aw[3], ax[3] = {m->axis[i][0], m->axis[i][1], m->axis[i][2]};
        m3v(k->Rw[i], ax, aw);
        real rr[3] = {p[0] - k->pw[i][0], p[1] - k->pw[i][1], p[2] - k->pw[i][2]}, c[3];
        v3cross(aw, rr, c);
        J[6 + i - 1] = v3dot(n, c);
    }
}

/* ------------------------------------------------------------------------------------------- */
/* ground query: z=0 half-space (plane.urdf box top face, rex_gym/util/pybullet_data/plane.urdf) */
/* or heightfield triangle mesh (rex_gym/model/terrain.py:32-53; btHeightfieldTerrainShape)      */
/* ------------------------------------------------------------------------------------------- */
static void ground_query(const RexoSim* s, const RexoEnv* e, const real* p, real* dist, real* n) {
    if (s->c.terrain == REXO_TERRAIN_PLANE) { *dist = p[2]; n[0] = 0; n[1] = 0; n[2] = 1; return; }
    const float* h = s->c.fields + (size_t)e->field_id * 65536;
    const double cell = 0.05;
    double fx = p[0] / cell + 127.5, fy = p[1] / cell + 127.5;
    if (fx < 0) fx = 0; if (fy < 0) fy = 0; if (fx > 254.999) fx = 254.999; if (fy > 254.999) fy = 254.999;
    int ix = (int)floor(fx), iy = (int)floor(fy);
    double u = fx - ix, v = fy - iy;
    double h00 = h[iy * 256 + ix], h10 = h[iy * 256 + ix + 1], h01 = h[(iy + 1) * 256 + ix], h11 = h[(iy + 1) * 256 + ix + 1];
    double hx, hy, hh;
    if (v >= u) { hx = h11 - h01; hy = h01 - h00; }   /* triangle (x,j),(x,j+1),(x+1,j+1) */
    else { hx = h10 - h00; hy = h11 - h10; }          /* triangle (x,j),(x+1,j+1),(x+1,j) */
    hh = h00 + hx * u + hy * v - s->field_zoff[e->field_id];
    double nx = -hx / cell, ny = -hy / cell, nz = 1.0;
    double inv = 1.0 / sqrt(nx * nx + ny * ny + nz * nz);
    n[0] = nx * inv; n[1] = ny * inv; n[2] = nz * inv;
    *dist = (p[2] - hh) * n[2];
}
/* btPlaneSpace1 */
static void plane_space(const real* n, real* p, real* q) {
    if (fabs(n[2]) > 0.7071067811865475244008443621048490) {
        real a = n[1] * n[1] + n[2] * n[2], k = 1.0 / sqrt(a);
        p[0] = 0; p[1] = -n[2] * k; p[2] = n[1] * k;
        q[0] = a * k; q[1] = -n[0] * p[2]; q[2] = n[0] * p[1];
    } else {
        real a = n[0] * n[0] + n[1] * n[1], k = 1.0 / sqrt(a);
        p[0] = -n[1] * k; p[1] = n[0] * k; p[2] = 0;
        q[0] = -n[2] * p[1]; q[1] = n[2] * p[0]; q[2] = a * k;
    }
}

/* ------------------------------------------------------------------------------------------- */
/* one pybullet.stepSimulation (call site rex_gym/model/rex.py:161) with joint torques tau       */
/* ------------------------------------------------------------------------------------------- */
typedef struct { real J[6 + REXO_MAXDOF], W[6 + REXO_MAXDOF]; real dinv, rhs, lo, hi, applied, mu; int normal_row; } Row;

static void step_simulation(RexoSim* s, RexoEnv* e, const real* tau) {
    const RexoModel* m = &s->m;
    const RexoConfig* c = &s->c;
    const real dt = c->sim_dt;
    const int nd = 6 + m->ndof;
    static _Thread_local Scratch K;
    static _Thread_local Row lim[2 * REXO_MAXDOF], nrm[REXO_MAXSHAPE], fri[2 * REXO_MAXSHAPE];
    Scratch* k = &K;
    kinematics(s, e, k);
    /* 1. unconstrained velocity update (btMultiBodyDynamicsWorld::solveConstraints: ABA then v += a*dt) */
    real acc[6 + REXO_MAXDOF], vel[6 + REXO_MAXDOF];
    aba(s, e, k, tau, acc);
    for (int a = 0; a < 3; a++) { vel[a] = e->angvel[a] + dt * acc[a]; vel[3 + a] = e->linvel[a] + dt * acc[3 + a]; }
    for (int j = 0; j < m->ndof; j++) vel[6 + j] = e->qd[j] + dt * acc[6 + j];
    /* btMultiBody::applyDeltaVeeMultiDof clamps every generalised velocity (base included) to +-m_maxCoordinateVelocity
     * (100, PyBullet's documented maxJointVelocity default) whenever a velocity change is applied */
    const real vmax = c->max_coordinate_velocity;
    for (int a = 0; a < nd; a++) { if (vel[a] > vmax) vel[a] = vmax; if (vel[a] < -vmax) vel[a] = -vmax; }

    /* 2. constraint rows at the start-of-step configuration */
    int nlim = 0, nn = 0, nf = 0;
    for (int j = 0; j < m->ndof; j++) {         /* btMultiBodyJointLimitConstraint: rows only when violated */
        for (int side = 0; side < 2; side++) {
            real pen = side == 0 ? (e->q[j] - m->lower[j + 1]) : (m->upper[j + 1] - e->q[j]);
            if (pen > 0) continue;
            Row* r = &lim[nlim++];
            for (int a = 0; a < nd; a++) r->J[a] = 0;
            r->J[6 + j] = side == 0 ? 1.0 : -1.0;
            delta_response(s, k, r->J, r->W);
            real den = 0, rel = 0; for (int a = 0; a < nd; a++) { den += r->J[a] * r->W[a]; rel += r->J[a] * vel[a]; }
            r->dinv = 1.0 / den;
            /* btMultiBodyJointLimitConstraint::createConstraintRows with m_splitImpulse (Bullet default): a violation deeper than
             * m_splitImpulsePenetrationThreshold (-0.04) moves the positional term to m_rhsPenetration, which the multibody solver
             * never applies -- the row then only stops further motion (an overshoot > 0.04 rad is permanent) */
            r->rhs = (pen > -0.04) ? (-pen * c->erp_joint / dt - rel) * r->dinv : -rel * r->dinv;
            r->lo = 0; r->hi = 1e10; r->applied = 0; r->normal_row = -1;
        }
    }
    e->limit_rows = nlim;
    e->contact_mask = 0;
    /* contact exists while the distance is below the manifold's breaking threshold: btCollisionDispatcher::getNewManifold with
     * CD_USE_RELATIVE_CONTACT_BREAKING_THRESHOLD = min over the two shapes of getAngularMotionDisc() * gContactBreakingThreshold
     * (0.02); for the toe link's compound shape that is 0.81 mm (rex_gym_b200/model_tables.py::contact_breaking_distance) */
    const real breaking = c->contact_breaking, slop = 1e-5;
    for (int sh = 0; sh < m->nshape; sh++) {    /* deepest sample point of each contact group vs ground */
        e->contact_vertex[sh] = -1;
        if (!m->shape_enabled[sh]) continue;
        int b = 0;
        real best = 1e30, bp[3] = {0, 0, 0}, bn[3] = {0, 0, 1}; int bi = -1;
        for (int v = 0; v < m->shape_npts[sh]; v++) {
            const int pi = m->shape_start[sh] + v;
            const int pb = m->pt_body[pi];
            if (c->terrain == REXO_TERRAIN_RANDOM && !m->pt_terrain[pi]) continue;
            const double* pl = m->pts[pi];
            real lp[3] = {pl[0], pl[1], pl[2]}, wp[3], n[3], d;
            m3v(k->Rw[pb], lp, wp);
            for (int a = 0; a < 3; a++) wp[a] += k->pw[pb][a];
            ground_query(s, e, wp, &d, n);
            d -= m->pt_margin[pi];
            if (d < best) { best = d; bi = v; b = pb; for (int a = 0; a < 3; a++) { bp[a] = wp[a]; bn[a] = n[a]; } }
        }
        if (bi < 0 || best > breaking) continue;
        e->contact_mask |= (1 << sh);
        e->contact_vertex[sh] = bi;
        Row* r = &nrm[nn];
        contact_jacobian(s, k, b, bp, bn, r->J);
        delta_response(s, k, r->J, r->W);
        real den = 0, rel = 0; for (int a = 0; a < nd; a++) { den += r->J[a] * r->W[a]; rel += r->J[a] * vel[a]; }
        r->dinv = 1.0 / den;
        real pen = best + slop;
        real poserr = 0, velerr = -rel;
        if (pen > 0) velerr -= pen / dt; else poserr = -pen * c->erp_contact / dt;
        r->rhs = (pen > -0.04) ? (poserr + velerr) * r->dinv : velerr * r->dinv;   /* split-impulse threshold */
        r->lo = 0; r->hi = 1e10; r->applied = 0; r->normal_row = -1;
        real t1[3], t2[3]; plane_space(bn, t1, t2);
        for (int d2 = 0; d2 < 2; d2++) {
            Row* f = &fri[nf++];
            contact_jacobian(s, k, b, bp, d2 == 0 ? t1 : t2, f->J);
            delta_response(s, k, f->J, f->W);
            real dn = 0, rl = 0; for (int a = 0; a < nd; a++) { dn += f->J[a] * f->W[a]; rl += f->J[a] * vel[a]; }
            f->dinv = 1.0 / dn; f->rhs = -rl * f->dinv; f->applied = 0; f->mu = c->friction; f->normal_row = nn;
            f->lo = 0; f->hi = 0;
        }
        nn++;
    }
    /* 3. PGS (btMultiBodyConstraintSolver::solveSingleIteration ordering), residual early-out */
    real dV[6 + REXO_MAXDOF];
    for (int a = 0; a < nd; a++) dV[a] = 0;
    int it = 0;
    if (nlim + nn > 0) {
        for (it = 0; it < c->solver_iterations; it++) {
            real resid = 0;
            for (int jj = 0; jj < nlim + nn + nf; jj++) {
                Row* r;
                if (jj < nlim) { int idx = (it & 1) ? jj : nlim - 1 - jj; r = &lim[idx]; }
                else if (jj < nlim + nn) r = &nrm[jj - nlim];
                else {
                    r = &fri[jj - nlim - nn];
                    real tot = nrm[r->normal_row].applied;
                    if (!(tot > 0)) continue;
                    r->lo = -r->mu * tot; r->hi = r->mu * tot;
                }
                real dvn = 0; for (int a = 0; a < nd; a++) dvn += r->J[a] * dV[a];
                real dI = r->rhs - dvn * r->dinv;
                real sum = r->applied + dI;
                if (sum < r->lo) { dI = r->lo - r->applied; r->applied = r->lo; }
                else if (sum > r->hi) { dI = r->hi - r->applied; r->applied = r->hi; }
                else r->applied = sum;
                for (int a = 0; a < nd; a++) dV[a] += r->W[a] * dI;
                real rs = dI / r->dinv;
                if (rs * rs > resid) resid = rs * rs;
            }
            if (resid <= c->residual_threshold || it >= c->solver_iterations - 1) { it++; break; }
        }
    }
    e->solver_iters = it;
    /* 4. integrate (btMultiBody::stepPositionsMultiDof) */
    for (int a = 0; a < nd; a++) { vel[a] += dV[a]; if (vel[a] > vmax) vel[a] = vmax; if (vel[a] < -vmax) vel[a] = -vmax; }   /* processDeltaVeeMultiDof2 */
    for (int a = 0; a < 3; a++) { e->angvel[a] = vel[a]; e->linvel[a] = vel[3 + a]; e->pos[a] += dt * vel[3 + a]; }
    for (int j = 0; j < m->ndof; j++) { e->qd[j] = vel[6 + j]; e->q[j] += dt * vel[6 + j]; }
    {   /* exponential-map quaternion update, base body branch of pQuatUpdateFun */
        real w[3] = {vel[0], vel[1], vel[2]};
        real fa = sqrt(v3dot(w, w));
        if (fa * dt > 0.7853981633974483) fa = 0.5 * 1.5707963267948966 / dt;   /* ANGULAR_MOTION_THRESHOLD */
        real ax[3];
        if (fa < 0.001) { real sc = 0.5 * dt - dt * dt * dt * 0.020833333333 * fa * fa; for (int a = 0; a < 3; a++) ax[a] = w[a] * sc; }
        else { real sc = sin(0.5 * fa * dt) / fa; for (int a = 0; a < 3; a++) ax[a] = w[a] * sc; }
        real dq[4] = {ax[0], ax[1], ax[2], cos(fa * dt * 0.5)};
        real q0[4] = {e->quat[0], e->quat[1], e->quat[2], e->quat[3]}, qn[4];
        /* world-frame omega: q_new = dq * q */
        qn[3] = dq[3] * q0[3] - dq[0] * q0[0] - dq[1] * q0[1] - dq[2] * q0[2];
        qn[0] = dq[3] * q0[0] + dq[0] * q0[3] + dq[1] * q0[2] - dq[2] * q0[1];
        qn[1] = dq[3] * q0[1] - dq[0] * q0[2] + dq[1] * q0[3] + dq[2] * q0[0];
        qn[2] = dq[3] * q0[2] + dq[0] * q0[1] - dq[1] * q0[0] + dq[2] * q0[3];
        real nrmq = sqrt(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3]);
        for (int a = 0; a < 4; a++) e->quat[a] = qn[a] / nrmq;
    }
}

/* ------------------------------------------------------------------------------------------- */
/* sensor history, latency and noise: rex_gym/model/rex.py:717-769                               */
/* ------------------------------------------------------------------------------------------- */
static Hist* hist_of(RexoSim* s, const RexoEnv* e) {
    if (e >= s->env && e < s->env + s->c.num_envs) return &s->hist[e - s->env];
    return &s->hist[s->c.num_envs + (e - s->snapshot)];
}
static double* ctrl_of(RexoSim* s, const RexoEnv* e) {
    if (e >= s->env && e < s->env + s->c.num_envs) return s->ctrl[e - s->env];
    return s->ctrl[s->c.num_envs + (e - s->snapshot)];
}
static void hist_push(Hist* h, const double* obs, int w) {        /* deque.appendleft, maxlen 100 (rex.py:122,733) */
    h->head = (h->head + 1) % REXO_HIST;
    memcpy(h->buf[h->head], obs, sizeof(double) * w);
    if (h->len < REXO_HIST) h->len++;
}
static const double* hist_at(const Hist* h, int k) { return h->buf[(h->head - k + 2 * REXO_HIST) % REXO_HIST]; }   /* history[k] */
static void hist_delayed(const Hist* h, double latency, double dt, int w, double* out) {   /* _GetDelayedObservation rex.py:735-753 */
    if (latency <= 0 || h->len == 1) { memcpy(out, hist_at(h, 0), sizeof(double) * w); return; }
    int n = (int)(latency / dt);
    if (n + 1 >= h->len) { memcpy(out, hist_at(h, h->len - 1), sizeof(double) * w); return; }
    double remaining = latency - n * dt;
    double alpha = remaining / dt;
    const double* a = hist_at(h, n); const double* b = hist_at(h, n + 1);
    for (int i = 0; i < w; i++) out[i] = (1.0 - alpha) * a[i] + alpha * b[i];
}
static void true_observation(const RexoSim* s, const RexoEnv* e, double* o) {     /* GetTrueObservation rex.py:717-724 */
    const RexoModel* m = &s->m; int n = m->nmotor;
    for (int i = 0; i < n; i++) { o[i] = e->q[m->motor_dof[i]]; o[n + i] = e->qd[m->motor_dof[i]]; o[2 * n + i] = e->tau_obs[i]; }
    for (int a = 0; a < 4; a++) o[3 * n + a] = e->quat[a];
    for (int a = 0; a < 3; a++) o[3 * n + 4 + a] = e->angvel[a];
}
static void receive_observation(RexoSim* s, RexoEnv* e) {                          /* ReceiveObservation rex.py:726-733 */
    if (!s->sensor_on) return;
    double o[REXO_OBSW]; true_observation(s, e, o);
    Hist* h = hist_of(s, e);
    hist_push(h, o, 3 * s->m.nmotor + 7);
    hist_delayed(h, s->c.control_latency, s->c.sim_dt, 3 * s->m.nmotor + 7, ctrl_of(s, e));
}
/* Counter-based N(0,1) (Box-Muller on two draws of the reset generator) replacing the unseeded np.random.normal of
 * _AddSensorNoise (rex.py:763-769).  Keyed on (seed, global env, reset count, control step since reset, call site, component);
 * sites: 0 observation rpy, 1 observation rpy rate, 2 observation motor angles, 3 reward orientation, 4 reward torques,
 * 5 reward velocities, 6 termination orientation, 7 turn goal-check orientation */
double rexo_noise(uint64_t seed, uint32_t env, uint32_t reset_count, uint32_t step, uint32_t site, uint32_t comp) {
    uint32_t slot = 1024u + (((step * 8u + site) * 32u + comp) << 1);
    double u1 = ((double)(rexo_rand_u32(seed, env, reset_count, slot) >> 8) + 1.0) * (1.0 / 16777216.0);
    double u2 = (double)(rexo_rand_u32(seed, env, reset_count, slot + 1u) >> 8) * (1.0 / 16777216.0);
    return sqrt(-2.0 * log(u1)) * cos(2.0 * PI * u2);
}
static double noise(const RexoSim* s, const RexoEnv* e, int group, uint32_t site, uint32_t comp) {
    double sd = s->c.noise_stdev[group];
    if (sd <= 0) return 0.0;
    uint32_t genv = (uint32_t)(e - s->env) + (uint32_t)s->c.env_offset;
    return sd * rexo_noise(s->c.seed, genv, e->reset_count, (uint32_t)e->env_step_counter, site, comp);
}
/* Rex.GetBaseRollPitchYaw (rex.py:429-442): Euler angles of the DELAYED orientation + noise; GetBaseOrientation (:530-537) turns
 * them back into a quaternion.  With the sensor model off this is the true orientation (no round trip: bit-stable with round 1). */
static void sensed_quat(RexoSim* s, RexoEnv* e, uint32_t site, real* q4) {
    if (!s->sensor_on) { for (int a = 0; a < 4; a++) q4[a] = e->quat[a]; return; }
    const double* c = ctrl_of(s, e) + 3 * s->m.nmotor;
    real d4[4] = {c[0], c[1], c[2], c[3]}, rpy[3];
    quat_to_euler(d4, rpy);
    for (int a = 0; a < 3; a++) rpy[a] += noise(s, e, 3, site, a);
    euler_to_quat(rpy, q4);
}

/* ------------------------------------------------------------------------------------------- */
/* Rex.ApplyAction + stepSimulation + ReceiveObservation: rex_gym/model/rex.py:158-163,568-641   */
/* ------------------------------------------------------------------------------------------- */
static void apply_action(RexoSim* s, RexoEnv* e, const double* cmd, real* tau) {       /* Rex.ApplyAction rex.py:568-641 */
    const RexoModel* m = &s->m;
    int n = m->nmotor;
    double q[REXO_MAXDOF], qd[REXO_MAXDOF], kp[REXO_MAXDOF], kd[REXO_MAXDOF], ta[REXO_MAXDOF], to[REXO_MAXDOF];
    double qd_true[REXO_MAXDOF];
    for (int i = 0; i < n; i++) { q[i] = e->q[m->motor_dof[i]]; qd[i] = e->qd[m->motor_dof[i]]; qd_true[i] = qd[i]; kp[i] = e->kp; kd[i] = e->kd; }
    if (s->sensor_on && s->c.pd_latency > 0 && hist_of(s, e)->len > 0) {       /* _GetPDObservation rex.py:755-759 */
        double pdo[REXO_OBSW];
        hist_delayed(hist_of(s, e), s->c.pd_latency, s->c.sim_dt, 3 * n + 7, pdo);
        for (int i = 0; i < n; i++) { q[i] = pdo[i]; qd[i] = pdo[n + i]; }
    }
    rexo_motor_torque(n, cmd, q, qd, qd_true, kp, kd, ta, to);   /* rex.py:596-600 */
    for (int j = 0; j < m->ndof; j++) tau[j] = 0;
    for (int i = 0; i < n; i++) {                                /* overheat protection rex.py:601-608 */
        if (fabs(ta[i]) > 2.45) e->overheat[i] += 1; else e->overheat[i] = 0;
        if (e->overheat[i] > 1.0 / s->c.sim_dt) e->enabled[i] = 0;
        e->tau_obs[i] = to[i];                                   /* rex.py:612 */
        tau[m->motor_dof[i]] = e->enabled[i] ? ta[i] : 0.0;      /* rex.py:617-623 */
        e->cmd[i] = cmd[i];
    }
}
static void apply_action_and_step(RexoSim* s, RexoEnv* e, const double* cmd) {            /* one pass of Rex.Step's loop rex.py:158-163 */
    real tau[REXO_MAXDOF];
    apply_action(s, e, cmd, tau);
    step_simulation(s, e, tau);
    receive_observation(s, e);                                   /* rex.py:162 */
}
/* ApplyAction alone (no physics): the torque each motor joint would be driven with, for tests/golden/apply_action_golden.json.gz */
void rexo_apply_action(RexoSim* s, int i, const double* cmd, double* tau_motor) {
    real tau[REXO_MAXDOF];
    apply_action(s, &s->env[i], cmd, tau);
    for (int k = 0; k < s->m.nmotor; k++) tau_motor[k] = tau[s->m.motor_dof[k]];
}
void rexo_substep(RexoSim* s, int i, const double* cmd) { apply_action_and_step(s, &s->env[i], cmd); }
void rexo_physics_only(RexoSim* s, int i, const double* tau) {
    real t[REXO_MAXDOF]; for (int j = 0; j < s->m.ndof; j++) t[j] = tau[j];
    step_simulation(s, &s->env[i], t);
}

/* ------------------------------------------------------------------------------------------- */
/* task signals                                                                                 */
/* ------------------------------------------------------------------------------------------- */
static double stage_sigmoid(double t, double end_t, double width) {   /* walk_env.py:217-226 etc. */
    double beta = width, p = width;
    if (p - beta + end_t <= t && t <= p - (beta / 2) + end_t) return (2 / (beta * beta)) * (t - p + beta) * (t - p + beta);
    else if (p - (beta / 2) + end_t <= t && t <= p + end_t) return 1 - (2 / (beta * beta)) * (t - p) * (t - p);
    return 1;
}
static void ik_signal_common(RexoEnv* e, int gallop, double now, const double* pos, const double* rpy,
                             double step_length, double step_angle, double step_rotation, double step_period,
                             double direction, double* signal) {
    double frames[12], ang[12];
    rexo_gait_loop(&e->gp_phi, &e->gp_last_time, &e->gp_alpha, gallop, now, step_length, step_angle, step_rotation,
                   step_period, direction, NULL, frames);
    rexo_ik_solve(rpy, pos, frames, ang);
    /* reorder FR,FL,RR,RL -> FL,FR,RL,RR (walk_env.py:284-289) */
    for (int k = 0; k < 3; k++) { signal[k] = ang[3 + k]; signal[3 + k] = ang[k]; signal[6 + k] = ang[9 + k]; signal[9 + k] = ang[6 + k]; }
}
/* RexWalkEnv._transform_action_to_motor_command: walk_env.py:207-324 */
static void walk_command(RexoSim* s, RexoEnv* e, const double* action, double* cmd) {
    const double* init = s->c.signal == REXO_SIGNAL_OL ? POSE_STAND_OL : POSE_STAND;
    if (e->stay_still) { for (int i = 0; i < 12; i++) cmd[i] = init[i]; return; }
    double t = e->step_counter * s->c.sim_dt;
    if (e->target_position != 0) {     /* _check_target_position :207-215 */
        double cx = fabs(e->pos[0]);
        if (cx >= fabs(e->target_position) - 0.15) {
            e->goal_reached = 1;
            if (!e->is_terminating) { e->end_time = t; e->is_terminating = 1; }
        }
    }
    if (s->c.signal == REXO_SIGNAL_IK) {   /* _IK_signal :252-290 */
        double base_coeff = stage_sigmoid(t, 0.0, 1.5);
        double p = 0.8 + action[0];
        double gait_coeff = (0.0 <= t && t <= p) ? t : 1.0;                 /* :228-235 */
        double step = 0.6, period = 0.65, base_x = 0.01;
        if (e->backwards) { step = -.3; period = .5; base_x = .0; }
        double pos[3] = {base_x, 0.0 * base_coeff, 0.0 * base_coeff}, rpy[3] = {0.0 * base_coeff, 0.0 * base_coeff, 0.0 * base_coeff};
        double step_length = step * gait_coeff;
        if (e->goal_reached) {
            double pb = 0.8 + action[1];
            double brakes = (e->end_time <= t && t <= pb + e->end_time) ? 1 - (t - e->end_time) : 0.0;   /* :237-244 */
            step_length *= brakes;
            if (brakes == 0.0) e->stay_still = 1;
        }
        double direction = step_length < 0 ? -1.0 : 1.0;
        ik_signal_common(e, 0, t * s->c.gait_clock_scale, pos, rpy, step_length, 0.0, 0.0, period, direction, cmd);
    } else {                               /* _open_loop_signal :292-315 */
        double period = 1.0 / 8, l_a = 0.1, f_a = l_a * 2;
        if (e->goal_reached) {
            double pb = 0.8 + 0.;
            double coeff = (e->end_time <= t && t <= pb + e->end_time) ? 1 - (t - e->end_time) : 0.0;
            l_a *= coeff; f_a *= coeff;
            if (coeff == 0.0) e->stay_still = 1;
        }
        double p0 = 0.8 + 0.0;
        double start = (0.0 <= t && t <= p0) ? t : 1.0;
        l_a *= start; f_a *= start;
        double l_ext = l_a * cos(2 * PI / period * t), f_ext = f_a * cos(2 * PI / period * t);
        double l_sw = -l_ext, sw = -f_ext;
        double pose[12] = {0.0, l_ext + action[0], f_ext + action[1], 0.0, l_sw + action[2], sw + action[3],
                           0.0, l_sw + action[4], sw + action[5], 0.0, l_ext + action[6], f_ext + action[7]};
        for (int i = 0; i < 12; i++) cmd[i] = init[i] + pose[i];
    }
}
/* RexReactiveEnv._transform_action_to_motor_command: gallop_env.py:212-313 */
static void gallop_command(RexoSim* s, RexoEnv* e, double* action, double* cmd) {
    const double* init = s->c.signal == REXO_SIGNAL_OL ? POSE_STAND_OL : POSE_STAND;
    if (e->stay_still) { for (int i = 0; i < 12; i++) cmd[i] = POSE_STAND[i]; return; }   /* rex.initial_pose :307-308 */
    double t = e->step_counter * s->c.sim_dt;
    if (e->target_position != 0) {     /* :212-220 (no stop space) */
        double cx = fabs(e->pos[0]);
        if (cx >= fabs(e->target_position)) {
            e->goal_reached = 1;
            if (!e->is_terminating) { e->end_time = t; e->is_terminating = 1; }
        }
    }
    if (s->c.signal == REXO_SIGNAL_IK) {   /* :257-285 */
        double base_coeff = stage_sigmoid(t, 0.0, 1.5);
        double p = 1. + action[1];
        double gait_coeff = (0.0 <= t && t <= p) ? t : 1.0;                 /* :241-248 */
        double pos[3] = {0.01, 0.0 * base_coeff, -0.007}, rpy[3] = {0.0 * base_coeff, 0.0 * base_coeff, 0.0 * base_coeff};
        double step_length = 1.3 * gait_coeff;
        if (e->goal_reached) {
            double pb = 1. + action[0];
            double brakes = (e->end_time <= t && t <= pb + e->end_time) ? 1 - (t - e->end_time) : 0.0;   /* :232-239 */
            step_length *= brakes;
        }
        ik_signal_common(e, 1, t * s->c.gait_clock_scale, pos, rpy, step_length, 0.0, 0.0, 0.3, 1.0, cmd);
    } else {                               /* :287-304 */
        if (e->goal_reached) {
            double pb = 1. + .0;
            double coeff = (e->end_time <= t && t <= pb + e->end_time) ? 1 - (t - e->end_time) : 0.0;
            for (int i = 0; i < 4; i++) action[i] *= coeff;
            if (coeff == 0.0) e->stay_still = 1;
        }
        for (int i = 0; i < 4; i++) {
            cmd[3 * i] = init[3 * i];
            if (i == 0 || i == 1) { cmd[3 * i + 1] = init[3 * i + 1] + action[0]; cmd[3 * i + 2] = init[3 * i + 2] + action[1]; }
            else { cmd[3 * i + 1] = init[3 * i + 1] + action[2]; cmd[3 * i + 2] = init[3 * i + 2] + action[3]; }
        }
    }
}
/* RexTurnEnv._transform_action_to_motor_command: turn_env.py:230-346 */
static void turn_command(RexoSim* s, RexoEnv* e, const double* action, double* cmd) {
    const double* init = s->c.signal == REXO_SIGNAL_OL ? POSE_STAND_OL : POSE_STAND;
    double t = e->step_counter * s->c.sim_dt;
    if (e->stay_still) {
        if (t - e->end_time >= 1.) e->env_goal_reached = 1;     /* _terminate_with_delay :334-336 */
        for (int i = 0; i < 12; i++) cmd[i] = init[i];
        return;
    }
    {   /* _check_target_position :324-332 */
        real q4[4], rpy[3];
        sensed_quat(s, e, 7, q4);                                  /* rex.GetBaseOrientation() turn_env.py:325 */
        quat_to_euler(q4, rpy);
        double cz = rpy[2];
        if (cz < 0) cz += 6.28;
        if (fabs(e->target_orient - cz) <= 0.01) {
            e->goal_reached = 1;
            if (!e->is_terminating) { e->end_time = t; e->is_terminating = 1; }
        }
    }
    if (s->c.signal == REXO_SIGNAL_IK) {   /* :239-269 */
        double base_coeff = stage_sigmoid(t, 0.0, 1.5);
        double gait_coeff = (0.0 <= t && t <= .8) ? t : 1.0;                 /* :230-237 */
        double dirv = -0.5 * gait_coeff;
        if (e->clockwise) dirv *= -1;
        double pos[3] = {0.009, 0.0 * base_coeff, 0.0 * base_coeff}, rpy[3] = {0.0 * base_coeff, 0.0 * base_coeff, 0.0 * base_coeff};
        double step_rotation = dirv + action[0];
        double step_period = 0.75 + action[1];
        if (e->goal_reached) e->stay_still = 1;
        ik_signal_common(e, 0, t * s->c.gait_clock_scale, pos, rpy, 0.02, 0.0, step_rotation, step_period, 1.0, cmd);
    } else {                               /* :271-311 */
        if (e->goal_reached) e->stay_still = 1;
        const double period = 1.0 / 10.0;  /* STEP_PERIOD turn_env.py:17 */
        double extension = 0.1, swing = 0.03 + action[0], swipe = 0.05 + action[1];
        int ith = ((int)(t / period)) % 2;
        double L0[12] = {swipe, extension, -swing, -swipe, extension, swing, swipe, -extension, swing, -swipe, -extension, -swing};
        double L1[12] = {-swipe, 0, swing, swipe, 0, -swing, -swipe, 0, -swing, swipe, 0, swing};
        double R0[12] = {swipe, extension, swing, -swipe, extension, -swing, swipe, -extension, -swing, -swipe, -extension, swing};
        double R1[12] = {-swipe, 0, -swing, swipe, 0, swing, -swipe, 0, swing, swipe, 0, -swing};
        const double* first = e->clockwise ? R0 : L0; const double* second = e->clockwise ? R1 : L1;
        const double* sel = ith ? second : first;
        for (int i = 0; i < 12; i++) cmd[i] = POSE_STAND_OL[i] + sel[i];
    }
}
/* RexStandupEnv._signal: standup_env.py:113-134 */
static void standup_command(RexoSim* s, RexoEnv* e, const double* action, double* cmd) {
    double t = e->step_counter * s->c.sim_dt;
    if (t > 0.1) { for (int i = 0; i < 12; i++) cmd[i] = POSE_STAND[i]; return; }
    t += 1;
    for (int i = 0; i < 12; i++) cmd[i] = POSE_STAND[i] * ((.1 + action[0]) / t + 1.5);
}

/* RexPosesEnv._signal: poses_env.py:187-225 (ramp :178-185; Kinematics.solve on the staged base pose) */
static const double POSE_RANGE[5][2] = {{-0.007, 0.007}, {-0.048, 0.021}, {-PI / 4, PI / 4}, {-PI / 4, PI / 4}, {-PI / 4, PI / 4}};  /* rex_gym_env.py:260-267 */
static void poses_command(RexoSim* s, RexoEnv* e, const double* action, double* cmd) {
    static const double FRAMES[12] = {0.115, -0.0925, -0.2, 0.115, 0.0925, -0.2, -0.115, -0.0925, -0.2, -0.115, 0.0925, -0.2};
    double t = e->step_counter * s->c.sim_dt;
    double p = 0.8 + action[0], end_t = 0.0;
    double coeff = (end_t <= t && t <= p + end_t) ? t : 1.0;
    double staged = e->target_value * coeff;
    double pos[3] = {0.01, 0, 0}, rpy[3] = {0, 0, 0}, ang[12];       /* _ranges defaults: base_x 0.01, others 0 */
    if (e->next_pose == 0) pos[1] = staged; else if (e->next_pose == 1) pos[2] = staged;
    else rpy[e->next_pose - 2] = staged;
    rexo_ik_solve(rpy, pos, FRAMES, ang);
    for (int k = 0; k < 3; k++) { cmd[k] = ang[3 + k]; cmd[3 + k] = ang[k]; cmd[6 + k] = ang[9 + k]; cmd[9 + k] = ang[6 + k]; }   /* :209-214 */
}

/* ------------------------------------------------------------------------------------------- */
/* reward / termination / observation                                                           */
/* ------------------------------------------------------------------------------------------- */
static double env_reward(RexoSim* s, RexoEnv* e) {
    const RexoConfig* c = &s->c;
    if (c->task == REXO_TASK_POSES) return 1.0;                                        /* poses_env.py:256-258 */
    if (c->task == REXO_TASK_TURN) return 0.035 - fabs(e->pos[0]) - fabs(e->pos[1]);   /* turn_env.py:362-367 */
    if (c->task == REXO_TASK_STANDUP) {                                                /* standup_env.py:151-167 */
        double pr = fabs(0.0 - e->pos[0]) + fabs(0.0 - e->pos[1]) + fabs(0.21 - e->pos[2]);
        if (fabs(pr) < 0.1) pr = 1.0 - pr; else pr = -pr;
        if (e->pos[2] > 0.21) pr = -1.0 - pr;
        return pr;
    }
    /* RexGymEnv._reward: rex_gym_env.py:501-542 */
    double cx = -e->pos[0];
    if (c->backwards == 1) cx = -cx;      /* `self._backwards`, the constructor argument (rex_gym_env.py:269,506): a direction drawn
                                           * at reset (walk_env.py:133-136 `self.backwards`) does not flip the objective */
    double fwd;
    e->target_position = fabs(e->target_position);
    double tp = e->target_position;
    if (cx > tp + 0.15) fwd = tp - cx;
    else if (tp <= cx && cx <= tp + 0.15) fwd = 1.0;
    else if (cx <= 0.05) fwd = 0.0;
    else fwd = cx / tp;
    double drift = -fabs(e->pos[1]);
    real q4[4], R[9];
    sensed_quat(s, e, 3, q4);                                      /* rex.GetBaseOrientation() rex_gym_env.py:530 */
    quat_to_mat(q4, R);
    double shake = -fabs(1 * R[6] + 1 * R[7] + 0 * R[8]);
    double dot = 0;
    if (s->sensor_on) {                                            /* GetMotorTorques() . GetMotorVelocities() :536-537 */
        const double* co = ctrl_of(s, e); int n = s->m.nmotor;
        for (int i = 0; i < n; i++) dot += (co[2 * n + i] + noise(s, e, 2, 4, i)) * (co[n + i] + noise(s, e, 1, 5, i));
    } else
    for (int i = 0; i < s->m.nmotor; i++) dot += e->tau_obs[i] * e->qd[s->m.motor_dof[i]];
    double energy = -fabs(dot) * c->sim_dt;
    /* objectives [forward, energy, drift, shake] x weights [distance, energy, drift, shake] (:56-59,191,538-540) */
    return fwd * c->w_distance + energy * c->w_energy + drift * c->w_drift + shake * c->w_shake;
}
static int env_done(RexoSim* s, RexoEnv* e) {
    const RexoConfig* c = &s->c;
    real q4[4] = {e->quat[0], e->quat[1], e->quat[2], e->quat[3]};
    if (c->task == REXO_TASK_POSES) return e->env_goal_reached;      /* is_fallen -> False (poses_env.py:247-254) */
    if (c->task == REXO_TASK_WALK || c->task == REXO_TASK_TURN) {    /* walk_env.py:326-338, rex_gym_env.py:490-495 */
        real qs[4], R[9];
        sensed_quat(s, e, 6, qs);                                    /* rex.GetBaseOrientation(): delayed + noisy */
        quat_to_mat(qs, R);
        return (R[8] < 0.85) || e->env_goal_reached;
    }
    real rpy[3]; quat_to_euler(q4, rpy);
    int fallen = fabs(rpy[0]) > 0.3 || fabs(rpy[1]) > 0.5;           /* gallop_env.py:319-329, standup_env.py:139-149 */
    if (c->task == REXO_TASK_STANDUP) return fallen;
    return fallen || e->env_goal_reached || (e->pos[1] > 0.3);       /* gallop_env.py:315-317 */
}
static double map_pi(double a) {   /* MapToMinusPiToPi rex.py:26-41 */
    double r = fmod(a, 2 * PI);
    if (r >= PI) r -= 2 * PI; else if (r < -PI) r += 2 * PI;
    return r;
}
static void env_observation(RexoSim* s, RexoEnv* e, double* o) {   /* walk_env.py:356-362, gallop_env.py:349-356 */
    if (s->sensor_on) {       /* GetBaseRollPitchYaw / GetBaseRollPitchYawRate / GetMotorAngles: delayed + noise (rex.py:429-442,548-558,457-468) */
        const double* co = ctrl_of(s, e); int n = s->m.nmotor;
        real d4[4] = {co[3 * n], co[3 * n + 1], co[3 * n + 2], co[3 * n + 3]}, rp[3];
        quat_to_euler(d4, rp);
        o[0] = rp[0] + noise(s, e, 3, 0, 0); o[1] = rp[1] + noise(s, e, 3, 0, 1);
        o[2] = co[3 * n + 4] + noise(s, e, 4, 1, 0); o[3] = co[3 * n + 5] + noise(s, e, 4, 1, 1);
        if (s->c.task == REXO_TASK_GALLOP) for (int i = 0; i < n; i++) o[4 + i] = map_pi(co[i] + noise(s, e, 0, 2, i));
        return;
    }
    real q4[4] = {e->quat[0], e->quat[1], e->quat[2], e->quat[3]}, rpy[3];
    quat_to_euler(q4, rpy);
    o[0] = rpy[0]; o[1] = rpy[1]; o[2] = e->angvel[0]; o[3] = e->angvel[1];
    if (s->c.task == REXO_TASK_GALLOP) for (int i = 0; i < s->m.nmotor; i++) o[4 + i] = map_pi(e->q[s->m.motor_dof[i]]);
}
static void obs_bounds(const RexoSim* s, int j, double* lo, double* hi) {   /* walk_env.py:364-374 (+0.01 rex_gym_env.py:277-278) */
    double ub = (j == 2 || j == 3) ? 2 * PI / s->c.sim_dt : 2 * PI;
    *hi = ub + 0.01; *lo = -ub - 0.01;
}
static void action_bounds(const RexoSim* s, int j, double* lo, double* hi) {
    const RexoConfig* c = &s->c; double b; (void)j;
    switch (c->task) {
        case REXO_TASK_WALK: b = c->signal == REXO_SIGNAL_IK ? 0.4 : 0.01; *lo = -b; *hi = b; break;   /* walk_env.py:104-114 */
        case REXO_TASK_GALLOP: b = c->signal == REXO_SIGNAL_IK ? 0.4 : 0.3; *lo = b; *hi = -b; break;  /* inverted Box gallop_env.py:128-130 */
        case REXO_TASK_TURN: *lo = -0.01; *hi = 0.01; break;                                           /* turn_env.py:100-110 */
        case REXO_TASK_POSES: *lo = -0.1; *hi = 0.1; break;                                            /* poses_env.py:118-120 */
        default: *lo = -0.1; *hi = 0.1; break;                                                         /* standup_env.py:99-101 */
    }
}
/* RangeNormalize._normalize_observ (wrappers.py:238-242) then ConvertTo32Bit._convert_observ (:522-527) */
void rexo_wrap_observation(const RexoSim* s, const double* raw, float* out) {
    for (int j = 0; j < s->obs_dim; j++) {
        double v = raw[j];
        if (s->c.normalize) { double lo, hi; obs_bounds(s, j, &lo, &hi); v = 2 * (v - lo) / (hi - lo) - 1; }
        out[j] = (float)v;
    }
}
/* ClipAction.step (wrappers.py:262-265: clip to the [-1, 1] box RangeNormalize shows) then RangeNormalize._denormalize_action
 * (:232-236) onto the task env's own Box -- gallop's has low > high (gallop_env.py:128-130), so the map turns into -b * a */
void rexo_wrap_action(const RexoSim* s, const double* act, double* out) {
    for (int j = 0; j < s->act_dim; j++) {
        double v = act[j];
        if (s->c.normalize) {
            double lo, hi; action_bounds(s, j, &lo, &hi);
            v = clipd(v, -1.0, 1.0);
            v = (v + 1) / 2 * (hi - lo) + lo;
        }
        out[j] = v;
    }
}
static void write_obs(RexoSim* s, RexoEnv* e, float* out) {
    double o[4 + REXO_MAXDOF];
    env_observation(s, e, o);
    rexo_wrap_observation(s, o, out);
}

/* ------------------------------------------------------------------------------------------- */
/* reset                                                                                        */
/* ------------------------------------------------------------------------------------------- */
static void settle_state(RexoSim* s, RexoEnv* e) {   /* Rex.Reset: rex.py:296-324 */
    const RexoModel* m = &s->m;
    e->pos[0] = 0; e->pos[1] = 0; e->pos[2] = 0.21;                 /* terrain.py:14-20 */
    e->quat[0] = 0; e->quat[1] = 0; e->quat[2] = 0; e->quat[3] = 1;
    for (int a = 0; a < 3; a++) { e->linvel[a] = 0; e->angvel[a] = 0; }
    for (int j = 0; j < m->ndof; j++) { e->q[j] = 0; e->qd[j] = 0; }
    for (int i = 0; i < m->nmotor; i++) {                            /* ResetPose :344-372 */
        e->q[m->motor_dof[i]] = s->stand_pose[i];
        e->overheat[i] = 0; e->enabled[i] = 1; e->tau_obs[i] = 0; e->cmd[i] = 0;
    }
    e->step_counter = 0;
    if (s->sensor_on) { Hist* h = hist_of(s, e); h->len = 0; h->head = REXO_HIST - 1; }      /* _observation_history.clear() rex.py:303 */
    /* settle_on_reset == 2: pristine start -- joints placed at the task's init pose, no holding phase.  This is the state the
     * PyBullet trajectories recovered from the reference's checkpoints start from (tools/extract_memory_golden.py). */
    if (s->c.settle_on_reset == 2) for (int i = 0; i < m->nmotor; i++) e->q[m->motor_dof[i]] = s->init_pose[i];
    /* RexPosesEnv.reset calls RexGymEnv.reset() with initial_motor_angles=None: no holding phase (rex.py:307) */
    if (s->c.settle_on_reset == 1 && s->c.task != REXO_TASK_POSES) {
        receive_observation(s, e);                                                       /* :313 */
        for (int it = 0; it < 100; it++) apply_action_and_step(s, e, s->stand_pose);     /* :315-318 */
        int n2 = (int)(0.5 / s->c.sim_dt);                                               /* reset_duration=0.5 */
        for (int it = 0; it < n2; it++) apply_action_and_step(s, e, s->init_pose);       /* :319-323 */
    }
    receive_observation(s, e);                                                           /* :324 */
}
static void reset_env(RexoSim* s, int i) {
    RexoEnv* e = &s->env[i];
    const RexoConfig* c = &s->c;
    uint32_t rc = e->reset_count + 1;
    int field = (c->terrain == REXO_TERRAIN_RANDOM) ? (int)(((uint32_t)i + (uint32_t)c->env_offset + rc) % (uint32_t)c->nfields) : 0;
    RexoEnv* snap = &s->snapshot[field];
    double kp = c->kp_lo == c->kp_hi ? c->motor_kp : rand_uniform(s, i, rc, 4, c->kp_lo, c->kp_hi);
    double kd = c->kd_lo == c->kd_hi ? c->motor_kd : rand_uniform(s, i, rc, 5, c->kd_lo, c->kd_hi);
    /* the C ABI carries gains as float32: drawn gains are rounded the same way so they compare bit-exactly */
    if (c->kp_lo != c->kp_hi) kp = (double)(float)kp;
    if (c->kd_lo != c->kd_hi) kd = (double)(float)kd;
    /* the settle (rex.py:314-323) runs with the nominal gains; per-env randomised gains (ours, the
     * reference ships no randomizer) apply from the first control step on, so the settled state only
     * depends on (init pose, field) and is computed once per field */
    if (snap->reset_count == 0) {
        snap->field_id = field; snap->kp = c->motor_kp; snap->kd = c->motor_kd;
        settle_state(s, snap); snap->reset_count = 1;
    }
    *e = *snap;
    if (s->sensor_on) {       /* the history the reset hold left behind (it only depends on the field, like the settled state) */
        s->hist[i] = s->hist[c->num_envs + field];
        memcpy(s->ctrl[i], s->ctrl[c->num_envs + field], sizeof(double) * REXO_OBSW);
    }
    e->reset_count = rc; e->field_id = field; e->kp = kp; e->kd = kd;
    e->env_step_counter = 0; e->limit_step = 0;
    e->gp_phi = 0; e->gp_last_time = 0; e->gp_alpha = 0;
    e->goal_reached = 0; e->is_terminating = 0; e->stay_still = 0; e->env_goal_reached = 0;
    e->backwards = 0; e->clockwise = 0; e->end_time = 0;
    e->target_position = 0; e->target_orient = 0; e->init_orient = 0;
    if (c->task == REXO_TASK_WALK) {   /* walk_env.py:125-154 */
        if (c->backwards < 0) e->backwards = (rexo_rand_u32(c->seed, (uint32_t)i + (uint32_t)c->env_offset, rc, 0) >> 31) ? 1 : 0;
        else e->backwards = c->backwards;
        if (isnan(c->target_position)) {
            double bound = e->backwards ? -3 : 3, half = e->backwards ? -2 : 1;   /* bound//2 floor-div */
            e->target_position = rand_uniform(s, i, rc, 1, half, bound);
        } else e->target_position = c->target_position;
    } else if (c->task == REXO_TASK_GALLOP) {   /* gallop_env.py:142-160 */
        e->target_position = isnan(c->target_position) ? rand_uniform(s, i, rc, 1, 1, 3) : c->target_position;
    } else if (c->task == REXO_TASK_TURN) {     /* turn_env.py:129-160 */
        e->target_orient = isnan(c->target_orient) ? rand_uniform(s, i, rc, 2, 0.2, 6) : c->target_orient;
        e->init_orient = isnan(c->init_orient) ? rand_uniform(s, i, rc, 3, 0.2, 6) : c->init_orient;
        double diff = fabs(e->init_orient - e->target_orient);   /* _solve_direction :313-322 */
        e->clockwise = 0;
        if (e->init_orient < e->target_orient) { if (diff > 3.14) e->clockwise = 1; }
        else { if (diff < 3.14) e->clockwise = 1; }
        real rpy[3] = {0, 0, e->init_orient}, q4[4];
        euler_to_quat(rpy, q4);                                  /* :157-159 */
        e->pos[0] = 0; e->pos[1] = 0; e->pos[2] = 0.21;
        for (int a = 0; a < 4; a++) e->quat[a] = q4[a];
    } else if (c->task == REXO_TASK_POSES) {    /* poses_env.py:148-176 */
        int any = 0;
        for (int k = 0; k < 5; k++) any |= !isnan(c->pose_values[k]);
        if (any) {                               /* fill_next_pose_and_target (a None argument counts as 0.0) */
            e->next_pose = 4;
            for (int k = 0; k < 4; k++) if (!isnan(c->pose_values[k]) && c->pose_values[k] != 0.0) { e->next_pose = k; break; }
            double v = c->pose_values[e->next_pose];
            e->target_value = isnan(v) ? 0.0 : v;
        } else {                                 /* deque rotation: the constructor's own reset() consumed 'base_y' */
            e->next_pose = (int)(rc % 5u);
            e->target_value = rand_uniform(s, i, rc, 6, POSE_RANGE[e->next_pose][0], POSE_RANGE[e->next_pose][1]);
        }
    }
}

/* ------------------------------------------------------------------------------------------- */
/* public API                                                                                   */
/* ------------------------------------------------------------------------------------------- */
RexoSim* rexo_create(const RexoModel* model, const RexoConfig* cfg) {
    RexoSim* s = (RexoSim*)calloc(1, sizeof(RexoSim));
    s->m = *model; s->c = *cfg;
    s->env = (RexoEnv*)calloc(cfg->num_envs, sizeof(RexoEnv));
    s->nsnap = cfg->terrain == REXO_TERRAIN_RANDOM ? cfg->nfields : 1;
    s->snapshot = (RexoEnv*)calloc(s->nsnap, sizeof(RexoEnv));
    s->sensor_on = cfg->control_latency > 0 || cfg->pd_latency > 0;
    for (int k = 0; k < 5; k++) s->sensor_on |= cfg->noise_stdev[k] > 0;
    {   /* rings exist when the sensor model is on, and always for small batches (unit entry points) */
        int nh = (s->sensor_on || cfg->num_envs <= 64) ? cfg->num_envs + s->nsnap : 0;
        s->hist = nh ? (Hist*)calloc(nh, sizeof(Hist)) : NULL;
        s->ctrl = nh ? (double (*)[REXO_OBSW])calloc(nh, sizeof(double[REXO_OBSW])) : NULL;
        for (int k = 0; k < nh; k++) s->hist[k].head = REXO_HIST - 1;
    }
    switch (cfg->task) {
        case REXO_TASK_WALK: s->act_dim = cfg->signal == REXO_SIGNAL_IK ? 2 : 8; s->obs_dim = 4; break;
        case REXO_TASK_GALLOP: s->act_dim = cfg->signal == REXO_SIGNAL_IK ? 2 : 4; s->obs_dim = 4 + model->nmotor; break;
        case REXO_TASK_TURN: s->act_dim = 2; s->obs_dim = 4; break;
        case REXO_TASK_POSES: s->act_dim = 1; s->obs_dim = 4; break;
        default: s->act_dim = 1; s->obs_dim = 4; break;
    }
    const double* ip = POSE_STAND;
    if (cfg->task == REXO_TASK_STANDUP) ip = POSE_REST;
    else if (cfg->signal == REXO_SIGNAL_OL) ip = POSE_STAND_OL;
    for (int i = 0; i < 12; i++) { s->init_pose[i] = ip[i]; s->stand_pose[i] = POSE_STAND[i]; }
    for (int i = 12; i < model->nmotor; i++) { s->init_pose[i] = ARM_REST[i - 12]; s->stand_pose[i] = ARM_REST[i - 12]; }
    s->field_zoff = (double*)calloc(cfg->nfields > 0 ? cfg->nfields : 1, sizeof(double));
    for (int f = 0; f < cfg->nfields && cfg->fields; f++) {
        float lo = 1e30f, hi = -1e30f;
        for (int a = 0; a < 65536; a++) { float h = cfg->fields[(size_t)f * 65536 + a]; if (h < lo) lo = h; if (h > hi) hi = h; }
        s->field_zoff[f] = 0.5 * ((double)lo + (double)hi);
    }
    return s;
}
void rexo_destroy(RexoSim* s) { if (!s) return; free(s->env); free(s->snapshot); free(s->hist); free(s->ctrl); free(s->field_zoff); free(s); }
void rexo_sensor_clear(RexoSim* s, int i) { if (s->hist) { s->hist[i].len = 0; s->hist[i].head = REXO_HIST - 1; } }
void rexo_sensor_push(RexoSim* s, int i, const double* obs) { if (s->hist) hist_push(&s->hist[i], obs, 3 * s->m.nmotor + 7); }
void rexo_sensor_delayed(RexoSim* s, int i, double latency, double* out) {
    if (s->hist) hist_delayed(&s->hist[i], latency, s->c.sim_dt, 3 * s->m.nmotor + 7, out);
}
int rexo_sensor_row(RexoSim* s, int i, int k, double* out) {
    if (!s->hist) return 0;
    if (k >= 0 && k < s->hist[i].len) memcpy(out, hist_at(&s->hist[i], k), sizeof(double) * (3 * s->m.nmotor + 7));
    return s->hist[i].len;
}
int rexo_obs_dim(const RexoSim* s) { return s->obs_dim; }
int rexo_action_dim(const RexoSim* s) { return s->act_dim; }
RexoEnv* rexo_env(RexoSim* s, int i) { return &s->env[i]; }

void rexo_reset(RexoSim* s, const int32_t* idx, int k, float* obs_out) {
    int n = idx ? k : s->c.num_envs;
    for (int j = 0; j < n; j++) {
        int i = idx ? idx[j] : j;
        reset_env(s, i);
        if (obs_out) write_obs(s, &s->env[i], obs_out + (size_t)j * s->obs_dim);
    }
}
/* <task>._transform_action_to_motor_command incl. the wrapper maths on the action */
static void transform_action(RexoSim* s, RexoEnv* e, const double* act, double* cmd) {
    const RexoConfig* c = &s->c;
    double a[8] = {0};
    rexo_wrap_action(s, act, a);
    switch (c->task) {
        case REXO_TASK_WALK: walk_command(s, e, a, cmd); break;
        case REXO_TASK_GALLOP: gallop_command(s, e, a, cmd); break;
        case REXO_TASK_TURN: turn_command(s, e, a, cmd); break;
        case REXO_TASK_POSES: poses_command(s, e, a, cmd); break;
        default: standup_command(s, e, a, cmd); break;
    }
    for (int j = 12; j < s->m.nmotor; j++) cmd[j] = ARM_REST[j - 12];   /* rex_gym_env.py:363-367 */
}
void rexo_transform_action(RexoSim* s, int i, const double* act, double* cmd) { transform_action(s, &s->env[i], act, cmd); }
void rexo_reward_done_obs(RexoSim* s, int i, double* reward, int* done, double* obs) {
    *reward = env_reward(s, &s->env[i]); *done = env_done(s, &s->env[i]); env_observation(s, &s->env[i], obs);
}
static void step_env(RexoSim* s, int i, const float* act, float* obs, float* reward, uint8_t* done) {
    RexoEnv* e = &s->env[i];
    const RexoConfig* c = &s->c;
    double a[8] = {0}, cmd[REXO_MAXDOF];
    for (int j = 0; j < s->act_dim; j++) a[j] = act[j];
    transform_action(s, e, a, cmd);
    for (int r = 0; r < c->action_repeat; r++) {                        /* Rex.Step rex.py:158-163 */
        apply_action_and_step(s, e, cmd);
        e->step_counter += 1;
    }
    double rew = env_reward(s, e);
    int d = env_done(s, e);
    e->env_step_counter += 1;
    e->limit_step += 1;
    if (c->max_episode_steps > 0 && e->limit_step >= c->max_episode_steps) d = 1;   /* LimitDuration */
    write_obs(s, e, obs);
    *reward = (float)rew;
    *done = (uint8_t)(d ? 1 : 0);
}
void rexo_step(RexoSim* s, const float* actions, float* obs, float* reward, uint8_t* done, int nthreads) {
    int n = s->c.num_envs;
    (void)nthreads;
#ifdef _OPENMP
#pragma omp parallel for num_threads(nthreads) schedule(static) if (nthreads > 1)
#endif
    for (int i = 0; i < n; i++)
        step_env(s, i, actions + (size_t)i * s->act_dim, obs + (size_t)i * s->obs_dim, reward + i, done + i);
}

/* ------------------------------------------------------------------------------------------- */
/* diagnostics for invariant tests                                                              */
/* ------------------------------------------------------------------------------------------- */
void rexo_aba(RexoSim* s, int i, const double* tau, double* qdd) {
    static _Thread_local Scratch K;
    real t[REXO_MAXDOF], acc[6 + REXO_MAXDOF];
    for (int j = 0; j < s->m.ndof; j++) t[j] = tau[j];
    kinematics(s, &s->env[i], &K);
    aba(s, &s->env[i], &K, t, acc);
    for (int j = 0; j < 6 + s->m.ndof; j++) qdd[j] = acc[j];
}
void rexo_mass_matrix(RexoSim* s, int i, double* M) {
    static _Thread_local Scratch K;
    int nd = 6 + s->m.ndof;
    real t[REXO_MAXDOF] = {0}, acc[6 + REXO_MAXDOF];
    kinematics(s, &s->env[i], &K);
    aba(s, &s->env[i], &K, t, acc);
    /* M^-1 column by column through the impulse response, then invert numerically on the Python side */
    for (int c = 0; c < nd; c++) {
        real f[6 + REXO_MAXDOF] = {0}, dv[6 + REXO_MAXDOF];
        f[c] = 1;
        delta_response(s, &K, f, dv);
        for (int r = 0; r < nd; r++) M[r * nd + c] = dv[r];
    }
}
void rexo_kinetic_momentum(RexoSim* s, int i, double* ke, double* lin, double* ang, double* com) {
    static _Thread_local Scratch K;
    const RexoModel* m = &s->m; RexoEnv* e = &s->env[i];
    kinematics(s, e, &K);
    real ww[3] = {e->angvel[0], e->angvel[1], e->angvel[2]}, vw[3] = {e->linvel[0], e->linvel[1], e->linvel[2]};
    m3tv(K.Rw[0], ww, K.v[0]); m3tv(K.Rw[0], vw, K.v[0] + 3);
    double T = 0, P[3] = {0, 0, 0}, L[3] = {0, 0, 0}, C[3] = {0, 0, 0}, Mt = 0;
    for (int b = 0; b < m->nb; b++) {
        if (b > 0) {
            real vp[6]; m6v(K.Xup[b], K.v[m->parent[b]], vp);
            for (int a = 0; a < 6; a++) K.v[b][a] = vp[a] + K.S[b][a] * e->qd[b - 1];
        }
        real I6[36], Iv[6]; body_inertia6(m, b, I6); m6v(I6, K.v[b], Iv);
        T += 0.5 * v6dot(K.v[b], Iv);
        /* world COM velocity and angular velocity */
        real wb[3] = {K.v[b][0], K.v[b][1], K.v[b][2]}, vb[3] = {K.v[b][3], K.v[b][4], K.v[b][5]};
        real c[3] = {m->com[b][0], m->com[b][1], m->com[b][2]}, wxc[3], vc[3], vcw[3], cw[3], wwb[3];
        v3cross(wb, c, wxc); for (int a = 0; a < 3; a++) vc[a] = vb[a] + wxc[a];
        m3v(K.Rw[b], vc, vcw); m3v(K.Rw[b], c, cw); m3v(K.Rw[b], wb, wwb);
        for (int a = 0; a < 3; a++) cw[a] += K.pw[b][a];
        real Ic[9], Iw[3], t3[3]; for (int a = 0; a < 9; a++) Ic[a] = m->inertia[b][a];
        m3v(Ic, wb, t3); m3v(K.Rw[b], t3, Iw);
        real mv[3] = {m->mass[b] * vcw[0], m->mass[b] * vcw[1], m->mass[b] * vcw[2]}, rxp[3];
        v3cross(cw, mv, rxp);
        for (int a = 0; a < 3; a++) { P[a] += mv[a]; L[a] += Iw[a] + rxp[a]; C[a] += m->mass[b] * cw[a]; }
        Mt += m->mass[b];
    }
    *ke = T;
    for (int a = 0; a < 3; a++) { lin[a] = P[a]; ang[a] = L[a]; com[a] = C[a] / Mt; }
}

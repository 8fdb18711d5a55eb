// rexsim_render.cu -- rgb_array frames of chosen environments, ray-cast on the device from the SoA state
// (RexGymEnv.render(mode="rgb_array"), rex_gym/envs/rex_gym_env.py:416-439).
//
// What is drawn is the collision geometry the contact model collides with, not the URDF visual meshes: the base and
// chassis boxes, the 12 leg boxes, the four toe prisms, with mark 'arm' the six arm cylinders and arm_section_4's box, and
// the ground (plane z = 0, or the env's heightfield).  Each shape takes its link's URDF visual colour from the render table
// (include/rexsim.h REXSIM_RT_*, packed by rex_gym_b200/model_tables.py pack_render_tables), which also holds the light,
// the checker tones of the ground and the sky.
//
// Grid: one CTA of 16 x 16 threads per 16 x 16 pixel tile of one image, blockIdx.x = tile, blockIdx.y = image.  Warp 0
// poses the robot (forward kinematics over the model table, 19 bodies: cheap enough to redo per CTA, and it keeps the
// library free of allocations after rexsim_create), writes every shape as world-space geometry + bounding sphere into
// shared memory, and culls the spheres against the tile's frustum.  Then every thread casts its pixel's ray against
// the surviving shapes and the ground.  The kernel only reads the state.
#include "rexsim_kernel.cuh"
#include "rexsim_arm.cuh"

namespace rexsim {

struct RenderArgs {
    const float* __restrict__ sf;       // [NF][N]
    const int32_t* __restrict__ si;     // [NI][N]
    const float* __restrict__ model;    // model table
    const float* __restrict__ rt;       // render table, REXSIM_RT_FLOATS
    const float* __restrict__ fields;   // [nfields][256*256] (terrain RANDOM)
    const float* __restrict__ zoff;     // [nfields] vertical centring of each field
    const float* __restrict__ zrange;   // [nfields][2] lowest / highest centred height
    const int32_t* __restrict__ idx;    // [k] env of each image
    uint8_t* __restrict__ rgb;          // [k][H][W][3]
    int32_t* __restrict__ err;          // [N + 1]: word N = aggregate error bits
    int N, terrain, arm, toe_npts;
    int W, H, tiles_x, image0;
    float dist, yaw, pitch;             // radians
};

enum { RT_TILE = 16, SHAPE_FLOATS = 20, MAX_SHAPES = REXSIM_RT_NSHAPES };
// shape record: [0..2] centre (box, cylinder) or body origin (toe); [3..11] three unit axes (box axes, foot frame columns,
// cylinder axis in [9..11]); [12..14] half extents (box) or radius, half length (cylinder); [15..17] bounding sphere centre, [18] radius
enum { SH_C = 0, SH_A0 = 3, SH_A1 = 6, SH_A2 = 9, SH_H = 12, SH_S = 15, SH_R = 18 };

// Bullet's computeViewMatrixFromYawPitchRoll (up axis z) followed by computeViewMatrixFromPositions (gluLookAt) and
// computeProjectionMatrixFOV (pybullet client API, the calls of rex_gym_env.py:420-436): R = Rz(yaw) Rx(pitch),
// eye = target + R (0, -d, 0), up = R (0, 0, 1); f = normalize(target - eye), s = normalize(f x up), u = s x f.
// The ray of pixel (row, col) is f + x tan(fov/2) (W/H) s + y tan(fov/2) u with x = (2 col + 1)/W - 1, y = 1 - (2 row + 1)/H;
// its f component is 1, so the ray parameter of a hit is its depth along the view axis (what near / far clip).
struct Camera { V3 eye, f, s, u; };
__device__ __forceinline__ Camera make_camera(V3 target, float d, float yaw, float pitch, float tan_half, float aspect) {
    float sy, cy, sp, cp;
    sincosf(yaw, &sy, &cy); sincosf(pitch, &sp, &cp);
    // Rx(pitch) (0, -d, 0) = (0, -d cp, -d sp); Rz(yaw) of that
    V3 off = mk(d * cp * sy, -d * cp * cy, -d * sp);
    V3 up = mk(sp * sy, -sp * cy, cp);
    Camera C;
    C.eye = target + off;
    V3 f = mk(-off.x, -off.y, -off.z);
    f = rsqrtf(dot(f, f)) * f;
    V3 s = cross(f, up);
    s = rsqrtf(dot(s, s)) * s;
    C.u = (tan_half) * cross(s, f);
    C.s = (tan_half * aspect) * s;
    C.f = f;
    return C;
}
__device__ __forceinline__ V3 pixel_ray(const Camera& C, float x, float y) { return fma3(x, C.s, fma3(y, C.u, C.f)); }

// box from its 8 body-frame corners (index 4 ix + 2 iy + iz, tools/compile_urdf.py shape_points) placed by (R, p)
__device__ void write_box(float* rec, const float* corners, const M3& R, V3 p) {
    V3 c0 = mk(corners[0], corners[1], corners[2]);
    V3 ex = 0.5f * (mk(corners[12], corners[13], corners[14]) - c0);
    V3 ey = 0.5f * (mk(corners[6], corners[7], corners[8]) - c0);
    V3 ez = 0.5f * (mk(corners[3], corners[4], corners[5]) - c0);
    V3 c = p + mul(R, c0 + ex + ey + ez);
    float hx = sqrtf(dot(ex, ex)), hy = sqrtf(dot(ey, ey)), hz = sqrtf(dot(ez, ez));
    V3 ax = mul(R, (1.f / hx) * ex), ay = mul(R, (1.f / hy) * ey), az = mul(R, (1.f / hz) * ez);
    rec[SH_C] = c.x; rec[SH_C + 1] = c.y; rec[SH_C + 2] = c.z;
    rec[SH_A0] = ax.x; rec[SH_A0 + 1] = ax.y; rec[SH_A0 + 2] = ax.z;
    rec[SH_A1] = ay.x; rec[SH_A1 + 1] = ay.y; rec[SH_A1 + 2] = ay.z;
    rec[SH_A2] = az.x; rec[SH_A2 + 1] = az.y; rec[SH_A2 + 2] = az.z;
    rec[SH_H] = hx; rec[SH_H + 1] = hy; rec[SH_H + 2] = hz;
    rec[SH_S] = c.x; rec[SH_S + 1] = c.y; rec[SH_S + 2] = c.z; rec[SH_R] = sqrtf(hx * hx + hy * hy + hz * hz);
}
__device__ void write_frame(float* rec, const M3& R, V3 p) {
    rec[SH_C] = p.x; rec[SH_C + 1] = p.y; rec[SH_C + 2] = p.z;
    rec[SH_A0] = R.c0.x; rec[SH_A0 + 1] = R.c0.y; rec[SH_A0 + 2] = R.c0.z;
    rec[SH_A1] = R.c1.x; rec[SH_A1 + 1] = R.c1.y; rec[SH_A1 + 2] = R.c1.z;
    rec[SH_A2] = R.c2.x; rec[SH_A2 + 1] = R.c2.y; rec[SH_A2 + 2] = R.c2.z;
}
__device__ __forceinline__ void write_sphere(float* rec, V3 c, float r) {
    rec[SH_S] = c.x; rec[SH_S + 1] = c.y; rec[SH_S + 2] = c.z; rec[SH_R] = r;
}
__device__ __forceinline__ V3 ld3(const float* p) { return mk(p[0], p[1], p[2]); }

// warp 0: pose every shape of env `env` into `shapes` (world frame)
__device__ void pose_shapes(const RenderArgs& A, int env, float* shapes, int lane) {
    const size_t N = A.N;
    const float* sf = A.sf;
    const V3 pos = mk(sf[(F_POS + 0) * N + env], sf[(F_POS + 1) * N + env], sf[(F_POS + 2) * N + env]);
    const M3 R0 = quat_to_mat(sf[(F_QUAT + 0) * N + env], sf[(F_QUAT + 1) * N + env], sf[(F_QUAT + 2) * N + env],
                              sf[(F_QUAT + 3) * N + env]);
    const float* mt = A.model;
    if (lane < 4) {            // leg `lane`: the step kernel's frames, origins moved from the base position to the world's
        const int leg = lane;
        const float q[3] = {sf[(F_Q + 3 * leg + 0) * N + env], sf[(F_Q + 3 * leg + 1) * N + env], sf[(F_Q + 3 * leg + 2) * N + env]};
        M3 R1, R2, R3; V3 p1, p2, p3;
        leg_frames(R0, mt + REXSIM_MT_LEG + leg * 48, q, R1, R2, R3, p1, p2, p3);
        p1 = pos + p1; p2 = pos + p2; p3 = pos + p3;
        const float* BX = mt + REXSIM_MT_BOX + leg * 72;
        write_box(shapes + (3 + 3 * leg + 0) * SHAPE_FLOATS, BX, R1, p1);
        write_box(shapes + (3 + 3 * leg + 1) * SHAPE_FLOATS, BX + 24, R2, p2);
        write_box(shapes + (3 + 3 * leg + 2) * SHAPE_FLOATS, BX + 48, R3, p3);
        float* toe = shapes + (15 + leg) * SHAPE_FLOATS;
        write_frame(toe, R3, p3);
        const float* ts = A.rt + REXSIM_RT_TOESPH;
        write_sphere(toe, p3 + mul(R3, mk(ts[0], 0.f, ts[1])), ts[2]);
    } else if (lane < 7) {     // base and chassis boxes
        write_box(shapes + (lane - 4) * SHAPE_FLOATS, mt + REXSIM_MT_BASEBOX + 24 * (lane - 4), R0, pos);
    } else if (lane == 7 && A.arm) {   // the arm: one serial chain with general joint frames (rexsim_arm.cuh layout)
        M3 Rp = R0; V3 pp = pos;
        for (int j = 0; j < ARM_NJ; j++) {
            M3 Rj; V3 pj;
            arm_joint_frame(mt + REXSIM_MT_ARM + ARM_STRIDE * j, Rp, pp, sf[(F_AQ + j) * N + env], Rj, pj);
            const float* cy = A.rt + REXSIM_RT_CYL + 8 * j;
            float* rec = shapes + (19 + j) * SHAPE_FLOATS;
            V3 c = pj + mul(Rj, ld3(cy)), ax = mul(Rj, ld3(cy + 3));
            rec[SH_C] = c.x; rec[SH_C + 1] = c.y; rec[SH_C + 2] = c.z;
            rec[SH_A2] = ax.x; rec[SH_A2 + 1] = ax.y; rec[SH_A2 + 2] = ax.z;
            rec[SH_H] = cy[6]; rec[SH_H + 1] = cy[7];
            write_sphere(rec, c, sqrtf(cy[6] * cy[6] + cy[7] * cy[7]));
            if (j == (int)A.rt[REXSIM_RT_ARMBOX]) write_box(shapes + 25 * SHAPE_FLOATS, A.rt + REXSIM_RT_ARMBOX + 1, Rj, pj);
            Rp = Rj; pp = pj;
        }
    }
}

// entering parameter of the ray o + t r into the slab |a . (p - c)| <= h: clips [t0, t1], remembers the entering face
__device__ __forceinline__ void clip_plane(float denom, float dist, float& t0, float& t1, int& face, int f) {
    // inside where denom t <= dist
    if (denom < 0.f) { float t = dist / denom; if (t > t0) { t0 = t; face = f; } }
    else if (denom > 0.f) { float t = dist / denom; t1 = fminf(t1, t); }
    else if (dist < 0.f) t1 = -1.f;
}

// ray against one posed shape; on a nearer hit updates best t and the outward normal
__device__ __forceinline__ void hit_box(const float* rec, V3 o, V3 r, float& best, V3& nrm) {
    V3 w = o - ld3(rec + SH_C);
    float t0 = 0.f, t1 = best; int face = -1;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        V3 a = ld3(rec + SH_A0 + 3 * k);
        float h = rec[SH_H + k], ow = dot(a, w), ra = dot(a, r);
        clip_plane(ra, h - ow, t0, t1, face, 2 * k + 1);
        clip_plane(-ra, h + ow, t0, t1, face, 2 * k);
    }
    if (face >= 0 && t0 <= t1) {
        best = t0;
        V3 a = ld3(rec + SH_A0 + 3 * (face >> 1));
        nrm = (face & 1) ? a : mk(-a.x, -a.y, -a.z);
    }
}
// toe prism: the convex (x, z) profile of the foot frame extruded over y in [-w, w] (REXSIM_MT_TOE); planes n . (x, z) <= d
__device__ __forceinline__ void hit_toe(const float* rec, const float* planes, int np, float w, V3 o, V3 r, float& best, V3& nrm) {
    V3 dw = o - ld3(rec + SH_C);
    V3 a0 = ld3(rec + SH_A0), a1 = ld3(rec + SH_A1), a2 = ld3(rec + SH_A2);
    float ox = dot(a0, dw), oy = dot(a1, dw), oz = dot(a2, dw);
    float rx = dot(a0, r), ry = dot(a1, r), rz = dot(a2, r);
    float t0 = 0.f, t1 = best; int face = -1;
    clip_plane(ry, w - oy, t0, t1, face, np + 1);
    clip_plane(-ry, w + oy, t0, t1, face, np);
    for (int e = 0; e < np && t0 <= t1; e++) {
        const float* P = planes + 3 * e;
        clip_plane(fmaf(P[0], rx, P[1] * rz), P[2] - fmaf(P[0], ox, P[1] * oz), t0, t1, face, e);
    }
    if (face >= 0 && t0 <= t1) {
        best = t0;
        nrm = face == np ? mk(-a1.x, -a1.y, -a1.z) : face == np + 1 ? a1 : fma3(planes[3 * face], a0, planes[3 * face + 1] * a2);
    }
}
// capped cylinder: the slab |axial| <= half length intersected with the infinite cylinder of the radius
__device__ __forceinline__ void hit_cylinder(const float* rec, V3 o, V3 r, float& best, V3& nrm) {
    V3 ax = ld3(rec + SH_A2);
    V3 w = o - ld3(rec + SH_C);
    float R = rec[SH_H], h = rec[SH_H + 1];
    float oa = dot(ax, w), ra = dot(ax, r);
    float t0 = 0.f, t1 = best; int face = -1;
    clip_plane(ra, h - oa, t0, t1, face, 1);
    clip_plane(-ra, h + oa, t0, t1, face, 0);
    V3 wp = fma3(-oa, ax, w), rp = fma3(-ra, ax, r);
    float a = dot(rp, rp), b = dot(wp, rp), c = dot(wp, wp) - R * R;
    if (a > 0.f) {
        float disc = b * b - a * c;
        if (disc < 0.f) return;
        float sq = sqrtf(disc), te = (-b - sq) / a, tx = (-b + sq) / a;
        if (te > t0) { t0 = te; face = 2; }
        t1 = fminf(t1, tx);
    } else if (c > 0.f) return;
    if (face >= 0 && t0 <= t1) {
        best = t0;
        if (face == 2) { V3 q = fma3(t0, rp, wp); nrm = rsqrtf(dot(q, q)) * q; }
        else nrm = face ? ax : mk(-ax.x, -ax.y, -ax.z);
    }
}

// ground: the plane z = 0, or the env's heightfield (rexsim_kernel.cu ground_query: vertex (ix, iy) at x = (ix - 127.5) * 0.05,
// height h[iy][ix] - zoff, cell split v >= u).  The ray is marched cell by cell (2-D DDA) over the part of it that lies inside
// the field's square and inside the slab of the field's heights.  Outside the square the ground is the horizontal plane at
// the field's lowest centred height (the physics clamps its queries to the border cells instead; DESIGN.md section 5).
__device__ __forceinline__ void hit_ground(const RenderArgs& A, const float* h, float zoff, float zlo, float zhi, V3 o, V3 r,
                                           float& best, V3& nrm) {
    if (A.terrain != REXSIM_TERRAIN_RANDOM) {
        if (r.z < 0.f) { float t = -o.z / r.z; if (t > 0.f && t < best) { best = t; nrm = mk(0.f, 0.f, 1.f); } }
        return;
    }
    const float gx0 = fmaf(o.x, 20.f, 127.5f), gy0 = fmaf(o.y, 20.f, 127.5f), dgx = r.x * 20.f, dgy = r.y * 20.f;
    if (r.z < 0.f) {           // the plane outside the square
        float t = (zlo - o.z) / r.z;
        float gx = fmaf(t, dgx, gx0), gy = fmaf(t, dgy, gy0);
        if (t > 0.f && t < best && (gx < 0.f || gx > 255.f || gy < 0.f || gy > 255.f)) { best = t; nrm = mk(0.f, 0.f, 1.f); }
    }
    float ta = 0.f, tb = best; int dummy = 0;
    clip_plane(r.z, zhi - o.z, ta, tb, dummy, 0);
    clip_plane(-r.z, o.z - zlo, ta, tb, dummy, 0);
    clip_plane(dgx, 255.f - gx0, ta, tb, dummy, 0);
    clip_plane(-dgx, gx0, ta, tb, dummy, 0);
    clip_plane(dgy, 255.f - gy0, ta, tb, dummy, 0);
    clip_plane(-dgy, gy0, ta, tb, dummy, 0);
    if (!(ta <= tb)) return;
    int ix = min(max((int)floorf(fmaf(ta, dgx, gx0)), 0), 254), iy = min(max((int)floorf(fmaf(ta, dgy, gy0)), 0), 254);
    const int sx = dgx > 0.f ? 1 : -1, sy = dgy > 0.f ? 1 : -1;
    const float ez = o.z + zoff;          // heights are compared uncentred
    // g = ray height - ground height along the ray is evaluated once at every boundary the ray crosses (cell edges, cell
    // diagonals) and carried into the next piece, so the march is watertight: a crossing of the ground cannot fall between
    // two pieces through rounding.  The hit is the crossing piece's triangle plane, its ray parameter clamped into the piece.
    float t = ta, g = NAN;
    for (;;) {
        const float tx = dgx != 0.f ? ((float)(ix + (sx > 0)) - gx0) / dgx : INFINITY;
        const float ty = dgy != 0.f ? ((float)(iy + (sy > 0)) - gy0) / dgy : INFINITY;
        const float tn = fminf(fminf(tx, ty), tb);
        const float* c = h + iy * 256 + ix;
        const float h00 = __ldg(c), h10 = __ldg(c + 1), h01 = __ldg(c + 256), h11 = __ldg(c + 257);
        const float u0 = gx0 - (float)ix, v0 = gy0 - (float)iy;
        const float dd = dgy - dgx, td = dd != 0.f ? (u0 - v0) / dd : INFINITY;      // v = u on the ray
        const bool split = td > t && td < tn;
        float ts = t;
        for (int piece = 0; piece <= (int)split; piece++) {
            const float te = split && piece == 0 ? td : tn, tm = 0.5f * (ts + te);
            // tri 0: v >= u, z = h00 + (h11 - h01) u + (h01 - h00) v;  tri 1: v < u, z = h00 + (h10 - h00) u + (h11 - h10) v
            const bool tri0 = fmaf(tm, dgy, v0) >= fmaf(tm, dgx, u0);
            const float a = tri0 ? h11 - h01 : h10 - h00, b = tri0 ? h01 - h00 : h11 - h10;
            if (g != g) g = fmaf(ts, r.z, ez) - (h00 + a * fmaf(ts, dgx, u0) + b * fmaf(ts, dgy, v0));
            const float ge = fmaf(te, r.z, ez) - (h00 + a * fmaf(te, dgx, u0) + b * fmaf(te, dgy, v0));
            if (g == 0.f || (g > 0.f) != (ge > 0.f)) {
                const float f0 = ez - h00 - a * u0 - b * v0, f1 = r.z - a * dgx - b * dgy;
                best = fminf(fmaxf(f1 != 0.f ? -f0 / f1 : ts, ts), te);
                float nx = -a * 20.f, ny = -b * 20.f, inv = rsqrtf(nx * nx + ny * ny + 1.f);
                nrm = mk(nx * inv, ny * inv, inv);
                return;
            }
            g = ge; ts = te;
        }
        if (tn >= tb) return;
        t = tn;
        if (tx <= ty) ix += sx; else iy += sy;
        if (ix < 0 || ix > 254 || iy < 0 || iy > 254) return;
    }
}

__global__ void __launch_bounds__(RT_TILE * RT_TILE) render_kernel(const RenderArgs A) {
    __shared__ float rt[REXSIM_RT_FLOATS];
    __shared__ float shapes[MAX_SHAPES * SHAPE_FLOATS];
    __shared__ unsigned live;
    const int tid = threadIdx.y * RT_TILE + threadIdx.x;
    const int img = A.image0 + blockIdx.y;
    const int env = A.idx[img];
    const bool valid = env >= 0 && env < A.N;
    for (int i = tid; i < REXSIM_RT_FLOATS; i += RT_TILE * RT_TILE) rt[i] = A.rt[i];
    const int tile = blockIdx.x, c0 = (tile % A.tiles_x) * RT_TILE, r0 = (tile / A.tiles_x) * RT_TILE;
    const float tan_half = tanf(0.5f * A.rt[REXSIM_RT_CAM] * (3.14159265358979323846f / 180.f)), aspect = (float)A.W / (float)A.H;
    const float inv_w = 1.f / (float)A.W, inv_h = 1.f / (float)A.H;
    const int nshapes = A.arm ? REXSIM_RT_NSHAPES : 19;
    Camera C;
    if (valid) C = make_camera(mk(A.sf[(F_POS + 0) * (size_t)A.N + env], A.sf[(F_POS + 1) * (size_t)A.N + env],
                                  A.sf[(F_POS + 2) * (size_t)A.N + env]), A.dist, A.yaw, A.pitch, tan_half, aspect);
    if (tid < 32) {
        if (valid) {
            pose_shapes(A, env, shapes, tid);
            __syncwarp();
            // frustum of the tile: the four planes through the eye spanned by its extreme pixel rays
            const int c1 = min(c0 + RT_TILE, A.W) - 1, r1 = min(r0 + RT_TILE, A.H) - 1;
            const float xl = (2 * c0 + 1) * inv_w - 1.f, xr = (2 * c1 + 1) * inv_w - 1.f;
            const float yt = 1.f - (2 * r0 + 1) * inv_h, yb = 1.f - (2 * r1 + 1) * inv_h;
            const V3 tl = pixel_ray(C, xl, yt), tr = pixel_ray(C, xr, yt), bl = pixel_ray(C, xl, yb), br = pixel_ray(C, xr, yb);
            const V3 mid = pixel_ray(C, 0.5f * (xl + xr), 0.5f * (yt + yb));
            bool keep = tid < nshapes;
            if (keep) {
                const float* rec = shapes + tid * SHAPE_FLOATS;
                const V3 d = ld3(rec + SH_S) - C.eye;
                const float rad = rec[SH_R];
                const V3 edges[4][2] = {{bl, tl}, {tl, tr}, {tr, br}, {br, bl}};
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    V3 n = cross(edges[k][0], edges[k][1]);
                    const float nn = dot(n, n);
                    if (!(nn > 1e-20f)) continue;         // a one-pixel-wide tile: no plane on that side
                    n = rsqrtf(nn) * n;
                    if (dot(n, mid) < 0.f) n = mk(-n.x, -n.y, -n.z);
                    if (dot(n, d) < -rad) keep = false;
                }
            }
            const unsigned m = __ballot_sync(0xffffffffu, keep);
            if (tid == 0) live = m;
        } else if (tid == 0) {
            live = 0;
            if (blockIdx.x == 0) atomicOr(A.err + A.N, REXSIM_FLAG_BAD_INDEX);
        }
    }
    __syncthreads();
    const int col = c0 + threadIdx.x, row = r0 + threadIdx.y;
    if (col >= A.W || row >= A.H) return;
    float rgbf[3] = {rt[REXSIM_RT_SKY], rt[REXSIM_RT_SKY + 1], rt[REXSIM_RT_SKY + 2]};
    if (valid) {
        const V3 r = pixel_ray(C, (2 * col + 1) * inv_w - 1.f, 1.f - (2 * row + 1) * inv_h);
        const V3 o = C.eye;
        const float rr = dot(r, r);
        float best = INFINITY; V3 nrm = mk(0.f, 0.f, 1.f); int who = -1;
        for (unsigned m = live; m; m &= m - 1) {
            const int s = __ffs(m) - 1;
            const float* rec = shapes + s * SHAPE_FLOATS;
            const V3 d = ld3(rec + SH_S) - o;                 // bounding sphere first
            const float tc = dot(d, r), rad = rec[SH_R];
            if (dot(d, d) * rr - tc * tc > rad * rad * rr) continue;
            const float prev = best;
            if (s < 15 || s == 25) hit_box(rec, o, r, best, nrm);
            else if (s < 19) hit_toe(rec, rt + REXSIM_RT_TOE, A.toe_npts, A.model[REXSIM_MT_BASE + 15], o, r, best, nrm);
            else hit_cylinder(rec, o, r, best, nrm);
            if (best < prev) who = s;
        }
        if (A.terrain == REXSIM_TERRAIN_RANDOM) {
            const int field = A.si[I_FIELD * (size_t)A.N + env];
            const float prev = best;
            hit_ground(A, A.fields + (size_t)field * 65536, A.zoff[field], A.zrange[2 * field], A.zrange[2 * field + 1], o, r, best, nrm);
            if (best < prev) who = -2;
        } else {
            const float prev = best;
            hit_ground(A, nullptr, 0.f, 0.f, 0.f, o, r, best, nrm);
            if (best < prev) who = -2;
        }
        if (who != -1 && best >= rt[REXSIM_RT_CAM + 1] && best <= rt[REXSIM_RT_CAM + 2]) {
            const float* col3;
            if (who == -2) {
                const V3 p = fma3(best, r, o);
                const float inv_sq = 1.f / rt[REXSIM_RT_CHECK + 6];
                const int parity = ((int)floorf(p.x * inv_sq) + (int)floorf(p.y * inv_sq)) & 1;
                col3 = rt + REXSIM_RT_CHECK + 3 * parity;
            } else {
                col3 = rt + REXSIM_RT_COLOR + 3 * who;
            }
            const float lam = fmaxf(0.f, dot(nrm, mk(rt[REXSIM_RT_LIGHT], rt[REXSIM_RT_LIGHT + 1], rt[REXSIM_RT_LIGHT + 2])));
            const float shade = fmaf(rt[REXSIM_RT_LIGHT + 4], lam, rt[REXSIM_RT_LIGHT + 3]);
            rgbf[0] = col3[0] * shade; rgbf[1] = col3[1] * shade; rgbf[2] = col3[2] * shade;
        }
    }
    uint8_t* out = A.rgb + (((size_t)blockIdx.y * A.H + row) * A.W + col) * 3;
#pragma unroll
    for (int c = 0; c < 3; c++) out[c] = (uint8_t)fminf(fmaxf(rgbf[c] * 255.f + 0.5f, 0.f), 255.f);
}

cudaError_t launch_render(const Params& P, const float* rt, const float* zrange, const int32_t* idx, int k, int W, int H,
                          float distance, float yaw_deg, float pitch_deg, uint8_t* rgb, cudaStream_t st, int* launches) {
    RenderArgs A;
    A.sf = P.sf; A.si = P.si; A.model = P.model; A.rt = rt; A.fields = P.cfg.fields; A.zoff = P.field_zoff; A.zrange = zrange;
    A.idx = idx; A.err = P.err; A.N = P.N; A.terrain = P.cfg.terrain; A.arm = P.cfg.num_motors == 18; A.toe_npts = P.cfg.toe_npts;
    A.W = W; A.H = H; A.dist = distance;
    A.yaw = yaw_deg * (float)(3.14159265358979323846 / 180.0); A.pitch = pitch_deg * (float)(3.14159265358979323846 / 180.0);
    const int tiles_y = (H + RT_TILE - 1) / RT_TILE;
    A.tiles_x = (W + RT_TILE - 1) / RT_TILE;
    for (int i0 = 0; i0 < k; i0 += 65535) {          // gridDim.y <= 65535 images per launch
        const int n = min(k - i0, 65535);
        A.image0 = i0;
        A.rgb = rgb + (size_t)i0 * H * W * 3;
        render_kernel<<<dim3(A.tiles_x * tiles_y, n), dim3(RT_TILE, RT_TILE), 0, st>>>(A);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        ++*launches;
    }
    return cudaSuccess;
}

}  // namespace rexsim

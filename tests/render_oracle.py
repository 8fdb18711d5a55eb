"""fp64 numpy oracle of the rgb_array renderer (rex_gym_b200/csrc/rexsim_render.cu).  Test infrastructure only.

It draws the same picture as the kernel from the fp64 oracle's own kinematics (oracle/rexsim_oracle.c kinematics(), reached
through render_oracle_poses.c) and the model JSON's collision geometry, written independently of the kernel: every convex
shape is the intersection of its convex hull's face planes (scipy), cylinders are solved as quadrics, and the heightfield
is marched over all rays at once.  Colours, light, checker, sky and lens come from the same render table the kernel reads
(rex_gym_b200.model_tables.pack_render_tables).

Besides the image it returns a per-pixel surface-patch id: -1 sky; shape s, face f -> (s + 1) * 1000 + f (shape order of the
kernel: 3 base boxes, 12 leg boxes, 4 toes, 6 arm cylinders, arm box); ground -> 2**50 + checker square and heightfield
triangle.  Within one patch the shade is constant (flat faces) or smooth (cylinder sides), so where fp32 and fp64 disagree on
a pixel's colour the id image changes within one pixel of it.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
from scipy.spatial import ConvexHull

from oracle import oracle as O
from rex_gym_b200 import model_tables as MT

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_LIB = None
_SIMS = {}


def _lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="render_oracle_"), "librender_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-std=c11", "-fopenmp", "-ffp-contract=off", "-w",
                               "-I", os.path.join(ROOT, "oracle"), "-o", out, os.path.join(HERE, "render_oracle_poses.c"), "-lm"])
        _LIB = C.CDLL(out)
        _LIB.rexo_create.restype = C.c_void_p
        _LIB.rexo_create.argtypes = [C.POINTER(O.RexoModel), C.POINTER(O.RexoConfig)]
        _LIB.rexo_env.restype = C.POINTER(O.RexoEnv)
        _LIB.rexo_env.argtypes = [C.c_void_p, C.c_int]
        _LIB.rexo_link_poses.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return _LIB


def link_poses(mark, pos, quat, q):
    """[nb][3][3] body -> world rotations and [nb][3] origins of a robot at base pose (pos, quat xyzw) and joint angles q."""
    L = _lib()
    if mark not in _SIMS:
        model, j = O.load_model(mark)
        c = O.RexoConfig()
        c.num_envs, c.task, c.signal, c.terrain = 1, O.TASKS["standup" if mark == "arm" else "walk"], O.SIGNALS["ol"], 0
        c.action_repeat, c.solver_iterations, c.sim_dt, c.settle_on_reset, c.gait_clock_scale = 5, 60, 0.001, 0, 1.0
        _SIMS[mark] = (model, c, L.rexo_create(C.byref(model), C.byref(c)))
    model, _, h = _SIMS[mark]
    e = L.rexo_env(h, 0).contents
    for a in range(3):
        e.pos[a] = float(pos[a])
    for a in range(4):
        e.quat[a] = float(quat[a])
    for a in range(len(q)):
        e.q[a] = float(q[a])
    nb = model.nb
    R, p = np.zeros((nb, 9)), np.zeros((nb, 3))
    L.rexo_link_poses(h, 0, R.ctypes.data, p.ctypes.data)
    return R.reshape(nb, 3, 3), p


def camera(target, distance=1.0, yaw=0.0, pitch=-30.0):
    """Bullet computeViewMatrixFromYawPitchRoll (up axis z) + computeViewMatrixFromPositions: eye, forward, side, up."""
    y, p = np.radians(yaw), np.radians(pitch)
    Rz = np.array([[np.cos(y), -np.sin(y), 0], [np.sin(y), np.cos(y), 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, np.cos(p), -np.sin(p)], [0, np.sin(p), np.cos(p)]])
    R = Rz @ Rx
    target = np.asarray(target, dtype=np.float64)
    eye = target + R @ np.array([0.0, -distance, 0.0])
    up = R @ np.array([0.0, 0.0, 1.0])
    f = (target - eye) / np.linalg.norm(target - eye)
    s = np.cross(f, up)
    s /= np.linalg.norm(s)
    u = np.cross(s, f)
    return eye, f, s, u, up


def rays(f, s, u, width, height, fov_deg=MT.CAMERA_FOV_DEG):
    """[H][W][3] pixel rays, f component 1 (the ray parameter of a hit is its view depth)."""
    th = np.tan(np.radians(fov_deg) / 2)
    x = (2 * np.arange(width) + 1) / width - 1
    y = 1 - (2 * np.arange(height) + 1) / height
    return f + (x[None, :, None] * th * width / height) * s + (y[:, None, None] * th) * u


def _planes(points):
    """Unique outward face planes (n, d) of the convex hull of points: inside where n . x <= d."""
    eq = ConvexHull(points).equations
    out = []
    for e in eq:
        if not any(np.dot(e[:3], o[:3]) > 1 - 1e-9 and abs(e[3] - o[3]) < 1e-12 for o in out):
            out.append(e)
    out = np.array(out)
    return out[:, :3], -out[:, 3]


def world_shapes(mark, pos, quat, q):
    """Posed shapes in the kernel's order: ("poly", normals, offsets, centre, radius) or ("cyl", centre, axis, radius, half)."""
    j = MT.load_model_json(mark)
    bodies = j["bodies"]
    R, p = link_poses(mark, pos, quat, q)

    def poly(b, s):
        P = np.asarray(s["points"]) @ R[b].T + p[b]
        n, d = _planes(P)
        c = 0.5 * (P.min(0) + P.max(0))
        return ("poly", n, d, c, np.linalg.norm(P - c, axis=1).max())
    shapes = [poly(0, s) for s in bodies[0]["shapes"] if s["kind"] == "box"]
    for leg in range(4):
        for bi in range(3):
            b = 1 + 3 * leg + bi
            shapes.append(poly(b, [s for s in bodies[b]["shapes"] if s["kind"] == "box"][0]))
    for leg in range(4):
        b = 3 + 3 * leg
        shapes.append(poly(b, [s for s in bodies[b]["shapes"] if s["kind"] == "hull"][0]))
    if mark == "arm":
        for k in range(6):
            b = 13 + k
            s = [s for s in bodies[b]["shapes"] if s["kind"] == "cylinder"][0]
            c = R[b] @ np.asarray(s["origin_xyz"]) + p[b]
            a = R[b] @ np.asarray(s["origin_rot"])[:, 2]
            shapes.append(("cyl", c, a, s["radius"], 0.5 * s["length"]))
        b = 17
        shapes.append(poly(b, [s for s in bodies[b]["shapes"] if s["kind"] == "box"][0]))
    return shapes


def _hit_poly(eye, r, n, d):
    denom = r @ n.T                         # [P][K]
    dist = d - n @ eye                      # [K]
    with np.errstate(divide="ignore", invalid="ignore"):
        t = dist / denom
    t_in = np.where(denom < 0, t, -np.inf)
    t_out = np.where(denom > 0, t, np.inf)
    para_out = ((denom == 0) & (dist < 0)).any(1)
    te, face = t_in.max(1), t_in.argmax(1)
    ok = (te > 0) & (te <= t_out.min(1)) & ~para_out
    return np.where(ok, te, np.inf), n[face], face


def _hit_cyl(eye, r, c, a, rad, half):
    w = eye - c
    oa, ra = w @ a, r @ a
    wp = np.broadcast_to(w - oa * a, r.shape)
    rp = r - ra[:, None] * a
    A = (rp * rp).sum(1)
    B = (wp * rp).sum(1)
    Cc = (wp * wp).sum(1) - rad * rad
    with np.errstate(divide="ignore", invalid="ignore"):
        t1, t2 = (half - oa) / ra, (-half - oa) / ra
        cap_in = np.where(ra != 0, np.minimum(t1, t2), np.where(abs(oa) <= half, -np.inf, np.nan))
        cap_out = np.where(ra != 0, np.maximum(t1, t2), np.where(abs(oa) <= half, np.inf, np.nan))
        disc = B * B - A * Cc
        sq = np.sqrt(np.maximum(disc, 0))
        side_in = np.where(A > 0, (-B - sq) / A, np.where(Cc <= 0, -np.inf, np.nan))
        side_out = np.where(A > 0, (-B + sq) / A, np.where(Cc <= 0, np.inf, np.nan))
    side_in = np.where((A > 0) & (disc < 0), np.nan, side_in)
    te = np.maximum(cap_in, side_in)
    tx = np.minimum(cap_out, side_out)
    ok = (te > 0) & (te <= tx) & np.isfinite(te)
    side = side_in > cap_in
    qpt = wp + te[:, None] * rp
    with np.errstate(divide="ignore", invalid="ignore"):
        nside = qpt / np.linalg.norm(qpt, axis=1, keepdims=True)
    ncap = np.where((ra < 0)[:, None], a, -a)       # the cap the ray enters faces against it
    nrm = np.where(side[:, None], nside, ncap)
    face = np.where(side, 2, np.where(ra < 0, 1, 0))
    return np.where(ok, te, np.inf), nrm, face


GROUND_ID = 1 << 50


def _ground(eye, r, best, terrain, heights, zoff, zlo, zhi):
    """Nearest ground hit below best: t, normal, heightfield triangle id (-1 plane / outside the field)."""
    P = len(r)
    t_hit = np.full(P, np.inf)
    nrm = np.tile([0.0, 0.0, 1.0], (P, 1))
    tri_id = np.full(P, -1, np.int64)
    if terrain != "random":
        with np.errstate(divide="ignore", invalid="ignore"):
            t = -eye[2] / r[:, 2]
        ok = (r[:, 2] < 0) & (t > 0) & (t < best)
        t_hit[ok] = t[ok]
        return t_hit, nrm, tri_id
    g0 = eye[:2] * 20 + 127.5
    dg = r[:, :2] * 20
    with np.errstate(divide="ignore", invalid="ignore"):
        tp = (zlo - eye[2]) / r[:, 2]
    gp = g0 + tp[:, None] * dg
    outside = (gp < 0).any(1) | (gp > 255).any(1)
    ok = (r[:, 2] < 0) & (tp > 0) & (tp < best) & outside
    t_hit[ok] = tp[ok]
    best = np.minimum(best, t_hit)
    ta, tb = np.zeros(P), best.copy()
    for denom, dist in ((r[:, 2], zhi - eye[2]), (-r[:, 2], eye[2] - zlo), (dg[:, 0], 255 - g0[0]), (-dg[:, 0], np.full(P, g0[0])),
                        (dg[:, 1], 255 - g0[1]), (-dg[:, 1], np.full(P, g0[1]))):
        dist = np.broadcast_to(dist, (P,))
        with np.errstate(divide="ignore", invalid="ignore"):
            t = dist / denom
        ta = np.where(denom < 0, np.maximum(ta, t), ta)
        tb = np.where(denom > 0, np.minimum(tb, t), tb)
        tb = np.where((denom == 0) & (dist < 0), -1.0, tb)
    act = np.nonzero(ta <= tb)[0]
    ix = np.clip(np.floor(g0[0] + ta[act] * dg[act, 0]), 0, 254).astype(np.int64)
    iy = np.clip(np.floor(g0[1] + ta[act] * dg[act, 1]), 0, 254).astype(np.int64)
    t = ta[act]
    h = heights.astype(np.float64)
    while act.size:
        dx, dy, rz = dg[act, 0], dg[act, 1], r[act, 2]
        with np.errstate(divide="ignore", invalid="ignore"):
            tx = np.where(dx != 0, (ix + (dx > 0) - g0[0]) / dx, np.inf)
            ty = np.where(dy != 0, (iy + (dy > 0) - g0[1]) / dy, np.inf)
        tn = np.minimum(np.minimum(tx, ty), tb[act])
        h00, h10, h01, h11 = h[iy, ix], h[iy, ix + 1], h[iy + 1, ix], h[iy + 1, ix + 1]
        u0, v0 = g0[0] - ix, g0[1] - iy
        th = np.full(act.size, np.inf)
        hx, hy, tri = np.zeros(act.size), np.zeros(act.size), np.zeros(act.size, np.int64)
        for k, (a, b) in enumerate(((h11 - h01, h01 - h00), (h10 - h00, h11 - h10))):
            f0 = eye[2] + zoff - h00 - a * u0 - b * v0
            f1 = rz - a * dx - b * dy
            with np.errstate(divide="ignore", invalid="ignore"):
                tt = -f0 / f1
            u, v = u0 + tt * dx, v0 + tt * dy
            ok = (f1 != 0) & (tt >= t) & (tt <= tn) & (tt < th) & ((v >= u) == (k == 0))
            th = np.where(ok, tt, th)
            hx, hy, tri = np.where(ok, a, hx), np.where(ok, b, hy), np.where(ok, k, tri)
        hit = np.isfinite(th)
        if hit.any():
            i = act[hit]
            t_hit[i] = th[hit]
            nn = np.stack([-hx[hit] * 20, -hy[hit] * 20, np.ones(hit.sum())], 1)
            nrm[i] = nn / np.linalg.norm(nn, axis=1, keepdims=True)
            tri_id[i] = (iy[hit] * 255 + ix[hit]) * 2 + tri[hit]
        go = ~hit & (tn < tb[act])
        stepx = tx <= ty
        ix = np.where(stepx, ix + np.where(dx > 0, 1, -1), ix)
        iy = np.where(stepx, iy, iy + np.where(dy > 0, 1, -1))
        go &= (ix >= 0) & (ix <= 254) & (iy >= 0) & (iy <= 254)
        act, ix, iy, t = act[go], ix[go], iy[go], tn[go]
    return t_hit, nrm, tri_id


def render(mark, pos, quat, q, width=480, height=360, distance=1.0, yaw=0.0, pitch=-30.0, terrain="plane", heights=None,
           draw_robot=True):
    """(rgb uint8 [H][W][3], surface-patch id int64 [H][W]) of one robot.  heights: the env's [256][256] field (terrain 'random').
    draw_robot=False: the same camera over the ground alone."""
    table = MT.pack_render_tables(mark).astype(np.float64)
    eye, f, s, u, _ = camera(pos, distance, yaw, pitch)
    r = rays(f, s, u, width, height, table[MT.RT_CAM]).reshape(-1, 3)
    P = len(r)
    best = np.full(P, np.inf)
    nrm = np.zeros((P, 3))
    ids = np.full(P, -1, np.int64)
    rr = (r * r).sum(1)
    for k, sh in enumerate(world_shapes(mark, pos, quat, q) if draw_robot else []):
        c, rad = (sh[3], sh[4]) if sh[0] == "poly" else (sh[1], np.hypot(sh[3], sh[4]))
        d = c - eye
        tc = r @ d
        sel = np.nonzero(d @ d * rr - tc * tc <= rad * rad * rr * (1 + 1e-6))[0]
        if not sel.size:
            continue
        if sh[0] == "poly":
            t, n, face = _hit_poly(eye, r[sel], sh[1], sh[2])
        else:
            t, n, face = _hit_cyl(eye, r[sel], sh[1], sh[2], sh[3], sh[4])
        better = t < best[sel]
        i = sel[better]
        best[i], nrm[i], ids[i] = t[better], n[better], (k + 1) * 1000 + face[better]
    zoff = zlo = zhi = 0.0
    if terrain == "random":
        hmin, hmax = float(heights.min()), float(heights.max())
        zoff = 0.5 * (hmin + hmax)
        zlo, zhi = hmin - zoff, hmax - zoff
    tg, ng, tri = _ground(eye, r, best.copy(), terrain, heights, zoff, zlo, zhi)
    g = tg < best
    best[g], nrm[g] = tg[g], ng[g]
    pg = eye + best[:, None] * r
    with np.errstate(invalid="ignore"):
        cx = np.floor(pg[:, 0] / table[MT.RT_CHECK + 6]).astype(np.int64, copy=False) if g.any() else np.zeros(P, np.int64)
        cy = np.floor(pg[:, 1] / table[MT.RT_CHECK + 6]).astype(np.int64, copy=False) if g.any() else np.zeros(P, np.int64)
    ids[g] = GROUND_ID + ((cx[g] & 0x3FF) << 30) + ((cy[g] & 0x3FF) << 20) + (tri[g] + 1)
    near, far = table[MT.RT_CAM + 1], table[MT.RT_CAM + 2]
    vis = np.isfinite(best) & (best >= near) & (best <= far)
    ids[~vis] = -1
    cols = table[MT.RT_COLOR:MT.RT_COLOR + 3 * MT.RT_NSHAPES].reshape(-1, 3)
    base = np.tile(table[MT.RT_SKY:MT.RT_SKY + 3], (P, 1))
    shape_idx = ids // 1000 - 1
    sh = vis & ~g
    base[sh] = cols[shape_idx[sh]]
    gv = vis & g
    par = ((cx + cy) & 1)[gv]
    base[gv] = table[MT.RT_CHECK:MT.RT_CHECK + 6].reshape(2, 3)[par]
    light = table[MT.RT_LIGHT:MT.RT_LIGHT + 3]
    shade = table[MT.RT_LIGHT + 3] + table[MT.RT_LIGHT + 4] * np.maximum(0.0, nrm @ light)
    rgb = np.where(vis[:, None], base * shade[:, None], base)
    img = np.clip(np.floor(rgb * 255 + 0.5), 0, 255).astype(np.uint8)
    return img.reshape(height, width, 3), ids.reshape(height, width)

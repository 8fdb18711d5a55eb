"""Pack the URDF-derived tables (model/rex_<mark>.json, produced by tools/compile_urdf.py from
rex_gym/util/pybullet_data/assets/urdf/rex.urdf) into the flat float32 table the kernels TMA-load
(layout: include/rexsim.h REXSIM_MT_*)."""
import json
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
MT_BASE, MT_LEG, MT_TOE, MT_BOX, MT_BASEBOX, MT_FLOATS = 0, 16, 208, 592, 880, 952
MT_ARM, ARM_STRIDE, MT_ARMPTS, ARMPTS_N = 952, 32, 952 + 192, 104
MT_FLOATS_ARM = MT_ARMPTS + 3 * ARMPTS_N
# render table (include/rexsim.h REXSIM_RT_*): light, sky, ground checker, camera lens, shape colours and the fixed geometry the
# renderer needs beyond the model table
RT_LIGHT, RT_SKY, RT_CHECK, RT_CAM, RT_COLOR, RT_TOE, RT_TOESPH, RT_CYL, RT_ARMBOX, RT_FLOATS = 0, 5, 8, 15, 18, 96, 384, 388, 436, 464
RT_NSHAPES = 26
# What is not URDF data: a light from above, behind the default camera's left shoulder; Lambert + ambient weights; a grey 1 m
# checker on the ground; a pale sky.  The camera lens is the reference's (rex_gym_env.py:428-431: fov 60, near 0.1, far 100).
LIGHT_DIR = (-0.4, -0.6, 1.0)
AMBIENT, DIFFUSE = 0.35, 0.65
SKY_RGB = (0.62, 0.76, 0.92)
CHECKER_RGB = ((0.80, 0.80, 0.80), (0.55, 0.55, 0.55))
CHECKER_SIZE = 1.0
CAMERA_FOV_DEG, CAMERA_NEAR, CAMERA_FAR = 60.0, 0.1, 100.0
MAX_TOE_PTS = 96     # profile vertices of the toe prism ((x, z) pairs: 2 * 96 floats fit the 384-float toe block)
# Margin added to the toe hull's reach.  Bullet's URDF importer puts 1 mm on convex hulls, but the PyBullet trajectories
# recovered from the reference's checkpoints (25 episodes, identical free fall from z = 0.21) put the touchdown where the
# exact hull reaches 0.25 mm LESS than its vertices (one 1 ms sub-step of the 0.32 m/s fall): -0.25 mm halves the joint
# error of the touchdown steps (3.0e-3 -> 1.9e-3 rad) and lowers the 300-step replay error by 6 %; +1 mm doubles it.
# One scalar fitted to one datum; a spawn height of 0.21025 m would be indistinguishable (tests/test_pybullet_goldens.py).
TOE_MARGIN = -0.00025
LINK_DAMPING = 0.04               # btMultiBody m_linearDamping = m_angularDamping, applied to every link
MAX_COORDINATE_VELOCITY = 100.0   # btMultiBody m_maxCoordinateVelocity


def _rpy_to_mat(rpy):
    r, p, y = rpy
    cr, sr, cp, sp, cy, sy = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
    rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    return rz @ ry @ rx          # URDF fixed-axis roll, pitch, yaw


def _is_diag(I):
    I = np.asarray(I, dtype=np.float64)
    return bool(np.all(I[~np.eye(3, dtype=bool)] == 0.0))


def _sym6(I):
    I = np.asarray(I, dtype=np.float64)
    return [I[0, 0], I[1, 1], I[2, 2], I[0, 1], I[0, 2], I[1, 2]]


def load_model_json(mark="base"):
    with open(os.path.join(HERE, "model", f"rex_{mark}.json")) as f:
        return json.load(f)


def pack_model_tables(mark="base"):
    """Returns (float32[MT_FLOATS], toe_npts).  Raises ValueError when the model does not have the leg
    structure the kernels assume (x-axis shoulder, y-axis leg and foot, unrotated joint frames)."""
    j = load_model_json(mark)
    bodies = j["bodies"]
    if len(bodies) < 13:
        raise ValueError("model must have a base and four 3-joint legs")
    arm = mark == "arm"
    if arm and len(bodies) != 19:
        raise ValueError("arm model must have six arm bodies after the legs")
    t = np.zeros(MT_FLOATS_ARM if arm else MT_FLOATS, dtype=np.float64)
    b0 = bodies[0]
    t[MT_BASE + 0] = b0["mass"]
    t[MT_BASE + 1:MT_BASE + 4] = b0["com"]
    t[MT_BASE + 4:MT_BASE + 10] = _sym6(b0["inertia"])
    t[MT_BASE + 10] = j["root_mass"]
    t[MT_BASE + 11:MT_BASE + 14] = j["root_inertia"]
    t[MT_BASE + 14] = 1.0 if _is_diag(b0["inertia"]) else 0.0       # flag: inertia tensor diagonal in the body frame
    boxes = [s for s in b0["shapes"] if s["kind"] == "box"]
    if len(boxes) != 3:
        raise ValueError("expected base + 2 chassis collision boxes")
    for k, s in enumerate(boxes):
        t[MT_BASEBOX + 24 * k:MT_BASEBOX + 24 * (k + 1)] = np.asarray(s["points"]).reshape(-1)
    axes = ([1, 0, 0], [0, 1, 0], [0, 1, 0])
    npts = None
    for leg in range(4):
        for bi in range(3):
            b = bodies[1 + 3 * leg + bi]
            if b["parent"] != (0 if bi == 0 else 3 * leg + bi):
                raise ValueError("unexpected kinematic tree")
            if not np.allclose(b["axis"], axes[bi]) or np.any(np.abs(b["joint_rpy"]) > 0):
                raise ValueError("kernels assume x/y/y joint axes and unrotated joint frames")
            o = MT_LEG + 48 * leg + 16 * bi
            t[o:o + 3] = b["joint_xyz"]
            t[o + 3] = b["mass"]
            t[o + 4:o + 7] = b["com"]
            t[o + 7] = b["lower"]
            t[o + 8:o + 14] = _sym6(b["inertia"])
            t[o + 14] = b["upper"]
            t[o + 15] = 1.0 if _is_diag(b["inertia"]) else 0.0
            box = [s for s in b["shapes"] if s["kind"] == "box"]
            if len(box) != 1:
                raise ValueError("expected one collision box per leg body")
            ob = MT_BOX + 72 * leg + 24 * bi
            t[ob:ob + 24] = np.asarray(box[0]["points"]).reshape(-1)
            hull = [s for s in b["shapes"] if s["kind"] == "hull"]
            if bi == 2:
                # the toe is a prism (tools/compile_urdf.py support_polytope): a convex (x, z) profile extruded over
                # y in [-w, +w] in the foot body frame, identical on the four feet -> one shared [npts][2] profile + w
                if len(hull) != 1 or "prism_profile_points" not in hull[0]:
                    raise ValueError("expected one prism toe hull on the foot body")
                pts = np.asarray(hull[0]["points"])
                n = int(hull[0]["prism_profile_points"])
                lo, hi = pts[:n], pts[n:]
                if len(pts) != 2 * n or n > MAX_TOE_PTS or not np.allclose(lo[:, [0, 2]], hi[:, [0, 2]], atol=1e-12):
                    raise ValueError("toe hull is not a prism of <= %d profile vertices" % MAX_TOE_PTS)
                w = float(hi[0, 1])
                if not (np.allclose(lo[:, 1], -w, atol=1e-9) and np.allclose(hi[:, 1], w, atol=1e-9) and w > 0):
                    raise ValueError("toe prism must be centred on y = 0 in the foot frame")
                prof = lo[:, [0, 2]]
                if npts is None:
                    npts, prof0, w0 = n, prof, w
                    t[MT_TOE:MT_TOE + 2 * n] = prof.reshape(-1)
                    t[MT_BASE + 15] = w            # toe half width (the pad word of the base block)
                elif n != npts or not np.allclose(prof, prof0, atol=1e-12) or abs(w - w0) > 1e-12:
                    raise ValueError("the four toe hulls must be identical in their foot frames")
    if arm:
        # collision points of each arm body, in the order the oracle scans them (oracle.load_model: contact group 9 + k)
        pts = [np.asarray(s["points"], dtype=np.float64).reshape(-1, 3) for k in range(6) for s in bodies[13 + k]["shapes"]]
        if sum(len(p) for p in pts) != ARMPTS_N:
            raise ValueError("expected %d arm collision points" % ARMPTS_N)
        start = 0
        for k in range(6):
            b = bodies[13 + k]
            if b["parent"] != (0 if k == 0 else 12 + k):
                raise ValueError("the arm must be one serial chain attached to the base")
            o = MT_ARM + ARM_STRIDE * k
            t[o:o + 3] = b["joint_xyz"]
            t[o + 3:o + 12] = _rpy_to_mat(b["joint_rpy"]).reshape(-1)      # child -> parent, row-major
            t[o + 12:o + 15] = b["axis"]
            t[o + 15] = b["mass"]
            t[o + 16:o + 19] = b["com"]
            t[o + 19:o + 25] = _sym6(b["inertia"])
            t[o + 25], t[o + 26] = b["lower"], b["upper"]
            p = np.concatenate([np.asarray(s["points"], dtype=np.float64).reshape(-1, 3) for s in b["shapes"]])
            t[o + 27], t[o + 28], t[o + 29] = len(p), start, np.linalg.norm(p, axis=1).max()
            t[MT_ARMPTS + 3 * start:MT_ARMPTS + 3 * (start + len(p))] = p.reshape(-1)
            start += len(p)
    return t.astype(np.float32), int(npts)


def contact_breaking_distance(mark="base"):
    """Manifold breaking distance of the toe / ground pair the way Bullet derives it: btCollisionDispatcher::getNewManifold with
    CD_USE_RELATIVE_CONTACT_BREAKING_THRESHOLD (the dispatcher default) takes min over the two shapes of
    getAngularMotionDisc() * gContactBreakingThreshold (0.02).  The toe link's collider is a btCompoundShape holding the hull
    under the URDF collision origin (rex.urdf:193: rpy 0 -0.4001 0, xyz 0 -0.01 0), so its disc comes from the compound's AABB:
    the hull's mesh-frame AABB grown by the importer margin (1 mm), pushed through btTransformAabb (|R| * half extents);
    disc = |centre| + |half extents|.  The 30 x 30 x 10 m ground box is far larger, so the toe decides: 0.81 mm."""
    j = load_model_json(mark)
    hull = [s for s in j["bodies"][3]["shapes"] if s["kind"] == "hull"][0]
    pts = np.asarray(hull["points"], dtype=np.float64) - np.array([0.0, 0.0, -0.115])        # foot body frame -> toe link frame (rex.urdf:233)
    R = _rpy_to_mat((0.0, -0.40010, 0.0)); t = np.array([0.0, -0.01, 0.0])
    mesh = (pts - t) @ R                                                                    # R^T (p - t): back to the stl frame
    lo, hi = mesh.min(0) - 0.001, mesh.max(0) + 0.001                                       # gUrdfDefaultCollisionMargin
    half, centre = 0.5 * (hi - lo), 0.5 * (hi + lo)
    half_w = np.abs(R) @ half                                                               # btTransformAabb
    centre_w = R @ centre + t
    return float((np.linalg.norm(centre_w) + np.linalg.norm(half_w)) * 0.02)


def toe_profile_planes(profile):
    """Edge planes of the convex toe profile ((x, z) vertices in order along its boundary, closed by the chord from the last to
    the first): [n][3] rows (nx, nz, d), outward unit normal and offset, inside where nx x + nz z <= d."""
    P = np.asarray(profile, dtype=np.float64)
    c = P.mean(0)
    out = []
    for i in range(len(P)):
        a, b = P[i], P[(i + 1) % len(P)]
        n = np.array([b[1] - a[1], a[0] - b[0]])
        n /= np.linalg.norm(n)
        if n @ (a - c) < 0:
            n = -n
        out.append([n[0], n[1], n @ a])
    out = np.array(out)
    if np.any(P @ out[:, :2].T - out[:, 2] > 1e-9):
        raise ValueError("toe profile is not convex in its stored order")
    return out


def render_shape_colors(mark="base"):
    """[26][3] rgb of the rendered shapes (URDF visual material of each shape's link), in the renderer's shape order: base +
    two chassis boxes, the 12 leg boxes (leg-major: shoulder, leg, foot), the four toes, the six arm cylinders, arm box."""
    j = load_model_json(mark)
    bodies = j["bodies"]
    cols = np.zeros((RT_NSHAPES, 3))

    def col(b, kind):
        shapes = [s for s in b["shapes"] if s["kind"] == kind]
        rgba = b["link_rgba"][shapes[0]["link"]]
        if rgba is None:
            raise ValueError("link %s has no visual material" % shapes[0]["link"])
        return rgba[:3]
    cols[0:3] = [b["link_rgba"][s["link"]][:3] for b in bodies[:1] for s in b["shapes"] if s["kind"] == "box"]
    for leg in range(4):
        for bi in range(3):
            cols[3 + 3 * leg + bi] = col(bodies[1 + 3 * leg + bi], "box")
        cols[15 + leg] = col(bodies[3 + 3 * leg], "hull")
    if mark == "arm":
        for k in range(6):
            cols[19 + k] = col(bodies[13 + k], "cylinder")
        cols[25] = col(bodies[17], "box")
    return cols


def pack_render_tables(mark="base"):
    """float32[RT_FLOATS] render table of `mark` (layout: include/rexsim.h REXSIM_RT_*), uploaded by rexsim_set_render_tables."""
    j = load_model_json(mark)
    bodies = j["bodies"]
    mt, npts = pack_model_tables(mark)
    t = np.zeros(RT_FLOATS, dtype=np.float64)
    L = np.asarray(LIGHT_DIR, dtype=np.float64)
    t[RT_LIGHT:RT_LIGHT + 3] = L / np.linalg.norm(L)
    t[RT_LIGHT + 3], t[RT_LIGHT + 4] = AMBIENT, DIFFUSE
    t[RT_SKY:RT_SKY + 3] = SKY_RGB
    t[RT_CHECK:RT_CHECK + 6] = np.asarray(CHECKER_RGB).reshape(-1)
    t[RT_CHECK + 6] = CHECKER_SIZE
    t[RT_CAM:RT_CAM + 3] = CAMERA_FOV_DEG, CAMERA_NEAR, CAMERA_FAR
    t[RT_COLOR:RT_COLOR + 3 * RT_NSHAPES] = render_shape_colors(mark).reshape(-1)
    prof = mt[MT_TOE:MT_TOE + 2 * npts].astype(np.float64).reshape(-1, 2)
    t[RT_TOE:RT_TOE + 3 * npts] = toe_profile_planes(prof).reshape(-1)
    w = float(mt[MT_BASE + 15])
    c = 0.5 * (prof.min(0) + prof.max(0))
    t[RT_TOESPH:RT_TOESPH + 3] = c[0], c[1], np.sqrt(((prof - c) ** 2).sum(1).max() + w * w) * (1 + 1e-5)
    if mark == "arm":
        for k in range(6):
            cyl = [s for s in bodies[13 + k]["shapes"] if s["kind"] == "cylinder"]
            if len(cyl) != 1:
                raise ValueError("expected one cylinder per arm body")
            s = cyl[0]
            o = RT_CYL + 8 * k
            t[o:o + 3] = s["origin_xyz"]
            t[o + 3:o + 6] = np.asarray(s["origin_rot"])[:, 2]          # cylinder axis = z of its origin frame
            t[o + 6], t[o + 7] = s["radius"], 0.5 * s["length"]
        boxes = [(k, s) for k in range(6) for s in bodies[13 + k]["shapes"] if s["kind"] == "box"]
        if len(boxes) != 1:
            raise ValueError("expected one arm box")
        t[RT_ARMBOX] = boxes[0][0]
        t[RT_ARMBOX + 1:RT_ARMBOX + 25] = np.asarray(boxes[0][1]["points"]).reshape(-1)
    return t.astype(np.float32)

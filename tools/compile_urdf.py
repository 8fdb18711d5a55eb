#!/usr/bin/env python3
"""URDF compiler: rex.urdf / rex_arm.urdf -> flat link/inertia/contact tables.

Reads the reference robot description where it lies (read-only) and emits the
*derived* tables the simulator consumes (rex_gym_b200/model/rex_<mark>.json).
Nothing from the URDF text is copied; the output is a merged-fixed-link tree with
composite masses, centres of mass, inertia tensors and contact sample points.

Rules restated from the reference call sites and Bullet's URDF importer
(pybullet==2.8.3, not vendored):

* `loadURDF` is called WITHOUT `URDF_USE_INERTIA_FROM_FILE`
  (rex_gym/model/rex.py:276-287), so the `<inertia ixx="100" ...>` values are
  dead: Bullet recomputes the inertia diagonal from the collision shape
  (box: m/12*(b^2+c^2); compound / convex hull: same formula on the local AABB;
  a link without collision shape gets a zero rotational inertia).
* No `<inertial><origin>` anywhere -> every URDF link's COM is its own origin.
* Fixed joints (chassis parts, leg covers, toes, arm tips) are kept by Bullet as
  0-DOF links; rigidly merging them into the parent is dynamically identical and
  is what we do here (13 moving bodies for `base`, 19 for `arm`).
* Toe collision = convex hull of stl/foot.stl (10 750 vertices).  We keep a
  K-point support polytope of that hull (extreme vertices in K directions).

Usage: python tools/compile_urdf.py [--ref /root/reference] [--out rex_gym_b200/model]
"""
import argparse
import json
import os
import struct
import xml.etree.ElementTree as ET

import numpy as np

URDF_MARGIN = 0.001  # Bullet gUrdfDefaultCollisionMargin (convex hull AABB inflation)


def rpy_to_mat(rpy):
    r, p, y = rpy
    cr, sr, cp, sp, cy, sy = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
    rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    return rz @ ry @ rx  # URDF fixed-axis roll, pitch, yaw


def vec(s, default=(0.0, 0.0, 0.0)):
    return np.array([float(x) for x in s.split()]) if s else np.array(default, dtype=float)


def load_stl_vertices(path, scale):
    data = open(path, "rb").read()
    n = struct.unpack("<I", data[80:84])[0]
    rec = np.dtype([("n", "<f4", 3), ("v", "<f4", (3, 3)), ("a", "<u2")])
    tri = np.frombuffer(data[84:84 + 50 * n], dtype=rec)
    v = tri["v"].reshape(-1, 3).astype(np.float64) * scale
    return np.unique(v, axis=0)


def support_polytope(verts):
    """Exact support set of the toe hull.  stl/foot.stl is a prism: a convex 2-D profile in the mesh x-z plane extruded
    along y (672 y-layers of the same tyre profile).  Its convex hull is therefore {profile hull vertices} x {y_min, y_max}:
    74 profile vertices; the ones on the flat top (mesh z == 0) can never be the deepest point against a ground below the
    robot and are dropped, leaving the curved part.  Every retained vertex is a true hull vertex, so the support function
    (deepest point along any downward direction) is exact -- an earlier 27-point subset under-estimated the reach by up
    to 0.4 mm between samples, which PyBullet trajectories recovered from the reference's checkpoints exposed as a
    touchdown that came one control step late (tools/dev_pybullet_replay.py)."""
    from scipy.spatial import ConvexHull
    xz = verts[:, [0, 2]]
    prof = xz[ConvexHull(xz).vertices]
    prof = prof[prof[:, 1] < -1e-4]                                  # drop the flat top edge
    prof = prof[np.argsort(np.arctan2(prof[:, 1], prof[:, 0]))]      # ordered along the arc
    y0, y1 = verts[:, 1].min(), verts[:, 1].max()
    return np.array([[x, y, z] for y in (y0, y1) for x, z in prof])


def parse_urdf(path, stl_dir):
    root = ET.parse(path).getroot()
    materials = {m.get("name"): vec(m.find("color").get("rgba")) for m in root.findall("material") if m.find("color") is not None}
    links = {}
    for ln in root.findall("link"):
        name = ln.get("name")
        mass = float(ln.find("inertial/mass").get("value"))
        # visual material: a named robot-level material or an inline colour; None for a link without a visual
        rgba = None
        mat = ln.find("visual/material")
        if mat is not None:
            rgba = vec(mat.find("color").get("rgba")) if mat.find("color") is not None else materials.get(mat.get("name"))
        shapes = []
        for col in ln.findall("collision"):
            org = col.find("origin")
            xyz = vec(org.get("xyz") if org is not None else None)
            rpy = vec(org.get("rpy") if org is not None else None)
            geom = col.find("geometry")
            for g in geom:
                if g.tag == "box":
                    shapes.append(dict(kind="box", size=vec(g.get("size")), xyz=xyz, rpy=rpy))
                elif g.tag == "cylinder":
                    shapes.append(dict(kind="cylinder", radius=float(g.get("radius")),
                                       length=float(g.get("length")), xyz=xyz, rpy=rpy))
                elif g.tag == "mesh":
                    fn = os.path.join(stl_dir, os.path.basename(g.get("filename")))
                    sc = vec(g.get("scale"), (1, 1, 1))[0]
                    shapes.append(dict(kind="hull", verts=load_stl_vertices(fn, sc), xyz=xyz, rpy=rpy))
        links[name] = dict(name=name, mass=mass, shapes=shapes, rgba=None if rgba is None else rgba.tolist())
    joints = []
    for jn in root.findall("joint"):
        org = jn.find("origin")
        ax = jn.find("axis")
        lim = jn.find("limit")
        joints.append(dict(
            name=jn.get("name"), type=jn.get("type"),
            parent=jn.find("parent").get("link"), child=jn.find("child").get("link"),
            xyz=vec(org.get("xyz") if org is not None else None),
            rpy=vec(org.get("rpy") if org is not None else None),
            axis=vec(ax.get("xyz")) if ax is not None else np.array([1.0, 0, 0]),
            lower=float(lim.get("lower")) if lim is not None else 0.0,
            upper=float(lim.get("upper")) if lim is not None else 0.0))
    return links, joints


def shape_local_aabb_halfext(sh):
    """Half extents of the shape's own local AABB (before the collision origin)."""
    if sh["kind"] == "box":
        return 0.5 * sh["size"], np.zeros(3)
    if sh["kind"] == "cylinder":  # URDF cylinder axis = z
        return np.array([sh["radius"], sh["radius"], 0.5 * sh["length"]]), np.zeros(3)
    v = sh["verts"]
    return 0.5 * (v.max(0) - v.min(0)) + URDF_MARGIN, 0.5 * (v.max(0) + v.min(0))


def link_inertia_diag(link):
    """Bullet shape-derived inertia diagonal (see module docstring)."""
    m, shapes = link["mass"], link["shapes"]
    if not shapes:      # an empty btCompoundShape: its AABB is the margin alone (2 mm cube) -- 3.3e-7 kg m^2 for the 0.5 kg leg covers
        l = 2 * URDF_MARGIN
        return m / 12.0 * np.array([2 * l * l, 2 * l * l, 2 * l * l])
    ident = len(shapes) == 1 and not shapes[0]["xyz"].any() and not shapes[0]["rpy"].any()
    if ident and shapes[0]["kind"] == "box":
        lx, ly, lz = shapes[0]["size"]
    else:  # compound: AABB of the children's (rotated) local AABBs
        lo, hi = np.full(3, np.inf), np.full(3, -np.inf)
        for sh in shapes:
            he, ce = shape_local_aabb_halfext(sh)
            R = rpy_to_mat(sh["rpy"])
            c = R @ ce + sh["xyz"]
            e = np.abs(R) @ he
            lo, hi = np.minimum(lo, c - e), np.maximum(hi, c + e)
        # btCompoundShape::getAabb grows the children's box by the compound's own margin, and the URDF importer gives every link
        # compound gUrdfDefaultCollisionMargin (BulletUrdfImporter::convertLinkCollisionShapes).  The recorded PyBullet episodes
        # select it: with the 1 mm the gallop-ol replay error drops by 30 % over the first 150 steps (3.3e-3 -> 2.3e-3 rad), walk-ol
        # roll/pitch by 16 % (tests/test_pybullet_goldens.py)
        lx, ly, lz = hi - lo + 2 * URDF_MARGIN
    return m / 12.0 * np.array([ly * ly + lz * lz, lx * lx + lz * lz, lx * lx + ly * ly])


def shape_points(sh):
    """Contact sample points of a shape in its link frame."""
    R = rpy_to_mat(sh["rpy"])
    if sh["kind"] == "box":
        h = 0.5 * sh["size"]
        P = np.array([[sx * h[0], sy * h[1], sz * h[2]] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)])
    elif sh["kind"] == "cylinder":
        r, h = sh["radius"], 0.5 * sh["length"]
        P = np.array([[r * np.cos(a), r * np.sin(a), s * h] for s in (-1, 1) for a in np.arange(8) * np.pi / 4])
    else:
        P = support_polytope(sh["verts"])
    return P @ R.T + sh["xyz"]


def compile_model(urdf_path, stl_dir, motor_names):
    links, joints = parse_urdf(urdf_path, stl_dir)
    child_joint = {j["child"]: j for j in joints}
    root = [n for n in links if n not in child_joint][0]
    bodies = []  # merged moving bodies

    def add_body(link_name, parent_body, joint):
        # gather this link + all fixed descendants into one rigid body
        parts = []  # (link, R, t) placement of the link frame in the body frame

        def gather(name, R, t):
            parts.append((links[name], R, t))
            for j in joints:
                if j["parent"] == name and j["type"] == "fixed":
                    Rj = rpy_to_mat(j["rpy"])
                    gather(j["child"], R @ Rj, R @ j["xyz"] + t)
        gather(link_name, np.eye(3), np.zeros(3))
        mass = sum(p[0]["mass"] for p in parts)
        com = sum(p[0]["mass"] * p[2] for p in parts) / mass
        I = np.zeros((3, 3))
        shapes = []
        for lk, R, t in parts:
            Il = R @ np.diag(link_inertia_diag(lk)) @ R.T
            d = t - com
            I += Il + lk["mass"] * (d @ d * np.eye(3) - np.outer(d, d))
            for sh in lk["shapes"]:
                shapes.append(dict(link=lk["name"], kind=sh["kind"],
                                   points=(shape_points(sh) @ R.T + t).tolist()))
                if sh["kind"] == "hull":     # prism: first half = profile on the y_min face, second half = y_max face
                    shapes[-1]["prism_profile_points"] = len(shapes[-1]["points"]) // 2
                if sh["kind"] == "cylinder":  # the renderer draws true capped cylinders: axis = z of the origin frame
                    shapes[-1].update(radius=sh["radius"], length=sh["length"], origin_xyz=(R @ sh["xyz"] + t).tolist(),
                                      origin_rot=(R @ rpy_to_mat(sh["rpy"])).tolist())
        b = dict(name=link_name, parent=parent_body, mass=mass, com=com.tolist(), inertia=I.tolist(),
                 shapes=shapes, links=[p[0]["name"] for p in parts])
        b["link_rgba"] = {p[0]["name"]: p[0]["rgba"] for p in parts}      # URDF visual material of every merged link
        if joint is not None:
            b.update(joint=joint["name"], joint_xyz=joint["xyz"].tolist(), joint_rpy=joint["rpy"].tolist(),
                     axis=joint["axis"].tolist(), lower=joint["lower"], upper=joint["upper"])
        idx = len(bodies)
        bodies.append(b)
        for j in joints:
            if j["type"] != "fixed" and any(j["parent"] == p[0]["name"] for p in parts):
                # joint frame placement in this merged body's frame
                for lk, R, t in parts:
                    if lk["name"] == j["parent"]:
                        jj = dict(j)
                        jj["xyz"] = R @ j["xyz"] + t
                        # rotation of the parent part is identity for every movable joint in both URDFs
                        assert np.allclose(R, np.eye(3))
                        add_body(j["child"], idx, jj)
        return idx

    add_body(root, -1, None)
    jname_to_body = {b["joint"]: i for i, b in enumerate(bodies) if "joint" in b}
    # Bullet applies its default base damping (0.04) with the un-merged root link's own mass/inertia
    return dict(bodies=bodies, motor_bodies=[jname_to_body[n] for n in motor_names],
                motor_names=motor_names, total_mass=sum(b["mass"] for b in bodies),
                root_mass=links[root]["mass"], root_inertia=link_inertia_diag(links[root]).tolist())


BASE_MOTORS = [f"{p}{leg}{s}" for leg in ("front_left", "front_right", "rear_left", "rear_right")
               for p, s in (("motor_", "_shoulder"), ("motor_", "_leg"), ("foot_motor_", ""))]
ARM_MOTORS = [f"motor_arm_m{i}" for i in range(1, 7)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    ap.add_argument("--out", default=os.path.join(os.path.dirname(__file__), "..", "rex_gym_b200", "model"))
    a = ap.parse_args()
    udir = os.path.join(a.ref, "rex_gym/util/pybullet_data/assets/urdf")
    for mark, fn, motors in (("base", "rex.urdf", BASE_MOTORS), ("arm", "rex_arm.urdf", BASE_MOTORS + ARM_MOTORS)):
        model = compile_model(os.path.join(udir, fn), os.path.join(udir, "stl"), motors)
        model["mark"] = mark
        model["source"] = f"rex_gym/util/pybullet_data/assets/urdf/{fn} (derived tables, not a copy)"
        out = os.path.join(a.out, f"rex_{mark}.json")
        with open(out, "w") as f:
            json.dump(model, f, indent=1)
        print(mark, "bodies", len(model["bodies"]), "mass %.4f" % model["total_mass"], "->", out)


if __name__ == "__main__":
    main()

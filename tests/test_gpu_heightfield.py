"""Heightfield contact of the step kernel against the fp64 oracle, over the whole field, at its borders and beyond them.

On random terrain the step kernel (rex_gym_b200/csrc/rexsim_kernel.cu, "ground query") stages a 17 x 17-vertex window of the env's
field in shared memory once per control step (load_tile) and answers every contact query of the step's sub-steps from it
(ground_query<RANDOM>): near a border the window's origin is clamped into the field, a query beyond a border is clamped to the
border cell, and a query outside the window is clamped to the window and flagged with REXSIM_FLAG_TILE_MISS.  The oracle reads
the whole field.  So the start states here are placed where those differences would show:

  interior     points spread over the field, each at its own yaw
  cell         the base at cell fractions 0.01 / 0.5 / 0.99 in x and in y, and 1e-8 cells below a vertex line (where the
               fp32 and fp64 cell indices of the base differ by one)
  inside       5-10 cm inside each border and each corner (window origin clamped to 0 or 239)
  on           exactly on each border
  beyond       0.2 m beyond each border (every query clamped to the border cell)
  fallen       on its back, side, nose, knees (the poses of test_gpu_generic_path.py)
  stretch      on its back or side with one rear leg straight (foot at its lower limit) along +x or +y, the base at cell
               fraction 0.99 along that axis: the leg's end lies in the window's last cell, 0.347 m ahead of the base
               against a margin of 0.3505 m.  These are not dropped (the leg's motor would fold it back first): they start
               lowered to within the breaking distance of the ground, the leg straight at the first sub-step

on three banks: the default random bank (64 fields), a 300-field bank reached through env_offset (fields 256-299; field k is
field k % 4 of the random bank with one vertex 1 m from every placement raised by k mm, so every field has its own vertical offset), and synthetic
slopes (planes at 10 and 25 degrees in +x, +y and diagonally, restricted to +-1 m around the origin, and a 10-degree plane whose
two triangles per cell have different slopes): tilted normals, both plane_space branches and sliding (friction 0.25).  The step
kernel tests only sample points below z = 0.06 m, which holds the random bank's ground (within +-0.025 m of z = 0) with room to
spare; the slope fields keep their ground below z = -0.02 m around the placements through their vertical offset.

Every start state is dropped on the oracle from 1.5 cm above its local ground until its contacts exist (standing: all four toes
on the slopes, three on the random blocks) and taken from the sub-step before; test_placements_reach_their_contacts (CPU) pins
that.  No placement raises TILE_MISS, the stretched leg included: the window (origin floor(fx) - 8, 7-8 cells ahead of the base)
holds every query of these states.  Over the whole joint range no sampled point of an upright robot lies more than 0.348 m ahead
of its base, 2 mm inside the smallest margin ahead (7 cells, 0.35 m); with the body tilted a point can lie up to 0.362 m from the
base horizontally, so a tilted robot with a straight leg, its base at the top of its cell, can still leave the window (flagged).
"""
import math

import numpy as np
import pytest

from twin import (BODY_BITS, BUILDS, FOLDED, LAYOUT, NOISE, STATE_KEYS, SUB, TOE_BITS, UPPER_BITS, IterationBand,
                  compare_control_steps, compare_substeps, force_build, launched, make_env, make_oracle, qmul, quat, rot,
                  state_errors, sync)

CELL = 0.05
EDGE = 127.5 * CELL                                     # vertex 0 / 255 of a field: its borders at x, y = -+6.375 m
TILE_MISS = 8                                           # REXSIM_FLAG_TILE_MISS
BANKS = {"default": (64, 0), "big": (300, 255), "slopes": (7, 0)}   # (fields, env_offset): env i starts on (i + offset + 1) % fields
CLEAR = 0.015                                           # drop height above the local ground
STRETCH_CLEAR = 4e-4                                    # the stretched poses' lowest point: inside the 0.81 mm breaking distance


# ---- banks ---------------------------------------------------------------------------------------------------------
_FIELDS = {}


def _fields(bank):
    if bank in _FIELDS:
        return _FIELDS[bank]
    from oracle.oracle import make_fields
    if bank == "default":
        f = make_fields(64)
    elif bank == "big":
        base = make_fields(4)
        f = np.stack([base[k % 4] for k in range(300)])
        # vertex (ix 40, iy 200), at (-4.375, 3.625) m, more than 1 m from every placement, raised by k mm on field k
        f[:, 200, 40] += np.float32(1e-3) * np.arange(300, dtype=np.float32)
    else:
        c = (np.arange(256) - 127.5) * CELL
        x, y = np.meshgrid(c, c)                        # field[iy][ix]
        f = []
        for deg in (10, 25):
            t = math.tan(math.radians(deg))
            for s in (x, y, (x + y) / math.sqrt(2)):
                f.append(t * np.clip(s, -1, 1))
        ii, jj = np.meshgrid(np.arange(256), np.arange(256))
        inside = (np.abs(x) <= 1) & (np.abs(y) <= 1)
        f.append(math.tan(math.radians(10)) * np.clip(x, -1, 1) + 0.004 * ((ii + jj) % 2) * inside)   # checkerboard of 4 mm
        # the step kernel only tests sample points below z = 0.06 m (the random bank's ground lies within +-0.025 m): a spike at
        # vertex (0, 0) sets each field's vertical offset so that the ground within 0.4 m of the origin lies below z = -0.02 m
        near = (np.abs(x) <= 0.4) & (np.abs(y) <= 0.4)
        for g in f:
            g[0, 0] = 2 * (g[near].max() + 0.02) - g.min()
        f = np.stack(f) + 1.0
    f = np.ascontiguousarray(f, np.float32)
    _FIELDS[bank] = f
    return f


def _zoff(f):
    return 0.5 * (float(f.min()) + float(f.max()))


def _ground(f, zoff, px, py):
    """The oracle's triangle height and normal (fp64) at world points px, py of field f ([256][256], f[iy][ix])."""
    fx = np.clip(np.asarray(px) / CELL + 127.5, 0, 254.999)
    fy = np.clip(np.asarray(py) / CELL + 127.5, 0, 254.999)
    ix, iy = np.floor(fx).astype(int), np.floor(fy).astype(int)
    u, v = fx - ix, fy - iy
    h00, h10, h01, h11 = (f[iy + b, ix + a].astype(np.float64) for a, b in ((0, 0), (1, 0), (0, 1), (1, 1)))
    upper = v >= u
    hx = np.where(upper, h11 - h01, h10 - h00)
    hy = np.where(upper, h01 - h00, h11 - h10)
    n = np.stack([-hx / CELL, -hy / CELL, np.ones_like(hx)], -1)
    return h00 + hx * u + hy * v - zoff, n / np.linalg.norm(n, axis=-1, keepdims=True)


# ---- kinematics of the contact sample points (oracle model tables, fp64) --------------------------------------------------
_MODEL = {}


def _model():
    if not _MODEL:
        from oracle.oracle import load_model
        m, _ = load_model("base")
        npt = m.shape_start[m.nshape - 1] + m.shape_npts[m.nshape - 1]
        group = np.zeros(npt, int)
        for g in range(m.nshape):
            group[m.shape_start[g]:m.shape_start[g] + m.shape_npts[g]] = g
        sel = np.array([m.pt_terrain[i] for i in range(npt)], bool)
        _MODEL.update(m=m, pts=np.array([list(m.pts[i]) for i in range(npt)])[sel], body=np.array(m.pt_body[:npt])[sel],
                      margin=np.array(m.pt_margin[:npt])[sel], group=group[sel],
                      jpos=np.array([list(m.jpos[i]) for i in range(m.nb)]), jrot=np.array([list(m.jrot[i]) for i in range(m.nb)]).reshape(-1, 3, 3),
                      axis=np.array([list(m.axis[i]) for i in range(m.nb)]), parent=list(m.parent[:m.nb]))
    return _MODEL


def _axis_angle(a, t):
    a = np.asarray(a, float)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(t) * K + (1 - math.cos(t)) * K @ K


def _points(s):
    """World positions [P][3] and contact groups [P] of the points the heightfield contact samples, in state s."""
    M = _model()
    Rw, pw = [rot(s["quat"])], [np.asarray(s["pos"], float)]
    for i in range(1, len(M["parent"])):
        p = M["parent"][i]
        Rw.append(Rw[p] @ M["jrot"][i] @ _axis_angle(M["axis"][i], s["q"][i - 1]))
        pw.append(pw[p] + Rw[p] @ M["jpos"][i])
    Rw, pw = np.array(Rw), np.array(pw)
    return np.einsum("pab,pb->pa", Rw[M["body"]], M["pts"]) + pw[M["body"]], M["group"]


def _clearance(s, f, zoff):
    """Smallest distance of a sampled point above the ground (the oracle's d - margin)."""
    wp, _ = _points(s)
    hh, n = _ground(f, zoff, wp[:, 0], wp[:, 1])
    return ((wp[:, 2] - hh) * n[:, 2] - _model()["margin"]).min()


def _toes_down(s, f):
    """Toes whose deepest sampled point lies within the contact breaking distance of the ground (the oracle's rule)."""
    from rex_gym_b200.model_tables import contact_breaking_distance
    wp, g = _points(s)
    hh, n = _ground(f, _zoff(f), wp[:, 0], wp[:, 1])
    d = (wp[:, 2] - hh) * n[:, 2] - _model()["margin"]
    return sum(d[g == t].min() <= contact_breaking_distance("base") for t in (2, 4, 6, 8))


def _window_origin(px):
    """load_tile's fp32 window origin along one axis for a base at px."""
    c = math.floor(np.float32(px) * np.float32(20.0) + np.float32(127.5))
    return min(max(c - 8, 0), 239)


# ---- placements ------------------------------------------------------------------------------------------------------
def _at(frac, cell=0):
    """World coordinate of cell fraction `frac` of the cell `cell` cells above the middle one."""
    return (127 + cell + frac - 127.5) * CELL


def _layout(bank):
    """-> [(kind, pose, x, y, yaw)], one per env (the env's field is (i + offset + 1) % fields)."""
    if bank == "slopes":
        out = []
        for i in range(35):
            pose = ("stand", "stand", "back", "side", "nose")[i // 7]
            fr = (0.01, 0.5, 0.99)[i % 3]
            out.append(("slope", pose, _at(fr, i % 5 - 2), _at(1 - fr, 2 - i % 4), 2 * math.pi * i / 35))
        return out
    yaws = iter(2 * math.pi * np.arange(40) / 40)
    out = [("interior", "stand", x, y, next(yaws)) for x, y in
           ((-4.5, -3.2), (3.1, -5.0), (0.7, 4.4), (-2.2, 1.3), (5.3, 2.6), (-5.6, 5.1))]
    out += [("cell", "stand", _at(fx, 3), _at(fy, -5), next(yaws)) for fx in (0.01, 0.5, 0.99) for fy in (0.01, 0.5, 0.99)]
    out += [("cell", "stand", _at(1 - 1e-8, 40), _at(1 - 1e-8, 17), next(yaws))]
    d = EDGE - 0.07
    out += [("inside", "stand", x, y, next(yaws)) for x, y in ((d, 1.0), (-d, -2.0), (0.5, d), (-1.5, -d),
                                                              (d + 0.02, d), (-d, d - 0.02), (d, -d + 0.01), (-d + 0.01, -d))]
    out += [("on", "stand", x, y, next(yaws)) for x, y in ((EDGE, 2.0), (-EDGE, 0.3), (-3.0, EDGE), (1.2, -EDGE))]
    b = EDGE + 0.2
    out += [("beyond", "stand", x, y, next(yaws)) for x, y in ((b, -1.0), (-b, 3.0), (2.5, b), (-0.8, -b))]
    out += [("fallen", p, x, y, next(yaws)) for p, x, y in (("back", 2.0, 2.0), ("side", -3.0, -1.0), ("nose", 1.0, -2.5),
                                                          ("knees", -1.0, 3.5))]
    out += [("stretch", "stretch-" + p, _at(0.99, 10) if ax == "x" else -2.6, _at(0.99, -30) if ax == "y" else 1.6, 0.0 if ax == "x" else math.pi / 2)
            for p, ax in (("back", "x"), ("back", "y"), ("side", "x"), ("side", "y"))]
    return out


STRETCH_LEG = 2                                         # rear left: its hip is at body +x
FALLEN = {"back": (math.pi + 0.04, 0.03), "side": (math.pi / 2 + 0.05, 0.02), "nose": (0.03, 1.2), "knees": (0.02, 0.015)}


def _want(pose, m, bank):
    """The contacts a placement is dropped until: standing, all four toes on the slopes and three on the random blocks (10 cm
    blocks up to 5 cm apart in height rarely carry all four feet at once); a shoulder or leg box on the knees; else the fallen
    scenario's groups of test_gpu_generic_path.WANT (back: the base box; side: a shoulder or leg box; nose: either)."""
    if pose == "stand":
        return bin(m & TOE_BITS).count("1") >= (4 if bank == "slopes" else 3)
    if pose == "knees":
        return bool(m & UPPER_BITS)
    if pose.startswith("stretch"):
        return m != 0
    return bool(m & {"back": 1, "side": UPPER_BITS, "nose": BODY_BITS}[pose])


def _kw(bank, sub=True, build=None):
    """The keywords of a placement batch, the same for the GPU env and its oracle; the sensor build: observation noise only."""
    nf, off = BANKS[bank]
    kw = dict(signal_type="ik", terrain_type="random", num_fields=nf, env_offset=off, mark="base", seed=21, target_position=2.0,
              backwards=False)
    if sub:
        kw.update(SUB)
    if build == "sensor":
        kw["observation_noise_stdev"] = NOISE
    return kw


def _oracle(bank, n, sub=True, build=None, **extra):
    return make_oracle("walk", n, fields=_fields(bank), **_kw(bank, sub, build), **extra)


_CACHE = {}


def _batch(bank):
    """-> (layout, start state {key: [N][...]}, fields of the envs)."""
    if bank in _CACHE:
        return _CACHE[bank]
    lay = _layout(bank)
    n = len(lay)
    F = _fields(bank)
    o = _oracle(bank, n)
    o.reset()
    fid = [o.env(i).field_id for i in range(n)]
    settled = [o.state(i) for i in range(n)]
    st = [None] * n
    # a standing placement that does not bring its toes down is placed again at the same point, turned a further 0.5 rad
    # the stretched leg would fold back to its stance pose under its motor while dropping: those envs start from the placed
    # state, lowered to within the breaking distance of the ground, so the leg is straight at the first sub-step
    pending = {i for i in range(n) if lay[i][0] != "stretch"}
    for i in set(range(n)) - pending:
        st[i] = _place(bank, lay[i], settled[i], F[fid[i]], 0.0, STRETCH_CLEAR)
    for attempt in range(24):
        for i in pending:
            if attempt == 0 or lay[i][1] == "stand":
                st[i] = _place(bank, lay[i], settled[i], F[fid[i]], 0.5 * attempt)
                o.set_state(i, st[i])
        for _ in range(150):
            prev = {i: o.state(i) for i in pending}
            o.step(np.zeros((n, o.A), np.float32))
            for i in list(pending):
                if not _want(lay[i][1], o.env(i).contact_mask, bank):
                    continue
                if lay[i][0] == "cell":                 # the drop moves the base by about 1 mm: put it back where it belongs,
                    prev[i]["pos"][:2] = lay[i][2:4]    # as long as its toes stay down
                    if _toes_down(prev[i], F[fid[i]]) < 3:
                        continue
                st[i] = prev[i]
                pending.discard(i)
            if not pending:
                break
        if not pending:
            break
    assert not pending, [lay[i][:2] for i in pending]
    out = lay, {k: np.stack([s[k] for s in st]) for k in st[0]}, fid
    _CACHE[bank] = out
    return out


def _place(bank, where, settled, f, turn, clear=CLEAR):
    """The settled state turned to its yaw (+ turn), moved to (x, y) and raised `clear` above the local ground; fallen poses are
    laid down in their roll and pitch."""
    kind, pose, x, y, yaw = where
    zo = _zoff(f)
    s = {k: np.array(v, np.float64) for k, v in settled.items()}
    qy = quat(0, 0, yaw + turn)
    s["linvel"], s["angvel"], s["qd"] = np.zeros(3), np.zeros(3), np.zeros_like(s["qd"])
    if pose == "stand":                                 # upright with the settled joints (some fields settle the robot fallen)
        s["quat"] = qy
        if bank == "slopes":                       # stand square on the plane under the base
            _, nrm = _ground(f, zo, x, y)
            ax = np.cross([0, 0, 1], nrm)
            if np.linalg.norm(ax) > 1e-12:
                a = math.acos(nrm[2]) / 2
                t = ax / np.linalg.norm(ax) * math.sin(a)
                s["quat"] = qmul([t[0], t[1], t[2], math.cos(a)], s["quat"])
    else:
        r, p = FALLEN[pose.split("-")[-1]]
        s["quat"] = qmul(qy, quat(r, p, 0.0))
        if pose == "knees":
            s["q"][:12] = FOLDED
        if kind == "stretch":
            s["q"][3 * STRETCH_LEG + 1] = -math.pi / 2       # leg along body +x
            s["q"][3 * STRETCH_LEG + 2] = -0.1               # foot at its lower limit: the leg straight
    s["pos"][:2] = x, y
    for _ in range(50):                                 # the distance along a block face's normal is not linear in the height
        gap = clear - _clearance(s, f, zo)
        s["pos"][2] += gap
        if abs(gap) < 2e-5:
            break
    assert abs(gap) < 2e-5, where
    return s


# ---- CPU ---------------------------------------------------------------------------------------------------------------
def test_oracle_takes_banks_beyond_256_fields():
    """CPU: the oracle runs on a 300-field bank.  A robot settled on field 3, 255, 256 or 299 (chosen through env_offset) ends
    exactly where it ends on a bank holding that field alone.  Fields 3, 255 and 299 share their heights around the robot and
    differ in their vertical offset only (the settle starts at the same absolute height, so they settle differently): field 3's
    settled state, moved down by the offsets' difference and stepped 50 sub-steps on fields 255 and 299, keeps its base height
    exactly that much lower (1e-9 m) and the same joints (1e-12)."""
    from oracle.oracle import OracleSim
    F = _fields("big")
    kw = dict(terrain="random", target_position=2.0, backwards=False, **SUB)
    got = {}
    for fid in (3, 255, 256, 299):
        o = OracleSim(1, "walk", "ik", fields=F, env_offset=fid - 1, **kw)
        o.reset()
        assert o.env(0).field_id == fid
        got[fid] = o.state(0)
        one = OracleSim(1, "walk", "ik", fields=F[fid:fid + 1], **kw)
        one.reset()
        for k, v in one.state(0).items():
            np.testing.assert_allclose(got[fid][k], v, rtol=0, atol=1e-12, err_msg=f"field {fid}: {k}")
    assert len({_zoff(F[k]) for k in (3, 255, 256, 299)}) == 4
    a = np.zeros((3, 2), np.float32)
    o = OracleSim(3, "walk", "ik", fields=F, env_offset=2, **kw)          # env 0 on field 3
    o.reset()
    for i, fid in ((0, 3), (1, 255), (2, 299)):
        s = {k: v.copy() for k, v in got[3].items()}
        s["pos"][2] -= _zoff(F[fid]) - _zoff(F[3])
        o.env(i).field_id = fid
        o.set_state(i, s)
    for _ in range(50):
        o.step(a)
    s0 = o.state(0)
    assert (o.env(0).contact_mask & TOE_BITS) == TOE_BITS
    for i, fid in ((1, 255), (2, 299)):
        s = o.state(i)
        assert abs(s0["pos"][2] - s["pos"][2] - (_zoff(F[fid]) - _zoff(F[3]))) < 1e-9, fid
        np.testing.assert_allclose(s["q"], s0["q"], rtol=0, atol=1e-12)


@pytest.mark.parametrize("bank", list(BANKS))
def test_placements_reach_their_contacts(bank):
    """CPU: every start state, one sub-step on the oracle, has the contacts it is there for (three or four toes standing; the
    base / body boxes fallen), its field is the one the bank puts it on, the border placements put the window where they should,
    the cell placements sit at their cell fractions, and the stretched leg is straight with its end in the window's last cell."""
    lay, st, fid = _batch(bank)
    nf, off = BANKS[bank]
    n = len(lay)
    np.testing.assert_array_equal(fid, [(i + off + 1) % nf for i in range(n)])
    if bank == "big":
        assert min(fid) >= 256
    o = _oracle(bank, n)
    o.reset()
    for i in range(n):
        o.set_state(i, {k: v[i] for k, v in st.items()})
    o.step(np.zeros((n, o.A), np.float32))
    for i, (kind, pose, *_r) in enumerate(lay):
        assert _want(pose, o.env(i).contact_mask, bank), (i, kind, pose, bin(o.env(i).contact_mask))
        x, y = st["pos"][i][:2]
        if kind == "inside":
            assert max(abs(x), abs(y)) < EDGE - 0.04
            assert {_window_origin(x), _window_origin(y)} & {0, 239}
        elif kind == "beyond":
            assert max(abs(x), abs(y)) > EDGE + 0.15
        elif kind == "stretch":                         # the leg is straight and its end lies in the window's last cell
            s = {k: v[i] for k, v in st.items()}
            assert s["q"][3 * STRETCH_LEG + 1] == -math.pi / 2 and s["q"][3 * STRETCH_LEG + 2] == -0.1
            ax = 0 if lay[i][4] == 0.0 else 1
            assert abs((s["pos"][ax] / CELL + 127.5) % 1 - 0.99) < 1e-9
            wp, _ = _points(s)
            low = wp[wp[:, 2] <= 0.06, ax]               # the points the kernel queries
            lead = math.floor(np.float32(low.max()) * np.float32(20.0) + np.float32(127.5))
            assert lead == _window_origin(s["pos"][ax]) + 15, (pose, lead, _window_origin(s["pos"][ax]))
    if bank != "slopes":
        kinds = [k for k, *_r in lay]
        assert [kinds.count(k) for k in ("interior", "cell", "inside", "on", "beyond", "fallen", "stretch")] == [6, 10, 8, 4, 4, 4, 4]
        # the cell placements: base at the bottom, middle and top of a cell, and one whose fp32 cell index is one above fp64's
        cell = [i for i in range(n) if lay[i][0] == "cell"]
        fr = sorted({round((st["pos"][i][a] / CELL + 127.5) % 1, 6) for i in cell[:9] for a in (0, 1)})
        assert fr == [0.01, 0.5, 0.99], fr
        for a in (0, 1):                                # the last one: fp32 cell index one above fp64's
            p = st["pos"][cell[9]][a]
            assert math.floor(np.float32(p) * np.float32(20.0) + np.float32(127.5)) == math.floor(p / CELL + 127.5) + 1
    else:
        slopes = [math.degrees(math.acos(_ground(_fields(bank)[fid[i]], _zoff(_fields(bank)[fid[i]]), *st["pos"][i][:2])[1][2]))
                  for i in range(n)]
        assert max(slopes) > 24 and min(slopes) > 5, slopes


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def _gpu_env(bank, build, monkeypatch, n, sub=True):
    from rex_gym_b200.envs import batched_env
    F = _fields(bank)
    monkeypatch.setattr(batched_env, "make_random_fields", lambda k, seed=10: F[:k].copy())
    force_build(monkeypatch, build)
    return make_env("walk", n, **_kw(bank, sub, build))


def _mask_exception(s, i, groups, f, zoff, breaking):
    """True when every group in `groups` has its deepest sampled point within float rounding of the breaking distance, or within
    1e-4 m of it and within 1e-4 cells of a crease or vertex line (where the fp32 and fp64 triangles differ)."""
    wp, g = _points({k: v[i] for k, v in s.items()})
    hh, nrm = _ground(f, zoff, wp[:, 0], wp[:, 1])
    d = (wp[:, 2] - hh) * nrm[:, 2] - _model()["margin"]
    for gr in groups:
        sel = np.nonzero(g == gr)[0]
        k = sel[np.argmin(d[sel])]
        gap = abs(d[k] - breaking)
        fx, fy = wp[k, 0] / CELL + 127.5, wp[k, 1] / CELL + 127.5
        u, v = fx % 1, fy % 1
        crease = min(u, 1 - u, v, 1 - v, abs(u - v)) < 1e-4
        if not (gap < 2e-6 or (gap < 1e-4 and crease)):
            return False
    return True


SUB_CONFIGS = [(b, bd) for b in BANKS for bd in ("small", "big", "sensor")]


@pytest.mark.gpu
@pytest.mark.parametrize("bank,build", SUB_CONFIGS, ids=["-".join(c) for c in SUB_CONFIGS])
def test_heightfield_substeps_against_the_oracle(monkeypatch, bank, build):
    """One control step = one physics sub-step (1 ms, 60 PGS iterations), 30 of them from the placed start states, the CUDA state
    re-synchronised to the oracle before each.  Per sub-step: the contact mask equals the oracle's on every group (a difference is
    accepted only where the numpy restatement finds the group's deepest point within float rounding of the breaking distance, or
    of it and of a crease); the solver path is the oracle's predicate and the PGS iterations lie in the oracle's band over
    early-out thresholds 0.8-1.2e-7 in fp64 and fp32; no env raises TILE_MISS; q and pos meet
    test_generic_substeps_against_the_oracle's bounds (90th percentile 2e-5 rad / 2e-6 m, none beyond 3e-3).
    Measured on an H100 SXM (700 W), 30 sub-steps x the bank's envs; the three builds of a bank agree bit for bit:
      default  q median 3.7e-7, p90 2.0e-6, max 1.0e-5 rad; pos median 8e-8, p90 2.8e-7, max 4.6e-7 m; 0 off the band
      big      q median 4.6e-7, p90 1.9e-6, max 9.9e-6 rad; pos median 9e-8, p90 2.9e-7, max 4.7e-7 m; 0 off the band
      slopes   q median 7.6e-7, p90 2.1e-6, max 9.8e-5 rad; pos median 5e-9, p90 2.4e-8, max 1.6e-7 m; 1 off the band
    and no contact-mask exception in any of them."""
    from rex_gym_b200.model_tables import contact_breaking_distance
    lay, st, fid = _batch(bank)
    n = len(lay)
    F = _fields(bank)
    env, ora = _gpu_env(bank, build, monkeypatch, n), _oracle(bank, n, build=build)
    band = IterationBand(lambda **b: _oracle(bank, n, build=build, **b))
    env.reset(); ora.reset(); band.reset()
    np.testing.assert_array_equal(env._state_i.cpu().numpy()[LAYOUT.I_FIELD], fid)
    breaking = contact_breaking_distance("base")
    eq, ep, off_band, generic_steps, excused, flags = compare_substeps(
        env, ora, band, st, build, [w[:2] for w in lay],
        exception=lambda so, i, groups: _mask_exception(so, i, groups, F[fid[i]], _zoff(F[fid[i]]), breaking))
    miss = np.argwhere(flags & TILE_MISS)
    assert not len(miss), ("TILE_MISS", [(k, lay[i][:2]) for k, i in miss])
    stats = (np.median(eq), np.percentile(eq, 90), eq.max(), np.median(ep), np.percentile(ep, 90), ep.max(), off_band, excused)
    print("heightfield sub-steps q (median, p90, max), pos (median, p90, max), iterations off the band, mask exceptions:", stats)
    assert generic_steps >= 30 * 8 * 0.5, generic_steps
    assert off_band <= 3 and excused <= 3, stats
    assert np.percentile(eq, 90) < 2e-5 and np.percentile(ep, 90) < 2e-6 and eq.max() < 3e-3 and ep.max() < 3e-3, stats
    assert env.check_errors() == 0
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bank,build", SUB_CONFIGS, ids=["-".join(c) for c in SUB_CONFIGS])
def test_heightfield_control_steps_against_the_oracle(monkeypatch, bank, build):
    """The task configuration (5 sub-steps per control step): 20 control steps of random actions inside walk-ik's bound from the
    placed states, re-synchronised every 5, within test_generic_control_steps_against_the_oracle's window (90th percentile
    1e-3 rad / 1e-3 m, none beyond 5e-2 / 5e-3); every output finite, no error bit on any step.
    Measured on an H100 SXM (700 W) over the 20 x N samples (q median / p90 / max in rad, pos max in m; the builds agree bit for bit):
      default 9.4e-7 / 3.8e-6 / 2.8e-4, 1.9e-6;  big 7.5e-7 / 4.1e-6 / 3.4e-4, 1.9e-6;  slopes 1.2e-6 / 4.6e-6 / 9.4e-4, 5.1e-5."""
    lay, st, fid = _batch(bank)
    n = len(lay)
    env, ora = _gpu_env(bank, build, monkeypatch, n, sub=False), _oracle(bank, n, sub=False, build=build)
    env.reset(); ora.reset()
    eqs, eps_, flags = compare_control_steps(env, ora, st, build, [w[:2] for w in lay], q90=1e-3, p90=1e-3, qmax=5e-2, pmax=5e-3)
    assert not flags.any(), np.argwhere(flags)
    print("heightfield control steps q (median, p90, max), pos (median, p90, max):",
          (np.median(eqs), np.percentile(eqs, 90), eqs.max(), np.median(eps_), np.percentile(eps_, 90), eps_.max()))
    assert env.check_errors() == 0
    env.close()


FLY = [(0.0, 0.0)] + [(s * dx, s * dy) for s in (1.0, 40.0) for dx, dy in ((1, 0), (-1, 0), (0, 1), (0, -1))]


@pytest.mark.gpu
@pytest.mark.parametrize("build", ["small", "big", "sensor"])
def test_tile_miss_flags_exactly_the_envs_that_leave_the_window(monkeypatch, build):
    """A flat field, one 20 ms control step of 20 sub-steps: robots fly 3.5 cm above the ground, no contact on any sub-step (checked
    on the oracle), at 0, 1 m/s (2 cm per step) and 40 m/s (0.8 m per step) in +-x and +-y.  The 40 m/s envs leave the window
    staged at the start of the step and raise TILE_MISS, the others do not; with no contact the states still match the oracle.
    After set_state with zero velocity, the next step clears the per-env word."""
    from rex_gym_b200.envs import batched_env
    n = len(FLY)
    F = np.zeros((1, 256, 256), np.float32)
    monkeypatch.setattr(batched_env, "make_random_fields", lambda k, seed=10: F.copy())
    force_build(monkeypatch, build)
    kw = dict(signal_type="ik", terrain_type="random", num_fields=1, seed=21, target_position=2.0, backwards=False,
              control_time_step=0.02, action_repeat=20)
    if build == "sensor":
        kw["observation_noise_stdev"] = NOISE
    env, ora, chk = make_env("walk", n, **kw), make_oracle("walk", n, fields=F, **kw), make_oracle("walk", n, fields=F, **kw)
    env.reset(); ora.reset(); chk.reset()
    so = ora.states()
    so["pos"][:, 2] += 0.035
    so["linvel"][:, :2] = FLY
    so["linvel"][:, 2] = 0.0
    for i in range(n):
        ora.set_state(i, {k: v[i] for k, v in so.items()})
        chk.set_state(i, {k: v[i] for k, v in so.items()})
    sync(env, ora)
    a = np.zeros((n, env.action_dim), np.float32)
    for i in range(n):                                  # the same control step, sub-step by sub-step: no contact anywhere
        cmd = chk.transform_action(a[i], i)
        for _ in range(20):
            chk.substep(i, cmd)
            assert chk.env(i).contact_mask == 0, (i, FLY[i])
    ora.step(a)
    env.step(a)
    assert launched(env) == BUILDS[build], launched(env)
    flags = env.error_flags().cpu().numpy()
    fast = np.array([math.hypot(*v) > 10 for v in FLY])
    np.testing.assert_array_equal((flags & TILE_MISS) != 0, fast)
    assert not (flags & ~TILE_MISS).any(), flags
    assert (env.get_state()["contact_mask"] == 0).all() and all(ora.env(i).contact_mask == 0 for i in range(n))
    eq, ep = state_errors(env, ora)
    assert eq.max() < 1e-4 and ep.max() < 1e-5
    assert env.check_errors() == TILE_MISS
    s2 = ora.states()
    for k in ("linvel", "angvel", "qd"):
        s2[k][:] = 0.0
    env.set_state(*(s2[k] for k in STATE_KEYS))
    env.step(a)
    assert not env.error_flags().cpu().numpy().any()
    assert env.check_errors() == 0
    env.close()

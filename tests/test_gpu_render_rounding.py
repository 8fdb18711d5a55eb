"""The renderer (rex_gym_b200/csrc/rexsim_render.cu) at rounding level: every pixel of every frame against the fp64 render
oracle's 9 jittered rays (render_oracle.check_pixels: the byte of a robust pixel exactly, any other pixel inside one ray's
colour box; render_oracle.EPS and DELTA carry the fp32 error budget), with no fraction of pixels excused.

Scenes: {base, arm} x {plane, the default 64-field bank}, each at a stepped state and at hand-set placements (standing,
fallen on the side, upside down, partly below the ground, 5 cm inside a field border, on it, 0.2 m beyond it where the plane at
the field's lowest height takes over, and at x = +-100 m); a 300-field bank reached through env_offset (fields 256-265); a
25 degree plane in x, one along the diagonal and a field whose two triangles per cell differ.  Cameras: 20 chosen (distance,
yaw, pitch) combinations, from the eye inside the base (0.05 m) to a far plane that cuts the ground, looking straight down,
level and up.  Sizes: the reference's 480 x 360, one-pixel last tiles (17 x 17, 33 x 47), 1 x 360, 480 x 1, 4096 x 16 and
4096 x 4096 on oracle windows.  Calls of 65 535, 65 536 and 131 071 images (more than one launch) against one-image renders.

The CPU tests show the criterion has teeth: it rejects the oracle rendered half a pixel off, with a truncating quantiser and with
the heightfield normal missing its x20 grid scale; it accepts the oracle under 2^-22 relative perturbations of pose and camera;
and every planned scene is at least render_oracle.MIN_ROBUST robust."""
import math

import numpy as np
import pytest

import render_oracle as RO

EDGE = 127.5 * 0.05                                     # a field's borders at x, y = -+6.375 m
STAND = np.tile([0.0, -0.88643435, 1.30197369], 4)      # INIT_POSES['stand']
N_PLACED = 10


def _quat(axis, deg):
    a = np.radians(deg) / 2
    return np.concatenate([np.sin(a) * np.asarray(axis, np.float64), [np.cos(a)]])


# (name, base position with z above the local ground, quaternion xyzw); index 0 keeps the stepped state
PLACEMENTS = [
    ("stepped", None, None),
    ("standing", (0.3, -0.2, 0.21), _quat((0, 0, 1), 30)),
    ("side", (0.5, -0.3, 0.08), _quat((1, 0, 0), 90)),
    ("upside down", (-0.4, 0.6, 0.15), _quat((1, 0, 0), 180)),
    ("below ground", (0.1, 0.2, 0.04), _quat((0, 0, 1), -60)),
    ("5 cm inside border", (EDGE - 0.05, 1.0, 0.21), _quat((0, 0, 1), 0)),
    ("on border", (-2.0, EDGE, 0.21), _quat((0, 0, 1), 90)),
    ("0.2 m beyond border", (EDGE + 0.2, 0.5, 0.21), _quat((0, 0, 1), 180)),
    ("x = +100 m", (100.0, 0.3, 0.21), _quat((0, 0, 1), 45)),
    ("x = -100 m", (-100.0, -0.3, 0.21), _quat((0, 0, 1), -135)),
]
# (distance m, yaw deg, pitch deg): the reference's camera, the eye inside the base (0.05 m: parts of the robot inside the near
# plane), 0.3 / 1 / 3 m, horizon, level and sky rays (pitch -5, 0, +15), straight down (-89.9), and far planes at 100 m that
# cut the ground (20 m at -10, 60 m at -30)
CAMERAS = [
    (1.0, 0.0, -30.0), (0.05, 0.0, -30.0), (0.05, 90.0, 0.0), (0.05, -135.0, -60.0), (0.3, 37.0, -60.0),
    (0.3, 180.0, -5.0), (0.3, 0.0, 15.0), (1.0, 37.0, -89.9), (1.0, -135.0, 15.0), (1.0, 90.0, 0.0),
    (1.0, 180.0, -5.0), (1.0, 37.0, -30.0), (3.0, 180.0, -30.0), (3.0, -135.0, -5.0), (3.0, 0.0, 15.0),
    (3.0, 90.0, -60.0), (3.0, 37.0, 0.0), (20.0, 0.0, -10.0), (60.0, 37.0, -30.0), (1.0, -135.0, -89.9),
]
SWEEP = (160, 120)


def placements_of(cam):
    """The three placements camera `cam` is checked on (every placement meets six cameras)."""
    return sorted({cam % N_PLACED, (cam + 3) % N_PLACED, (cam + 7) % N_PLACED})


def place(mark, terrain, heights, st, k):
    """(pos, quat) of placement k: z is taken above the ground under the base (the field's triangle, or the plane at its
    lowest height beyond the border)."""
    name, pos, quat = PLACEMENTS[k]
    if pos is None:
        return st["pos"][0].copy(), st["quat"][0].copy()
    pos = np.array(pos, np.float64)
    if terrain == "random":
        zoff = 0.5 * (float(heights.min()) + float(heights.max()))
        gx, gy = pos[0] * 20 + 127.5, pos[1] * 20 + 127.5
        if 0 <= gx <= 255 and 0 <= gy <= 255:
            ix, iy = min(int(gx), 254), min(int(gy), 254)
            pos[2] += float(heights[iy:iy + 2, ix:ix + 2].max()) - zoff
        else:
            pos[2] += float(heights.min()) - zoff
    return pos, quat


# ---- CPU: the criterion has teeth ------------------------------------------------------------------------------------
def _cpu_scene(mark, terrain, k):
    from rex_gym_b200.terrain import make_random_fields
    heights = make_random_fields(1)[0].astype(np.float64) if terrain == "random" else None
    q = np.concatenate([STAND, np.zeros(6)]) if mark == "arm" else STAND
    st = {"pos": np.array([[0.0, 0.0, 0.2]]), "quat": np.array([[0.0, 0.0, 0.0, 1.0]])}
    pos, quat = place(mark, terrain, heights, st, k)
    return dict(mark=mark, pos=pos, quat=quat, q=q, terrain=terrain, heights=heights)


KIND_MARKS = {"base-plane": ("base", "plane"), "base-random": ("base", "random"), "arm-plane": ("arm", "plane"),
              "arm-random": ("arm", "random")}
SWEEP_CASES = [(kind, c) for kind in KIND_MARKS for c in range(len(CAMERAS))]
SWEEP_IDS = ["%s-d%g-y%g-p%g" % ((k,) + CAMERAS[c]) for k, c in SWEEP_CASES]


def _samples(sc, cam, eps=RO.EPS, **kw):
    d, y, p = cam
    return RO.render_values(width=SWEEP[0], height=SWEEP[1], distance=d, yaw=y, pitch=p, offset=RO.jitter(eps), **sc, **kw)


@pytest.mark.parametrize("kind,cam", SWEEP_CASES, ids=SWEEP_IDS)
def test_planned_scenes_are_robust(kind, cam):
    """CPU: every scene of the camera sweep (the stepped state replaced by the standing pose) keeps MIN_ROBUST of its pixels
    robust, and the oracle's own bytes pass."""
    for k in placements_of(cam):
        sc = _cpu_scene(*KIND_MARKS[kind], k)
        val, ids = _samples(sc, CAMERAS[cam])
        RO.assert_pixels(np.clip(np.floor(val[0]), 0, 255), val, ids, "%s %s" % (kind, PLACEMENTS[k][0]))


@pytest.mark.parametrize("mark,terrain,k,cam", [("base", "plane", 1, 0), ("base", "random", 4, 11), ("arm", "plane", 2, 4),
                                                ("arm", "random", 0, 12), ("base", "random", 7, 13), ("base", "plane", 8, 18)])
def test_criterion_accepts_fp32_sized_perturbations(mark, terrain, k, cam):
    """CPU: the pose and the camera angles moved by 2^-22 relative (a few fp32 roundings) still pass."""
    sc = _cpu_scene(mark, terrain, k)
    val, ids = _samples(sc, CAMERAS[cam])
    rng = np.random.default_rng(k + 17 * cam)
    e = 2.0 ** -22
    jig = lambda x: np.asarray(x, np.float64) * (1 + e * rng.choice([-1.0, 1.0], np.shape(x)))
    sc2 = dict(sc, pos=jig(sc["pos"]), quat=jig(sc["quat"]), q=jig(sc["q"]))
    d, y, p = CAMERAS[cam]
    v2, _ = RO.render_values(width=SWEEP[0], height=SWEEP[1], distance=jig(d), yaw=jig(y), pitch=jig(p), **sc2)
    RO.assert_pixels(np.clip(np.floor(v2), 0, 255), val, ids, "perturbed")


def _fails(got, val, ids):
    frac, err, bad = RO.check_pixels(got, val, ids)
    return len(bad) > 0


@pytest.mark.parametrize("mark,terrain,k,cam", [("base", "plane", 1, 0), ("base", "random", 4, 11), ("arm", "plane", 2, 4),
                                                ("arm", "random", 0, 12), ("base", "random", 5, 13)])
def test_criterion_rejects_oracle_mutants(mark, terrain, k, cam):
    """CPU: the oracle itself with the ray half a pixel off centre, with a quantiser that truncates, and (on the heightfield)
    with the normal missing its x20 grid scale fails against the unmutated oracle."""
    sc = _cpu_scene(mark, terrain, k)
    val, ids = _samples(sc, CAMERAS[cam])
    d, y, p = CAMERAS[cam]
    kw = dict(width=SWEEP[0], height=SWEEP[1], distance=d, yaw=y, pitch=p, **sc)
    half, _ = RO.render_values(offset=(0.5, 0.5), **kw)
    assert _fails(np.clip(np.floor(half), 0, 255), val, ids), "half-pixel offset"
    assert _fails(np.clip(np.floor(val[0] - 0.5), 0, 255), val, ids), "truncating quantiser"
    if terrain == "random":
        flat, _ = RO.render_values(normal_scale=1.0, **kw)
        assert _fails(np.clip(np.floor(flat), 0, 255), val, ids), "normal without the grid scale"


def test_jitter_and_budget():
    """CPU: 9 rays, the centre and 8 on a circle of EPS at 45 degrees; EPS at most 0.05 px (10x below a half-pixel error)."""
    j = RO.jitter()
    assert j.shape == (9, 2) and (j[0] == 0).all()
    assert np.allclose(np.hypot(j[1:, 0], j[1:, 1]), RO.EPS) and RO.EPS <= 0.05 and RO.DELTA <= 0.01
    ang = np.degrees(np.arctan2(j[1:, 1], j[1:, 0])) % 360
    assert np.allclose(np.sort(ang), np.arange(0, 360, 45))


def test_windows_and_offsets_match_the_full_frame():
    """CPU: a window of render_values is the same pixels of the full frame, and render() is its floor."""
    sc = _cpu_scene("base", "random", 1)
    full, fid = RO.render_values(width=64, height=48, **sc)
    win, wid = RO.render_values(width=64, height=48, rows=range(40, 48), cols=range(3, 20), **sc)
    assert np.array_equal(win, full[40:48, 3:20]) and np.array_equal(wid, fid[40:48, 3:20])
    img, ids = RO.render(width=64, height=48, **sc)
    assert np.array_equal(img, np.clip(np.floor(full), 0, 255).astype(np.uint8)) and np.array_equal(ids, fid)
    both, bid = RO.render_values(width=64, height=48, offset=[(0, 0), (0.25, -0.5)], **sc)
    one, _ = RO.render_values(width=64, height=48, offset=(0.25, -0.5), **sc)
    assert np.array_equal(both[0], full) and np.array_equal(both[1], one)


# ---- GPU ---------------------------------------------------------------------------------------------------------------
STATS = {"robust": 1.0, "err": 0, "frames": 0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if STATS["frames"]:
        print("\nrender rounding: %d frames, minimum robust fraction %.4f, largest |device - oracle| on robust pixels %d LSB"
              % (STATS["frames"], STATS["robust"], STATS["err"]))


def _check(got, val, ids, what, min_robust=RO.MIN_ROBUST):
    frac, err = RO.assert_pixels(got, val, ids, what, min_robust)
    if min_robust:
        STATS["robust"] = min(STATS["robust"], frac)
    STATS["err"] = max(STATS["err"], err)
    STATS["frames"] += 1


def _slope_fields():
    c = (np.arange(256) - 127.5) * 0.05
    x, y = np.meshgrid(c, c)                                        # field[iy][ix]
    t = math.tan(math.radians(25))
    ii, jj = np.meshgrid(np.arange(256), np.arange(256))
    two = 0.1 * x + 0.02 * ((ii + jj) % 2)                          # per cell: the two triangles slope apart
    return np.ascontiguousarray(np.stack([t * x, t * (x + y) / math.sqrt(2), two]) + 1.0, np.float32)


def _big_bank():
    from rex_gym_b200.terrain import make_random_fields
    base = make_random_fields(4)
    f = np.stack([base[k % 4] for k in range(300)])
    f[:, 200, 40] += np.float32(1e-3) * np.arange(300, dtype=np.float32)   # every field its own vertical offset
    return np.ascontiguousarray(f, np.float32)


# (mark, terrain, bank): bank None = the product's default bank
KINDS = {"base-plane": ("base", "plane", None), "base-random": ("base", "random", None), "arm-plane": ("arm", "plane", None),
         "arm-random": ("arm", "random", None), "base-300": ("base", "random", "big"), "base-slopes": ("base", "random", "slopes")}
_ENVS = {}


def _env(kind):
    """A batch of N_PLACED envs, stepped from reset, then envs 1.. moved to the hand-set placements."""
    if kind in _ENVS:
        return _ENVS[kind]
    from rex_gym_b200.envs import batched_env
    mark, terrain, bank = KINDS[kind]
    kw = dict(terrain_type=terrain, mark=mark, seed=5)
    with pytest.MonkeyPatch.context() as mp:
        if bank == "big":
            F = _big_bank()
            mp.setattr(batched_env, "make_random_fields", lambda k, seed=10: F[:k].copy())
            kw.update(num_fields=300, env_offset=255)                  # env i on field (i + 256) % 300
        elif bank == "slopes":
            F = _slope_fields()
            mp.setattr(batched_env, "make_random_fields", lambda k, seed=10: F[:k].copy())
            kw.update(num_fields=3)
        if mark == "arm":
            env = batched_env.RexStandupBatchEnv(num_envs=N_PLACED, **kw)
            bound, n = 0.1, 30
        else:
            env = batched_env.RexWalkBatchEnv(num_envs=N_PLACED, signal_type="ik", target_position=2.0, backwards=False, **kw)
            bound, n = 0.4, 40
    rng = np.random.default_rng(len(_ENVS))
    env.reset()
    for _ in range(n):
        env.step(rng.uniform(-bound, bound, size=(env.num_envs, env.action_dim)).astype(np.float32))
    st = env.get_state()
    pos, quat = st["pos"].copy(), st["quat"].copy()
    for i in range(1, N_PLACED):
        heights = RO.scene(env, i, st)["heights"]
        pos[i], quat[i] = place(mark, terrain, heights, st, i)
    env.set_state(pos, quat, np.zeros_like(st["linvel"]), np.zeros_like(st["angvel"]), st["q"], np.zeros_like(st["qd"]))
    _ENVS[kind] = env
    return env


@pytest.fixture(scope="module", autouse=True)
def _close_envs():
    yield
    for env in _ENVS.values():
        env.close()
    _ENVS.clear()


def _frames(env, envs, width, height, cam, rows=None, cols=None):
    d, y, p = cam
    img = env.render_batch(list(envs), width=width, height=height, distance=d, yaw=y, pitch=p).cpu().numpy()
    st = env.get_state()
    for k, i in enumerate(envs):
        val, ids = RO.render_values(width=width, height=height, distance=d, yaw=y, pitch=p, offset=RO.jitter(), rows=rows,
                                    cols=cols, **RO.scene(env, i, st))
        got = img[k] if rows is None else img[k][np.ix_(np.asarray(rows), np.asarray(cols))]
        yield i, got, val, ids


@pytest.mark.gpu
@pytest.mark.parametrize("kind,cam", SWEEP_CASES, ids=SWEEP_IDS)
def test_camera_sweep(kind, cam):
    """160 x 120 frames of three placements per camera, every pixel held to the oracle's 9 rays."""
    env = _env(kind)
    for i, got, val, ids in _frames(env, placements_of(cam), *SWEEP, CAMERAS[cam]):
        _check(got, val, ids, "%s %s camera %s" % (kind, PLACEMENTS[i][0], CAMERAS[cam]))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["base-300", "base-slopes"])
@pytest.mark.parametrize("cam", [0, 12, 17, 7])
def test_custom_banks(kind, cam):
    """Fields 256-265 of a 300-field bank reached through env_offset; the 25 degree planes in x and along the diagonal and the
    field whose two triangles per cell differ: the stepped env and the placements on and around a field (3 or 10 envs)."""
    env = _env(kind)
    if kind == "base-300":
        assert (env._state_i[RO._layout().I_FIELD].cpu().numpy() >= 256).all()
        envs = placements_of(cam)
    else:
        assert sorted(env._state_i[RO._layout().I_FIELD, :3].cpu().numpy().tolist()) == [0, 1, 2]
        envs = [0, 1, 2]
    for i, got, val, ids in _frames(env, envs, *SWEEP, CAMERAS[cam]):
        _check(got, val, ids, "%s env %d camera %s" % (kind, i, CAMERAS[cam]))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["base-plane", "arm-random"])
@pytest.mark.parametrize("size", [(480, 360), (17, 17), (33, 47), (1, 360), (480, 1), (4096, 16)],
                         ids=lambda s: "%dx%d" % s)
def test_image_shapes(kind, size):
    """The reference's size, one-pixel last tiles in both directions (17 x 17, 33 x 47: the frustum's one-pixel branch), one
    row, one column and a 4096-pixel side, whole frames of the stepped env and one placement."""
    env = _env(kind)
    # a pixel of a frame with a side under 48 pixels spans degrees of the view (up to 60 along a one-pixel side): most of them
    # lie within EPS of some patch edge, so these frames are held pixel by pixel with no robust floor
    floor = RO.MIN_ROBUST if min(size) >= 48 else 0.0
    for i, got, val, ids in _frames(env, [0, 1], *size, CAMERAS[0]):
        _check(got, val, ids, "%s %dx%d env %d" % ((kind,) + size + (i,)), floor)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["base-plane", "base-random"])
def test_4096_square_on_windows(kind):
    """4096 x 4096 frames checked on oracle windows: the image centre, the last tile row, the last tile column and the corner."""
    env = _env(kind)
    n = 4096
    for rows, cols in ((range(2032, 2064), range(2032, 2064)), (range(n - 16, n), range(1900, 2200)),
                       (range(1900, 2200), range(n - 16, n)), (range(n - 16, n), range(n - 16, n))):
        for i, got, val, ids in _frames(env, [0], n, n, CAMERAS[0], rows, cols):
            _check(got, val, ids, "%s 4096 window rows %s cols %s" % (kind, rows, cols))


@pytest.fixture(scope="module")
def crowd():
    """1009 envs (a prime: the image pattern below is not periodic in 65 535), every one at its own pose, and each env's 2 x 2
    image from 0.3 m rendered alone."""
    from rex_gym_b200.envs.batched_env import RexWalkBatchEnv
    env = RexWalkBatchEnv(num_envs=1009, signal_type="ik", target_position=2.0, backwards=False, seed=9)
    env.reset()
    st = env.get_state()
    rng = np.random.default_rng(4)
    pos = st["pos"] + rng.uniform(-0.05, 0.05, st["pos"].shape)
    q = st["q"] + rng.uniform(-0.3, 0.3, st["q"].shape)
    quat = st["quat"] + rng.uniform(-0.2, 0.2, st["quat"].shape)
    quat /= np.linalg.norm(quat, axis=1, keepdims=True)
    env.set_state(pos, quat, st["linvel"], st["angvel"], q, st["qd"])
    one = np.stack([env.render_batch([e], width=2, height=2, distance=0.3)[0].cpu().numpy() for e in range(env.num_envs)])
    assert len({x.tobytes() for x in one}) > 250                    # the poses give different 2 x 2 images
    yield env, one
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("k", [65535, 65536, 131071])
def test_many_images_in_one_call(crowd, k):
    """One call of k 2 x 2 images, env (i * i + 7) % 1009 for image i: every image equals the one-image render of its env, and
    the call issues ceil(k / 65 535) launches."""
    import torch
    env, one = crowd
    idx = (np.arange(k, dtype=np.int64) ** 2 + 7) % env.num_envs
    n0 = env.launch_count
    img = env.render_batch(torch.from_numpy(idx.astype(np.int32)).cuda(), width=2, height=2, distance=0.3).cpu().numpy()
    assert env.launch_count - n0 == -(-k // 65535)
    same = (img == one[idx]).all((1, 2, 3))
    assert same.all(), "images differ from their one-image render, first at %s" % np.nonzero(~same)[0][:5]


@pytest.mark.gpu
def test_out_of_range_device_indices_in_a_long_call(crowd):
    """Device indices outside the batch scattered through a 70 001-image call: those images are sky, every other image is
    its one-image render, and check_errors() raises IndexError once."""
    import torch
    from rex_gym_b200 import model_tables as MT
    env, one = crowd
    k = 70001
    idx = (np.arange(k, dtype=np.int64) ** 2 + 7) % env.num_envs
    bad = np.zeros(k, bool)
    bad[[0, 5, 65534, 65535, 65536, k - 1]] = True
    bad[np.random.default_rng(1).choice(k, 200, replace=False)] = True
    idx = np.where(bad, np.where(np.arange(k) % 2, env.num_envs + np.arange(k) % 7, -1 - np.arange(k) % 5), idx)
    assert env.check_errors() == 0
    img = env.render_batch(torch.from_numpy(idx.astype(np.int32)).cuda(), width=2, height=2, distance=0.3).cpu().numpy()
    sky = np.floor(MT.pack_render_tables("base")[MT.RT_SKY:MT.RT_SKY + 3].astype(np.float64) * 255 + 0.5).astype(np.uint8)
    assert (img[bad] == sky).all()
    assert (img[~bad] == one[idx[~bad]]).all()
    with pytest.raises(IndexError):
        env.check_errors()
    assert env.check_errors() == 0

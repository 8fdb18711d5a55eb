"""rgb_array renderer on the device against the fp64 render oracle (tests/render_oracle.py, per pixel through its 9 jittered rays:
render_oracle.check_pixels), and its contract: deterministic, independent of the other images of a call, free of side effects,
index checks."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def oracle_samples(env, i, width=480, height=360, distance=1.0, yaw=0.0, pitch=-30.0, st=None, draw_robot=True):
    """The oracle's 9 jittered rays of every pixel of env i's frame: value [9][H][W][3], id [9][H][W] (render_oracle.check_pixels)."""
    import render_oracle as RO
    return RO.render_values(width=width, height=height, distance=distance, yaw=yaw, pitch=pitch, draw_robot=draw_robot,
                            offset=RO.jitter(), **RO.scene(env, i, st))


def assert_frame(got, env, i, what, **kw):
    import render_oracle as RO
    val, ids = oracle_samples(env, i, **kw)
    RO.assert_pixels(got, val, ids, what, RO.MIN_ROBUST if min(val.shape[1:3]) >= 48 else 0.0)   # a 1 x 1 frame: no floor
    return ids[0]


def stepped(env, n_steps, bound, seed=0):
    rng = np.random.default_rng(seed)
    env.reset()
    for _ in range(n_steps):
        env.step(rng.uniform(-bound, bound, size=(env.num_envs, env.action_dim)).astype(np.float32))
    return env


@pytest.fixture(scope="module")
def walk():
    from rex_gym_b200.envs.batched_env import RexWalkBatchEnv
    env = stepped(RexWalkBatchEnv(num_envs=4, signal_type="ik", target_position=2.0, backwards=False), 60, 0.4)
    yield env
    env.close()


def test_walk_ik_flat_matches_oracle(walk):
    img = walk.render_batch(np.arange(4)).cpu().numpy()
    for i in range(4):
        assert_frame(img[i], walk, i, "walk env %d" % i)


def test_turn_ik_heightfield_with_border_and_fallen_envs():
    from rex_gym_b200.envs.batched_env import RexTurnBatchEnv
    env = stepped(RexTurnBatchEnv(num_envs=4, signal_type="ik", terrain_type="random", num_fields=4), 80, 0.01, seed=1)
    st = env.get_state()
    st["pos"][2] = [6.3, 0.2, 0.25]                          # at the field's border (the square ends at 6.375 m)
    st["pos"][3] = [0.5, -0.3, 0.08]
    st["quat"][3] = [np.sin(np.pi / 4), 0.0, 0.0, np.cos(np.pi / 4)]   # lying on its side
    env.set_state(st["pos"], st["quat"], st["linvel"], st["angvel"], st["q"], st["qd"])
    img = env.render_batch(np.arange(4)).cpu().numpy()
    st = env.get_state()
    for i in range(4):
        assert_frame(img[i], env, i, "turn env %d" % i, st=st)
    env.close()


def test_standup_with_the_arm_matches_oracle():
    from rex_gym_b200.envs.batched_env import RexStandupBatchEnv
    env = stepped(RexStandupBatchEnv(num_envs=2, mark="arm"), 50, 0.1, seed=2)
    img = env.render_batch([0, 1]).cpu().numpy()
    import render_oracle as RO
    for i in range(2):
        ids = assert_frame(img[i], env, i, "standup arm env %d" % i)
        shapes = set((ids[(ids >= 0) & (ids < RO.GROUND_ID)] // 1000 - 1).tolist())
        assert any(s >= 19 for s in shapes)                 # the arm is in the picture
    env.close()


def test_top_down_camera_and_odd_sizes(walk):
    img = walk.render_batch([1], distance=3.0, yaw=90.0, pitch=-89.0).cpu().numpy()[0]
    assert_frame(img, walk, 1, "yaw 90 pitch -89", distance=3.0, yaw=90.0, pitch=-89.0)
    for w, h in ((97, 61), (1, 1)):
        img = walk.render_batch([0, 3], width=w, height=h).cpu().numpy()
        assert img.shape == (2, h, w, 3)
        for k, i in enumerate((0, 3)):
            assert_frame(img[k], walk, i, "%dx%d env %d" % (w, h, i), width=w, height=h)


def test_deterministic_and_independent_of_the_other_images(walk):
    import torch
    a = walk.render_batch([0, 1, 2, 3])
    b = walk.render_batch([0, 1, 2, 3])
    assert torch.equal(a, b)
    assert torch.equal(walk.render_batch([2])[0], a[2])
    c = walk.render_batch(torch.tensor([3, 2, 2, 0], device="cuda"))
    assert torch.equal(c[0], a[3]) and torch.equal(c[1], a[2]) and torch.equal(c[2], a[2]) and torch.equal(c[3], a[0])
    assert walk.render_batch([]).shape == (0, 360, 480, 3)


def test_render_has_no_side_effects():
    import torch
    from rex_gym_b200.envs.batched_env import RexWalkBatchEnv
    kw = dict(num_envs=8, signal_type="ik", target_position=2.0, backwards=False, seed=7)
    a, b = RexWalkBatchEnv(**kw), RexWalkBatchEnv(**kw)
    a.reset(); b.reset()
    rng = np.random.default_rng(3)
    for t in range(12):
        act = rng.uniform(-0.4, 0.4, size=(8, 2)).astype(np.float32)
        sd = a.state_dict()
        a.render_batch(np.arange(8), width=64, height=48)
        a.render()
        sd2 = a.state_dict()
        assert torch.equal(sd["state_f"], sd2["state_f"]) and torch.equal(sd["state_i"], sd2["state_i"])
        oa, ra, da, _ = a.step(act)
        ob, rb, db, _ = b.step(act)
        assert np.array_equal(oa, ob) and np.array_equal(ra, rb) and np.array_equal(da, db)
    assert a.check_errors() == 0
    a.close(); b.close()


def test_robot_far_away_leaves_the_oracle_ground(walk):
    st = walk.get_state()
    pos = st["pos"].copy()
    pos[0] = [100.0, 0.0, 0.2]
    walk.set_state(pos, st["quat"], st["linvel"], st["angvel"], st["q"], st["qd"])
    try:
        img = walk.render_batch([0]).cpu().numpy()[0]
        st2 = walk.get_state()
        assert_frame(img, walk, 0, "at x = 100 m", st=st2)
        import render_oracle as RO
        val, gids = oracle_samples(walk, 0, st=st2, draw_robot=False)
        _, rids = oracle_samples(walk, 0, st=st2)
        free = ((rids < 0) | (rids >= RO.GROUND_ID)).all(0)     # pixels none of whose rays meets the robot
        RO.assert_pixels(img[free], val[:, free], gids[:, free], "ground at x = 100 m")
    finally:
        walk.set_state(st["pos"], st["quat"], st["linvel"], st["angvel"], st["q"], st["qd"])


def test_render_surface(walk):
    from rex_gym_b200.envs.single_env import RexWalkEnv
    f = walk.render()
    assert isinstance(f, np.ndarray) and f.shape == (360, 480, 3) and f.dtype == np.uint8
    assert np.array_equal(f, walk.render_batch([0])[0].cpu().numpy())
    assert np.array_equal(walk[2].render(), walk.render_batch([2])[0].cpu().numpy())
    assert walk.render("human").size == 0 and walk[1].render("human").size == 0
    e = RexWalkEnv()
    e.reset()
    assert e.render().shape == (360, 480, 3) and e.render("human").size == 0
    e.close()


def test_index_checks(walk):
    import torch
    with pytest.raises(IndexError):
        walk.render_batch([0, 4])
    with pytest.raises(IndexError):
        walk.render_batch([-1])
    with pytest.raises(ValueError):
        walk.render_batch([0], width=0)
    walk.check_errors()
    img = walk.render_batch(torch.tensor([1, 7], device="cuda")).cpu().numpy()
    from rex_gym_b200 import model_tables as MT
    sky = np.floor(MT.pack_render_tables("base")[MT.RT_SKY:MT.RT_SKY + 3].astype(np.float64) * 255 + 0.5)
    assert (img[1] == sky.astype(np.uint8)).all()
    with pytest.raises(IndexError):
        walk.check_errors()
    assert walk.check_errors() == 0

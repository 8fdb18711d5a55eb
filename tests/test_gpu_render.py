"""rgb_array renderer on the device against the fp64 render oracle (tests/render_oracle.py), and its contract: deterministic,
independent of the other images of a call, free of side effects, index checks."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

I_FIELD = 4     # int state word of the env's heightfield (rexsim_kernel.cuh)


def assert_frames_match(got, ref, ids, what=""):
    """At most 0.5 % of pixels differ by more than 2/255 in a channel, and each such pixel lies within 1 px of a change of
    surface patch in the oracle's id image: fp32 / fp64 flips at silhouettes, face edges, checker lines and triangle edges."""
    assert got.shape == ref.shape and got.dtype == np.uint8
    bad = (np.abs(got.astype(np.int16) - ref.astype(np.int16)) > 2).any(-1)
    frac = bad.mean()
    assert frac <= 0.005, "%s: %.3f %% of pixels differ" % (what, 100 * frac)
    H, W = ids.shape
    pad = np.pad(ids, 1, mode="edge")
    edge = np.zeros((H, W), bool)
    for dy in (0, 1, 2):
        for dx in (0, 1, 2):
            edge |= pad[dy:dy + H, dx:dx + W] != ids
    off = bad & ~edge
    assert not off.any(), "%s: %d differing pixels away from any patch edge, first at %s" % (what, off.sum(), np.argwhere(off)[:3])


def oracle_frame(env, i, width=480, height=360, distance=1.0, yaw=0.0, pitch=-30.0, st=None, draw_robot=True):
    import render_oracle as RO
    st = st or env.get_state()
    heights = None
    if env.terrain_type == "random":
        field = int(env.state_dict()["state_i"][I_FIELD, i].item())
        heights = env._fields[field].cpu().numpy().reshape(256, 256)
    return RO.render(env.mark, st["pos"][i].astype(np.float64), st["quat"][i].astype(np.float64), st["q"][i].astype(np.float64),
                     width, height, distance, yaw, pitch, env.terrain_type, heights, draw_robot=draw_robot)


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
        ref, ids = oracle_frame(walk, i)
        assert_frames_match(img[i], ref, ids, "walk env %d" % i)


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
        ref, ids = oracle_frame(env, i, st=st)
        assert_frames_match(img[i], ref, ids, "turn env %d" % i)
    env.close()


def test_standup_with_the_arm_matches_oracle():
    from rex_gym_b200.envs.batched_env import RexStandupBatchEnv
    env = stepped(RexStandupBatchEnv(num_envs=2, mark="arm"), 50, 0.1, seed=2)
    img = env.render_batch([0, 1]).cpu().numpy()
    import render_oracle as RO
    for i in range(2):
        ref, ids = oracle_frame(env, i)
        assert_frames_match(img[i], ref, ids, "standup arm env %d" % i)
        shapes = set((ids[(ids >= 0) & (ids < RO.GROUND_ID)] // 1000 - 1).tolist())
        assert any(s >= 19 for s in shapes)                 # the arm is in the picture
    env.close()


def test_top_down_camera_and_odd_sizes(walk):
    img = walk.render_batch([1], distance=3.0, yaw=90.0, pitch=-89.0).cpu().numpy()[0]
    ref, ids = oracle_frame(walk, 1, distance=3.0, yaw=90.0, pitch=-89.0)
    assert_frames_match(img, ref, ids, "yaw 90 pitch -89")
    for w, h in ((97, 61), (1, 1)):
        img = walk.render_batch([0, 3], width=w, height=h).cpu().numpy()
        assert img.shape == (2, h, w, 3)
        for k, i in enumerate((0, 3)):
            ref, ids = oracle_frame(walk, i, width=w, height=h)
            assert_frames_match(img[k], ref, ids, "%dx%d env %d" % (w, h, i))


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
        ref, ids = oracle_frame(walk, 0, st=st2)
        assert_frames_match(img, ref, ids, "at x = 100 m")
        ground, gids = oracle_frame(walk, 0, st=st2, draw_robot=False)
        import render_oracle as RO
        robot = (ids >= 0) & (ids < RO.GROUND_ID)
        pad = np.pad(robot, 1)
        near = np.zeros_like(robot)
        for dy in (0, 1, 2):
            for dx in (0, 1, 2):
                near |= pad[dy:dy + robot.shape[0], dx:dx + robot.shape[1]]
        free = ~near                                             # pixels the robot's silhouette does not reach
        assert_frames_match(np.where(free[..., None], img, ground), ground, gids, "ground at x = 100 m")
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

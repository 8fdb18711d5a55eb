"""CPU suite: the C-ABI library loads and exports every symbol include/rexsim.h declares (no compute calls
without a GPU), host-only entry points, packer layout, no-CPU-fallback behaviour."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "rexsim.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(rexsim_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from rex_gym_b200 import _capi
    L = _capi.load()
    names = header_functions()
    assert len(names) >= 14
    for n in names:
        assert hasattr(L, n), n
    assert sorted(_capi.EXPORTS) == names


def test_host_only_entry_points():
    from rex_gym_b200 import _capi
    L = _capi.load()
    # widths of the reference spaces: walk_env.py:108-113, gallop_env.py:123-127,349-356, turn_env.py:104-108
    assert [L.rexsim_action_dim(t, s) for t, s in ((0, 0), (0, 1), (1, 0), (1, 1), (2, 0), (2, 1), (3, 1))] == [2, 8, 2, 4, 2, 2, 1]
    assert [L.rexsim_obs_dim(t, 12) for t in range(4)] == [4, 16, 4, 4]
    cfg = _capi.RexSimConfig()
    nf, ni = C.c_int32(), C.c_int32()
    assert L.rexsim_state_words(C.byref(cfg), C.byref(nf), C.byref(ni)) == 0
    assert nf.value == 55 and ni.value == 17          # + I_HPUSH (rows pushed into the sensor history)


def test_create_rejects_bad_arguments_without_touching_the_gpu():
    from rex_gym_b200 import _capi
    L = _capi.load()
    cfg = _capi.RexSimConfig()
    h = C.c_void_p()
    tb = np.zeros(952, np.float32)
    assert L.rexsim_create(C.byref(cfg), tb.ctypes.data, 952, C.byref(h)) == -1          # num_envs = 0
    cfg.num_envs, cfg.num_motors, cfg.task, cfg.action_repeat, cfg.solver_iterations, cfg.sim_dt_d, cfg.toe_npts = 8, 12, 0, 5, 60, 0.001, 27
    cfg.gait_clock_scale = 1.0
    assert L.rexsim_create(C.byref(cfg), tb.ctypes.data, 951, C.byref(h)) == -2          # model table size
    cfg.num_motors, cfg.task = 18, 1
    assert L.rexsim_create(C.byref(cfg), tb.ctypes.data, 952 + 192, C.byref(h)) == -4    # arm + gallop not built
    assert b"arm" in L.rexsim_last_error()
    with pytest.raises(ValueError):
        _capi.check(-4)


def test_rng_is_bit_identical_to_the_oracle():
    from rex_gym_b200 import _capi
    from oracle import oracle as O
    L, R = _capi.load(), O.lib()
    rng = np.random.default_rng(0)
    for _ in range(500):
        s, e, r, k = int(rng.integers(0, 2**63)), int(rng.integers(0, 2**31)), int(rng.integers(0, 2**31)), int(rng.integers(0, 8))
        assert L.rexsim_rand_u32(s, e, r, k) == R.rexo_rand_u32(s, e, r, k)


def test_sensor_noise_generator_matches_the_oracle():
    """Rex._AddSensorNoise (rex.py:763-769) draws from the unseeded np.random.normal; both sides replace it by the same
    counter-based Box-Muller draw.  The library evaluates it in float (as the device does), the oracle in double."""
    from rex_gym_b200 import _capi
    from oracle import oracle as O
    L, R = _capi.load(), O.lib()
    rng = np.random.default_rng(1)
    got, want = [], []
    for _ in range(4000):
        s, e, r = int(rng.integers(0, 2**63)), int(rng.integers(0, 2**20)), int(rng.integers(1, 2**16))
        st, site, comp = int(rng.integers(0, 3000)), int(rng.integers(0, 8)), int(rng.integers(0, 18))
        got.append(L.rexsim_noise(s, e, r, st, site, comp)); want.append(R.rexo_noise(s, e, r, st, site, comp))
    got, want = np.array(got), np.array(want)
    assert np.abs(got - want).max() < 5e-6
    assert abs(want.mean()) < 0.06 and abs(want.std() - 1.0) < 0.05          # N(0, 1)


def test_sensor_history_depth_follows_the_deque_reads():
    """_GetDelayedObservation (rex.py:735-753) reads history[n] and history[n + 1], n = int(latency / dt); the deque keeps 100."""
    from rex_gym_b200 import _capi
    L = _capi.load()
    cfg = _capi.RexSimConfig()
    cfg.sim_dt_d = 0.001
    assert L.rexsim_history_depth(C.byref(cfg)) == 0                       # reference default: no history at all
    cfg.noise_stdev[3] = 0.01
    assert L.rexsim_history_depth(C.byref(cfg)) == 2
    cfg.control_latency, cfg.pd_latency = 0.02, 0.003
    assert L.rexsim_history_depth(C.byref(cfg)) == 22
    cfg.pd_latency = 0.0305
    assert L.rexsim_history_depth(C.byref(cfg)) == 32
    cfg.control_latency = 0.2
    assert L.rexsim_history_depth(C.byref(cfg)) == 100
    cfg.control_latency = -1.0
    cfg.num_envs, cfg.num_motors, cfg.action_repeat, cfg.solver_iterations, cfg.toe_npts, cfg.gait_clock_scale = 8, 12, 5, 60, 27, 1.0
    h = C.c_void_p()
    tb = np.zeros(952, np.float32)
    assert L.rexsim_create(C.byref(cfg), tb.ctypes.data, 952, C.byref(h)) == -1 and b"latenc" in L.rexsim_last_error()


def test_model_table_packer_layout():
    from rex_gym_b200.model_tables import pack_model_tables, MT_LEG, MT_TOE, MT_BOX, MT_BASEBOX, MT_FLOATS
    t, npts = pack_model_tables("base")
    assert t.dtype == np.float32 and t.shape == (MT_FLOATS,) and MT_FLOATS * 4 % 16 == 0   # TMA bulk copy granularity
    assert npts == 68                                # profile vertices of the toe prism (exact hull of stl/foot.stl, curved part)
    assert abs(t[0] - 1.3) < 1e-6 and abs(t[10] - 1.2) < 1e-6                             # merged base / un-merged root mass
    legs = t[MT_LEG:MT_LEG + 192].reshape(4, 3, 16)
    np.testing.assert_allclose(legs[:, 0, :3], [[-0.093, -0.036, 0], [-0.093, 0.036, 0], [0.093, -0.036, 0], [0.093, 0.036, 0]], atol=1e-7)
    np.testing.assert_allclose(legs[:, 1, 3], 0.6, atol=1e-6)                            # leg link + 0.5 kg cover (rex.urdf)
    np.testing.assert_allclose(legs[:, 2, 7], -0.1, atol=1e-6); np.testing.assert_allclose(legs[:, 2, 14], 2.59, atol=1e-6)
    toe = t[MT_TOE:MT_TOE + 384].reshape(192, 2)         # (x, z) profile in the foot frame, shared by the four feet
    assert np.all(toe[npts:] == 0) and np.all(np.abs(toe[:npts, 0]) < 0.02) and np.all(toe[:npts, 1] < -0.10)
    assert abs(toe[:npts, 1].min() + 0.13444) < 1e-4                                        # lowest hull point: 134.4 mm below the knee
    assert abs(t[15] - 0.01) < 1e-7                                                         # prism half width
    assert t[MT_BOX:MT_BASEBOX].reshape(4, 3, 8, 3).shape == (4, 3, 8, 3)


def test_arm_collision_points_are_the_oracles():
    """The arm's collision points (mark 'arm': six contact groups, 16 per cylinder + the 8 corners of arm_section_4's box) are
    packed body by body in the order the oracle scans its contact groups 9-14, with each body's count, start and reach."""
    from oracle.oracle import load_model
    from rex_gym_b200.model_tables import pack_model_tables, MT_ARM, ARM_STRIDE, MT_ARMPTS, ARMPTS_N, MT_FLOATS_ARM
    t, _ = pack_model_tables("arm")
    assert t.shape == (MT_FLOATS_ARM,) and MT_FLOATS_ARM * 4 % 16 == 0 and ARMPTS_N == 104
    m, _ = load_model("arm")
    assert m.nshape == 15
    for k in range(6):
        o = MT_ARM + ARM_STRIDE * k
        g = 9 + k
        n, s = int(t[o + 27]), int(t[o + 28])
        assert n == m.shape_npts[g] == (24 if k == 4 else 16)
        ref = np.array([m.pts[m.shape_start[g] + v][:] for v in range(n)])
        assert all(m.pt_body[m.shape_start[g] + v] == 13 + k for v in range(n))
        np.testing.assert_array_equal(t[MT_ARMPTS + 3 * s:MT_ARMPTS + 3 * (s + n)].reshape(n, 3), ref.astype(np.float32))
        assert abs(t[o + 29] - np.linalg.norm(ref, axis=1).max()) < 1e-6
    assert int(t[MT_ARM + ARM_STRIDE * 5 + 28]) + int(t[MT_ARM + ARM_STRIDE * 5 + 27]) == ARMPTS_N


def test_no_cpu_fallback():
    import torch
    import rex_gym_b200 as R
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        R.make("RexWalk-v0", num_envs=4)


def test_reference_surface_names():
    import rex_gym_b200 as R
    assert set(R.ENV_IDS) == {"RexWalk-v0", "RexGalloping-v0", "RexTurn-v0", "RexStandup-v0", "RexPoses-v0"}       # playground/__init__.py:17-57
    for m in ("step", "reset", "close", "__len__", "__getitem__"):                  # batch_env.py:44-115
        assert hasattr(R.BatchedRexEnv, m)
    with pytest.raises(ValueError):
        R.make("RexGo-v0")
    from rex_gym_b200.envs.gym import walk_env, gallop_env, turn_env, standup_env     # the reference's module paths
    assert walk_env.RexWalkEnv and gallop_env.RexReactiveEnv and turn_env.RexTurnEnv and standup_env.RexStandupEnv


def test_terrain_bank_is_what_the_reference_hands_to_pybullet():
    """tests/golden/terrain_golden.json (tools/gen_terrain_golden.py): the heights the reference's unmodified Terrain class passed
    to createCollisionShape for its first three terrains (construction, then two update_terrain() = two resets), as float32
    hashes + samples.  Bank field k is bit-for-bit the k-th of them, in the product's bank and in the oracle's."""
    import hashlib
    import json
    from rex_gym_b200 import terrain as T
    from oracle.oracle import make_fields
    g = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "terrain_golden.json")))
    assert (g["rows"], g["columns"]) == (T.ROWS, T.COLUMNS) and g["mesh_scale"] == [T.CELL, T.CELL, 1] == g["update_mesh_scale"]
    assert g["init_position_random"] == [0, 0, 0.21]
    ours, orac = T.make_random_fields(3), make_fields(3)
    for k, want in enumerate(g["fields"]):
        for f in (ours[k], orac[k]):
            flat = np.ascontiguousarray(f, np.float32).reshape(-1)
            assert hashlib.sha256(flat.tobytes()).hexdigest() == want["sha256_float32"], k
            np.testing.assert_array_equal(flat[::257], np.array(want["every_257th"], np.float32))
        assert 0 <= want["min"] and want["max"] <= T.PERTURBATION


def test_terrain_bank_follows_the_reference_stream():
    """field 0 = first generate_terrain() of the reference: random.seed(10), 2x2 blocks of U(0, 0.05)
    (rex_gym/model/terrain.py:26,36-44)."""
    import random
    from rex_gym_b200.terrain import make_random_fields
    f = make_random_fields(2)
    rnd = random.Random(10)
    first = [rnd.uniform(0, 0.05) for _ in range(5)]
    assert f.shape == (2, 256, 256)
    np.testing.assert_allclose(f[0].reshape(-1)[[0, 1, 256, 257]], np.float32(first[0]))
    np.testing.assert_allclose(f[0].reshape(-1)[2], np.float32(first[1]))
    assert f.min() >= 0 and f.max() <= 0.05 and not np.array_equal(f[0], f[1])

"""rgb_array renderer, CPU side: the follow camera's convention, the model data the renderer reads, the C ABI symbols, and the
fp64 render oracle on the standing robot."""
import hashlib
import os

import numpy as np

from rex_gym_b200 import model_tables as MT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# sha256 of pack_model_tables(mark) before the renderer's JSON keys were added: the physics' table must not move
MODEL_TABLE_SHA256 = {"base": "24f040ebe8aaaad66fee8a8ef19c4e59248bd77eaf497e310d3a5959ffc94f70",
                      "arm": "cf551820d133bb44d4b3c4e00b3fce36371787df802e25fe3be1783218265a30"}


def test_camera_at_the_reference_parameters():
    import render_oracle as RO
    target = np.array([0.3, -0.2, 0.21])
    eye, f, s, u, up = RO.camera(target, 1.0, 0.0, -30.0)          # rex_gym_env.py:214-216
    assert np.allclose(eye - target, [0.0, -0.8660254, 0.5], atol=1e-7)
    assert np.allclose(up, [0.0, 0.5, 0.8660254], atol=1e-7)
    assert np.allclose(u, up, atol=1e-12)                            # the view's up is the camera's up at roll 0
    assert np.allclose(np.cross(s, f), u) and abs(f @ s) < 1e-15


def test_centre_ray_passes_through_the_target_and_ground_rows_lie_below_the_horizon():
    import render_oracle as RO
    target = np.array([1.0, 2.0, 0.2])
    eye, f, s, u, _ = RO.camera(target, 1.0, 0.0, -30.0)
    r = RO.rays(f, s, u, 481, 361)                                   # odd sides: one pixel centre on the optical axis
    c = r[180, 240]
    assert np.allclose(eye + 1.0 * c, target, atol=1e-12)
    r = RO.rays(f, s, u, 480, 360)
    assert (r[..., 2] < 0).all()                                     # every pixel of every row looks down at the ground
    assert r[0, :, 2].max() > -0.01                                  # ... and the horizon is the image's top edge
    rgb, ids = RO.render("base", target, [0, 0, 0, 1], np.zeros(12), 480, 360, draw_robot=False)
    ground = ids >= RO.GROUND_ID
    assert ground[-1].all() and ground[180].all()
    sky = MT.pack_render_tables("base")[MT.RT_SKY:MT.RT_SKY + 3]
    assert (ids[ground.sum(1) == 0] == -1).all()                     # rows beyond the far plane are sky
    assert np.abs(rgb[0, 0].astype(float) / 255 - sky).max() < 1 / 255


def test_standing_robot_is_centred_in_the_oracle_frame():
    import render_oracle as RO
    q = np.tile([0.0, -0.88643435, 1.30197369], 4)                   # INIT_POSES['stand']
    rgb, ids = RO.render("base", [0.0, 0.0, 0.21], [0, 0, 0, 1], q, 97, 61)
    assert 1000 <= ids[30, 48] < 4000                                # the optical axis meets the base / chassis boxes
    shapes = set((ids[(ids >= 0) & (ids < RO.GROUND_ID)] // 1000 - 1).tolist())
    assert set(range(0, 3)) <= shapes and any(15 <= s < 19 for s in shapes)
    assert rgb.dtype == np.uint8 and rgb.shape == (61, 97, 3)


def test_model_tables_unchanged_and_render_keys_present():
    for mark in ("base", "arm"):
        t, _ = MT.pack_model_tables(mark)
        assert hashlib.sha256(t.tobytes()).hexdigest() == MODEL_TABLE_SHA256[mark]
        j = MT.load_model_json(mark)
        for b in j["bodies"]:
            assert sorted(b["link_rgba"]) == sorted(b["links"])
            for s in b["shapes"]:
                assert b["link_rgba"][s["link"]] is not None and len(b["link_rgba"][s["link"]]) == 4
                if s["kind"] == "cylinder":
                    assert s["radius"] > 0 and s["length"] > 0 and len(s["origin_xyz"]) == 3
                    assert np.allclose(np.asarray(s["origin_rot"]) @ np.asarray(s["origin_rot"]).T, np.eye(3))
        rt = MT.pack_render_tables(mark)
        assert rt.shape == (MT.RT_FLOATS,) and rt.dtype == np.float32
        cols = rt[MT.RT_COLOR:MT.RT_COLOR + 3 * MT.RT_NSHAPES].reshape(-1, 3)
        assert np.allclose(cols[0], [0.1, 0.1, 0.1]) and np.allclose(cols[1], [0.92, 0.83, 0.0])   # black base, yellow chassis
        assert np.allclose(cols[15:19], 0.6)                                                        # grey toes


def test_render_table_layout_matches_the_header():
    src = open(os.path.join(ROOT, "include", "rexsim.h")).read()
    for name in ("LIGHT", "SKY", "CHECK", "CAM", "COLOR", "TOE", "TOESPH", "CYL", "ARMBOX", "FLOATS", "NSHAPES"):
        import re
        m = re.search(r"#define REXSIM_RT_%s (\d+)" % name, src)
        assert m and int(m.group(1)) == getattr(MT, "RT_" + name), name


def test_render_is_exported():
    from rex_gym_b200 import _capi
    L = _capi.load()
    assert hasattr(L, "rexsim_render") and hasattr(L, "rexsim_set_render_tables")

"""Per-env constructor values without a GPU: the keyword checks that come before any CUDA call, each entry's meaning, the
library's row layout and the sharding slices."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
NEW = ("rexsim_value_row", "rexsim_set_env_values", "rexsim_set_task_values", "rexsim_env_value_buffers")


def _no_cuda(monkeypatch):
    import torch
    from rex_gym_b200 import _capi

    def touched(*a, **k):
        raise AssertionError("CUDA touched before the keywords were checked")
    monkeypatch.setattr(torch.cuda, "is_available", touched)
    monkeypatch.setattr(_capi, "load", touched)


N = 4
REFUSED = [
    ("wrong length", dict(target_position=[1.0, 2.0])),
    ("wrong length of a tensor", dict(base_yaw=np.zeros((N, 2)))),
    ("wrong length of gains", dict(motor_kp=[1.0] * (N + 1))),
    ("backwards outside -1/0/1", dict(backwards=[0, 1, 2, -1])),
    ("backwards fraction", dict(backwards=[0, 0.5, 1, 1])),
    ("negative kp", dict(motor_kp=[1.0, -0.1, 1.0, 1.0])),
    ("negative kd", dict(motor_kd=[0.02, 0.02, -1e-3, 0.02])),
    ("non-finite kp", dict(motor_kp=[1.0, np.inf, 1.0, 1.0])),
    ("NaN kd", dict(motor_kd=[0.02, np.nan, 0.02, 0.02])),
    ("per-env kp with a kp range", dict(motor_kp=[1.0] * N, motor_kp_range=(0.8, 1.2))),
    ("per-env kd with a kd range", dict(motor_kd=[0.02] * N, motor_kd_range=(0.01, 0.03))),
    ("per-env kp with a kd range", dict(motor_kp=[1.0] * N, motor_kd_range=(0.01, 0.03))),
]


@pytest.mark.parametrize("why,kw", REFUSED, ids=[r[0] for r in REFUSED])
def test_refusals_come_before_any_cuda_call(why, kw, monkeypatch):
    import rex_gym_b200 as R
    _no_cuda(monkeypatch)
    with pytest.raises(ValueError):
        R.BatchedRexEnv(task="walk", num_envs=N, **kw)


def test_more_than_64_gain_pairs_are_refused_before_any_cuda_call(monkeypatch):
    import rex_gym_b200 as R
    _no_cuda(monkeypatch)
    n = 130
    kp = 1.0 + 0.01 * (np.arange(n) % 65)
    with pytest.raises(ValueError, match="64"):
        R.BatchedRexEnv(task="walk", num_envs=n, motor_kp=kp)
    # 64 pairs is the limit, not past it: the keywords pass and the first CUDA touch is reached
    with pytest.raises(AssertionError, match="CUDA touched"):
        R.BatchedRexEnv(task="walk", num_envs=n, motor_kp=1.0 + 0.01 * (np.arange(n) % 64))


def test_each_entry_means_what_the_scalar_means():
    import torch
    from rex_gym_b200.envs.batched_env import TASK_VALUE_KEYWORDS, check_env_values, task_value
    nan = float("nan")
    vals = dict(target_position=[None, 0.0, 2.0, nan], backwards=[None, False, True, -1], target_orient=torch.tensor([0.5, nan, 1.0, 2.0]),
                init_orient=1.5, base_y=None, base_z=np.array([0.0, 0.01, nan, 0.0]))
    rows, gains = check_env_values(N, vals, 1.0, 0.02)
    assert gains is None and set(rows) == set(TASK_VALUE_KEYWORDS)
    eq = np.testing.assert_array_equal
    eq(rows["target_position"], np.float32([nan, nan, 2.0, nan]))            # None and 0 draw, as the scalar
    eq(rows["backwards"], np.float32([-1, 0, 1, -1]))
    eq(rows["target_orient"], np.float32([0.5, nan, 1.0, 2.0]))
    eq(rows["init_orient"], np.full(N, 1.5, np.float32))                     # scalars are repeated
    eq(rows["base_z"], np.float32([0.0, 0.01, nan, 0.0]))
    for k in ("base_y", "base_roll", "base_pitch", "base_yaw"):
        assert np.isnan(rows[k]).all()
    # the scalar rule itself is today's
    assert np.isnan(task_value("target_position", 0)) and task_value("backwards", None) == -1 and task_value("backwards", 1) == 1


def test_scalars_switch_nothing_on_and_gains_alone_fill_every_row():
    from rex_gym_b200.envs.batched_env import TASK_VALUE_KEYWORDS, check_env_values
    assert check_env_values(N, dict(target_position=2.0, backwards=True), 1.0, 0.02) == (None, None)
    rows, (kp, kd) = check_env_values(N, dict(target_position=2.0, backwards=True), [1.0, 1.2, 1.0, 0.9], 0.03)
    assert set(rows) == set(TASK_VALUE_KEYWORDS)
    np.testing.assert_array_equal(rows["target_position"], np.full(N, 2.0, np.float32))
    np.testing.assert_array_equal(rows["backwards"], np.ones(N, np.float32))
    np.testing.assert_array_equal(kp, np.float32([1.0, 1.2, 1.0, 0.9]))
    np.testing.assert_array_equal(kd, np.full(N, 0.03, np.float32))


def test_the_library_owns_the_row_layout():
    from rex_gym_b200 import _capi
    from rex_gym_b200.envs.batched_env import TASK_VALUE_KEYWORDS
    L = _capi.load()
    rows = [L.rexsim_value_row(k.encode()) for k in TASK_VALUE_KEYWORDS]
    assert sorted(rows) == list(range(len(TASK_VALUE_KEYWORDS)))
    assert L.rexsim_value_row(b"motor_kp") == -1 and L.rexsim_value_row(b"energy_weight") == -1
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rexsim.h")).read(), flags=re.S)
    for name in NEW:
        assert name in _capi.SIGNATURES and name in _capi.EXPORTS
        assert re.search(r"\b%s\s*\(" % name, header), name
        assert hasattr(L, name)


def test_sharding_slices_global_arrays(monkeypatch):
    from rex_gym_b200 import sharding
    import rex_gym_b200.envs.batched_env as B
    seen = []
    monkeypatch.setattr(B, "BatchedRexEnv", lambda **kw: seen.append(kw) or kw)
    g = 8
    tp, kp = np.arange(g, dtype=np.float32) + 1, [1.0, 1.1] * 4
    for rank in range(2):
        sharding.make_sharded_env(g, rank, 2, task="walk", target_position=tp, backwards=[0, 1, -1, 0, 1, -1, 0, 1], motor_kp=kp,
                                  init_orient=0.5)
    a, b = seen
    assert (a["env_offset"], a["num_envs"], b["env_offset"], b["num_envs"]) == (0, 4, 4, 4)
    np.testing.assert_array_equal(a["target_position"], tp[:4])
    np.testing.assert_array_equal(b["target_position"], tp[4:])
    assert list(b["backwards"]) == [1, -1, 0, 1] and list(b["motor_kp"]) == [1.0, 1.1, 1.0, 1.1]
    assert a["init_orient"] == 0.5 and b["init_orient"] == 0.5                # scalars pass through

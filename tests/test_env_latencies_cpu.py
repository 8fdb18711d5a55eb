"""Per-env sensor latencies without a GPU: the keyword checks that come before any CUDA call, the values handed to the
library, the ABI symbols, the sharding slices and set_task_values' refusal."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
NEW = ("rexsim_set_env_latencies", "rexsim_env_latency_buffers")
N = 4


def _no_cuda(monkeypatch):
    import torch
    from rex_gym_b200 import _capi

    def touched(*a, **k):
        raise AssertionError("CUDA touched before the keywords were checked")
    monkeypatch.setattr(torch.cuda, "is_available", touched)
    monkeypatch.setattr(_capi, "load", touched)


REFUSED = [
    ("wrong length", dict(control_latency=[0.0, 0.01])),
    ("wrong length of pd", dict(pd_latency=np.zeros(N + 1))),
    ("two dimensions", dict(control_latency=np.zeros((N, 2)))),
    ("negative control latency", dict(control_latency=[0.0, -0.001, 0.0, 0.0])),
    ("negative pd latency", dict(pd_latency=[0.0, 0.0, -1e-4, 0.0])),
    ("NaN control latency", dict(control_latency=[0.0, np.nan, 0.0, 0.0])),
    ("NaN pd latency", dict(pd_latency=[np.nan, 0.0, 0.0, 0.0])),
    ("infinite pd latency", dict(pd_latency=[0.0, np.inf, 0.0, 0.0])),
    ("negative scalar beside an array", dict(control_latency=[0.0] * N, pd_latency=-0.001)),
]


@pytest.mark.parametrize("why,kw", REFUSED, ids=[r[0] for r in REFUSED])
def test_refusals_come_before_any_cuda_call(why, kw, monkeypatch):
    import rex_gym_b200 as R
    _no_cuda(monkeypatch)
    with pytest.raises(ValueError):
        R.BatchedRexEnv(task="walk", num_envs=N, **kw)


def test_more_than_64_hold_settings_are_refused_before_any_cuda_call(monkeypatch):
    import rex_gym_b200 as R
    _no_cuda(monkeypatch)
    n = 130
    with pytest.raises(ValueError, match="64"):
        R.BatchedRexEnv(task="walk", num_envs=n, pd_latency=1e-5 * (np.arange(n) % 65))
    # settings count (kp, kd, pd_latency) triples: 8 gain pairs x 9 latencies is 72, past the cap
    with pytest.raises(ValueError, match="64"):
        R.BatchedRexEnv(task="walk", num_envs=n, motor_kp=1.0 + 0.01 * (np.arange(n) % 8), pd_latency=1e-4 * (np.arange(n) % 9))
    # 64 settings is the limit, not past it; control latencies do not count
    with pytest.raises(AssertionError, match="CUDA touched"):
        R.BatchedRexEnv(task="walk", num_envs=n, pd_latency=1e-5 * (np.arange(n) % 64), control_latency=1e-3 * np.arange(n))
    with pytest.raises(AssertionError, match="CUDA touched"):
        R.BatchedRexEnv(task="walk", num_envs=n, motor_kp=1.0 + 0.01 * (np.arange(n) % 8), pd_latency=1e-4 * (np.arange(n) % 8))


def test_latencies_combine_with_gain_ranges(monkeypatch):
    """Drawn gains hold the reset at the scalar gains: one setting per distinct pd_latency."""
    import rex_gym_b200 as R
    _no_cuda(monkeypatch)
    with pytest.raises(AssertionError, match="CUDA touched"):
        R.BatchedRexEnv(task="gallop", signal_type="ol", num_envs=N, pd_latency=[0.0, 0.001, 0.0, 0.0005],
                        motor_kp_range=(0.8, 1.2), motor_kd_range=(0.01, 0.03))


def test_values_handed_to_the_library():
    import torch
    from rex_gym_b200.envs.batched_env import check_env_latencies
    assert check_env_latencies(N, 0.01, 0.0) is None                              # scalars switch nothing on
    ctl, pd = check_env_latencies(N, [0.0, 0.0105, 0.02, 0.0105], 0.001)
    assert ctl.dtype == np.float64 and pd.dtype == np.float64                     # fp64, as the config's scalars
    np.testing.assert_array_equal(ctl, [0.0, 0.0105, 0.02, 0.0105])               # the Python floats themselves, not fp32
    np.testing.assert_array_equal(pd, np.full(N, 0.001))                          # a scalar is repeated
    ctl, pd = check_env_latencies(N, 0.0, torch.tensor([0.0, 5e-4, 1e-3, 0.0], dtype=torch.float64))
    np.testing.assert_array_equal(ctl, np.zeros(N))
    np.testing.assert_array_equal(pd, [0.0, 5e-4, 1e-3, 0.0])


def test_set_task_values_refuses_latencies():
    from rex_gym_b200.envs.batched_env import BatchedRexEnv
    env = BatchedRexEnv.__new__(BatchedRexEnv)             # the keyword check comes before the batch is looked at
    for kw in (dict(control_latency=0.01), dict(pd_latency=[0.001] * N)):
        with pytest.raises(ValueError, match="fixed at construction"):
            env.set_task_values(**kw)


def test_the_library_exports_the_entry_points():
    from rex_gym_b200 import _capi
    L = _capi.load()
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rexsim.h")).read(), flags=re.S)
    for name in NEW:
        assert name in _capi.SIGNATURES and name in _capi.EXPORTS
        assert re.search(r"\b%s\s*\(" % name, header), name
        assert hasattr(L, name)
    assert L.rexsim_set_env_latencies(None, None, None) == -1                     # REXSIM_ERR_INVALID, no handle touched


def test_sharding_slices_global_latency_arrays(monkeypatch):
    from rex_gym_b200 import sharding
    import rex_gym_b200.envs.batched_env as B
    seen = []
    monkeypatch.setattr(B, "BatchedRexEnv", lambda **kw: seen.append(kw) or kw)
    g = 8
    ctl = np.arange(g) * 0.001
    for rank in range(2):
        sharding.make_sharded_env(g, rank, 2, task="walk", control_latency=ctl, pd_latency=[0.0, 0.001] * 4)
    a, b = seen
    np.testing.assert_array_equal(a["control_latency"], ctl[:4])
    np.testing.assert_array_equal(b["control_latency"], ctl[4:])
    assert list(b["pd_latency"]) == [0.0, 0.001, 0.0, 0.001]
    seen.clear()
    sharding.make_sharded_env(g, 1, 2, task="walk", control_latency=0.01)
    assert seen[0]["control_latency"] == 0.01                                    # scalars pass through

"""Per-env control rates without a GPU: the keyword checks that come before any CUDA call (one simulation time step for the
batch, positive integer repeats, one solver_iterations), the per-env int(300 / action_repeat) rule, the collapse of
all-equal arrays to the scalar construction, set_task_values' refusal, the sharding slices and the ABI symbols."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
NEW = ("rexsim_set_env_repeats", "rexsim_env_repeat_buffers", "rexsim_launch_groups", "rexsim_launch_group",
       "rexsim_slot_buffers")
N = 4


def _no_cuda(monkeypatch):
    import torch
    from rex_gym_b200 import _capi

    def touched(*a, **k):
        raise AssertionError("CUDA touched before the keywords were checked")
    monkeypatch.setattr(torch.cuda, "is_available", touched)
    monkeypatch.setattr(_capi, "load", touched)


REFUSED = [
    ("time steps differ", dict(control_time_step=[0.005, 0.006, 0.005, 0.005], action_repeat=5), "simulation time steps differ"),
    ("repeat alone differs", dict(control_time_step=0.005, action_repeat=[5, 5, 10, 5]), "BatchEnv refuses the mix"),
    ("per-env solver_iterations", dict(action_repeat=[5, 10, 5, 10], control_time_step=[0.005, 0.01, 0.005, 0.01],
                                       solver_iterations=[60, 30, 60, 30]), "solver_iterations takes one value"),
    ("zero repeat entry", dict(action_repeat=[5, 0, 5, 5]), "not a positive integer"),
    ("negative repeat", dict(action_repeat=-5), "not a positive integer"),
    ("fractional repeat", dict(action_repeat=[5, 2.5, 5, 5]), "not a positive integer"),
    ("bool repeat", dict(action_repeat=[5, True, 5, 5]), "not a positive integer"),
    ("None repeat entry", dict(action_repeat=[5, None, 5, 5]), "not a positive integer"),
    ("negative time step", dict(control_time_step=[0.005, -0.005, 0.005, 0.005]), "positive finite"),
    ("infinite time step", dict(control_time_step=[0.005, float("inf"), 0.005, 0.005]), "positive finite"),
    ("NaN time step", dict(control_time_step=np.array([0.005, np.nan, 0.005, 0.005])), "positive finite"),
    ("string time step", dict(control_time_step=["0.005"] * N), "positive finite"),
    ("wrong length", dict(control_time_step=[0.005, 0.01], action_repeat=[5, 10]), "one entry per env"),
    ("two dimensions", dict(action_repeat=np.full((N, 1), 5)), "one entry per env"),
]


@pytest.mark.parametrize("why,kw,msg", REFUSED, ids=[r[0] for r in REFUSED])
def test_refusals_come_before_any_cuda_call(why, kw, msg, monkeypatch):
    import rex_gym_b200 as R
    _no_cuda(monkeypatch)
    with pytest.raises(ValueError, match=msg):
        R.BatchedRexEnv(task="walk", num_envs=N, **kw)


def test_more_than_eight_rates_are_refused(monkeypatch):
    import rex_gym_b200 as R
    _no_cuda(monkeypatch)
    n = 9
    with pytest.raises(ValueError, match="9 distinct"):
        R.BatchedRexEnv(task="walk", num_envs=n, control_time_step=[r / 1000 for r in range(1, 10)], action_repeat=list(range(1, 10)))


@pytest.mark.parametrize("kw", [dict(control_time_step=[0.005, 0.01, 0.006, 0.001], action_repeat=[5, 10, 6, 1]),
                                dict(control_time_step=np.array([0.012, 0.006, 0.006, 0.012]), action_repeat=(12, 6, 6, 12)),
                                dict(control_time_step=(0.004,) * N, action_repeat=np.full(N, 4))])
def test_accepted_arrays_reach_cuda(kw, monkeypatch):
    import rex_gym_b200 as R
    _no_cuda(monkeypatch)
    with pytest.raises(AssertionError, match="CUDA touched"):
        R.BatchedRexEnv(task="walk", num_envs=N, **kw)
    with pytest.raises(AssertionError, match="CUDA touched"):
        R.make("RexGalloping-v0", num_envs=N, **kw)


def test_every_millisecond_rate_up_to_twenty_is_one_time_step():
    assert all(r / 1000 / r == 0.001 for r in range(1, 21))           # fp64, as rex_gym_env.py:173 divides
    from rex_gym_b200.envs.batched_env import check_env_repeats
    for lo in (1, 9, 13):
        r = list(range(lo, lo + 8))
        cts, rep, dt, per_env = check_env_repeats(8, "walk", [x / 1000 for x in r], r)
        assert dt == 0.001 and rep == tuple(r) and per_env[0].tolist() == r


def test_iterations_follow_each_envs_repeat_unless_given():
    from rex_gym_b200.envs.batched_env import check_env_repeats
    cts, rep, dt, (r, it) = check_env_repeats(N, "walk", [0.005, 0.010, 0.006, 0.001], [5, 10, 6, 1])
    assert cts == (0.005, 0.010, 0.006, 0.001) and rep == (5, 10, 6, 1) and dt == 0.001
    assert r.dtype == it.dtype == np.int32 and r.flags["C_CONTIGUOUS"] and it.flags["C_CONTIGUOUS"]
    assert it.tolist() == [int(300 / x) for x in (5, 10, 6, 1)] == [60, 30, 50, 300]
    _, _, _, (r, it) = check_env_repeats(N, "walk", [0.005, 0.010, 0.006, 0.001], [5, 10, 6, 1], solver_iterations=40)
    assert it.tolist() == [40] * N and r.tolist() == [5, 10, 6, 1]
    # the task's defaults fill a scalar None, so a per-env action_repeat can pair with the default control step
    _, rep, dt, per_env = check_env_repeats(N, "gallop", [0.006, 0.012, 0.006, 0.012], [6, 12, 6, 12])
    assert dt == 0.001 and per_env[1].tolist() == [50, 25, 50, 25]


def test_all_equal_arrays_collapse_to_the_scalar():
    from rex_gym_b200.envs.batched_env import check_env_repeats
    assert check_env_repeats(N, "walk", None, None) == (0.005, 5, 0.001, None)
    assert check_env_repeats(N, "poses", None, None) == (0.006, 6, 0.006 / 6, None)
    for cts, rep in (([0.01] * N, [10] * N), (np.full(N, 0.01), np.full(N, 10)), ((0.01,) * N, 10), (0.01, (10,) * N)):
        c, r, dt, per_env = check_env_repeats(N, "walk", cts, rep)
        assert (c, r, dt, per_env) == (0.01, 10, 0.001, None) and type(c) is float and type(r) is int


def test_set_task_values_refuses_the_rate_keywords():
    from rex_gym_b200.envs.batched_env import BatchedRexEnv
    env = BatchedRexEnv.__new__(BatchedRexEnv)             # the keyword check comes before the batch is looked at
    for kw in (dict(control_time_step=0.01), dict(action_repeat=[10] * N)):
        with pytest.raises(ValueError, match="control rates and terrains are fixed at construction"):
            env.set_task_values(**kw)


def test_sharding_slices_global_rate_arrays(monkeypatch):
    from rex_gym_b200 import sharding
    import rex_gym_b200.envs.batched_env as B
    seen = []
    monkeypatch.setattr(B, "BatchedRexEnv", lambda **kw: seen.append(kw) or kw)
    g = 8
    cts, rep = [0.005, 0.01, 0.01, 0.005, 0.006, 0.006, 0.01, 0.005], [5, 10, 10, 5, 6, 6, 10, 5]
    for rank in range(2):
        sharding.make_sharded_env(g, rank, 2, task="walk", control_time_step=cts, action_repeat=np.array(rep))
    a, b = seen
    assert list(a["control_time_step"]) == cts[:4] and list(a["action_repeat"]) == rep[:4] and a["env_offset"] == 0
    assert list(b["control_time_step"]) == cts[4:] and list(b["action_repeat"]) == rep[4:] and b["env_offset"] == 4
    seen.clear()
    sharding.make_sharded_env(g, 1, 2, task="walk", control_time_step=0.01, action_repeat=10)
    assert seen[0]["control_time_step"] == 0.01 and seen[0]["action_repeat"] == 10          # scalars pass through


def test_the_library_exports_the_entry_points():
    from rex_gym_b200 import _capi
    L = _capi.load()
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rexsim.h")).read(), flags=re.S)
    for name in NEW:
        assert name in _capi.SIGNATURES and name in _capi.EXPORTS
        assert re.search(r"\b%s\s*\(" % name, header), name
        assert hasattr(L, name)
    assert L.rexsim_set_env_repeats(None, None, None) == -1                       # REXSIM_ERR_INVALID, no handle touched
    assert L.rexsim_env_repeat_buffers(None, None) == -1
    assert L.rexsim_launch_groups(None) == 0
    assert L.rexsim_launch_group(None, 0, None) == -1
    assert L.rexsim_slot_buffers(None, None, None) == -1

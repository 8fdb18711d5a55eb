"""Per-env terrains without a GPU: the keyword checks that come before any CUDA call, the collapse of all-equal arrays to the
scalar construction, set_task_values' refusal, the sharding slices and the ABI symbols."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
NEW = ("rexsim_set_env_terrains", "rexsim_env_terrain_buffers", "rexsim_last_terrain_build")
N = 4


def _no_cuda(monkeypatch):
    import torch
    from rex_gym_b200 import _capi

    def touched(*a, **k):
        raise AssertionError("CUDA touched before the keywords were checked")
    monkeypatch.setattr(torch.cuda, "is_available", touched)
    monkeypatch.setattr(_capi, "load", touched)


REFUSED = [
    ("unknown entry", ["plane", "hills", "random", "plane"], ValueError, "only 'plane' and 'random' are built"),
    ("csv entry", np.array(["plane", "csv", "plane", "plane"]), ValueError, "only 'plane' and 'random' are built"),
    ("non-string entry", ["plane", 1, "random", "plane"], ValueError, "only 'plane' and 'random' are built"),
    ("None entry", ["plane", None, "random", "plane"], ValueError, "only 'plane' and 'random' are built"),
    ("wrong length", ["plane", "random"], ValueError, "one entry per env"),
    ("too long", ("plane", "random") * 3, ValueError, "one entry per env"),
    ("two dimensions", np.array([["plane", "random"]] * N), ValueError, "one entry per env"),
    ("unknown scalar", "hills", ValueError, "only 'plane' and 'random' are built"),
]


@pytest.mark.parametrize("why,terrain,exc,msg", REFUSED, ids=[r[0] for r in REFUSED])
def test_refusals_come_before_any_cuda_call(why, terrain, exc, msg, monkeypatch):
    import rex_gym_b200 as R
    _no_cuda(monkeypatch)
    with pytest.raises(exc, match=msg):
        R.BatchedRexEnv(task="walk", num_envs=N, terrain_type=terrain)


@pytest.mark.parametrize("terrain", [["plane", "random"] * 2, ("random", "plane", "plane", "plane"),
                                     np.array(["random", "random", "plane", "random"])])
def test_accepted_arrays_reach_cuda(terrain, monkeypatch):
    import rex_gym_b200 as R
    _no_cuda(monkeypatch)
    with pytest.raises(AssertionError, match="CUDA touched"):
        R.BatchedRexEnv(task="walk", num_envs=N, terrain_type=terrain)
    with pytest.raises(AssertionError, match="CUDA touched"):
        R.make("RexTurn-v0", num_envs=N, terrain_type=terrain)


def test_all_equal_arrays_collapse_to_the_scalar():
    from rex_gym_b200.envs.batched_env import check_env_terrains
    assert check_env_terrains(N, "plane") == ("plane", None)
    assert check_env_terrains(N, "random") == ("random", None)
    for t in ("plane", "random"):
        assert check_env_terrains(N, [t] * N) == (t, None)
        assert check_env_terrains(N, np.array([t] * N)) == (t, None)
        assert check_env_terrains(N, tuple([t] * N)) == (t, None)
    scalar, ids = check_env_terrains(N, np.array(["random", "plane", "plane", "random"]))
    assert scalar is None and ids.dtype == np.int32 and ids.tolist() == [1, 0, 0, 1]
    assert ids.flags["C_CONTIGUOUS"]


def test_set_task_values_refuses_terrain_type():
    from rex_gym_b200.envs.batched_env import BatchedRexEnv
    env = BatchedRexEnv.__new__(BatchedRexEnv)             # the keyword check comes before the batch is looked at
    for kw in (dict(terrain_type="random"), dict(terrain_type=["plane"] * N)):
        with pytest.raises(ValueError, match="terrains are fixed at construction"):
            env.set_task_values(**kw)


def test_sharding_slices_global_terrain_arrays(monkeypatch):
    from rex_gym_b200 import sharding
    import rex_gym_b200.envs.batched_env as B
    seen = []
    monkeypatch.setattr(B, "BatchedRexEnv", lambda **kw: seen.append(kw) or kw)
    g = 8
    terrain = ["plane", "random", "random", "plane", "random", "random", "random", "plane"]
    for rank in range(2):
        sharding.make_sharded_env(g, rank, 2, task="walk", terrain_type=terrain)
    a, b = seen
    assert list(a["terrain_type"]) == terrain[:4] and a["env_offset"] == 0
    assert list(b["terrain_type"]) == terrain[4:] and b["env_offset"] == 4
    seen.clear()
    sharding.make_sharded_env(g, 1, 2, task="walk", terrain_type=np.array(terrain))
    assert list(seen[0]["terrain_type"]) == terrain[4:]
    seen.clear()
    sharding.make_sharded_env(g, 1, 2, task="walk", terrain_type="random")
    assert seen[0]["terrain_type"] == "random"                                   # scalars pass through


def test_the_library_exports_the_entry_points():
    from rex_gym_b200 import _capi
    L = _capi.load()
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rexsim.h")).read(), flags=re.S)
    for name in NEW:
        assert name in _capi.SIGNATURES and name in _capi.EXPORTS
        assert re.search(r"\b%s\s*\(" % name, header), name
        assert hasattr(L, name)
    assert L.rexsim_set_env_terrains(None, None, 0.5) == -1                       # REXSIM_ERR_INVALID, no handle touched
    assert L.rexsim_env_terrain_buffers(None, None, None) == -1
    assert L.rexsim_last_terrain_build(None, 0, None, None, None) == -1

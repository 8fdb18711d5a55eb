"""Per-env tasks and signals without a GPU: the space rule that comes before any CUDA call (the mixes whose spaces agree are
accepted, the others refused with the reference's BatchEnv message), the per-env default control rates, the collapse of
all-equal pairs to the scalar construction, the sharding slices, the ABI symbols and the ABI's refusals that need no device."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
NEW = ("rexsim_set_env_tasks", "rexsim_env_task_buffers", "rexsim_launch_group_task")
N = 4


def _no_cuda(monkeypatch):
    import torch
    from rex_gym_b200 import _capi

    def touched(*a, **k):
        raise AssertionError("CUDA touched before the keywords were checked")
    monkeypatch.setattr(torch.cuda, "is_available", touched)
    monkeypatch.setattr(_capi, "load", touched)


def alternate(a, b, n=N):
    return [(a, b)[i % 2] for i in range(n)]


ACCEPTED = [
    ("turn ik + turn ol, raw", dict(task="turn", signal_type=["ik", "ol", "ik", "ol"])),
    ("standup + poses, ol", dict(task=alternate("standup", "poses"), signal_type="ol")),
    ("standup + poses, either signal", dict(task=alternate("standup", "poses"), signal_type=["ik", "ik", "ol", "ol"])),
    ("walk ik + turn ik + turn ol, normalized", dict(task=["walk", "turn", "turn", "walk"], signal_type=["ik", "ik", "ol", "ik"],
                                                     normalize=True)),
    ("turn mix with frame wrappers", dict(task="turn", signal_type=alternate("ik", "ol"), frame_history=[0, 2], frame_delta=True)),
    ("turn mix with the arm", dict(task="turn", signal_type=alternate("ik", "ol"), mark="arm")),
    ("numpy entries", dict(task=np.array(["walk", "turn"] * 2), signal_type=np.array(["ik"] * N), normalize=True)),
]
REFUSED = [
    ("walk ik + turn ik, raw", dict(task=alternate("walk", "turn"), signal_type="ik"), "same observation space"),
    ("walk ik + walk ol", dict(task="walk", signal_type=alternate("ik", "ol"), normalize=True), "same observation space"),
    ("walk ol + turn ol", dict(task=alternate("walk", "turn"), signal_type="ol", normalize=True), "same observation space"),
    ("gallop + walk", dict(task=alternate("gallop", "walk"), signal_type="ik", normalize=True, control_time_step=0.005,
                           action_repeat=5), "same observation space"),
    ("gallop ik + gallop ol", dict(task="gallop", signal_type=alternate("ik", "ol"), normalize=True), "same observation space"),
    ("walk + standup", dict(task=alternate("walk", "standup"), signal_type="ik", normalize=True), "same observation space"),
    ("unknown task entry", dict(task=["walk", "run", "walk", "walk"]), "unknown task"),
    ("unknown signal entry", dict(task="turn", signal_type=["ik", "cpg", "ik", "ik"]), "unknown signal_type"),
    ("wrong length", dict(task=["turn", "turn"], signal_type="ik"), "one entry per env"),
    ("two dimensions", dict(task=np.array([["turn"]] * N), signal_type="ik"), "one entry per env"),
    ("standup + poses at one given rate pair", dict(task=alternate("standup", "poses"), control_time_step=[0.005, 0.006] * 2,
                                                    action_repeat=5), "simulation time steps differ"),
]


@pytest.mark.parametrize("why,kw", ACCEPTED, ids=[a[0] for a in ACCEPTED])
def test_accepted_mixes_reach_cuda(why, kw, monkeypatch):
    import rex_gym_b200 as R
    _no_cuda(monkeypatch)
    with pytest.raises(AssertionError, match="CUDA touched"):
        R.BatchedRexEnv(num_envs=N, **kw)


@pytest.mark.parametrize("why,kw,msg", REFUSED, ids=[r[0] for r in REFUSED])
def test_refusals_come_before_any_cuda_call(why, kw, msg, monkeypatch):
    import rex_gym_b200 as R
    _no_cuda(monkeypatch)
    with pytest.raises(ValueError, match=msg):
        R.BatchedRexEnv(num_envs=N, **kw)


def test_the_space_rule_is_the_task_spaces():
    """check_env_tasks refuses exactly the pairs whose task_spaces differ from env 0's, shapes before bounds."""
    from rex_gym_b200.envs.batched_env import SIGNALS, TASKS, check_env_tasks, task_spaces, _same_box
    pairs = [(t, s) for t in TASKS for s in SIGNALS]
    for normalize in (False, True):
        for p in pairs:
            for q in pairs:
                sp, sq = (task_spaces(*x, normalize, 0.001) for x in (p, q))
                same = _same_box(sp[0], sq[0]) and _same_box(sp[1], sq[1])
                args = (2, [p[0], q[0]], [p[1], q[1]], 0.001, normalize)
                if same:
                    check_env_tasks(*args)
                else:
                    with pytest.raises(ValueError, match="All environments must use the same observation space"):
                        check_env_tasks(*args)
    # the table of mixes that agree
    agree = lambda normalize: {frozenset((p, q)) for p in pairs for q in pairs if p < q and
                               all(_same_box(x, y) for x, y in zip(task_spaces(*p, normalize, 0.001), task_spaces(*q, normalize, 0.001)))}
    raw = {frozenset((("turn", "ik"), ("turn", "ol")))} | {frozenset((p, q)) for p in pairs for q in pairs
                                                          if p < q and p[0] in ("standup", "poses") and q[0] in ("standup", "poses")}
    assert agree(False) == raw
    walk_turn = [("walk", "ik"), ("turn", "ik"), ("turn", "ol")]
    assert agree(True) == raw | {frozenset((p, q)) for p in walk_turn for q in walk_turn if p < q}


def test_spaces_are_the_scalar_constructions():
    from rex_gym_b200.envs.batched_env import task_spaces
    a, o = task_spaces("gallop", "ol", False, 0.001)
    assert a.shape == (4,) and (a.low == np.float32(0.3)).all() and o.shape == (16,)
    a, o = task_spaces("turn", "ik", False, 0.001, frames=[0, 1, 3], frame_delta=True)
    assert o.shape == (12,) and (o.high[2:4] > 0).all()
    a, o = task_spaces("walk", "ol", True, 0.001)
    assert a.shape == (8,) and np.isinf(a.high).all() and (o.high == 1).all()


def test_all_equal_pairs_collapse_to_the_scalar():
    from rex_gym_b200.envs.batched_env import check_env_tasks
    assert check_env_tasks(N, "turn", "ol") == ("turn", "ol", None)
    assert check_env_tasks(N, ["turn"] * N, ("ol",) * N) == ("turn", "ol", None)
    assert check_env_tasks(N, np.array(["walk"] * N), "ik", normalize=True) == ("walk", "ik", None)
    t, s, (ti, si) = check_env_tasks(N, "standup", ["ik", "ol", "ol", "ik"])
    assert t == ("standup",) * N and s == ("ik", "ol", "ol", "ik")
    assert ti.dtype == si.dtype == np.int32 and ti.tolist() == [3] * N and si.tolist() == [0, 1, 1, 0]
    assert ti.flags["C_CONTIGUOUS"] and si.flags["C_CONTIGUOUS"]


def test_default_rates_follow_each_envs_task():
    from rex_gym_b200.envs.batched_env import check_env_repeats
    tasks = ["standup", "poses", "poses", "standup"]
    cts, rep, dt, (r, it) = check_env_repeats(N, tasks, None, None)
    assert cts == (0.005, 0.006, 0.006, 0.005) and rep == (5, 6, 6, 5) and dt == 0.001
    assert r.tolist() == [5, 6, 6, 5] and it.tolist() == [60, 50, 50, 60]
    assert check_env_repeats(N, ["poses"] * N, None, None) == (0.006, 6, 0.006 / 6, None)
    assert check_env_repeats(N, ["walk", "turn", "turn", "walk"], None, None) == (0.005, 5, 0.001, None)
    assert check_env_repeats(N, tasks, 0.01, 10) == (0.01, 10, 0.001, None)          # given scalars override every default


def test_default_rates_refuse_a_repeat_that_splits_the_time_step():
    from rex_gym_b200.envs.batched_env import check_env_repeats
    with pytest.raises(ValueError, match="simulation time steps differ"):
        check_env_repeats(N, ["standup", "poses", "poses", "standup"], None, 6)


def test_sharding_slices_global_task_arrays(monkeypatch):
    from rex_gym_b200 import sharding
    import rex_gym_b200.envs.batched_env as B
    seen = []
    monkeypatch.setattr(B, "BatchedRexEnv", lambda **kw: seen.append(kw) or kw)
    g = 8
    tasks, sigs = ["walk", "turn", "turn", "walk", "turn", "walk", "walk", "turn"], ["ik", "ik", "ol", "ik", "ol", "ik", "ik", "ik"]
    for rank in range(2):
        sharding.make_sharded_env(g, rank, 2, task=tasks, signal_type=np.array(sigs), normalize=True)
    a, b = seen
    assert list(a["task"]) == tasks[:4] and list(a["signal_type"]) == sigs[:4] and a["env_offset"] == 0
    assert list(b["task"]) == tasks[4:] and list(b["signal_type"]) == sigs[4:] and b["env_offset"] == 4
    seen.clear()
    sharding.make_sharded_env(g, 1, 2, task="turn", signal_type="ol")
    assert seen[0]["task"] == "turn" and seen[0]["signal_type"] == "ol"          # scalars pass through


def test_the_library_exports_the_entry_points():
    from rex_gym_b200 import _capi
    L = _capi.load()
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rexsim.h")).read(), flags=re.S)
    for name in NEW:
        assert name in _capi.SIGNATURES and name in _capi.EXPORTS
        assert re.search(r"\b%s\s*\(" % name, header), name
        assert hasattr(L, name)
    assert re.search(r"REXSIM_MAX_LAUNCH_GROUPS\s*=\s*16\b", header)
    assert re.search(r"REXSIM_GROUP_WORDS\s*=\s*8\b", header)                  # rexsim_launch_group's layout is unchanged
    t = np.zeros(N, np.int32)
    assert L.rexsim_set_env_tasks(None, t.ctypes.data, t.ctypes.data) == -1     # REXSIM_ERR_INVALID, no handle touched
    assert L.rexsim_env_task_buffers(None, None) == -1
    assert L.rexsim_launch_group_task(None, 0, None, None) == -1

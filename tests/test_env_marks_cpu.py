"""Per-env marks without a GPU: the table facts a batch of both marks rests on (the arm's model table starts with the base's,
its render table differs only in the arm's shapes), the space rule over every (task, signal) x mark mix before any CUDA call,
the collapse of all-equal arrays to the scalar construction, the sharding slices and the ABI symbols."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
NEW = ("rexsim_set_env_marks", "rexsim_env_mark_buffers", "rexsim_launch_group_mark")
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


def test_the_arm_tables_serve_the_base_envs():
    """The base step, settle and render read the first MT_FLOATS floats of the model table, the renderer draws 19 shapes for a
    base env: a handle built on the arm's tables runs its base envs as the base's tables would."""
    from rex_gym_b200 import model_tables as M
    base, npts_base = M.pack_model_tables("base")
    arm, npts_arm = M.pack_model_tables("arm")
    assert base.size == M.MT_FLOATS and arm.size == M.MT_FLOATS_ARM
    np.testing.assert_array_equal(arm[:M.MT_FLOATS].view(np.int32), base.view(np.int32))
    assert npts_arm == npts_base
    assert M.contact_breaking_distance("arm") == M.contact_breaking_distance("base")
    rb, ra = M.pack_render_tables("base"), M.pack_render_tables("arm")
    assert rb.size == ra.size == M.RT_FLOATS
    arm_only = np.zeros(M.RT_FLOATS, bool)
    arm_only[M.RT_COLOR + 3 * 19:M.RT_COLOR + 3 * M.RT_NSHAPES] = True        # the colours of shapes 19..25
    arm_only[M.RT_CYL:M.RT_FLOATS] = True                                     # the arm's cylinders and box
    np.testing.assert_array_equal(ra[~arm_only].view(np.int32), rb[~arm_only].view(np.int32))
    assert (ra[arm_only] != rb[arm_only]).any()


PAIRS = [(t, s) for t in ("walk", "gallop", "turn", "standup", "poses") for s in ("ik", "ol")]


@pytest.mark.parametrize("normalize", [False, True])
def test_the_space_rule_over_every_pair_and_mark(normalize):
    """Base and arm envs of one (task, signal) pair are one batch for every task but gallop; a gallop env with the arm is
    refused with the library's message, and a base gallop env differs from any arm env's spaces."""
    from rex_gym_b200.envs.batched_env import check_env_tasks
    for t, s in PAIRS:
        args = (2, t, s, 0.001, normalize)
        if t == "gallop":
            with pytest.raises(ValueError, match="mark='arm' is built for every task but gallop"):
                check_env_tasks(*args, mark=("base", "arm"))
        else:
            assert check_env_tasks(*args, mark=("base", "arm")) == (t, s, None)
            assert check_env_tasks(*args, mark=("arm", "base")) == (t, s, None)
    # a mix of pairs and marks: the same as the pairs alone once the gallop envs are out
    for p in PAIRS:
        for q in PAIRS:
            if "gallop" in (p[0], q[0]) or p == q:
                continue
            args = (2, [p[0], q[0]], [p[1], q[1]], 0.001, normalize)
            try:
                check_env_tasks(*args)
                agree = True
            except ValueError:
                agree = False
            if agree:
                check_env_tasks(*args, mark=("base", "arm"))
            else:
                with pytest.raises(ValueError, match="All environments must use the same observation space"):
                    check_env_tasks(*args, mark=("base", "arm"))
    # a base gallop env next to an arm env of another task: the spaces differ
    with pytest.raises(ValueError, match="same observation space|but gallop"):
        check_env_tasks(2, ["gallop", "walk"], "ik", 0.001, True, mark=("base", "arm"))


ACCEPTED = [
    ("walk ik", dict(task="walk", mark=alternate("base", "arm"))),
    ("walk ol", dict(task="walk", signal_type="ol", mark=alternate("arm", "base"))),
    ("turn", dict(task="turn", mark=np.array(["base", "arm", "arm", "base"]))),
    ("standup", dict(task="standup", signal_type="ol", mark=("arm", "base", "base", "base"))),
    ("poses", dict(task="poses", mark=alternate("base", "arm"))),
    ("turn ik + ol with both marks", dict(task="turn", signal_type=alternate("ik", "ol"), mark=["base", "base", "arm", "arm"])),
]
REFUSED = [
    ("gallop with both marks", dict(task="gallop", mark=alternate("base", "arm")), "but gallop"),
    ("gallop env beside arm walk", dict(task=alternate("gallop", "walk"), normalize=True, control_time_step=0.005, action_repeat=5,
                                        mark=alternate("base", "arm")), "same observation space"),
    ("unknown entry", dict(task="walk", mark=["base", "arms", "base", "base"]), "mark must be 'base' or 'arm'"),
    ("non-string entry", dict(task="walk", mark=["base", 1, "base", "base"]), "mark must be 'base' or 'arm'"),
    ("unknown scalar", dict(task="walk", mark="legs"), "mark must be 'base' or 'arm'"),
    ("wrong length", dict(task="walk", mark=["base", "arm"]), "one entry per env"),
    ("two dimensions", dict(task="walk", mark=np.array([["base"]] * N)), "one entry per env"),
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


def test_all_equal_arrays_collapse_to_the_scalar():
    from rex_gym_b200.envs.batched_env import check_env_marks
    assert check_env_marks(N, "base") == ("base", None)
    assert check_env_marks(N, "arm") == ("arm", None)
    assert check_env_marks(N, ["arm"] * N) == ("arm", None)
    assert check_env_marks(N, np.array(["base"] * N)) == ("base", None)
    s, nm = check_env_marks(N, ("base", "arm", "arm", "base"))
    assert s is None and nm.dtype == np.int32 and nm.flags["C_CONTIGUOUS"] and nm.tolist() == [12, 18, 18, 12]


def test_sharding_slices_global_mark_arrays(monkeypatch):
    from rex_gym_b200 import sharding
    import rex_gym_b200.envs.batched_env as B
    seen = []
    monkeypatch.setattr(B, "BatchedRexEnv", lambda **kw: seen.append(kw) or kw)
    g = 8
    marks = ["base", "arm", "arm", "base", "arm", "base", "base", "base"]
    for rank in range(2):
        sharding.make_sharded_env(g, rank, 2, task="walk", mark=marks)
    a, b = seen
    assert list(a["mark"]) == marks[:4] and a["env_offset"] == 0
    assert list(b["mark"]) == marks[4:] and b["env_offset"] == 4
    seen.clear()
    sharding.make_sharded_env(g, 1, 2, task="walk", mark="arm")
    assert seen[0]["mark"] == "arm"                                              # a scalar passes through


def test_the_library_exports_the_entry_points():
    from rex_gym_b200 import _capi
    L = _capi.load()
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rexsim.h")).read(), flags=re.S)
    for name in NEW:
        assert name in _capi.SIGNATURES and name in _capi.EXPORTS
        assert re.search(r"\b%s\s*\(" % name, header), name
        assert hasattr(L, name)
    assert re.search(r"REXSIM_GROUP_WORDS\s*=\s*8\b", header)                  # rexsim_launch_group's layout is unchanged
    nm = np.full(N, 12, np.int32)
    assert L.rexsim_set_env_marks(None, nm.ctypes.data) == -1                  # REXSIM_ERR_INVALID, no handle touched
    assert L.rexsim_env_mark_buffers(None, None) == -1
    assert L.rexsim_launch_group_mark(None, 0, None) == -1

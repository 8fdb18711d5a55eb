"""The frame wrappers (BatchedRexEnv(frame_history=..., frame_delta=...)): the reference's FrameHistory and FrameDelta
(rex_gym/agents/tools/wrappers.py:93-181) fused into the step and reset kernels.

CPU: oracle/frame_oracle.py, the fp64 restatement, reproduces every output and space of tests/golden/frame_wrapper_golden.json.gz
(tools/gen_frame_wrapper_golden.py ran the reference's own classes); every refusal happens before any CUDA call; the entry points
are declared and exported.

GPU: twin batches with the same seed and actions, wrappers off and on.  The "on" twin's rewards, dones, state, sensor ring and
episode books equal the "off" twin's bit for bit, and its observations equal the fp32 restatement applied to the "off" twin's
observation stream bit for bit, in every step-kernel instance, through auto-resets, explicit resets, a checkpoint, the host-buffer
step and a graph-captured Rollout."""
import ctypes as C
import gzip
import json
import os
import re

import numpy as np
import pytest

from oracle.frame_oracle import FrameWrappers, frame_spaces

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
G = json.load(gzip.open(os.path.join(HERE, "golden", "frame_wrapper_golden.json.gz"), "rt"))
NEW = ("rexsim_set_frames", "rexsim_out_dim", "rexsim_frame_buffers")
MISSING_ZERO = "Past indices should include 0 for the current frame."


# ---- CPU -----------------------------------------------------------------------------------------------------------------
def _case_id(c):
    return "%s-%s-%s%s" % (c["task"], "norm" if c["normalize"] else "raw", "-".join(map(str, c["past_indices"] or ["none"])),
                           "-delta" if c["delta"] else "")


def _inner(c, row):
    """The observation FrameDelta / FrameHistory are handed: the raw row, through RangeNormalize in fp64 when it is on
    (wrappers.py:238-242)."""
    x = np.array(c["raw_observs"][row], np.float64)
    if c["normalize"]:
        lo, hi = (np.array(b, np.float64) for b in c["observ_box"])
        x = 2 * (x - lo) / (hi - lo) - 1
    return x


def test_fixture_covers_what_the_fused_stack_must_reproduce():
    assert G["wrapper_order"] == ["LimitDuration", "RangeNormalize", "ClipAction", "FrameDelta", "FrameHistory", "ConvertTo32Bit"]
    assert G["missing_zero_error"] == MISSING_ZERO
    cases = G["cases"]
    assert {c["task"] for c in cases} == {"walk", "gallop"} and {c["normalize"] for c in cases} == {False, True}
    lists = [c["past_indices"] for c in cases]
    assert [0, 1, 2] in lists                                   # an index equal to the capacity
    assert any(p and len(set(p)) < len(p) for p in lists)       # duplicates
    assert any(p and p != sorted(p) for p in lists)             # an unordered list
    assert any(p is None and c["delta"] for p, c in zip(lists, cases))           # delta alone
    assert any(p and c["delta"] for p, c in zip(lists, cases))                   # delta under history
    assert all(sum(k == "reset" for k, _ in c["events"]) >= 3 for c in cases)    # resets mid-stream


@pytest.mark.parametrize("c", G["cases"], ids=[_case_id(c) for c in G["cases"]])
def test_fp64_restatement_reproduces_the_reference(c):
    fw = FrameWrappers(1, c["O"], c["past_indices"], c["delta"], np.float64)
    assert fw.out_dim == len(c["observs"][0])
    for (kind, row), want in zip(c["events"], c["observs"]):
        x = _inner(c, row)[None]
        got = fw.reset(x) if kind == "reset" else fw.step(x)
        np.testing.assert_array_equal(got[0], np.array(want, np.float32), err_msg="%s row %d" % (kind, row))
    if c["past_indices"] == [0, 1, 2]:
        # the aliasing pinned: index 2 = capacity reads the current slot, so the third frame repeats the first
        out = np.array(c["observs"][-1], np.float32).reshape(3, -1)
        np.testing.assert_array_equal(out[2], out[0])
    lo, hi = frame_spaces(*c["inner_space"], past_indices=c["past_indices"], delta=c["delta"])
    np.testing.assert_array_equal(lo, c["space"][0])
    np.testing.assert_array_equal(hi, c["space"][1])


@pytest.mark.parametrize("c", G["cases"], ids=[_case_id(c) for c in G["cases"]])
def test_batch_spaces_follow_the_reference(c):
    """BatchedRexEnv's float32 Box: exact where the bounds are (normalize: [-1, 1] gives [-2, 2]), to float32 rounding on the
    raw task bounds."""
    from rex_gym_b200.envs.batched_env import frame_space
    lo, hi = frame_space(*(np.array(b, np.float32) for b in c["inner_space"]), c["past_indices"] or [], c["delta"])
    assert lo.dtype == np.float32 and lo.shape == (len(c["observs"][0]),)
    rtol = 0 if c["normalize"] else 1e-6
    np.testing.assert_allclose(lo, c["space"][0], rtol=rtol)
    np.testing.assert_allclose(hi, c["space"][1], rtol=rtol)


@pytest.mark.parametrize("past,error", [([1, 2], KeyError), ([], KeyError), ([0, -1, 2], ValueError), ([0], ValueError),
                                        ([0, 0], ValueError), (list(range(17)), ValueError), ([0, 65], ValueError),
                                        ([0, 1.5], ValueError)])
def test_refusals_come_before_any_cuda_call(past, error, monkeypatch):
    import torch
    import rex_gym_b200 as R
    from rex_gym_b200 import _capi

    def touched(*a, **k):
        raise AssertionError("CUDA touched before the keywords were checked")
    monkeypatch.setattr(torch.cuda, "is_available", touched)
    monkeypatch.setattr(_capi, "load", touched)
    with pytest.raises(error) as e:
        R.BatchedRexEnv(task="walk", num_envs=4, frame_history=past)
    if error is KeyError:
        assert e.value.args[0] == MISSING_ZERO


def test_entry_points_are_declared_and_exported():
    from rex_gym_b200 import _capi
    L = _capi.load()
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rexsim.h")).read(), flags=re.S)
    for name in NEW:
        assert name in _capi.SIGNATURES and name in _capi.EXPORTS
        assert re.search(r"\b%s\s*\(" % name, header), name
        assert hasattr(L, name)
    # a null handle is refused, and has no width
    assert L.rexsim_set_frames(None, None, 0, 1) == -1
    assert L.rexsim_out_dim(None) == 0
    p, q, a, b = C.c_void_p(), C.c_void_p(), C.c_int64(), C.c_int64()
    assert L.rexsim_frame_buffers(None, C.byref(p), C.byref(a), C.byref(q), C.byref(b)) == -1


# ---- GPU: helpers ----------------------------------------------------------------------------------------------------------
def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _words(env):
    out = dict(state_f=_np(env._state_f), state_i=_np(env._state_i), cmd=_np(env.last_command()))
    if env._ring is not None:
        out["sensor_history"] = _np(env._ring)
    if env._episode is not None:
        out["episode_statistics"] = _np(env._episode["block"])
    return out


def _twins(task, n, past, delta, **kw):
    from twin import make_env
    off = make_env(task, n, **kw)
    on = make_env(task, n, frame_history=past, frame_delta=delta, **kw)
    fw = FrameWrappers(n, off.obs_dim, past, delta, np.float32)
    assert on.obs_dim == fw.out_dim and on.observation_space.shape == (fw.out_dim,)
    return off, on, fw


# ---- GPU: every step-kernel instance ----------------------------------------------------------------------------------------
from twin import BUILDS, INSTANCES, bound, force_build, instance_config, launched, row_id  # noqa: E402


@pytest.mark.gpu
@pytest.mark.parametrize("row", INSTANCES, ids=[row_id(r) for r in INSTANCES])
def test_every_instance_matches_the_restatement_of_its_twin(row, monkeypatch):
    """48 auto-resetting steps of 15-step episodes (three in-kernel resets per env) with frame_history=[0, 1, 2, 3] (index 3 =
    capacity) and delta: rewards, dones, state words, sensor ring and episode books bit-identical to the wrappers-off twin, every
    observation word the fp32 restatement of the twin's observation stream bit for bit."""
    task, sig, arm, terrain, build = row
    force_build(monkeypatch, build)
    n = 19
    kw = dict(instance_config(row), auto_reset=True, episode_statistics=True, normalize=INSTANCES.index(row) % 2 == 0)
    off, on, fw = _twins(task, n, [0, 1, 2, 3], True, **kw)
    np.testing.assert_array_equal(on.reset(), fw.reset(off.reset()))
    rng = np.random.default_rng(11)
    b = bound(task, sig) * (1.0 if not kw["normalize"] else 1.5)
    for k in range(48):
        a = rng.uniform(-b, b, size=(n, off.action_dim)).astype(np.float32)
        o0, r0, d0, _ = off.step(a)
        o1, r1, d1, _ = on.step(a)
        assert launched(off) == launched(on) == BUILDS[build]
        np.testing.assert_array_equal(r0, r1, err_msg=f"reward, step {k}")
        np.testing.assert_array_equal(d0, d1, err_msg=f"done, step {k}")
        np.testing.assert_array_equal(o1, fw.step(o0, first=d0), err_msg=f"obs, step {k}")
    w0, w1 = _words(off), _words(on)
    for key in w0:
        np.testing.assert_array_equal(w0[key], w1[key], err_msg=key)
    assert set(on.state_dict()) - set(off.state_dict()) == {"frame_history", "frame_delta"}
    assert (fw.t < 15).all()
    off.close(); on.close()


# ---- GPU: explicit resets, checkpoint, host path ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("task,past,delta", [("walk", [0, 2, 1], True), ("gallop", [3, 0, 3, 1], False), ("gallop", None, True)])
def test_explicit_reset_restarts_only_the_listed_envs(task, past, delta):
    """auto_reset=False: host and device reset(indices) restart the listed envs' frames; out-of-range device indices leave every
    buffer untouched (IndexError from check_errors, as for the state)."""
    import torch
    n = 24
    off, on, fw = _twins(task, n, past, delta, seed=5, normalize=True)
    np.testing.assert_array_equal(on.reset(), fw.reset(off.reset()))
    rng = np.random.default_rng(3)
    for k in range(30):
        if k in (4, 11):
            idx = rng.choice(n, size=5, replace=False)
            got, want = on.reset(idx), off.reset(idx)
            np.testing.assert_array_equal(got, fw.reset(want, idx))
        if k == 17:
            dev = torch.tensor([2, -1, n + 3, 9], dtype=torch.int32, device="cuda")
            before = {key: v.clone() for key, v in on._frames.items()}
            got, want = _np(on.reset(dev)), _np(off.reset(dev))
            np.testing.assert_array_equal(got[[0, 3]], fw.reset(want[[0, 3]], [2, 9]))
            for key, v in on._frames.items():
                w = v.view(-1, n).cpu().numpy()
                w0 = before[key].view(-1, n).cpu().numpy()
                keep = np.setdiff1d(np.arange(n), [2, 9])
                np.testing.assert_array_equal(w[:, keep], w0[:, keep])
            for e in (off, on):
                with pytest.raises(IndexError):
                    e.check_errors()
        a = rng.uniform(-1.5, 1.5, size=(n, off.action_dim)).astype(np.float32)
        o0, r0, d0, _ = off.step(a)
        o1, r1, d1, _ = on.step(a)
        np.testing.assert_array_equal(r0, r1); np.testing.assert_array_equal(d0, d1)
        np.testing.assert_array_equal(o1, fw.step(o0), err_msg=f"step {k}")
    off.close(); on.close()


@pytest.mark.gpu
def test_state_dict_resumes_mid_episode_exactly():
    from twin import make_env
    kw = dict(seed=9, normalize=True, auto_reset=True, max_episode_steps=40, frame_history=[0, 1, 5], frame_delta=True)
    n = 32
    a = make_env("gallop", n, **kw)
    a.reset()
    rng = np.random.default_rng(8)
    acts = rng.uniform(-1, 1, size=(40, n, a.action_dim)).astype(np.float32)
    for k in range(13):
        a.step(acts[k])
    sd = {k: v.clone() for k, v in a.state_dict().items()}
    assert {"frame_history", "frame_delta"} <= set(sd)
    ref = [a.step(acts[k])[:3] for k in range(13, 40)]
    b = make_env("gallop", n, **kw)
    b.reset()
    b.load_state_dict(sd)
    for k, want in zip(range(13, 40), ref):
        got = b.step(acts[k])[:3]
        for x, y in zip(got, want):
            np.testing.assert_array_equal(x, y, err_msg=f"step {k}")
    a.close(); b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [64, 16500], ids=["zero-copy", "staged"])
def test_host_step_returns_the_device_bytes(n):
    import torch
    from twin import make_env
    kw = dict(seed=4, normalize=True, auto_reset=True, max_episode_steps=7, frame_history=[0, 2, 1, 2], frame_delta=True)
    h, d = make_env("walk", n, **kw), make_env("walk", n, **kw)
    assert int(h._L.rexsim_host_out_bytes(h._h)) == h._h_out.numel()
    np.testing.assert_array_equal(h.reset(), d.reset())
    rng = np.random.default_rng(1)
    for k in range(12):
        a = rng.uniform(-1, 1, size=(n, 2)).astype(np.float32)
        oh, rh, dh, _ = h.step(a)
        od, rd, dd, _ = d.step(torch.from_numpy(a).cuda())
        np.testing.assert_array_equal(oh, _np(od), err_msg=f"obs {k}")
        np.testing.assert_array_equal(rh, _np(rd)); np.testing.assert_array_equal(dh, _np(dd))
    h.close(); d.close()


# ---- GPU: Rollout ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tensor_cores", [False, True], ids=["fp32", "tensor-cores"])
def test_rollout_records_the_restated_stream(tensor_cores):
    """A T = 32 graph-captured Rollout of walk-ik with frame_history=[0, 1, 2, 3] (16 observation words): the observations it
    recorded, its rewards and dones equal the restatement of a wrappers-off twin replaying the recorded actions."""
    import torch
    from rex_gym_b200.agents import ForwardGaussianPolicy, Rollout
    from twin import make_env
    n, T = 512, 32
    kw = dict(signal_type="ik", normalize=True, auto_reset=True, max_episode_steps=25, target_position=2.0, backwards=False)
    env = make_env("walk", n, frame_history=[0, 1, 2, 3], **kw)
    assert env.obs_dim == 16
    net = ForwardGaussianPolicy(env.obs_dim, env.action_dim, seed=3, tensor_cores=tensor_cores)
    ro = Rollout(env, net, T, seed=17, training=True, use_graph=True)
    out = {k: _np(v).copy() for k, v in ro.collect().items()}
    twin = make_env("walk", n, **kw)
    fw = FrameWrappers(n, twin.obs_dim, [0, 1, 2, 3], False, np.float32)
    cur = fw.reset(_np(twin.reset(torch.arange(n, dtype=torch.int32, device="cuda"))))
    for t in range(T):
        np.testing.assert_array_equal(out["observ"][t], cur, err_msg=f"observ {t}")
        o, r, d, _ = twin.step(torch.from_numpy(out["action"][t]).cuda())
        np.testing.assert_array_equal(out["reward"][t], _np(r), err_msg=f"reward {t}")
        np.testing.assert_array_equal(out["done"][t], _np(d), err_msg=f"done {t}")
        cur = fw.step(_np(o), first=_np(d))
    assert out["done"].any()
    env.close(); twin.close(); net.close()


# ---- GPU: the entry point's refusals -----------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_set_frames_refuses_malformed_indices_and_a_started_handle():
    from twin import make_env
    env = make_env("walk", 8, seed=1)
    L = env._L

    def call(idx, delta=0, count=None):
        a = np.ascontiguousarray(idx, np.int32)
        return L.rexsim_set_frames(env._h, a.ctypes.data if a.size else None, len(a) if count is None else count, delta)
    for idx, delta in (([1, 2], 0), ([0, -1], 0), ([0], 0), ([0, 65], 0), (list(range(17)), 0), ([0, 1], 2)):
        assert call(idx, delta) == -1, (idx, delta)
    assert call([0, 1], 0, count=-1) == -1
    call([1, 2])
    assert MISSING_ZERO.encode() in L.rexsim_last_error()
    assert L.rexsim_out_dim(env._h) == 4                               # nothing was switched on
    env.reset()
    assert call([0, 1], 1) == -1
    assert b"before the first reset or step" in L.rexsim_last_error()
    assert L.rexsim_out_dim(env._h) == 4
    env.close()

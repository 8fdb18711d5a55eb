"""GPU: the replicated PGS loop of the 255-register build against the shuffle loop of the 128-register build, bit for bit.

With REXSIM_PGS_REPLICATED (rex_gym_b200/csrc/rexsim_kernel.cu) the small build on flat ground solves the 12 foot-contact rows of
an env on each of its 4 lanes, while the big build hands every impulse change from lane to lane.  Both perform the same fmaf
sequence per row, and
walk-ik and turn-ik already agreed bit for bit between the two builds before the replicated loop existed
(test_gpu_builds.py::test_the_dispatcher_switches_builds_at_its_thresholds).  So the forced small and big builds must keep agreeing
on everything a step writes: obs, reward, done, the whole SoA state and the per-env solver cost (PGS iterations), which also pins
that both loops leave at the same iteration.
"""
import pytest
import torch
from twin import BUILDS, force_build, launched, make_env, solver_cost

CASES = [  # (envs, solver_iterations): None = the task's default, int(300 / action_repeat)
    (8449, None),      # 265 CTAs of the small build: more than one wave, one env in the last CTA
    (1003, None),      # the last warp holds 3 of its 8 envs
    (1003, 1),         # one iteration: the loop body runs once, every env leaves at the cap
    (1003, 60),        # the default cap of walk-ik / turn-ik written out
]


@pytest.mark.gpu
@pytest.mark.parametrize("n,iters", CASES, ids=["n8449", "n1003", "n1003-iters1", "n1003-iters60"])
@pytest.mark.parametrize("task", ["walk", "turn"])
def test_replicated_and_shuffle_solvers_agree_bit_for_bit(monkeypatch, task, n, iters):
    """60 auto-resetting control steps with episode phases staggered by partial resets; the two builds alternate step by step."""
    kw = dict(signal_type="ik", normalize=True, auto_reset=True, max_episode_steps=25, seed=17, solver_iterations=iters)
    envs = {b: make_env(task, n, **kw) for b in ("small", "big")}
    for e in envs.values():
        e.reset()
    gen = torch.Generator(device="cuda").manual_seed(5)
    iterations = set()
    for k in range(60):
        act = torch.rand((n, envs["small"].action_dim), device="cuda", generator=gen) * 2 - 1
        if k % 9 == 4:
            idx = torch.randperm(n, device="cuda", generator=gen)[:n // 4].to(torch.int32)
            for e in envs.values():
                e.reset(idx)
        out = {}
        for b, e in envs.items():
            force_build(monkeypatch, b)
            out[b] = [t.clone() for t in e.step(act)[:3]] + [torch.from_numpy(solver_cost(e)), e._state_f.clone(), e._state_i.clone()]
        assert launched(envs["small"]) == BUILDS["small"] and launched(envs["big"]) == BUILDS["big"]
        for name, x, y in zip(("obs", "reward", "done", "cost", "state_f", "state_i"), out["small"], out["big"]):
            assert torch.equal(x, y), f"{name} differs at step {k}"
        iterations.update(out["small"][3].unique().tolist())
    assert max(iterations) > 0                   # the solver ran
    for e in envs.values():
        assert (e.check_errors() & 1) == 0
        e.close()

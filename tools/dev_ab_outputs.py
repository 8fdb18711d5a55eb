#!/usr/bin/env python3
"""A/B bit identity of library builds (the outputs half of dev_ab.py's timing A/B).

    python tools/dev_ab_outputs.py rex_gym_b200/librexsim_parent.so rex_gym_b200/librexsim.so [more.so ...]

Runs all 72 step-kernel instances of tests/twin.INSTANCES (forced build, 37 envs, 40 steps of seeded random actions,
auto-reset after 15 steps), walk-ik on flat ground at 8449 and 65 536 envs and turn-ik on heightfields at 16 897 envs (the
big build, warp re-grouping on) once per library, each library in its own process (REXSIM_LIB).  After every step it hashes
obs, reward, done, last_command, the error words, the whole SoA state and the sensor ring; then bench.py --dump-outputs.
Random actions from reset rarely reach the generic solver path, so every configuration of tests/test_gpu_generic_path.CONFIGS
also runs from that test's start states (body, arm and multi-limit contacts): 4 single sub-steps, then 4 control steps of the
task configuration, hashing the solver cost as well.  Last, render_batch frames of a few envs of walk-ik on flat ground,
turn-ik on the random heightfields and standup with the arm, with the default camera and at 97 x 61.  Then the agent kernels:
every network of tests/test_gpu_agent_shapes.ROWS in its precision at that test's batch sizes (perform's four outputs, noise-free
and sampled), the filter update (whole batch and partial + finalize: filter state and counters) and the reward transform, and
the three scans on seeded inputs.
Every later library is compared with the first: each array that is not bit-identical is reported, and for a frame the number
of pixels that differ."""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]


def cases():
    from twin import INSTANCES, instance_config, row_id
    out = [(row_id(r), r[0], None if r[4] == "sensor" else r[4], 37, instance_config(r)) for r in INSTANCES]
    for n in (8449, 65536):
        out.append((f"walk-ik-plane-n{n}", "walk", None, n, dict(signal_type="ik", seed=13, max_episode_steps=15)))
    out.append(("turn-ik-random-n16897", "turn", None, 16897,
                dict(signal_type="ik", seed=13, max_episode_steps=15, terrain_type="random", num_fields=64)))
    return out


def digest(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(str((a.dtype.str, a.shape)).encode() + a.tobytes()).hexdigest()


def _force_build(build):
    import pytest
    import twin
    twin.force_build(pytest.MonkeyPatch(), build)


def _record(env, rec, k, ret, cost=False):
    """Hash what step `k` returned (`ret`) and left in the library's buffers into `rec`."""
    o, r, d = ret[:3]
    arrs = dict(obs=o, reward=r, done=d, cmd=env.last_command(), err=env._err, sf=env._state_f, si=env._state_i)
    if env._ring is not None:
        arrs["ring"] = env._ring
    for name, v in arrs.items():
        rec[f"{k:02d}_{name}"] = digest(v if isinstance(v, np.ndarray) else v.cpu().numpy())
    if cost:
        import twin
        rec[f"{k:02d}_cost"] = digest(twin.solver_cost(env))


def generic_cases(res):
    """tests/test_gpu_generic_path start states, every CONFIGS entry: single sub-steps, then control steps."""
    import test_gpu_generic_path as G
    import twin
    for mark, terrain, build in G.CONFIGS:
        ids, st = G._batch(mark, terrain)
        for sub, steps in ((True, 4), (False, 4)):
            _force_build(build)
            env = twin.make_env("walk", G.N, **G._kw(mark, terrain, sub, build))
            env.reset()
            env.set_state(*(st[k] for k in twin.STATE_KEYS))
            rng = np.random.default_rng(7)
            rec = res[f"generic-{mark}-{terrain}-{build}-{'substep' if sub else 'control'}"] = {}
            for k in range(steps):
                ret = env.step(rng.uniform(-0.4, 0.4, size=(G.N, env.action_dim)).astype(np.float32))
                _record(env, rec, k, ret, cost=True)
            env.close()


def render_cases(R, res, frames):
    """render_batch of a few stepped envs: default camera and an odd size."""
    import torch
    _force_build(None)
    for cid, task, kw in (("render-walk-ik-plane", "walk", dict(signal_type="ik")),
                          ("render-turn-ik-random", "turn", dict(signal_type="ik", terrain_type="random", num_fields=4)),
                          ("render-standup-ol-arm", "standup", dict(signal_type="ol", mark="arm"))):
        env = R.BatchedRexEnv(task=task, num_envs=8, seed=5, **kw)
        env.reset()
        rng = np.random.default_rng(2)
        for _ in range(30):
            env.step(rng.uniform(-0.1, 0.1, size=(8, env.action_dim)).astype(np.float32))
        for size, (w, h) in (("480x360", (480, 360)), ("97x61", (97, 61))):
            img = env.render_batch(torch.arange(4, device="cuda"), width=w, height=h).cpu().numpy()
            res[f"{cid}-{size}"] = {"frames": digest(img)}
            frames[f"{cid}-{size}"] = img
        env.close()


def agent_cases(res):
    """perform, experience, transform_reward of every tests/test_gpu_agent_shapes row; the three scans."""
    import torch
    import test_gpu_agent_shapes as S
    from rex_gym_b200.agents import utility
    sizes = S.batch_sizes(S._half())
    for row in S.ROWS:
        _, _, obs, nets = S._setup(row, max(sizes))
        net = nets[-1]
        x_all = torch.from_numpy(obs).cuda()
        rew_all = torch.from_numpy(np.random.default_rng(3).normal(0.1, 0.5, max(sizes)).astype(np.float32)).cuda()
        rec = res["agent-" + S.row_id(row)] = {}
        for n in sizes:
            for training in (False, True):
                out = net.perform(x_all[:n], training=training, seed=S.SEED, step=S.STEP, env_offset=S.OFFSET)
                for k, t in out.items():
                    rec[f"n{n}_{'sampled' if training else 'mean'}_{k}"] = digest(t.cpu().numpy())
        for n in sizes:
            net.experience(x_all[:n], rew_all[:n])
            rec[f"n{n}_experience"] = digest(np.r_[net._filt.cpu().numpy().view(np.int32), net._cnt.cpu().numpy().view(np.int32)])
            S._experience_split(net, x_all[:n], rew_all[:n])
            rec[f"n{n}_partial_finalize"] = digest(np.r_[net._filt.cpu().numpy().view(np.int32), net._cnt.cpu().numpy().view(np.int32)])
            rec[f"n{n}_transform_reward"] = digest(net.transform_reward(rew_all[:n]).cpu().numpy())
        for nt in nets:
            nt.close()
    rng = np.random.default_rng(17)
    rec = res["agent-scans"] = {}
    for L in S.SCAN_LENGTHS:
        r, v = (torch.from_numpy(rng.normal(size=(300, L)).astype(np.float32)).cuda() for _ in range(2))
        length = torch.from_numpy(rng.integers(0, L + 1, 300).astype(np.int32)).cuda()
        rec[f"L{L}_return"] = digest(utility.discounted_return(r, length, 0.985).cpu().numpy())
        rec[f"L{L}_advantage"] = digest(utility.lambda_advantage(r, v, length, 0.985).cpu().numpy())
        v1 = torch.from_numpy(rng.normal(size=(L + 1, 300)).astype(np.float32)).cuda()
        done = torch.from_numpy(rng.random((L, 300)) < 0.05).cuda()
        ret, adv = utility.gae_segments(r.t().contiguous(), v1, done, 0.985, 0.95)
        rec[f"L{L}_gae"] = digest(np.r_[ret.cpu().numpy(), adv.cpu().numpy()])


def run(out):
    """Child process: every case with the library REXSIM_LIB names; {case: {step_array: sha256}} to `out`, the render frames
    beside it (frames.npz)."""
    import torch
    import rex_gym_b200 as R
    from rex_gym_b200.envs.batched_env import ACTION_BOUND
    res = {}
    for cid, task, build, n, kw in cases():
        _force_build(build)
        env = R.BatchedRexEnv(task=task, num_envs=n, auto_reset=True, **kw)
        env.reset()
        rng = np.random.default_rng(11)
        b = ACTION_BOUND[(task, kw["signal_type"])]
        rec = res[cid] = {}
        for k in range(40):
            ret = env.step(torch.as_tensor(rng.uniform(-b, b, size=(n, env.action_dim)).astype(np.float32), device="cuda"))
            _record(env, rec, k, ret)
        env.close()
    generic_cases(res)
    frames = {}
    render_cases(R, res, frames)
    agent_cases(res)
    with open(out, "w") as f:
        json.dump(res, f)
    np.savez(os.path.join(os.path.dirname(out), "frames.npz"), **frames)


def outputs(lib):
    """{case: {step_array: sha256}} of every case and of bench.py --dump-outputs with library `lib`, and the render frames."""
    env = dict(os.environ, REXSIM_LIB=os.path.abspath(lib))
    with tempfile.TemporaryDirectory(prefix="ab_outputs_") as d:
        subprocess.run([sys.executable, os.path.abspath(__file__), "--child", os.path.join(d, "steps.json")], env=env,
                       check=True, cwd=ROOT)
        subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--steps", "20", "--warmup", "5", "--no-extras",
                        "--dump-outputs", os.path.join(d, "bench")], env=env, check=True, cwd=ROOT, stdout=subprocess.DEVNULL)
        with open(os.path.join(d, "steps.json")) as f:
            steps = json.load(f)
        for f in sorted(os.listdir(os.path.join(d, "bench"))):
            steps["bench " + f] = {"array": digest(np.load(os.path.join(d, "bench", f)))}
        with np.load(os.path.join(d, "frames.npz")) as z:
            frames = {k: z[k] for k in z.files}
    return steps, frames


def main(libs):
    runs = [outputs(lib) for lib in libs]
    (ref_steps, ref_frames), status = runs[0], 0
    for lib, (other, frames) in zip(libs[1:], runs[1:]):
        print(f"== {libs[0]} vs {lib}")
        nbad = 0
        for cid, ref in ref_steps.items():
            bad = [k for k in ref if other.get(cid, {}).get(k) != ref[k]]
            nbad += bool(bad)
            what = "identical" if not bad else "DIFFERS in %d arrays, first %s" % (len(bad), bad[0])
            if bad and cid in ref_frames:
                px = (ref_frames[cid] != frames[cid]).any(-1).reshape(len(ref_frames[cid]), -1).sum(1)
                what += f", differing pixels per image {px.tolist()} of {ref_frames[cid][0, ..., 0].size}"
            print(f"{cid:40s} {what}")
        print(f"{len(ref_steps) - nbad} of {len(ref_steps)} runs bit-identical\n")
        status |= nbad > 0
    return status


if __name__ == "__main__":
    if sys.argv[1] == "--child":
        sys.path.insert(0, ROOT)
        run(sys.argv[2])
    else:
        sys.exit(main(sys.argv[1:]))

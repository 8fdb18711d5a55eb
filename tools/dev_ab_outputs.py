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
every network of tests/agent_twin.FF_ROWS in its precision at the feed-forward batch sizes, on agent_twin.ff_setup's inputs
(perform's four outputs, noise-free and sampled), the filter update (whole batch and partial + finalize: filter state and
counters) and the reward transform, and the three scans on seeded inputs.
Then the mixed batches of the per-env keywords (mixed_cases, as tests/test_gpu_env_*.py build them, up to the 16-group and
64-setting caps): the launch groups' words, the slot buffers, the hold table, the latency buffer and the launch count after
construction, then every output of 30 steps after a full reset and the state and ring words after them.
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


def mixed_cases():
    """(case id, task, n, action bound, keywords) of mixed batches: each per-env keyword alone, then together, at the caps."""
    gains = [(1.0, 0.02), (1.3, 0.03), (0.8, 0.015)]
    cyc = lambda vals, n, k=1: [vals[(e // k) % len(vals)] for e in range(n)]
    cfg = dict(seed=13, max_episode_steps=15, num_fields=4)
    out = [("mixed-values", "walk", 24, 0.4, dict(cfg, target_position=cyc([None, 1.5, 3.0], 24), backwards=cyc([None, 0, 1], 24, 2),
                                                   motor_kp=[g[0] for g in cyc(gains, 24, 3)], motor_kd=[g[1] for g in cyc(gains, 24, 3)])),
           ("mixed-latencies", "walk", 27, 0.4, dict(cfg, control_latency=cyc([0.0, 0.0105, 0.02], 27), pd_latency=cyc([0.0, 0.0005, 0.001], 27, 3),
                                                      motor_kp=[g[0] for g in cyc(gains, 27, 9)], motor_kd=[g[1] for g in cyc(gains, 27, 9)])),
           ("mixed-terrains", "walk", 27, 0.4, dict(cfg, terrain_type=cyc(["plane", "random", "random"], 27), pd_latency=cyc([0.0, 0.001], 27))),
           ("mixed-repeats", "gallop", 24, 0.3, dict(cfg, signal_type="ol", control_time_step=cyc([0.005, 0.006, 0.010], 24),
                                                      action_repeat=cyc([5, 6, 10], 24), terrain_type=cyc(["plane", "random"], 24, 4))),
           ("mixed-tasks-turn", "turn", 24, 0.01, dict(cfg, signal_type=cyc(["ik", "ol"], 24), terrain_type=cyc(["plane", "random"], 24, 3))),
           ("mixed-tasks-walk-turn", None, 24, 1.0, dict(cfg, normalize=True, task=cyc(["walk", "turn", "turn"], 24),
                                                          signal_type=cyc(["ik", "ik", "ol"], 24))),
           ("mixed-tasks-standup-poses", None, 24, 0.1, dict(cfg, task=cyc(["standup", "poses", "standup"], 24), signal_type=cyc(["ol", "ik", "ik"], 24),
                                                              motor_kp=[g[0] for g in cyc(gains, 24, 2)], motor_kd=[g[1] for g in cyc(gains, 24, 2)])),
           ("mixed-marks", "walk", 24, 0.4, dict(cfg, mark=cyc(["base", "arm"], 24, 5), pd_latency=cyc([0.0, 0.001], 24, 3),
                                                  observation_noise_stdev=(0.01, 0.01, 0.01, 0.01, 0.01)))]
    # the 16 groups of the cap: 2 terrains x 2 marks x 2 rates x 2 step units
    combos = [(t, m, r, sg) for t in ("plane", "random") for m in ("base", "arm") for r in ((0.005, 5), (0.010, 10)) for sg in ("ik", "ol")]
    labels = [combos[(i + i // 16) % 16] for i in range(64)]
    out.append(("mixed-16-groups", "turn", 64, 0.01, dict(cfg, terrain_type=[l[0] for l in labels], mark=[l[1] for l in labels],
                                                          control_time_step=[l[2][0] for l in labels],
                                                          action_repeat=[l[2][1] for l in labels], signal_type=[l[3] for l in labels])))
    # the 64 hold settings of the cap: 8 gains x 2 marks x 2 PD latencies x 2 start poses, on both terrains
    out.append(("mixed-64-settings", None, 128, 0.1, dict(cfg, task=cyc(["standup", "poses"], 128, 64), signal_type="ol",
                                                          motor_kp=cyc([1.0 + 0.01 * k for k in range(8)], 128),
                                                          mark=cyc(["base", "arm"], 128, 16), pd_latency=cyc([0.0, 0.001], 128, 32),
                                                          terrain_type=cyc(["plane", "random"], 128, 3))))
    return out


def mixed_run(R, res):
    """mixed_cases: what the handle holds after construction, then 30 steps after a full reset."""
    import ctypes as C
    import torch
    from rex_gym_b200 import _capi
    _force_build(None)
    for cid, task, n, b, kw in mixed_cases():
        env = R.BatchedRexEnv(num_envs=n, auto_reset=True, **(dict(task=task) if task else {}), **kw)
        L, h = env._L, env._h
        view = lambda p, shape, typestr: _capi.device_view(p.value, shape, typestr, env, "cuda").cpu().numpy()
        rec = res[cid] = {"launch_count": str(env.launch_count)}

        def groups(when):
            words = []
            for g in range(L.rexsim_launch_groups(h)):
                info, t, sg, m = np.zeros(8, np.int32), C.c_int32(), C.c_int32(), C.c_int32()
                assert L.rexsim_launch_group(h, g, info.ctypes.data) == 0
                assert L.rexsim_launch_group_task(h, g, C.byref(t), C.byref(sg)) == 0
                assert L.rexsim_launch_group_mark(h, g, C.byref(m)) == 0
                words.append(info.tolist() + [t.value, sg.value, m.value])
            rec[when + "_groups"] = digest(np.array(words, np.int32))
        groups("built")
        p, q, g, k = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_int32()
        assert L.rexsim_slot_buffers(h, C.byref(p), C.byref(q)) == 0
        rec["perm"] = digest(view(p, (n,), "<i4")) if p.value else "identity"
        rec["group"] = digest(view(q, (n,), "|u1")) if q.value else "one group"
        if env._values is not None:
            assert L.rexsim_env_value_buffers(h, C.byref(p), C.byref(q), C.byref(g), C.byref(k)) == 0
            rec["pair"], rec["gains"], rec["npairs"] = digest(view(q, (n,), "<i4")), digest(view(g, (k.value, 2), "<f4")), str(k.value)
        if env._latency is not None:
            assert L.rexsim_env_latency_buffers(h, C.byref(p), C.byref(k)) == 0
            rec["latency"], rec["depth"] = digest(view(p, (2, n), "<f8")), str(k.value)
        env.reset()
        rng = np.random.default_rng(11)
        for s in range(30):
            ret = env.step(torch.as_tensor(rng.uniform(-b, b, size=(n, env.action_dim)).astype(np.float32), device="cuda"))
            _record(env, rec, s, ret)
        groups("stepped")
        env.close()


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
    """perform, experience, transform_reward of every tests/agent_twin.FF_ROWS row; the three scans."""
    import torch
    import agent_twin as T
    from rex_gym_b200.agents import utility
    sizes = T.ff_batch_sizes(T.half_sm())
    for row in T.FF_ROWS:
        _, _, obs, nets = T.ff_setup(row, max(sizes))
        net = nets[-1]
        x_all = torch.from_numpy(obs).cuda()
        rew_all = torch.from_numpy(np.random.default_rng(3).normal(0.1, 0.5, max(sizes)).astype(np.float32)).cuda()
        rec = res["agent-" + T.ff_id(row)] = {}
        for n in sizes:
            for training in (False, True):
                out = net.perform(x_all[:n], training=training, seed=T.SEED, step=T.STEP, env_offset=T.OFFSET)
                for k, t in out.items():
                    rec[f"n{n}_{'sampled' if training else 'mean'}_{k}"] = digest(t.cpu().numpy())
        for n in sizes:
            net.experience(x_all[:n], rew_all[:n])
            rec[f"n{n}_experience"] = digest(np.r_[net._filt.cpu().numpy().view(np.int32), net._cnt.cpu().numpy().view(np.int32)])
            T.experience_split(net, x_all[:n], rew_all[:n])
            rec[f"n{n}_partial_finalize"] = digest(np.r_[net._filt.cpu().numpy().view(np.int32), net._cnt.cpu().numpy().view(np.int32)])
            rec[f"n{n}_transform_reward"] = digest(net.transform_reward(rew_all[:n]).cpu().numpy())
        for nt in nets:
            nt.close()
    rng = np.random.default_rng(17)
    rec = res["agent-scans"] = {}
    for L in T.SCAN_LENGTHS:
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
    mixed_run(R, res)
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

#!/usr/bin/env python3
"""A/B bit identity of library builds (the outputs half of dev_ab.py's timing A/B).

    python tools/dev_ab_outputs.py rex_gym_b200/librexsim_parent.so rex_gym_b200/librexsim.so [more.so ...]

Runs every step-kernel instance of tests/test_gpu_builds.INSTANCES (forced build, 37 envs, 40 steps of seeded random actions,
auto-reset after 15 steps), walk-ik on flat ground at 8449 and 65 536 envs and turn-ik on heightfields at 16 897 envs (the
big build, warp re-grouping on) once per library, each library in its own process (REXSIM_LIB).  After every step it hashes
obs, reward, done, last_command, the error words, the whole SoA state and the sensor ring; then bench.py --dump-outputs.
Every later library is compared with the first: each array that is not bit-identical is reported."""
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
    from test_gpu_builds import INSTANCES, _config, _row_id
    out = [(_row_id(r), r[0], None if r[4] == "sensor" else r[4], 37, _config(*r[:5])) for r in INSTANCES]
    for n in (8449, 65536):
        out.append((f"walk-ik-plane-n{n}", "walk", None, n, dict(signal_type="ik", seed=13, max_episode_steps=15)))
    out.append(("turn-ik-random-n16897", "turn", None, 16897,
                dict(signal_type="ik", seed=13, max_episode_steps=15, terrain_type="random", num_fields=64)))
    return out


def digest(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(str((a.dtype.str, a.shape)).encode() + a.tobytes()).hexdigest()


def run(out):
    """Child process: every case with the library REXSIM_LIB names; {case: {step_array: sha256}} to `out`."""
    import torch
    import rex_gym_b200 as R
    from rex_gym_b200.envs.batched_env import ACTION_BOUND
    res = {}
    for cid, task, build, n, kw in cases():
        if build:
            os.environ["REXSIM_FORCE_BUILD"] = build
        else:
            os.environ.pop("REXSIM_FORCE_BUILD", None)
        env = R.BatchedRexEnv(task=task, num_envs=n, auto_reset=True, **kw)
        env.reset()
        rng = np.random.default_rng(11)
        b = ACTION_BOUND[(task, kw["signal_type"])]
        rec = res[cid] = {}
        for k in range(40):
            a = torch.as_tensor(rng.uniform(-b, b, size=(n, env.action_dim)).astype(np.float32), device="cuda")
            o, r, d = env.step(a)[:3]
            arrs = dict(obs=o, reward=r, done=d, cmd=env.last_command(), err=env._err, sf=env._state_f, si=env._state_i)
            if env._ring is not None:
                arrs["ring"] = env._ring
            for name, v in arrs.items():
                rec[f"{k:02d}_{name}"] = digest(v.cpu().numpy())
        env.close()
    with open(out, "w") as f:
        json.dump(res, f)


def outputs(lib):
    """{case: {step_array: sha256}} of every case and of bench.py --dump-outputs with library `lib`."""
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
    return steps


def main(libs):
    runs = [outputs(lib) for lib in libs]
    status = 0
    for lib, other in zip(libs[1:], runs[1:]):
        print(f"== {libs[0]} vs {lib}")
        nbad = 0
        for cid, ref in runs[0].items():
            bad = [k for k in ref if other.get(cid, {}).get(k) != ref[k]]
            nbad += bool(bad)
            print(f"{cid:32s} {'identical' if not bad else 'DIFFERS in %d arrays, first %s' % (len(bad), bad[0])}")
        print(f"{len(runs[0]) - nbad} of {len(runs[0])} runs bit-identical\n")
        status |= nbad > 0
    return status


if __name__ == "__main__":
    if sys.argv[1] == "--child":
        sys.path.insert(0, ROOT)
        run(sys.argv[2])
    else:
        sys.exit(main(sys.argv[1:]))

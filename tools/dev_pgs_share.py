#!/usr/bin/env python3
"""The PGS solver's share of the step: the bench.py headline timed at several solver_iterations caps.

    python tools/dev_pgs_share.py [--steps 200] [--warmup 20] [--envs 4096,8448,65536] [--iters 60,30,15,1]

Each batch size runs bench.py's headline workload (walk-ik on flat ground, staggered episode ages, L2 flushed between device-timed
steps, bench.Timer) once per cap.  The time the step loses between the default cap (60) and a single iteration is the solver loop's
share of the critical path.  Prints one line per run and a JSON summary with the GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_name_and_power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as ex:
        return "unknown (%r)" % ex


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--envs", default="4096,8448,65536")
    ap.add_argument("--iters", default="60,30,15,1")
    args = ap.parse_args()
    import torch
    import bench
    import rex_gym_b200 as R
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    T = bench.Timer(dev, 1, flush)
    res = {"gpu": gpu_name_and_power_limit(), "lib": os.environ.get("REXSIM_LIB", "librexsim.so").split("/")[-1], "runs": []}
    for n in [int(x) for x in args.envs.split(",")]:
        times = {}
        for it in [int(x) for x in args.iters.split(",")]:
            gen = torch.Generator(device=dev); gen.manual_seed(1234)
            env = R.BatchedRexEnv(num_envs=n, device="cuda:0", seed=1234, solver_iterations=it, **bench.WORKLOAD)
            env.reset()
            acts = torch.rand((max(32, min(args.warmup + args.steps, 256)), n, env.action_dim), device=dev, generator=gen) * 2 - 1
            bench.stagger_episodes(env, acts)
            for k in range(args.warmup):
                env.step(acts[k % acts.shape[0]])
            r = T.run(env, acts, args.warmup, args.steps)
            err = env.check_errors()
            env.close()
            times[it] = r["ms_per_step"]
            print(f"{res['lib']} n={n:6d} iters={it:3d} {r['ms_per_step']:.4f} ms/step (median {r['median_step_ms']:.4f}) err={err}",
                  flush=True)
            res["runs"].append(dict(envs=n, solver_iterations=it, ms_per_step=r["ms_per_step"], median_step_ms=r["median_step_ms"]))
        hi, lo = max(times), min(times)
        share = (times[hi] - times[lo]) / times[hi]
        print(f"n={n}: solver share of the step (cap {hi} vs {lo}) = {100 * share:.1f} %", flush=True)
        res.setdefault("share", {})[n] = share
    print(json.dumps(res))


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Frames per second of BatchedRexEnv.render_batch (480 x 360 rgb_array, rex_gym_b200/csrc/rexsim_render.cu) for k = 1, 16, 256
images per call, on flat ground and on the random heightfield, with mark 'base' and 'arm'.  CUDA events around >= 1 s of calls
after a warm-up; prints the card and its power limit from the same run, then one JSON line per configuration.

Usage: python tools/bench_render.py [--seconds 1.0] [--out results/bench_render.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:       # the numbers still stand with the torch device name
        q = "%s (nvidia-smi unavailable: %s)" % (torch.cuda.get_device_name(0), e)
    return q


def measure(env, k, seconds):
    idx = torch.arange(k, dtype=torch.int32, device="cuda") % env.num_envs
    for _ in range(3):
        env.render_batch(idx)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(20):
        env.render_batch(idx)
    b.record()
    torch.cuda.synchronize()
    calls = max(20, int(1.25 * seconds * 1000.0 * 20 / max(a.elapsed_time(b), 1e-3)) + 1)
    a.record()
    for _ in range(calls):
        env.render_batch(idx)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b)
    if ms < 1000.0 * seconds:
        return measure(env, k, 2 * seconds)
    return dict(calls=calls, seconds=ms / 1000.0, frames_per_s=calls * k / (ms / 1000.0), ms_per_call=ms / calls)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_render needs a CUDA device")
    from rex_gym_b200.envs.batched_env import BatchedRexEnv
    print("card: name, power limit, max SM clock =", card(), flush=True)
    rows = []
    for terrain in ("plane", "random"):
        for mark in ("base", "arm"):
            task = "walk" if mark == "base" else "standup"
            env = BatchedRexEnv(task=task, num_envs=256, terrain_type=terrain, mark=mark, num_fields=4,
                                signal_type="ik" if task == "walk" else "ol")
            env.reset()
            rng = np.random.default_rng(0)
            b = 0.4 if task == "walk" else 0.1
            for _ in range(50):
                env.step(rng.uniform(-b, b, size=(256, env.action_dim)).astype(np.float32))
            for k in (1, 16, 256):
                r = dict(terrain=terrain, mark=mark, k=k, width=480, height=360, **measure(env, k, a.seconds))
                rows.append(r)
                print(json.dumps(r), flush=True)
            env.close()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()

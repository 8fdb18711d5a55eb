#!/usr/bin/env python3
"""What the fused frame wrappers (BatchedRexEnv(frame_history=[0, 1, 2, 3], frame_delta=True)) cost per control step: walk-ik at
4096 and 65 536 envs, C3 (gallop-ol, random gains, 16 observation words) and C5 (standup with the arm), off and on alternately
in one process, three rounds each.  Same workload as tools/bench_configs.py (normalized actions, auto-reset, staggered
episodes); CUDA events around `steps` device-path steps.  Prints the card and its power limit from the same run, then one JSON
line per configuration.

Usage: python tools/bench_frame_wrappers.py [--steps 200] [--rounds 3]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from bench import stagger_episodes  # noqa: E402
from bench_configs import CONFIGS  # noqa: E402
from bench_render import card  # noqa: E402

NAMES = ("C2 ", "C2' ", "C3 ", "C5 ")           # walk-ik 4096, walk-ik 65536, gallop-ol rand kp/kd, standup arm
FRAMES = dict(frame_history=[0, 1, 2, 3], frame_delta=True)


def ms_per_step(kw, on, steps):
    import rex_gym_b200 as R
    env = R.BatchedRexEnv(normalize=True, auto_reset=True, max_episode_steps=2000, **(FRAMES if on else {}), **kw)
    env.reset()
    g = torch.Generator(device="cuda"); g.manual_seed(3)
    acts = torch.rand((30, env.num_envs, env.action_dim), device="cuda", generator=g) * 2 - 1
    stagger_episodes(env, acts)
    for k in range(20):
        env.step(acts[k % 30])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for k in range(steps):
        env.step(acts[k % 30])
    e1.record()
    torch.cuda.synchronize()
    width = env.obs_dim
    env.close()
    return e0.elapsed_time(e1) / steps, width


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frame_wrappers needs a CUDA device")
    print("card: name, power limit, max SM clock =", card(), flush=True)
    for prefix in NAMES:
        name, kw = next(c for c in CONFIGS if c[0].startswith(prefix))
        off, on, width = [], [], None
        for _ in range(a.rounds):
            off.append(ms_per_step(kw, False, a.steps)[0])
            t, width = ms_per_step(kw, True, a.steps)
            on.append(t)
        row = dict(config=name, envs=kw["num_envs"], steps=a.steps, obs_words_on=width, ms_off=[round(x, 4) for x in off],
                   ms_on=[round(x, 4) for x in on],
                   median_cost_pct=round(100 * (sorted(on)[len(on) // 2] / sorted(off)[len(off) // 2] - 1), 2))
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""What the final observations and time-limit bytes (BatchedRexEnv(final_observation=True)) cost per control step: walk-ik at
4096 and 65 536 envs, C3 (gallop-ol, random gains) and C5 (standup with the arm), the switch off and on alternately in one
process, medians over rounds.  Same workload as tools/bench_episode_stats.py (normalized actions, auto-reset, staggered
episodes); CUDA events around `steps` device-path steps.  Then a 65 536-env walk-ik Rollout (T = 32, feed-forward network):
collect with final_observation off and on, and returns_and_advantages plain against bootstrap_truncated=True (the gather, the
value pass on the truncated rows and its one host sync included).  Episodes of max_episode_steps = 100 there, so that a
32-step window holds truncations.  Prints the card and its power limit from the same run, then one JSON line per row.

Usage: python tools/bench_final_observation.py [--steps 200] [--rounds 3]"""
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


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def ms_per_step(kw, on, steps):
    import rex_gym_b200 as R
    env = R.BatchedRexEnv(normalize=True, auto_reset=True, max_episode_steps=2000, final_observation=on, **kw)
    env.reset()
    g = torch.Generator(device="cuda"); g.manual_seed(3)
    acts = torch.rand((30, env.num_envs, env.action_dim), device="cuda", generator=g) * 2 - 1
    stagger_episodes(env, acts)
    for k in range(20):
        env.step(acts[k % 30])
    k = [0]

    def step():
        env.step(acts[k[0] % 30]); k[0] += 1
    ms = timed(step, steps)
    env.close()
    return ms


def rollout_ms(on, reps):
    import rex_gym_b200 as R
    from rex_gym_b200.agents import ForwardGaussianPolicy, Rollout
    env = R.BatchedRexEnv(task="walk", num_envs=65536, signal_type="ik", target_position=2.0, backwards=False, normalize=True,
                          auto_reset=True, max_episode_steps=100)
    net = ForwardGaussianPolicy(env.obs_dim, env.action_dim, seed=1)
    ro = Rollout(env, net, 32, seed=2, training=True, final_observation=on)
    for _ in range(4):                                 # capture, and episodes spread over the limit
        ro.collect()
    collect = timed(ro.collect, reps)
    ro.collect()
    scan = timed(lambda: ro.returns_and_advantages(0.985, 0.95), reps)
    boot = timed(lambda: ro.returns_and_advantages(0.985, 0.95, bootstrap_truncated=True), reps) if on else None
    truncated = int(ro.truncated.sum()) if on else None
    env.close(); net.close()
    return collect, scan, boot, truncated


def median(x):
    return sorted(x)[len(x) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_final_observation needs a CUDA device")
    print("card: name, power limit, max SM clock =", card(), flush=True)
    for prefix in NAMES:
        name, kw = next(c for c in CONFIGS if c[0].startswith(prefix))
        off, on = [], []
        for _ in range(a.rounds):
            off.append(ms_per_step(kw, False, a.steps))
            on.append(ms_per_step(kw, True, a.steps))
        print(json.dumps(dict(config=name, envs=kw["num_envs"], steps=a.steps, ms_off=[round(x, 4) for x in off],
                              ms_on=[round(x, 4) for x in on], median_cost_pct=round(100 * (median(on) / median(off) - 1), 2))),
              flush=True)
    rows = {False: [], True: []}
    for _ in range(a.rounds):
        for sw in (False, True):
            rows[sw].append(rollout_ms(sw, 5))
    off, on = rows[False], rows[True]
    print(json.dumps(dict(config="walk-ik 65536 Rollout T=32 (ff)", collect_ms_off=[round(r[0], 3) for r in off],
                          collect_ms_on=[round(r[0], 3) for r in on],
                          collect_cost_pct=round(100 * (median([r[0] for r in on]) / median([r[0] for r in off]) - 1), 2),
                          scan_ms=round(median([r[1] for r in on]), 4), bootstrap_ms=round(median([r[2] for r in on]), 4),
                          truncated_steps=on[-1][3])), flush=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Workload for ncu captures of the BASELINE configs: a de-synchronised batch (episode ages staggered like bench.py) stepping on
random actions.  The first entry of bench_configs.CONFIGS whose name starts with the config argument (C2, C3, C4, C5, standup),
with the envs given here.  Usage under ncu:
  ncu --set full --clock-control none --import-source on -k regex:step_kernel -s <skip> -c 1 -o out python tools/prof_cfg.py C5 16384
The staggering takes 256 launches (+ 32 resets); captures should skip ~300 step_kernel launches."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402
import rex_gym_b200 as R  # noqa: E402
from bench import stagger_episodes  # noqa: E402
from bench_configs import CONFIGS  # noqa: E402

cfg = sys.argv[1] if len(sys.argv) > 1 else "C5"
n = int(sys.argv[2]) if len(sys.argv) > 2 else 16384
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 20
common = dict(normalize=True, auto_reset=True, max_episode_steps=2000)
kw = dict(next(kw for name, kw in CONFIGS if name.startswith(cfg)), num_envs=n)
if len(sys.argv) > 4:
    common["rebalance_every"] = int(sys.argv[4])
env = R.BatchedRexEnv(**common, **kw)
env.reset()
acts = torch.rand((64, n, env.action_dim), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1234)) * 2 - 1
stagger_episodes(env, acts)
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
torch.cuda.synchronize(); a.record()
for r in range(5):
    for k in range(steps):
        env.step(acts[k % 64])
b.record(); torch.cuda.synchronize()
print(cfg, n, "rebalance_every", common.get("rebalance_every", "default"), "ms/step %.4f" % (a.elapsed_time(b) / (5 * steps)), "errors", env.check_errors())

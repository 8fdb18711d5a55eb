#!/usr/bin/env python3
"""A/B timing of library builds (REXSIM_LIB=...): steady-state ms/step at several batch sizes, device path."""
import sys, os, time
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import torch
import rex_gym_b200 as R
tag = os.environ.get("REXSIM_LIB", "default").split("/")[-1]
for task, kw in (("walk", dict(target_position=2.0, backwards=False)), ("gallop", dict(signal_type="ol", target_position=2.0))):
    for n in (4096, 8448, 65536):        # one wave of the 255-register build, the largest batch it takes, the 128-register build
        env = R.BatchedRexEnv(task=task, num_envs=n, normalize=True, auto_reset=True, max_episode_steps=2000, **kw)
        env.reset()
        acts = torch.rand((40, n, env.action_dim), device="cuda") * 2 - 1
        for k in range(10): env.step(acts[k])
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); a.record()
        for r in range(5):
            for k in range(10, 40): env.step(acts[k])
        b.record(); torch.cuda.synchronize()
        ms = a.elapsed_time(b) / 150
        print(f"{tag} {task:6s} n={n:6d} {ms:8.4f} ms/step {n/ms/1e3:8.2f} M env-steps/s err={env.check_errors()}", flush=True)
        env.close()

#!/usr/bin/env python3
"""Device-timed throughput of the BASELINE.json configs that are built, on one GPU (not the bench.py contract;
a developer table for DESIGN.md).  Usage: python tools/bench_configs.py [--steps 100]"""
import argparse, json, os, sys
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import torch
import rex_gym_b200 as R
from bench import stagger_episodes

CONFIGS = [
    ("C2 walk-ik flat 4096", dict(task="walk", num_envs=4096, signal_type="ik", target_position=2.0, backwards=False)),
    ("C2' walk-ik flat 65536", dict(task="walk", num_envs=65536, signal_type="ik", target_position=2.0, backwards=False)),
    ("C3 gallop-ol rand kp/kd 16384", dict(task="gallop", num_envs=16384, signal_type="ol", motor_kp_range=(0.8, 1.2), motor_kd_range=(0.01, 0.03))),
    ("C4 turn-ik heightfield 16384 (per-GPU share of 65536 on 4)", dict(task="turn", num_envs=16384, signal_type="ik", terrain_type="random", num_fields=64)),
    ("C4' turn-ik heightfield 65536 on one GPU", dict(task="turn", num_envs=65536, signal_type="ik", terrain_type="random", num_fields=64)),
    ("standup (base mark) 16384", dict(task="standup", num_envs=16384, signal_type="ol")),
    ("C5 standup arm (18-DOF) 16384 (per-GPU share of 131072 on 8)", dict(task="standup", num_envs=16384, signal_type="ol", mark="arm")),
    ("turn-ik heightfield arm (18-DOF) 16384", dict(task="turn", num_envs=16384, signal_type="ik", terrain_type="random", num_fields=64, mark="arm")),
    ("walk-ol flat arm (18-DOF) 16384", dict(task="walk", num_envs=16384, signal_type="ol", target_position=2.0, backwards=False, mark="arm")),
    ("poses arm (18-DOF) 16384", dict(task="poses", num_envs=16384, signal_type="ik", mark="arm")),
]

def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--steps", type=int, default=100); a = ap.parse_args()
    out = []
    for name, kw in CONFIGS:
        env = R.BatchedRexEnv(normalize=True, auto_reset=True, max_episode_steps=2000, **kw)
        env.reset()
        n = env.num_envs
        acts = torch.rand((30, n, env.action_dim), device="cuda") * 2 - 1
        stagger_episodes(env, acts)          # de-synchronised episode phases, as under auto-reset (see bench.py)
        for k in range(20): env.step(acts[k % 30])
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record()
        dones = 0
        for k in range(a.steps):
            _, _, d, _ = env.step(acts[k % 30])
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.steps
        row = dict(config=name, envs=n, ms_per_step=round(ms, 4), M_env_steps_per_s=round(n / ms / 1e3, 2), error_flags_or=env.check_errors())
        print(json.dumps(row), flush=True); out.append(row)
        env.close()

if __name__ == "__main__":
    main()

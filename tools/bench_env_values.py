#!/usr/bin/env python3
"""What per-env constructor values cost.  Step time: walk-ik at 4096 and 65 536 envs and C5 (standup with the arm), the batch
built with scalars (off) and with one value per env (on), alternately in one process, medians over rounds.  On: walk cycles
its envs through targets 1.5 / 2.0 / 2.5 / drawn and directions -1 / 0 / 1 plus three gain pairs; C5 through three gain pairs.
Same workload as tools/bench_final_observation.py (normalized actions, auto-reset, staggered episodes); CUDA events around
`steps` device-path steps.  Creation time (host clock around the constructor, which ends in a device synchronise): walk-ik
at 4096 envs with 1 gain pair through the scalar keywords, and 1, 8 and 64 pairs through per-env gains, on flat ground and
on the 64-field heightfield.  Prints the card and its power limit from the same run, then one JSON line per row.

Also an "equal values" column: every scalar given as an array of equal entries, the same physics through the value block.

Latencies (--workload latencies): walk-ik at 16 384 and 65 536 envs with control_latency 20 ms and pd_latency 1 ms as scalars
against a mixed batch cycling its envs through control latencies 0 / 10.5 / 20 ms and pd latencies 0 / 0.5 / 1 ms (the same
deepest history row), alternately in one process.

Terrains (--workload terrains): walk-ik and turn-ik at 16 384 and 65 536 envs on the 64-field bank, all on the plane, all on
the heightfield, a 50/50 mix (every other env) stepped as two slot ranges of one batch, and the sum of an all-plane and an
all-heightfield batch of N/2 each, alternately in one process.

Repeats (--workload repeats): walk-ik at 16 384 and 65 536 envs, the scalar 5 ms / 5 sub-step batch, a 50/50 mix (every
other env) of (5 ms, 5) and (10 ms, 10) stepped as two slot ranges of one batch, the same mix with each rate on one
contiguous half of the envs ("blocked"), and the sum of a (5 ms, 5) and a (10 ms, 10)
batch of N/2 each, alternately in one process; ms per control step and env-steps/s.  Creation time of walk-ik at 4096 envs
with 1 rate (scalar) and with 8 rates (r ms, r sub-steps for r = 1..8: 8 settle caps).

Tasks (--workload tasks): normalized walk-ik and turn-ik at 16 384 and 65 536 envs, all walk, all turn, a 50/50 mix (every
other env) stepped as two slot ranges of one batch, and the sum of an all-walk and an all-turn batch of N/2 each, alternately
in one process.

Marks (--workload marks): normalized walk-ik at 16 384 and 65 536 envs, all base, all arm, a 50/50 mix (every other env)
stepped as two slot ranges of one batch, and the sum of an all-base and an all-arm batch of N/2 each, alternately in one
process.  Creation time of walk-ik at 4096 envs, all base, all arm and the 50/50 mix.

Usage: python tools/bench_env_values.py [--steps 200] [--rounds 3] [--workload all|values|latencies|terrains|repeats|tasks|marks]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from bench import stagger_episodes  # noqa: E402
from bench_configs import CONFIGS  # noqa: E402
from bench_final_observation import median, timed  # noqa: E402
from bench_render import card  # noqa: E402

NAMES = ("C2 ", "C2' ", "C5 ")                # walk-ik 4096, walk-ik 65536, standup arm 16384
GAINS = [(1.0, 0.02), (1.2, 0.025), (0.8, 0.015)]


def same_values(kw):
    """The config with every scalar given as one equal value per env: the same physics as the scalars, through the block."""
    n, kw = kw["num_envs"], dict(kw)
    for k in ("target_position", "backwards"):
        if k in kw:
            kw[k] = [kw[k]] * n
    kw["motor_kp"], kw["motor_kd"] = np.full(n, 1.0, np.float32), np.full(n, 0.02, np.float32)
    return kw


def per_env(kw):
    """The config with one value per env: targets, directions and gain pairs cycling over the envs."""
    n, kw = kw["num_envs"], dict(kw)
    i = np.arange(n)
    if kw["task"] == "walk":
        kw["target_position"] = np.array([1.5, 2.0, 2.5, np.nan], np.float32)[i % 4]
        kw["backwards"] = (i % 3) - 1
    kw["motor_kp"] = np.array([g[0] for g in GAINS], np.float32)[i % 3]
    kw["motor_kd"] = np.array([g[1] for g in GAINS], np.float32)[i % 3]
    return kw


def mixed_latencies(kw):
    """The config with each env's (control_latency, pd_latency) one of nine, the deepest the scalar row's."""
    i = np.arange(kw["num_envs"])
    return dict(kw, control_latency=np.array([0.0, 0.0105, 0.02])[i % 3], pd_latency=np.array([0.0, 0.0005, 0.001])[(i // 3) % 3])


def ms_per_step(kw, steps):
    import rex_gym_b200 as R
    env = R.BatchedRexEnv(normalize=True, auto_reset=True, max_episode_steps=2000, **kw)
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


def create_ms(kw):
    import rex_gym_b200 as R
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    env = R.BatchedRexEnv(**kw)
    torch.cuda.synchronize()
    ms = 1e3 * (time.perf_counter() - t0)
    env.close()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3, help="step rounds; creation rows take the median of 2 x rounds + 1")
    ap.add_argument("--workload", choices=("all", "values", "latencies", "terrains", "repeats", "tasks", "marks"), default="all")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_env_values needs a CUDA device")
    print("card: name, power limit, max SM clock =", card(), flush=True)
    if a.workload in ("all", "latencies"):
        name, c2 = next(c for c in CONFIGS if c[0].startswith("C2 "))
        for n in (16384, 65536):
            kw = dict(c2, num_envs=n, control_latency=0.02, pd_latency=0.001)
            scalar, mixed = [], []
            for _ in range(a.rounds):
                scalar.append(ms_per_step(kw, a.steps))
                mixed.append(ms_per_step(mixed_latencies(kw), a.steps))
            print(json.dumps(dict(config="walk-ik latencies", envs=n, steps=a.steps, ms_scalar=[round(x, 4) for x in scalar],
                                  ms_mixed=[round(x, 4) for x in mixed],
                                  mixed_cost_pct=round(100 * (median(mixed) / median(scalar) - 1), 2))), flush=True)
    if a.workload in ("all", "terrains"):
        for task in ("walk", "turn"):
            for n in (16384, 65536):
                kw = dict(task=task, signal_type="ik", num_fields=64)
                mix = ["plane", "random"] * (n // 2)
                rows = {}
                for _ in range(a.rounds):
                    for name, k in (("plane", dict(kw, num_envs=n, terrain_type="plane")),
                                    ("random", dict(kw, num_envs=n, terrain_type="random")),
                                    ("mixed", dict(kw, num_envs=n, terrain_type=mix)),
                                    ("half_plane", dict(kw, num_envs=n // 2, terrain_type="plane")),
                                    ("half_random", dict(kw, num_envs=n // 2, terrain_type="random"))):
                        rows.setdefault(name, []).append(ms_per_step(k, a.steps))
                halves = median(rows["half_plane"]) + median(rows["half_random"])
                print(json.dumps(dict(config="%s-ik terrains" % task, envs=n, steps=a.steps,
                                      **{"ms_" + k: [round(x, 4) for x in v] for k, v in rows.items()},
                                      ms_halves_sum=round(halves, 4),
                                      mixed_vs_halves_pct=round(100 * (median(rows["mixed"]) / halves - 1), 2))), flush=True)
    if a.workload in ("all", "repeats"):
        for n in (16384, 65536):
            kw = dict(task="walk", signal_type="ik")
            mix = [(0.005, 5), (0.010, 10)] * (n // 2)
            rows = {}
            for _ in range(a.rounds):
                for name, k in (("scalar", dict(kw, num_envs=n, control_time_step=0.005, action_repeat=5)),
                                ("mixed", dict(kw, num_envs=n, control_time_step=[c for c, _ in mix],
                                               action_repeat=[r for _, r in mix])),
                                ("mixed_blocked", dict(kw, num_envs=n, control_time_step=[0.005] * (n // 2) + [0.010] * (n // 2),
                                                       action_repeat=[5] * (n // 2) + [10] * (n // 2))),
                                ("half_5", dict(kw, num_envs=n // 2, control_time_step=0.005, action_repeat=5)),
                                ("half_10", dict(kw, num_envs=n // 2, control_time_step=0.010, action_repeat=10))):
                    rows.setdefault(name, []).append(ms_per_step(k, a.steps))
            halves = median(rows["half_5"]) + median(rows["half_10"])
            print(json.dumps(dict(config="walk-ik repeats", envs=n, steps=a.steps,
                                  **{"ms_" + k: [round(x, 4) for x in v] for k, v in rows.items()},
                                  ms_halves_sum=round(halves, 4),
                                  env_steps_per_s={"scalar": round(n / median(rows["scalar"]) * 1e3),
                                                   "mixed": round(n / median(rows["mixed"]) * 1e3),
                                                   "halves": round(n / halves * 1e3)},
                                  mixed_vs_halves_pct=round(100 * (median(rows["mixed"]) / halves - 1), 2))), flush=True)
        n = 4096
        base = dict(task="walk", num_envs=n, signal_type="ik", target_position=2.0, backwards=False)
        create_ms(base)                                      # module load and first-launch costs out of the timed rows
        rates = [(r / 1000, r) for r in range(1, 9)]
        eight = dict(base, control_time_step=[rates[e % 8][0] for e in range(n)], action_repeat=[rates[e % 8][1] for e in range(n)])
        rows = {"1_rate": [], "8_rates": []}
        for _ in range(2 * a.rounds + 1):
            rows["1_rate"].append(create_ms(base))
            rows["8_rates"].append(create_ms(eight))
        print(json.dumps(dict(config="create walk-ik %d envs, plane" % n, **{"ms_" + k: round(median(v), 1) for k, v in rows.items()})),
              flush=True)
    if a.workload in ("all", "tasks"):
        for n in (16384, 65536):
            kw = dict(signal_type="ik")
            rows = {}
            for _ in range(a.rounds):
                for name, k in (("walk", dict(kw, num_envs=n, task="walk")),
                                ("turn", dict(kw, num_envs=n, task="turn")),
                                ("mixed", dict(kw, num_envs=n, task=["walk", "turn"] * (n // 2))),
                                ("half_walk", dict(kw, num_envs=n // 2, task="walk")),
                                ("half_turn", dict(kw, num_envs=n // 2, task="turn"))):
                    rows.setdefault(name, []).append(ms_per_step(k, a.steps))
            halves = median(rows["half_walk"]) + median(rows["half_turn"])
            print(json.dumps(dict(config="walk-ik + turn-ik tasks, normalized", envs=n, steps=a.steps,
                                  **{"ms_" + k: [round(x, 4) for x in v] for k, v in rows.items()},
                                  ms_halves_sum=round(halves, 4),
                                  mixed_vs_halves_pct=round(100 * (median(rows["mixed"]) / halves - 1), 2))), flush=True)
    if a.workload in ("all", "marks"):
        for n in (16384, 65536):
            kw = dict(task="walk", signal_type="ik")
            rows = {}
            for _ in range(a.rounds):
                for name, k in (("base", dict(kw, num_envs=n, mark="base")),
                                ("arm", dict(kw, num_envs=n, mark="arm")),
                                ("mixed", dict(kw, num_envs=n, mark=["base", "arm"] * (n // 2))),
                                ("half_base", dict(kw, num_envs=n // 2, mark="base")),
                                ("half_arm", dict(kw, num_envs=n // 2, mark="arm"))):
                    rows.setdefault(name, []).append(ms_per_step(k, a.steps))
            halves = median(rows["half_base"]) + median(rows["half_arm"])
            print(json.dumps(dict(config="walk-ik marks, normalized", envs=n, steps=a.steps,
                                  **{"ms_" + k: [round(x, 4) for x in v] for k, v in rows.items()},
                                  ms_halves_sum=round(halves, 4),
                                  mixed_vs_halves_pct=round(100 * (median(rows["mixed"]) / halves - 1), 2))), flush=True)
        n = 4096
        base = dict(task="walk", num_envs=n, signal_type="ik", target_position=2.0, backwards=False)
        create_ms(base)                                      # module load and first-launch costs out of the timed rows
        rows = {"base": [], "arm": [], "mixed": []}
        for _ in range(2 * a.rounds + 1):
            rows["base"].append(create_ms(dict(base, mark="base")))
            rows["arm"].append(create_ms(dict(base, mark="arm")))
            rows["mixed"].append(create_ms(dict(base, mark=["base", "arm"] * (n // 2))))
        print(json.dumps(dict(config="create walk-ik %d envs, marks" % n, **{"ms_" + k: round(median(v), 1) for k, v in rows.items()})),
              flush=True)
    if a.workload in ("latencies", "terrains", "repeats", "tasks", "marks"):
        return
    for prefix in NAMES:
        name, kw = next(c for c in CONFIGS if c[0].startswith(prefix))
        off, same, on = [], [], []
        for _ in range(a.rounds):
            off.append(ms_per_step(kw, a.steps))
            same.append(ms_per_step(same_values(kw), a.steps))
            on.append(ms_per_step(per_env(kw), a.steps))
        # same: the feature's own cost (identical physics); on: a mixed batch, whose envs also walk, fall and reset differently
        print(json.dumps(dict(config=name, envs=kw["num_envs"], steps=a.steps, ms_off=[round(x, 4) for x in off],
                              ms_same=[round(x, 4) for x in same], ms_on=[round(x, 4) for x in on],
                              same_cost_pct=round(100 * (median(same) / median(off) - 1), 2),
                              mixed_cost_pct=round(100 * (median(on) / median(off) - 1), 2))), flush=True)
    n = 4096
    base = dict(task="walk", num_envs=n, signal_type="ik", target_position=2.0, backwards=False)
    create_ms(base)                                          # module load and first-launch costs out of the timed rows
    for terrain in ("plane", "random"):
        kw = dict(base, terrain_type=terrain, num_fields=64)
        rows = {"scalar": []}
        for _ in range(2 * a.rounds + 1):
            rows["scalar"].append(create_ms(kw))
            for pairs in (1, 8, 64):
                kp = (1.0 + 0.005 * (np.arange(n) % pairs)).astype(np.float32)
                rows.setdefault(pairs, []).append(create_ms(dict(kw, motor_kp=kp)))
        print(json.dumps(dict(config="create walk-ik %d envs, %s" % (n, terrain),
                              **{("ms_%s" % k if k == "scalar" else "ms_%d_pairs" % k): round(median(v), 1) for k, v in rows.items()})),
              flush=True)


if __name__ == "__main__":
    main()

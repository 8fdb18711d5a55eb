#!/usr/bin/env python3
"""Device-timed numbers for the agent glue (developer table for DESIGN.md): perform (feed-forward, recurrent and linear policy
cells), experience, the scans and the graph-captured rollout (policy + env step + filter update per control step), with the
card name and power limit read in the same run.  Usage: python tools/bench_agent.py [--cells: the policy-cell rows alone]"""
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402
import rex_gym_b200 as R  # noqa: E402
from rex_gym_b200.agents import ForwardGaussianPolicy, LinearGaussianPolicy, RecurrentGaussianPolicy, Rollout, utility  # noqa: E402


def timed(fn, reps=50, warm=5):
    for _ in range(warm):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); a.record()
    for _ in range(reps):
        fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def card():
    """The device name and its enforced power limit (nvidia-smi query, read only), as the numbers' context."""
    import subprocess
    row = dict(kernel="card", name=torch.cuda.get_device_name(0))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        row["power_limit_and_max_sm_clock"] = q
    except Exception as e:                                  # the name alone still says what was measured
        row["power_limit_and_max_sm_clock"] = "unavailable: %s" % e
    return row


def policy_flops(cell, O, A, H1=200, H2=100, G=100):
    """Multiply-adds x 2 per env of one perform: the policy (dense, cell, head) plus the value MLP O-H1-H2-1."""
    value = O * H1 + H1 * H2 + H2
    policy = dict(forward=O * H1 + H1 * H2 + H2 * A, recurrent=O * H1 + (H1 + G) * 3 * G + G * A, linear=O * A)[cell]
    return 2.0 * (policy + value)


def perform_rows():
    rows = []
    for O, A in ((4, 2), (16, 4)):
        for n in (4096, 16384, 65536):
            for cell in ("forward", "recurrent", "linear"):
                if cell == "forward":
                    net = ForwardGaussianPolicy(O, A)
                elif cell == "recurrent":
                    net = RecurrentGaussianPolicy(O, A, num_envs=n)
                else:
                    net = LinearGaussianPolicy(O, A, num_envs=n)
                x = torch.randn((n, O), device="cuda")
                out = net.perform(x, training=True)
                ms = timed(lambda: net.perform(x, training=True, out=out))
                fl = n * policy_flops(cell, O, A)
                rows.append(dict(kernel="perform", cell=cell, O=O, A=A, n=n, ms=round(ms, 4), gflops=round(fl / ms / 1e6, 1)))
                net.close()
    return rows


def rollout_rows():
    rows = []
    for n in (4096, 65536):
        for cell in (ForwardGaussianPolicy, RecurrentGaussianPolicy):
            env = R.BatchedRexEnv(task="walk", num_envs=n, signal_type="ik", normalize=True, auto_reset=True,
                                  max_episode_steps=2000, target_position=2.0, backwards=False)
            net = cell(env.obs_dim, env.action_dim) if cell is ForwardGaussianPolicy else cell(env.obs_dim, env.action_dim, num_envs=n)
            T = 32
            ro = Rollout(env, net, T, training=True, use_graph=True)
            ms = timed(ro.collect, reps=10, warm=2)
            rows.append(dict(kernel="rollout(perform+step+experience)", cell=cell.__name__, graph=True, n=n, T=T,
                             ms_per_control_step=round(ms / T, 4), M_env_steps_per_s=round(n * T / ms / 1e3, 2)))
            env.close(); net.close()
    return rows


def main():
    if "--cells" in sys.argv:                               # only the policy-cell rows (perform and rollout per cell)
        for r in [card()] + perform_rows() + rollout_rows():
            print(json.dumps(r), flush=True)
        return
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm = float(peaks.get("hbm_gbs", 3350.0))
    rows = []
    for O, A, n in ((4, 2, 4096), (4, 2, 65536), (16, 4, 65536)):
        net = ForwardGaussianPolicy(O, A)
        x = torch.randn((n, O), device="cuda")
        out = net.perform(x, training=True)
        ms = timed(lambda: net.perform(x, training=True, out=out))
        flops = 2.0 * n * 2 * (O * 200 + 200 * 100 + 100 * (A + 1) / 2)
        rows.append(dict(kernel="perform", O=O, A=A, n=n, ms=round(ms, 4), gflops=round(flops / ms / 1e6, 1),
                         frac_fp32_peak=round(flops / ms / 1e6 / 74400.0, 3)))
        r = torch.randn((n,), device="cuda")
        ms = timed(lambda: net.experience(x, r))
        rows.append(dict(kernel="experience", O=O, n=n, ms=round(ms, 4)))
        net.close()
    for T, n in ((64, 65536), (256, 65536)):
        rw, v = torch.randn((T, n), device="cuda"), torch.randn((T + 1, n), device="cuda")
        d = (torch.rand((T, n), device="cuda") < 0.01)
        ms = timed(lambda: utility.gae_segments(rw, v, d, 0.985, 0.95), reps=20)
        byt = T * n * (4 + 4 + 1 + 4 + 4)
        rows.append(dict(kernel="gae_segments", T=T, n=n, ms=round(ms, 4), GBps=round(byt / ms / 1e6, 1), frac_hbm=round(byt / ms / 1e6 / hbm, 3)))
        ln = torch.full((n,), T, dtype=torch.int32, device="cuda")
        rt, vt = rw.t(), v[:T].t()                          # [E][L] views of time-major storage
        ms = timed(lambda: utility.lambda_advantage(rt, vt, ln, 0.985), reps=20)
        byt = T * n * 12
        rows.append(dict(kernel="lambda_advantage", L=T, episodes=n, ms=round(ms, 4), GBps=round(byt / ms / 1e6, 1), frac_hbm=round(byt / ms / 1e6 / hbm, 3)))
    for n in (4096, 65536):
        env = R.BatchedRexEnv(task="walk", num_envs=n, signal_type="ik", normalize=True, auto_reset=True, max_episode_steps=2000,
                              target_position=2.0, backwards=False)
        net = ForwardGaussianPolicy(env.obs_dim, env.action_dim)
        T = 32
        for graph in (False, True):
            ro = Rollout(env, net, T, training=True, use_graph=graph)
            ms = timed(ro.collect, reps=10, warm=2)
            rows.append(dict(kernel="rollout(perform+step+experience)", graph=graph, n=n, T=T, ms_per_control_step=round(ms / T, 4),
                             M_env_steps_per_s=round(n * T / ms / 1e3, 2)))
        env.close(); net.close()
    rows = [card()] + rows + perform_rows() + rollout_rows()
    for r in rows:
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Find the first env/step where GPU and oracle part ways and print what happened around it."""
import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np
from twin import bound, make_env, make_oracle, state_errors, toe_masks

def run(task, sig, n, steps, seed, thr=2e-4, **kw):
    env, ora = make_env(task, n, signal_type=sig, seed=seed, **kw), make_oracle(task, n, signal_type=sig, seed=seed, **kw)
    env.reset(); ora.reset()
    print(f"[{task}-{sig}] reset dq {state_errors(env, ora)[0].max():.2e}")
    rng = np.random.default_rng(11); b = bound(task, sig)
    hist = []
    for k in range(steps):
        a = rng.uniform(-b, b, size=(n, env.action_dim)).astype(np.float32)
        env.step(a); ora.step(a)
        eq = state_errors(env, ora)[0]
        lim = np.array([ora.env(i).limit_rows for i in range(n)])
        it = np.array([ora.env(i).solver_iters for i in range(n)])
        hist.append((eq, toe_masks(ora), env.get_state()['contact_mask'].copy(), lim, it))
        bad = np.nonzero(eq > thr)[0]
        if len(bad):
            i = bad[0]
            print(f"  first divergence: env {i} at step {k}: dq {eq[i]:.2e}; flags {int(env.error_flags()[i])}")
            for kk in range(max(0, k - 8), k + 1):
                h = hist[kk]
                print(f"   step {kk}: dq {h[0][i]:.2e} oracle mask {h[1][i]:09b} gpu mask {h[2][i]:09b} limit rows {h[3][i]} iters {h[4][i]} pos z {ora.env(i).pos[2]:.3f}")
            break
    else:
        print("  no divergence above", thr, "max", max(h[0].max() for h in hist))
    env.close()

if __name__ == "__main__":
    run("gallop", "ol", 32, 120, 3, target_position=2.0, motor_kp_range=(0.8, 1.2), motor_kd_range=(0.01, 0.03))
    run("turn", "ik", 16, 30, 9, terrain_type="random", num_fields=4)
    run("standup", "ol", 16, 60, 3)

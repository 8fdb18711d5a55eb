"""Dev: CUDA sensor model vs oracle, per-step error table for several configurations (run on the GPU box)."""
import sys, os
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from twin import NOISE, bound, make_env, make_oracle, state_errors, sync

CASES = [("walk", "ik", dict(target_position=2.0, backwards=False, control_latency=0.0125)),
         ("walk", "ik", dict(target_position=2.0, backwards=False, observation_noise_stdev=NOISE)),
         ("walk", "ik", dict(target_position=2.0, backwards=False, pd_latency=0.0005)),
         ("walk", "ik", dict(target_position=2.0, backwards=False, pd_latency=0.001)),
         ("walk", "ik", dict(target_position=2.0, backwards=False, pd_latency=0.003)),
         ("gallop", "ol", dict(target_position=2.0, control_latency=0.0105, observation_noise_stdev=NOISE)),
         ("poses", "ik", dict(control_latency=0.03)),
         ("poses", "ik", dict(pd_latency=0.001)),
         ("standup", "ol", dict(mark="arm", control_latency=0.01, observation_noise_stdev=(0, 0.05, 0.1, 0, 0))),
         ("walk", "ik", dict(control_latency=0.0125, terrain_type="random", num_fields=4))]
n = 16
for task, sig, kw in CASES:
    env, ora = make_env(task, n, signal_type=sig, seed=5, **kw), make_oracle(task, n, signal_type=sig, seed=5, **kw)
    og, oc = env.reset(), ora.reset()
    print(task, sig, kw)
    print("  reset |dobs| max per column:", np.abs(og - oc).max(0)[:6])
    if task == "standup":
        sync(env, ora)
    rng = np.random.default_rng(4)
    b = bound(task, sig)
    for k in range(40):
        a = rng.uniform(-b, b, size=(n, env.action_dim)).astype(np.float32)
        o, r, d, _ = env.step(a)
        oc, rc, dc = ora.step(a)
        if k % 5 == 0 or k < 3:
            dq = state_errors(env, ora)[0].max()
            print("  step %2d  ang %.2e  rate %.2e  rest %.2e  rew %.2e  state-q %.2e  done %s" % (
                k, np.abs(o[:, :2] - oc[:, :2]).max(), np.abs(o[:, 2:4] - oc[:, 2:4]).max(),
                np.abs(o[:, 4:] - oc[:, 4:]).max() if o.shape[1] > 4 else 0.0, np.abs(r - rc).max(), dq, (d != dc).sum()))
    env.close()

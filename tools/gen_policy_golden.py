"""Write tests/golden/policies/*.npz: what the tests need from the TF checkpoints the reference ships under
rex_gym/policies/<task>/<signal>/, small enough to commit.

Per checkpoint:
  * the checkpoint's own .index file, byte for byte, and the shard bytes of the tensors the tests read -- the global step,
    both streaming-normaliser states and the policy network -- at their original offsets.  tests/golden/tf_policies.py
    rebuilds a sparse checkpoint from them, so the pure-Python reader (rex_gym_b200/agents/tf_checkpoint.py) still parses
    the real index and reads the real tensors.  The value network and the PPO episode memory are not stored: they read as
    zeros from the rebuilt shard.
  * a fixed, seeded sample of the episode memory TensorFlow recorded (observation, sampled action, action mean, log-stddev,
    reward): all 25 episodes at MEM_STEPS of the first 400 control steps.

Usage: python tools/gen_policy_golden.py [--ref <rex-gym checkout>]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rex_gym_b200.agents import networks, tf_checkpoint as tfc  # noqa: E402

CHECKPOINTS = ["gallop/ik", "gallop/ol", "standup/ol", "turn/ik", "turn/ol", "walk/ik", "walk/ol", "poses"]
MEM_STEPS = 96
FILTERS = ["global_step", "normalize_observ/Variable", "normalize_observ/Variable_1", "normalize_observ/Variable_2",
           "normalize_reward/Variable", "normalize_reward/Variable_1", "normalize_reward/Variable_2"]
POLICY = [networks._TF + n for _, block, n, _ in networks._PARAMS if block == networks.POLICY]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", required=True, help="root of a rex-gym checkout")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "policies"))
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    steps = np.sort(np.random.default_rng(0).choice(400, MEM_STEPS, replace=False)).astype(np.int32)
    for rel in CHECKPOINTS:
        prefix = tfc.latest_checkpoint(os.path.join(a.ref, "rex_gym", "policies", rel))
        ents = tfc.list_variables(prefix)
        shard = "%s.data-00000-of-00001" % prefix
        data = np.fromfile(shard, dtype=np.uint8)
        names = FILTERS + POLICY
        ranges = np.array(sorted((ents[n][3], ents[n][4]) for n in names), dtype=np.int64)
        out = dict(name=np.array(os.path.basename(prefix)), index=np.fromfile(prefix + ".index", dtype=np.uint8),
                   data_size=np.int64(data.size), ranges=ranges, chunks=np.concatenate([data[o:o + s] for o, s in ranges]))
        if rel != "poses":
            m = tfc.load_variables(prefix, ["memory/Variable_%d" % k for k in (1, 2, 3, 4, 5)])
            out.update(mem_steps=steps, mem_observ=m["memory/Variable_1"][:, steps], mem_action=m["memory/Variable_2"][:, steps],
                       mem_mean=m["memory/Variable_3"][:, steps], mem_logstd=m["memory/Variable_4"][:, steps],
                       mem_reward=m["memory/Variable_5"][:, steps])
        path = os.path.join(a.out, rel.replace("/", "_") + ".npz")
        np.savez_compressed(path, **out)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()

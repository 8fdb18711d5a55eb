#!/usr/bin/env python3
"""Golden vectors for the frame wrappers, produced by running the reference's own code from /root/reference (read-only):

  rex_gym.agents.tools.wrappers.{FrameHistory, FrameDelta, RangeNormalize, ClipAction, LimitDuration, ConvertTo32Bit}
      (wrappers.py:93-181,183-291,461-544) stacked as the step kernel fuses them,
          ConvertTo32Bit(FrameHistory(FrameDelta(ClipAction(RangeNormalize(LimitDuration(env))))))
      (RangeNormalize and ClipAction only with normalize; either frame wrapper alone too), around the scripted inner env of
      tools/gen_wrapper_golden.py, whose Boxes come from the walk and gallop envs' own constructor lines.

Shims as in tools/gen_wrapper_golden.py (stub gym / pybullet / pybullet_data / tensorflow, RexGymEnv.__init__ -> keyword
recorder).  Each case resets mid-stream; the cases cover an index equal to the capacity, duplicates, an unordered list, delta
alone, delta under history and both normalize settings.

Output: tests/golden/frame_wrapper_golden.json.gz (committed; the GPU box has no /root/reference).
"""
import gzip
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gen_golden import install_stubs, FakeRex  # noqa: E402
from gen_wrapper_golden import install_tf_stub, ScriptedEnv  # noqa: E402

OUT = os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "frame_wrapper_golden.json.gz")

# (past_indices or None, delta)
FRAMES = [([0, 1, 2, 3], True), ([0, 1, 2], False), ([3, 0, 1, 1], False), ([0, 4, 0, 2], True), (None, True), ([0, 1], False)]
RESETS = (6, 13)              # the stack is reset again before these steps


class ContinuingEnv(ScriptedEnv):
    """The scripted inner env, whose reset after the first returns the next row of its script instead of row 0."""

    def reset(self):
        if self.seen or self.k:
            self.k += 1
        return np.array(self._o[self.k], np.float64)


def main():
    install_stubs()
    install_tf_stub()
    import rex_gym.envs.rex_gym_env as rge
    from rex_gym.agents.tools import wrappers

    def recorder_init(self, **kw):
        self._kw = kw
        self._signal_type = kw.get("signal_type")
        self._time_step = kw["control_time_step"] / kw["action_repeat"]
        self.mark = kw.get("mark", "base")
        self._on_rack = kw.get("on_rack", False)
        self.num_motors = 12
        self.rex = FakeRex(self._time_step, self.num_motors)
        self.rex.num_motors = self.num_motors
    rge.RexGymEnv.__init__ = recorder_init
    from rex_gym.envs.gym import walk_env, gallop_env
    classes = {"walk": walk_env.RexWalkEnv, "gallop": gallop_env.RexReactiveEnv}
    gold = {"reference": "nicrusso7/rex-gym @ /root/reference",
            "shims": ["stub gym/pybullet/pybullet_data/tensorflow", "RexGymEnv.__init__ -> keyword recorder"],
            "wrapper_order": ["LimitDuration", "RangeNormalize", "ClipAction", "FrameDelta", "FrameHistory", "ConvertTo32Bit"],
            "cases": []}
    rng = np.random.default_rng(20261017)
    for task, cls in classes.items():
        env = cls.__new__(cls)
        env.__init__(signal_type="ik")
        asp = env.action_space
        hi = env._get_observation_upper_bound() + rge.OBSERVATION_EPS
        lo = env._get_observation_lower_bound() - rge.OBSERVATION_EPS
        osp = sys.modules["gym.spaces"].Box(lo, hi)
        A, O = asp.shape[0], osp.shape[0]
        for normalize in (False, True):
            for past, delta in FRAMES:
                T, duration = 20, 50
                obs = rng.uniform(-1, 1, (T + 1, O)) * hi * rng.choice([1e-3, 0.1, 1.0], (T + 1, 1))
                rew = rng.normal(0, 1, T + 1)
                inner = ContinuingEnv(asp, osp, obs, rew, np.zeros(T + 1, bool))
                w = wrappers.LimitDuration(inner, duration)
                if normalize:
                    w = wrappers.ClipAction(wrappers.RangeNormalize(w))
                inner_space = (np.asarray(w.observation_space.low).tolist(), np.asarray(w.observation_space.high).tolist())
                if delta:
                    w = wrappers.FrameDelta(w)
                if past is not None:
                    w = wrappers.FrameHistory(w, past, True)
                w = wrappers.ConvertTo32Bit(w)
                acts = rng.uniform(-1, 1, (T, A))
                # the stream: a reset, then steps, the stack reset again before the steps in RESETS; every event consumes the
                # next row of the inner script (events[j] = [kind, row])
                events, out = [], []
                o = w.reset()
                events.append(["reset", inner.k]); out.append(np.asarray(o, np.float64).tolist())
                for t in range(T - len(RESETS)):
                    if t in RESETS:
                        o = w.reset()
                        events.append(["reset", inner.k]); out.append(np.asarray(o, np.float64).tolist())
                    o, r, d, _ = w.step(acts[t])
                    events.append(["step", inner.k]); out.append(np.asarray(o, np.float64).tolist())
                assert all(np.asarray(x, np.float32).dtype == np.float32 for x in out)
                sp = w.observation_space
                gold["cases"].append(dict(task=task, O=O, normalize=normalize, past_indices=past, delta=delta,
                                          sim_dt=env._time_step, raw_observs=obs.tolist(), events=events, observs=out,
                                          observ_box=[lo.tolist(), hi.tolist()], inner_space=inner_space,
                                          space=[np.asarray(sp.low, np.float64).tolist(), np.asarray(sp.high, np.float64).tolist()]))
                print(task, "normalize" if normalize else "raw", past, "delta" if delta else "", "width", len(out[-1]))
    # FrameHistory's own refusal of a list without the current frame (wrappers.py:108-109)
    try:
        wrappers.FrameHistory(None, [1, 2], True)
    except KeyError as e:
        gold["missing_zero_error"] = str(e.args[0])
    with gzip.open(OUT, "wt") as f:
        json.dump(gold, f)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

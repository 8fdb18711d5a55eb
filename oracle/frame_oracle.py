"""Host restatement of the reference's FrameHistory and FrameDelta wrappers (rex_gym/agents/tools/wrappers.py:93-181) for a
batch, stacked as the step kernel fuses them around the oracle's wrapper arithmetic (oracle.py wrap_observation):

    ConvertTo32Bit(FrameHistory(FrameDelta(ClipAction(RangeNormalize(LimitDuration(env))))))

dtype=np.float64 restates the reference (FrameDelta subtracts the float64 observations, ConvertTo32Bit casts the result);
dtype=np.float32 restates the kernel, which subtracts the float32 observations it writes without the wrappers."""
import numpy as np


class FrameWrappers:
    """FrameHistory(past_indices, flatten=True) over FrameDelta, per env of a batch of n.  Either may be off: past_indices None
    (or empty) for no history, delta False for no delta."""

    def __init__(self, n, obs_dim, past_indices=None, delta=False, dtype=np.float64):
        self.n, self.O, self.dtype = n, obs_dim, dtype
        self.idx = list(past_indices or [])
        self.delta = bool(delta)
        self.C = max(self.idx) if self.idx else 0
        self.ring = np.zeros((n, max(self.C, 1), obs_dim), dtype)      # FrameHistory._buffer per env
        self.last = np.zeros((n, obs_dim), dtype)                       # FrameDelta._last per env
        self.t = np.zeros(n, np.int64)                                  # FrameHistory._step per env

    @property
    def out_dim(self):
        return self.O * (len(self.idx) if self.idx else 1)

    def _select(self, e):
        if not self.idx:
            return self.ring[e, 0]
        return np.concatenate([self.ring[e, (self.t[e] - i) % self.C] for i in self.idx])

    def reset(self, obs, envs=None):
        """obs [k, O] the inner observations of a reset of envs (default: all) -> [k, out_dim] float32."""
        envs = np.arange(self.n) if envs is None else np.asarray(envs)
        out = np.zeros((len(envs), self.out_dim), np.float32)
        for j, e in enumerate(envs):
            x = np.asarray(obs[j], self.dtype)
            self.last[e] = x                                            # FrameDelta.reset: last = observ, returns observ
            self.ring[e, :] = x                                         # FrameHistory.reset: every slot, step = 0
            self.t[e] = 0
            out[j] = self._select(e).astype(np.float32)
        return out

    def step(self, obs, first=None):
        """obs [n, O] the inner observations of a step of every env -> [n, out_dim] float32.  first [n] bool marks envs whose
        observation is the first of a new episode (an auto-reset step): they restart as in reset()."""
        out = np.zeros((self.n, self.out_dim), np.float32)
        for e in range(self.n):
            x = np.asarray(obs[e], self.dtype)
            if first is not None and first[e]:
                out[e] = self.reset(x[None], [e])[0]
                continue
            d = x
            if self.delta:                                              # FrameDelta.step: observ - last, then last = observ
                d = x - self.last[e]
                self.last[e] = x
            self.t[e] += 1                                              # FrameHistory.step: buffer[step % capacity] = observ
            if self.idx:
                self.ring[e, self.t[e] % self.C] = d
            else:
                self.ring[e, 0] = d
            out[e] = self._select(e).astype(np.float32)
        return out


def frame_spaces(low, high, past_indices=None, delta=False):
    """The observation Box through FrameDelta (wrappers.py:163-168) and FrameHistory (:116-125), in the inputs' dtype."""
    low, high = np.asarray(low), np.asarray(high)
    if delta:
        low, high = low - high, high - low
    if past_indices:
        low = np.repeat(low[None, ...], len(past_indices), 0).reshape(-1)
        high = np.repeat(high[None, ...], len(past_indices), 0).reshape(-1)
    return low, high

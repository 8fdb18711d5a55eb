"""CPU ORACLE (test infrastructure, NOT the product path) for the agent glue around the step kernel: a numpy restatement
of the TensorFlow-1 graph pieces of rex_gym/agents that rex_gym_b200/csrc/rexsim_agent.cu replaces.

Only tests/ may import this module.

PARITY STATUS: pinned statistically, not bit-wise, against TensorFlow outputs.  tensorflow==1.15 is not installable here, but
the shipped checkpoints' EpisodeMemory keeps what TF itself computed during the last training episodes: per stored observation the
action mean and log-stddev (memory/Variable_3 / _4) and the sampled action.  They come from the weights of one to three optimiser
updates BEFORE the saved ones (the stored log-stddevs differ from the checkpoint's by ~3e-3), so they cannot be exact goldens of
the saved weights; the forward pass below reproduces them to an rms of 0.02-0.08 (policy stddev 0.39) on all seven checkpoints
that carry a memory, and every architectural alternative tried is 2-25x worse (tests/test_tf_recorded_policy_outputs.py).
Also checked: the network against an independent torch fp32 MLP built from the same TF variables, the normaliser against the
two-pass definition, the scans against brute-force sums, and that all ten shipped checkpoints load into this layout
(tests/test_agent_oracle.py).
"""
import math

import numpy as np


# ---- agents/ppo/normalize.py -----------------------------------------------------------------------------------------
class StreamingNormalize(object):
    """normalize.py:22-144 (count, mean, var_sum; transform / update / _std)."""

    def __init__(self, shape, center=True, scale=True, clip=10, dtype=np.float64):
        self.center, self.scale, self.clip = center, scale, clip
        self.count = 0
        self.mean = np.zeros(shape, dtype)
        self.var_sum = np.zeros(shape, dtype)
        self.dtype = dtype

    def std(self):                                         # :131-144
        if self.count > 1:
            return np.sqrt(self.var_sum / self.dtype(self.count - 1) + self.dtype(1e-4))
        return np.full_like(self.var_sum, np.nan)

    def transform(self, value):                            # :43-71
        v = np.array(value, self.dtype)
        if self.center:
            v = v - self.mean
        if self.scale:
            v = v / ((self.std() + self.dtype(1e-8)) if self.count > 1 else np.ones_like(self.var_sum))
        if self.clip:
            v = np.clip(v, -self.clip, self.clip)
        return v

    def update(self, value):                               # :73-99 (batch form)
        v = np.array(value, self.dtype)
        if v.ndim == self.mean.ndim:
            v = v[None, ...]
        self.count += v.shape[0]
        step = self.dtype(self.count)
        mean_delta = (v - self.mean[None, ...]).sum(0)
        new_mean = self.mean + mean_delta / step
        if not self.count > 1:
            new_mean = v[0]
        var_delta = (v - self.mean[None, ...]) * (v - new_mean[None, ...])
        self.var_sum = self.var_sum + var_delta.sum(0)
        self.mean = new_mean


# ---- agents/scripts/networks.py:66-110 ForwardGaussianPolicy -------------------------------------------------------------
def unpack_params(params, O, A, H1, H2):
    """Packed block of include/rexsim_agent.h -> dict of arrays."""
    p = np.asarray(params)
    pad4 = lambda n: (n + 3) & ~3
    npol = pad4(O * H1 + H1 + H1 * H2 + H2 + H2 * A + A + A)
    out, o = {}, 0
    for name, shape in (("pW1", (O, H1)), ("pb1", (H1,)), ("pW2", (H1, H2)), ("pb2", (H2,)), ("pW3", (H2, A)), ("pb3", (A,)), ("logstd", (A,))):
        n = int(np.prod(shape)); out[name] = p[o:o + n].reshape(shape); o += n
    o = npol
    for name, shape in (("vW1", (O, H1)), ("vb1", (H1,)), ("vW2", (H1, H2)), ("vb2", (H2,)), ("vW3", (H2, 1)), ("vb3", (1,))):
        n = int(np.prod(shape)); out[name] = p[o:o + n].reshape(shape); o += n
    return out


def pack_params(d, O, A, H1, H2):
    pad4 = lambda n: (n + 3) & ~3
    pol = np.concatenate([np.asarray(d[k], np.float32).reshape(-1) for k in ("pW1", "pb1", "pW2", "pb2", "pW3", "pb3", "logstd")])
    val = np.concatenate([np.asarray(d[k], np.float32).reshape(-1) for k in ("vW1", "vb1", "vW2", "vb2", "vW3", "vb3")])
    out = np.zeros(pad4(pol.size) + pad4(val.size), np.float32)
    out[:pol.size] = pol
    out[pad4(pol.size):pad4(pol.size) + val.size] = val
    return out


def forward_gaussian_policy(w, x, dtype=np.float64):
    """x: normalised observations [n][O] -> mean [n][A], logstd [A], value [n]   (fully_connected = x @ W + b, then act)."""
    x = np.asarray(x, dtype)
    W = {k: np.asarray(v, dtype) for k, v in w.items()}
    h = np.maximum(x @ W["pW1"] + W["pb1"], 0)
    h = np.maximum(h @ W["pW2"] + W["pb2"], 0)
    mean = np.tanh(h @ W["pW3"] + W["pb3"])
    g = np.maximum(x @ W["vW1"] + W["vb1"], 0)
    g = np.maximum(g @ W["vW2"] + W["vb2"], 0)
    value = (g @ W["vW3"] + W["vb3"])[:, 0]
    return mean, W["logstd"], value


# ---- sampling: the counter-based generator shared with the kernels (rexsim_kernel.cuh rand_u32) --------------------------
_M64 = (1 << 64) - 1


def rand_u32(seed, env, counter, slot):
    z = (seed + 0x9E3779B97F4A7C15 * (env + 1)) & _M64
    z ^= ((counter << 32) | slot) & _M64
    z = (z + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    z = z ^ (z >> 31)
    return (z >> 32) & 0xFFFFFFFF


def uniform_pair(seed, env, step, a):
    """The sampler's (u1, u2) of action a (rexsim_agent.cu head_outputs): (k + 1/2) / 2^23 for the top 23 bits k of a draw,
    which the kernel computes exactly in fp32."""
    return tuple(((rand_u32(seed, env, step, 2 * a + i) >> 9) + 0.5) / 8388608.0 for i in (0, 1))


def normal_noise(seed, env, step, a):
    u1, u2 = uniform_pair(seed, env, step, a)
    return math.sqrt(-2.0 * math.log(u1)) * math.cos(2.0 * math.pi * u2)


def perform(w, filt, observ, training, seed=0, step=0, env_offset=0):
    """PPOAlgorithm.perform (algorithm.py:105-135): action, mean, logprob, value."""
    x = filt.transform(observ)
    mean, logstd, value = forward_gaussian_policy(w, x)
    n, A = mean.shape
    z = np.zeros((n, A))
    if training:
        for e in range(n):
            for a in range(A):
                z[e, a] = normal_noise(seed, env_offset + e, step, a)
    action = mean + np.exp(logstd)[None, :] * z
    logprob = (-0.5 * z * z - logstd[None, :] - 0.5 * math.log(2 * math.pi)).sum(1)
    return action, mean, logprob, value


# ---- agents/ppo/utility.py:72-124 ------------------------------------------------------------------------------------------
def discounted_return(reward, length, discount):
    reward = np.asarray(reward, np.float64)
    E, L = reward.shape
    mask = (np.arange(L)[None, :] < np.asarray(length)[:, None]).astype(np.float64)
    out = np.zeros_like(reward)
    agg = np.zeros(E)
    for t in range(L - 1, -1, -1):
        agg = mask[:, t] * reward[:, t] + discount * agg
        out[:, t] = agg
    return out


def lambda_advantage(reward, value, length, discount):
    reward, value = np.asarray(reward, np.float64), np.asarray(value, np.float64)
    E, L = reward.shape
    mask = (np.arange(L)[None, :] < np.asarray(length)[:, None]).astype(np.float64)
    next_value = np.concatenate([value[:, 1:], np.zeros((E, 1))], 1)
    delta = reward + discount * next_value - value
    out = np.zeros_like(reward)
    agg = np.zeros(E)
    for t in range(L - 1, -1, -1):
        agg = mask[:, t] * delta[:, t] + discount * agg
        out[:, t] = agg
    return out


def gae_segments(reward, value, done, discount, lam):
    """time-major [T][N] (+ bootstrap row in value): see include/rexsim_agent.h rexagent_gae_segments."""
    reward, value = np.asarray(reward, np.float64), np.asarray(value, np.float64)
    T, n = reward.shape
    nd = 1.0 - np.asarray(done, np.float64)
    ret, adv = np.zeros((T, n)), np.zeros((T, n))
    r_next, a_next, v_next = value[T].copy(), np.zeros(n), value[T].copy()
    for t in range(T - 1, -1, -1):
        delta = reward[t] + discount * v_next * nd[t] - value[t]
        a_next = delta + discount * lam * nd[t] * a_next
        r_next = reward[t] + discount * nd[t] * r_next
        adv[t], ret[t] = a_next, r_next
        v_next = value[t]
    return ret, adv

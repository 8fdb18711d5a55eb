"""CPU ORACLE (test infrastructure, NOT the product path) for the reference's RecurrentGaussianPolicy and LinearGaussianPolicy
(rex_gym/agents/scripts/networks.py:113-159 and :21-63) and the per-environment state PPOAlgorithm keeps for them
(agents/ppo/algorithm.py:74, :90-135); fp64 numpy, beside oracle/agent_oracle.py whose filter, value network and sampling it
reuses.

Only tests/ may import this module.

PARITY STATUS: restated from documentation, not pinned to TensorFlow output.  The cell is tf.contrib.rnn.GRUBlockCell as the
TensorFlow 1.15 op documentation defines it:
    [r | u] = sigmoid([x, h] . w_ru + b_ru)     (r: the first G columns)
    c       = tanh([x, r * h] . w_c + b_c)
    h'      = u * h + (1 - u) * c
tensorflow==1.15 is not installable here, and no shipped checkpoint is recurrent (every config.yaml the reference ships names
ForwardGaussianPolicy), so no recorded output can pin it.  It is NOT torch.nn.GRUCell: that cell applies r after the hidden
matmul (n = tanh(W_in x + b_in + r * (W_hn h + b_hn))) and puts u's complement on the other term, so it is a different
function and is not used as a check (tests/test_recurrent_oracle.py shows a case where the two differ).
"""
import math

import numpy as np

from . import agent_oracle as AO


def _pad4(n):
    return (n + 3) & ~3


def gru_shapes(O, A, H1, G):
    """The policy block of include/rexsim_recurrent.h in its order: (key, shape)."""
    return (("pW1", (O, H1)), ("pb1", (H1,)), ("w_ru", (H1 + G, 2 * G)), ("b_ru", (2 * G,)), ("w_c", (H1 + G, G)), ("b_c", (G,)),
            ("pW3", (G, A)), ("pb3", (A,)), ("logstd", (A,)))


def linear_shapes(O, A):
    return (("pW", (O, A)), ("pb", (A,)), ("logstd", (A,)))


def pack_policy(w, shapes):
    flat = np.concatenate([np.asarray(w[k], np.float32).reshape(-1) for k, _ in shapes])
    out = np.zeros(_pad4(flat.size), np.float32)
    out[:flat.size] = flat
    return out


def unpack_policy(block, shapes):
    out, o = {}, 0
    for k, s in shapes:
        n = int(np.prod(s))
        out[k] = np.asarray(block)[o:o + n].reshape(s)
        o += n
    return out


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def gru_block_cell(x, h, w_ru, b_ru, w_c, b_c):
    """GRUBlockCell: x [n][I], h [n][G] -> h' [n][G] (the cell's output and new state), fp64."""
    x, h = np.asarray(x, np.float64), np.asarray(h, np.float64)
    G = h.shape[1]
    ru = sigmoid(np.concatenate([x, h], 1) @ np.asarray(w_ru, np.float64) + np.asarray(b_ru, np.float64))
    r, u = ru[:, :G], ru[:, G:]
    c = np.tanh(np.concatenate([x, r * h], 1) @ np.asarray(w_c, np.float64) + np.asarray(b_c, np.float64))
    return u * h + (1.0 - u) * c


def value_network(w, x):
    """ForwardGaussianPolicy's value MLP (agent_oracle.forward_gaussian_policy's value half)."""
    W = {k: np.asarray(w[k], np.float64) for k in ("vW1", "vb1", "vW2", "vb2", "vW3", "vb3")}
    g = np.maximum(np.asarray(x, np.float64) @ W["vW1"] + W["vb1"], 0)
    g = np.maximum(g @ W["vW2"] + W["vb2"], 0)
    return (g @ W["vW3"] + W["vb3"])[:, 0]


def recurrent_gaussian_policy(w, x, h):
    """networks.py:140-159: x normalised observations [n][O], h state [n][G] -> mean [n][A], logstd [A], value [n], h'."""
    W = {k: np.asarray(v, np.float64) for k, v in w.items()}
    a1 = np.maximum(np.asarray(x, np.float64) @ W["pW1"] + W["pb1"], 0)
    h2 = gru_block_cell(a1, h, W["w_ru"], W["b_ru"], W["w_c"], W["b_c"])
    return np.tanh(h2 @ W["pW3"] + W["pb3"]), W["logstd"], value_network(w, x), h2


def linear_gaussian_policy(w, x):
    """networks.py:48-63: mean = tanh(x . W + b), logstd, the value MLP."""
    W = {k: np.asarray(v, np.float64) for k, v in w.items()}
    x = np.asarray(x, np.float64)
    return np.tanh(x @ W["pW"] + W["pb"]), W["logstd"], value_network(w, x)


def perform(w, filt, observ, training, seed=0, step=0, env_offset=0, state=None, begin=None):
    """PPOAlgorithm.perform with a recurrent (state [n][G] given) or linear (state None) policy: action, mean, logprob, value and
    the new state.  Rows with begin set start from zero (begin_episode)."""
    x = filt.transform(observ)
    if state is None:
        mean, logstd, value = linear_gaussian_policy(w, x)
        h2 = None
    else:
        h = np.array(state, np.float64)
        if begin is not None:
            h[np.asarray(begin, bool)] = 0.0
        mean, logstd, value, h2 = recurrent_gaussian_policy(w, x, h)
    n, A = mean.shape
    z = np.zeros((n, A))
    if training:
        for e in range(n):
            for a in range(A):
                z[e, a] = AO.normal_noise(seed, env_offset + e, step, a)
    action = mean + np.exp(logstd)[None, :] * z
    logprob = (-0.5 * z * z - logstd[None, :] - 0.5 * math.log(2 * math.pi)).sum(1)
    return action, mean, logprob, value, h2

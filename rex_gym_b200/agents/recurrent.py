"""RecurrentGaussianPolicy and LinearGaussianPolicy on the GPU: the reference's two other policy cells
(rex_gym/agents/scripts/networks.py:113-159 and :21-63), fused with PPOAlgorithm.perform's observation filter and sampling
(agents/ppo/algorithm.py:105-135) like ForwardGaussianPolicy (csrc/rexsim_agent.cu, C ABI include/rexsim_recurrent.h).

Both keep ForwardGaussianPolicy's value network, observation and reward filters and noise step counter: they live in a
ForwardGaussianPolicy held by the network (its own policy block is unused).  The recurrent network also keeps
PPOAlgorithm's per-environment cell state (_last_state, algorithm.py:74): perform advances it, `begin` rows and
begin_episode() restart it from zero.  There is no CPU fallback."""
import ctypes as C

import numpy as np
import torch

from .. import _capi
from .networks import ForwardGaussianPolicy, check_observ

_VALUE_KEYS = ("vW1", "vb1", "vW2", "vb2", "vW3", "vb3")


def _glorot(rng, i, o):
    lim = np.sqrt(6.0 / (i + o))
    return rng.uniform(-lim, lim, (i, o)).astype(np.float32)


class _PolicyCell(object):
    """What both networks share: the handle, the parameter blocks, perform and the agent-side calls."""
    recurrent = False

    def __init__(self, observ_size, action_size, value_layers, kind, hidden1, cell, num_envs, init_logstd, init_mean_factor,
                 device, seed):
        self._ff = ForwardGaussianPolicy(observ_size, action_size, value_layers, value_layers, init_logstd, init_mean_factor,
                                         device, seed)
        ff = self._ff
        self._L, self.device, self._call = ff._L, ff.device, ff._call
        self.O, self.A, self.num_envs = ff.O, ff.A, int(num_envs)
        self.observ_filter, self.reward_filter = ff.observ_filter, ff.reward_filter
        self._rcfg = _capi.RexRnnConfig(kind, int(hidden1), int(cell), self.num_envs)
        self.n_policy = int(self._L.rexrnn_policy_floats(C.byref(ff._cfg), C.byref(self._rcfg)))
        h = C.c_void_p()
        self._call(self._L.rexrnn_create, ff._h, C.byref(self._rcfg), C.byref(h), stream=False)
        self._h = h
        self._state = None
        if kind == _capi.REXRNN_GRU:
            p = C.c_void_p()
            _capi.check(self._L.rexrnn_state_buffer(self._h, C.byref(p)))
            self._state = _capi.device_view(p.value, (self.num_envs, int(cell)), "<f4", self, self.device)

    # ---- parameters: the policy block of include/rexsim_recurrent.h, the value block of the ForwardGaussianPolicy ----------
    def _layout(self):
        o = 0
        for k, s in self._policy_shapes():
            yield k, s, o
            o += int(np.prod(s))

    def set_weights(self, w):
        block = np.zeros(self.n_policy, np.float32)
        for k, s, o in self._layout():
            a = np.asarray(w[k], np.float32)
            if a.shape != s:
                raise ValueError("weight %s has shape %s, expected %s" % (k, a.shape, s))
            block[o:o + a.size] = a.reshape(-1)
        self._call(self._L.rexrnn_set_params, self._h, block.ctypes.data, block.size, stream=False)
        ffw = self._ff.get_weights()
        ffw.update({k: w[k] for k in _VALUE_KEYS})
        self._ff.set_weights(ffw)

    def get_weights(self):
        block = np.zeros(self.n_policy, np.float32)
        self._call(self._L.rexrnn_get_params, self._h, block.ctypes.data, block.size, stream=False)
        w = {k: block[o:o + int(np.prod(s))].reshape(s).copy() for k, s, o in self._layout()}
        ffw = self._ff.get_weights()
        w.update({k: ffw[k] for k in _VALUE_KEYS})
        return w

    def set_filters(self, *args, **kwargs):
        self._ff.set_filters(*args, **kwargs)

    def get_filters(self):
        return self._ff.get_filters()

    # ---- PPOAlgorithm.begin_episode / perform / experience ------------------------------------------------------------
    def begin_episode(self, indices):
        """algorithm.begin_episode (algorithm.py:90-103): the cell state of these environments restarts from zero."""
        if self._state is not None:
            self._state[torch.as_tensor(indices, device=self.device, dtype=torch.long)] = 0.0

    def perform(self, observ, training=False, seed=0, step=0, env_offset=0, out=None, observ_copy=None, begin=None):
        """ForwardGaussianPolicy.perform for the first n <= num_envs environments, plus `begin` (CUDA uint8 or bool [n], or
        None): rows with begin set start from the zero state.  A call that asks for an action, mean or log-prob advances the
        state of rows 0..n-1; a call for the value alone leaves it untouched."""
        n = check_observ(observ, self.O)
        if out is None:
            dev = observ.device
            out = dict(action=torch.empty((n, self.A), device=dev), mean=torch.empty((n, self.A), device=dev),
                       logprob=torch.empty((n,), device=dev), value=torch.empty((n,), device=dev))
        if begin is not None:
            if not (isinstance(begin, torch.Tensor) and begin.is_cuda and begin.dtype in (torch.uint8, torch.bool)
                    and begin.shape == (n,) and begin.is_contiguous()):
                raise ValueError("begin must be a contiguous CUDA uint8 or bool tensor of shape (%d,)" % n)
            begin = begin.view(torch.uint8)
        ptr = lambda t: None if t is None else t.data_ptr()
        self._call(self._L.rexrnn_perform, self._h, observ.data_ptr(), ptr(begin), n, int(bool(training)), int(seed), int(step),
                   int(env_offset), ptr(out.get("action")), ptr(out.get("mean")), ptr(out.get("logprob")), ptr(out.get("value")),
                   ptr(observ_copy))
        return out

    def value(self, observ, out=None):
        """The value block alone (the ForwardGaussianPolicy's) on observ [n][O], any n: the cell state is not touched."""
        return self._ff.value(observ, out)

    def experience(self, observ, reward, group=None):
        self._ff.experience(observ, reward, group)

    def transform_reward(self, reward, out=None):
        return self._ff.transform_reward(reward, out)

    def state_dict(self):
        """Filter statistics, counters and the cell state (device tensors): with get_weights() the complete agent state."""
        sd = self._ff.state_dict()
        if self._state is not None:
            sd["hidden"] = self._state.clone()
        return sd

    def load_state_dict(self, sd):
        self._ff.load_state_dict(sd)
        if self._state is not None:
            self._state.copy_(sd["hidden"])

    @property
    def launch_count(self):
        return self._ff.launch_count + int(self._L.rexrnn_launch_count(self._h))

    def close(self):
        if self._h is not None:
            torch.cuda.synchronize(self.device)
            self._L.rexrnn_destroy(self._h)
            self._h = None
        self._ff.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class RecurrentGaussianPolicy(_PolicyCell):
    """networks.py:113-159: normalised observation -> dense policy_layers[0] ReLU -> GRUBlockCell(cell_size) -> dense tanh mean,
    free logstd; the value network of ForwardGaussianPolicy.  policy_layers must have two entries, as the reference's configs do:
    the reference builds the dense layers of policy_layers[:-1] and a cell of 100 units whatever policy_layers[-1] says
    (networks.py:132), so cell_size defaults to 100.  Weights (TF variables under network/rnn/policy/): pW1, pb1
    (fully_connected), w_ru, b_ru, w_c, b_c (gru_cell), pW3, pb3 (fully_connected_1), logstd; vW1 .. vb3 as
    ForwardGaussianPolicy.  num_envs: rows of the cell state."""
    recurrent = True

    def __init__(self, observ_size, action_size, policy_layers=(200, 100), value_layers=(200, 100), init_logstd=-1.0,
                 init_mean_factor=0.1, device="cuda:0", seed=0, num_envs=1, cell_size=100):
        if len(policy_layers) != 2:
            raise ValueError("policy_layers must have two sizes: the dense layer and the (unused) last entry")
        self.H1, self.G = int(policy_layers[0]), int(cell_size)
        super().__init__(observ_size, action_size, value_layers, _capi.REXRNN_GRU, self.H1, self.G, num_envs, init_logstd,
                         init_mean_factor, device, seed)
        # TF defaults: glorot-uniform kernels (fully_connected and GRUBlockCell), zero biases but b_ru = 1 (gru_ops.py),
        # variance_scaling(factor=init_mean_factor) on the mean layer, logstd = init_logstd
        rng = np.random.default_rng([seed, 1])
        O, A, H1, G = self.O, self.A, self.H1, self.G
        w = {k: v for k, v in self._ff.get_weights().items() if k in _VALUE_KEYS}
        w.update(pW1=_glorot(rng, O, H1), pb1=np.zeros(H1), w_ru=_glorot(rng, H1 + G, 2 * G), b_ru=np.ones(2 * G),
                 w_c=_glorot(rng, H1 + G, G), b_c=np.zeros(G),
                 pW3=(rng.standard_normal((G, A)) * np.sqrt(init_mean_factor / G)).astype(np.float32), pb3=np.zeros(A),
                 logstd=np.full(A, init_logstd))
        self.set_weights(w)

    def _policy_shapes(self):
        O, A, H1, G = self.O, self.A, self.H1, self.G
        return (("pW1", (O, H1)), ("pb1", (H1,)), ("w_ru", (H1 + G, 2 * G)), ("b_ru", (2 * G,)), ("w_c", (H1 + G, G)),
                ("b_c", (G,)), ("pW3", (G, A)), ("pb3", (A,)), ("logstd", (A,)))


class LinearGaussianPolicy(_PolicyCell):
    """networks.py:21-63: mean = tanh(normalised observation . pW + pb), free logstd; the value network of
    ForwardGaussianPolicy.  The reference ignores policy_layers here; it is accepted for the same signature.  No state: `begin`
    and begin_episode() change nothing."""

    def __init__(self, observ_size, action_size, policy_layers=(200, 100), value_layers=(200, 100), init_logstd=-1.0,
                 init_mean_factor=0.1, device="cuda:0", seed=0, num_envs=1):
        super().__init__(observ_size, action_size, value_layers, _capi.REXRNN_LINEAR, 0, 0, num_envs, init_logstd,
                         init_mean_factor, device, seed)
        rng = np.random.default_rng([seed, 1])
        O, A = self.O, self.A
        w = {k: v for k, v in self._ff.get_weights().items() if k in _VALUE_KEYS}
        w.update(pW=(rng.standard_normal((O, A)) * np.sqrt(init_mean_factor / O)).astype(np.float32), pb=np.zeros(A),
                 logstd=np.full(A, init_logstd))
        self.set_weights(w)

    def _policy_shapes(self):
        return (("pW", (self.O, self.A)), ("pb", (self.A,)), ("logstd", (self.A,)))

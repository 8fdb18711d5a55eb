"""ForwardGaussianPolicy on the GPU: rex_gym/agents/scripts/networks.py:66-110 (policy MLP -> tanh mean, free log-stddev
vector, value MLP) fused with PPOAlgorithm.perform's observation filter and sampling (agents/ppo/algorithm.py:105-135) in
one CUDA kernel (csrc/rexsim_agent.cu, C ABI include/rexsim_agent.h).  There is no CPU fallback."""
import ctypes as C
import functools
import os

import numpy as np
import torch

from .. import _capi
from . import tf_checkpoint as tfc
from .normalize import StreamingNormalize

_TF = "network/rnn/"
POLICY, VALUE = 0, 1
# the parameter block in its order (include/rexsim_agent.h): key, block, TF variable name under _TF, shape from (O, A, H1, H2)
_PARAMS = (
    ("pW1", POLICY, "policy/fully_connected/weights", lambda O, A, H1, H2: (O, H1)),
    ("pb1", POLICY, "policy/fully_connected/biases", lambda O, A, H1, H2: (H1,)),
    ("pW2", POLICY, "policy/fully_connected_1/weights", lambda O, A, H1, H2: (H1, H2)),
    ("pb2", POLICY, "policy/fully_connected_1/biases", lambda O, A, H1, H2: (H2,)),
    ("pW3", POLICY, "policy/fully_connected_2/weights", lambda O, A, H1, H2: (H2, A)),
    ("pb3", POLICY, "policy/fully_connected_2/biases", lambda O, A, H1, H2: (A,)),
    ("logstd", POLICY, "policy/logstd", lambda O, A, H1, H2: (A,)),
    ("vW1", VALUE, "value/fully_connected/weights", lambda O, A, H1, H2: (O, H1)),
    ("vb1", VALUE, "value/fully_connected/biases", lambda O, A, H1, H2: (H1,)),
    ("vW2", VALUE, "value/fully_connected_1/weights", lambda O, A, H1, H2: (H1, H2)),
    ("vb2", VALUE, "value/fully_connected_1/biases", lambda O, A, H1, H2: (H2,)),
    ("vW3", VALUE, "value/fully_connected_2/weights", lambda O, A, H1, H2: (H2, 1)),
    ("vb3", VALUE, "value/fully_connected_2/biases", lambda O, A, H1, H2: (1,)),
)


class ForwardGaussianPolicy(object):
    """policy_layers / value_layers must both be (H1, H2) (every config the reference ships uses (200, 100))."""

    def __init__(self, observ_size, action_size, policy_layers=(200, 100), value_layers=(200, 100), init_logstd=-1.0,
                 init_mean_factor=0.1, device="cuda:0", seed=0, tensor_cores=False):
        if tuple(policy_layers) != tuple(value_layers) or len(policy_layers) != 2:
            raise ValueError("policy_layers and value_layers must be the same two sizes")
        if not torch.cuda.is_available():
            raise RuntimeError("rex_gym_b200 needs a CUDA device: there is no CPU fallback")
        self._L = _capi.load()
        self.device = torch.device(device)
        self.O, self.A, (self.H1, self.H2) = int(observ_size), int(action_size), [int(x) for x in policy_layers]
        c = _capi.RexAgentConfig(self.O, self.A, self.H1, self.H2, 5.0, 10.0)       # clips: algorithm.py:49-58
        self._cfg = c
        self.n_policy = int(self._L.rexagent_policy_floats(C.byref(c)))
        self.n_value = int(self._L.rexagent_value_floats(C.byref(c)))
        index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        # every library call: on this network's device and torch's current stream there, a non-zero status raised
        self._call = functools.partial(_capi.call, index)
        h = C.c_void_p()
        self._call(self._L.rexagent_create, C.byref(c), C.byref(h), stream=False)
        self._h = h
        # tensor_cores=True: layer 2 (97 % of the flops) as wgmma tf32 with fp32 accumulation in registers; operands keep 11
        # significant bits (error vs the fp32 kernel: DESIGN.md section 5).  False (default): fp32 on the CUDA cores.
        self.tensor_cores = bool(tensor_cores)
        if self.tensor_cores:
            self._call(self._L.rexagent_set_precision, self._h, 1, stream=False)
        pf, pc = C.c_void_p(), C.c_void_p()
        _capi.check(self._L.rexagent_state_buffers(self._h, C.byref(pf), C.byref(pc)))
        self._filt = _capi.device_view(pf.value, (2 * self.O + 2,), "<f4", self, self.device)
        self._cnt = _capi.device_view(pc.value, (4,), "<i8", self, self.device)                    # int64: counts pass 2^31
        self.observ_filter = StreamingNormalize(self, "observ")
        self.reward_filter = StreamingNormalize(self, "reward")
        # initialisers of networks.py:18-19 and tf.contrib.layers defaults: xavier-uniform hidden layers, zero biases,
        # variance_scaling(factor=init_mean_factor) on the mean layer, logstd = init_logstd
        rng = np.random.default_rng(seed)

        def xavier(i, o):
            lim = np.sqrt(6.0 / (i + o))
            return rng.uniform(-lim, lim, (i, o)).astype(np.float32)
        O, A, H1, H2 = self.O, self.A, self.H1, self.H2
        self.set_weights(dict(
            pW1=xavier(O, H1), pb1=np.zeros(H1), pW2=xavier(H1, H2), pb2=np.zeros(H2),
            pW3=(rng.standard_normal((H2, A)) * np.sqrt(init_mean_factor / H2)).astype(np.float32), pb3=np.zeros(A),
            logstd=np.full(A, init_logstd), vW1=xavier(O, H1), vb1=np.zeros(H1), vW2=xavier(H1, H2), vb2=np.zeros(H2),
            vW3=xavier(H2, 1), vb3=np.zeros(1)))

    # ---- parameters ----------------------------------------------------------------------------------------------
    def _layout(self):
        """(key, shape, offset) of every parameter in the block: the policy's from 0, the value network's from n_policy."""
        o = [0, self.n_policy]
        for k, block, _, shape in _PARAMS:
            s = shape(self.O, self.A, self.H1, self.H2)
            yield k, s, o[block]
            o[block] += int(np.prod(s))

    def set_weights(self, w):
        block = np.zeros(self.n_policy + self.n_value, np.float32)
        for k, s, o in self._layout():
            a = np.asarray(w[k], np.float32)
            if a.shape != s:
                raise ValueError("weight %s has shape %s, expected %s" % (k, a.shape, s))
            block[o:o + a.size] = a.reshape(-1)
        self._call(self._L.rexagent_set_params, self._h, block.ctypes.data, block.size, stream=False)

    def get_weights(self):
        block = np.zeros(self.n_policy + self.n_value, np.float32)
        self._call(self._L.rexagent_get_params, self._h, block.ctypes.data, block.size, stream=False)
        return {k: block[o:o + int(np.prod(s))].reshape(s).copy() for k, s, o in self._layout()}

    @classmethod
    def from_tf_checkpoint(cls, directory_or_prefix, device="cuda:0"):
        """Load one of the policies the reference ships (rex_gym/policies/<task>/<signal>/model.ckpt-N.*): network weights
        and both streaming-normaliser states, exactly what PolicyPlayer restores (playground/policy_player.py:35-41)."""
        w, filters = read_tf_policy(directory_or_prefix)
        O, H1 = w["pW1"].shape
        H2, A = w["pW3"].shape
        net = cls(O, A, (H1, H2), (H1, H2), device=device)
        net.set_weights(w)
        net.set_filters(*filters)
        return net

    def set_filters(self, observ_count, observ_mean, observ_var_sum, reward_count=0, reward_mean=0.0, reward_var_sum=0.0):
        m = np.ascontiguousarray(observ_mean, np.float32); v = np.ascontiguousarray(observ_var_sum, np.float32)
        if m.shape != (self.O,) or v.shape != (self.O,):
            raise ValueError("filter statistics must have shape (%d,)" % self.O)
        self._call(self._L.rexagent_set_filters, self._h, int(observ_count), m.ctypes.data, v.ctypes.data, int(reward_count),
                   float(reward_mean), float(reward_var_sum), stream=False)

    def get_filters(self):
        counts = np.zeros(2, np.int64); m = np.zeros(self.O, np.float32); v = np.zeros(self.O, np.float32); r = np.zeros(2, np.float32)
        self._call(self._L.rexagent_get_filters, self._h, counts.ctypes.data, m.ctypes.data, v.ctypes.data, r.ctypes.data, stream=False)
        return dict(observ_count=int(counts[0]), observ_mean=m, observ_var_sum=v, reward_count=int(counts[1]),
                    reward_mean=float(r[0]), reward_var_sum=float(r[1]))

    # ---- PPOAlgorithm.perform / experience -----------------------------------------------------------------------------
    def _stream(self):
        return _capi.stream_ptr(self.device)

    def perform(self, observ, training=False, seed=0, step=0, env_offset=0, out=None, observ_copy=None):
        """observ: CUDA float32 [n][O].  Returns dict(action [n][A], mean [n][A], logprob [n], value [n]) of CUDA tensors
        (pass `out` to reuse buffers, e.g. slices of a rollout)."""
        n = check_observ(observ, self.O)
        if out is None:
            dev = observ.device
            out = dict(action=torch.empty((n, self.A), device=dev), mean=torch.empty((n, self.A), device=dev),
                       logprob=torch.empty((n,), device=dev), value=torch.empty((n,), device=dev))
        ptr = lambda t: None if t is None else t.data_ptr()
        self._call(self._L.rexagent_perform, self._h, observ.data_ptr(), n, int(bool(training)), int(seed), int(step), int(env_offset),
                   ptr(out.get("action")), ptr(out.get("mean")), ptr(out.get("logprob")), ptr(out.get("value")), ptr(observ_copy))
        return out

    def value(self, observ, out=None):
        """The value network alone on observ [n][O] (filtered as perform filters it): CUDA float32 [n]."""
        out = torch.empty((observ.shape[0],), dtype=torch.float32, device=observ.device) if out is None else out
        return self.perform(observ, out=dict(value=out))["value"]

    def experience(self, observ, reward, group=None):
        """PPOAlgorithm._define_experience's filter updates (algorithm.py:157-161) for one batch; advances the device-side
        step counter that keys the next perform's noise.  With torch.distributed initialised (env-sharded rollout, one rank per
        GPU) the batch statistics are summed over the ranks first -- one all-reduce of 2*(O+1) floats, the only exchange
        step of this path -- so every rank keeps the filter state of the whole batch."""
        import torch.distributed as dist
        n = observ.shape[0]
        sharded = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
        if not sharded:
            self._call(self._L.rexagent_experience, self._h, observ.data_ptr(), reward.data_ptr(), n)
            return
        if getattr(self, "_sums", None) is None:
            self._sums = torch.zeros((self.O + 1, 2), dtype=torch.float32, device=self.device)
        self._call(self._L.rexagent_experience_partial, self._h, observ.data_ptr(), reward.data_ptr(), n, self._sums.data_ptr())
        with torch.cuda.device(self.device):
            dist.all_reduce(self._sums, op=dist.ReduceOp.SUM, group=group)
        self._call(self._L.rexagent_experience_finalize, self._h, self._sums.data_ptr(), n * dist.get_world_size(group),
                   observ.data_ptr(), reward.data_ptr())

    def transform_reward(self, reward, out=None):
        out = torch.empty_like(reward) if out is None else out
        self._call(self._L.rexagent_transform_reward, self._h, reward.data_ptr(), reward.numel(), out.data_ptr())
        return out

    def state_dict(self):
        """Filter statistics and counters (device tensors): with get_weights() the complete agent state."""
        return {"filters": self._filt.clone(), "counters": self._cnt.clone()}

    def load_state_dict(self, sd):
        self._filt.copy_(sd["filters"]); self._cnt.copy_(sd["counters"])

    @property
    def launch_count(self):
        return int(self._L.rexagent_launch_count(self._h))

    def close(self):
        if self._h is not None:
            torch.cuda.synchronize(self.device)
            self._L.rexagent_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def check_observ(observ, O):
    """The batch size of a perform call's observations; raises unless they are a contiguous CUDA float32 [n][O] tensor."""
    if not (isinstance(observ, torch.Tensor) and observ.is_cuda and observ.dtype == torch.float32 and observ.is_contiguous()):
        raise ValueError("observ must be a contiguous CUDA float32 tensor")
    if observ.dim() != 2 or observ.shape[1] != O:
        raise ValueError("Invalid observation shape %s, expected (n, %d)" % (tuple(observ.shape), O))
    return observ.shape[0]


def read_tf_policy(directory_or_prefix):
    """(weights dict, (observ_count, observ_mean, observ_var_sum, reward_count, reward_mean, reward_var_sum)) from a TF checkpoint."""
    prefix = tfc.latest_checkpoint(directory_or_prefix) if os.path.isdir(directory_or_prefix) else directory_or_prefix
    names = [_TF + n for _, _, n, _ in _PARAMS] + ["normalize_observ/Variable", "normalize_observ/Variable_1", "normalize_observ/Variable_2",
                                               "normalize_reward/Variable", "normalize_reward/Variable_1", "normalize_reward/Variable_2"]
    v = tfc.load_variables(prefix, names)
    missing = [n for n in names if n not in v]
    if missing:
        raise ValueError("checkpoint %s is not a ForwardGaussianPolicy PPO checkpoint (missing %s)" % (prefix, missing[:3]))
    w = {k: v[_TF + n] for k, _, n, _ in _PARAMS}
    filt = (int(v["normalize_observ/Variable"]), v["normalize_observ/Variable_1"], v["normalize_observ/Variable_2"],
            int(v["normalize_reward/Variable"]), float(v["normalize_reward/Variable_1"]), float(v["normalize_reward/Variable_2"]))
    return w, filt

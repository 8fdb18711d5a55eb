"""discounted_return / lambda_advantage (rex_gym/agents/ppo/utility.py:72-82,112-124) as CUDA scans; tensors stay on
the device.  Rows are episodes ([E][L] like the reference's EpisodeMemory) in any strided layout -- pass a transposed view of
a time-major buffer and the kernel reads it coalesced."""
import torch

from .. import _capi


def _check(t, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.dim() == 2):
        raise ValueError("%s must be a 2-D CUDA float32 tensor" % name)


def discounted_return(reward, length, discount):
    _check(reward, "reward")
    E, L = reward.shape
    length = length.to(device=reward.device, dtype=torch.int32).contiguous()
    out = torch.empty_strided(reward.shape, reward.stride(), dtype=torch.float32, device=reward.device)
    _capi.call(reward.device.index, _capi.load().rexagent_discounted_return, reward.data_ptr(), length.data_ptr(), E, L,
               reward.stride(0), reward.stride(1), float(discount), out.data_ptr())
    return out


def lambda_advantage(reward, value, length, discount):
    _check(reward, "reward"); _check(value, "value")
    if value.shape != reward.shape or value.stride() != reward.stride():
        raise ValueError("value must have the shape and strides of reward")
    E, L = reward.shape
    length = length.to(device=reward.device, dtype=torch.int32).contiguous()
    out = torch.empty_strided(reward.shape, reward.stride(), dtype=torch.float32, device=reward.device)
    _capi.call(reward.device.index, _capi.load().rexagent_lambda_advantage, reward.data_ptr(), value.data_ptr(), length.data_ptr(),
               E, L, reward.stride(0), reward.stride(1), float(discount), out.data_ptr())
    return out


def gae_segments(reward, value, done, discount, lam=1.0):
    """Time-major rollout of an auto-resetting batch: reward, done [T][N], value [T+1][N] -> (return, advantage) [T][N]."""
    T, n = reward.shape
    if tuple(value.shape) != (T + 1, n) or tuple(done.shape) != (T, n):
        raise ValueError("value must be [T+1][N] and done [T][N]")
    reward, value = reward.contiguous(), value.contiguous()
    d8 = done.contiguous().view(torch.uint8) if done.dtype == torch.bool else done.to(torch.uint8).contiguous()
    ret, adv = torch.empty_like(reward), torch.empty_like(reward)
    _capi.call(reward.device.index, _capi.load().rexagent_gae_segments, reward.data_ptr(), value.data_ptr(), d8.data_ptr(), T, n,
               float(discount), float(lam), ret.data_ptr(), adv.data_ptr())
    return ret, adv

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


def gae_segments(reward, value, done, discount, lam=1.0, truncated=None, final_value=None):
    """Time-major rollout of an auto-resetting batch: reward, done [T][N], value [T+1][N] -> (return, advantage) [T][N].
    truncated [T][N] (bool or uint8) and final_value [T][N], both or neither: a done step that is truncated (cut by the time
    limit) bootstraps from final_value, the value of its final observation, instead of ending at value 0
    (rexsim_gae_segments_bootstrap); every other step is computed bit for bit as without them."""
    T, n = reward.shape
    if tuple(value.shape) != (T + 1, n) or tuple(done.shape) != (T, n):
        raise ValueError("value must be [T+1][N] and done [T][N]")
    if (truncated is None) != (final_value is None):
        raise ValueError("truncated and final_value go together")
    if truncated is not None and (tuple(truncated.shape) != (T, n) or tuple(final_value.shape) != (T, n)):
        raise ValueError("truncated and final_value must be [T][N]")
    reward, value = reward.contiguous(), value.contiguous()
    u8 = lambda t: t.contiguous().view(torch.uint8) if t.dtype == torch.bool else t.to(torch.uint8).contiguous()
    d8 = u8(done)
    ret, adv = torch.empty_like(reward), torch.empty_like(reward)
    L = _capi.load()
    if truncated is None:
        _capi.call(reward.device.index, L.rexagent_gae_segments, reward.data_ptr(), value.data_ptr(), d8.data_ptr(), T, n,
                   float(discount), float(lam), ret.data_ptr(), adv.data_ptr())
    else:
        tr8, fv = u8(truncated), final_value.to(torch.float32).contiguous()
        _capi.call(reward.device.index, L.rexsim_gae_segments_bootstrap, reward.data_ptr(), value.data_ptr(), d8.data_ptr(),
                   tr8.data_ptr(), fv.data_ptr(), T, n, float(discount), float(lam), ret.data_ptr(), adv.data_ptr())
    return ret, adv

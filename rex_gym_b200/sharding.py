"""Env sharding across the GPUs of one box (SURVEY.md section 8(e)).

Environments are independent, so each rank owns a contiguous block of global env ids and steps it with
no data-path collective.  Reset draws key on the GLOBAL env id (RexSimConfig.env_offset), so a sharded run
produces exactly the trajectories of the single-GPU run.  The one optional collective is an all-gather
of the packed per-rank outputs [n, O + 2] = (obs | reward | done) for a learner that wants the whole batch on
every rank; it is a single NCCL call on the step stream (torch.distributed, backend nccl on GPUs, gloo in the
CPU tests).  The other is an all-reduce of the four episode totals (episode_summary) when the summary is logged."""
import torch
import torch.distributed as dist


def shard_range(global_envs, rank, world):
    """Contiguous partition of [0, global_envs): (offset, count) of `rank`."""
    if global_envs % world:
        raise ValueError("global_envs must be divisible by the number of ranks")
    n = global_envs // world
    return rank * n, n


def pack_outputs(obs, reward, done):
    """[n, O] f32, [n] f32, [n] bool/u8 -> [n, O + 2] f32 (one message per rank)."""
    return torch.cat([obs, reward.reshape(-1, 1).to(obs.dtype), done.reshape(-1, 1).to(obs.dtype)], dim=1).contiguous()


def unpack_outputs(packed):
    return packed[:, :-2], packed[:, -2], packed[:, -1] > 0.5


def all_gather_outputs(obs, reward, done, group=None):
    """One all-gather of the packed outputs; returns (obs_all [G*n, O], reward_all, done_all) on every rank."""
    packed = pack_outputs(obs, reward, done)
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return unpack_outputs(packed)
    out = torch.empty((world * packed.shape[0], packed.shape[1]), dtype=packed.dtype, device=packed.device)
    dist.all_gather_into_tensor(out, packed, group=group)
    return unpack_outputs(out)


def episode_summary(env, group=None, clear=True):
    """simulate()'s episode summary over every rank's shard: one all-reduce (sum) of the shards' episode totals, then the
    means of the whole batch on every rank (BatchedRexEnv.episode_summary of a single-GPU run)."""
    from .envs.batched_env import summarize_episodes
    totals = env.episode_totals(clear).clone()
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(totals, op=dist.ReduceOp.SUM, group=group)
    return summarize_episodes(totals)


def make_sharded_env(global_envs, rank=None, world=None, **kwargs):
    """BatchedRexEnv for this rank's block of a `global_envs`-sized batch."""
    from .envs.batched_env import BatchedRexEnv
    if rank is None:
        rank = dist.get_rank() if dist.is_initialized() else 0
    if world is None:
        world = dist.get_world_size() if dist.is_initialized() else 1
    from .envs.batched_env import PER_ENV_KEYWORDS, is_per_env
    off, n = shard_range(global_envs, rank, world)
    # per-env constructor values of the whole batch: this rank's slice
    for k in PER_ENV_KEYWORDS:
        if k in kwargs and is_per_env(kwargs[k]) and len(kwargs[k]) == global_envs:
            kwargs[k] = kwargs[k][off:off + n]
    return BatchedRexEnv(num_envs=n, env_offset=off, **kwargs)

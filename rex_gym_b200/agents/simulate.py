"""The rollout loop of rex_gym/agents/tools/simulate.py:57-123 on the device: per control step

    prevob -> PPOAlgorithm.perform (filter + policy + value + sample)   one kernel   (csrc/rexsim_agent.cu)
           -> BatchEnv.step (RexGymEnv.step for every env)              one kernel   (csrc/rexsim_kernel.cu)
           -> PPOAlgorithm.experience (filter updates) + memory append  one kernel; the "append" is the kernels writing
                                                                        straight into the [T][N] rollout buffers

Environments that finish are restarted inside the step kernel (auto_reset), which is what simulate() does at the top of
the next iteration (`begin_episode`, :117-120): the observation stored after a `done` is the first one of the new episode.
A recurrent network (RecurrentGaussianPolicy) gets the matching episode-start mask with every perform: all ones after
reset(), else the `done` row of the previous control step -- for the first step of a collect, the last row of the previous
one, kept in a buffer the captured graph owns.
The whole T-step loop is captured once into a CUDA graph and replayed: no host round trip per step (SURVEY.md 8(f) row 1).

With final_observation=True the step kernel also writes, into two more [T][N] buffers of the graph, what the auto-reset would
lose: the final observation of every env that ended (the `nextob` simulate() hands to algo.experience, simulate.py:67-75) and
its time-limit byte (gym TimeLimit's 'TimeLimit.truncated').  returns_and_advantages(bootstrap_truncated=True) then bootstraps
the episodes the time limit cut from the value of their final observation instead of treating them as terminal.
"""
import torch

from . import utility


class Rollout(object):
    def __init__(self, env, network, horizon, seed=0, training=True, use_graph=True, final_observation=False):
        if not getattr(env._cfg, "auto_reset", 0):
            raise ValueError("Rollout needs an env created with auto_reset=True")
        if network.O != env.obs_dim or network.A != env.action_dim:
            raise ValueError("network (%d -> %d) does not fit the env (%d -> %d)" % (network.O, network.A, env.obs_dim, env.action_dim))
        if getattr(network, "recurrent", False) and network.num_envs < env.num_envs:
            raise ValueError("the network keeps cell state for %d envs, the env has %d" % (network.num_envs, env.num_envs))
        self.env, self.net, self.T, self.seed, self.training = env, network, int(horizon), int(seed), bool(training)
        N, O, A, T, dev = env.num_envs, env.obs_dim, env.action_dim, self.T, env.device
        f32 = dict(dtype=torch.float32, device=dev)
        self.observ = torch.zeros((T, N, O), **f32)
        self.action = torch.zeros((T, N, A), **f32)
        self.mean = torch.zeros((T, N, A), **f32)
        self.logprob = torch.zeros((T, N), **f32)
        self.value = torch.zeros((T + 1, N), **f32)
        self.reward = torch.zeros((T, N), **f32)
        self.done = torch.zeros((T, N), dtype=torch.uint8, device=dev)
        self._cur = torch.zeros((N, O), **f32)             # observation the next action is computed from
        self.final_observ = self.limit = self.truncated = None
        if final_observation:
            self.final_observ = torch.zeros((T, N, O), **f32)                     # valid where done
            self.limit = torch.zeros((T, N), dtype=torch.uint8, device=dev)       # step kernel's time-limit bytes
            self.truncated = torch.zeros((T, N), dtype=torch.bool, device=dev)    # limit == 1: cut by the time limit alone
        self._recurrent = bool(getattr(network, "recurrent", False))
        self._begin = torch.ones((N,), dtype=torch.uint8, device=dev) if self._recurrent else None    # episode starts of step 0
        self._graph = None
        import torch.distributed as dist
        if use_graph and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            use_graph = False      # env-sharded: the per-step filter all-reduce runs through c10d; the plain loop is used
        self._use_graph = use_graph
        self.reset()

    def reset(self):
        """simulate(reset=True): restart every environment."""
        idx = torch.arange(self.env.num_envs, device=self.env.device, dtype=torch.int32)
        self._cur.copy_(self.env.reset(idx))
        if self._recurrent:
            self._begin.fill_(1)

    def _loop(self):
        env, net, T = self.env, self.net, self.T
        for t in range(T):
            step = dict(training=self.training, seed=self.seed, step=0, env_offset=env._cfg.env_offset,
                        out=dict(action=self.action[t], mean=self.mean[t], logprob=self.logprob[t], value=self.value[t]),
                        observ_copy=self.observ[t])
            if self._recurrent:
                step["begin"] = self._begin if t == 0 else self.done[t - 1]
            net.perform(self._cur, **step)
            if self.final_observ is None:
                env.step_into(self.action[t], self._cur, self.reward[t], self.done[t])
            else:
                env.step_into(self.action[t], self._cur, self.reward[t], self.done[t], self.final_observ[t], self.limit[t])
            if self.training:
                net.experience(self.observ[t], self.reward[t])
        net.perform(self._cur, training=False, out=dict(value=self.value[T]))       # bootstrap value of the last observation
        if self.limit is not None:
            torch.eq(self.limit, 1, out=self.truncated)
        if self._recurrent:
            self._begin.copy_(self.done[T - 1])

    def collect(self):
        """Run T control steps for every env; returns views of the rollout buffers (valid until the next collect)."""
        if not self._use_graph:
            self._loop()
        else:
            if self._graph is None:
                torch.cuda.synchronize(self.env.device)
                side = torch.cuda.Stream(device=self.env.device)
                side.wait_stream(torch.cuda.current_stream(self.env.device))
                # warm-up outside capture (lazy kernel loading must not happen while capturing); the warm-up advances the
                # environments and the filters, so everything is snapshotted first and put back afterwards
                snap = (self.env.state_dict(), self.net.state_dict(), self._cur.clone(),
                        None if self._begin is None else self._begin.clone())
                with torch.cuda.stream(side):
                    self._loop()
                torch.cuda.current_stream(self.env.device).wait_stream(side)
                torch.cuda.synchronize(self.env.device)
                self.env.load_state_dict(snap[0]); self.net.load_state_dict(snap[1]); self._cur.copy_(snap[2])
                if self._begin is not None:
                    self._begin.copy_(snap[3])
                torch.cuda.synchronize(self.env.device)
                self._graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self._graph):
                    self._loop()
            self._graph.replay()
        out = dict(observ=self.observ, action=self.action, mean=self.mean, logprob=self.logprob, value=self.value,
                   reward=self.reward, done=self.done.view(torch.bool))
        if self.final_observ is not None:
            out.update(final_observ=self.final_observ, truncated=self.truncated)
        return out

    def summary(self, clear=True):
        """simulate()'s mean_score / mean_length (simulate.py:95-106) over the episodes that ended since the last clear: the step
        kernel keeps the bookkeeping of an env created with episode_statistics=True, inside the captured graph as well
        (BatchedRexEnv.episode_summary)."""
        return self.env.episode_summary(clear)

    def returns_and_advantages(self, discount, lam=1.0, bootstrap_truncated=False):
        """Done-aware discounted return and GAE over the last rollout (utility.gae_segments).  bootstrap_truncated=True (needs
        final_observation=True) bootstraps the steps the time limit cut from the value of their final observation: the value
        network runs once, value only, on those rows (one host sync for their count).  Off by default, as in the reference,
        whose PPO has no final observation to bootstrap from."""
        if not bootstrap_truncated:
            return utility.gae_segments(self.reward, self.value, self.done, discount, lam)
        if self.final_observ is None:
            raise ValueError("bootstrap_truncated needs a Rollout created with final_observation=True")
        final_value = torch.zeros_like(self.reward)
        rows = self.final_observ[self.truncated]          # a truncated step is a done step
        if rows.shape[0]:
            final_value[self.truncated] = self.net.value(rows)
        return utility.gae_segments(self.reward, self.value, self.done, discount, lam, truncated=self.truncated,
                                    final_value=final_value)

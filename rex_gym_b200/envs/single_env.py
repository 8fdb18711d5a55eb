"""Single-environment gym.Env facade over the batched kernel (N = 1), with the reference's class names and constructor
kwargs so `PolicyPlayer` / user scripts written against rex_gym.envs.gym.* keep working
(rex_gym/playground/policy_player.py:43-46; rex_gym/envs/rex_gym_env.py:287-414)."""
import numpy as np

from .batched_env import BatchedRexEnv

try:  # pragma: no cover - gym is absent in the build image
    import gym  # type: ignore
    _Base = gym.Env
except Exception:
    _Base = object


class SingleRexEnv(_Base):
    """gym.Env surface: reset() -> obs[O]; step(a[A]) -> (obs[O], reward, done, {'action': cmd[nm]}).  With
    final_observation=True the info also carries gym TimeLimit's 'TimeLimit.truncated' on the step that reaches
    max_episode_steps (BatchedRexEnv)."""
    metadata = {"render.modes": ["human", "rgb_array"], "video.frames_per_second": 66}
    _task = "walk"

    def __init__(self, **kwargs):
        kwargs.pop("num_envs", None)
        kwargs.setdefault("render", False)
        self._batch = BatchedRexEnv(task=self._task, num_envs=1, **kwargs)
        self.action_space = self._batch.action_space
        self.observation_space = self._batch.observation_space
        self.mark = self._batch.mark
        self.num_motors = self._batch.num_motors
        self.control_time_step = self._batch.control_time_step

    def reset(self):
        return self._batch.reset()[0]

    def step(self, action):
        a = np.asarray(action, dtype=np.float32).reshape(1, -1)
        obs, reward, done, info = self._batch.step(a)
        return obs[0], float(reward[0]), bool(done[0]), info[0]

    def render(self, mode="rgb_array", close=False):
        """(360, 480, 3) uint8 frame for 'rgb_array'; rex_gym_env.py:416-418 returns an empty array for the other modes."""
        return self._batch.render(mode, close)

    def seed(self, seed=None):
        return [seed]

    def close(self):
        self._batch.close()

    @property
    def env_step_counter(self):
        return int(self._batch.get_state()["env_step_counter"][0])

    @property
    def rex(self):
        """Minimal stand-in for env.rex getters used by user scripts (model/rex.py:410-558)."""
        return _RexView(self._batch)


class _RexView(object):
    def __init__(self, batch):
        self._b = batch

    def GetBasePosition(self):
        return tuple(self._b.get_state()["pos"][0])

    def GetBaseOrientation(self):
        return tuple(self._b.get_state()["quat"][0])

    def GetMotorAngles(self):
        return self._b.get_state()["q"][0]

    def GetMotorVelocities(self):
        return self._b.get_state()["qd"][0]

    def GetTimeSinceReset(self):
        return float(self._b.get_state()["step_counter"][0]) * self._b._time_step


class RexWalkEnv(SingleRexEnv):
    """rex_gym/envs/gym/walk_env.py:16"""
    _task = "walk"


class RexReactiveEnv(SingleRexEnv):
    """rex_gym/envs/gym/gallop_env.py:28"""
    _task = "gallop"


class RexTurnEnv(SingleRexEnv):
    """rex_gym/envs/gym/turn_env.py:20"""
    _task = "turn"


class RexStandupEnv(SingleRexEnv):
    """rex_gym/envs/gym/standup_env.py:17"""
    _task = "standup"

    def __init__(self, **kwargs):
        kwargs.setdefault("signal_type", "ol")
        super().__init__(**kwargs)


class RexPosesEnv(SingleRexEnv):
    """rex_gym/envs/gym/poses_env.py:21"""
    _task = "poses"


def register_with_gym():
    """The reference registers its ids at import of rex_gym.playground (playground/__init__.py:17-57); call this to
    register the same ids against the batched CUDA envs when gym is installed."""
    from gym.envs.registration import register  # type: ignore
    for env_id, entry, steps in (("RexWalk-v0", "RexWalkEnv", 2500), ("RexGalloping-v0", "RexReactiveEnv", 1000),
                                 ("RexTurn-v0", "RexTurnEnv", 1000), ("RexStandup-v0", "RexStandupEnv", 400),
                                 ("RexPoses-v0", "RexPosesEnv", 400)):
        register(id=env_id, entry_point="rex_gym_b200.envs.single_env:" + entry, max_episode_steps=steps, reward_threshold=5.0)

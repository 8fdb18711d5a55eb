"""Device-side agent glue around the step kernel (SURVEY.md section 8(f) rows 1-2), mirroring the module names of
rex_gym/agents: networks.ForwardGaussianPolicy (and RecurrentGaussianPolicy / LinearGaussianPolicy in recurrent),
normalize.StreamingNormalize, utility.{discounted_return,lambda_advantage}, simulate (the rollout loop).  The PPO learner itself is out of scope."""
from .networks import ForwardGaussianPolicy  # noqa: F401
from .recurrent import RecurrentGaussianPolicy, LinearGaussianPolicy  # noqa: F401
from .simulate import Rollout  # noqa: F401
from . import utility, tf_checkpoint  # noqa: F401

"""`rlinf_b200.algorithms` - the reference's `rlinf.algorithms` plugin surface, CUDA-backed.

Importing the package fills the registries, like rlinf/algorithms/__init__.py:16.
"""
from . import advantages, loss_scales, losses  # noqa: F401  (registration side effects)
from .loss_scales import LOSS_SCALE_REGISTRY, get_loss_scales, register_loss_scale  # noqa: F401
from .losses import reasoning_actor_loss, reasoning_critic_loss  # noqa: F401
from .megatron_epilogue import MegatronLossEpilogue, step_metrics, valid_token_count  # noqa: F401
from .registry import (  # noqa: F401
    ADV_REGISTRY,
    LOSS_REGISTRY,
    calculate_adv_and_returns,
    get_adv_and_returns,
    get_policy_loss,
    policy_loss,
    register_advantage,
    register_policy_loss,
)

from .base_policy import ActorCritic, BasePolicy, DeviceBatch
from .lagrangian_base import LagrangianPolicy
from .ppo_lag import PPOLagrangian
from .sac_lag import SACLagrangian
from .ddpg_lag import DDPGLagrangian, GaussianNoise
from .cpo import CPO
from .trpo_lag import TRPOLagrangian
from .focops import FOCOPS
from .cvpo import CVPO

__all__ = ["ActorCritic", "BasePolicy", "DeviceBatch", "LagrangianPolicy", "PPOLagrangian",
           "SACLagrangian", "DDPGLagrangian", "GaussianNoise", "CPO", "TRPOLagrangian", "FOCOPS", "CVPO"]

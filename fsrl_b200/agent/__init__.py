from .base_agent import BaseAgent, OffpolicyAgent, OnpolicyAgent
from .cpo_agent import CPOAgent
from .ddpg_lag_agent import DDPGLagAgent
from .ppo_lag_agent import PPOLagAgent
from .sac_lag_agent import SACLagAgent
from .trpo_lag_agent import TRPOLagAgent
from .focops_agent import FOCOPSAgent
from .cvpo_agent import CVPOAgent

__all__ = ["BaseAgent", "OffpolicyAgent", "OnpolicyAgent", "PPOLagAgent", "SACLagAgent", "DDPGLagAgent", "CPOAgent", "TRPOLagAgent", "FOCOPSAgent", "CVPOAgent"]

from mjlab_b200.envs.tracking_env import TrackingEnvCfg, TrackingFlatEnv
from mjlab_b200.envs.velocity_env import VelocityCommandCfg, VelocityEnvCfg, VelocityFlatEnv, velocity_task_cfg

__all__ = ["TrackingEnvCfg", "TrackingFlatEnv", "VelocityCommandCfg", "VelocityEnvCfg", "VelocityFlatEnv", "velocity_task_cfg"]

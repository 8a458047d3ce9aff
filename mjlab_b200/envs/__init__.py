from mjlab_b200.envs.events import EventsCfg, RandomizeFieldCfg
from mjlab_b200.envs.noise import (ConstantNoiseCfg, GaussianNoiseCfg, NoiseModelCfg, NoiseModelWithAdditiveBiasCfg,
                                   UniformNoiseCfg)
from mjlab_b200.envs.obs_history import ObservationsCfg, ObsGroupCfg
from mjlab_b200.envs.tracking_env import (TrackingEnvCfg, TrackingFlatEnv, TrackingRewardsCfg, TrackingTerminationsCfg,
                                          tracking_task_cfg)
from mjlab_b200.envs.velocity_env import VelocityCommandCfg, VelocityEnvCfg, VelocityFlatEnv, velocity_task_cfg

__all__ = ["ConstantNoiseCfg", "EventsCfg", "GaussianNoiseCfg", "NoiseModelCfg", "NoiseModelWithAdditiveBiasCfg",
           "ObsGroupCfg", "ObservationsCfg", "RandomizeFieldCfg", "TrackingEnvCfg", "TrackingFlatEnv",
           "TrackingRewardsCfg", "TrackingTerminationsCfg", "UniformNoiseCfg", "VelocityCommandCfg", "VelocityEnvCfg",
           "VelocityFlatEnv", "tracking_task_cfg", "velocity_task_cfg"]

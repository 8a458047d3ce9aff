from mjlab_b200.envs.events import EventsCfg, RandomizeFieldCfg
from mjlab_b200.envs.obs_history import ObservationsCfg, ObsGroupCfg
from mjlab_b200.envs.tracking_env import (TrackingEnvCfg, TrackingFlatEnv, TrackingRewardsCfg, TrackingTerminationsCfg,
                                          tracking_task_cfg)
from mjlab_b200.envs.velocity_env import VelocityCommandCfg, VelocityEnvCfg, VelocityFlatEnv, velocity_task_cfg

__all__ = ["EventsCfg", "ObsGroupCfg", "ObservationsCfg", "RandomizeFieldCfg", "TrackingEnvCfg", "TrackingFlatEnv",
           "TrackingRewardsCfg", "TrackingTerminationsCfg", "VelocityCommandCfg", "VelocityEnvCfg", "VelocityFlatEnv",
           "tracking_task_cfg", "velocity_task_cfg"]

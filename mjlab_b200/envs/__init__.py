from mjlab_b200.envs.events import (ApplyExternalForceTorqueCfg, EventsCfg, PushBySettingVelocityCfg,
                                    RandomizeFieldCfg, ResetJointsByScaleCfg, ResetRootStateUniformCfg)
from mjlab_b200.envs.noise import (ConstantNoiseCfg, GaussianNoiseCfg, NoiseModelCfg, NoiseModelWithAdditiveBiasCfg,
                                   UniformNoiseCfg)
from mjlab_b200.envs.obs_history import ObservationsCfg, ObsGroupCfg
from mjlab_b200.envs.tracking_env import (TrackingEnvCfg, TrackingFlatEnv, TrackingRewardsCfg, TrackingTerminationsCfg,
                                          tracking_task_cfg)
from mjlab_b200.envs.velocity_env import VelocityCommandCfg, VelocityEnvCfg, VelocityFlatEnv, velocity_task_cfg

__all__ = ["ApplyExternalForceTorqueCfg", "ConstantNoiseCfg", "EventsCfg", "GaussianNoiseCfg", "NoiseModelCfg", "NoiseModelWithAdditiveBiasCfg",
           "ObsGroupCfg", "ObservationsCfg", "PushBySettingVelocityCfg", "RandomizeFieldCfg", "ResetJointsByScaleCfg", "ResetRootStateUniformCfg", "TrackingEnvCfg", "TrackingFlatEnv",
           "TrackingRewardsCfg", "TrackingTerminationsCfg", "UniformNoiseCfg", "VelocityCommandCfg", "VelocityEnvCfg",
           "VelocityFlatEnv", "tracking_task_cfg", "velocity_task_cfg"]

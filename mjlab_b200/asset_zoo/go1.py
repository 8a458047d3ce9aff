"""Unitree Go1 robot configuration (restates ``unitree_go1/go1_constants.py``)."""

from __future__ import annotations

from mjlab_b200.compiler.spec_cfg import (
  ActuatorCfg,
  CollisionCfg,
  ContactSensorCfg,
  InitialStateCfg,
  RobotCfg,
)

# go1_constants.py:38-60: single-stage reflected inertia = rotor * gear^2
_ROTOR = 0.000111842
ARM_HIP = _ROTOR * 6**2
ARM_KNEE = _ROTOR * (6 * 1.5) ** 2
_W = 10 * 2.0 * 3.1415926535
_Z = 2.0

ACTUATORS = (
  ActuatorCfg(
    joint_names_expr=[".*_hip_joint", ".*_thigh_joint"], effort_limit=23.7,
    stiffness=ARM_HIP * _W**2, damping=2 * _Z * ARM_HIP * _W, armature=ARM_HIP,
  ),
  ActuatorCfg(
    joint_names_expr=[".*_calf_joint"], effort_limit=35.55,
    stiffness=ARM_KNEE * _W**2, damping=2 * _Z * ARM_KNEE * _W, armature=ARM_KNEE,
  ),
)

# go1_constants.py:88-97
INIT_STATE = InitialStateCfg(
  pos=(0.0, 0.0, 0.278),
  joint_pos={".*thigh_joint": 0.9, ".*calf_joint": -1.8, ".*R_hip_joint": 0.1,
             ".*L_hip_joint": -0.1},
)

_FOOT = "^[FR][LR]_foot_collision$"
# go1_constants.py:130-138: no self collision (contype 1, conaffinity 0)
FULL_COLLISION = CollisionCfg(
  geom_names_expr=[".*_collision"],
  condim={_FOOT: 3, ".*_collision": 1},
  priority={_FOOT: 1},
  friction={_FOOT: (0.6,)},
  solimp={_FOOT: (0.9, 0.95, 0.023)},
  contype=1,
  conaffinity=0,
)

ACTION_SCALE = {n: 0.25 * a.effort_limit / a.stiffness for a in ACTUATORS for n in a.joint_names_expr}
FOOT_GEOMS = [f"{leg}_foot_collision" for leg in ("FR", "FL", "RR", "RL")]
# posture reward widths per joint (tasks/velocity/config/go1/rough_env_cfg.py:39-42): {regex: std}
POSTURE_STD = {r".*(FR|FL|RR|RL)_(hip|thigh)_joint.*": 0.3, r".*(FR|FL|RR|RL)_calf_joint.*": 0.6}


def velocity_sensors():
  # tasks/velocity/config/go1/rough_env_cfg.py:18-28
  return tuple(
    ContactSensorCfg(
      name=f"{leg}_foot_ground_contact", geom1=f"{leg}_foot_collision", body2="terrain",
      num=1, data=("found",), reduce="netforce",
    )
    for leg in ("FR", "FL", "RR", "RL")
  )


def robot_cfg(xml: str, sensors=()) -> RobotCfg:
  return RobotCfg(
    xml=xml, init_state=INIT_STATE, collisions=(FULL_COLLISION,), actuators=ACTUATORS,
    sensors=tuple(sensors), soft_joint_pos_limit_factor=0.9, action_scale=ACTION_SCALE,
  )

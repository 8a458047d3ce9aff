"""Unitree G1 (29 dof) robot configuration.

Values restate the reference's ``asset_zoo/robots/unitree_g1/g1_constants.py`` (line numbers
cited per block); formulas are re-derived here rather than imported.
"""

from __future__ import annotations

import math

from mjlab_b200.compiler.spec_cfg import (
  ActuatorCfg,
  CollisionCfg,
  ContactSensorCfg,
  InitialStateCfg,
  RobotCfg,
)


def _two_stage_planetary(rotor, gear):
  # utils/actuator.py:26-35: inertia of each stage reflected to the output shaft
  return rotor[0] * (gear[1] * gear[2]) ** 2 + rotor[1] * gear[2] ** 2 + rotor[2]


# g1_constants.py:43-101 motor data (rotor inertias kg m^2, stage gear ratios)
ARM_5020 = _two_stage_planetary((0.139e-4, 0.017e-4, 0.169e-4), (1, 1 + 46 / 18, 1 + 56 / 16))
ARM_7520_14 = _two_stage_planetary((0.489e-4, 0.098e-4, 0.533e-4), (1, 4.5, 1 + 48 / 22))
ARM_7520_22 = _two_stage_planetary((0.489e-4, 0.109e-4, 0.738e-4), (1, 4.5, 5))
ARM_4010 = _two_stage_planetary((0.068e-4, 0.0, 0.0), (1, 5, 5))

# g1_constants.py:124-135: PD gains from a 10 Hz natural frequency, damping ratio 2
_W = 10 * 2.0 * 3.1415926535
_Z = 2.0


def _pd(arm):
  return arm * _W**2, 2.0 * _Z * arm * _W


def _act(exprs, arm, effort, mult=1):
  kp, kd = _pd(arm)
  return ActuatorCfg(
    joint_names_expr=exprs, effort_limit=effort * mult, armature=arm * mult,
    stiffness=kp * mult, damping=kd * mult,
  )


# g1_constants.py:137-186 (waist pitch/roll and ankles: two 5020s on a linkage -> x2)
ACTUATORS = (
  _act([".*_elbow_joint", ".*_shoulder_pitch_joint", ".*_shoulder_roll_joint",
        ".*_shoulder_yaw_joint", ".*_wrist_roll_joint"], ARM_5020, 25.0),
  _act([".*_hip_pitch_joint", ".*_hip_yaw_joint", "waist_yaw_joint"], ARM_7520_14, 88.0),
  _act([".*_hip_roll_joint", ".*_knee_joint"], ARM_7520_22, 139.0),
  _act([".*_wrist_pitch_joint", ".*_wrist_yaw_joint"], ARM_4010, 5.0),
  _act(["waist_pitch_joint", "waist_roll_joint"], ARM_5020, 25.0, mult=2),
  _act([".*_ankle_pitch_joint", ".*_ankle_roll_joint"], ARM_5020, 25.0, mult=2),
)

# g1_constants.py:206-219
KNEES_BENT = InitialStateCfg(
  pos=(0, 0, 0.76),
  joint_pos={
    ".*_hip_pitch_joint": -0.312, ".*_knee_joint": 0.669, ".*_ankle_pitch_joint": -0.363,
    ".*_elbow_joint": 0.6, "left_shoulder_roll_joint": 0.2, "left_shoulder_pitch_joint": 0.2,
    "right_shoulder_roll_joint": -0.2, "right_shoulder_pitch_joint": 0.2,
  },
)

_FOOT = r"^(left|right)_foot[1-7]_collision$"
# g1_constants.py:228-233: everything collides; feet condim 3 / priority 1 / mu 0.6
FULL_COLLISION = CollisionCfg(
  geom_names_expr=[".*_collision"],
  condim={_FOOT: 3, ".*_collision": 1},
  priority={_FOOT: 1},
  friction={_FOOT: (0.6,)},
)

# g1_constants.py:278-289: action scale = 0.25 * effort / stiffness per joint pattern
ACTION_SCALE = {n: 0.25 * a.effort_limit / a.stiffness for a in ACTUATORS for n in a.joint_names_expr}

FOOT_GEOMS = [f"{s}_foot{i}_collision" for s in ("left", "right") for i in range(1, 8)]

# posture reward widths per joint (tasks/velocity/config/g1/rough_env_cfg.py:51-69): {regex: std}
POSTURE_STD = {
  # lower body
  r".*hip_pitch.*": 0.3, r".*hip_roll.*": 0.15, r".*hip_yaw.*": 0.15, r".*knee.*": 0.35, r".*ankle_pitch.*": 0.25,
  r".*ankle_roll.*": 0.1,
  # waist
  r".*waist_yaw.*": 0.15, r".*waist_roll.*": 0.08, r".*waist_pitch.*": 0.1,
  # arms
  r".*shoulder_pitch.*": 0.35, r".*shoulder_roll.*": 0.15, r".*shoulder_yaw.*": 0.1, r".*elbow.*": 0.25,
  r".*wrist.*": 0.3,
}


def velocity_sensors():
  # tasks/velocity/config/g1/rough_env_cfg.py:18-28
  return tuple(
    ContactSensorCfg(
      name=f"{side}_foot_ground_contact", body1=f"{side}_ankle_roll_link", body2="terrain",
      num=1, data=("found",), reduce="netforce",
    )
    for side in ("left", "right")
  )


def tracking_sensors():
  # tasks/tracking/config/g1/flat_env_cfg.py:11-20 (self-collision counter, 10 slots)
  return (
    ContactSensorCfg(
      name="self_collision", subtree1="pelvis", subtree2="pelvis",
      data=("found",), reduce="netforce", num=10,
    ),
  )


def robot_cfg(xml: str, sensors=()) -> RobotCfg:
  return RobotCfg(
    xml=xml, init_state=KNEES_BENT, collisions=(FULL_COLLISION,), actuators=ACTUATORS,
    sensors=tuple(sensors), soft_joint_pos_limit_factor=0.9, action_scale=ACTION_SCALE,
  )


assert math.isclose(_pd(ARM_5020)[0], 14.25, rel_tol=2e-3)  # SURVEY.md Appendix B table

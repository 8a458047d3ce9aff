"""Run by tests/test_velocity_command.py through tests/ref_runner.py (not collected by the main suite: it needs the
stand-ins ref_runner installs).  Instantiates the reference's cfg classes of the three velocity tasks that have a model
here and writes the fields velocity_task_cfg sets, as JSON, to the file named by B2_TASK_CFGS."""
import json
import os


def _fields(cfg):
  tw = cfg.commands.twist
  cv = cfg.curriculum.command_vel
  terrain = cfg.scene.terrain
  return dict(
    robot=cfg.scene.entities["robot"].spec_fn.__module__.rsplit(".", 1)[-1] if hasattr(cfg.scene.entities["robot"],
                                                                                    "spec_fn") else None,
    action_scale=dict(cfg.actions.joint_pos.scale),
    terrain_type=terrain.terrain_type, terrain_generator=terrain.terrain_generator is not None,
    terrain_curriculum=cfg.curriculum.terrain_levels is not None,
    command_curriculum=None if cv is None else [[s["step"], list(s["range"])] for s in cv.params["velocity_stages"]],
    push=cfg.events.push_robot.params["velocity_range"],
    posture_std=cfg.rewards.pose.params["std"],
    lin_vel_x=list(tw.ranges.lin_vel_x), lin_vel_y=list(tw.ranges.lin_vel_y), ang_vel_z=list(tw.ranges.ang_vel_z),
    heading=list(tw.ranges.heading), heading_command=tw.heading_command,
    heading_control_stiffness=tw.heading_control_stiffness, rel_standing_envs=tw.rel_standing_envs,
    rel_heading_envs=tw.rel_heading_envs, init_velocity_prob=tw.init_velocity_prob,
    resampling_time_range=list(tw.resampling_time_range), episode_length_s=cfg.episode_length_s,
    decimation=cfg.decimation)


def test_write_task_cfgs():
  from mjlab.tasks.velocity.config.g1.flat_env_cfg import UnitreeG1FlatEnvCfg
  from mjlab.tasks.velocity.config.go1.flat_env_cfg import UnitreeGo1FlatEnvCfg
  from mjlab.tasks.velocity.config.go1.rough_env_cfg import UnitreeGo1RoughEnvCfg

  # Each cfg is read as soon as it is built, in this order: the cfgs share their default scene and event instances,
  # and the flat tasks write their plane terrain (and G1 its push velocity) into them
  out = {"Mjlab-Velocity-Rough-Unitree-Go1": _fields(UnitreeGo1RoughEnvCfg()),
         "Mjlab-Velocity-Flat-Unitree-Go1": _fields(UnitreeGo1FlatEnvCfg()),
         "Mjlab-Velocity-Flat-Unitree-G1": _fields(UnitreeG1FlatEnvCfg())}
  with open(os.environ["B2_TASK_CFGS"], "w") as f:
    json.dump(out, f)

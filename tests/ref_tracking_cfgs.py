"""Run by tests/test_tracking_task.py through tests/ref_runner.py (not collected by the main suite: it needs the
stand-ins ref_runner installs).  Instantiates the reference's cfg classes of the four G1 tracking tasks and writes the
fields tracking_task_cfg sets, as JSON, to the file named by B2_TASK_CFGS."""
import json
import os

KEYS = ("x", "y", "z", "roll", "pitch", "yaw")


def _range6(d):
  return None if d is None else [list(d.get(k, (0.0, 0.0))) for k in KEYS]


def _noise(t):
  return None if t is None or t.noise is None else [t.noise.n_min, t.noise.n_max]


def _fields(cfg):
  mo = cfg.commands.motion
  pol = cfg.observations.policy
  push = cfg.events.push_robot
  r, t = cfg.rewards, cfg.terminations
  rewards = {k: dict(weight=getattr(r, k).weight, std=getattr(r, k).params.get("std"))
             for k in ("motion_global_root_pos", "motion_global_root_ori", "motion_body_pos", "motion_body_ori",
                       "motion_body_lin_vel", "motion_body_ang_vel", "action_rate_l2", "joint_limit", "self_collisions")}
  terms = {k: (None if getattr(t, k) is None else getattr(t, k).params.get("threshold"))
           for k in ("anchor_pos", "anchor_ori", "ee_body_pos")}
  policy = {k: (None if getattr(pol, k) is None else _noise(getattr(pol, k)))
            for k in ("command", "motion_anchor_pos_b", "motion_anchor_ori_b", "base_lin_vel", "base_ang_vel",
                      "joint_pos", "joint_vel", "actions")}
  return dict(
    rewards=rewards, terminations=terms, time_out=t.time_out is not None, pose_range=_range6(mo.pose_range),
    velocity_range=_range6(mo.velocity_range), joint_position_range=list(mo.joint_position_range),
    push=None if push is None else _range6(push.params["velocity_range"]),
    push_interval_s=None if push is None else list(push.interval_range_s), policy_terms=policy,
    enable_corruption=pol.enable_corruption, disable_adaptive_sampling=mo.disable_adaptive_sampling,
    episode_length_s=cfg.episode_length_s, decimation=cfg.decimation, body_names=list(mo.body_names),
    anchor=mo.anchor_body_name, ee_body_names=list(t.ee_body_pos.params["body_names"]))


def test_write_task_cfgs():
  from mjlab.tasks.tracking.config.g1 import flat_env_cfg as f

  # each cfg is read as soon as it is built: the cfgs share their default term instances
  out = {}
  for name, cls in (("Mjlab-Tracking-Flat-Unitree-G1", f.G1FlatEnvCfg),
                    ("Mjlab-Tracking-Flat-Unitree-G1-Play", f.G1FlatEnvCfg_PLAY),
                    ("Mjlab-Tracking-Flat-Unitree-G1-No-State-Estimation", f.G1FlatNoStateEstimationEnvCfg),
                    ("Mjlab-Tracking-Flat-Unitree-G1-No-State-Estimation-Play", f.G1FlatNoStateEstimationEnvCfg_PLAY)):
    out[name] = _fields(cls())
  with open(os.environ["B2_TASK_CFGS"], "w") as fh:
    json.dump(out, fh)

"""Slim motion-tracking flat-terrain environment (BASELINE.json configs[2], SURVEY.md §8d config C): the
*caller* of the hot path for the task with self-collision sensing and the higher contact count.

Follows ``ManagerBasedRlEnv.step`` (``src/mjlab/envs/manager_based_rl_env.py:106-147``) with the terms of
``tasks/tracking/tracking_env_cfg.py`` / ``tasks/tracking/config/g1/flat_env_cfg.py``: action -> 4 x {ctrl,
``sim.step``} -> terminations (time-out, anchor height / orientation, end-effector height) -> rewards (six
tracking terms, action rate, joint limits, self-collision count) -> reset of finished envs onto the motion
clip (RSI: clip frame + pose / velocity / joint noise, ``mdp/commands.py:283-352``) + forward -> command update
(``commands.py:354-388``: time step, anchor-relative body targets) -> interval push -> observations (policy
group with noise, critic group privileged).

The clip is ``cfg.motion_file``, a ``.npz`` in the reference's layout (``mjlab_b200.envs.motion``; one can be
generated with ``tools/make_motion_clip.py``).  Start frames of resets and clip restarts then come from the
reference's adaptive failure-bin sampler (``commands.py:256-297``, EMA ``:394-398``): the clip is cut into
``T // (1 / step_dt) + 1`` bins, terminations are counted in the bin of the frame the env reached, their EMA plus a
uniform floor, smoothed by the kernel ``lambda^i``, is the distribution of the next env step's start bins, and the
frame is uniform inside the bin.  Each draw inverts that distribution's CDF at the step's own uniform, so the draws
stay one uniform each; ``sampling_entropy`` / ``sampling_top1_prob`` / ``sampling_top1_bin`` of the distribution
the step drew from are in its extras.  ``disable_adaptive_sampling`` starts every episode at frame 0.

Without a file the clip is the synthetic one SURVEY.md §8d specifies for the benchmark: the KNEES_BENT pose held
for ``clip_frames`` frames, start frames uniform (the sampler has no effect on the physics load of a static clip).
Everything is mask-based torch code (or the fused kernels of ``csrc/b2_trackenv.cuh`` with the sampler's one-CTA
``b2_trackenv_bins``), so one env step is CUDA-graph capturable.
"""

from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
import torch
import torch.nn.functional as F

from mjlab_b200.asset_zoo import g1, load_compiled
from mjlab_b200.entity_data import EntityData, EntityIndexing, quat_apply, quat_apply_inverse, quat_mul
from mjlab_b200.envs.events import (RESET_STATE_TERMS, ApplyExternalForceTorqueCfg, Events, EventsCfg,
                                    PushBySettingVelocityCfg, RandomizeFieldCfg)
from mjlab_b200.envs.motion import MotionClip
from mjlab_b200.envs.noise import TaskNoise, tracking_defaults
from mjlab_b200.envs.obs_history import Observations, ObservationsCfg
from mjlab_b200.render import RENDER_MODES, ViewerConfig, check_render_mode, env_render, env_renderer, task_viewer
from mjlab_b200.envs.velocity_env import _resolve
from mjlab_b200.sim import MujocoCfg, Simulation, SimulationCfg, native

VELOCITY_RANGE = ((-0.5, 0.5), (-0.5, 0.5), (-0.2, 0.2), (-0.52, 0.52), (-0.52, 0.52), (-0.78, 0.78))  # tracking_env_cfg.py:30-37
POSE_RANGE = ((-0.05, 0.05), (-0.05, 0.05), (-0.01, 0.01), (-0.1, 0.1), (-0.1, 0.1), (-0.2, 0.2))       # :61-68
BODY_NAMES = ("pelvis", "left_hip_roll_link", "left_knee_link", "left_ankle_roll_link", "right_hip_roll_link",
              "right_knee_link", "right_ankle_roll_link", "torso_link", "left_shoulder_roll_link", "left_elbow_link",
              "left_wrist_yaw_link", "right_shoulder_roll_link", "right_elbow_link", "right_wrist_yaw_link")  # g1/flat_env_cfg.py:26-41
EE_NAMES = ("left_ankle_roll_link", "right_ankle_roll_link", "left_wrist_yaw_link", "right_wrist_yaw_link")  # :48-53
# the columns of the episode logs (B2_TRACKENV_NREW / NTERM / NMETRIC of include/b2sim.h)
TRACKING_TERMS = ("motion_global_root_pos", "motion_global_root_ori", "motion_body_pos", "motion_body_ori",
                  "motion_body_lin_vel", "motion_body_ang_vel")
REWARD_TERMS = TRACKING_TERMS + ("action_rate_l2", "joint_limit", "self_collisions")
TERMINATION_TERMS = ("time_out", "anchor_pos", "anchor_ori", "ee_body_pos")
METRICS = ("error_anchor_pos", "error_anchor_rot", "error_anchor_lin_vel", "error_anchor_ang_vel", "error_body_pos",
           "error_body_rot", "error_body_lin_vel", "error_body_ang_vel", "error_joint_pos", "error_joint_vel")
INT32_MAX = 2**31 - 1


def obs_terms(nu: int, nb: int, state_estimation: bool = True) -> dict:
  """{group: [(term, elements), ...]} in frame order (tracking_env_cfg.py:88-150); without state estimation the policy
  group has no motion_anchor_pos_b and no base_lin_vel."""
  policy = [("command", 2 * nu), ("motion_anchor_pos_b", 3), ("motion_anchor_ori_b", 6), ("base_lin_vel", 3),
            ("base_ang_vel", 3), ("joint_pos", nu), ("joint_vel", nu), ("actions", nu)]
  critic = policy[:3] + [("body_pos", 3 * nb), ("body_ori", 6 * nb)] + policy[3:]
  if not state_estimation:
    policy = [t for t in policy if t[0] not in ("motion_anchor_pos_b", "base_lin_vel")]
  return {"policy": policy, "critic": critic}


@dataclass
class TrackingRewardsCfg:
  """Weights and stds of the task's reward terms (tracking_env_cfg.py:201-252), the reference's defaults.  A term at
  weight 0 is not evaluated and its episode sum stays 0 (reward_manager.py:82-84); it is still logged."""

  motion_global_root_pos: float = 0.5
  motion_global_root_ori: float = 0.5
  motion_body_pos: float = 1.0
  motion_body_ori: float = 1.0
  motion_body_lin_vel: float = 1.0
  motion_body_ang_vel: float = 1.0
  action_rate_l2: float = -0.1
  joint_limit: float = -10.0
  self_collisions: float = -10.0
  motion_global_root_pos_std: float = 0.3
  motion_global_root_ori_std: float = 0.4
  motion_body_pos_std: float = 0.3
  motion_body_ori_std: float = 0.4
  motion_body_lin_vel_std: float = 1.0
  motion_body_ang_vel_std: float = 3.14

  def check(self) -> None:
    for t in TRACKING_TERMS:
      s = getattr(self, t + "_std")
      if not (math.isfinite(s) and s > 0.0):
        raise ValueError(f"rewards {t}_std must be positive and finite, not {s}")
    for t in REWARD_TERMS:
      if not math.isfinite(getattr(self, t)):
        raise ValueError(f"rewards {t}: the weight must be finite")


@dataclass
class TrackingTerminationsCfg:
  """Thresholds of the task's termination terms (tracking_env_cfg.py:253-278): anchor_pos (bad_anchor_pos_z_only),
  anchor_ori (bad_anchor_ori) and ee_body_pos (bad_motion_body_pos_z_only on EE_NAMES).  None removes a term;
  time_out always stays."""

  anchor_pos: float | None = 0.25
  anchor_ori: float | None = 0.8
  ee_body_pos: float | None = 0.25

  def check(self) -> None:
    for t in TERMINATION_TERMS[1:]:
      v = getattr(self, t)
      if v is not None and not (math.isfinite(v) and v > 0.0):
        raise ValueError(f"terminations {t}: the threshold must be positive and finite (or None), not {v}")


def _check_range6(name: str, r) -> None:
  try:
    pairs = [(float(lo), float(hi)) for lo, hi in r]
  except (TypeError, ValueError):  # not a sequence of pairs of numbers
    pairs = None
  if pairs is None or len(pairs) != 6:
    raise ValueError(f"{name} needs six (lo, hi) pairs (x, y, z, roll, pitch, yaw), got {r!r}")
  for k, (lo, hi) in enumerate(pairs):
    if not (math.isfinite(lo) and math.isfinite(hi) and lo <= hi):
      raise ValueError(f"{name}[{k}]: ({lo}, {hi}) is not a finite range with lo <= hi")


@dataclass
class TrackingEnvCfg:
  num_envs: int = 4096
  decimation: int = 4                 # tracking_env_cfg.py:305
  episode_length_s: float = 10.0      # :306
  clip_frames: int = 500              # synthetic static clip (SURVEY.md §8d config C); unused with a motion_file
  push_interval_s: tuple = (1.0, 3.0)
  friction_range: tuple = (0.3, 1.2)
  joint_position_range: tuple = (-0.1, 0.1)
  env_spacing: float = 2.5
  seed: int = 42
  motion_file: str | None = None      # reference-layout .npz (mjlab_b200.envs.motion); None: the synthetic clip
  adaptive_kernel_size: int = 1       # commands.py:429-433
  adaptive_lambda: float = 0.8
  adaptive_uniform_ratio: float = 0.1
  adaptive_alpha: float = 0.001
  disable_adaptive_sampling: bool = False
  sim: SimulationCfg = field(
    default_factory=lambda: SimulationCfg(
      nconmax=150_000, njmax=250, mujoco=MujocoCfg(timestep=0.005, iterations=10, ls_iterations=20)))  # :283-291
  rewards: TrackingRewardsCfg = field(default_factory=TrackingRewardsCfg)
  terminations: TrackingTerminationsCfg = field(default_factory=TrackingTerminationsCfg)
  pose_range: tuple = POSE_RANGE           # RSI offsets of the root pose, (lo, hi) of x, y, z, roll, pitch, yaw
  velocity_range: tuple = VELOCITY_RANGE   # RSI offsets of the root velocity
  push_velocity_range: tuple | None = VELOCITY_RANGE  # push_by_setting_velocity; None: no push event
  policy_state_estimation: bool = True     # False: no motion_anchor_pos_b and no base_lin_vel in the policy group
  policy_corruption: bool = True           # the policy group's enable_corruption
  # per-episode logs of the reward, termination and command managers (reward_log, termination_log, command_log)
  episode_logs: bool = False
  # clip, scale and history of the policy and critic groups (terms: obs_terms); the defaults leave both as computed
  observations: ObservationsCfg = field(default_factory=ObservationsCfg)
  # randomize_field events (envs/events.py), run after the task's startup randomisation (startup_events)
  events: EventsCfg = field(default_factory=EventsCfg)
  # the camera of env.render() with render_mode="rgb_array" (tracking_env_cfg.py:45-52; the robot's cfg names the body,
  # tracking_task_cfg sets it)
  viewer: ViewerConfig = field(default_factory=task_viewer)
  # the motion command's ghost in env.render() frames (commands.py:400-416): the robot posed at the clip's current
  # frame of cfg.viewer.env_idx, drawn translucent in ghost_color (MotionCommandCfg.VizCfg, commands.py:436-439)
  debug_vis: bool = False
  ghost_color: tuple = (0.5, 0.7, 0.5, 0.5)

  def __post_init__(self):
    self.check()

  def check(self) -> None:
    self.rewards.check()
    self.terminations.check()
    self.events.check()
    for t in self.events.terms:
      if isinstance(t, PushBySettingVelocityCfg) and self.push_velocity_range is not None:
        raise ValueError("a PushBySettingVelocityCfg term needs push_velocity_range=None: the built-in push also "
                         "writes the root velocity, and it cannot take the term's place in the list order")
      if isinstance(t, RESET_STATE_TERMS) or (isinstance(t, ApplyExternalForceTorqueCfg) and t.mode == "reset"):
        raise ValueError(f"a {type(t).__name__} term of mode 'reset' is a no-op in the tracking env: the motion "
                         "command's RSI rewrites the root, the joints and clears the wrenches (clear_state) after the "
                         "reset events")
    _check_range6("pose_range", self.pose_range)
    _check_range6("velocity_range", self.velocity_range)
    if self.push_velocity_range is not None:
      _check_range6("push_velocity_range", self.push_velocity_range)
    if not self.episode_length_s > 0:
      raise ValueError(f"episode_length_s must be positive, not {self.episode_length_s}")
    on = self.observations.policy.enable_corruption
    if on is not None and bool(on) != bool(self.policy_corruption):
      raise ValueError(f"observations.policy.enable_corruption={on} contradicts policy_corruption="
                       f"{self.policy_corruption}; set one of them")


_NO_RSI = ((0.0, 0.0),) * 6  # an empty pose_range / velocity_range dict of MotionCommandCfg: every offset 0
_PLAY = dict(policy_corruption=False, push_velocity_range=None, pose_range=_NO_RSI, velocity_range=_NO_RSI,
             disable_adaptive_sampling=True, episode_length_s=int(1e9))
# the reference's four G1 tracking tasks (tasks/tracking/config/g1/__init__.py), as their cfg classes set them
# (G1FlatEnvCfg, G1FlatEnvCfg_PLAY, G1FlatNoStateEstimationEnvCfg, G1FlatNoStateEstimationEnvCfg_PLAY:
# config/g1/flat_env_cfg.py), with the episode logs on
TRACKING_TASKS = {
  "Mjlab-Tracking-Flat-Unitree-G1": dict(),
  "Mjlab-Tracking-Flat-Unitree-G1-Play": dict(_PLAY),
  "Mjlab-Tracking-Flat-Unitree-G1-No-State-Estimation": dict(policy_state_estimation=False),
  "Mjlab-Tracking-Flat-Unitree-G1-No-State-Estimation-Play": dict(_PLAY, policy_state_estimation=False),
}


def startup_events(cfg: TrackingEnvCfg) -> tuple:
  """The task's startup randomisation (tracking_env_cfg.py:162-198): the torso's COM offset, the joints' default
  positions and the feet's friction (friction_range)."""
  return (RandomizeFieldCfg("body_ipos", {0: (-0.025, 0.025), 1: (-0.05, 0.05), 2: (-0.05, 0.05)}, operation="add",
                            names="torso_link"),
          RandomizeFieldCfg("qpos0", (-0.01, 0.01), operation="add"),
          RandomizeFieldCfg("geom_friction", tuple(cfg.friction_range), operation="abs", names=tuple(g1.FOOT_GEOMS)))


def tracking_task_cfg(name: str, **overrides) -> TrackingEnvCfg:
  """The TrackingEnvCfg of one of the reference's tracking tasks by its registered name, with `overrides` (any
  TrackingEnvCfg field) on top.  As in the reference, whose robot cfg leaves it empty, the clip comes in as the
  `motion_file` override (without one the env runs the synthetic clip).  The presets leave the motion's ghost off,
  so their frames show the scene alone; the reference's tasks turn it on, which `debug_vis=True` does here."""
  if name not in TRACKING_TASKS:
    raise ValueError(f"unknown tracking task {name!r}; known: {', '.join(TRACKING_TASKS)}")
  # (the G1's camera override: tracking/config/g1/flat_env_cfg.py:54)
  return TrackingEnvCfg(**{"episode_logs": True, "viewer": task_viewer(body_name="torso_link"), **TRACKING_TASKS[name],
                           **overrides})


def quat_inv(q):
  return torch.cat([q[..., 0:1], -q[..., 1:4]], dim=-1)


def yaw_quat(q):
  w, x, y, z = q.unbind(-1)
  yaw = torch.atan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z))
  out = torch.zeros_like(q)
  out[..., 0] = torch.cos(yaw / 2)
  out[..., 3] = torch.sin(yaw / 2)
  return out


def quat_from_euler_xyz(r, p, y):
  cy, sy, cr, sr, cp, sp = torch.cos(y / 2), torch.sin(y / 2), torch.cos(r / 2), torch.sin(r / 2), torch.cos(p / 2), torch.sin(p / 2)
  return torch.stack([cy * cr * cp + sy * sr * sp, cy * sr * cp - sy * cr * sp, cy * cr * sp + sy * sr * cp,
                      sy * cr * cp - cy * sr * sp], dim=-1)


def quat_error_magnitude(a, b):
  d = quat_mul(a, quat_inv(b))
  return 2.0 * torch.atan2(d[..., 1:4].norm(dim=-1), d[..., 0].abs())


def rot6(q):
  """First two columns of R(q), flattened row-major over (3, 2) (``matrix_from_quat(q)[..., :2]``)."""
  w, x, y, z = q.unbind(-1)
  c0 = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + w * z), 2 * (x * z - w * y)], dim=-1)
  c1 = torch.stack([2 * (x * y - w * z), 1 - 2 * (x * x + z * z), 2 * (y * z + w * x)], dim=-1)
  return torch.stack([c0, c1], dim=-1).flatten(-2)


class TrackingFlatEnv:
  metadata = {"render_modes": RENDER_MODES}

  def __init__(self, cfg: TrackingEnvCfg, device: str = "cuda:0", model=None, native_mdp: bool = True,
               render_mode: str | None = None):
    check_render_mode(render_mode)
    self.cfg, self.device = cfg, device
    self.native_mdp = native_mdp  # fused CUDA kernels (csrc/b2_trackenv.cuh) or the torch reference below
    self.model = m = model if model is not None else load_compiled("g1_tracking_flat")
    n = self.num_envs = cfg.num_envs
    self.sim = Simulation(n, cfg.sim, m, device)
    self._nan_guard = getattr(self.sim, "nan_guard", None)  # (None on a Simulation stand-in without the guard)
    dev = torch.device(device)
    f32 = dict(dtype=torch.float32, device=dev)
    self.nq, self.nv, self.nu = int(m.nq), int(m.nv), int(m.nu)
    self.step_dt = cfg.decimation * float(m.opt_timestep)
    cfg.check()
    # clamped to the episode counter's int32 range: an "effectively infinite" episode (the play tasks' 1e9 s) never
    # truncates, on both paths, instead of wrapping to a negative limit
    self.max_episode_length = min(math.ceil(cfg.episode_length_s / self.step_dt), INT32_MAX)
    self.gen = torch.Generator(device=dev)
    self.gen.manual_seed(cfg.seed)
    key = m.keys["robot/init_state"]
    self.default_qpos = torch.tensor(key["qpos"], **f32)
    self.default_joint_pos = self.default_qpos[7:].clone()
    ix = EntityIndexing.from_model(m, "robot", device)
    self.robot = EntityData(ix, self.sim.data, self.sim.model, device, n, soft_joint_pos_limit_factor=0.9)
    self.action_scale = torch.tensor(_resolve(g1.ACTION_SCALE, list(ix.joint_names), 0.5), **f32)
    self.body_idx = torch.tensor([ix.body_names.index(b) for b in BODY_NAMES], device=dev)
    self.anchor = BODY_NAMES.index("torso_link")
    self.ee_idx = torch.tensor([BODY_NAMES.index(b) for b in EE_NAMES], device=dev)
    self.self_collision_adr = [int(v) for v in ix.sensor_adr["self_collision"]]  # python ints: graph-capturable indexing
    cols = math.ceil(math.sqrt(n))
    idx = torch.arange(n, device=dev)
    self.env_origins = torch.stack(
      [(idx // cols - (cols - 1) / 2) * cfg.env_spacing, (idx % cols - (cols - 1) / 2) * cfg.env_spacing,
       torch.zeros(n, device=dev)], dim=1).float()
    # ---- domain randomisation: the task's startup terms, then cfg.events; the fields they name get a per-world copy
    self.events = Events(startup_events(cfg) + tuple(cfg.events.terms), ix, self.sim, n, self.step_dt, device,
                         clear_xfrc=False)  # (the RSI of _resample clears the wrenches)
    self.sim.expand_model_fields(self.events.fields())
    self.events.run_startup(self._rand)
    self.events.draw_timers(self._rand)
    self.sim.data.qpos[:] = self.default_qpos
    self.sim.data.qvel[:] = 0.0
    self.sim.forward()
    nbk = len(BODY_NAMES)
    if cfg.motion_file is None:  # synthetic clip: the keyframe held static (keys of commands.py:34-50)
      T = cfg.clip_frames
      pose0 = self.robot.body_link_pose_w[0:1, self.body_idx].clone()  # (1, 14, 7) at the world origin
      self.motion = dict(
        joint_pos=self.default_joint_pos.expand(T, -1).contiguous(), joint_vel=torch.zeros(T, self.nu, **f32),
        body_pos_w=pose0[:, :, 0:3].expand(T, -1, -1).contiguous(), body_quat_w=pose0[:, :, 3:7].expand(T, -1, -1).contiguous(),
        body_lin_vel_w=torch.zeros(T, nbk, 3, **f32), body_ang_vel_w=torch.zeros(T, nbk, 3, **f32))
      self.start_mode = native.START_UNIFORM
    else:
      self.motion = MotionClip.load(cfg.motion_file, ix, BODY_NAMES, self.step_dt, dev).as_dict()
      T = self.motion["joint_pos"].shape[0]
      self.start_mode = native.START_FIRST if cfg.disable_adaptive_sampling else native.START_ADAPTIVE
    self.T = T
    self._sampler_setup()
    self.time_steps = torch.zeros(n, dtype=torch.long, device=dev)
    self.episode_length_buf = torch.zeros(n, dtype=torch.int32, device=dev)
    self.last_action = torch.zeros(n, self.nu, **f32)
    self.push_time_left = torch.zeros(n, **f32)
    lo_t, hi_t = cfg.push_interval_s
    self.push_time_left.copy_(self._rand(n) * (hi_t - lo_t) + lo_t)
    self.body_pos_relative_w = torch.zeros(n, nbk, 3, **f32)
    self.body_quat_relative_w = torch.zeros(n, nbk, 4, **f32)
    self._done_buf = torch.zeros(n, dtype=torch.bool, device=dev)
    self.log_row = torch.zeros(n, 3, **f32)  # (reward, terminated, truncated) for the rank-0 log gather
    self._vr = torch.tensor(cfg.velocity_range, **f32)
    self._pr = torch.tensor(cfg.pose_range, **f32)
    self._init_task()
    self._graph = None
    self.reset()
    self.render_mode = render_mode
    self.metadata = {**self.metadata, "render_fps": 1.0 / self.step_dt}
    self._offline_renderer = env_renderer(self.sim, cfg.viewer, render_mode)

  # -- helpers -------------------------------------------------------------------------------------
  def _rand(self, *shape):
    return torch.rand(shape, generator=self.gen, device=self.device)

  def _randn(self, *shape):
    return torch.randn(shape, generator=self.gen, device=self.device)

  def _clip(self, name):
    return self.motion[name][self.time_steps]

  # -- task configuration and episode logs ---------------------------------------------------------------------------
  def _init_task(self) -> None:
    """The configured terms as both paths use them, and the per-env log state (columns: REWARD_TERMS,
    TERMINATION_TERMS, METRICS)."""
    cfg, n = self.cfg, self.num_envs
    f32 = dict(dtype=torch.float32, device=self.device)
    rc, tc = cfg.rewards, cfg.terminations
    self.reward_weights = [float(getattr(rc, t)) for t in REWARD_TERMS]
    self.reward_stds = [float(getattr(rc, t + "_std")) for t in TRACKING_TERMS]
    self.term_thresholds = [getattr(tc, t) for t in TERMINATION_TERMS[1:]]
    self._push_r = None if cfg.push_velocity_range is None else torch.tensor(cfg.push_velocity_range, **f32)
    terms = obs_terms(self.nu, len(BODY_NAMES), cfg.policy_state_estimation)
    # noise-configured groups: the task's default noise (policy as policy_corruption, critic none) on the critic frame
    task_noise = TaskNoise(tracking_defaults(), {"policy": bool(cfg.policy_corruption), "critic": False},
                           terms["critic"])
    self.obs_groups = Observations(cfg.observations, terms, n, self.device, task_noise)
    self.nobs, self.nobs_critic = self.obs_groups.width("policy"), self.obs_groups.width("critic")  # elements per env
    self.episode_sums = torch.zeros(n, len(REWARD_TERMS), **f32)
    self.finished_sums = torch.zeros(n, len(REWARD_TERMS), **f32)
    self.term_flags = torch.zeros(n, len(TERMINATION_TERMS), **f32)
    self.motion_metrics = torch.zeros(n, len(METRICS), **f32)
    self.finished_metrics = torch.zeros(n, len(METRICS), **f32)

  def _ended(self):
    """[n, 1] envs whose episode ended in the last step (terminated | truncated, the reference's reset_buf; clip
    restarts are internal to the command) and their count."""
    ended = (self.term_flags != 0).any(dim=1, keepdim=True)
    return ended, ended.sum()

  def _need_logs(self) -> None:
    if not self.cfg.episode_logs:
      raise RuntimeError("episode logs are off: build the env with TrackingEnvCfg(episode_logs=True)")

  def reward_log(self) -> dict:
    """``Episode_Reward/<term>`` of RewardManager.reset (managers/reward_manager.py:61-75) for the envs whose episode
    ended in the last step: the mean of their episode sums over episode_length_s (NaN when none ended), for all nine
    terms.  Device tensors, no host synchronisation."""
    self._need_logs()
    ended, k = self._ended()
    mean = torch.where(ended, self.finished_sums, 0.0).sum(0) / k / self.cfg.episode_length_s
    return {f"Episode_Reward/{t}": mean[i] for i, t in enumerate(REWARD_TERMS)}

  def termination_log(self) -> dict:
    """``Episode_Termination/<term>`` of TerminationManager.reset (managers/termination_manager.py:73-85): how many of
    the envs whose episode ended in the last step that term fired for (NaN when none ended); a removed term has no
    key.  Device tensors, no host synchronisation."""
    self._need_logs()
    ended, k = self._ended()
    count = torch.count_nonzero(self.term_flags, dim=0).float()
    count = torch.where(k > 0, count, math.nan)
    on = [True] + [t is not None for t in self.term_thresholds]
    return {f"Episode_Termination/{t}": count[i] for i, t in enumerate(TERMINATION_TERMS) if on[i]}

  def command_log(self) -> dict:
    """``Metrics/motion/<error>`` of CommandManager.reset (managers/command_manager.py:128-134, the errors of
    MotionCommand._update_metrics, tasks/tracking/mdp/commands.py:221-255) for the envs whose episode ended in the last
    step: the mean of the errors of their last command update (NaN when none ended); with the adaptive sampler also
    ``sampling_entropy`` / ``sampling_top1_prob`` / ``sampling_top1_bin``.  Device tensors, no host synchronisation."""
    self._need_logs()
    ended, k = self._ended()
    mean = torch.where(ended, self.finished_metrics, 0.0).sum(0) / k
    out = {f"Metrics/motion/{t}": mean[i] for i, t in enumerate(METRICS)}
    if self.start_mode == native.START_ADAPTIVE:
      for i, t in enumerate(("sampling_entropy", "sampling_top1_prob", "sampling_top1_bin")):
        out[f"Metrics/motion/{t}"] = self._metrics[i]
    return out

  def _motion_errors(self, frame, pos, quat, lin, ang):
    """[n, 10] MotionCommand._update_metrics (commands.py:221-255) at clip frames `frame` against the robot's tracked
    bodies and joints and the current relative targets."""
    d, a = self.sim.data, self.anchor
    clip = {k: v[frame] for k, v in self.motion.items()}
    a_pos = clip["body_pos_w"][:, a] + self.env_origins
    return torch.stack([
      (a_pos - pos[:, a]).norm(dim=-1), quat_error_magnitude(clip["body_quat_w"][:, a], quat[:, a]),
      (clip["body_lin_vel_w"][:, a] - lin[:, a]).norm(dim=-1), (clip["body_ang_vel_w"][:, a] - ang[:, a]).norm(dim=-1),
      (self.body_pos_relative_w - pos).norm(dim=-1).mean(-1),
      quat_error_magnitude(self.body_quat_relative_w, quat).mean(-1),
      (clip["body_lin_vel_w"] - lin).norm(dim=-1).mean(-1), (clip["body_ang_vel_w"] - ang).norm(dim=-1).mean(-1),
      (clip["joint_pos"] - d.qpos[:, 7:]).norm(dim=-1), (clip["joint_vel"] - d.qvel[:, 6:]).norm(dim=-1)], dim=1)

  # -- adaptive start-frame sampler (commands.py:99-110, 256-297, 394-398) -------------------------------
  def _sampler_setup(self) -> None:
    cfg, dev = self.cfg, torch.device(self.device)
    B = self.bin_count = int(self.T // (1 / self.step_dt)) + 1
    if self.start_mode != native.START_ADAPTIVE:
      return
    if cfg.adaptive_kernel_size < 1 or not cfg.adaptive_lambda > 0 or not cfg.adaptive_uniform_ratio > 0 \
       or not 0.0 <= cfg.adaptive_alpha <= 1.0:
      raise ValueError("adaptive sampling needs adaptive_kernel_size >= 1, adaptive_lambda > 0, "
                       "adaptive_uniform_ratio > 0 and 0 <= adaptive_alpha <= 1")
    k = torch.tensor([cfg.adaptive_lambda**i for i in range(cfg.adaptive_kernel_size)], device=dev)
    self._bin_kernel = k / k.sum()
    self.bin_failed_count = torch.zeros(B, device=dev)   # EMA of terminations per bin
    self._bin_failed_cur = torch.zeros(B, device=dev)    # terminations per bin in the current env step
    self._metrics = torch.zeros(3, device=dev)            # entropy, top-1 prob, top-1 bin of the last step's draws
    self._cdf = self._start_distribution()[1].contiguous()  # CDF the next draws invert

  def _start_distribution(self):
    """(p, CDF) of the start bins from the failure EMA; the CDF's last entry is 1 so that every u < 1 finds a bin."""
    cfg, B = self.cfg, self.bin_count
    p = (self.bin_failed_count + cfg.adaptive_uniform_ratio / float(B)).view(1, 1, -1)
    p = F.conv1d(F.pad(p, (0, cfg.adaptive_kernel_size - 1), mode="replicate"), self._bin_kernel.view(1, 1, -1)).view(-1)
    p = p / p.sum()
    cdf = p.cumsum(0)
    cdf[-1] = 1.0
    return p, cdf

  def _start_frames(self, u: torch.Tensor) -> torch.Tensor:
    """Start frame of each env for its uniform ``u`` (B2_START_* of include/b2sim.h)."""
    T = self.T
    if self.start_mode == native.START_FIRST:
      return torch.zeros_like(u, dtype=torch.long)
    if self.start_mode == native.START_UNIFORM:
      return (u * (T - 1)).long()
    B, cdf = self.bin_count, self._cdf
    b = torch.searchsorted(cdf, u.contiguous(), right=True).clamp_(max=B - 1)  # first bin with cdf > u
    c0 = torch.where(b > 0, cdf[(b - 1).clamp(min=0)], torch.zeros_like(u))
    frac = (u - c0) / (cdf[b] - c0)
    return ((b + frac) / B * (T - 1)).long().clamp_(max=T - 1)

  def _sampler_step(self) -> None:
    """End of an env step: metrics of the distribution the step drew from, EMA update, CDF for the next step."""
    B, a = self.bin_count, self.cfg.adaptive_alpha
    p, _ = self._start_distribution()
    H = -(p * (p + 1e-12).log()).sum()
    pmax, imax = p.max(dim=0)
    self._metrics.copy_(torch.stack([H / math.log(B) if B > 1 else torch.ones_like(H), pmax, imax.float() / B]))
    self.bin_failed_count.copy_(a * self._bin_failed_cur + (1 - a) * self.bin_failed_count)
    self._bin_failed_cur.zero_()
    self._cdf.copy_(self._start_distribution()[1])

  def _extras(self, critic):
    x = {"critic": critic}
    if self.start_mode == native.START_ADAPTIVE:
      x.update(sampling_entropy=self._metrics[0], sampling_top1_prob=self._metrics[1], sampling_top1_bin=self._metrics[2])
    return x

  def _resample(self, mask: torch.Tensor, restart_clip: torch.Tensor, Ub: torch.Tensor) -> None:
    """``MotionCommand._resample_command`` for the masked envs: new clip frame, RSI noise, state write.  ``Ub``:
    this call's uniforms ``[n, 13 + nu]`` (0 clip frame, 1-6 pose, 7-12 velocity, 13.. joints; include/b2sim.h)."""
    n, d = self.num_envs, self.sim.data
    ts = self._start_frames(Ub[:, 0])
    self.time_steps.copy_(torch.where(restart_clip, ts, self.time_steps))
    pose_n = Ub[:, 1:7] * (self._pr[:, 1] - self._pr[:, 0]) + self._pr[:, 0]
    vel_n = Ub[:, 7:13] * (self._vr[:, 1] - self._vr[:, 0]) + self._vr[:, 0]
    root_pos = self._clip("body_pos_w")[:, 0] + self.env_origins + pose_n[:, 0:3]
    root_ori = quat_mul(quat_from_euler_xyz(pose_n[:, 3], pose_n[:, 4], pose_n[:, 5]), self._clip("body_quat_w")[:, 0])
    lin = self._clip("body_lin_vel_w")[:, 0] + vel_n[:, 0:3]
    ang = self._clip("body_ang_vel_w")[:, 0] + vel_n[:, 3:6]
    lo, hi = self.cfg.joint_position_range
    jp = self._clip("joint_pos") + Ub[:, 13:13 + self.nu] * (hi - lo) + lo
    lim = self.robot.soft_joint_pos_limits
    jp = torch.minimum(torch.maximum(jp, lim[..., 0]), lim[..., 1])
    qpos = torch.cat([root_pos, root_ori, jp], dim=1)
    qvel = torch.cat([lin, quat_apply_inverse(root_ori, ang), self._clip("joint_vel")], dim=1)
    mk = mask.unsqueeze(1)
    d.qpos[:] = torch.where(mk, qpos, d.qpos[:])
    d.qvel[:] = torch.where(mk, qvel, d.qvel[:])
    d.ctrl[:] = torch.where(mk, torch.zeros_like(d.ctrl[:]), d.ctrl[:])  # clear_state (data.py:170-178)
    d.xfrc_applied[:] = torch.where(mask.view(n, 1, 1), torch.zeros_like(d.xfrc_applied[:]), d.xfrc_applied[:])

  def _robot_bodies(self):
    pose = self.robot.body_link_pose_w[:, self.body_idx]
    vel = self.robot.body_link_vel_w[:, self.body_idx]
    return pose[..., 0:3], pose[..., 3:7], vel[..., 0:3], vel[..., 3:6]

  def _update_command(self) -> None:
    """``MotionCommand._update_command``: anchor-relative targets (yaw-aligned, height from the clip)."""
    pos, quat, _, _ = self._robot_bodies()
    nbk = len(BODY_NAMES)
    a_pos = (self._clip("body_pos_w")[:, self.anchor] + self.env_origins)[:, None, :].expand(-1, nbk, -1)
    a_quat = self._clip("body_quat_w")[:, self.anchor][:, None, :].expand(-1, nbk, -1)
    r_pos = pos[:, self.anchor][:, None, :].expand(-1, nbk, -1)
    r_quat = quat[:, self.anchor][:, None, :].expand(-1, nbk, -1)
    delta_pos = torch.cat([r_pos[..., 0:2], a_pos[..., 2:3]], dim=-1)
    delta_ori = yaw_quat(quat_mul(r_quat, quat_inv(a_quat)))
    # (in place: the fused kernels hold pointers to these two tensors)
    self.body_quat_relative_w.copy_(quat_mul(delta_ori, self._clip("body_quat_w")))
    self.body_pos_relative_w.copy_(delta_pos + quat_apply(delta_ori, self._clip("body_pos_w") + self.env_origins[:, None, :] - a_pos))

  def observations(self, Z: torch.Tensor | None = None):
    """(policy, critic) groups of tracking_env_cfg.py:88-150; uniform noise on the policy group from the draws
    ``Z[n, 15 + 2 nu]`` (anchor pos 3, anchor ori 6, base lin 3, base ang 3, joint pos, joint vel)."""
    d = self.sim.data
    if Z is None:
      Z = self._rand(self.num_envs, 15 + 2 * self.nu)
    pos, quat, _, _ = self._robot_bodies()
    a_pos = self._clip("body_pos_w")[:, self.anchor] + self.env_origins
    a_quat = self._clip("body_quat_w")[:, self.anchor]
    r_pos, r_quat = pos[:, self.anchor], quat[:, self.anchor]
    command = torch.cat([self._clip("joint_pos"), self._clip("joint_vel")], dim=1)
    anchor_pos_b = quat_apply_inverse(r_quat, a_pos - r_pos)
    anchor_ori_b = rot6(quat_mul(quat_inv(r_quat), a_quat))
    base_lin, base_ang = self.robot.root_link_lin_vel_b, self.robot.root_link_ang_vel_b
    jp, jv = d.qpos[:, 7:] - self.default_joint_pos, d.qvel[:, 6:]
    terms = [command, anchor_pos_b, anchor_ori_b, base_lin, base_ang, jp, jv, self.last_action]
    amp = (0.0, 0.25, 0.05, 0.5, 0.2, 0.01, 0.5, 0.0)
    # each noised term has its own columns of Z, drawn whether or not the term is in the policy group
    se, noise_on = self.cfg.policy_state_estimation, self.cfg.policy_corruption
    noisy, k = [], 0
    for i, (t, a) in enumerate(zip(terms, amp)):
      if se or i not in (1, 3):  # without state estimation: no motion_anchor_pos_b, no base_lin_vel
        noisy.append(t if a == 0.0 or not noise_on else t + (Z[:, k:k + t.shape[1]] * 2 - 1) * a)
      if a != 0.0:
        k += t.shape[1]
    rq = r_quat[:, None, :].expand(-1, len(BODY_NAMES), -1)
    body_pos_b = quat_apply_inverse(rq, pos - r_pos[:, None, :]).flatten(1)
    body_ori_b = rot6(quat_mul(quat_inv(rq), quat)).flatten(1)
    critic = torch.cat(terms[:3] + [body_pos_b, body_ori_b] + terms[3:], dim=1)
    return torch.cat(noisy, dim=1), critic

  # -- API -----------------------------------------------------------------------------------------
  def reset(self):
    for t in (self.episode_sums, self.term_flags, self.motion_metrics):  # the logs start over
      t.zero_()
    all_ = torch.ones(self.num_envs, dtype=torch.bool, device=self.device)
    self._resample(all_, all_, self._rand(self.num_envs, 13 + self.nu))
    self.events.reset_all(self._rand)
    self.sim.forward()
    self._update_command()
    policy, critic = self.observations()
    out = self.obs_groups.fill({"policy": policy, "critic": critic}, self._rand, self._randn)
    return out["policy"], out["critic"]

  def enable_cuda_graph(self) -> None:
    dev = torch.device(self.device)
    self._action_buf = torch.zeros(self.num_envs, self.nu, device=dev)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
      for _ in range(2):
        self._step_impl(self._action_buf)
      g = torch.cuda.CUDAGraph()
      g.register_generator_state(self.gen)
      with torch.cuda.graph(g, stream=side):
        self._graph_out = self._step_impl(self._action_buf)
    torch.cuda.current_stream(dev).wait_stream(side)
    self._graph = g

  def step(self, action: torch.Tensor):
    """One env step (the captured graph's replay after ``enable_cuda_graph``).  With the sim's NaN guard enabled it then
    polls the guard without synchronising: a NaN the GPU found in this step's sub-steps is dumped by this call or, when
    the GPU has not got there yet, by a later step (usually one or two later) or by ``close()``.  The dump's content
    does not depend on which, because the guard's ring and flags freeze on the device at the detection sub-step."""
    if self._graph is not None:
      self._action_buf.copy_(action, non_blocking=True)
      self._graph.replay()
      out = self._graph_out
    else:
      out = self._step_impl(action)
    if self._nan_guard is not None:
      self._nan_guard.poll()
    return out

  def _step_impl(self, action: torch.Tensor):
    n = self.num_envs
    U = self._rand(n, 48 + 4 * self.nu)  # B2_TRACKENV_NU: every random number of this env step (include/b2sim.h)
    self.events.draw(self._rand)         # (and those of the reset and interval events, when there are any)
    self.obs_groups.draw(self._rand, self._randn)  # (and the observation noise's, when a term draws)
    if self.native_mdp:
      return self._step_native(action, U)
    return self._step_torch(action, U)

  def _native_setup(self) -> None:
    """Argument block of the fused kernels: device pointers of the env's own tensors (all persistent)."""
    n, nu, dev = self.num_envs, self.nu, torch.device(self.device)
    f32 = dict(dtype=torch.float32, device=dev)
    nb = len(BODY_NAMES)
    self._U = torch.zeros(n, 48 + 4 * nu, **f32)
    self._act = torch.zeros(n, nu, **f32)
    self._reward = torch.zeros(n, **f32)
    self._term = torch.zeros(n, dtype=torch.bool, device=dev)
    self._trunc = torch.zeros(n, dtype=torch.bool, device=dev)
    self._obs = torch.zeros(n, 5 * nu + (15 if self.cfg.policy_state_estimation else 9), **f32)
    self._critic = torch.zeros(n, 5 * nu + 15 + 9 * nb, **f32)
    self._body_idx32 = self.robot.indexing.body_ids[self.body_idx].to(torch.int32).contiguous()
    self._ee_idx32 = self.ee_idx.to(torch.int32).contiguous()
    lim = self.robot.soft_joint_pos_limits
    self._soft_lo, self._soft_hi = lim[0, :, 0].contiguous(), lim[0, :, 1].contiguous()
    self.body_pos_relative_w = self.body_pos_relative_w.contiguous()
    self.body_quat_relative_w = self.body_quat_relative_w.contiguous()
    A = native.B2TrackEnvArgs()
    ptr = dict(action=self._act, U=self._U, default_joint_pos=self.default_joint_pos, soft_lo=self._soft_lo,
               soft_hi=self._soft_hi, env_origins=self.env_origins, m_joint_pos=self.motion["joint_pos"],
               m_joint_vel=self.motion["joint_vel"], m_body_pos=self.motion["body_pos_w"],
               m_body_quat=self.motion["body_quat_w"], m_body_lin=self.motion["body_lin_vel_w"],
               m_body_ang=self.motion["body_ang_vel_w"], body_idx=self._body_idx32, ee_idx=self._ee_idx32,
               time_steps=self.time_steps, episode_length=self.episode_length_buf, last_action=self.last_action,
               push_time_left=self.push_time_left, body_pos_rel=self.body_pos_relative_w,
               body_quat_rel=self.body_quat_relative_w, reward=self._reward, terminated=self._term,
               truncated=self._trunc, mask=self._done_buf, log_row=self.log_row, obs=self._obs, critic=self._critic)
    for k, t in ptr.items():
      assert t.is_contiguous(), k
      setattr(A, k, t.data_ptr())
    for k in range(6):
      A.pose_range[2 * k], A.pose_range[2 * k + 1] = self.cfg.pose_range[k]
      A.vel_range[2 * k], A.vel_range[2 * k + 1] = self.cfg.velocity_range[k]
    A.step_dt = self.step_dt
    A.jp_lo, A.jp_hi = self.cfg.joint_position_range
    A.push_lo, A.push_hi = self.cfg.push_interval_s
    A.nb, A.nee, A.anchor, A.T = nb, len(EE_NAMES), self.anchor, self.T
    A.self_collision_adr = self.self_collision_adr[0]
    A.root_body = int(self.robot.indexing.root_body_id)
    A.max_episode_length = self.max_episode_length
    A.adaptive = self.start_mode
    if self.start_mode == native.START_ADAPTIVE:
      sampler = dict(adaptive_kernel=self._bin_kernel, cdf=self._cdf, bin_fail_ema=self.bin_failed_count,
                     bin_fail_cur=self._bin_failed_cur, metrics=self._metrics)
      for k, t in sampler.items():
        assert t.is_contiguous() and t.dtype == torch.float32, k
        setattr(A, k, t.data_ptr())
      ptr.update(sampler)
      A.adaptive_alpha, A.adaptive_uniform_ratio = self.cfg.adaptive_alpha, self.cfg.adaptive_uniform_ratio
      A.nbins, A.adaptive_kernel_size = self.bin_count, self.cfg.adaptive_kernel_size
    A.weight[:] = self.reward_weights
    A.std2[:] = [s**2 for s in self.reward_stds]  # (the fp32 value of the double the torch path divides by)
    for k, v in enumerate(self.term_thresholds):
      A.term_on[k], A.term_threshold[k] = v is not None, 0.0 if v is None else v
    if self.cfg.push_velocity_range is not None:
      A.push_on = 1
      for k in range(6):
        A.push_range[2 * k], A.push_range[2 * k + 1] = self.cfg.push_velocity_range[k]
    A.policy_state_estimation, A.policy_corruption = self.cfg.policy_state_estimation, self.cfg.policy_corruption
    if self.cfg.episode_logs:
      logs = dict(episode_sums=self.episode_sums, finished_sums=self.finished_sums, term_flags=self.term_flags,
                  motion_metrics=self.motion_metrics, finished_metrics=self.finished_metrics)
      for k, t in logs.items():
        assert t.is_contiguous() and t.dtype == torch.float32, k
        setattr(A, k, t.data_ptr())
      ptr.update(logs)
    self._native_args = A
    self._keep = ptr
    self.obs_groups.bind({"policy": self._obs, "critic": self._critic}, self._term, self._trunc)
    # (the interval push and wrench run after post2's observations, from the forward's cvel)
    self.events.bind(self._term, self._trunc, self._done_buf, interval_after_obs=True)

  def _step_native(self, action: torch.Tensor, U: torch.Tensor):
    """Two fused kernels around the masked forward (csrc/b2_trackenv.cuh) instead of ~150 torch launches."""
    import ctypes

    if getattr(self, "_native_args", None) is None:
      self._native_setup()
    sim = self.sim
    self._U.copy_(U)
    self._act.copy_(action)
    native.check(sim._lib.b2_velenv_pre(sim._h, ctypes.c_void_p(self._act.data_ptr()),
                                        ctypes.c_void_p(self.default_joint_pos.data_ptr()),
                                        ctypes.c_void_p(self.action_scale.data_ptr()), sim._stream()))
    sim.step_n(self.cfg.decimation)
    return self._mdp_native(self._act, self._U)

  def _mdp_native(self, action: torch.Tensor, U: torch.Tensor):
    """Everything after the sub-steps on the fused path: post1 (and the sampler's bins), the reset and interval
    events (b2_events, when configured), the forward of the reset envs, post2, and the observation groups' clip, scale
    and history (b2_obs_history, when configured)."""
    import ctypes

    if getattr(self, "_native_args", None) is None:
      self._native_setup()
    sim = self.sim
    st = sim._stream()
    if action is not self._act:  # (the kernels read their own two input buffers)
      self._act.copy_(action)
    if U is not self._U:
      self._U.copy_(U)
    native.check(sim._lib.b2_trackenv_post1(sim._h, ctypes.byref(self._native_args), st))
    if self.start_mode == native.START_ADAPTIVE:
      native.check(sim._lib.b2_trackenv_bins(sim._h, ctypes.byref(self._native_args), st))
    self.events.run_native(sim)
    sim.forward(env_mask=self._done_buf)
    native.check(sim._lib.b2_trackenv_post2(sim._h, ctypes.byref(self._native_args), st))
    self.events.run_native_after_obs(sim)
    out = self.obs_groups.run_native(sim, {"policy": self._obs, "critic": self._critic})
    return out["policy"], self._reward, self._term, self._trunc, self._extras(out["critic"])

  def _step_torch(self, action: torch.Tensor, U: torch.Tensor):
    self.sim.data.ctrl[:] = self.default_joint_pos + self.action_scale * action  # JointPositionAction, use_default_offset
    self.sim.step_n(self.cfg.decimation)
    return self._mdp_torch(action, U)

  def _mdp_torch(self, action: torch.Tensor, U: torch.Tensor):
    """Everything after the sub-steps, in torch ops on the env's own tensors.  It returns fresh tensors and leaves the
    fused path's output buffers alone, so an env built with ``native_mdp=True`` can run it too (the tests compare the
    two on one state)."""
    cfg, d, n, nu = self.cfg, self.sim.data, self.num_envs, self.nu
    S = 13 + nu
    self.episode_length_buf += 1
    pos, quat, lin, ang = self._robot_bodies()
    a_pos = self._clip("body_pos_w")[:, self.anchor] + self.env_origins
    a_quat = self._clip("body_quat_w")[:, self.anchor]
    r_pos, r_quat = pos[:, self.anchor], quat[:, self.anchor]
    # terminations (tracking_env_cfg.py:253-278); a removed term never fires
    truncated = self.episode_length_buf >= self.max_episode_length
    th, never = self.term_thresholds, torch.zeros_like(truncated)
    bad_z = (a_pos[:, 2] - r_pos[:, 2]).abs() > th[0] if th[0] is not None else never
    g = self.robot.gravity_vec_w
    bad_ori = ((quat_apply_inverse(a_quat, g)[:, 2] - quat_apply_inverse(r_quat, g)[:, 2]).abs() > th[1]
               if th[1] is not None else never)
    ee_err = (self.body_pos_relative_w[:, self.ee_idx, 2] - pos[:, self.ee_idx, 2]).abs()
    bad_ee = (ee_err > th[2]).any(dim=1) if th[2] is not None else never
    terminated = bad_z | bad_ori | bad_ee
    if self.start_mode == native.START_ADAPTIVE:  # failures, in the bin of the frame reached (commands.py:257-265)
      fail_bin = (self.time_steps * self.bin_count // self.T).clamp_(0, self.bin_count - 1)
      self._bin_failed_cur.index_add_(0, fail_bin, terminated.float())
    # rewards (:200-250): each term times its weight; a term at weight 0 is not evaluated
    W, sd = self.reward_weights, self.reward_stds
    jp, lim = d.qpos[:, 7:], self.robot.soft_joint_pos_limits
    terms = (
      lambda: torch.exp(-((a_pos - r_pos) ** 2).sum(-1) / sd[0]**2),
      lambda: torch.exp(-quat_error_magnitude(a_quat, r_quat) ** 2 / sd[1]**2),
      lambda: torch.exp(-((self.body_pos_relative_w - pos) ** 2).sum(-1).mean(-1) / sd[2]**2),
      lambda: torch.exp(-(quat_error_magnitude(self.body_quat_relative_w, quat) ** 2).mean(-1) / sd[3]**2),
      lambda: torch.exp(-((self._clip("body_lin_vel_w") - lin) ** 2).sum(-1).mean(-1) / sd[4]**2),
      lambda: torch.exp(-((self._clip("body_ang_vel_w") - ang) ** 2).sum(-1).mean(-1) / sd[5]**2),
      lambda: ((action - self.last_action) ** 2).sum(1),
      lambda: ((lim[..., 0] - jp).clamp(min=0) + (jp - lim[..., 1]).clamp(min=0)).sum(1),
      lambda: d.sensordata[:, self.self_collision_adr[0]])
    zero = torch.zeros(n, device=self.device)
    vals = [W[i] * f() if W[i] != 0.0 else zero for i, f in enumerate(terms)]
    r = None
    for i, v in enumerate(vals):
      if W[i] != 0.0:
        r = v if r is None else r + v
    reward = (zero if r is None else r) * self.step_dt
    self.last_action.copy_(action)
    done = terminated | truncated
    self.log_row.copy_(torch.stack([reward, terminated.float(), truncated.float()], dim=1))
    # episode logs (RewardManager / TerminationManager), kept only with episode_logs, as on the fused kernels: a done
    # env's sums end their episode
    dk = done.unsqueeze(1)
    if cfg.episode_logs:
      sums = self.episode_sums + torch.stack(vals, dim=1) * self.step_dt
      self.finished_sums.copy_(torch.where(dk, sums, self.finished_sums))
      self.episode_sums.copy_(torch.where(dk, 0.0, sums))
      self.term_flags.copy_(torch.stack([truncated, bad_z, bad_ori, bad_ee], dim=1).float())
      # motion errors (MotionCommand._update_metrics): a done env hands over those of the last update; every other
      # env takes them now, at its frame before the clip steps (a done env takes its own after the forward, below)
      self.finished_metrics.copy_(torch.where(dk, self.motion_metrics, self.finished_metrics))
      e = self._motion_errors(self.time_steps, pos, quat, lin, ang)
      self.motion_metrics.copy_(torch.where(dk, self.motion_metrics, e))
    # reset onto the clip (RSI); then the clip's time step: envs that ran off its end restart on it.  Both rewrite
    # the whole state of their envs, so one forward over the union follows (the reference runs one per event).  An
    # env reset onto the clip's last frame is restarted in the same step, so its state is written twice before that
    # forward and the motion errors it takes after it see the second state (the reference sees the first)
    self._resample(done, done, U[:, 0:S])
    self.episode_length_buf.copy_(torch.where(done, torch.zeros_like(self.episode_length_buf), self.episode_length_buf))
    self.last_action.copy_(torch.where(done.unsqueeze(1), torch.zeros_like(self.last_action), self.last_action))
    self.time_steps += 1
    ended = self.time_steps >= self.T
    self._resample(ended, ended, U[:, S:2 * S])
    if self.start_mode == native.START_ADAPTIVE:
      self._sampler_step()
    self.events.step_torch(terminated, truncated)  # reset, then interval events (before the forward, as b2_events)
    self._done_buf.copy_(done | ended)
    self.sim.forward(env_mask=self._done_buf)
    # a done env's motion errors: its reset state against the frame before the clip stepped and the stale targets
    if cfg.episode_logs:
      e = self._motion_errors((self.time_steps - 1).clamp(min=0), *self._robot_bodies())
      self.motion_metrics.copy_(torch.where(dk, e, self.motion_metrics))
    self._update_command()
    # interval push (push_by_setting_velocity, tracking_env_cfg.py:155-161); none without a push range
    if self._push_r is not None:
      pr = self._push_r
      self.push_time_left -= self.step_dt
      push = self.push_time_left <= 0
      P = U[:, 2 * S:2 * S + 7]
      vel_w = self.robot.root_link_vel_w + P[:, 0:6] * (pr[:, 1] - pr[:, 0]) + pr[:, 0]
      vel = torch.cat([vel_w[:, 0:3], quat_apply_inverse(self.robot.root_link_quat_w, vel_w[:, 3:6])], dim=1)
      d.qvel[:, 0:6] = torch.where(push.unsqueeze(1), vel, d.qvel[:, 0:6])
      lo_t, hi_t = cfg.push_interval_s
      self.push_time_left.copy_(torch.where(push, P[:, 6] * (hi_t - lo_t) + lo_t, self.push_time_left))
    policy, critic = self.observations(U[:, 2 * S + 7:])
    out = self.obs_groups.update({"policy": policy, "critic": critic}, terminated | truncated)
    self.events.step_interval_state()  # the interval push and wrench terms, after the observations
    return out["policy"], reward, terminated, truncated, self._extras(out["critic"])

  def render(self) -> np.ndarray | None:
    """The reference's ``env.render()``: None with ``render_mode=None``, else an (height, width, 3) uint8 frame of
    ``cfg.viewer``'s camera, drawn on the GPU after the last step."""
    return env_render(self._offline_renderer, self.update_visualizers if self.cfg.debug_vis else None)

  def ghost_qpos(self, env_idx: int) -> torch.Tensor:
    """(nq,) pose of the motion's current frame for one env (commands.py:410-414): the first tracked body's (the
    pelvis's) position plus the env origin and its orientation as the free joint, the clip's joint positions."""
    ix = self.robot.indexing
    ts = self.time_steps[env_idx:env_idx + 1]
    q = torch.zeros(self.nq, dtype=torch.float32, device=self.device)
    q[ix.free_joint_q_adr[:3]] = self.motion["body_pos_w"][ts, 0][0] + self.env_origins[env_idx]
    q[ix.free_joint_q_adr[3:7]] = self.motion["body_quat_w"][ts, 0][0]
    q[ix.joint_q_adr] = self.motion["joint_pos"][ts][0]
    return q

  def update_visualizers(self, visualizer) -> None:
    """The motion command's ghost for ``visualizer.env_idx`` (commands.py:400-416), built on the device."""
    if visualizer.env_idx >= self.num_envs:
      return
    visualizer.add_ghost_mesh(self.ghost_qpos(visualizer.env_idx), self.cfg.ghost_color)

  def close(self):
    if self._offline_renderer is not None:
      self._offline_renderer.close()
    self.sim.close()

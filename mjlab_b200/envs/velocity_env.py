"""Slim velocity-tracking flat-terrain environment: the *caller* of the hot path.

Follows the control flow of the reference's ``ManagerBasedRlEnv.step``
(``src/mjlab/envs/manager_based_rl_env.py:106-147``) for the velocity task
(``tasks/velocity/velocity_env_cfg.py``): process action -> ``decimation`` x {write ctrl,
``sim.step``} -> terminations -> rewards -> reset terminated envs + ``sim.forward`` -> commands
-> interval push event -> observations.  The manager/term machinery is not rebuilt (out of scope,
SURVEY.md §2 rows 6-8); terms are fused torch expressions and resets are mask-based so the step
has no host synchronisation.
"""

from __future__ import annotations

import math
import re
from dataclasses import dataclass, field

import numpy as np
import torch

from mjlab_b200.asset_zoo import g1, go1, load_compiled
from mjlab_b200.entity_data import EntityIndexing, quat_apply
from mjlab_b200.envs import events as evm
from mjlab_b200.envs.events import Events, EventsCfg, PushBySettingVelocityCfg, RandomizeFieldCfg
from mjlab_b200.envs.noise import TaskNoise, velocity_defaults
from mjlab_b200.envs.obs_history import Observations, ObservationsCfg
from mjlab_b200.render import RENDER_MODES, ViewerConfig, check_render_mode, env_render, env_renderer, task_viewer
from mjlab_b200.sim import MujocoCfg, Simulation, SimulationCfg


REWARD_TERMS = ("track_lin_vel_exp", "track_ang_vel_exp", "pose", "dof_pos_limits", "action_rate_l2",  # fixed
                "air_time", "feet_slide", "foot_clearance", "is_alive", "is_terminated", "joint_torques_l2",
                "joint_acc_l2", "electrical_power_cost", "flat_orientation_l2")  # opt-in (VelocityRewardsCfg)
NFIXED = 5
# the terms of both observation groups, in frame order (velocity_env_cfg.py:86-131); elements per term
OBS_TERMS = ("base_lin_vel", "base_ang_vel", "projected_gravity", "joint_pos", "joint_vel", "actions", "command")


def obs_terms(nu: int) -> list[tuple[str, int]]:
  return list(zip(OBS_TERMS, (3, 3, 3, nu, nu, nu, 3)))


@dataclass
class VelocityRewardsCfg:
  """Reward terms the reference's velocity task offers beside the five fixed ones (tasks/velocity/mdp/rewards.py:52-190,
  envs/mdp/rewards.py:22-127), each off at weight 0: a term at weight 0 is not evaluated and its state does not
  advance (reward_manager.py:82-84).  Sensor and geom names are the robot's own (without the ``robot/`` prefix)."""

  air_time: float = 0.0
  feet_slide: float = 0.0
  foot_clearance: float = 0.0
  is_alive: float = 0.0
  is_terminated: float = 0.0
  joint_torques_l2: float = 0.0
  joint_acc_l2: float = 0.0
  electrical_power_cost: float = 0.0
  flat_orientation_l2: float = 0.0
  # feet_air_time (velocity_env_cfg.py:201-214); sensor_names None: the model's *_foot_ground_contact sensors
  air_time_sensor_names: tuple | None = None
  threshold_min: float = 0.05
  threshold_max: float = 0.15
  command_threshold: float = 0.05
  reward_mode: str = "on_landing"          # "on_landing" | "continuous"
  command_scale_type: str = "smooth"       # "smooth" | "hard"
  command_scale_width: float = 0.2
  # feet_slide: one geom per contact sensor
  feet_slide_sensor_names: tuple = ()
  feet_slide_geom_names: tuple = ()
  # foot_clearance_reward: no defaults in the reference, required at a non-zero weight
  target_height: float | None = None
  std: float | None = None
  tanh_mult: float | None = None
  foot_clearance_geom_names: tuple = ()


@dataclass
class VelocityCommandCfg:
  """The task's UniformVelocityCommandCfg (velocity_env_cfg.py:66-83, tasks/velocity/mdp/velocity_command.py:179-203):
  (lo, hi) ranges of the commanded body-frame velocities and the heading target, the heading controller's gain, the
  share of standing envs (zero command) and the resampling timer in seconds.  Every env is a heading env
  (rel_heading_envs 1) and none starts at its command's velocity (init_velocity_prob 0), as in all of the reference's
  velocity tasks."""

  lin_vel_x: tuple = (-1.0, 1.0)
  lin_vel_y: tuple = (-0.5, 0.5)
  ang_vel_z: tuple = (-1.0, 1.0)
  heading: tuple = (-math.pi, math.pi)
  heading_control_stiffness: float = 0.5
  rel_standing_envs: float = 0.1
  resampling_time_range: tuple = (3.0, 8.0)
  # the command's arrows in env.render() frames (velocity_command.py:106-177): commanded and actual planar velocity
  # and yaw rate of cfg.viewer.env_idx, drawn viz.z_offset above the root and scaled by viz.scale
  debug_vis: bool = False

  @dataclass
  class VizCfg:
    z_offset: float = 0.2
    scale: float = 0.75

  viz: VizCfg = field(default_factory=VizCfg)

  def __post_init__(self):
    self.check()

  def check(self) -> None:
    for k in ("lin_vel_x", "lin_vel_y", "ang_vel_z", "heading", "resampling_time_range"):
      lo, hi = getattr(self, k)
      if not lo <= hi:
        raise ValueError(f"command {k}: lo {lo} > hi {hi}")
    if not 0.0 <= self.rel_standing_envs <= 1.0:
      raise ValueError(f"command rel_standing_envs must lie in [0, 1], not {self.rel_standing_envs}")
    if not self.resampling_time_range[0] > 0.0:
      raise ValueError(f"command resampling_time_range must be positive, not {self.resampling_time_range}")


@dataclass
class VelocityEnvCfg:
  robot: str = "g1"
  num_envs: int = 4096
  decimation: int = 4                      # velocity_env_cfg.py:271
  episode_length_s: float = 20.0           # :272
  fall_angle: float = math.radians(70.0)   # :241-243
  push_interval_s: tuple = (1.0, 3.0)      # :156-161
  push_vel: float | None = 0.5             # flat_env_cfg.py:20-24; None: no built-in push
  friction_range: tuple = (0.3, 1.2)       # :162-172
  env_spacing: float = 2.5
  terrain: str = "flat"                    # "flat" (plane) | "rough" (box terrain, velocity_env_cfg.py:274-278)
  max_init_terrain_level: int = 5          # terrain_importer.py:203-223
  # terrain-level curriculum (velocity_env_cfg.py:228-230, mdp/curriculums.py:18-52): after every episode a robot
  # moves a row up or down the terrain grid by how far it walked; needs a terrain with sub-terrain origins
  terrain_curriculum: bool = False
  terrain_size: tuple = (8.0, 8.0)         # sub-terrain size the model's terrain grid was generated with
  seed: int = 42
  sim: SimulationCfg = field(
    default_factory=lambda: SimulationCfg(
      nconmax=140_000, njmax=300,
      mujoco=MujocoCfg(timestep=0.005, iterations=10, ls_iterations=20),
    )
  )
  rewards: VelocityRewardsCfg = field(default_factory=VelocityRewardsCfg)  # opt-in terms beside the fixed five
  command: VelocityCommandCfg = field(default_factory=VelocityCommandCfg)
  # command-velocity curriculum (commands_vel, tasks/velocity/mdp/curriculums.py:55-74): (step, (lo, hi)) stages; in
  # a step, lin_vel_x and ang_vel_z take the range of the last stage in list order whose step is below the step's
  # common_step_counter.  Empty: off
  command_curriculum: tuple = ()
  # per-joint widths of the posture reward (posture, envs/mdp/rewards.py:73-104): {joint regex: std}, every joint
  # matched by exactly one pattern and every pattern by some joint.  None: one width of 0.3 for every joint
  posture_std: dict | None = None
  # clip, scale and history of the policy and critic groups (terms: OBS_TERMS); the defaults leave both as computed
  observations: ObservationsCfg = field(default_factory=ObservationsCfg)
  # event terms (envs/events.py), run after the startup foot friction of friction_range: randomize_field, and the
  # state terms push_by_setting_velocity (needs push_vel=None) and apply_external_force_torque
  events: EventsCfg = field(default_factory=EventsCfg)
  # the camera of env.render() with render_mode="rgb_array" (velocity_env_cfg.py:41-48; the robot's cfg names the body,
  # velocity_task_cfg sets it)
  viewer: ViewerConfig = field(default_factory=task_viewer)

  def __post_init__(self):
    self.check()

  def check(self) -> None:
    self.events.check()
    if self.push_vel is not None and self.events.has(PushBySettingVelocityCfg):
      raise ValueError("a PushBySettingVelocityCfg term needs push_vel=None: the built-in push also writes the root "
                       "velocity, and it runs before the observations, where it cannot take the term's place in the "
                       "list order")


def _float32(x) -> float:
  return float(np.float32(x))


def _mid_half(lo: float, hi: float) -> tuple[float, float]:
  """A range as the kernel draws it, mid + (2u - 1) half, in fp32."""
  return _float32((lo + hi) / 2), _float32((hi - lo) / 2)


# the reference's velocity tasks with a model here (tasks/velocity/config/*/__init__.py), as their cfg classes set them
# (UnitreeG1FlatEnvCfg, UnitreeGo1FlatEnvCfg, UnitreeGo1RoughEnvCfg; the command curriculum of velocity_env_cfg.py:232-241)
_GO1_COMMAND_STAGES = ((500 * 24, (-3.0, 3.0)),)
VELOCITY_TASKS = {
  "Mjlab-Velocity-Flat-Unitree-G1": dict(robot="g1", terrain="flat", push_vel=0.5, posture_std=g1.POSTURE_STD),
  "Mjlab-Velocity-Flat-Unitree-Go1": dict(robot="go1", terrain="flat", push_vel=1.0, posture_std=go1.POSTURE_STD,
                                          command_curriculum=_GO1_COMMAND_STAGES),
  "Mjlab-Velocity-Rough-Unitree-Go1": dict(robot="go1", terrain="rough", terrain_curriculum=True, push_vel=1.0,
                                           posture_std=go1.POSTURE_STD, command_curriculum=_GO1_COMMAND_STAGES),
}


# the robots' camera overrides (config/g1/rough_env_cfg.py:71, config/go1/rough_env_cfg.py:46-48)
VIEWERS = {"g1": dict(body_name="torso_link"), "go1": dict(body_name="trunk", distance=1.5, elevation=-10.0)}


def velocity_task_cfg(name: str, **overrides) -> VelocityEnvCfg:
  """The VelocityEnvCfg of one of the reference's velocity tasks by its registered name, with `overrides` (any
  VelocityEnvCfg field, e.g. num_envs) on top.  The presets leave the command's debug visualisation off, so their
  frames show the scene alone; the reference's tasks turn it on, which `command=VelocityCommandCfg(debug_vis=True)`
  does here."""
  if name not in VELOCITY_TASKS:
    raise ValueError(f"unknown velocity task {name!r}; known: {', '.join(VELOCITY_TASKS)}")
  preset = dict(VELOCITY_TASKS[name])
  preset["posture_std"] = dict(preset["posture_std"])
  preset["viewer"] = task_viewer(**VIEWERS[preset["robot"]])
  return VelocityEnvCfg(**{**preset, **overrides})


def resolve_posture_std(posture_std: dict, joint_names: list[str]) -> list[float]:
  """One std per joint from {regex: std}, by resolve_matching_names_values' rules (re.fullmatch): a joint matched by
  two patterns or by none, or a pattern that matches no joint, is a ValueError."""
  out = []
  used = set()
  for j in joint_names:
    hits = [p for p in posture_std if re.fullmatch(p, j)]
    if len(hits) != 1:
      raise ValueError(f"posture_std: joint '{j}' is matched by {len(hits)} patterns {hits}, not exactly one")
    used.add(hits[0])
    out.append(float(posture_std[hits[0]]))
  unused = [p for p in posture_std if p not in used]
  if unused:
    raise ValueError(f"posture_std: patterns {unused} match no joint")
  if not all(v > 0.0 for v in out):
    raise ValueError("posture_std: every std must be positive")
  return out


def _resolve(pattern_map: dict, names: list[str], default: float) -> list[float]:
  out = []
  for n in names:
    for pat, v in pattern_map.items():
      if re.match(pat, n):
        out.append(v)
        break
    else:
      out.append(default)
  return out


# (rgba of the commanded and actual planar velocity and yaw rate arrows, velocity_command.py:146-177; width 0.015)
VELOCITY_ARROW_COLORS = ((0.2, 0.2, 0.6, 0.6), (0.2, 0.6, 0.2, 0.6), (0.0, 0.6, 1.0, 0.7), (0.0, 1.0, 0.4, 0.7))
VELOCITY_ARROW_WIDTH = 0.015


def velocity_arrows(pos, quat, cmd, lin_vel_b, ang_vel_b, z_offset: float, scale: float) -> torch.Tensor:
  """(4, 2, 3) world (from, to) of the command's arrows for one env (velocity_command.py:135-177): commanded and
  actual planar velocity, commanded and actual yaw rate, from (0, 0, z_offset)·scale in the root frame."""
  z = torch.zeros(4, 2, 3, dtype=pos.dtype, device=pos.device)
  z[..., 2] = z_offset
  z[0, 1, :2], z[2, 1, :2] = cmd[:2], lin_vel_b[:2]
  z[1, 1, 2] += cmd[2]
  z[3, 1, 2] += ang_vel_b[2]
  return pos + quat_apply(quat.expand(8, 4), (z * scale).reshape(8, 3)).reshape(4, 2, 3)


def quat_rotate_inverse(q: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
  w, u = q[:, 0:1], q[:, 1:4]
  t = 2.0 * torch.cross(u, v, dim=-1)
  return v - w * t + torch.cross(u, t, dim=-1)


class VelocityFlatEnv:
  metadata = {"render_modes": RENDER_MODES}

  def __init__(self, cfg: VelocityEnvCfg, device: str = "cuda:0", model=None, native_mdp: bool = True,
               render_mode: str | None = None):
    check_render_mode(render_mode)
    self.cfg = cfg
    self.device = device
    zoo = g1 if cfg.robot == "g1" else go1
    self.model = model if model is not None else load_compiled(f"{cfg.robot}_{cfg.terrain}")
    m = self.model
    self.terrain_curriculum = bool(cfg.terrain_curriculum)
    if self.terrain_curriculum and "terrain_origins" not in m.arrays:
      raise ValueError(f"terrain_curriculum needs a terrain with sub-terrain origins; '{cfg.terrain}' has none")
    self.num_envs = cfg.num_envs
    self.sim = Simulation(cfg.num_envs, cfg.sim, m, device)
    self._nan_guard = getattr(self.sim, "nan_guard", None)  # (None on a Simulation stand-in without the guard)
    self.nq, self.nv, self.nu = int(m.nq), int(m.nv), int(m.nu)
    self.step_dt = cfg.decimation * float(m.opt_timestep)
    self.max_episode_length = math.ceil(cfg.episode_length_s / self.step_dt)
    dev = torch.device(device)
    self.gen = torch.Generator(device=dev)
    self.gen.manual_seed(cfg.seed)
    key = m.keys["robot/init_state"]
    f32 = dict(dtype=torch.float32, device=dev)
    self.default_qpos = torch.tensor(key["qpos"], **f32)
    self.default_joint_pos = self.default_qpos[7:].clone()
    jnames = [n.split("/")[-1] for n in m.names["joint"][1:]]
    self.action_scale = torch.tensor(_resolve(zoo.ACTION_SCALE, jnames, 0.5), **f32)
    rng = torch.tensor(m.jnt_range[1:], **f32)
    mid, half = rng.mean(dim=1), 0.5 * (rng[:, 1] - rng[:, 0]) * 0.9  # soft limits (entity.py:372-380)
    self.soft_lo, self.soft_hi = mid - half, mid + half
    # env origins on a grid (terrain_importer.py:203-223 for the flat case)
    n = cfg.num_envs
    cols = math.ceil(math.sqrt(n))
    idx = torch.arange(n, device=dev)
    self.env_origins = torch.stack(
      [(idx // cols - (cols - 1) / 2) * cfg.env_spacing, (idx % cols - (cols - 1) / 2) * cfg.env_spacing,
       torch.zeros(n, device=dev)], dim=1).float()
    if "terrain_origins" in m.arrays:
      # sub-terrain grid: spawn on the sub-terrain origins, level <= max_init_terrain_level, types round-robin
      # (terrain_importer.py:203-223)
      from mjlab_b200.terrains import env_origins_curriculum

      origins = np.asarray(m.arrays["terrain_origins"])
      # origins sit at the sub-terrain centres, so consecutive rows are one sub-terrain length apart
      if self.terrain_curriculum and not np.allclose(np.diff(origins[:, :, 0], axis=0), cfg.terrain_size[0]):
        raise ValueError(f"terrain_size {cfg.terrain_size} does not match the model's terrain grid")
      org, levels, types = env_origins_curriculum(n, origins, cfg.max_init_terrain_level, cfg.seed)
      self.env_origins = torch.tensor(org, dtype=torch.float32, device=dev)
      self.terrain_origins = torch.tensor(origins, dtype=torch.float32, device=dev).contiguous()  # [rows, cols, 3]
      self.terrain_levels = torch.tensor(levels, dtype=torch.int32, device=dev)
      self.terrain_types = torch.tensor(types, dtype=torch.int32, device=dev)
      self.max_terrain_level = int(origins.shape[0])
      self.move_up_dist = 0.5 * float(cfg.terrain_size[0])
      # the mean level terrain_levels_vel returns for logging, kept on the device (updated by the curriculum)
      self.terrain_level_mean = self.terrain_levels.float().mean()
    # domain randomisation: the task's startup foot friction (velocity_env_cfg.py:162-172), then cfg.events; the
    # fields they name get a per-world copy first
    cfg.check()
    feet = RandomizeFieldCfg("geom_friction", tuple(cfg.friction_range), operation="abs", names=tuple(zoo.FOOT_GEOMS))
    self.events = Events((feet,) + tuple(cfg.events.terms), EntityIndexing.from_model(m, "robot", device), self.sim,
                         n, self.step_dt, device)
    self.events.set_reset_state(self.default_qpos, self.env_origins, self.soft_lo, self.soft_hi)
    self.sim.expand_model_fields(self.events.fields())
    self.events.run_startup(self._rand)
    self.events.draw_timers(self._rand)
    self.episode_length_buf = torch.zeros(n, dtype=torch.int32, device=dev)
    self.last_action = torch.zeros(n, self.nu, **f32)
    self.command = torch.zeros(n, 3, **f32)
    # UniformVelocityCommand state (velocity_env_cfg.py:66-83): resampling timer 3..8 s, heading control, 10 % standing
    self.cmd_time_left = torch.zeros(n, **f32)
    self.heading_target = torch.zeros(n, **f32)
    self.is_standing = torch.zeros(n, dtype=torch.bool, device=dev)
    self.log_row = torch.zeros(n, 3, **f32)  # (reward, terminated, truncated): the rank-0 log gather reads this
    self.push_time_left = torch.zeros(n, **f32)
    self._down = torch.tensor([0.0, 0.0, -1.0], **f32).expand(n, 3)  # gravity direction (world)
    self.native_mdp = bool(native_mdp)
    self._graph = None
    self._done_buf = torch.zeros(n, dtype=torch.bool, device=dev)  # fixed address (graph capture / native)
    lo_t, hi_t = cfg.push_interval_s
    self.push_time_left.copy_(self._rand(n) * (hi_t - lo_t) + lo_t)
    self._init_rewards()
    self._init_command(jnames)
    # noise-configured groups: the task's default noise (policy corrupted, critic not) on the noise-free critic frame
    task_noise = TaskNoise(velocity_defaults(), {"policy": True, "critic": False}, obs_terms(self.nu))
    self.obs_groups = Observations(cfg.observations, {g: obs_terms(self.nu) for g in ("policy", "critic")}, n, device,
                                   task_noise)
    self.nobs, self.nobs_critic = self.obs_groups.width("policy"), self.obs_groups.width("critic")  # elements per env
    if self.native_mdp:
      self._init_native()
    self._reset_all(curriculum=False)  # no episode has ended yet: the initial levels stand
    self.render_mode = render_mode
    self.metadata = {**self.metadata, "render_fps": 1.0 / self.step_dt}
    self._offline_renderer = env_renderer(self.sim, cfg.viewer, render_mode)
    self._vis = None  # the debug visualisation's EntityData and arrow colours, made at its first frame

  # -- helpers -----------------------------------------------------------------------------------
  def _rand(self, *shape):
    return torch.rand(shape, generator=self.gen, device=self.device)

  def _randn(self, *shape):
    return torch.randn(shape, generator=self.gen, device=self.device)

  def _draw(self) -> torch.Tensor:
    """The step's uniform numbers, one launch (layout: include/b2sim.h B2VelEnvArgs.U): 0-1 reset xy, 2 yaw,
    3-5 command, 6 heading target, 7 standing draw, 8 command timer, 9-10 push, 11 push timer, 12 terrain level
    redraw, 16.. obs noise."""
    return self._rand(self.num_envs, 16 + 9 + 2 * self.nu)

  def _init_rewards(self) -> None:
    """Resolve VelocityRewardsCfg against the model and allocate the air-time state and the episode sums."""
    rc, m, n = self.cfg.rewards, self.model, self.num_envs
    if rc.reward_mode not in ("on_landing", "continuous"):
      raise ValueError(f"reward_mode must be 'on_landing' or 'continuous', not {rc.reward_mode!r}")
    if rc.command_scale_type not in ("smooth", "hard"):
      raise ValueError(f"command_scale_type must be 'smooth' or 'hard', not {rc.command_scale_type!r}")
    self.reward_weights = [float(getattr(rc, t)) for t in REWARD_TERMS[NFIXED:]]
    sensors, geoms, intprm = m.names["sensor"], m.names["geom"], np.asarray(m.arrays["sensor_intprm"]).reshape(-1, 3)

    def lookup(kind, names, table):
      if len(names) > 32:
        raise ValueError(f"at most 32 feet per reward term, got {len(names)} {kind}s")
      ids = []
      for s in names:
        if f"robot/{s}" not in table:
          raise ValueError(f"unknown {kind} '{s}'")
        ids.append(table.index(f"robot/{s}"))
      return ids

    def contact_adr(names):
      ids = lookup("sensor", names, sensors)
      for s, i in zip(names, ids):
        if not intprm[i, 0] & 1:  # the data fields are packed found, force, ... (compiler/spec.py CONTACT_DATA)
          raise ValueError(f"sensor '{s}': its first data field is not 'found'")
      return [int(m.arrays["sensor_adr"][i]) for i in ids]

    air_names = rc.air_time_sensor_names
    if air_names is None:
      air_names = [s.split("/", 1)[1] for s in sensors if s.startswith("robot/") and s.endswith("_foot_ground_contact")]
    if len(rc.feet_slide_sensor_names) != len(rc.feet_slide_geom_names):
      raise ValueError(f"feet_slide needs one geom per sensor: {len(rc.feet_slide_sensor_names)} sensors, "
                       f"{len(rc.feet_slide_geom_names)} geoms")
    w_air, w_slide, w_clear = self.reward_weights[:3]
    if w_clear != 0.0 and None in (rc.target_height, rc.std, rc.tanh_mult):
      raise ValueError("foot_clearance needs target_height, std and tanh_mult")
    for w_, k, names in ((w_air, "air_time", air_names), (w_slide, "feet_slide", rc.feet_slide_sensor_names),
                         (w_clear, "foot_clearance", rc.foot_clearance_geom_names)):
      if w_ != 0.0 and not names:
        raise ValueError(f"{k} has a non-zero weight and no feet")
    i32 = dict(dtype=torch.int32, device=self.device)
    body = np.asarray(m.arrays["geom_bodyid"])
    self._air_adr = torch.tensor(contact_adr(air_names), **i32)
    self._slide_adr = torch.tensor(contact_adr(rc.feet_slide_sensor_names), **i32)
    self._slide_geom = torch.tensor(lookup("geom", rc.feet_slide_geom_names, geoms), **i32)
    self._clear_geom = torch.tensor(lookup("geom", rc.foot_clearance_geom_names, geoms), **i32)
    self._slide_body, self._clear_body = (torch.tensor(body[g.cpu().numpy()], **i32)
                                          for g in (self._slide_geom, self._clear_geom))
    self._root_body = int(m.arrays["body_rootid"][m.arrays["jnt_bodyid"][0]])  # the floating base's tree
    f32 = dict(dtype=torch.float32, device=self.device)
    nf = len(air_names)
    self.air_time, self.contact_time, self.last_air_time = (torch.zeros(n, nf, **f32) for _ in range(3))
    self.episode_sums = torch.zeros(n, len(REWARD_TERMS), **f32)
    self.finished_sums = torch.zeros(n, len(REWARD_TERMS), **f32)

  def _init_command(self, joint_names: list[str]) -> None:
    """The command's ranges in fp32 as the kernel draws them, the curriculum's stage table and counter, the posture
    widths, and the command's metrics."""
    cfg, n, dev = self.cfg, self.num_envs, self.device
    cc = cfg.command
    cc.check()
    self._cmd_mid_half = [_mid_half(*getattr(cc, k)) for k in ("lin_vel_x", "lin_vel_y", "ang_vel_z", "heading")]
    stages = list(cfg.command_curriculum)
    if len(stages) > 8:
      raise ValueError(f"command_curriculum: at most 8 stages, got {len(stages)}")
    for step, (lo, hi) in stages:
      if int(step) != step or not 0 <= step < 2 ** 31 or not lo <= hi:
        raise ValueError(f"command_curriculum: stage ({step}, ({lo}, {hi})) needs an integer step in [0, 2^31) and "
                         "lo <= hi")
    f32 = dict(dtype=torch.float32, device=dev)
    # (mid, half, lo, hi) of lin_vel_x and ang_vel_z as configured, and of each stage
    self._cmd_base = torch.tensor([[*self._cmd_mid_half[k], *getattr(cc, r)] for k, r in ((0, "lin_vel_x"),
                                                                                        (2, "ang_vel_z"))], **f32)
    self._stages = [(int(st), *_mid_half(lo, hi), _float32(lo), _float32(hi)) for st, (lo, hi) in stages]
    self._stage_step = torch.tensor([st[0] for st in self._stages], dtype=torch.int32, device=dev)
    self._stage_vals = torch.tensor([st[1:] for st in self._stages], **f32).reshape(-1, 4)
    # common_step_counter (manager_based_rl_env.py:117); it only advances with the command curriculum on, the one
    # thing that reads it
    self.common_step_counter = torch.zeros(1, dtype=torch.int32, device=dev)
    std = [0.3] * len(joint_names) if cfg.posture_std is None else resolve_posture_std(cfg.posture_std, joint_names)
    self.posture_inv_std2 = torch.tensor(1.0 / np.asarray(std, dtype=np.float64) ** 2, **f32)
    self.metric_steps = _float32(cc.resampling_time_range[1] / self.step_dt)
    self.metric_xy = torch.zeros(n, **f32)
    self.metric_yaw = torch.zeros(n, **f32)
    self.finished_metrics = torch.zeros(n, 2, **f32)

  def _command_ranges(self, counter: torch.Tensor):
    """[2, 4] (mid, half, lo, hi) of lin_vel_x and ang_vel_z at common_step_counter `counter`: those of the last stage
    in list order whose step is below it, or the cfg's (commands_vel, curriculums.py:55-74, which writes the stage's
    range into the cfg for good)."""
    if not self._stages:
      return self._cmd_base
    idx = torch.arange(len(self._stages), device=self.device)
    last = torch.where(counter > self._stage_step, idx, -1).max()
    return torch.where(last >= 0, self._stage_vals[last.clamp(min=0)], self._cmd_base)

  def command_log(self) -> dict:
    """``Metrics/twist/error_vel_xy`` and ``error_vel_yaw`` of CommandManager.reset (managers/command_manager.py:128-134,
    velocity_command.py:43-62) for the envs whose episode ended in the last step: the mean of their accumulated errors
    (NaN when none ended); with the command curriculum on also ``Curriculum/command_vel``, the upper lin_vel_x bound in
    effect.  Device tensors, no host synchronisation."""
    done = self._done_buf.unsqueeze(1)
    mean = torch.where(done, self.finished_metrics, 0.0).sum(0) / done.sum()
    out = {"Metrics/twist/error_vel_xy": mean[0], "Metrics/twist/error_vel_yaw": mean[1]}
    if self._stages:
      out["Curriculum/command_vel"] = self._command_ranges(self.common_step_counter)[0, 3]
    return out

  def reward_log(self) -> dict:
    """``Episode_Reward/<term>`` of RewardManager.reset (managers/reward_manager.py:61-75) for the envs whose episode
    ended in the last step: the mean of their episode sums over episode_length_s (NaN when none ended), for the fixed
    terms and the enabled ones.  Device tensors, no host synchronisation."""
    done = self._done_buf.unsqueeze(1)
    mean = torch.where(done, self.finished_sums, 0.0).sum(0) / done.sum() / self.cfg.episode_length_s
    return {f"Episode_Reward/{t}": mean[i] for i, t in enumerate(REWARD_TERMS)
            if i < NFIXED or self.reward_weights[i - NFIXED] != 0.0}

  def termination_log(self) -> dict:
    """``Episode_Termination/time_out`` and ``fell_over`` of TerminationManager.reset
    (managers/termination_manager.py:73-85): how many of the envs whose episode ended in the last step that term fired
    for (NaN when none ended).  Device tensors, no host synchronisation."""
    done = self._done_buf
    flags = torch.stack([self.log_row[:, 2], self.log_row[:, 1]], dim=1)  # (truncated, terminated) of the last step
    count = torch.where(done.any(), torch.count_nonzero(flags, dim=0).float(), math.nan)
    return {"Episode_Termination/time_out": count[0], "Episode_Termination/fell_over": count[1]}

  def _init_native(self) -> None:
    from mjlab_b200.sim import native

    n, dev = self.num_envs, self.device
    nframe = 9 + 3 * self.nu + 3
    self._obs = torch.zeros(n, nframe, device=dev)
    self._reward = torch.zeros(n, device=dev)
    self._term = torch.zeros(n, dtype=torch.bool, device=dev)
    self._trunc = torch.zeros(n, dtype=torch.bool, device=dev)
    self._U = torch.zeros(n, 16 + 9 + 2 * self.nu, device=dev)
    self._critic = torch.zeros(n, nframe, device=dev)
    self._action_in = torch.zeros(n, self.nu, device=dev)
    self._origins = self.env_origins.contiguous()
    a = native.B2VelEnvArgs()
    for name, t in (
      ("action", self._action_in), ("U", self._U), ("default_qpos", self.default_qpos),
      ("default_joint_pos", self.default_joint_pos), ("action_scale", self.action_scale),
      ("soft_lo", self.soft_lo), ("soft_hi", self.soft_hi), ("env_origins", self._origins),
      ("episode_length", self.episode_length_buf), ("last_action", self.last_action),
      ("command", self.command), ("push_time_left", self.push_time_left), ("obs", self._obs),
      ("reward", self._reward), ("terminated", self._term), ("truncated", self._trunc), ("done", self._done_buf),
      ("cmd_time_left", self.cmd_time_left), ("heading_target", self.heading_target),
      ("is_standing", self.is_standing), ("critic", self._critic), ("log_row", self.log_row),
    ):
      assert t.is_contiguous()
      setattr(a, name, t.data_ptr())
    a.step_dt, a.fall_angle = self.step_dt, self.cfg.fall_angle
    a.push_vel, a.push_off = (0.0, 1) if self.cfg.push_vel is None else (self.cfg.push_vel, 0)
    a.push_lo, a.push_hi = self.cfg.push_interval_s
    a.max_episode_length = self.max_episode_length
    if self.terrain_curriculum:
      for name, t in (("terrain_origins", self.terrain_origins), ("terrain_levels", self.terrain_levels),
                      ("terrain_types", self.terrain_types), ("terrain_level_mean", self.terrain_level_mean)):
        assert t.is_contiguous()
        setattr(a, name, t.data_ptr())
      a.move_up_dist, a.episode_length_s = self.move_up_dist, self.cfg.episode_length_s
      a.rows, a.cols = self.terrain_origins.shape[:2]
      a.curriculum = 1
    rc = self.cfg.rewards
    for name, t in (("air_sensor_adr", self._air_adr), ("slide_sensor_adr", self._slide_adr),
                    ("slide_geom", self._slide_geom), ("slide_body", self._slide_body), ("clear_geom", self._clear_geom),
                    ("clear_body", self._clear_body), ("air_time", self.air_time), ("contact_time", self.contact_time),
                    ("last_air_time", self.last_air_time), ("episode_sums", self.episode_sums),
                    ("finished_sums", self.finished_sums)):
      assert t.is_contiguous()
      setattr(a, name, t.data_ptr())
    a.weight[:] = self.reward_weights
    a.air_threshold_min, a.air_threshold_max = rc.threshold_min, rc.threshold_max
    a.air_command_threshold, a.air_command_scale_width = rc.command_threshold, rc.command_scale_width
    a.clearance_target_height, a.clearance_std, a.clearance_tanh_mult = (
      0.0 if v is None else v for v in (rc.target_height, rc.std, rc.tanh_mult))
    a.air_continuous, a.air_hard_scale = rc.reward_mode == "continuous", rc.command_scale_type == "hard"
    a.n_air, a.n_slide, a.n_clear = len(self._air_adr), len(self._slide_adr), len(self._clear_geom)
    a.root_body = self._root_body
    cc = self.cfg.command
    for k, (mid, half) in enumerate(self._cmd_mid_half):
      a.cmd_mid[k], a.cmd_half[k] = mid, half
    a.ang_lo, a.ang_hi = cc.ang_vel_z
    a.heading_stiffness, a.rel_standing = cc.heading_control_stiffness, cc.rel_standing_envs
    lo_t, hi_t = cc.resampling_time_range
    a.resample_lo, a.resample_span = lo_t, _float32(np.float32(hi_t) - np.float32(lo_t))
    a.n_stage = len(self._stages)
    for s, (step, mid, half, lo, hi) in enumerate(self._stages):
      a.stage_step[s], a.stage_mid[s], a.stage_half[s], a.stage_lo[s], a.stage_hi[s] = step, mid, half, lo, hi
    for name, t in (("step_counter", self.common_step_counter), ("posture_inv_std2", self.posture_inv_std2),
                    ("metric_xy", self.metric_xy), ("metric_yaw", self.metric_yaw),
                    ("finished_metrics", self.finished_metrics)):
      assert t.is_contiguous()
      setattr(a, name, t.data_ptr())
    a.metric_steps = self.metric_steps
    resets = self.events.reset_state_terms()  # reset_root_state_uniform / reset_joints_by_scale, in the reset branch
    if len(resets) > native.VELENV_NRESET:
      raise ValueError(f"at most {native.VELENV_NRESET} reset root and joint terms, got {len(resets)}")
    if resets:
      a.ev_V, a.ev_v_width, a.n_reset = self.events.V.data_ptr(), self.events.v_width, len(resets)
    for k, t in enumerate(resets):
      T = a.reset_term[k]
      T.kind = native.RESET_ROOT if t.kind == evm.ROOT else native.RESET_JOINTS
      T.col, T.count = t.col, t.count
      T.joint[:t.count if t.kind == evm.JOINTS else 0] = t.bodies
      T.lo[:len(t.lo)], T.span[:len(t.span)] = t.lo, t.span
    self._native_args = a
    self.obs_groups.bind({"policy": self._obs, "critic": self._critic}, self._term, self._trunc)
    self.events.bind(self._term, self._trunc, self._done_buf)

  def _reset_where(self, mask: torch.Tensor, U: torch.Tensor) -> None:
    """reset_root_state_uniform + reset_joints_by_scale (envs/mdp/events.py:43-124) for masked envs."""
    d = self.sim.data
    n = self.num_envs
    qpos = self.default_qpos.expand(n, -1).clone()
    qpos[:, 0:2] += (U[:, 0:2] - 0.5) + self.env_origins[:, 0:2]
    qpos[:, 2] += self.env_origins[:, 2]
    yaw = (U[:, 2] * 2 - 1) * 3.14
    qpos[:, 3] = torch.cos(0.5 * yaw)
    qpos[:, 6] = torch.sin(0.5 * yaw)
    qpos[:, 7:] = torch.minimum(torch.maximum(qpos[:, 7:], self.soft_lo), self.soft_hi)
    mk = mask.unsqueeze(1)
    # in-place updates everywhere: the step may be replayed from a CUDA graph (fixed addresses)
    d.qpos[:] = torch.where(mk, qpos, d.qpos[:])
    d.qvel[:] = torch.where(mk, torch.zeros_like(d.qvel[:]), d.qvel[:])
    d.ctrl[:] = torch.where(mk, self.default_joint_pos.expand(n, -1), d.ctrl[:])
    self.episode_length_buf.copy_(torch.where(mask, torch.zeros_like(self.episode_length_buf), self.episode_length_buf))
    self.last_action.copy_(torch.where(mk, torch.zeros_like(self.last_action), self.last_action))

  def _terrain_curriculum(self, mask: torch.Tensor, U: torch.Tensor) -> None:
    """terrain_levels_vel (tasks/velocity/mdp/curriculums.py:18-52) and TerrainImporter.update_env_origins
    (terrains/terrain_importer.py:186-201) for the masked envs, from the state of the episode that just ended: a robot
    that walked further than half a sub-terrain moves a row up, one that walked less than half of what its command
    asked for moves a row down, one past the last row is redrawn from U[:, 12].  Its reset spawns at the new origin."""
    o, c, root = self.env_origins, self.command, self.sim.data.qpos[:, 0:2]
    dx, dy = root[:, 0] - o[:, 0], root[:, 1] - o[:, 1]
    dist = torch.sqrt(dx * dx + dy * dy)
    up = dist > self.move_up_dist
    down = (dist < torch.sqrt(c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1]) * self.cfg.episode_length_s * 0.5) & ~up
    top = self.max_terrain_level
    level = self.terrain_levels + up.int() - down.int()
    redraw = torch.floor(U[:, 12] * top).int().clamp(max=top - 1)
    level = torch.where(level >= top, redraw, level.clamp(min=0))
    self.terrain_levels.copy_(torch.where(mask, level, self.terrain_levels))
    new = self.terrain_origins[self.terrain_levels.long(), self.terrain_types.long()]
    self.env_origins.copy_(torch.where(mask.unsqueeze(1), new, o))
    self.terrain_level_mean.copy_(self.terrain_levels.float().mean())

  def _geom_vel(self, geoms: torch.Tensor, bodies: torch.Tensor):
    """Height and world-frame linear velocity of geoms (EntityData.geom_vel_w, entity/data.py:20-31, 282-288)."""
    d = self.sim.data
    pos = d.geom_xpos[:, geoms.long()]
    cvel = d.cvel[:, bodies.long()]
    com = d.subtree_com[:, self._root_body].unsqueeze(1)
    return pos[..., 2], cvel[..., 3:6] - torch.cross(cvel[..., 0:3], com - pos, dim=-1)

  def _opt_in_rewards(self, terminated: torch.Tensor, done: torch.Tensor, grav_b: torch.Tensor) -> torch.Tensor:
    """The VelocityRewardsCfg terms from the pre-reset state, weighted ([n, 9]; zero for a term at weight 0, which is
    not evaluated).  Advances the air-time state, and zeroes it for the done envs (feet_air_time.reset)."""
    rc, d, W = self.cfg.rewards, self.sim.data, self.reward_weights
    out = torch.zeros(self.num_envs, len(W), device=self.device)
    if W[0] != 0.0:  # feet_air_time (tasks/velocity/mdp/rewards.py:84-146)
      contact = d.sensordata[:, self._air_adr.long()] > 0
      first = (self.air_time > 0) & contact
      last = torch.where(first, self.air_time, self.last_air_time)
      air = torch.where(contact, 0.0, self.air_time + self.step_dt)
      ct = torch.where(contact, self.contact_time + self.step_dt, 0.0)
      if rc.reward_mode == "continuous":
        r = (~contact & (air > rc.threshold_min) & (air <= rc.threshold_max)).float().sum(1)
      else:  # the span as the kernel forms it: one fp32 subtraction
        span = float(np.float32(rc.threshold_max) - np.float32(rc.threshold_min))
        r = ((last - rc.threshold_min).clamp(min=0.0).clamp(max=span) * first).sum(1) / self.step_dt
      c = self.command
      cn = torch.sqrt(c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1])
      if rc.command_scale_type == "smooth":
        r = r * (0.5 * (1.0 + torch.tanh((cn - rc.command_threshold) / rc.command_scale_width)))
      else:
        r = r * (cn > rc.command_threshold)
      out[:, 0] = r
      keep = ~done.unsqueeze(1)
      for t, v in ((self.air_time, air), (self.contact_time, ct), (self.last_air_time, last)):
        t.copy_(torch.where(keep, v, 0.0))
    if W[1] != 0.0:  # feet_slide (:174-187)
      _, v = self._geom_vel(self._slide_geom, self._slide_body)
      out[:, 1] = (v[..., :2].norm(dim=-1) * (d.sensordata[:, self._slide_adr.long()] > 0)).sum(1)
    if W[2] != 0.0:  # foot_clearance_reward (:156-171)
      z, v = self._geom_vel(self._clear_geom, self._clear_body)
      err = (z - rc.target_height) ** 2 * torch.tanh(rc.tanh_mult * v[..., :2].norm(dim=-1))
      out[:, 2] = torch.exp(-err.sum(1) / rc.std)
    nu = self.nu
    tau, qd = d.actuator_force[:, :nu], d.qvel[:, 6:]
    for i, f in ((3, lambda: (~terminated).float()), (4, lambda: terminated.float()),  # envs/mdp/rewards.py:22-127
                 (5, lambda: (tau ** 2).sum(1)), (6, lambda: (d.qacc[:, 6:] ** 2).sum(1)),
                 (7, lambda: (tau * qd).clamp(min=0.0).sum(1)), (8, lambda: (grav_b[:, :2] ** 2).sum(1))):
      if W[i] != 0.0:
        out[:, i] = f()
    return out * torch.tensor(W, device=self.device)

  def _posture(self, jp: torch.Tensor) -> torch.Tensor:
    """The pose reward (posture, envs/mdp/rewards.py:73-104): exp(-mean(d^2 / std^2)) with the per-joint widths of
    posture_std (0.3 for every joint without one)."""
    d2 = (jp - self.default_joint_pos) ** 2
    return torch.exp(-(d2 * self.posture_inv_std2).mean(1))

  def _update_command(self, done: torch.Tensor, U: torch.Tensor, metrics: bool = True) -> None:
    """CommandTerm.compute + UniformVelocityCommand (tasks/velocity/mdp/velocity_command.py:43-110): resample on
    reset and on timer expiry, heading control on every env, standing envs get a zero command.  A component is drawn
    as mid + (2u - 1) half.  With `metrics`, the command's error metrics first take this step's increment (a done env
    hands its sums over and restarts them)."""
    cc = self.cfg.command
    rng = self._command_ranges(self.common_step_counter)
    (ym, yh), (hm, hh) = self._cmd_mid_half[1], self._cmd_mid_half[3]
    ctl = self.cmd_time_left - self.step_dt
    rs = done | (ctl <= 0)
    cmd = torch.stack([rng[0, 0] + (U[:, 3] * 2 - 1) * rng[0, 1], ym + (U[:, 4] * 2 - 1) * yh,
                       rng[1, 0] + (U[:, 5] * 2 - 1) * rng[1, 1]], dim=1)
    old = self.command.clone()
    self.command.copy_(torch.where(rs.unsqueeze(1), cmd, self.command))
    self.heading_target.copy_(torch.where(rs, hm + (U[:, 6] * 2 - 1) * hh, self.heading_target))
    self.is_standing.copy_(torch.where(rs, U[:, 7] <= _float32(cc.rel_standing_envs), self.is_standing))
    lo_t, hi_t = cc.resampling_time_range
    span = _float32(np.float32(hi_t) - np.float32(lo_t))
    self.cmd_time_left.copy_(torch.where(rs, lo_t + span * U[:, 8], ctl))
    q = self.sim.data.qpos[:, 3:7]
    if metrics:  # _update_metrics (velocity_command.py:49-62) after CommandTerm.reset of the done envs
      d = self.sim.data
      m = torch.where(done.unsqueeze(1), cmd, old)
      vb = quat_rotate_inverse(q, d.qvel[:, 0:3])
      exy = (m[:, :2] - vb[:, :2]).norm(dim=1) / self.metric_steps
      eyaw = (m[:, 2] - d.qvel[:, 5]).abs() / self.metric_steps
      self.finished_metrics.copy_(torch.where(done.unsqueeze(1), torch.stack([self.metric_xy, self.metric_yaw], 1),
                                              self.finished_metrics))
      self.metric_xy.copy_(torch.where(done, 0.0, self.metric_xy) + exy)
      self.metric_yaw.copy_(torch.where(done, 0.0, self.metric_yaw) + eyaw)
    fx = 1 - 2 * (q[:, 2] ** 2 + q[:, 3] ** 2)
    fy = 2 * (q[:, 1] * q[:, 2] + q[:, 0] * q[:, 3])
    err = self.heading_target - torch.atan2(fy, fx)
    err = err - 2 * math.pi * torch.floor((err + math.pi) / (2 * math.pi))
    self.command[:, 2] = torch.minimum(torch.maximum(cc.heading_control_stiffness * err, rng[1, 2]), rng[1, 3])
    self.command.copy_(torch.where(self.is_standing.unsqueeze(1), torch.zeros_like(self.command), self.command))

  def observations(self, U: torch.Tensor | None = None):
    """Policy group (uniform noise per term, velocity_env_cfg.py:86-118); ``critic`` is the noise-free copy."""
    d = self.sim.data
    q = d.qpos[:, 3:7]
    lin_b = quat_rotate_inverse(q, d.qvel[:, 0:3])
    terms = [lin_b, d.qvel[:, 3:6], quat_rotate_inverse(q, self._down), d.qpos[:, 7:] - self.default_joint_pos,
             d.qvel[:, 6:], self.last_action, self.command]
    self.critic_obs = torch.cat(terms, dim=1)
    if U is None:
      return self.critic_obs
    Z, nu = U[:, 16:] * 2 - 1, self.nu
    noise = [Z[:, 0:3] * 0.1, Z[:, 3:6] * 0.2, Z[:, 6:9] * 0.05, Z[:, 9:9 + nu] * 0.01, Z[:, 9 + nu:9 + 2 * nu] * 1.5]
    return torch.cat([t + z for t, z in zip(terms[:5], noise)] + terms[5:], dim=1)

  # -- API ---------------------------------------------------------------------------------------
  def reset(self):
    """End every episode and start new ones (with the terrain curriculum on, each env first moves rows by how its
    episode went)."""
    return self._reset_all(curriculum=self.terrain_curriculum)

  def _reset_all(self, curriculum: bool):
    all_ = torch.ones(self.num_envs, dtype=torch.bool, device=self.device)
    self.finished_sums.copy_(self.episode_sums)  # RewardManager.reset of every env
    self.finished_metrics.copy_(torch.stack([self.metric_xy, self.metric_yaw], 1))  # CommandTerm.reset of every env
    self.metric_xy.zero_(); self.metric_yaw.zero_()
    for t in (self.episode_sums, self.air_time, self.contact_time, self.last_air_time):
      t.zero_()
    U = self._draw()
    if curriculum:
      self._terrain_curriculum(all_, U)
    self._reset_where(all_, U)
    self.events.reset_all(self._rand)
    self.sim.forward()
    self._update_command(all_, U, metrics=False)
    frame = self.observations()
    return self.obs_groups.fill({"policy": frame, "critic": frame}, self._rand, self._randn)["policy"]

  def enable_cuda_graph(self) -> None:
    """Capture one whole env step (ctrl write, 4 sub-steps, MDP glue, masked reset + forward) in a
    CUDA graph.  The step has no host synchronisation, so replay is a single launch; inputs and
    outputs live in static buffers (``step`` copies the action in and returns the static outputs)."""
    dev = torch.device(self.device)
    self._action_buf = torch.zeros(self.num_envs, self.nu, device=dev)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
      for _ in range(2):  # warm-up on the side stream (allocator, lazy inits)
        self._step_impl(self._action_buf)
      g = torch.cuda.CUDAGraph()
      g.register_generator_state(self.gen)  # torch.rand(generator=self.gen) inside the capture
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
    return self._step_native(action) if self.native_mdp else self._step_torch(action)

  def _step_native(self, action: torch.Tensor):
    """Two fused kernels (b2_velenv_pre / b2_velenv_post) instead of ~90 torch launches."""
    import ctypes

    from mjlab_b200.sim import native

    sim = self.sim
    self._action_in.copy_(action)
    self._U.copy_(self._draw())
    self.events.draw(self._rand)
    self.obs_groups.draw(self._rand, self._randn)
    native.check(sim._lib.b2_velenv_pre(
      sim._h, ctypes.c_void_p(self._action_in.data_ptr()), ctypes.c_void_p(self.default_joint_pos.data_ptr()),
      ctypes.c_void_p(self.action_scale.data_ptr()), sim._stream()))
    sim.step_n(self.cfg.decimation)
    return self._mdp_native(self._action_in, self._U)

  def _mdp_native(self, action: torch.Tensor, U: torch.Tensor):
    """Everything after the sub-steps on the fused path: b2_velenv_post, the reset and interval events (b2_events,
    when configured), then the forward of the reset envs and the observation groups' clip, scale and history
    (b2_obs_history, when configured)."""
    import ctypes

    from mjlab_b200.sim import native

    sim = self.sim
    if action is not self._action_in:  # (the kernel reads its own two input buffers)
      self._action_in.copy_(action)
    if U is not self._U:
      self._U.copy_(U)
    native.check(sim._lib.b2_velenv_post(sim._h, ctypes.byref(self._native_args), sim._stream()))
    self.events.run_native(sim)
    sim.forward(env_mask=self._done_buf)
    out = self.obs_groups.run_native(sim, {"policy": self._obs, "critic": self._critic})
    return out["policy"], self._reward, self._term, self._trunc, {"critic": out["critic"]}

  def _step_torch(self, action: torch.Tensor):
    """Reference implementation of the same step in torch ops (also the checker of the fused kernels)."""
    U = self._draw()
    self.events.draw(self._rand)
    self.obs_groups.draw(self._rand, self._randn)
    # JointPositionAction: target = default + scale * action (joint_actions.py:85-103)
    self.sim.data.ctrl[:] = self.default_joint_pos + self.action_scale * action
    self.sim.step_n(self.cfg.decimation)
    return self._mdp_torch(action, U)

  def _mdp_torch(self, action: torch.Tensor, U: torch.Tensor):
    """Everything after the sub-steps, in torch ops on the env's own tensors.  It returns fresh tensors and leaves the
    fused path's output buffers alone, so an env built with ``native_mdp=True`` can run it too (the tests compare the
    two on one state)."""
    cfg, d = self.cfg, self.sim.data
    self.episode_length_buf += 1
    if self._stages:
      self.common_step_counter += 1
    q = d.qpos[:, 3:7]
    grav_b = quat_rotate_inverse(q, self._down)
    terminated = torch.acos((-grav_b[:, 2]).clamp(-1.0, 1.0)) > cfg.fall_angle  # bad_orientation
    truncated = self.episode_length_buf >= self.max_episode_length              # time_out
    # rewards (velocity_env_cfg.py:183-214): tracking, posture, limits, action rate
    lin_b = quat_rotate_inverse(q, d.qvel[:, 0:3])
    r_lin = torch.exp(-((self.command[:, :2] - lin_b[:, :2]) ** 2).sum(1) / 0.25)
    r_ang = torch.exp(-((self.command[:, 2] - d.qvel[:, 5]) ** 2) / 0.25)
    jp = d.qpos[:, 7:]
    r_pose = self._posture(jp)
    r_lim = -((self.soft_lo - jp).clamp(min=0) + (jp - self.soft_hi).clamp(min=0)).sum(1)
    r_rate = -0.1 * ((action - self.last_action) ** 2).sum(1)
    done = terminated | truncated
    extra = self._opt_in_rewards(terminated, done, grav_b)  # [n, 9] weighted values of the opt-in terms
    if any(w != 0.0 for w in self.reward_weights):
      reward = (r_lin + r_ang + r_pose + r_lim + r_rate + extra.sum(1)) * self.step_dt
    else:
      reward = (r_lin + r_ang + r_pose + r_lim + r_rate) * self.step_dt
    # episode sums (RewardManager.compute / reset): a done env's row ends its episode
    sums = self.episode_sums + torch.cat([torch.stack([r_lin, r_ang, r_pose, r_lim, r_rate], 1), extra], 1) * self.step_dt
    self.finished_sums.copy_(torch.where(done.unsqueeze(1), sums, self.finished_sums))
    self.episode_sums.copy_(torch.where(done.unsqueeze(1), 0.0, sums))
    self.last_action.copy_(action)
    # partial reset + forward (manager_based_rl_env.py:128-132), mask-based: no host sync; the curriculum runs
    # before the reset events (_reset_idx, :205-208)
    if self.terrain_curriculum:
      self._terrain_curriculum(done, U)
    self._reset_where(done, U)
    self.events.step_torch(terminated, truncated)  # reset, then interval events (before the forward, as b2_events)
    self._done_buf.copy_(done)
    self.sim.forward(env_mask=self._done_buf)  # only the reset envs need new derived quantities here
    self._update_command(done, U)
    self.log_row.copy_(torch.stack([reward, terminated.float(), truncated.float()], dim=1))
    # interval event: push_by_setting_velocity (events.py:127-143), unless push_vel is None
    if cfg.push_vel is not None:
      self.push_time_left -= self.step_dt
      push = self.push_time_left <= 0
      pv = (U[:, 9:11] * 2 - 1) * cfg.push_vel
      d.qvel[:, 0:2] = torch.where(push.unsqueeze(1), pv, d.qvel[:, 0:2])
      lo_t, hi_t = cfg.push_interval_s
      self.push_time_left.copy_(torch.where(push, U[:, 11] * (hi_t - lo_t) + lo_t, self.push_time_left))
    out = self.obs_groups.update({"policy": self.observations(U), "critic": self.critic_obs}, terminated | truncated)
    self.events.step_interval_state()  # the interval push and wrench terms, after the observations
    return out["policy"], reward, terminated, truncated, {"critic": out["critic"]}

  def render(self) -> np.ndarray | None:
    """The reference's ``env.render()``: None with ``render_mode=None``, else an (height, width, 3) uint8 frame of
    ``cfg.viewer``'s camera, drawn on the GPU after the last step."""
    return env_render(self._offline_renderer, self.update_visualizers if self.cfg.command.debug_vis else None)

  def update_visualizers(self, visualizer) -> None:
    """The velocity command's arrows for ``visualizer.env_idx`` (velocity_command.py:106-177), from the root link's
    pose and body-frame velocity and the command, computed on the device.  A root at the world origin (an env not yet
    placed) draws its arrows with alpha 0, i.e. not at all."""
    e = visualizer.env_idx
    if e >= self.num_envs:
      return
    if self._vis is None:
      from mjlab_b200.entity_data import EntityData

      ix = EntityIndexing.from_model(self.model, "robot", self.device)
      colors = torch.tensor(VELOCITY_ARROW_COLORS, dtype=torch.float32, device=self.device)
      self._vis = (EntityData(ix, self.sim.data, self.sim.model, self.device, self.num_envs), colors)
    robot, colors = self._vis
    pos = robot.root_link_pos_w[e]
    viz = self.cfg.command.viz
    ends = velocity_arrows(pos, robot.root_link_quat_w[e], self.command[e], robot.root_link_lin_vel_b[e],
                           robot.root_link_ang_vel_b[e], viz.z_offset, viz.scale)
    colors = torch.cat([colors[:, :3], colors[:, 3:] * (pos.norm() >= 1e-6)], dim=1)
    for k in range(4):
      visualizer.add_arrow(ends[k, 0], ends[k, 1], colors[k], width=VELOCITY_ARROW_WIDTH)

  def close(self):
    if self._offline_renderer is not None:
      self._offline_renderer.close()
    self.sim.close()

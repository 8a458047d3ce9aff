"""Domain randomisation of model fields in the fused environments, as the reference's EventManager runs its
``randomize_field`` terms (EventTermCfg, managers/manager_term_config.py; EventManager, managers/event_manager.py;
randomize_field, FIELD_SPECS, _determine_target_axes and _get_entity_indices, envs/mdp/events.py:184-397).

A term redraws one model field of the robot's joints, bodies, geoms or sites.  Each selected (element, axis) entry
draws ``x = lo + u span`` (``log_uniform``: ``exp`` of that, in the logarithms of the bounds) and writes ``field + x``
(``add``), ``field * x`` (``scale``) or ``x`` (``abs``) into the env's own copy of the field.  The operations read the
field's current value, as the reference's do, so ``add`` and ``scale`` terms of mode ``reset`` compound over episodes.

* ``startup``: every env, once, when the env is built, in list order.
* ``reset``: the envs in the step's ``terminated | truncated`` (the reference's ``reset_buf``; a tracking clip restart
  is not a reset), in list order; ``reset()`` of the env resets every env and runs them on all of them.
* ``interval``: after the reset terms, in list order (``EventManager.apply("interval")`` after ``_reset_idx``).  Each
  term keeps a per-env timer, drawn when the env is built: every env takes ``step_dt`` off it, and an env whose timer
  fell below 1e-6 redraws it and fires the term.  A reset does not redraw a timer: ``EventManager.reset`` redraws only
  those of class-based terms, and ``randomize_field`` is a function.

Draws: a uniform is ``lo + u span`` with ``u`` from the env's generator, one fp32 product then one fp32 sum, where
``span`` is ``hi - lo`` taken in double and rounded to fp32 once (the timers, as EventManager's
``rand * (hi - lo) + lo``, take the same form).  ``log_uniform`` draws ``lo, span`` of ``log(lo), log(hi)``, computed
once on the host, and takes ``exp``.  Startup terms draw ``rand(n, entries)`` each, in list order.  Reset and interval
terms read one block ``V`` that the env draws right after the step's own uniforms (only when such terms exist): each
term owns a contiguous run of its columns, one per (element, axis) entry, element-major, and an interval term one
more, the redraw of its timer when it fires.

Deviations from the reference:
* Only the target axes of an element are written; the reference's ``add`` / ``scale`` also double or square the other
  axes of a partly targeted element (``_generate_random_values`` clones them into the draws).
* An env that both resets and fires an interval term in one step runs the forward of its reset after both, so that
  forward sees the interval draw too (the fused step has one masked forward, after its event launch).
* Values the env or the model derived from a field are not recomputed: soft joint limits, the default pose,
  ``body_subtreemass``, ``*_invweight0``.  The reference computes its soft limits once (``Entity.initialize``) and has
  no ``set_const`` on this path either.
* ``gaussian`` is not offered: the reference's ``sample_gaussian`` with tensor bounds draws one value that every env
  and element shares.  ``dof_frictionloss`` is refused: the engine has no friction loss, so the value would be ignored.

State terms (``ResetRootStateUniformCfg``, ``ResetJointsByScaleCfg``, ``PushBySettingVelocityCfg``,
``ApplyExternalForceTorqueCfg``: envs/mdp/events.py:43-164) write qpos, qvel and xfrc_applied.  Their V columns and
timer rows follow the field terms', in list order (the kinds write disjoint state, so only the draw layout differs from
the reference's one list).  Reset root, joint and wrench terms run after the env's own reset (a reset env's
xfrc_applied first zeroed, as clear_state does; the root and joint terms in the velocity env's post kernel), interval
pushes and wrenches after the env has built the step's observations (DESIGN §4.2).

The fused path runs every reset and interval term of a step in one ``b2_events`` launch (``csrc/b2_events.cuh``); the
torch path below is its reference and runs the startup terms on both paths.
"""

from __future__ import annotations

import ctypes
import math
import re
from dataclasses import dataclass, field

import numpy as np
import torch

from mjlab_b200.entity_data import quat_apply_inverse, quat_mul
from mjlab_b200.sim import native

MODES = ("startup", "reset", "interval")
DISTRIBUTIONS = ("uniform", "log_uniform")
OPERATIONS = ("add", "scale", "abs")
# field: (entity kind, axes per element, default axes, valid axes), as FIELD_SPECS (events.py:184-209); kind "dof"
# addresses through joint_v_adr, "qpos" through joint_q_adr, the others by id
FIELD_SPECS = {
  "dof_armature": ("dof", 1, None, None),
  "dof_frictionloss": ("dof", 1, None, None),
  "dof_damping": ("dof", 1, None, None),
  "jnt_range": ("joint", 2, None, None),
  "jnt_stiffness": ("joint", 1, None, None),
  "body_mass": ("body", 1, None, None),
  "body_ipos": ("body", 3, (0, 1, 2), None),
  "body_iquat": ("body", 4, (0, 1, 2, 3), None),
  "body_inertia": ("body", 3, None, None),
  "body_pos": ("body", 3, (0, 1, 2), None),
  "body_quat": ("body", 4, (0, 1, 2, 3), None),
  "geom_friction": ("geom", 3, (0,), (0, 1, 2)),
  "geom_pos": ("geom", 3, (0, 1, 2), None),
  "geom_quat": ("geom", 4, (0, 1, 2, 3), None),
  "geom_rgba": ("geom", 4, (0, 1, 2, 3), None),
  "site_pos": ("site", 3, (0, 1, 2), None),
  "site_quat": ("site", 4, (0, 1, 2, 3), None),
  "qpos0": ("qpos", 1, None, None),
}
_NAMES = {"dof": "joint_names", "qpos": "joint_names", "joint": "joint_names", "body": "body_names",
          "geom": "geom_names", "site": "site_names"}
_IDS = {"dof": "joint_v_adr", "qpos": "joint_q_adr", "joint": "joint_ids", "body": "body_ids", "geom": "geom_ids",
        "site": "site_ids"}
_F32_MAX = float(np.finfo(np.float32).max)


def _f32(x) -> float:
  return float(np.float32(x))


def _finite32(x) -> bool:
  try:
    x = float(x)
  except (TypeError, ValueError):
    return False
  return math.isfinite(x) and abs(x) <= _F32_MAX


def _pair(name: str, r) -> tuple[float, float]:
  try:
    lo, hi = r
  except (TypeError, ValueError):
    raise ValueError(f"{name} must be a (lo, hi) pair, not {r!r}") from None
  if not (_finite32(lo) and _finite32(hi) and float(lo) <= float(hi)):
    raise ValueError(f"{name} = {r!r} needs finite bounds with lo <= hi")
  return float(lo), float(hi)


@dataclass
class RandomizeFieldCfg:
  """One ``randomize_field`` event term, with the reference's parameter names.  ``names``: regexes (re.fullmatch)
  over the robot's joints, bodies, geoms or sites, whichever kind the field has; None selects all of them."""

  field: str
  ranges: tuple | dict                    # (lo, hi) for every target axis, or {axis: (lo, hi)}
  mode: str = "startup"                   # "startup" | "reset" | "interval"
  distribution: str = "uniform"           # "uniform" | "log_uniform"
  operation: str = "abs"                  # "add" | "scale" | "abs"
  axes: tuple | list | None = None        # None: the keys of a ranges dict, else the field's default axes
  names: tuple | list | str | None = None
  interval_range_s: tuple | None = None   # "interval": (lo, hi) seconds between firings, 0 <= lo <= hi

  def __post_init__(self):
    self.check()

  def target_axes(self) -> list[int]:
    """_determine_target_axes (events.py:291-324)."""
    _, width, default, _ = FIELD_SPECS[self.field]
    if self.axes is not None:
      return list(self.axes)
    if isinstance(self.ranges, dict):
      return list(self.ranges)
    return list(default) if default is not None else list(range(width))

  def axis_ranges(self) -> list[tuple[float, float]]:
    """(lo, hi) of each target axis (_prepare_axis_ranges, events.py:327-346)."""
    axes = self.target_axes()
    if isinstance(self.ranges, dict):
      return [_pair(f"{self.field} ranges[{a}]", self.ranges[a]) for a in axes]
    r = _pair(f"{self.field} ranges", self.ranges)
    return [r] * len(axes)

  def check(self) -> None:
    """ValueError for a malformed term (everything but the names, which need the model)."""
    if self.field not in FIELD_SPECS:
      raise ValueError(f"unknown field {self.field!r}; randomize_field supports {list(FIELD_SPECS)}")
    if self.field == "dof_frictionloss":
      raise ValueError("dof_frictionloss: the engine has no joint friction loss, so the randomised value would be "
                       "ignored")
    if self.mode not in MODES:
      raise ValueError(f"{self.field}: mode must be one of {MODES}, not {self.mode!r}")
    if self.distribution == "gaussian":
      raise ValueError(f"{self.field}: 'gaussian' is not offered: the reference's sample_gaussian with tensor bounds "
                       "draws one value that every env and element shares")
    if self.distribution not in DISTRIBUTIONS:
      raise ValueError(f"{self.field}: distribution must be one of {DISTRIBUTIONS}, not {self.distribution!r}")
    if self.operation not in OPERATIONS:
      raise ValueError(f"{self.field}: operation must be one of {OPERATIONS}, not {self.operation!r}")
    if not isinstance(self.ranges, (tuple, list, dict)):
      raise ValueError(f"{self.field}: ranges must be a (lo, hi) pair or {{axis: (lo, hi)}}, not {self.ranges!r}")
    _, width, _, valid = FIELD_SPECS[self.field]
    axes = self.target_axes()
    if not axes:
      raise ValueError(f"{self.field}: no target axes")
    for a in axes:
      if not isinstance(a, (int, np.integer)) or isinstance(a, bool) or not 0 <= a < width:
        raise ValueError(f"{self.field}: axis {a!r} is outside the field's {width} axes")
      if valid is not None and a not in valid:
        raise ValueError(f"{self.field}: invalid axis {a}; valid axes: {list(valid)}")
    if len(set(axes)) != len(axes):
      raise ValueError(f"{self.field}: axes {axes} repeat an axis")
    if isinstance(self.ranges, dict):
      missing = [a for a in axes if a not in self.ranges]
      if missing:
        raise ValueError(f"{self.field}: ranges has no entry for target axes {missing}")
    for lo, hi in self.axis_ranges():
      if self.distribution == "log_uniform" and not lo > 0.0:
        raise ValueError(f"{self.field}: log_uniform needs lo > 0, not {lo}")
    if self.mode == "interval":
      if self.interval_range_s is None:
        raise ValueError(f"{self.field}: mode 'interval' needs interval_range_s")
      lo, hi = _pair(f"{self.field} interval_range_s", self.interval_range_s)
      if lo < 0.0:
        raise ValueError(f"{self.field}: interval_range_s {self.interval_range_s!r} needs 0 <= lo <= hi")
    if self.names is not None:
      names = [self.names] if isinstance(self.names, str) else self.names
      if not isinstance(names, (tuple, list)) or not names or not all(isinstance(p, str) for p in names):
        raise ValueError(f"{self.field}: names must be a regex or a sequence of regexes, not {self.names!r}")


AXES6 = ("x", "y", "z", "roll", "pitch", "yaw")


def _check_mode(what: str, mode, allowed: tuple, interval_range_s) -> None:
  if mode == "startup":
    raise ValueError(f"{what}: mode 'startup' writes state that the env's first reset() overwrites, as it does in the "
                     "reference; use mode 'reset' or 'interval'")
  if mode not in allowed:
    raise ValueError(f"{what}: mode must be one of {allowed}, not {mode!r}")
  if mode == "interval":
    if interval_range_s is None:
      raise ValueError(f"{what}: mode 'interval' needs interval_range_s")
    lo, _ = _pair(f"{what} interval_range_s", interval_range_s)
    if lo < 0.0:
      raise ValueError(f"{what}: interval_range_s {interval_range_s!r} needs 0 <= lo <= hi")


def _names(what: str, names) -> None:
  if names is not None:
    pats = [names] if isinstance(names, str) else names
    if not isinstance(pats, (tuple, list)) or not pats or not all(isinstance(p, str) for p in pats):
      raise ValueError(f"{what}: names must be a regex or a sequence of regexes, not {names!r}")


@dataclass
class PushBySettingVelocityCfg:
  """``push_by_setting_velocity`` (envs/mdp/events.py:127-143) as an interval term: adds a uniform draw per axis of
  ``velocity_range`` ({"x" "y" "z" "roll" "pitch" "yaw": (lo, hi)}, a missing axis draws 0) to the root link's world
  velocity and writes it back to qvel."""

  velocity_range: dict
  interval_range_s: tuple | None = None
  mode: str = "interval"

  def __post_init__(self):
    self.check()

  def ranges(self) -> list[tuple[float, float]]:
    return [_pair(f"push velocity_range[{k!r}]", self.velocity_range.get(k, (0.0, 0.0))) for k in AXES6]

  def check(self) -> None:
    if not isinstance(self.velocity_range, dict):
      raise ValueError(f"push: velocity_range must be a dict over {AXES6}, not {self.velocity_range!r}")
    bad = [k for k in self.velocity_range if k not in AXES6]
    if bad:
      raise ValueError(f"push: unknown velocity_range keys {bad}; known: {list(AXES6)}")
    self.ranges()
    _check_mode("push", self.mode, ("interval",), self.interval_range_s)


@dataclass
class ApplyExternalForceTorqueCfg:
  """``apply_external_force_torque`` (envs/mdp/events.py:146-164): writes a uniform force and torque per axis to
  ``xfrc_applied`` of the robot's bodies matched by ``names`` (regexes, re.fullmatch; None: every body)."""

  force_range: tuple
  torque_range: tuple
  names: tuple | list | str | None = None
  mode: str = "interval"                  # "interval" | "reset"
  interval_range_s: tuple | None = None

  def __post_init__(self):
    self.check()

  def check(self) -> None:
    _pair("external wrench force_range", self.force_range)
    _pair("external wrench torque_range", self.torque_range)
    _check_mode("external wrench", self.mode, ("reset", "interval"), self.interval_range_s)
    _names("external wrench", self.names)


@dataclass
class ResetRootStateUniformCfg:
  """``reset_root_state_uniform`` (envs/mdp/events.py:43-86) as a reset term: the default root pose plus the env
  origin, offset by a uniform draw per key of ``pose_range`` (position ``x y z``, orientation ``roll pitch yaw``
  composed onto the default orientation), and a root velocity drawn from ``velocity_range`` (its angular part given
  in the world frame).  A missing key draws 0.  Velocity env only."""

  pose_range: dict
  velocity_range: dict
  mode: str = "reset"

  def __post_init__(self):
    self.check()

  def ranges(self) -> list[tuple[float, float]]:
    return [_pair(f"reset_root {name}[{k!r}]", r.get(k, (0.0, 0.0)))
            for name, r in (("pose_range", self.pose_range), ("velocity_range", self.velocity_range)) for k in AXES6]

  def check(self) -> None:
    for name, r in (("pose_range", self.pose_range), ("velocity_range", self.velocity_range)):
      if not isinstance(r, dict):
        raise ValueError(f"reset_root: {name} must be a dict over {AXES6}, not {r!r}")
      bad = [k for k in r if k not in AXES6]
      if bad:
        raise ValueError(f"reset_root: unknown {name} keys {bad}; known: {list(AXES6)}")
    self.ranges()
    _check_mode("reset_root", self.mode, ("reset",), None)


@dataclass
class ResetJointsByScaleCfg:
  """``reset_joints_by_scale`` (envs/mdp/events.py:89-124) as a reset term: the default joint positions of the joints
  matched by ``names`` (regexes, re.fullmatch; None: every joint) times a uniform scale from ``position_range``,
  clamped to the soft joint limits, and the default joint velocities (0) times a scale from ``velocity_range``.
  Velocity env only."""

  position_range: tuple
  velocity_range: tuple
  names: tuple | list | str | None = None
  mode: str = "reset"

  def __post_init__(self):
    self.check()

  def check(self) -> None:
    _pair("reset_joints position_range", self.position_range)
    _pair("reset_joints velocity_range", self.velocity_range)
    _check_mode("reset_joints", self.mode, ("reset",), None)
    _names("reset_joints", self.names)


STATE_TERMS = (PushBySettingVelocityCfg, ApplyExternalForceTorqueCfg, ResetRootStateUniformCfg, ResetJointsByScaleCfg)
RESET_STATE_TERMS = (ResetRootStateUniformCfg, ResetJointsByScaleCfg)
ROOT, JOINTS = 10, 11  # _StateTerm.kind of the reset state terms (run in the env's post kernel, not in b2_events)


@dataclass
class EventsCfg:
  """The env's event terms, run after its built-in startup randomisation: randomize_field terms, and the state terms
  push_by_setting_velocity and apply_external_force_torque."""

  terms: tuple = ()

  def __post_init__(self):
    self.check()

  def check(self) -> None:
    for t in self.terms:
      if not isinstance(t, (RandomizeFieldCfg,) + STATE_TERMS):
        raise ValueError(f"events: every term must be a RandomizeFieldCfg, PushBySettingVelocityCfg, "
                         f"ApplyExternalForceTorqueCfg, ResetRootStateUniformCfg or ResetJointsByScaleCfg, not "
                         f"{type(t).__name__}")
      t.check()

  def has(self, kind) -> bool:
    return any(isinstance(t, kind) for t in self.terms)


def _resolve_names(patterns, names: tuple, what: str) -> list[int]:
  """Indices (entity order) of `names` matched by the regexes (resolve_matching_names: re.fullmatch, a name matched
  by two patterns and a pattern that matches nothing are errors)."""
  if patterns is None:
    return list(range(len(names)))
  pats = [patterns] if isinstance(patterns, str) else list(patterns)
  hit, used = [], set()
  for i, n in enumerate(names):
    m = [p for p in pats if re.fullmatch(p, n)]
    if len(m) > 1:
      raise ValueError(f"{what}: '{n}' is matched by several patterns {m}")
    if m:
      hit.append(i)
      used.add(m[0])
  unused = [p for p in pats if p not in used]
  if unused:
    raise ValueError(f"{what}: patterns {unused} match no {what.split()[-1]} of the robot")
  return hit


@dataclass
class _Term:
  cfg: RandomizeFieldCfg
  offsets: list          # element * width + axis in the world's row, element-major
  idx: torch.Tensor      # the offsets as a device index
  lo: torch.Tensor       # [count] fp32
  span: torch.Tensor     # [count] fp32
  col: int = -1          # first V column (reset / interval terms)
  timer: int = -1        # row of the timers (interval terms)
  interval: tuple = (0.0, 0.0)  # fp32 (lo, span) of the timer

  @property
  def count(self) -> int:
    return len(self.offsets)


def quat_from_euler_xyz(roll: torch.Tensor, pitch: torch.Tensor, yaw: torch.Tensor) -> torch.Tensor:
  """(w, x, y, z) of the rotation by roll about x, then pitch about y, then yaw about z (extrinsic xyz)."""
  cr, sr = torch.cos(roll * 0.5), torch.sin(roll * 0.5)
  cp, sp = torch.cos(pitch * 0.5), torch.sin(pitch * 0.5)
  cy, sy = torch.cos(yaw * 0.5), torch.sin(yaw * 0.5)
  return torch.stack([cy * cr * cp + sy * sr * sp, cy * sr * cp - sy * cr * sp, cy * cr * sp + sy * sr * cp,
                      sy * cr * cp - cy * sr * sp], dim=-1)


def _draw_bounds(lo: float, hi: float, log: bool) -> tuple[float, float]:
  if log:
    lo, hi = math.log(lo), math.log(hi)
  return _f32(lo), _f32(hi - lo)


@dataclass
class _StateTerm:
  cfg: object
  kind: int                 # native.EVENT_PUSH / EVENT_WRENCH
  count: int                # PUSH: 6 axes; WRENCH: bodies
  bodies: list              # WRENCH: global body ids
  lo: list                  # PUSH: 6 fp32 bounds; WRENCH: (force, torque)
  span: list
  col: int = -1
  timer: int = -1
  interval: tuple = (0.0, 0.0)

  @property
  def draws(self) -> int:
    return {native.EVENT_PUSH: 6, native.EVENT_WRENCH: 6 * self.count, ROOT: 12, JOINTS: 2 * self.count}[self.kind]


class Events:
  """The env's terms resolved against its robot: the startup run, the per-step torch path and the fused path's
  argument block."""

  def __init__(self, terms, indexing, sim, num_envs: int, step_dt: float, device, clear_xfrc: bool = True):
    self.sim, self.num_envs, self.step_dt, self.device = sim, num_envs, float(step_dt), torch.device(device)
    self.indexing = indexing
    self.terms: list[_Term] = []
    self.state: list[_StateTerm] = []
    for t in terms:
      if isinstance(t, STATE_TERMS):
        self.state.append(self._state_term(t))
        continue
      t.check()
      kind, width, _, _ = FIELD_SPECS[t.field]
      what = f"{t.field} names"
      ids = getattr(indexing, _IDS[kind])
      elems = [int(ids[i]) for i in _resolve_names(t.names, getattr(indexing, _NAMES[kind]), f"{what} over {kind}")]
      if not elems:
        raise ValueError(f"{t.field}: the robot has no {kind} to randomise")
      axes, rng = t.target_axes(), t.axis_ranges()
      bounds = [_draw_bounds(lo, hi, t.distribution == "log_uniform") for lo, hi in rng]
      offsets = [e * width + a for e in elems for a in axes]
      lo = torch.tensor([b[0] for _ in elems for b in bounds], dtype=torch.float32, device=self.device)
      span = torch.tensor([b[1] for _ in elems for b in bounds], dtype=torch.float32, device=self.device)
      idx = torch.tensor(offsets, dtype=torch.long, device=self.device)
      self.terms.append(_Term(t, offsets, idx, lo, span))
    # the per-step terms: reset terms, then interval terms, each in list order; their V columns in that order
    self.startup = [t for t in self.terms if t.cfg.mode == "startup"]
    self.stepped = ([t for t in self.terms if t.cfg.mode == "reset"] +
                    [t for t in self.terms if t.cfg.mode == "interval"])
    col = ntimer = 0
    for t in self.stepped:
      t.col = col
      col += t.count
      if t.cfg.mode == "interval":
        t.timer, ntimer = ntimer, ntimer + 1
        t.interval = _draw_bounds(*t.cfg.interval_range_s, log=False)
        col += 1
    # the state terms' columns and timer rows follow those of the field terms, in list order
    for t in self.state:
      t.col = col
      col += t.draws
      if t.cfg.mode == "interval":
        t.timer, ntimer = ntimer, ntimer + 1
        t.interval = _draw_bounds(*t.cfg.interval_range_s, log=False)
        col += 1
    # a reset env's wrenches are cleared before its reset terms (Entity.reset -> clear_state); the tracking env's RSI
    # clears them itself
    self.clear_xfrc = bool(clear_xfrc) and any(t.kind == native.EVENT_WRENCH for t in self.state)
    # V columns and timer rows: the field terms' (reset, then interval, each in list order), then the state terms' in
    # list order.  The kinds write disjoint state, so this layout is the only difference from the reference's one
    # list; the first timers are drawn in the same order (draw_timers)
    self.v_width = col
    self.reset_ctx = None  # set_reset_state: what the reset root and joint terms start from
    n = num_envs
    self.V = torch.zeros(n, max(col, 1), dtype=torch.float32, device=self.device) if col else None
    self.timers = torch.zeros(ntimer, n, dtype=torch.float32, device=self.device)
    self._args = self._args_after = None

  def _state_term(self, t) -> _StateTerm:
    ix = self.indexing
    if isinstance(t, ResetRootStateUniformCfg):
      lo, span = [], []
      for a, b in t.ranges():  # tensor bounds: the fp32 difference of the fp32 bounds
        lo.append(_f32(a))
        span.append(_f32(np.float32(b) - np.float32(a)))
      return _StateTerm(t, ROOT, 12, [], lo, span)
    if isinstance(t, ResetJointsByScaleCfg):
      hit = _resolve_names(t.names, ix.joint_names, "reset_joints names over joint")
      if not hit:
        raise ValueError("reset_joints: the robot has no joint to reset")
      if len(hit) > 32:
        raise ValueError(f"reset_joints: at most 32 joints per term, got {len(hit)}")
      bounds = [_draw_bounds(*_pair("position_range", t.position_range), log=False),
                _draw_bounds(*_pair("velocity_range", t.velocity_range), log=False)]  # float bounds
      return _StateTerm(t, JOINTS, len(hit), hit, [b[0] for b in bounds], [b[1] for b in bounds])
    if isinstance(t, PushBySettingVelocityCfg):
      lo, span = [], []
      for a, b in t.ranges():  # tensor bounds: the fp32 difference of the fp32 bounds
        lo.append(_f32(a))
        span.append(_f32(np.float32(b) - np.float32(a)))
      return _StateTerm(t, native.EVENT_PUSH, 6, [], lo, span)
    hit = _resolve_names(t.names, ix.body_names, "external wrench names over body")
    if not hit:
      raise ValueError("external wrench: the robot has no body to push on")
    bounds = [_draw_bounds(*_pair("force_range", t.force_range), log=False),
              _draw_bounds(*_pair("torque_range", t.torque_range), log=False)]  # float bounds: fp32 of the double span
    return _StateTerm(t, native.EVENT_WRENCH, len(hit), [int(ix.body_ids[i]) for i in hit], [b[0] for b in bounds],
                      [b[1] for b in bounds])

  def fields(self) -> list[str]:
    """The fields any term names, in order of first use (the reference's domain_randomization_fields)."""
    return list(dict.fromkeys(t.cfg.field for t in self.terms))

  @property
  def active(self) -> bool:
    """Whether a step has work: reset or interval terms."""
    return bool(self.stepped or self.state)

  def _row(self, t: _Term) -> torch.Tensor:
    """[n, row] view of the env's copy of t's field."""
    return getattr(self.sim.model, t.cfg.field).view(self.num_envs, -1)

  def _apply(self, t: _Term, mask: torch.Tensor | None, u: torch.Tensor) -> None:
    """Write t's draws from the uniforms `u` [n, count] into the envs of `mask` (None: every env)."""
    x = u * t.span + t.lo
    if t.cfg.distribution == "log_uniform":
      x = torch.exp(x)
    row = self._row(t)
    old = row[:, t.idx]
    op = t.cfg.operation
    new = old + x if op == "add" else old * x if op == "scale" else x
    row[:, t.idx] = new if mask is None else torch.where(mask.unsqueeze(1), new, old)

  def _timer_draw(self, t: _Term, u: torch.Tensor) -> torch.Tensor:
    lo, span = t.interval
    return u * span + lo

  # -- the env's calls -----------------------------------------------------------------------------------------------
  def run_startup(self, rand) -> None:
    """The startup terms on every env, in list order; `rand(*shape)` is the env's generator."""
    for t in self.startup:
      self._apply(t, None, rand(self.num_envs, t.count))

  def draw_timers(self, rand) -> None:
    """The interval terms' first timers (EventManager._prepare_terms), one rand(n) each: the field terms', then the
    state terms', each in list order."""
    for t in self.stepped + self.state:
      if t.timer >= 0:
        self.timers[t.timer].copy_(self._timer_draw(t, rand(self.num_envs)))

  def draw(self, rand) -> None:
    """This step's block V, when there are reset or interval terms (the env calls it right after its own draws)."""
    if self.V is not None:
      self.V.copy_(rand(self.num_envs, self.v_width))

  def reset_all(self, rand) -> None:
    """reset() of every env: a fresh V and the reset terms on every env (_reset_idx(all)); the timers run on."""
    if self.clear_xfrc:
      self.sim.data.xfrc_applied[:] = 0.0
    if not any(t.cfg.mode == "reset" for t in self.stepped + self.state):
      return
    self.draw(rand)
    for t in self.stepped:
      if t.cfg.mode == "reset":
        self._apply(t, None, self.V[:, t.col:t.col + t.count])
    for t in self.state:
      if t.cfg.mode == "reset":
        self._apply_state(t, None)

  def _fire(self, t) -> torch.Tensor:
    """Advance t's timer by one step and return the envs it fires on (EventManager.apply("interval"))."""
    tl = self.timers[t.timer] - self.step_dt
    fire = tl < 1e-6
    col = t.col + (t.count if isinstance(t, _Term) else t.draws)
    self.timers[t.timer].copy_(torch.where(fire, self._timer_draw(t, self.V[:, col]), tl))
    return fire

  def set_reset_state(self, default_qpos, env_origins, soft_lo, soft_hi) -> None:
    """The env's default pose, its env origins (updated in place by a terrain curriculum) and soft joint limits, which
    the reset root and joint terms start from."""
    self.reset_ctx = (default_qpos, env_origins, soft_lo, soft_hi)

  def reset_state_terms(self) -> list:
    return [t for t in self.state if t.kind in (ROOT, JOINTS)]

  def _apply_state(self, t: _StateTerm, mask: torch.Tensor | None) -> None:
    """Write state term t's draws from V into the envs of `mask` (None: every env)."""
    d, n = self.sim.data, self.num_envs
    u = self.V[:, t.col:t.col + t.draws]
    keep = (lambda new, old: new) if mask is None else (
      lambda new, old: torch.where(mask.view(-1, *([1] * (new.dim() - 1))), new, old))
    f32 = dict(dtype=torch.float32, device=self.device)
    if t.kind == ROOT:  # reset_root_state_uniform from the default root state plus the env origin
      q0, org, _, _ = self.reset_ctx
      x = u * torch.tensor(t.span, **f32) + torch.tensor(t.lo, **f32)
      pos = q0[0:3] + x[:, 0:3] + org
      quat = quat_mul(q0[3:7].expand(n, 4), quat_from_euler_xyz(x[:, 3], x[:, 4], x[:, 5]))
      vel = torch.zeros(n, 6, **f32) + x[:, 6:12]
      d.qpos[:, 0:7] = keep(torch.cat([pos, quat], dim=1), d.qpos[:, 0:7])
      d.qvel[:, 0:6] = keep(torch.cat([vel[:, 0:3], quat_apply_inverse(quat, vel[:, 3:6])], dim=1), d.qvel[:, 0:6])
      return
    if t.kind == JOINTS:  # reset_joints_by_scale, clamped to the soft joint limits
      q0, _, lo, hi = self.reset_ctx
      k, j = t.count, torch.tensor(t.bodies, dtype=torch.long, device=self.device)
      jp = q0[7:][j] * (u[:, :k] * t.span[0] + t.lo[0])
      jv = torch.zeros(n, k, **f32) * (u[:, k:] * t.span[1] + t.lo[1])
      jp = torch.minimum(torch.maximum(jp, lo[j]), hi[j])
      d.qpos[:, 7 + j] = keep(jp, d.qpos[:, 7 + j])
      d.qvel[:, 6 + j] = keep(jv, d.qvel[:, 6 + j])
      return
    if t.kind == native.EVENT_WRENCH:
      k = t.count
      f = (u[:, :3 * k] * t.span[0] + t.lo[0]).view(n, k, 3)
      tq = (u[:, 3 * k:] * t.span[1] + t.lo[1]).view(n, k, 3)
      b = torch.tensor(t.bodies, dtype=torch.long, device=self.device)
      d.xfrc_applied[:, b] = keep(torch.cat([f, tq], dim=2), d.xfrc_applied[:, b])
      return
    # push_by_setting_velocity: root_link_vel_w (compute_velocity_from_cvel) plus the draw, the angular part back in
    # the body frame of root_link_quat_w
    rb = self.indexing.root_body_id
    c, pos, com = d.cvel[:, rb], d.xpos[:, rb], d.subtree_com[:, rb]
    vel = torch.cat([c[:, 3:6] - torch.cross(c[:, 0:3], com - pos, dim=-1), c[:, 0:3]], dim=1)
    lo = torch.tensor(t.lo, dtype=torch.float32, device=self.device)
    span = torch.tensor(t.span, dtype=torch.float32, device=self.device)
    vel = vel + (u * span + lo)
    new = torch.cat([vel[:, 0:3], quat_apply_inverse(d.xquat[:, rb], vel[:, 3:6])], dim=1)
    d.qvel[:, 0:6] = keep(new, d.qvel[:, 0:6])

  def step_torch(self, terminated: torch.Tensor, truncated: torch.Tensor) -> None:
    """The step's reset terms and interval field terms in torch ops (with step_interval_state, the reference of
    b2_events); the env calls it right after its own reset."""
    if not self.active:
      return
    reset, V = terminated | truncated, self.V
    for t in self.stepped:
      u = V[:, t.col:t.col + t.count]
      if t.cfg.mode == "reset":
        self._apply(t, reset, u)
        continue
      self._apply(t, self._fire(t), u)
    if self.clear_xfrc:
      d = self.sim.data
      d.xfrc_applied[:] = torch.where(reset.view(-1, 1, 1), 0.0, d.xfrc_applied[:])
    for t in self.state:
      if t.cfg.mode == "reset":
        self._apply_state(t, reset)

  def step_interval_state(self) -> None:
    """The interval state terms in torch ops, in list order; the env calls it after it has built the step's
    observations (EventManager.apply("interval") after command_manager.compute)."""
    for t in self.state:
      if t.cfg.mode == "interval":
        self._apply_state(t, self._fire(t))

  # -- the fused path ------------------------------------------------------------------------------------------------

  def bind(self, terminated: torch.Tensor, truncated: torch.Tensor, refreshed: torch.Tensor | None = None,
           interval_after_obs: bool = False) -> None:
    """Build the argument blocks of b2_events over the env's persistent buffers (nothing without such terms).
    `refreshed`: the mask of the masked forward that follows the launch (a push reads those envs' root from qvel).
    `interval_after_obs`: the interval push and wrench terms go into a second block, launched after the env's
    observations (run_native_after_obs), when the forward has refreshed every env."""
    launched = [t for t in self.state if t.kind in (native.EVENT_PUSH, native.EVENT_WRENCH)]
    later = [t for t in launched if interval_after_obs and t.cfg.mode == "interval"]
    now = [t for t in launched if t not in later]
    if len(self.stepped) > native.EVENTS_NTERM:
      raise ValueError(f"at most {native.EVENTS_NTERM} reset and interval terms, got {len(self.stepped)}")
    if max(len(now), len(later)) > native.EVENTS_NSTATE:
      raise ValueError(f"at most {native.EVENTS_NSTATE} push and external wrench terms, got {len(launched)}")
    self._keep = []  # (the first block's entry and body tables first)
    if self.stepped or now:
      self._args = self._block(self.stepped, now, terminated, truncated, refreshed, self.clear_xfrc)
    if later:
      self._no_env = torch.zeros_like(terminated)  # (after the forward: no env is stale, none resets here)
      self._args_after = self._block([], later, self._no_env, self._no_env, self._no_env, False)
    self._keep += [terminated, truncated, refreshed]

  def _block(self, fields, state, terminated, truncated, refreshed, clear_xfrc):
    lib, h = self.sim._lib, self.sim._h
    table = [lib.b2_field_name(h, 1, i).decode() for i in range(lib.b2_num_fields(h, 1))]  # B2_MODEL
    elem = torch.cat([torch.stack([torch.tensor(t.offsets, dtype=torch.int32, device=self.device).view(torch.float32),
                                   t.lo, t.span], dim=1) for t in fields]).contiguous() if fields else None
    bodies = torch.tensor([b for t in state for b in t.bodies] or [0], dtype=torch.int32, device=self.device)
    A = native.B2EventArgs()
    A.terminated, A.truncated = terminated.data_ptr(), truncated.data_ptr()
    A.V, A.v_width = self.V.data_ptr(), self.v_width
    if elem is not None:
      A.elem, A.nelem = elem.data_ptr(), elem.shape[0]
    if self.timers.numel():
      A.timers = self.timers.data_ptr()
    A.ninterval, A.nterm, A.step_dt = self.timers.shape[0], len(fields), self.step_dt
    for k, t in enumerate(fields):
      T = A.term[k]
      T.mode = native.EVENT_INTERVAL if t.cfg.mode == "interval" else native.EVENT_RESET
      T.operation = OPERATIONS.index(t.cfg.operation)
      T.distribution = DISTRIBUTIONS.index(t.cfg.distribution)
      T.field, T.count, T.col = table.index(t.cfg.field), t.count, t.col
      T.interval_lo, T.interval_span = t.interval
    first = 0
    for k, t in enumerate(state):
      S = A.state[k]
      S.kind, S.mode, S.col, S.count, S.timer = t.kind, native.EVENT_INTERVAL if t.cfg.mode == "interval" else \
        native.EVENT_RESET, t.col, t.count, t.timer
      if t.kind == native.EVENT_WRENCH:
        S.first, first = first, first + t.count
        S.lo[:], S.span[:] = t.lo, t.span
      else:
        S.lo6[:], S.span6[:] = t.lo, t.span
      S.interval_lo, S.interval_span = t.interval
    A.nstate, A.nbodies, A.clear_xfrc = len(state), first, int(clear_xfrc)
    A.bodies, A.root_body = bodies.data_ptr(), self.indexing.root_body_id
    if refreshed is not None:
      A.refreshed = refreshed.data_ptr()
    self._keep += [elem, bodies]
    return A

  def run_native(self, sim) -> None:
    """The fused path: one b2_events launch (none without reset or interval terms)."""
    if self._args is not None:
      native.check(sim._lib.b2_events(sim._h, ctypes.byref(self._args), sim._stream()))

  def run_native_after_obs(self, sim) -> None:
    """The second launch of bind(interval_after_obs=True): the interval push and wrench terms."""
    if self._args_after is not None:
      native.check(sim._lib.b2_events(sim._h, ctypes.byref(self._args_after), sim._stream()))

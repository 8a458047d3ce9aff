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


@dataclass
class EventsCfg:
  """The env's randomize_field terms, run after its built-in startup randomisation."""

  terms: tuple = ()

  def __post_init__(self):
    self.check()

  def check(self) -> None:
    for t in self.terms:
      if not isinstance(t, RandomizeFieldCfg):
        raise ValueError(f"events: every term must be a RandomizeFieldCfg, not {type(t).__name__}")
      t.check()


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


def _draw_bounds(lo: float, hi: float, log: bool) -> tuple[float, float]:
  if log:
    lo, hi = math.log(lo), math.log(hi)
  return _f32(lo), _f32(hi - lo)


class Events:
  """The env's terms resolved against its robot: the startup run, the per-step torch path and the fused path's
  argument block."""

  def __init__(self, terms, indexing, sim, num_envs: int, step_dt: float, device):
    self.sim, self.num_envs, self.step_dt, self.device = sim, num_envs, float(step_dt), torch.device(device)
    self.indexing = indexing
    self.terms: list[_Term] = []
    for t in terms:
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
    self.v_width = col
    n = num_envs
    self.V = torch.zeros(n, max(col, 1), dtype=torch.float32, device=self.device) if col else None
    self.timers = torch.zeros(ntimer, n, dtype=torch.float32, device=self.device)
    self._args = None

  def fields(self) -> list[str]:
    """The fields any term names, in order of first use (the reference's domain_randomization_fields)."""
    return list(dict.fromkeys(t.cfg.field for t in self.terms))

  @property
  def active(self) -> bool:
    """Whether a step has work: reset or interval terms."""
    return bool(self.stepped)

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
    """The interval terms' first timers (EventManager._prepare_terms), one rand(n) each."""
    for t in self.stepped:
      if t.timer >= 0:
        self.timers[t.timer].copy_(self._timer_draw(t, rand(self.num_envs)))

  def draw(self, rand) -> None:
    """This step's block V, when there are reset or interval terms (the env calls it right after its own draws)."""
    if self.V is not None:
      self.V.copy_(rand(self.num_envs, self.v_width))

  def reset_all(self, rand) -> None:
    """reset() of every env: a fresh V and the reset terms on every env (_reset_idx(all)); the timers run on."""
    if not any(t.cfg.mode == "reset" for t in self.stepped):
      return
    self.draw(rand)
    for t in self.stepped:
      if t.cfg.mode == "reset":
        self._apply(t, None, self.V[:, t.col:t.col + t.count])

  def step_torch(self, terminated: torch.Tensor, truncated: torch.Tensor) -> None:
    """The step's reset and interval terms in torch ops (the reference of b2_events)."""
    if not self.active:
      return
    reset, V = terminated | truncated, self.V
    for t in self.stepped:
      u = V[:, t.col:t.col + t.count]
      if t.cfg.mode == "reset":
        self._apply(t, reset, u)
        continue
      tl = self.timers[t.timer] - self.step_dt
      fire = tl < 1e-6
      self.timers[t.timer].copy_(torch.where(fire, self._timer_draw(t, V[:, t.col + t.count]), tl))
      self._apply(t, fire, u)

  # -- the fused path ------------------------------------------------------------------------------------------------
  def bind(self, terminated: torch.Tensor, truncated: torch.Tensor) -> None:
    """Build the argument block of b2_events over the env's persistent buffers (nothing without per-step terms)."""
    if not self.active:
      return
    if len(self.stepped) > native.EVENTS_NTERM:
      raise ValueError(f"at most {native.EVENTS_NTERM} reset and interval terms, got {len(self.stepped)}")
    lib, h = self.sim._lib, self.sim._h
    table = [lib.b2_field_name(h, 1, i).decode() for i in range(lib.b2_num_fields(h, 1))]  # B2_MODEL
    elem = torch.cat([torch.stack([torch.tensor(t.offsets, dtype=torch.int32, device=self.device).view(torch.float32),
                                   t.lo, t.span], dim=1) for t in self.stepped]).contiguous()
    A = native.B2EventArgs()
    A.terminated, A.truncated = terminated.data_ptr(), truncated.data_ptr()
    A.V, A.v_width, A.elem, A.nelem = self.V.data_ptr(), self.v_width, elem.data_ptr(), elem.shape[0]
    if self.timers.numel():
      A.timers = self.timers.data_ptr()
    A.ninterval, A.nterm, A.step_dt = self.timers.shape[0], len(self.stepped), self.step_dt
    for k, t in enumerate(self.stepped):
      T = A.term[k]
      T.mode = native.EVENT_INTERVAL if t.cfg.mode == "interval" else native.EVENT_RESET
      T.operation = OPERATIONS.index(t.cfg.operation)
      T.distribution = DISTRIBUTIONS.index(t.cfg.distribution)
      T.field, T.count, T.col = table.index(t.cfg.field), t.count, t.col
      T.interval_lo, T.interval_span = t.interval
    self._args, self._keep = A, (elem, terminated, truncated)

  def run_native(self, sim) -> None:
    """The fused path: one b2_events launch (none without reset or interval terms)."""
    if self._args is not None:
      native.check(sim._lib.b2_events(sim._h, ctypes.byref(self._args), sim._stream()))

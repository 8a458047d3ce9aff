"""Per-term observation noise of the fused environments, as the reference configures it (ObservationTermCfg.noise and
ObservationGroupCfg.enable_corruption, managers/manager_term_config.py:88-111; ObservationManager.compute_group and
_prepare_terms, managers/observation_manager.py:153-172, 229-256; the noise classes and models, utils/noise/).

The classes below stand in for the reference's, with its names and fields.  A parameter is a number or a tuple with
one value per element of the term.  What a term computes from its noise-free value ``x``, in fp32 with one rounding
per operation, as torch computes the reference's expressions:

* ``UniformNoiseCfg``: ``noise = u * span + n_min``, ``u`` uniform in [0, 1).  ``span`` is the fp32 rounding of the
  double ``n_max - n_min`` when both bounds are numbers (torch rounds the Python scalar once), and the fp32 difference
  of the fp32 bounds when either is a tuple (a tensor subtraction).  The two can differ in the last bit.
* ``GaussianNoiseCfg``: ``noise = std * z + mean``, ``z`` standard normal (torch.randn).
* ``ConstantNoiseCfg``: ``noise = bias``.
* ``operation``: ``add`` gives ``x + noise``, ``scale`` gives ``x * noise``, ``abs`` gives ``noise`` (``0 + bias`` for a
  constant, as ``torch.zeros_like(x) + bias``).
* ``NoiseModelWithAdditiveBiasCfg`` adds a per-(env, element) bias after the noise.  On every env that resets
  (``terminated | truncated``) the bias is redrawn as ``bias = bias_noise_cfg.apply(bias)`` before the new observation
  is computed, so an ``add`` bias accumulates over episodes.  ``sample_bias_per_component=False`` shares one draw
  across the term's elements.  Its parameters must be numbers: the reference applies it to an ``(n, 1)`` bias on the
  first reset.

The draws of a step are one uniform block ``W`` and one normal block ``N`` of the env's generator; each random term
owns ``dim`` columns of its block for the per-step noise and, for a bias model, ``dim`` (or 1, shared) columns for the
reset redraw, which are drawn every step and read by reset envs only.
"""

from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

_F32_MAX = float(np.finfo(np.float32).max)
OPERATIONS = ("add", "scale", "abs")  # B2_NOISE_ADD / SCALE / ABS
CONSTANT, UNIFORM, GAUSSIAN = 1, 2, 3  # B2_NOISE_CONSTANT / UNIFORM / GAUSSIAN (0: none)


def _finite32(x) -> bool:
  try:
    x = float(x)
  except (TypeError, ValueError):
    return False
  return math.isfinite(x) and abs(x) <= _F32_MAX


def _values(name: str, p) -> list[float]:
  """The values of parameter `p` (a number or a non-empty tuple), each finite in fp32."""
  vals = list(p) if isinstance(p, (tuple, list)) else [p]
  if not vals or isinstance(p, (bool, np.bool_)) or not all(_finite32(v) and not isinstance(v, (bool, np.bool_))
                                                            for v in vals):
    raise ValueError(f"{name} = {p!r} must be a number or a tuple of numbers, finite in fp32")
  return [float(v) for v in vals]


@dataclass(kw_only=True)
class NoiseCfg:
  """Base of the three noise classes (noise_cfg.py NoiseCfg)."""

  operation: str = "add"

  def params(self) -> dict:
    return {}

  def check(self, dim: int | None = None, name: str = "noise") -> None:
    if type(self) not in (ConstantNoiseCfg, UniformNoiseCfg, GaussianNoiseCfg):
      raise ValueError(f"{name}: {type(self).__name__} is not a noise class")
    if self.operation not in OPERATIONS:
      raise ValueError(f"{name}: operation must be one of {OPERATIONS}, not {self.operation!r}")
    vals = {k: _values(f"{name}.{k}", p) for k, p in self.params().items()}
    if dim is not None:
      for k, p in self.params().items():
        if isinstance(p, (tuple, list)) and len(p) != dim:
          raise ValueError(f"{name}.{k} has {len(p)} values, the term has {dim} elements")
    if isinstance(self, UniformNoiseCfg):
      lo, hi = vals["n_min"], vals["n_max"]
      if len(lo) != len(hi) and 1 not in (len(lo), len(hi)):
        raise ValueError(f"{name}: n_min and n_max have {len(lo)} and {len(hi)} values")
      m = max(len(lo), len(hi))
      if any(a >= b for a, b in zip(lo * m if len(lo) == 1 else lo, hi * m if len(hi) == 1 else hi)):
        raise ValueError(f"{name}: n_min must be below n_max, element by element ({self.n_min!r}, {self.n_max!r})")
    if isinstance(self, GaussianNoiseCfg) and any(s <= 0 for s in vals["std"]):
      raise ValueError(f"{name}: std must be positive, not {self.std!r}")


@dataclass
class ConstantNoiseCfg(NoiseCfg):
  bias: float | tuple = 0.0

  def __post_init__(self):
    self.check()

  def params(self) -> dict:
    return {"bias": self.bias}


@dataclass
class UniformNoiseCfg(NoiseCfg):
  n_min: float | tuple = -1.0
  n_max: float | tuple = 1.0

  def __post_init__(self):
    self.check()

  def params(self) -> dict:
    return {"n_min": self.n_min, "n_max": self.n_max}


@dataclass
class GaussianNoiseCfg(NoiseCfg):
  mean: float | tuple = 0.0
  std: float | tuple = 1.0

  def __post_init__(self):
    self.check()

  def params(self) -> dict:
    return {"mean": self.mean, "std": self.std}


@dataclass(kw_only=True)
class NoiseModelCfg:
  """A noise class applied through a model (noise_cfg.py NoiseModelCfg): the same per-step noise."""

  noise_cfg: NoiseCfg

  def __post_init__(self):
    self.check()

  def check(self, dim: int | None = None, name: str = "noise") -> None:
    if type(self) not in (NoiseModelCfg, NoiseModelWithAdditiveBiasCfg):
      raise ValueError(f"{name}: {type(self).__name__} is not a noise model")
    if not isinstance(self.noise_cfg, NoiseCfg):
      raise ValueError(f"{name}: noise_cfg must be a noise class, not {self.noise_cfg!r}")
    self.noise_cfg.check(dim, name + ".noise_cfg")


@dataclass(kw_only=True)
class NoiseModelWithAdditiveBiasCfg(NoiseModelCfg):
  """Per-step noise plus a bias redrawn on reset (noise_model.py NoiseModelWithAdditiveBias)."""

  bias_noise_cfg: NoiseCfg | None = None
  sample_bias_per_component: bool = True

  def check(self, dim: int | None = None, name: str = "noise") -> None:
    super().check(dim, name)
    if not isinstance(self.bias_noise_cfg, NoiseCfg):
      raise ValueError(f"{name}: bias_noise_cfg must be specified for NoiseModelWithAdditiveBiasCfg (a noise class)")
    self.bias_noise_cfg.check(None, name + ".bias_noise_cfg")
    if any(isinstance(p, (tuple, list)) for p in self.bias_noise_cfg.params().values()):
      raise ValueError(f"{name}: the parameters of bias_noise_cfg must be numbers (the first reset draws an (n, 1) bias)")
    if not isinstance(self.sample_bias_per_component, (bool, np.bool_)):
      raise ValueError(f"{name}: sample_bias_per_component must be a bool")


def check_term_noise(cfg, dim: int | None = None, name: str = "noise") -> None:
  """ValueError unless `cfg` is None, a noise class or a noise model whose parameters fit `dim` elements."""
  if cfg is None:
    return
  if not isinstance(cfg, (NoiseCfg, NoiseModelCfg)):
    raise ValueError(f"{name}: {cfg!r} is not a noise class or a noise model")
  cfg.check(dim, name)


# ---- the tasks' defaults -----------------------------------------------------------------------------------------------
def _u(a: float) -> UniformNoiseCfg:
  return UniformNoiseCfg(n_min=-a, n_max=a)


def velocity_defaults() -> dict:
  """{group: {term: noise}} of the velocity task (velocity_env_cfg.py:90-114); the critic (PrivilegedCfg(PolicyCfg))
  inherits the policy's terms."""
  policy = {"base_lin_vel": _u(0.1), "base_ang_vel": _u(0.2), "projected_gravity": _u(0.05), "joint_pos": _u(0.01),
            "joint_vel": _u(1.5)}
  return {"policy": policy, "critic": dict(policy)}


def tracking_defaults() -> dict:
  """{group: {term: noise}} of the tracking task (tracking_env_cfg.py:93-124); its critic has no noise."""
  return {"policy": {"motion_anchor_pos_b": _u(0.25), "motion_anchor_ori_b": _u(0.05), "base_lin_vel": _u(0.5),
                     "base_ang_vel": _u(0.2), "joint_pos": _u(0.01), "joint_vel": _u(0.5)},
          "critic": {}}


@dataclass
class TaskNoise:
  """What the env tells the groups about noise: the task's default term noise and enable_corruption per group, and
  the terms of the noise-free source row (the critic frame, which holds every term of both groups)."""

  defaults: dict     # {group: {term: NoiseCfg | NoiseModelCfg}}
  corruption: dict   # {group: bool}
  source: list       # [(term, elements), ...] of the source row, in order


# ---- one term's noise, resolved ---------------------------------------------------------------------------------------
class Draw:
  """One noise class resolved for a term of `dim` elements: fp32 parameter rows and its columns in W or N."""

  def __init__(self, cfg: NoiseCfg, dim: int, device, per_element_draws: bool = True):
    self.kind = {ConstantNoiseCfg: CONSTANT, UniformNoiseCfg: UNIFORM, GaussianNoiseCfg: GAUSSIAN}[type(cfg)]
    self.op = OPERATIONS.index(cfg.operation)
    self.ndraw = 0 if self.kind == CONSTANT else (dim if per_element_draws else 1)
    self.col = -1  # first column in W (uniform) or N (gaussian); set by the layout

    def row(p):
      return np.asarray(list(p) if isinstance(p, (tuple, list)) else [p] * dim, dtype=np.float32)

    if self.kind == CONSTANT:
      p0, p1 = row(cfg.bias), None
    elif self.kind == UNIFORM:
      p0 = row(cfg.n_min)
      if isinstance(cfg.n_min, (tuple, list)) or isinstance(cfg.n_max, (tuple, list)):
        p1 = row(cfg.n_max) - p0                                       # fp32 - fp32 (a tensor subtraction)
      else:
        p1 = np.full(dim, np.float32(float(cfg.n_max) - float(cfg.n_min)), dtype=np.float32)  # double, rounded once
    else:
      p0, p1 = row(cfg.mean), row(cfg.std)
    self.p0 = torch.tensor(p0, dtype=torch.float32, device=device)
    self.p1 = None if p1 is None else torch.tensor(p1, dtype=torch.float32, device=device)
    self.p0_at = self.p1_at = -1  # offsets in the parameter row; set by the layout

  @property
  def block(self) -> str:
    return "W" if self.kind == UNIFORM else "N"

  def apply(self, x: torch.Tensor, r: torch.Tensor | None) -> torch.Tensor:
    """The class's `apply` on `x` with the draws `r` (broadcast against x)."""
    if self.kind == CONSTANT:
      noise = self.p0
      if self.op == 2:
        return torch.zeros_like(x) + noise
    else:
      noise = r * self.p1 + self.p0
    return x + noise if self.op == 0 else x * noise if self.op == 1 else noise.expand_as(x).clone()


class TermNoise:
  """The effective noise of one term: the per-step draw and, for a bias model, the bias redraw."""

  def __init__(self, cfg, dim: int, device):
    self.dim = dim
    base = cfg.noise_cfg if isinstance(cfg, NoiseModelCfg) else cfg
    self.noise = Draw(base, dim, device)
    self.bias = None
    self.shared = False
    if isinstance(cfg, NoiseModelWithAdditiveBiasCfg):
      self.shared = not bool(cfg.sample_bias_per_component)
      self.bias = Draw(cfg.bias_noise_cfg, dim, device, per_element_draws=not self.shared)

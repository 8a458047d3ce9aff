"""Clip, scale and history of the fused environments' observation groups, as the reference's ObservationManager
configures them (ObservationTermCfg / ObservationGroupCfg, managers/manager_term_config.py:87-111;
ObservationManager.compute_group and _prepare_terms, managers/observation_manager.py:153-188, 229-270; the history's
CircularBuffer, utils/buffers/circular_buffer.py).

Each env computes the frame of a group (its terms concatenated in cfg order, noise applied) as before.  A configured
group then takes every term of that frame through, in order: clip to ``(lo, hi)``, multiply by ``scale``, append to
the term's history.  The group's output is

* ``flatten_history_dim=True``: ``(n, sum_t max(H_t, 1) D_t)``, the terms in cfg order, each term's frames contiguous,
  oldest first, newest last (a term without history appears once);
* ``flatten_history_dim=False``: ``(n, H, sum_t D_t)``, time-major; every term has the same ``H >= 1``.

In every env step an env drops its oldest frame and appends the new one; an env in the step's ``terminated |
truncated`` (the reference's ``reset_buf``, whose envs ``_reset_idx`` hands to ``ObservationManager.reset``) gets the
new frame in every slot, as ``CircularBuffer.append`` backfills a reset row.  ``reset()`` of an env fills every env's
history with the frame it computes.

The output tensor is the history: the fused path's ``b2_obs_history`` kernel (``csrc/b2_obshist.cuh``) and the torch
path below both update it in place.  A group left at its defaults is not processed at all: the env returns its frame,
as it did before this existed.

Noise (``envs/noise.py``).  A group is noise-configured when its ``noise`` dict is not empty or its
``enable_corruption`` is set.  Such a group does not take the env's frame (whose built-in noise stays as it was for the
groups that are not): each term reads its noise-free values from the env's critic frame, gets its effective noise (the
task's default, replaced by a ``noise`` entry, none when the group's corruption is off), then the clip, scale and
history above.  A group that is not noise-configured is untouched: same outputs, launches and draws.
"""

from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass, field

import numpy as np
import torch

from mjlab_b200.envs import noise as nz
from mjlab_b200.sim import native

_F32_MAX = float(np.finfo(np.float32).max)
GROUPS = ("policy", "critic")


def _is_length(h) -> bool:
  return isinstance(h, (int, np.integer)) and not isinstance(h, (bool, np.bool_)) and h >= 0


def _finite32(x) -> bool:
  """A real number that is finite in fp32 (NaN fails)."""
  try:
    x = float(x)
  except (TypeError, ValueError):
    return False
  return math.isfinite(x) and abs(x) <= _F32_MAX


@dataclass
class ObsGroupCfg:
  """Clip, scale and history of one observation group (ObservationGroupCfg and the ObservationTermCfg fields of its
  terms).  Terms are named as in the reference's task cfg.  The defaults leave the group as the env computes it."""

  history_length: int | None = None   # the group's history length: when set it overrides every term's
  flatten_history_dim: bool = True    # False: (n, H, sum D); needs one history length >= 1 for every term
  term_history: dict = field(default_factory=dict)  # {term: history length}; 0: no history
  clip: dict = field(default_factory=dict)          # {term: (lo, hi)}
  scale: dict = field(default_factory=dict)         # {term: factor, or one factor per element of the term}
  # {term: NoiseCfg | NoiseModelCfg | None} (envs/noise.py): replaces the task's default noise of the term; None: none
  noise: dict = field(default_factory=dict)
  enable_corruption: bool | None = None  # None: the task's setting for the group; False drops every term's noise

  def __post_init__(self):
    self.check()

  def lengths(self, names) -> list[int]:
    """The history length of each term (observation_manager.py:231-233)."""
    if self.history_length is not None:
      return [int(self.history_length)] * len(names)
    return [int(self.term_history.get(t, 0)) for t in names]

  def check(self, terms: dict | None = None, group: str = "observations") -> None:
    """ValueError for a malformed block; with `terms` ({name: elements}, in cfg order) also for one that does not fit
    the group's terms."""
    if self.history_length is not None and not _is_length(self.history_length):
      raise ValueError(f"{group}: history_length must be an integer >= 0 or None, not {self.history_length!r}")
    if not isinstance(self.flatten_history_dim, (bool, np.bool_)):
      raise ValueError(f"{group}: flatten_history_dim must be a bool, not {self.flatten_history_dim!r}")
    for k in ("term_history", "clip", "scale", "noise"):
      if not isinstance(getattr(self, k), dict):
        raise ValueError(f"{group}: {k} must be a dict keyed by term name")
    for t, h in self.term_history.items():
      if not _is_length(h):
        raise ValueError(f"{group}: term_history[{t!r}] must be an integer >= 0, not {h!r}")
    for t, c in self.clip.items():
      try:
        lo, hi = c
      except (TypeError, ValueError):
        raise ValueError(f"{group}: clip[{t!r}] must be a (lo, hi) pair, not {c!r}") from None
      if not (_finite32(lo) and _finite32(hi) and float(lo) <= float(hi)):
        raise ValueError(f"{group}: clip[{t!r}] = {c!r} needs finite bounds with lo <= hi")
    for t, s in self.scale.items():
      vals = list(s) if isinstance(s, (tuple, list)) else [s]
      if not vals or not all(_finite32(v) for v in vals):
        raise ValueError(f"{group}: scale[{t!r}] = {s!r} must be a finite number or a tuple of finite numbers")
    if self.enable_corruption is not None and not isinstance(self.enable_corruption, (bool, np.bool_)):
      raise ValueError(f"{group}: enable_corruption must be a bool or None, not {self.enable_corruption!r}")
    for t, c in self.noise.items():
      nz.check_term_noise(c, terms[t] if terms is not None and t in terms else None, f"{group}: noise[{t!r}]")
    if terms is None:
      return
    for k in ("term_history", "clip", "scale", "noise"):
      unknown = [t for t in getattr(self, k) if t not in terms]
      if unknown:
        raise ValueError(f"{group}: {k} names unknown terms {unknown}; the group's terms are {list(terms)}")
    for t, s in self.scale.items():
      if isinstance(s, (tuple, list)) and len(s) != terms[t]:
        raise ValueError(f"{group}: scale[{t!r}] has {len(s)} factors, the term has {terms[t]} elements")
    H = self.lengths(list(terms))
    if not self.flatten_history_dim and (len(set(H)) != 1 or H[0] < 1):
      raise ValueError(f"{group}: flatten_history_dim=False needs one history length >= 1 for every term, not {H}")


@dataclass
class ObservationsCfg:
  """The blocks of the env's two observation groups."""

  policy: ObsGroupCfg = field(default_factory=ObsGroupCfg)
  critic: ObsGroupCfg = field(default_factory=ObsGroupCfg)


@dataclass
class _Term:
  name: str
  src: int                    # first column in the frame
  dim: int
  frames: int                 # history length as configured (0: none)
  dst: int                    # column of the oldest frame in the output row
  stride: int                 # columns between consecutive frames
  clip: tuple | None          # fp32 bounds
  scale: torch.Tensor | None  # [dim] fp32 factors
  scale_at: int               # offset in the env's scale row, -1: none
  col: int = 0                # first column in the noise source row (noise-configured groups)
  noise: nz.TermNoise | None = None  # effective noise


class ObsGroup:
  """One group resolved against the env's terms: the layout of its output and the history buffer."""

  def __init__(self, cfg: ObsGroupCfg, group: str, terms: list[tuple[str, int]], num_envs: int, device,
               scale_at: int = 0, task_noise: nz.TaskNoise | None = None):
    cfg.check(dict(terms), group)
    H = cfg.lengths([t for t, _ in terms])
    # noise-configured: read the noise-free source row and apply the effective noise (module docstring)
    self.noisy = bool(cfg.noise) or cfg.enable_corruption is not None
    self.active = any(h > 0 for h in H) or bool(cfg.clip) or bool(cfg.scale) or self.noisy
    self.flatten = bool(cfg.flatten_history_dim)
    self.num_envs, self.frame_width = num_envs, sum(d for _, d in terms)
    dev = torch.device(device)
    self.terms: list[_Term] = []
    src = dst = 0
    for (name, dim), h in zip(terms, H):
      s = cfg.scale.get(name)
      if s is not None:
        s = torch.tensor(list(s) if isinstance(s, (tuple, list)) else [s] * dim, dtype=torch.float32, device=dev)
      c = cfg.clip.get(name)
      c = None if c is None else (float(np.float32(c[0])), float(np.float32(c[1])))
      if self.flatten:
        t = _Term(name, src, dim, h, dst, dim, c, s, -1)
        dst += max(h, 1) * dim
      else:
        t = _Term(name, src, dim, h, src, self.frame_width, c, s, -1)
      if s is not None:
        t.scale_at, scale_at = scale_at, scale_at + dim
      self.terms.append(t)
      src += dim
    self.scale_end = scale_at
    self.bias = None  # [n, frame_width] the bias models' state, element e at column e
    if self.noisy:
      source = task_noise.source if task_noise is not None else terms
      cols, c = {}, 0
      for name, dim in source:
        cols[name], c = c, c + dim
      self.source_width = c
      on = cfg.enable_corruption
      if on is None:
        on = bool(task_noise.corruption.get(group, False)) if task_noise is not None else False
      defaults = task_noise.defaults.get(group, {}) if task_noise is not None else {}
      for t in self.terms:
        if t.name not in cols or dict(source)[t.name] != t.dim:
          raise ValueError(f"{group}: the noise source row has no term {t.name!r} of {t.dim} elements")
        t.col = cols[t.name]
        eff = cfg.noise[t.name] if t.name in cfg.noise else defaults.get(t.name)
        if on and eff is not None:
          nz.check_term_noise(eff, t.dim, f"{group}: noise of {t.name!r}")
          t.noise = nz.TermNoise(eff, t.dim, dev)
      if any(t.noise is not None and t.noise.bias is not None for t in self.terms):
        self.bias = torch.zeros(num_envs, self.frame_width, dtype=torch.float32, device=dev)
    self.shape = (num_envs, dst) if self.flatten else (num_envs, H[0], self.frame_width)
    self.width = int(np.prod(self.shape[1:]))  # elements per env
    self.out = torch.zeros(num_envs, self.width, dtype=torch.float32, device=dev) if self.active else None

  def output(self) -> torch.Tensor:
    return self.out.view(self.shape)

  def _frames(self, t: _Term) -> torch.Tensor:
    """[n, max(H, 1), D] view of term t's frames in the output buffer."""
    if self.flatten:
      return self.out[:, t.dst:t.dst + max(t.frames, 1) * t.dim].unflatten(1, (max(t.frames, 1), t.dim))
    return self.out.view(self.shape)[:, :, t.src:t.src + t.dim]

  def _bias(self, t: _Term) -> torch.Tensor:
    return self.bias[:, t.src:t.src + t.dim]

  def redraw_bias(self, mask: torch.Tensor | None, W, N, first: bool = False, shape: bool = False) -> None:
    """Redraw the bias of every bias model in the envs of `mask` (None: all) from the draws W, N.  `first`: the
    reference's first reset(all), when every bias is still (n, 1) and draws one column; `shape`: the first compute's
    reshape of a per-component bias, which draws again per element (noise_model.py _initialize_bias_shape)."""
    for t in self.terms:
      d = t.noise.bias if t.noise is not None else None
      if d is None or (shape and t.noise.shared):
        continue
      b = self._bias(t)
      new = d.apply(b, _cols(d, W, N, 1 if first else None))
      b.copy_(new if mask is None else torch.where(mask.view(-1, 1), new, b))

  def update(self, frame: torch.Tensor, reset: torch.Tensor, source: torch.Tensor | None = None, W=None, N=None,
             redraw: bool = True) -> torch.Tensor:
    """The torch path: clip, scale and append `frame` [n, frame_width]; `reset` [n] bool backfills.  A
    noise-configured group reads `source` instead and first redraws the biases of the reset envs (unless not
    `redraw`) and adds the noise, from this step's draws W, N.  Returns a fresh copy of the output."""
    r = reset.view(-1, 1, 1)
    if self.noisy and redraw and self.bias is not None:
      self.redraw_bias(reset, W, N)
    for t in self.terms:
      if self.noisy:
        v = source[:, t.col:t.col + t.dim]
        if t.noise is not None:
          v = t.noise.noise.apply(v, _cols(t.noise.noise, W, N))
          if t.noise.bias is not None:
            v = v + self._bias(t)
      else:
        v = frame[:, t.src:t.src + t.dim]
      if t.clip is not None:
        v = v.clamp(t.clip[0], t.clip[1])
      if t.scale is not None:
        v = v * t.scale
      hist = self._frames(t)
      v = v.unsqueeze(1)
      hist.copy_(torch.where(r, v.expand_as(hist), torch.cat([hist[:, 1:], v], dim=1)))
    return self.output().clone()

  def native_group(self, G: native.B2ObsHistGroup, frame: torch.Tensor) -> None:
    assert frame.is_contiguous() and frame.shape == (self.num_envs, self.frame_width)
    G.frame, G.out = frame.data_ptr(), self.out.data_ptr()
    G.frame_width, G.out_width, G.nterm = self.frame_width, self.width, len(self.terms)
    if len(self.terms) > native.OBSHIST_NTERM:
      raise ValueError(f"at most {native.OBSHIST_NTERM} terms per group")
    for k, t in enumerate(self.terms):
      T = G.term[k]
      T.src, T.dim, T.frames, T.dst, T.stride, T.scale = t.src, t.dim, t.frames, t.dst, t.stride, t.scale_at
      T.clip = t.clip is not None
      T.lo, T.hi = t.clip if t.clip is not None else (0.0, 0.0)

  def native_noise(self, Z: native.B2ObsNoiseGroup, source: torch.Tensor) -> None:
    assert source.is_contiguous() and source.shape == (self.num_envs, self.source_width)
    Z.source, Z.source_width = source.data_ptr(), self.source_width
    if self.bias is not None:
      Z.bias = self.bias.data_ptr()
    for k, t in enumerate(self.terms):
      M = Z.term[k]
      M.col = t.col
      if t.noise is None:
        continue
      d = t.noise.noise
      M.noise, M.noise_op, M.noise_p0, M.noise_p1, M.noise_draw = d.kind, d.op, d.p0_at, d.p1_at, d.col
      if t.noise.bias is not None:
        d = t.noise.bias
        M.bias, M.bias_op, M.bias_p0, M.bias_p1, M.bias_draw = d.kind, d.op, d.p0_at, d.p1_at, d.col
        M.bias_shared = int(t.noise.shared)


def _cols(d: nz.Draw, W, N, count: int | None = None):
  """The draws of `d` (its first `count` columns; all by default), None for a constant."""
  if d.kind == nz.CONSTANT:
    return None
  block = W if d.kind == nz.UNIFORM else N
  return block[:, d.col:d.col + (d.ndraw if count is None else count)]


class Observations:
  """The env's policy and critic groups: their outputs on both paths and the fused path's argument block."""

  def __init__(self, cfg: ObservationsCfg, terms: dict, num_envs: int, device, task_noise: nz.TaskNoise | None = None):
    """`terms`: {group: [(term name, elements), ...]} in the order of the group's frame; `task_noise`: the task's
    default noise and its noise-free source row (without it a noise-configured group reads its own frame and has no
    default noise)."""
    self.groups, at = {}, 0
    for g in GROUPS:
      self.groups[g] = ObsGroup(getattr(cfg, g), g, terms[g], num_envs, device, scale_at=at, task_noise=task_noise)
      at = self.groups[g].scale_end
    scales = [t.scale for grp in self.groups.values() for t in grp.terms if t.scale is not None]
    self.scale_row = torch.cat(scales) if scales else None
    self.active = [g for g in GROUPS if self.groups[g].active]
    self._args = None
    self._layout_noise(num_envs, device)

  def _layout_noise(self, n: int, device) -> None:
    """Columns of W and N and offsets in the parameter row of every term's noise, group by group, term by term: a
    term's per-step draws, then its bias redraw."""
    both = [t.name for g in GROUPS for t in self.groups[g].terms if t.noise is not None and t.noise.bias is not None]
    if len(both) != len(set(both)):
      raise ValueError("a bias model on the same term in both groups is not supported (the reference keys a bias "
                       "model's state by term name, so both groups would share one)")
    width, params, at = {"W": 0, "N": 0}, [], 0
    for g in GROUPS:
      for t in self.groups[g].terms:
        if t.noise is None:
          continue
        for d in (t.noise.noise, t.noise.bias):
          if d is None:
            continue
          if d.ndraw:
            d.col, width[d.block] = width[d.block], width[d.block] + d.ndraw
          for k, p in (("p0_at", d.p0), ("p1_at", d.p1)):
            if p is not None:
              setattr(d, k, at)
              params.append(p)
              at += p.numel()
    self.nW, self.nN = width["W"], width["N"]
    dev = torch.device(device)
    self.W = torch.zeros(n, self.nW, dtype=torch.float32, device=dev) if self.nW else None
    self.N = torch.zeros(n, self.nN, dtype=torch.float32, device=dev) if self.nN else None
    self.param_row = torch.cat(params).contiguous() if params else None
    self.noisy = [g for g in GROUPS if self.groups[g].noisy]
    self._shaped = False  # whether the first reset reshaped the per-component biases

  def draw(self, rand, randn) -> None:
    """This step's blocks W (rand) and N (randn), when a term draws (the env calls it right after the events')."""
    if self.W is not None:
      self.W.copy_(rand(*self.W.shape))
    if self.N is not None:
      self.N.copy_(randn(*self.N.shape))

  def width(self, g: str) -> int:
    """Elements per env of group g's output."""
    return self.groups[g].width

  def update(self, frames: dict, reset: torch.Tensor, redraw: bool = True) -> dict:
    """The torch path: each group's output from its frame (the frame itself for a group at its defaults); a
    noise-configured group reads the critic frame, the noise-free source, with this step's W and N."""
    return {g: self.groups[g].update(frames[g], reset, frames["critic"], self.W, self.N, redraw)
            if self.groups[g].active else frames[g] for g in GROUPS}

  def fill(self, frames: dict, rand=None, randn=None) -> dict:
    """reset() of the env: the reference's reset(all) then compute, so every env's bias is redrawn, the noise drawn
    (from fresh W, N of rand and randn) and every env's history is the frame.  The first call also does what the
    reference's first reset(all) and first compute do to a bias: one draw per env into the (n, 1) bias, then a
    per-element draw on top of it for a per-component bias (noise_model.py _initialize_bias_shape)."""
    f = frames["policy"]
    all_ = torch.ones(f.shape[0], dtype=torch.bool, device=f.device)
    if not self.noisy:
      return self.update(frames, all_)
    self.draw(rand, randn)
    if self._shaped:
      return self.update(frames, all_)
    for g in self.noisy:
      if self.groups[g].bias is not None:
        self.groups[g].redraw_bias(None, self.W, self.N, first=True)
    self.draw(rand, randn)
    for g in self.noisy:
      if self.groups[g].bias is not None:
        self.groups[g].redraw_bias(None, self.W, self.N, shape=True)
    self._shaped = True
    return self.update(frames, all_, redraw=False)

  def bind(self, frames: dict, terminated: torch.Tensor, truncated: torch.Tensor) -> None:
    """Build the argument block of b2_obs_history over the fused path's frame buffers (persistent tensors)."""
    if not self.active:
      return
    A = native.B2ObsHistArgs()
    A.terminated, A.truncated = terminated.data_ptr(), truncated.data_ptr()
    if self.scale_row is not None:
      A.scale, A.nscale = self.scale_row.data_ptr(), self.scale_row.numel()
    A.ngroup = len(self.active)
    for k, g in enumerate(self.active):
      self.groups[g].native_group(A.group[k], frames[g])
      if self.groups[g].noisy:
        self.groups[g].native_noise(A.noise[k], frames["critic"])
    for name, t in (("W", self.W), ("N", self.N), ("param", self.param_row)):
      if t is not None:
        setattr(A, name, t.data_ptr())
    A.nW, A.nN = self.nW, self.nN
    A.nparam = 0 if self.param_row is None else self.param_row.numel()
    self._args, self._keep = A, (frames, terminated, truncated)

  def run_native(self, sim, frames: dict) -> dict:
    """The fused path: one b2_obs_history launch for the configured groups (none when every group is at its
    defaults); returns each group's output buffer (the frame buffer for a group at its defaults)."""
    if self._args is not None:
      native.check(sim._lib.b2_obs_history(sim._h, ctypes.byref(self._args), sim._stream()))
    return {g: self.groups[g].output() if self.groups[g].active else frames[g] for g in GROUPS}

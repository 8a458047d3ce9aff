"""Offscreen frames of the batched scene: the reference's ``ViewerConfig`` (``viewer/viewer_config.py``) and
``OffscreenRenderer`` (``viewer/offscreen_renderer.py``), drawn by the ray-casting kernel ``b2_render``
(``csrc/b2_render.cuh``) from the geom poses the engine holds on the device, instead of by OpenGL from a CPU
``mj_forward`` per drawn env.

Differences from the reference: robots are drawn from their primitive geoms (mesh geoms are not drawn), there are no
reflections or textures (``enable_reflections`` is accepted and has no effect), and shading is the fixed model of
DESIGN.md §4.
"""

from __future__ import annotations

import ctypes
import enum
import math
from dataclasses import dataclass

import numpy as np
import torch

from mjlab_b200.sim import native

MAX_ENVS = 32  # worlds 0..MAX_ENVS-1 are drawn besides env_idx (the reference's _MAX_ENVS)


@dataclass
class ViewerConfig:
  lookat: tuple[float, float, float] = (0.0, 0.0, 0.0)
  distance: float = 5.0
  elevation: float = -45.0
  azimuth: float = 90.0

  class OriginType(enum.Enum):
    """The frame in which the camera position and target are defined."""

    WORLD = enum.auto()
    """The origin of the world."""
    ASSET_ROOT = enum.auto()
    """The center of the asset defined by asset_name."""
    ASSET_BODY = enum.auto()
    """The center of the body defined by body_name in asset defined by asset_name."""

  origin_type: OriginType = OriginType.WORLD
  asset_name: str | None = None
  body_name: str | None = None
  env_idx: int = 0
  enable_reflections: bool = True  # accepted for compatibility; the ray caster draws no reflections
  enable_shadows: bool = True
  height: int = 240
  width: int = 320


def tracked_body(model, cfg: ViewerConfig) -> int:
  """Engine body id the camera tracks (its subtree_com is the target), or -1 for a free camera at ``cfg.lookat``.
  Entities are the body-name prefixes (``robot/...``), as the compiled scenes name them."""
  O = ViewerConfig.OriginType
  if cfg.origin_type == O.WORLD:
    return -1
  bodies = list(model.names["body"])
  entities = sorted({b.split("/", 1)[0] for b in bodies if "/" in b})
  if cfg.origin_type == O.ASSET_ROOT:
    if cfg.asset_name:
      asset = cfg.asset_name
    elif len(entities) == 1:
      asset = entities[0]
    else:
      raise ValueError(f"Multiple entities in scene ({len(entities)}). Specify asset_name to choose which one.")
    if asset not in entities:
      raise KeyError(f"Scene element '{asset}' not found. Available: {entities}")
    parent = np.asarray(model.arrays["body_parentid"])
    return next(i for i, b in enumerate(bodies) if b.startswith(asset + "/") and not bodies[parent[i]].startswith(asset + "/"))
  if not cfg.asset_name or not cfg.body_name:
    raise ValueError("asset_name/body_name required for ASSET_BODY origin type")
  if cfg.asset_name not in entities:
    raise KeyError(f"Scene element '{cfg.asset_name}' not found. Available: {entities}")
  name = f"{cfg.asset_name}/{cfg.body_name}"
  if name not in bodies:
    raise ValueError(f"Body '{cfg.body_name}' not found in asset '{cfg.asset_name}'")
  return bodies.index(name)


class OffscreenRenderer:
  """Frames of ``sim`` (a ``Simulation``) as ``cfg`` sets the camera.  ``update()`` enqueues one frame on the sim's
  stream after whatever work is queued there (the step); ``render()`` copies it to the host.  The output buffers are
  allocated once, here; ``extra_outputs`` also allocates the depth and segmentation buffers (``depth()``,
  ``segmentation()``: the distance along the camera axis, +inf for the background, and (world, geom) pairs, (-1, -1)
  for the background)."""

  def __init__(self, sim, cfg: ViewerConfig, extra_outputs: bool = False):
    if not (1 <= cfg.width <= 4096 and 1 <= cfg.height <= 4096):
      raise ValueError(f"width and height must lie in 1..4096, got {cfg.width} x {cfg.height}")
    if not 0 <= cfg.env_idx < sim.num_envs:
      raise ValueError(f"env_idx {cfg.env_idx} outside [0, {sim.num_envs})")
    self._cfg, self._sim = cfg, sim
    body = tracked_body(sim.mj_model, cfg)
    dev = torch.device(sim.device)
    h, w = cfg.height, cfg.width
    self._rgb = torch.zeros((h, w, 3), dtype=torch.uint8, device=dev)
    self._depth = torch.zeros((h, w), dtype=torch.float32, device=dev) if extra_outputs else None
    self._seg = torch.zeros((h, w, 2), dtype=torch.int32, device=dev) if extra_outputs else None
    a = self._args = native.B2RenderArgs()
    a.width, a.height = w, h
    a.lookat[:] = [float(x) for x in cfg.lookat]
    a.track_body = body
    a.distance, a.azimuth, a.elevation = float(cfg.distance), float(cfg.azimuth), float(cfg.elevation)
    a.env_idx, a.noverlay, a.shadows, a.brute = int(cfg.env_idx), MAX_ENVS, int(bool(cfg.enable_shadows)), 0
    a.rgb = self._rgb.data_ptr()
    a.depth = self._depth.data_ptr() if extra_outputs else None
    a.seg = self._seg.data_ptr() if extra_outputs else None
    # debug visualisation: the arrow records (filled on the device by DebugVisualizer.add_arrow) and the ghost's
    # one-world engine, made at the first add_ghost_mesh
    self._decor = torch.zeros((native.RENDER_MAXDECOR, native.RENDER_DECOR), dtype=torch.float32, device=dev)
    self._ghost = self._ghost_qpos = None

  def update(self, data=None, debug_vis_callback=None) -> None:
    """Enqueue a frame of the sim's current state (``data`` is accepted for the reference's signature; the kernel
    reads the engine's state on the device).  ``debug_vis_callback(visualizer)`` adds this frame's decoration through
    a ``DebugVisualizer``; decoration does not carry over to the next frame."""
    if self._rgb is None:
      raise ValueError("Renderer closed.")
    a, s = self._args, self._sim
    a.decor, a.ndecor, a.ghost_xpos, a.ghost_xmat = None, 0, None, None
    a.ghost_rgba[:] = [0.0] * 4
    if debug_vis_callback is not None:
      vis = DebugVisualizer(self)
      debug_vis_callback(vis)
      if vis._narrow:
        a.decor, a.ndecor = self._decor.data_ptr(), vis._narrow
    if s._lib.b2_render(s._h, ctypes.byref(a), s._stream()) != 0:
      raise RuntimeError(f"b2sim: {s._lib.b2_last_error().decode()}")

  def _ghost_pose(self, qpos) -> None:
    """Forward kinematics of ``qpos`` in the ghost's one-world engine (same library and model as the sim), enqueued
    on the sim's stream; points the frame's ghost fields at its geom poses."""
    s = self._sim
    if self._ghost is None:
      dev = torch.device(s.device)
      self._ghost = native.Engine(s._lib, s.mj_model, 1, cuda_device=dev.index or 0)
      self._ghost_qpos = _engine_tensor(self._ghost, "qpos", dev)[0]
      self._ghost_xpos = self._ghost.get_field(0, "geom_xpos").ptr
      self._ghost_xmat = self._ghost.get_field(0, "geom_xmat").ptr
    self._ghost_qpos.copy_(_as_device(qpos, self._ghost_qpos.device), non_blocking=True)
    self._ghost.check(s._lib.b2_forward(self._ghost.h, s._stream()))
    self._args.ghost_xpos, self._args.ghost_xmat = self._ghost_xpos, self._ghost_xmat

  def render(self) -> np.ndarray:
    """The last frame as a host ``(height, width, 3)`` uint8 array (waits for it)."""
    if self._rgb is None:
      raise ValueError("Renderer closed.")
    return self._rgb.cpu().numpy().copy()

  def depth(self) -> np.ndarray:
    return self._depth.cpu().numpy().copy()

  def segmentation(self) -> np.ndarray:
    return self._seg.cpu().numpy().copy()

  def close(self) -> None:
    self._rgb = self._depth = self._seg = self._decor = None
    if self._ghost is not None:
      self._ghost.close()
      self._ghost = self._ghost_qpos = None


def _engine_tensor(engine, name: str, dev: torch.device) -> torch.Tensor:
  """A Data field of ``engine`` as a tensor sharing its memory (device memory, or host memory for the host-emulated
  library)."""
  t = engine.get_field(0, name)
  if dev.type == "cuda":
    from mjlab_b200.sim.sim_data import tensor_from_b2

    return tensor_from_b2(t, engine)
  shape = tuple(int(t.shape[k]) for k in range(t.ndim))
  stride = tuple(int(t.stride[k]) for k in range(t.ndim))
  span = 1 + sum((n - 1) * st for n, st in zip(shape, stride))
  buf = (ctypes.c_float * span).from_address(t.ptr)
  return torch.from_numpy(np.frombuffer(buf, dtype=np.float32)).as_strided(shape, stride)


def _as_device(x, dev: torch.device) -> torch.Tensor:
  """``x`` (a tensor or a sequence) as fp32 on ``dev``; host values go through pinned memory, so the copy is enqueued
  without waiting for the stream."""
  if isinstance(x, torch.Tensor) and x.device == dev:
    return x.to(torch.float32)
  t = torch.as_tensor(np.asarray(x.cpu() if isinstance(x, torch.Tensor) else x, dtype=np.float32))
  if dev.type == "cuda":
    t = t.pin_memory().to(dev, non_blocking=True)
  return t


def _check_color(color) -> tuple:
  c = tuple(float(x) for x in color)
  if len(c) != 4 or not all(math.isfinite(x) and 0.0 <= x <= 1.0 for x in c):
    raise ValueError(f"color must be four finite values in [0, 1] (rgba), got {tuple(color)}")
  return c


class DebugVisualizer:
  """What a debug-vis callback draws into one frame (the reference's ``DebugVisualizer``,
  ``viewer/debug_visualizer.py``, as its ``MujocoNativeDebugVisualizer`` draws it): arrows and a ghost of the robot,
  blended over the scene as one translucent layer (DESIGN.md §4.4).  Nothing here waits for the device: device tensors
  are copied on the sim's stream."""

  def __init__(self, renderer: OffscreenRenderer):
    self.env_idx = renderer._cfg.env_idx
    self._r = renderer
    self._narrow = 0
    self._ghosted = False

  def add_arrow(self, start, end, color, width: float = 0.015) -> None:
    """An arrow from ``start`` to ``end`` (world, 3 values each: tensors or sequences), ``width`` the shaft's radius.
    ``color`` is rgba in [0, 1], or a device tensor of 4 (taken as given, e.g. alpha 0 to hide the arrow)."""
    if self._narrow >= native.RENDER_MAXDECOR:
      raise ValueError(f"at most {native.RENDER_MAXDECOR} arrows per frame")
    if not (math.isfinite(width) and width > 0.0):
      raise ValueError(f"width must be positive and finite, got {width}")
    row = self._r._decor[self._narrow]
    dev = row.device
    for k, (x, what) in enumerate(((start, "start"), (end, "end"))):
      if (x.numel() if isinstance(x, torch.Tensor) else len(x)) != 3:
        raise ValueError(f"{what} must have 3 values")
      row[3 * k:3 * k + 3].copy_(_as_device(x, dev).reshape(3), non_blocking=True)
    if isinstance(color, torch.Tensor) and color.device == dev:
      row[6:7].copy_(_as_device([width], dev), non_blocking=True)
      row[7:11].copy_(color.reshape(4))
    else:
      row[6:11].copy_(_as_device([width, *_check_color(color)], dev), non_blocking=True)
    self._narrow += 1

  def add_ghost_mesh(self, qpos, color) -> None:
    """The robot's dynamic geoms posed at ``qpos`` (the model's nq values: a tensor or a sequence), all drawn in
    ``color`` (rgba in [0, 1]).  Its forward kinematics runs in a one-world engine of the sim's model."""
    n = qpos.numel() if isinstance(qpos, torch.Tensor) else len(qpos)
    nq = int(self._r._sim.mj_model.nq)
    if n != nq:
      raise ValueError(f"qpos has {n} values, the model has nq = {nq}")
    c = _check_color(color)
    if self._ghosted:
      raise ValueError("one ghost per frame")
    self._r._ghost_pose(qpos.reshape(-1) if isinstance(qpos, torch.Tensor) else qpos)
    self._r._args.ghost_rgba[:] = c
    self._ghosted = True


RENDER_MODES = [None, "rgb_array"]  # the reference ManagerBasedRlEnv's metadata["render_modes"]


def task_viewer(**overrides) -> ViewerConfig:
  """The velocity and tracking tasks' camera (velocity_env_cfg.py:41-48, tracking_env_cfg.py:45-52): tracks a body of
  the robot, whose name the robot's cfg sets (``body_name``), with ``overrides`` on top."""
  return ViewerConfig(**{**dict(origin_type=ViewerConfig.OriginType.ASSET_BODY, asset_name="robot", body_name="",
                                distance=3.0, elevation=-5.0, azimuth=90.0), **overrides})


def check_render_mode(render_mode) -> None:
  if render_mode not in RENDER_MODES:
    raise ValueError(f"Render mode {render_mode} is not supported. Please use: {RENDER_MODES}.")


def env_renderer(sim, cfg: ViewerConfig, render_mode) -> OffscreenRenderer | None:
  """The renderer of an env made with ``render_mode`` (None: no renderer, nothing allocated)."""
  check_render_mode(render_mode)
  return OffscreenRenderer(sim, cfg) if render_mode == "rgb_array" else None


def env_render(renderer: OffscreenRenderer | None, debug_vis_callback=None) -> np.ndarray | None:
  """``env.render()``: None without a renderer, else a frame of the state after the last step, with the decoration
  ``debug_vis_callback`` adds (the env's ``update_visualizers``)."""
  if renderer is None:
    return None
  renderer.update(debug_vis_callback=debug_vis_callback)
  return renderer.render()

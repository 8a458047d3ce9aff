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

  def update(self, data=None) -> None:
    """Enqueue a frame of the sim's current state (``data`` is accepted for the reference's signature; the kernel
    reads the engine's state on the device)."""
    if self._rgb is None:
      raise ValueError("Renderer closed.")
    s = self._sim
    if s._lib.b2_render(s._h, ctypes.byref(self._args), s._stream()) != 0:
      raise RuntimeError(f"b2sim: {s._lib.b2_last_error().decode()}")

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
    self._rgb = self._depth = self._seg = None


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


def env_render(renderer: OffscreenRenderer | None) -> np.ndarray | None:
  """``env.render()``: None without a renderer, else a frame of the state after the last step."""
  if renderer is None:
    return None
  renderer.update()
  return renderer.render()

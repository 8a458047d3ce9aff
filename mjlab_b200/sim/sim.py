"""`Simulation` — the drop-in for the reference's ``mjlab.sim.Simulation``
(``src/mjlab/sim/sim.py:94-198``) backed by libb2sim.so instead of mujoco_warp.

Same constructor and methods (``step / forward / create_graph / expand_model_fields / reset /
close``), same properties (``data / model / mj_model / mj_data / wp_model / wp_data``), same
error behaviour (``ValueError("Fields not found in model: ...")``, read-only bridges).
There is no CPU path: constructing a ``Simulation`` without a CUDA device, or without the built
extension, raises.
"""

from __future__ import annotations

import ctypes
from dataclasses import dataclass, field
from types import SimpleNamespace
from typing import Any, Literal

import numpy as np
import torch

from mjlab_b200.compiler.compile import Model
from mjlab_b200.sim import native
from mjlab_b200.sim.sim_data import Bridge, EngineStruct
from mjlab_b200.utils.nan_guard import NanGuard, NanGuardCfg


@dataclass
class MujocoCfg:
  """Physics options; mirrors ``MujocoCfg`` (reference ``sim/sim.py:43-82``)."""

  timestep: float = 0.002
  integrator: Literal["euler", "implicitfast"] = "implicitfast"
  impratio: float = 1.0
  cone: Literal["pyramidal", "elliptic"] = "pyramidal"
  jacobian: Literal["auto", "dense", "sparse"] = "auto"
  solver: Literal["newton", "cg", "pgs"] = "newton"
  iterations: int = 100
  tolerance: float = 1e-8
  ls_iterations: int = 50
  ls_tolerance: float = 0.01
  gravity: tuple = (0, 0, -9.81)

  def validate(self) -> None:
    if self.timestep <= 0:
      raise ValueError("timestep must be positive")

  def edit_spec(self, spec) -> None:
    from mjlab_b200.asset_zoo.scene import apply_mujoco_cfg

    self.validate()
    apply_mujoco_cfg(spec, self)


@dataclass(kw_only=True)
class SimulationCfg:
  nconmax: int | None = None
  njmax: int | None = None
  ls_parallel: bool = True
  mujoco: MujocoCfg = field(default_factory=MujocoCfg)
  nan_guard: NanGuardCfg = field(default_factory=NanGuardCfg)


class Simulation:
  """GPU-resident batched simulation on one H100."""

  def __init__(self, num_envs: int, cfg: SimulationCfg, model: Model, device: str):
    self.cfg = cfg
    self.device = device
    self.num_envs = num_envs
    dev = torch.device(device)
    if dev.type != "cuda":
      raise RuntimeError(
        f"Simulation(device={device!r}): the H100 engine has no CPU path; pass 'cuda:N'"
      )
    if not torch.cuda.is_available():
      raise RuntimeError("Simulation: no CUDA device is available")
    self._dev_index = dev.index if dev.index is not None else torch.cuda.current_device()
    self._mj_model = model
    self._mj_data = SimpleNamespace(
      qpos=np.array(model.qpos0, dtype=np.float64), qvel=np.zeros(int(model.nv)), time=0.0
    )
    lib = native.load_library()
    torch.cuda.synchronize(self._dev_index)
    self._engine = native.Engine(lib, model, num_envs, cfg.nconmax, cfg.njmax, self._dev_index)
    # the env drivers launch their kernels on this library and sim
    self._lib, self._h = lib, self._engine.h

    opt = SimpleNamespace(
      ls_parallel=cfg.ls_parallel, timestep=float(model.opt_timestep),
      iterations=int(model.opt_iterations), ls_iterations=int(model.opt_ls_iterations),
    )
    self._wp_data = EngineStruct(self, 0, {"nworld": num_envs})
    self._wp_model = EngineStruct(
      self, 1, {"opt": opt, "nq": int(model.nq), "nv": int(model.nv), "nu": int(model.nu),
                "nbody": int(model.nbody), "ngeom": int(model.ngeom), "nsite": int(model.nsite)},
    )
    self._model_bridge = Bridge(self._wp_model)
    self._data_bridge = Bridge(self._wp_data)

    # One physics step is one kernel launch, so CUDA graphs buy little; they stay available
    # through create_graph() for API parity and are re-captured lazily after model expansion.
    self.use_cuda_graph = False
    self.step_graph = None
    self.forward_graph = None
    self._graph_dirty = False
    # armed before any graph can be captured, so every graph of this sim carries the guard's stream work
    self.nan_guard = NanGuard(cfg.nan_guard, self._engine, self._mj_model, self._stream)

  # -- plumbing ----------------------------------------------------------------------------------
  def _stream(self) -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream(self._dev_index).cuda_stream)

  def set_option(self, key: str, value: float) -> None:
    self._engine.set_option(key, value)

  def get_option(self, key: str) -> float:
    return self._engine.get_option(key)

  def create_graph(self) -> None:
    """Capture ``step`` and ``forward`` as CUDA graphs (reference ``sim.py:131-140``)."""
    self.step_graph = None
    self.forward_graph = None
    self._graph_dirty = False
    if not self.use_cuda_graph:
      return
    side = torch.cuda.Stream(self._dev_index)
    side.wait_stream(torch.cuda.current_stream(self._dev_index))
    with torch.cuda.stream(side):
      g1 = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g1, stream=side):
        native.check(self._lib.b2_step(self._h, ctypes.c_void_p(side.cuda_stream)))
      g2 = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g2, stream=side):
        native.check(self._lib.b2_forward(self._h, ctypes.c_void_p(side.cuda_stream)))
    torch.cuda.current_stream(self._dev_index).wait_stream(side)
    self.step_graph, self.forward_graph = g1, g2

  # -- properties ---------------------------------------------------------------------------------
  @property
  def mj_model(self) -> Model:
    return self._mj_model

  @property
  def mj_data(self) -> Any:
    return self._mj_data

  @property
  def wp_model(self) -> EngineStruct:
    return self._wp_model

  @property
  def wp_data(self) -> EngineStruct:
    return self._wp_data

  @property
  def data(self) -> Bridge:
    return self._data_bridge

  @property
  def model(self) -> Bridge:
    return self._model_bridge

  # -- methods ------------------------------------------------------------------------------------
  def expand_model_fields(self, fields: list[str]) -> None:
    """Give the named model fields a real per-world leading dimension
    (reference ``sim.py:170-176`` + ``sim/randomization.py:20-55``)."""
    invalid = [f for f in fields if f not in self._mj_model.arrays]
    if invalid:
      raise ValueError(f"Fields not found in model: {invalid}")
    for f in fields:
      native.check(
        self._lib.b2_expand_model_field(self._h, f.encode(), self._stream(), None)
      )
      self._wp_model._drop(f)
      self._model_bridge._invalidate(f)
    self._graph_dirty = True

  def reset(self) -> None:
    pass

  def forward(self, env_mask: torch.Tensor | None = None) -> None:
    """``mjwarp.forward`` for all worlds, or only those selected by a bool ``env_mask`` (extension)."""
    if env_mask is not None:
      if env_mask.dtype != torch.bool or env_mask.numel() != self.num_envs or not env_mask.is_contiguous():
        raise ValueError("env_mask must be a contiguous bool tensor with one entry per env")
      native.check(
        self._lib.b2_forward_masked(self._h, ctypes.c_void_p(env_mask.data_ptr()), self._stream())
      )
      return
    if self.use_cuda_graph and self._graph_dirty:
      self.create_graph()
    if self.use_cuda_graph and self.forward_graph is not None:
      self.forward_graph.replay()
    else:
      native.check(self._lib.b2_forward(self._h, self._stream()))

  def step(self) -> None:
    """One sub-step.  With the NaN guard enabled, and outside a stream capture, it synchronises once at the end and
    writes the guard's dump if this or an earlier sub-step produced NaN/Inf."""
    if self.use_cuda_graph and self._graph_dirty:
      self.create_graph()
    if self.use_cuda_graph and self.step_graph is not None:
      self.step_graph.replay()
    else:
      native.check(self._lib.b2_step(self._h, self._stream()))
    self._check_nan_guard()

  def step_n(self, n: int) -> None:
    """``n`` sub-steps with ``ctrl`` held (the decimation loop of
    ``envs/manager_based_rl_env.py:109-114``) in one library call; the NaN guard as in ``step``."""
    native.check(self._lib.b2_step_n(self._h, int(n), self._stream()))
    self._check_nan_guard()

  def _check_nan_guard(self) -> None:
    if self.nan_guard.enabled and not torch.cuda.is_current_stream_capturing():
      self.nan_guard.check_and_dump()

  def stats(self) -> native.B2Stats:
    st = native.B2Stats()
    native.check(self._lib.b2_stats(self._h, self._stream(), ctypes.byref(st)))
    return st

  def launch_count(self) -> int:
    return int(self._lib.b2_launch_count(self._h))

  def close(self) -> None:
    h = getattr(self, "_h", None)
    if h:
      torch.cuda.synchronize(self._dev_index)
      self.nan_guard.check_and_dump()  # what graphed steps since the last poll found
      # engine memory is about to be freed: drop every cached view and make later field access fail loudly
      for st, br in ((self._wp_data, self._data_bridge), (self._wp_model, self._model_bridge)):
        st._tensors.clear()
        st._closed = True
        object.__getattribute__(br, "_wrapped_cache").clear()
      self._engine.close()
      self._h = None

"""``mujoco_warp`` stand-in over libb2sim.so: the four calls mjlab makes at the engine boundary
(``src/mjlab/sim/sim.py:110`` ``put_model``, ``:113`` ``put_data``, ``:136/195`` ``step``, ``:139/187`` ``forward``)
and the ``Model`` / ``Data`` structs whose array attributes are ``wp.array`` views of engine memory
(``[nworld, ...]``; model fields are shared by all worlds, leading stride 0, until one is assigned a tiled
array — what ``sim/randomization.py:52-55`` does — which switches the engine to a per-world copy).

``put_model`` cannot allocate anything yet (the engine sizes its memory for ``nworld`` worlds, which only
``put_data`` knows), so the ``Model`` it returns binds to the engine when ``put_data`` is called for the same
``mjModel``.
"""

from __future__ import annotations

import ctypes
from types import SimpleNamespace

import torch

from mjlab_b200.sim import native
from mjlab_b200.sim.sim_data import tensor_from_b2

from . import warp_shim as wp

__b2_compat__ = True
__version__ = "0.0-b2compat (libb2sim)"


class _Engine(native.Engine):
  """The engine on the current CUDA device: fields are torch tensors over device memory.  The functions below use only
  lib / h / nworld / device / names / tensor / stream, so that a test double with that interface can stand in."""

  def __init__(self, mjm, nworld: int, nconmax, njmax):
    if not torch.cuda.is_available():
      raise RuntimeError("mujoco_warp (H100 engine): no CUDA device is available; there is no CPU path")
    lib = native.load_library()
    self.device = torch.cuda.current_device()
    torch.cuda.synchronize(self.device)
    super().__init__(lib, mjm, nworld, nconmax, njmax, self.device)

  def tensor(self, which: int, name: str) -> torch.Tensor:
    return tensor_from_b2(self.get_field(which, name), self)

  def stream(self) -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)


class _Struct:
  _which = 0

  def __init__(self):
    object.__setattr__(self, "_engine", None)
    object.__setattr__(self, "_arrays", {})
    object.__setattr__(self, "_plain", {})
    object.__setattr__(self, "__dataclass_fields__", {})

  def _bind(self, engine: _Engine) -> None:
    object.__setattr__(self, "_engine", engine)
    object.__setattr__(self, "__dataclass_fields__", {n: None for n in engine.names(self._which)})

  def __getattr__(self, name):
    if name.startswith("__"):
      raise AttributeError(name)
    plain = object.__getattribute__(self, "_plain")
    if name in plain:
      return plain[name]
    arrays = object.__getattribute__(self, "_arrays")
    if name in arrays:
      return arrays[name]
    eng = object.__getattribute__(self, "_engine")
    if eng is None:
      raise AttributeError(f"'{name}': this Model is not bound to an engine yet (call put_data first)")
    if name not in object.__getattribute__(self, "__dataclass_fields__"):
      raise AttributeError(f"{type(self).__name__} has no field '{name}'")
    a = wp.array(eng.tensor(self._which, name))
    arrays[name] = a
    return a

  def __dir__(self):
    return list(object.__getattribute__(self, "__dataclass_fields__")) + list(object.__getattribute__(self, "_plain"))


class Model(_Struct):
  _which = 1

  def __init__(self, mjm):
    super().__init__()
    self._plain.update(
      mjm=mjm, nq=int(mjm.nq), nv=int(mjm.nv), nu=int(mjm.nu), nbody=int(mjm.nbody), ngeom=int(mjm.ngeom),
      nsite=int(mjm.nsite), njnt=int(mjm.njnt),
      opt=SimpleNamespace(ls_parallel=True, timestep=float(mjm.opt_timestep), iterations=int(mjm.opt_iterations),
                          ls_iterations=int(mjm.opt_ls_iterations)),
    )

  def __setattr__(self, name, value):
    fields = object.__getattribute__(self, "__dataclass_fields__")
    if name in fields and isinstance(value, wp.array):
      # a tiled [nworld, ...] array replaces the shared one: the engine gets a per-world copy of it
      eng = self._engine
      native.check(eng.lib.b2_expand_model_field(eng.h, name.encode(), eng.stream(), None))
      own = eng.tensor(1, name)
      own.copy_(value._t.reshape(own.shape))
      self._arrays[name] = wp.array(own)
      return
    self._plain[name] = value


class Data(_Struct):
  _which = 0

  def __init__(self, nworld: int):
    super().__init__()
    self._plain.update(nworld=int(nworld))


_pending: dict[int, Model] = {}


def put_model(mjm) -> Model:
  m = Model(mjm)
  _pending[id(mjm)] = m
  return m


def put_data(mjm, mjd=None, nworld: int = 1, nconmax=None, njmax=None, **_) -> Data:
  eng = _Engine(mjm, nworld, nconmax, njmax)
  m = _pending.pop(id(mjm), None)
  d = Data(nworld)
  d._bind(eng)
  if m is not None:
    m._bind(eng)
  object.__setattr__(d, "_model", m)
  if mjd is not None and hasattr(mjd, "qpos"):
    import numpy as np

    q = np.asarray(mjd.qpos, dtype=np.float64)
    if q.shape == (int(mjm.nq),) and not np.allclose(q, np.asarray(mjm.qpos0)):
      d.qpos._t[:] = torch.as_tensor(q, dtype=torch.float32, device=d.qpos._t.device)
      native.check(eng.lib.b2_forward(eng.h, eng.stream()))
  return d


def make_data(mjm, nworld: int = 1, nconmax=None, njmax=None, **kw) -> Data:
  return put_data(mjm, None, nworld=nworld, nconmax=nconmax, njmax=njmax, **kw)


def _engine_of(m, d) -> _Engine:
  eng = object.__getattribute__(d, "_engine")
  if m is not None and object.__getattribute__(m, "_engine") is None:
    m._bind(eng)  # a Model made by put_model after its Data (or for a different mjModel object)
  return eng


def step(m: Model, d: Data) -> None:
  eng = _engine_of(m, d)
  native.check(eng.lib.b2_step(eng.h, eng.stream()))


def forward(m: Model, d: Data) -> None:
  eng = _engine_of(m, d)
  native.check(eng.lib.b2_forward(eng.h, eng.stream()))

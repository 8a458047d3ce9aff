"""ctypes loader for the CPU oracle (TEST INFRASTRUCTURE — see oracle/b2_oracle.c header).

Importable only from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / reference arm.
"""

from __future__ import annotations

import ctypes
import subprocess
from pathlib import Path

import numpy as np

from mjlab_b200.sim.native import make_model_desc

_DIR = Path(__file__).parent
_REAL = {"f64": ctypes.c_double, "f32": ctypes.c_float}


def build(force: bool = False) -> None:
  if force or not (_DIR / "libb2oracle64.so").exists() or not (_DIR / "libb2oracle32.so").exists():
    subprocess.check_call(["make", "-C", str(_DIR), "-s"] + (["-B"] if force else []))


def _bind(L: ctypes.CDLL, real) -> ctypes.CDLL:
  """Declare the signature of every b2o_* function of b2_oracle.c on ``L``.

  Without ``argtypes`` ctypes passes a Python int as a C ``int``, which truncates a 64-bit pointer, and a float as a
  double whatever the precision. Pointers are ``c_void_p``, which takes ``None``, a ``c_void_p``, a ``byref`` or any
  ctypes pointer."""
  vp, ci, cd, cs = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_char_p
  signatures = {
    "b2o_create": ([vp, ci, ci, ci], vp),
    "b2o_destroy": ([vp], None),
    "b2o_real_size": ([], ci),
    "b2o_field": ([vp, cs, vp, vp], vp),
    "b2o_model_field": ([vp, cs, vp], vp),
    "b2o_set_option": ([vp, cs, cd], ci),
    "b2o_forward": ([vp, ci], None),
    "b2o_step": ([vp, ci], None),
    "b2o_max_threads": ([], ci),
    "b2o_prim_sphere_box": ([vp, real, vp, vp, vp, real, vp], ci),
    "b2o_prim_capsule_box": ([vp] * 6 + [real, vp], ci),
    "b2o_prim_box_box": ([vp] * 6 + [real, vp], ci),
    "b2o_prim_convex": ([ci, vp, vp, vp, vp, ci, ci, vp, vp, vp, vp, ci, real, real, vp], ci),
    "b2o_prim_plane_mesh": ([vp] * 5 + [ci, real, vp], ci),
    "b2o_prim_plane_smooth": ([vp, vp, ci, vp, vp, vp, real, vp], ci),
    "b2o_prim_hfield": ([vp, vp, vp, ci, ci, vp, ci, vp, vp, vp, vp, ci, real, real, vp], ci),
  }
  for name, (args, res) in signatures.items():
    fn = getattr(L, name)
    fn.argtypes, fn.restype = args, res
  return L


_libs: dict[str, ctypes.CDLL] = {}


def load_library(precision: str = "f64") -> ctypes.CDLL:
  """The oracle library of one precision ("f64" or "f32"), built if needed, loaded once, every function declared."""
  if precision not in _libs:
    real = _REAL[precision]
    build()
    L = _bind(ctypes.CDLL(str(_DIR / f"libb2oracle{precision[1:]}.so")), real)
    if L.b2o_real_size() != ctypes.sizeof(real):
      raise RuntimeError(f"libb2oracle{precision[1:]}.so computes in {L.b2o_real_size()}-byte reals, not {precision}")
    _libs[precision] = L
  return _libs[precision]


class Oracle:
  """One batched oracle instance. Fields are numpy views ``[nworld, n]`` of its memory."""

  def __init__(self, model, nworld: int = 1, maxcon: int = 64, njmax: int = 300,
               precision: str = "f64"):
    self.lib = load_library(precision)
    self._real = _REAL[precision]
    self.dtype = np.float64 if precision == "f64" else np.float32
    self.model = model
    self.nworld = nworld
    desc, self._keep = make_model_desc(model)
    self.h = ctypes.c_void_p(self.lib.b2o_create(ctypes.byref(desc), nworld, maxcon, njmax))
    self._cache = {}

  def __del__(self):
    try:
      self.lib.b2o_destroy(self.h)
    except Exception:
      pass

  def _view(self, p, ct, n: int) -> np.ndarray:
    return np.ctypeslib.as_array((ct * (self.nworld * n)).from_address(p)).reshape(self.nworld, n)

  def field(self, name: str) -> np.ndarray:
    if name in self._cache:
      return self._cache[name]
    n, is_int = ctypes.c_int(0), ctypes.c_int(0)
    p = self.lib.b2o_field(self.h, name.encode(), ctypes.byref(n), ctypes.byref(is_int))
    if not p:
      raise KeyError(name)
    arr = self._view(p, ctypes.c_int if is_int.value else self._real, n.value)
    self._cache[name] = arr
    return arr

  def __getattr__(self, name):
    if name.startswith("_") or name in ("lib", "h", "model", "nworld", "dtype"):
      raise AttributeError(name)
    return self.field(name)

  def model_field(self, name: str) -> np.ndarray:
    n = ctypes.c_int(0)
    p = self.lib.b2o_model_field(self.h, name.encode(), ctypes.byref(n))
    if not p:
      raise KeyError(name)
    return self._view(p, self._real, n.value)

  def set_option(self, key: str, value: float) -> None:
    if self.lib.b2o_set_option(self.h, key.encode(), value):
      raise ValueError(f"the oracle has no option {key!r}")

  def forward(self, nthread: int = 0) -> None:
    self.lib.b2o_forward(self.h, nthread)

  def step(self, nthread: int = 0) -> None:
    self.lib.b2o_step(self.h, nthread)

  def max_threads(self) -> int:
    return int(self.lib.b2o_max_threads())

"""Test double for ``mjlab_b200.compat.mujoco_warp_shim._Engine`` backed by the host-emulated library
(tests/emul/build.py): same C ABI, "device" memory is host memory, fields are torch CPU tensors aliasing it.

Lets the CPU suite run the reference's own ``Simulation`` / ``Entity`` / event code against the product's kernels
(tests/test_reference_dropin.py, backend "emul").  Test infrastructure only: the product's ``_Engine`` refuses to
start without a CUDA device.
"""
import ctypes
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))

from mjlab_b200.sim import native  # noqa: E402

_LIB = None


def load_emul_library(defines=()):
  from build import build

  return native.bind(ctypes.CDLL(str(build(defines=defines))))


def host_tensor(t: native.B2Tensor) -> torch.Tensor:
  """A torch CPU tensor over the (host) memory a B2Tensor of the emulated library describes."""
  shape = tuple(int(t.shape[k]) for k in range(t.ndim))
  stride = tuple(int(t.stride[k]) for k in range(t.ndim))
  dtype = torch.int32 if t.dtype == 1 else torch.float32
  if any(s == 0 for s in shape) or not t.ptr:
    return torch.empty(shape, dtype=dtype)
  span = 1 + sum((s - 1) * st for s, st in zip(shape, stride))
  buf = (ctypes.c_byte * (span * 4)).from_address(t.ptr)
  flat = torch.from_numpy(np.frombuffer(buf, dtype=np.int32 if t.dtype == 1 else np.float32))
  return flat.as_strided(shape, stride)


class EmulEngine(native.Engine):
  """Drop-in for ``_Engine`` (lib / h / nworld / device / names / tensor / stream) on the emulated library."""

  def __init__(self, mjm, nworld: int, nconmax, njmax):
    global _LIB
    if _LIB is None:
      _LIB = load_emul_library()
    super().__init__(_LIB, mjm, nworld, nconmax, njmax)
    self.device = "cpu"
    self.set_option("sorted_dispatch", 0.0)  # (the 1024-thread sort kernel is slow to emulate)

  def tensor(self, which: int, name: str) -> torch.Tensor:
    return host_tensor(self.get_field(which, name))

  def stream(self) -> ctypes.c_void_p:
    return ctypes.c_void_p(0)

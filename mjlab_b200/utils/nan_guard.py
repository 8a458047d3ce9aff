"""NaN guard with the behaviour of the reference's ``utils/nan_guard.py:29-158``: when enabled, keep a short ring buffer
of pre-step states for the first few envs and, the first time a step produces NaN/Inf in
``qpos/qvel/qacc/qacc_warmstart``, dump them to an ``.npz``.  Disabled by default (SURVEY.md §8a S8).

The guard runs on the GPU inside the physics step (``b2_nan_guard``, include/b2sim.h; DESIGN.md §4.3): every sub-step
of ``b2_step`` / ``b2_step_n`` records and checks as stream work, so it also watches steps replayed from a CUDA graph.
The host only reads the result: ``check_and_dump`` synchronises once, ``poll`` reads a host-visible word and
synchronises only when the device has found something.  The ring and the flags freeze at the detection sub-step, so the
dump's content does not depend on when the host looks.

Dump layout: ``nan_env_ids`` (every env non-finite after the detection sub-step), ``num_envs_captured``, and
``qpos_step_%06d`` / ``qvel_step_%06d`` ([num_envs_captured, nq] / [.., nv] float32) for the last ``buffer_size``
sub-steps up to and including the detection sub-step, numbered by sub-step from the guard's start (the state before
that sub-step).
"""

from __future__ import annotations

import ctypes
import os
import tempfile
import time
from collections.abc import Callable
from dataclasses import dataclass
from typing import TYPE_CHECKING

import numpy as np

if TYPE_CHECKING:
  from mjlab_b200.sim import native


@dataclass
class NanGuardCfg:
  enabled: bool = False
  buffer_size: int = 100
  output_dir: str = os.path.join(tempfile.gettempdir(), "mjlab", "nan_dumps")
  max_envs_to_capture: int = 5


class NanGuard:
  """The device guard of one engine (``native.Engine``), armed at construction when ``cfg.enabled``.  ``stream``
  returns the stream the engine's steps run on (``check_and_dump`` synchronises it)."""

  def __init__(self, cfg: NanGuardCfg, engine: native.Engine, model, stream: Callable[[], ctypes.c_void_p]) -> None:
    self.cfg = cfg
    self.enabled = cfg.enabled
    self.num_envs = engine.nworld
    self.num_envs_to_capture = min(self.num_envs, cfg.max_envs_to_capture)
    self._engine, self._stream = engine, stream
    self._nq, self._nv = int(model.nq), int(model.nv)
    self._dumped = False
    self.last_dump_path: str | None = None
    self._word = None
    if self.enabled:
      from mjlab_b200.sim import native  # (the sim package imports this module)

      lib, h = engine.lib, engine.h
      engine.check(lib.b2_nan_guard(h, self.num_envs_to_capture, int(cfg.buffer_size), native.NAN_GUARD_ON))
      self._word = ctypes.c_int32.from_address(lib.b2_nan_guard_word(h))

  def poll(self) -> bool:
    """Dump if the device has found a non-finite state, without synchronising while it has not.  Work still in flight
    is seen by a later call.  Returns whether this call wrote the dump."""
    if not self.enabled or self._dumped or not self._word.value:
      return False
    return self.check_and_dump()

  def check_and_dump(self) -> bool:
    """Synchronise the stream once and dump if the device has found a non-finite state (once per guard)."""
    if not self.enabled or self._dumped:
      return False
    detected = self._read()
    if detected < 0:
      return False
    n, first = self.num_envs_to_capture, max(0, detected - int(self.cfg.buffer_size) + 1)
    states = np.empty((detected - first + 1, n, self._nq + self._nv), dtype=np.float32)
    flags = np.empty(self.num_envs, dtype=np.uint8)
    self._read(states, flags)
    self._dump(np.flatnonzero(flags), first, states)
    self._dumped = True
    return True

  def _read(self, states: np.ndarray | None = None, flags: np.ndarray | None = None) -> int:
    e = self._engine
    d = ctypes.c_int64()
    e.check(e.lib.b2_nan_guard_read(e.h, self._stream(), ctypes.byref(d),
                                    None if states is None else states.ctypes.data,
                                    None if flags is None else flags.ctypes.data))
    return int(d.value)

  def _dump(self, nan_env_ids: np.ndarray, first: int, states: np.ndarray) -> None:
    os.makedirs(self.cfg.output_dir, exist_ok=True)
    stamp = time.strftime("%Y%m%d_%H%M%S")
    path = os.path.join(self.cfg.output_dir, f"nan_dump_{stamp}_{os.getpid()}.npz")
    out = {"nan_env_ids": nan_env_ids, "num_envs_captured": self.num_envs_to_capture}
    for i, s in enumerate(states):
      out[f"qpos_step_{first + i:06d}"] = s[:, :self._nq]
      out[f"qvel_step_{first + i:06d}"] = s[:, self._nq:]
    np.savez_compressed(path, **out)
    self.last_dump_path = path
    print(f"[NanGuard] NaN/Inf detected in envs {nan_env_ids[:10].tolist()}; dumped {path}")

"""Motion clips for the tracking task in the reference's file layout (``tasks/tracking/mdp/commands.py:30-66``,
``MotionLoader``; written by ``scripts/csv_to_npz.py``).

A ``.npz`` holds, for T frames and the entity's bodies in ``EntityIndexing.body_names`` order:
``joint_pos`` / ``joint_vel`` ``[T, nu]`` (entity joint order), ``body_pos_w`` / ``body_lin_vel_w`` /
``body_ang_vel_w`` ``[T, nbody, 3]``, ``body_quat_w`` ``[T, nbody, 4]`` (wxyz), and optionally ``fps``.
"""

from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from mjlab_b200.entity_data import EntityIndexing

KEYS = ("joint_pos", "joint_vel", "body_pos_w", "body_quat_w", "body_lin_vel_w", "body_ang_vel_w")


@dataclass
class MotionClip:
  """A clip restricted to the tracked bodies: contiguous float32 tensors ``[T, nu]`` and ``[T, nb, 3|4]`` (the layout
  the fused tracking kernels index, ``B2TrackEnvArgs.m_*``)."""

  joint_pos: torch.Tensor
  joint_vel: torch.Tensor
  body_pos_w: torch.Tensor
  body_quat_w: torch.Tensor
  body_lin_vel_w: torch.Tensor
  body_ang_vel_w: torch.Tensor

  @property
  def num_frames(self) -> int:
    return int(self.joint_pos.shape[0])

  def as_dict(self) -> dict:
    return {k: getattr(self, k) for k in KEYS}

  @staticmethod
  def load(path, indexing: EntityIndexing, body_names, step_dt: float, device) -> "MotionClip":
    """Read ``path``, check every array against the entity, keep ``body_names`` (in that order).  Raises
    ``ValueError`` naming the offending key and the expected shape."""
    nu, nbody = len(indexing.joint_names), len(indexing.body_names)
    missing = [b for b in body_names if b not in indexing.body_names]
    if missing:
      raise ValueError(f"motion: tracked bodies {missing} are not bodies of the entity")
    with np.load(path) as f:
      data = {k: f[k] for k in f.files}
    T = None
    for k in KEYS:
      if k not in data:
        raise ValueError(f"motion file {path}: missing key '{k}'")
      want = (nu,) if k.startswith("joint") else (nbody, 4 if k == "body_quat_w" else 3)
      a = data[k]
      if a.ndim != 1 + len(want) or tuple(a.shape[1:]) != want or (T is not None and a.shape[0] != T):
        exp = ", ".join(["T" if T is None else str(T)] + [str(s) for s in want])
        raise ValueError(f"motion file {path}: '{k}' has shape {tuple(a.shape)}, expected [{exp}]")
      T = a.shape[0]
      if not np.issubdtype(a.dtype, np.number) or not np.isfinite(a).all():
        raise ValueError(f"motion file {path}: '{k}' holds non-finite or non-numeric values")
    if T < 2:
      raise ValueError(f"motion file {path}: 'joint_pos' has {T} frame(s), expected T >= 2")
    if "fps" in data:
      fps = np.asarray(data["fps"], dtype=np.float64).reshape(-1)
      if fps.size != 1 or not abs(fps[0] * step_dt - 1.0) < 1e-6:
        raise ValueError(f"motion file {path}: 'fps' is {fps.tolist()}, expected [{1.0 / step_dt:g}] (1 / env step_dt)")
    sel = np.array([indexing.body_names.index(b) for b in body_names])
    out = {}
    for k in KEYS:
      a = data[k] if k.startswith("joint") else data[k][:, sel]
      out[k] = torch.tensor(np.ascontiguousarray(a, dtype=np.float32), device=device)
    return MotionClip(**out)

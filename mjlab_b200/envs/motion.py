"""Motion clips for the tracking task in the reference's file layout (``tasks/tracking/mdp/commands.py:30-66``,
``MotionLoader``; written by ``scripts/csv_to_npz.py``), and the converter from CSV recordings to that layout.

A ``.npz`` holds, for T frames and the entity's bodies in ``EntityIndexing.body_names`` order:
``joint_pos`` / ``joint_vel`` ``[T, nu]`` (entity joint order), ``body_pos_w`` / ``body_lin_vel_w`` /
``body_ang_vel_w`` ``[T, nbody, 3]``, ``body_quat_w`` ``[T, nbody, 4]`` (wxyz), and optionally ``fps``.

A CSV recording (e.g. the retargeted LAFAN1 clips for the G1) has one row per frame: root position, root quaternion
(xyzw) and one angle per joint of ``joint_names``.  ``convert_csv`` resamples it to the output rate, differentiates
it, and runs every output frame as one world of a single engine forward to record the body states:

  python -m mjlab_b200.envs.motion IN.csv [IN2.csv ...] --output-dir DIR [--input-fps 30] [--output-fps 50]
                                   [--line-range FIRST LAST] [--device cuda:0]
"""

from __future__ import annotations

import argparse
import warnings
from dataclasses import dataclass
from pathlib import Path

import numpy as np
import torch

from mjlab_b200.entity_data import EntityData, EntityIndexing, quat_apply_inverse, quat_mul

KEYS = ("joint_pos", "joint_vel", "body_pos_w", "body_quat_w", "body_lin_vel_w", "body_ang_vel_w")

# the joint columns of the G1 CSV recordings, in file order (the reference's scripts/csv_to_npz.py)
G1_CSV_JOINTS = (
  "left_hip_pitch_joint", "left_hip_roll_joint", "left_hip_yaw_joint", "left_knee_joint", "left_ankle_pitch_joint",
  "left_ankle_roll_joint", "right_hip_pitch_joint", "right_hip_roll_joint", "right_hip_yaw_joint", "right_knee_joint",
  "right_ankle_pitch_joint", "right_ankle_roll_joint", "waist_yaw_joint", "waist_roll_joint", "waist_pitch_joint",
  "left_shoulder_pitch_joint", "left_shoulder_roll_joint", "left_shoulder_yaw_joint", "left_elbow_joint",
  "left_wrist_roll_joint", "left_wrist_pitch_joint", "left_wrist_yaw_joint", "right_shoulder_pitch_joint",
  "right_shoulder_roll_joint", "right_shoulder_yaw_joint", "right_elbow_joint", "right_wrist_roll_joint",
  "right_wrist_pitch_joint", "right_wrist_yaw_joint")


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


# ---- CSV recordings -> motion files ---------------------------------------------------------------------------------
def read_csv(path, input_fps: float, line_range: tuple[int, int] | None = None, joint_names=G1_CSV_JOINTS,
             device="cpu") -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
  """Rows of a motion CSV as float32 ``(root_pos [N, 3], root_quat [N, 4] wxyz, joint_pos [N, len(joint_names)])``.

  ``line_range=(first, last)`` keeps lines ``first..last`` (1-based, inclusive).  Raises ``ValueError`` naming the
  file and the offending line or column for a bad rate or range, a wrong column count, a non-finite value, a root
  quaternion whose norm is more than 1e-3 from 1 (the engine would normalise it, the finite-difference velocities
  would not match it) and fewer than 2 rows."""
  if not input_fps > 0:
    raise ValueError(f"{path}: input_fps is {input_fps}, expected > 0")
  first, kw = 1, {}
  if line_range is not None:
    first, last = (int(v) for v in line_range)
    if first < 1 or last < first:
      raise ValueError(f"{path}: line_range ({first}, {last}) is reversed or starts before line 1")
    kw = dict(skiprows=first - 1, max_rows=last - first + 1)
  try:
    with warnings.catch_warnings():
      warnings.simplefilter("ignore")  # (loadtxt warns on a range past the end; that is refused below)
      a = np.loadtxt(path, delimiter=",", ndmin=2, **kw)
  except ValueError as e:
    raise ValueError(f"{path}: {e}") from None
  if line_range is not None and a.shape[0] < last - first + 1:
    raise ValueError(f"{path}: line_range ({first}, {last}) is outside the file, which has "
                     f"{first - 1 + a.shape[0]} line(s)")
  if a.shape[0] < 2:
    raise ValueError(f"{path}: {a.shape[0]} frame(s), expected at least 2")
  ncol = 7 + len(joint_names)
  if a.shape[1] != ncol:
    raise ValueError(f"{path}: {a.shape[1]} columns, expected {ncol} (root position 3, root quaternion xyzw 4, "
                     f"joints {len(joint_names)})")
  bad = np.argwhere(~np.isfinite(a))
  if len(bad):
    r, c = bad[0]
    raise ValueError(f"{path}: line {first + r}, column {c + 1} is not finite ({a[r, c]})")
  off = np.abs(np.linalg.norm(a[:, 3:7], axis=1) - 1.0)
  if (off > 1e-3).any():
    r = int(np.argmax(off > 1e-3))
    raise ValueError(f"{path}: line {first + r}: the root quaternion (columns 4-7) has norm "
                     f"{np.linalg.norm(a[r, 3:7]):.6g}, more than 1e-3 from 1")
  m = torch.from_numpy(a).to(torch.float32).to(device)
  return m[:, 0:3], m[:, [6, 3, 4, 5]], m[:, 7:]


def _slerp(a: torch.Tensor, b: torch.Tensor, tau: torch.Tensor) -> torch.Tensor:
  """Row-wise slerp with the branches of the reference's per-frame ``quat_slerp``: ``a`` at ``tau == 0``, at
  ``||a.b| - 1| < 4 eps`` and at an angle below ``4 eps``; ``b`` unchanged at ``tau == 1``; ``b`` negated when
  ``a.b < 0``."""
  eps4 = torch.finfo(a.dtype).eps * 4.0
  d = (a * b).sum(-1)
  flip = d < 0
  b2 = torch.where(flip[:, None], -b, b)
  d = torch.where(flip, -d, d)
  angle = torch.acos(d.clamp(-1, 1))
  isin = 1.0 / torch.sin(angle)
  s = a * torch.sin((1.0 - tau) * angle)[:, None] * isin[:, None] + b2 * torch.sin(tau * angle)[:, None] * isin[:, None]
  s = torch.where((((d - 1.0).abs() < eps4) | (angle < eps4))[:, None], a, s)
  s = torch.where((tau == 1)[:, None], b, s)
  return torch.where((tau == 0)[:, None], a, s)


def _axis_angle(q: torch.Tensor, eps: float = 1.0e-6) -> torch.Tensor:
  """Rotation vectors of unit quaternions (wxyz), with a Taylor form below ``eps`` rad."""
  q = torch.where(q[:, 0:1] < 0, -q, q)
  half = torch.atan2(q[:, 1:].norm(dim=-1), q[:, 0])
  ang = 2.0 * half
  k = torch.where(ang.abs() > eps, torch.sin(half) / ang, 0.5 - ang * ang / 48)
  return q[:, 1:] / k[:, None]


def frame_blend(n: int, input_fps: float, output_fps: float, device) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
  """For each output frame of an ``n``-frame recording: the input frames before and after it and the blend weight of
  the second (the reference's ``MotionLoader._compute_frame_blend``)."""
  if not output_fps > 0:
    raise ValueError(f"output_fps is {output_fps}, expected > 0")
  duration = (n - 1) * (1.0 / input_fps)
  times = torch.arange(0, duration, 1.0 / output_fps, device=device, dtype=torch.float32)
  if times.shape[0] < 3:
    raise ValueError(f"{n} input frames at {input_fps:g} fps give {times.shape[0]} output frame(s) at "
                     f"{output_fps:g} fps, expected at least 3 (the angular velocity is a central difference)")
  phase = times / duration
  i0 = (phase * (n - 1)).floor().long()
  return i0, (i0 + 1).clamp(max=n - 1), phase * (n - 1) - i0


def resample(root_pos: torch.Tensor, root_quat: torch.Tensor, joint_pos: torch.Tensor, input_fps: float,
             output_fps: float) -> dict:
  """The recording at ``output_fps`` with its velocities, as the reference's ``MotionLoader`` computes them: frames at
  ``arange(0, duration, 1 / output_fps)`` (fp32), lerp of positions and joint angles and slerp of the quaternion
  between the two neighbouring input frames, ``torch.gradient`` for the linear and joint velocities, and the SO(3)
  central difference for the angular velocity (world frame) with its first and last samples repeated.

  Returns ``root_pos``, ``root_quat``, ``root_lin_vel_w``, ``root_ang_vel_w``, ``joint_pos``, ``joint_vel``."""
  i0, i1, blend = frame_blend(root_pos.shape[0], input_fps, output_fps, root_pos.device)
  out_dt = 1.0 / output_fps
  w = blend[:, None]
  pos = root_pos[i0] * (1 - w) + root_pos[i1] * w
  jp = joint_pos[i0] * (1 - w) + joint_pos[i1] * w
  quat = _slerp(root_quat[i0], root_quat[i1], blend)
  rel = quat_mul(quat[2:], quat[:-2] * torch.tensor([1.0, -1.0, -1.0, -1.0], device=quat.device))
  ang = _axis_angle(rel) / (2.0 * out_dt)
  return dict(root_pos=pos, root_quat=quat, root_lin_vel_w=torch.gradient(pos, spacing=out_dt, dim=0)[0],
              root_ang_vel_w=torch.cat([ang[:1], ang, ang[-1:]]), joint_pos=jp,
              joint_vel=torch.gradient(jp, spacing=out_dt, dim=0)[0])


def forward_frames(sim, robot: EntityData, root_pos, root_quat, root_lin_vel_w, root_ang_vel_w, joint_pos,
                   joint_vel) -> tuple[dict, np.ndarray]:
  """Body states of T frames, each frame one world of ``sim`` (chunks of its world count; the last chunk is padded
  with its final frame and the padding discarded).  Joint arrays are ``[T, nu]`` in entity joint order.

  Returns the file layout's arrays (host float32) and, per frame, whether the root link's world velocities read back
  after the forward equal the motion's (``torch.testing.assert_close``'s fp32 tolerances)."""
  W, T = sim.data.qpos.shape[0], root_pos.shape[0]
  parts, ok = {k: [] for k in KEYS}, []
  for s in range(0, T, W):
    idx = torch.arange(s, s + W, device=root_pos.device).clamp(max=T - 1)
    q, lin, ang = root_quat[idx], root_lin_vel_w[idx], root_ang_vel_w[idx]
    # free joint: linear velocity in the world frame, angular velocity in the body frame
    robot.write_root_state(torch.cat([root_pos[idx], q, lin, quat_apply_inverse(q, ang)], dim=1))
    robot.write_joint_state(joint_pos[idx], joint_vel[idx])
    sim.forward()
    k = min(W, T - s)
    pose, vel = robot.body_link_pose_w[:k], robot.body_link_vel_w[:k]
    for key, x in (("joint_pos", robot.joint_pos[:k]), ("joint_vel", robot.joint_vel[:k]),
                   ("body_pos_w", pose[..., 0:3]), ("body_quat_w", pose[..., 3:7]),
                   ("body_lin_vel_w", vel[..., 0:3]), ("body_ang_vel_w", vel[..., 3:6])):
      parts[key].append(x.detach().to("cpu", torch.float32).numpy().copy())
    root = robot.root_link_vel_w[:k]
    ok.append(torch.isclose(root, torch.cat([lin, ang], dim=1)[:k], rtol=1.3e-6, atol=1e-5).all(dim=1).cpu())
  return {k: np.concatenate(v) for k, v in parts.items()}, torch.cat(ok).numpy()


def _check_root_velocity(ok: np.ndarray, name) -> None:
  if not ok.all():
    raise ValueError(f"{name}: frame {int(np.argmin(ok))}: the root link's velocity after the forward differs from "
                     f"the motion's (root quaternion not unit, or the entity's root is not its free joint's body)")


def write_motion(path, fps: float, arrays: dict) -> str:
  """Write ``arrays`` (the ``KEYS``) and ``fps=[fps]`` to ``path`` in the reference's layout."""
  np.savez(path, fps=np.array([fps]), **{k: arrays[k] for k in KEYS})
  return str(path)


def record_motion(sim, robot: EntityData, root_pos, root_quat, root_lin_vel_w, root_ang_vel_w, joint_pos, joint_vel,
                  fps: float, path) -> str:
  """Set each frame's state on its own world of ``sim``, run one forward per chunk of worlds, check the root
  velocities read back, and write the motion file ``path`` (every body of the entity, ``body_names`` order)."""
  arrays, ok = forward_frames(sim, robot, root_pos, root_quat, root_lin_vel_w, root_ang_vel_w, joint_pos, joint_vel)
  _check_root_velocity(ok, path)
  return write_motion(path, fps, arrays)


def convert_csv(paths, output_dir, input_fps: float = 30.0, output_fps: float = 50.0,
                line_range: tuple[int, int] | None = None, device="cuda:0", chunk: int = 4096,
                joint_names=G1_CSV_JOINTS, simulation=None) -> list[str]:
  """Convert CSV recordings of the G1 into motion files ``output_dir/<stem>.npz`` for ``TrackingEnvCfg(motion_file=)``.

  Every output frame of every file is one world of a single ``Simulation`` of at most ``chunk`` worlds on
  ``device``.  CSV columns map to the entity's joints by ``joint_names``; joints the CSV lacks keep their
  ``default_joint_pos`` and zero velocity.  ``simulation`` replaces the ``Simulation`` class (same signature).
  Returns the written paths."""
  from mjlab_b200.asset_zoo import load_compiled
  from mjlab_b200.sim import Simulation, SimulationCfg

  paths = [Path(p) for p in ([paths] if isinstance(paths, (str, Path)) else paths)]
  if not paths:
    raise ValueError("convert_csv: no input files")
  if chunk < 1:
    raise ValueError(f"convert_csv: chunk is {chunk}, expected >= 1")
  outs = [Path(output_dir) / f"{p.stem}.npz" for p in paths]
  if len(set(outs)) != len(outs):
    raise ValueError(f"convert_csv: input files share a stem, their outputs would collide: {[str(p) for p in paths]}")
  m = load_compiled("g1_tracking_flat")
  ix = EntityIndexing.from_model(m, "robot", "cpu")
  unknown = [j for j in joint_names if j not in ix.joint_names]
  if unknown:
    raise ValueError(f"convert_csv: CSV joints {unknown} are not joints of the G1")
  cols = torch.tensor([ix.joint_names.index(j) for j in joint_names], device=device)
  default = torch.tensor(m.keys["robot/init_state"]["qpos"], dtype=torch.float32)[ix.joint_q_adr.long()].to(device)
  clips = []
  for p in paths:
    c = resample(*read_csv(p, input_fps, line_range, joint_names, device), input_fps, output_fps)
    T = c["joint_pos"].shape[0]
    jp, jv = default.expand(T, -1).clone(), torch.zeros(T, len(default), device=device)
    jp[:, cols], jv[:, cols] = c["joint_pos"], c["joint_vel"]
    c["joint_pos"], c["joint_vel"] = jp, jv
    clips.append(c)
  frames = [c["joint_pos"].shape[0] for c in clips]
  order = ("root_pos", "root_quat", "root_lin_vel_w", "root_ang_vel_w", "joint_pos", "joint_vel")
  motion = [torch.cat([c[k] for c in clips]) for k in order]
  worlds = min(chunk, sum(frames))
  sim = (simulation or Simulation)(worlds, SimulationCfg(), m, device)
  try:
    robot = EntityData(EntityIndexing.from_model(m, "robot", device), sim.data, sim.model, device, worlds)
    arrays, ok = forward_frames(sim, robot, *motion)
  finally:
    sim.close()
  Path(output_dir).mkdir(parents=True, exist_ok=True)
  start = 0
  for p, out, T in zip(paths, outs, frames):
    _check_root_velocity(ok[start:start + T], p)
    write_motion(out, output_fps, {k: v[start:start + T] for k, v in arrays.items()})
    start += T
  return [str(o) for o in outs]


def main(argv=None) -> None:
  ap = argparse.ArgumentParser(prog="python -m mjlab_b200.envs.motion",
                               description="Convert G1 motion CSVs (root position, root quaternion xyzw, 29 joint "
                                           "angles per row) into motion files for the tracking task.")
  ap.add_argument("inputs", nargs="+", help="CSV files; each is written to OUTPUT_DIR/<stem>.npz")
  ap.add_argument("--output-dir", required=True)
  ap.add_argument("--input-fps", type=float, default=30.0)
  ap.add_argument("--output-fps", type=float, default=50.0)
  ap.add_argument("--line-range", type=int, nargs=2, metavar=("FIRST", "LAST"),
                  help="keep lines FIRST..LAST of each file (1-based, inclusive)")
  ap.add_argument("--device", default="cuda:0")
  a = ap.parse_args(argv)
  for out in convert_csv(a.inputs, a.output_dir, a.input_fps, a.output_fps, a.line_range, a.device):
    print(out)


if __name__ == "__main__":
  main()

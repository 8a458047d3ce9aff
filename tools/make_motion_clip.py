"""Write a time-varying G1 motion clip in the reference's file layout (tasks/tracking/mdp/commands.py:30-66):
  python tools/make_motion_clip.py OUT.npz [--frames 960] [--device cuda:0]

The motion: every joint swings sinusoidally about the KNEES_BENT keyframe, inside its soft limits (the legs only a
little, so the feet stay near the ground), with the analytic joint velocity; the pelvis drifts forward, bobs and
turns slowly.  Body poses and velocities come from one forward with one world per frame, as the reference's
scripts/csv_to_npz.py does (`mjlab_b200.envs.motion.record_motion`: set qpos / qvel, forward, read the link states).  `sim` may be any object with the `Simulation` interface (e.g. one on the host-emulated library)."""

from __future__ import annotations

import argparse
import math
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from mjlab_b200.asset_zoo import load_compiled  # noqa: E402
from mjlab_b200.entity_data import EntityData, EntityIndexing, quat_mul  # noqa: E402
from mjlab_b200.envs.motion import record_motion  # noqa: E402
from mjlab_b200.sim import Simulation, SimulationCfg  # noqa: E402


def motion_law(m, ix: EntityIndexing, soft_limits: torch.Tensor, frames: int, fps: float, device: str):
  """The clip's root and joint states at ``frames`` samples ``1 / fps`` apart, float32: root position, root quaternion
  (wxyz), root linear and angular velocity (world frame), joint positions and velocities (entity joint order).
  ``soft_limits`` is the entity's ``[nu, 2]`` soft joint range."""
  dev = torch.device(device)
  key = torch.tensor(m.keys["robot/init_state"]["qpos"], dtype=torch.float32, device=dev)
  nu = len(ix.joint_names)
  t = torch.arange(frames, dtype=torch.float64, device=dev)[:, None] / fps
  # joints: one sinusoid each (0.3-0.8 Hz, staggered phases), amplitude within the soft limits about the keyframe
  lim = soft_limits.double()
  q0 = key[7:].double().clamp(lim[:, 0], lim[:, 1])
  # (legs swing little, so that the feet stay on the ground: RSI puts the robot in the clip's pose)
  cap = torch.tensor([0.04 if any(s in nm for s in ("hip", "knee", "ankle")) else 0.35 for nm in ix.joint_names],
                     dtype=torch.float64, device=dev)
  amp = torch.minimum(torch.minimum((q0 - lim[:, 0]).clamp(min=0), (lim[:, 1] - q0).clamp(min=0)) * 0.9, cap)
  j = torch.arange(nu, dtype=torch.float64, device=dev)
  w = 2 * math.pi * (0.3 + 0.5 * j / max(nu - 1, 1))
  ph = 0.7 * j
  jp = q0 + amp * torch.sin(w * t + ph)
  jv = amp * w * torch.cos(w * t + ph)
  # root: forward drift 0.3 m/s, 5 mm bob at 1 Hz, yaw rate 0.2 rad/s
  vx, bob, wb, wz = 0.3, 0.005, 2 * math.pi * 1.0, 0.2
  yaw = wz * t[:, 0]
  pos = key[0:3].double().expand(frames, 3).clone()
  pos[:, 0] += vx * t[:, 0]
  pos[:, 2] += bob * torch.sin(wb * t[:, 0])
  qyaw = torch.stack([torch.cos(yaw / 2), 0 * yaw, 0 * yaw, torch.sin(yaw / 2)], dim=1)
  quat = quat_mul(qyaw.float(), key[3:7].expand(frames, 4))
  lin = torch.zeros(frames, 3, dtype=torch.float64, device=dev)
  lin[:, 0] = vx
  lin[:, 2] = bob * wb * torch.cos(wb * t[:, 0])
  ang_w = torch.zeros(frames, 3, device=dev)
  ang_w[:, 2] = wz
  return pos.float(), quat, lin.float(), ang_w, jp.float(), jv.float()


def make_clip(path, frames: int = 960, fps: float = 50.0, device: str = "cuda:0", sim=None, model=None) -> str:
  m = model if model is not None else load_compiled("g1_tracking_flat")
  if sim is None:
    sim = Simulation(frames, SimulationCfg(), m, device)
  ix = EntityIndexing.from_model(m, "robot", device)
  robot = EntityData(ix, sim.data, sim.model, device, frames, soft_joint_pos_limit_factor=0.9)
  motion = motion_law(m, ix, robot.soft_joint_pos_limits[0], frames, fps, device)
  return record_motion(sim, robot, *motion, fps, path)


if __name__ == "__main__":
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("out")
  ap.add_argument("--frames", type=int, default=960)
  ap.add_argument("--fps", type=float, default=50.0)
  ap.add_argument("--device", default="cuda:0")
  a = ap.parse_args()
  print(make_clip(a.out, a.frames, a.fps, a.device))

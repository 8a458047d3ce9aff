"""Speed of the CSV-to-motion-file converter (mjlab_b200.envs.motion.convert_csv) on a GPU: a 20,000-frame G1 clip at
50 fps, written as a 30 fps CSV from tools/make_motion_clip.py's motion law with seeded joint jitter.  Reports output
frames per second end to end and the time split into reading and resampling, engine forwards (chunks of 4096 worlds,
host copies included) and writing, as the median of --reps runs after one warm-up, with the card's name and power
limit read in the same run.  Prints one JSON line.
  python tools/time_motion_csv.py [--frames 20000] [--reps 3] [--device cuda:0]"""

from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import tempfile
import time
import types
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from make_motion_clip import motion_law  # noqa: E402

from mjlab_b200.asset_zoo import load_compiled  # noqa: E402
from mjlab_b200.entity_data import EntityData, EntityIndexing  # noqa: E402
from mjlab_b200.envs.motion import convert_csv, forward_frames, read_csv, resample, write_motion  # noqa: E402
from mjlab_b200.sim import Simulation, SimulationCfg  # noqa: E402


def write_csv(path, frames: int) -> None:
  """``frames`` output frames at 50 fps need ``frames * 30 / 50 + 1`` rows at 30 fps."""
  m = load_compiled("g1_tracking_flat")
  ix = EntityIndexing.from_model(m, "robot", "cpu")
  lim = EntityData(ix, None, types.SimpleNamespace(jnt_range=torch.tensor(m.jnt_range)[None]), "cpu", 1,
                   soft_joint_pos_limit_factor=0.9).soft_joint_pos_limits[0]
  rows = frames * 3 // 5 + 1
  pos, quat, _, _, jp, _ = motion_law(m, ix, lim, rows, 30.0, "cpu")
  jp = jp + torch.from_numpy(np.random.default_rng(0).normal(0.0, 0.01, jp.shape)).float()
  np.savetxt(path, torch.cat([pos, quat[:, [1, 2, 3, 0]], jp], dim=1).double().numpy(), delimiter=",", fmt="%.9g")


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--frames", type=int, default=20000)
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--device", default="cuda:0")
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("time_motion_csv: no CUDA device")
  dev = a.device
  gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
  with tempfile.TemporaryDirectory() as td:
    csv = Path(td) / "clip.csv"
    write_csv(csv, a.frames)
    m = load_compiled("g1_tracking_flat")
    total, read, fwd, write = [], [], [], []
    for rep in range(a.reps + 1):  # rep 0 warms up
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      out = convert_csv([csv], td, device=dev)[0]
      t1 = time.perf_counter()
      c = resample(*read_csv(csv, 30.0, device=dev), 30.0, 50.0)
      torch.cuda.synchronize()
      t2 = time.perf_counter()
      T = c["joint_pos"].shape[0]
      sim = Simulation(min(4096, T), SimulationCfg(), m, dev)
      robot = EntityData(EntityIndexing.from_model(m, "robot", dev), sim.data, sim.model, dev, min(4096, T))
      torch.cuda.synchronize()
      t3 = time.perf_counter()
      arrays, ok = forward_frames(sim, robot, c["root_pos"], c["root_quat"], c["root_lin_vel_w"], c["root_ang_vel_w"],
                                  c["joint_pos"], c["joint_vel"])
      t4 = time.perf_counter()
      write_motion(Path(td) / "again.npz", 50.0, arrays)
      t5 = time.perf_counter()
      sim.close()
      assert ok.all() and T == a.frames, (T, a.frames)
      if rep:
        total.append(t1 - t0); read.append(t2 - t1); fwd.append(t4 - t3); write.append(t5 - t4)
    nbytes = Path(out).stat().st_size
  med = statistics.median
  print(json.dumps(dict(
    gpu=gpu, frames=a.frames, output_frames_per_s=round(a.frames / med(total)), total_s=round(med(total), 4),
    read_and_resample_s=round(med(read), 4), forwards_s=round(med(fwd), 4), write_s=round(med(write), 4),
    file_mb=round(nbytes / 2**20, 1), reps=a.reps, total_s_all=[round(t, 4) for t in total])))


if __name__ == "__main__":
  main()

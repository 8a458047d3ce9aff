"""Cost of the NaN guard on the device: env-steps/s of workload B (G1 velocity, flat) at 4096 envs through the CUDA graph
with the guard off and on (SimulationCfg.nan_guard, the defaults: 5 captured envs, 100 entries), the two envs
alternating in one run so that drift of a shared machine hits them alike.  The guarded env polls the guard after every
step, as it does in training.  Prints one JSON line with the GPU name, its power limit and SM clock, every rate and the
spread.
  python tools/time_nan_guard.py [--envs 4096] [--steps 200] [--warmup 20] [--reps 5]"""

from __future__ import annotations

import argparse
import dataclasses
import json
import subprocess
import sys
import tempfile
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from time_curriculum import steps_per_s  # noqa: E402

from mjlab_b200.envs import VelocityEnvCfg, VelocityFlatEnv  # noqa: E402
from mjlab_b200.utils.nan_guard import NanGuardCfg  # noqa: E402

DEV = "cuda:0"


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--envs", type=int, default=4096)
  ap.add_argument("--steps", type=int, default=200)
  ap.add_argument("--warmup", type=int, default=20)
  ap.add_argument("--preroll", type=int, default=100, help="untimed env steps to the steady mix of resets")
  ap.add_argument("--reps", type=int, default=5)
  a = ap.parse_args()
  query = "name,power.limit,clocks.max.sm,clocks.sm"
  gpu = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
  out_dir = tempfile.mkdtemp(prefix="nan_guard_")
  envs = {}
  for case, on in (("off", False), ("on", True)):  # bench.make_env's B
    cfg = VelocityEnvCfg(num_envs=a.envs, seed=42)
    cfg = dataclasses.replace(cfg, sim=dataclasses.replace(cfg.sim, nan_guard=NanGuardCfg(enabled=on, output_dir=out_dir)))
    envs[case] = VelocityFlatEnv(cfg, device=DEV)
  g = torch.Generator(device=DEV)
  g.manual_seed(0)
  for e in envs.values():
    e.enable_cuda_graph()
  acts = [torch.rand((a.envs, envs["off"].nu), generator=g, device=DEV) * 2 - 1 for _ in range(8)]
  launches = {}
  for k, e in envs.items():
    steps_per_s(e, acts, a.preroll, 0)
    n0 = e.sim.launch_count()
    e.sim.step_n(e.cfg.decimation)  # (one eager decimation loop: the library's launches, which the graph replays)
    launches[k] = e.sim.launch_count() - n0
  rates = {k: [] for k in envs}
  for _ in range(a.reps):
    for k, e in envs.items():
      rates[k].append(steps_per_s(e, acts, a.steps, a.warmup))
  med = {k: sorted(v)[len(v) // 2] for k, v in rates.items()}
  clock = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
  dumped = envs["on"].sim.nan_guard.last_dump_path
  print(json.dumps(dict(
    gpu=gpu, sm_clock_after=clock, envs=a.envs, steps=a.steps, reps=a.reps,
    launches_per_decimation_loop=launches,
    env_steps_per_s={k: [round(x) for x in v] for k, v in rates.items()},
    median_env_steps_per_s={k: round(v) for k, v in med.items()},
    spread={k: round((max(v) - min(v)) / max(v), 5) for k, v in rates.items()},
    cost_on_vs_off_median=round(1 - med["on"] / med["off"], 5),
    dump_written=dumped)))
  for e in envs.values():
    e.close()


if __name__ == "__main__":
  main()

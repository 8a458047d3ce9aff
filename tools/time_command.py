"""Env-steps/s of workloads B (G1 flat) and E (Go1 rough) at 4096 envs through the CUDA graph, each with its defaults
and with the preset of the same robot and terrain (B: Mjlab-Velocity-Flat-Unitree-G1; E: Mjlab-Velocity-Rough-Unitree-Go1
with its terrain and command curricula), alternating the four envs in one run so that drift of a shared machine hits
them alike; plus the time of one b2_velenv_post call from CUDA events.  Prints one JSON line with the GPU name, its
power limit and SM clock, every rate and the spread.
  python tools/time_command.py [--envs 4096] [--steps 200] [--warmup 20] [--reps 3]"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from time_curriculum import post_ms, steps_per_s  # noqa: E402

from mjlab_b200.envs import VelocityEnvCfg, VelocityFlatEnv, velocity_task_cfg  # noqa: E402

DEV = "cuda:0"
WORKLOADS = {  # bench.make_env's B and E, and the preset of the same robot and terrain
  "B": (dict(robot="g1"), "Mjlab-Velocity-Flat-Unitree-G1"),
  "E": (dict(robot="go1", terrain="rough"), "Mjlab-Velocity-Rough-Unitree-Go1"),
}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--envs", type=int, default=4096)
  ap.add_argument("--steps", type=int, default=200)
  ap.add_argument("--warmup", type=int, default=20)
  ap.add_argument("--preroll", type=int, default=100, help="untimed env steps to the steady mix of resets")
  ap.add_argument("--reps", type=int, default=3)
  a = ap.parse_args()
  query = "name,power.limit,clocks.max.sm,clocks.sm"
  gpu = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
  g = torch.Generator(device=DEV)
  g.manual_seed(0)
  envs = {}
  for wl, (kw, task) in WORKLOADS.items():
    envs[f"{wl}_default"] = VelocityFlatEnv(VelocityEnvCfg(num_envs=a.envs, seed=42, **kw), device=DEV)
    envs[f"{wl}_preset"] = VelocityFlatEnv(velocity_task_cfg(task, num_envs=a.envs, seed=42), device=DEV)
  for e in envs.values():
    e.enable_cuda_graph()
  acts = {k: [torch.rand((a.envs, e.nu), generator=g, device=DEV) * 2 - 1 for _ in range(8)] for k, e in envs.items()}
  for k, e in envs.items():
    steps_per_s(e, acts[k], a.preroll, 0)
  rates = {k: [] for k in envs}
  for _ in range(a.reps):
    for k, e in envs.items():
      rates[k].append(steps_per_s(e, acts[k], a.steps, a.warmup))
  med = {k: sorted(v)[len(v) // 2] for k, v in rates.items()}
  logs = {k: {t: round(float(v), 6) for t, v in e.command_log().items()} for k, e in envs.items()}
  post = {k: post_ms(e) for k, e in envs.items()}
  clock = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
  print(json.dumps(dict(
    gpu=gpu, sm_clock_after=clock, envs=a.envs, steps=a.steps, reps=a.reps,
    env_steps_per_s={k: [round(x) for x in v] for k, v in rates.items()},
    median_env_steps_per_s={k: round(v) for k, v in med.items()},
    spread={k: round((max(v) - min(v)) / max(v), 5) for k, v in rates.items()},
    cost_of_preset_median={wl: round(1 - med[f"{wl}_preset"] / med[f"{wl}_default"], 5) for wl in WORKLOADS},
    post_call_us={k: round(1000 * v, 3) for k, v in post.items()}, command_log=logs)))
  for e in envs.values():
    e.close()


if __name__ == "__main__":
  main()

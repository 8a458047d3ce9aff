"""Env-steps/s of workload E (Go1 velocity on the rough box terrain, 4096 envs, through the CUDA graph) with the
terrain-level curriculum off and on, alternating the two in one run so that drift of a shared machine hits both alike;
plus the time of one b2_velenv_post call (the post kernel and, with the curriculum, the one-CTA level mean) from CUDA
events.  Prints one JSON line with the GPU name, its power limit, every rate and the spread.
  python tools/time_curriculum.py [--envs 4096] [--steps 200] [--warmup 20] [--reps 5]"""

from __future__ import annotations

import argparse
import ctypes
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from mjlab_b200.envs import VelocityEnvCfg, VelocityFlatEnv  # noqa: E402
from mjlab_b200.sim import native  # noqa: E402

DEV = "cuda:0"


def steps_per_s(env, acts, steps, warmup):
  for k in range(warmup):
    env.step(acts[k % len(acts)])
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for k in range(steps):
    env.step(acts[k % len(acts)])
  torch.cuda.synchronize()
  return env.num_envs * steps / (time.perf_counter() - t0)


def post_ms(env, launches=2000):
  """One b2_velenv_post call on the env's current state (it rewrites the MDP state; timing only)."""
  sim, A = env.sim, env._native_args
  st = sim._stream()
  call = lambda: native.check(sim._lib.b2_velenv_post(sim._h, ctypes.byref(A), st))  # noqa: E731
  for _ in range(50):
    call()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(launches):
    call()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / launches


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--envs", type=int, default=4096)
  ap.add_argument("--steps", type=int, default=200)
  ap.add_argument("--warmup", type=int, default=20)
  ap.add_argument("--preroll", type=int, default=100, help="untimed env steps to the steady mix of resets")
  ap.add_argument("--reps", type=int, default=5)
  a = ap.parse_args()
  gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
  g = torch.Generator(device=DEV)
  g.manual_seed(0)
  envs = {}
  for name, on in (("off", False), ("on", True)):
    e = VelocityFlatEnv(VelocityEnvCfg(robot="go1", terrain="rough", num_envs=a.envs, seed=42, terrain_curriculum=on),
                        device=DEV)
    e.enable_cuda_graph()
    envs[name] = e
  acts = [torch.rand((a.envs, envs["off"].nu), generator=g, device=DEV) * 2 - 1 for _ in range(8)]
  for e in envs.values():
    steps_per_s(e, acts, a.preroll, 0)
  rates = {name: [] for name in envs}
  for _ in range(a.reps):
    for name, e in envs.items():
      rates[name].append(steps_per_s(e, acts, a.steps, a.warmup))
  best = {k: max(v) for k, v in rates.items()}
  med = {k: sorted(v)[len(v) // 2] for k, v in rates.items()}
  on = envs["on"]
  levels = dict(terrain_level_mean=float(on.terrain_level_mean),
                level_histogram=torch.bincount(on.terrain_levels.long(), minlength=on.max_terrain_level).tolist())
  post = {name: post_ms(e) for name, e in envs.items()}
  print(json.dumps(dict(
    gpu=gpu, envs=a.envs, steps=a.steps, reps=a.reps,
    env_steps_per_s={k: [round(x) for x in v] for k, v in rates.items()},
    best_env_steps_per_s={k: round(v) for k, v in best.items()},
    median_env_steps_per_s={k: round(v) for k, v in med.items()},
    spread={k: round((max(v) - min(v)) / max(v), 5) for k, v in rates.items()},
    cost_of_curriculum_median=round(1 - med["on"] / med["off"], 5),
    env_step_ms={k: round(a.envs / v * 1e3, 4) for k, v in med.items()},
    post_call_ms={k: round(v, 5) for k, v in post.items()}, **levels)))
  for e in envs.values():
    e.close()


if __name__ == "__main__":
  main()

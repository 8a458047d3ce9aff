"""Cost of the observation groups' history on the fused path: env-steps/s of workload B (G1 velocity, flat) and C (G1
tracking, synthetic clip) at 4096 envs through the CUDA graph with their default groups and with a history of
--frames frames on the policy and the critic group, alternating the four envs in one run so that drift of a shared
machine hits them alike; plus the time of one b2_obs_history call from CUDA events, and the bytes it moves from the
shapes (each output element is read once from the old history and written once; each frame element is read once).
Prints one JSON line with the GPU name, its power limit and SM clock, every rate and the spread.
  python tools/time_obs_history.py [--envs 4096] [--frames 5] [--steps 200] [--warmup 20] [--reps 3]"""

from __future__ import annotations

import argparse
import ctypes
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from time_curriculum import steps_per_s  # noqa: E402

from mjlab_b200.envs import (ObservationsCfg, ObsGroupCfg, TrackingEnvCfg, TrackingFlatEnv, VelocityEnvCfg,  # noqa: E402
                             VelocityFlatEnv)
from mjlab_b200.sim import native  # noqa: E402

DEV = "cuda:0"


def history_call(env, launches=2000):
  """(us per b2_obs_history call, bytes it moves) on the env's current state; the call shifts the histories."""
  sim, A = env.sim, env.obs_groups._args
  st = sim._stream()
  call = lambda: native.check(sim._lib.b2_obs_history(sim._h, ctypes.byref(A), st))  # noqa: E731
  for _ in range(50):
    call()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(launches):
    call()
  e1.record()
  torch.cuda.synchronize()
  nbytes = 0
  for g in env.obs_groups.active:
    grp = env.obs_groups.groups[g]
    frames = sum(max(t.frames, 1) * t.dim for t in grp.terms)  # elements of the output row
    shifted = sum((max(t.frames, 1) - 1) * t.dim for t in grp.terms)  # of those, read back from the old history
    nbytes += 4 * env.num_envs * (grp.frame_width + shifted + frames)
  nbytes += 2 * env.num_envs  # terminated, truncated
  return 1000 * e0.elapsed_time(e1) / launches, nbytes


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--envs", type=int, default=4096)
  ap.add_argument("--frames", type=int, default=5)
  ap.add_argument("--steps", type=int, default=200)
  ap.add_argument("--warmup", type=int, default=20)
  ap.add_argument("--preroll", type=int, default=100, help="untimed env steps to the steady mix of resets")
  ap.add_argument("--reps", type=int, default=3)
  a = ap.parse_args()
  query = "name,power.limit,clocks.max.sm,clocks.sm"
  gpu = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
  hist = ObservationsCfg(policy=ObsGroupCfg(history_length=a.frames), critic=ObsGroupCfg(history_length=a.frames))
  envs = {  # bench.make_env's B and C, with default groups and with the history
    "B_default": VelocityFlatEnv(VelocityEnvCfg(num_envs=a.envs, seed=42), device=DEV),
    "B_history": VelocityFlatEnv(VelocityEnvCfg(num_envs=a.envs, seed=42, observations=hist), device=DEV),
    "C_default": TrackingFlatEnv(TrackingEnvCfg(num_envs=a.envs, seed=42), device=DEV),
    "C_history": TrackingFlatEnv(TrackingEnvCfg(num_envs=a.envs, seed=42, observations=hist), device=DEV),
  }
  g = torch.Generator(device=DEV)
  g.manual_seed(0)
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
  calls = {}
  for k in ("B_history", "C_history"):
    us, nbytes = history_call(envs[k])
    calls[k] = dict(us=round(us, 3), bytes=nbytes, gb_per_s=round(nbytes / us / 1e3, 1),
                    widths={gr: envs[k].obs_groups.width(gr) for gr in ("policy", "critic")})
  clock = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
  print(json.dumps(dict(
    gpu=gpu, sm_clock_after=clock, envs=a.envs, frames=a.frames, steps=a.steps, reps=a.reps,
    env_steps_per_s={k: [round(x) for x in v] for k, v in rates.items()},
    median_env_steps_per_s={k: round(v) for k, v in med.items()},
    spread={k: round((max(v) - min(v)) / max(v), 5) for k, v in rates.items()},
    cost_vs_default_median={w: round(1 - med[f"{w}_history"] / med[f"{w}_default"], 5) for w in ("B", "C")},
    b2_obs_history=calls)))
  for e in envs.values():
    e.close()


if __name__ == "__main__":
  main()

"""Env-steps/s of workload C (G1 tracking, synthetic clip) at 4096 envs through the CUDA graph with its defaults, with
the Mjlab-Tracking-Flat-Unitree-G1 preset (the configured kernel path with the episode logs on) and with the
No-State-Estimation preset, alternating the three envs in one run so that drift of a shared machine hits them alike;
plus the time of one b2_trackenv_post1 / post2 call from CUDA events.  Prints one JSON line with the GPU name, its
power limit and SM clock, every rate and the spread.
  python tools/time_tracking_terms.py [--envs 4096] [--steps 200] [--warmup 20] [--reps 3]"""

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

from mjlab_b200.envs import TrackingEnvCfg, TrackingFlatEnv, tracking_task_cfg  # noqa: E402
from mjlab_b200.sim import native  # noqa: E402

DEV = "cuda:0"


def call_us(env, name, launches=2000):
  """One b2_trackenv_<name> call on the env's current state (it rewrites the MDP state; timing only)."""
  sim, A = env.sim, env._native_args
  fn, st = getattr(sim._lib, f"b2_trackenv_{name}"), sim._stream()
  call = lambda: native.check(fn(sim._h, ctypes.byref(A), st))  # noqa: E731
  for _ in range(50):
    call()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(launches):
    call()
  e1.record()
  torch.cuda.synchronize()
  return 1000 * e0.elapsed_time(e1) / launches


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
  envs = {  # bench.make_env's C, and the presets on the same synthetic clip
    "C_default": TrackingFlatEnv(TrackingEnvCfg(num_envs=a.envs, seed=42), device=DEV),
    "C_preset_logs": TrackingFlatEnv(tracking_task_cfg("Mjlab-Tracking-Flat-Unitree-G1", num_envs=a.envs, seed=42),
                                     device=DEV),
    "C_no_state_estimation": TrackingFlatEnv(
      tracking_task_cfg("Mjlab-Tracking-Flat-Unitree-G1-No-State-Estimation", num_envs=a.envs, seed=42), device=DEV),
  }
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
  logs = {k: {t: round(float(v), 6) for f in (e.reward_log, e.termination_log, e.command_log) for t, v in f().items()}
          for k, e in envs.items() if e.cfg.episode_logs}
  calls = {k: {c: round(call_us(e, c), 3) for c in ("post1", "post2")} for k, e in envs.items()}
  clock = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
  print(json.dumps(dict(
    gpu=gpu, sm_clock_after=clock, envs=a.envs, steps=a.steps, reps=a.reps,
    env_steps_per_s={k: [round(x) for x in v] for k, v in rates.items()},
    median_env_steps_per_s={k: round(v) for k, v in med.items()},
    spread={k: round((max(v) - min(v)) / max(v), 5) for k, v in rates.items()},
    cost_vs_default_median={k: round(1 - med[k] / med["C_default"], 5) for k in envs if k != "C_default"},
    call_us=calls, logs=logs)))
  for e in envs.values():
    e.close()


if __name__ == "__main__":
  main()

"""Cost of the reset root and joint, push and external-wrench event terms on the fused path: env-steps/s of workload B (G1 velocity, flat)
and C (G1 tracking, synthetic clip) at 4096 envs through the CUDA graph, default against configured:
  B: the reference-style reset_base (x, y in +-0.5, yaw in +-3.14, a velocity range on every axis),
     reset_robot_joints at scale (0.5, 1.5), push_vel=None with the reference's G1 flat push (x, y in +-0.5 every 1 to
     3 s) as a term, and an interval torso wrench;
  C: push_velocity_range=None with an interval push on every axis, and an interval wrench on the torso and ankles.
The envs alternate in one run, so that drift of a shared machine hits them alike.  Also the time of one b2_events call
of each configured env and of one b2_velenv_post call of B (default and configured, on a state with resets) from
CUDA events over many launches.  Prints one JSON line with the GPU name, its power limit and
SM clock, every rate and the spread.
  python tools/time_state_events.py [--envs 4096] [--steps 200] [--warmup 20] [--reps 3]"""

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

from mjlab_b200.envs import (ApplyExternalForceTorqueCfg, EventsCfg, PushBySettingVelocityCfg,  # noqa: E402
                             ResetJointsByScaleCfg, ResetRootStateUniformCfg, TrackingEnvCfg, TrackingFlatEnv,
                             VelocityEnvCfg, VelocityFlatEnv)
from mjlab_b200.sim import native  # noqa: E402

DEV = "cuda:0"
W = ApplyExternalForceTorqueCfg
V5 = {k: (-0.5, 0.5) for k in ("x", "y", "z", "roll", "pitch", "yaw")}
B_TERMS = (ResetRootStateUniformCfg({"x": (-0.5, 0.5), "y": (-0.5, 0.5), "yaw": (-3.14, 3.14)}, V5),
           ResetJointsByScaleCfg((0.5, 1.5), (0.0, 0.0)),
           PushBySettingVelocityCfg({"x": (-0.5, 0.5), "y": (-0.5, 0.5)}, interval_range_s=(1.0, 3.0)),
           W((-10.0, 10.0), (-1.0, 1.0), names="torso_link", interval_range_s=(1.0, 3.0)))
C_TERMS = (PushBySettingVelocityCfg(V5, interval_range_s=(1.0, 3.0)),
           W((-10.0, 10.0), (-1.0, 1.0), names=("torso_link", ".*_ankle_roll_link"), interval_range_s=(1.0, 3.0)))


def events_call(env, A, launches=2000):
  """us per b2_events call of argument block A on the env's current state."""
  sim, st = env.sim, env.sim._stream()
  call = lambda: native.check(sim._lib.b2_events(sim._h, ctypes.byref(A), st))  # noqa: E731
  for _ in range(50):
    call()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(launches):
    call()
  e1.record()
  torch.cuda.synchronize()
  return 1000 * e0.elapsed_time(e1) / launches


def post_call(env, launches=2000):
  """us per b2_velenv_post call on the env's current state (timing only: the call rewrites the MDP state)."""
  sim, A = env.sim, env._native_args
  st = sim._stream()
  env.episode_length_buf.fill_(env.max_episode_length - 1)  # every call resets every env: the reset branch runs
  call = lambda: native.check(sim._lib.b2_velenv_post(sim._h, ctypes.byref(A), st))  # noqa: E731
  for _ in range(50):
    call()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(launches):
    env.episode_length_buf.fill_(env.max_episode_length - 1)
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
  envs = {
    "B_default": VelocityFlatEnv(VelocityEnvCfg(num_envs=a.envs, seed=42), device=DEV),
    "B_state": VelocityFlatEnv(VelocityEnvCfg(num_envs=a.envs, seed=42, push_vel=None,
                                              events=EventsCfg(terms=B_TERMS)), device=DEV),
    "C_default": TrackingFlatEnv(TrackingEnvCfg(num_envs=a.envs, seed=42), device=DEV),
    "C_state": TrackingFlatEnv(TrackingEnvCfg(num_envs=a.envs, seed=42, push_velocity_range=None,
                                              events=EventsCfg(terms=C_TERMS)), device=DEV),
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
  # B: the launch before the forward; C: the launch after the observations (its pushes and wrenches)
  calls = {"B_state": round(events_call(envs["B_state"], envs["B_state"].events._args), 3),
           "C_state": round(events_call(envs["C_state"], envs["C_state"].events._args_after), 3)}
  # (a fill_ per call in both: it is timed alike for default and configured)
  post = {k: round(post_call(envs[k]), 3) for k in ("B_default", "B_state")}
  clock = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
  print(json.dumps(dict(
    gpu=gpu, sm_clock_after=clock, envs=a.envs, steps=a.steps, reps=a.reps,
    env_steps_per_s={k: [round(x) for x in v] for k, v in rates.items()},
    median_env_steps_per_s={k: round(v) for k, v in med.items()},
    spread={k: round((max(v) - min(v)) / max(v), 5) for k, v in rates.items()},
    cost_vs_default_median={w: round(1 - med[f"{w}_state"] / med[f"{w}_default"], 5) for w in ("B", "C")},
    b2_events_us=calls, b2_velenv_post_all_reset_us=post)))
  for e in envs.values():
    e.close()


if __name__ == "__main__":
  main()

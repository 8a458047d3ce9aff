"""Cost of per-term observation noise on the fused path: env-steps/s of workload B (G1 velocity, flat) and C (G1
tracking, synthetic clip) at 4096 envs through the CUDA graph with their default groups and with a noise-configured
policy group (the task's default uniform noise re-expressed through the noise path, a Gaussian base_ang_vel and a
per-component additive bias on projected_gravity (B) / joint_pos (C)), alternating the four envs in one run so that
drift of a shared machine hits them alike; plus the time of one b2_obs_history call from CUDA events over --launches
calls, and the bytes it moves from the shapes (per element: the source value and the output written once, the draw it
reads and, for a bias term, the bias read and written; terminated and truncated once per env).
Prints one JSON line with the GPU name, its power limit and SM clock, every rate and the spread.
  python tools/time_obs_noise.py [--envs 4096] [--steps 200] [--warmup 20] [--reps 3] [--launches 2000]"""

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

from mjlab_b200.envs import (GaussianNoiseCfg, NoiseModelWithAdditiveBiasCfg, ObservationsCfg,  # noqa: E402
                             ObsGroupCfg, TrackingEnvCfg, TrackingFlatEnv, UniformNoiseCfg, VelocityEnvCfg,
                             VelocityFlatEnv)
from mjlab_b200.sim import native  # noqa: E402

DEV = "cuda:0"


def configured(bias_term: str) -> ObservationsCfg:
  bias = NoiseModelWithAdditiveBiasCfg(noise_cfg=UniformNoiseCfg(n_min=-0.05, n_max=0.05),
                                       bias_noise_cfg=UniformNoiseCfg(n_min=-0.02, n_max=0.02))
  return ObservationsCfg(policy=ObsGroupCfg(noise={"base_ang_vel": GaussianNoiseCfg(mean=0.0, std=0.2),
                                                   bias_term: bias}))


def noise_call(env, launches):
  """(us per b2_obs_history call, bytes it moves) on the env's current state (the call redraws the biases of the
  state's reset envs)."""
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
  nbytes = 2 * env.num_envs  # terminated, truncated
  for g in env.obs_groups.active:
    grp = env.obs_groups.groups[g]
    for t in grp.terms:
      per = 2 * max(t.frames, 1) - 1 + 1  # history shifted (read + write of the older frames, the new one written), source
      if t.noise is not None:
        per += t.noise.noise.ndraw > 0
        per += 2 * (t.noise.bias is not None)
      nbytes += 4 * env.num_envs * t.dim * per
  return 1000 * e0.elapsed_time(e1) / launches, nbytes


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--envs", type=int, default=4096)
  ap.add_argument("--steps", type=int, default=200)
  ap.add_argument("--warmup", type=int, default=20)
  ap.add_argument("--preroll", type=int, default=100, help="untimed env steps to the steady mix of resets")
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--launches", type=int, default=2000)
  a = ap.parse_args()
  query = "name,power.limit,clocks.max.sm,clocks.sm"
  gpu = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
  envs = {  # bench.make_env's B and C, with default groups and with the noise-configured policy group
    "B_default": VelocityFlatEnv(VelocityEnvCfg(num_envs=a.envs, seed=42), device=DEV),
    "B_noise": VelocityFlatEnv(VelocityEnvCfg(num_envs=a.envs, seed=42, observations=configured("projected_gravity")),
                               device=DEV),
    "C_default": TrackingFlatEnv(TrackingEnvCfg(num_envs=a.envs, seed=42), device=DEV),
    "C_noise": TrackingFlatEnv(TrackingEnvCfg(num_envs=a.envs, seed=42, observations=configured("joint_pos")),
                               device=DEV),
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
  for k in ("B_noise", "C_noise"):
    us, nbytes = noise_call(envs[k], a.launches)
    calls[k] = dict(us=round(us, 3), bytes=nbytes, gb_per_s=round(nbytes / us / 1e3, 1),
                    widths={gr: envs[k].obs_groups.width(gr) for gr in ("policy", "critic")},
                    draws=dict(W=envs[k].obs_groups.nW, N=envs[k].obs_groups.nN))
  clock = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
  print(json.dumps(dict(
    gpu=gpu, sm_clock_after=clock, envs=a.envs, steps=a.steps, reps=a.reps,
    env_steps_per_s={k: [round(x) for x in v] for k, v in rates.items()},
    median_env_steps_per_s={k: round(v) for k, v in med.items()},
    spread={k: round((max(v) - min(v)) / max(v), 5) for k, v in rates.items()},
    cost_vs_default_median={w: round(1 - med[f"{w}_noise"] / med[f"{w}_default"], 5) for w in ("B", "C")},
    b2_obs_history=calls)))
  for e in envs.values():
    e.close()


if __name__ == "__main__":
  main()

"""Env-steps/s of workloads E (Go1 rough, terrain curriculum) and B (G1 flat) at 4096 envs through the CUDA graph with
every opt-in reward term (VelocityEnvCfg.rewards) off and on, alternating the four envs in one run so that drift of a
shared machine hits them alike; plus the time of one b2_velenv_post call from CUDA events.  Prints one JSON line with
the GPU name, its power limit, every rate and the spread.
  python tools/time_rewards.py [--envs 4096] [--steps 200] [--warmup 20] [--reps 5]"""

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

from mjlab_b200.envs import VelocityEnvCfg, VelocityFlatEnv  # noqa: E402
from mjlab_b200.envs.velocity_env import VelocityRewardsCfg  # noqa: E402

DEV = "cuda:0"
FEET = {"go1": ("FR", "FL", "RR", "RL"), "g1": ("left", "right")}
GEOM = {"go1": "{}_foot_collision", "g1": "{}_foot1_collision"}


def all_terms(robot: str) -> VelocityRewardsCfg:
  """Every opt-in term at a non-zero weight, feet_slide and foot_clearance on the robot's feet."""
  feet = FEET[robot]
  return VelocityRewardsCfg(
    air_time=1.0, feet_slide=-0.25, foot_clearance=0.5, is_alive=0.1, is_terminated=-1.0, joint_torques_l2=-1e-4,
    joint_acc_l2=-2.5e-7, electrical_power_cost=-2e-3, flat_orientation_l2=-1.0,
    feet_slide_sensor_names=tuple(f"{f}_foot_ground_contact" for f in feet),
    feet_slide_geom_names=tuple(GEOM[robot].format(f) for f in feet),
    foot_clearance_geom_names=tuple(GEOM[robot].format(f) for f in feet), target_height=0.1, std=0.05, tanh_mult=2.0)


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
  workloads = {"E": dict(robot="go1", terrain="rough", terrain_curriculum=True), "B": dict(robot="g1")}
  envs = {}
  for wl, kw in workloads.items():
    for name, on in (("off", False), ("on", True)):
      cfg = VelocityEnvCfg(num_envs=a.envs, seed=42, **kw)
      if on:
        cfg.rewards = all_terms(kw["robot"])
      e = VelocityFlatEnv(cfg, device=DEV)
      e.enable_cuda_graph()
      envs[f"{wl}_{name}"] = e
  acts = {k: [torch.rand((a.envs, e.nu), generator=g, device=DEV) * 2 - 1 for _ in range(8)] for k, e in envs.items()}
  for k, e in envs.items():
    steps_per_s(e, acts[k], a.preroll, 0)
  rates = {k: [] for k in envs}
  for _ in range(a.reps):
    for k, e in envs.items():
      rates[k].append(steps_per_s(e, acts[k], a.steps, a.warmup))
  med = {k: sorted(v)[len(v) // 2] for k, v in rates.items()}
  logs = {k: {t: round(float(v), 6) for t, v in e.reward_log().items()} for k, e in envs.items() if k.endswith("_on")}
  post = {k: post_ms(e) for k, e in envs.items()}
  print(json.dumps(dict(
    gpu=gpu, envs=a.envs, steps=a.steps, reps=a.reps,
    env_steps_per_s={k: [round(x) for x in v] for k, v in rates.items()},
    median_env_steps_per_s={k: round(v) for k, v in med.items()},
    spread={k: round((max(v) - min(v)) / max(v), 5) for k, v in rates.items()},
    cost_of_terms_median={wl: round(1 - med[f"{wl}_on"] / med[f"{wl}_off"], 5) for wl in workloads},
    post_call_ms={k: round(v, 5) for k, v in post.items()}, reward_log=logs)))
  for e in envs.values():
    e.close()


if __name__ == "__main__":
  main()

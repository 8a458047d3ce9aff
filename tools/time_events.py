"""Cost of the reset and interval randomize_field events on the fused path: env-steps/s of workload B (G1 velocity,
flat) and C (G1 tracking, synthetic clip) at 4096 envs through the CUDA graph with their default events and with
(i) a reset-mode body_mass scale on every body, a feet geom_friction abs and an interval dof_damping scale, and
(ii) the same plus a reset-mode body_pos add.  Case (ii) expands body_pos, which takes the step kernel off its compact
kinematic records (DESIGN.md §4.3), so its rate includes that physics cost and is reported on its own.  The envs
alternate in one run, so that drift of a shared machine hits them alike.  Also the time of one b2_events call from
CUDA events over many launches.  Prints one JSON line with the GPU name, its power limit and SM clock, every rate and
the spread.
  python tools/time_events.py [--envs 4096] [--steps 200] [--warmup 20] [--reps 3]"""

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

from mjlab_b200.asset_zoo import g1  # noqa: E402
from mjlab_b200.envs import (EventsCfg, RandomizeFieldCfg, TrackingEnvCfg, TrackingFlatEnv, VelocityEnvCfg,  # noqa: E402
                             VelocityFlatEnv)
from mjlab_b200.sim import native  # noqa: E402

DEV = "cuda:0"
R = RandomizeFieldCfg
EVENTS = (R("body_mass", (0.8, 1.2), mode="reset", operation="scale"),
          R("geom_friction", (0.3, 1.2), mode="reset", operation="abs", names=tuple(g1.FOOT_GEOMS)),
          R("dof_damping", (0.8, 1.25), mode="interval", operation="scale", interval_range_s=(1.0, 3.0)))
BODY_POS = R("body_pos", (-0.005, 0.005), mode="reset", operation="add", names=".*_ankle_roll_link")


def events_call(env, launches=2000):
  """us per b2_events call on the env's current state (the call rewrites the fields of the envs in reset_buf)."""
  sim, A = env.sim, env.events._args
  st = sim._stream()
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
  cases = {"default": EventsCfg(), "events": EventsCfg(terms=EVENTS), "events_body_pos": EventsCfg(terms=EVENTS + (BODY_POS,))}
  envs = {}
  for c, ev in cases.items():  # bench.make_env's B and C
    envs[f"B_{c}"] = VelocityFlatEnv(VelocityEnvCfg(num_envs=a.envs, seed=42, events=ev), device=DEV)
    envs[f"C_{c}"] = TrackingFlatEnv(TrackingEnvCfg(num_envs=a.envs, seed=42, events=ev), device=DEV)
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
  calls = {k: dict(us=round(events_call(envs[k]), 3), entries=int(envs[k].events._args.nelem))
           for k in ("B_events", "C_events")}
  clock = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
  print(json.dumps(dict(
    gpu=gpu, sm_clock_after=clock, envs=a.envs, steps=a.steps, reps=a.reps,
    env_steps_per_s={k: [round(x) for x in v] for k, v in rates.items()},
    median_env_steps_per_s={k: round(v) for k, v in med.items()},
    spread={k: round((max(v) - min(v)) / max(v), 5) for k, v in rates.items()},
    cost_vs_default_median={f"{w}_{c}": round(1 - med[f"{w}_{c}"] / med[f"{w}_default"], 5)
                            for w in ("B", "C") for c in ("events", "events_body_pos")},
    b2_events=calls)))
  for e in envs.values():
    e.close()


if __name__ == "__main__":
  main()

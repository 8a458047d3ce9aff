"""Env-steps/s of the motion-tracking task at 4096 envs through the CUDA graph, for the synthetic static clip, a
generated moving clip (tools/make_motion_clip.py) with uniform start frames (the sampler switched off), and the same
clip with the adaptive sampler; plus the time of one b2_trackenv_bins launch from CUDA events.  Prints one JSON line with the GPU name and
power limit.
  python tools/time_tracking_clip.py [--envs 4096] [--steps 200] [--warmup 20] [--frames 960] [--reps 3]"""

from __future__ import annotations

import argparse
import ctypes
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from make_motion_clip import make_clip  # noqa: E402

from mjlab_b200.envs.tracking_env import TrackingEnvCfg, TrackingFlatEnv  # noqa: E402
from mjlab_b200.sim import native  # noqa: E402

DEV = "cuda:0"


def steps_per_s(env, steps, warmup):
  g = torch.Generator(device=DEV)
  g.manual_seed(0)
  acts = [torch.rand((env.num_envs, env.nu), generator=g, device=DEV) * 2 - 1 for _ in range(8)]
  for k in range(warmup):
    env.step(acts[k % 8])
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for k in range(steps):
    env.step(acts[k % 8])
  torch.cuda.synchronize()
  return env.num_envs * steps / (time.perf_counter() - t0)


def bins_kernel_ms(env, launches=2000):
  sim, A = env.sim, env._native_args
  st = sim._stream()
  call = lambda: native.check(sim._lib.b2_trackenv_bins(sim._h, ctypes.byref(A), st))  # noqa: E731
  for _ in range(50):
    call()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()  # (the sim launches on the current stream)
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
  ap.add_argument("--frames", type=int, default=960)
  ap.add_argument("--reps", type=int, default=3)
  a = ap.parse_args()
  gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
  with tempfile.TemporaryDirectory() as tmp:
    clip = make_clip(Path(tmp) / "clip.npz", frames=a.frames, device=DEV)
    torch.cuda.empty_cache()
    cases = {"synthetic": dict(), "clip_uniform": dict(motion_file=clip), "clip_adaptive": dict(motion_file=clip)}
    envs = {}
    for name, kw in cases.items():
      e = TrackingFlatEnv(TrackingEnvCfg(num_envs=a.envs, **kw), device=DEV)
      if name == "clip_uniform":  # the same clip with the sampler off: uniform start frames, no b2_trackenv_bins
        e.start_mode = native.START_UNIFORM
      e.enable_cuda_graph()
      envs[name] = e
    rates = {name: [] for name in cases}
    for _ in range(a.reps):  # alternate the cases, so that drift of the shared machine hits all three alike
      for name, e in envs.items():
        rates[name].append(steps_per_s(e, a.steps, a.warmup))
    ad = envs["clip_adaptive"]
    ms = bins_kernel_ms(ad)
    best = {k: max(v) for k, v in rates.items()}
    step_ms = a.envs / best["clip_adaptive"] * 1e3
    print(json.dumps(dict(
      gpu=gpu, envs=a.envs, clip_frames=a.frames, nbins=ad.bin_count, steps=a.steps, reps=a.reps,
      env_steps_per_s={k: [round(x) for x in v] for k, v in rates.items()},
      best_env_steps_per_s={k: round(v) for k, v in best.items()},
      env_step_ms_adaptive=round(step_ms, 4), bins_kernel_ms=round(ms, 5),
      bins_kernel_share_of_env_step=round(ms / step_ms, 5),
      sampling=dict(entropy=float(ad._metrics[0]), top1_prob=float(ad._metrics[1]), top1_bin=float(ad._metrics[2])))))
    for e in envs.values():
      e.close()


if __name__ == "__main__":
  main()

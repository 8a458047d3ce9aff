"""Cost of the debug visualisation in offscreen frames (csrc/b2_render.cuh's decoration items, mjlab_b200/render.py's
DebugVisualizer).  For the G1 velocity env (the command's four arrows) and the G1 tracking env (the motion's ghost), at
--envs envs after 20 zero-action steps, with the task presets' camera, at 320 x 240 and 1280 x 720:
  - kernel_ms: b2_render kernel time per frame, CUDA events over --frames launches after 20 warm-up launches, without
    and with the decoration the env's update_visualizers adds (filled once, then the same launch repeated);
  - update_ms: OffscreenRenderer.update() per frame with the callback (the decoration's small torch kernels and, for
    the ghost, its forward kinematics), CUDA events;
  - render_ms: env.render() end to end (host clock, ending in the copy to the host), debug_vis off and on.
Prints one JSON line per measurement with the GPU's name and power limit.
  python tools/time_render_debug_vis.py [--envs 4096] [--frames 200]"""

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

from mjlab_b200.envs import (TrackingFlatEnv, VelocityCommandCfg, VelocityFlatEnv, tracking_task_cfg,  # noqa: E402
                             velocity_task_cfg)

DEV = "cuda:0"
SIZES = ((320, 240), (1280, 720))


def make_env(kind: str, envs: int, debug_vis: bool, w: int, h: int):
  if kind == "velocity":
    cfg = velocity_task_cfg("Mjlab-Velocity-Flat-Unitree-G1", num_envs=envs,
                            command=VelocityCommandCfg(debug_vis=debug_vis))
    cls = VelocityFlatEnv
  else:
    cfg = tracking_task_cfg("Mjlab-Tracking-Flat-Unitree-G1", num_envs=envs, debug_vis=debug_vis)
    cls = TrackingFlatEnv
  cfg.viewer.width, cfg.viewer.height = w, h
  env = cls(cfg, render_mode="rgb_array")
  act = torch.zeros(envs, env.nu, device=DEV)
  for _ in range(20):
    env.step(act)
  return env


def events_ms(fn, frames: int) -> float:
  for _ in range(20):
    fn()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(frames):
    fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b) / frames


def measure(kind: str, envs: int, frames: int, w: int, h: int, debug_vis: bool) -> dict:
  env = make_env(kind, envs, debug_vis, w, h)
  r, s = env._offline_renderer, env.sim
  cb = env.update_visualizers if debug_vis else None
  r.update(debug_vis_callback=cb)  # leaves this frame's decoration in the launch arguments

  def launch():
    if s._lib.b2_render(s._h, ctypes.byref(r._args), s._stream()) != 0:
      raise RuntimeError(s._lib.b2_last_error().decode())

  row = dict(kernel_ms=events_ms(launch, frames), ndecor=int(r._args.ndecor), ghost=bool(r._args.ghost_xpos),
             update_ms=events_ms(lambda: r.update(debug_vis_callback=cb), frames))
  env.render()
  torch.cuda.synchronize()
  t = time.perf_counter()
  for _ in range(50):
    env.render()
  row["render_ms"] = (time.perf_counter() - t) * 1e3 / 50
  env.close()
  del env
  torch.cuda.empty_cache()
  return row


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--envs", type=int, default=4096)
  ap.add_argument("--frames", type=int, default=200)
  a = ap.parse_args()
  gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()[0]
  for kind in ("velocity", "tracking"):
    for w, h in SIZES:
      for debug_vis in (False, True, False, True):
        row = dict(gpu=gpu, env=kind, envs=a.envs, width=w, height=h, debug_vis=debug_vis,
                   **measure(kind, a.envs, a.frames, w, h, debug_vis))
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
  main()

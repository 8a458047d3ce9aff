"""Cost of offscreen frames (b2_render, csrc/b2_render.cuh) on the GPU.  For each workload (G1 flat and Go1 on the
height-field terrain, both at --envs worlds after a short random-control rollout, the task presets' tracking camera)
and each image size (320 x 240, 1280 x 720): kernel time per frame (CUDA events over --frames launches after
warm-up) with the tile cull and with the brute-force loop (B2RenderArgs.brute), and OffscreenRenderer.update() +
render() end to end (host clock, ending in the copy to the host).  Then the G1 velocity env's env-steps/s with and
without one env.render() per step.  Prints one JSON line per measurement with the GPU's name and power limit, and saves
each workload's first frame as PNG under --out when PIL imports.
  python tools/time_render.py [--envs 4096] [--frames 200] [--out DIR]  (default DIR: time_render in the temp dir)"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from mjlab_b200.asset_zoo import load_compiled  # noqa: E402
from mjlab_b200.envs import VelocityFlatEnv, velocity_task_cfg  # noqa: E402
from mjlab_b200.render import OffscreenRenderer, ViewerConfig  # noqa: E402
from mjlab_b200.sim import Simulation, SimulationCfg  # noqa: E402

DEV = "cuda:0"
WORKLOADS = (("g1_flat", "torso_link", 3.0, -5.0), ("go1_rough_hf", "trunk", 1.5, -10.0))
SIZES = ((320, 240), (1280, 720))


def kernel_ms(r: OffscreenRenderer, frames: int, brute: int) -> float:
  r._args.brute = brute
  for _ in range(20):
    r.update()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(frames):
    r.update()
  b.record()
  b.synchronize()
  r._args.brute = 0
  return a.elapsed_time(b) / frames


def end_to_end_ms(r: OffscreenRenderer, frames: int) -> float:
  r.update()
  r.render()
  torch.cuda.synchronize()
  t = time.perf_counter()
  for _ in range(frames):
    r.update()
    r.render()
  return (time.perf_counter() - t) * 1e3 / frames


def env_rate(render: bool, envs: int, steps: int) -> float:
  env = VelocityFlatEnv(velocity_task_cfg("Mjlab-Velocity-Flat-Unitree-G1", num_envs=envs),
                        render_mode="rgb_array" if render else None)
  env.enable_cuda_graph()
  act = torch.zeros(envs, env.nu, device=DEV)
  for _ in range(20):
    env.step(act)
    env.render()
  torch.cuda.synchronize()
  t = time.perf_counter()
  for _ in range(steps):
    env.step(act)
    env.render()
  torch.cuda.synchronize()
  rate = envs * steps / (time.perf_counter() - t)
  env.close()
  return rate


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--envs", type=int, default=4096)
  ap.add_argument("--frames", type=int, default=200)
  ap.add_argument("--steps", type=int, default=200)
  ap.add_argument("--out", default=str(Path(tempfile.gettempdir()) / "time_render"))
  a = ap.parse_args()
  gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()[0]
  out = Path(a.out)
  out.mkdir(parents=True, exist_ok=True)
  try:
    from PIL import Image
  except ImportError:
    Image = None
  for name, body, distance, elevation in WORKLOADS:
    m = load_compiled(name)
    sim = Simulation(a.envs, SimulationCfg(), m, DEV)
    key = m.keys["robot/init_state"]
    sim.data.qpos[:] = torch.tensor(key["qpos"], dtype=torch.float32, device=DEV)
    sim.forward()
    g = torch.Generator(device=DEV).manual_seed(0)
    for _ in range(20):
      sim.data.ctrl[:] = torch.tensor(key["ctrl"], dtype=torch.float32, device=DEV) + 0.3 * (
        2 * torch.rand(a.envs, int(m.nu), device=DEV, generator=g) - 1)
      sim.step()
    for w, h in SIZES:
      cfg = ViewerConfig(origin_type=ViewerConfig.OriginType.ASSET_BODY, asset_name="robot", body_name=body,
                         distance=distance, elevation=elevation, width=w, height=h)
      r = OffscreenRenderer(sim, cfg)
      row = dict(gpu=gpu, workload=name, envs=a.envs, ngeom=int(m.ngeom), width=w, height=h,
                 kernel_ms=kernel_ms(r, a.frames, 0), kernel_brute_ms=kernel_ms(r, a.frames, 1),
                 render_ms=end_to_end_ms(r, 50))
      print(json.dumps(row), flush=True)
      if Image is not None:
        r.update()
        Image.fromarray(r.render()).save(out / f"{name}_{w}x{h}.png")
      r.close()
    sim.close()
    del sim
    torch.cuda.empty_cache()
  for render in (False, True, False, True):
    print(json.dumps(dict(gpu=gpu, workload="velocity G1 flat env", envs=a.envs, render_per_step=render,
                          env_steps_per_s=env_rate(render, a.envs, a.steps))), flush=True)


if __name__ == "__main__":
  main()

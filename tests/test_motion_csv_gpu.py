"""CSV recordings converted into motion files on the H100 (mjlab_b200.envs.motion.convert_csv): the same file as the
host-emulated library's, a long clip in several chunks, and the tracking env running on it through its CUDA graph
with the NaN guard armed."""

import dataclasses

import numpy as np
import pytest
import torch

from mjlab_b200.sim import Simulation, native
from test_motion_csv import convert, csv_joints, write_csv

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


class CountingSimulation(Simulation):
  worlds, forwards = [], 0

  def __init__(self, num_envs, *a, **k):
    CountingSimulation.worlds.append(num_envs)
    super().__init__(num_envs, *a, **k)

  def forward(self, env_mask=None):
    CountingSimulation.forwards += 1
    super().forward(env_mask)


def test_fixture_on_the_h100_matches_the_emulated_library(tmp_path, monkeypatch):
  from mjlab_b200.envs.motion import convert_csv

  path = write_csv(tmp_path / "clip.csv")
  gpu = dict(np.load(convert_csv([path], tmp_path / "gpu", device=DEV, joint_names=csv_joints())[0]))
  monkeypatch.setattr(native, "check", lambda rc: (_ for _ in ()).throw(RuntimeError("b2sim call failed")) if rc else None)
  emu = dict(np.load(convert([path], tmp_path / "emul")[0]))
  assert list(gpu) == list(emu) and gpu["fps"].tolist() == [50.0]
  for k in ("joint_pos", "joint_vel", "body_pos_w", "body_quat_w", "body_lin_vel_w", "body_ang_vel_w"):
    assert gpu[k].shape == emu[k].shape and gpu[k].dtype == np.float32, k
    tol = 1e-5 if k in ("joint_pos", "body_pos_w", "body_quat_w") else 1e-4
    assert np.abs(gpu[k] - emu[k]).max() <= tol, (k, np.abs(gpu[k] - emu[k]).max())


@pytest.fixture(scope="module")
def long_clip(tmp_path_factory):
  """9001 rows at 30 fps: 15000 frames at 50 fps, converted in chunks of 4096 worlds."""
  from mjlab_b200.envs.motion import convert_csv

  d = tmp_path_factory.mktemp("long")
  path = write_csv(d / "long.csv", frames=9001, flip=None, repeat=None)
  CountingSimulation.worlds, CountingSimulation.forwards = [], 0
  out = convert_csv([path], d, device=DEV, joint_names=csv_joints(), simulation=CountingSimulation)[0]
  assert CountingSimulation.worlds == [4096] and CountingSimulation.forwards == 4
  return path, out


def test_long_clip_converts_in_four_chunks(long_clip, tmp_path):
  from mjlab_b200.envs.motion import convert_csv

  path, out = long_clip
  chunked = dict(np.load(out))
  assert chunked["joint_pos"].shape == (15000, 29)
  CountingSimulation.worlds, CountingSimulation.forwards = [], 0
  whole = dict(np.load(convert_csv([path], tmp_path, device=DEV, joint_names=csv_joints(), chunk=15000,
                                   simulation=CountingSimulation)[0]))
  assert CountingSimulation.worlds == [15000] and CountingSimulation.forwards == 1
  for k, v in whole.items():  # each world's forward is its own: the chunking changes no bit
    assert np.array_equal(v, chunked[k]), k


def test_tracking_env_runs_on_the_converted_clip_through_its_cuda_graph(long_clip, tmp_path):
  from mjlab_b200.envs import TrackingEnvCfg, TrackingFlatEnv
  from mjlab_b200.utils.nan_guard import NanGuardCfg

  n = 4096
  cfg = TrackingEnvCfg(num_envs=n, seed=7, motion_file=long_clip[1])
  guard = NanGuardCfg(enabled=True, output_dir=str(tmp_path / "dumps"))
  e = TrackingFlatEnv(dataclasses.replace(cfg, sim=dataclasses.replace(cfg.sim, nan_guard=guard)), device=DEV)
  assert e.T == 15000 and e.sim.nan_guard.enabled
  e.enable_cuda_graph()
  g = torch.Generator(device=DEV)
  g.manual_seed(3)
  for _ in range(200):
    ob, rb, tb, ub, x = e.step(torch.rand((n, e.nu), generator=g, device=DEV) * 2 - 1)
  torch.cuda.synchronize()
  assert torch.isfinite(ob).all() and torch.isfinite(rb).all() and torch.isfinite(x["critic"]).all()
  assert (e.time_steps >= 0).all() and (e.time_steps < e.T).all()
  assert not e.sim.nan_guard.check_and_dump() and not (tmp_path / "dumps").exists()
  e.close()

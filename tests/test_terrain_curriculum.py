"""Terrain-level curriculum of the velocity task (VelocityEnvCfg.terrain_curriculum): the torch restatement against
the reference's own terrain_levels_vel / TerrainImporter.update_env_origins, the fused post kernel against the torch
path (host-emulated library here, the GPU under -m gpu), and on the GPU that pushed robots move up, held robots move
down and robots past the last row are redrawn."""

import ctypes
import importlib.util
import math
import sys
import types

import numpy as np
import pytest
import torch

import refload
from mjlab_b200.sim import native


def _stand_in(origins, levels, types_, env_origins, root_xy, command, episode_length_s=20.0, size=8.0):
  """The attributes of VelocityFlatEnv that its curriculum step reads and writes."""
  rows = origins.shape[0]
  qpos = torch.zeros(len(levels), 19)
  qpos[:, 0:2] = root_xy
  return types.SimpleNamespace(
    env_origins=env_origins.clone(), command=command.clone(), sim=types.SimpleNamespace(data=types.SimpleNamespace(qpos=qpos)),
    cfg=types.SimpleNamespace(episode_length_s=episode_length_s), move_up_dist=size / 2, max_terrain_level=rows,
    terrain_origins=origins, terrain_levels=levels.to(torch.int32).clone(), terrain_types=types_.to(torch.int32).clone(),
    terrain_level_mean=torch.zeros(()))


def _seeded_states(n=600, seed=0):
  """Origins of the go1_rough grid, levels at 0 / in the middle / at the last row, roots at 0..9 m from their origins
  (some exactly at the thresholds), commands with standing (zero) rows, a done mask and the step's uniforms."""
  from mjlab_b200.asset_zoo import load_compiled

  g = torch.Generator().manual_seed(seed)
  origins = torch.tensor(np.asarray(load_compiled("go1_rough").arrays["terrain_origins"]), dtype=torch.float32)
  rows, cols = origins.shape[:2]
  levels = torch.randint(0, rows, (n,), generator=g)
  levels[: n // 4] = 0
  levels[n // 4: n // 2] = rows - 1
  types_ = torch.randint(0, cols, (n,), generator=g)
  env_origins = origins[levels, types_]
  ang = torch.rand(n, generator=g) * 2 * math.pi
  r = torch.rand(n, generator=g) * 9.0
  command = torch.stack([torch.rand(n, generator=g) * 2 - 1, torch.rand(n, generator=g) - 0.5, torch.zeros(n)], 1)
  command[::5] = 0.0
  root_xy = env_origins[:, 0:2] + torch.stack([r * torch.cos(ang), r * torch.sin(ang)], 1)
  root_xy[0::7] = env_origins[0::7, 0:2] + torch.tensor([4.0, 0.0])  # exactly half a sub-terrain: not a move up
  root_xy[1::7] = env_origins[1::7, 0:2] + torch.tensor([1.0, 0.0])
  command[1::7] = torch.tensor([0.1, 0.0, 0.0])  # exactly the move-down threshold (1 m at 20 s): not a move down
  done = torch.rand(n, generator=g) < 0.7
  U = torch.rand(n, 16, generator=g)
  return origins, levels, types_, env_origins, root_xy, command, done, U


def _ref_curriculum(monkeypatch):
  """The reference's tasks/velocity/mdp/curriculums.py and terrains/terrain_importer.py, executed from oracle/_ref."""
  if not refload.available():
    pytest.skip("the reference package is not installed (oracle/install_reference.py)")
  refload.load()
  from mjlab.terrains.terrain_importer import TerrainImporter

  vc = types.ModuleType("mjlab.tasks.velocity.mdp.velocity_command")  # only a type cast of commands_vel
  vc.UniformVelocityCommandCfg = type("UniformVelocityCommandCfg", (), {})
  monkeypatch.setitem(sys.modules, vc.__name__, vc)
  name = "mjlab.tasks.velocity.mdp.curriculums"
  spec = importlib.util.spec_from_file_location(name, refload.REF / "mjlab" / "tasks" / "velocity" / "mdp" / "curriculums.py")
  mod = importlib.util.module_from_spec(spec)
  monkeypatch.setitem(sys.modules, name, mod)
  spec.loader.exec_module(mod)
  return mod, TerrainImporter


def _ref_env(TerrainImporter, origins, levels, types_, env_origins, root_xy, command, episode_length_s=20.0):
  """A minimal ManagerBasedRlEnv for terrain_levels_vel: the robot's root position, the command, and a
  TerrainImporter holding the grid, the levels and the origins (its update_env_origins is the reference's)."""
  terrain = object.__new__(TerrainImporter)
  terrain.cfg = types.SimpleNamespace(terrain_generator=types.SimpleNamespace(size=(8.0, 8.0)))
  terrain.terrain_origins = origins
  terrain.env_origins = env_origins.clone()
  terrain.terrain_levels = levels.clone()
  terrain.terrain_types = types_.clone()
  terrain.max_terrain_level = origins.shape[0]
  robot = types.SimpleNamespace(data=types.SimpleNamespace(root_link_pos_w=torch.cat([root_xy, torch.zeros(len(levels), 1)], 1)))

  class Scene(dict):
    pass

  scene = Scene(robot=robot)
  scene.terrain = terrain
  scene.env_origins = terrain.env_origins
  cmd = command.clone()
  return types.SimpleNamespace(scene=scene, command_manager=types.SimpleNamespace(get_command=lambda name: cmd),
                               max_episode_length_s=episode_length_s)


def test_torch_curriculum_matches_reference_terrain_levels_vel(monkeypatch):
  from mjlab_b200.envs.velocity_env import VelocityFlatEnv

  mod, TerrainImporter = _ref_curriculum(monkeypatch)
  origins, levels, types_, env_origins, root_xy, command, done, U = _seeded_states()
  rows = origins.shape[0]
  ref = _ref_env(TerrainImporter, origins, levels, types_, env_origins, root_xy, command)
  mod.terrain_levels_vel(ref, torch.nonzero(done).squeeze(1), "twist")
  ours = _stand_in(origins, levels, types_, env_origins, root_xy, command)
  VelocityFlatEnv._terrain_curriculum(ours, done, torch.cat([U, torch.rand(len(U), 30)], 1))
  ref_lv, ref_org = ref.scene.terrain.terrain_levels, ref.scene.terrain.env_origins
  lv = ours.terrain_levels.long()
  dist = (root_xy - env_origins[:, 0:2]).norm(dim=1)
  redrawn = done & (levels == rows - 1) & (dist > 4.0)
  same = ~redrawn
  assert torch.equal(lv[same], ref_lv[same]) and torch.equal(ours.env_origins[same], ref_org[same])
  # the redraw: torch.randint_like there, floor(U[:, 12] rows) here - both a row of the grid
  assert redrawn.sum() > 20
  assert ((ref_lv[redrawn] >= 0) & (ref_lv[redrawn] < rows)).all()
  assert torch.equal(lv[redrawn], (U[redrawn, 12] * rows).floor().long().clamp(max=rows - 1))
  assert torch.equal(ours.env_origins, origins[lv, types_])
  assert float(ours.terrain_level_mean) == float(lv.float().mean())
  # every branch was taken, and the not-done envs kept their level and origin
  moved = lv - levels
  assert ((moved == 1) & same & done).sum() > 20 and ((moved == -1) & done).sum() > 20
  assert ((moved == 0) & (levels == 0) & done & (dist < 1.0)).sum() > 5  # a move down clipped at row 0
  assert ((moved == 0) & done & ~redrawn).sum() > 20
  assert torch.equal(lv[~done], levels[~done]) and torch.equal(ours.env_origins[~done], env_origins[~done])
  # the mean the reference logs, where nothing is redrawn
  keep = levels < rows - 1
  ref = _ref_env(TerrainImporter, origins, levels[keep], types_[keep], env_origins[keep], root_xy[keep], command[keep])
  mean = mod.terrain_levels_vel(ref, torch.nonzero(done[keep]).squeeze(1), "twist")
  ours = _stand_in(origins, levels[keep], types_[keep], env_origins[keep], root_xy[keep], command[keep])
  VelocityFlatEnv._terrain_curriculum(ours, done[keep], U[keep])
  assert torch.equal(ours.terrain_levels.long(), ref.scene.terrain.terrain_levels)
  assert float(ours.terrain_level_mean) == float(mean)


def test_curriculum_needs_a_terrain_grid():
  from mjlab_b200.envs import VelocityEnvCfg, VelocityFlatEnv

  with pytest.raises(ValueError, match="sub-terrain origins"):
    VelocityFlatEnv(VelocityEnvCfg(robot="go1", terrain="flat", num_envs=2, terrain_curriculum=True), device="cpu")


def test_post_kernel_refuses_curriculum_without_tables():
  """The curriculum without its tables is refused, and so are a zeroed command block and a block without the arrays
  every step writes."""
  sys.path.insert(0, str(refload.ROOT / "tests" / "emul"))
  from engine import load_emul_library

  from mjlab_b200.asset_zoo import load_compiled

  lib = load_emul_library(())
  e = native.Engine(lib, load_compiled("go1_flat"), 1)
  curriculum, zeroed, no_arrays = native.B2VelEnvArgs(), native.B2VelEnvArgs(), native.B2VelEnvArgs()
  curriculum.curriculum, curriculum.rows, curriculum.cols = 1, 10, 20
  no_arrays.resample_lo = 3.0
  for a, match in ((curriculum, b"terrain curriculum"), (zeroed, b"the command needs"),
                   (no_arrays, b"needs episode_sums")):
    assert lib.b2_velenv_post(e.h, ctypes.byref(a), None) != 0
    assert match in lib.b2_last_error()
  e.close()


def _twin_envs(make, cfg):
  """The same env on the torch path (a) and the fused kernels (b), with a few envs moved to the last row."""
  a, b = make(cfg, native_mdp=False), make(cfg, native_mdp=True)
  top = a.max_terrain_level - 1
  for e in (a, b):
    e.terrain_levels[::5] = top
    e.env_origins[::5] = e.terrain_origins[top, e.terrain_types[::5].long()]
  return a, b


def _run_twins(a, b, steps, p_teleport, teleport_every=3):
  """Zero actions (the same ctrl on both paths, so the same physics); every few steps some robots are moved 5 m along
  x and dropped from 1 m, so that they move up at their next reset.  Levels, origins, done and the reset root
  positions must be identical; b is re-synchronised to a after every step (the reset yaw uses fast-math sines)."""
  n, dev = a.num_envs, a.device
  g = torch.Generator(device="cpu").manual_seed(7)
  act = torch.zeros(n, a.nu, device=dev)
  top = a.max_terrain_level - 1
  counts = dict(up=0, down=0, redraw=0, done=0)
  for k in range(steps):
    if k % teleport_every == 0:
      sel = (torch.rand(n, generator=g) < p_teleport).to(dev)
      for e in (a, b):
        e.sim.data.qpos[:, 0] = torch.where(sel, e.sim.data.qpos[:, 0] + 5.0, e.sim.data.qpos[:, 0])
        e.sim.data.qpos[:, 2] = torch.where(sel, e.sim.data.qpos[:, 2] + 1.0, e.sim.data.qpos[:, 2])
    lv0 = a.terrain_levels.clone()
    _, _, ta, ua, _ = a.step(act)
    _, _, tb, ub, _ = b.step(act)
    da, db = ta | ua, tb | ub
    assert torch.equal(da, db), k
    assert torch.equal(a.terrain_levels, b.terrain_levels), k
    assert torch.equal(a.env_origins, b.env_origins), k
    assert torch.equal(a.sim.data.qpos[:][da, 0:3], b.sim.data.qpos[:][db, 0:3]), k
    assert torch.allclose(a.terrain_level_mean, b.terrain_level_mean, rtol=1e-6, atol=0), k
    d = a.terrain_levels - lv0
    counts["up"] += int((da & (d == 1)).sum())
    counts["down"] += int((da & (d == -1)).sum())
    counts["redraw"] += int((da & (lv0 == top) & (a.terrain_levels < top - 1)).sum())  # below a move down: redrawn
    counts["done"] += int(da.sum())
    for f in ("qpos", "qvel", "qacc_warmstart", "ctrl"):
      getattr(b.sim.data, f)[:] = getattr(a.sim.data, f)[:]
    b.command.copy_(a.command)
    b.heading_target.copy_(a.heading_target)
  return counts


def test_emulated_post_kernel_curriculum_matches_torch(monkeypatch):
  """The fused post kernel on the host-emulated library against the torch path, go1_rough, sharing U."""
  from test_kernel_emul import EmulSimulation

  import mjlab_b200.envs.velocity_env as ve

  monkeypatch.setattr(ve, "Simulation", EmulSimulation)
  monkeypatch.setattr(native, "check", lambda rc: (_ for _ in ()).throw(RuntimeError("b2sim call failed")) if rc else None)
  cfg = ve.VelocityEnvCfg(robot="go1", terrain="rough", num_envs=10, episode_length_s=1.0, terrain_curriculum=True)
  a, b = _twin_envs(lambda c, native_mdp: ve.VelocityFlatEnv(c, device="cpu", native_mdp=native_mdp), cfg)
  # full-length episodes (the move-down distance scales with it) that time out within the run
  ep = torch.randint(a.max_episode_length - 10, a.max_episode_length, (10,), generator=torch.Generator().manual_seed(3))
  for e in (a, b):
    e.episode_length_buf.copy_(ep.int())
  counts = _run_twins(a, b, 10, p_teleport=0.15)
  assert counts["up"] > 0 and counts["down"] > 0 and counts["redraw"] > 0, counts
  a.close()
  b.close()


@pytest.mark.gpu
def test_post_kernel_curriculum_matches_torch_gpu():
  from mjlab_b200.envs import VelocityEnvCfg, VelocityFlatEnv

  cfg = VelocityEnvCfg(robot="go1", terrain="rough", num_envs=256, episode_length_s=1.0, terrain_curriculum=True)
  a, b = _twin_envs(lambda c, native_mdp: VelocityFlatEnv(c, device="cuda:0", native_mdp=native_mdp), cfg)
  counts = _run_twins(a, b, 300, p_teleport=0.03)
  assert counts["up"] > 100 and counts["down"] > 100 and counts["redraw"] > 10, counts
  a.close()
  b.close()


def _flat_columns(env):
  return (env.terrain_origins[:, :, 2] == 0).all(dim=0)


@pytest.mark.gpu
def test_curriculum_moves_levels_gpu():
  """Pushed robots go a row up, robots held still under a command go a row down (or stay at row 0), robots pushed
  off the last row are redrawn from U[:, 12]; all at their first time-out, with the step captured in a CUDA graph."""
  from mjlab_b200.envs import VelocityEnvCfg, VelocityFlatEnv

  n = 256
  env = VelocityFlatEnv(VelocityEnvCfg(robot="go1", terrain="rough", num_envs=n, episode_length_s=2.0, fall_angle=4.0,
                                       terrain_curriculum=True), device="cuda:0")
  rows = env.max_terrain_level
  flat = _flat_columns(env)[env.terrain_types.long()]
  idx = torch.arange(n, device="cuda:0")
  push, hold = flat & (idx % 2 == 0), flat & (idx % 2 == 1)
  last = push & (idx % 6 == 0)
  assert push.sum() > 20 and hold.sum() > 20 and last.sum() > 5
  # robots of `last` start on the last row: same column, same offset from their origin
  new_org = env.terrain_origins[rows - 1, env.terrain_types.long()]
  d = env.sim.data
  d.qpos[:, 0:3] = torch.where(last.unsqueeze(1), d.qpos[:, 0:3] + new_org - env.env_origins, d.qpos[:, 0:3])
  env.env_origins.copy_(torch.where(last.unsqueeze(1), new_org, env.env_origins))
  env.terrain_levels.copy_(torch.where(last, rows - 1, env.terrain_levels))
  env.enable_cuda_graph()  # (its warm-up runs two steps)
  lv0 = env.terrain_levels.clone()
  act = torch.zeros(n, env.nu, device="cuda:0")
  ep_left = env.max_episode_length - int(env.episode_length_buf.max())
  assert ep_left > 10 and bool((env.episode_length_buf == env.episode_length_buf[0]).all())
  for k in range(ep_left):
    d.qvel[:, 0] = torch.where(push, 5.0, d.qvel[:, 0])
    d.qvel[:] = torch.where(hold.unsqueeze(1), 0.0, d.qvel[:])
    env.command[:] = torch.where(hold.unsqueeze(1), torch.tensor([1.0, 0.0, 0.0], device="cuda:0"), env.command)
    _, _, term, trunc, _ = env.step(act)
    if k < ep_left - 1:
      assert not bool((term | trunc).any()) and torch.equal(env.terrain_levels, lv0)
  torch.cuda.synchronize()
  assert bool(trunc.all())
  lv = env.terrain_levels
  up = push & ~last
  assert torch.equal(lv[up], lv0[up] + 1)
  assert torch.equal(lv[hold], (lv0[hold] - 1).clamp(min=0))
  assert torch.equal(lv[last], (env._U[last, 12] * rows).floor().int().clamp(max=rows - 1))
  assert ((lv >= 0) & (lv < rows)).all()
  assert torch.equal(env.env_origins, env.terrain_origins[lv.long(), env.terrain_types.long()])
  assert float(env.terrain_level_mean) == pytest.approx(float(lv.float().mean()), rel=1e-6)
  # every reset spawned within the reset's +-0.5 m of its new origin
  assert ((d.qpos[:, 0:2] - env.env_origins[:, 0:2]).abs() <= 0.5).all()
  env.close()

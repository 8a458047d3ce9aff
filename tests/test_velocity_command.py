"""The velocity command as the reference's tasks configure it (VelocityEnvCfg.command, command_curriculum, posture_std,
velocity_task_cfg, env.command_log()): the torch path against the reference's own code (commands_vel, posture,
UniformVelocityCommand, run from oracle/_ref), the presets against the reference's cfg classes, the fused post kernel
against the torch path on one saved state (the Harness of test_mdp_kernels.py; emul here, the H100 under -m gpu), and
the configurations the env refuses."""

import importlib.util
import json
import math
import os
import subprocess
import sys
import types
from pathlib import Path

import numpy as np
import pytest
import torch

import refload
import test_mdp_kernels as tmk

ROOT = Path(__file__).resolve().parents[1]
BACKENDS = tmk.BACKENDS
COMMAND_ENV = ["common_step_counter", "metric_xy", "metric_yaw", "finished_metrics"]
TASKS = ("Mjlab-Velocity-Flat-Unitree-G1", "Mjlab-Velocity-Flat-Unitree-Go1", "Mjlab-Velocity-Rough-Unitree-Go1")


def _ve():
  import mjlab_b200.envs.velocity_env as ve

  return ve


def _command(**kw):
  base = dict(lin_vel_x=(-0.3, 2.1), lin_vel_y=(0.2, 0.9), ang_vel_z=(-2.0, 0.5), heading=(-1.0, 2.0),
              heading_control_stiffness=0.8, rel_standing_envs=0.3, resampling_time_range=(0.05, 0.15))
  base.update(kw)
  return _ve().VelocityCommandCfg(**base)


def _harness(backend, monkeypatch, task=None, **cfg):
  if task is not None:
    if backend == "emul":
      tmk._patch_emul(monkeypatch, _ve())
    c = _ve().velocity_task_cfg(task, **cfg)
    env = _ve().VelocityFlatEnv(c, device="cpu" if backend == "emul" else "cuda:0", native_mdp=True)
    H = tmk.Harness(env, backend, tmk.VEL_ENV)
  else:
    H = tmk._velocity(backend, monkeypatch, **cfg)
  H.env_fields += COMMAND_ENV
  return H


def _pose64(env, S):
  """Float64 pose term of the saved state: with the env's per-joint widths, and with the default single width."""
  d2 = (S["data.qpos"][:, 7:].double() - env.default_joint_pos.double()) ** 2
  return torch.exp(-(d2 * env.posture_inv_std2.double()).mean(1)), torch.exp(-d2.mean(1) / 0.09)


def _ranges64(env, counter):
  """(x lo, x hi, z lo, z hi) in effect at common_step_counter `counter`, from the cfg (the rule, not the env's table)."""
  cc = env.cfg.command
  x, z = cc.lin_vel_x, cc.ang_vel_z
  for step, rng in env.cfg.command_curriculum:
    if counter > step:
      x = z = rng
  return (*x, *z)


def check(H, S, T, N, action, U):
  """Every output and piece of post-state of the two paths for every env, and each path against the configured
  command: draws inside the ranges in effect, the heading command clamped to the yaw range, the timer inside its
  range, the counter advanced, the metrics handed over."""
  env, tol, c = H.env, H.tol, H.counts
  nu = env.nu
  cc = env.cfg.command
  margin, reward64, scale64 = tmk._velocity_reference(env, S, action)
  pose, single = _pose64(env, S)
  reward64 = reward64 + (pose - single) * env.step_dt
  inband = margin.abs() < tol["band"]
  for R in (T, N):
    H.equal("terminated vs float64", R["out.terminated"][~inband], (margin > 0)[~inband])
  keep = T["out.terminated"] == N["out.terminated"]
  c["in_band"] += int(inband.sum())
  done = T["out.terminated"] | T["out.truncated"]
  dt = np.float32(env.step_dt)
  ctl = S["env.cmd_time_left"].cpu().numpy().astype(np.float32) - dt
  resample = done | torch.from_numpy(ctl <= 0).to(done.device)
  c["done"] += int(done.sum()); c["resample"] += int(resample.sum())
  stages = bool(env.cfg.command_curriculum)
  counter = int(S["env.common_step_counter"][0]) + (1 if stages else 0)
  xlo, xhi, zlo, zhi = _ranges64(env, counter)
  f = lambda v: float(np.float32(v))  # noqa: E731
  for R in (T, N):
    H.equal("counter", R["env.common_step_counter"], torch.full_like(S["env.common_step_counter"], counter))
    H.close("reward vs float64", R["out.reward"], reward64, rowwise=False, scale=scale64)
    cmd, ht, st = R["env.command"], R["env.heading_target"], R["env.is_standing"]
    moving = resample & ~st
    for k, (lo, hi) in enumerate(((xlo, xhi), tuple(cc.lin_vel_y))):
      v = cmd[moving, k]
      assert bool(((v >= f(lo)) & (v <= f(hi))).all()), ("command range", k, v.min(), v.max(), lo, hi)
    h = ht[resample]
    assert bool(((h >= f(cc.heading[0])) & (h <= f(cc.heading[1]))).all()), "heading target range"
    yaw = cmd[~st, 2]
    assert bool(((yaw >= f(zlo)) & (yaw <= f(zhi))).all()), ("yaw clamp", yaw.min(), yaw.max(), zlo, zhi)
    c["yaw_at_bound"] += int(((yaw == f(zlo)) | (yaw == f(zhi))).sum()) if R is N else 0
    assert bool((cmd[st] == 0).all())
    tl = R["env.cmd_time_left"][resample]
    lo_t, hi_t = cc.resampling_time_range
    assert bool(((tl >= f(lo_t)) & (tl <= f(hi_t) * (1 + 1e-6))).all()), "timer range"
    # a done env hands the sums of its command episode over and restarts them with one increment
    H.equal("finished metrics of done envs", R["env.finished_metrics"][done],
            torch.stack([S["env.metric_xy"], S["env.metric_yaw"]], 1)[done])
    H.equal("finished metrics of the others", R["env.finished_metrics"][~done], S["env.finished_metrics"][~done])
    assert bool((R["env.metric_xy"][~done] >= S["env.metric_xy"][~done]).all())
  # equal: ints, bools, copies, IEEE-exact values (mid + (2u - 1) half is rounded as written on both paths)
  for k in ("out.truncated", "env.episode_length_buf", "env._done_buf", "env.is_standing", "env.last_action",
            "env.heading_target", "env.env_origins", "env.terrain_levels", "data.ctrl", "data.qvel",
            "env.common_step_counter", "env.finished_metrics"):
    if k in T:
      H.equal(k, T[k], N[k], keep)
  H.equal("command xy", T["env.command"][:, :2], N["env.command"][:, :2], keep)
  H.equal("joint positions", T["data.qpos"][:, 7:], N["data.qpos"][:, 7:], keep)
  H.ulps("cmd_time_left", T["env.cmd_time_left"], N["env.cmd_time_left"], tol["fma_ulp"], keep)
  H.ulps("push_time_left", T["env.push_time_left"], N["env.push_time_left"], tol["fma_ulp"], keep)
  H.close("reward", T["out.reward"], N["out.reward"], keep, rowwise=False, scale=scale64)
  # yaw: path against path away from the wrap_to_pi seam, where the two may land on opposite bounds
  not_seam = keep & ((T["env.command"][:, 2] - N["env.command"][:, 2]).abs() < 0.5 * (zhi - zlo))
  c["seam"] += int((keep & ~not_seam).sum())
  H.close("yaw command", T["env.command"][:, 2], N["env.command"][:, 2], not_seam, floor=1.0, rowwise=False,
          rel=4 * tol["heading"])
  # metrics: errors of order one velocity over metric_steps
  for k in ("env.metric_xy", "env.metric_yaw"):
    H.close(k, T[k], N[k], keep, floor=4.0 / env.metric_steps, rowwise=False)
  for name, sl, amp in (("lin vel", slice(0, 3), 0.1), ("ang vel", slice(3, 6), 0.2), ("gravity", slice(6, 9), 0.05),
                        ("joint pos", slice(9, 9 + nu), 0.01), ("joint vel", slice(9 + nu, 9 + 2 * nu), 1.5)):
    H.close("obs " + name, T["out.obs"][:, sl], N["out.obs"][:, sl], keep, floor=amp)
  for R in (T, N):
    H.equal("obs command is the command", R["out.obs"][:, 9 + 3 * nu:], R["env.command"])


def _step(H, g, resample_all=False):
  env = H.env
  act = torch.rand((env.num_envs, env.nu), generator=g, device=env.device) * 2 - 1
  tmk._pre(env, act)
  env.sim.step_n(env.cfg.decimation)
  if resample_all:
    env.cmd_time_left.zero_()
  U = env._draw()
  S, T, N = H.both(act, U)
  check(H, S, T, N, act, U)
  return S, T, N


def _rollout(H, steps, seed, resample_all=False):
  """Command timers that run out during the run and first episodes of different lengths."""
  env = H.env
  g = tmk._gen(env, seed)
  env.cmd_time_left.copy_(torch.rand(env.num_envs, generator=g, device=env.device) * steps * env.step_dt)
  env.episode_length_buf.copy_(torch.randint(0, env.max_episode_length, (env.num_envs,), generator=g,
                                             device=env.device).int())
  for _ in range(steps):
    _step(H, g, resample_all)


# ---- the torch path against the reference's code -----------------------------------------------------------------
def _ref_module(monkeypatch, name, rel):
  if not refload.available():
    pytest.skip("the reference package is not installed (oracle/install_reference.py)")
  monkeypatch.syspath_prepend(str(ROOT / "tests" / "stubs"))  # prettytable stand-in (managers package)
  refload.load()
  for pkg in ("mjlab.tasks", "mjlab.tasks.velocity", "mjlab.tasks.velocity.mdp"):  # without their __init__
    if pkg not in sys.modules:
      mod = types.ModuleType(pkg)
      mod.__path__ = [str(refload.REF / Path(*pkg.split(".")))]
      monkeypatch.setitem(sys.modules, pkg, mod)
  spec = importlib.util.spec_from_file_location(name, refload.REF / "mjlab" / Path(*rel))
  mod = importlib.util.module_from_spec(spec)
  monkeypatch.setitem(sys.modules, name, mod)
  spec.loader.exec_module(mod)
  return mod


def _velocity_command_module(monkeypatch):
  return _ref_module(monkeypatch, "mjlab.tasks.velocity.mdp.velocity_command",
                     ("tasks", "velocity", "mdp", "velocity_command.py"))


def _ref_twist(vc, cc):
  return vc.UniformVelocityCommandCfg(
    asset_name="robot", resampling_time_range=tuple(cc.resampling_time_range), rel_standing_envs=cc.rel_standing_envs,
    rel_heading_envs=1.0, heading_command=True, heading_control_stiffness=cc.heading_control_stiffness,
    ranges=vc.UniformVelocityCommandCfg.Ranges(lin_vel_x=tuple(cc.lin_vel_x), lin_vel_y=tuple(cc.lin_vel_y),
                                               ang_vel_z=tuple(cc.ang_vel_z), heading=tuple(cc.heading)))


@pytest.mark.parametrize("stages", [
  ((12000, (-3.0, 3.0)),),
  ((40, (-2.0, 2.5)), (10, (-1.5, 1.5)), (25, (-0.5, 3.0))),
  ((10, (-1.5, 1.5)), (10, (-2.0, 0.0)), (0, (-0.2, 0.2)), (30, (-3.0, 3.0))),
])
def test_commands_vel_matches_reference(stages, monkeypatch):
  """The ranges in effect at counters on both sides of every stage's step, against commands_vel walking the same
  counters on one cfg (which it mutates, so stages persist)."""
  _velocity_command_module(monkeypatch)
  cur = _ref_module(monkeypatch, "mjlab.tasks.velocity.mdp.curriculums", ("tasks", "velocity", "mdp", "curriculums.py"))
  vc = sys.modules["mjlab.tasks.velocity.mdp.velocity_command"]
  H = _harness("emul", monkeypatch, robot="go1", num_envs=2, command_curriculum=stages)
  env = H.env
  twist = _ref_twist(vc, env.cfg.command)
  renv = types.SimpleNamespace(common_step_counter=0, command_manager=types.SimpleNamespace(
    get_term=lambda name: types.SimpleNamespace(cfg=twist)))
  counters = sorted({max(0, s + k) for s, _ in stages for k in (-1, 0, 1, 2)} | {0})
  for cnt in counters:
    renv.common_step_counter = cnt
    log = cur.commands_vel(renv, None, "twist", [{"step": s, "range": r} for s, r in stages])
    got = env._command_ranges(torch.tensor([cnt], dtype=torch.int32))
    want = [*twist.ranges.lin_vel_x, *twist.ranges.ang_vel_z]
    assert [float(got[0, 2]), float(got[0, 3]), float(got[1, 2]), float(got[1, 3])] == [float(np.float32(v)) for v in want], cnt
    assert float(got[0, 3]) == float(np.float32(float(log[0]))), cnt
    mid, half = float(got[0, 0]), float(got[0, 1])
    assert abs(mid - (want[0] + want[1]) / 2) <= 1e-6 and abs(half - (want[1] - want[0]) / 2) <= 1e-6
  env.close()


@pytest.mark.parametrize("robot", ["g1", "go1"])
def test_posture_matches_reference(robot, monkeypatch):
  """The pose reward with each robot's width table against the reference's posture class on the same joints."""
  er = _ref_module(monkeypatch, "mjlab.envs.mdp.rewards", ("envs", "mdp", "rewards.py"))
  from mjlab.managers.manager_term_config import RewardTermCfg

  from mjlab_b200.asset_zoo import g1, go1

  table = (g1 if robot == "g1" else go1).POSTURE_STD
  H = _harness("emul", monkeypatch, robot=robot, num_envs=16, posture_std=table)
  env = H.env
  names = [n.split("/")[-1] for n in env.model.names["joint"][1:]]
  g = tmk._gen(env, 3)
  jp = env.default_joint_pos + (torch.rand((16, env.nu), generator=g) * 2 - 1) * torch.linspace(0.0, 0.8, 16).unsqueeze(1)

  def find_joints(expr):
    assert expr == (".*",)
    return list(range(len(names))), names

  data = types.SimpleNamespace(default_joint_pos=env.default_joint_pos.expand(16, -1).clone(), joint_pos=jp)
  renv = types.SimpleNamespace(scene={"robot": types.SimpleNamespace(data=data, find_joints=find_joints)},
                               device="cpu")
  asset_cfg = types.SimpleNamespace(name="robot", joint_names=(".*",), joint_ids=slice(None))
  term = er.posture(RewardTermCfg(func=er.posture, weight=1.0, params=dict(asset_cfg=asset_cfg, std=dict(table))), renv)
  want = term(renv, std=None, asset_cfg=asset_cfg)
  got = env._posture(jp)
  assert float(got.min()) < 0.5 < float(got.max())
  torch.testing.assert_close(got, want, rtol=2e-6, atol=1e-7)
  env.close()


@pytest.mark.parametrize("standing", [0.0, 0.3])
def test_command_term_matches_reference(standing, monkeypatch):
  """One step of the command on the same state: CommandTerm.reset of the done envs, then compute (_update_metrics,
  the timer resample, _update_command) of UniformVelocityCommand, its uniform_ draws replaced by the env's U columns,
  against the torch path's _update_command."""
  vc = _velocity_command_module(monkeypatch)
  from mjlab_b200.envs.velocity_env import quat_rotate_inverse

  H = _harness("emul", monkeypatch, robot="go1", num_envs=48, command=_command(rel_standing_envs=standing,
                                                                               heading=(-3.0, 3.0)))
  env = H.env
  n, d = env.num_envs, env.sim.data
  g = tmk._gen(env, 9)
  for _ in range(2):  # some motion, so that the velocities are not zero
    tmk._pre(env, torch.rand((n, env.nu), generator=g) * 2 - 1)
    env.sim.step_n(1)
  d.qvel[:, 0:6] += torch.rand((n, 6), generator=g) * 2 - 1
  env.command.copy_(torch.rand((n, 3), generator=g) * 2 - 1)
  env.heading_target.copy_(torch.rand(n, generator=g) * 6 - 3)
  env.is_standing.copy_(torch.rand(n, generator=g) < 0.2)
  env.cmd_time_left.copy_(torch.where(torch.arange(n) % 3 == 0, 0.01, 1.0))  # every third env resamples by its timer
  env.metric_xy.copy_(torch.rand(n, generator=g)); env.metric_yaw.copy_(torch.rand(n, generator=g))
  done = torch.arange(n) % 4 == 1
  U = env._draw()
  # the reference term on the same state
  q = d.qpos[:, 3:7]
  heading = torch.atan2(2 * (q[:, 1] * q[:, 2] + q[:, 0] * q[:, 3]), 1 - 2 * (q[:, 2] ** 2 + q[:, 3] ** 2))
  data = types.SimpleNamespace(heading_w=heading, root_link_lin_vel_b=quat_rotate_inverse(q, d.qvel[:, 0:3]),
                               root_link_ang_vel_b=d.qvel[:, 3:6].clone())
  renv = types.SimpleNamespace(num_envs=n, device="cpu", step_dt=env.step_dt, scene={"robot": types.SimpleNamespace(data=data)})
  term = vc.UniformVelocityCommand(_ref_twist(vc, env.cfg.command), renv)
  term.vel_command_b.copy_(env.command); term.heading_target.copy_(env.heading_target)
  term.is_heading_env.fill_(True); term.is_standing_env.copy_(env.is_standing)
  term.time_left.copy_(env.cmd_time_left)
  term.metrics["error_vel_xy"].copy_(env.metric_xy); term.metrics["error_vel_yaw"].copy_(env.metric_yaw)
  # uniform_ draws of _resample / _resample_command, in their order: timer, x, y, z, heading, heading env, standing,
  # initial velocity
  cols = [8, 3, 4, 5, 6, None, 7, None]
  state = {"ids": None, "k": 0}
  orig_resample, orig_uniform = term._resample, torch.Tensor.uniform_

  def resample(ids):
    state["ids"], state["k"] = ids, 0
    orig_resample(ids)

  def uniform(t, lo=0.0, hi=1.0):
    col = cols[state["k"] % len(cols)]
    state["k"] += 1
    u = U[state["ids"], col].double() if col is not None else torch.full((len(state["ids"]),), 0.5, dtype=torch.float64)
    return t.copy_(lo + (hi - lo) * u)

  term._resample = resample
  monkeypatch.setattr(torch.Tensor, "uniform_", uniform)
  ids = done.nonzero().flatten()
  extras = term.reset(env_ids=ids)
  term.compute(dt=env.step_dt)
  monkeypatch.setattr(torch.Tensor, "uniform_", orig_uniform)
  before = (env.metric_xy.clone(), env.metric_yaw.clone())
  env._update_command(done, U)
  rs = done | (torch.arange(n) % 3 == 0)
  torch.testing.assert_close(env.heading_target, term.heading_target, rtol=0, atol=1e-6)
  H.equal("standing", env.is_standing, term.is_standing_env)
  torch.testing.assert_close(env.command, term.vel_command_b, rtol=0, atol=2e-6)
  torch.testing.assert_close(env.metric_xy, term.metrics["error_vel_xy"], rtol=1e-6, atol=1e-7)
  torch.testing.assert_close(env.metric_yaw, term.metrics["error_vel_yaw"], rtol=1e-6, atol=1e-7)
  torch.testing.assert_close(env.cmd_time_left[rs & ~done], term.time_left[rs & ~done], rtol=0, atol=1e-6)
  for k, m in enumerate(("error_vel_xy", "error_vel_yaw")):
    assert abs(float(env.finished_metrics[done, k].mean()) - extras[m]) <= 1e-6
    assert bool((env.finished_metrics[done, k] == before[k][done]).all())
  yaw = env.command[~env.is_standing, 2]
  assert bool(((yaw == -2.0) | (yaw == 0.5)).any()) and int(rs.sum()) > 12
  env.close()


# ---- presets against the reference's cfg classes -----------------------------------------------------------------
def test_presets_match_reference_cfgs(tmp_path):
  if not refload.available():
    pytest.skip("the reference package is not installed (oracle/install_reference.py)")
  out = tmp_path / "cfgs.json"
  here = str(Path(__file__).parent)
  cmd = [sys.executable, str(Path(__file__).with_name("ref_runner.py")), "--rootdir", here, "--confcutdir", here,
         str(Path(__file__).with_name("ref_task_cfgs.py"))]
  r = subprocess.run(cmd, capture_output=True, text=True, cwd=tmp_path, timeout=900,
                     env=dict(os.environ, B2_TASK_CFGS=str(out)))
  assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
  ref = json.loads(out.read_text())
  ve = _ve()
  from mjlab_b200.asset_zoo import g1, go1

  for name in TASKS:
    want, cfg = ref[name], ve.velocity_task_cfg(name)
    zoo = g1 if cfg.robot == "g1" else go1
    assert want["robot"] == f"{cfg.robot}_constants", name
    assert {k: pytest.approx(v) for k, v in want["action_scale"].items()} == zoo.ACTION_SCALE, name
    assert (cfg.terrain == "flat") == (want["terrain_type"] == "plane" and not want["terrain_generator"]), name
    assert (cfg.terrain == "rough") == want["terrain_generator"], name
    assert cfg.terrain_curriculum == want["terrain_curriculum"], name
    stages = [[s, list(r)] for s, r in cfg.command_curriculum] or None
    assert stages == want["command_curriculum"], name
    assert want["push"] == {"x": [-cfg.push_vel, cfg.push_vel], "y": [-cfg.push_vel, cfg.push_vel]}, name
    assert cfg.posture_std == want["posture_std"], name
    cc = cfg.command
    for k in ("lin_vel_x", "lin_vel_y", "ang_vel_z", "heading", "resampling_time_range"):
      assert list(getattr(cc, k)) == want[k], (name, k)
    assert (cc.heading_control_stiffness, cc.rel_standing_envs) == (want["heading_control_stiffness"],
                                                                    want["rel_standing_envs"]), name
    assert want["heading_command"] and want["rel_heading_envs"] == 1.0 and want["init_velocity_prob"] == 0.0, name
    assert (cfg.episode_length_s, cfg.decimation) == (want["episode_length_s"], want["decimation"]), name


def test_preset_overrides_and_defaults():
  ve = _ve()
  cfg = ve.velocity_task_cfg("Mjlab-Velocity-Flat-Unitree-Go1", num_envs=8, push_vel=0.25)
  assert (cfg.num_envs, cfg.push_vel, cfg.robot) == (8, 0.25, "go1")
  default = ve.VelocityEnvCfg()
  assert default.command == ve.VelocityCommandCfg() and default.command_curriculum == () and default.posture_std is None
  cc = default.command
  assert (cc.lin_vel_x, cc.lin_vel_y, cc.ang_vel_z, cc.heading) == ((-1.0, 1.0), (-0.5, 0.5), (-1.0, 1.0),
                                                                    (-math.pi, math.pi))
  assert (cc.heading_control_stiffness, cc.rel_standing_envs, cc.resampling_time_range) == (0.5, 0.1, (3.0, 8.0))


# ---- the fused kernel against the torch path ---------------------------------------------------------------------
@pytest.mark.parametrize("backend", BACKENDS)
def test_configured_command(backend, monkeypatch):
  """Non-default ranges, stiffness, standing share and timer over a rollout with short timers and episodes."""
  big = backend == "cuda"
  H = _harness(backend, monkeypatch, robot="go1", num_envs=512 if big else 8, decimation=4 if big else 1,
               episode_length_s=0.2 if big else 0.03, command=_command())
  _rollout(H, 12 if big else 5, seed=31)
  H.report("configured command")
  c = H.counts
  assert c["done"] > 0 and c["resample"] > c["done"] and c["yaw_at_bound"] > 0, c
  H.env.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_curriculum_stage_boundary(backend, monkeypatch):
  """Unsorted stages, the counter walking from 1 to 6 with every env resampling every step: the ranges are the cfg's
  at counter 1, stage (1)'s from counter 2 (the later-listed stage (1) keeps winning over stage (3) once both have
  passed), and stage (5)'s at counter 6 but not yet at counter 5.  A saturating heading controller shows the yaw
  clamp at the bounds in effect: ±1.5, then ±3."""
  big = backend == "cuda"
  stages = ((3, (-0.25, 0.75)), (1, (-1.5, 1.5)), (5, (-3.0, 3.0)))
  H = _harness(backend, monkeypatch, robot="go1", num_envs=256 if big else 6, decimation=4 if big else 1,
               command=_command(heading_control_stiffness=4.0, heading=(-3.0, 3.0), rel_standing_envs=0.0),
               command_curriculum=stages)
  env = H.env
  g = tmk._gen(env, 5)
  env.common_step_counter.fill_(0)
  want = {1: (-0.3, 2.1), 2: (-1.5, 1.5), 3: (-1.5, 1.5), 4: (-1.5, 1.5), 5: (-1.5, 1.5), 6: (-3.0, 3.0)}
  for counter in range(1, 7):
    S, T, N = _step(H, g, resample_all=True)  # (check holds every draw to _ranges64 of this counter)
    assert _ranges64(env, counter)[:2] == want[counter]
    assert float(env.command_log()["Curriculum/command_vel"]) == float(np.float32(want[counter][1])), counter
    yaw = N["env.command"][:, 2].abs()
    if counter >= 2:
      assert float(yaw.max()) == want[counter][1], (counter, yaw)
  H.report("curriculum stage boundary")
  env.close()


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("task", TASKS)
def test_presets_rollout(backend, task, monkeypatch):
  """Each preset (its posture table, push velocity, curricula) over a rollout with short episodes."""
  big = backend == "cuda"
  H = _harness(backend, monkeypatch, task=task, num_envs=512 if big else 4, decimation=4 if big else 1,
               episode_length_s=0.2 if big else 0.03, push_interval_s=(0.02, 0.08))
  _rollout(H, 10 if big else 4, seed=17)
  H.report(task)
  assert H.counts["done"] > 0, H.counts
  H.env.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_metrics_and_command_log(backend, monkeypatch):
  """Metric accumulation and hand-off: done envs, envs resampled by their timer, the others; each increment against
  float64 from the saved state; command_log() is the mean over the done envs, NaN when none ended."""
  H = _harness(backend, monkeypatch, robot="go1", num_envs=24, command=_command(rel_standing_envs=0.0))
  env = H.env
  mx = env.max_episode_length
  rows = [dict(episode_length_buf=mx - 1) if i % 3 == 0 else dict(cmd_time_left=0.0) if i % 3 == 1 else dict()
          for i in range(24)]
  action, U = tmk._fill(H, rows)
  g = tmk._gen(env, 4)
  d = env.sim.data
  d.qvel[:, 0:6] = torch.rand((24, 6), generator=g, device=env.device) * 2 - 1
  env.metric_xy.copy_(torch.rand(24, generator=g, device=env.device))
  env.metric_yaw.copy_(torch.rand(24, generator=g, device=env.device))
  env.finished_metrics.fill_(7.0)
  S, T, N = H.both(action, U)
  check(H, S, T, N, action, U)
  done = N["out.truncated"]
  assert int(done.sum()) == 8
  steps = env.metric_steps
  cc = env.cfg.command
  u = U.double()
  fresh = torch.stack([sum(cc.lin_vel_x) / 2 + (u[:, 3] * 2 - 1) * (cc.lin_vel_x[1] - cc.lin_vel_x[0]) / 2,
                       sum(cc.lin_vel_y) / 2 + (u[:, 4] * 2 - 1) * (cc.lin_vel_y[1] - cc.lin_vel_y[0]) / 2,
                       sum(cc.ang_vel_z) / 2 + (u[:, 5] * 2 - 1) * (cc.ang_vel_z[1] - cc.ang_vel_z[0]) / 2], 1)
  q = S["data.qpos"][:, 3:7].double()
  vb = tmk._rot_inv64(q, S["data.qvel"][:, 0:3].double())
  old = S["env.command"].double()
  inc_xy = torch.where(done, fresh[:, :2].norm(dim=1), (old[:, :2] - vb[:, :2]).norm(dim=1)) / steps
  inc_yaw = torch.where(done, fresh[:, 2].abs(), (old[:, 2] - S["data.qvel"][:, 5].double()).abs()) / steps
  for R in (T, N):
    want_xy = torch.where(done, 0.0, S["env.metric_xy"].double()) + inc_xy
    want_yaw = torch.where(done, 0.0, S["env.metric_yaw"].double()) + inc_yaw
    H.close("metric_xy vs float64", R["env.metric_xy"], want_xy, floor=4.0 / steps, rowwise=False)
    H.close("metric_yaw vs float64", R["env.metric_yaw"], want_yaw, floor=4.0 / steps, rowwise=False)
  log = env.command_log()
  assert set(log) == {"Metrics/twist/error_vel_xy", "Metrics/twist/error_vel_yaw"}
  assert log["Metrics/twist/error_vel_xy"].device == env._done_buf.device
  for k, name in enumerate(("error_vel_xy", "error_vel_yaw")):
    want = float(S["env.metric_" + name[10:]][done].double().mean())
    assert abs(float(log["Metrics/twist/" + name]) - want) <= 1e-6 * max(1.0, want)
  action, U = tmk._fill(H, [dict() for _ in range(24)])
  H.both(action, U)
  assert all(math.isnan(float(v)) for v in env.command_log().values())
  H.report("metrics")
  env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 3, 130, 4096])
def test_world_counts(n, monkeypatch):
  H = _harness("cuda", monkeypatch, task="Mjlab-Velocity-Rough-Unitree-Go1", num_envs=n, episode_length_s=0.1,
               command_curriculum=((3, (-3.0, 3.0)),))
  _rollout(H, 6, seed=n)
  H.report(f"command {n} envs")
  assert H.counts["done"] > 0, H.counts
  H.env.close()


@pytest.mark.gpu
def test_cuda_graph_across_a_stage_boundary():
  """Replays of the captured step advance the device counter (no host synchronisation in the step): the commands
  drawn before the stage's step stay in the cfg's range, those after it reach the stage's, and command_log() follows."""
  ve = _ve()
  cfg = ve.velocity_task_cfg("Mjlab-Velocity-Flat-Unitree-Go1", num_envs=1024, command_curriculum=((6, (-3.0, 3.0)),),
                             command=_command(lin_vel_x=(-1.0, 1.0), rel_standing_envs=0.0))
  env = ve.VelocityFlatEnv(cfg, device="cuda:0")
  env.enable_cuda_graph()  # (its two warm-up steps ran the counter on)
  start = int(env.common_step_counter[0])
  act = torch.zeros((env.num_envs, env.nu), device="cuda:0")
  for k in range(1, 9):
    env.cmd_time_left.zero_()  # every env resamples in this step
    env.step(act)
    counter = start + k
    assert int(env.common_step_counter[0]) == counter
    x = env.command[:, 0]
    hi = 3.0 if counter > 6 else 1.0
    assert float(x.abs().max()) <= hi and (counter <= 6 or float(x.abs().max()) > 1.0), (counter, float(x.abs().max()))
    assert float(env.command_log()["Curriculum/command_vel"]) == hi
  env.close()


# ---- configurations the env refuses ------------------------------------------------------------------------------
def test_unknown_preset():
  with pytest.raises(ValueError, match="Mjlab-Velocity-Flat-Unitree-G1, Mjlab-Velocity-Flat-Unitree-Go1, "
                                       "Mjlab-Velocity-Rough-Unitree-Go1"):
    _ve().velocity_task_cfg("Mjlab-Velocity-Rough-Unitree-G1")


@pytest.mark.parametrize("bad, match", [
  (dict(lin_vel_x=(1.0, -1.0)), "lin_vel_x"), (dict(lin_vel_y=(0.5, 0.4)), "lin_vel_y"),
  (dict(ang_vel_z=(2.0, 1.0)), "ang_vel_z"), (dict(heading=(1.0, -1.0)), "heading"),
  (dict(rel_standing_envs=-0.1), "rel_standing_envs"), (dict(rel_standing_envs=1.5), "rel_standing_envs"),
  (dict(resampling_time_range=(0.0, 8.0)), "positive"), (dict(resampling_time_range=(-1.0, 2.0)), "positive"),
  (dict(resampling_time_range=(5.0, 3.0)), "resampling_time_range"),
])
def test_invalid_command(bad, match):
  with pytest.raises(ValueError, match=match):
    _ve().VelocityCommandCfg(**bad)


@pytest.mark.parametrize("cfg, match", [
  (dict(posture_std={r".*(hip|thigh)_joint": 0.3}), "matched by 0 patterns"),
  (dict(posture_std={r".*_joint": 0.3, r".*calf.*": 0.6}), "matched by 2 patterns"),
  (dict(posture_std={r".*(hip|thigh)_joint": 0.3, r".*calf_joint": 0.6, r".*elbow.*": 0.2}), "match no joint"),
  (dict(posture_std={r".*(hip|thigh)_joint": 0.3, r".*calf_joint": 0.0}), "positive"),
  (dict(command_curriculum=((10, (1.0, -1.0)),)), "lo <= hi"),
  (dict(command_curriculum=((-1, (-1.0, 1.0)),)), "integer step"),
  (dict(command_curriculum=tuple((k, (-1.0, 1.0)) for k in range(9))), "at most 8"),
])
def test_invalid_configuration(cfg, match, monkeypatch):
  ve = _ve()
  tmk._patch_emul(monkeypatch, ve)
  with pytest.raises(ValueError, match=match):
    ve.VelocityFlatEnv(ve.VelocityEnvCfg(robot="go1", num_envs=2, **cfg), device="cpu")


def test_command_after_construction_is_checked(monkeypatch):
  """A cfg changed after it was built is checked again when the env is."""
  ve = _ve()
  tmk._patch_emul(monkeypatch, ve)
  cfg = ve.VelocityEnvCfg(robot="go1", num_envs=2)
  cfg.command.lin_vel_x = (2.0, 1.0)
  with pytest.raises(ValueError, match="lin_vel_x"):
    ve.VelocityFlatEnv(cfg, device="cpu")

"""The fused environment kernels (csrc/b2_env.cuh: b2_velenv_pre / b2_velenv_post; csrc/b2_trackenv.cuh:
b2_trackenv_post1 / bins / post2) against the torch path, on ONE post-physics state.

One env is built with ``native_mdp=True``.  After the physics sub-steps (or after a state is written by hand) every
Data field the engine lists and every env tensor the MDP touches is saved; ``_mdp_torch`` runs, its outputs and the
whole post-state are collected, the save is restored, ``_mdp_native`` runs on the very same state and the same is
collected.  Physics ran once, nothing is copied from one path to the other, and every item is compared for every
environment: there is no agreement fraction in this file.  Backends: ``emul`` (the host-emulated library, CPU suite)
and ``cuda`` (marked gpu; the only build that sees --use_fast_math).

Tolerances (``TOL``), and why:

* Integers and bools (terminated, truncated, done mask, episode_length, time_steps, terrain_levels, is_standing,
  start frames): equal.
* A termination is a threshold on a float.  Its margin is recomputed here in float64 from the saved state; the two
  paths may disagree only where |margin| < ``band``, an absolute width of 1e-6 on both backends: about 8 fp32 ulp
  of the compared quantity where that is of order 1 (the tracking thresholds, an angle near 1.2 rad), more ulps of a
  smaller one (fall_angle = 0.12 in the rollouts).  Both must equal the float64 decision outside it, and every test bounds the number of environments inside it.
  Timers are decided by one IEEE subtraction on both sides, so they have no band: ``timer - step_dt <= 0`` is
  recomputed in fp32 here and must be matched exactly.
* Copies and IEEE-exact arithmetic (reset root x, y, z, joint resets, ctrl, qvel of the velocity task, last_action,
  heading_target, env_origins, the command's x and y, log_row's flags, the unnoised critic terms that are copies or
  one subtraction): equal.  ``a * b + c`` with a drawn ``a`` (resampled timers) is one rounding on the GPU (FMA) and
  two in torch: ``fma_ulp`` = 0 on the host, 1 on the GPU.
* Everything through exp, sin / cos, acos, atan2, a rotation or a division: |a - b| <= ``rel`` * s per element, where
  s is the larger magnitude of the two values and of the row of inputs the element was rotated or summed from (a
  rotated component can cancel to zero).  The reward is also held to the float64 value of the same formula, within
  ``rel`` of the sum of the magnitudes of its terms times step_dt - relative to its own size, not an absolute 1e-4.
  ``rel``: 2e-6 on the host (IEEE fp32 both sides, libm against torch's vectorised functions; largest seen 3e-7).
  On the GPU (__expf, __sinf / __cosf, approximate division under --use_fast_math) the largest error measured on an
  NVIDIA H100 80GB HBM3 (700 W) over every case of this file was 1.6e-6 (a body-frame velocity of the policy group);
  the reward stayed below 7e-7 of its terms' size.  ``rel`` there is 4e-6.  Rows behind the masked forward (derived
  kinematics, the tracking targets and the observations built from them) carry a kinematic chain on top of the
  reset state's rounding and are held to ``kin``: 2e-5 on the host (largest seen 2e-7), 1e-4 on the GPU (3.8e-5).
* wrap_to_pi maps a heading error at the seam to +pi or -pi, and the command's yaw (clamped to +-1) flips sign there.
  Each path's yaw command is compared with clamp(0.5 wrap(heading_target - heading)) in float64 from its own
  post-state; inside ``seam`` of the seam only |yaw| = 1 is required.  Those environments are counted.
* pre: ctrl within 1 ulp (of the largest of the sum and its operands) of default + scale * action in float64 (FMA
  against mul + add).

Not covered: a robot with nu > 32 (the second trip of ``for (a = lane; a < nu; a += 32)``).  VelocityFlatEnv resolves
action scales and foot geoms from the asset zoo of its two robots, so a synthetic robot needs more than a fixture.
"""

import ctypes
import math
import sys
from collections import Counter
from pathlib import Path

import numpy as np
import pytest
import torch

from mjlab_b200.sim import native

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tools"))

BACKENDS = ["emul", pytest.param("cuda", marks=pytest.mark.gpu)]
# rel / kin / band / seam / heading / fma_ulp as described above
TOL = {
  "emul": dict(rel=2e-6, kin=2e-5, band=1e-6, seam=4e-6, heading=2e-6, fma_ulp=0),
  "cuda": dict(rel=4e-6, kin=1e-4, band=1e-6, seam=4e-6, heading=2e-6, fma_ulp=1),
}
BELOW_ONE = float(np.nextafter(np.float32(1.0), np.float32(0.0)))
VEL_ENV = ("episode_length_buf last_action command cmd_time_left heading_target is_standing push_time_left log_row "
           "_done_buf env_origins terrain_levels terrain_level_mean").split()
TRK_ENV = ("time_steps episode_length_buf last_action push_time_left body_pos_relative_w body_quat_relative_w log_row "
           "_done_buf bin_failed_count _bin_failed_cur _cdf _metrics").split()
DERIVED = ("xpos", "xquat", "link_vel_w", "link_state_b")


def _ulp(x, k=1):
  """x moved by k fp32 ulps."""
  x = np.float32(x)
  for _ in range(abs(k)):
    x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf))
  return float(x)


# ---- harness -----------------------------------------------------------------------------------------------------
class Harness:
  """One native_mdp=True env; runs both MDP halves on one saved state (module docstring)."""

  def __init__(self, env, backend, env_fields):
    self.env, self.backend, self.tol = env, backend, TOL[backend]
    self.env_fields = [f for f in env_fields if hasattr(env, f)]
    eng = env.sim._e if backend == "emul" else env.sim._engine
    self.data_fields = [f for f in eng.names(0) if getattr(env.sim.data, f)[...].numel() > 0]
    self.worst = Counter()   # largest error / bound seen per compared item
    self.counts = Counter()  # events and in-band decisions

  def snapshot(self):
    s = {"data." + f: getattr(self.env.sim.data, f)[...].clone() for f in self.data_fields}
    s.update({"env." + f: getattr(self.env, f).clone() for f in self.env_fields})
    return s

  def restore(self, snap):
    for k, v in snap.items():
      kind, f = k.split(".", 1)
      if kind == "data":
        getattr(self.env.sim.data, f)[...] = v
      else:
        getattr(self.env, f).copy_(v)

  def _collect(self, out):
    obs, reward, term, trunc, extras = out
    r = self.snapshot()
    r.update({"out.obs": obs.clone(), "out.reward": reward.clone(), "out.terminated": term.clone(),
              "out.truncated": trunc.clone()})
    r.update({"out." + k: v.clone() for k, v in extras.items()})
    return r

  def both(self, action, U):
    """(saved state, torch path's results, fused path's results); the env is left in the fused path's post-state."""
    snap = self.snapshot()
    t = self._collect(self.env._mdp_torch(action, U))
    self.restore(snap)
    n = self._collect(self.env._mdp_native(action, U))
    return snap, t, n

  # -- comparisons --
  def equal(self, name, a, b, rows=None):
    if rows is not None and a.dim() > 0 and a.shape[0] == len(rows):
      a, b = a[rows], b[rows]
    assert a.shape == b.shape and a.dtype == b.dtype, name
    bad = a != b
    assert not bool(bad.any()), (name, int(bad.sum()), a[bad][:4], b[bad][:4])

  def ulps(self, name, a, b, k, rows=None):
    """|a - b| <= k fp32 ulps of the larger (k = 0: equal)."""
    if rows is not None:
      a, b = a[rows], b[rows]
    big = torch.maximum(a.abs(), b.abs()).clamp(min=1e-30)
    lim = k * (torch.nextafter(big, torch.full_like(big, math.inf)) - big)
    bad = (a - b).abs() > lim
    assert not bool(bad.any()), (name, int(bad.sum()), a[bad][:4], b[bad][:4])

  def close(self, name, a, b, rows=None, floor=0.0, rowwise=True, rel=None, scale=None):
    """|a - b| <= rel * max(|a|, |b|, scale): scale is the row's largest magnitude (rowwise), ``floor``, and the
    per-element ``scale`` (the size of the terms an element was summed from)."""
    rel = self.tol["rel"] if rel is None else rel
    if rows is not None:
      a, b = a[rows], b[rows]
      scale = scale[rows] if scale is not None else None
    if a.numel() == 0:
      return
    a, b = a.double(), b.double()
    s = torch.maximum(a.abs(), b.abs())
    if rowwise and a.dim() > 1:
      s = s.flatten(1).amax(dim=1).view(-1, *([1] * (a.dim() - 1))).expand_as(a)
    s = s.clamp(min=max(floor, 1e-30))
    if scale is not None:
      s = torch.maximum(s, scale.double())
    err = ((a - b).abs() / s).max().item()
    self.worst[name] = max(self.worst[name], err / rel)
    assert err <= rel, (name, err, rel)

  def report(self, label):
    """Largest error seen per item as a fraction of its bound, and the counts (shown with pytest -rP)."""
    top = ", ".join(f"{k}={v:.2f}" for k, v in sorted(self.worst.items(), key=lambda kv: -kv[1])[:8])
    print(f"[{label}/{self.backend}] counts {dict(self.counts)}; largest error / bound: {top}")


def _patch_emul(monkeypatch, module):
  from test_kernel_emul import EmulSimulation

  monkeypatch.setattr(module, "Simulation", EmulSimulation)
  monkeypatch.setattr(native, "check", lambda rc: (_ for _ in ()).throw(RuntimeError("b2sim call failed")) if rc else None)


def _velocity(backend, monkeypatch, **cfg):
  import mjlab_b200.envs.velocity_env as ve

  if backend == "emul":
    _patch_emul(monkeypatch, ve)
  env = ve.VelocityFlatEnv(ve.VelocityEnvCfg(**cfg), device="cpu" if backend == "emul" else "cuda:0", native_mdp=True)
  return Harness(env, backend, VEL_ENV)


def _tracking(backend, monkeypatch, **cfg):
  import mjlab_b200.envs.tracking_env as te

  if backend == "emul":
    _patch_emul(monkeypatch, te)
  env = te.TrackingFlatEnv(te.TrackingEnvCfg(**cfg), device="cpu" if backend == "emul" else "cuda:0", native_mdp=True)
  env._native_setup()
  return Harness(env, backend, TRK_ENV)


def _gen(env, seed):
  g = torch.Generator(device=env.device)
  g.manual_seed(seed)
  return g


def _rot_inv64(q, v):
  w, u = q[..., 0:1], q[..., 1:4]
  t = 2.0 * torch.cross(u, v.expand_as(u), dim=-1)
  return v - w * t + torch.cross(u, t, dim=-1)


def _wrap64(x):
  return x - 2 * math.pi * torch.floor((x + math.pi) / (2 * math.pi))


# ---- velocity task: the checks ---------------------------------------------------------------------------------------
def _velocity_reference(env, S, action):
  """Terminations' margin and the reward of velocity_env_cfg.py:183-214 in float64 from the saved state."""
  qpos, qvel = S["data.qpos"].double(), S["data.qvel"].double()
  q = qpos[:, 3:7]
  down = torch.tensor([0.0, 0.0, -1.0], dtype=torch.float64, device=qpos.device)
  angle = torch.acos((-_rot_inv64(q, down)[:, 2]).clamp(-1.0, 1.0))
  lin_b = _rot_inv64(q, qvel[:, 0:3])
  cmd = S["env.command"].double()
  jp = qpos[:, 7:]
  terms = torch.stack([
    torch.exp(-((cmd[:, :2] - lin_b[:, :2]) ** 2).sum(1) / 0.25),
    torch.exp(-((cmd[:, 2] - qvel[:, 5]) ** 2) / 0.25),
    torch.exp(-((jp - env.default_joint_pos.double()) ** 2).mean(1) / 0.09),
    -((env.soft_lo.double() - jp).clamp(min=0) + (jp - env.soft_hi.double()).clamp(min=0)).sum(1),
    -0.1 * ((action.double() - S["env.last_action"].double()) ** 2).sum(1)], dim=1)
  return angle - float(np.float32(env.cfg.fall_angle)), terms.sum(1) * env.step_dt, terms.abs().sum(1) * env.step_dt


def check_velocity(H, S, T, N, action, U):
  """Every output and every piece of post-state of the two paths, for every env; counts go to H.counts."""
  env, tol, c = H.env, H.tol, H.counts
  nu, dt = env.nu, np.float32(env.step_dt)
  f32 = lambda x: x.cpu().numpy().astype(np.float32)
  margin, reward64, scale64 = _velocity_reference(env, S, action)
  # decisions
  inband = margin.abs() < tol["band"]
  for R in (T, N):
    H.equal("terminated vs float64", R["out.terminated"][~inband], (margin > 0)[~inband])
    H.equal("truncated", R["out.truncated"], S["env.episode_length_buf"] + 1 >= env.max_episode_length)
  keep = T["out.terminated"] == N["out.terminated"]  # (False only inside the band, by the two asserts above)
  c["in_band"] += int(inband.sum())
  c["split"] += int((~keep).sum())
  done = (T["out.terminated"] | T["out.truncated"])
  ctl, ptl = f32(S["env.cmd_time_left"]) - dt, f32(S["env.push_time_left"]) - dt
  by_timer = torch.from_numpy(ctl <= 0).to(done.device)
  push = torch.from_numpy(ptl <= 0).to(done.device)
  resample = done | by_timer
  c["terminated"] += int(T["out.terminated"].sum()); c["truncated"] += int(T["out.truncated"].sum())
  c["both"] += int((T["out.terminated"] & T["out.truncated"]).sum())
  c["push"] += int(push.sum()); c["reset_and_push"] += int((push & done).sum())
  c["resample_by_timer"] += int((by_timer & ~done).sum())
  for R in (T, N):  # each path against the fp32 timer decisions recomputed here
    H.equal("push fired", R["env.push_time_left"][keep & ~push], torch.from_numpy(ptl).to(done.device)[keep & ~push])
    assert bool((R["env.push_time_left"][push] >= env.cfg.push_interval_s[0]).all())
    H.equal("timer kept", R["env.cmd_time_left"][keep & ~resample], torch.from_numpy(ctl).to(done.device)[keep & ~resample])
    assert bool((R["env.cmd_time_left"][keep & resample] >= 3.0).all())
    H.equal("log_row reward", R["env.log_row"][:, 0], R["out.reward"])
    H.close("reward vs float64", R["out.reward"], reward64, rowwise=False, scale=scale64)
  # equal: ints, bools, copies, IEEE-exact values
  for k in ("out.truncated", "env.episode_length_buf", "env._done_buf", "env.is_standing", "env.last_action",
            "env.heading_target", "env.env_origins", "env.terrain_levels", "data.ctrl", "data.qvel"):
    if k in T:
      H.equal(k, T[k], N[k], keep)
  H.equal("log_row flags", T["env.log_row"][:, 1:], N["env.log_row"][:, 1:], keep)
  H.equal("reset root xyz", T["data.qpos"][:, 0:3], N["data.qpos"][:, 0:3], keep)
  H.equal("joint positions", T["data.qpos"][:, 7:], N["data.qpos"][:, 7:], keep)
  H.equal("root quat of envs not reset", T["data.qpos"][:, 3:7], N["data.qpos"][:, 3:7], keep & ~done)
  H.equal("command xy", T["env.command"][:, :2], N["env.command"][:, :2], keep)
  H.ulps("cmd_time_left", T["env.cmd_time_left"], N["env.cmd_time_left"], tol["fma_ulp"], keep)
  H.ulps("push_time_left", T["env.push_time_left"], N["env.push_time_left"], tol["fma_ulp"], keep)
  if "env.terrain_level_mean" in T and bool(keep.all()):
    H.ulps("terrain_level_mean", T["env.terrain_level_mean"], N["env.terrain_level_mean"], 1)
  cr, ob = "out.critic", "out.obs"
  H.equal("critic ang vel (copy)", T[cr][:, 3:6], N[cr][:, 3:6], keep)
  H.equal("critic joint pos, joint vel, last action", T[cr][:, 9:9 + 3 * nu], N[cr][:, 9:9 + 3 * nu], keep)
  H.equal("obs last action", T[ob][:, 9 + 2 * nu:9 + 3 * nu], N[ob][:, 9 + 2 * nu:9 + 3 * nu], keep)
  for R in (T, N):
    H.equal("obs command is the command", R[ob][:, 9 + 3 * nu:], R["env.command"])
    H.equal("critic command is the command", R[cr][:, 9 + 3 * nu:], R["env.command"])
    H.equal("obs last action is last_action", R[ob][:, 9 + 2 * nu:9 + 3 * nu], R["env.last_action"])
    H.equal("critic joint vel is qvel", R[cr][:, 9 + nu:9 + 2 * nu], R["data.qvel"][:, 6:])
  # through transcendental functions, rotations, noise arithmetic
  H.close("reward", T["out.reward"], N["out.reward"], keep, rowwise=False, scale=scale64)
  H.close("reset root quat", T["data.qpos"][:, 3:7], N["data.qpos"][:, 3:7], keep & done)
  for name, sl, amp in (("lin vel", slice(0, 3), 0.1), ("ang vel", slice(3, 6), 0.2), ("gravity", slice(6, 9), 0.05),
                        ("joint pos", slice(9, 9 + nu), 0.01), ("joint vel", slice(9 + nu, 9 + 2 * nu), 1.5)):
    H.close("obs " + name, T[ob][:, sl], N[ob][:, sl], keep, floor=amp)
    H.close("critic " + name, T[cr][:, sl], N[cr][:, sl], keep, floor=1e-3 if sl.start == 0 else amp)
  # The masked forward ran on (nearly) the same reset state.  One difference is by construction: the post kernel
  # writes a push into qvel before that forward and the torch path (as the reference) after it, so for an env reset
  # and pushed in one step the fused path's derived velocity rows hold the push and the torch path's hold zero.
  # Neither env reads those rows and the next physics step recomputes them from qvel, which is equal.
  for f in DERIVED:
    rows = keep & ~(done & push) if f in ("link_vel_w", "link_state_b") else keep
    H.close("data." + f, T["data." + f], N["data." + f], rows, floor=1.0, rel=tol["kin"])
  same_state = keep & (T["data.qpos"] == N["data.qpos"]).all(dim=1)
  H.equal("sensordata where the state is bit-equal", T["data.sensordata"], N["data.sensordata"], same_state)
  # the yaw command: each path against float64 from its own post-state
  for R in (T, N):
    q = R["data.qpos"][:, 3:7].double()
    heading = torch.atan2(2 * (q[:, 1] * q[:, 2] + q[:, 0] * q[:, 3]), 1 - 2 * (q[:, 2] ** 2 + q[:, 3] ** 2))
    raw = R["env.heading_target"].double() - heading
    err = _wrap64(raw)
    at_seam = (math.pi - err.abs()) < tol["seam"]
    want = torch.where(R["env.is_standing"], torch.zeros_like(err), (0.5 * err).clamp(-1.0, 1.0))
    yaw = R["env.command"][:, 2].double()
    d = torch.where(at_seam & ~R["env.is_standing"], (yaw.abs() - 1.0).abs(), (yaw - want).abs())
    H.worst["yaw command"] = max(H.worst["yaw command"], d.max().item() / tol["heading"])
    assert bool((d <= tol["heading"]).all()), ("yaw command", d.max().item())
    if R is N:
      c["seam"] += int(at_seam.sum())
  not_seam = keep & ((T["env.command"][:, 2] - N["env.command"][:, 2]).abs() < 1.0)
  H.close("yaw command, path against path", T["env.command"][:, 2], N["env.command"][:, 2], not_seam,
          floor=1.0, rowwise=False, rel=tol["heading"])
  c["standing"] += int(N["env.is_standing"].sum())
  if "env.terrain_levels" in T:
    d = N["env.terrain_levels"] - S["env.terrain_levels"]
    top = env.max_terrain_level - 1
    c["level_up"] += int((d == 1).sum()); c["level_down"] += int((d == -1).sum())
    c["level_redraw"] += int((done & (S["env.terrain_levels"] == top) & (d != -1) & (d != 0)).sum())
    c["level_redraw"] += int((done & (S["env.terrain_levels"] == top) & (N["env.terrain_levels"] == top) &
                              (_dist_from_origin(S) > env.move_up_dist)).sum())
    H.equal("origins follow levels", N["env.env_origins"],
            env.terrain_origins[N["env.terrain_levels"].long(), env.terrain_types.long()])
    assert bool((T["env.terrain_levels"][~done] == S["env.terrain_levels"][~done]).all())


def _dist_from_origin(S):
  return (S["data.qpos"][:, 0:2] - S["env.env_origins"][:, 0:2]).norm(dim=1)


def _pre(env, action):
  """b2_velenv_pre: ctrl = default + scale * action, checked to 1 ulp of the float64 value."""
  sim = env.sim
  act = action.contiguous()
  native.check(sim._lib.b2_velenv_pre(sim._h, ctypes.c_void_p(act.data_ptr()), ctypes.c_void_p(env.default_joint_pos.data_ptr()),
                                      ctypes.c_void_p(env.action_scale.data_ptr()), sim._stream()))
  prod = env.action_scale.double() * act.double()
  want = env.default_joint_pos.double() + prod
  got = sim.data.ctrl[...].double()
  # one ulp of the largest of the sum and its two operands: mul + add rounds the product too, and the sum can cancel
  big = torch.maximum(torch.maximum(want.abs(), prod.abs()), env.default_joint_pos.double().abs().expand_as(prod)).float()
  ulp = (torch.nextafter(big, torch.full_like(big, math.inf)) - big).double()
  assert bool(((got - want).abs() <= ulp).all()), (got - want).abs().max()


def _velocity_rollout(H, steps, seed, full_length=False):
  """Command timers that run out during the run; first episodes of different lengths, or (full_length) long episodes
  that all time out within the run."""
  env = H.env
  n, g, mx = env.num_envs, _gen(env, seed), env.max_episode_length
  env.cmd_time_left.copy_(torch.rand(n, generator=g, device=env.device) * steps * env.step_dt)
  ep = torch.randint(mx - steps if full_length else 0, mx, (n,), generator=g, device=env.device)
  env.episode_length_buf.copy_(ep.int())
  for _ in range(steps):
    act = torch.rand((n, env.nu), generator=g, device=env.device) * 2 - 1
    _pre(env, act)
    env.sim.step_n(env.cfg.decimation)
    U = env._draw()
    S, T, N = H.both(act, U)
    check_velocity(H, S, T, N, act, U)


# ---- velocity task: the cases ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("backend", BACKENDS)
def test_velocity_flat_rollout(backend, monkeypatch):
  """Workload B (G1 flat): random actions, physics once per env step, short episodes and push intervals."""
  big = backend == "cuda"
  H = _velocity(backend, monkeypatch, num_envs=1024 if big else 4, decimation=4 if big else 1, fall_angle=0.12,
                push_interval_s=(0.02, 0.08) if big else (0.005, 0.02), episode_length_s=0.2 if big else 0.03)
  _velocity_rollout(H, 40 if big else 6, seed=11)
  H.report("velocity flat rollout")
  c = H.counts
  assert c["truncated"] > 0 and c["push"] > 0 and c["resample_by_timer"] > 0 and c["reset_and_push"] > 0, c
  if big:
    assert c["terminated"] > 0, c
  assert c["in_band"] <= 2 and c["split"] <= c["in_band"], c
  H.env.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_velocity_rough_curriculum_rollout(backend, monkeypatch):
  """Workload E (Go1 rough, terrain curriculum): some robots are carried 5 m from their origin before an episode
  ends, some start on the last row, so levels move up, down and are redrawn."""
  big = backend == "cuda"
  n = 1024 if big else 8
  H = _velocity(backend, monkeypatch, robot="go1", terrain="rough", terrain_curriculum=True, num_envs=n,
                decimation=4 if big else 1, push_interval_s=(0.02, 0.08) if big else (0.005, 0.02),
                episode_length_s=2.0 if big else 1.0)  # (the move-down distance scales with the episode length)
  env = H.env
  top = env.max_terrain_level - 1
  env.terrain_levels[::3] = top
  env.env_origins[::3] = env.terrain_origins[top, env.terrain_types[::3].long()]
  env.sim.data.qpos[::3, 0:3] = env.env_origins[::3] + torch.tensor([0.0, 0.0, 0.4], device=env.device)
  env.sim.data.qpos[::2, 0] += 5.0
  env.sim.forward()
  _velocity_rollout(H, 40 if big else 5, seed=13, full_length=True)
  H.report("velocity rough rollout")
  c = H.counts
  assert c["level_up"] > 0 and c["level_down"] > 0 and c["level_redraw"] > 0 and c["truncated"] > 0, c
  assert c["in_band"] <= 2 and c["split"] <= c["in_band"], c
  env.close()


def _tilted(angle, yaw=0.0):
  """Root quaternion (w, x, y, z): a tilt of `angle` about x after a yaw."""
  return np.array([math.cos(yaw / 2) * math.cos(angle / 2), math.cos(yaw / 2) * math.sin(angle / 2),
                   math.sin(yaw / 2) * math.sin(angle / 2), math.sin(yaw / 2) * math.cos(angle / 2)], dtype=np.float64)


def _fill(H, rows):
  """Write hand-made environments: `rows` is a list of dicts of overrides (qpos / qvel slices, env tensors, U
  columns) applied on top of the standing default state, one env each; the rest of the batch keeps the default."""
  env = H.env
  n = env.num_envs
  assert len(rows) <= n, (len(rows), n)
  d = env.sim.data
  dev = env.device
  qpos = env.default_qpos.expand(n, -1).clone()
  qpos[:, 0:3] += env.env_origins
  d.qpos[...] = qpos
  d.qvel[...] = 0.0
  d.ctrl[...] = env.default_joint_pos
  env.episode_length_buf.fill_(3)
  env.last_action.zero_()
  env.command.copy_(torch.tensor([0.3, -0.1, 0.2], device=dev).expand(n, 3))
  env.cmd_time_left.fill_(5.0); env.push_time_left.fill_(5.0)
  env.heading_target.fill_(0.3); env.is_standing.fill_(False)
  U = torch.full((n, 16 + 9 + 2 * env.nu), 0.5, device=dev)
  U[:, 7] = 0.7
  action = torch.zeros(n, env.nu, device=dev)
  for i, row in enumerate(rows):
    for k, v in row.items():
      if k == "U":
        for col, val in v.items():
          U[i, col] = val
        continue
      v = torch.as_tensor(np.asarray(v), device=dev)
      if k == "quat":
        d.qpos[i, 3:7] = v.float()
      elif k == "xy":
        d.qpos[i, 0:2] = env.env_origins[i, 0:2] + v.float()
      elif k == "joints":
        d.qpos[i, 7:] = v.float()
      elif k == "qvel":
        d.qvel[i, :len(v)] = v.float()
      elif k == "action":
        action[i] = v.float()
      else:
        getattr(env, k)[i] = v.to(getattr(env, k).dtype)
  return action, U


def _velocity_edge_rows(env):
  fa, dt, mx = float(np.float32(env.cfg.fall_angle)), float(np.float32(env.step_dt)), env.max_episode_length
  rows = []
  # fall angle: around the threshold in steps of an fp32 ulp of the cosine, far above, upside down, upright
  for k in (-64, -8, -2, -1, 0, 1, 2, 8, 64):
    rows.append(dict(quat=_tilted(fa + k * 1.2e-7)))
  for yaw in (0.7, -2.9):
    rows += [dict(quat=_tilted(fa - 1e-3, yaw)), dict(quat=_tilted(fa + 1e-3, yaw))]
  rows += [dict(quat=_tilted(math.pi)), dict(quat=_tilted(0.0)), dict(quat=[0.0, 1.0, 0.0, 0.0])]
  # episode length
  rows += [dict(episode_length_buf=mx - 3), dict(episode_length_buf=mx - 2), dict(episode_length_buf=mx - 1),
           dict(episode_length_buf=mx), dict(episode_length_buf=mx - 1, quat=_tilted(fa + 0.2))]
  # timers: exactly step_dt (the difference is 0: fires), one ulp either side, negative
  for t in (dt, _ulp(dt, 1), _ulp(dt, -1), -0.5, 2 * dt):
    rows += [dict(cmd_time_left=t), dict(push_time_left=t), dict(cmd_time_left=t, push_time_left=t)]
  # reset and push in one step (the pushed velocity survives the qvel zeroing); reset and timer together
  rows += [dict(episode_length_buf=mx - 1, push_time_left=dt, qvel=[0.4, -0.3, 0.1, 0.2, 0.1, -0.3], U={9: 0.9, 10: 0.1}),
           dict(quat=_tilted(fa + 0.3), push_time_left=-1.0, qvel=[1.0, 1.0, 1.0], U={9: 0.0, 10: BELOW_ONE, 11: 0.0}),
           dict(episode_length_buf=mx - 1, cmd_time_left=dt), dict(push_time_left=dt, U={11: BELOW_ONE})]
  # standing <-> moving through a resample; the standing draw at 0.1 exactly and one ulp either side
  for u7 in (0.0, _ulp(0.1, -1), float(np.float32(0.1)), _ulp(0.1, 1), BELOW_ONE):
    rows += [dict(cmd_time_left=dt, is_standing=False, U={7: u7}), dict(cmd_time_left=dt, is_standing=True, U={7: u7}),
             dict(is_standing=True, U={7: u7})]
  # uniforms at 0 and at the largest float below 1
  for u in (0.0, BELOW_ONE):
    rows += [dict(episode_length_buf=mx - 1, U={c: u for c in range(0, 13)}),
             dict(episode_length_buf=mx - 1, U={2: u}), dict(cmd_time_left=dt, U={c: u for c in (3, 4, 5, 6, 8)}),
             dict(U={c: u for c in range(16, 16 + 9 + 2 * env.nu)})]
  # heading error swept across +-pi (robot yaw 0.4 -> heading 0.4), heading_target at +-pi
  for k in (-40, -3, -1, 0, 1, 3, 40):
    for sgn in (1.0, -1.0):
      rows.append(dict(quat=_tilted(0.0, 0.4), heading_target=float(np.float32(0.4 + sgn * math.pi + k * 2.4e-7))))
  for ht in (math.pi, -math.pi, float(np.float32(math.pi)), -float(np.float32(math.pi))):
    rows += [dict(heading_target=ht), dict(quat=_tilted(0.0, 3.1), heading_target=ht),
             dict(quat=_tilted(0.0, math.pi), heading_target=ht)]
  rows += [dict(cmd_time_left=dt, U={6: 0.0}), dict(cmd_time_left=dt, U={6: BELOW_ONE}), dict(cmd_time_left=dt, U={6: 0.5})]
  # joints below, on and above the soft limits (limit reward), and a reset from there
  lo, hi, dflt = env.soft_lo.cpu().numpy(), env.soft_hi.cpu().numpy(), env.default_joint_pos.cpu().numpy()
  for j in sorted({0, 1, env.nu // 2, env.nu - 1}):
    for v in (lo[j] - 0.05, lo[j], hi[j], hi[j] + 0.05, _ulp(lo[j], -1), _ulp(hi[j], 1)):
      jp = dflt.copy()
      jp[j] = v
      rows += [dict(joints=jp), dict(joints=jp, episode_length_buf=mx - 1)]
  return rows


@pytest.mark.parametrize("backend", BACKENDS)
def test_velocity_decision_edges(backend, monkeypatch):
  """Hand-written states, one environment per edge value (the velocity kernels read only qpos, qvel and env tensors)."""
  # the default state is clamped into the soft limits first, as a reset does, so that the limit term is 0 by default
  H = _velocity(backend, monkeypatch, robot="go1", num_envs=176)
  env = H.env
  env.default_qpos[7:] = torch.minimum(torch.maximum(env.default_qpos[7:], env.soft_lo), env.soft_hi)
  rows = _velocity_edge_rows(env)
  action, U = _fill(H, rows)
  action[1::2] = 0.25
  S, T, N = H.both(action, U)
  check_velocity(H, S, T, N, action, U)
  H.report("velocity edges")
  c = H.counts
  assert c["terminated"] >= 8 and c["truncated"] >= 10 and c["both"] >= 1 and c["push"] >= 8, c
  assert c["resample_by_timer"] >= 10 and c["reset_and_push"] >= 2 and c["seam"] >= 2 and c["standing"] >= 4, c
  assert c["in_band"] <= 7 and c["split"] <= c["in_band"], c  # (the seven tilts written within 8 ulp of the angle)
  # the edges, by name, on the fused path's results
  dt = float(np.float32(env.step_dt))
  for i, r in enumerate(rows):
    done = bool(N["out.terminated"][i] | N["out.truncated"][i])
    if set(r) == {"cmd_time_left"}:
      assert (float(N["env.cmd_time_left"][i]) >= 3.0) == (np.float32(r["cmd_time_left"]) - np.float32(dt) <= 0), r
    if set(r) == {"push_time_left"}:
      assert (float(N["env.push_time_left"][i]) >= 1.0) == (np.float32(r["push_time_left"]) - np.float32(dt) <= 0), r
    if "qvel" in r and done:  # reset and push together: the push is in qvel and in both observation groups
      assert float(N["data.qvel"][i, 0:2].abs().min()) > 0.1 and float(N["data.qvel"][i, 2:].abs().max()) == 0.0
      assert float(N["out.critic"][i, 0:2].abs().max()) > 0.1 and float(T["out.critic"][i, 0:2].abs().max()) > 0.1
      assert float((N["out.obs"][i, 0:3] - N["out.critic"][i, 0:3]).abs().max()) <= 0.1 + 1e-6
    if set(r) == {"cmd_time_left", "is_standing", "U"}:
      assert bool(N["env.is_standing"][i]) == (np.float32(r["U"][7]) <= np.float32(0.1)), r
    if set(r) == {"is_standing", "U"}:
      assert bool(N["env.is_standing"][i]), r  # no resample: the state stands
  env.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_velocity_reset_clamps_joints(backend, monkeypatch):
  """A default pose with joints below soft_lo and above soft_hi: the reset writes them clamped onto the limits."""
  H = _velocity(backend, monkeypatch, robot="go1", num_envs=6)
  env = H.env
  env.default_qpos[7] = env.soft_lo[0] - 0.1
  env.default_qpos[8] = env.soft_hi[1] + 0.1
  env.default_qpos[7 + env.nu - 1] = env.soft_hi[env.nu - 1] + 0.05
  rows = [dict(episode_length_buf=env.max_episode_length - 1) for _ in range(4)] + [dict(), dict()]
  action, U = _fill(H, rows)
  S, T, N = H.both(action, U)
  check_velocity(H, S, T, N, action, U)
  for R in (T, N):
    jp = R["data.qpos"][:, 7:]
    assert bool(R["out.truncated"][:4].all()) and not bool(R["out.truncated"][4:].any())
    H.equal("clamped onto soft_lo", jp[:4, 0], env.soft_lo[0].expand(4))
    H.equal("clamped onto soft_hi", jp[:4, 1], env.soft_hi[1].expand(4))
    H.equal("clamped onto soft_hi, last joint", jp[:4, -1], env.soft_hi[-1].expand(4))
    H.equal("not reset: as written", jp[4:], S["data.qpos"][4:, 7:])
    assert float(jp[4, 0]) < float(env.soft_lo[0]) and float(jp[4, 1]) > float(env.soft_hi[1])
  env.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_velocity_curriculum_edges(backend, monkeypatch):
  """Distance walked at the move-up bound and either side, at the move-down bound, level 0 moving down, last row
  moving up (redraw from U[12] at 0, mid, just below 1: the last clamps to rows - 1)."""
  H = _velocity(backend, monkeypatch, robot="go1", terrain="rough", terrain_curriculum=True, num_envs=40)
  env = H.env
  rows_, mx, up = env.max_terrain_level, env.max_episode_length, env.move_up_dist
  rows = []
  for lvl in (0, 3, rows_ - 1):
    for dist in (up, _ulp(up, 1), _ulp(up, -1), up + 1.0):
      for u in ((0.0, 0.5, BELOW_ONE) if lvl == rows_ - 1 and dist > up else (0.5,)):
        rows.append(dict(terrain_levels=lvl, xy=[dist, 0.0], U={12: u}))
    # the move-down bound: |command| * episode_length_s / 2 = 1 m at |command| = 0.1
    for dist in (1.0, _ulp(1.0, -1), _ulp(1.0, 1), 0.2):
      rows.append(dict(terrain_levels=lvl, xy=[0.0, dist], command=[0.1, 0.0, 0.0]))
  for r in rows:
    r["episode_length_buf"] = mx - 1
  rows.append(dict(terrain_levels=2, xy=[6.0, 0.0]))  # not done: stays
  for i, r in enumerate(rows):  # the origin of the row the env is on
    env.terrain_levels[i] = r["terrain_levels"]
  env.env_origins.copy_(env.terrain_origins[env.terrain_levels.long(), env.terrain_types.long()])
  assert env.cfg.episode_length_s == 20.0
  action, U = _fill(H, rows)
  S, T, N = H.both(action, U)
  check_velocity(H, S, T, N, action, U)
  H.report("velocity curriculum edges")
  c = H.counts
  assert c["level_up"] >= 2 and c["level_down"] >= 2 and c["level_redraw"] >= 2, c
  # each row against the rule in fp32 from the saved state (an ulp written next to a far origin may round away)
  lv0, lv = S["env.terrain_levels"], N["env.terrain_levels"]
  for i, r in enumerate(rows[:-1]):
    dx, dy = np.float32(S["data.qpos"][i, 0].item()) - np.float32(S["env.env_origins"][i, 0].item()), \
        np.float32(S["data.qpos"][i, 1].item()) - np.float32(S["env.env_origins"][i, 1].item())
    dist = np.sqrt(dx * dx + dy * dy, dtype=np.float32)
    cmd = np.float32(abs(float(S["env.command"][i, 0])))
    goes_up = dist > np.float32(up)
    goes_down = (not goes_up) and dist < cmd * np.float32(env.cfg.episode_length_s) * np.float32(0.5)
    want = int(lv0[i]) + int(goes_up) - int(goes_down)
    if want >= rows_:
      want = min(int(math.floor(np.float32(r["U"][12]) * np.float32(rows_))), rows_ - 1)
    assert int(lv[i]) == max(want, 0), (i, r, dist, int(lv[i]), want)
  assert int(lv[len(rows) - 1]) == 2
  env.close()


def _velocity_isolated(H, term, g):
  """A batch in which only the inputs of one reward term vary; the others sit where their term is constant
  (pose error 0, inside the limits, action = last action, velocity = command)."""
  env = H.env
  n, nu, dev = env.num_envs, env.nu, env.device
  action, U = _fill(H, [])
  r = lambda *s: torch.rand(s, generator=g, device=dev) * 2 - 1
  d = env.sim.data
  if term == "lin":
    d.qvel[:, 0:2] = r(n, 2) * 1.5
  elif term == "ang":
    d.qvel[:, 5] = r(n) * 1.5
  elif term == "pose":
    span = torch.minimum(env.default_joint_pos - env.soft_lo, env.soft_hi - env.default_joint_pos).clamp(min=0)
    d.qpos[:, 7:] = env.default_joint_pos + r(n, nu) * span
  elif term == "limits":
    j = torch.arange(n, device=dev) % nu
    jp = d.qpos[:, 7:].clone()
    jp[torch.arange(n, device=dev), j] = torch.where(torch.arange(n, device=dev) % 2 == 0, env.soft_lo[j] - 0.01 - 0.1 * r(n).abs(),
                                                     env.soft_hi[j] + 0.01 + 0.1 * r(n).abs())
    d.qpos[:, 7:] = jp
  elif term == "rate":
    action = r(n, nu)
    env.last_action.copy_(r(n, nu))
  return action, U


@pytest.mark.parametrize("backend", BACKENDS)
def test_velocity_reward_terms_in_isolation(backend, monkeypatch):
  H = _velocity(backend, monkeypatch, robot="go1", num_envs=48)
  env = H.env
  env.default_qpos[7:] = torch.minimum(torch.maximum(env.default_qpos[7:], env.soft_lo), env.soft_hi)
  g = _gen(env, 3)
  for term in ("lin", "ang", "pose", "limits", "rate"):
    action, U = _velocity_isolated(H, term, g)
    S, T, N = H.both(action, U)
    check_velocity(H, S, T, N, action, U)
    r = N["out.reward"]
    assert float(r.max() - r.min()) > 1e-3 * env.step_dt, term  # the term did vary
  H.report("velocity reward terms")
  env.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_velocity_observation_noise_columns(backend, monkeypatch):
  """Each noise column alone at 0, 0.5 and just below 1 while the others are at 0.5 (no noise): the policy group
  differs from the critic group in exactly that element, by exactly the amplitude of its term."""
  H = _velocity(backend, monkeypatch, robot="go1", num_envs=3 * 33)
  env = H.env
  nu = env.nu
  action, U = _fill(H, [])
  env.sim.data.qvel[...] = torch.rand(env.sim.data.qvel[...].shape, generator=_gen(env, 5), device=env.device) - 0.5
  amp = [0.1] * 3 + [0.2] * 3 + [0.05] * 3 + [0.01] * nu + [1.5] * nu
  vals = (0.0, 0.5, BELOW_ONE)
  for c in range(9 + 2 * nu):
    for k, v in enumerate(vals):
      U[3 * c + k, 16 + c] = v
  S, T, N = H.both(action, U)
  check_velocity(H, S, T, N, action, U)
  for R in (T, N):
    diff = (R["out.obs"] - R["out.critic"]).double()
    for c in range(9 + 2 * nu):
      for k, v in enumerate(vals):
        row = diff[3 * c + k]
        want = (2.0 * np.float32(v) - 1.0) * amp[c]
        assert abs(float(row[c]) - want) <= 1e-6 * max(1.0, float(R["out.critic"][3 * c + k, c].abs())), (c, v)
        row = row.clone()
        row[c] = 0.0
        assert float(row.abs().max()) == 0.0, (c, v)
  H.report("velocity noise columns")
  env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 3, 5, 130, 4096])
def test_velocity_world_counts(n, monkeypatch):
  """Partial CTAs (four warps, one env each), a single warp, and 4096 envs once (workload B)."""
  H = _velocity("cuda", monkeypatch, num_envs=n, fall_angle=0.12, push_interval_s=(0.02, 0.08), episode_length_s=0.1)
  _velocity_rollout(H, 8, seed=n)
  H.report(f"velocity {n} envs")
  assert H.counts["truncated"] > 0 and H.counts["in_band"] <= 2, H.counts
  H.env.close()


# ---- tracking task: the checks ---------------------------------------------------------------------------------------
def _tracking_reference(env, S, action):
  """The three termination margins and the reward of tracking_env_cfg.py:200-278 in float64 from the saved state."""
  import mjlab_b200.envs.tracking_env as te
  from mjlab_b200.entity_data import quat_apply_inverse

  dd = lambda x: x.double()
  bid = env.robot.indexing.body_ids[env.body_idx].long()
  pos, quat = dd(S["data.xpos"][:, bid]), dd(S["data.xquat"][:, bid])
  vel = dd(S["data.link_vel_w"][:, bid])
  lin, ang = vel[..., 0:3], vel[..., 3:6]
  ts = S["env.time_steps"]
  clip = {k: dd(v[ts]) for k, v in env.motion.items()}
  a_pos = clip["body_pos_w"][:, env.anchor] + dd(env.env_origins)
  a_quat = clip["body_quat_w"][:, env.anchor]
  r_pos, r_quat = pos[:, env.anchor], quat[:, env.anchor]
  g = torch.tensor([0.0, 0.0, -1.0], dtype=torch.float64, device=pos.device).expand(len(ts), 3)
  rel_p, rel_q = dd(S["env.body_pos_relative_w"]), dd(S["env.body_quat_relative_w"])
  margins = torch.cat([
    ((a_pos[:, 2] - r_pos[:, 2]).abs() - 0.25)[:, None],
    ((quat_apply_inverse(a_quat, g)[:, 2] - quat_apply_inverse(r_quat, g)[:, 2]).abs() - 0.8)[:, None],
    (rel_p[:, env.ee_idx, 2] - pos[:, env.ee_idx, 2]).abs() - 0.25], dim=1)
  qe = te.quat_error_magnitude
  jp, lim = dd(S["data.qpos"][:, 7:]), dd(env.robot.soft_joint_pos_limits)
  terms = torch.stack([
    0.5 * torch.exp(-((a_pos - r_pos) ** 2).sum(-1) / 0.3**2),
    0.5 * torch.exp(-qe(a_quat, r_quat) ** 2 / 0.4**2),
    torch.exp(-((rel_p - pos) ** 2).sum(-1).mean(-1) / 0.3**2),
    torch.exp(-(qe(rel_q, quat) ** 2).mean(-1) / 0.4**2),
    torch.exp(-((clip["body_lin_vel_w"] - lin) ** 2).sum(-1).mean(-1) / 1.0**2),
    torch.exp(-((clip["body_ang_vel_w"] - ang) ** 2).sum(-1).mean(-1) / 3.14**2),
    -0.1 * ((dd(action) - dd(S["env.last_action"])) ** 2).sum(1),
    -10.0 * ((lim[..., 0] - jp).clamp(min=0) + (jp - lim[..., 1]).clamp(min=0)).sum(1),
    -10.0 * dd(S["data.sensordata"][:, env.self_collision_adr[0]])], dim=1)
  return margins, terms.sum(1) * env.step_dt, terms.abs().sum(1) * env.step_dt


def _drawn_frames(env, S, u):
  """Start frames of the draws u under the distribution the step drew from (the saved CDF)."""
  if "env._cdf" not in S:
    return env._start_frames(u)
  now = env._cdf.clone()
  env._cdf.copy_(S["env._cdf"])
  frames = env._start_frames(u.contiguous())
  env._cdf.copy_(now)
  return frames


def check_tracking(H, S, T, N, action, U):
  env, tol, c = H.env, H.tol, H.counts
  nu, dt = env.nu, np.float32(env.step_dt)
  Sn = 13 + nu
  margins, reward64, scale64 = _tracking_reference(env, S, action)
  near = margins.abs() < tol["band"]
  # in the band only if no other threshold decides: a margin clearly above 0 terminates whatever the near one does
  inband = near.any(dim=1) & ~((margins > 0) & ~near).any(dim=1)
  term64 = (margins > 0).any(dim=1)
  trunc = S["env.episode_length_buf"] + 1 >= env.max_episode_length
  for R in (T, N):
    H.equal("terminated vs float64", R["out.terminated"][~inband], term64[~inband])
    H.equal("truncated", R["out.truncated"], trunc)
    H.close("reward vs float64", R["out.reward"], reward64, rowwise=False, scale=scale64)
    H.equal("log_row reward", R["env.log_row"][:, 0], R["out.reward"])
  keep = T["out.terminated"] == N["out.terminated"]
  c["in_band"] += int(inband.sum()); c["split"] += int((~keep).sum())
  term = N["out.terminated"]
  done = term | trunc
  ended = N["env._done_buf"] & ~done
  ptl = S["env.push_time_left"].cpu().numpy().astype(np.float32) - dt
  push = torch.from_numpy(ptl <= 0).to(done.device)
  c["terminated"] += int(term.sum()); c["truncated"] += int(trunc.sum()); c["push"] += int(push.sum())
  c["clip_restart"] += int(ended.sum()); c["both"] += int((term & trunc).sum())
  for k in range(margins.shape[1]):
    c[f"term{k}"] += int((margins[:, k] > 0).sum())
  for R in (T, N):
    H.equal("push fired", R["env.push_time_left"][~push], torch.from_numpy(ptl).to(done.device)[~push])
    assert bool((R["env.push_time_left"][push] >= env.cfg.push_interval_s[0]).all())
    assert bool(((R["env.time_steps"] >= 0) & (R["env.time_steps"] < env.T)).all())
  # the clip's time step: a finished env starts on the frame of U[:, 0] and moves on one frame; an env then at the
  # clip's end (a reset onto the last frame too: two resamples in one step) restarts on the frame of U[:, S]
  first = _drawn_frames(env, S, U[:, 0])
  want_ts = torch.where(done, first, S["env.time_steps"]) + 1
  restart = want_ts >= env.T
  want_ts = torch.where(restart, _drawn_frames(env, S, U[:, Sn]), want_ts)
  c["double_resample"] += int((done & restart).sum())
  H.equal("time_steps vs the draws", N["env.time_steps"], want_ts)
  H.equal("done mask vs the draws", N["env._done_buf"], done | restart)
  # ... and its state comes from that block of U: the joints are the frame's plus the block's joint noise
  cols = torch.where(restart, Sn, 0)[:, None] + 13 + torch.arange(nu, device=U.device)[None, :]
  lo, hi = env.cfg.joint_position_range
  lim = env.robot.soft_joint_pos_limits.double()
  frame = torch.where(restart, want_ts, (want_ts - 1).clamp(min=0))  # (a reset writes its frame, then the clip steps)
  want_jp = env.motion["joint_pos"][frame].double() + U.gather(1, cols).double() * (hi - lo) + lo
  want_jp = torch.minimum(torch.maximum(want_jp, lim[..., 0]), lim[..., 1])
  for R, rows in ((T, keep & (done | restart)), (N, done | restart)):
    H.close("reset joints vs their block of U", R["data.qpos"][:, 7:], want_jp, rows, floor=1.0)
  same = bool(keep.all())
  for k in ("out.truncated", "env._done_buf", "env.episode_length_buf", "env.time_steps", "env.last_action", "data.ctrl",
            "data.xfrc_applied"):
    H.equal(k, T[k], N[k], keep)
  H.equal("log_row flags", T["env.log_row"][:, 1:], N["env.log_row"][:, 1:], keep)
  H.ulps("push_time_left", T["env.push_time_left"], N["env.push_time_left"], tol["fma_ulp"], keep)
  not_reset = keep & ~N["env._done_buf"]
  H.equal("joint state of envs not reset", T["data.qpos"][:, 7:], N["data.qpos"][:, 7:], not_reset)
  H.equal("qpos of envs not reset", T["data.qpos"], N["data.qpos"], not_reset)
  H.equal("joint velocities (clip copies or untouched)", T["data.qvel"][:, 6:], N["data.qvel"][:, 6:], keep)
  if same and "env._cdf" in T:
    for k in ("env.bin_failed_count", "env._bin_failed_cur", "env._cdf", "env._metrics"):
      H.close(k, T[k], N[k], floor=1.0, rowwise=False, rel=1e-6)
    H.equal("failure counts cleared", N["env._bin_failed_cur"], torch.zeros_like(N["env._bin_failed_cur"]))
    for k in ("sampling_entropy", "sampling_top1_prob", "sampling_top1_bin"):
      H.close(k, T["out." + k], N["out." + k], floor=1.0, rowwise=False, rel=1e-6)
  ob, cr = "out.obs", "out.critic"
  nb = len(env.body_idx)
  ct = 2 * nu + 9 + 9 * nb
  H.equal("obs command (clip copies)", T[ob][:, 0:2 * nu], N[ob][:, 0:2 * nu], keep)
  H.equal("critic command (clip copies)", T[cr][:, 0:2 * nu], N[cr][:, 0:2 * nu], keep)
  H.equal("obs last action", T[ob][:, 4 * nu + 15:], N[ob][:, 4 * nu + 15:], keep)
  H.equal("critic last action", T[cr][:, ct + 6 + 2 * nu:], N[cr][:, ct + 6 + 2 * nu:], keep)
  for R in (T, N):
    H.equal("obs last action is last_action", R[ob][:, 4 * nu + 15:], R["env.last_action"])
    H.equal("critic joint vel is qvel", R[cr][:, ct + 6 + nu:ct + 6 + 2 * nu], R["data.qvel"][:, 6:])
    H.equal("obs command is the clip frame", R[ob][:, 0:nu], env.motion["joint_pos"][R["env.time_steps"]])
  H.close("reward", T["out.reward"], N["out.reward"], keep, rowwise=False, scale=scale64)
  H.close("qpos root", T["data.qpos"][:, 0:7], N["data.qpos"][:, 0:7], keep, floor=1.0)
  H.close("qpos joints", T["data.qpos"][:, 7:], N["data.qpos"][:, 7:], keep, floor=1.0)
  H.close("qvel root", T["data.qvel"][:, 0:6], N["data.qvel"][:, 0:6], keep, floor=0.1)
  loose = tol["kin"]  # behind the masked forward: a kinematic chain on top of the reset state's rounding
  for f in DERIVED:
    H.close("data." + f, T["data." + f], N["data." + f], keep, floor=1.0, rel=loose)
  H.close("body_pos_relative_w", T["env.body_pos_relative_w"], N["env.body_pos_relative_w"], keep, floor=1.0, rel=loose)
  H.close("body_quat_relative_w", T["env.body_quat_relative_w"], N["env.body_quat_relative_w"], keep, floor=1.0, rel=loose)
  groups = [("anchor pos", 2 * nu, 3, 0.25), ("anchor ori", 2 * nu + 3, 6, 1.0), ("base lin", 2 * nu + 9, 3, 0.5),
            ("base ang", 2 * nu + 12, 3, 0.2), ("joint pos", 2 * nu + 15, nu, 0.01), ("joint vel", 3 * nu + 15, nu, 0.5)]
  for name, a, w, amp in groups:
    H.close("obs " + name, T[ob][:, a:a + w], N[ob][:, a:a + w], keep, floor=amp, rel=loose)
  for name, a, w in (("anchor", 2 * nu, 9), ("body pos", 2 * nu + 9, 3 * nb), ("body ori", 2 * nu + 9 + 3 * nb, 6 * nb),
                     ("base vel", ct, 6), ("joint pos", ct + 6, nu), ("joint vel", ct + 6 + nu, nu)):
    H.close("critic " + name, T[cr][:, a:a + w], N[cr][:, a:a + w], keep, floor=0.1, rel=loose)
  same_state = keep & (T["data.qpos"] == N["data.qpos"]).all(dim=1) & (T["data.qvel"] == N["data.qvel"]).all(dim=1)
  H.equal("sensordata where the state is bit-equal", T["data.sensordata"], N["data.sensordata"], same_state)
  return dict(done=done, ended=ended, term=term, margins=margins)


def _tracking_rollout(H, steps, seed, drop_every=3):
  env = H.env
  n, g = env.num_envs, _gen(env, seed)
  env.episode_length_buf.copy_(torch.randint(0, env.max_episode_length, (n,), generator=g, device=env.device).int())
  for k in range(steps):
    act = torch.rand((n, env.nu), generator=g, device=env.device) * 2 - 1
    if k % drop_every == 1:  # falls: some anchors drop below the clip's by more than 0.25 m
      env.sim.data.qpos[k % 4::4, 2] -= 0.4
    if k % drop_every == 2:
      env.time_steps[(k + 1) % 4::4] = env.T - 1
    _pre(env, act)
    env.sim.step_n(env.cfg.decimation)
    U = env._rand(n, 48 + 4 * env.nu)
    U[::5, 0] = BELOW_ONE  # the largest draw: with the adaptive sampler it can land on the clip's last frame
    S, T, N = H.both(act, U)
    check_tracking(H, S, T, N, act, U)


_CLIPS = {}


def _make_clip(backend, tmp_path, frames):
  """A generated motion file, made once per backend and length."""
  if (backend, frames) not in _CLIPS:
    _CLIPS[backend, frames] = _generate_clip(backend, tmp_path, frames)
  return _CLIPS[backend, frames]


def _generate_clip(backend, tmp_path, frames):
  from make_motion_clip import make_clip

  if backend == "cuda":
    return make_clip(tmp_path / "clip.npz", frames=frames, device="cuda:0")
  from test_kernel_emul import EmulSimulation

  from mjlab_b200.asset_zoo import load_compiled
  from mjlab_b200.sim import SimulationCfg

  m = load_compiled("g1_tracking_flat")
  sim = EmulSimulation(frames, SimulationCfg(), m, "cpu")
  path = make_clip(tmp_path / "clip.npz", frames=frames, device="cpu", sim=sim, model=m)
  sim.close()
  return path


@pytest.mark.parametrize("clip", ["synthetic", "motion_file"])
@pytest.mark.parametrize("backend", BACKENDS)
def test_tracking_rollout(backend, clip, monkeypatch, tmp_path):
  """Workload C (G1 tracking): the synthetic static clip, and a motion file with the adaptive start-frame sampler."""
  big = backend == "cuda"
  cfg = dict(num_envs=1024 if big else 4, episode_length_s=0.3 if big else 0.06,
             push_interval_s=(0.05, 0.15) if big else (0.02, 0.06))
  if clip == "synthetic":
    cfg["clip_frames"] = 30 if big else 6
  else:
    cfg.update(motion_file=_make_clip(backend, tmp_path, 960 if big else 120), adaptive_kernel_size=3, adaptive_alpha=0.2)
  H = _tracking(backend, monkeypatch, **cfg)
  _tracking_rollout(H, 40 if big else 6, seed=17)
  H.report(f"tracking rollout, {clip}")
  c = H.counts
  assert c["terminated"] > 0 and c["truncated"] > 0 and c["push"] > 0 and c["clip_restart"] > 0, c
  assert c["in_band"] <= 2 and c["split"] <= c["in_band"], c
  if clip == "motion_file":
    assert float(H.env.bin_failed_count.sum()) > 0
    assert c["double_resample"] > 0 or not big, c  # (a handful of envs on the host: the edge test has the case)
  H.env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 3, 5, 130])
def test_tracking_world_counts(n, monkeypatch):
  H = _tracking("cuda", monkeypatch, num_envs=n, episode_length_s=0.1, push_interval_s=(0.02, 0.08), clip_frames=12)
  _tracking_rollout(H, 8, seed=n)
  H.report(f"tracking {n} envs")
  assert H.counts["truncated"] > 0 and H.counts["in_band"] <= 2, H.counts
  H.env.close()


def _tracking_base(H):
  """Every env on its clip frame, at rest: the derived rows both paths read are the clip's own (all errors 0)."""
  env = H.env
  n, dev = env.num_envs, env.device
  U = torch.full((n, 48 + 4 * env.nu), 0.5, device=dev)
  all_ = torch.ones(n, dtype=torch.bool, device=dev)
  env.time_steps.fill_(1)
  env._resample(all_, ~all_, U[:, 0:13 + env.nu])  # (all draws 0.5: no RSI noise; the frame stays)
  env.sim.forward()
  env._update_command()
  env.episode_length_buf.fill_(2)
  env.last_action.zero_()
  env.push_time_left.fill_(5.0)
  return torch.zeros(n, env.nu, device=dev), U


@pytest.mark.parametrize("backend", BACKENDS)
def test_tracking_decision_edges(backend, monkeypatch, tmp_path):
  """Thresholds written into the derived rows the kernels read: anchor height 0.25 +- d, gravity projection 0.8 +- d,
  each end effector alone at 0.25 +- d, time_steps at T-2 / T-1, an episode ending on the clip's last frame, the
  self-collision count, an episode end whose reset lands on the last frame (two resamples in one step, the second from
  the second block of U), failures in the first and last bin and either side of the bin boundaries, start-frame draws
  at 0 and just below 1."""
  H = _tracking(backend, monkeypatch, num_envs=64, motion_file=_make_clip(backend, tmp_path, 120),
                adaptive_kernel_size=2, adaptive_alpha=0.5, episode_length_s=1.0)
  env = H.env
  action, U = _tracking_base(H)
  d, dev = env.sim.data, env.device
  bid = env.robot.indexing.body_ids[env.body_idx].long()
  anchor, T_, mx, Sn = int(bid[env.anchor]), env.T, env.max_episode_length, 13 + env.nu
  # a failure history under which the largest draw lands on the clip's last frame (cdf[-1] is 1 and the division
  # inside the last bin rounds up to it): a reset with that draw runs off the clip in the same step
  g = torch.Generator().manual_seed(0)
  below_one = torch.tensor([BELOW_ONE], device=dev)
  for _ in range(400):
    env.bin_failed_count.copy_((torch.rand(env.bin_count, generator=g) * 3).to(dev))
    env._cdf.copy_(env._start_distribution()[1])
    if int(env._start_frames(below_one)[0]) == T_ - 1:
      break
  else:
    pytest.fail("no failure history puts the largest draw on the last frame")
  ema0 = env.bin_failed_count.clone()
  i = 0
  deltas = (-1e-3, -3e-7, 3e-7, 1e-3)
  want_term = {}
  a_z = env.motion["body_pos_w"][env.time_steps, env.anchor, 2] + env.env_origins[:, 2]
  for dz in deltas:  # anchor height error 0.25 + dz, the robot's anchor above and below the clip's
    for sgn in (1.0, -1.0):
      d.xpos[i, anchor, 2] = a_z[i] + sgn * (0.25 + dz)
      want_term[i] = dz > 0 if abs(dz) > 1e-6 else None
      i += 1
  for e, ee in enumerate(env.ee_idx.tolist()):  # each end effector alone
    for dz in deltas:
      d.xpos[i, int(bid[ee]), 2] = env.body_pos_relative_w[i, ee, 2] + 0.25 + dz
      want_term[i] = dz > 0 if abs(dz) > 1e-6 else None
      i += 1
  for b in range(len(env.body_idx)):  # a body that is not an end effector never terminates
    if b not in env.ee_idx.tolist() and b != env.anchor and i < 34:
      d.xpos[i, int(bid[b]), 2] += 0.2
      want_term[i] = False
      i += 1
  # gravity projection: tilt the robot's anchor about x from the clip's orientation until the z difference is 0.8 + dz
  from mjlab_b200.entity_data import quat_mul
  for dz in deltas:
    a_quat = env.motion["body_quat_w"][env.time_steps[i], env.anchor].double()
    lo_, hi_ = 0.0, math.pi
    for _ in range(80):  # bisection on the tilt angle, float64
      mid = 0.5 * (lo_ + hi_)
      tq = torch.tensor([math.cos(mid / 2), math.sin(mid / 2), 0.0, 0.0], dtype=torch.float64, device=dev)
      q = quat_mul(a_quat[None], tq[None])[0]
      gz = lambda qq: -(1 - 2 * (qq[1] ** 2 + qq[2] ** 2))
      if abs(float(gz(a_quat) - gz(q))) > 0.8 + dz:
        hi_ = mid
      else:
        lo_ = mid
    d.xquat[i, anchor] = q.float()
    want_term[i] = dz > 0 if abs(dz) > 1e-6 else None
    i += 1
  edge0 = i
  # clip time: T-2 (no restart), T-1 (restart, draws 0 and just below 1), an episode end on the last frame
  env.time_steps[i] = T_ - 2; i += 1
  env.time_steps[i] = T_ - 1; U[i, 13 + env.nu] = 0.0; i += 1
  env.time_steps[i] = T_ - 1; U[i, 13 + env.nu] = BELOW_ONE; i += 1
  env.episode_length_buf[i] = mx - 1; env.time_steps[i] = T_ - 1; U[i, 0] = 0.25; U[i, 13 + env.nu] = 0.75; two = i; i += 1
  env.episode_length_buf[i] = mx - 1; U[i, 0] = 0.0; i += 1
  env.episode_length_buf[i] = mx - 2; i += 1
  # failures in the first and the last bin; term && trunc
  env.time_steps[i] = 0; d.xpos[i, anchor, 2] -= 0.4; i += 1
  env.time_steps[i] = T_ - 1; d.xpos[i, anchor, 2] -= 0.4; i += 1
  env.episode_length_buf[i] = mx - 1; d.xpos[i, anchor, 2] -= 0.4; i += 1
  # self-collision count 0 / 1 / 10
  adr = env.self_collision_adr[0]
  for v in (0.0, 1.0, 10.0):
    d.sensordata[i, adr] = v; i += 1
  # push timer at step_dt exactly and one ulp either side
  dt = float(np.float32(env.step_dt))
  for t in (dt, _ulp(dt, 1), _ulp(dt, -1), -0.3):
    env.push_time_left[i] = t; i += 1
  # episode end and clip end in one step: the reset draws the last frame, the clip's step runs off it, and the env is
  # resampled again from the second block of U (whose joint noise differs from the first block's); timed out, and fallen
  twice = i
  for fallen in (False, True):
    U[i, 0] = BELOW_ONE; U[i, Sn] = 0.3; U[i, Sn + 13:Sn + 13 + env.nu] = 0.9
    if fallen:
      d.xpos[i, anchor, 2] -= 0.4
    else:
      env.episode_length_buf[i] = mx - 1
    i += 1
  # failures on the last frame of a bin and the first of the next (120 frames, 3 bins: 39 | 40, 79 | 80)
  bins0 = i
  for ts_ in (39, 40, 40, 79, 80):
    env.time_steps[i] = ts_; d.xpos[i, anchor, 2] -= 0.4; i += 1
  assert i <= env.num_envs and env.bin_count == 3 and T_ == 120
  S, T, N = H.both(action, U)
  info = check_tracking(H, S, T, N, action, U)
  H.report("tracking edges")
  for k, w in want_term.items():
    if w is not None:
      assert bool(N["out.terminated"][k]) == w and bool(T["out.terminated"][k]) == w, (k, w, info["margins"][k])
  c = H.counts
  assert c["in_band"] <= 14 and c["split"] <= c["in_band"], c  # (the 14 margins written at +-3e-7)
  assert all(c[f"term{k}"] >= 2 for k in range(6)), c  # every threshold terminated somebody
  assert c["clip_restart"] >= 2 and c["both"] >= 1 and c["push"] >= 3, c
  ts = N["env.time_steps"]
  assert int(ts[edge0]) == T_ - 1 and int(ts[edge0 + 1]) == 0 and int(ts[edge0 + 2]) == T_ - 1
  # episode end on the clip's last frame with a middling draw: one resample, from the first block, then one frame on
  assert int(ts[two]) == int(_drawn_frames(env, S, U[two:two + 1, 0])[0]) + 1 and 1 < int(ts[two]) < T_ - 1
  assert int(ts[two + 1]) == 1
  # the two resamples: the frame is the second block's draw (no further step), the joints carry its noise (0.9, not 0.5)
  assert c["double_resample"] >= 2, c
  lo, hi = env.cfg.joint_position_range
  for k in (twice, twice + 1):
    assert int(_drawn_frames(env, S, U[k:k + 1, 0])[0]) == T_ - 1
    assert int(ts[k]) == int(_drawn_frames(env, S, U[k:k + 1, Sn])[0]) and 0 < int(ts[k]) < T_ - 1
    for R in (T, N):
      noise = (R["data.qpos"][k, 7:] - env.motion["joint_pos"][ts[k]]).double()
      inside = (R["data.qpos"][k, 7:] > env._soft_lo) & (R["data.qpos"][k, 7:] < env._soft_hi)
      assert bool(inside.sum() > env.nu // 2) and float((noise[inside] - (0.9 * (hi - lo) + lo)).abs().max()) < 1e-6
  # failure counts per bin: each terminated env in the bin of the frame it had reached, EMA with alpha 0.5
  B = env.bin_count
  counts = torch.zeros(B, dtype=torch.float64, device=dev)
  for k in torch.nonzero(N["out.terminated"]).flatten().tolist():
    counts[min(int(S["env.time_steps"][k]) * B // T_, B - 1)] += 1
  for R in (T, N):
    H.close("bin_failed_count per bin", R["env.bin_failed_count"], 0.5 * counts + 0.5 * ema0.double(), floor=1.0,
            rowwise=False, rel=1e-6)
  assert [min(int(S["env.time_steps"][k]) * B // T_, B - 1) for k in range(bins0, bins0 + 5)] == [0, 1, 1, 1, 2]
  assert bool(N["out.terminated"][bins0:bins0 + 5].all()) and float(counts.min()) >= 1
  r = N["out.reward"]
  base = edge0 + 9
  assert float(r[base] - r[base + 1]) == pytest.approx(10.0 * env.step_dt, rel=1e-4)
  assert float(r[base] - r[base + 2]) == pytest.approx(100.0 * env.step_dt, rel=1e-4)
  env.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_tracking_reward_terms_in_isolation(backend, monkeypatch, tmp_path):
  """Only one reward term's inputs vary per batch; the rest of the state is the clip's own frame (errors 0)."""
  H = _tracking(backend, monkeypatch, num_envs=16, motion_file=_make_clip(backend, tmp_path, 120), episode_length_s=1.0)
  env = H.env
  dev, n = env.device, env.num_envs
  g = _gen(env, 23)
  r = lambda *s: torch.rand(s, generator=g, device=dev) * 2 - 1
  bid = env.robot.indexing.body_ids[env.body_idx].long()
  others = torch.tensor([int(b) for k, b in enumerate(bid) if k != env.anchor], device=dev)
  for term in ("anchor_pos", "anchor_ori", "body_pos", "body_ori", "lin_vel", "ang_vel", "rate", "limits", "collision"):
    action, U = _tracking_base(H)
    d = env.sim.data
    if term == "anchor_pos":
      d.xpos[:, int(bid[env.anchor]), 0:2] += 0.1 * r(n, 2)
    elif term == "anchor_ori":
      q = d.xquat[:, int(bid[env.anchor])] + 0.1 * r(n, 4)
      d.xquat[:, int(bid[env.anchor])] = q / q.norm(dim=1, keepdim=True)
    elif term == "body_pos":
      d.xpos[:, others, 0:2] += 0.1 * r(n, len(others), 2)
    elif term == "body_ori":
      q = d.xquat[:, others] + 0.1 * r(n, len(others), 4)
      d.xquat[:, others] = q / q.norm(dim=-1, keepdim=True)
    elif term == "lin_vel":
      d.link_vel_w[:, bid, 0:3] += r(n, len(bid), 3)
    elif term == "ang_vel":
      d.link_vel_w[:, bid, 3:6] += 3.0 * r(n, len(bid), 3)
    elif term == "rate":
      action = r(n, env.nu)
      env.last_action.copy_(r(n, env.nu))
    elif term == "limits":
      j = torch.arange(n, device=dev) % env.nu
      d.qpos[torch.arange(n, device=dev), 7 + j] = env._soft_hi[j] + 0.02 * r(n).abs() + 1e-3
    elif term == "collision":
      d.sensordata[:, env.self_collision_adr[0]] = torch.arange(n, device=dev).float() % 4
    S, T, N = H.both(action, U)
    check_tracking(H, S, T, N, action, U)
    rw = N["out.reward"]
    assert float(rw.max() - rw.min()) > 1e-3 * env.step_dt, term
    assert not bool(N["out.terminated"].any()), term
  H.report("tracking reward terms")
  env.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_tracking_observation_noise_columns(backend, monkeypatch):
  """Each noise column alone at 0 and just below 1, the others at 0.5: the policy group moves in that element only,
  by the amplitude of its term."""
  H = _tracking(backend, monkeypatch, num_envs=2 * (15 + 2 * 29), clip_frames=8, episode_length_s=1.0)
  env = H.env
  nu = env.nu
  action, U = _tracking_base(H)
  Z0 = 2 * (13 + nu) + 7
  amp = [0.25] * 3 + [0.05] * 6 + [0.5] * 3 + [0.2] * 3 + [0.01] * nu + [0.5] * nu
  vals = (0.0, BELOW_ONE)
  for c in range(15 + 2 * nu):
    for k, v in enumerate(vals):
      U[2 * c + k, Z0 + c] = v
  base_action, base_U = action, torch.full_like(U, 0.5)
  S, T0, N0 = H.both(base_action, base_U)
  check_tracking(H, S, T0, N0, base_action, base_U)
  _tracking_base(H)
  S, T, N = H.both(action, U)
  check_tracking(H, S, T, N, action, U)
  for R, R0 in ((T, T0), (N, N0)):
    H.equal("critic carries no noise", R["out.critic"], R0["out.critic"])
    diff = (R["out.obs"] - R0["out.obs"]).double()
    for c in range(15 + 2 * nu):
      for k, v in enumerate(vals):
        row = diff[2 * c + k].clone()
        want = (2.0 * np.float32(v) - 1.0) * amp[c]
        assert abs(float(row[2 * nu + c]) - want) <= 2e-6 * max(1.0, abs(float(R0["out.obs"][2 * c + k, 2 * nu + c]))), (c, v)
        row[2 * nu + c] = 0.0
        assert float(row.abs().max()) == 0.0, (c, v)
  H.report("tracking noise columns")
  env.close()

"""Push and external-wrench event terms (PushBySettingVelocityCfg, ApplyExternalForceTorqueCfg in
mjlab_b200/envs/events.py; the state block of csrc/b2_events.cuh).

* The torch path against the reference's own ``push_by_setting_velocity`` and ``apply_external_force_torque``,
  executed from oracle/_ref at every call of a torch-path rollout of workloads B and C (resets, a mid-run ``reset()``
  and, for C, clip restarts) on the host emulation.  The reference's ``sample_uniform`` is fed the env's V columns and
  its entity stand-in computes ``root_link_vel_w`` with the reference's ``compute_velocity_from_cvel`` over the env's
  ``sim.data``; qvel and xfrc_applied must be equal after every call.
* b2_events against the torch path on the fused path's own post-physics state, at 1 and 33 envs on the host emulation
  and 1, 33 and 4096 on the H100: timers and wrenches bit-identical; a pushed root velocity within PUSH_TOL (below);
  rows of envs that neither reset nor fired untouched.
* Under CUDA graph replay, the fused step writes what the eager fused step writes.
* Defaults: no new draw or launch without state terms, and ``push_vel=None`` turns the built-in push off on both paths.
* Every refusal of the cfg, of the envs and of the C entry.
"""

import ctypes
import types

import numpy as np
import pytest
import torch

import test_events as tev
import test_mdp_kernels as tmk
from mjlab_b200.envs import ApplyExternalForceTorqueCfg as W
from mjlab_b200.envs import EventsCfg, PushBySettingVelocityCfg as P, RandomizeFieldCfg as R
from mjlab_b200.envs import ResetJointsByScaleCfg as J, ResetRootStateUniformCfg as RR
from mjlab_b200.envs import events as evm
from mjlab_b200.envs import tracking_env as te
from mjlab_b200.envs import velocity_env as ve
from mjlab_b200.sim import native

# |kernel - torch| of a pushed root velocity: the kernel's cross product and quaternion rotation contract into FMAs
# under --use_fast_math, and an env the step reset reads its root from qvel and the normalised qpos quaternion (the
# masked forward has not run yet) where the torch path reads the forward's cvel and xquat.  Both are a few fp32
# roundings of values below 10 in magnitude.
PUSH_TOL = dict(atol=2e-5, rtol=2e-5)
# the reset root orientation and the angular velocity rotated by it, against the reference: its quat_mul takes a
# factored form of the Hamilton product (three sums folded into products) that rounds differently from the direct form
# used here; both are a few fp32 roundings of unit-magnitude values
QUAT_TOL = dict(atol=1e-6, rtol=1e-6)
# |kernel - torch| of a reset root on the fused path: the kernel's sinf / cosf under --use_fast_math are within 2 ulps
# of the correctly rounded values for |x| <= pi, and its products contract into FMAs; a few ulps of values below 10
RESET_TOL = dict(atol=4e-6, rtol=4e-6)
I = (0.0, 0.012)  # interval_range_s of the rollouts (step_dt 0.005: fires every one to three steps)
ALL6 = {k: (-0.3 * (i + 1), 0.2 * (i + 1)) for i, k in enumerate(evm.AXES6)}


def _cases(kind: str) -> dict:
  if kind == "C":  # the tracking env offers interval pushes and wrenches (reset state terms are no-ops there)
    return {"push": (P(ALL6, interval_range_s=I),),
            "wrench": (W((-20.0, 20.0), (-2.0, 3.0), names=(".*_ankle_roll_link", "torso_link"), interval_range_s=I),
                       P({"x": (-0.5, 0.5), "yaw": (-1.0, 1.0)}, interval_range_s=(0.0, 0.004))),
            "two": (W((-5.0, 5.0), (-1.0, 1.0), interval_range_s=(0.0, 0.004)),
                    W((1.0, 2.0), (0.0, 0.0), names="pelvis", interval_range_s=I),
                    R("body_mass", (0.9, 1.1), mode="reset", operation="scale", names="pelvis"))}
  cases = {f"push_{k}": (P({k: ALL6[k]}, interval_range_s=I),) for k in evm.AXES6}
  cases["push_all"] = (P(ALL6, interval_range_s=I),)
  cases.update({f"root_pose_{k}": (RR({k: ALL6[k]}, {}),) for k in evm.AXES6})
  cases.update({f"root_vel_{k}": (RR({}, {k: ALL6[k]}),) for k in evm.AXES6})
  cases["root_all"] = (RR({"x": (-0.5, 0.5), "y": (-0.5, 0.5), "yaw": (-3.14, 3.14), "roll": (-0.1, 0.1)}, ALL6),
                       J((0.5, 1.5), (-1.0, 1.0)))
  cases["joints"] = (J((0.8, 1.2), (0.0, 0.0), names=(".*_knee_joint", ".*_hip_pitch_joint")),
                     J((0.0, 10.0), (-1.0, 1.0), names=".*_elbow_joint"),  # scales that hit the soft limits
                     P({"x": (-0.5, 0.5)}, interval_range_s=I))
  cases["wrench"] = (W((-20.0, 20.0), (-2.0, 3.0), names="torso_link", mode="reset"),
                     W((-5.0, 5.0), (-1.0, 1.0), names=".*_ankle_roll_link", interval_range_s=I))
  cases["two"] = (P({"x": (-0.5, 0.5), "y": (-0.5, 0.5)}, interval_range_s=(0.0, 0.004)),  # shorter than step_dt
                  W((-5.0, 5.0), (-1.0, 1.0), interval_range_s=I),
                  R("dof_damping", (0.5, 2.0), mode="reset", operation="scale"))
  return cases


def _env(kind, terms, n, device="cpu", native_mdp=False, **kw):
  ev = EventsCfg(terms=terms)
  if kind == "B":
    cfg = dict(num_envs=n, decimation=1, fall_angle=0.12, episode_length_s=0.03, push_vel=None, events=ev)
    return ve.VelocityFlatEnv(ve.VelocityEnvCfg(**{**cfg, **kw}), device=device, native_mdp=native_mdp)
  cfg = dict(num_envs=n, decimation=1, clip_frames=7, episode_length_s=0.04, push_velocity_range=None, events=ev)
  return te.TrackingFlatEnv(te.TrackingEnvCfg(**{**cfg, **kw}), device=device, native_mdp=native_mdp)


# ---- the torch path against the reference's functions -------------------------------------------------------------------
class _RefEntity:
  """The slice of the reference's Entity that push_by_setting_velocity and apply_external_force_torque use, over the
  env's sim.data (a copy of it, which the reference's writes go to)."""

  def __init__(self, ref_data, ix, d):
    self.ix, self.d = ix, d
    rb = ix.root_body_id
    self.num_bodies = len(ix.body_names)
    vel = ref_data.compute_velocity_from_cvel(d["xpos"][:, rb], d["subtree_com"][:, rb], d["cvel"][:, rb])
    self.data = types.SimpleNamespace(root_link_vel_w=vel, root_link_quat_w=d["xquat"][:, rb])

  def write_root_link_pose_to_sim(self, pose, env_ids):
    self.d["qpos"][env_ids, 0:7] = pose

  def write_joint_state_to_sim(self, pos, vel, env_ids, joint_ids):
    rows_q, rows_v = self.d["qpos"][env_ids], self.d["qvel"][env_ids]
    rows_q[:, 7 + joint_ids], rows_v[:, 6 + joint_ids] = pos, vel
    self.d["qpos"][env_ids], self.d["qvel"][env_ids] = rows_q, rows_v

  def write_root_link_velocity_to_sim(self, vel, env_ids):
    self.d["qvel"][env_ids, 0:6] = vel

  def write_external_wrench_to_sim(self, forces, torques, env_ids, body_ids):
    g = self.ix.body_ids[body_ids if body_ids is not None else slice(None)]
    x = self.d["xfrc_applied"]
    rows = x[env_ids]
    rows[:, g, 0:3] = forces
    rows[:, g, 3:6] = torques
    x[env_ids] = rows


def _reference_call(ref, E, t, mask, monkeypatch):
  """qvel and xfrc_applied after the reference's function runs term t on the envs of `mask` of the env's current
  state, its sampler fed the env's V columns."""
  import mjlab.entity.data as ref_data

  d = E.sim.data
  state = {k: getattr(d, k)[:].clone() for k in ("qpos", "qvel", "xfrc_applied", "xpos", "xquat", "subtree_com",
                                                 "cvel")}
  ix = E.indexing
  ent = _RefEntity(ref_data, ix, state)
  n = E.num_envs
  if E.reset_ctx is not None:
    q0, org, lo, hi = E.reset_ctx
    ent.data.default_root_state = torch.cat([q0[0:7], torch.zeros(6)]).expand(n, 13)
    ent.data.default_joint_pos, ent.data.default_joint_vel = q0[7:].expand(n, -1), torch.zeros(n, len(lo))
    ent.data.soft_joint_pos_limits = torch.stack([lo, hi], dim=-1).expand(n, -1, 2)
  ids = torch.arange(E.num_envs) if mask is None else mask.nonzero().flatten()
  step = {native.EVENT_PUSH: 6, evm.ROOT: 6, evm.JOINTS: t.count}.get(t.kind, 3 * t.count)
  cols = iter(range(t.col, t.col + t.draws, step))
  V = E.V

  def sample(lower, upper, size, device):
    c = next(cols)
    u = V[ids, c:c + int(np.prod(size[1:]))].reshape(size)
    return u * (upper - lower) + lower

  monkeypatch.setattr(ref.events, "sample_uniform", sample)
  scene = {"robot": ent}
  renv = types.SimpleNamespace(num_envs=E.num_envs, device="cpu",
                               scene=_Scene(scene, None if E.reset_ctx is None else E.reset_ctx[1]))
  if len(ids):
    c = t.cfg
    if t.kind == evm.ROOT:
      ref.events.reset_root_state_uniform(renv, ids, c.pose_range, c.velocity_range)
    elif t.kind == evm.JOINTS:
      cfg = types.SimpleNamespace(name="robot", joint_ids=list(t.bodies))
      ref.events.reset_joints_by_scale(renv, ids, c.position_range, c.velocity_range, asset_cfg=cfg)
    elif t.kind == native.EVENT_PUSH:
      ref.events.push_by_setting_velocity(renv, ids, c.velocity_range)
    else:
      names = list(ix.body_names)
      hit = evm._resolve_names(c.names, names, "body") if c.names is not None else slice(None)
      cfg = types.SimpleNamespace(name="robot", body_ids=hit)
      ref.events.apply_external_force_torque(renv, ids, c.force_range, c.torque_range, asset_cfg=cfg)
  return state["qpos"], state["qvel"], state["xfrc_applied"]


class _Scene(dict):
  def __init__(self, entities, env_origins):
    super().__init__(entities)
    self.env_origins = env_origins


CASES_B, CASES_C = list(_cases("B")), list(_cases("C"))


def _reference_rollout(kind, case, monkeypatch):
  ref = tev._reference(monkeypatch)
  tmk._patch_emul(monkeypatch, ve if kind == "B" else te)
  checked = {"calls": 0, "fired": 0}
  apply_state = evm.Events._apply_state

  def rec(self, t, mask):
    want_qpos, want_qvel, want_x = _reference_call(ref, self, t, mask, monkeypatch)
    apply_state(self, t, mask)
    d = self.sim.data
    if t.kind == evm.ROOT:  # the orientation: see QUAT_TOL
      torch.testing.assert_close(d.qpos[:, 3:7], want_qpos[:, 3:7], **QUAT_TOL)
      torch.testing.assert_close(d.qvel[:, 3:6], want_qvel[:, 3:6], **QUAT_TOL)
      want_qpos, want_qvel = want_qpos.clone(), want_qvel.clone()
      want_qpos[:, 3:7], want_qvel[:, 3:6] = d.qpos[:, 3:7], d.qvel[:, 3:6]
    assert torch.equal(d.qpos[:], want_qpos), (case, t.cfg, (d.qpos[:] != want_qpos).nonzero()[:4])
    assert torch.equal(d.qvel[:], want_qvel), (case, t.cfg, (d.qvel[:] != want_qvel).nonzero()[:4])
    assert torch.equal(d.xfrc_applied[:], want_x), (case, t.cfg)
    checked["calls"] += 1
    checked["fired"] += self.num_envs if mask is None else int(mask.sum())

  monkeypatch.setattr(evm.Events, "_apply_state", rec)
  env = _env(kind, _cases(kind)[case], 6)
  g = torch.Generator().manual_seed(7)
  resets = restarts = 0
  for k in range(30):
    if k == 15:
      env.reset()
    _, _, term, trunc, _ = env.step(torch.rand((env.num_envs, env.nu), generator=g) * 2 - 1)
    resets += int((term | trunc).sum())
    if kind == "C":
      restarts += int((env._done_buf & ~(term | trunc)).sum())
  assert checked["fired"] > 0 and resets > 0 and (kind == "B" or restarts > 0), (checked, resets, restarts)
  env.close()


@pytest.mark.parametrize("case", CASES_B)
def test_torch_path_matches_reference_functions_B(case, monkeypatch):
  _reference_rollout("B", case, monkeypatch)


@pytest.mark.parametrize("case", CASES_C)
def test_torch_path_matches_reference_functions_C(case, monkeypatch):
  _reference_rollout("C", case, monkeypatch)


def test_g1_flat_push_robot_as_a_term(monkeypatch):
  """push_vel=None plus the reference's G1 flat push_robot term (velocity x, y in +-0.5, every 1 to 3 s) on the torch
  path: each firing writes what the reference's push_by_setting_velocity writes (checked inside the rollout), and
  the built-in push timer stands still."""
  ref = tev._reference(monkeypatch)
  tmk._patch_emul(monkeypatch, ve)
  env = ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=8, decimation=1, push_vel=None, events=EventsCfg(terms=(
    P({"x": (-0.5, 0.5), "y": (-0.5, 0.5)}, interval_range_s=(1.0, 3.0)),))), device="cpu", native_mdp=False)
  t = env.events.state[0]
  before = env.push_time_left.clone()
  fired = 0
  for _ in range(12):
    env.events.timers[t.timer] = torch.where(torch.rand(env.num_envs) < 0.5, 0.0, env.events.timers[t.timer])
    fire = (env.events.timers[t.timer] - env.step_dt) < 1e-6
    env.step(torch.zeros(env.num_envs, env.nu))
    fired += int(fire.sum())
  assert fired > 0 and torch.equal(env.push_time_left, before)
  # one more firing, checked against the reference's function on the state it read
  env.events.timers[t.timer] = 0.0
  E = env.events
  _, want_qvel, _ = _reference_call(ref, E, t, torch.ones(env.num_envs, dtype=torch.bool), monkeypatch)
  E._apply_state(t, E._fire(t))
  assert torch.equal(env.sim.data.qvel[:], want_qvel)
  env.close()


# ---- b2_events against the torch path on one saved state ---------------------------------------------------------------
def _kernel_case(kind, backend, monkeypatch, case, n, steps):
  mod = ve if kind == "B" else te
  if backend == "emul":
    tmk._patch_emul(monkeypatch, mod)
  env = _env(kind, _cases(kind)[case], n, device="cpu" if backend == "emul" else "cuda:0", native_mdp=True,
             episode_length_s=0.03)
  if kind == "C":
    env._native_setup()
  E, d, sim = env.events, env.sim.data, env.sim
  g = tmk._gen(env, n)
  counts = dict(reset=0, fired=0, kept=0)
  for k in range(steps):
    act = torch.rand((n, env.nu), generator=g, device=env.device) * 2 - 1
    # the fused step up to b2_events, then b2_events against the torch reset and interval parts
    post, forward, run_native = E.run_native, sim.forward, None
    saved = {}

    def stop(sim_):
      saved.update(qvel=d.qvel[:].clone(), xfrc=d.xfrc_applied[:].clone(), timers=E.timers.clone(),
                   qpos=d.qpos[:].clone())
      post(sim_)

    E.run_native = stop
    if kind == "B":  # (the masked forward runs below, after the comparison; C's pushes run after it)
      sim.forward = lambda env_mask=None: None
    env.step(act)
    E.run_native, sim.forward = post, forward
    term, trunc, done = env._term.clone(), env._trunc.clone(), env._done_buf.clone()
    got = dict(qvel=d.qvel[:].clone(), xfrc=d.xfrc_applied[:].clone(), timers=E.timers.clone())
    d.qvel[:] = saved["qvel"]
    d.xfrc_applied[:] = saved["xfrc"]
    E.timers.copy_(saved["timers"])
    E.step_torch(term, trunc)
    if E.reset_state_terms():  # the post kernel's reset root and joint terms against the torch ones, from one V
      r = term | trunc
      torch.testing.assert_close(d.qpos[:][r], saved["qpos"][r], **RESET_TOL)
      torch.testing.assert_close(d.qvel[:][r], saved["qvel"][r], **RESET_TOL)
      assert torch.equal(d.qpos[:][~r], saved["qpos"][~r])
      d.qpos[:], d.qvel[:] = saved["qpos"], saved["qvel"]  # (on from the fused path's values)
      counts["reset_terms"] = counts.get("reset_terms", 0) + int(r.sum())
    sim.forward(env_mask=done)
    E.step_interval_state()
    assert torch.equal(E.timers, got["timers"]), (case, k)
    assert torch.equal(d.xfrc_applied[:], got["xfrc"]), (case, k)
    fired = (got["timers"] != saved["timers"] - env.step_dt).any(0) if E.timers.numel() else torch.zeros_like(done)
    hit = term | trunc | fired
    pushed = any(t.kind == native.EVENT_PUSH for t in E.state)
    if pushed:
      torch.testing.assert_close(d.qvel[:][hit], got["qvel"][hit], **PUSH_TOL)
    assert torch.equal(got["qvel"][~hit], saved["qvel"][~hit]), (case, k)  # rows that neither reset nor fired
    assert torch.equal(got["xfrc"][~hit], saved["xfrc"][~hit]), (case, k)
    # continue from the fused path's state, with the env's own forward
    d.qvel[:] = got["qvel"]
    sim.forward(env_mask=done)
    counts["reset"] += int((term | trunc).sum())
    counts["fired"] += int((fired & ~(term | trunc)).sum())
    counts["kept"] += int((~hit).sum())
  assert (counts["fired"] > 0 or case == "root_all") and (n < 33 or counts["reset"] > 0), counts
  env.close()


KERNEL_B = ["push_all", "wrench", "two", "root_all", "joints"]


@pytest.mark.parametrize("case", KERNEL_B)
@pytest.mark.parametrize("n", [1, 33])
def test_kernel_matches_torch_emul_B(case, n, monkeypatch):
  _kernel_case("B", "emul", monkeypatch, case, n, steps=12 if n == 1 else 8)


@pytest.mark.parametrize("case", CASES_C)
@pytest.mark.parametrize("n", [1, 33])
def test_kernel_matches_torch_emul_C(case, n, monkeypatch):
  _kernel_case("C", "emul", monkeypatch, case, n, steps=12 if n == 1 else 8)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,case", [("B", c) for c in KERNEL_B] + [("C", c) for c in CASES_C])
@pytest.mark.parametrize("n", [1, 33, 4096])
def test_kernel_matches_torch_cuda(kind, case, n, monkeypatch):
  _kernel_case(kind, "cuda", monkeypatch, case, n, steps=12 if n == 1 else 8)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["B", "C"])
def test_graph_replay_matches_eager(kind):
  """Two envs from one seed, one stepped through the captured graph and one eagerly, write the same state."""
  n, case = 512, "two"
  envs = [_env(kind, _cases(kind)[case], n, device="cuda:0", native_mdp=True, episode_length_s=0.2) for _ in range(2)]
  envs[0].enable_cuda_graph()
  envs[1].enable_cuda_graph()  # (the same warm-up steps), then stepped eagerly
  envs[1]._graph = None
  g = torch.Generator(device="cuda:0").manual_seed(3)
  for _ in range(10):
    a = torch.rand((n, envs[0].nu), generator=g, device="cuda:0") * 2 - 1
    outs = [e.step(a) for e in envs]
    assert torch.equal(outs[0][0], outs[1][0])
    for f in ("qpos", "qvel", "xfrc_applied"):
      assert torch.equal(getattr(envs[0].sim.data, f)[:], getattr(envs[1].sim.data, f)[:]), f
    assert torch.equal(envs[0].events.timers, envs[1].events.timers)
  assert (envs[0].sim.data.xfrc_applied[:] != 0).any()
  for e in envs:
    e.close()


@pytest.mark.gpu
def test_physics_sees_the_state_writes():
  """A velocity env with reset root and joint terms, a reset and an interval wrench and an interval push, through its
  CUDA graph: after steps with resets, pushes and wrenches, the next sub-step of those worlds matches the oracle loaded
  with the same qpos, qvel, ctrl and xfrc_applied."""
  from util import load_oracle, relerr

  from oracle.oracle import Oracle

  n = 64
  terms = (RR({"x": (-0.3, 0.3), "yaw": (-3.14, 3.14), "roll": (-0.1, 0.1)}, {"x": (-0.5, 0.5), "yaw": (-1.0, 1.0)}),
           J((0.5, 1.5), (-1.0, 1.0)), W((-30.0, 30.0), (-3.0, 3.0), names="torso_link", mode="reset"),
           W((-20.0, 20.0), (-2.0, 2.0), names=".*_ankle_roll_link", interval_range_s=(0.0, 0.03)),
           P({"x": (-0.5, 0.5), "y": (-0.5, 0.5), "yaw": (-0.5, 0.5)}, interval_range_s=(0.0, 0.03)))
  env = ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=n, fall_angle=0.12, episode_length_s=0.2, push_vel=None,
                                             events=EventsCfg(terms=terms)))
  env.enable_cuda_graph()
  done = torch.zeros(n, dtype=torch.bool, device="cuda:0")
  for _ in range(60):
    _, _, term, trunc, _ = env.step(torch.zeros(n, env.nu, device="cuda:0"))
    done |= term | trunc
    if int(done.sum()) >= 8:
      break
  assert int(done.sum()) >= 8
  sim, m = env.sim, env.model
  assert bool((sim.data.xfrc_applied[:] != 0).any())
  o = Oracle(m, nworld=n, maxcon=int(sim.get_option("maxcon")))
  sim.set_option("iterations", 50)  # converged answers do not depend on the path that reached them
  for k in ("timestep", "iterations", "ls_iterations", "tolerance", "ls_tolerance", "integrator"):
    o.set_option(k, sim.get_option(k))
  load_oracle(o, {f: getattr(sim.data, f)[:].cpu().numpy() for f in ("qpos", "qvel", "ctrl", "qacc_warmstart")})
  o.field("xfrc_applied")[:] = sim.data.xfrc_applied[:].cpu().numpy().reshape(n, -1)
  o.model_field("geom_friction")[:] = sim.model.geom_friction[...].cpu().numpy().reshape(n, -1)
  o.step()
  sim.step()
  torch.cuda.synchronize()
  for f in ("qpos", "qvel"):
    e = relerr(getattr(sim.data, f)[:].cpu().numpy(), o.field(f)).max()
    assert e < 1e-3, (f, e)
  env.close()


# ---- defaults -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["B", "C"])
def test_no_state_terms_draw_and_launch_nothing_new(kind, monkeypatch):
  tmk._patch_emul(monkeypatch, ve if kind == "B" else te)
  mod = ve.VelocityFlatEnv if kind == "B" else te.TrackingFlatEnv
  cfg = (ve.VelocityEnvCfg if kind == "B" else te.TrackingEnvCfg)(num_envs=3)
  env = mod(cfg, device="cpu", native_mdp=True)
  assert env.events.V is None and not env.events.state and not env.events.clear_xfrc
  if kind == "C":
    env._native_setup()
  assert env.events._args is None  # (no b2_events launch)
  env.close()


@pytest.mark.parametrize("native_mdp", [False, True])
def test_push_vel_none_turns_the_builtin_push_off(native_mdp, monkeypatch):
  tmk._patch_emul(monkeypatch, ve)
  env = ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=4, decimation=1, push_vel=None, push_interval_s=(0.0, 0.0)),
                           device="cpu", native_mdp=native_mdp)
  t0 = env.push_time_left.clone()
  for _ in range(3):
    env.step(torch.zeros(4, env.nu))
  assert torch.equal(env.push_time_left, t0)
  assert ve.VelocityEnvCfg().push_vel == 0.5
  env.close()


# ---- refusals -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("make,match", [
  (lambda: P({"forward": (0, 1)}, interval_range_s=I), "unknown velocity_range keys"),
  (lambda: P({"x": (1, 0)}, interval_range_s=I), "lo <= hi"),
  (lambda: P({"x": (0, float("inf"))}, interval_range_s=I), "finite"),
  (lambda: P({"x": (0, 1)}, interval_range_s=I, mode="reset"), "mode must be one of"),
  (lambda: P({"x": (0, 1)}, interval_range_s=I, mode="startup"), "first reset"),
  (lambda: P({"x": (0, 1)}), "needs interval_range_s"),
  (lambda: P({"x": (0, 1)}, interval_range_s=(-1.0, 1.0)), "0 <= lo"),
  (lambda: W((1, 0), (0, 1)), "lo <= hi"),
  (lambda: W((0, 1), (0, float("nan")), mode="reset"), "finite"),
  (lambda: W((0, 1), (0, 1), mode="startup"), "first reset"),
  (lambda: W((0, 1), (0, 1), mode="sometimes"), "mode must be one of"),
  (lambda: W((0, 1), (0, 1)), "needs interval_range_s"),
  (lambda: W((0, 1), (0, 1), mode="reset", names=3), "names must be"),
  (lambda: EventsCfg(terms=("push",)), "every term must be"),
  (lambda: RR({"z": (0, 1), "w": (0, 1)}, {}), "unknown pose_range keys"),
  (lambda: RR({}, {"x": (1, 0)}), "lo <= hi"),
  (lambda: RR({}, {"yaw": (0, float("inf"))}), "finite"),
  (lambda: RR({}, {}, mode="interval"), "mode must be one of"),
  (lambda: RR({}, {}, mode="startup"), "first reset"),
  (lambda: J((1.5, 0.5), (0, 0)), "lo <= hi"),
  (lambda: J((0.5, 1.5), (0, 0), mode="startup"), "first reset"),
  (lambda: J((0.5, 1.5), (0, 0), mode="interval"), "mode must be one of"),
])
def test_cfg_refusals(make, match):
  with pytest.raises(ValueError, match=match):
    make()


def test_env_refusals(monkeypatch):
  push = P({"x": (-0.5, 0.5)}, interval_range_s=I)
  with pytest.raises(ValueError, match="needs push_vel=None"):
    ve.VelocityEnvCfg(events=EventsCfg(terms=(push,)))
  with pytest.raises(ValueError, match="needs push_velocity_range=None"):
    te.TrackingEnvCfg(events=EventsCfg(terms=(push,)))
  te.TrackingEnvCfg(push_velocity_range=None, events=EventsCfg(terms=(push,)))
  for t in (W((0, 1), (0, 1), mode="reset"), RR({"x": (0, 1)}, {}), J((0.5, 1.5), (0, 0))):
    with pytest.raises(ValueError, match="no-op in the tracking env"):
      te.TrackingEnvCfg(events=EventsCfg(terms=(t,)))
  tmk._patch_emul(monkeypatch, ve)
  with pytest.raises(ValueError, match="match no body"):
    ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=2, events=EventsCfg(terms=(W((0, 1), (0, 1), mode="reset",
                                                                              names="no_such_link"),))), device="cpu")
  with pytest.raises(ValueError, match="match no joint"):
    ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=2, events=EventsCfg(terms=(J((0.5, 1.5), (0, 0),
                                                                              names="no_such_joint"),))), device="cpu")
  cfg = ve.VelocityEnvCfg(num_envs=2)
  cfg.events = EventsCfg(terms=(push,))  # (set after the cfg's own check: the env checks again)
  with pytest.raises(ValueError, match="needs push_vel=None"):
    ve.VelocityFlatEnv(cfg, device="cpu")


def test_c_entry_refusals(monkeypatch):
  """b2_events refuses every malformed state block before it launches (host emulation)."""
  tmk._patch_emul(monkeypatch, ve)
  env = _env("B", _cases("B")["two"], 3, native_mdp=True)
  lib, h = env.sim._lib, env.sim._h
  A = env.events._args
  call = lambda a: lib.b2_events(h, ctypes.byref(a), None)  # noqa: E731
  assert call(A) == 0
  push, wrench = 0, 1  # (the "two" case: a push, then an interval wrench)
  cases = [
    ("unknown kind", lambda a: setattr(a.state[push], "kind", 7)),
    ("unknown mode", lambda a: setattr(a.state[wrench], "mode", 5)),
    ("reset push", lambda a: setattr(a.state[push], "mode", native.EVENT_RESET)),
    ("push count", lambda a: setattr(a.state[push], "count", 5)),
    ("V column outside the row", lambda a: setattr(a.state[wrench], "col", a.v_width - 3)),
    ("negative column", lambda a: setattr(a.state[push], "col", -1)),
    ("body table counts", lambda a: setattr(a, "nbodies", a.nbodies + 1)),
    ("body table order", lambda a: setattr(a.state[wrench], "first", 1)),
    ("no body table", lambda a: setattr(a, "bodies", None)),
    ("timer row", lambda a: setattr(a.state[wrench], "timer", a.state[push].timer)),
    ("timer past ninterval", lambda a: setattr(a, "ninterval", a.ninterval - 1)),
    ("negative interval", lambda a: setattr(a.state[push], "interval_lo", -1.0)),
    ("no refreshed mask", lambda a: setattr(a, "refreshed", None)),
    ("root body", lambda a: setattr(a, "root_body", 0)),
    ("too many state terms", lambda a: setattr(a, "nstate", native.EVENTS_NSTATE + 1)),
    ("no term at all", lambda a: (setattr(a, "nstate", 0), setattr(a, "nterm", 0))),
  ]
  for label, edit in cases:
    a = native.B2EventArgs.from_buffer_copy(A)
    edit(a)
    assert call(a) != 0, label
    assert b"b2_events" in lib.b2_last_error(), label
  # a body id outside the model, read back from the device table (a new table address: the entry checks it afresh)
  bad = env.events._keep[1].clone()
  bad[-1] = 10_000
  a = native.B2EventArgs.from_buffer_copy(A)
  a.bodies = bad.data_ptr()
  assert call(a) != 0 and b"outside the model's bodies" in lib.b2_last_error()
  env.close()


def test_c_entry_refuses_bad_reset_terms(monkeypatch):
  """b2_velenv_post refuses a malformed reset-term table before it launches (host emulation)."""
  tmk._patch_emul(monkeypatch, ve)
  env = _env("B", _cases("B")["root_all"], 3, native_mdp=True)
  lib, h, A = env.sim._lib, env.sim._h, env._native_args
  call = lambda a: lib.b2_velenv_post(h, ctypes.byref(a), None)  # noqa: E731
  for label, edit in [
    ("unknown kind", lambda a: setattr(a.reset_term[0], "kind", 9)),
    ("root count", lambda a: setattr(a.reset_term[0], "count", 11)),
    ("V column outside the row", lambda a: setattr(a.reset_term[1], "col", a.ev_v_width - 1)),
    ("joint outside nu", lambda a: a.reset_term[1].joint.__setitem__(0, env.nu)),
    ("joint count", lambda a: setattr(a.reset_term[1], "count", 33)),
    ("too many terms", lambda a: setattr(a, "n_reset", native.VELENV_NRESET + 1)),
    ("no V", lambda a: setattr(a, "ev_V", None)),
  ]:
    a = native.B2VelEnvArgs.from_buffer_copy(A)
    edit(a)
    assert call(a) != 0, label
    assert b"b2_velenv_post" in lib.b2_last_error(), label
  env.close()


def test_c_layout_of_the_state_block():
  """The ctypes mirrors of B2EventStateTerm and the appended B2EventArgs fields have the C structs' offsets, and no
  earlier field of B2EventArgs moved."""
  import subprocess
  from pathlib import Path

  root = Path(__file__).resolve().parents[1]
  structs = (native.B2EventStateTerm, native.B2EventArgs, native.B2VelResetTerm)
  src = '#include <stdio.h>\n#include <stddef.h>\n#include "b2sim.h"\nint main(void) {\n'
  want = []
  for S in structs:
    src += f'  printf("%zu\\n", sizeof({S.__name__}));\n'
    want.append(ctypes.sizeof(S))
    for f, _ in S._fields_:
      src += f'  printf("%zu\\n", offsetof({S.__name__}, {f}));\n'
      want.append(getattr(S, f).offset)
  src += ('  printf("%d %d %d\\n", B2_EVENTS_NSTATE, B2_EVENT_PUSH, B2_EVENT_WRENCH);\n  return 0;\n}\n')
  import tempfile

  with tempfile.TemporaryDirectory() as tmp:
    c = Path(tmp) / "layout.c"
    c.write_text(src)
    exe = Path(tmp) / "layout"
    subprocess.run(["cc", "-I", str(root / "include"), str(c), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
  assert [int(x) for x in out[:-3]] == want
  assert [int(x) for x in out[-3:]] == [native.EVENTS_NSTATE, native.EVENT_PUSH, native.EVENT_WRENCH]
  # the block starts after the last field it was appended to (at the pointer alignment)
  assert native.B2EventArgs.refreshed.offset == (native.B2EventArgs.term.offset + ctypes.sizeof(native.B2EventTerm)
                                                 * native.EVENTS_NTERM + 7) // 8 * 8

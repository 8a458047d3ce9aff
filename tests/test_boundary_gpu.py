"""Boundary contract on the GPU: what the reference pins in tests/test_sim_data.py,
tests/test_entity.py:292-388, tests/smoke_test.py:21-22 and tests/test_nan_guard.py, restated
against our Simulation."""

import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

BOX_XML = """
<mujoco>
  <worldbody>
    <body name="box" pos="0 0 1">
      <freejoint name="free"/>
      <geom name="box_geom" type="box" size="0.1 0.1 0.1" mass="1.0"/>
    </body>
  </worldbody>
</mujoco>
"""


def _box_sim(n=3):
  from mjlab_b200.compiler import Spec
  from mjlab_b200.sim import Simulation, SimulationCfg

  m = Spec.from_string(BOX_XML).compile()
  return Simulation(n, SimulationCfg(), m, "cuda:0"), m


def test_time_zero_and_derived_fields_valid_after_construction(g1_model):
  from mjlab_b200.sim import Simulation, SimulationCfg

  sim = Simulation(2, SimulationCfg(), g1_model, "cuda:0")
  assert float(sim.data.time[0]) == 0.0  # tests/smoke_test.py:22
  assert sim.data.nworld == 2
  # forward ran at qpos0: pelvis at its XML height, kinematics populated (SURVEY §8a S1b)
  assert float(sim.data.xpos[0, 2, 2]) == pytest.approx(0.793, abs=1e-5)
  assert float(sim.data.xquat[0, 2, 0]) == pytest.approx(1.0)
  sim.close()


def test_bridge_is_read_only_and_views_share_memory():
  sim, _ = _box_sim()
  with pytest.raises(AttributeError, match="Cannot set attribute"):
    sim.data.qpos = torch.zeros(1)
  q = sim.data.qpos
  assert q is sim.data.qpos  # wrapper cache
  ptr = q.data_ptr()
  q[:] = 7.0
  assert q.data_ptr() == ptr  # slice-assign keeps the address (CUDA-graph safety)
  assert float(sim.wp_data.qpos[1, 0]) == 7.0
  assert torch.sum(q).item() == pytest.approx(7.0 * 3 * 7)  # torch functions accept the wrapper
  assert ((q + 1)[0, 0]).item() == 8.0
  sim.close()


def test_free_fall_and_applied_wrench_qualitative():
  """tests/test_entity.py:292-330: gravity pulls down; +x force moves +x; z torque spins about z."""
  sim, m = _box_sim(3)
  sim.step()
  assert (sim.data.qvel[:, 2] < 0).all()
  sim.data.qvel[:] = 0
  sim.data.xfrc_applied[:, 1, 0] = 10.0
  x0 = sim.data.qpos[:, 0].clone()
  for _ in range(10):
    sim.step()
  assert (sim.data.qpos[:, 0] > x0).all()
  sim.data.xfrc_applied[:] = 0
  sim.data.qvel[:] = 0
  sim.data.xfrc_applied[:, 1, 5] = 1.0
  for _ in range(10):
    sim.step()
  w = sim.data.qvel[0, 3:6].abs()
  assert w[2] > 5 * max(w[0], w[1])
  # a huge force does not produce NaN (tests/test_entity.py:378-388)
  sim.data.xfrc_applied[:, 1, 0] = 1e6
  sim.step()
  assert torch.isfinite(sim.data.qpos[:]).all()
  sim.close()


def test_free_fall_matches_analytic():
  sim, m = _box_sim(1)
  sim.data.qpos[:, 2] = 5.0
  n = 50
  for _ in range(n):
    sim.step()
  h = float(m.opt_timestep)
  # semi-implicit Euler: v_k = -g k h, z_k = z0 - g h^2 k(k+1)/2
  assert float(sim.data.qvel[0, 2]) == pytest.approx(-9.81 * n * h, rel=1e-5)
  assert float(sim.data.qpos[0, 2]) == pytest.approx(5.0 - 9.81 * h * h * n * (n + 1) / 2, rel=1e-5)
  sim.close()


def test_nan_guard_dumps_once(tmp_path):
  from mjlab_b200.compiler import Spec
  from mjlab_b200.sim import Simulation, SimulationCfg
  from mjlab_b200.utils.nan_guard import NanGuardCfg

  m = Spec.from_string(BOX_XML).compile()
  cfg = SimulationCfg(nan_guard=NanGuardCfg(enabled=True, output_dir=str(tmp_path)))
  sim = Simulation(4, cfg, m, "cuda:0")
  sim.step()
  assert not list(tmp_path.glob("*.npz"))
  sim.data.qpos[1, 0] = float("nan")  # fault injection as in tests/test_nan_guard.py:70
  sim.step()
  dumps = list(tmp_path.glob("*.npz"))
  assert len(dumps) == 1
  z = np.load(dumps[0])
  assert 1 in z["nan_env_ids"]
  sim.step()
  assert len(list(tmp_path.glob("*.npz"))) == 1
  sim.close()


def test_c_abi_host_buffer_step(g1_model):
  """b2_step_host: host ctrl in, qpos/qvel out, equals the device-side path."""
  from mjlab_b200.sim import Simulation, SimulationCfg

  n = 16
  a = Simulation(n, SimulationCfg(), g1_model, "cuda:0")
  b = Simulation(n, SimulationCfg(), g1_model, "cuda:0")
  key = g1_model.keys["robot/init_state"]
  for s in (a, b):
    s.data.qpos[:] = torch.tensor(key["qpos"], device="cuda:0", dtype=torch.float32)
  ctrl = (np.tile(key["ctrl"], (n, 1)) + 0.1).astype(np.float32)
  nq, nv = int(g1_model.nq), int(g1_model.nv)
  qpos = np.zeros((n, nq), np.float32)
  qvel = np.zeros((n, nv), np.float32)
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
  rc = a._lib.b2_step_host(a._h, ctrl.ctypes.data_as(ctypes.c_void_p), 4,
                           qpos.ctypes.data_as(ctypes.c_void_p), qvel.ctypes.data_as(ctypes.c_void_p), stream)
  assert rc == 0
  torch.cuda.synchronize()
  b.data.ctrl[:] = torch.tensor(ctrl, device="cuda:0")
  b.step_n(4)
  torch.cuda.synchronize()
  assert (qpos == b.data.qpos[:].cpu().numpy()).all()
  assert (qvel == b.data.qvel[:].cpu().numpy()).all()
  assert a.launch_count() >= 4
  a.close()
  b.close()


def test_cuda_graph_replay_matches_eager(g1_model):
  from mjlab_b200.sim import Simulation, SimulationCfg
  from util import load_sim, make_states

  st = make_states(g1_model, 8, seed=3)
  a = Simulation(8, SimulationCfg(), g1_model, "cuda:0")
  b = Simulation(8, SimulationCfg(), g1_model, "cuda:0")
  b.use_cuda_graph = True
  b.create_graph()
  load_sim(a, st)
  load_sim(b, st)
  for _ in range(3):
    a.step()
    b.step()
  b.expand_model_fields(["geom_friction"])  # graphs are re-captured lazily after expansion
  a.expand_model_fields(["geom_friction"])
  a.step()
  b.step()
  torch.cuda.synchronize()
  assert (a.data.qpos[:] == b.data.qpos[:]).all()
  a.close()
  b.close()


def test_velocity_env_runs_and_resets():
  from mjlab_b200.envs import VelocityEnvCfg, VelocityFlatEnv

  env = VelocityFlatEnv(VelocityEnvCfg(num_envs=64), device="cuda:0")
  obs = env.reset()
  assert obs.shape == (64, 3 + 3 + 3 + 29 + 29 + 29 + 3)
  total_done = 0
  g = torch.Generator(device="cuda:0")
  g.manual_seed(11)
  for _ in range(150):
    a = torch.rand((64, 29), generator=g, device="cuda:0") * 2 - 1
    obs, r, term, trunc, _ = env.step(a)
    total_done += int(term.sum())
  assert torch.isfinite(obs).all() and torch.isfinite(r).all()
  assert total_done > 0  # random actions make G1 fall within a few seconds; those envs were reset
  assert (env.sim.data.qpos[:, 2] > 0.2).all()
  env.close()


def test_velocity_env_cuda_graph_matches_eager():
  from mjlab_b200.envs import VelocityEnvCfg, VelocityFlatEnv

  a = VelocityFlatEnv(VelocityEnvCfg(num_envs=32, push_interval_s=(1e9, 2e9)), device="cuda:0")
  b = VelocityFlatEnv(VelocityEnvCfg(num_envs=32, push_interval_s=(1e9, 2e9)), device="cuda:0")
  b.enable_cuda_graph()
  # graph warm-up advanced b by two (zero-action) steps: bring both to the same state again
  for f in ("qpos", "qvel", "qacc_warmstart", "ctrl"):
    getattr(b.sim.data, f)[:] = getattr(a.sim.data, f)[:]
  b.episode_length_buf[:] = a.episode_length_buf
  b.last_action[:] = a.last_action
  b.command[:] = a.command
  b.push_time_left[:] = a.push_time_left
  b.cmd_time_left[:] = a.cmd_time_left
  b.heading_target[:] = a.heading_target
  b.is_standing[:] = a.is_standing
  g = torch.Generator(device="cuda:0")
  g.manual_seed(5)
  for _ in range(5):  # short horizon: nobody falls, so no (differently seeded) resets happen
    act = (torch.rand((32, 29), generator=g, device="cuda:0") * 2 - 1) * 0.2
    oa = a.step(act)
    ob = b.step(act)
    # the policy observation carries noise drawn from generators that are in different states after the capture
    # warm-up; the critic group is the same terms without noise
    assert torch.allclose(oa[4]["critic"], ob[4]["critic"], atol=1e-5) and torch.allclose(oa[1], ob[1], atol=1e-6)
    assert (oa[0] - oa[4]["critic"]).abs().max() > 0.05 and (ob[0] - ob[4]["critic"]).abs().max() > 0.05
    assert torch.equal(b.log_row[:, 0], ob[1])
  a.close()
  b.close()


def test_long_rollout_stays_finite_and_within_capacity():
  """Soak: 300 env steps (1200 physics steps) of the benchmark workload at 1024 envs."""
  from mjlab_b200.envs import VelocityEnvCfg, VelocityFlatEnv

  env = VelocityFlatEnv(VelocityEnvCfg(num_envs=1024), device="cuda:0")
  env.enable_cuda_graph()
  g = torch.Generator(device="cuda:0")
  g.manual_seed(9)
  resets = 0
  for k in range(300):
    obs, r, term, trunc, _ = env.step(torch.rand((1024, 29), generator=g, device="cuda:0") * 2 - 1)
    resets += int(term.sum())
  d = env.sim.data
  assert torch.isfinite(d.qpos[:]).all() and torch.isfinite(d.qvel[:]).all() and torch.isfinite(obs).all()
  assert (d.qvel[:].abs() < 200).all()  # nothing exploded
  st = env.sim.stats()
  assert st.overflow_worlds == 0 and st.ncon_max <= st.ncon_cap
  assert resets > 1024  # every env fell and was reset at least once on average
  env.close()


def test_entity_data_over_engine_views(g1_model):
  """EntityData (S7) on the real strided engine tensors: int32 index tensors, (N,1) env ids."""
  from mjlab_b200.entity_data import EntityData, EntityIndexing
  from mjlab_b200.sim import Simulation, SimulationCfg
  from util import load_sim, make_states

  n = 16
  sim = Simulation(n, SimulationCfg(), g1_model, "cuda:0")
  st = make_states(g1_model, n, seed=2, vel=1.0)
  load_sim(sim, st)
  sim.forward()
  ed = EntityData(EntityIndexing.from_model(g1_model, "robot", "cuda:0"), sim.data, sim.model, "cuda:0", n)
  qvel = torch.tensor(st["qvel"], dtype=torch.float32, device="cuda:0")
  assert torch.allclose(ed.root_link_lin_vel_w, qvel[:, 0:3], atol=1e-4)   # csv_to_npz.py:279-284
  assert torch.allclose(ed.root_link_ang_vel_b, qvel[:, 3:6], atol=1e-4)
  assert ed.body_link_vel_w.shape == (n, 30, 6) and ed.geom_pose_w.shape == (n, 68, 7)
  env_ids = torch.tensor([3, 7], device="cuda:0")
  state = torch.arange(26, dtype=torch.float32, device="cuda:0").reshape(2, 13)
  ed.write_root_state(state, env_ids)
  assert torch.equal(sim.data.qpos[env_ids][:, :7], state[:, :7])
  ed.write_joint_position(torch.full((2, 2), 0.1, device="cuda:0"), joint_ids=torch.tensor([1, 4], device="cuda:0"), env_ids=env_ids)
  assert torch.allclose(sim.data.qpos[env_ids][:, [8, 11]], torch.full((2, 2), 0.1, device="cuda:0"))
  ed.write_external_wrench(torch.ones(n, 30, 3, device="cuda:0"), None)
  sim.step()
  assert torch.isfinite(sim.data.qpos[:]).all()
  ed.clear_state()
  assert (sim.data.xfrc_applied[:] == 0).all()
  sim.close()


def test_native_mdp_kernels_match_torch_reference():
  """b2_velenv_pre/post (fused MDP glue) vs the torch implementation through step() end to end, same seeds and
  uniforms.  Two simulations run the physics separately and b is re-synchronised to a after every step, so this
  comparison is loose (an agreement fraction, absolute tolerances); the strict one, on one saved state, every output
  and every environment, is tests/test_mdp_kernels.py."""
  from mjlab_b200.envs import VelocityEnvCfg, VelocityFlatEnv

  cfg = dict(num_envs=128, fall_angle=0.12, push_interval_s=(0.02, 0.08), episode_length_s=0.2)
  a = VelocityFlatEnv(VelocityEnvCfg(**cfg), device="cuda:0", native_mdp=False)
  b = VelocityFlatEnv(VelocityEnvCfg(**cfg), device="cuda:0", native_mdp=True)
  assert torch.equal(a.sim.data.qpos[:], b.sim.data.qpos[:])
  g = torch.Generator(device="cuda:0")
  g.manual_seed(11)
  n_term = n_trunc = 0
  for k in range(14):
    act = torch.rand((128, 29), generator=g, device="cuda:0") * 2 - 1
    oa, ra, ta, ua, _ = a.step(act)
    ob, rb, tb, ub, _ = b.step(act)
    # physics runs separately in the two sims from identical states with ctrl equal up to 1 ulp (FMA vs
    # mul+add), so a few contact-rich envs may differ slightly: require agreement on >= 97 % of the envs
    ok = (ta == tb) & (ua == ub) & ((ra - rb).abs() < 1e-4) & ((oa - ob).abs().amax(dim=1) < 2e-3)
    assert ok.float().mean() >= 0.97, (k, float(ok.float().mean()))
    assert torch.equal(ua, ub)  # time-outs do not depend on the physics
    same = ta == tb
    assert torch.equal(a.episode_length_buf[same], b.episode_length_buf[same])
    assert torch.allclose(a.command[same], b.command[same], atol=1e-6)
    assert torch.allclose(a.push_time_left, b.push_time_left, atol=1e-6)
    # re-synchronise so that differences never accumulate (the MDP logic is what is under test)
    for f in ("qpos", "qvel", "qacc_warmstart", "ctrl"):
      getattr(b.sim.data, f)[:] = getattr(a.sim.data, f)[:]
    b.episode_length_buf.copy_(a.episode_length_buf)
    b.last_action.copy_(a.last_action)
    b.command.copy_(a.command)
    n_term += int(ta.sum())
    n_trunc += int(ua.sum())
  assert n_term > 20 and n_trunc > 20  # both reset paths were exercised
  a.close()
  b.close()


def test_engine_side_entity_quantities_match_torch_derivation(g1_model):
  """SURVEY.md §8f-2: link / com velocities, body-frame velocities, projected gravity and heading written by the
  step kernel equal what EntityData derives from (xpos, xquat, subtree_com, cvel) with torch ops; in a decimation
  loop only the last sub-step writes the consumer-visible kinematics, with the same final values."""
  from mjlab_b200.entity_data import EntityData, EntityIndexing
  from mjlab_b200.sim import Simulation, SimulationCfg
  from util import load_sim, make_states

  n = 64
  st = make_states(g1_model, n, seed=41, vel=2.0, tilt=0.8)
  sim = Simulation(n, SimulationCfg(), g1_model, "cuda:0")
  load_sim(sim, st)
  sim.forward()
  ix = EntityIndexing.from_model(g1_model, "robot", "cuda:0")
  a = EntityData(ix, sim.data, sim.model, "cuda:0", n, native=True)
  b = EntityData(ix, sim.data, sim.model, "cuda:0", n, native=False)
  assert a._native and not b._native
  for name in ("root_link_vel_w", "root_com_vel_w", "body_link_vel_w", "body_com_vel_w", "projected_gravity_b",
               "heading_w", "root_link_lin_vel_b", "root_link_ang_vel_b", "root_com_lin_vel_b", "root_com_ang_vel_b"):
    x, y = getattr(a, name), getattr(b, name)
    assert x.shape == y.shape and torch.allclose(x, y, atol=2e-5, rtol=1e-5), (name, float((x - y).abs().max()))
  # step_n(4) == 4 x step(): state and the (last sub-step's) kinematics outputs
  sim2 = Simulation(n, SimulationCfg(), g1_model, "cuda:0")
  load_sim(sim, st)
  load_sim(sim2, st)
  sim.step_n(4)
  for _ in range(4):
    sim2.step()
  torch.cuda.synchronize()
  for f in ("qpos", "qvel", "xpos", "xquat", "xmat", "geom_xpos", "geom_xmat", "site_xpos", "cvel", "subtree_com",
            "link_vel_w", "com_vel_w", "link_state_b"):
    assert torch.equal(getattr(sim.data, f)[:], getattr(sim2.data, f)[:]), f
  sim.close()
  sim2.close()

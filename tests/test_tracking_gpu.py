"""Config C (BASELINE.json configs[2]): G1 motion tracking on flat ground — the env-level caller and one-step
parity against the fp64 oracle at the contact-rich, self-colliding states the random-action agent produces
(per-world domain randomisation of body_ipos / qpos0 / geom_friction included)."""

import numpy as np
import pytest
import torch

from util import relerr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def T(x):
  return x[:].detach().cpu().numpy()


@pytest.fixture(scope="module")
def env():
  from mjlab_b200.envs import TrackingEnvCfg, TrackingFlatEnv

  e = TrackingFlatEnv(TrackingEnvCfg(num_envs=256, seed=7), device=DEV)
  yield e
  e.close()


def test_tracking_env_steps_and_resets(env):
  n = env.num_envs
  g = torch.Generator(device=DEV)
  g.manual_seed(0)
  pol, crit = env.observations()
  assert pol.shape == (n, 58 + 3 + 6 + 3 + 3 + 29 + 29 + 29) and crit.shape == (n, pol.shape[1] + 14 * 3 + 14 * 6)
  resets, selfcol, maxcon = 0, 0.0, 0
  for _ in range(40):
    obs, rew, term, trunc, extra = env.step(torch.rand((n, 29), generator=g, device=DEV) * 2 - 1)
    assert torch.isfinite(obs).all() and torch.isfinite(rew).all() and torch.isfinite(extra["critic"]).all()
    resets += int((term | trunc).sum())
    selfcol = max(selfcol, float(env.sim.data.sensordata[:, env.self_collision_adr[0]].max()))
    maxcon = max(maxcon, int(env.sim.data.ncon[:].max()))
  assert resets > 0          # flailing robots leave the reference pose and are put back on the clip
  assert selfcol >= 1.0      # the self-collision sensor (num=10 slots, slot 0 = count) sees contacts
  assert maxcon >= 12
  assert (env.time_steps >= 0).all() and (env.time_steps < env.cfg.clip_frames).all()
  assert int(env.sim.stats().overflow_worlds) == 0
  # per-world DR is in place: torso com offsets, joint zero offsets and foot friction differ between worlds
  assert env.sim.model.body_ipos[:].std(dim=0).max() > 1e-3 and env.sim.model.qpos0[:].std(dim=0).max() > 1e-3


def test_tracking_step_parity_at_self_collision_states(env):
  """One physics step from the env's own mid-rollout states (many contacts, self-collisions, active limits)."""
  from oracle.oracle import Oracle

  sim, m, n = env.sim, env.model, env.num_envs
  o = Oracle(m, nworld=n, maxcon=int(sim.get_option("maxcon")))
  for f in ("body_ipos", "qpos0", "geom_friction"):
    o.model_field(f)[:] = T(getattr(sim.model, f)).reshape(n, -1)
  for f in ("qpos", "qvel", "ctrl", "qacc_warmstart"):
    o.field(f)[:] = T(getattr(sim.data, f))
  o.field("xfrc_applied")[:] = T(sim.data.xfrc_applied).reshape(n, -1)
  o.step()
  sim.step()
  torch.cuda.synchronize()
  d = sim.data
  same = T(d.ncon).ravel() == o.ncon.ravel()
  assert same.mean() > 0.97  # a contact at the detection threshold may appear on one side only
  assert o.ncon.max() >= 12 and o.sensordata[:, 0].max() >= 1
  assert (T(d.sensordata)[same] == o.sensordata[same]).all()  # self-collision counts are integers: exact
  for f, p99, mx in (("qpos", 1e-5, 1e-4), ("qvel", 1e-4, 1e-3), ("qacc_warmstart", 1e-4, 1e-3)):
    e = relerr(T(getattr(d, f))[same], o.field(f)[same], floor=1e-9)
    assert np.percentile(e, 99) < p99 * 3 and e.max() < mx * 3, (f, np.percentile(e, 99), e.max())


def test_tracking_env_step_is_graph_capturable():
  """One whole env step (ctrl, 4 sub-steps, terminations, rewards, RSI resets + masked forwards, command update,
  push, both observation groups) replays from a CUDA graph: no host synchronisation anywhere in the step."""
  from mjlab_b200.envs import TrackingEnvCfg, TrackingFlatEnv

  b = TrackingFlatEnv(TrackingEnvCfg(num_envs=64, seed=3), device=DEV)
  b.enable_cuda_graph()
  g = torch.Generator(device=DEV)
  g.manual_seed(1)
  q0 = b.sim.data.qpos[:].clone()
  done = 0
  for _ in range(30):
    ob, rb, tb, ub, info = b.step(torch.rand((64, 29), generator=g, device=DEV) * 2 - 1)
    assert torch.isfinite(ob).all() and torch.isfinite(rb).all() and torch.isfinite(info["critic"]).all()
    done += int((tb | ub).sum())
    assert torch.equal(b.log_row[:, 0], rb)
  assert not torch.equal(b.sim.data.qpos[:], q0) and done > 0
  b.close()


def test_tracking_native_mdp_kernels_match_torch_reference():
  """csrc/b2_trackenv.cuh (two fused kernels around the masked forward) against the torch implementation through
  step() end to end, on the same uniforms.  Two simulations run the physics separately and are re-synchronised after
  every step, so this comparison is loose; the strict one, on one saved state, every output and every environment, is
  tests/test_mdp_kernels.py."""
  from mjlab_b200.envs import TrackingEnvCfg, TrackingFlatEnv

  n = 128
  cfg = dict(num_envs=n, seed=5, episode_length_s=0.3, clip_frames=12, push_interval_s=(0.05, 0.15))
  a = TrackingFlatEnv(TrackingEnvCfg(**cfg), device=DEV, native_mdp=False)
  b = TrackingFlatEnv(TrackingEnvCfg(**cfg), device=DEV, native_mdp=True)
  assert torch.equal(a.sim.data.qpos[:], b.sim.data.qpos[:])
  g = torch.Generator(device=DEV)
  g.manual_seed(2)
  term = trunc = 0
  for k in range(25):
    act = torch.rand((n, 29), generator=g, device=DEV) * 2 - 1
    if k == 5:  # falls: the anchors of the first envs drop below the clip's by more than 0.25 m
      for e in (a, b):
        e.sim.data.qpos[:8, 2] -= 0.4
    oa, ra, ta, ua, xa = a.step(act)
    ob, rb, tb, ub, xb = b.step(act)
    # a termination threshold crossed within fp32 rounding may differ between two runs of the physics: compare the
    # envs whose flags agree, and require that to be nearly all of them
    same = (ta == tb) & (ua == ub) & (a._done_buf == b._done_buf)
    assert same.float().mean() > 0.97, (k, same.float().mean())
    assert torch.allclose(ra[same], rb[same], atol=5e-4), (k, (ra - rb)[same].abs().max())
    assert torch.equal(a.time_steps[same], b.time_steps[same])
    assert torch.allclose(oa[same], ob[same], atol=5e-3), (k, (oa - ob)[same].abs().max())
    assert torch.allclose(xa["critic"][same], xb["critic"][same], atol=5e-3)
    assert torch.allclose(a.body_pos_relative_w[same], b.body_pos_relative_w[same], atol=1e-4)
    term += int(ta.sum())
    trunc += int(ua.sum())
    for f in ("qpos", "qvel", "qacc_warmstart", "ctrl"):  # resynchronise: the MDP logic is what is under test
      getattr(b.sim.data, f)[:] = getattr(a.sim.data, f)[:]
    for f in ("time_steps", "episode_length_buf", "last_action", "push_time_left", "body_pos_relative_w", "body_quat_relative_w"):
      getattr(b, f).copy_(getattr(a, f))
  assert term > 0 and trunc > 0
  a.close()
  b.close()

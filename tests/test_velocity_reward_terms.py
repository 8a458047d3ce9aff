"""Opt-in reward terms of the velocity task (VelocityEnvCfg.rewards) and their episode logs: the torch path against the
reference's own functions (tasks/velocity/mdp/rewards.py, envs/mdp/rewards.py, run from oracle/_ref), the fused post
kernel against the torch path on one saved state (the Harness of test_mdp_kernels.py; emul here, the H100 under
-m gpu), and the configurations the env refuses.

Where terms are enabled, check_velocity's float64 reward (five fixed terms) is extended by the opt-in terms' weighted
values as the torch path logged them: those are held to the reference's functions in the first test."""

import ctypes
import importlib.util
import math
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import refload
import test_mdp_kernels as tmk
from mjlab_b200.sim import native

ROOT = Path(__file__).resolve().parents[1]
BACKENDS = tmk.BACKENDS
REWARD_ENV = ["air_time", "contact_time", "last_air_time", "episode_sums", "finished_sums"]
GO1_FEET = ("FR", "FL", "RR", "RL")
NEW = ("air_time", "feet_slide", "foot_clearance", "is_alive", "is_terminated", "joint_torques_l2", "joint_acc_l2",
       "electrical_power_cost", "flat_orientation_l2")


def _rewards(**kw):
  import mjlab_b200.envs.velocity_env as ve

  base = dict(feet_slide_sensor_names=tuple(f"{f}_foot_ground_contact" for f in GO1_FEET),
              feet_slide_geom_names=tuple(f"{f}_foot_collision" for f in GO1_FEET),
              foot_clearance_geom_names=tuple(f"{f}_foot_collision" for f in GO1_FEET),
              target_height=0.1, std=0.05, tanh_mult=2.0)
  base.update(kw)
  return ve.VelocityRewardsCfg(**base)


def _all_on(**kw):
  w = dict(air_time=1.0, feet_slide=-0.25, foot_clearance=0.5, is_alive=0.3, is_terminated=-2.0,
           joint_torques_l2=-1e-4, joint_acc_l2=-2.5e-7, electrical_power_cost=-2e-3, flat_orientation_l2=-1.0)
  w.update(kw)
  return _rewards(**w)


def _harness(backend, monkeypatch, **cfg):
  H = tmk._velocity(backend, monkeypatch, **cfg)
  H.env_fields += REWARD_ENV
  return H


def _extra_from_log(S, T):
  """Weighted opt-in terms times step_dt, [n, 9], as the torch path added them to its episode sums."""
  done = (T["out.terminated"] | T["out.truncated"]).unsqueeze(1)
  after = torch.where(done, T["env.finished_sums"], T["env.episode_sums"])
  return (after - S["env.episode_sums"]).double()[:, 5:]


def check(H, S, T, N, action, U, monkeypatch):
  """check_velocity with the opt-in terms in its float64 reward, then the reward state of the two paths."""
  orig = tmk._velocity_reference
  extra = _extra_from_log(S, T)

  def ref(env, S_, action_):
    margin, r64, s64 = orig(env, S_, action_)
    return margin, r64 + extra.sum(1), s64 + extra.abs().sum(1)

  monkeypatch.setattr(tmk, "_velocity_reference", ref)
  tmk.check_velocity(H, S, T, N, action, U)
  monkeypatch.setattr(tmk, "_velocity_reference", orig)
  for k in ("env.air_time", "env.contact_time", "env.last_air_time"):
    H.equal(k, T[k], N[k])
  for k in ("env.episode_sums", "env.finished_sums"):
    H.close(k, T[k], N[k], floor=1e-6, rowwise=False, scale=T[k].abs().amax(0, keepdim=True).expand_as(T[k]))


def _rollout(H, steps, seed, monkeypatch):
  env = H.env
  n, g = env.num_envs, tmk._gen(env, seed)
  env.episode_length_buf.copy_(torch.randint(0, env.max_episode_length, (n,), generator=g, device=env.device).int())
  for _ in range(steps):
    act = torch.rand((n, env.nu), generator=g, device=env.device) * 2 - 1
    tmk._pre(env, act)
    env.sim.step_n(env.cfg.decimation)
    U = env._draw()
    # the sums restart each step, so that the step's values read back from them exactly (_extra_from_log);
    # accumulation is checked in test_episode_sums_and_reward_log
    env.episode_sums.zero_()
    S, T, N = H.both(act, U)
    check(H, S, T, N, act, U, monkeypatch)


# ---- the torch path against the reference's functions ------------------------------------------------------------
def _ref_modules(monkeypatch):
  if not refload.available():
    pytest.skip("the reference package is not installed (oracle/install_reference.py)")
  monkeypatch.syspath_prepend(str(ROOT / "tests" / "stubs"))  # prettytable stand-in (managers package)
  ns = refload.load()
  mods = []
  for name, rel in (("mjlab.tasks.velocity.mdp.rewards", ("tasks", "velocity", "mdp", "rewards.py")),
                    ("mjlab.envs.mdp.rewards", ("envs", "mdp", "rewards.py"))):
    spec = importlib.util.spec_from_file_location(name, refload.REF / "mjlab" / Path(*rel))
    mod = importlib.util.module_from_spec(spec)
    monkeypatch.setitem(sys.modules, name, mod)
    spec.loader.exec_module(mod)
    mods.append(mod)
  return ns, mods[0], mods[1]


def _ref_env(ns, env, terminated):
  """A ManagerBasedRlEnv with the fields the reward functions read, from the env's Data (the geom velocities through
  the reference's own compute_velocity_from_cvel)."""
  import types

  from mjlab_b200.envs.velocity_env import quat_rotate_inverse

  m, d = env.model, env.sim.data
  sensors = {s.split("/", 1)[1]: int(m.arrays["sensor_adr"][i]) for i, s in enumerate(m.names["sensor"])}
  body = torch.as_tensor(np.asarray(m.arrays["geom_bodyid"]), dtype=torch.long)
  pos = d.geom_xpos[...].clone()
  vel = ns.entity_data.compute_velocity_from_cvel(pos, d.subtree_com[:, env._root_body].unsqueeze(1),
                                                  d.cvel[:, body])
  data = types.SimpleNamespace(
    sensor_data={s: d.sensordata[:, a:a + 1].clone() for s, a in sensors.items()}, geom_pos_w=pos,
    geom_lin_vel_w=vel[..., 0:3], actuator_force=d.actuator_force[...].clone(), joint_acc=d.qacc[:, 6:].clone(),
    joint_vel=d.qvel[:, 6:].clone(), projected_gravity_b=quat_rotate_inverse(d.qpos[:, 3:7], env._down))
  robot = types.SimpleNamespace(data=data, sensor_names=list(sensors))
  return types.SimpleNamespace(
    scene={"robot": robot}, num_envs=env.num_envs, device=env.device, step_dt=env.step_dt,
    command_manager=types.SimpleNamespace(get_command=lambda name: env.command),
    termination_manager=types.SimpleNamespace(terminated=terminated))


def _ours(env, terminated):
  from mjlab_b200.envs.velocity_env import quat_rotate_inverse

  d = env.sim.data
  done = torch.zeros(env.num_envs, dtype=torch.bool)
  return env._opt_in_rewards(terminated, done, quat_rotate_inverse(d.qpos[:, 3:7], env._down))


@pytest.mark.parametrize("mode", ["on_landing", "continuous"])
@pytest.mark.parametrize("scale", ["smooth", "hard"])
def test_torch_terms_match_reference_functions(mode, scale, monkeypatch):
  """feet_air_time over a contact sequence with landings (both modes, both command scales), feet_slide,
  foot_clearance_reward and the six penalties of envs/mdp/rewards.py, each at weight 1 on the same Data."""
  ns, vr, er = _ref_modules(monkeypatch)
  from mjlab.managers.manager_term_config import RewardTermCfg

  H = _harness("emul", monkeypatch, robot="go1", num_envs=24, decimation=1,
               rewards=_rewards(**{t: 1.0 for t in NEW}, reward_mode=mode, command_scale_type=scale))
  env = H.env
  g = tmk._gen(env, 7)
  d = env.sim.data
  # some physics so that velocities, forces and accelerations are not zero
  for _ in range(3):
    tmk._pre(env, torch.rand((env.num_envs, env.nu), generator=g) * 2 - 1)
    env.sim.step_n(1)
  env.command.copy_(torch.rand((env.num_envs, 3), generator=g) * 2 - 1)
  env.command[::4, :2] = 0.0  # standing: the smooth scale is small, the hard one 0
  env.command[1::4, 0] = 0.05  # at the command threshold
  sensors = [f"{f}_foot_ground_contact" for f in GO1_FEET]
  adr = env._air_adr.long()
  terminated = torch.rand(env.num_envs, generator=g) < 0.3
  air_cfg = RewardTermCfg(func=vr.feet_air_time, weight=1.0, params=dict(
    asset_name="robot", threshold_min=0.05, threshold_max=0.15, command_name="twist", command_threshold=0.05,
    sensor_names=sensors, reward_mode=mode, command_scale_type=scale, command_scale_width=0.2))
  ref_air = vr.feet_air_time(air_cfg, _ref_env(ns, env, terminated))
  landings = 0
  for k in range(40):  # feet in the air for 1..12 steps (0.02 .. 0.24 s at step_dt 0.02) between contacts
    period = torch.arange(env.num_envs * 4).view(env.num_envs, 4) % 12 + 1
    contact = ((k // period) % 2 == 0) | (torch.rand((env.num_envs, 4), generator=g) < 0.05)
    d.sensordata[:, adr] = contact.float() * torch.rand((env.num_envs, 4), generator=g)  # 0 or found > 0 (a count)
    renv = _ref_env(ns, env, terminated)
    want = ref_air(renv)
    landings += int(((env.air_time > 0) & (d.sensordata[:, adr] > 0)).sum())
    got = _ours(env, terminated)
    torch.testing.assert_close(got[:, 0], want.float(), rtol=2e-6, atol=1e-6)
    torch.testing.assert_close(env.air_time, ref_air.current_air_time, rtol=0, atol=0)
    torch.testing.assert_close(env.last_air_time, ref_air.last_air_time, rtol=0, atol=0)
    torch.testing.assert_close(env.contact_time, ref_air.current_contact_time, rtol=0, atol=0)
  assert landings > 50
  renv = _ref_env(ns, env, terminated)
  geoms = env._slide_geom.long().tolist()
  asset = types_ns(name="robot", geom_ids=geoms)
  want = {
    "feet_slide": vr.feet_slide(renv, sensors, asset),
    "foot_clearance": vr.foot_clearance_reward(renv, 0.1, 0.05, 2.0, asset),
    "is_alive": er.is_alive(renv), "is_terminated": er.is_terminated(renv),
    "joint_torques_l2": er.joint_torques_l2(renv), "electrical_power_cost": er.electrical_power_cost(renv),
    "joint_acc_l2": er.joint_acc_l2(renv, types_ns(name="robot", joint_ids=slice(None))),
    "flat_orientation_l2": er.flat_orientation_l2(renv)}
  got = _ours(env, terminated)
  for t, w in want.items():
    v = got[:, NEW.index(t)]
    assert float(v.abs().max()) > 0, t
    torch.testing.assert_close(v, w.float(), rtol=4e-6, atol=1e-7, msg=t)
  env.close()


def types_ns(**kw):
  import types

  return types.SimpleNamespace(**kw)


# ---- the fused kernel against the torch path ---------------------------------------------------------------------
@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("term", NEW)
def test_each_term_alone(backend, term, monkeypatch):
  """One opt-in term at weight 1, the others off, over a short rollout with physics (feet leave the ground under
  random actions; short episodes reset envs inside it)."""
  big = backend == "cuda"
  kw = {term: 1.0}
  if term == "air_time":
    kw.update(reward_mode="continuous", threshold_min=0.0)
  H = _harness(backend, monkeypatch, robot="go1", num_envs=256 if big else 6, decimation=4 if big else 1,
               episode_length_s=0.2 if big else 0.02, fall_angle=0.3, rewards=_rewards(**kw))
  _rollout(H, 12 if big else 6, seed=21, monkeypatch=monkeypatch)
  log = H.env.reward_log()
  assert set(log) == {f"Episode_Reward/{t}" for t in ("track_lin_vel_exp", "track_ang_vel_exp", "pose",
                                                        "dof_pos_limits", "action_rate_l2", term)}
  H.report(f"term {term}")
  H.env.close()


def _edge_env(backend, monkeypatch, mode, scale, dt_steps=1):
  H = _harness(backend, monkeypatch, robot="go1", num_envs=24, rewards=_rewards(
    air_time=1.0, reward_mode=mode, command_scale_type=scale, threshold_min=0.06, threshold_max=0.16))
  env = H.env
  env.default_qpos[7:] = torch.minimum(torch.maximum(env.default_qpos[7:], env.soft_lo), env.soft_hi)
  return H


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("mode", ["on_landing", "continuous"])
@pytest.mark.parametrize("scale", ["smooth", "hard"])
def test_air_time_edges(backend, mode, scale, monkeypatch):
  """Air time that reaches threshold_min or threshold_max exactly this step (one IEEE + step_dt) and one ulp either
  side, a landing (first contact) against a foot that stays down, the command norm at command_threshold and one ulp
  above, and done envs whose foot state is zeroed after their reward."""
  H = _edge_env(backend, monkeypatch, mode, scale)
  env = H.env
  rc = env.cfg.rewards
  dt = np.float32(env.step_dt)
  lo, hi = np.float32(rc.threshold_min), np.float32(rc.threshold_max)
  thr = np.float32(rc.command_threshold)
  mx = env.max_episode_length

  def before(t):  # the air time a foot in the air needs before this step to reach t after it
    a = np.float32(t - dt)
    while np.float32(a + dt) > t:
      a = np.nextafter(a, np.float32(-1))
    while np.float32(a + dt) < t:
      a = np.nextafter(a, np.float32(1))
    assert np.float32(a + dt) == t
    return float(a)

  # (air before, contact now, command x, done): one foot per row written, the others down and at rest
  cases = []
  for t in (lo, hi):
    a = before(t)
    for k in (-1, 0, 1):
      cases.append((tmk._ulp(a, k), False, 0.5, False))  # in the air: continuous edges
      cases.append((float(np.float32(tmk._ulp(a, k) + dt)), True, 0.5, False))  # landing with air time t +- ulp
  cases += [(0.0, True, 0.5, False), (0.1, True, float(thr), False), (0.1, True, tmk._ulp(thr, 1), False),
            (0.1, False, float(thr), False), (0.1, False, tmk._ulp(thr, 1), False), (0.1, True, 0.5, True),
            (0.1, False, 0.5, True), (0.3, True, 0.5, False)]
  rows = [dict(command=[c, 0.0, 0.0], **({"episode_length_buf": mx - 1} if done else {})) for _, _, c, done in cases]
  action, U = tmk._fill(H, rows)
  adr = env._air_adr.long()
  d = env.sim.data
  d.sensordata[:, adr] = 1.0
  env.air_time.zero_(); env.contact_time.fill_(0.5); env.last_air_time.fill_(0.02)
  for i, (a, contact, _, _) in enumerate(cases):
    env.air_time[i, 0] = a
    env.contact_time[i, 0] = 0.0 if a > 0 else 0.5
    d.sensordata[i, adr[0]] = 1.0 if contact else 0.0
  S, T, N = H.both(action, U)
  check(H, S, T, N, action, U, monkeypatch)
  air = _extra_from_log(S, N)[:, 0] / float(dt)
  done = N["out.terminated"] | N["out.truncated"]
  for i, (a, contact, c, dn) in enumerate(cases):
    new = np.float32(0.0) if contact else np.float32(np.float32(a) + dt)
    first = a > 0 and contact
    if mode == "continuous":
      per = float(not contact and lo < new <= hi)
    else:
      per = float(min(max(np.float32(a) - lo, 0), np.float32(hi - lo)) / dt) if first else 0.0
    cn = np.float32(c)
    s = float(cn > thr) if scale == "hard" else 0.5 * (1 + math.tanh((float(cn) - float(thr)) / rc.command_scale_width))
    assert abs(float(air[i]) - per * s) <= 2e-5 * max(1.0, per), (i, cases[i], float(air[i]), per * s)
    if scale == "hard" and c in (float(thr), tmk._ulp(thr, 1)) and per > 0:
      assert (float(air[i]) > 0) == (cn > thr), (i, cases[i])
    assert bool(done[i]) == dn, i
    if dn:
      for k in ("env.air_time", "env.contact_time", "env.last_air_time"):
        assert float(N[k][i].abs().max()) == 0.0, (k, i)
    else:
      assert float(N["env.air_time"][i, 0]) == float(new), i
      if first:
        assert float(N["env.last_air_time"][i, 0]) == float(np.float32(a)), i
  H.report(f"air time edges {mode} {scale}")
  env.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_episode_sums_and_reward_log(backend, monkeypatch):
  """finished_sums holds the sums of the episode a done env just ended (this step included) and episode_sums restarts
  at 0; reward_log() is their mean over the done envs over episode_length_s, NaN when no env ended."""
  H = _harness(backend, monkeypatch, robot="go1", num_envs=12, rewards=_all_on())
  env = H.env
  mx = env.max_episode_length
  rows = [dict(episode_length_buf=mx - 1) if i % 3 == 0 else dict() for i in range(12)]
  action, U = tmk._fill(H, rows)
  g = tmk._gen(env, 4)
  env.episode_sums.copy_(torch.rand(env.episode_sums.shape, generator=g, device=env.device))
  env.finished_sums.fill_(123.0)
  S, T, N = H.both(action, U)
  check(H, S, T, N, action, U, monkeypatch)
  done = N["out.truncated"]
  assert int(done.sum()) == 4
  for R in (T, N):
    assert float(R["env.episode_sums"][done].abs().max()) == 0.0
    assert bool((R["env.finished_sums"][~done] == 123.0).all())
    assert bool((R["env.finished_sums"][done] != S["env.episode_sums"][done]).any())
  log = env.reward_log()
  names = ("track_lin_vel_exp", "track_ang_vel_exp", "pose", "dof_pos_limits", "action_rate_l2") + NEW
  assert list(log) == [f"Episode_Reward/{t}" for t in names]
  want = N["env.finished_sums"][done].double().mean(0) / env.cfg.episode_length_s
  for i, t in enumerate(names):
    assert log[f"Episode_Reward/{t}"].device == env._done_buf.device
    assert abs(float(log[f"Episode_Reward/{t}"]) - float(want[i])) <= 1e-6 * max(1.0, abs(float(want[i]))), t
  # a step in which no env ends: NaN, as the mean over no envs is
  action, U = tmk._fill(H, [dict() for _ in range(12)])
  H.both(action, U)
  assert all(math.isnan(float(v)) for v in env.reward_log().values())
  env.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_rollout_workload_e_all_terms(backend, monkeypatch):
  """Workload E (Go1 rough, terrain curriculum) with every opt-in term on, 50 env steps (fewer on the host)."""
  big = backend == "cuda"
  H = _harness(backend, monkeypatch, robot="go1", terrain="rough", terrain_curriculum=True,
               num_envs=1024 if big else 4, decimation=4 if big else 1, push_interval_s=(0.02, 0.08),
               episode_length_s=0.5 if big else 0.03, rewards=_all_on(reward_mode="on_landing"))
  _rollout(H, 50 if big else 4, seed=5, monkeypatch=monkeypatch)
  H.report("workload E, all terms")
  assert H.counts["truncated"] > 0 and H.counts["in_band"] <= 2, H.counts
  H.env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 3, 130, 4096])
def test_world_counts(n, monkeypatch):
  H = _harness("cuda", monkeypatch, robot="go1", num_envs=n, fall_angle=0.3, episode_length_s=0.1,
               rewards=_all_on(reward_mode="continuous", threshold_min=0.0))
  _rollout(H, 8, seed=n, monkeypatch=monkeypatch)
  H.report(f"reward terms {n} envs")
  assert H.counts["truncated"] > 0, H.counts
  H.env.close()


# ---- configurations the env refuses ------------------------------------------------------------------------------
@pytest.mark.parametrize("bad, match", [
  (dict(air_time_sensor_names=("nope_contact",)), "unknown sensor"),
  (dict(feet_slide_geom_names=("FR_foot_collision", "FL_foot_collision", "RR_foot_collision", "nope")), "unknown geom"),
  (dict(foot_clearance_geom_names=("nope",)), "unknown geom"),
  (dict(feet_slide_geom_names=("FR_foot_collision",)), "one geom per sensor"),
  (dict(foot_clearance_geom_names=("FR_foot_collision",) * 33), "at most 32"),
  (dict(air_time_sensor_names=("FR_foot_ground_contact",) * 33), "at most 32"),
  (dict(reward_mode="sometimes"), "reward_mode"),
  (dict(command_scale_type="soft"), "command_scale_type"),
  (dict(foot_clearance=1.0, std=None), "target_height, std and tanh_mult"),
])
def test_invalid_configuration(bad, match, monkeypatch):
  import mjlab_b200.envs.velocity_env as ve

  tmk._patch_emul(monkeypatch, ve)
  with pytest.raises(ValueError, match=match):
    ve.VelocityFlatEnv(ve.VelocityEnvCfg(robot="go1", num_envs=2, rewards=_rewards(**bad)), device="cpu")


def test_sensor_without_found_is_refused(monkeypatch):
  """A contact sensor whose first data field is not 'found' (here: force only) cannot say whether a foot is down."""
  import mjlab_b200.envs.velocity_env as ve
  from mjlab_b200.asset_zoo import load_compiled

  tmk._patch_emul(monkeypatch, ve)
  m = load_compiled("go1_flat")
  intprm = np.array(m.arrays["sensor_intprm"]).copy()
  intprm[1, 0] = 2
  m.arrays["sensor_intprm"] = intprm
  with pytest.raises(ValueError, match="first data field is not 'found'"):
    ve.VelocityFlatEnv(ve.VelocityEnvCfg(robot="go1", num_envs=2), device="cpu", model=m)


def test_c_abi_layout(tmp_path):
  """The ctypes mirror of B2VelEnvArgs has the C struct's size and field offsets (the block is appended at the end)."""
  fields = [f[0] for f in native.B2VelEnvArgs._fields_]
  src = "#include <stdio.h>\n#include <stddef.h>\n#include \"b2sim.h\"\nint main(void) {\n"
  src += f'  printf("%zu\\n", sizeof(B2VelEnvArgs));\n'
  src += "".join(f'  printf("%zu\\n", offsetof(B2VelEnvArgs, {f}));\n' for f in fields) + "  return 0;\n}\n"
  (tmp_path / "layout.c").write_text(src)
  subprocess.check_call(["cc", "-I", str(ROOT / "include"), "-o", str(tmp_path / "layout"), str(tmp_path / "layout.c")])
  got = [int(x) for x in subprocess.check_output([str(tmp_path / "layout")]).split()]
  want = [ctypes.sizeof(native.B2VelEnvArgs)] + [getattr(native.B2VelEnvArgs, f).offset for f in fields]
  assert got == want

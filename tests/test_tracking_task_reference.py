"""The tracking torch path against the reference's own code, executed from oracle/_ref: the reward functions of
tasks/tracking/mdp/rewards.py and envs/mdp/rewards.py with non-default stds and weights, the termination functions of
tasks/tracking/mdp/terminations.py and envs/mdp/terminations.py with non-default thresholds, driven through
RewardManager.compute / reset and TerminationManager.compute / reset (a weight-0 term, a removed termination term), and
MotionCommand._update_metrics through CommandManager.reset, on saved states with terminations, time-outs and clip
restarts.  The managers and the command run as the reference's unbound methods on stand-in objects that hold the saved
state; nothing of this repository's formulas is restated here.  The fused kernels are held to the torch path by
tests/test_tracking_task.py."""

import importlib.util
import sys
import types
from pathlib import Path

import pytest
import torch

import refload
import test_mdp_kernels as tmk
import test_motion_clip
from mjlab_b200.envs import tracking_env as te

ROOT = Path(__file__).resolve().parents[1]


def _load(monkeypatch, name, *rel):
  spec = importlib.util.spec_from_file_location(name, refload.REF / "mjlab" / Path(*rel))
  mod = importlib.util.module_from_spec(spec)
  monkeypatch.setitem(sys.modules, name, mod)
  spec.loader.exec_module(mod)
  return mod


def _reference(monkeypatch):
  """(commands, tracking rewards, tracking terminations, envs rewards, envs terminations, managers) of the reference."""
  cmds = test_motion_clip._ref_commands(monkeypatch)  # (skips when the reference is not installed)
  for pkg in ("mjlab.tasks", "mjlab.tasks.tracking", "mjlab.tasks.tracking.mdp", "mjlab.envs.mdp"):
    if pkg not in sys.modules:
      mod = types.ModuleType(pkg)
      mod.__path__ = [str(refload.REF / Path(*pkg.split(".")))]
      monkeypatch.setitem(sys.modules, pkg, mod)
  tr = _load(monkeypatch, "mjlab.tasks.tracking.mdp.rewards", "tasks", "tracking", "mdp", "rewards.py")
  tt = _load(monkeypatch, "mjlab.tasks.tracking.mdp.terminations", "tasks", "tracking", "mdp", "terminations.py")
  er = _load(monkeypatch, "mjlab.envs.mdp.rewards", "envs", "mdp", "rewards.py")
  et = _load(monkeypatch, "mjlab.envs.mdp.terminations", "envs", "mdp", "terminations.py")
  from mjlab.managers.command_manager import CommandManager
  from mjlab.managers.reward_manager import RewardManager
  from mjlab.managers.termination_manager import TerminationManager

  return cmds, tr, tt, er, et, types.SimpleNamespace(cmd=CommandManager, rew=RewardManager, term=TerminationManager)


def _command(cmds, env, ts, pos, quat, lin, ang, jp, jv, rel_p, rel_q, metrics):
  """A MotionCommand of the reference holding one state: robot rows already gathered to the tracked bodies."""
  c = object.__new__(cmds.MotionCommand)
  n, nb = env.num_envs, len(te.BODY_NAMES)
  c.cfg = types.SimpleNamespace(body_names=list(te.BODY_NAMES), anchor_body_name="torso_link")
  c.motion = types.SimpleNamespace(**env.motion)
  c.time_steps = ts.clone()
  c._env = types.SimpleNamespace(scene=types.SimpleNamespace(env_origins=env.env_origins))
  c.robot = types.SimpleNamespace(data=types.SimpleNamespace(
    body_link_pos_w=pos, body_link_quat_w=quat, body_link_lin_vel_w=lin, body_link_ang_vel_w=ang, joint_pos=jp,
    joint_vel=jv))
  c.body_indexes = torch.arange(nb)
  c.robot_anchor_body_index = c.motion_anchor_body_index = env.anchor
  c.body_pos_relative_w, c.body_quat_relative_w = rel_p.clone(), rel_q.clone()
  c.metrics = {m: metrics[:, i].clone() for i, m in enumerate(te.METRICS)}
  c.command_counter = torch.zeros(n, dtype=torch.long)
  c._resample = lambda env_ids: None  # (the reset's resample is the state the torch path wrote; it is read back below)
  return c


def _robot(env, S, prefix):
  bid = env.robot.indexing.body_ids[env.body_idx].long()
  vel = S[prefix + "link_vel_w"][:, bid]
  return (S[prefix + "xpos"][:, bid], S[prefix + "xquat"][:, bid], vel[..., 0:3], vel[..., 3:6],
          S[prefix + "qpos"][:, 7:], S[prefix + "qvel"][:, 6:])


def _managers(ref, mods, env, S, action, command):
  """The reference's RewardManager and TerminationManager (their own compute / reset) on the saved state."""
  cmds, tr, tt, er, et = mods
  rc, tc = env.cfg.rewards, env.cfg.terminations
  n = env.num_envs
  pos, quat, lin, ang, jp, jv = _robot(env, S, "data.")
  asset = types.SimpleNamespace(sensor_names=["self_collision"], data=types.SimpleNamespace(
    joint_pos=jp, soft_joint_pos_limits=env.robot.soft_joint_pos_limits.expand(n, -1, -1),
    gravity_vec_w=env.robot.gravity_vec_w,
    sensor_data={"self_collision": S["data.sensordata"][:, env.self_collision_adr]}))
  renv = types.SimpleNamespace(
    command_manager=types.SimpleNamespace(get_term=lambda name: command), scene={"robot": asset},
    action_manager=types.SimpleNamespace(action=action, prev_action=S["env.last_action"]),
    episode_length_buf=S["env.episode_length_buf"] + 1, max_episode_length=env.max_episode_length,
    max_episode_length_s=env.cfg.episode_length_s)
  asset_cfg = types.SimpleNamespace(name="robot", joint_ids=slice(None))
  funcs = dict(motion_global_root_pos=tr.motion_global_anchor_position_error_exp,
               motion_global_root_ori=tr.motion_global_anchor_orientation_error_exp,
               motion_body_pos=tr.motion_relative_body_position_error_exp,
               motion_body_ori=tr.motion_relative_body_orientation_error_exp,
               motion_body_lin_vel=tr.motion_global_body_linear_velocity_error_exp,
               motion_body_ang_vel=tr.motion_global_body_angular_velocity_error_exp)
  cfgs = [types.SimpleNamespace(func=funcs[t], weight=getattr(rc, t),
                                params=dict(command_name="motion", std=getattr(rc, t + "_std"))) for t in te.TRACKING_TERMS]
  cfgs += [types.SimpleNamespace(func=er.action_rate_l2, weight=rc.action_rate_l2, params={}),
           types.SimpleNamespace(func=er.joint_pos_limits, weight=rc.joint_limit, params=dict(asset_cfg=asset_cfg)),
           types.SimpleNamespace(func=tr.self_collision_cost, weight=rc.self_collisions,
                                 params=dict(sensor_name="self_collision", asset_cfg=asset_cfg))]
  rm = types.SimpleNamespace(
    _env=renv, _term_names=list(te.REWARD_TERMS), _term_cfgs=cfgs, _class_term_cfgs=[],
    _reward_buf=torch.zeros(n), _step_reward=torch.zeros(n, len(cfgs)),
    _episode_sums={t: S["env.episode_sums"][:, i].clone() for i, t in enumerate(te.REWARD_TERMS)})
  reward = ref.rew.compute(rm, dt=env.step_dt).clone()
  tcfgs = {"time_out": types.SimpleNamespace(func=et.time_out, params={}, time_out=True)}
  if tc.anchor_pos is not None:
    tcfgs["anchor_pos"] = types.SimpleNamespace(func=tt.bad_anchor_pos_z_only, time_out=False,
                                                params=dict(command_name="motion", threshold=tc.anchor_pos))
  if tc.anchor_ori is not None:
    tcfgs["anchor_ori"] = types.SimpleNamespace(func=tt.bad_anchor_ori, time_out=False,
                                                params=dict(asset_cfg=asset_cfg, command_name="motion",
                                                            threshold=tc.anchor_ori))
  if tc.ee_body_pos is not None:
    tcfgs["ee_body_pos"] = types.SimpleNamespace(func=tt.bad_motion_body_pos_z_only, time_out=False,
                                                 params=dict(command_name="motion", threshold=tc.ee_body_pos,
                                                             body_names=list(te.EE_NAMES)))
  tm = types.SimpleNamespace(
    _env=renv, _term_names=list(tcfgs), _term_cfgs=list(tcfgs.values()), _class_term_cfgs=[],
    _truncated_buf=torch.zeros(n, dtype=torch.bool), _terminated_buf=torch.zeros(n, dtype=torch.bool),
    _term_dones={k: torch.zeros(n, dtype=torch.bool) for k in tcfgs})
  ref.term.compute(tm)
  return rm, reward, tm


def _close(a, b, rel=2e-5, floor=1e-6):
  a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
  assert a.shape == b.shape
  err = (a - b).abs() / torch.maximum(torch.maximum(a.abs(), b.abs()), torch.tensor(floor, dtype=torch.float64))
  assert float(err.max()) <= rel, (float(err.max()), a, b)


CFG = dict(rewards=te.TrackingRewardsCfg(motion_global_root_pos=0.7, motion_body_ori=0.0, motion_body_lin_vel=1.3,
                                         action_rate_l2=-0.3, joint_limit=-4.0, self_collisions=-2.0,
                                         motion_global_root_pos_std=0.2, motion_global_root_ori_std=0.7,
                                         motion_body_pos_std=0.15, motion_body_ori_std=0.5,
                                         motion_body_lin_vel_std=2.0, motion_body_ang_vel_std=1.5),
           terminations=te.TrackingTerminationsCfg(anchor_pos=0.2, anchor_ori=None, ee_body_pos=0.3))


@pytest.mark.parametrize("clip", ["synthetic", "motion_file"])
def test_torch_path_matches_reference_code(clip, monkeypatch, tmp_path):
  """Each step of a short rollout: the reward, every episode sum, the termination flags and the three logs of the
  torch path against the reference's managers, and the motion errors against MotionCommand._update_metrics at the
  reference's point of the step (before _update_command; a done env after its reset, against the stale targets)."""
  cmds, tr, tt, er, et, ref = _reference(monkeypatch)
  cfg = dict(num_envs=12, episode_length_s=0.1, push_interval_s=(0.02, 0.06), episode_logs=True, **CFG)
  if clip == "synthetic":
    cfg["clip_frames"] = 8
  else:
    cfg.update(motion_file=tmk._make_clip("emul", tmp_path, 120), adaptive_kernel_size=2, adaptive_alpha=0.3)
  H = tmk._tracking("emul", monkeypatch, **cfg)
  H.env_fields += ["episode_sums", "finished_sums", "term_flags", "motion_metrics", "finished_metrics"]
  env = H.env
  n, g = env.num_envs, tmk._gen(env, 29)
  seen = dict(ended=0, time_out=0, fell=0, restart=0, metric_rows=0)
  for k in range(8):
    act = torch.rand((n, env.nu), generator=g) * 2 - 1
    if k % 2 == 1:
      env.sim.data.qpos[k % 3::3, 2] -= 0.35
    if k % 3 == 2:
      env.time_steps[(k + 1) % 4::4] = env.T - 1
    tmk._pre(env, act)
    env.sim.step_n(env.cfg.decimation)
    U = env._rand(n, 48 + 4 * env.nu)
    S = H.snapshot()
    out = env._mdp_torch(act, U)
    T = H.snapshot()
    pos, quat, lin, ang, jp, jv = _robot(env, S, "data.")
    rel_p, rel_q = S["env.body_pos_relative_w"], S["env.body_quat_relative_w"]
    command = _command(cmds, env, S["env.time_steps"], pos, quat, lin, ang, jp, jv, rel_p, rel_q, S["env.motion_metrics"])
    rm, reward, tm = _managers(ref, (cmds, tr, tt, er, et), env, S, act, command)
    # terminations and the reward
    assert torch.equal(out[2], tm._terminated_buf) and torch.equal(out[3], tm._truncated_buf), k
    _close(out[1], reward, floor=1e-3 * env.step_dt)
    done = tm._terminated_buf | tm._truncated_buf
    ids = torch.nonzero(done).flatten()
    # the episode sums: a done env's sum is its finished one, every other env's runs on
    for i, t in enumerate(te.REWARD_TERMS):
      got = torch.where(done, T["env.finished_sums"][:, i], T["env.episode_sums"][:, i])
      _close(got, rm._episode_sums[t], floor=1e-4 * env.step_dt)
      if getattr(env.cfg.rewards, t) == 0.0:
        assert not bool(T["env.episode_sums"][:, i].any()) and not bool(T["env.finished_sums"][:, i].any())
    # the resets' logs: CommandManager.reset (the errors of the last update), RewardManager / TerminationManager.reset
    mgr = types.SimpleNamespace(_terms={"motion": command})
    if len(ids):
      logs = {**ref.cmd.reset(mgr, ids), **ref.rew.reset(rm, ids), **ref.term.reset(tm, ids)}
      ours = {**env.command_log(), **env.reward_log(), **env.termination_log()}
      ours = {k_: v for k_, v in ours.items() if "sampling_" not in k_}
      assert set(logs) == set(ours), set(logs) ^ set(ours)
      for k_, v in logs.items():
        _close(ours[k_], float(v), floor=1e-6), k_
      seen["ended"] += len(ids)
      seen["time_out"] += int(logs["Episode_Termination/time_out"])
      seen["fell"] += int(logs.get("Episode_Termination/anchor_pos", 0)) + int(logs.get("Episode_Termination/ee_body_pos", 0))
    else:
      assert all(torch.isnan(v) for v in env.reward_log().values())
    # _update_metrics where the reference runs it: after the reset and the forward, before _update_command.  A done
    # env: its reset state (the torch path's post-forward rows) at its start frame, the targets of the last update.
    # Not compared: an env reset onto the clip's last frame and restarted in the same step (written twice before the
    # one forward, DESIGN.md section 4.2)
    start = tmk._drawn_frames(env, S, U[:, 0])
    twice = done & (start + 1 >= env.T)
    seen["restart"] += int((T["env._done_buf"] & ~done).sum())
    post = _robot(env, T, "data.")
    d1 = done.view(-1, 1)
    mixed = [torch.where(d1.view(-1, *([1] * (a.dim() - 1))), b, a) for a, b in zip((pos, quat, lin, ang, jp, jv), post)]
    after = _command(cmds, env, torch.where(done, start, S["env.time_steps"]), *mixed, rel_p, rel_q,
                     torch.zeros(n, len(te.METRICS)))
    after._update_metrics()
    want = torch.stack([after.metrics[m] for m in te.METRICS], dim=1)
    rows = ~twice
    seen["metric_rows"] += int((rows & done).sum())
    _close(T["env.motion_metrics"][rows], want[rows], rel=1e-4, floor=1e-4)
  assert seen["ended"] > 0 and seen["time_out"] > 0 and seen["fell"] > 0 and seen["restart"] > 0, seen
  assert seen["metric_rows"] > 0, seen
  env.close()


@pytest.mark.parametrize("term", ["anchor_pos", "anchor_ori", "ee_body_pos"])
def test_terminations_at_thresholds_match_reference_code(term, monkeypatch):
  """Each termination alone (the others removed), its error below, exactly at and just across its non-default
  threshold: the torch path's flags against the reference's termination functions through TerminationManager."""
  import test_tracking_task as ttt

  cmds, tr, tt, er, et, ref = _reference(monkeypatch)
  terms = {t: (v if t == term else None) for t, v in ttt.THRESHOLDS.items()}
  H = tmk._tracking("emul", monkeypatch, num_envs=32, clip_frames=6, episode_length_s=1.0, episode_logs=True,
                    terminations=te.TrackingTerminationsCfg(**terms))
  H.env_fields += ["episode_sums", "term_flags", "motion_metrics"]
  env = H.env
  action, U, want = ttt.threshold_state(H, term)
  S = H.snapshot()
  out = env._mdp_torch(action, U)
  command = _command(cmds, env, S["env.time_steps"], *_robot(env, S, "data."), S["env.body_pos_relative_w"],
                     S["env.body_quat_relative_w"], S["env.motion_metrics"])
  _, _, tm = _managers(ref, (cmds, tr, tt, er, et), env, S, action, command)
  assert list(tm._term_dones) == ["time_out", term]
  assert torch.equal(out[2], tm._terminated_buf)
  assert torch.equal(env.term_flags[:, te.TERMINATION_TERMS.index(term)] != 0, tm._term_dones[term])
  assert [bool(tm._term_dones[term][r]) for r in want] == list(want.values())
  env.close()

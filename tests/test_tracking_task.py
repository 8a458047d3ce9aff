"""The tracking task as the reference's four G1 tracking tasks configure it: TrackingRewardsCfg, TrackingTerminationsCfg,
the RSI / push ranges, the two policy-group switches, tracking_task_cfg and the episode logs (reward_log,
termination_log, command_log).

* The presets against the reference's cfg classes (read through tests/ref_tracking_cfgs.py under tests/ref_runner.py).
* The fused kernels' configured terms and logs against the torch path on one saved state per step
  (test_mdp_kernels.Harness): emulated backend in the CPU suite, the H100 under -m gpu.
* The play tasks: never truncated, frame-0 starts without RSI offsets, no push, policy = critic on the shared terms.
* Refused configurations, the C ABI of the appended block.
"""

import ctypes
import json
import math
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import refload
import test_mdp_kernels as tmk
from mjlab_b200.envs import tracking_env as te
from mjlab_b200.sim import native

ROOT = Path(__file__).resolve().parents[1]
LOGS = "episode_sums finished_sums term_flags motion_metrics finished_metrics".split()
BACKENDS = tmk.BACKENDS


def _harness(backend, monkeypatch, **cfg):
  H = tmk._tracking(backend, monkeypatch, **cfg)
  H.env_fields += [f for f in LOGS]
  return H


def _compare(H, S, T, N):
  """Every output and every env tensor of the two paths on one saved state; a termination decided inside the float
  band of one path only is excluded row-wise (counted in H.counts["split"])."""
  env, tol = H.env, H.tol
  keep = T["out.terminated"] == N["out.terminated"]
  H.counts["split"] += int((~keep).sum())
  assert int((~keep).sum()) <= 2, "terminations differ in more than the band allows"
  for k in ("out.truncated", "env._done_buf", "env.time_steps", "env.episode_length_buf", "env.term_flags"):
    H.equal(k, T[k], N[k], keep)
  H.ulps("push_time_left", T["env.push_time_left"], N["env.push_time_left"], tol["fma_ulp"], keep)
  H.close("reward", T["out.reward"], N["out.reward"], keep, rowwise=False, floor=env.step_dt)
  loose = tol["kin"]
  for k in ("env.episode_sums", "env.finished_sums"):
    H.close(k, T[k], N[k], keep, floor=env.step_dt, rel=loose)
  for k in ("env.motion_metrics", "env.finished_metrics"):
    H.close(k, T[k], N[k], keep, floor=1.0, rel=loose)
  H.close("qpos", T["data.qpos"], N["data.qpos"], keep, floor=1.0)
  H.close("qvel", T["data.qvel"], N["data.qvel"], keep, floor=1.0, rel=loose)
  assert T["out.obs"].shape == N["out.obs"].shape == (env.num_envs, env.nobs)
  H.close("obs", T["out.obs"], N["out.obs"], keep, floor=1.0, rel=loose)
  H.close("critic", T["out.critic"], N["out.critic"], keep, floor=1.0, rel=loose)


def _rollout(H, steps, seed, drop_every=3):
  """Random actions, anchors dropped (terminations), clips run to their end (restarts), episodes near their limit."""
  env = H.env
  n, g = env.num_envs, tmk._gen(env, seed)
  env.episode_length_buf.copy_(torch.randint(0, env.max_episode_length, (n,), generator=g, device=env.device).int()
                               .clamp(max=max(env.max_episode_length - 1, 0)))
  for k in range(steps):
    act = torch.rand((n, env.nu), generator=g, device=env.device) * 2 - 1
    if k % drop_every == 1:
      env.sim.data.qpos[k % 4::4, 2] -= 0.4
    if k % drop_every == 2:
      env.time_steps[(k + 1) % 4::4] = env.T - 1
    tmk._pre(env, act)
    env.sim.step_n(env.cfg.decimation)
    U = env._rand(n, 48 + 4 * env.nu)
    S, T, N = H.both(act, U)
    _compare(H, S, T, N)
    H.counts["ended"] += int((N["env.term_flags"] != 0).any(1).sum())
    H.counts["done"] += int(N["env._done_buf"].sum())


R = te.TrackingRewardsCfg
K = te.TrackingTerminationsCfg
CASES = {
  "weights_and_stds": dict(rewards=R(motion_global_root_pos=0.7, motion_global_root_ori=0.2, motion_body_pos=1.5,
                                     motion_body_ori=0.6, motion_body_lin_vel=0.9, motion_body_ang_vel=1.3,
                                     action_rate_l2=-0.3, joint_limit=-4.0, self_collisions=-2.0,
                                     motion_global_root_pos_std=0.2, motion_global_root_ori_std=0.7,
                                     motion_body_pos_std=0.15, motion_body_ori_std=0.5, motion_body_lin_vel_std=2.0,
                                     motion_body_ang_vel_std=1.5)),
  "terminations": dict(terminations=K(anchor_pos=0.1, anchor_ori=None, ee_body_pos=0.3)),
  "terminations_removed": dict(terminations=K(anchor_pos=None, anchor_ori=0.5, ee_body_pos=None)),
  "ranges": dict(pose_range=((-0.1, 0.2), (0.0, 0.0), (-0.02, 0.03), (-0.2, 0.1), (0.0, 0.3), (-0.5, 0.5)),
                 velocity_range=((-1.0, 0.5), (0.0, 0.2), (-0.3, 0.3), (0.0, 0.0), (-0.2, 0.7), (-1.0, 1.0)),
                 push_velocity_range=((-0.2, 0.2), (-1.0, 0.0), (0.0, 0.0), (-0.3, 0.3), (-0.1, 0.1), (0.5, 0.9))),
  "no_push": dict(push_velocity_range=None),
  "no_state_estimation": dict(policy_state_estimation=False),
  "no_corruption": dict(policy_corruption=False),
  "logs_only": dict(episode_logs=True),
}
CASES.update({f"weight0_{t}": dict(rewards=R(**{t: 0.0})) for t in te.REWARD_TERMS})  # each term off alone


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("backend", BACKENDS)
def test_configured_terms_match_torch(backend, case, monkeypatch):
  big = backend == "cuda"
  cfg = dict(num_envs=1024 if big else 8, episode_length_s=0.3 if big else 0.06, clip_frames=30 if big else 6,
             push_interval_s=(0.05, 0.15) if big else (0.02, 0.06))
  cfg.update({"episode_logs": True, **CASES[case]})
  H = _harness(backend, monkeypatch, **cfg)
  assert all(getattr(H.env._native_args, f) for f in LOGS)
  _rollout(H, 30 if big else 5, seed=11)
  H.report(f"configured {case}")
  c = H.counts
  assert c["ended"] > 0 and c["done"] >= c["ended"], c
  if case.startswith("weight0_"):  # a term at weight 0 is not evaluated: its sums stay 0
    i = te.REWARD_TERMS.index(case[len("weight0_"):])
    assert not bool(H.env.episode_sums[:, i].any()) and not bool(H.env.finished_sums[:, i].any())
  H.env.close()


# ---- each termination term alone, at and just across its threshold ---------------------------------------------------
THRESHOLDS = dict(anchor_pos=0.125, anchor_ori=0.5, ee_body_pos=0.375)  # (dyadic: an fp32 difference can equal them)


def _f32_at(a, thr, sign):
  """(b, b_across): fp32 b near a + sign thr with fp32 |a - b| == thr exactly (None where the fp32 grid has no such
  b), and the next fp32 b beyond the threshold (|a - b| > thr)."""
  a, t = torch.tensor(a, dtype=torch.float32), torch.tensor(thr, dtype=torch.float32)
  step = torch.tensor(sign * math.inf, dtype=torch.float32)
  b = lo = a + sign * t
  for _ in range(8):
    lo = torch.nextafter(lo, -step)
  b, at = lo, None
  for _ in range(16):
    e = (a - b).abs()
    if e == t:
      at = float(b)
    if e > t:
      return at, float(b)
    b = torch.nextafter(b, step)
  raise AssertionError("no fp32 value across the threshold")


def threshold_state(H, term):
  """A base state (every env on its clip frame, all errors 0) with `term`'s error placed in rows 0.. at 1e-3 below,
  exactly at (fp32) and just across (next fp32) its THRESHOLDS value, each side; returns (action, U, {row: fires})."""
  env = H.env
  action, U = tmk._tracking_base(H)
  d, thr = env.sim.data, THRESHOLDS[term]
  bid = env.robot.indexing.body_ids[env.body_idx].long()
  anchor = int(bid[env.anchor])
  want, i = {}, 0
  if term in ("anchor_pos", "ee_body_pos"):
    for sign in (1.0, -1.0):
      for k in ([env.anchor] if term == "anchor_pos" else env.ee_idx.tolist()):
        if term == "anchor_pos":
          a = float(env.motion["body_pos_w"][env.time_steps[i], env.anchor, 2] + env.env_origins[i, 2])
        else:
          a = float(env.body_pos_relative_w[i, k, 2])
        at, across = _f32_at(a, thr, sign)
        for z, fires in ((a + sign * (thr - 1e-3), False), (at, False), (across, True)):
          if z is None:
            continue
          d.xpos[i, int(bid[k]), 2] = z
          want[i] = fires
          H.counts["exact"] += z is at
          i += 1
  else:  # gravity projection: tilt the anchor about x until the z difference is thr + dz (float64 bisection)
    from mjlab_b200.entity_data import quat_mul
    for dz in (-1e-3, -1e-5, 1e-5, 1e-3):
      a_quat = env.motion["body_quat_w"][env.time_steps[i], env.anchor].double()
      lo_, hi_ = 0.0, math.pi
      for _ in range(80):
        mid = 0.5 * (lo_ + hi_)
        tq = torch.tensor([math.cos(mid / 2), math.sin(mid / 2), 0.0, 0.0], dtype=torch.float64, device=env.device)
        q = quat_mul(a_quat[None], tq[None])[0]
        gz = lambda qq: -(1 - 2 * (qq[1] ** 2 + qq[2] ** 2))
        if abs(float(gz(a_quat) - gz(q))) > thr + dz:
          hi_ = mid
        else:
          lo_ = mid
      d.xquat[i, anchor] = q.float()
      want[i] = dz > 0
      i += 1
  return action, U, want


@pytest.mark.parametrize("removed", [False, True])
@pytest.mark.parametrize("term", list(THRESHOLDS))
@pytest.mark.parametrize("backend", BACKENDS)
def test_termination_term_alone_at_its_threshold(backend, term, removed, monkeypatch):
  """One termination term on (the others removed), its error at, below and just across its threshold: the flag and
  the decision on both paths; removed, it never fires."""
  terms = {t: (None if t != term or removed else v) for t, v in THRESHOLDS.items()}
  H = _harness(backend, monkeypatch, num_envs=32, clip_frames=6, episode_length_s=1.0, episode_logs=True,
               terminations=K(**terms))
  action, U, want = threshold_state(H, term)
  assert term == "anchor_ori" or H.counts["exact"] >= 1  # (an angle error cannot be placed on an fp32 value)
  S, T, N = H.both(action, U)
  _compare(H, S, T, N)
  col = te.TERMINATION_TERMS.index(term)
  for R in (T, N):
    for row, fires in want.items():
      assert bool(R["out.terminated"][row]) == (fires and not removed), (row, fires)
      assert float(R["env.term_flags"][row, col]) == float(fires and not removed), row
    assert not bool(R["out.terminated"][len(want):].any())
  keys = set(H.env.termination_log())
  assert (f"Episode_Termination/{term}" in keys) == (not removed)
  H.env.close()


@pytest.mark.parametrize("name", list(te.TRACKING_TASKS))
@pytest.mark.parametrize("backend", BACKENDS)
def test_presets_match_torch(backend, name, monkeypatch, tmp_path):
  """Each preset on a motion file with its own sampler (adaptive, or frame 0 in play)."""
  big = backend == "cuda"
  clip = tmk._make_clip(backend, tmp_path, 960 if big else 120)
  cfg = te.tracking_task_cfg(name, motion_file=clip, num_envs=512 if big else 6, adaptive_kernel_size=3,
                             adaptive_alpha=0.2)
  kw = {f: getattr(cfg, f) for f in cfg.__dataclass_fields__}
  H = _harness(backend, monkeypatch, **kw)
  if "Play" not in name:
    H.env.max_episode_length = 15  # (episodes short enough to time out in the rollout; the kernel's limit too)
    H.env._native_args.max_episode_length = 15
  _rollout(H, 20 if big else 4, seed=5)
  H.report(f"preset {name}")
  H.env.close()


def test_configured_path_at_reset_hands_over_logs(monkeypatch):
  """The logs of an episode end: the finished sums and errors move over, the sums restart, and the log methods report
  the means over the ended envs only (clip restarts excluded)."""
  H = _harness("emul", monkeypatch, num_envs=8, clip_frames=6, episode_length_s=1.0, episode_logs=True)
  env = H.env
  action, U = tmk._tracking_base(H)
  env.episode_sums.copy_(torch.rand(8, 9))
  env.motion_metrics.copy_(torch.rand(8, 10))
  before_sums, before_metrics = env.episode_sums.clone(), env.motion_metrics.clone()
  env.episode_length_buf[0] = env.max_episode_length - 1            # time out
  env.sim.data.xpos[1, int(env.robot.indexing.body_ids[env.body_idx][env.anchor]), 2] -= 0.4  # falls
  env.time_steps[2] = env.T - 1                                      # clip restart only
  S, T, N = H.both(action, U)
  _compare(H, S, T, N)
  for R in (T, N):
    ended = (R["env.term_flags"] != 0).any(1)
    assert ended.tolist() == [True, True] + [False] * 6
    assert bool(R["env._done_buf"][2])
    assert R["env.term_flags"][0].tolist() == [1.0, 0.0, 0.0, 0.0] and R["env.term_flags"][1, 1] == 1.0
    assert torch.equal(R["env.finished_metrics"][:2], before_metrics[:2])
    assert bool((R["env.episode_sums"][:2] == 0).all())
  H.close("finished sums", N["env.finished_sums"][:2], T["env.finished_sums"][:2], floor=1.0)
  assert bool((N["env.finished_sums"][:2] - before_sums[:2]).abs().max() < 1.0)
  log = env.reward_log()
  want = N["env.finished_sums"][:2].mean(0) / env.cfg.episode_length_s
  assert torch.allclose(torch.stack([log[f"Episode_Reward/{t}"] for t in te.REWARD_TERMS]), want)
  tl = env.termination_log()
  assert {k: float(v) for k, v in tl.items()} == {"Episode_Termination/time_out": 1.0, "Episode_Termination/anchor_pos": 1.0,
                                                  "Episode_Termination/anchor_ori": 0.0, "Episode_Termination/ee_body_pos": 0.0}
  cl = env.command_log()
  assert torch.allclose(torch.stack([cl[f"Metrics/motion/{t}"] for t in te.METRICS]), before_metrics[:2].mean(0))
  # (the errors a done env takes after the forward are held to the reference's _update_metrics in
  # tests/test_tracking_task_reference.py)
  env.term_flags.zero_()
  assert all(math.isnan(float(v)) for v in list(env.reward_log().values()) + list(env.termination_log().values()))
  env.close()


def test_play_never_truncates_and_starts_at_frame_zero(monkeypatch, tmp_path):
  clip = tmk._make_clip("emul", tmp_path, 120)
  cfg = te.tracking_task_cfg("Mjlab-Tracking-Flat-Unitree-G1-Play", motion_file=clip, num_envs=6)
  kw = {f: getattr(cfg, f) for f in cfg.__dataclass_fields__}
  H = _harness("emul", monkeypatch, **kw)
  env = H.env
  assert env.max_episode_length == te.INT32_MAX and env._native_args.max_episode_length == te.INT32_MAX
  env.episode_length_buf.fill_(te.INT32_MAX - 4)  # (3 steps: up to INT32_MAX - 1)
  ptl = env.push_time_left.clone()
  n, g = env.num_envs, tmk._gen(env, 3)
  for k in range(3):
    act = torch.rand((n, env.nu), generator=g) * 2 - 1
    env.sim.data.qpos[k::3, 2] -= 0.4  # some fall: their reset starts at frame 0, without RSI offsets
    tmk._pre(env, act)
    env.sim.step_n(env.cfg.decimation)
    U = env._rand(n, 48 + 4 * env.nu)
    S, T, N = H.both(act, U)
    _compare(H, S, T, N)
    for R in (T, N):
      assert not bool(R["out.truncated"].any())
      done = R["out.terminated"]
      H.counts["resets"] += int(done.sum())
      assert bool((R["env.time_steps"][done] == 1).all())
      root = env.motion["body_pos_w"][0, 0] + env.env_origins[done]
      assert torch.equal(R["data.qpos"][done, 0:3], root)
      assert torch.equal(R["env.push_time_left"], ptl)
      nu = env.nu
      pol, cr = R["out.obs"], R["out.critic"]
      ct = 2 * nu + 9 + 9 * len(te.BODY_NAMES)
      assert torch.equal(pol[:, :2 * nu + 9], cr[:, :2 * nu + 9])
      assert torch.equal(pol[:, 2 * nu + 9:2 * nu + 15], cr[:, ct:ct + 6])
      assert torch.equal(pol[:, 2 * nu + 15:], cr[:, ct + 6:])
  assert H.counts["resets"] > 0
  env.close()


def test_observation_switches_columns(monkeypatch):
  """Without state estimation the policy row is 5 nu + 9 wide in the reference's order, and each remaining noise
  column still moves only its own element, by its term's amplitude; the dropped terms' columns move nothing."""
  n_cols = 15 + 2 * 29
  H = _harness("emul", monkeypatch, num_envs=2 * n_cols, clip_frames=8, episode_length_s=1.0,
               policy_state_estimation=False)
  env = H.env
  nu = env.nu
  action, U = tmk._tracking_base(H)
  Z0 = 2 * (13 + nu) + 7
  amp = [0.25] * 3 + [0.05] * 6 + [0.5] * 3 + [0.2] * 3 + [0.01] * nu + [0.5] * nu
  dest = [None] * 3 + [2 * nu + k for k in range(6)] + [None] * 3 + [2 * nu + 6 + k for k in range(3)] + \
         [2 * nu + 9 + k for k in range(2 * nu)]
  vals = (0.0, tmk.BELOW_ONE)
  for c in range(n_cols):
    for k, v in enumerate(vals):
      U[2 * c + k, Z0 + c] = v
  S, T0, N0 = H.both(action, torch.full_like(U, 0.5))
  tmk._tracking_base(H)
  S, T, N = H.both(action, U)
  _compare(H, S, T, N)
  for R, R0 in ((T, T0), (N, N0)):
    assert R["out.obs"].shape[1] == 5 * nu + 9
    diff = (R["out.obs"] - R0["out.obs"]).double()
    for c in range(n_cols):
      for k, v in enumerate(vals):
        row = diff[2 * c + k].clone()
        if dest[c] is not None:
          want = (2.0 * np.float32(v) - 1.0) * amp[c]
          assert abs(float(row[dest[c]]) - want) <= 2e-6 * max(1.0, abs(float(R0["out.obs"][2 * c + k, dest[c]]))), c
          row[dest[c]] = 0.0
        assert float(row.abs().max()) == 0.0, (c, v)
  env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 5, 4096])
def test_preset_world_counts(n, monkeypatch):
  cfg = te.tracking_task_cfg("Mjlab-Tracking-Flat-Unitree-G1-No-State-Estimation", num_envs=n, clip_frames=12,
                             episode_length_s=0.1, push_interval_s=(0.02, 0.08))
  H = _harness("cuda", monkeypatch, **{f: getattr(cfg, f) for f in cfg.__dataclass_fields__})
  _rollout(H, 8, seed=n)
  H.report(f"preset {n} envs")
  H.env.close()


@pytest.mark.gpu
def test_logs_under_cuda_graph_replay():
  """The logs advance under replay of the captured step: the kernels write them through the captured pointers."""
  cfg = te.tracking_task_cfg("Mjlab-Tracking-Flat-Unitree-G1", num_envs=256, clip_frames=30, episode_length_s=0.1)
  env = te.TrackingFlatEnv(cfg, device="cuda:0")
  env.enable_cuda_graph()
  g = torch.Generator(device="cuda:0").manual_seed(0)
  seen = 0.0
  for _ in range(20):
    env.step(torch.rand((256, env.nu), generator=g, device="cuda:0") * 2 - 1)
    tl = env.termination_log()["Episode_Termination/time_out"]
    seen += float(torch.nan_to_num(tl, nan=0.0))
    rl = env.reward_log()
    if not math.isnan(float(rl["Episode_Reward/motion_body_pos"])):
      assert all(math.isfinite(float(v)) for v in rl.values())
      assert all(math.isfinite(float(v)) for v in env.command_log().values())
  assert seen >= 256
  env.close()


# ---- refusals -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [
  dict(rewards=R(motion_body_pos_std=0.0)), dict(rewards=R(motion_global_root_ori_std=-0.4)),
  dict(rewards=R(motion_body_lin_vel_std=math.inf)), dict(rewards=R(action_rate_l2=math.nan)),
  dict(terminations=K(anchor_pos=0.0)), dict(terminations=K(anchor_ori=-0.8)), dict(terminations=K(ee_body_pos=math.inf)),
  dict(terminations=K(anchor_pos=math.nan)),
  dict(pose_range=((0.1, -0.1),) + te.POSE_RANGE[1:]), dict(velocity_range=te.VELOCITY_RANGE[:5]),
  dict(push_velocity_range=te.VELOCITY_RANGE + ((0.0, 1.0),)), dict(push_velocity_range=((0.0, 1.0, 2.0),) * 6),
  dict(push_velocity_range=((1.0, 0.0),) * 6), dict(episode_length_s=0.0),
  dict(pose_range=(0.1, 0.2, 0.3, 0.4, 0.5, 0.6)), dict(velocity_range=(("a", "b"),) * 6), dict(pose_range=None),
])
def test_refused_configurations(kw):
  with pytest.raises(ValueError):
    te.TrackingEnvCfg(**kw)


def test_unknown_task_name_lists_the_known_ones():
  with pytest.raises(ValueError, match="Mjlab-Tracking-Flat-Unitree-G1-No-State-Estimation-Play"):
    te.tracking_task_cfg("Mjlab-Tracking-Rough-Unitree-G1")


def test_inconsistent_block_is_refused(monkeypatch):
  H = _harness("emul", monkeypatch, num_envs=2, clip_frames=4, episode_length_s=1.0, episode_logs=True)
  env = H.env
  A = env._native_args
  logs = {f: getattr(A, f) for f in LOGS}
  for nulls in (["term_flags"], ["finished_metrics"], LOGS[1:]):  # some log arrays set, some null
    for f in nulls:
      setattr(A, f, None)
    with pytest.raises(RuntimeError):
      env._mdp_native(torch.zeros(2, env.nu), torch.rand(2, 48 + 4 * env.nu))
    for f, p in logs.items():
      setattr(A, f, p)
  for arr, k, bad in (("std2", 3, 0.0), ("term_threshold", 1, -1.0), ("push_range", 0, 5.0)):
    keep = getattr(A, arr)[k]
    getattr(A, arr)[k] = bad
    with pytest.raises(RuntimeError):
      env._mdp_native(torch.zeros(2, env.nu), torch.rand(2, 48 + 4 * env.nu))
    getattr(A, arr)[k] = keep
  env._mdp_native(torch.zeros(2, env.nu), torch.rand(2, 48 + 4 * env.nu))  # restored: accepted
  env.close()


def test_log_methods_need_episode_logs(monkeypatch):
  H = _harness("emul", monkeypatch, num_envs=2, clip_frames=4)
  assert not any(getattr(H.env._native_args, f) for f in LOGS)
  for f in (H.env.reward_log, H.env.termination_log, H.env.command_log):
    with pytest.raises(RuntimeError):
      f()
  H.env.close()


def test_c_abi_layout(tmp_path):
  """The ctypes mirror of B2TrackEnvArgs has the C struct's size and field offsets (the block is appended at the end)."""
  fields = [f[0] for f in native.B2TrackEnvArgs._fields_]
  src = "#include <stdio.h>\n#include <stddef.h>\n#include \"b2sim.h\"\nint main(void) {\n"
  src += '  printf("%zu\\n", sizeof(B2TrackEnvArgs));\n'
  src += "".join(f'  printf("%zu\\n", offsetof(B2TrackEnvArgs, {f}));\n' for f in fields) + "  return 0;\n}\n"
  (tmp_path / "layout.c").write_text(src)
  subprocess.check_call(["cc", "-I", str(ROOT / "include"), "-o", str(tmp_path / "layout"), str(tmp_path / "layout.c")])
  got = [int(x) for x in subprocess.check_output([str(tmp_path / "layout")]).split()]
  want = [ctypes.sizeof(native.B2TrackEnvArgs)] + [getattr(native.B2TrackEnvArgs, f).offset for f in fields]
  assert got == want


# ---- presets against the reference's cfg classes ----------------------------------------------------------------------
def test_presets_match_reference_cfgs(tmp_path):
  if not refload.available():
    pytest.skip("the reference package is not installed (oracle/install_reference.py)")
  out = tmp_path / "cfgs.json"
  here = str(Path(__file__).parent)
  cmd = [sys.executable, str(Path(__file__).with_name("ref_runner.py")), "--rootdir", here, "--confcutdir", here,
         str(Path(__file__).with_name("ref_tracking_cfgs.py"))]
  r = subprocess.run(cmd, capture_output=True, text=True, cwd=tmp_path, timeout=900,
                     env=dict(os.environ, B2_TASK_CFGS=str(out)))
  assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
  ref = json.loads(out.read_text())
  assert set(ref) == set(te.TRACKING_TASKS)
  amp = dict(motion_anchor_pos_b=0.25, motion_anchor_ori_b=0.05, base_lin_vel=0.5, base_ang_vel=0.2, joint_pos=0.01,
             joint_vel=0.5)
  for name, want in ref.items():
    cfg = te.tracking_task_cfg(name)
    for t in te.REWARD_TERMS:
      assert getattr(cfg.rewards, t) == want["rewards"][t]["weight"], (name, t)
      if t in te.TRACKING_TERMS:
        assert getattr(cfg.rewards, t + "_std") == want["rewards"][t]["std"], (name, t)
    assert {t: getattr(cfg.terminations, t) for t in te.TERMINATION_TERMS[1:]} == want["terminations"], name
    assert want["time_out"]
    as_list = lambda r: None if r is None else [list(p) for p in r]
    assert as_list(cfg.pose_range) == want["pose_range"] and as_list(cfg.velocity_range) == want["velocity_range"], name
    assert as_list(cfg.push_velocity_range) == want["push"], name
    if want["push_interval_s"] is not None:
      assert list(cfg.push_interval_s) == want["push_interval_s"]
    assert list(cfg.joint_position_range) == want["joint_position_range"]
    pol = want["policy_terms"]
    dropped = {k for k, v in pol.items() if v is None and k in ("motion_anchor_pos_b", "base_lin_vel")}
    assert (not dropped) == cfg.policy_state_estimation and dropped in (set(), {"motion_anchor_pos_b", "base_lin_vel"})
    for k, a in amp.items():
      if k not in dropped:
        assert pol[k] == [-a, a], (name, k)
    assert pol["command"] is None and pol["actions"] is None
    assert cfg.policy_corruption == want["enable_corruption"], name
    assert cfg.disable_adaptive_sampling == want["disable_adaptive_sampling"], name
    assert cfg.episode_length_s == want["episode_length_s"] and cfg.decimation == want["decimation"], name
    assert list(te.BODY_NAMES) == want["body_names"] and want["anchor"] == "torso_link"
    assert list(te.EE_NAMES) == want["ee_body_names"]


@pytest.mark.parametrize("backend", BACKENDS)
def test_velocity_termination_log(backend, monkeypatch):
  """VelocityFlatEnv.termination_log on both paths: a time-out, a fall, both in one env, and NaN when none ended."""
  H = tmk._velocity(backend, monkeypatch, num_envs=8, episode_length_s=1.0)
  env = H.env
  n, dev = env.num_envs, env.device
  d = env.sim.data
  tilt = torch.tensor([math.cos(math.pi / 4), math.sin(math.pi / 4), 0.0, 0.0], device=dev)  # 90 deg: past fall_angle
  env.episode_length_buf.fill_(1)
  env.episode_length_buf[[0, 2]] = env.max_episode_length - 1  # time out: envs 0 and 2
  d.qpos[[1, 2], 3:7] = tilt                                   # fall: envs 1 and 2
  action, U = torch.zeros(n, env.nu, device=dev), torch.full((n, 16 + 9 + 2 * env.nu), 0.5, device=dev)
  snap = H.snapshot()
  for mdp in (env._mdp_torch, env._mdp_native):
    H.restore(snap)
    mdp(action, U)
    log = {k: float(v) for k, v in env.termination_log().items()}
    assert log == {"Episode_Termination/time_out": 2.0, "Episode_Termination/fell_over": 2.0}, (mdp.__name__, log)
  env.episode_length_buf.fill_(1)
  env._mdp_native(action, U)
  assert all(math.isnan(float(v)) for v in env.termination_log().values())
  env.close()

"""Clip, scale and history of the observation groups (mjlab_b200/envs/obs_history.py, csrc/b2_obshist.cuh).

* The torch path against the reference's own ObservationManager and CircularBuffer, executed from oracle/_ref: the
  reference's term functions return, at each step, the per-term frames the env's torch path computed (noise already
  in them, so the reference's noise is None); each step is ``reset(ids of reset_buf)`` then
  ``compute(update_history=True)``, as ``ManagerBasedRlEnv.step`` runs them.  Outputs must be equal: both sides do the
  same fp32 clamp and product and copy frames.
* b2_obs_history against the torch path on one saved post-physics state (the Harness of test_mdp_kernels.py), whose
  histories hold several distinct frames and which has envs in reset_buf and, for workload C, clip restarts outside
  it.  The expected output is the torch update of the saved history by the fused path's own frames and reset_buf, so
  it is bit-identical on both backends (a clamp, one IEEE product and copies).
* With default groups nothing new is launched and the env returns the buffers it returned before.
* Every refusal of the cfg, of the env and of the C entry, and the C layout of the argument block.
"""

import ctypes
import dataclasses
import subprocess
from pathlib import Path
from unittest.mock import Mock

import pytest
import torch

import refload
import test_mdp_kernels as tmk
from mjlab_b200.envs import ObservationsCfg, ObsGroupCfg
from mjlab_b200.envs import obs_history as oh
from mjlab_b200.envs import tracking_env as te
from mjlab_b200.envs import velocity_env as ve
from mjlab_b200.sim import native

ROOT = Path(__file__).resolve().parents[1]
GROUPS = oh.GROUPS
NB = len(te.BODY_NAMES)


def _configs(nu: int) -> dict:
  """The configurations every check runs: group-level H; mixed per-term H (0, 1, 4); clip on two terms; a scalar and a
  per-element scale (one of them on a clipped term, so the order clip -> scale shows); time-major history."""
  per_joint = tuple(0.05 * (k + 1) for k in range(nu))
  G = ObsGroupCfg
  return {
    "group_h3": ObservationsCfg(policy=G(history_length=3), critic=G(history_length=3)),
    "mixed_h": ObservationsCfg(policy=G(term_history={"base_ang_vel": 1, "joint_pos": 4, "actions": 0}),
                               critic=G(term_history={"joint_vel": 4, "base_ang_vel": 1, "joint_pos": 0})),
    "clip": ObservationsCfg(policy=G(clip={"joint_vel": (-1.0, 1.0), "base_ang_vel": (-0.3, 0.2)}),
                            critic=G(clip={"joint_vel": (-2.0, 0.5), "actions": (-0.5, 0.5)})),
    "scale": ObservationsCfg(policy=G(scale={"base_ang_vel": 0.25, "joint_pos": per_joint}, clip={"base_ang_vel": (-0.1, 0.1)},
                                      term_history={"joint_pos": 2}),
                             critic=G(scale={"joint_vel": 0.05, "actions": per_joint})),
    "time_major": ObservationsCfg(policy=G(history_length=2, flatten_history_dim=False, clip={"joint_vel": (-1.0, 1.0)}),
                                  critic=G(term_history={t: 3 for t in ve.OBS_TERMS + ("motion_anchor_pos_b",
                                           "motion_anchor_ori_b", "body_pos", "body_ori")}, flatten_history_dim=False,
                                           scale={"joint_pos": per_joint})),
  }


def _for(kind, cfg: ObservationsCfg, nu) -> ObservationsCfg:
  """cfg restricted to the terms of workload `kind` (the time-major critic names every term of both tasks)."""
  terms = _terms(kind, nu)
  out = {}
  for g in GROUPS:
    c = getattr(cfg, g)
    names = dict(terms[g])
    out[g] = dataclasses.replace(c, term_history={t: h for t, h in c.term_history.items() if t in names},
                                 clip={t: v for t, v in c.clip.items() if t in names},
                                 scale={t: v for t, v in c.scale.items() if t in names})
  return ObservationsCfg(**out)


def _terms(kind, nu):
  return {g: ve.obs_terms(nu) for g in GROUPS} if kind == "B" else te.obs_terms(nu, NB)


CONFIGS = list(_configs(1))  # (their names)


# ---- the torch path against the reference's ObservationManager -----------------------------------------------------
def _reference(monkeypatch):
  if not refload.available():
    pytest.skip("the reference package is not installed under oracle/_ref")
  monkeypatch.syspath_prepend(str(ROOT / "tests" / "stubs"))  # (prettytable stand-in)
  refload.load()
  from mjlab.managers.manager_term_config import ObservationGroupCfg, ObservationTermCfg
  from mjlab.managers.observation_manager import ObservationManager
  from mjlab.utils.buffers import CircularBuffer

  import mjlab.managers.observation_manager as om
  assert Path(om.__file__).resolve().is_relative_to(refload.REF.resolve())
  assert om.CircularBuffer is CircularBuffer
  return ObservationGroupCfg, ObservationTermCfg, ObservationManager


def _ref_manager(ref, cfg: ObservationsCfg, terms: dict, n: int, box: dict):
  """The reference's ObservationManager over the groups of `cfg`; term t of group g returns box[g][t]."""
  OGC, OTC, OM = ref

  def group(g):
    gc = getattr(cfg, g)
    fields = []
    for name, _ in terms[g]:
      kw = dict(func=lambda env, _g=g, _t=name: box[_g][_t].clone(), params={}, noise=None,
                history_length=gc.term_history.get(name, 0), flatten_history_dim=gc.flatten_history_dim)
      if name in gc.clip:
        kw["clip"] = tuple(gc.clip[name])
      if name in gc.scale:
        kw["scale"] = gc.scale[name]
      fields.append((name, OTC, dataclasses.field(default_factory=lambda kw=kw: OTC(**kw))))
    cls = dataclasses.make_dataclass(f"{g.title()}Cfg", fields, bases=(OGC,))
    return cls(history_length=gc.history_length, flatten_history_dim=gc.flatten_history_dim)

  cls = dataclasses.make_dataclass("ObsCfg", [(g, object, dataclasses.field(default_factory=lambda g=g: group(g)))
                                              for g in GROUPS])
  env = Mock()
  env.num_envs, env.device = n, "cpu"
  return OM(cls(), env)


def _split(frames: dict, terms: dict) -> dict:
  out = {}
  for g in GROUPS:
    k, out[g] = 0, {}
    for name, dim in terms[g]:
      out[g][name] = frames[g][:, k:k + dim].clone()
      k += dim
  return out


def _record_rollout(kind, monkeypatch, cfg, steps):
  """A torch-path rollout of workload `kind` on the host emulation with `cfg` as the env's observations: the frames
  and reset_buf every update saw, the env's outputs, and the clip restarts (C) outside reset_buf."""
  mod = ve if kind == "B" else te
  tmk._patch_emul(monkeypatch, mod)
  if kind == "B":
    env = ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=6, decimation=1, fall_angle=0.12, episode_length_s=0.04,
                                               push_interval_s=(0.005, 0.02), observations=cfg),
                             device="cpu", native_mdp=False)
  else:
    env = te.TrackingFlatEnv(te.TrackingEnvCfg(num_envs=6, decimation=1, clip_frames=7, episode_length_s=0.06,
                                               push_interval_s=(0.02, 0.06), observations=cfg),
                             device="cpu", native_mdp=False)
  seen = []
  update = env.obs_groups.update

  def record(frames, reset):
    seen.append(({g: f.clone() for g, f in frames.items()}, reset.clone()))
    return update(frames, reset)

  env.obs_groups.update = record
  r = env.reset()
  outs = [r if kind == "C" else (r, None)]  # (the velocity env's reset() returns the policy group only)
  restarts = 0
  g = torch.Generator().manual_seed(5)
  for _ in range(steps):
    act = torch.rand((env.num_envs, env.nu), generator=g) * 2 - 1
    obs, _, term, trunc, extras = env.step(act)
    outs.append((obs, extras["critic"]))
    if kind == "C":
      restarts += int((env._done_buf & ~(term | trunc)).sum())
  env.close()
  return seen, outs, restarts, env.nu


@pytest.mark.parametrize("kind", ["B", "C"])
def test_torch_path_matches_reference_manager(kind, monkeypatch):
  """64 env steps with resets (and clip restarts, C); the env runs the mixed configuration, every configuration is
  driven by the frames and reset_buf of that rollout."""
  ref = _reference(monkeypatch)
  seen, outs, restarts, nu = _record_rollout(kind, monkeypatch, _for(kind, _configs(1)["mixed_h"], 1), steps=64)
  terms = _terms(kind, nu)
  n = seen[0][1].shape[0]
  resets = sum(int(r.sum()) for _, r in seen[1:])
  assert resets >= 4 and (kind == "B" or restarts >= 2), (resets, restarts)
  for name, cfg in _configs(nu).items():
    cfg = _for(kind, cfg, nu)
    mine = oh.Observations(cfg, terms, n, "cpu")
    box = _split(seen[0][0], terms)
    ref_m = _ref_manager(ref, cfg, terms, n, box)
    for k, (frames, reset) in enumerate(seen):
      box.update(_split(frames, terms))
      ref_m.reset(None if k == 0 else torch.nonzero(reset).flatten())  # (k = 0: the env's reset())
      want = ref_m.compute(update_history=True)
      got = mine.update(frames, reset)
      for g in GROUPS:
        assert mine.groups[g].active
        assert got[g].shape == want[g].shape, (name, g, got[g].shape, want[g].shape)
        assert torch.equal(got[g], want[g]), (name, g, k)
      if name == "mixed_h":  # what the env built with this configuration returned
        pol, cri = outs[k]
        assert torch.equal(pol, got["policy"]), (name, k)
        assert cri is None or torch.equal(cri, got["critic"]), (name, k)


# ---- b2_obs_history against the torch path on one saved state ---------------------------------------------------------
class _Harness(tmk.Harness):
  """test_mdp_kernels' Harness that also saves and restores the groups' histories."""

  def snapshot(self):
    s = super().snapshot()
    s.update({"hist." + g: grp.out.clone() for g, grp in self.env.obs_groups.groups.items() if grp.active})
    return s

  def restore(self, snap):
    for k, v in snap.items():
      if k.startswith("hist."):
        self.env.obs_groups.groups[k[5:]].out.copy_(v)
    super().restore({k: v for k, v in snap.items() if not k.startswith("hist.")})


def _env(kind, backend, monkeypatch, cfg_name, n):
  nu = 29  # (G1 in both workloads)
  cfg = _for(kind, _configs(nu)[cfg_name], nu)
  if kind == "B":
    H = tmk._velocity(backend, monkeypatch, num_envs=n, decimation=1, fall_angle=0.12, episode_length_s=0.2,
                      observations=cfg)
    fields = tmk.VEL_ENV
  else:
    H = tmk._tracking(backend, monkeypatch, num_envs=n, decimation=1, clip_frames=9, episode_length_s=0.2,
                      observations=cfg)
    fields = tmk.TRK_ENV
  assert H.env.nu == nu
  return _Harness(H.env, backend, fields)


def _kernel_rollout(H, kind, steps, seed):
  """`steps` env steps of both paths from one saved state each; the fused path's output must be the torch update of
  the saved history by the fused path's own frames and reset_buf."""
  env = H.env
  n, g = env.num_envs, tmk._gen(env, seed)
  # every env times out once within the run, at a step of its own
  ep = env.max_episode_length - 1 - (torch.arange(n, device=env.device) * 7 + 2) % steps
  env.episode_length_buf.copy_(ep.int())
  counts = dict(reset=0, restart=0, kept=0)
  tmk._pre(env, torch.zeros(n, env.nu, device=env.device))
  env.sim.step_n(env.cfg.decimation)  # (a post-physics state; the steps below change it through resets and pushes)
  for k in range(steps):
    act = torch.rand((n, env.nu), generator=g, device=env.device) * 2 - 1
    if kind == "B":
      U = env._draw()
    else:
      U = env._rand(n, 48 + 4 * env.nu)
      if k % 3 == 2:  # clip restarts: some envs on the clip's last frame
        env.time_steps[k % 2::3] = env.T - 1
    S, T, N = H.both(act, U)
    reset = N["out.terminated"] | N["out.truncated"]
    counts["reset"] += int(reset.sum())
    counts["kept"] += int((~reset).sum())
    if kind == "C":
      counts["restart"] += int((N["env._done_buf"] & ~reset).sum())
    frames = {"policy": env._obs, "critic": env._critic}
    for grp_name, out in (("policy", "out.obs"), ("critic", "out.critic")):
      grp = env.obs_groups.groups[grp_name]
      post = grp.out.clone()
      grp.out.copy_(S["hist." + grp_name])
      want = grp.update(frames[grp_name], reset)
      grp.out.copy_(post)
      assert N[out].shape == want.shape == grp.shape, (grp_name, N[out].shape, want.shape)
      bad = N[out] != want
      assert not bool(bad.any()), (grp_name, k, int(bad.sum()), torch.nonzero(bad)[:4])
      assert T[out].shape == want.shape
  return counts


def _kernel_case(kind, backend, monkeypatch, cfg_name, n, steps=5):
  H = _env(kind, backend, monkeypatch, cfg_name, n)
  counts = _kernel_rollout(H, kind, steps, seed=n)
  assert counts["reset"] > 0 and counts["kept"] > 0, counts
  if kind == "C":
    assert counts["restart"] > 0, counts
  H.env.close()


@pytest.mark.parametrize("cfg_name", CONFIGS)
@pytest.mark.parametrize("kind", ["B", "C"])
@pytest.mark.parametrize("n", [1, 33])
def test_kernel_matches_torch_emul(kind, cfg_name, n, monkeypatch):
  _kernel_case(kind, "emul", monkeypatch, cfg_name, n, steps=5 if n > 1 else 12)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name", CONFIGS)
@pytest.mark.parametrize("kind", ["B", "C"])
@pytest.mark.parametrize("n", [1, 33, 4096])
def test_kernel_matches_torch_cuda(kind, cfg_name, n, monkeypatch):
  _kernel_case(kind, "cuda", monkeypatch, cfg_name, n, steps=6 if n > 1 else 16)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["B", "C"])
def test_kernel_under_graph_replay(kind):
  """The captured env step updates the histories: each replay's output is the torch update of the history before it
  by the frames and reset_buf the replay wrote."""
  nu, n = 29, 512
  cfg = _for(kind, _configs(nu)["scale"], nu)
  cfg.critic.history_length = 4
  if kind == "B":
    env = ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=n, fall_angle=0.12, episode_length_s=0.2, observations=cfg))
  else:
    env = te.TrackingFlatEnv(te.TrackingEnvCfg(num_envs=n, clip_frames=12, episode_length_s=0.2, observations=cfg))
  env.enable_cuda_graph()
  g = torch.Generator(device="cuda:0").manual_seed(3)
  resets = 0
  for _ in range(12):
    before = {grp: env.obs_groups.groups[grp].out.clone() for grp in GROUPS}
    obs, _, term, trunc, extras = env.step(torch.rand((n, env.nu), generator=g, device="cuda:0") * 2 - 1)
    got = {"policy": obs.clone(), "critic": extras["critic"].clone()}
    reset = term | trunc
    resets += int(reset.sum())
    for grp, frame in (("policy", env._obs), ("critic", env._critic)):
      G = env.obs_groups.groups[grp]
      post = G.out.clone()
      G.out.copy_(before[grp])
      assert torch.equal(G.update(frame, reset), got[grp]), grp
      G.out.copy_(post)
  assert resets > 0
  env.close()


# ---- default off ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["B", "C"])
def test_default_groups_launch_nothing_and_return_the_frames(kind, monkeypatch):
  """Default cfg: a step launches what it launched before and returns the post kernels' own buffers; a configured
  group adds exactly one launch for both groups."""
  launches = {}
  for name in ("default", "configured"):
    if name == "configured":
      H = _env(kind, "emul", monkeypatch, "mixed_h", 4)
    else:
      H = (tmk._velocity("emul", monkeypatch, num_envs=4, decimation=1) if kind == "B"
           else tmk._tracking("emul", monkeypatch, num_envs=4, decimation=1))
      assert H.env.cfg.observations == ObservationsCfg()
    env = H.env
    count = lambda: env.sim._lib.b2_launch_count(env.sim._h)  # noqa: E731
    act = torch.zeros(env.num_envs, env.nu)
    env.step(act)
    before = count()
    obs, _, _, _, extras = env.step(act)
    launches[name] = count() - before
    frame_w = 9 + 3 * env.nu + 3 if kind == "B" else 5 * env.nu + 15
    if name == "default":
      assert obs is env._obs and extras["critic"] is env._critic
      assert env.obs_groups._args is None and env.nobs == frame_w == obs.shape[1]
      assert env.nobs_critic == env._critic.shape[1]
      out = env._mdp_torch(act, env._draw() if kind == "B" else env._rand(env.num_envs, 48 + 4 * env.nu))
      assert out[0].shape == obs.shape and out[4]["critic"].shape == extras["critic"].shape
    else:
      assert obs.data_ptr() == env.obs_groups.groups["policy"].out.data_ptr()
      assert env.nobs == obs.shape[1] > frame_w and env.nobs_critic == extras["critic"].shape[1]
    env.close()
  assert launches["configured"] == launches["default"] + 1, launches


def test_output_widths():
  """nobs / the output shapes from the layout: flattened sum_t max(H_t, 1) D_t, time-major (H, sum D)."""
  terms = {g: ve.obs_terms(12) for g in GROUPS}
  cfg = ObservationsCfg(policy=ObsGroupCfg(term_history={"joint_pos": 4, "base_ang_vel": 1, "actions": 0}),
                        critic=ObsGroupCfg(history_length=5, flatten_history_dim=False))
  o = oh.Observations(cfg, terms, 3, "cpu")
  assert o.groups["policy"].shape == (3, 9 + 3 * 12 + 3 + 3 * 12)
  assert o.groups["critic"].shape == (3, 5, 9 + 3 * 12 + 3) and o.width("critic") == 5 * (9 + 3 * 12 + 3)
  # the layout: joint_pos's four frames follow projected_gravity, oldest first
  f = torch.arange(3 * (9 + 36 + 3), dtype=torch.float32).view(3, -1)
  o.fill({"policy": f, "critic": f})
  out = o.update({"policy": f + 1000, "critic": f + 1000}, torch.tensor([False, True, False]))
  p = out["policy"]
  jp = p[:, 9:9 + 48].view(3, 4, 12)
  assert torch.equal(jp[0, :3], f[0, 9:21].expand(3, 12)) and torch.equal(jp[0, 3], f[0, 9:21] + 1000)
  assert torch.equal(jp[1], (f[1, 9:21] + 1000).expand(4, 12))  # reset: backfilled
  assert torch.equal(p[:, 0:9], f[:, 0:9] + 1000) and torch.equal(p[:, 57:], f[:, 21:] + 1000)
  assert torch.equal(out["critic"][0, :4], f[0].expand(4, -1)) and torch.equal(out["critic"][0, 4], f[0] + 1000)


# ---- refusals ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [
  dict(history_length=-1), dict(history_length=2.0), dict(history_length=True), dict(history_length="3"),
  dict(term_history={"joint_pos": -2}), dict(term_history={"joint_pos": 1.5}), dict(flatten_history_dim=0),
  dict(clip={"joint_pos": (1.0, -1.0)}), dict(clip={"joint_pos": (-float("inf"), 1.0)}),
  dict(clip={"joint_pos": (0.0, float("nan"))}), dict(clip={"joint_pos": (0.0, 1e39)}), dict(clip={"joint_pos": 1.0}),
  dict(scale={"joint_pos": float("nan")}), dict(scale={"joint_pos": float("inf")}), dict(scale={"joint_pos": ()}),
  dict(scale={"joint_pos": (1.0, float("inf"))}), dict(scale={"joint_pos": "x"}), dict(clip=[("joint_pos", (0, 1))]),
])
def test_cfg_refusals(kw):
  with pytest.raises(ValueError):
    ObsGroupCfg(**kw)


@pytest.mark.parametrize("kw", [
  dict(term_history={"joint_position": 2}), dict(clip={"foot_height": (0.0, 1.0)}), dict(scale={"body_pos": 2.0}),
  dict(scale={"joint_pos": (1.0,) * 11}), dict(scale={"command": (1.0, 2.0)}),
  dict(flatten_history_dim=False), dict(flatten_history_dim=False, history_length=0),
  dict(flatten_history_dim=False, term_history={t: 2 for t in ve.OBS_TERMS[:-1]}),
  dict(flatten_history_dim=False, term_history={t: 2 if t != "actions" else 3 for t in ve.OBS_TERMS}),
])
def test_group_refusals(kw):
  """What only the group's terms decide: names, per-element scale lengths, a time-major group without one H >= 1."""
  with pytest.raises(ValueError):
    oh.Observations(ObservationsCfg(critic=ObsGroupCfg(**kw)), {g: ve.obs_terms(12) for g in GROUPS}, 2, "cpu")


def test_env_refusals(monkeypatch):
  """The envs refuse at build: the velocity groups have no body_pos, the tracking policy without state estimation has
  no base_lin_vel; a cfg edited after it was made is checked again."""
  tmk._patch_emul(monkeypatch, ve)
  tmk._patch_emul(monkeypatch, te)
  with pytest.raises(ValueError, match="unknown terms"):
    ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=2, observations=ObservationsCfg(
      critic=ObsGroupCfg(term_history={"body_pos": 2}))), device="cpu")
  with pytest.raises(ValueError, match="unknown terms"):
    te.TrackingFlatEnv(te.TrackingEnvCfg(num_envs=2, clip_frames=4, policy_state_estimation=False, observations=ObservationsCfg(
      policy=ObsGroupCfg(clip={"base_lin_vel": (-1.0, 1.0)}))), device="cpu")
  cfg = ObservationsCfg(policy=ObsGroupCfg(history_length=2))
  cfg.policy.history_length = -3
  with pytest.raises(ValueError, match="history_length"):
    ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=2, observations=cfg), device="cpu")
  # (with state estimation the same clip is fine)
  env = te.TrackingFlatEnv(te.TrackingEnvCfg(num_envs=2, clip_frames=4, observations=ObservationsCfg(
    policy=ObsGroupCfg(clip={"base_lin_vel": (-1.0, 1.0)}))), device="cpu")
  env.close()


def _bad_blocks(A):
  """(label, edit) of malformed argument blocks, each on a copy of the env's own."""
  def term(f):
    return lambda a: f(a.group[0].term[3])  # (joint_pos: two frames, scaled)
  return [
    ("null terminated", lambda a: setattr(a, "terminated", None)),
    ("null truncated", lambda a: setattr(a, "truncated", None)),
    ("no groups", lambda a: setattr(a, "ngroup", 0)),
    ("three groups", lambda a: setattr(a, "ngroup", 3)),
    ("null frame", lambda a: setattr(a.group[0], "frame", None)),
    ("null out", lambda a: setattr(a.group[1], "out", None)),
    ("no terms", lambda a: setattr(a.group[0], "nterm", 0)),
    ("too many terms", lambda a: setattr(a.group[0], "nterm", native.OBSHIST_NTERM + 1)),
    ("frame width off", lambda a: setattr(a.group[0], "frame_width", a.group[0].frame_width + 1)),
    ("out width short", lambda a: setattr(a.group[0], "out_width", a.group[0].out_width - 1)),
    ("out width long", lambda a: setattr(a.group[0], "out_width", a.group[0].out_width + 1)),
    ("negative H", term(lambda t: setattr(t, "frames", -1))),
    ("H beyond the row", term(lambda t: setattr(t, "frames", t.frames + 1))),
    ("terms not contiguous", term(lambda t: setattr(t, "src", t.src + 1))),
    ("zero dim", term(lambda t: setattr(t, "dim", 0))),
    ("overlapping frames", term(lambda t: setattr(t, "stride", t.stride - 1))),
    ("dst outside", term(lambda t: setattr(t, "dst", -1))),
    ("clip lo > hi", term(lambda t: (setattr(t, "clip", 1), setattr(t, "lo", 1.0), setattr(t, "hi", -1.0)))),
    ("clip not finite", term(lambda t: (setattr(t, "clip", 1), setattr(t, "lo", -float("inf")), setattr(t, "hi", 0.0)))),
    ("clip nan", term(lambda t: (setattr(t, "clip", 1), setattr(t, "lo", float("nan")), setattr(t, "hi", 0.0)))),
    ("clip flag", term(lambda t: setattr(t, "clip", 2))),
    ("scale outside the row", term(lambda t: setattr(t, "scale", A.nscale))),
    ("scale offset", term(lambda t: setattr(t, "scale", -2))),
    ("scale row null", lambda a: setattr(a, "scale", None)),
    ("scale row negative", lambda a: setattr(a, "nscale", -1)),
  ]


def test_c_entry_refusals(monkeypatch):
  """b2_obs_history refuses every malformed block before it launches (host emulation)."""
  H = _env("B", "emul", monkeypatch, "scale", 3)
  env, sim = H.env, H.env.sim
  A = env.obs_groups._args
  assert A is not None and A.ngroup == 2 and A.nscale > 0 and A.group[0].term[3].frames == 2
  call = lambda a: sim._lib.b2_obs_history(sim._h, ctypes.byref(a), None)  # noqa: E731
  assert call(A) == 0
  n0 = sim._lib.b2_launch_count(sim._h)
  for label, edit in _bad_blocks(A):
    a = native.B2ObsHistArgs.from_buffer_copy(A)
    edit(a)
    assert call(a) != 0, label
    assert b"b2_obs_history" in sim._lib.b2_last_error(), label
  assert sim._lib.b2_launch_count(sim._h) == n0
  assert sim._lib.b2_obs_history(None, ctypes.byref(A), None) != 0
  assert sim._lib.b2_obs_history(sim._h, None, None) != 0
  env.close()


def test_c_abi_layout(tmp_path):
  """The ctypes mirrors of B2ObsHistTerm, B2ObsHistGroup and B2ObsHistArgs have the C structs' sizes and offsets."""
  structs = (native.B2ObsHistTerm, native.B2ObsHistGroup, native.B2ObsHistArgs)
  src = "#include <stdio.h>\n#include <stddef.h>\n#include \"b2sim.h\"\nint main(void) {\n"
  want = []
  for S in structs:
    src += f'  printf("%zu\\n", sizeof({S.__name__}));\n'
    want.append(ctypes.sizeof(S))
    for f, _ in S._fields_:
      src += f'  printf("%zu\\n", offsetof({S.__name__}, {f}));\n'
      want.append(getattr(S, f).offset)
  src += '  printf("%d\\n%d\\n", B2_OBSHIST_NTERM, B2_OBSHIST_NGROUP);\n  return 0;\n}\n'
  want += [native.OBSHIST_NTERM, native.OBSHIST_NGROUP]
  (tmp_path / "layout.c").write_text(src)
  subprocess.check_call(["cc", "-I", str(ROOT / "include"), "-o", str(tmp_path / "layout"), str(tmp_path / "layout.c")])
  got = [int(x) for x in subprocess.check_output([str(tmp_path / "layout")]).split()]
  assert got == want

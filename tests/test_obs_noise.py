"""Per-term observation noise of the observation groups (mjlab_b200/envs/noise.py, envs/obs_history.py,
csrc/b2_obshist.cuh).

* The torch path against the reference's own ObservationManager, noise classes and noise models, executed from
  oracle/_ref.  The reference's term functions return the noise-free values the env read (the critic frame's columns),
  and its ``torch.rand_like`` / ``torch.randn_like`` (of ``mjlab.utils.noise.noise_cfg``) hand out the env's W and N
  columns in the order it asks for them.  Each step is ``reset(ids of reset_buf)`` then ``compute(update_history=True)``;
  the env's reset() is ``reset(all)`` then ``compute``.  Outputs and biases must be equal after every call.
* The default noise tables against the reference's cfg classes.
* b2_obs_history against the torch path on one saved state (test_mdp_kernels' Harness), from the fused path's own
  frames: outputs and bias state bit-identical.
* With default groups nothing is drawn or launched, and the env returns the post kernels' buffers.
* Every refusal of the cfg, the env and the C entry, and the C layout of the extended argument block.
"""

import ctypes
import dataclasses
import json
import os
import subprocess
import sys
import types
from pathlib import Path

import pytest
import torch

import refload
import test_mdp_kernels as tmk
import test_obs_history as toh
from mjlab_b200.envs import (ConstantNoiseCfg, GaussianNoiseCfg, NoiseModelCfg, NoiseModelWithAdditiveBiasCfg,
                             ObservationsCfg, ObsGroupCfg, UniformNoiseCfg)
from mjlab_b200.envs import noise as nz
from mjlab_b200.envs import obs_history as oh
from mjlab_b200.envs import tracking_env as te
from mjlab_b200.envs import velocity_env as ve
from mjlab_b200.sim import native

ROOT = Path(__file__).resolve().parents[1]
GROUPS = oh.GROUPS
NB = len(te.BODY_NAMES)
G = ObsGroupCfg
U, Gs, C = UniformNoiseCfg, GaussianNoiseCfg, ConstantNoiseCfg


def _per(nu, f):
  return tuple(float(f(k)) for k in range(nu))


def _configs(nu: int) -> dict:
  """Every configuration the checks run, on terms both tasks have (base_lin_vel, base_ang_vel: 3; joint_pos,
  joint_vel, actions: nu)."""
  bias_pc = NoiseModelWithAdditiveBiasCfg(noise_cfg=Gs(mean=0.01, std=0.05),
                                          bias_noise_cfg=U(n_min=-0.1, n_max=0.1))  # per component, add: accumulates
  bias_sh = NoiseModelWithAdditiveBiasCfg(noise_cfg=U(n_min=-0.02, n_max=0.03),
                                          bias_noise_cfg=Gs(mean=0.0, std=0.2, operation="abs"),
                                          sample_bias_per_component=False)
  return {
    # uniform: scalar bounds (double span), per-element bounds (fp32 span), each operation; the velocity critic is
    # corrupted (its inherited defaults and an override)
    "uniform": ObservationsCfg(
      policy=G(noise={"base_ang_vel": U(n_min=-0.3, n_max=0.2),
                      "joint_pos": U(n_min=_per(nu, lambda k: -0.01 * (k + 1)), n_max=0.37, operation="scale"),
                      "joint_vel": U(n_min=-1.1, n_max=0.7, operation="abs")}),
      critic=G(enable_corruption=True, noise={"actions": U(n_min=_per(nu, lambda k: -0.1 - k / 64),
                                                           n_max=_per(nu, lambda k: 0.3 + k / 32))})),
    "gaussian": ObservationsCfg(
      policy=G(noise={"base_ang_vel": Gs(mean=0.0, std=0.3),
                      "joint_pos": Gs(mean=_per(nu, lambda k: 1.0 + k / 100), std=_per(nu, lambda k: 0.1 + k / 50),
                                      operation="scale"),
                      "base_lin_vel": Gs(mean=-0.2, std=0.7, operation="abs")}),
      critic=G(enable_corruption=True, noise={"joint_vel": Gs(mean=0.1, std=1.3)})),
    "constant": ObservationsCfg(
      policy=G(noise={"base_ang_vel": C(bias=0.125), "joint_pos": C(bias=_per(nu, lambda k: 1 - k / 10),
                                                                    operation="scale"),
                      "joint_vel": C(bias=_per(nu, lambda k: -0.0 if k % 2 else k / 7), operation="abs"),
                      "actions": NoiseModelCfg(noise_cfg=C(bias=-0.5))})),
    # bias models: per component with an add bias over several episodes, shared with an abs bias, constant bias
    "bias": ObservationsCfg(
      policy=G(noise={"joint_pos": bias_pc, "base_ang_vel": bias_sh,
                      "actions": NoiseModelWithAdditiveBiasCfg(noise_cfg=C(bias=0.0), bias_noise_cfg=C(bias=0.25))}),
      critic=G(enable_corruption=True, noise={"joint_vel": NoiseModelWithAdditiveBiasCfg(
        noise_cfg=U(n_min=-0.5, n_max=0.5), bias_noise_cfg=U(n_min=-0.3, n_max=0.1),
        sample_bias_per_component=False)})),
    # corruption off on a policy group with overrides: no noise at all, the clean values
    "off": ObservationsCfg(policy=G(enable_corruption=False, noise={"joint_vel": Gs(mean=0.0, std=1.0)})),
    # the defaults re-expressed, one term's removed; noise with clip, scale and history
    "defaults": ObservationsCfg(policy=G(enable_corruption=True, noise={"joint_pos": None})),
    "history": ObservationsCfg(
      policy=G(history_length=3, clip={"base_ang_vel": (-0.2, 0.25), "joint_vel": (-1.0, 1.0)},
               scale={"joint_pos": _per(nu, lambda k: 0.5 + k / 10), "base_ang_vel": 0.25},
               noise={"base_ang_vel": Gs(mean=0.0, std=0.4), "joint_vel": bias_pc}),
      critic=G(term_history={"joint_pos": 2}, noise={"joint_vel": U(n_min=-0.5, n_max=0.5)})),
  }



def _terms(kind, nu):
  return {g: ve.obs_terms(nu) for g in GROUPS} if kind == "B" else te.obs_terms(nu, NB)


def _task_noise(kind, nu, policy_corruption=True):
  if kind == "B":
    return nz.TaskNoise(nz.velocity_defaults(), {"policy": True, "critic": False}, ve.obs_terms(nu))
  return nz.TaskNoise(nz.tracking_defaults(), {"policy": policy_corruption, "critic": False}, _terms("C", nu)["critic"])


# ---- recording -------------------------------------------------------------------------------------------------------
def _patch_recorder(monkeypatch):
  """Every Observations logs its draws (W, N after each) and updates (frames, reset, redraw, outputs) on `_log`."""
  draw, update = oh.Observations.draw, oh.Observations.update

  def rec_draw(self, rand, randn):
    draw(self, rand, randn)
    self.__dict__.setdefault("_log", []).append(
      ("draw", None if self.W is None else self.W.clone(), None if self.N is None else self.N.clone()))

  def rec_update(self, frames, reset, redraw=True):
    out = update(self, frames, reset, redraw)
    self.__dict__.setdefault("_log", []).append(
      ("update", {g: f.clone() for g, f in frames.items()}, reset.clone(), redraw, {g: o.clone() for g, o in out.items()},
       {g: None if self.groups[g].bias is None else self.groups[g].bias.clone() for g in GROUPS}))
    return out

  monkeypatch.setattr(oh.Observations, "draw", rec_draw)
  monkeypatch.setattr(oh.Observations, "update", rec_update)


def _events(log):
  """[(draws, frames, reset, first, outputs, biases)]: one per update, with the draws made since the previous one."""
  out, draws = [], []
  for item in log:
    if item[0] == "draw":
      draws.append(item[1:])
    else:
      out.append(dict(draws=draws, frames=item[1], reset=item[2], first=not item[3], out=item[4], bias=item[5]))
      draws = []
  return out


def _rollout_env(kind, monkeypatch, cfg, steps, policy_corruption=True):
  """A torch-path rollout of workload `kind` on the host emulation with `cfg` as the env's observations (a second
  reset() halfway); returns the env's Observations (its `_log`) and nu."""
  _patch_recorder(monkeypatch)
  mod = ve if kind == "B" else te
  tmk._patch_emul(monkeypatch, mod)
  if kind == "B":
    env = ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=6, decimation=1, fall_angle=0.12, episode_length_s=0.04,
                                               push_interval_s=(0.005, 0.02), observations=cfg),
                             device="cpu", native_mdp=False)
  else:
    env = te.TrackingFlatEnv(te.TrackingEnvCfg(num_envs=6, decimation=1, clip_frames=7, episode_length_s=0.06,
                                               push_interval_s=(0.02, 0.06), policy_corruption=policy_corruption,
                                               observations=cfg),
                             device="cpu", native_mdp=False)
  g = torch.Generator().manual_seed(5)
  restarts = 0
  for k in range(steps):
    if k == steps // 2:
      env.reset()
    act = torch.rand((env.num_envs, env.nu), generator=g) * 2 - 1
    obs, _, term, trunc, extras = env.step(act)
    log = env.obs_groups._log[-1]
    assert torch.equal(obs, log[4]["policy"]) and torch.equal(extras["critic"], log[4]["critic"])
    if kind == "C":
      restarts += int((env._done_buf & ~(term | trunc)).sum())
  env.close()
  if kind == "C":
    assert restarts >= 2, restarts
  return env.obs_groups, env.nu


# ---- the reference ---------------------------------------------------------------------------------------------------
def _reference(monkeypatch):
  ref = toh._reference(monkeypatch)
  import mjlab.utils.noise.noise_cfg as ncfg
  import mjlab.utils.noise.noise_model as nmod

  assert Path(ncfg.__file__).resolve().is_relative_to(refload.REF.resolve())
  assert Path(nmod.__file__).resolve().is_relative_to(refload.REF.resolve())
  queue = {"rand": [], "randn": []}

  def pop(kind):
    def f(data, *a, **k):
      assert queue[kind], f"torch.{kind}_like with no draw left"
      r = queue[kind].pop(0)
      assert r.shape == data.shape, (kind, r.shape, data.shape)
      return r.clone()
    return f

  fake = types.SimpleNamespace(**{k: getattr(torch, k) for k in dir(torch) if not k.startswith("__")})
  fake.rand_like, fake.randn_like = pop("rand"), pop("randn")
  monkeypatch.setattr(ncfg, "torch", fake)
  return ref, ncfg, queue


def _to_ref(c, R):
  """A fresh reference noise cfg equal to `c` (tuples become fp32 tensors, as a user would pass them)."""
  if c is None:
    return None
  if isinstance(c, NoiseModelWithAdditiveBiasCfg):
    return R.NoiseModelWithAdditiveBiasCfg(noise_cfg=_to_ref(c.noise_cfg, R), bias_noise_cfg=_to_ref(c.bias_noise_cfg, R),
                                           sample_bias_per_component=c.sample_bias_per_component)
  if isinstance(c, NoiseModelCfg):
    return R.NoiseModelCfg(noise_cfg=_to_ref(c.noise_cfg, R))
  kw = {k: torch.tensor(v, dtype=torch.float32) if isinstance(v, tuple) else v for k, v in c.params().items()}
  return getattr(R, type(c).__name__)(operation=c.operation, **kw)


def _ref_manager(ref, R, cfg, terms, n, box, task_noise, mine):
  """The reference's ObservationManager over `cfg` as a user would write it in the reference: the task's term noise,
  replaced by the cfg's entries, and the group's enable_corruption (the task's when not set).  A group `mine` does not
  noise-configure reads the env's frame, without noise."""
  OGC, OTC, OM = ref

  def group(g):
    gc = getattr(cfg, g)
    noisy = mine.groups[g].noisy
    fields = []
    for name, _ in terms[g]:
      noise = gc.noise[name] if name in gc.noise else task_noise.defaults[g].get(name)
      kw = dict(func=lambda env, _g=g, _t=name: box[_g][_t].clone(), params={},
                noise=_to_ref(noise, R) if noisy else None,
                history_length=gc.term_history.get(name, 0), flatten_history_dim=gc.flatten_history_dim)
      if name in gc.clip:
        kw["clip"] = tuple(gc.clip[name])
      if name in gc.scale:
        kw["scale"] = gc.scale[name]
      fields.append((name, OTC, dataclasses.field(default_factory=lambda kw=kw: OTC(**kw))))
    cls = dataclasses.make_dataclass(f"{g.title()}Cfg", fields, bases=(OGC,))
    on = gc.enable_corruption if gc.enable_corruption is not None else task_noise.corruption[g]
    return cls(history_length=gc.history_length, flatten_history_dim=gc.flatten_history_dim,
               enable_corruption=bool(on) and noisy)

  cls = dataclasses.make_dataclass("ObsCfg", [(g, object, dataclasses.field(default_factory=lambda g=g: group(g)))
                                              for g in GROUPS])
  env = types.SimpleNamespace(num_envs=n, device="cpu")
  return OM(cls(), env)


def _box(ev, terms, mine, task_noise):
  """{group: {term: values}} the reference's term functions return: the clean source columns of a noise-configured
  group, the frame of one that is not."""
  src = ev["frames"]["critic"]
  cols, c = {}, 0
  for name, dim in task_noise.source:
    cols[name], c = c, c + dim
  out = {}
  for g in GROUPS:
    out[g], k = {}, 0
    for name, dim in terms[g]:
      if mine.groups[g].noisy:
        out[g][name] = src[:, cols[name]:cols[name] + dim].clone()
      else:
        out[g][name] = ev["frames"][g][:, k:k + dim].clone()
      k += dim
  return out


def _block(d, W, N):
  return W if d.kind == nz.UNIFORM else N


def _feed(queue, ev, mine, n):
  """Queue the draws the reference asks for in this event, in its order: the bias models' reset (instances in term
  order, policy first), then compute term by term (a per-component bias's first reshape, then the noise)."""
  W, N = ev["draws"][0] if ev["draws"] else (None, None)
  ids = torch.arange(n) if ev["first"] else torch.nonzero(ev["reset"]).flatten()
  live = [(g, t) for g in GROUPS for t in mine.groups[g].terms if t.noise is not None]
  for g, t in live:
    d = t.noise.bias
    if d is not None and d.kind != nz.CONSTANT:
      q = "rand" if d.kind == nz.UNIFORM else "randn"
      queue[q].append(_block(d, W, N)[ids][:, d.col:d.col + (1 if ev["first"] else d.ndraw)])
  W, N = ev["draws"][-1] if ev["draws"] else (None, None)
  for g, t in live:
    for d, first_only in ((t.noise.bias, True), (t.noise.noise, False)):
      if d is None or d.kind == nz.CONSTANT or (first_only and (not ev["first"] or t.noise.shared)):
        continue
      queue["rand" if d.kind == nz.UNIFORM else "randn"].append(_block(d, W, N)[:, d.col:d.col + d.ndraw])


def _check_against_reference(ref, R, queue, cfg, mine, events, terms, task_noise, n, label):
  box = _box(events[0], terms, mine, task_noise)
  ref_m = _ref_manager(ref, R, cfg, terms, n, box, task_noise, mine)
  for k, ev in enumerate(events):
    box.update(_box(ev, terms, mine, task_noise))
    _feed(queue, ev, mine, n)
    ref_m.reset(None if ev["first"] else torch.nonzero(ev["reset"]).flatten())
    want = ref_m.compute(update_history=True)
    assert not queue["rand"] and not queue["randn"], (label, k, "draws left over")
    for g in GROUPS:
      assert torch.equal(ev["out"][g], want[g]), (label, g, k, (ev["out"][g] - want[g]).abs().max())
      grp = mine.groups[g]
      for t in grp.terms:
        if t.noise is None or t.noise.bias is None:
          continue
        rb = ref_m._group_obs_class_instances[t.name]._bias
        assert torch.equal(ev["bias"][g][:, t.src:t.src + t.dim], rb.expand(n, t.dim)), (label, g, t.name, k)


def _drive(cfg, kind, nu, events, task_noise, seed):
  """Run Observations(cfg) over the frames and reset_bufs of a recorded rollout, with draws of its own (the rollout's
  second reset() as reset() again); returns it, its log in hand."""
  mine = oh.Observations(cfg, _terms(kind, nu), events[0]["reset"].shape[0], "cpu", task_noise)
  g = torch.Generator().manual_seed(seed)
  rand = lambda *s: torch.rand(s, generator=g)  # noqa: E731
  randn = lambda *s: torch.randn(s, generator=g)  # noqa: E731
  for k, ev in enumerate(events):
    if k == 0 or ev["reset"].all():
      mine.fill(ev["frames"], rand, randn)
    else:
      mine.draw(rand, randn)
      mine.update(ev["frames"], ev["reset"])
  return mine


@pytest.mark.parametrize("kind", ["B", "C"])
def test_torch_path_matches_reference_noise(kind, monkeypatch):
  """64-step rollouts with resets (and clip restarts, C): the env's own outputs under the bias configuration, then
  every configuration driven by the rollout's frames and reset_bufs with draws of its own."""
  ref, R, queue = _reference(monkeypatch)
  nu0 = 29
  mine_env, nu = _rollout_env(kind, monkeypatch, _configs(nu0)["bias"], steps=64)
  assert nu == nu0
  terms, tn = _terms(kind, nu), _task_noise(kind, nu)
  events = _events(mine_env._log)
  n = events[0]["reset"].shape[0]
  resets = sum(int(ev["reset"].sum()) for ev in events[1:])
  assert events[0]["first"] and len(events[0]["draws"]) == 2 and resets >= 4 * n, resets
  assert sum(bool(ev["reset"].all()) for ev in events[1:]) >= 1  # (the second reset())
  _check_against_reference(ref, R, queue, _configs(nu)["bias"], mine_env, events, terms, tn, n, "env")
  for name, cfg in _configs(nu).items():
    mine = _drive(cfg, kind, nu, events, tn, seed=len(name))
    _check_against_reference(ref, R, queue, cfg, mine, _events(mine._log), terms, tn, n, name)
    if name == "off":
      for ev in _events(mine._log):  # the clean values
        assert torch.equal(ev["out"]["policy"], torch.cat([v for v in _box(ev, terms, mine, tn)["policy"].values()], 1))


def test_tracking_policy_corruption_off_matches_reference(monkeypatch):
  """The tracking policy with policy_corruption=False and enable_corruption=False: its overrides are dropped."""
  ref, R, queue = _reference(monkeypatch)
  cfg = ObservationsCfg(policy=G(enable_corruption=False, noise={"joint_vel": U(n_min=-2.0, n_max=2.0)}),
                        critic=G(enable_corruption=True, noise={"joint_pos": Gs(mean=0.0, std=0.1)}))
  mine, nu = _rollout_env("C", monkeypatch, cfg, steps=24, policy_corruption=False)
  tn = _task_noise("C", nu, policy_corruption=False)
  events = _events(mine._log)
  _check_against_reference(ref, R, queue, cfg, mine, events, _terms("C", nu), tn, events[0]["reset"].shape[0], "off")


# ---- the defaults against the reference's cfg classes ------------------------------------------------------------------
_REF_NOISE = '''
import json, os


def _noise(t):
  n = t.noise
  return None if n is None else [type(n).__name__, n.operation, float(n.n_min), float(n.n_max)]


def _groups(o):
  return {g: {"enable_corruption": getattr(o, g).enable_corruption,
              "terms": {k: _noise(v) for k, v in vars(getattr(o, g)).items() if hasattr(v, "func")}}
          for g in ("policy", "critic")}


def test_write_noise():
  from mjlab.tasks.velocity.velocity_env_cfg import ObservationCfg as V
  from mjlab.tasks.tracking.tracking_env_cfg import ObservationCfg as T
  with open(os.environ["B2_NOISE_CFGS"], "w") as f:
    json.dump({"velocity": _groups(V()), "tracking": _groups(T())}, f)
'''


def test_default_noise_matches_reference_cfgs(tmp_path):
  """The default tables and group corruption equal the reference's ObservationCfg classes of both tasks, and the four
  tracking tasks' policy noise and enable_corruption (tests/ref_tracking_cfgs.py)."""
  if not refload.available():
    pytest.skip("the reference package is not installed (oracle/install_reference.py)")
  here = str(Path(__file__).parent)
  (tmp_path / "ref_noise_cfgs.py").write_text(_REF_NOISE)
  env = dict(os.environ, B2_TASK_CFGS=str(tmp_path / "tasks.json"), B2_NOISE_CFGS=str(tmp_path / "noise.json"))
  cmd = [sys.executable, str(Path(__file__).with_name("ref_runner.py")), "--rootdir", here, "--confcutdir", here,
         str(Path(__file__).with_name("ref_tracking_cfgs.py")), str(tmp_path / "ref_noise_cfgs.py")]
  r = subprocess.run(cmd, capture_output=True, text=True, cwd=tmp_path, timeout=900, env=env)
  assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
  ref = json.loads((tmp_path / "noise.json").read_text())
  mine = {"velocity": (nz.velocity_defaults(), {"policy": True, "critic": False}, ve.obs_terms(29)),
          "tracking": (nz.tracking_defaults(), {"policy": True, "critic": False}, _terms("C", 29)["critic"])}
  for task, (defaults, corruption, terms) in mine.items():
    for g in GROUPS:
      want = ref[task][g]
      assert want["enable_corruption"] == corruption[g], (task, g)
      got = {t: None if t not in defaults[g] else ["UniformNoiseCfg", defaults[g][t].operation, defaults[g][t].n_min,
                                                   defaults[g][t].n_max] for t in want["terms"]}
      assert got == want["terms"], (task, g)
      assert set(want["terms"]) >= set(defaults[g]) and set(want["terms"]) <= {t for t, _ in terms}, (task, g)
  tasks = json.loads((tmp_path / "tasks.json").read_text())
  for name, want in tasks.items():
    cfg = te.tracking_task_cfg(name)
    assert want["enable_corruption"] == cfg.policy_corruption, name
    pol = nz.tracking_defaults()["policy"]
    for t, v in want["policy_terms"].items():
      if v is not None:
        assert (v == [pol[t].n_min, pol[t].n_max]) if t in pol else v is None, (name, t)
      elif t in pol:
        assert t in ("motion_anchor_pos_b", "base_lin_vel") and not cfg.policy_state_estimation, (name, t)


# ---- b2_obs_history against the torch path on one saved state --------------------------------------------------------
class _Harness(toh._Harness):
  """Also saves and restores the groups' bias state and the noise draws."""

  def snapshot(self):
    s = super().snapshot()
    s.update({"bias." + g: grp.bias.clone() for g, grp in self.env.obs_groups.groups.items() if grp.bias is not None})
    return s

  def restore(self, snap):
    for k, v in snap.items():
      if k.startswith("bias."):
        self.env.obs_groups.groups[k[5:]].bias.copy_(v)
    super().restore({k: v for k, v in snap.items() if not k.startswith("bias.")})


def _env(kind, backend, monkeypatch, cfg_name, n):
  nu = 29
  cfg = _configs(nu)[cfg_name]
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


def _expected(env, S, reset):
  """The torch update of the saved histories and biases by the fused path's own frames, reset_buf and draws; leaves
  the fused path's post-state in place."""
  O = env.obs_groups
  post = {g: (grp.out.clone(), None if grp.bias is None else grp.bias.clone()) for g, grp in O.groups.items() if grp.active}
  for g, (out, bias) in post.items():
    O.groups[g].out.copy_(S["hist." + g])
    if bias is not None:
      O.groups[g].bias.copy_(S["bias." + g])
  want = O.update({"policy": env._obs, "critic": env._critic}, reset)
  want_bias = {g: None if O.groups[g].bias is None else O.groups[g].bias.clone() for g in post}
  for g, (out, bias) in post.items():
    O.groups[g].out.copy_(out)
    if bias is not None:
      O.groups[g].bias.copy_(bias)
  return want, want_bias, {g: b for g, (_, b) in post.items()}


def _kernel_rollout(H, kind, steps, seed):
  env = H.env
  n, g = env.num_envs, tmk._gen(env, seed)
  ep = env.max_episode_length - 1 - (torch.arange(n, device=env.device) * 7 + 2) % steps
  env.episode_length_buf.copy_(ep.int())
  counts = dict(reset=0, restart=0, kept=0)
  tmk._pre(env, torch.zeros(n, env.nu, device=env.device))
  env.sim.step_n(env.cfg.decimation)
  for k in range(steps):
    act = torch.rand((n, env.nu), generator=g, device=env.device) * 2 - 1
    if kind == "B":
      U_ = env._draw()
    else:
      U_ = env._rand(n, 48 + 4 * env.nu)
      if k % 3 == 2:
        env.time_steps[k % 2::3] = env.T - 1
    env.obs_groups.draw(env._rand, env._randn)
    S, T, N = H.both(act, U_)
    reset = N["out.terminated"] | N["out.truncated"]
    counts["reset"] += int(reset.sum())
    counts["kept"] += int((~reset).sum())
    if kind == "C":
      counts["restart"] += int((N["env._done_buf"] & ~reset).sum())
    want, want_bias, got_bias = _expected(env, S, reset)
    for grp, key in (("policy", "out.obs"), ("critic", "out.critic")):
      bad = N[key] != want[grp]
      assert N[key].shape == want[grp].shape and not bool(bad.any()), (grp, k, int(bad.sum()), torch.nonzero(bad)[:4])
      assert T[key].shape == want[grp].shape
      if want_bias.get(grp) is not None:
        assert torch.equal(got_bias[grp], want_bias[grp]), (grp, k)
  return counts


KERNEL_CONFIGS = ["uniform", "gaussian", "constant", "bias", "history"]


def _kernel_case(kind, backend, monkeypatch, cfg_name, n, steps):
  H = _env(kind, backend, monkeypatch, cfg_name, n)
  counts = _kernel_rollout(H, kind, steps, seed=n)
  assert counts["reset"] > 0 and counts["kept"] > 0, counts
  if kind == "C":
    assert counts["restart"] > 0, counts
  H.env.close()


@pytest.mark.parametrize("cfg_name", KERNEL_CONFIGS)
@pytest.mark.parametrize("kind", ["B", "C"])
@pytest.mark.parametrize("n", [1, 33])
def test_kernel_matches_torch_emul(kind, cfg_name, n, monkeypatch):
  _kernel_case(kind, "emul", monkeypatch, cfg_name, n, steps=5 if n > 1 else 12)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name", KERNEL_CONFIGS)
@pytest.mark.parametrize("kind", ["B", "C"])
@pytest.mark.parametrize("n", [1, 33, 4096])
def test_kernel_matches_torch_cuda(kind, cfg_name, n, monkeypatch):
  _kernel_case(kind, "cuda", monkeypatch, cfg_name, n, steps=6 if n > 1 else 16)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["B", "C"])
def test_kernel_under_graph_replay(kind):
  """The captured env step draws W and N and updates outputs and biases: each replay's result is the torch update of
  the state before it by the frames, reset_buf and draws the replay wrote."""
  nu, n = 29, 512
  cfg = _configs(nu)["bias"]
  cfg.policy.history_length = 2
  if kind == "B":
    env = ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=n, fall_angle=0.12, episode_length_s=0.2, observations=cfg))
  else:
    env = te.TrackingFlatEnv(te.TrackingEnvCfg(num_envs=n, clip_frames=12, episode_length_s=0.2, observations=cfg))
  env.enable_cuda_graph()
  O = env.obs_groups
  g = torch.Generator(device="cuda:0").manual_seed(3)
  resets, draws = 0, set()
  for _ in range(12):
    S = {"hist." + k: grp.out.clone() for k, grp in O.groups.items()}
    S.update({"bias." + k: grp.bias.clone() for k, grp in O.groups.items() if grp.bias is not None})
    obs, _, term, trunc, extras = env.step(torch.rand((n, env.nu), generator=g, device="cuda:0") * 2 - 1)
    got = {"policy": obs.clone(), "critic": extras["critic"].clone()}
    reset = term | trunc
    resets += int(reset.sum())
    draws.add(float(O.W.sum()) + float(O.N.sum()))
    want, want_bias, got_bias = _expected(env, S, reset)
    for grp in GROUPS:
      assert torch.equal(want[grp], got[grp]), grp
      if want_bias[grp] is not None:
        assert torch.equal(want_bias[grp], got_bias[grp]), grp
  assert resets > 0 and len(draws) == 12  # (fresh draws every replay)
  env.close()


# ---- default off ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["B", "C"])
def test_defaults_draw_and_launch_nothing(kind, monkeypatch):
  """Default groups: no W or N (the generator ends a step where an env whose noise draws nothing ends it), the
  launches of before, and the post kernels' own buffers; a random term draws, and adds the one launch."""
  states, launches = {}, {}
  for name, cfg in (("default", ObservationsCfg()),
                    ("constant", ObservationsCfg(critic=G(enable_corruption=False, noise={"actions": C(bias=0.5)}))),
                    ("random", ObservationsCfg(policy=G(noise={"joint_vel": Gs(mean=0.0, std=1.0)})))):
    if kind == "B":
      H = tmk._velocity("emul", monkeypatch, num_envs=4, decimation=1, observations=cfg)
    else:
      H = tmk._tracking("emul", monkeypatch, num_envs=4, decimation=1, observations=cfg)
    env = H.env
    count = lambda: env.sim._lib.b2_launch_count(env.sim._h)  # noqa: E731
    act = torch.zeros(env.num_envs, env.nu)
    env.step(act)
    before = count()
    obs, _, _, _, extras = env.step(act)
    launches[name] = count() - before
    states[name] = env.gen.get_state()
    if name == "default":
      assert env.obs_groups.W is None and env.obs_groups.N is None and not env.obs_groups.noisy
      assert obs is env._obs and extras["critic"] is env._critic and env.obs_groups._args is None
    else:
      noisy = "critic" if name == "constant" else "policy"
      out = obs if noisy == "policy" else extras["critic"]
      assert out.data_ptr() == env.obs_groups.groups[noisy].out.data_ptr() and env.obs_groups.noisy == [noisy]
      assert (env.obs_groups.N is None) == (env.obs_groups.W is None) == (name == "constant")
    env.close()
  assert torch.equal(states["default"], states["constant"]) and not torch.equal(states["default"], states["random"])
  assert launches["constant"] == launches["random"] == launches["default"] + 1, launches


def test_uniform_span_roundings():
  """A scalar range's span is the double n_max - n_min rounded once; per-element bounds give the fp32 difference of
  the fp32 bounds.  For (-0.02, 0.03) they differ in the last bit, and each matches what torch computes."""
  d_scalar = nz.Draw(U(n_min=-0.02, n_max=0.03), 1, "cpu")
  d_tuple = nz.Draw(U(n_min=(-0.02,), n_max=(0.03,)), 1, "cpu")
  s64 = torch.tensor(0.03 - -0.02, dtype=torch.float32)
  s32 = torch.tensor(0.03, dtype=torch.float32) - torch.tensor(-0.02, dtype=torch.float32)
  assert not torch.equal(s64, s32)
  assert torch.equal(d_scalar.p1[0], s64) and torch.equal(d_tuple.p1[0], s32)
  u = torch.rand(4096, 1, generator=torch.Generator().manual_seed(1))
  x = torch.zeros(4096, 1)
  assert torch.equal(d_scalar.apply(x, u), x + (u * (0.03 - -0.02) + -0.02))
  lo, hi = torch.tensor([-0.02]), torch.tensor([0.03])
  assert torch.equal(d_tuple.apply(x, u), x + (u * (hi - lo) + lo))


# ---- refusals ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("make", [
  lambda: U(n_min=0.5, n_max=0.5), lambda: U(n_min=1.0, n_max=-1.0), lambda: U(n_min=(0.0, 1.0), n_max=(1.0, 1.0)),
  lambda: U(n_min=(0.0, 2.0), n_max=1.0), lambda: Gs(std=0.0), lambda: Gs(std=(1.0, -1.0)), lambda: Gs(mean=float("nan")),
  lambda: C(bias=float("inf")), lambda: C(bias=1e39), lambda: U(n_min=-1.0, n_max=(1.0, 1e40)), lambda: C(bias=()),
  lambda: C(bias="x"), lambda: C(bias=True), lambda: U(operation="mul"), lambda: Gs(operation=None),
  lambda: NoiseModelWithAdditiveBiasCfg(noise_cfg=U()), lambda: NoiseModelCfg(noise_cfg=0.1),
  lambda: NoiseModelWithAdditiveBiasCfg(noise_cfg=U(), bias_noise_cfg=C(bias=(0.1, 0.2))),
  lambda: NoiseModelWithAdditiveBiasCfg(noise_cfg=U(), bias_noise_cfg=U(), sample_bias_per_component=1),
  lambda: G(noise={"joint_pos": 0.1}), lambda: G(noise={"joint_pos": "uniform"}), lambda: G(enable_corruption=1),
  lambda: G(noise=[("joint_pos", U())]), lambda: G(noise={"joint_pos": types.SimpleNamespace(operation="add")}),
])
def test_cfg_refusals(make):
  with pytest.raises(ValueError):
    make()


def test_cfg_refuses_an_edited_class():
  c = U(n_min=-1.0, n_max=1.0)
  c.operation = "abs "
  with pytest.raises(ValueError, match="operation"):
    G(noise={"joint_pos": c})
  c = Gs()
  c.std = -1.0
  with pytest.raises(ValueError, match="std"):
    G(noise={"joint_pos": c})


@pytest.mark.parametrize("kw", [
  dict(noise={"joint_position": U()}), dict(noise={"body_pos": U()}), dict(noise={"joint_pos": U(n_min=(0.0,) * 11)}),
  dict(noise={"base_ang_vel": Gs(std=(1.0, 1.0))}), dict(noise={"actions": C(bias=(1.0,) * 13)}),
])
def test_group_refusals(kw):
  with pytest.raises(ValueError):
    oh.Observations(ObservationsCfg(critic=G(**kw)), {g: ve.obs_terms(12) for g in GROUPS}, 2, "cpu",
                    _task_noise("B", 12))


def test_env_refusals(monkeypatch):
  """The envs refuse at build: unknown terms, the tracking policy's enable_corruption against policy_corruption (also
  after an edit), and a bias model on one term in both groups."""
  tmk._patch_emul(monkeypatch, ve)
  tmk._patch_emul(monkeypatch, te)
  with pytest.raises(ValueError, match="unknown terms"):
    ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=2, observations=ObservationsCfg(critic=G(noise={"body_pos": U()}))),
                       device="cpu")
  with pytest.raises(ValueError, match="unknown terms"):
    te.TrackingFlatEnv(te.TrackingEnvCfg(num_envs=2, clip_frames=4, policy_state_estimation=False,
                                         observations=ObservationsCfg(policy=G(noise={"base_lin_vel": U()}))),
                       device="cpu")
  with pytest.raises(ValueError, match="contradicts"):
    te.TrackingEnvCfg(policy_corruption=False, observations=ObservationsCfg(policy=G(enable_corruption=True)))
  with pytest.raises(ValueError, match="contradicts"):
    te.TrackingEnvCfg(observations=ObservationsCfg(policy=G(enable_corruption=False)))
  cfg = te.TrackingEnvCfg(num_envs=2, clip_frames=4)
  cfg.observations.policy.enable_corruption = False
  with pytest.raises(ValueError, match="contradicts"):
    te.TrackingFlatEnv(cfg, device="cpu")
  bias = NoiseModelWithAdditiveBiasCfg(noise_cfg=U(), bias_noise_cfg=U())
  with pytest.raises(ValueError, match="both groups"):
    ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=2, observations=ObservationsCfg(
      policy=G(noise={"joint_pos": bias}), critic=G(enable_corruption=True, noise={"joint_pos": bias}))), device="cpu")
  cfg = ObservationsCfg(policy=G(noise={"joint_pos": U()}))
  cfg.policy.noise["joint_pos"] = U(n_min=(0.0,) * 3, n_max=1.0)  # (edited after it was made: checked again)
  with pytest.raises(ValueError, match="elements"):
    ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=2, observations=cfg), device="cpu")
  env = te.TrackingFlatEnv(te.TrackingEnvCfg(num_envs=2, clip_frames=4, observations=ObservationsCfg(
    policy=G(enable_corruption=True, noise={"base_lin_vel": Gs()}))), device="cpu")
  env.close()


def _bad_blocks(A):
  """(label, edit) of malformed noise blocks, each on a copy of the env's own ("bias" configuration, velocity: policy
  base_ang_vel (term 1) a uniform noise with a shared gaussian bias, joint_pos (term 3) gaussian with a uniform bias,
  actions (term 5) constant with a constant bias; critic joint_vel (term 4) uniform with a shared uniform bias)."""
  def term(g, k, f):
    return lambda a: f(a.noise[g].term[k])
  return [
    ("unknown noise class", term(0, 3, lambda t: setattr(t, "noise", 4))),
    ("negative noise class", term(0, 3, lambda t: setattr(t, "noise", -1))),
    ("unknown noise op", term(0, 3, lambda t: setattr(t, "noise_op", 3))),
    ("unknown bias class", term(0, 3, lambda t: setattr(t, "bias", 7))),
    ("unknown bias op", term(0, 1, lambda t: setattr(t, "bias_op", -1))),
    ("bias_shared flag", term(0, 1, lambda t: setattr(t, "bias_shared", 2))),
    ("source column negative", term(0, 0, lambda t: setattr(t, "col", -1))),
    ("source column past the row", term(0, 6, lambda t: setattr(t, "col", t.col + 1))),
    ("noisy source column past the row", term(0, 3, lambda t: setattr(t, "col", A.noise[0].source_width))),
    ("source width short", lambda a: setattr(a.noise[1], "source_width", a.noise[1].source_width - 1)),
    ("no source", lambda a: setattr(a.noise[0], "source", None)),
    ("no bias row", lambda a: setattr(a.noise[1], "bias", None)),
    ("no W", lambda a: setattr(a, "W", None)),
    ("no N", lambda a: setattr(a, "N", None)),
    ("no param", lambda a: setattr(a, "param", None)),
    ("param p0 outside", term(0, 3, lambda t: setattr(t, "noise_p0", A.nparam - 1))),
    ("param p1 negative", term(0, 3, lambda t: setattr(t, "noise_p1", -1))),
    ("bias param outside", term(0, 5, lambda t: setattr(t, "bias_p0", A.nparam))),
    ("noise draw outside W", term(0, 1, lambda t: setattr(t, "noise_draw", A.nW - 1))),
    ("noise draw outside N", term(0, 3, lambda t: setattr(t, "noise_draw", A.nN - 1))),
    ("bias draw outside", term(1, 4, lambda t: setattr(t, "bias_draw", A.nW))),
    ("per-element bias draws outside", term(1, 4, lambda t: (setattr(t, "bias_shared", 0),
                                                             setattr(t, "bias_draw", A.nW - 1)))),
    ("negative draw", term(0, 1, lambda t: setattr(t, "noise_draw", -1))),
    ("nW negative", lambda a: setattr(a, "nW", -1)),
    ("nparam negative", lambda a: setattr(a, "nparam", -1)),
    ("a code without a source", lambda a: (setattr(a.noise[0], "source", None), setattr(a.noise[0].term[0], "noise", 1),
                                           setattr(a.noise[0].term[0], "noise_p0", 0))),
  ]


def test_c_entry_refusals(monkeypatch):
  """b2_obs_history refuses every malformed noise block before it launches (host emulation)."""
  H = _env("B", "emul", monkeypatch, "bias", 3)
  env, sim = H.env, H.env.sim
  A = env.obs_groups._args
  Z = A.noise
  assert A.ngroup == 2 and Z[0].term[3].noise == native.NOISE_GAUSSIAN and Z[0].term[3].bias == native.NOISE_UNIFORM
  assert Z[0].term[1].bias_shared == 1 and Z[0].term[5].noise == native.NOISE_CONSTANT and Z[1].term[4].bias_shared == 1
  assert Z[0].term[0].noise == native.NOISE_UNIFORM  # (the default base_lin_vel noise)
  call = lambda a: sim._lib.b2_obs_history(sim._h, ctypes.byref(a), None)  # noqa: E731
  assert call(A) == 0
  n0 = sim._lib.b2_launch_count(sim._h)
  for label, edit in _bad_blocks(A):
    a = native.B2ObsHistArgs.from_buffer_copy(A)
    edit(a)
    assert call(a) != 0, label
    assert b"b2_obs_history" in sim._lib.b2_last_error(), label
  assert sim._lib.b2_launch_count(sim._h) == n0
  env.close()


def test_c_abi_layout(tmp_path):
  """The ctypes mirrors of B2ObsNoiseTerm, B2ObsNoiseGroup and the extended B2ObsHistArgs have the C structs' sizes
  and offsets; the fields before the noise block did not move."""
  structs = (native.B2ObsNoiseTerm, native.B2ObsNoiseGroup, native.B2ObsHistArgs)
  src = "#include <stdio.h>\n#include <stddef.h>\n#include \"b2sim.h\"\nint main(void) {\n"
  want = []
  for S in structs:
    src += f'  printf("%zu\\n", sizeof({S.__name__}));\n'
    want.append(ctypes.sizeof(S))
    for f, _ in S._fields_:
      src += f'  printf("%zu\\n", offsetof({S.__name__}, {f}));\n'
      want.append(getattr(S, f).offset)
  src += ('  printf("%d %d %d %d %d %d %d\\n", B2_NOISE_NONE, B2_NOISE_CONSTANT, B2_NOISE_UNIFORM, B2_NOISE_GAUSSIAN, '
          'B2_NOISE_ADD, B2_NOISE_SCALE, B2_NOISE_ABS);\n  return 0;\n}\n')
  want += [native.NOISE_NONE, native.NOISE_CONSTANT, native.NOISE_UNIFORM, native.NOISE_GAUSSIAN,
           *range(len(nz.OPERATIONS))]
  assert (nz.CONSTANT, nz.UNIFORM, nz.GAUSSIAN) == (native.NOISE_CONSTANT, native.NOISE_UNIFORM, native.NOISE_GAUSSIAN)
  (tmp_path / "layout.c").write_text(src)
  subprocess.check_call(["cc", "-I", str(ROOT / "include"), "-o", str(tmp_path / "layout"), str(tmp_path / "layout.c")])
  got = [int(x) for x in subprocess.check_output([str(tmp_path / "layout")]).split()]
  assert got == want
  # the block before the noise fields is where it was: group[1] ends where W starts (up to alignment)
  A = native.B2ObsHistArgs
  assert A.group.offset == 32 and A.W.offset == A.group.offset + ctypes.sizeof(native.B2ObsHistGroup) * 2

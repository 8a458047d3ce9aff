"""Reset and interval randomize_field events (mjlab_b200/envs/events.py, csrc/b2_events.cuh).

* The torch path against the reference's own ``randomize_field`` and ``EventManager`` (``apply("reset")``,
  ``reset``, ``apply("interval")``), executed from oracle/_ref over torch-path rollouts of workloads B and C with
  resets, time-outs, clip restarts (C) and interval firings.  The reference's samplers are fed the env's draws
  (``sample_uniform`` / ``sample_log_uniform`` of ``mjlab.envs.mdp.events`` and ``torch.rand`` of
  ``managers.event_manager``), and it runs on its own copy of the fields from the state before the env's first
  ``reset()``, so ``add`` and ``scale`` compound over its episodes as they do in the env.  Every randomised entry and
  every timer must be equal after every step (only the target axes: the reference also writes the other axes of a
  partly targeted element).
* b2_events against the torch path on one saved post-physics state (the Harness of test_mdp_kernels.py), using the
  fused path's own terminated / truncated: uniform draws bit-identical, log-uniform within LOG_ULPS (the kernel's expf
  under --use_fast_math is not correctly rounded); rows of envs that neither reset nor fired are untouched.
* Through the CUDA graph, the written fields reach the physics: the next sub-step of the reset worlds matches the
  oracle loaded with them.
* Defaults: nothing new is launched or drawn, and the built-in startup terms reproduce the inline recipes they replace.
* Every refusal of the cfg, of the env and of the C entry, and the C layout of the argument block.
"""

import ctypes
import dataclasses
import subprocess
import types
from pathlib import Path

import numpy as np
import pytest
import torch

import refload
import test_mdp_kernels as tmk
from mjlab_b200.envs import EventsCfg, RandomizeFieldCfg as R
from mjlab_b200.envs import events as evm
from mjlab_b200.envs import tracking_env as te
from mjlab_b200.envs import velocity_env as ve
from mjlab_b200.sim import native

ROOT = Path(__file__).resolve().parents[1]
LOG_ULPS = 4  # |kernel - torch| of a log_uniform draw (|log| <= 0.7 here: __expf is within 2 + 1.16 |x| ulps)

# ---- configurations ---------------------------------------------------------------------------------------------------
FEET_RE = (r"left_foot[1-7]_collision", r"right_foot[1-7]_collision")


def _cases() -> dict:
  """Term lists the checks run (G1 names; the rollouts use decimation 1, step_dt 0.005)."""
  I = (0.01, 0.03)
  return {
    "fields_a": (R("dof_armature", (0.8, 1.25), mode="reset", operation="scale"),
                 R("dof_damping", (0.5, 2.0), mode="interval", operation="scale", interval_range_s=I),
                 R("jnt_range", (-0.01, 0.01), mode="reset", operation="add"),
                 R("jnt_stiffness", (0.0, 0.1), mode="interval", operation="abs", interval_range_s=I),
                 R("body_mass", (0.9, 1.1), mode="reset", operation="scale"),
                 R("body_ipos", (-0.01, 0.01), mode="interval", operation="add", interval_range_s=I),
                 R("body_iquat", (0.99, 1.01), mode="reset", operation="scale", names="torso_link"),
                 R("body_inertia", (0.9, 1.1), mode="reset", operation="scale"),
                 R("qpos0", (-0.01, 0.01), mode="reset", operation="add", names=".*_knee_joint")),
    "fields_b": (R("body_pos", (-0.001, 0.001), mode="reset", operation="add", names=".*_wrist_yaw_link"),
                 R("body_quat", (0.999, 1.001), mode="interval", operation="scale", names="torso_link",
                   interval_range_s=I),
                 R("geom_friction", (0.3, 1.2), mode="reset", operation="abs", names=FEET_RE),
                 R("geom_pos", (-0.001, 0.001), mode="interval", operation="add", names=FEET_RE, interval_range_s=I),
                 R("geom_quat", (0.999, 1.001), mode="reset", operation="scale", names="left_foot1_collision"),
                 R("geom_rgba", (0.0, 1.0), mode="reset", operation="abs"),
                 R("site_pos", (-0.01, 0.01), mode="interval", operation="add", interval_range_s=I),
                 R("site_quat", (0.99, 1.01), mode="reset", operation="scale")),
    "log_axes": (R("geom_friction", {0: (0.5, 1.5), 2: (0.8, 1.25)}, mode="reset", operation="scale",
                   distribution="log_uniform", names=FEET_RE),
                 R("body_ipos", (-0.01, 0.01), mode="reset", operation="add", axes=(0, 2), names=".*_link"),
                 R("body_mass", (0.5, 2.0), mode="interval", operation="scale", distribution="log_uniform",
                   names=("pelvis", "torso_link"), interval_range_s=(0.0, 0.02))),
    "order": (R("body_mass", (0.9, 1.1), mode="reset", operation="scale", names=".*_ankle_.*"),
              R("body_mass", (0.01, 0.02), mode="reset", operation="add", names=".*_ankle_.*"),
              R("body_mass", (1.0, 3.0), mode="interval", operation="abs", names=".*_ankle_roll_link",
                interval_range_s=(0.005, 0.015)),
              R("geom_friction", (0.95, 1.05), mode="interval", operation="scale", axes=(1,),
                interval_range_s=(0.0, 0.004))),  # (shorter than step_dt: fires every step)
  }


CASES = list(_cases())


def _draws(V, t, log: bool) -> torch.Tensor:
  """[n, count] values of term t from the block V, as Events._apply forms them."""
  x = V[:, t.col:t.col + t.count] * t.span + t.lo
  return torch.exp(x) if log else x


# ---- the torch path against the reference's EventManager -------------------------------------------------------------
def _reference(monkeypatch):
  if not refload.available():
    pytest.skip("the reference package is not installed under oracle/_ref")
  monkeypatch.syspath_prepend(str(ROOT / "tests" / "stubs"))  # (prettytable stand-in)
  refload.load()
  import mjlab.envs.mdp.events as rev
  import mjlab.managers.event_manager as rem
  from mjlab.managers.manager_term_config import EventTermCfg
  from mjlab.managers.scene_entity_config import SceneEntityCfg
  from mjlab.third_party.isaaclab.isaaclab.utils.string import resolve_matching_names

  assert Path(rev.__file__).resolve().is_relative_to(refload.REF.resolve())
  return types.SimpleNamespace(events=rev, em=rem, EventTermCfg=EventTermCfg, SceneEntityCfg=SceneEntityCfg,
                               resolve=resolve_matching_names)


class _Entity:
  """The slice of the reference's Entity that SceneEntityCfg.resolve and randomize_field read, over our indexing."""

  def __init__(self, ref, ix):
    self.indexing = ix
    for kind, plural in (("joint", "joints"), ("body", "bodies"), ("geom", "geoms"), ("site", "sites")):
      names = list(getattr(ix, f"{kind}_names"))
      setattr(self, f"{kind}_names", names)
      setattr(self, f"num_{plural}", len(names))
      setattr(self, f"find_{plural}", lambda keys, preserve_order=False, _n=names, **_: ref.resolve(keys, _n, preserve_order))


def _record(kind, monkeypatch, terms, steps):
  """A torch-path rollout on the host emulation with `terms`: the fields before the first reset(), then per call of the
  events (reset() and every step) the block V, reset_buf, the fields and the timers after it."""
  mod = ve if kind == "B" else te
  tmk._patch_emul(monkeypatch, mod)
  calls, first = [], {}
  reset_all, step_torch, draw_timers = evm.Events.reset_all, evm.Events.step_torch, evm.Events.draw_timers

  def fields(self):
    return {f: getattr(self.sim.model, f).clone() for f in self.fields()}

  def rec_reset_all(self, rand):
    first.setdefault("fields", fields(self))
    reset_all(self, rand)
    calls.append(("reset_all", self.V.clone(), None, fields(self), self.timers.clone()))

  def rec_step(self, terminated, truncated):
    step_torch(self, terminated, truncated)
    calls.append(("step", self.V.clone(), (terminated | truncated).clone(), fields(self), self.timers.clone()))

  def rec_draw_timers(self, rand):
    def rec(*shape):
      u = rand(*shape)
      first.setdefault("u", []).append(u.clone())
      return u
    draw_timers(self, rec)

  monkeypatch.setattr(evm.Events, "draw_timers", rec_draw_timers)
  monkeypatch.setattr(evm.Events, "reset_all", rec_reset_all)
  monkeypatch.setattr(evm.Events, "step_torch", rec_step)
  ev = EventsCfg(terms=terms)
  if kind == "B":
    env = ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=6, decimation=1, fall_angle=0.12, episode_length_s=0.03,
                                               events=ev), device="cpu", native_mdp=False)
  else:
    env = te.TrackingFlatEnv(te.TrackingEnvCfg(num_envs=6, decimation=1, clip_frames=7, episode_length_s=0.04,
                                               events=ev), device="cpu", native_mdp=False)
  restarts = 0
  g = torch.Generator().manual_seed(5)
  for k in range(steps):
    if k == steps // 2:
      env.reset()
    _, _, term, trunc, _ = env.step(torch.rand((env.num_envs, env.nu), generator=g) * 2 - 1)
    if kind == "C":
      restarts += int((env._done_buf & ~(term | trunc)).sum())
  return env, first, calls, restarts


def _ref_run(ref, env, start, calls, monkeypatch):
  """Replay `calls` through the reference's EventManager on a copy of `start`; yields after each call the
  reference's fields and timers."""
  E = env.events
  n = env.num_envs
  model = types.SimpleNamespace(**{f: v.clone() for f, v in start["fields"].items()})
  first_u = list(start.get("u", []))
  renv = types.SimpleNamespace(num_envs=n, device="cpu", scene={"robot": _Entity(ref, env_ix(env))},
                               sim=types.SimpleNamespace(model=model))
  cur = {}

  def wrap(t):
    def func(env_, env_ids, **params):
      cur.update(term=t, ids=env_ids, axis=0)
      return ref.events.randomize_field(env_, env_ids, **params)
    return func

  def sample(lower, upper, size, device):
    t, k = cur["term"], cur["axis"]
    cur["axis"] += 1
    naxes = len(t.cfg.target_axes())
    ids = cur["ids"]
    x = cur["X"][id(t)][ids if isinstance(ids, torch.Tensor) else slice(None)][:, k::naxes]
    return x.reshape(size)

  monkeypatch.setattr(ref.events, "sample_uniform", sample)
  monkeypatch.setattr(ref.events, "sample_log_uniform", sample)
  interval = [t for t in E.stepped if t.cfg.mode == "interval"]
  rng = {}

  def rand(*size, device=None, **_):
    size = size[0] if len(size) == 1 and isinstance(size[0], tuple) else size
    if "V" not in cur:  # EventManager._prepare_terms: the env's first timers
      return first_u.pop(0)
    V = cur["V"]
    assert cur["phase"] == "interval"  # (EventManager.reset redraws no timer of a function term)
    tl = em._interval_term_time_left
    for j in range(rng["i"], len(interval)):  # the next interval term with an env to fire
      valid = (tl[j] < 1e-6).nonzero().flatten()
      if len(valid):
        rng["i"] = j + 1
        assert len(valid) == size[0]
        t = interval[j]
        return V[valid, t.col + t.count]
    raise AssertionError("torch.rand without a firing interval term")

  fake_torch = types.SimpleNamespace(**{k: getattr(torch, k) for k in dir(torch) if not k.startswith("__")})
  fake_torch.rand = rand
  monkeypatch.setattr(ref.em, "torch", fake_torch)
  cfg_fields = []
  for i, t in enumerate(E.stepped):
    c = t.cfg
    names = {"dof": "joint_names", "qpos": "joint_names", "joint": "joint_names", "body": "body_names",
             "geom": "geom_names", "site": "site_names"}[evm.FIELD_SPECS[c.field][0]]
    asset = ref.SceneEntityCfg("robot", **({} if c.names is None else
                                           {names: [c.names] if isinstance(c.names, str) else list(c.names)}))
    params = dict(field=c.field, ranges=c.ranges, distribution=c.distribution, operation=c.operation,
                  asset_cfg=asset)
    if c.axes is not None:
      params["axes"] = list(c.axes)
    kw = dict(func=wrap(t), mode=c.mode, params=params)
    if c.mode == "interval":
      kw["interval_range_s"] = tuple(c.interval_range_s)
    cfg_fields.append((f"t{i}", ref.EventTermCfg, dataclasses.field(default_factory=lambda kw=kw: ref.EventTermCfg(**kw))))
  cls = dataclasses.make_dataclass("EvCfg", cfg_fields)
  em = ref.em.EventManager(cls(), renv)
  step = 0
  for what, V, reset, _, _ in calls:
    cur["V"] = V
    cur["X"] = {id(t): _draws(V, t, t.cfg.distribution == "log_uniform") for t in E.stepped}
    ids = torch.arange(n) if what == "reset_all" else reset.nonzero().flatten()
    if len(ids):
      if any(t.cfg.mode == "reset" for t in E.stepped):
        em.apply("reset", env_ids=ids, global_env_step_count=step)
      cur.update(phase="reset", reset_ids=ids)
      rng["i"] = 0
      em.reset(ids)
    if what == "step" and interval:
      cur["phase"], rng["i"] = "interval", 0
      em.apply("interval", dt=env.step_dt)
    step += 1
    yield model, em


def env_ix(env):
  return env.events.indexing


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("kind", ["B", "C"])
def test_torch_path_matches_reference_event_manager(kind, case, monkeypatch):
  ref = _reference(monkeypatch)
  terms = _cases()[case]
  env, start, calls, restarts = _record(kind, monkeypatch, terms, steps=40)
  E = env.events
  resets = torch.stack([c[2] for c in calls if c[0] == "step"])
  assert int(resets.sum()) >= 6 and (kind == "B" or restarts > 0), (int(resets.sum()), restarts)
  assert int(resets.sum(0).max()) >= 3  # some env resets three times: add / scale compound over its episodes
  fired = 0
  for (what, V, reset, mine, timers), (model, em) in zip(calls, _ref_run(ref, env, start, calls, monkeypatch)):
    for t in E.stepped:
      a = getattr(model, t.cfg.field).reshape(env.num_envs, -1)[:, t.idx]
      b = mine[t.cfg.field].reshape(env.num_envs, -1)[:, t.idx]
      assert torch.equal(a, b), (case, what, t.cfg.field, (a != b).nonzero()[:4])
    interval = [t for t in E.stepped if t.cfg.mode == "interval"]
    for j, t in enumerate(interval):
      assert torch.equal(em._interval_term_time_left[j], timers[t.timer]), (case, what, j)
      fired += int((timers[t.timer] > em._interval_term_time_left[j] - 1).sum()) if what == "step" else 0
  env.close()


# ---- b2_events against the torch path on one saved state ----------------------------------------------------------------
class _Harness(tmk.Harness):
  """test_mdp_kernels' Harness that also saves and restores the randomised fields and the timers."""

  def snapshot(self):
    s = super().snapshot()
    E = self.env.events
    s.update({"model." + f: getattr(self.env.sim.model, f).clone() for f in E.fields()})
    s["events.timers"] = E.timers.clone()
    return s

  def restore(self, snap):
    E = self.env.events
    for k, v in snap.items():
      if k.startswith("model."):
        getattr(self.env.sim.model, k[6:])[...] = v
    E.timers.copy_(snap["events.timers"])
    super().restore({k: v for k, v in snap.items() if k.split(".")[0] not in ("model", "events")})


def _env(kind, backend, monkeypatch, case, n):
  ev = EventsCfg(terms=_cases()[case])
  if kind == "B":
    H = tmk._velocity(backend, monkeypatch, num_envs=n, decimation=1, fall_angle=0.12, episode_length_s=0.2, events=ev)
    fields = tmk.VEL_ENV
  else:
    H = tmk._tracking(backend, monkeypatch, num_envs=n, decimation=1, clip_frames=9, episode_length_s=0.2, events=ev)
    fields = tmk.TRK_ENV
  return _Harness(H.env, backend, fields)


def _kernel_rollout(H, kind, steps, seed):
  env = H.env
  E = env.events
  n, g = env.num_envs, tmk._gen(env, seed)
  ep = env.max_episode_length - 1 - (torch.arange(n, device=env.device) * 7 + 2) % steps
  env.episode_length_buf.copy_(ep.int())
  counts = dict(reset=0, fired=0, kept=0)
  tmk._pre(env, torch.zeros(n, env.nu, device=env.device))
  env.sim.step_n(env.cfg.decimation)
  for k in range(steps):
    act = torch.rand((n, env.nu), generator=g, device=env.device) * 2 - 1
    U = env._draw() if kind == "B" else env._rand(n, 48 + 4 * env.nu)
    E.draw(env._rand)
    S, _, N = H.both(act, U)
    reset = N["out.terminated"] | N["out.truncated"]
    # the torch events on the saved fields and timers with the fused path's own reset_buf
    post = {f: getattr(env.sim.model, f).clone() for f in E.fields()}
    post_t = E.timers.clone()
    for f in E.fields():
      getattr(env.sim.model, f)[...] = S["model." + f]
    E.timers.copy_(S["events.timers"])
    E.step_torch(N["out.terminated"], N["out.truncated"])
    want = {f: getattr(env.sim.model, f).clone() for f in E.fields()}
    assert torch.equal(E.timers, post_t), (k, (E.timers != post_t).nonzero()[:4])
    hit = reset.clone()
    for t in E.stepped:
      a = post[t.cfg.field].reshape(n, -1)[:, t.idx]
      b = want[t.cfg.field].reshape(n, -1)[:, t.idx]
      if t.cfg.distribution == "log_uniform":
        H.ulps(t.cfg.field, a, b, LOG_ULPS)
      else:
        H.equal(t.cfg.field, a, b)
    fired = (post_t != S["events.timers"] - env.step_dt).any(0) if E.timers.numel() else torch.zeros_like(reset)
    hit = reset | fired
    for f in dict.fromkeys(t.cfg.field for t in E.stepped):  # untargeted entries, rows that neither reset nor fired
      targets = torch.cat([t.idx for t in E.stepped if t.cfg.field == f])
      rest = torch.ones(post[f].reshape(n, -1).shape[1], dtype=torch.bool, device=env.device)
      rest[targets] = False
      H.equal(f + " (untargeted)", post[f].reshape(n, -1)[:, rest], S["model." + f].reshape(n, -1)[:, rest])
      H.equal(f + " (untouched rows)", post[f][~hit], S["model." + f][~hit])
    for f in E.fields():
      getattr(env.sim.model, f)[...] = post[f]
    E.timers.copy_(post_t)
    counts["reset"] += int(reset.sum())
    counts["fired"] += int((hit & ~reset).sum())
    counts["kept"] += int((~hit).sum())
  return counts


def _kernel_case(kind, backend, monkeypatch, case, n, steps):
  H = _env(kind, backend, monkeypatch, case, n)
  counts = _kernel_rollout(H, kind, steps, seed=n)
  # (the "order" case has a term that fires in every step, so no env keeps its rows there)
  assert counts["reset"] > 0 and counts["fired"] > 0 and (counts["kept"] > 0 or case == "order"), counts
  H.env.close()


KERNEL_CASES = ["fields_a", "fields_b", "log_axes", "order"]


@pytest.mark.parametrize("case", KERNEL_CASES)
@pytest.mark.parametrize("kind", ["B", "C"])
@pytest.mark.parametrize("n", [1, 33])
def test_kernel_matches_torch_emul(kind, case, n, monkeypatch):
  _kernel_case(kind, "emul", monkeypatch, case, n, steps=5 if n > 1 else 16)


@pytest.mark.gpu
@pytest.mark.parametrize("case", KERNEL_CASES)
@pytest.mark.parametrize("kind", ["B", "C"])
@pytest.mark.parametrize("n", [1, 33, 4096])
def test_kernel_matches_torch_cuda(kind, case, n, monkeypatch):
  _kernel_case(kind, "cuda", monkeypatch, case, n, steps=6 if n > 1 else 16)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["B", "C"])
def test_kernel_under_graph_replay(kind):
  """Each replay of the captured step writes the torch update of the fields and timers before it, by the replay's
  own V and reset_buf."""
  n = 512
  ev = EventsCfg(terms=_cases()["order"] + _cases()["fields_a"][:2])
  if kind == "B":
    env = ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=n, fall_angle=0.12, episode_length_s=0.2, events=ev))
  else:
    env = te.TrackingFlatEnv(te.TrackingEnvCfg(num_envs=n, clip_frames=12, episode_length_s=0.2, events=ev))
  E = env.events
  env.enable_cuda_graph()
  g = torch.Generator(device="cuda:0").manual_seed(3)
  resets = fired = 0
  for _ in range(12):
    before = {f: getattr(env.sim.model, f).clone() for f in E.fields()}
    timers = E.timers.clone()
    _, _, term, trunc, _ = env.step(torch.rand((n, env.nu), generator=g, device="cuda:0") * 2 - 1)
    got = {f: getattr(env.sim.model, f).clone() for f in E.fields()}
    got_t = E.timers.clone()
    resets += int((term | trunc).sum())
    fired += int((got_t != timers - env.step_dt).sum())
    for f in E.fields():
      getattr(env.sim.model, f)[...] = before[f]
    E.timers.copy_(timers)
    E.step_torch(term, trunc)
    assert torch.equal(E.timers, got_t)
    for f in E.fields():
      assert torch.equal(getattr(env.sim.model, f), got[f]), f
      getattr(env.sim.model, f)[...] = got[f]
  assert resets > 0 and fired > 0
  env.close()


@pytest.mark.gpu
def test_physics_sees_the_reset_draws():
  """A velocity env with a reset-mode body_mass scale and a feet geom_friction abs term, through its CUDA graph: after
  a step with resets, the next sub-step of every world matches the oracle loaded with the fields the events wrote."""
  from util import load_oracle, relerr

  from oracle.oracle import Oracle

  n = 64
  ev = EventsCfg(terms=(R("body_mass", (0.5, 1.5), mode="reset", operation="scale"),
                        R("geom_friction", (0.2, 0.4), mode="reset", operation="abs", names=FEET_RE)))
  env = ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=n, fall_angle=0.12, episode_length_s=0.2, events=ev))
  env.enable_cuda_graph()
  mass0 = env.sim.model.body_mass.clone()
  done = torch.zeros(n, dtype=torch.bool, device="cuda:0")
  for _ in range(60):
    _, _, term, trunc, _ = env.step(torch.zeros(n, env.nu, device="cuda:0"))
    done |= term | trunc
    if int(done.sum()) >= 8:
      break
  assert int(done.sum()) >= 8
  mass = env.sim.model.body_mass.clone()
  assert bool((mass[done] != mass0[done]).any(1).all())
  sim, m = env.sim, env.model
  o = Oracle(m, nworld=n, maxcon=int(sim.get_option("maxcon")))
  sim.set_option("iterations", 50)  # converged answers do not depend on the path that reached them
  for k in ("timestep", "iterations", "ls_iterations", "tolerance", "ls_tolerance", "integrator"):
    o.set_option(k, sim.get_option(k))
  load_oracle(o, {f: getattr(sim.data, f)[:].cpu().numpy() for f in ("qpos", "qvel", "ctrl", "qacc_warmstart")})
  for f in ("body_mass", "geom_friction"):
    o.model_field(f)[:] = getattr(sim.model, f)[...].cpu().numpy().reshape(n, -1)
  o.step()
  sim.step()
  torch.cuda.synchronize()
  rows = done.cpu().numpy()
  for f in ("qpos", "qvel"):
    e = relerr(getattr(sim.data, f)[:].cpu().numpy()[rows], o.field(f)[rows]).max()
    assert e < 1e-3, (f, e)
  env.close()


# ---- defaults ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["B", "C"])
def test_default_events_launch_and_draw_nothing(kind, monkeypatch):
  """Without reset or interval terms a step launches what it did and draws no V; with them, one launch more."""
  launches = {}
  for name in ("default", "configured"):
    if name == "default":
      H = (tmk._velocity("emul", monkeypatch, num_envs=4, decimation=1) if kind == "B"
           else tmk._tracking("emul", monkeypatch, num_envs=4, decimation=1))
      assert H.env.cfg.events == EventsCfg()
    else:
      H = _env(kind, "emul", monkeypatch, "order", 4)
    env = H.env
    count = lambda: env.sim._lib.b2_launch_count(env.sim._h)  # noqa: E731
    act = torch.zeros(env.num_envs, env.nu)
    env.step(act)
    before = count()
    state = env.gen.get_state()
    env.step(act)
    launches[name] = count() - before
    if name == "default":
      assert env.events.V is None and env.events._args is None and not env.events.active
      # the step drew exactly its own uniforms
      g = torch.Generator().manual_seed(0)
      g.set_state(state)
      width = 16 + 9 + 2 * env.nu if kind == "B" else 48 + 4 * env.nu
      torch.rand((env.num_envs, width), generator=g)
      assert torch.equal(g.get_state(), env.gen.get_state())
    env.close()
  assert launches["configured"] == launches["default"] + 1, launches


@pytest.mark.parametrize("kind", ["B", "C"])
def test_default_startup_terms_reproduce_the_inline_recipes(kind, monkeypatch):
  """The built-in startup terms write the fields the inline recipes they replace wrote, from the same generator."""
  mod = ve if kind == "B" else te
  tmk._patch_emul(monkeypatch, mod)
  n = 5
  if kind == "B":
    env = ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=n, robot="go1", friction_range=(0.3, 1.2)), device="cpu")
  else:
    env = te.TrackingFlatEnv(te.TrackingEnvCfg(num_envs=n, clip_frames=4, friction_range=(0.4, 1.1)), device="cpu")
  m, cfg = env.model, env.cfg
  gen = torch.Generator().manual_seed(cfg.seed)

  def rand(*shape):
    return torch.rand(shape, generator=gen)

  def shared(f):
    return torch.tensor(np.asarray(m.arrays[f]), dtype=torch.float32).reshape(getattr(env.sim.model, f).shape[1:])

  from mjlab_b200.asset_zoo import g1, go1
  feet_names = (g1 if cfg.__class__ is te.TrackingEnvCfg or cfg.robot == "g1" else go1).FOOT_GEOMS
  feet = [m.names["geom"].index(f"robot/{g}") for g in feet_names]
  fr = shared("geom_friction").expand(n, -1, -1).clone()
  if kind == "B":
    lo, hi = cfg.friction_range
    fr[:, feet, 0] = rand(n, len(feet)) * (hi - lo) + lo
  else:
    ix = env.robot.indexing
    ipos = shared("body_ipos").expand(n, -1, -1).clone()
    torso = int(ix.body_ids[ix.body_names.index("torso_link")])
    rng = torch.tensor([[-0.025, 0.025], [-0.05, 0.05], [-0.05, 0.05]])
    ipos[:, torso] += rand(n, 3) * (rng[:, 1] - rng[:, 0]) + rng[:, 0]
    q0 = shared("qpos0").expand(n, -1).clone()
    q0[:, ix.joint_q_adr.long()] += rand(n, env.nu) * 0.02 - 0.01
    lo, hi = cfg.friction_range
    fr[:, feet, 0] = rand(n, len(feet)) * (hi - lo) + lo
    assert torch.equal(env.sim.model.body_ipos[...], ipos)
    assert torch.equal(env.sim.model.qpos0[...], q0)
  assert torch.equal(env.sim.model.geom_friction[...], fr)
  assert [t.cfg.field for t in env.events.startup] == (["geom_friction"] if kind == "B" else
                                                       ["body_ipos", "qpos0", "geom_friction"])
  env.close()


def test_reset_add_compounds_over_episodes(monkeypatch):
  """An add term of mode reset adds a fresh draw to the field's current value at every reset of an env."""
  tmk._patch_emul(monkeypatch, ve)
  term = R("body_mass", (0.1, 0.2), mode="reset", operation="add", names="torso_link")
  env = ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=3, decimation=1, episode_length_s=0.015,
                                             events=EventsCfg(terms=(term,))), device="cpu")
  t = env.events.stepped[0]
  row = lambda: env.sim.model.body_mass.reshape(3, -1)[:, t.idx[0]].clone()  # noqa: E731
  want, resets = row(), 0
  for _ in range(10):
    env.step(torch.zeros(3, env.nu))
    reset = env._term | env._trunc
    resets += int(reset.sum())
    want = torch.where(reset, want + (env.events.V[:, 0] * t.span[0] + t.lo[0]), want)
    assert torch.equal(row(), want)
  assert resets >= 9
  env.close()


# ---- refusals ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [
  dict(field="actuator_gainprm", ranges=(0.9, 1.1)), dict(field="dof_frictionloss", ranges=(0.0, 0.1)),
  dict(field="body_mass", ranges=(0.9, 1.1), mode="episode"),
  dict(field="body_mass", ranges=(0.9, 1.1), distribution="gaussian"),
  dict(field="body_mass", ranges=(0.9, 1.1), distribution="normal"),
  dict(field="body_mass", ranges=(0.9, 1.1), operation="mul"),
  dict(field="body_mass", ranges=(1.1, 0.9)), dict(field="body_mass", ranges=(0.0, float("inf"))),
  dict(field="body_mass", ranges=(float("nan"), 1.0)), dict(field="body_mass", ranges=(0.0, 1e39)),
  dict(field="body_mass", ranges=0.5), dict(field="body_mass", ranges=(0.0, 1.0), distribution="log_uniform"),
  dict(field="geom_friction", ranges={0: (0.5, 1.0), 1: (-1.0, 1.0)}, distribution="log_uniform"),
  dict(field="body_ipos", ranges=(0.0, 1.0), axes=(3,)), dict(field="body_mass", ranges=(0.0, 1.0), axes=(1,)),
  dict(field="geom_friction", ranges=(0.0, 1.0), axes=(3,)), dict(field="body_ipos", ranges=(0.0, 1.0), axes=(0, 0)),
  dict(field="geom_quat", ranges={0: (0.0, 1.0)}, axes=(0, 1)),
  dict(field="body_mass", ranges=(0.9, 1.1), mode="interval"),
  dict(field="body_mass", ranges=(0.9, 1.1), mode="interval", interval_range_s=(2.0, 1.0)),
  dict(field="body_mass", ranges=(0.9, 1.1), mode="interval", interval_range_s=(-1.0, 1.0)),
  dict(field="body_mass", ranges=(0.9, 1.1), mode="interval", interval_range_s=(0.0, float("inf"))),
  dict(field="body_mass", ranges=(0.9, 1.1), names=3),
])
def test_cfg_refusals(kw):
  with pytest.raises(ValueError):
    R(**kw)


@pytest.mark.parametrize("kind", ["B", "C"])
def test_env_refusals(kind, monkeypatch):
  """Names that match nothing or a name matched twice, and a cfg edited after it was made, raise when the env is
  built."""
  mod = ve if kind == "B" else te
  tmk._patch_emul(monkeypatch, mod)

  def build(*terms):
    ev = EventsCfg(terms=terms)
    if kind == "B":
      return ve.VelocityFlatEnv(ve.VelocityEnvCfg(num_envs=2, events=ev), device="cpu")
    return te.TrackingFlatEnv(te.TrackingEnvCfg(num_envs=2, clip_frames=4, events=ev), device="cpu")

  for terms in ((R("body_mass", (0.9, 1.1), names="no_such_body"),),
                (R("geom_friction", (0.5, 1.0), names=("left_foot1_collision", "left_foot[0-9]_collision")),),
                (R("dof_damping", (0.5, 1.0), names=(".*_knee_joint", "nope")),)):
    with pytest.raises(ValueError, match="match"):
      build(*terms)
  t = R("body_mass", (0.9, 1.1), mode="reset")
  t.distribution = "gaussian"
  with pytest.raises(ValueError, match="gaussian"):
    build(t)
  with pytest.raises(ValueError, match="RandomizeFieldCfg"):
    EventsCfg(terms=(dict(field="body_mass"),))


def _bad_blocks(nfields):
  def term(f):
    return lambda a, E: f(a.term[0])
  return [
    ("null terminated", lambda a, E: setattr(a, "terminated", None)),
    ("null truncated", lambda a, E: setattr(a, "truncated", None)),
    ("null V", lambda a, E: setattr(a, "V", None)),
    ("null table", lambda a, E: setattr(a, "elem", None)),
    ("no terms", lambda a, E: setattr(a, "nterm", 0)),
    ("too many terms", lambda a, E: setattr(a, "nterm", native.EVENTS_NTERM + 1)),
    ("zero step_dt", lambda a, E: setattr(a, "step_dt", 0.0)),
    ("missing timers", lambda a, E: setattr(a, "timers", None)),
    ("too few timer rows", lambda a, E: setattr(a, "ninterval", 0)),
    ("unknown mode", term(lambda t: setattr(t, "mode", 2))),
    ("unknown operation", term(lambda t: setattr(t, "operation", 3))),
    ("unknown distribution", term(lambda t: setattr(t, "distribution", -1))),
    ("field outside the table", term(lambda t: setattr(t, "field", nfields))),
    ("int field", term(lambda t: setattr(t, "field", E_INT_FIELD[0]))),
    ("shared field", term(lambda t: setattr(t, "field", E_SHARED_FIELD[0]))),
    ("V column outside", term(lambda t: setattr(t, "col", 10**6))),
    ("V column negative", term(lambda t: setattr(t, "col", -1))),
    ("zero count", term(lambda t: setattr(t, "count", 0))),
    ("counts off", lambda a, E: setattr(a, "nelem", a.nelem + 1)),
  ]


E_INT_FIELD, E_SHARED_FIELD = [0], [0]


def test_c_entry_refusals(monkeypatch):
  """b2_events refuses every malformed block before it launches (host emulation)."""
  H = _env("B", "emul", monkeypatch, "order", 3)
  env, sim = H.env, H.env.sim
  E = env.events
  A = E._args
  assert A is not None and A.ninterval == 2
  lib, h = sim._lib, sim._h
  names = [lib.b2_field_name(h, 1, i).decode() for i in range(lib.b2_num_fields(h, 1))]
  E_INT_FIELD[0] = names.index("jnt_type") if "jnt_type" in names else next(
    i for i, f in enumerate(names) if sim._lib.b2_expand_model_field(h, f.encode(), None, None) != 0)
  E_SHARED_FIELD[0] = names.index("dof_armature")
  call = lambda a: lib.b2_events(h, ctypes.byref(a), None)  # noqa: E731
  assert call(A) == 0
  n0 = lib.b2_launch_count(h)
  for label, edit in _bad_blocks(len(names)):
    a = native.B2EventArgs.from_buffer_copy(A)
    edit(a, E)
    assert call(a) != 0, label
    assert b"b2_events" in lib.b2_last_error(), label
  # an entry outside the field's row (a table of its own, so that the checked one is not taken as known)
  bad = E._keep[0].clone()
  bad.view(torch.int32)[0, 0] = env.sim.model.body_mass.shape[1]
  a = native.B2EventArgs.from_buffer_copy(A)
  a.elem = bad.data_ptr()
  assert call(a) != 0 and b"outside the row" in lib.b2_last_error()
  assert lib.b2_launch_count(h) == n0
  assert lib.b2_events(None, ctypes.byref(A), None) != 0
  assert lib.b2_events(h, None, None) != 0
  env.close()


def test_c_abi_layout(tmp_path):
  """The ctypes mirrors of B2EventTerm, B2EventElem and B2EventArgs have the C structs' sizes and offsets."""
  structs = (native.B2EventTerm, native.B2EventElem, native.B2EventArgs)
  src = "#include <stdio.h>\n#include <stddef.h>\n#include \"b2sim.h\"\nint main(void) {\n"
  want = []
  for S in structs:
    src += f'  printf("%zu\\n", sizeof({S.__name__}));\n'
    want.append(ctypes.sizeof(S))
    for f, _ in S._fields_:
      src += f'  printf("%zu\\n", offsetof({S.__name__}, {f}));\n'
      want.append(getattr(S, f).offset)
  src += ('  printf("%d %d %d %d %d %d %d %d %d\\n", B2_EVENTS_NTERM, B2_EVENT_RESET, B2_EVENT_INTERVAL, B2_EVENT_ADD, '
          'B2_EVENT_SCALE, B2_EVENT_ABS, B2_EVENT_UNIFORM, B2_EVENT_LOG_UNIFORM, 0);\n  return 0;\n}\n')
  want += [native.EVENTS_NTERM, native.EVENT_RESET, native.EVENT_INTERVAL, *range(3), *range(2), 0]
  (tmp_path / "layout.c").write_text(src)
  subprocess.check_call(["cc", "-I", str(ROOT / "include"), "-o", str(tmp_path / "layout"), str(tmp_path / "layout.c")])
  got = [int(x) for x in subprocess.check_output([str(tmp_path / "layout")]).split()]
  assert got == want
  assert [evm.OPERATIONS.index(o) for o in ("add", "scale", "abs")] == [0, 1, 2]
  assert [evm.DISTRIBUTIONS.index(d) for d in ("uniform", "log_uniform")] == [0, 1]

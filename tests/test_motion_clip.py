"""Motion clips in the reference's file layout and the adaptive start-frame sampler of the tracking task, on the
host-emulated library (tests/emul): the loader, the sampler kernel b2_trackenv_bins and the draws of
b2_trackenv_post1 against the torch implementation, and the sampler's metrics against the reference's own
``MotionCommand._adaptive_sampling`` where oracle/_ref is installed."""

import ctypes
import importlib.util
import sys
import types
from pathlib import Path

import numpy as np
import pytest
import torch

import refload
from mjlab_b200.sim import native
from test_kernel_emul import EmulSim, EmulSimulation, _load

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tools"))

FRAMES = 960  # 20 bins at the env step of 0.02 s


@pytest.fixture(scope="module")
def clip(tmp_path_factory):
  from make_motion_clip import make_clip

  from mjlab_b200.asset_zoo import load_compiled
  from mjlab_b200.sim import SimulationCfg

  m = load_compiled("g1_tracking_flat")
  sim = EmulSimulation(FRAMES, SimulationCfg(), m, "cpu")
  path = make_clip(tmp_path_factory.mktemp("clip") / "clip.npz", frames=FRAMES, device="cpu", sim=sim, model=m)
  sim.close()
  return path


def _indexing():
  from mjlab_b200.asset_zoo import load_compiled
  from mjlab_b200.entity_data import EntityIndexing

  return EntityIndexing.from_model(load_compiled("g1_tracking_flat"), "robot", "cpu")


def _emul_env(monkeypatch, **cfg):
  import mjlab_b200.envs.tracking_env as te

  monkeypatch.setattr(te, "Simulation", EmulSimulation)
  monkeypatch.setattr(native, "check", lambda rc: (_ for _ in ()).throw(RuntimeError("b2sim call failed")) if rc else None)
  native_mdp = cfg.pop("native_mdp")
  return te.TrackingFlatEnv(te.TrackingEnvCfg(**cfg), device="cpu", native_mdp=native_mdp)


# ---- loader ------------------------------------------------------------------------------------------------------
def test_loader_round_trips_a_generated_clip(clip):
  from mjlab_b200.envs.motion import MotionClip
  from mjlab_b200.envs.tracking_env import BODY_NAMES

  ix = _indexing()
  mc = MotionClip.load(clip, ix, BODY_NAMES, 0.02, "cpu")
  raw = np.load(clip)
  sel = [ix.body_names.index(b) for b in BODY_NAMES]
  assert mc.num_frames == FRAMES
  for k, t in mc.as_dict().items():
    assert t.dtype == torch.float32 and t.is_contiguous(), k
    want = raw[k] if k.startswith("joint") else raw[k][:, sel]
    assert np.array_equal(t.numpy(), want.astype(np.float32)), k
  # the clip moves: joints swing, the pelvis drifts, velocities are non-zero
  assert raw["joint_pos"].std(axis=0).min() > 1e-3 and np.abs(raw["body_lin_vel_w"][:, 0, 0] - 0.3).max() < 1e-4
  assert np.abs(raw["joint_vel"]).max() > 0.1 and np.abs(raw["body_ang_vel_w"]).max() > 0.1


def _bad_files(clip, tmp_path):
  raw = dict(np.load(clip))
  cases = {}
  d = dict(raw); del d["body_quat_w"]
  cases["missing"] = (d, r"missing key 'body_quat_w'")
  d = dict(raw); d["joint_vel"] = d["joint_vel"][:, :5]
  cases["shape"] = (d, rf"'joint_vel' has shape \({FRAMES}, 5\), expected \[{FRAMES}, 29\]")
  d = dict(raw); d["body_pos_w"] = d["body_pos_w"][:, :10]
  cases["bodies"] = (d, rf"'body_pos_w' has shape \({FRAMES}, 10, 3\), expected \[{FRAMES}, 30, 3\]")
  d = dict(raw); d["body_lin_vel_w"] = d["body_lin_vel_w"][:-1]
  cases["frames"] = (d, rf"'body_lin_vel_w' has shape \({FRAMES - 1}, 30, 3\), expected \[{FRAMES}, 30, 3\]")
  d = {k: (v[:1] if k != "fps" else v) for k, v in raw.items()}
  cases["one_frame"] = (d, r"'joint_pos' has 1 frame\(s\), expected T >= 2")
  d = dict(raw); d["body_ang_vel_w"] = d["body_ang_vel_w"].copy(); d["body_ang_vel_w"][7, 3, 1] = np.nan
  cases["nan"] = (d, r"'body_ang_vel_w' holds non-finite")
  d = dict(raw); d["fps"] = np.array([30])
  cases["fps"] = (d, r"'fps' is \[30.0\], expected \[50\]")
  out = {}
  for name, (arrays, msg) in cases.items():
    p = tmp_path / f"{name}.npz"
    np.savez(p, **arrays)
    out[name] = (p, msg)
  return out


def test_loader_refuses_malformed_files(clip, tmp_path):
  from mjlab_b200.envs.motion import MotionClip
  from mjlab_b200.envs.tracking_env import BODY_NAMES

  ix = _indexing()
  for name, (path, msg) in _bad_files(clip, tmp_path).items():
    with pytest.raises(ValueError, match=msg):
      MotionClip.load(path, ix, BODY_NAMES, 0.02, "cpu")
  with pytest.raises(ValueError, match=r"not bodies of the entity"):
    MotionClip.load(clip, ix, ("pelvis", "tail_link"), 0.02, "cpu")


def _ref_commands(monkeypatch):
  """The reference's tasks/tracking/mdp/commands.py, executed from oracle/_ref (its viewer import stubbed)."""
  if not refload.available():
    pytest.skip("the reference package is not installed (oracle/install_reference.py)")
  refload.load()
  monkeypatch.syspath_prepend(str(ROOT / "tests" / "stubs"))
  from mjlab.managers.command_manager import CommandTerm
  from mjlab.managers.manager_term_config import CommandTermCfg

  mgr = sys.modules["mjlab.managers"]
  monkeypatch.setattr(mgr, "CommandTerm", CommandTerm, raising=False)
  monkeypatch.setattr(mgr, "CommandTermCfg", CommandTermCfg, raising=False)
  dv = types.ModuleType("mjlab.viewer.debug_visualizer")
  dv.DebugVisualizer = type("DebugVisualizer", (), {})
  monkeypatch.setitem(sys.modules, "mjlab.viewer.debug_visualizer", dv)
  name = "mjlab.tasks.tracking.mdp.commands"
  spec = importlib.util.spec_from_file_location(name, refload.REF / "mjlab" / "tasks" / "tracking" / "mdp" / "commands.py")
  mod = importlib.util.module_from_spec(spec)
  monkeypatch.setitem(sys.modules, name, mod)
  spec.loader.exec_module(mod)
  return mod


def test_loader_reads_the_reference_layout_as_the_reference_does(clip, tmp_path, monkeypatch):
  from ref_env_cases import _static_clip

  from mjlab_b200.envs.motion import MotionClip
  from mjlab_b200.envs.tracking_env import BODY_NAMES

  ix = _indexing()
  static = _static_clip(tmp_path / "static.npz")
  ours = {p: MotionClip.load(p, ix, BODY_NAMES, 0.02, "cpu") for p in (static, clip)}
  assert ours[static].num_frames == 200 and float(ours[static].joint_vel.abs().max()) == 0.0
  mod = _ref_commands(monkeypatch)
  idx = torch.tensor([ix.body_names.index(b) for b in BODY_NAMES])
  for p, mc in ours.items():  # (the generated clip loads unchanged through the reference's MotionLoader too)
    ref = mod.MotionLoader(str(p), idx, device="cpu")
    assert ref.time_step_total == mc.num_frames
    for k in ("joint_pos", "joint_vel", "body_pos_w", "body_quat_w", "body_lin_vel_w", "body_ang_vel_w"):
      assert torch.equal(getattr(ref, k), getattr(mc, k)), (p, k)


# ---- the sampler kernel --------------------------------------------------------------------------------------------
class _Bins:
  """b2_trackenv_bins on the emulated library with its own sampler arrays."""

  def __init__(self, lib, nbins, ksize=1, lam=0.8, ratio=0.1, alpha=0.001):
    from mjlab_b200.asset_zoo import load_compiled

    self.lib, self.sim = lib, EmulSim(lib, load_compiled("g1_tracking_flat"), 1)
    k = torch.tensor([lam**i for i in range(ksize)])
    self.kernel = k / k.sum()
    self.ema, self.cur, self.cdf, self.metrics = torch.zeros(nbins), torch.zeros(nbins), torch.zeros(nbins), torch.zeros(3)
    A = self.A = native.B2TrackEnvArgs()
    A.nb, A.anchor, A.T, A.root_body = 1, 0, 2, 1
    A.adaptive, A.nbins, A.adaptive_kernel_size = native.START_ADAPTIVE, nbins, ksize
    A.adaptive_alpha, A.adaptive_uniform_ratio = alpha, ratio
    for f, t in (("adaptive_kernel", self.kernel), ("cdf", self.cdf), ("bin_fail_ema", self.ema),
                 ("bin_fail_cur", self.cur), ("metrics", self.metrics)):
      setattr(A, f, t.data_ptr())

  def run(self):
    assert self.lib.b2_trackenv_bins(self.sim.h, ctypes.byref(self.A), None) == 0, self.lib.b2_last_error()


def _ref_metrics(mod, bin_failed, ksize, lam=0.8, ratio=0.1):
  B = len(bin_failed)
  k = torch.tensor([lam**i for i in range(ksize)])
  stub = types.SimpleNamespace(
    _env=types.SimpleNamespace(termination_manager=types.SimpleNamespace(terminated=torch.zeros(1, dtype=torch.bool))),
    time_steps=torch.zeros(1, dtype=torch.long), bin_count=B, motion=types.SimpleNamespace(time_step_total=50 * B),
    _current_bin_failed=torch.zeros(B), bin_failed_count=torch.tensor(bin_failed, dtype=torch.float32),
    cfg=types.SimpleNamespace(adaptive_uniform_ratio=ratio, adaptive_kernel_size=ksize), kernel=k / k.sum(),
    device="cpu", metrics={n: torch.zeros(1) for n in ("sampling_entropy", "sampling_top1_prob", "sampling_top1_bin")})
  mod.MotionCommand._adaptive_sampling(stub, torch.zeros(1, dtype=torch.long))
  return [float(stub.metrics[n][0]) for n in ("sampling_entropy", "sampling_top1_prob", "sampling_top1_bin")]


def test_sampler_metrics_match_the_reference_formula(monkeypatch):
  mod = _ref_commands(monkeypatch)
  lib = _load()
  rng = np.random.default_rng(4)
  vectors = [np.zeros(20), rng.exponential(0.05, 20), np.eye(20)[13] * 0.3, rng.exponential(0.2, 7)]
  for v in vectors:
    for ksize in (1, 3, 8):
      b = _Bins(lib, len(v), ksize=ksize)
      b.ema[:] = torch.tensor(v, dtype=torch.float32)
      b.run()
      ref = _ref_metrics(mod, v, ksize)
      assert np.allclose(b.metrics.numpy(), ref, atol=1e-6, rtol=0), (ksize, b.metrics, ref)
  b.sim.close()


def test_sampler_kernel_update_and_large_bin_counts():
  """EMA update and CDF of b2_trackenv_bins against a float64 restatement, up to 65536 bins (18 h at 50 fps); one
  bin has entropy 1 by definition (the reference divides by log 1)."""
  lib = _load()
  rng = np.random.default_rng(7)
  for B, ksize in ((1, 1), (1, 4), (20, 3), (1000, 5), (65536, 2)):
    b = _Bins(lib, B, ksize=ksize, alpha=0.25)
    ema, cur = rng.exponential(0.1, B), rng.integers(0, 4, B).astype(float)
    b.ema[:] = torch.tensor(ema, dtype=torch.float32)
    b.cur[:] = torch.tensor(cur, dtype=torch.float32)
    b.run()
    ema_new = 0.25 * cur + 0.75 * ema
    assert np.allclose(b.ema.numpy(), ema_new, rtol=1e-5, atol=1e-7) and not b.cur.any()
    w = b.kernel.double().numpy()
    x = np.concatenate([ema_new + 0.1 / B, np.full(ksize - 1, ema_new[-1] + 0.1 / B)])
    p = np.array([x[i:i + ksize] @ w for i in range(B)])
    p /= p.sum()
    cdf = b.cdf.double().numpy()
    assert cdf[-1] == 1.0 and (np.diff(cdf) >= 0).all()
    assert np.abs(cdf - np.cumsum(p)).max() < 2e-5, B
    if B == 1:
      assert b.metrics[0] == 1.0 and b.metrics[1] == 1.0 and b.metrics[2] == 0.0
    b.sim.close()


def test_draws_follow_the_distribution(clip, monkeypatch):
  """Inverse-CDF draws on 20k uniforms: the frame histogram passes a chi-square test against p (bins uniform inside)."""
  from scipy.stats import chisquare

  env = _emul_env(monkeypatch, num_envs=2, motion_file=clip, native_mdp=False)
  B, T = env.bin_count, env.T
  assert B == 20 and T == FRAMES
  env.bin_failed_count.copy_(torch.linspace(0, 1, B) ** 2 * 0.05)
  env._cdf.copy_(env._start_distribution()[1])
  p = env._start_distribution()[0].double().numpy()
  g = torch.Generator()
  g.manual_seed(11)
  ts = env._start_frames(torch.rand(20000, generator=g)).numpy()
  assert ts.min() >= 0 and ts.max() <= T - 1
  # frame f collects the mass of [f, f + 1) under the piecewise-uniform density over (bin + frac) / B (T - 1)
  edges = np.arange(T + 1, dtype=float)
  cdf_pos = np.interp(np.clip(edges * B / (T - 1), 0, B), np.arange(B + 1), np.concatenate([[0], np.cumsum(p)]))
  expect = np.diff(cdf_pos)[: T - 1]
  expect[-1] += 1 - expect.sum()
  obs = np.bincount(ts, minlength=T)[: T - 1]
  # groups of 20 frames
  og = np.add.reduceat(obs, np.arange(0, T - 1, 20))
  eg = np.add.reduceat(expect, np.arange(0, T - 1, 20)) * len(ts)
  assert eg.min() > 20
  assert chisquare(og, eg).pvalue > 1e-3
  env.close()


# ---- the env: kernels against the torch path -----------------------------------------------------------------------
def test_adaptive_sampler_kernels_match_torch_reference(clip, monkeypatch):
  """The tracking env on a moving clip with adaptive start frames (20 bins, a 3-wide kernel, a fast EMA): the fused
  kernels + b2_trackenv_bins against the torch path on the same uniforms, over terminations (forced falls),
  time-outs and clip restarts."""
  n = 6
  cfg = dict(num_envs=n, episode_length_s=0.06, push_interval_s=(0.01, 0.05), motion_file=clip,
             adaptive_kernel_size=3, adaptive_alpha=0.3)
  a = _emul_env(monkeypatch, native_mdp=False, **cfg)
  b = _emul_env(monkeypatch, native_mdp=True, **cfg)
  assert a.T == FRAMES and a.bin_count == 20 and torch.equal(a.time_steps, b.time_steps)
  assert torch.equal(a.sim.data.qpos[:], b.sim.data.qpos[:])
  g = torch.Generator()
  g.manual_seed(5)
  S = 13 + a.nu
  events = dict(term=0, trunc=0, ended=0, draws=0)
  for k in range(10):
    act = torch.rand((n, a.nu), generator=g) * 2 - 1
    if k in (1, 4, 6):  # falls: the anchor drops below the clip's by more than 0.25 m
      for e in (a, b):
        e.sim.data.qpos[k % n, 2] -= 0.4
    if k in (3, 7):  # an env at the clip's last frame runs off its end
      for e in (a, b):
        e.time_steps[(k + 2) % n] = FRAMES - 1
    cdf0, ts0 = a._cdf.clone(), a.time_steps.clone()
    oa, ra, ta, ua, xa = a.step(act)
    ob, rb, tb, ub, xb = b.step(act)
    assert torch.equal(ta, tb) and torch.equal(ua, ub), (k, ta, tb, ua, ub)
    done = ta | ua
    # no draw of this step came within 1e-6 of a CDF step, where the two CDFs could disagree by rounding
    u = torch.cat([b._U[done, 0], b._U[b._done_buf & ~done, S]])
    if len(u):
      assert (u[:, None] - cdf0[None, :]).abs().min() > 1e-6, k
    assert torch.equal(a.time_steps, b.time_steps), (k, a.time_steps, b.time_steps)
    assert torch.allclose(a.bin_failed_count, b.bin_failed_count, atol=1e-6, rtol=0), k
    assert torch.allclose(a._cdf, b._cdf, atol=1e-6, rtol=0), (k, (a._cdf - b._cdf).abs().max())
    for m in ("sampling_entropy", "sampling_top1_prob", "sampling_top1_bin"):
      assert abs(float(xa[m]) - float(xb[m])) <= 1e-6, (k, m, xa[m], xb[m])
    assert torch.allclose(ra, rb, atol=2e-5), (k, ra, rb)
    assert torch.allclose(oa, ob, atol=1e-4), (k, (oa - ob).abs().max())
    assert torch.allclose(xa["critic"], xb["critic"], atol=1e-4), (k, (xa["critic"] - xb["critic"]).abs().max())
    events["term"] += int(ta.sum()); events["trunc"] += int(ua.sum())
    events["ended"] += int((b._done_buf & ~done).sum()); events["draws"] += len(u)
    for f in ("qpos", "qvel", "qacc_warmstart", "ctrl"):  # resynchronise: the MDP logic is what is under test
      getattr(b.sim.data, f)[:] = getattr(a.sim.data, f)[:]
  assert all(v > 0 for v in events.values()), events
  # the failures moved the distribution away from uniform
  assert float(a.bin_failed_count.sum()) > 0 and float(xb["sampling_entropy"]) < 1.0
  a.close()
  b.close()


def test_disabled_adaptive_sampling_starts_every_episode_at_frame_zero(clip, monkeypatch):
  for native_mdp in (False, True):
    e = _emul_env(monkeypatch, num_envs=3, episode_length_s=0.06, motion_file=clip,
                  disable_adaptive_sampling=True, native_mdp=native_mdp)
    assert (e.time_steps == 0).all()
    resets = 0
    for k in range(4):
      e.sim.data.qpos[k % 3, 2] -= 0.4
      _, _, t, u, x = e.step(torch.zeros(3, e.nu))
      d = t | u
      resets += int(d.sum())
      assert (e.time_steps[d] == 1).all()  # frame 0, then this step's advance
      assert "sampling_entropy" not in x
    assert resets > 0
    e.close()


def test_without_a_motion_file_the_sampler_fields_are_zero(monkeypatch):
  """motion_file=None: the argument block's sampler fields are all zero, and a run with those fields zeroed explicitly
  gives bit-identical outputs."""
  cfg = dict(num_envs=3, decimation=1, episode_length_s=0.015, clip_frames=4, native_mdp=True)
  a = _emul_env(monkeypatch, **dict(cfg))
  b = _emul_env(monkeypatch, **dict(cfg))
  a._native_setup()
  b._native_setup()
  A = b._native_args
  first, last = native.B2TrackEnvArgs.adaptive_kernel, native.B2TrackEnvArgs.adaptive_kernel_size
  ctypes.memset(ctypes.addressof(A) + first.offset, 0, last.offset + last.size - first.offset)
  for f in ("adaptive_kernel", "cdf", "bin_fail_ema", "bin_fail_cur", "metrics", "adaptive_alpha",
            "adaptive_uniform_ratio", "nbins", "adaptive", "adaptive_kernel_size"):
    assert not getattr(a._native_args, f), f
  g = torch.Generator()
  g.manual_seed(1)
  for k in range(5):
    act = torch.rand((3, a.nu), generator=g) * 2 - 1
    oa, ra, ta, ua, xa = a.step(act)
    ob, rb, tb, ub, xb = b.step(act)
    assert set(xa) == {"critic"}
    assert torch.equal(oa, ob) and torch.equal(ra, rb) and torch.equal(xa["critic"], xb["critic"])
    assert torch.equal(a.time_steps, b.time_steps) and torch.equal(ta | ua, tb | ub)
  a.close()
  b.close()

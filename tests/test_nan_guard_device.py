"""The NaN guard on the device (b2_nan_guard, csrc/b2_nanguard.cuh; mjlab_b200/utils/nan_guard.py).

* Host emulation: the dump of the device guard, armed under ``step_n(4)`` calls with a NaN written into one world's
  qpos between calls, is bit-equal to that of the host algorithm the guard replaces (restated below: record the first
  ``ncapture`` worlds, step one sub-step, check every world), with the ring wrapping, ``max_envs_to_capture`` above
  the number of worlds, and the two stream partitions of b2_step_n (2048 worlds, the NaN in the second); a second NaN
  after the dump writes nothing.  Never armed and armed-then-disarmed launch the same kernels and step to the same
  bits, and an armed guard that finds nothing changes no state.  The C entries refuse bad arguments.  The fused
  velocity and tracking envs run with the guard and a NaN written into one world's qvel, and dump by ``close()``.
* H100: ``Simulation.step()`` and ``step_n`` dump the same bits at 64 and 4096 worlds; the fused envs through their
  CUDA graph dump what they dump without it; an armed guard changes no output of 50 env steps.

The NaN is only ever written into plane / primitive models: on a static-grid or height-field model a NaN position
would become a cell index.
"""

import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from mjlab_b200.compiler import Spec
from mjlab_b200.sim import native
from mjlab_b200.utils.nan_guard import NanGuard, NanGuardCfg

sys.path.insert(0, str(Path(__file__).parent / "emul"))

BOX_XML = """
<mujoco>
  <worldbody>
    <geom name="floor" type="plane" size="5 5 0.1"/>
    <body name="box" pos="0 0 1">
      <freejoint name="free"/>
      <geom name="box_geom" type="box" size="0.1 0.1 0.1" mass="1.0"/>
    </body>
  </worldbody>
</mujoco>
"""


@pytest.fixture(scope="module")
def box():
  return Spec.from_string(BOX_XML).compile()


@pytest.fixture(scope="module")
def lib():
  from engine import load_emul_library

  return load_emul_library()


def _engine(lib, model, n, seed=0):
  """An emulated sim with seeded velocities: boxes tumbling down onto the floor."""
  from test_kernel_emul import EmulSim

  e = EmulSim(lib, model, n)
  rng = np.random.default_rng(seed)
  e.field("qvel")[:] = rng.uniform(-2.0, 2.0, e.field("qvel").shape).astype(np.float32)
  e.field("qpos")[:, 2] = rng.uniform(0.12, 0.6, n).astype(np.float32)
  e.forward()
  return e


def _load(path) -> dict:
  z = np.load(path)
  return {k: z[k] for k in z.files}


def _assert_same_dump(a: dict, b: dict) -> None:
  assert sorted(a) == sorted(b)
  for k in a:
    assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
    assert a[k].tobytes() == b[k].tobytes(), k


class HostGuard:
  """The host algorithm the device guard replaces (the reference's utils/nan_guard.py): before every sub-step, record
  qpos / qvel of the first ``ncapture`` worlds, keeping the last ``buffer_size``; after it, check every world; dump
  once, at the first sub-step with a non-finite value."""

  def __init__(self, engine, nworld, cfg: NanGuardCfg):
    self.e, self.cfg = engine, cfg
    self.n = min(nworld, cfg.max_envs_to_capture)
    self.buffer, self.step, self.dump = [], 0, None

  def sub_step(self):
    q, v = self.e.field("qpos"), self.e.field("qvel")
    self.buffer = (self.buffer + [(self.step, q[:self.n].copy(), v[:self.n].copy())])[-self.cfg.buffer_size:]
    self.step += 1
    assert self.e.lib.b2_step(self.e.h, None) == 0
    bad = np.zeros(self.e.n, bool)
    for f in ("qpos", "qvel", "qacc", "qacc_warmstart"):
      bad |= ~np.isfinite(self.e.field(f)).all(axis=1)
    if self.dump is None and bad.any():
      self.dump = {"nan_env_ids": np.flatnonzero(bad), "num_envs_captured": np.asarray(self.n)}
      for k, qk, vk in self.buffer:
        self.dump[f"qpos_step_{k:06d}"], self.dump[f"qvel_step_{k:06d}"] = qk, vk


def _guarded(lib, model, n, cfg):
  e = _engine(lib, model, n)
  return e, NanGuard(cfg, e, model, lambda: ctypes.c_void_p(0))


# (worlds, max_envs_to_capture, buffer_size, step_n(4) calls before the NaN, world of the NaN)
CASES = {
  "plain": (6, 5, 100, 2, 1),
  "ring_wraps": (6, 3, 3, 3, 4),
  "capture_above_nworld": (4, 10, 5, 1, 0),
  "two_partitions": (2048, 5, 2, 1, 1500),
}


@pytest.mark.parametrize("case", CASES)
def test_dump_matches_the_host_algorithm(case, lib, box, tmp_path):
  n, ncap, bsize, before, bad_world = CASES[case]
  cfg = NanGuardCfg(enabled=True, buffer_size=bsize, max_envs_to_capture=ncap, output_dir=str(tmp_path))
  dev, guard = _guarded(lib, box, n, cfg)
  host = HostGuard(_engine(lib, box, n), n, cfg)
  def call():
    assert lib.b2_step_n(dev.h, 4, None) == 0
    for _ in range(4):
      host.sub_step()
    return guard.poll()  # (the emulation runs the call before returning: the word is already set)

  for _ in range(before):
    assert not call()
  for e in (dev, host.e):
    e.field("qpos")[bad_world, 0] = np.nan
  assert call()
  assert host.dump is not None
  dumps = list(tmp_path.glob("nan_dump_*.npz"))
  assert len(dumps) == 1 and str(dumps[0]) == guard.last_dump_path
  got = _load(dumps[0])
  _assert_same_dump(got, host.dump)
  assert bad_world in got["nan_env_ids"] and int(got["num_envs_captured"]) == min(n, ncap)
  assert len([k for k in got if k.startswith("qpos_step_")]) == min(bsize, 4 * before + 1)
  # a second NaN in another world after the dump: the guard has fired, nothing more is written
  dev.field("qvel")[(bad_world + 1) % n, 3] = np.inf
  assert lib.b2_step_n(dev.h, 4, None) == 0
  assert not guard.poll() and not guard.check_and_dump()
  assert len(list(tmp_path.glob("nan_dump_*.npz"))) == 1
  dev.close()
  host.e.close()


def test_a_sub_step_at_a_time_dumps_what_step_n_dumps(lib, box, tmp_path):
  """b2_step per sub-step and b2_step_n number the sub-steps alike."""
  dumps = []
  for single in (True, False):
    out = tmp_path / str(single)
    e, guard = _guarded(lib, box, 6, NanGuardCfg(enabled=True, buffer_size=6, output_dir=str(out)))
    for k in range(3):
      if k == 2:
        e.field("qpos")[2, 1] = np.nan
      if single:
        for _ in range(4):
          assert lib.b2_step(e.h, None) == 0
      else:
        assert lib.b2_step_n(e.h, 4, None) == 0
    assert guard.check_and_dump()
    dumps.append(_load(guard.last_dump_path))
    e.close()
  _assert_same_dump(*dumps)
  assert sorted(k for k in dumps[0] if k.startswith("qpos")) == [f"qpos_step_{k:06d}" for k in range(3, 9)]


def test_disarmed_is_free_and_armed_only_reads(lib, box):
  never, disarmed, armed = (_engine(lib, box, 6) for _ in range(3))
  assert lib.b2_nan_guard(disarmed.h, 5, 10, native.NAN_GUARD_ON) == 0
  assert lib.b2_nan_guard(disarmed.h, 0, 0, 0) == 0
  assert lib.b2_nan_guard_word(disarmed.h) is None
  assert lib.b2_nan_guard(armed.h, 5, 10, native.NAN_GUARD_ON) == 0
  counts = [lib.b2_launch_count(e.h) for e in (never, disarmed, armed)]
  assert counts[0] == counts[1] == counts[2]
  for _ in range(3):
    for e in (never, disarmed, armed):
      assert lib.b2_step_n(e.h, 4, None) == 0 and lib.b2_step(e.h, None) == 0
  grown = [lib.b2_launch_count(e.h) - c for e, c in zip((never, disarmed, armed), counts)]
  # armed: one start kernel per call and one check kernel per sub-step
  assert grown[0] == grown[1] and grown[2] == grown[0] + 3 * ((1 + 4) + (1 + 1))
  for f in ("qpos", "qvel", "qacc", "qacc_warmstart", "time"):
    a = never.field(f).tobytes()
    assert disarmed.field(f).tobytes() == a and armed.field(f).tobytes() == a, f
  d = ctypes.c_int64()
  assert lib.b2_nan_guard_read(armed.h, None, ctypes.byref(d), None, None) == 0 and d.value == -1
  assert ctypes.c_int32.from_address(lib.b2_nan_guard_word(armed.h)).value == 0
  for e in (never, disarmed, armed):
    e.close()


def test_c_entry_refusals(lib, box):
  e = _engine(lib, box, 4)

  def refused(rc, match):
    assert rc != 0 and match in lib.b2_last_error().decode(), lib.b2_last_error()

  refused(lib.b2_nan_guard(None, 1, 1, native.NAN_GUARD_ON), "null sim")
  for ncap, bsize in ((0, 5), (5, 5), (-1, 5), (1, 0), (4, -3)):
    refused(lib.b2_nan_guard(e.h, ncap, bsize, native.NAN_GUARD_ON), "1 <= ncapture <= nworld (4) and buffer_size >= 1")
  refused(lib.b2_nan_guard(e.h, 1, 1, 2), "flags must be 0 or B2_NAN_GUARD_ON")
  refused(lib.b2_nan_guard(e.h, 4, 2**31 - 8, native.NAN_GUARD_ON), "too large")
  d = ctypes.c_int64()
  refused(lib.b2_nan_guard_read(e.h, None, ctypes.byref(d), None, None), "not armed")
  assert lib.b2_nan_guard(e.h, 4, 1, native.NAN_GUARD_ON) == 0
  refused(lib.b2_nan_guard_read(e.h, None, None, None, None), "bad arguments")
  refused(lib.b2_nan_guard_read(None, None, ctypes.byref(d), None, None), "bad arguments")
  assert lib.b2_nan_guard_word(None) is None
  e.close()


# ---- the fused environments -----------------------------------------------------------------------------------------
NAN_STEP = 3  # qvel[n - 3, 0] = NaN before this env step (in the second partition at 4096 envs)


def _env_run(kind, device, steps, graph, nan, out_dir, n):
  """`steps` seeded env steps of the G1 flat velocity (B) or tracking (C) env with the guard on; with `nan`, a NaN is
  written into world n - 3's qvel before step NAN_STEP.  With `graph` the steps replay the env's CUDA graph; without,
  the env still runs enable_cuda_graph's warm-up steps (on the GPU), so that both start from the same state.  Returns
  the outputs of every step and the env."""
  import dataclasses

  from mjlab_b200.envs import tracking_env as te
  from mjlab_b200.envs import velocity_env as ve

  guard = NanGuardCfg(enabled=True, buffer_size=6, max_envs_to_capture=3, output_dir=str(out_dir))
  cfg = (ve.VelocityEnvCfg if kind == "B" else te.TrackingEnvCfg)(num_envs=n, seed=5)
  cfg = dataclasses.replace(cfg, sim=dataclasses.replace(cfg.sim, nan_guard=guard))
  env = (ve.VelocityFlatEnv if kind == "B" else te.TrackingFlatEnv)(cfg, device=device, native_mdp=True)
  if device != "cpu":
    env.enable_cuda_graph()
    if not graph:
      env._graph = None
  g = torch.Generator(device=device).manual_seed(1)
  outs = []
  for k in range(steps):
    if nan and k == NAN_STEP:
      env.sim.data.qvel[n - 3, 0] = float("nan")
    a = torch.rand((n, env.nu), generator=g, device=device) * 2 - 1
    outs.append([t.clone() if torch.is_tensor(t) else {k2: v.clone() for k2, v in t.items()} for t in env.step(a)])
  return outs, env


class GuardedEmulSimulation:
  """The emulated Simulation stand-in of the env tests (tests/test_kernel_emul.py) with the device guard, as
  Simulation runs it: checked by the env's poll after each step and once more at close."""

  def __new__(cls, num_envs, cfg, model, device):
    from test_kernel_emul import EmulSimulation

    sim = EmulSimulation(num_envs, cfg, model, device)
    sim.nan_guard = NanGuard(cfg.nan_guard, sim._e, model, sim._stream)
    close = sim.close

    def closing():
      sim.nan_guard.check_and_dump()
      close()

    sim.close = closing
    return sim


@pytest.mark.parametrize("kind", ["B", "C"])
def test_fused_env_with_a_nan_dumps_on_the_emulation(kind, monkeypatch, tmp_path):
  """The NaN-injected env sequence of the H100 test below on the host emulation: it runs, and the env dumps."""
  from mjlab_b200.envs import tracking_env as te
  from mjlab_b200.envs import velocity_env as ve

  monkeypatch.setattr(ve if kind == "B" else te, "Simulation", GuardedEmulSimulation)
  monkeypatch.setattr(native, "check", lambda rc: (_ for _ in ()).throw(RuntimeError("b2sim call failed")) if rc else None)
  _, env = _env_run(kind, "cpu", NAN_STEP + 2, False, True, tmp_path, 4)
  env.close()
  dumps = list(tmp_path.glob("nan_dump_*.npz"))
  assert len(dumps) == 1
  z = _load(dumps[0])
  assert z["nan_env_ids"].tolist() == [1] and int(z["num_envs_captured"]) == 3
  assert np.isnan(z[max(k for k in z if k.startswith("qvel_step_"))][1, 0])


# ---- H100 -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [64, 4096])
def test_sim_step_and_step_n_dump_the_same(n, box, tmp_path):
  from mjlab_b200.sim import Simulation, SimulationCfg

  dumps = []
  for single in (True, False):
    out = tmp_path / str(single)
    cfg = SimulationCfg(nan_guard=NanGuardCfg(enabled=True, buffer_size=10, output_dir=str(out)))
    sim = Simulation(n, cfg, box, "cuda:0")
    g = torch.Generator(device="cuda:0").manual_seed(2)
    sim.data.qvel[:] = torch.rand(sim.data.qvel[:].shape, generator=g, device="cuda:0") * 4 - 2
    sim.forward()
    for k in range(4):
      if k == 3:
        sim.data.qpos[n - 3, 0] = float("nan")  # (in the second partition at 4096 worlds)
      if single:
        for _ in range(4):
          sim.step()
      else:
        sim.step_n(4)
    dumps.append(_load(sim.nan_guard.last_dump_path))
    assert len(list(out.glob("*.npz"))) == 1
    sim.close()
  _assert_same_dump(*dumps)
  assert dumps[0]["nan_env_ids"].tolist() == [n - 3]
  assert sorted(k for k in dumps[0] if k.startswith("qpos")) == [f"qpos_step_{k:06d}" for k in range(3, 13)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["B", "C"])
def test_fused_env_under_a_graph_dumps_what_it_dumps_without(kind, tmp_path):
  dumps = []
  for graph in (True, False):
    out = tmp_path / str(graph)
    _, env = _env_run(kind, "cuda:0", NAN_STEP + 2, graph, True, out, 4096)
    env.close()
    files = list(out.glob("nan_dump_*.npz"))
    assert len(files) == 1
    dumps.append(_load(files[0]))
  _assert_same_dump(*dumps)
  assert dumps[0]["nan_env_ids"].tolist() == [4096 - 3]


@pytest.mark.gpu
def test_armed_guard_changes_no_output(tmp_path):
  """50 seeded env steps of the G1 flat velocity env through its graph, guard on and off: bit-identical outputs."""
  from mjlab_b200.envs import VelocityEnvCfg, VelocityFlatEnv

  on, env = _env_run("B", "cuda:0", 50, True, False, tmp_path, 4096)
  env.close()
  ref = VelocityFlatEnv(VelocityEnvCfg(num_envs=4096, seed=5), device="cuda:0", native_mdp=True)
  ref.enable_cuda_graph()
  g = torch.Generator(device="cuda:0").manual_seed(1)
  for k in range(50):
    got = ref.step(torch.rand((4096, ref.nu), generator=g, device="cuda:0") * 2 - 1)
    for a, b in zip(on[k], got):
      if torch.is_tensor(a):
        assert torch.equal(a, b), k
      else:
        assert all(torch.equal(a[key], b[key]) for key in a), k
  ref.close()
  assert not list(tmp_path.glob("*.npz"))

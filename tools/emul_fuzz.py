"""Fuzz the fused kernel on the host emulation (tests/emul) against the oracle with synthetic robots.

  python tools/emul_fuzz.py [--seeds 5] [--limbs 5] [--joints 8] [--worlds 2] [--steps 2]
  python tools/emul_fuzz.py --scene obstacle [--seeds 6]      # free primitives among static boxes (grid + box routines)

Each seed builds a floating base with `limbs` chains of up to `joints` hinge joints (random axes, limits, capsule
links; nv <= 64, nbody <= 64), drops it on a plane in a random pose (self-collisions included), and compares one
forward pass and a few resynchronised steps of the emulated CUDA sources with the fp64 oracle.  No GPU needed;
functional check only."""
import argparse
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tests"), str(ROOT / "tests" / "emul")]

from mjlab_b200.compiler import Spec  # noqa: E402
from oracle.oracle import Oracle  # noqa: E402
from synth_models import robot_xml  # noqa: E402
from test_kernel_emul import EmulSim, _load  # noqa: E402
from util import relerr  # noqa: E402


def obstacle_runs(lib, seeds, worlds, steps, keep_going=False):
  """Free spheres / capsules / boxes in random orientations among 20+ static boxes, spheres and capsules on a plane
  (tests/test_boxes_terrain.py: obstacle_course_xml): pair table + static grid + every primitive pair type."""
  from test_boxes_terrain import obstacle_course_xml

  bad = []
  for seed in range(1, seeds + 1):
    m = Spec.from_string(obstacle_course_xml(seed=seed, nobst=20 + min(seed, 40), nobj=9)).compile()
    n = worlds
    sim = EmulSim(lib, m, n, ncon=96)
    o = Oracle(m, nworld=n, maxcon=int(sim.option("maxcon")), njmax=2000)
    rng = np.random.default_rng(seed)
    q = np.tile(m.qpos0, (n, 1))
    q += rng.uniform(-0.08, 0.08, q.shape) * (np.arange(q.shape[1]) % 7 < 3)
    q[:, 2::7] -= rng.uniform(0.3, 0.45)
    for b in range(q.shape[1] // 7):
      v = rng.normal(size=(n, 4))
      q[:, 7 * b + 3 : 7 * b + 7] = v / np.linalg.norm(v, axis=1, keepdims=True)
    st = dict(qpos=q, qvel=rng.uniform(-0.5, 0.5, (n, int(m.nv))))
    for k, v in st.items():
      o.field(k)[:] = v
    sim.load(st)
    worst, seen = 0.0, 0
    for _ in range(max(steps, 1) + 3):
      o.forward()
      sim.forward()
      if not (sim.field("ncon").ravel() == o.ncon.ravel()).all():
        # (a capsule lying along a box face reports one contact or one per end depending on which side of the
        # 1e-3 r length threshold the bisection lands: a tie of the rule, not an arithmetic difference)
        assert keep_going, (seed, sim.field("ncon").ravel(), o.ncon.ravel())
        bad.append(seed)
        break
      worst = max(worst, float(relerr(sim.field("qacc"), o.qacc, floor=10.0).max()))
      seen = max(seen, int(o.ncon.max()))
      o.step()
      sim.step(1)
      for f in ("qpos", "qvel", "qacc_warmstart"):
        sim.field(f)[...] = getattr(o, f)
    print(f"seed {seed}: nstatic={int(m.nstatic)} npair={int(m.npair)} max ncon {seen} worst qacc rel err {worst:.2e}")
    assert worst < 1e-2, seed  # (capsule-box contact ends are defined to ~1e-3 m)
    sim.close()
  print("ok" if not bad else f"contact-count ties in seeds {bad}")
  return bad


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--scene", choices=["robot", "obstacle"], default="robot")
  ap.add_argument("--seeds", type=int, default=5)
  ap.add_argument("--limbs", type=int, default=5)
  ap.add_argument("--joints", type=int, default=8)
  ap.add_argument("--worlds", type=int, default=2)
  ap.add_argument("--steps", type=int, default=2)
  ap.add_argument("--first", type=int, default=0, help="first seed")
  ap.add_argument("--keep-going", action="store_true", help="report every failing seed instead of stopping at the first")
  a = ap.parse_args()
  lib = _load()
  if a.scene == "obstacle":
    return obstacle_runs(lib, a.seeds, a.worlds, a.steps, a.keep_going)
  worst, bad = 0.0, []
  for seed in range(a.first, a.first + a.seeds):
    rng = np.random.default_rng(seed)
    m = Spec.from_string(robot_xml(rng, a.limbs, a.joints)).compile()
    n, nv = a.worlds, int(m.nv)
    sim = EmulSim(lib, m, n, ncon=96)
    o = Oracle(m, nworld=n, maxcon=int(sim.option("maxcon")), njmax=2000)  # (the engine never truncates at njmax)
    q = np.tile(m.qpos0, (n, 1))
    q[:, 2] += rng.uniform(-0.3, 0.3, n)
    q[:, 7:] += rng.uniform(-1.0, 1.0, (n, int(m.nq) - 7))
    st = dict(qpos=q, qvel=rng.uniform(-1, 1, (n, nv)), qacc_warmstart=rng.uniform(-1, 1, (n, nv)))
    if int(m.nu):
      st["ctrl"] = rng.uniform(-1, 1, (n, int(m.nu)))
    for k, v in st.items():
      o.field(k)[:] = v
    sim.load(st)
    o.forward()
    sim.forward()
    if not (sim.field("ncon").ravel() == o.ncon.ravel()).all() or not (sim.field("nefc").ravel() == o.nefc.ravel()).all():
      print(f"seed {seed}: contact / row counts differ: {sim.field('ncon').ravel().tolist()} vs {o.ncon.ravel().tolist()}")
      assert a.keep_going, seed
      bad.append((seed, "counts"))
      sim.close()
      continue
    e = float(relerr(sim.field("qacc"), o.qacc, floor=10.0).max())
    for _ in range(a.steps):
      o.step()
      sim.step(1)
      e = max(e, float(relerr(sim.field("qvel"), o.qvel).max()))
      for f in ("qpos", "qvel", "qacc_warmstart"):
        sim.field(f)[...] = getattr(o, f)
    worst = max(worst, e)
    print(f"seed {seed}: nv={nv} nbody={int(m.nbody)} npair={int(m.npair)} ncon={o.ncon.ravel().tolist()} "
          f"integrator={'Euler' if int(m.opt_integrator) == 0 else 'implicitfast'} max rel err {e:.2e}")
    if e >= 3e-3:
      assert a.keep_going, seed
      bad.append((seed, e))
    sim.close()
  print(f"{'ok' if not bad else 'FAILED ' + str(bad)}: worst relative error {worst:.2e} over {a.seeds} seeds")
  return bad


if __name__ == "__main__":
  main()

"""The step kernel on the H100 against the fp64 oracle at the model sizes, joint layouts and solver paths that the
asset-zoo models never reach: nv and nbody past one warp's 32 lanes and up to the 64 that b2_create accepts, more than
32 actuators (motor, velocity and position, gear != 1, ctrllimited), bodies with several joints (the generic
kinematics walk), more than 32 limit rows and more than 64 contacts (the line-search rows outside the register
window), the reduced and full Newton problems, the tree and dense factorisation schedules, and the independence of
a world from its neighbours in the 4-warp CTA.

The models come from tools/synth_models.py (the generator tools/emul_fuzz.py fuzzes on the host emulation), so the
tolerances are those of the emulated counterparts; every case asserts the size or path it exists for, so that a
change to the generator cannot make it vacuous."""

import functools
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from util import load_oracle, load_sim, make_states, relerr

sys.path.append(str(Path(__file__).resolve().parents[1] / "tools"))
from synth_models import robot_xml  # noqa: E402

pytestmark = pytest.mark.gpu

EFC_LIMIT = 3  # oracle efc_type of a joint-limit row

# name: (seed, limbs, joints, generator options)
MODELS = {
  "nv32": (1, 4, 10, dict(dofs=26)),
  "nv33_nbody33": (1, 4, 10, dict(dofs=27, feet=True)),
  "nv64_nbody64": (2, 4, 18, dict(dofs=58, feet=True)),
  "nu33": (1, 5, 9, dict(dofs=33, actuate_all=True, unlimited=True, offsets=True)),
  "nu58": (1, 6, 12, dict(dofs=58, actuate_all=True)),
  "multijoint": (2, 5, 5, dict(dofs=38, joints_per_body=3, offsets=True, actuate_all=True)),
  "nv37": (1, 5, 8, dict(dofs=31)),
  "boxes": (1, 6, 8, dict(dofs=50, box_links=True)),
}

# what each model of the shape matrix exists for
SHAPES = {
  "nv32": dict(nv=32),
  "nv33_nbody33": dict(nv=33, nbody=33),
  "nv64_nbody64": dict(nv=64, nbody=64),  # (b2_create refuses more)
  "nu33": dict(nu=33),
  "nu58": dict(nu=58),
  "multijoint": dict(max_body_joints=3),
}


@functools.cache
def _model(name):
  from mjlab_b200.compiler import Spec

  seed, limbs, joints, kw = MODELS[name]
  return Spec.from_string(robot_xml(np.random.default_rng(seed), limbs, joints, **kw)).compile()


def _sim(model, n, nconmax=None):
  from mjlab_b200.sim import Simulation, SimulationCfg

  sim = Simulation(n, SimulationCfg(nconmax=nconmax), model, "cuda:0")
  sim.set_option("debug_outputs", 1)  # (qacc_smooth and qfrc_constraint are written)
  return sim


def _oracle(model, n, sim, precision="f64"):
  from oracle.oracle import Oracle

  return Oracle(model, nworld=n, maxcon=int(sim.get_option("maxcon")), njmax=3000, precision=precision)


def F(sim, name):
  return getattr(sim.data, name)[:].detach().cpu().numpy()


def _depth(model):
  parent = np.asarray(model.body_parentid)
  d = np.zeros(len(parent), int)
  for b in range(1, len(parent)):
    d[b] = d[parent[b]] + 1
  return int(d.max())


def _states(model, n, seed, lift=True):
  """tools/emul_fuzz.py's random states (base height +-0.3 m, joints +-1 around qpos0, random velocities, warm
  starts and controls).  With `lift`, every third world is lifted clear of the floor with its joints nearer qpos0
  and its limited joints inside their ranges, so that CTAs mix warps with no constraint rows and heavy ones.  Returns the states and that mask."""
  rng = np.random.default_rng(seed)
  nq, nv, nu = int(model.nq), int(model.nv), int(model.nu)
  q = np.tile(np.asarray(model.qpos0, np.float64), (n, 1))
  q[:, 2] += rng.uniform(-0.3, 0.3, n)
  q[:, 7:] += rng.uniform(-1.0, 1.0, (n, nq - 7))
  st = dict(qpos=q, qvel=rng.uniform(-1, 1, (n, nv)), qacc_warmstart=rng.uniform(-1, 1, (n, nv)))
  if nu:
    st["ctrl"] = rng.uniform(-1, 1, (n, nu))
  up = np.zeros(n, bool)
  if lift:
    up[2::3] = True
    q[up, 2] = 0.3 + 0.15 * _depth(model)  # (every link is shorter than 0.15 m)
    q[up, 7:] = model.qpos0[7:] + 0.3 * (q[up, 7:] - model.qpos0[7:])  # (few self-contacts)
    rg, lim, qa = np.asarray(model.jnt_range), np.asarray(model.jnt_limited), np.asarray(model.jnt_qposadr)
    for j in np.nonzero(lim)[0]:
      q[up, qa[j]] = np.clip(q[up, qa[j]], 0.8 * rg[j, 0], 0.8 * rg[j, 1])
  return st, up


def _pair(model, n, st, nconmax=None):
  sim = _sim(model, n, nconmax)
  o = _oracle(model, n, sim)
  load_oracle(o, st)
  load_sim(sim, st)
  return sim, o


def _check_forward(sim, o, n, smooth_tol=1e-4):
  """tests/test_kernel_emul.py's _check_forward on the GPU: identical contact sets and row counts, kinematics,
  inertia, bias and actuator forces to 1e-5, the unconstrained acceleration to `smooth_tol` (1e-4, or per world),
  qacc to 1e-3 (floor 10)."""
  nc = o.ncon.ravel()
  assert (F(sim, "ncon").ravel() == nc).all(), np.nonzero(F(sim, "ncon").ravel() != nc)
  assert (F(sim, "nefc").ravel() == o.nefc.ravel()).all(), np.nonzero(F(sim, "nefc").ravel() != o.nefc.ravel())
  cg, og = F(sim, "contact_geom"), o.contact_geom.reshape(n, -1, 2)
  cd = F(sim, "contact_dist")
  for w in range(n):
    assert (cg[w, : nc[w]] == og[w, : nc[w]]).all(), w
    if nc[w]:
      assert np.abs(cd[w, : nc[w]] - o.contact_dist[w, : nc[w]]).max() < 1e-5, w
  tight = ["xpos", "xquat", "xmat", "xipos", "subtree_com", "cvel", "geom_xpos", "geom_xmat", "qfrc_bias",
           "qfrc_smooth", "qM"] + (["actuator_force"] if int(o.model.nu) else [])
  for f in tight:
    e = relerr(F(sim, f).reshape(n, -1), o.field(f).reshape(n, -1))
    assert e.max() < 1e-5, (f, int(e.argmax()), e.max())
  e = relerr(F(sim, "qacc_smooth"), o.qacc_smooth)
  assert (e < smooth_tol).all(), ("qacc_smooth", int((e / smooth_tol).argmax()), e.max())
  e = relerr(F(sim, "qacc"), o.qacc, floor=10.0)
  assert e.max() < 1e-3, ("qacc", int(e.argmax()), e.max())


@pytest.mark.parametrize("n", [128, 130])  # phase-synchronous CTAs; a partial last CTA
@pytest.mark.parametrize("name", list(SHAPES))
def test_shape_matrix_matches_the_oracle(name, n):
  """One forward, one step, then three steps resynchronised to the oracle, for each size of the shape matrix."""
  m = _model(name)
  shape = dict(nv=int(m.nv), nbody=int(m.nbody), nu=int(m.nu), max_body_joints=int(np.max(m.body_jntnum)))
  for k, v in SHAPES[name].items():
    assert shape[k] == v, (k, shape)
  if name == "multijoint":
    # b2_create keeps the compact one-joint kinematic records (fastkin) only when no body has two joints: this model
    # takes the generic walk, with hinges and slides mixed on a body and anchors off the body origin
    jt = np.asarray(m.jnt_type)
    assert (jt == 2).any() and (jt == 3).any() and np.abs(np.asarray(m.jnt_pos)).max() > 0.005
  if SHAPES[name].get("nu"):
    # motor, velocity and position actuators with gears off 1, control-limited; implicitfast adds the velocity
    # actuators' derivative to the implicit matrix (a second trip of that lane loop too)
    bias = np.asarray(m.actuator_biasprm).reshape(-1, 10)
    position, velocity = bias[:, 1] != 0, (bias[:, 1] == 0) & (bias[:, 2] != 0)
    assert position.any() and velocity.any() and (~position & ~velocity).any()  # (the rest are motors)
    gear = np.asarray(m.actuator_gear).ravel()
    assert np.asarray(m.actuator_ctrllimited).all() and gear.min() < 0.9 and gear.max() > 1.1
    assert int(m.opt_integrator) == 3
  st, up = _states(m, n, seed=7 + n)
  sim, o = _pair(m, n, st, nconmax=96 * n)
  o.forward()
  sim.forward()
  torch.cuda.synchronize()
  nefc = o.nefc.ravel()
  assert (nefc[up] == 0).sum() >= n // 12 and (nefc[~up] > 0).sum() >= n // 2, (nefc[up], nefc[~up])
  # M of the 64-dof robot is ill-conditioned for fp32 in a few worlds: the oracle's own fp32 build is up to 5e-5
  # off its fp64 unconstrained acceleration there, and the kernel (another summation order, approximate reciprocals)
  # lands within twice that, just over 1e-4 (measured on an H100).  Such worlds are bounded by 4x the fp32 oracle's
  # error instead
  o32 = _oracle(m, n, sim, precision="f32")
  load_oracle(o32, st)
  o32.forward()
  smooth_tol = np.maximum(1e-4, 4 * relerr(o32.qacc_smooth, o.qacc_smooth))
  _check_forward(sim, o, n, smooth_tol)
  for _ in range(4):
    o.step()
    sim.step()
    torch.cuda.synchronize()
    e = relerr(F(sim, "qvel"), o.qvel)
    assert e.max() < 3e-3, ("qvel", int(e.argmax()), e.max())
    for f in ("qpos", "qvel", "qacc_warmstart"):
      getattr(sim.data, f)[:] = torch.as_tensor(o.field(f), dtype=torch.float32, device=sim.device)
  sim.close()


def test_more_than_32_limit_rows():
  """Every world has 39-58 joints 0.01-0.05 past their limits: the line search reads the limit rows beyond the
  32-lane register window, and the Newton problem has more than 32 limit rows."""
  m = _model("nv64_nbody64")
  n = 128
  st, _ = _states(m, n, seed=3, lift=False)
  rng = np.random.default_rng(4)
  q = st["qpos"]
  q[:, 2] = 0.3 + 0.15 * _depth(m)  # clear of the floor: limit rows dominate
  lim, rg, qa = np.asarray(m.jnt_limited), np.asarray(m.jnt_range), np.asarray(m.jnt_qposadr)
  js = np.nonzero(lim)[0]
  assert len(js) >= 39
  for w in range(n):
    pick = rng.choice(js, size=int(rng.integers(39, len(js) + 1)), replace=False)
    side = rng.integers(0, 2, len(pick))
    past = rng.uniform(0.01, 0.05, len(pick))
    q[w, qa[pick]] = np.where(side == 1, rg[pick, 1] + past, rg[pick, 0] - past)
  sim, o = _pair(m, n, st)
  o.forward()
  sim.forward()
  torch.cuda.synchronize()
  nlim = np.array([(o.efc_type[w, : o.nefc[w, 0]] == EFC_LIMIT).sum() for w in range(n)])
  assert nlim.min() > 32, nlim.min()
  assert (F(sim, "nefc").ravel() == o.nefc.ravel()).all()
  e = relerr(F(sim, "qacc"), o.qacc, floor=10.0)
  assert e.max() < 1e-3, ("qacc", int(e.argmax()), e.max())
  e = relerr(F(sim, "qfrc_constraint"), o.qfrc_constraint)
  assert e.max() < 1e-3, ("qfrc_constraint", int(e.argmax()), e.max())
  sim.close()


@pytest.mark.parametrize("z,lo,hi", [(0.65, 32, 64), (0.52, 64, None)])
def test_more_than_64_contacts(z, lo, hi):
  """A box-link robot hanging into the floor (the submerged links give four box-plane contacts each): 32 < ncon <= 64
  (the second register half of the line search) and ncon > 64 (the rows outside the register window), no overflow."""
  m = _model("boxes")
  n = 128
  rng = np.random.default_rng(11)
  q = np.tile(np.asarray(m.qpos0, np.float64), (n, 1))
  q[:, 2] = z + rng.uniform(-0.02, 0.02, n)
  q[:, 7:] += rng.uniform(-0.03, 0.03, (n, int(m.nq) - 7))
  st = dict(qpos=q, qvel=rng.uniform(-0.5, 0.5, (n, int(m.nv))), ctrl=rng.uniform(-1, 1, (n, int(m.nu))))
  sim, o = _pair(m, n, st, nconmax=128 * n)
  maxcon = int(sim.get_option("maxcon"))
  o.forward()
  sim.forward()
  torch.cuda.synchronize()
  nc = o.ncon.ravel()
  inside = (nc > lo) & (nc < (maxcon if hi is None else hi + 1))
  assert inside.mean() > 0.5 and nc.max() < maxcon, (np.sort(nc), maxcon)
  assert not o.overflow.any() and not F(sim, "overflow").any()
  _check_forward(sim, o, n)
  e = relerr(F(sim, "qfrc_constraint"), o.qfrc_constraint, floor=10.0)
  assert e.max() < 1e-3, ("qfrc_constraint", int(e.argmax()), e.max())
  sim.close()


def _reduced_block_cap(nv):
  """b2sim.cu's rule: the largest leading block nv - 4k (k >= 1, at least 6) whose packed triangle fits 200 floats."""
  for k in range(1, nv):
    c = nv - 4 * k
    if c < 6:
      return 0
    if c * (c + 1) // 2 <= 200:
      return c
  return 0


@pytest.mark.parametrize("name", ["g1_flat", "nv37", "nv64_nbody64"])
def test_reduced_and_full_newton_match_the_oracle(name):
  """The Newton solver on the constrained leading block (Schur complement of M, the rest by back-substitution) and
  on all dofs give the oracle's answer; the leading-block cap depends on nv (19 for G1, 17 at nv 37, 16 at nv 64)."""
  n = 128
  if name == "g1_flat":
    from mjlab_b200.asset_zoo import load_compiled

    m = load_compiled(name)
    st = make_states(m, n, seed=5)
  else:
    m = _model(name)
    st, up = _states(m, n, seed=21)
    # lifted worlds with one joint of the first limb past its limit: the only constrained dofs are low ones
    j = 1 + np.arange(n) % 3
    qa, rg = np.asarray(m.jnt_qposadr), np.asarray(m.jnt_range)
    st["qpos"][up, qa[j[up]]] = rg[j[up], 1] + 0.03
  nv = int(m.nv)
  cap = {"g1_flat": 19, "nv37": 17, "nv64_nbody64": 16}[name]
  assert _reduced_block_cap(nv) == cap
  sim, o = _pair(m, n, st)
  assert int(sim.get_option("reduced_block_cap")) == cap
  o.forward()
  nefc = o.nefc.ravel()
  res = {}
  for full in (0, 1):
    sim.set_option("full_solver", full)
    load_sim(sim, st)
    sim.forward()
    torch.cuda.synchronize()
    nd = F(sim, "solver_nd").ravel()
    if full:
      assert (nd[nefc > 0] == nv).all()
    else:
      assert ((nd > 0) & (nd < nv)).sum() >= 8, np.bincount(nd)
      assert (nd[(nd > 0) & (nd < nv)] <= cap).all()
    res[full] = F(sim, "qacc").copy()
    e = relerr(res[full], o.qacc, floor=10.0)
    assert e.max() < 1e-3, (full, "qacc", int(e.argmax()), e.max())
    e = relerr(F(sim, "qfrc_constraint"), o.qfrc_constraint, floor=10.0)
    assert e.max() < 1e-3, (full, "qfrc_constraint", int(e.argmax()), e.max())
  assert relerr(res[0], res[1], floor=10.0).max() < 1e-3
  sim.close()


def test_tree_and_dense_schedules_on_the_64_dof_robot():
  """The dof-tree L^T D L schedule and the dense one (taken when a contact couples two branches, or forced) give the
  oracle's step on the nv 64 robot, with self-contacts between its limbs in the batch."""
  m = _model("nv64_nbody64")
  n = 128
  st, _ = _states(m, n, seed=31)
  a, o = _pair(m, n, st)
  b = _sim(m, n)
  b.set_option("dense_factor", 1)
  load_sim(b, st)
  o.step()
  a.step()
  b.step()
  torch.cuda.synchronize()
  # contacts between two limbs (neither body an ancestor of the other): the default path takes the dense schedule
  parent = np.asarray(m.body_parentid)

  def chain(b):
    out = {b}
    while b:
      b = int(parent[b])
      out.add(b)
    return out

  gb = np.asarray(m.geom_bodyid)
  cg = o.contact_geom.reshape(n, -1, 2)
  cross = 0
  for w in range(n):
    for g1, g2 in cg[w, : o.ncon[w, 0]]:
      b1, b2 = int(gb[g1]), int(gb[g2])
      cross += b1 > 1 and b2 > 1 and b1 not in chain(b2) and b2 not in chain(b1)
  assert cross >= 5, cross
  ea, eb = relerr(F(a, "qvel"), o.qvel), relerr(F(b, "qvel"), o.qvel)
  assert ea.max() < 3e-3 and eb.max() < 3e-3, (ea.max(), eb.max())
  assert relerr(F(a, "qvel"), F(b, "qvel")).max() < 3e-3
  a.close()
  b.close()


STATE = ("qpos", "qvel", "qacc_warmstart", "ncon", "contact_geom")


def _run(model, st, n, steps=3, **options):
  sim = _sim(model, n)
  for k, v in options.items():
    sim.set_option(k, v)
  load_sim(sim, st)
  for _ in range(steps):
    sim.step()
  torch.cuda.synchronize()
  out = {f: F(sim, f).copy() for f in STATE}
  out["niter"] = F(sim, "solver_niter").ravel().copy()
  sim.close()
  return out


def test_worlds_do_not_depend_on_their_neighbours():
  """A world's result does not depend on which warp of which CTA steps it, on the worlds next to it, on the
  heavy-first dispatch order or on whether the CTAs run phase-synchronously: bit for bit, on the nv 64 robot
  (the largest per-warp shared-memory block)."""
  m = _model("nv64_nbody64")
  n = 520
  st, _ = _states(m, n + 1, seed=41)
  base = {k: v[:n] for k, v in st.items()}
  perm = np.random.default_rng(42).permutation(n)
  ref = _run(m, base, n)
  assert len(np.unique(ref["niter"])) > 2  # (the dispatch sort key takes several values)
  runs = {
    "permuted": (_run(m, {k: v[perm] for k, v in base.items()}, n), perm),
    "unsorted": (_run(m, base, n, sorted_dispatch=0), np.arange(n)),
    "521 worlds": (_run(m, st, n + 1), np.arange(n)),  # (partial last CTA: phase synchronisation off)
  }
  for what, (out, p) in runs.items():
    for f in STATE:
      got = out[f][np.argsort(p)][:n] if what == "permuted" else out[f][:n]
      assert np.array_equal(got, ref[f]), (what, f)

"""The constraint solver of the step kernel and of the oracle (oracle/b2_oracle.c) against an independent fp64 solution
of the soft-constraint problem.

The kernel and the oracle build their constraint rows the same way, and the parity tests compare the two with each
other, so a convention both got wrong would pass them all.  Here the rows are built again from the model's arrays, one
world's rows of the per-world fields, the state and the backend's contact list (the narrowphase is pinned by other
files, so the list is input), and the problem is solved in plain dense fp64:

  limit rows     hinges and slides with dist = +-(range - q) < jnt_margin: J = -+e_dof, diagApprox = dof_invweight0
  contact rows   J = frame (J_b2 - J_b1) from the `Rigid` point Jacobians at contact_pos; condim 1 one row, condim 3
                 the four pyramid edges J_n +- mu J_t; a contact with dist >= margin - gap has no row
  parameters     mj_contactParam: the geom of higher priority decides; at equal priority the larger condim and
                 friction (floored at MINMU), solref and solimp mixed by solmix weights, or the element-wise min of
                 solref when either is not positive; margin the larger, gap the larger
  impedance      the solimp sigmoid (power and mid); K, B from a positive solref with the time constant raised to 2h
                 (refsafe) or from a negative one; R = max(eps, (1-d)/d diagApprox), D = 1/R,
                 aref = -B J v - K d (dist - margin)
  minimiser      c(a) = 1/2 (a-a_s)^T M (a-a_s) + sum_{Ja-aref<0} 1/2 D (Ja-aref)^2 by Newton with an exact line
                 search, then certified: the linear system of the final active set is solved directly, and the active
                 set and the gradient are checked at that point (the cost is strictly convex: it is the minimiser)

The limit and contact rows, mj_contactParam's rules, the impedance sigmoid, refsafe and the negative-solref stiffness
and damping are restated from MuJoCo's documentation (Computation: Constraint model, Solver parameters, Contact
parameters).  Recalled, not restated: the pyramid edges' diagApprox tran (1 + mu^2) with tran the sum of the two
bodies' translational invweight0, and their R = 2 mu'^2 R with mu' = mu / sqrt(impratio) (SURVEY.md Appendix A marks
both (?)).  This file pins the kernel and the oracle to this formulation; it does not pin the formulation to MuJoCo.

Three backends: the fp64 oracle and the host-emulated library (CPU suite), and the H100 (`-m gpu`).  Every case
asserts the condition it exists for.  Every input is rounded to fp32 first, so that all backends and the reference
see the same numbers.  The oracle runs with tolerance 1e-14 and 100 iterations; the kernel with each solver path.
"""

import functools
import sys
from pathlib import Path

import numpy as np
import pytest

from test_rigid_body_reference import (EULER, FREE, HINGE, IMPLICITFAST, SLIDE, SYNTH, Backend, Rigid, arr, f32, f32_model,
                                       free_joints)
from util import convex_scene, convex_states, make_states, relerr

sys.path.append(str(Path(__file__).resolve().parents[1] / "tools"))
from synth_models import robot_xml  # noqa: E402

MINVAL, MINIMP, MAXIMP, MINMU = 1e-15, 1e-4, 0.9999, 1e-5
HFIELD, SPHERE, CAPSULE, ELLIPSOID, CYLINDER, BOX, MESH = 1, 2, 3, 4, 5, 6, 7

BACKENDS = ["oracle", "emul", pytest.param("cuda", marks=pytest.mark.gpu)]
ENGINES = ["emul", pytest.param("cuda", marks=pytest.mark.gpu)]
NWORLD = {"oracle": 4, "emul": 4, "cuda": 32}
CASES = ["g1", "go1", "multijoint", "nu58", "nv64_nbody64", "convex", "round", "stairs"]
# solver paths of the kernel, on the same states: options set before the forward
PATHS = {"newton": {}, "full": {"full_solver": 1}, "dense": {"dense_factor": 1}, "cg": {"solver": 1, "iterations": 100},
         "precise": {"iterations": 200, "tolerance": 1e-12}}
ORACLE_OPTS = {"iterations": 100, "tolerance": 1e-14}
NCON = 96  # contacts per world (the engine's largest per-world capacity)

# ---- tolerances ----------------------------------------------------------------------------------------------------
# qacc: ||qacc - a*||_M / ||a* - a_s||_M; qfrc: qfrc_constraint against J^T f*; force: contact_force against f* in the
# contact frame, over the world's largest normal force; cost: solver_cost against c(qacc); subopt: (c(qacc) - c*) /
# (meaninertia nv); qvel, qpos: one step against the reference integrator driven by f*.
# fp64 oracle (tolerance 1e-14): limited by the reference's own bias forces (central differences, ~1e-8 in a_s).
# Measured worst cases: qacc 9.0e-8, qfrc 8.4e-8, force 5.9e-8, cost 1.6e-8, subopt 2.5e-9, qvel 5.5e-8, qpos 1.3e-9,
# qacc against a* norm-wise 5.8e-8.  rows: the oracle's efc arrays; J and aref to 2e-7 only: the oracle turns hinge
# axes by the product of the body quaternions before normalising it, and the fp32-rounded body_quat of the robots are
# unit only to |q|^2 - 1 ~ 1e-7 (G1's wrist columns differ by 1.1e-8, multijoint's by 5.7e-8); the reference
# normalises every quaternion.
ORACLE_TOL = dict(rows=1e-12, rows_J=2e-7, rows_qacc=1e-9, qacc=3.6e-7, qfrc=3.4e-7, force=2.4e-7, cost=6e-8, subopt=1e-8, qvel=2.2e-7,
                  qpos=5e-9)
# fp32 kernel, Newton (default, full, dense factor, 200 iterations at tolerance 1e-12).  Measured worst cases over every
# case, host emulation (4 worlds) | NVIDIA H100 80GB HBM3 at a 700 W power limit (32 worlds): qacc 4.2e-5 | 1.9e-4,
# qfrc 2.5e-5 | 1.4e-4, force 5.9e-5 | 8.4e-5, cost 3.4e-5 | 8.6e-5, subopt 3.2e-3 | 7.9e-4 (the stairs world with 81
# contacts | the convex scene), qvel 1.2e-4 | 5.0e-4, qpos 3.3e-6 | 6.5e-6.
KERNEL_TOL = dict(qacc=7e-4, qfrc=5.5e-4, force=3.3e-4, cost=3.4e-4, subopt=1.2e-2, qvel=2e-3, qpos=2.5e-5)
# CG (100 iterations) stops on its own improvement test, farther from the minimiser than Newton.  Measured on G1 and
# the 64-dof robot, emulation | H100: qacc 1.8e-4 | 6.0e-4, qfrc 3.3e-4 | 2.1e-3, force 3.3e-4 | 8.5e-4, cost 1.0e-6 |
# 8.3e-5, subopt 2.5e-3 | 1.0e-2.
CG_TOL = dict(KERNEL_TOL, qacc=2.4e-3, qfrc=8.4e-3, force=3.4e-3, cost=3.3e-4, subopt=4e-2)


def tol(backend, path="newton"):
  return ORACLE_TOL if backend == "oracle" else CG_TOL if path == "cg" else KERNEL_TOL


# ---- the reference problem -----------------------------------------------------------------------------------------


class Params:
  """The constraint parameters of one world: the model's arrays, the world's rows (field -> values) where given."""

  def __init__(self, m, row):
    def f(k, width=0):
      v = np.asarray(row.get(k, m.arrays[k]), np.float64)
      return v.reshape(-1, width) if width else v.ravel()

    self.priority, self.condim = arr(m, "geom_priority").astype(int), arr(m, "geom_condim").astype(int)
    self.friction, self.solref, self.solimp = f("geom_friction", 3), f("geom_solref", 2), f("geom_solimp", 5)
    self.solmix, self.margin, self.gap = f("geom_solmix"), f("geom_margin"), f("geom_gap")
    self.jlimited = arr(m, "jnt_limited") != 0
    self.jrange, self.jmargin = f("jnt_range", 2), f("jnt_margin")
    self.jsolref, self.jsolimp = f("jnt_solref", 2), f("jnt_solimp", 5)
    self.dinv, self.binv = f("dof_invweight0"), f("body_invweight0", 2)
    self.h, self.impratio = float(m.opt_timestep), float(m.opt_impratio)


def contact_param(P, g1, g2, drop):
  """condim, friction, solref, solimp of a geom pair (mj_contactParam)."""
  if P.priority[g1] != P.priority[g2] and "priority" not in drop:
    g = g1 if P.priority[g1] > P.priority[g2] else g2
    return P.condim[g], P.friction[g, 0], P.solref[g], P.solimp[g]
  s1, s2 = P.solmix[g1], P.solmix[g2]
  if "solmix" in drop or (s1 < MINVAL and s2 < MINVAL):
    mix = 0.5
  elif s1 >= MINVAL and s2 >= MINVAL:
    mix = s1 / (s1 + s2)
  else:
    mix = 0.0 if s1 < MINVAL else 1.0
  r1, r2 = P.solref[g1], P.solref[g2]
  solref = mix * r1 + (1 - mix) * r2 if r1[0] > 0 and r2[0] > 0 else np.minimum(r1, r2)
  return (max(P.condim[g1], P.condim[g2]), max(P.friction[g1, 0], P.friction[g2, 0]), solref,
          mix * P.solimp[g1] + (1 - mix) * P.solimp[g2])


def impedance(si, x, drop):
  """The solimp sigmoid at |pos - margin| = x, and dmax."""
  dmin, dmax = np.clip(si[0], MINIMP, MAXIMP), np.clip(si[1], MINIMP, MAXIMP)
  width, mid = max(si[2], MINVAL), np.clip(si[3], MINIMP, MAXIMP)
  power = 1.0 if "power" in drop else max(si[4], 1.0)
  x = x / width
  if x >= 1:
    return dmax, dmax
  if x <= 0:
    return dmin, dmax
  y = x if power == 1 else (x**power / mid**(power - 1) if x <= mid else 1 - (1 - x)**power / (1 - mid)**(power - 1))
  return dmin + y * (dmax - dmin), dmax


def stiffness(sr, dmax, h, drop):
  """K, B of a solref."""
  if sr[0] > 0:
    tc = sr[0] if "refsafe" in drop else max(sr[0], 2 * h)
    return 1 / max(MINVAL, dmax * dmax * tc * tc * sr[1] * sr[1]), 2 / max(MINVAL, dmax * tc)
  return -sr[0] / (dmax * dmax), -sr[1] / dmax


def build(r, P, q, v, con, drop=()):
  """Every constraint row of one world: limits (joint order, lower side first), then contacts in list order."""
  K = r.kin(q)
  J, pos, mar, par, diag, pyr, meta = [], [], [], [], [], [], []
  for j in range(len(r.jtype)):
    if not P.jlimited[j] or r.jtype[j] not in (HINGE, SLIDE):
      continue
    d = r.dadr[j]
    for side in (-1, 1):
      dist = side * (P.jrange[j, (side + 1) // 2] - q[r.qadr[j]])
      if dist < P.jmargin[j]:
        row = np.zeros(r.nv)
        row[d] = -side
        J.append(row), pos.append(dist), mar.append(P.jmargin[j]), par.append((P.jsolref[j], P.jsolimp[j]))
        diag.append(P.dinv[d]), pyr.append(0.0)
        meta.append(dict(kind="limit", side=side, slide=r.jtype[j] == SLIDE, solref=P.jsolref[j][0]))
  contacts = []
  for c, (g1, g2) in enumerate(con["geom"]):
    dist = con["dist"][c]
    condim, fri, sr, si = contact_param(P, g1, g2, drop)
    assert condim in (1, 3), condim
    mu = max(fri, MINMU)
    gap = 0.0 if "gap" in drop else max(P.gap[g1], P.gap[g2])
    margin = max(P.margin[g1], P.margin[g2])
    incm = margin - gap
    b1, b2 = r.geom_body[g1], r.geom_body[g2]
    cm = dict(first=len(J), dim=condim, mu=mu, dist=dist, margin=margin, incm=incm, b1=b1, b2=b2, g=(g1, g2))
    contacts.append(cm)
    if dist >= incm:
      cm["dim"] = 0
      continue
    Jp = r.jac(K, np.tile(con["pos"][c], (r.nb, 1)))[0]
    dif = Jp[b2] - (0.0 if "body1" in drop else Jp[b1])  # (nv, 3)
    fr = np.asarray(con["frame"][c], np.float64).reshape(3, 3)
    jn, jt = dif @ fr[0], dif @ fr[1:].T
    tran = P.binv[b1, 0] + P.binv[b2, 0]
    sgn = -1.0 if "tangent" in drop else 1.0
    if condim == 1:
      rows, dg = [jn], tran
    else:
      rows = [jn + sgn * mu * jt[:, 0], jn - sgn * mu * jt[:, 0], jn + sgn * mu * jt[:, 1], jn - sgn * mu * jt[:, 1]]
      dg = tran * (1 + mu * mu)
    for row in rows:
      J.append(row), pos.append(dist), mar.append(incm), par.append((sr, si)), diag.append(dg)
      pyr.append(mu if condim > 1 else 0.0)
      meta.append(dict(kind="contact", contact=c, solref=sr[0]))
  nefc = len(J)
  J = np.array(J).reshape(nefc, r.nv)
  pos, mar, diag, pyr = (np.array(x, np.float64) for x in (pos, mar, diag, pyr))
  R, aref = np.zeros(nefc), np.zeros(nefc)
  jv = J @ v
  for i in range(nefc):
    sr, si = par[i]
    imp, dmax = impedance(si, abs(pos[i] - mar[i]), drop)
    k, b = stiffness(sr, dmax, P.h, drop)
    R[i] = max(MINVAL, (1 - imp) / imp * diag[i])
    if pyr[i] > 0 and "pyramid" not in drop:
      mup = pyr[i] if "impratio" in drop else pyr[i] / np.sqrt(P.impratio)
      R[i] = max(MINVAL, 2 * mup * mup * R[i])
    aref[i] = -b * jv[i] - k * imp * (pos[i] - mar[i])
    meta[i].update(x=abs(pos[i] - mar[i]) / max(si[2], MINVAL), power=si[4])
  return dict(J=J, pos=pos, margin=mar, R=R, D=1 / R, aref=aref, contacts=contacts, meta=meta, nefc=nefc)


def cost(S, a):
  d = a - S["a_s"]
  jar = S["J"] @ a - S["aref"]
  return 0.5 * d @ S["M"] @ d + 0.5 * np.sum(S["D"] * np.minimum(jar, 0.0)**2)


def gradient(S, a):
  jar = S["J"] @ a - S["aref"]
  return S["M"] @ (a - S["a_s"]) + S["J"].T @ (S["D"] * np.minimum(jar, 0.0))


def line_search(S, a, s):
  """The exact minimiser along s of the piecewise quadratic cost: the root of its piecewise linear derivative."""
  jar, jv = S["J"] @ a - S["aref"], S["J"] @ s
  g0, g2 = s @ S["M"] @ (a - S["a_s"]), s @ S["M"] @ s

  def slope(t):
    x = jar + t * jv
    on = x < 0
    return g0 + t * g2 + np.sum(S["D"][on] * x[on] * jv[on])

  with np.errstate(divide="ignore", invalid="ignore"):
    bps = np.sort(np.unique((-jar / jv)[(jv != 0) & (-jar / jv > 0)]))
  lo = 0.0
  for hi in list(bps) + [np.inf]:
    if hi == np.inf or slope(hi) >= 0:
      t = lo + 1.0 if hi == np.inf else 0.5 * (lo + hi)  # the active set inside (lo, hi)
      on = (jar + t * jv) < 0
      return -(g0 + np.sum(S["D"][on] * jar[on] * jv[on])) / (g2 + np.sum(S["D"][on] * jv[on]**2))
    lo = hi


def minimise(S, iterations=100):
  a = S["a_s"].copy()
  prev = None
  for _ in range(iterations):
    jar = S["J"] @ a - S["aref"]
    on = jar < 0
    if prev is not None and (on == prev).all():
      break
    H = S["M"] + S["J"][on].T @ (S["D"][on, None] * S["J"][on])
    s = -np.linalg.solve(H, gradient(S, a))
    if not s.any():
      break
    a = a + line_search(S, a, s) * s
    prev = on
  return a


def certify(S, a):
  """The minimiser: the linear system of a's active set solved directly, the active set and the gradient checked."""
  J, D, aref = S["J"], S["D"], S["aref"]
  on = (J @ a - aref) < 0
  H = S["M"] + J[on].T @ (D[on, None] * J[on])
  a = np.linalg.solve(H, S["M"] @ S["a_s"] + J[on].T @ (D[on] * aref[on]))
  jar = J @ a - aref
  scale = max(np.abs(aref).max(initial=0.0), np.abs(J @ a).max(initial=0.0), 1e-300)
  assert (jar[on] <= 1e-10 * scale).all() and (jar[~on] >= -1e-10 * scale).all(), "inconsistent active set"
  f = -D * np.minimum(jar, 0.0)
  g = gradient(S, a)
  assert np.abs(g).max() <= 1e-9 * max(np.abs(S["M"] @ S["a_s"]).max(), np.abs(J.T @ f).max(), 1.0), np.abs(g).max()
  return a


def solve(S, drop=()):
  """a*, f*, qfrc_constraint*, contact_force* and c* of a built problem (stopped after one Newton iteration, not
  certified, when `drop` holds "newton")."""
  if S["nefc"] == 0:
    a = S["a_s"].copy()
  elif "newton" in drop:
    a = minimise(S, iterations=1)
  else:
    a = certify(S, minimise(S))
  jar = S["J"] @ a - S["aref"]
  f = -S["D"] * np.minimum(jar, 0.0)
  cf = np.zeros((len(S["contacts"]), 3))
  for c, cm in enumerate(S["contacts"]):
    k = cm["first"]
    if cm["dim"] == 1:
      cf[c, 0] = f[k]
    elif cm["dim"] == 3:
      cf[c] = [f[k:k + 4].sum(), cm["mu"] * (f[k] - f[k + 1]), cm["mu"] * (f[k + 2] - f[k + 3])]
  return dict(a=a, jar=jar, f=f, qfrc=S["J"].T @ f, cf=cf, cost=cost(S, a))


# ---- cases: models, per-world rows, states ------------------------------------------------------------------------


@functools.cache
def model(case):
  """The case's model, every float rounded to fp32.  The synthetic robots keep their self- and floor contacts;
  multijoint's floor has a higher priority than the robot, nu58 is compiled with impratio 4.  "round": free cylinders
  and ellipsoids on a floor and a block; "stairs": Go1 on the rough box terrain (stairs and boxes out to 76 m)."""
  from mjlab_b200.asset_zoo import load_compiled
  from mjlab_b200.compiler import Spec

  if case in ("g1", "go1"):
    m = load_compiled(case + "_flat")
  elif case in SYNTH:
    seed, limbs, joints, kw = SYNTH[case]
    xml = robot_xml(np.random.default_rng(seed), limbs, joints, **kw)
    if case == "multijoint":
      xml = xml.replace('<geom name="floor"', '<geom name="floor" priority="1"')
    if case == "nu58":
      xml = xml.replace("<option ", '<option impratio="4" ')
    m = Spec.from_string(xml).compile()
  elif case == "round":
    m = Spec.from_string(ROUND_XML).compile()
  elif case == "stairs":
    m = load_compiled("go1_rough")
  else:
    m = convex_scene()[0]
  return f32_model(m)


ROUND_XML = """<mujoco><option timestep="0.004"/><worldbody><geom name="floor" type="plane" size="0 0 1"/>
 <geom name="block" type="box" pos="0.3 0 0.08" size="0.1 0.1 0.08"/>
 <body name="c1" pos="0 0 0.06"><freejoint/><geom type="cylinder" size="0.07 0.05" mass="1"/></body>
 <body name="e1" pos="0.08 0.03 0.13"><freejoint/><geom type="ellipsoid" size="0.09 0.06 0.045" mass="0.8"/></body>
 <body name="c2" pos="-0.08 0.06 0.08"><freejoint/><geom type="cylinder" size="0.04 0.08" mass="0.6"/></body>
 <body name="e2" pos="0.02 -0.09 0.07"><freejoint/><geom type="ellipsoid" size="0.06 0.07 0.05" mass="0.7"/></body>
 <body name="bx" pos="0.3 0.02 0.19"><freejoint/><geom type="box" size="0.05 0.04 0.03" mass="0.5"/></body>
 <body name="e3" pos="0.26 -0.06 0.2"><freejoint/><geom type="ellipsoid" size="0.05 0.04 0.06" mass="0.4"/></body>
</worldbody></mujoco>"""


def solref_rows(rng, k, h):
  """(k, 2) solrefs: a third positive, a third positive with a time constant below 2h (refsafe), a third negative."""
  kind = rng.integers(0, 3, k)[:, None]
  pos = np.c_[rng.uniform(0.01, 0.04, k), rng.uniform(0.6, 1.4, k)]
  fast = np.c_[rng.uniform(0.2, 0.9, k) * 2 * h, rng.uniform(0.6, 1.4, k)]
  neg = np.c_[-rng.uniform(1e3, 1e4, k), -rng.uniform(20.0, 200.0, k)]
  return np.where(kind == 0, pos, np.where(kind == 1, fast, neg))


def solimp_rows(rng, k):
  """(k, 5) solimps: widths of 5 to 50 mm (penetrations land inside the sigmoid), power 1 to 3, mid 0.2 to 0.8."""
  return np.c_[rng.uniform(0.5, 0.9, k), rng.uniform(0.9, 0.99, k), rng.uniform(0.005, 0.05, k),
               rng.uniform(0.2, 0.8, k), rng.uniform(1.0, 3.0, k)]


def constraint_rows(m, n, rng):
  """Per-world values of every expandable field the constraint rows read: (n, count * width) rows.  Odd worlds give
  every geom a margin of 5 to 30 mm and a gap of up to 70% of it; limited joints get narrowed ranges and margins."""
  h, ng, nj = float(m.opt_timestep), int(m.ngeom), int(m.njnt)
  lim = (arr(m, "jnt_limited") != 0) & (arr(m, "jnt_type") != FREE)
  rows = {}
  for w in range(n):
    r = {}
    fr = arr(m, "geom_friction", 3).copy()
    fr[:, 0] = rng.uniform(0.2, 1.5, ng)
    r["geom_friction"] = fr
    r["geom_solref"], r["geom_solimp"] = solref_rows(rng, ng, h), solimp_rows(rng, ng)
    r["geom_solmix"] = rng.uniform(0.1, 3.0, ng)
    r["geom_margin"] = rng.uniform(0.005, 0.03, ng) * (w % 2)
    r["geom_gap"] = r["geom_margin"] * rng.uniform(0.0, 0.7, ng)
    rg = arr(m, "jnt_range", 2).copy()
    width = rg[:, 1] - rg[:, 0]
    rg[lim, 0] += rng.uniform(0.0, 0.1, lim.sum()) * width[lim]
    rg[lim, 1] -= rng.uniform(0.0, 0.1, lim.sum()) * width[lim]
    r["jnt_range"] = rg
    r["jnt_margin"] = np.where(lim, rng.uniform(0.0, 0.05, nj) * width, 0.0)
    r["jnt_solref"], r["jnt_solimp"] = solref_rows(rng, nj, h), solimp_rows(rng, nj)
    for k, v in r.items():
      rows.setdefault(k, []).append(np.asarray(v, np.float64).ravel())
  return {k: np.stack(v) for k, v in rows.items()}


def lowest_point(m, r, q):
  """Height of the lowest point of the colliding geoms of the moving bodies (spheres, capsules, boxes)."""
  K = r.kin(q)
  gt, size = arr(m, "geom_type"), arr(m, "geom_size", 3)
  coll = (arr(m, "geom_contype") != 0) | (arr(m, "geom_conaffinity") != 0)
  z = np.inf
  for g in np.nonzero(coll & np.isin(gt, (SPHERE, CAPSULE, BOX)) & r.moves.any(1)[r.geom_body])[0]:
    c, R, s = K["geom_xpos"][g], K["geom_xmat"][g], size[g]
    ext = {SPHERE: s[0], CAPSULE: s[0] + abs(R[2, 2]) * s[1], BOX: np.abs(R[2]) @ s}[gt[g]]
    z = min(z, c[2] - ext)
  return z


def synth_states(m, n, rng):
  """Joints near and past both ends of their (model) ranges, the base tilted and lowered until its lowest point is
  0 to 30 mm inside the floor."""
  nv, nb = int(m.nv), int(m.nbody)
  jt, qa = arr(m, "jnt_type"), arr(m, "jnt_qposadr")
  rg = arr(m, "jnt_range", 2)
  r = Rigid(m)
  q = np.tile(arr(m, "qpos0"), (n, 1))
  for w in range(n):
    for j in np.nonzero(jt != FREE)[0]:
      lo, hi = rg[j]
      u = rng.uniform()
      q[w, qa[j]] = (rng.uniform(lo, hi) if u < 0.4 else
                     lo + rng.uniform(-0.08, 0.05) * (hi - lo) if u < 0.7 else hi + rng.uniform(-0.05, 0.08) * (hi - lo))
    ax = rng.normal(size=3)
    t = rng.uniform(-0.2, 0.2)
    q[w, 3:7] = np.r_[np.cos(t / 2), np.sin(t / 2) * ax / np.linalg.norm(ax)]
    q[w, 2] += rng.uniform(-0.03, 0.0) - lowest_point(m, r, q[w])
  return dict(qpos=q, qvel=rng.uniform(-0.5, 0.5, (n, nv)), qacc_warmstart=np.zeros((n, nv)),
              ctrl=rng.uniform(-1.0, 1.0, (n, int(m.nu))), xfrc_applied=np.zeros((n, 6 * nb)))


def round_states(m, n, rng):
  """Every free body within 20 mm of its place and turned at random: the cylinders and ellipsoids press into the
  floor, the block and each other."""
  nv, nb = int(m.nv), int(m.nbody)
  q = np.tile(arr(m, "qpos0"), (n, 1))
  for a in arr(m, "jnt_qposadr")[free_joints(m)]:
    q[:, a:a + 3] += rng.normal(0.0, 0.02, (n, 3))
    quat = rng.normal(size=(n, 4))
    q[:, a + 3:a + 7] = quat / np.linalg.norm(quat, axis=1, keepdims=True)
  return dict(qpos=q, qvel=rng.uniform(-0.5, 0.5, (n, nv)), ctrl=np.zeros((n, 0)), xfrc_applied=np.zeros((n, 6 * nb)))


def stairs_states(m, rows, n, rng):
  """Go1 on sub-terrain origins of the rough box terrain: the first half of the worlds within 20 m of the origin, the
  second half 55 to 65 m out, where the kernel's reference point c0 (the com of the moving bodies) lies.  In the last
  world the robot is turned at random and lowered onto the boxes with every margin at 0.1 m, in the first pose
  (searched with the fp64 oracle) that makes 70 to 88 contacts: more than the 64 the solver keeps in registers."""
  from oracle.oracle import Oracle

  org = np.asarray(m.arrays["terrain_origins"]).reshape(-1, 3)
  d = np.linalg.norm(org[:, :2], axis=1)
  near, far = org[d < 20.0], org[(d > 55.0) & (d < 65.0)]
  st = make_states(m, n, seed=int(rng.integers(1 << 30)), z_range=(-0.05, 0.0), joint_noise=0.3)
  h = n // 2
  spots = np.concatenate([near[rng.integers(0, len(near), h)], far[rng.integers(0, len(far), n - h)]])
  st["qpos"][:, 0:2] = spots[:, 0:2] + rng.uniform(-0.5, 0.5, (n, 2))
  st["qpos"][:, 2] += spots[:, 2]
  st["xfrc_applied"] = np.zeros((n, 6 * int(m.nbody)))
  w = n - 1
  rows["geom_margin"][w] = 0.1
  rows["geom_gap"][w] = 0.1 * rng.uniform(0.0, 0.5, int(m.ngeom))
  o = Oracle(m, nworld=1, maxcon=NCON, njmax=4 * NCON + 128)
  for k, v in rows.items():
    o.model_field(k)[:] = f32(v[w])
  for k in ("qvel", "ctrl"):
    o.field(k)[:] = f32(st[k][w])
  for _ in range(500):
    q = st["qpos"][w].copy()
    q[0:2] = far[rng.integers(0, len(far))][0:2] + rng.uniform(-2.0, 2.0, 2)
    quat = rng.normal(size=4)
    q[3:7] = quat / np.linalg.norm(quat)
    q[2] = org[np.argmin(np.linalg.norm(org[:, :2] - q[:2], axis=1)), 2] + rng.uniform(-0.1, 0.1)
    o.field("qpos")[:] = f32(q)
    o.forward()
    if 70 <= int(o.ncon[0, 0]) <= 88 and not int(o.overflow[0, 0]):
      st["qpos"][w] = q
      return st
  raise AssertionError("no pose with 70 to 88 contacts")


@functools.cache
def case_data(case, n, seed=1):
  """The model, per-world rows and states of a case, every value rounded to fp32."""
  m = model(case)
  rng = np.random.default_rng(seed)
  rows = constraint_rows(m, n, rng)
  nv, nb = int(m.nv), int(m.nbody)
  if case in ("g1", "go1"):
    st = make_states(m, n, seed=seed, z_range=(-0.04, 0.0), joint_noise=0.3)
    st["xfrc_applied"] = np.zeros((n, 6 * nb))
    hinge = np.nonzero(arr(m, "jnt_type") == HINGE)[0][:6]  # (one leg: the rest of G1 stays free for the reduced solver)
    for w in range(n):  # two joints of every world up to 50 mrad past either end of the world's range
      for j in rng.choice(hinge, 2, replace=False):
        lo, hi = rows["jnt_range"][w].reshape(-1, 2)[j]
        st["qpos"][w, arr(m, "jnt_qposadr")[j]] = lo - rng.uniform(0, 0.05) if rng.uniform() < 0.5 else hi + rng.uniform(0, 0.05)
    if case == "go1":
      # world 1: margins of 20 mm, gaps of 14, pitched nose-down by 0.3 rad and lifted until its lowest point is 12 mm
      # up (in the band); its rear legs are then free, and the solver works on the leading block of dofs only
      rows["geom_margin"][1], rows["geom_gap"][1] = 0.02, 0.014
      st["qpos"][1, 3:7] = [np.cos(0.15), 0.0, np.sin(0.15), 0.0]
      st["qpos"][1, 2] += 0.012 - lowest_point(m, Rigid(m), st["qpos"][1])
  elif case in SYNTH:
    st = synth_states(m, n, rng)
  elif case == "round":
    st = round_states(m, n, rng)
  elif case == "stairs":
    st = stairs_states(m, rows, n, rng)
  else:
    st = convex_states(m, *convex_scene()[1:], n, seed=seed)
    st["xfrc_applied"] = np.zeros((n, 6 * nb))
  st["qfrc_applied"] = rng.normal(0.0, 2.0, (n, nv))
  st["qacc_warmstart"] = np.zeros((n, nv))
  return m, {k: f32(v) for k, v in rows.items()}, {k: f32(v) for k, v in st.items()}


@functools.cache
def smooth_parts(case, n):
  """Per world: the Rigid model, the constraint parameters and the reference's M, qfrc_smooth and a_s."""
  m, rows, st = case_data(case, n)
  out = []
  for w in range(n):
    row = {k: v[w] for k, v in rows.items()}
    r, P = Rigid(m, row), Params(m, row)
    F = r.forward(st["qpos"][w], st["qvel"][w], st["ctrl"][w] if r.nu else [], st["qfrc_applied"][w],
                  st["xfrc_applied"][w])
    out.append((r, P, dict(M=F["qM"], qfrc_smooth=F["qfrc_smooth"], a_s=F["qacc_smooth"])))
  return out


# ---- backends ------------------------------------------------------------------------------------------------------

OUT = ("ncon", "nefc", "qacc", "qfrc_constraint", "contact_force", "contact_geom", "contact_dist", "contact_pos",
       "contact_frame", "solver_cost", "overflow", "solver_niter")


def open_backend(backend, case, opts):
  n = NWORLD[backend]
  m, rows, st = case_data(case, n)
  be = Backend(backend, m, n, nconmax=NCON * n)
  be.rows(rows)
  be.load(st)
  for k, v in (ORACLE_OPTS if backend == "oracle" else opts).items():
    be.set(k, v)
  return be, m, rows, st


def outputs(be):
  out = {f: be.a(f) for f in OUT}
  if be.e is not None:
    out["solver_nd"] = be.a("solver_nd")
  else:
    out.update({f: be.a(f) for f in ("efc_J", "efc_pos", "efc_margin", "efc_R", "efc_D", "efc_aref")})
  # (a world whose broadphase finds more candidate pairs than the engine holds, 128 without static geoms, keeps the
  # contacts of the first 128: the synthetic robots' limbs overlap that much in a few worlds.  The contact list is the
  # reference's input, so such a world is still one well-defined problem, and it is compared like every other.)
  return out


@functools.cache
def run(backend, case, path="newton"):
  """One forward of a case on a backend: its outputs."""
  be, *_ = open_backend(backend, case, PATHS[path])
  try:
    be.forward()
    out = outputs(be)
    if be.e is not None:
      out["options"] = {k: be.e.opt(k) for k in PATHS[path]}
    return out
  finally:
    be.close()


def contact_list(out, w):
  k = int(out["ncon"][w, 0])
  return dict(geom=out["contact_geom"][w, :2 * k].reshape(k, 2).astype(int), dist=out["contact_dist"][w, :k],
              pos=out["contact_pos"][w, :3 * k].reshape(k, 3), frame=out["contact_frame"][w, :9 * k].reshape(k, 9))


def references(backend, case, out, drop=()):
  """The reference problem and its solution in every world, on the backend's contact lists."""
  m, rows, st = case_data(case, len(out["qacc"]))
  res = []
  for w, (r, P, sm) in enumerate(smooth_parts(case, len(out["qacc"]))):
    S = build(r, P, st["qpos"][w], st["qvel"][w], contact_list(out, w), drop)
    S.update(sm)
    S.update(solve(S, drop))
    S["scale"] = 1.0 / (float(m.stat_meaninertia) * max(1, r.nv))
    res.append(S)
  return res


def mnorm(M, x):
  return float(np.sqrt(max(x @ M @ x, 0.0)))


def errors(out, refs):
  """Per world and per assertion: the backend's error against the reference (nefc: rows of difference).  In a world
  whose constraints barely move the acceleration the qacc and cost errors are relative to 5% of a*'s M-norm (and the
  cost of that) instead."""
  E = {k: [] for k in ("nefc", "qacc", "qfrc", "force", "cost", "subopt")}
  for w, S in enumerate(refs):
    qacc = out["qacc"][w]
    E["nefc"].append(abs(int(out["nefc"][w, 0]) - S["nefc"]))
    floor = 0.05 * mnorm(S["M"], S["a"])
    E["qacc"].append(mnorm(S["M"], qacc - S["a"]) / max(mnorm(S["M"], S["a"] - S["a_s"]), floor))
    E["qfrc"].append(relerr(out["qfrc_constraint"][w:w + 1], S["qfrc"][None])[0])
    k = len(S["contacts"])
    cf = out["contact_force"][w, :3 * k].reshape(k, 3)
    E["force"].append(np.abs(cf - S["cf"]).max(initial=0.0) / max(S["cf"][:, 0].max(initial=0.0), 1e-9))
    c = cost(S, qacc)
    E["cost"].append(abs(out["solver_cost"][w, 0] - c) / max(abs(c), 0.5 * floor * floor))
    E["subopt"].append((c - S["cost"]) * S["scale"])
  return {k: np.array(v, np.float64) for k, v in E.items()}


def exact_zeros(out, refs):
  """Excluded contacts, and contacts whose every row is inactive at a* by more than 1e-3 of the world's largest
  |aref|, have a contact force of exactly 0."""
  for w, S in enumerate(refs):
    k = len(S["contacts"])
    cf = out["contact_force"][w, :3 * k].reshape(k, 3)
    big = 1e-3 * np.abs(S["aref"]).max(initial=0.0)
    for c, cm in enumerate(S["contacts"]):
      rows = {0: 0, 1: 1, 3: 4}[cm["dim"]]
      if cm["dim"] == 0 or (S["jar"][cm["first"]:cm["first"] + rows] > big).all():
        assert (cf[c] == 0).all(), (w, c, cm["dim"], cf[c])


def check(backend, out, refs, path="newton", keys=("qacc", "qfrc", "force", "cost", "subopt")):
  E = errors(out, refs)
  assert (E["nefc"] == 0).all(), ("nefc", out["nefc"].ravel(), [S["nefc"] for S in refs])
  T = tol(backend, path)
  for k in keys:
    assert (E[k] <= T[k]).all(), (k, int(np.argmax(E[k])), E[k].max(), T[k])
  exact_zeros(out, refs)


# ---- what each case exists for -------------------------------------------------------------------------------------


def features(m, out, refs):
  """What the case's rows hold, over all worlds."""
  F = dict(constrained=np.mean([S["nefc"] > 0 for S in refs]), nlim=max(sum(x["kind"] == "limit" for x in S["meta"]) for S in refs))
  meta = [x for S in refs for x in S["meta"]]
  cons = [cm for S in refs for cm in S["contacts"]]
  gt = arr(m, "geom_type")
  lims = [x for x in meta if x["kind"] == "limit"]
  F["past_lower"] = any(x["side"] == -1 for x in lims)
  F["past_upper"] = any(x["side"] == 1 for x in lims)
  F["slide_limits"] = any(x["slide"] for x in lims)
  F["margin_dist"] = any(cm["dim"] and cm["dist"] > 0 for cm in cons)
  F["band"] = any(cm["dim"] == 0 and cm["dist"] < cm["margin"] for cm in cons)
  F["refsafe"] = any(0 < x["solref"] < 2 * float(m.opt_timestep) for x in meta)
  F["neg_solref"] = any(x["solref"] < 0 for x in meta)
  F["sigmoid"] = any(0 < x["x"] < 1 and x["power"] > 1.5 for x in meta)
  F["mixed_dims"] = any({1, 3} <= {cm["dim"] for cm in S["contacts"]} for S in refs)
  moving = Rigid(m).moves.any(1)  # (bodies some dof moves)
  F["two_bodies"] = any(cm["dim"] and moving[cm["b1"]] and moving[cm["b2"]] for cm in cons)
  F["types"] = {int(gt[g]) for cm in cons if cm["dim"] for g in cm["g"]}
  pr = arr(m, "geom_priority")
  F["priority"] = any(cm["dim"] and pr[cm["g"][0]] != pr[cm["g"][1]] for cm in cons)
  F["ncon"] = int(out["ncon"].max())
  F["far"] = max(np.linalg.norm(contact_list(out, w)["pos"][:, :2], axis=1).min(initial=np.inf)
                 for w in range(len(refs)) if out["ncon"][w, 0] > 0)
  F["static_boxes"] = any(cm["dim"] and not moving[cm["b1"]] and gt[cm["g"][0]] == BOX for cm in cons)
  if "solver_nd" in out:
    F["reduced"] = bool((out["solver_nd"] < int(m.nv)).any())
  return F


def assert_case(case, m, out, refs):
  F = features(m, out, refs)
  assert F["constrained"] >= 0.75 and F["margin_dist"] and F["refsafe"] and F["neg_solref"] and F["sigmoid"], F
  if case in ("g1", "go1"):
    assert F["priority"] and F["past_lower"] and F["past_upper"] and F["band"] and F.get("reduced", True), F
  elif case == "multijoint":
    assert F["priority"] and F["slide_limits"] and F["two_bodies"], F
  elif case == "nu58":
    assert float(m.opt_impratio) != 1 and 3 in {cm["dim"] for S in refs for cm in S["contacts"]}, F
  elif case == "nv64_nbody64":
    assert F["nlim"] > 32 and F["mixed_dims"] and F["slide_limits"], F
  elif case == "convex":
    assert F["two_bodies"] and {MESH, HFIELD} <= F["types"], F
  elif case == "round":
    assert F["two_bodies"] and {CYLINDER, ELLIPSOID} <= F["types"], F
  elif case == "stairs":
    # box contacts, a world whose every contact lies 55 m or more from the origin, and one with more than 64
    assert F["static_boxes"] and F["far"] > 55.0 and F["ncon"] > 64, F
  return F


# ---- 1.-6. one forward ---------------------------------------------------------------------------------------------


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("backend", BACKENDS)
def test_forward_reaches_the_minimiser(backend, case):
  """Row count, acceleration, constraint force, contact forces, cost and suboptimality of one forward against the
  certified fp64 minimiser, world by world."""
  out = run(backend, case)
  m = model(case)
  refs = references(backend, case, out)
  assert_case(case, m, out, refs)
  check(backend, out, refs)


@pytest.mark.parametrize("path", [p for p in PATHS if p != "newton"])
@pytest.mark.parametrize("case", ["g1", "nv64_nbody64"])
@pytest.mark.parametrize("backend", ENGINES)
def test_every_solver_path_reaches_the_minimiser(backend, case, path):
  """The full Newton problem, the dense factorisation, CG and a tiny tolerance on the states of the default path."""
  out = run(backend, case, path)
  refs = references(backend, case, out)
  assert out["options"] == {k: float(np.float32(v)) for k, v in PATHS[path].items()}, out["options"]
  if path == "full":
    assert (out["solver_nd"][out["nefc"] > 0] == int(model(case).nv)).all()
  if path == "cg":  # (the same stop rules on another direction: more, cheaper iterations than Newton)
    assert out["solver_niter"].sum() > run(backend, case)["solver_niter"].sum()
  check(backend, out, refs, path)


def test_the_oracle_builds_the_reference_rows():
  """The oracle's efc_J, efc_pos, efc_margin, efc_R, efc_D, efc_aref (limits first, then contacts in list order) equal
  the reference's to 1e-12, and its qacc at tolerance 1e-14 is the minimiser of the reference's rows with the oracle's
  own M and qfrc_smooth to 1e-9.  On G1 and multijoint, whose fp32-rounded body quaternions are not unit, J, aref and
  qacc are held to ORACLE_TOL's looser bounds (see there)."""
  for case in CASES:
    m = model(case)
    quat = arr(m, "body_quat", 4)[1:]
    unit = np.abs((quat**2).sum(1) - 1).max() < 1e-12
    assert unit == (case not in ("g1", "multijoint")), case
    be, *_ = open_backend("oracle", case, {})
    try:
      be.forward()
      out = outputs(be)
      qM, qfrc = be.a("qM"), be.a("qfrc_smooth")
    finally:
      be.close()
    refs = references("oracle", case, out)
    nv = int(m.nv)
    for w, S in enumerate(refs):
      k = S["nefc"]
      got = dict(J=out["efc_J"][w, :k * nv].reshape(k, nv), pos=out["efc_pos"][w, :k], margin=out["efc_margin"][w, :k],
                 R=out["efc_R"][w, :k], D=out["efc_D"][w, :k], aref=out["efc_aref"][w, :k])
      for f, v in got.items():
        e = relerr(v.reshape(1, -1), S[f].reshape(1, -1))[0]
        assert e <= ORACLE_TOL["rows" if unit or f not in ("J", "aref") else "rows_J"], (case, w, f, e)
      M = qM[w].reshape(nv, nv)
      own = dict(S, M=M, a_s=np.linalg.solve(M, qfrc[w]))
      a = solve(own)["a"]
      e = relerr(out["qacc"][w:w + 1], a[None])[0]
      assert e <= (ORACLE_TOL["rows_qacc"] if unit else ORACLE_TOL["qacc"]), (case, w, e)


# ---- 7. warm starts ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("backend", ENGINES)
def test_the_answer_does_not_depend_on_the_warm_start(backend):
  """G1 from qacc_warmstart 0, a_s, a* and a* + d (d of 10x max|a*|), and through step with a changed control: every
  run meets the acceleration tolerance.  Which start survives MuJoCo's rule (start from a_s when it is cheaper) shows
  in the iteration count: a* + d is dropped (the iterations of the start from a_s), a* is kept (at most one).  The
  shifted start of step adds a_s - qacc_smooth_prev to the warm start: with qacc_warmstart = a* + d and
  qacc_smooth_prev = a_s + d it lands on a* and is kept; with the control unchanged the same inputs get no shift and
  fall back to a_s."""
  case = "g1"
  refs = references(backend, case, run(backend, case))
  a_star = np.stack([S["a"] for S in refs])
  a_s = np.stack([S["a_s"] for S in refs])
  d = np.random.default_rng(11).normal(0.0, 10.0 * np.abs(a_star).max(), a_star.shape)
  be, m, rows, st = open_backend(backend, case, {})
  niter = {}
  try:
    for name, ws in {"zero": 0 * a_star, "smooth": a_s, "star": a_star, "far": a_star + d}.items():
      be.load(dict(st, qacc_warmstart=f32(ws)))
      be.forward()
      check(backend, outputs(be), refs, keys=("qacc",))
      niter[name] = be.a("solver_niter").ravel()
    assert int(m.nu) > 0
    for shifted in (True, False):
      be.load(dict(st, ctrl_prev=st["ctrl"] + (0.1 if shifted else 0.0), qacc_smooth_prev=f32(a_s + d),
                   qacc_warmstart=f32(a_star + d)))
      be.step_n(1)
      check(backend, outputs(be), refs, keys=("qacc",))
      niter[shifted] = be.a("solver_niter").ravel()
  finally:
    be.close()
  assert (niter["far"] == niter["smooth"]).all() and (niter[False] == niter["smooth"]).all(), niter
  assert (niter["star"] <= 1).all() and (niter[True] <= 1).all() and (niter["smooth"] > 1).any(), niter


# ---- 8. one step ---------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("integrator", [EULER, IMPLICITFAST])
@pytest.mark.parametrize("case", ["g1", "nu58", "convex"])
@pytest.mark.parametrize("backend", BACKENDS)
def test_one_step_follows_the_reference_forces(backend, case, integrator):
  """qvel and qpos after one step against the reference integrator driven by f*."""
  be, m, rows, st = open_backend(backend, case, {})
  try:
    be.set("integrator", integrator)
    be.step_n(1)
    q1, v1 = be.a("qpos"), be.a("qvel")
  finally:
    be.close()
  refs = references(backend, case, run(backend, case))
  h = float(m.opt_timestep)
  T = tol(backend)
  for w, (r, _, _) in enumerate(smooth_parts(case, len(q1))):
    q, v = r.step(st["qpos"][w], st["qvel"][w], st["ctrl"][w] if r.nu else [], st["qfrc_applied"][w],
                  st["xfrc_applied"][w], h, integrator, qfrc_constraint=refs[w]["qfrc"])
    ev, eq = relerr(v1[w:w + 1], v[None])[0], relerr(q1[w:w + 1], q[None])[0]
    assert ev <= T["qvel"] and eq <= T["qpos"], (w, ev, eq)


# ---- 9. the tolerances are tight enough to matter -------------------------------------------------------------------

PERTURBATIONS = ["pyramid", "impratio", "refsafe", "power", "solmix", "priority", "gap", "body1", "tangent", "newton"]


@pytest.mark.parametrize("drop", PERTURBATIONS)
def test_every_reference_perturbation_is_detected(drop):
  """With one formula of the reference changed, some case's kernel comparison (host emulation) fails by at least 10x
  its tolerance, or the row count differs."""
  worst = 0.0
  for case in CASES:
    out = run("emul", case)
    E = errors(out, references("emul", case, out, drop=(drop,)))
    if (E["nefc"] > 0).any():
      worst = np.inf
      break
    worst = max(worst, *(E[k].max() / KERNEL_TOL[k] for k in ("qacc", "qfrc", "force")))
  assert worst >= 10.0, (drop, worst)

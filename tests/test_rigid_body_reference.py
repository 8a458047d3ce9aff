"""The contact-free dynamics of the step kernel and of the oracle (oracle/b2_oracle.c) against an independent fp64
rigid-body model.

The kernel and the oracle compute the smooth dynamics the same way: com-based motion vectors (`cdof`, `cvel`),
composite rigid-body inertias and a recursive Newton-Euler pass.  The other tests compare the two with each other, so
a convention both got wrong would pass them all.  `Rigid` below is a second formulation, written from rigid-body
mechanics and reading nothing but the model's arrays and one world's rows of the per-world fields:

  kinematics   body frames by rotation matrices (Rodrigues for hinges), joint by joint in body order
  velocities   point Jacobians: a dof moves a point of body b when it is on b's chain; a hinge or a free joint's
               angular dof (body-frame axis, through the body origin) by axis x (point - anchor), a slide or a free
               joint's linear dof (world axis) by its axis
  M            sum over bodies of m Jp^T Jp + Jr^T I_w Jr, plus the armature
  qfrc_bias    Newton-Euler on every body along q(t) = q (+) v t (the motion with qacc = 0): the com acceleration and
               the angular acceleration are central differences of Jp(q(t)) v and Jr(q(t)) v, Richardson-extrapolated
  forces       actuators (gain, bias, gear, ctrl and force clamps), damping and stiffness, qfrc_applied, and
               xfrc_applied as a force at the body com and a torque
  step         v' = v + h (M + h D - h sum gear^2 b2)^-1 qfrc_smooth (the actuator sum for implicitfast only, without
               clamped actuators), q' = q (+) h v'

It is compared with three backends: the fp64 oracle and the host-emulated library (CPU suite), and the H100 (`-m gpu`).
Every case asserts the condition it exists for.  Errors are norm-wise relative per world (`util.relerr`).  Every input
(model arrays, per-world rows, states) is rounded to fp32 first, so that all backends and the reference see the same
numbers.
"""

import copy
import functools
import re
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle.oracle import Oracle
from test_model_fields import Eng
from util import _quat_mul, convex_scene, convex_states, make_states, relerr

sys.path.append(str(Path(__file__).resolve().parents[1] / "tools"))
from synth_models import robot_xml  # noqa: E402

MINVAL = 1e-15  # mjMINVAL
FREE, SLIDE, HINGE = 0, 2, 3
EULER, IMPLICITFAST = 0, 3

BACKENDS = ["oracle", "emul", pytest.param("cuda", marks=pytest.mark.gpu)]
ENGINES = ["emul", pytest.param("cuda", marks=pytest.mark.gpu)]
NWORLD = {"oracle": 4, "emul": 4, "cuda": 8}
NWIDE = 130  # G1 on the GPU: the last CTA is partial

# ---- tolerances ----------------------------------------------------------------------------------------------------
# fp64 oracle: kinematics, M and forces are the same sums in another order; the bias carries the reference's
# difference error (the Richardson step below gives <= 3e-11 on these cases)
ORACLE_TOL = dict(kin=1e-12, qM=1e-12, bias=1e-8, qacc=1e-8, qpos=1e-10, qvel=1e-8)
# fp32 kernel near the origin.  Measured worst cases over every case here, host emulation | H100 80GB HBM3 (approximate
# sincos, reciprocals and square roots): kinematics 4.9e-7 | 1.8e-6, cvel and derived velocities 9.0e-7 | 1.9e-6,
# qM 1.1e-6 | 1.3e-6, qfrc_bias and qfrc_smooth 2.7e-6 | 3.3e-6, qacc_smooth 6.8e-5 | 6.3e-5 (M of the convex scene's
# light bodies and the 64-dof robot is ill-conditioned), qpos after one step 1.2e-7 | 1.7e-7 and after four 1.8e-6 |
# 1.5e-6, qvel after one step 8.8e-5 | 1.2e-4 and after four 5.7e-5 | 5.8e-5 (qvel and qpos bounds scale with steps)
KERNEL_TOL = dict(kin=5e-6, vel=6e-6, qM=4e-6, bias=1e-5, qacc=2e-4, qpos=1e-6, qvel=5e-4)
# the identity M qacc = qfrc_smooth + qfrc_constraint on constrained worlds (fp32 solve of M against the forces)
IDENTITY_TOL = {"oracle": 1e-10, "kernel": 1e-5}


# ---- the reference -------------------------------------------------------------------------------------------------


def qmat(q):
  """Rotation matrix of a quaternion (w, x, y, z), normalised first."""
  w, x, y, z = np.asarray(q, np.float64) / np.linalg.norm(q)
  return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                   [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                   [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def rodrigues(axis, ang):
  a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
  K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
  return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


class Rigid:
  """fp64 rigid-body model of one world: the model's arrays, with the per-world fields taken from `row` (field ->
  that world's values) where given."""

  def __init__(self, m, row=None):
    row = row or {}

    def i(k):
      return np.asarray(m.arrays[k]).astype(int).ravel()

    def f(k, width=0):  # the world's row where given, else the model's values; (count, width) or (count,)
      v = np.asarray(row.get(k, m.arrays[k]), np.float64)
      return v.reshape(-1, width) if width else v.ravel()

    self.nb, self.nv, self.nu = int(m.nbody), int(m.nv), int(m.nu)
    self.parent, self.rootid = i("body_parentid"), i("body_rootid")
    self.jntadr, self.jntnum = i("body_jntadr"), i("body_jntnum")
    self.jtype, self.qadr, self.dadr = i("jnt_type"), i("jnt_qposadr"), i("jnt_dofadr")
    self.body_pos, self.body_quat = f("body_pos", 3), f("body_quat", 4)
    self.ipos, self.iquat, self.inertia = f("body_ipos", 3), f("body_iquat", 4), f("body_inertia", 3)
    self.mass, self.subtreemass = f("body_mass"), f("body_subtreemass")
    self.jnt_pos, self.jnt_axis, self.stiffness = f("jnt_pos", 3), f("jnt_axis", 3), f("jnt_stiffness")
    self.qpos0, self.armature, self.damping = f("qpos0"), f("dof_armature"), f("dof_damping")
    self.geom_body, self.geom_pos, self.geom_quat = i("geom_bodyid"), f("geom_pos", 3), f("geom_quat", 4)
    self.site_body, self.site_pos, self.site_quat = i("site_bodyid"), f("site_pos", 3), f("site_quat", 4)
    if self.nu:
      self.trn, self.gear = i("actuator_trnid"), f("actuator_gear")
      self.gainprm, self.biasprm = f("actuator_gainprm", 10), f("actuator_biasprm", 10)
      self.ctrllimited, self.forcelimited = i("actuator_ctrllimited") != 0, i("actuator_forcelimited") != 0
      self.ctrlrange, self.forcerange = f("actuator_ctrlrange", 2), f("actuator_forcerange", 2)
    self.gravity = np.asarray(m.opt_gravity, np.float64)
    # on[b, c]: body c is b or one of its ancestors (parents precede their children); a dof moves body b when it
    # belongs to a body on b's chain
    on = np.eye(self.nb, dtype=bool)
    for b in range(1, self.nb):
      on[b] |= on[self.parent[b]]
    self.chain = on
    self.moves = on[:, i("dof_bodyid")]  # (nb, nv)

  # -- kinematics --

  def kin(self, q):
    nb, nv = self.nb, self.nv
    P, R = np.zeros((nb, 3)), np.zeros((nb, 3, 3))
    R[0] = np.eye(3)
    axis, anchor, rot = np.zeros((nv, 3)), np.zeros((nv, 3)), np.zeros(nv, bool)
    for b in range(1, nb):
      p, r = P[self.parent[b]] + R[self.parent[b]] @ self.body_pos[b], R[self.parent[b]] @ qmat(self.body_quat[b])
      for j in range(self.jntadr[b], self.jntadr[b] + self.jntnum[b]):
        a, d = self.qadr[j], self.dadr[j]
        if self.jtype[j] == FREE:
          p, r = q[a:a + 3].copy(), qmat(q[a + 3:a + 7])
          axis[d:d + 3] = np.eye(3)
          axis[d + 3:d + 6], anchor[d + 3:d + 6], rot[d + 3:d + 6] = r.T, p, True  # body-frame axes, at the origin
          continue
        an, ax, dq = p + r @ self.jnt_pos[j], r @ self.jnt_axis[j], q[a] - self.qpos0[a]
        axis[d] = ax
        if self.jtype[j] == SLIDE:
          p = p + ax * dq
        else:
          assert self.jtype[j] == HINGE, self.jtype[j]
          anchor[d], rot[d] = an, True
          r = rodrigues(ax, dq) @ r
          p = an - r @ self.jnt_pos[j]
      P[b], R[b] = p, r
    xipos = P + np.einsum("bij,bj->bi", R, self.ipos)
    ximat = np.einsum("bij,bjk->bik", R, np.array([qmat(x) for x in self.iquat]))
    desc = self.chain.T * self.mass[None, :]  # desc[b, c] = mass of c when c is in b's subtree
    big = self.subtreemass >= MINVAL
    scom = xipos.copy()
    scom[big] = (desc @ xipos)[big] / self.subtreemass[big, None]
    gm = np.array([qmat(x) for x in self.geom_quat]) if len(self.geom_quat) else np.zeros((0, 3, 3))
    sm = np.array([qmat(x) for x in self.site_quat]) if len(self.site_quat) else np.zeros((0, 3, 3))
    gb, sb = self.geom_body, self.site_body
    return dict(xpos=P, xmat=R, xipos=xipos, ximat=ximat, subtree_com=scom,
                geom_xpos=P[gb] + np.einsum("gij,gj->gi", R[gb], self.geom_pos),
                geom_xmat=np.einsum("gij,gjk->gik", R[gb], gm),
                site_xpos=P[sb] + np.einsum("gij,gj->gi", R[sb], self.site_pos),
                site_xmat=np.einsum("gij,gjk->gik", R[sb], sm), axis=axis, anchor=anchor, rot=rot)

  def jac(self, K, pts):
    """Point Jacobians (nb, nv, 3) of the body-fixed points `pts` (nb, 3) of every body: linear and angular."""
    ax, rot = K["axis"][None], K["rot"][None, :, None]
    lin = np.where(rot, np.cross(ax, pts[:, None, :] - K["anchor"][None]), ax)
    mv = self.moves[:, :, None]
    return mv * lin, mv * rot * ax

  def inertia_w(self, K):
    return np.einsum("bij,bj,bkj->bik", K["ximat"], self.inertia, K["ximat"])

  def mass_matrix(self, K):
    Jp, Jr = self.jac(K, K["xipos"])
    return (np.diag(self.armature) + np.einsum("b,bvk,bwk->vw", self.mass, Jp, Jp) +
            np.einsum("bvk,bkl,bwl->vw", Jr, self.inertia_w(K), Jr))

  def integrate(self, q, v, t):
    """q (+) v t: linear dofs and joints add, a free joint's quaternion turns by its body-frame rate."""
    q = np.array(q, np.float64)
    for j in range(len(self.jtype)):
      a, d = self.qadr[j], self.dadr[j]
      if self.jtype[j] != FREE:
        q[a] += t * v[d]
        continue
      q[a:a + 3] += t * v[d:d + 3]
      w = np.asarray(v[d + 3:d + 6], np.float64)
      n = np.linalg.norm(w)
      quat = q[a + 3:a + 7] / np.linalg.norm(q[a + 3:a + 7])
      if n > 0:
        quat = _quat_mul(quat, np.r_[np.cos(0.5 * n * t), np.sin(0.5 * n * t) * w / n])
      q[a + 3:a + 7] = quat / np.linalg.norm(quat)
    return q

  def bias(self, q, v):
    """Newton-Euler forces of the motion with qacc = 0, mapped to the dofs by the com Jacobians."""
    v = np.asarray(v, np.float64)

    def rates(t):
      K = self.kin(self.integrate(q, v, t))
      Jp, Jr = self.jac(K, K["xipos"])
      return np.einsum("bvk,v->bk", Jp, v), np.einsum("bvk,v->bk", Jr, v)

    _, w = rates(0.0)
    # the step scales with the fastest rate (joint speeds, and body spins that the joints' sum makes): h * rate = 1e-2
    # keeps the Richardson-extrapolated central difference (error h^4) near 1e-11 at every speed
    h = 1e-2 / max(1.0, np.abs(v).max(), np.linalg.norm(w, axis=1).max())

    def central(hh):
      (pa, wa), (pb, wb) = rates(hh), rates(-hh)
      return (pa - pb) / (2 * hh), (wa - wb) / (2 * hh)

    (a1, al1), (a2, al2) = central(h), central(h / 2)
    acc, alpha = (4 * a2 - a1) / 3, (4 * al2 - al1) / 3
    K = self.kin(q)
    Jp, Jr = self.jac(K, K["xipos"])
    I = self.inertia_w(K)
    F = self.mass[:, None] * (acc - self.gravity)
    T = np.einsum("bij,bj->bi", I, alpha) + np.cross(w, np.einsum("bij,bj->bi", I, w))
    return np.einsum("bvk,bk->v", Jp, F) + np.einsum("bvk,bk->v", Jr, T)

  # -- forces --

  def actuation(self, q, v, ctrl):
    """Actuator forces, their generalised sum and which of them sit at a force limit."""
    if not self.nu:
      return np.zeros(0), np.zeros(self.nv), np.zeros(0, bool)
    qa, da = self.qadr[self.trn], self.dadr[self.trn]
    c = np.asarray(ctrl, np.float64)
    c = np.where(self.ctrllimited, np.clip(c, self.ctrlrange[:, 0], self.ctrlrange[:, 1]), c)
    f = (self.gainprm[:, 0] * c + self.biasprm[:, 0] + self.biasprm[:, 1] * self.gear * q[qa] +
         self.biasprm[:, 2] * self.gear * v[da])
    lo, hi = self.forcerange[:, 0], self.forcerange[:, 1]
    clamped = self.forcelimited & ((f <= lo) | (f >= hi))
    f = np.where(self.forcelimited, np.clip(f, lo, hi), f)
    qf = np.zeros(self.nv)
    np.add.at(qf, da, self.gear * f)
    return f, qf, clamped

  def forward(self, q, v, ctrl, qfrc_applied, xfrc_applied):
    """Every compared output of a forward at one state."""
    q, v = np.asarray(q, np.float64), np.asarray(v, np.float64)
    K = self.kin(q)
    Jp, Jr = self.jac(K, K["xipos"])
    M = self.mass_matrix(K)
    bias = self.bias(q, v)
    passive = -self.damping * v
    hs = (self.jtype != FREE)
    np.add.at(passive, self.dadr[hs], -self.stiffness[hs] * (q[self.qadr[hs]] - self.qpos0[self.qadr[hs]]))
    force, qact, clamped = self.actuation(q, v, ctrl)
    xf = np.asarray(xfrc_applied, np.float64).reshape(self.nb, 6)
    ext = np.einsum("bvk,bk->v", Jp, xf[:, :3]) + np.einsum("bvk,bk->v", Jr, xf[:, 3:])
    smooth = passive - bias + qfrc_applied + qact + ext
    w = np.einsum("bvk,v->bk", Jr, v)
    at = lambda pts: np.einsum("bvk,v->bk", self.jac(K, pts)[0], v)  # noqa: E731  velocity of body-fixed points
    R = K["xmat"]
    lin = at(K["xpos"])
    out = {k: K[k] for k in ("xpos", "xmat", "xipos", "ximat", "subtree_com", "geom_xpos", "geom_xmat", "site_xpos",
                             "site_xmat")}
    out.update(
        cvel=np.concatenate([w, at(K["subtree_com"][self.rootid])], axis=1),
        link_vel_w=np.concatenate([lin, w], axis=1),
        com_vel_w=np.concatenate([at(K["xipos"]), w], axis=1),
        link_state_b=np.concatenate([np.einsum("bji,bj->bi", R, lin), np.einsum("bji,bj->bi", R, w),
                                     np.einsum("bji,j->bi", R, np.array([0.0, 0.0, -1.0]))], axis=1),
        heading=np.arctan2(R[:, 1, 0], R[:, 0, 0]), heading_weight=np.hypot(R[:, 1, 0], R[:, 0, 0]),
        qM=M, qfrc_bias=bias, qfrc_smooth=smooth, qacc_smooth=np.linalg.solve(M, smooth), actuator_force=force,
        clamped=clamped)
    return out

  def step(self, q, v, ctrl, qfrc_applied, xfrc_applied, h, integrator, qfrc_constraint=0.0):
    """One step; `qfrc_constraint` (a given constraint force) is added to the smooth forces."""
    S = self.forward(q, v, ctrl, qfrc_applied, xfrc_applied)
    A = S["qM"] + h * np.diag(self.damping)
    if integrator == IMPLICITFAST and self.nu:
      free = ~S["clamped"]
      np.add.at(A, (self.dadr[self.trn][free],) * 2, -h * (self.gear**2 * self.biasprm[:, 2])[free])
    v1 = np.asarray(v, np.float64) + h * np.linalg.solve(A, S["qfrc_smooth"] + qfrc_constraint)
    return self.integrate(q, v1, h), v1


# ---- models, per-world rows and states -----------------------------------------------------------------------------


def f32(v):
  return np.asarray(v, dtype=np.float32).astype(np.float64)


def f32_model(m):
  """The model with every float array rounded to fp32, as the engine holds it."""
  m = copy.copy(m)
  m.arrays = {k: (f32(v) if np.asarray(v).dtype.kind == "f" else v) for k, v in m.arrays.items()}
  m.opt_gravity = f32(m.opt_gravity)
  return m


FIXED_XML = """<mujoco><compiler angle="radian"/><option timestep="0.004" integrator="implicitfast"/>
<worldbody><geom name="floor" type="plane" size="0 0 1"/>
 <body name="cart" pos="0.1 -0.2 1.5" quat="0.95 0.1 -0.2 0.2">
  <joint name="s0" type="slide" axis="1 0 0" range="-5 5" limited="false" damping="0.3" stiffness="4" armature="0.02"/>
  <geom type="box" size="0.1 0.05 0.04" mass="2" contype="0" conaffinity="0"/>
  <body name="arm" pos="0.05 0.02 -0.03" quat="0.9 0.3 0.1 -0.2">
   <joint name="h1" pos="0.02 -0.03 0.01" axis="0.3 1 0.2" limited="false" damping="0.2" stiffness="3"/>
   <geom type="capsule" fromto="0 0 0 0.02 0 -0.25" size="0.03" mass="0.7" contype="0" conaffinity="0"/>
   <site name="tip" pos="0 0.01 -0.25" quat="0.8 0 0.6 0"/>
   <body name="fore" pos="0.01 0.02 -0.25">
    <joint name="h2" pos="0.01 0 0.02" axis="1 0 0" limited="false" armature="0.01"/>
    <joint name="s2" type="slide" axis="0 0.6 0.8" limited="false" damping="0.5"/>
    <geom type="capsule" fromto="0 0 0 0 0.03 -0.2" size="0.025" mass="0.5" contype="0" conaffinity="0"/>
   </body>
  </body>
 </body>
 <body name="wheel" pos="-0.4 0.3 1.2" quat="0.7 0 0.7 0">
  <joint name="h3" axis="0 0 1" pos="0.03 0 0" limited="false"/>
  <geom type="box" size="0.12 0.05 0.02" pos="0.05 0 0" mass="1" contype="0" conaffinity="0"/>
 </body>
 <body name="mount" pos="0.3 0.3 2.0"><site name="hook" pos="0 0 0.1"/></body>
</worldbody>
<actuator>
 <motor joint="s0" gear="1.7" ctrllimited="true" ctrlrange="-1 1" forcelimited="true" forcerange="-0.8 0.8"/>
 <velocity joint="h1" kv="2" gear="0.6"/>
 <position joint="h2" kp="30" kv="1.5" gear="1.3" ctrllimited="true" ctrlrange="-0.5 0.5"/>
 <motor joint="h3" gear="0.8"/>
</actuator></mujoco>"""

SYNTH = {  # tools/synth_models.py robots of test_model_shapes_gpu: (seed, limbs, joints, options)
  "multijoint": (2, 5, 5, dict(dofs=38, joints_per_body=3, offsets=True, actuate_all=True)),
  "nu58": (1, 6, 12, dict(dofs=58, actuate_all=True)),
  "nv64_nbody64": (2, 4, 18, dict(dofs=58, feet=True)),
}
CASES = ["g1", "go1", "multijoint", "nu58", "nv64_nbody64", "convex", "fixed"]


@functools.cache
def model(case):
  from mjlab_b200.asset_zoo import load_compiled
  from mjlab_b200.compiler import Spec

  if case in ("g1", "go1"):
    m = load_compiled(case + "_flat")
  elif case in SYNTH:
    seed, limbs, joints, kw = SYNTH[case]
    # (the robot's own geoms made visual-only: its limbs overlap at qpos0, and contacts are not this file's subject)
    xml = re.sub(r'<geom (?!name="floor")', '<geom contype="0" conaffinity="0" ',
                 robot_xml(np.random.default_rng(seed), limbs, joints, **kw))
    m = Spec.from_string(xml).compile()
  elif case == "convex":
    m = convex_scene()[0]
  else:
    m = Spec.from_string(FIXED_XML).compile()
  return m


@functools.cache
def model32(case):
  return f32_model(model(case))


def arr(m, k, w=None):
  a = np.asarray(m.arrays[k])
  return a.reshape(len(a), -1) if w else a.ravel()


def turn(q, ang, rng):
  """Unit quaternions `q` (k, 4) turned by up to `ang` radians about random axes."""
  ax = rng.normal(size=(len(q), 3))
  ax /= np.linalg.norm(ax, axis=1, keepdims=True)
  t = rng.uniform(-ang, ang, (len(q), 1))
  r = _quat_mul(q, np.concatenate([np.cos(t / 2), ax * np.sin(t / 2)], axis=1))
  return r / np.linalg.norm(r, axis=1, keepdims=True)


def world_rows(m, n, rng):
  """Per-world values of the fields the dynamics read: (n, count * width) rows, each world its own draw."""
  jt = arr(m, "jnt_type")
  nb = int(m.nbody)
  parent = arr(m, "body_parentid")
  massive = arr(m, "body_mass") > 0
  joint = np.nonzero(jt != FREE)[0]
  jdof, jq = arr(m, "jnt_dofadr")[joint], arr(m, "jnt_qposadr")[joint]
  rows = {}
  for w in range(n):
    r = {}
    r["body_mass"] = np.where(massive, arr(m, "body_mass") * rng.uniform(0.8, 1.25, nb), 0.0)
    sub = r["body_mass"].copy()
    for b in range(nb - 1, 0, -1):
      sub[parent[b]] += sub[b]
    r["body_subtreemass"] = sub  # (consistent with the masses: subtree_com stays the com)
    r["body_ipos"] = arr(m, "body_ipos", 3) + rng.uniform(-0.01, 0.01, (nb, 3)) * massive[:, None]
    r["body_iquat"] = turn(arr(m, "body_iquat", 4), 0.6, rng)
    r["body_inertia"] = arr(m, "body_inertia", 3) * rng.uniform(0.7, 1.4, (nb, 3))
    r["dof_armature"] = arr(m, "dof_armature") + rng.uniform(0.0, 0.05, int(m.nv))
    r["dof_damping"] = arr(m, "dof_damping").copy()
    r["dof_damping"][jdof] += rng.uniform(0.0, 1.0, len(jdof))
    r["jnt_stiffness"] = arr(m, "jnt_stiffness").copy()
    r["jnt_stiffness"][joint] += rng.uniform(0.0, 5.0, len(joint))
    r["body_pos"] = arr(m, "body_pos", 3) + rng.uniform(-0.01, 0.01, (nb, 3))  # (a free joint's body ignores it)
    r["jnt_pos"] = arr(m, "jnt_pos", 3).copy()
    r["jnt_pos"][joint] += rng.uniform(-0.01, 0.01, (len(joint), 3))
    r["qpos0"] = arr(m, "qpos0").copy()
    r["qpos0"][jq] += rng.uniform(-0.05, 0.05, len(jq))
    if int(m.nu):
      r["actuator_gainprm"] = arr(m, "actuator_gainprm", 10) * np.r_[rng.uniform(0.8, 1.25), np.ones(9)]
      r["actuator_biasprm"] = arr(m, "actuator_biasprm", 10) * np.r_[1.0, rng.uniform(0.8, 1.25, 2), np.ones(7)]
      r["actuator_gear"] = arr(m, "actuator_gear") * rng.uniform(0.7, 1.4, int(m.nu))
    for k, v in r.items():
      rows.setdefault(k, []).append(np.asarray(v, np.float64).ravel())
  return {k: np.stack(v) for k, v in rows.items()}


def free_joints(m):
  return np.nonzero(arr(m, "jnt_type") == FREE)[0]


def lifted_states(m, n, seed, far=0.0, spin=10.0):
  """States high above the floor (moved `far` metres along x), every limited joint in the middle of its range,
  unlimited hinges beyond +-pi, free quaternions of norm ~0.5 or ~1.8.  Every odd world is fast: bases spin at `spin`
  rad/s and joints move at up to 20 rad/s (limited ones no faster than keeps them inside their range for four steps).
  Controls fall outside their ranges, forces reach their limits, and qfrc_applied and xfrc_applied (on five bodies)
  are non-zero."""
  rng = np.random.default_rng(seed)
  nv, nu, nb = int(m.nv), int(m.nu), int(m.nbody)
  key = m.keys.get("robot/init_state")  # (the robots' standing pose is free of self-contacts; qpos0 need not be)
  q = np.tile(np.asarray(key["qpos"] if key else arr(m, "qpos0"), np.float64), (n, 1))
  depth = np.zeros(nb, int)
  for b in range(1, nb):
    depth[b] = depth[arr(m, "body_parentid")[b]] + 1
  jt, qa, da = arr(m, "jnt_type"), arr(m, "jnt_qposadr"), arr(m, "jnt_dofadr")
  lim, rg = arr(m, "jnt_limited") != 0, arr(m, "jnt_range", 2)
  v = rng.uniform(-1.0, 1.0, (n, nv))
  for j in range(len(jt)):
    a, d = qa[j], da[j]
    if jt[j] == FREE:
      q[:, a:a + 3] += rng.uniform(-0.3, 0.3, (n, 3))
      q[:, a + 2] = 1.0 + 0.15 * depth.max()  # (any pose: no link is longer than 0.15 m)
      q[:, a] += far
      quat = turn(np.tile([1.0, 0.0, 0.0, 0.0], (n, 1)), np.pi, rng)
      q[:, a + 3:a + 7] = quat * rng.choice([0.5, 1.8], (n, 1)) * rng.uniform(0.9, 1.1, (n, 1))
      ax = rng.normal(size=(len(v[1::2]), 3))
      v[1::2, d + 3:d + 6] = spin * ax / np.linalg.norm(ax, axis=1, keepdims=True)
      continue
    top = 20.0
    if lim[j]:
      # within the middle 30% of the range, and no faster than leaves it within the middle 80% after four steps
      lo, hi = rg[j]
      r = hi - lo
      q[:, a] = np.clip(q[:, a], lo + 0.35 * r, hi - 0.35 * r) + rng.uniform(-0.05, 0.05, n) * r
      top = min(top, 0.25 * r / (4 * float(m.opt_timestep)))
    else:
      q[:, a] += rng.uniform(-5.0, 5.0, n)  # beyond +-pi
    v[1::2, d] = rng.uniform(-top, top, len(v[1::2]))
  st = dict(qpos=q, qvel=v, qacc_warmstart=np.zeros((n, nv)), qfrc_applied=rng.normal(0.0, 2.0, (n, nv)))
  xf = np.zeros((n, nb, 6))
  moving = np.nonzero(arr(m, "body_mass") > 0)[0]
  for w in range(n):
    bs = rng.choice(moving, size=min(5, len(moving)), replace=False)
    xf[w, bs, :3] = rng.normal(0.0, 10.0, (len(bs), 3))
    xf[w, bs, 3:] = rng.normal(0.0, 1.0, (len(bs), 3))
  st["xfrc_applied"] = xf.reshape(n, -1)
  if nu:
    cr = arr(m, "actuator_ctrlrange", 2)
    mid, half = cr.mean(axis=1), np.maximum(0.5 * (cr[:, 1] - cr[:, 0]), 0.5)
    st["ctrl"] = mid + rng.uniform(-1.6, 1.6, (n, nu)) * half  # (about a third outside the range)
  return st


def contact_free(m, rows, st, steps=4):
  """Which worlds have no constraint row at their state and over `steps` steps of either integrator.  (The fp64
  oracle only picks the states; what is compared is each backend against the reference.)"""
  n = len(st["qpos"])
  o = Oracle(m, nworld=n)
  for k, v in rows.items():
    o.model_field(k)[:] = v
  ok = np.ones(n, bool)
  for integrator in (EULER, IMPLICITFAST):
    o.set_option("integrator", integrator)
    for k, v in st.items():
      o.field(k)[:] = v
    o.forward()
    ok &= o.nefc.ravel() == 0
    for _ in range(steps):
      o.step()
      ok &= o.nefc.ravel() == 0
  return ok


def draw(case, m, n, seed, far):
  rows = world_rows(m, n, np.random.default_rng(seed))
  if case != "convex":
    # (the 64-body robot's long chains carry slides: spun at 10 rad/s they reach their limits within four steps)
    return rows, lifted_states(m, n, seed, far=far, spin=2.0 if case == "nv64_nbody64" else 10.0)
  st = convex_states(m, *convex_scene()[1:], n, seed=seed, drop=True)
  rng = np.random.default_rng(seed)
  st["qvel"] = rng.uniform(-1, 1, st["qvel"].shape)
  st["qvel"][1::2] *= 10.0
  quat = st["qpos"].reshape(n, -1, 7)[:, :, 3:]  # (a view: nine free joints, one after the other)
  quat *= 1.7  # non-unit quaternions
  st["qfrc_applied"] = rng.normal(0.0, 2.0, st["qvel"].shape)
  xf = np.zeros((n, int(m.nbody), 6))
  xf[:, 1:] = rng.normal(0.0, 2.0, (n, int(m.nbody) - 1, 6))
  st["xfrc_applied"] = xf.reshape(n, -1)
  return rows, st


def case_setup(case, n, seed=1, far=0.0, fp32=True):
  """The model, per-world rows and lifted states of a case, after asserting what the case exists for.  The states
  are the first `n` of 4n draws that stay free of contacts and limits for four steps.  With `fp32` every value is
  rounded to fp32 (the engine's inputs); the fp64 oracle is given the model's own values."""
  m = model32(case) if fp32 else model(case)
  rnd = f32 if fp32 else (lambda v: np.asarray(v, np.float64))
  rows, st = draw(case, m, 4 * n, seed, far)
  rows, st = ({k: rnd(v) for k, v in d.items()} for d in (rows, st))
  keep = np.nonzero(contact_free(m, rows, st))[0]
  assert len(keep) >= n, f"{len(keep)} contact-free states of {4 * n}"
  rows, st = ({k: v[keep[:n]] for k, v in d.items()} for d in (rows, st))
  jt = arr(m, "jnt_type")
  for a in arr(m, "jnt_qposadr")[jt == FREE]:
    st["qpos"][1::2, a + 3:a + 7] *= -1  # (the same rotations: still free of contacts)
  if case in ("g1", "go1"):
    assert (jt[1:] == HINGE).all() and (arr(m, "actuator_forcelimited") != 0).all()
  elif case == "multijoint":
    # the generic kinematics walk: up to three joints on a body, hinges and slides mixed, anchors off the origin
    assert arr(m, "body_jntnum").max() == 3 and (jt == SLIDE).any() and np.abs(arr(m, "jnt_pos")).max() > 0.005
  elif case == "nu58":
    bias = arr(m, "actuator_biasprm", 10)
    position, velocity = bias[:, 1] != 0, (bias[:, 1] == 0) & (bias[:, 2] != 0)
    assert int(m.nu) == 58 and position.any() and velocity.any() and (~position & ~velocity).any()
    assert (arr(m, "actuator_ctrllimited") != 0).all() and np.abs(arr(m, "actuator_gear") - 1).min() > 0.0
  elif case == "nv64_nbody64":
    assert int(m.nv) == 64 and int(m.nbody) == 64
  elif case == "convex":
    assert len(free_joints(m)) == 9 and len(np.unique(arr(m, "body_rootid")[1:])) == 9
  else:
    # fixed base: slides and unlimited hinges, angles beyond +-pi, a massless static body (subtree_com = xipos)
    assert not len(free_joints(m)) and (jt == SLIDE).any() and (jt == HINGE).any()
    hq = arr(m, "jnt_qposadr")[jt == HINGE]
    assert (np.abs(st["qpos"][:, hq] - arr(m, "qpos0")[hq]) > np.pi).any()
    assert (arr(m, "body_subtreemass")[1:] < MINVAL).any()
  fj = free_joints(m)
  if len(fj):
    # non-unit quaternions of both signs, and fast worlds: a base spin of ~10 rad/s, joints at up to 20 rad/s
    fq, fd = arr(m, "jnt_qposadr")[fj], arr(m, "jnt_dofadr")[fj]
    quat = np.stack([st["qpos"][:, a + 3:a + 7] for a in fq], 1)
    assert np.abs(np.linalg.norm(quat, axis=2) - 1).min() > 0.05
    assert (quat[..., 0] < 0).any() and (quat[..., 0] > 0).any()
    spin = np.linalg.norm(np.stack([st["qvel"][:, d + 3:d + 6] for d in fd], 1), axis=2).max(axis=1)
    jd = arr(m, "jnt_dofadr")[jt != FREE]
    fast = spin > 9.0
    assert case == "nv64_nbody64" or (fast.any() and (~fast).any())
    if len(jd) and fast.any():
      assert np.abs(st["qvel"][fast][:, jd]).max() > 15.0
  return m, rows, st


def references(m, rows, st):
  """One Rigid per world, on that world's rows."""
  n = len(st["qpos"])
  return [Rigid(m, {k: v[w] for k, v in rows.items()}) for w in range(n)]


def ref_forward(refs, st):
  """The reference's forward outputs, (n, -1) per field."""
  n, nu = len(refs), refs[0].nu
  outs = [r.forward(st["qpos"][w], st["qvel"][w], st["ctrl"][w] if nu else [], st["qfrc_applied"][w],
                    st["xfrc_applied"][w]) for w, r in enumerate(refs)]
  return {k: np.stack([o[k] for o in outs]).reshape(n, -1) for k in outs[0]}


# ---- backends ------------------------------------------------------------------------------------------------------


class Backend:
  """The fp64 oracle or an engine (Eng: host emulation or H100) behind one interface."""

  def __init__(self, name, m, n, precision="f64", nconmax=None):
    """`nconmax`: the engine's contact pool over all worlds (the oracle holds the per-world share, and room for
    four rows per contact)."""
    self.name, self.n = name, n
    if name == "oracle":
      maxcon = -(-nconmax // n) if nconmax else 64
      self.o, self.e = Oracle(m, nworld=n, precision=precision, maxcon=maxcon, njmax=max(300, 4 * maxcon + 128)), None
    else:
      self.o, self.e = None, Eng(name, m, n, nconmax)

  def rows(self, rows):
    for k, v in rows.items():
      if self.e is None:
        self.o.model_field(k)[:] = v
      else:
        self.e.expand(k)
        self.e.model_rows(k, v)

  def load(self, st):
    for k, v in st.items():
      if self.e is None:
        self.o.field(k)[:] = v
      else:
        t = self.e.t(k)
        t[...] = torch.as_tensor(v, dtype=torch.float32, device=self.e.dev).reshape(t.shape)

  def set(self, key, value):
    (self.o.set_option if self.e is None else self.e.set)(key, value)

  def forward(self):
    self.o.forward() if self.e is None else self.e.forward()

  def step_n(self, k):
    if self.e is None:
      for _ in range(k):
        self.o.step()
    elif k == 1:
      self.e.step()
    else:
      self.e.step_n(k)

  def a(self, f):
    v = self.o.field(f) if self.e is None else self.e.a(f)
    return np.asarray(v, np.float64).reshape(self.n, -1).copy()

  def close(self):
    if self.e is not None:
      self.e.close()


def quat_mats(xq):
  """Rotation matrices of the rows of quaternions (n, 4k), flattened per world."""
  q = xq.reshape(len(xq), -1, 4)
  return np.stack([[qmat(x) if np.linalg.norm(x) > 0 else np.eye(3) for x in w] for w in q]).reshape(len(xq), -1)


KIN = ("xpos", "xmat", "xipos", "subtree_com", "geom_xpos", "geom_xmat", "site_xpos", "site_xmat")
VEL = ("cvel", "link_vel_w", "com_vel_w", "link_state_b")
DYN = ("qM", "qfrc_bias", "qfrc_smooth", "qacc_smooth", "actuator_force")


def tol_of(backend, field):
  T = ORACLE_TOL if backend == "oracle" else KERNEL_TOL
  kind = {"qM": "qM", "qfrc_bias": "bias", "qfrc_smooth": "bias", "qacc_smooth": "qacc", "actuator_force": "kin"}
  if field in VEL:
    return T.get("vel", T["kin"])
  return T[kind.get(field, "kin")]


def compare(be, ref, fields, tols=None, report=None):
  """Engine outputs against the reference world by world; returns the worst error of every field."""
  worst = {}
  for f in fields:
    if be.name == "oracle" and f in ("link_vel_w", "com_vel_w", "link_state_b"):
      continue
    if not ref[f].size:  # (no actuators, or no sites)
      continue
    got = be.a(f)
    want = ref[f]
    if f == "link_state_b":
      g = got.reshape(be.n, -1, 10)
      got = g[:, :, :9].reshape(be.n, -1)
      dh = np.angle(np.exp(1j * (g[:, :, 9] - ref["heading"])))
      eh = np.abs(dh * ref["heading_weight"]).max(axis=1)
      tol = tols[f] if tols else tol_of(be.name, f)
      assert (eh < tol).all(), ("heading", int(eh.argmax()), eh.max())
    e = relerr(got, want)
    tol = tols[f] if tols else tol_of(be.name, f)
    assert (e < tol).all(), (f, int(np.argmax(e / tol)), e.max())
    worst[f] = e.max()
  if be.name == "oracle":
    e = relerr(be.a("ximat"), ref["ximat"])
    assert e.max() < ORACLE_TOL["kin"], ("ximat", e.max())
  if "xmat" in fields:  # the quaternions (any norm and sign on input) turn the frames the matrices hold
    e = relerr(quat_mats(be.a("xquat")), ref["xmat"])
    assert e.max() < (tols["xmat"] if tols else tol_of(be.name, "xmat")), ("xquat", e.max())
    worst["xquat"] = e.max()
  if report is not None:
    report.update({k: max(v, report.get(k, 0.0)) for k, v in worst.items()})
  return worst


def setup(backend, case, seed=1, far=0.0):
  n = NWIDE if backend == "cuda" and case == "g1" else NWORLD[backend]
  m, rows, st = case_setup(case, n, seed=seed, far=far, fp32=backend != "oracle")
  be = Backend(backend, m, n)
  be.rows(rows)
  be.load(st)
  return m, rows, st, be


# ---- 1. forward ----------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("backend", BACKENDS)
def test_forward_matches_the_rigid_body_reference(backend, case):
  """Kinematics, velocities, M, bias, actuator and smooth forces after a forward, world by world, each world on its
  own model rows."""
  m, rows, st, be = setup(backend, case)
  try:
    be.forward()
    ref = ref_forward(references(m, rows, st), st)
    if int(m.nu):
      # controls outside their ranges, and forces at their limits, in the state set
      cr = arr(m, "actuator_ctrlrange", 2)
      outside = (st["ctrl"] < cr[:, 0]) | (st["ctrl"] > cr[:, 1])
      limited = arr(m, "actuator_ctrllimited") != 0
      assert (outside & limited).any() or not limited.any()
      if (arr(m, "actuator_forcelimited") != 0).any():
        assert ref["clamped"].any() and (~ref["clamped"]).any()
    compare(be, ref, KIN + VEL + DYN)
  finally:
    be.close()


def test_the_convex_scene_reference_point_lies_in_no_tree():
  """In the convex scene the com of all moving bodies (the kernel's internal reference point) is far from every
  tree's subtree com, so cvel's shift to subtree_com[root] is exercised."""
  m, rows, st = case_setup("convex", 2)
  r = references(m, rows, st)[0]
  K = r.kin(st["qpos"][0])
  c0 = (r.mass[:, None] * K["xipos"]).sum(0) / r.mass.sum()
  roots = np.unique(r.rootid[1:])
  assert np.linalg.norm(K["subtree_com"][roots] - c0, axis=1).min() > 0.1


# ---- 2. steps ------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("integrator", [EULER, IMPLICITFAST])
@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("backend", BACKENDS)
def test_contact_free_steps_match_the_reference_integrator(backend, case, integrator):
  """One step and step_n(4) from lifted states (no constraint row in any world) against the reference integrator."""
  m, rows, st, be = setup(backend, case, seed=2)
  refs = references(m, rows, st)
  h = float(m.opt_timestep)
  try:
    be.set("integrator", integrator)
    T = ORACLE_TOL if backend == "oracle" else KERNEL_TOL
    for k in (1, 4):
      be.load(st)
      be.step_n(k)
      assert (be.a("nefc") == 0).all(), be.a("nefc").ravel()
      q, v = [], []
      for w, r in enumerate(refs):
        qw, vw = st["qpos"][w], st["qvel"][w]
        for _ in range(k):
          qw, vw = r.step(qw, vw, st["ctrl"][w] if r.nu else [], st["qfrc_applied"][w], st["xfrc_applied"][w], h,
                          integrator)
        q.append(qw)
        v.append(vw)
      # (the step growth of fp32 rounding over four steps is bounded by 4x the one-step bound)
      for f, want, tol in (("qpos", np.array(q), T["qpos"] * k), ("qvel", np.array(v), T["qvel"] * k)):
        e = relerr(be.a(f), want)
        assert (e < tol).all(), (f, k, int(e.argmax()), e.max())
  finally:
    be.close()


# ---- 3. the outputs of step_n ----------------------------------------------------------------------------------------


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("backend", ENGINES)
def test_step_n_outputs_the_last_substeps_kinematics(backend, case):
  """Only the last sub-step of step_n stores poses, cvel and the derived velocities (and poses the geoms that cannot
  collide).  After step_n(4) they are the reference's at the state the last sub-step started from: the state a
  second engine reaches with step_n(3) from the same input (the kernel is bit-deterministic)."""
  m, rows, st, be = setup(backend, case, seed=3)
  twin = Backend(backend, m, be.n)
  try:
    gt = (arr(m, "geom_contype") == 0) & (arr(m, "geom_conaffinity") == 0)
    assert gt.any() or case == "convex", "no visual-only geom"
    twin.rows(rows)
    twin.load(st)
    twin.step_n(3)
    be.step_n(4)
    s3 = dict(st, qpos=twin.a("qpos"), qvel=twin.a("qvel"))
    assert relerr(s3["qpos"], st["qpos"]).min() > 1e-4  # (the outputs of an earlier state would be told apart)
    ref = ref_forward(references(m, rows, s3), s3)
    compare(be, ref, KIN + VEL)
  finally:
    be.close()
    twin.close()


# ---- 4. far from the origin ------------------------------------------------------------------------------------------


# Fields whose fp32 error grows with the distance from the origin: the arms of the dofs and the com offsets are
# differences of positions that carry fewer digits there.  60 m out they are bounded by FAR_FACTOR x the fp32 oracle's
# worst error on the same states where that exceeds their bound near the origin (test_model_shapes_gpu's rule).
# Measured worst cases, kernel | fp32 oracle, host emulation (4 worlds): cvel 1.0e-5 | 6.0e-6, qM 3.6e-6 | 3.6e-6,
# qfrc_bias 1.3e-5 | 1.3e-5, qacc_smooth 2.8e-5 | 2.7e-5; H100 80GB HBM3 (130 worlds): cvel 1.6e-5 | 1.1e-5, qM 3.9e-6
# | 3.8e-6, qfrc_bias 6.0e-5 | 5.9e-5, qacc_smooth 4.7e-5 | 4.6e-5.  (World by world the ratio of the two is noisy: up
# to 11 for cvel on the H100, in a world where the oracle happens to round well.)
FAR_FIELDS = ("cvel", "qM", "qfrc_bias", "qfrc_smooth", "qacc_smooth")
FAR_FACTOR = 4.0


@pytest.mark.parametrize("backend", ENGINES)
def test_far_from_the_origin(backend):
  """G1 60 m from the origin, the scale of the rough-terrain grid, where the positions' rounding dominates: the
  distance-dependent fields are bounded by FAR_FACTOR x the fp32 oracle's worst error, the others keep their
  bounds."""
  m, rows, st, be = setup(backend, "g1", seed=4, far=60.0)
  o32 = Backend("oracle", m, be.n, precision="f32")
  try:
    assert (st["qpos"][:, 0] > 59.0).all()
    o32.rows(rows)
    o32.load(st)
    o32.forward()
    be.forward()
    ref = ref_forward(references(m, rows, st), st)
    tols = {f: tol_of(backend, f) for f in KIN + VEL + DYN}
    far = {f: FAR_FACTOR * relerr(o32.a(f), ref[f]).max() for f in FAR_FIELDS}
    assert far["qM"] > tols["qM"] and far["qfrc_bias"] > tols["qfrc_bias"]  # (the positions' rounding dominates)
    tols.update({f: max(tols[f], far[f]) for f in FAR_FIELDS})
    tols.update({f: tols["cvel"] for f in ("link_vel_w", "com_vel_w", "link_state_b")})
    compare(be, ref, KIN + VEL + DYN, tols=tols)
  finally:
    be.close()


# ---- 5. constrained worlds -------------------------------------------------------------------------------------------


@pytest.mark.parametrize("backend", BACKENDS)
def test_constrained_worlds_satisfy_the_equations_of_motion(backend):
  """G1 on the floor with joints at and past their limits: the backend's own qacc and qfrc_constraint satisfy
  M_ref qacc = qfrc_smooth_ref + qfrc_constraint in every world."""
  n = NWORLD[backend]
  fp32 = backend != "oracle"
  m = model32("g1") if fp32 else model("g1")
  rnd = f32 if fp32 else (lambda v: np.asarray(v, np.float64))
  rows = {k: rnd(v) for k, v in world_rows(m, n, np.random.default_rng(5)).items()}
  st = make_states(m, n, seed=5, z_range=(-0.06, -0.02))  # (every world presses into the floor)
  st.update(qfrc_applied=np.zeros((n, int(m.nv))), xfrc_applied=np.zeros((n, 6 * int(m.nbody))))
  st = {k: rnd(v) for k, v in st.items()}
  be = Backend(backend, m, n)
  try:
    be.rows(rows)
    be.load(st)
    be.forward()
    assert (be.a("nefc") > 0).all()
    refs = references(m, rows, st)
    ref = ref_forward(refs, st)
    qacc, fc = be.a("qacc"), be.a("qfrc_constraint")
    lhs = np.stack([r.mass_matrix(r.kin(st["qpos"][w])) @ qacc[w] for w, r in enumerate(refs)])
    e = relerr(lhs, ref["qfrc_smooth"] + fc)
    tol = IDENTITY_TOL["oracle" if backend == "oracle" else "kernel"]
    assert (e < tol).all(), (int(e.argmax()), e.max())
  finally:
    be.close()

"""The CPU oracle against analytic cases, invariants and its committed golden vectors.

The reference holds no known-answer tests for this path (SURVEY.md §4, §8c: parity unpinned), so
these are what pin the restated algorithm."""

import json
import re
from pathlib import Path

import numpy as np
import pytest

from mjlab_b200.compiler import Spec
from oracle.oracle import _DIR, Oracle, load_library
from util import convex_scene, load_oracle, make_states, terrain_states

GOLDEN = Path(__file__).parent / "golden"

FREE_BODY = """
<mujoco><option timestep="0.002" integrator="Euler"/>
  <worldbody><body name="b" pos="0 0 1"><freejoint/>
    <geom type="box" size="0.1 0.2 0.3" mass="3"/></body></worldbody></mujoco>
"""
PENDULUM = """
<mujoco><option timestep="0.0005" integrator="Euler"/>
  <worldbody><body name="p" pos="0 0 2"><joint name="h" axis="0 1 0"/>
    <geom type="sphere" size="0.01" pos="0 0 -1" mass="1"/></body></worldbody></mujoco>
"""
BALL_ON_PLANE = """
<mujoco><option timestep="0.002"/>
  <worldbody><geom name="floor" type="plane" size="0 0 1"/>
    <body name="ball" pos="0 0 0.099"><freejoint/><geom type="sphere" size="0.1" mass="2"/></body>
  </worldbody></mujoco>
"""


def test_oracle_field_surface():
  """Every Data field keeps its name, element type and row length (tests/golden/oracle_fields.json), for a humanoid,
  a quadruped on a height field and the mesh / height-field scene; an unknown name raises."""
  from mjlab_b200.asset_zoo import load_compiled

  golden = json.loads((GOLDEN / "oracle_fields.json").read_text())
  assert sorted(golden) == ["convex_scene", "g1_flat", "go1_rough_hf"]
  for name, rows in golden.items():
    m = convex_scene()[0] if name == "convex_scene" else load_compiled(name)
    for prec in ("f64", "f32"):
      o = Oracle(m, nworld=2, maxcon=40, njmax=120, precision=prec)
      got = []
      for f, _, _ in rows:
        a = o.field(f)
        assert a.shape[0] == 2 and a.dtype in (np.int32, o.dtype), (name, f, a.shape, a.dtype)
        got.append([f, "int" if a.dtype == np.int32 else "real", a.shape[1]])
      assert got == rows, name
      with pytest.raises(KeyError):
        o.field("qpos0")  # a model array, not a Data field


def test_oracle_options():
  m = Spec.from_string(PENDULUM).compile()
  o = Oracle(m)
  for k, v in (("iterations", 7), ("ls_iterations", 9), ("tolerance", 1e-6), ("ls_tolerance", 1e-3),
               ("timestep", 1e-3), ("integrator", 0)):
    o.set_option(k, v)
  o.step()
  assert o.time[0, 0] == 1e-3
  for k in ("solver", "iteration"):
    with pytest.raises(ValueError, match=f"'{k}'"):
      o.set_option(k, 1)


def test_oracle_library_binds_every_entry_point():
  """load_library declares the signature of every b2o_* function b2_oracle.c exports, in both precisions."""
  src = (_DIR / "b2_oracle.c").read_text()
  defined = set(re.findall(r"^(?!static)\w[\w \t*]*?\b(b2o_\w+)\s*\(", src, re.M))
  assert {"b2o_create", "b2o_field", "b2o_set_option", "b2o_prim_hfield"} <= defined
  for prec in ("f64", "f32"):
    lib = load_library(prec)
    for fn in defined:
      assert hasattr(lib, fn), f"{fn} is defined in b2_oracle.c but not exported by the {prec} library"
    assert {fn for fn in defined if getattr(lib, fn).argtypes is not None} == defined, prec


def test_free_fall_and_momentum():
  m = Spec.from_string(FREE_BODY).compile()
  o = Oracle(m)
  o.forward()
  assert o.qacc[0] == pytest.approx([0, 0, -9.81, 0, 0, 0], abs=1e-12)
  # torque-free tumbling: angular momentum (world frame) is conserved, energy nearly
  o.qvel[0] = [0.3, -0.2, 0.1, 1.0, 2.0, 3.0]
  o.set_option("timestep", 1e-4)

  def ang_mom():
    o.forward()
    R = o.xmat[0].reshape(-1, 3, 3)[1]
    Ib = np.diag(m.body_inertia[1])
    Rb = R @ _quat_mat(m.body_iquat[1])
    return Rb @ Ib @ Rb.T @ (R @ o.qvel[0][3:6])

  L0 = ang_mom()
  for _ in range(2000):
    o.step()
  assert ang_mom() == pytest.approx(L0, rel=2e-3)
  assert o.qvel[0][:2] == pytest.approx([0.3, -0.2], abs=1e-12)  # linear momentum in x,y


def _quat_mat(q):
  w, x, y, z = q
  return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                   [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                   [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def test_pendulum_period():
  m = Spec.from_string(PENDULUM).compile()
  o = Oracle(m)
  o.qpos[0] = [0.05]
  h, t, crossings, prev = float(m.opt_timestep), 0.0, [], 0.05
  for _ in range(9000):
    o.step()
    t += h
    if prev > 0 >= o.qpos[0, 0]:
      crossings.append(t)
    prev = o.qpos[0, 0]
  period = np.diff(crossings).mean()
  # point mass on a massless rod of length 1 (sphere inertia 0.4 m r^2 is negligible)
  assert period == pytest.approx(2 * np.pi * np.sqrt(1.0 / 9.81), rel=2e-3)


def test_resting_contact_force_equals_weight():
  m = Spec.from_string(BALL_ON_PLANE).compile()
  o = Oracle(m)
  for _ in range(1500):
    o.step()
  assert int(o.ncon[0, 0]) == 1
  assert abs(o.qvel[0]).max() < 1e-6
  assert o.contact_force[0, 0] == pytest.approx(2 * 9.81, rel=1e-6)  # normal force = m g
  assert abs(o.contact_force[0, 1:3]).max() < 1e-9
  # frame: normal of the plane, tangents orthonormal (mju_makeFrame)
  fr = o.contact_frame[0, :9].reshape(3, 3)
  assert fr @ fr.T == pytest.approx(np.eye(3), abs=1e-12) and fr[0] == pytest.approx([0, 0, 1])


def test_mass_matrix_and_smooth_dynamics_identities(g1_model):
  n = 6
  o = Oracle(g1_model, nworld=n)
  load_oracle(o, make_states(g1_model, n, seed=5))
  o.forward()
  nv = int(g1_model.nv)
  for w in range(n):
    M = o.qM[w].reshape(nv, nv)
    assert M == pytest.approx(M.T, abs=1e-12)
    assert np.linalg.eigvalsh(M).min() > 0
    assert M @ o.qacc_smooth[w] == pytest.approx(o.qfrc_smooth[w], rel=1e-9, abs=1e-9)
    # total mass seen by the translational free-joint dofs
    assert M[0, 0] == pytest.approx(g1_model.body_mass.sum(), rel=1e-12)


def test_solver_kkt_and_constraint_signs(g1_model):
  n = 8
  o = Oracle(g1_model, nworld=n)
  load_oracle(o, make_states(g1_model, n, seed=6))
  o.set_option("tolerance", 1e-14)
  o.set_option("iterations", 60)
  o.forward()
  nv = int(g1_model.nv)
  assert int(o.nefc.max()) > 20
  for w in range(n):
    ne = int(o.nefc[w, 0])
    M = o.qM[w].reshape(nv, nv)
    J = o.efc_J[w][: ne * nv].reshape(ne, nv)
    f = o.efc_force[w][:ne]
    # stationarity: M a = qfrc_smooth + J^T f ; forces non-negative ; complementarity with Jaref
    res = M @ o.qacc[w] - o.qfrc_smooth[w] - J.T @ f
    assert abs(res).max() < 1e-6 * max(1.0, abs(o.qfrc_smooth[w]).max())
    assert (f >= 0).all()
    jar = J @ o.qacc[w] - o.efc_aref[w][:ne]
    assert f == pytest.approx(np.where(jar < 0, -o.efc_D[w][:ne] * jar, 0.0), rel=1e-9, abs=1e-9)
    assert o.qfrc_constraint[w] == pytest.approx(J.T @ f, rel=1e-9, abs=1e-9)


def test_pyramid_rows_share_regulariser(g1_model):
  o = Oracle(g1_model, nworld=1)
  load_oracle(o, make_states(g1_model, 1, seed=8, z_range=(-0.03, -0.03)))
  o.forward()
  ne = int(o.nefc[0, 0])
  types, ids, R = o.efc_type[0][:ne], o.efc_id[0][:ne], o.efc_R[0][:ne]
  pyr = np.nonzero(types == 5)[0]
  assert len(pyr) >= 4
  for c in np.unique(ids[pyr]):
    rows = pyr[ids[pyr] == c]
    assert len(rows) == 4 and np.ptp(R[rows]) == 0.0  # R = 2 mu^2 R_first on all four edges


@pytest.mark.parametrize("name", ["g1_flat_seed101", "go1_flat_seed102", "g1_tracking_flat_seed103",
                                  "go1_stairs_small_seed104"])
def test_oracle_reproduces_golden(name):
  from mjlab_b200.asset_zoo import load_compiled

  z = np.load(GOLDEN / f"{name}.npz")
  m = load_compiled(name.rsplit("_seed", 1)[0])
  n = int(z["n"])
  seed = int(z["seed"])
  st = terrain_states(m, n, seed, 1.4) if "terrain_origins" in m.arrays else make_states(m, n, seed=seed)
  for k, v in st.items():
    assert v == pytest.approx(z[f"in_{k}"], abs=0)  # the seeded inputs themselves are reproducible
  o = Oracle(m, nworld=n, maxcon=48)
  load_oracle(o, st)
  o.forward()
  assert (o.ncon == z["fwd_ncon"]).all() and (o.contact_geom == z["fwd_contact_geom"]).all()
  for f in ("qacc", "qfrc_constraint", "cvel", "sensordata", "contact_force"):
    assert o.field(f) == pytest.approx(z[f"fwd_{f}"], rel=1e-9, abs=1e-9), f
  load_oracle(o, st)
  for _ in range(3):
    o.step()
  assert o.qpos == pytest.approx(z["step3_qpos"], rel=1e-10, abs=1e-10)
  assert o.qvel == pytest.approx(z["step3_qvel"], rel=1e-8, abs=1e-8)


def test_fp32_oracle_tracks_fp64(g1_model):
  n = 4
  st = make_states(g1_model, n, seed=12)
  a, b = Oracle(g1_model, nworld=n), Oracle(g1_model, nworld=n, precision="f32")
  load_oracle(a, st)
  load_oracle(b, st)
  a.step()
  b.step()
  assert (a.ncon == b.ncon).all()
  assert np.abs(a.qvel - b.qvel).max() < 2e-3 * max(1.0, np.abs(a.qvel).max())


INCLINE = """
<mujoco><option timestep="0.002"/>
  <worldbody><geom name="floor" type="plane" size="0 0 1" friction="{mu} 0.005 0.0001"/>
    <body name="box" pos="0 0 0.0195"><freejoint/>
      <geom type="box" size="0.2 0.2 0.02" mass="1" friction="{mu} 0.005 0.0001"/></body>
  </worldbody></mujoco>
"""


@pytest.mark.parametrize("mu,theta_deg,slides", [(0.3, 30.0, True), (0.8, 20.0, False)])
def test_coulomb_friction_on_incline(mu, theta_deg, slides):
  """Known-answer check of the pyramidal friction model: a box on a plane tilted by theta (gravity is
  tilted instead of the plane) slides with a = g (sin(theta) - mu cos(theta)) along a pyramid axis when
  mu < tan(theta) and sticks otherwise."""
  from mjlab_b200.compiler import Spec

  sp = Spec.from_string(INCLINE.format(mu=mu))
  th = np.radians(theta_deg)
  sp.option.gravity = (9.81 * np.sin(th), 0.0, -9.81 * np.cos(th))
  m = sp.compile()
  o = Oracle(m)
  for _ in range(300):  # 0.6 s: let the normal direction settle
    o.step()
  v0, t0 = o.qvel[0, 0], o.time[0, 0]
  fn = []
  for _ in range(500):
    o.step()
    nc = int(o.ncon[0, 0])
    fn.append(o.contact_force[0, 0 : 3 * nc : 3].sum())
  a = (o.qvel[0, 0] - v0) / (o.time[0, 0] - t0)
  if slides:
    assert a == pytest.approx(9.81 * (np.sin(th) - mu * np.cos(th)), rel=0.03)
  else:
    assert abs(o.qvel[0, 0]) < 0.02 and abs(a) < 0.02  # held by friction (soft-constraint creep only)
  # time-averaged normal force carries the weight component perpendicular to the plane
  assert np.mean(fn) == pytest.approx(9.81 * np.cos(th), rel=0.03)


ARM = """
<mujoco><compiler angle="radian"/><option timestep="0.002" integrator="{integ}"/>
  <worldbody><body name="arm" pos="0 0 1"><joint name="h" axis="0 1 0" range="-0.5 0.5" limited="{limited}" damping="{damping}"/>
    <geom type="capsule" fromto="0 0 0 0.5 0 0" size="0.02" mass="1"/></body></worldbody>
  {actuator}
</mujoco>
"""


def test_position_actuator_steady_state_and_clamps():
  """Affine-bias position actuator (force = kp (ctrl - q) - kd qdot): a horizontal 1 kg arm (com at 0.25 m)
  settles where kp (target - q) balances gravity; a force range clamps the actuator output."""
  act = '<actuator><position joint="h" kp="{kp}" kv="2" {fr}/></actuator>'
  m = Spec.from_string(ARM.format(integ="implicitfast", limited="false", damping="0", actuator=act.format(kp=200, fr=""))).compile()
  o = Oracle(m)
  o.ctrl[:] = 0.1
  for _ in range(4000):
    o.step()
  q = o.qpos[0, 0]
  # axis +y: positive q lowers the tip; gravity torque about y for the com at 0.25 cos(q) ahead of the hinge
  tau_g = 1.0 * 9.81 * 0.25 * np.cos(q)
  assert abs(o.qvel[0, 0]) < 1e-6
  assert 200 * (0.1 - q) == pytest.approx(-tau_g, rel=1e-4)
  assert o.actuator_force[0, 0] == pytest.approx(-tau_g, rel=1e-4)
  # forcerange +-1 N m cannot hold the arm: the output sits on the clamp while the arm falls
  m = Spec.from_string(ARM.format(integ="implicitfast", limited="false", damping="0",
                                  actuator=act.format(kp=200, fr='forcerange="-1 1" forcelimited="true"'))).compile()
  o = Oracle(m)
  o.ctrl[:] = 0.0
  for _ in range(100):
    o.step()
  assert o.actuator_force[0, 0] == pytest.approx(-1.0) and o.qpos[0, 0] > 0.05


def test_joint_limit_holds_against_gravity():
  """The arm falls onto its upper limit (0.5 rad) and rests there: limit force = gravity torque, penetration
  follows the soft-constraint law f = (1/R) k imp (-r) with R = (1 - imp)/imp * dof_invweight0."""
  m = Spec.from_string(ARM.format(integ="implicitfast", limited="true", damping="0.05", actuator="")).compile()
  o = Oracle(m)
  for _ in range(6000):
    o.step()
  q = o.qpos[0, 0]
  assert abs(o.qvel[0, 0]) < 1e-5 and int(o.nefc[0, 0]) == 1
  r = 0.5 - q
  assert -2e-3 < r < 0.0  # slightly beyond the limit
  tau_g = 9.81 * 0.25 * np.cos(q)
  # default solref (0.02, 1), solimp (0.9, 0.95, 0.001, 0.5, 2): stiffness k = 1/(dmax^2 tc^2 dr^2)
  k = 1.0 / (0.95**2 * 0.02**2 * 1.0)
  x = abs(r) / 0.001
  y = x**2 / 0.5 if x <= 0.5 else 1 - (1 - x) ** 2 / 0.5
  imp = 0.95 if x >= 1 else 0.9 + y * 0.05
  R = (1 - imp) / imp * float(m.dof_invweight0[0])
  assert tau_g == pytest.approx(k * imp * (-r) / R, rel=2e-3)
  assert o.qfrc_constraint[0, 0] == pytest.approx(-tau_g, rel=1e-4)


@pytest.mark.parametrize("integ", ["Euler", "implicitfast"])
def test_joint_damping_decay_rate(integ):
  """Zero-gravity spin with viscous joint damping b: omega decays as exp(-b t / I); both integrators treat
  damping implicitly (MuJoCo's Euler does so for joint damping), so the discrete rate is 1 / (1 + h b / I)."""
  sp = Spec.from_string(ARM.format(integ=integ, limited="false", damping="0.3", actuator=""))
  sp.option.gravity = (0.0, 0.0, 0.0)
  m = sp.compile()
  o = Oracle(m)
  o.qvel[:] = 2.0
  o.forward()
  inertia = float(o.qM[0, 0])
  for _ in range(500):
    o.step()
  expect = 2.0 * (1.0 / (1.0 + 0.002 * 0.3 / inertia)) ** 500
  assert o.qvel[0, 0] == pytest.approx(expect, rel=1e-6)
  assert expect == pytest.approx(2.0 * np.exp(-0.3 * 1.0 / inertia), rel=2e-2)  # backward-Euler discretisation error


def test_resting_contact_penetration_follows_soft_constraint_law():
  """Ball on a plane at rest: depth r solves m g = (1/R) k imp(r) (-r), R = (1-imp)/imp (invweight_ball + 0);
  checks impedance, reference acceleration and regulariser together (MuJoCo 'Computation' chapter)."""
  m = Spec.from_string(BALL_ON_PLANE).compile()
  o = Oracle(m)
  for _ in range(3000):
    o.step()
  assert abs(o.qvel[0]).max() < 1e-6 and int(o.ncon[0, 0]) == 1
  r = float(o.contact_dist[0, 0])
  assert -1e-3 < r < 0
  k = 1.0 / (0.95**2 * 0.02**2)
  x = abs(r) / 0.001
  y = x**2 / 0.5 if x <= 0.5 else 1 - (1 - x) ** 2 / 0.5
  imp = 0.95 if x >= 1 else 0.9 + y * 0.05
  ball = [i for i, n in enumerate(m.names["body"]) if n == "ball"][0]
  # the four pyramid rows share D: the normal force is the sum of four equal row forces, each (1/R_row) k imp (-r)
  mu = float(o.contact_friction[0, 0])
  Rrow = 2 * mu * mu * (1 - imp) / imp * float(m.body_invweight0[ball, 0]) * (1 + mu * mu)
  assert 2 * 9.81 == pytest.approx(4 * k * imp * (-r) / Rrow, rel=2e-3)

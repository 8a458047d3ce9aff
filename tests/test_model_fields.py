"""Per-world model fields against the fp64 oracle (oracle/b2_oracle.c).

Domain randomisation changes the model after b2_create through the expandable float arrays (kFloatArrays in
mjlab_b200/csrc/b2sim.cu); the step kernel reads each of them through a {pointer, per-world stride} pair.  Every case
writes model values into the engine and the same values into the oracle's per-world model arrays (`Oracle.model_field`),
then compares forward and step outputs world by world.  The file runs on the host-emulated library (CPU suite) and on
the GPU (`-m gpu`).  Tolerances are those of test_kernel_emul._check_forward.

A case must prove that it tests something: in the oracle, every perturbed world has to move some compared output by at
least 100x that output's tolerance (or change the contact set); otherwise the case fails as vacuous.  Two fields are
inert by the engine's scope (DESIGN.md §6): `geom_rgba` (rendering only) and `dof_frictionloss` (friction loss is not
modelled; the oracle ignores it too).  For those, the perturbed worlds must be bit-identical to the unperturbed one.

The states and model setups (identical in every world) are chosen so that every field matters: frame perturbations go
to non-root bodies (a free joint ignores its body's frame), joint ranges are set so that joints sit past their limits
or within a margin of them, feet and a leg press on the ground, geoms come within a perturbed margin, the ground has
the feet's contact priority and its own solref (so that `geom_solmix` weighs two different values), controls fall
outside a narrowed control range, narrowed force ranges saturate the actuators, and shrunken bounding radii make the
broadphase drop contacts.  The per-field cases use Go1; the all-fields case uses G1.
"""

import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from mjlab_b200.sim import native
from oracle.oracle import Oracle
from util import _quat_mul, load_oracle, make_states, relerr

sys.path.insert(0, str(Path(__file__).parent / "emul"))

BACKENDS = [pytest.param("cuda", marks=pytest.mark.gpu), "emul"]
INERT = ("geom_rgba", "dof_frictionloss")
KINREC = ("body_pos", "body_quat", "jnt_pos", "jnt_axis", "qpos0")  # also copied into the fast kinematic records

# (field, relative tolerance) of a forward; qacc and sensordata are checked as in _check_forward
FWD = [(f, 1e-5) for f in ("xpos", "xquat", "xipos", "subtree_com", "cvel", "geom_xpos", "geom_xmat", "site_xpos",
                           "site_xmat", "qM", "qfrc_bias", "qfrc_smooth", "actuator_force")]
QACC_TOL, QACC_FLOOR, SENSOR_TOL, QPOS_TOL, QVEL_TOL = 1e-3, 10.0, 1e-3, 1e-4, 5e-3


# ---- backends ----------------------------------------------------------------------------------------------------

_emul = None


def _emul_lib():
  global _emul
  if _emul is None:
    from engine import load_emul_library

    _emul = load_emul_library()
  return _emul


class Eng:
  """One b2_sim on either backend.  Fields are fetched afresh on every access (an expansion moves a model field), as
  torch tensors over engine memory: device memory on "cuda", host memory on "emul"."""

  def __init__(self, backend, model, n, nconmax=None):
    self.n = n
    if backend == "emul":
      from engine import host_tensor

      self.sim, self.e, self.dev = None, native.Engine(_emul_lib(), model, n, nconmax), "cpu"
      self._wrap = host_tensor
    else:
      from mjlab_b200.sim import Simulation, SimulationCfg
      from mjlab_b200.sim.sim_data import tensor_from_b2

      self.sim = Simulation(n, SimulationCfg(nconmax=nconmax), model, "cuda:0")
      self.e, self.dev = self.sim._engine, "cuda:0"
      self._wrap = lambda t: tensor_from_b2(t, self.sim)
    self.lib, self.h = self.e.lib, self.e.h
    self.e.set_option("debug_outputs", 1)  # qM, qfrc_bias, qfrc_smooth

  def stream(self):
    return None if self.sim is None else ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

  def t(self, name, which=0):
    return self._wrap(self.e.get_field(which, name))

  def a(self, name):
    return self.t(name).cpu().numpy()

  def opt(self, key):
    return self.e.get_option(key)

  def set(self, key, value):
    self.e.set_option(key, value)

  def load(self, st):
    for k, v in st.items():
      self.t(k)[...] = torch.as_tensor(v, dtype=torch.float32, device=self.dev)

  def model_rows(self, name, rows):
    """One row per world (the field must be expanded)."""
    t = self.t(name, 1)
    assert t.stride(0) > 0, name
    t[...] = torch.as_tensor(np.asarray(rows).reshape(t.shape), dtype=torch.float32, device=self.dev)

  def shared_row(self, name, row):
    """Write the row every world reads while the field is not expanded (at one world: the only row)."""
    t = self.t(name, 1)
    t[0] = torch.as_tensor(np.asarray(row).reshape(t.shape[1:]), dtype=torch.float32, device=self.dev)

  def expand(self, name):
    self.e.check(self.lib.b2_expand_model_field(self.h, name.encode(), self.stream(), None))

  def forward(self):
    self.e.check(self.lib.b2_forward(self.h, self.stream()))

  def step(self):
    self.e.check(self.lib.b2_step(self.h, self.stream()))

  def step_n(self, k):
    self.e.check(self.lib.b2_step_n(self.h, k, self.stream()))

  def forward_masked(self, mask):
    m = torch.as_tensor(mask.astype(np.uint8), device=self.dev)
    self.e.check(self.lib.b2_forward_masked(self.h, ctypes.c_void_p(m.data_ptr()), self.stream()))
    if self.sim is not None:
      torch.cuda.synchronize()

  def close(self):
    if self.sim is not None:
      self.sim.close()
    else:
      self.e.close()


def expandable_fields(eng):
  """The model fields b2_expand_model_field accepts, read from the library."""
  out = []
  for name in eng.e.names(1):
    t = native.B2Tensor()
    if eng.lib.b2_expand_model_field(eng.h, name.encode(), None, ctypes.byref(t)) == 0:
      out.append(name)
  return out


# ---- comparisons -------------------------------------------------------------------------------------------------


def _contacts(ncon, nefc, geom, w):
  return int(ncon[w]), int(nefc[w]), geom[w, : 2 * int(ncon[w])].tolist()


def check_forward(eng, o, worlds=None):
  """Engine against oracle after a forward, world by world: contact sets identical, fields within tolerance."""
  n = eng.n
  worlds = np.arange(n) if worlds is None else np.asarray(worlds)
  en, ee, eg = eng.a("ncon").ravel(), eng.a("nefc").ravel(), eng.a("contact_geom").reshape(n, -1)
  og = o.contact_geom.reshape(n, -1)
  for w in worlds:
    assert _contacts(en, ee, eg, w) == _contacts(o.ncon.ravel(), o.nefc.ravel(), og, w), f"contact set of world {w}"
  for f, tol in FWD:
    e = relerr(eng.a(f).reshape(n, -1)[worlds], o.field(f).reshape(n, -1)[worlds])
    assert e.max() < tol, (f, int(worlds[e.argmax()]), e.max())
  e = relerr(eng.a("qacc")[worlds], o.qacc[worlds], floor=QACC_FLOOR)
  assert e.max() < QACC_TOL, ("qacc", int(worlds[e.argmax()]), e.max())
  assert np.abs(eng.a("sensordata")[worlds] - o.sensordata[worlds]).max(initial=0.0) < SENSOR_TOL


def check_state(eng, o, worlds=None):
  worlds = np.arange(eng.n) if worlds is None else np.asarray(worlds)
  for f, tol in (("qpos", QPOS_TOL), ("qvel", QVEL_TOL)):
    e = relerr(eng.a(f)[worlds], o.field(f)[worlds])
    assert e.max() < tol, (f, int(worlds[e.argmax()]), e.max())


def forward_effect(o, w, ob, wb):
  """How far world `w` of oracle `o` lies from world `wb` of `ob` after a forward, in units of the tolerance
  (inf when the contact sets differ)."""
  oc = _contacts(o.ncon.ravel(), o.nefc.ravel(), o.contact_geom.reshape(o.nworld, -1), w)
  if oc != _contacts(ob.ncon.ravel(), ob.nefc.ravel(), ob.contact_geom.reshape(ob.nworld, -1), wb):
    return np.inf
  r = [relerr(o.field(f)[w:w + 1], ob.field(f)[wb:wb + 1])[0] / tol for f, tol in FWD]
  r.append(relerr(o.qacc[w:w + 1], ob.qacc[wb:wb + 1], floor=QACC_FLOOR)[0] / QACC_TOL)
  r.append(np.abs(o.sensordata[w] - ob.sensordata[wb]).max(initial=0.0) / SENSOR_TOL)
  return max(r)


def state_effect(o, w, ob, wb):
  return max(relerr(o.field(f)[w:w + 1], ob.field(f)[wb:wb + 1])[0] / tol for f, tol in (("qpos", QPOS_TOL),
                                                                                         ("qvel", QVEL_TOL)))


# ---- the model setups and perturbations --------------------------------------------------------------------------


def _dirs(rng, n, dim=3):
  d = rng.normal(size=(n, dim))
  return d / np.linalg.norm(d, axis=1, keepdims=True)


def _unit(v):
  return v / np.linalg.norm(v, axis=1, keepdims=True)


def _turn(q, ang, rng):
  """Quaternions `q` turned by `ang` radians about random axes."""
  ax = _dirs(rng, len(q))
  dq = np.concatenate([np.full((len(q), 1), np.cos(ang / 2)), ax * np.sin(ang / 2)], axis=1)
  r = _quat_mul(q, dq)
  return r / np.linalg.norm(r, axis=1, keepdims=True)


class Parts:
  """Index sets of a robot scene: its bodies below the floating base, its bodies, hinge joints and their dofs and
  qpos addresses, its geoms, and the geoms of the collision pairs."""

  def __init__(self, m):
    a = {k: np.asarray(v) for k, v in m.arrays.items()}
    root = int(a["jnt_bodyid"][a["jnt_type"] == 0][0])
    self.robot = np.nonzero(a["body_rootid"] == root)[0]
    self.nonroot = self.robot[self.robot != root]
    self.hinge = np.nonzero(a["jnt_type"] != 0)[0]
    self.hinge_dof = a["jnt_dofadr"][self.hinge]
    self.hinge_q = a["jnt_qposadr"][self.hinge]
    self.geoms = np.nonzero(np.isin(a["geom_bodyid"], self.robot))[0]
    self.colliding = np.intersect1d(np.union1d(a["pair_geom1"], a["pair_geom2"]), self.geoms)
    self.ctrl = np.asarray(m.keys["robot/init_state"]["ctrl"], dtype=np.float64)


def _at(v, idx, fn):
  v = v.copy()
  v[idx] = fn(v[idx])
  return v


# field -> perturb(parts, rows, k, rng): the model rows (count, width) of one world with strength k (0 < k <= 2)
PERTURB = {
    "body_pos": lambda p, v, k, r: _at(v, p.nonroot, lambda x: x + 0.01 * k * _dirs(r, len(x))),
    "body_quat": lambda p, v, k, r: _at(v, p.nonroot, lambda x: _turn(x, 0.05 * k, r)),
    "body_ipos": lambda p, v, k, r: _at(v, p.robot, lambda x: x + 0.01 * k * _dirs(r, len(x))),
    "body_iquat": lambda p, v, k, r: _at(v, p.robot, lambda x: _turn(x, 0.5 * k, r)),
    "body_mass": lambda p, v, k, r: _at(v, p.robot, lambda x: x * (1 + 0.2 * k)),
    "body_subtreemass": lambda p, v, k, r: _at(v, p.robot, lambda x: x * (1 + 0.2 * k)),
    "body_inertia": lambda p, v, k, r: _at(v, p.robot, lambda x: x * (1 + 0.3 * k * r.uniform(0.5, 1.0, x.shape))),
    "body_invweight0": lambda p, v, k, r: _at(v, p.robot, lambda x: x * (1 + 2.0 * k)),
    "jnt_pos": lambda p, v, k, r: _at(v, p.hinge, lambda x: x + 0.01 * k * _dirs(r, len(x))),
    "jnt_axis": lambda p, v, k, r: _at(v, p.hinge, lambda x: _unit(x + 0.05 * k * _dirs(r, len(x)))),
    "jnt_range": lambda p, v, k, r: _at(v, p.hinge, lambda x: x + 0.07 * k * np.array([-1.0, 1.0])),
    "jnt_solref": lambda p, v, k, r: _at(v, p.hinge, lambda x: x * np.array([1 + 5.0 * k, 1.0])),
    "jnt_solimp": lambda p, v, k, r: _at(v, p.hinge, lambda x: np.concatenate(
        [x[:, :2] * (1 - 0.45 * k), x[:, 2:]], axis=1)),
    "jnt_margin": lambda p, v, k, r: _at(v, p.hinge, lambda x: x + 0.04 * k),
    "jnt_stiffness": lambda p, v, k, r: _at(v, p.hinge, lambda x: x + 10.0 * k),
    "dof_armature": lambda p, v, k, r: v + 0.02 * k,
    "dof_damping": lambda p, v, k, r: _at(v, p.hinge_dof, lambda x: x + 2.0 * k),
    "dof_frictionloss": lambda p, v, k, r: v + 0.5 * k,
    "dof_invweight0": lambda p, v, k, r: v * (1 + 2.0 * k),
    "geom_size": lambda p, v, k, r: _at(v, p.colliding, lambda x: x * (1 + 0.6 * k)),
    "geom_pos": lambda p, v, k, r: _at(v, p.geoms, lambda x: x + 0.01 * k * _dirs(r, len(x))),
    "geom_quat": lambda p, v, k, r: _at(v, p.geoms, lambda x: _turn(x, 0.1 * k, r)),
    "geom_friction": lambda p, v, k, r: v * np.array([1 - 0.45 * k, 1.0, 1.0]),
    "geom_solref": lambda p, v, k, r: v * np.array([1 + 1.0 * k, 1.0]),
    "geom_solimp": lambda p, v, k, r: np.concatenate([v[:, :2] * (1 - 0.48 * k), v[:, 2:]], axis=1),
    "geom_solmix": lambda p, v, k, r: _at(v, p.colliding, lambda x: x * (1 + 2.0 * k)),
    "geom_margin": lambda p, v, k, r: _at(v, p.colliding, lambda x: x + 0.03 * k),
    "geom_gap": lambda p, v, k, r: _at(v, p.colliding, lambda x: x + 0.02 * k),
    "geom_rbound": lambda p, v, k, r: _at(v, p.colliding, lambda x: x * 1e-3 * k),
    "geom_rgba": lambda p, v, k, r: np.clip(v + 0.2 * k, 0.0, 1.0),
    "site_pos": lambda p, v, k, r: v + 0.01 * k * _dirs(r, len(v)),
    "site_quat": lambda p, v, k, r: _turn(v, 0.1 * k, r),
    "actuator_gainprm": lambda p, v, k, r: _at(v, (slice(None), 0), lambda x: x * (1 + 0.3 * k)),
    "actuator_biasprm": lambda p, v, k, r: _at(v, (slice(None), slice(1, 3)), lambda x: x * (1 + 0.3 * k)),
    "actuator_ctrlrange": lambda p, v, k, r: p.ctrl[:, None] + 0.05 * k * np.array([-1.0, 1.0]),
    "actuator_forcerange": lambda p, v, k, r: v * 0.1 / k,
    "actuator_gear": lambda p, v, k, r: v * (1 + 0.5 * k),
    "qpos0": lambda p, v, k, r: _at(v, p.hinge_q, lambda x: x + 0.05 * k * r.choice([-1.0, 1.0], x.shape)),
}

def _limits(p, v, q):
  """Joint ranges around the joint angles `q`: a third of the hinges 0.05 below their range, a third 0.05 above it,
  a third 0.03 inside it (within reach of a joint margin)."""
  v = v.copy()
  for i, (j, a) in enumerate(zip(p.hinge, p.hinge_q)):
    v[j] = q[a] + [[0.05, 0.5], [-0.5, -0.05], [-0.5, 0.03]][i % 3]
  return v


# setup writes, identical in every world, that make the fields matter (the field under test is written over them):
# the limits above; soft limits and contacts (solimp 0.5-0.7), so that the regularisation weights (dof_invweight0,
# body_invweight0) count; a ground whose solref differs from the robot's, so that geom_solmix weighs two values
SETUP = {
    "jnt_range": lambda p, rows, q: _limits(p, rows["jnt_range"], q),
    "jnt_solimp": lambda p, rows, q: _at(rows["jnt_solimp"], p.hinge, lambda x: [0.5, 0.7, 0.001, 0.5, 2.0]),
    "geom_solimp": lambda p, rows, q: np.tile([0.5, 0.7, 0.001, 0.5, 2.0], (len(rows["geom_solimp"]), 1)),
    "geom_solref": lambda p, rows, q: _at(rows["geom_solref"], 0, lambda x: np.array([0.06, 0.5])),
}
# and for one field only: a margin for the gap to cut into
FIELD_SETUP = {"geom_gap": {"geom_margin": lambda p, rows, q: _at(rows["geom_margin"], p.colliding, lambda x: x + 0.04)}}


def model_rows(m, name):
  """The model's values of a float field as (count, width) float64."""
  v = np.asarray(m.arrays[name], dtype=np.float64)
  return v.reshape(len(v), -1)


def f32(v):
  return np.asarray(v, dtype=np.float32).astype(np.float64)


def tiled_state(m, n, seed=7):
  """One state copied into every world (world 0 is then the unperturbed twin of the rest): the base lowered 2 cm
  and rolled so that feet and a leg of the same priority as the ground touch it, sliding."""
  st = make_states(m, 1, seed=seed, z_range=(-0.02, -0.02), tilt=0.0, joint_noise=0.1, vel=0.5)
  roll = 0.3
  st["qpos"][:, 3:7] = _quat_mul(st["qpos"][:, 3:7], np.array([[np.cos(roll / 2), np.sin(roll / 2), 0.0, 0.0]]))
  return {k: np.repeat(v, n, axis=0) for k, v in st.items()}


def apply_setup(eng, o, m, p, field, q):
  """The setup writes (for joint angles `q`), to the shared rows of the engine and to every world of the oracle(s);
  returns every field's rows after them."""
  rows = {k: model_rows(m, k) for k in PERTURB}
  writes = {g: fn(p, rows, q) for g, fn in SETUP.items()}
  writes.update({g: fn(p, rows, q) for g, fn in FIELD_SETUP.get(field, {}).items()})
  for g, v in writes.items():
    v = f32(v)
    if eng is not None:
      eng.shared_row(g, v)
    for oo in o:
      oo.model_field(g)[:] = v.reshape(1, -1)
    rows[g] = v
  return rows


def go1_scene():
  """Go1 flat with the ground at the feet's contact priority, so that every contact mixes the two geoms' solver
  parameters by their geom_solmix weights (a higher-priority foot would impose its own)."""
  import copy

  from mjlab_b200.asset_zoo import load_compiled

  m = copy.deepcopy(load_compiled("go1_flat"))
  m.arrays = dict(m.arrays)
  prio = np.array(m.arrays["geom_priority"], dtype=np.int32)
  prio[0] = prio.max()
  m.arrays["geom_priority"] = prio
  return m


@pytest.fixture(scope="module")
def go1():
  m = go1_scene()
  return m, Parts(m)


# ---- a. one case per expandable field ---------------------------------------------------------------------------


@pytest.mark.parametrize("backend", BACKENDS)
def test_every_expandable_field_has_a_case(backend, go1):
  """The cases below cover exactly the fields the library lets callers expand."""
  eng = Eng(backend, go1[0], 2)
  try:
    assert sorted(expandable_fields(eng)) == sorted(PERTURB)
  finally:
    eng.close()


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("field", sorted(PERTURB))
def test_expanded_field_matches_oracle(backend, field, go1):
  """World 0 keeps the model value, worlds 1 and 2 get their own perturbation; forward and two steps agree with the
  oracle world by world, and the perturbation visibly moves the oracle's answer."""
  m, p = go1
  n = 3
  eng = Eng(backend, m, n)
  o = Oracle(m, nworld=n, maxcon=int(eng.opt("maxcon")))
  st = tiled_state(m, n)
  rows = apply_setup(eng, [o], m, p, field, st["qpos"][0])
  eng.expand(field)
  vals = np.stack([f32(rows[field])] + [f32(PERTURB[field](p, rows[field], k, np.random.default_rng(k)))
                                         for k in (1, 2)])
  eng.model_rows(field, vals)
  o.model_field(field)[:] = vals.reshape(n, -1)
  eng.load(st)
  load_oracle(o, st)
  eng.forward()
  o.forward()
  check_forward(eng, o)
  fwd = [forward_effect(o, w, o, 0) for w in (1, 2)]
  out0 = {f: eng.a(f) for f, _ in FWD + [("qacc", 0), ("sensordata", 0)]}
  eng.step_n(2)
  o.step()
  o.step()
  check_state(eng, o)
  eff = [max(fwd[w - 1], state_effect(o, w, o, 0)) for w in (1, 2)]
  if field in INERT:
    assert max(eff) == 0.0, eff
    for f, v in out0.items():
      assert all(np.array_equal(v[w], v[0]) for w in (1, 2)), f
    q = eng.a("qpos"), eng.a("qvel")
    assert all(np.array_equal(x[w], x[0]) for x in q for w in (1, 2))
  else:
    assert min(eff) >= 100.0, f"vacuous: the perturbation of {field} moves no output by 100x its tolerance ({eff})"
  eng.close()


# ---- b. the same perturbations written to the shared row --------------------------------------------------------


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("n", [3, 1])
@pytest.mark.parametrize("field", sorted(PERTURB))
def test_shared_row_write_reaches_every_world(backend, field, n, go1):
  """A write to the shared row (no expansion; at one world after an expansion, which is then a no-op) reaches every
  world, kinematics included: the engine agrees with an oracle holding the written value in every world."""
  m, p = go1
  eng = Eng(backend, m, n)
  o = Oracle(m, nworld=n, maxcon=int(eng.opt("maxcon")))
  base = Oracle(m, nworld=1, maxcon=int(eng.opt("maxcon")))
  st = tiled_state(m, n)
  rows = apply_setup(eng, [o, base], m, p, field, st["qpos"][0])
  if n == 1:
    eng.expand(field)
  assert eng.t(field, 1).stride(0) == 0
  row = f32(PERTURB[field](p, rows[field], 1, np.random.default_rng(1)))
  eng.shared_row(field, row)
  o.model_field(field)[:] = row.reshape(1, -1)
  eng.load(st)
  load_oracle(o, st)
  load_oracle(base, {k: v[:1] for k, v in st.items()})
  eng.forward()
  o.forward()
  base.forward()
  check_forward(eng, o)
  fwd = forward_effect(o, 0, base, 0)
  eng.step_n(2)
  for oo in (o, base):
    oo.step()
    oo.step()
  check_state(eng, o)
  eff = max(fwd, state_effect(o, 0, base, 0))
  assert eff == 0.0 if field in INERT else eff >= 100.0, eff
  eng.close()


# ---- c. expansion semantics --------------------------------------------------------------------------------------


@pytest.mark.parametrize("backend", BACKENDS)
def test_expansion_tiles_keeps_and_isolates(backend, go1):
  """Expanding after a shared-row write tiles the written value; a second expansion is a no-op that keeps the
  per-world values (and the memory); expanding one field leaves every other field shared."""
  m, p = go1
  n = 3
  eng = Eng(backend, m, n)
  row = f32(model_rows(m, "body_mass") * 1.5)
  eng.shared_row("body_mass", row)
  eng.expand("body_mass")
  t = eng.t("body_mass", 1)
  assert t.stride(0) > 0
  assert np.array_equal(t.cpu().numpy(), np.repeat(row.reshape(1, -1), n, axis=0).astype(np.float32))
  t[1] = t[1] * 2.0
  t[2] = t[2] * 3.0
  before, ptr = t.cpu().numpy().copy(), eng.e.get_field(1, "body_mass").ptr
  eng.expand("body_mass")
  t = eng.t("body_mass", 1)
  assert eng.e.get_field(1, "body_mass").ptr == ptr and np.array_equal(t.cpu().numpy(), before)
  for f in PERTURB:
    if f != "body_mass":
      assert eng.t(f, 1).stride(0) == 0, f
  # and the kernel reads what the expansions left: the oracle with the same three rows agrees
  o = Oracle(m, nworld=n, maxcon=int(eng.opt("maxcon")))
  o.model_field("body_mass")[:] = before
  st = tiled_state(m, n)
  eng.load(st)
  load_oracle(o, st)
  eng.forward()
  o.forward()
  check_forward(eng, o)
  eng.close()


# ---- d. every field randomised per world at once -----------------------------------------------------------------


def randomize_all(eng, o, m, p, seed):
  """Every field expanded with its own perturbation in every world (strengths 0.2-1), around the model's values
  (the joint-limit setup needs one state; the worlds here have their own)."""
  rows = {k: model_rows(m, k) for k in PERTURB}
  for g, fn in SETUP.items():
    if g != "jnt_range":
      rows[g] = fn(p, rows, None)
  for g, fn in FIELD_SETUP["geom_gap"].items():
    rows[g] = fn(p, rows, None)
  rng = np.random.default_rng(seed)
  n = eng.n
  for field in sorted(PERTURB):
    vals = np.stack([f32(PERTURB[field](p, rows[field], rng.uniform(0.2, 1.0), rng)) for _ in range(n)])
    eng.expand(field)
    eng.model_rows(field, vals)
    o.model_field(field)[:] = vals.reshape(n, -1)


@pytest.mark.parametrize("backend,n", [pytest.param("cuda", 5, marks=pytest.mark.gpu), ("emul", 3)])
def test_all_fields_randomised_per_world(backend, n, g1_model):
  """G1 with all fields per world at once, distinct states; on the GPU 5 worlds leave a CTA partly empty."""
  m = g1_model
  eng = Eng(backend, m, n)
  o = Oracle(m, nworld=n, maxcon=int(eng.opt("maxcon")))
  randomize_all(eng, o, m, Parts(m), seed=3)
  st = make_states(m, n, seed=12)
  eng.load(st)
  load_oracle(o, st)
  eng.forward()
  o.forward()
  check_forward(eng, o)
  eng.step_n(2)
  o.step()
  o.step()
  check_state(eng, o)
  eng.close()


@pytest.mark.gpu
def test_all_fields_randomised_on_partitioned_masked_and_graph_paths(g1_model):
  """2048 G1 worlds, every field per world, against the oracle world by world on each path that remaps or partitions
  worlds: step_n(4) (two stream partitions of 1024 worlds, each in heavy-first order), a masked forward, and a
  CUDA-graph replay after a further model write."""
  m = g1_model
  n = 2048
  eng = Eng("cuda", m, n)
  o = Oracle(m, nworld=n, maxcon=int(eng.opt("maxcon")))
  p = Parts(m)
  randomize_all(eng, o, m, p, seed=4)
  for k in ("iterations",):  # converged answers do not depend on the path that reached them
    eng.set(k, 50)
    o.set_option(k, 50)
  assert eng.opt("sorted_dispatch") == 1
  st = make_states(m, n, seed=13)
  load_oracle(o, st)
  for _ in range(4):
    o.step()
  ref = {f: o.field(f).copy() for f in ("qpos", "qvel")}

  class Ref:  # the oracle's state after the four steps, as check_state reads it
    nworld = n

    @staticmethod
    def field(f):
      return ref[f]

  eng.load(st)
  eng.step_n(4)
  check_state(eng, Ref)
  # masked forward: the unselected worlds keep their outputs bit for bit, the selected ones match the oracle
  st2 = make_states(m, n, seed=14)
  eng.load(st2)
  load_oracle(o, st2)
  keep = {f: eng.a(f) for f in ("xpos", "qacc", "ncon", "qM")}
  mask = np.random.default_rng(5).random(n) < 0.5
  eng.forward_masked(mask)
  o.forward()
  for f, v in keep.items():
    assert np.array_equal(eng.a(f)[~mask], v[~mask]), f
  check_forward(eng, o, np.nonzero(mask)[0])
  # a CUDA graph of the step, replayed after the per-world values changed in place
  sim = eng.sim
  sim.use_cuda_graph = True
  sim.create_graph()
  rng = np.random.default_rng(6)
  rows = {k: model_rows(m, k) for k in PERTURB}
  for field in ("body_mass", "qpos0", "body_pos", "geom_friction"):
    vals = np.stack([f32(PERTURB[field](p, rows[field], rng.uniform(0.2, 1.0), rng)) for _ in range(n)])
    eng.model_rows(field, vals)
    o.model_field(field)[:] = vals.reshape(n, -1)
  eng.load(st)
  load_oracle(o, st)
  sim.step()
  o.step()
  check_state(eng, o)
  eng.close()


@pytest.mark.gpu
def test_graph_replay_sees_shared_row_writes(go1):
  """Shared-row writes of the five fields the fast kinematics keep a copy of, made after a CUDA graph of
  b2_step_n was captured, reach every world of every stream partition when the graph is replayed."""
  m, p = go1
  n = 2048
  eng = Eng("cuda", m, n)
  o = Oracle(m, nworld=n, maxcon=int(eng.opt("maxcon")))
  st = make_states(m, n, seed=15)
  g = torch.cuda.CUDAGraph()
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    with torch.cuda.graph(g, stream=side):
      eng.e.check(eng.lib.b2_step_n(eng.h, 2, ctypes.c_void_p(side.cuda_stream)))
  torch.cuda.current_stream().wait_stream(side)
  rows = {k: model_rows(m, k) for k in PERTURB}
  for field in KINREC:
    row = f32(PERTURB[field](p, rows[field], 1, np.random.default_rng(1)))
    eng.shared_row(field, row)
    o.model_field(field)[:] = row.reshape(1, -1)
  eng.load(st)
  load_oracle(o, st)
  g.replay()
  o.step()
  o.step()
  check_state(eng, o)
  eng.close()


# ---- e. the reference's own randomisation code -------------------------------------------------------------------


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("field", ["qpos0", "body_pos"])
def test_reference_randomize_field(backend, field, n, g1_model):
  """The reference's `expand_model_fields` and `randomize_field` (envs/mdp/events.py) through its own
  `mjlab.sim.Simulation` at one and three worlds: the engine agrees with the oracle given the values the event wrote."""
  import refload

  if not refload.available():
    pytest.skip("oracle/_ref not installed")
  ref = refload.load()
  mp = pytest.MonkeyPatch()
  dev = "cuda:0"
  if backend == "emul":
    import mjlab_b200.compat.mujoco_warp_shim as mw
    from engine import EmulEngine

    mp.setattr(mw, "_Engine", EmulEngine)
    mp.setattr(native, "check", lambda rc: (_ for _ in ()).throw(RuntimeError("b2sim call failed")) if rc else None)
    dev = "cpu"
  try:
    _reference_randomize_field(ref, dev, field, n, g1_model)
  finally:
    mp.undo()


def _reference_randomize_field(ref, dev, field, n, m):
  import mujoco  # the compat stand-in

  sim = ref.sim.Simulation(n, ref.sim.SimulationCfg(), m, dev)
  E = ref.entity
  ent = E.Entity.__new__(E.Entity)  # (as test_reference_dropin: the scene is already compiled)
  ent.cfg = E.EntityCfg()
  ent._spec = mujoco.EntitySpecView(m, "robot/")
  ent._free_joint = ent._spec.joints[0]
  ent._non_free_joints = tuple(ent._spec.joints[1:])
  ent.initialize(sim.mj_model, sim.model, sim.data, dev)

  class Scene:
    entities = {"robot": ent}

    def __getitem__(self, k):
      return self.entities[k]

  import types

  env = types.SimpleNamespace(sim=sim, device=dev, num_envs=n, scene=Scene())
  sim.expand_model_fields([field])  # what the reference's event manager does for a randomised field (no-op at n=1)
  sim.create_graph()  # (the reference captures its graphs after the expansion: the expanded arrays are new memory)
  cfg = ref.scene_entity_config.SceneEntityCfg("robot", joint_names=[".*"], body_names=[".*"])
  cfg.resolve(env.scene)
  torch.manual_seed(2)
  if field == "qpos0":
    ref.events.randomize_field(env, None, "qpos0", ranges=(-0.05, 0.05), operation="add", asset_cfg=cfg)
  else:
    ref.events.randomize_field(env, None, "body_pos", ranges=(-0.01, 0.01), operation="add", asset_cfg=cfg)
  written = getattr(sim.model, field)[:].cpu().numpy().reshape(n, -1).astype(np.float64)
  assert np.abs(written - model_rows(m, field).reshape(1, -1)).max() > 1e-3  # the event wrote something
  o = Oracle(m, nworld=n, maxcon=int(object.__getattribute__(sim.wp_data, "_engine").get_option("maxcon")))
  o.model_field(field)[:] = written
  st = make_states(m, n, seed=16, joint_noise=0.6)
  for k, v in st.items():
    getattr(sim.data, k)[:] = torch.as_tensor(v, dtype=torch.float32, device=dev)
  load_oracle(o, st)
  sim.forward()
  o.forward()
  if dev != "cpu":
    torch.cuda.synchronize()
  for f, tol in FWD:
    if f in ("qM", "qfrc_bias", "qfrc_smooth"):  # (debug outputs, off in the reference's Simulation)
      continue
    e = relerr(getattr(sim.data, f)[:].cpu().numpy().reshape(n, -1), o.field(f).reshape(n, -1))
    assert e.max() < tol, (f, e.max())
  assert np.array_equal(sim.data.ncon[:].cpu().numpy().ravel(), o.ncon.ravel())
  e = relerr(sim.data.qacc[:].cpu().numpy(), o.qacc, floor=QACC_FLOOR)
  assert e.max() < QACC_TOL, e.max()

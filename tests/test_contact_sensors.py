"""Contact sensors (phase 9 of the step kernel, `sensors()` of oracle/b2_oracle.c) against an fp64 evaluation of
their definition, for every option b2_create accepts: data in {found, force, dist, pos, normal} (all 31 ordered
subsets), reduce `none` (num 1, 8, 40) and `netforce`, primary and secondary objects given as a geom, a body or a
subtree, and no secondary object.

Three comparisons per state:
  1. the engine's sensordata against `evaluate()` on the engine's own contacts (ncon, contact_geom / dist / pos /
     frame / force), with the exclusion rule recomputed in fp32 as the kernel makes it.  This isolates the sensor code
     from solver noise: `found` and every reduce-none column are gathers and sign flips of the same fp32 values and
     must be bit-equal; the netforce sums get fp32 bounds.
  2. the oracle's sensordata against `evaluate()` on the oracle's contacts (exclusion from contact_efc), in fp64.
  3. the engine's contacts against the oracle's: identical sets and exclusions world by world, dist / pos / normals
     within 1e-5, forces within 1e-3 of the world's largest contact force (floor 10 N, as qfrc_constraint in
     test_model_shapes_gpu).  After step_n(4) the fp32 and fp64 trajectories have parted for four steps, so there
     only the sensor counts are compared, in the worlds whose contact sets still agree.

The file runs on the host-emulated library (CPU suite) and on the GPU (`-m gpu`).  Every case asserts the condition
it exists for (more than 32 and more than `num` matches, a dir = -1 match, an excluded contact between matched
objects, a condim-1 match, a stale slot that was cleared), so that no change of model or state makes it vacuous.
"""

import itertools
import sys
from pathlib import Path

import numpy as np
import pytest

from mjlab_b200.compiler.spec import OBJ_BODY, OBJ_GEOM, OBJ_XBODY, Spec
from mjlab_b200.compiler.spec_cfg import ContactSensorCfg
from mjlab_b200.sim import native
from oracle.oracle import Oracle
from test_model_fields import Eng, _emul_lib
from util import convex_scene, convex_states, load_oracle, make_states, relerr

sys.path.append(str(Path(__file__).resolve().parents[1] / "tools"))
from synth_models import robot_xml  # noqa: E402

BACKENDS = [pytest.param("cuda", marks=pytest.mark.gpu), "emul"]

# the accepted data fields: intprm bit and width (torque, bit 2, and tangent, bit 6, are refused)
FIELDS = (("found", 1, 1), ("force", 2, 3), ("dist", 8, 1), ("pos", 16, 3), ("normal", 32, 3))
SUBSETS = [tuple(f for f, _, _ in c) for r in range(1, 6) for c in itertools.combinations(FIELDS, r)]
assert len(SUBSETS) == 31

# kernel-vs-evaluation bounds of the netforce columns (comparison 1; comparison 2 is fp64 and gets 1e-6 of them)
NET_FORCE, NET_POS, NET_NORMAL, NET_NORMAL_MIN = 1e-6, 1e-6, 1e-5, 1e-2
# engine-vs-oracle contact bounds (comparison 3)
CON_TOL, FORCE_TOL, FORCE_FLOOR = 1e-5, 1e-3, 10.0


# ---- the fp64 evaluation of the sensor definitions ---------------------------------------------------------------


class Sensors:
  """The model's sensor tables, and which geoms each sensor's primary and secondary objects cover."""

  def __init__(self, m):
    a = lambda k: np.asarray(m.arrays[k])  # noqa: E731
    self.n = int(m.nsensor)
    self.nsensordata = int(m.nsensordata)
    self.intprm = a("sensor_intprm").reshape(-1, 3)
    self.adr, self.dim = a("sensor_adr").ravel(), a("sensor_dim").ravel()
    parent, gbody = a("body_parentid").ravel(), a("geom_bodyid").ravel()
    self.margin = a("geom_margin").astype(np.float32).ravel()
    self.gap = a("geom_gap").astype(np.float32).ravel()
    self.condim, self.priority = a("geom_condim").ravel(), a("geom_priority").ravel()

    def subtree(b, root):  # body b in the subtree rooted at `root`, walking body_parentid
      while b != root and b != 0:
        b = parent[b]
      return b == root

    def covers(t, i):
      if t < 0:
        return np.ones(len(gbody), bool)
      if t == OBJ_GEOM:
        return np.arange(len(gbody)) == i
      if t == OBJ_BODY:
        return gbody == i
      assert t == OBJ_XBODY, t
      return np.array([subtree(int(b), int(i)) for b in gbody])

    self.obj = [covers(int(t), int(i)) for t, i in zip(a("sensor_objtype").ravel(), a("sensor_objid").ravel())]
    self.ref = [covers(int(t), int(i)) for t, i in zip(a("sensor_reftype").ravel(), a("sensor_refid").ravel())]

  def included32(self, geom, dist):
    """The kernel's exclusion rule in fp32: a contact is a constraint when dist < max(margins) - max(gaps)."""
    g1, g2 = geom[:, 0], geom[:, 1]
    incm = np.maximum(self.margin[g1], self.margin[g2]) - np.maximum(self.gap[g1], self.gap[g2])
    return np.asarray(dist, np.float32) < incm

  def contact_condim(self, geom):
    g1, g2 = geom[:, 0], geom[:, 1]
    p1, p2 = self.priority[g1], self.priority[g2]
    return np.where(p1 > p2, self.condim[g1], np.where(p2 > p1, self.condim[g2], np.maximum(self.condim[g1],
                                                                                            self.condim[g2])))


def evaluate(S, geom, dist, pos, frame, force, incl, scale=1.0):
  """fp64 sensordata of one world from its contacts (arrays over its ncon contacts), the bound of every element
  (0: must be bit-equal; inf: not compared) and per-sensor facts for the vacuity checks.  `scale` multiplies the
  netforce bounds."""
  geom = np.asarray(geom).reshape(-1, 2)
  out, tol = np.zeros(S.nsensordata), np.zeros(S.nsensordata)
  dist, pos = np.asarray(dist, np.float64), np.asarray(pos, np.float64).reshape(-1, 3)
  frame, force = np.asarray(frame, np.float64).reshape(-1, 3, 3), np.asarray(force, np.float64).reshape(-1, 3)
  cdim = S.contact_condim(geom)
  facts = []
  for s in range(S.n):
    ds, red, num = (int(x) for x in S.intprm[s])
    adr, dim = int(S.adr[s]), int(S.dim[s])
    slot = dim // max(num, 1)
    om, rm = S.obj[s], S.ref[s]
    d = np.where(om[geom[:, 0]] & rm[geom[:, 1]], 1, np.where(om[geom[:, 1]] & rm[geom[:, 0]], -1, 0))
    pair = np.nonzero(d != 0)[0]
    c = pair[incl[pair]]
    dc = d[c].astype(np.float64)
    q, qt = out[adr:adr + dim], tol[adr:adr + dim]
    cols, a = {}, 0
    for f, bit, w in FIELDS:
      if ds & bit:
        cols[f] = a
        a += w
    assert a == slot, (s, a, slot)
    nm = len(c)
    fw = dc[:, None] * np.einsum("crk,cr->ck", frame[c], force[c])  # contact force in the world frame
    mag = np.linalg.norm(fw, axis=1)
    if red == 0:
      for i in range(min(nm, num)):
        k, row = c[i], q[i * slot:(i + 1) * slot]
        if "found" in cols:
          row[cols["found"]] = nm
        if "force" in cols:
          row[cols["force"]:cols["force"] + 3] = force[k] * [1.0, dc[i], dc[i]]
        if "dist" in cols:
          row[cols["dist"]] = dist[k]
        if "pos" in cols:
          row[cols["pos"]:cols["pos"] + 3] = pos[k]
        if "normal" in cols:
          row[cols["normal"]:cols["normal"] + 3] = dc[i] * frame[k, 0]
    else:
      assert red == 3, red
      net, sumf = fw.sum(axis=0), mag.sum()
      if nm:
        if "found" in cols:
          q[cols["found"]] = nm
        if "force" in cols:
          q[cols["force"]:cols["force"] + 3] = net
          qt[cols["force"]:cols["force"] + 3] = scale * NET_FORCE * sumf
        if "pos" in cols:
          q[cols["pos"]:cols["pos"] + 3] = (mag[:, None] * pos[c]).sum(axis=0) / sumf if sumf > 0 else 0.0
          qt[cols["pos"]:cols["pos"] + 3] = scale * NET_POS
        if "normal" in cols:
          big = np.linalg.norm(net) > NET_NORMAL_MIN * sumf
          q[cols["normal"]:cols["normal"] + 3] = net / np.linalg.norm(net) if big else 0.0
          qt[cols["normal"]:cols["normal"] + 3] = scale * NET_NORMAL if big else np.inf
    facts.append(dict(s=s, reduce=red, num=num, data=ds, nmatch=nm, neg=int((dc < 0).sum()),
                      excluded=int((~incl[pair]).sum()), condim1=int((cdim[c] == 1).sum()),
                      normal_checked=red == 3 and "normal" in cols and nm > 0 and np.isfinite(qt[cols["normal"]])))
  return out, tol, facts


def engine_contacts(eng):
  n = eng.n
  nc = eng.a("ncon").ravel()
  return nc, dict(geom=eng.a("contact_geom").reshape(n, -1, 2), dist=eng.a("contact_dist").reshape(n, -1),
                  pos=eng.a("contact_pos").reshape(n, -1, 3), frame=eng.a("contact_frame").reshape(n, -1, 9),
                  force=eng.a("contact_force").reshape(n, -1, 3))


def oracle_contacts(o):
  n = o.nworld
  return o.ncon.ravel(), dict(geom=o.contact_geom.reshape(n, -1, 2), dist=o.contact_dist, pos=o.contact_pos.reshape(
      n, -1, 3), frame=o.contact_frame.reshape(n, -1, 9), force=o.contact_force.reshape(n, -1, 3))


def _world(nc, con, w):
  return {k: v[w, :nc[w]] for k, v in con.items()}


def check_engine(S, eng, worlds=None):
  """Comparison 1; returns the per-sensor facts of every compared world."""
  nc, con = engine_contacts(eng)
  sd = eng.a("sensordata").astype(np.float64)
  facts = []
  for w in range(eng.n) if worlds is None else worlds:
    c = _world(nc, con, w)
    exp, tol, f = evaluate(S, incl=S.included32(c["geom"], c["dist"]), **c)
    err = np.abs(sd[w] - exp)
    bad = ~(err <= tol)
    assert not bad.any(), ("engine", w, np.nonzero(bad)[0][:8], sd[w][bad][:8], exp[bad][:8])
    facts += f
  return facts


def check_oracle(S, o):
  """Comparison 2 (fp64: the gathers exact, the netforce sums to 1e-6 of the fp32 bounds)."""
  nc, con = oracle_contacts(o)
  facts = []
  for w in range(o.nworld):
    c = _world(nc, con, w)
    exp, tol, f = evaluate(S, incl=o.contact_efc[w, :nc[w]] >= 0, scale=1e-6, **c)
    err = np.abs(o.sensordata[w] - exp)
    bad = ~(err <= tol)
    assert not bad.any(), ("oracle", w, np.nonzero(bad)[0][:8], o.sensordata[w][bad][:8], exp[bad][:8])
    facts += f
  return facts


def same_contact_sets(S, eng, o):
  """Worlds whose engine and oracle contacts are the same pairs in the same order, with the same exclusions."""
  en, ec = engine_contacts(eng)
  on, oc = oracle_contacts(o)
  same = []
  for w in range(eng.n):
    if en[w] == on[w] and np.array_equal(ec["geom"][w, :en[w]], oc["geom"][w, :on[w]]) and np.array_equal(
        S.included32(ec["geom"][w, :en[w]], ec["dist"][w, :en[w]]), o.contact_efc[w, :on[w]] >= 0):
      same.append(w)
  return same


def check_against_oracle(S, eng, o, dist_tol=CON_TOL, pos_tol=CON_TOL, normal_tol=CON_TOL):
  """Comparison 3: identical contact sets and exclusions, contact values within tolerance, the same counts."""
  assert same_contact_sets(S, eng, o) == list(range(eng.n))
  en, ec = engine_contacts(eng)
  _, oc = oracle_contacts(o)
  for w in range(eng.n):
    k = en[w]
    if k == 0:
      continue
    for f, tol in (("dist", dist_tol), ("pos", pos_tol)):
      assert np.abs(ec[f][w, :k] - oc[f][w, :k]).max() < tol, (f, w)
    assert np.abs(ec["frame"][w, :k, :3] - oc["frame"][w, :k, :3]).max() < normal_tol, ("normal", w)
    e = relerr(ec["force"][w:w + 1, :k], oc["force"][w:w + 1, :k], floor=FORCE_FLOOR)[0]
    assert e < FORCE_TOL, ("force", w, e)
  counts_agree(S, eng, o, range(eng.n))


def counts_agree(S, eng, o, worlds):
  sd = eng.a("sensordata")
  for s in range(S.n):
    ds, red, num = S.intprm[s]
    if ds & 1:
      idx = S.adr[s] + (S.dim[s] // num) * np.arange(num if red == 0 else 1)
      assert np.array_equal(sd[np.ix_(list(worlds), idx)], o.sensordata[np.ix_(list(worlds), idx)]), s


# ---- sentinel in the row padding: phase 9 writes nothing outside the sensors' slots ------------------------------

SENTINEL = 12345.0


def _padded_rows(eng):
  t = eng.e.get_field(0, "sensordata")
  raw = native.B2Tensor.from_buffer_copy(t)
  raw.shape[1] = raw.stride[0]
  return eng._wrap(raw)


def arm_padding(eng):
  rows = _padded_rows(eng)
  rows[:, eng.e.get_field(0, "sensordata").shape[1]:] = SENTINEL


def check_padding(eng):
  rows = _padded_rows(eng).cpu().numpy()
  assert (rows[:, int(eng.e.get_field(0, "sensordata").shape[1]):] == SENTINEL).all(), "write past the last sensor"


# ---- the synthetic robot -----------------------------------------------------------------------------------------

LINK = "l3_5"  # a lower link of the fourth chain: often on the floor
OBJECTS = [
  dict(subtree1="base"),  # every contact of the robot, no secondary object
  dict(geom1="floor", subtree2="base"),  # dir = +1 (the plane is the first geom of its contacts)
  dict(subtree1="base", geom2="floor"),  # dir = -1
  dict(body1=LINK, body2="world"),  # body against body (the floor's), dir = -1
  dict(geom1=LINK + "_box"),  # a geom, no secondary object
  dict(geom1="floor", subtree2="l3_0"),  # a chain's subtree as the secondary object
  dict(subtree1="base", subtree2="base"),  # self contacts: both orientations match, dir = +1
  dict(subtree1="l3_0", subtree2="base"),  # the chain against the rest: both dirs, and its own self contacts
]
REDUCE = [("none", 1), ("none", 8), ("none", 40), ("netforce", 1)]


def robot_sensors():
  """Every object pair with every reduction; the 31 data subsets in turn (the full set twice); last a two-float
  sensor matching every contact, whose slot fits the row padding, so that nsensordata leaves row padding for a write past its one slot to land in."""
  out = []
  for i, (obj, (red, num)) in enumerate(itertools.product(OBJECTS, REDUCE)):
    out.append(ContactSensorCfg(name=f"s{i}", data=SUBSETS[(i + 30) % 31], reduce=red, num=num, **obj))
  out.append(ContactSensorCfg(name="tail", subtree1="base", data=("found", "dist"), num=1))
  return out


def robot_spec():
  return Spec.from_string(robot_xml(np.random.default_rng(1), 6, 8, dofs=50, box_links=True))


def robot_model():
  """tools/synth_models.py's box-link robot (six chains of eight links: up to four box-plane contacts each), its link
  geoms named after their bodies, the floor frictionless (condim 1) so that condim-1 geoms give condim-1 contacts,
  a margin and gap on the floor so that every floor contact has an excluded band, and the sensors above added
  through ContactSensorCfg.edit_spec."""
  sp = robot_spec()
  for b in sp.bodies:
    for g in b.geoms:
      g.name = g.name or b.name + "_box"
  floor = sp.geom("floor")
  floor.condim, floor.margin, floor.gap = 1, 0.004, 0.002
  for c in robot_sensors():
    c.edit_spec(sp)
  return sp.compile()


_STATES = {}


def _robot_states(m, seed):
  """Base heights 0.6-0.8 m with the joints 0.3 rad off their rest angles: 20-90 contacts, tens of them between
  links.  World 0 hangs lowest, world 1 highest.  Worlds where the fp64 oracle finds more than 88 contacts are raised 3 cm at a time
  (the engine keeps 96 per world here)."""
  if (id(m), seed) in _STATES:
    return _STATES[id(m), seed]
  n = 130
  rng = np.random.default_rng(seed)
  q = np.tile(np.asarray(m.qpos0, np.float64), (n, 1))
  q[:, 2] = rng.uniform(0.6, 0.8, n)
  q[0, 2], q[1, 2] = 0.6, 0.8
  q[:, 7:] += rng.uniform(-0.3, 0.3, (n, int(m.nq) - 7))
  st = dict(qpos=q, qvel=rng.uniform(-0.5, 0.5, (n, int(m.nv))), ctrl=rng.uniform(-1, 1, (n, int(m.nu))),
            qacc_warmstart=np.zeros((n, int(m.nv))))
  while True:
    o = Oracle(m, nworld=n, maxcon=200)
    load_oracle(o, st)
    o.forward()
    over = o.ncon.ravel() > 88
    if not over.any():
      _STATES[id(m), seed] = st
      return st
    q[over, 2] += 0.03


def robot_states(m, n, seed=21):
  """The first `n` worlds of _robot_states (world 0 has more than 64 contacts with seed 21)."""
  return {k: v[:n].copy() for k, v in _robot_states(m, seed).items()}


@pytest.fixture(scope="module")
def robot():
  m = robot_model()
  return m, Sensors(m)


def _pair(backend, m, n, st, maxcon=160):
  eng = Eng(backend, m, n, nconmax=maxcon * n)
  o = Oracle(m, nworld=n, maxcon=int(eng.opt("maxcon")), njmax=3000)
  eng.load(st)
  load_oracle(o, st)
  return eng, o


def require(facts, n):
  """The conditions the robot cases exist for, over the facts of all their comparisons."""
  net40 = [f["nmatch"] for f in facts if f["reduce"] == 0 and f["num"] == 40]
  assert max(net40) > 40 and any(32 < k < 40 or k > 64 for k in net40), sorted(set(net40))
  assert any(f["neg"] and f["data"] & (2 | 32) and f["reduce"] == 0 for f in facts), "no dir = -1 match"
  assert any(f["neg"] and f["data"] & 2 and f["reduce"] == 3 for f in facts), "no dir = -1 netforce"
  assert any(f["excluded"] for f in facts), "no excluded contact between matched objects"
  assert any(f["condim1"] and f["data"] & 2 for f in facts), "no condim-1 match"
  assert any(f["normal_checked"] for f in facts), "no netforce normal compared"
  if n > 1:
    assert any(0 < f["nmatch"] < f["num"] for f in facts if f["reduce"] == 0 and f["num"] == 40)
    assert any(f["nmatch"] > 8 for f in facts if f["reduce"] == 0 and f["num"] == 8)


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("n", [1, 3, 130])  # 130: the last 4-warp CTA on the GPU is half empty
def test_robot_sensors(backend, n, robot):
  """forward, step (the sensors of the pre-integration state) and step_n(4) (the last sub-step): comparisons 1-3
  on the box-link robot, with sentinels in the sensordata row padding."""
  m, S = robot
  st = robot_states(m, n)
  eng, o = _pair(backend, m, n, st)
  assert int(m.nsensordata) % 4 != 0 and S.intprm[-1].tolist() == [9, 0, 1]
  facts = []
  arm_padding(eng)
  eng.forward()
  o.forward()
  facts += check_engine(S, eng)
  facts += check_oracle(S, o)
  check_against_oracle(S, eng, o)
  assert int(eng.a("ncon").max()) > 64 and not eng.a("overflow").any()
  eng.step()
  o.step()
  facts += check_engine(S, eng)
  facts += check_oracle(S, o)
  check_against_oracle(S, eng, o)
  eng.step_n(4)
  for _ in range(4):
    o.step()
  facts += check_engine(S, eng)
  facts += check_oracle(S, o)
  same = same_contact_sets(S, eng, o)
  assert 2 * len(same) >= n, same
  counts_agree(S, eng, o, same)
  check_padding(eng)
  require(facts, n)
  eng.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_masked_forward_keeps_unselected_sensors(backend, robot):
  """A masked forward evaluates the sensors of the selected worlds only: the others keep their sensordata bit for
  bit (here the values of an earlier, different state)."""
  m, S = robot
  n = 6
  eng, _ = _pair(backend, m, n, robot_states(m, n, seed=3))
  eng.forward()
  before = eng.a("sensordata").copy()
  assert (before != 0).any(axis=1).all()
  eng.load(robot_states(m, n, seed=4))
  mask = np.arange(n) % 2 == 1
  eng.forward_masked(mask)
  after = eng.a("sensordata")
  assert np.array_equal(after[~mask], before[~mask])
  assert not np.array_equal(after[mask], before[mask])
  check_engine(S, eng, np.nonzero(mask)[0])
  eng.close()


@pytest.mark.parametrize("backend", BACKENDS)
def test_stale_slots_are_cleared(backend, robot):
  """A step with many contacts, then a forward of the robot lifted clear of the floor with its joints at rest (no
  contacts): every slot that held data reads zero, including the first values of the sensors, in the engine and in
  the oracle."""
  m, S = robot
  n = 3
  st = robot_states(m, n)
  eng, o = _pair(backend, m, n, st)
  eng.step()
  o.step()
  held = eng.a("sensordata") != 0
  assert held[:, S.adr].any(axis=0).sum() >= S.n // 2, "the first value of most sensors held data"
  held_o = o.sensordata != 0
  assert held_o[:, S.adr].any(axis=0).sum() >= S.n // 2
  up = robot_states(m, n)
  up["qpos"][:, 2] = 3.0
  up["qpos"][:, 7:] = np.asarray(m.qpos0)[7:]
  eng.load(up)
  load_oracle(o, up)
  eng.forward()
  o.forward()
  assert int(eng.a("ncon").max()) == 0 and int(o.ncon.max()) == 0
  assert (eng.a("sensordata")[held] == 0).all() and (o.sensordata[held_o] == 0).all()
  eng.close()


# ---- the mesh / height-field scene (the convex step kernel) -------------------------------------------------------


CONVEX_SENSORS = (
  ContactSensorCfg(name="m1", body1="m1", data=("found", "force", "dist", "pos", "normal"), num=8),
  ContactSensorCfg(name="m1_net", body1="m1", data=("found", "force", "pos", "normal"), reduce="netforce"),
  ContactSensorCfg(name="field", geom1="terrain", data=("found", "force", "dist", "pos", "normal"), num=8),
  ContactSensorCfg(name="field_net", geom1="terrain", data=("found", "force", "pos", "normal"), reduce="netforce"),
  ContactSensorCfg(name="hm_field", subtree1="hm", geom2="terrain", data=("found", "force", "normal"), num=2),
  ContactSensorCfg(name="floor_bx", geom1="floor", body2="bx", data=("found", "dist"), num=1),
)


@pytest.mark.parametrize("backend", BACKENDS)
def test_convex_scene_sensors(backend):
  """Sensors on a mesh body and on the height field, in the scene of tests/util.convex_scene: comparisons 1-3 after
  a forward and a step; the contacts of the convex routines against the oracle's at the bounds of
  test_convex_scene."""
  m, anchors, hf = convex_scene(sensors=CONVEX_SENSORS)
  S = Sensors(m)
  n = 8
  eng, o = _pair(backend, m, n, convex_states(m, anchors, hf, n, seed=9), maxcon=64)
  facts = []
  for entry in ("forward", "step"):
    getattr(eng, entry)()
    getattr(o, entry)()
    facts += check_engine(S, eng)
    facts += check_oracle(S, o)
    check_against_oracle(S, eng, o, dist_tol=2e-5, pos_tol=2e-4, normal_tol=5e-3)
  for s in range(S.n):
    assert any(f["nmatch"] for f in facts if f["s"] == s), f"sensor {s} never matched"
  assert any(f["neg"] for f in facts if f["s"] == 4), "hm_field: the field is the first geom, dir = -1 expected"
  eng.close()


# ---- the shipped G1 tracking model ------------------------------------------------------------------------------


@pytest.mark.parametrize("backend", BACKENDS)
def test_g1_self_collision_counter(backend):
  """The 10-slot self-collision sensor of g1_tracking_flat (subtree pelvis against itself, netforce) in states with
  many self contacts: comparisons 1-3 after a forward and a step."""
  from mjlab_b200.asset_zoo import load_compiled

  m = load_compiled("g1_tracking_flat")
  S = Sensors(m)
  assert S.n == 1 and S.intprm[0].tolist() == [1, 3, 10]
  n = 16
  eng, o = _pair(backend, m, n, make_states(m, n, seed=21, joint_noise=1.5), maxcon=96)
  counts = []
  for entry in ("forward", "step"):
    getattr(eng, entry)()
    getattr(o, entry)()
    counts += [f["nmatch"] for f in check_engine(S, eng)]
    check_oracle(S, o)
    check_against_oracle(S, eng, o)
  assert max(counts) >= 3 and sum(k > 0 for k in counts) >= n // 2, counts
  eng.close()


# ---- refusals and the encoding -----------------------------------------------------------------------------------


@pytest.mark.parametrize("opt", [dict(data=("found", "torque")), dict(data=("tangent",)), dict(reduce="mindist"),
                                 dict(reduce="maxforce")], ids=["torque", "tangent", "mindist", "maxforce"])
def test_unsupported_options_are_refused(opt):
  """b2_create refuses the contact-sensor options the engine does not evaluate, each with its message."""
  sp = Spec.from_string(robot_xml(np.random.default_rng(1), 2, 2, dofs=4))
  ContactSensorCfg(name="s", subtree1="base", **opt).edit_spec(sp)
  with pytest.raises(RuntimeError, match="contact sensor data/reduce combination not implemented"):
    native.Engine(_emul_lib(), sp.compile(), 1)


def test_non_contact_sensor_types_are_refused():
  """add_sensor with an mjtSensor type other than contact (here accelerometer, 1) is refused by compile(), not
  evaluated as a contact sensor."""
  sp = robot_spec()
  sp.add_sensor(name="acc", type=1, objtype=OBJ_BODY, objname="base")
  with pytest.raises(NotImplementedError, match="sensor 'acc' \\(type 1\\): the engine evaluates contact sensors only"):
    sp.compile()


ENCODING_CASES = [
  dict(subtree1="base", geom2="floor", data=("found", "force", "pos"), num=8),
  dict(body1="l0_1", data=("normal",), reduce="netforce"),
  dict(geom1="floor", subtree2="l1_0", data=("found", "force", "dist", "pos", "normal"), num=40),
  dict(subtree1="base", subtree2="base", data=("found",), reduce="netforce", num=10),
  dict(body1="l1_1", body2="world", data=("dist", "normal"), num=3),
]


def test_encoding_matches_the_reference_cfg():
  """The reference's own ContactSensorCfg (utils/spec_config.py, on the MjSpec stand-in, which passes MuJoCo's
  mjSENS_CONTACT) and mjlab_b200.compiler.spec_cfg.ContactSensorCfg compile to the same sensor tables."""
  import refload

  if not refload.available():
    pytest.skip("oracle/_ref not installed")
  refload.load()
  import mjlab.utils.spec_config as ref_cfg

  tables = []
  for cfg in (ref_cfg.ContactSensorCfg, ContactSensorCfg):
    sp = robot_spec()
    for i, kw in enumerate(ENCODING_CASES):
      cfg(name=f"s{i}", **kw).edit_spec(sp)
    m = sp.compile()
    tables.append({k: np.asarray(m.arrays[k]).tolist() for k in ("sensor_type", "sensor_objtype", "sensor_objid",
                   "sensor_reftype", "sensor_refid", "sensor_intprm", "sensor_dim", "sensor_adr")})
  assert tables[0] == tables[1]

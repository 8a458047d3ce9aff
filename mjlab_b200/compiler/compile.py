"""Spec -> flat compiled :class:`Model` (the subset of ``mj_compile`` + ``mj_setConst`` the hot path needs).

Id ordering reproduces what the reference's compiler yields because ids leak into
``EntityIndexing`` (reference ``src/mjlab/entity/entity.py:588-652``): bodies depth-first in
spec order, geoms/sites/joints grouped by body in that order, dofs in joint order, actuators
in creation order (SURVEY.md Appendix D).

Derived constants (``body_subtreemass``, ``dof_invweight0``, ``body_invweight0``,
``stat.meaninertia``, ``geom_rbound``, the candidate collision-pair table) are computed here in
float64 numpy at ``qpos0``; they follow MuJoCo's documented ``mj_setConst`` semantics
(SURVEY.md Appendix A.5, restated from the public "Computation" chapter).
"""

from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import NamedTuple

import numpy as np

from mjlab_b200.compiler import spec as S
from mjlab_b200.compiler.spec import quat_mul, quat_to_mat, mat_to_quat

MINVAL = 1e-15


class ModelArray(NamedTuple):
  name: str
  dtype: type  # float64 arrays are narrowed to fp32 by the CUDA library on upload
  width: int | None = None  # row width of a 2-D array; None: 1-D
  set_const: bool = False  # computed by _set_const from the packed model, not by a compile stage


# Every array that travels through the C ABI (include/b2sim.h: B2Array), in descriptor order.
I, F, SET_CONST = np.int32, np.float64, True
MODEL_ARRAYS = [ModelArray(*row) for row in [
  ("body_parentid", I), ("body_rootid", I), ("body_weldid", I),
  ("body_jntadr", I), ("body_jntnum", I), ("body_dofadr", I), ("body_dofnum", I),
  ("body_pos", F, 3), ("body_quat", F, 4), ("body_ipos", F, 3), ("body_iquat", F, 4),
  ("body_mass", F), ("body_subtreemass", F, None, SET_CONST), ("body_inertia", F, 3),
  ("body_invweight0", F, 2, SET_CONST),
  ("jnt_type", I), ("jnt_qposadr", I), ("jnt_dofadr", I), ("jnt_bodyid", I),
  ("jnt_limited", I), ("jnt_pos", F, 3), ("jnt_axis", F, 3), ("jnt_range", F, 2),
  ("jnt_solref", F, 2), ("jnt_solimp", F, 5), ("jnt_margin", F), ("jnt_stiffness", F),
  ("dof_bodyid", I), ("dof_jntid", I), ("dof_parentid", I),
  ("dof_armature", F), ("dof_damping", F), ("dof_frictionloss", F),
  ("dof_invweight0", F, None, SET_CONST),
  ("geom_type", I), ("geom_bodyid", I), ("geom_contype", I),
  ("geom_conaffinity", I), ("geom_condim", I), ("geom_priority", I),
  ("geom_size", F, 3), ("geom_pos", F, 3), ("geom_quat", F, 4), ("geom_friction", F, 3),
  ("geom_solref", F, 2), ("geom_solimp", F, 5), ("geom_solmix", F), ("geom_margin", F),
  ("geom_gap", F), ("geom_rbound", F), ("geom_rgba", F, 4),
  ("site_bodyid", I), ("site_pos", F, 3), ("site_quat", F, 4),
  ("actuator_trnid", I), ("actuator_ctrllimited", I), ("actuator_forcelimited", I),
  ("actuator_gainprm", F, 10), ("actuator_biasprm", F, 10), ("actuator_ctrlrange", F, 2),
  ("actuator_forcerange", F, 2), ("actuator_gear", F),
  ("pair_geom1", I), ("pair_geom2", I),
  # static (world-welded, non-plane) collision geoms found through a uniform xy grid instead of the pair table
  ("static_geom", I), ("static_cell0", I, 2), ("dyn_cgeom", I), ("grid_start", I), ("grid_items", I),
  ("grid_params", F),
  # mesh / height-field assets (csrc/b2_convex.h): geom_dataid -> mesh id (mesh geoms) or hfield id (hfield geoms)
  ("geom_dataid", I), ("mesh_vertadr", I), ("mesh_vertnum", I), ("mesh_vert", F, 3),
  ("hfield_adr", I), ("hfield_nrow", I), ("hfield_ncol", I), ("hfield_size", F, 4), ("hfield_data", F),
  ("sensor_type", I), ("sensor_objtype", I), ("sensor_objid", I),
  ("sensor_reftype", I), ("sensor_refid", I), ("sensor_intprm", I, 3),
  ("sensor_adr", I), ("sensor_dim", I),
  ("qpos0", F),
]]
MODEL_SCALARS_I = [
  "nq", "nv", "nu", "nbody", "njnt", "ngeom", "nsite", "nsensor", "nsensordata", "npair", "nstatic",
  "opt_integrator", "opt_cone", "opt_solver", "opt_iterations", "opt_ls_iterations",
]
MODEL_SCALARS_F = [
  "opt_timestep", "opt_tolerance", "opt_ls_tolerance", "opt_impratio", "stat_meaninertia",
]
# (qpos width, dof width) of each joint type the engine compiles (ball joints are refused)
JOINT_WIDTH = {S.JNT_FREE: (7, 6), S.JNT_SLIDE: (1, 1), S.JNT_HINGE: (1, 1)}


class _Accessor:
  def __init__(self, **kw):
    self.__dict__.update(kw)


@dataclass
class Model:
  """Compiled model: plain numpy arrays named after ``mjModel`` fields."""

  arrays: dict = field(default_factory=dict)
  names: dict = field(default_factory=dict)  # kind -> list[str]
  keys: dict = field(default_factory=dict)  # key name -> dict(qpos, qvel, ctrl)
  opt_gravity: np.ndarray = field(default_factory=lambda: np.array([0, 0, -9.81]))

  def __getattr__(self, name):
    arrays = object.__getattribute__(self, "arrays")
    if name in arrays:
      return arrays[name]
    if name in ("na", "nmocap", "ntendon", "neq"):
      return 0  # mjModel sizes of features outside the compiled subset (read by NanGuard / viewers)
    raise AttributeError(name)

  # name -> id helpers (mirror model.body(name).id style accessors, Appendix D)
  def name2id(self, kind: str, name: str) -> int:
    try:
      return self.names[kind].index(name)
    except ValueError:
      raise KeyError(f"{kind} '{name}' not found") from None

  def body(self, name):
    i = int(name) if isinstance(name, (int, np.integer)) else self.name2id("body", name)
    return _Accessor(id=i, name=self.names["body"][i], mass=np.array([float(self.body_mass[i])]),
                     pos=np.asarray(self.body_pos)[i], parentid=np.array([int(self.body_parentid[i])]))

  # (scalar attributes come back as 1-element arrays, as the MuJoCo bindings return them: `jnt.dofadr[0]`)
  def joint(self, name):
    i = int(name) if isinstance(name, (int, np.integer)) else self.name2id("joint", name)
    return _Accessor(
      id=i, name=self.names["joint"][i], type=np.array([int(self.jnt_type[i])]),
      qposadr=np.array([int(self.jnt_qposadr[i])]), dofadr=np.array([int(self.jnt_dofadr[i])]),
      range=np.asarray(self.jnt_range)[i],
    )

  def geom(self, key):
    i = int(key) if isinstance(key, (int, np.integer)) else self.name2id("geom", key)
    return _Accessor(
      id=i, name=self.names["geom"][i], condim=np.array([int(self.geom_condim[i])]),
      priority=np.array([int(self.geom_priority[i])]), friction=self.geom_friction[i],
    )

  def actuator(self, key):
    i = int(key) if isinstance(key, (int, np.integer)) else self.name2id("actuator", key)
    return _Accessor(
      id=i, name=self.names["actuator"][i], gainprm=self.actuator_gainprm[i],
      biasprm=self.actuator_biasprm[i], forcerange=self.actuator_forcerange[i],
    )

  def sensor(self, name):
    i = int(name) if isinstance(name, (int, np.integer)) else self.name2id("sensor", name)
    return _Accessor(id=i, name=self.names["sensor"][i], adr=np.array([int(self.sensor_adr[i])]),
                     dim=np.array([int(self.sensor_dim[i])]))

  def key(self, name):
    return _Accessor(**self.keys[name])

  # -- persistence (compiled blobs ship in mjlab_b200/asset_zoo/compiled) -------------------
  def save(self, path) -> None:
    import json

    meta = {
      "names": self.names,
      "keys": {k: {n: (None if v is None else list(map(float, v))) for n, v in d.items()}
               for k, d in self.keys.items()},
      "gravity": list(map(float, self.opt_gravity)),
    }
    np.savez_compressed(path, __meta__=np.array(json.dumps(meta)), **self.arrays)

  @staticmethod
  def from_binary_path(path) -> "Model":
    """``mujoco.MjModel.from_binary_path``: the blob ``mj_saveModel`` wrote (this engine's npz, whatever its suffix)."""
    return Model.load(path)

  @staticmethod
  def load(path) -> "Model":
    import json

    z = np.load(path, allow_pickle=False)
    meta = json.loads(str(z["__meta__"]))
    m = Model()
    m.arrays = {k: z[k] for k in z.files if k != "__meta__"}
    m.names = meta["names"]
    m.keys = {
      k: {n: (None if v is None else np.array(v)) for n, v in d.items()}
      for k, d in meta["keys"].items()
    }
    m.opt_gravity = np.array(meta["gravity"])
    return m


# ---------------------------------------------------------------------------------------
# geometry-derived inertia (bodies without <inertial>)
# ---------------------------------------------------------------------------------------


def mesh_volume_inertia(vertex: np.ndarray, face: np.ndarray | None):
  """(volume, centre of mass, 3x3 unit-density inertia about the com) of a closed triangle mesh (signed
  tetrahedra against the origin); without faces the convex hull is used, which is also what collides."""
  if face is None:
    from scipy.spatial import ConvexHull

    hull = ConvexHull(vertex)
    face = hull.simplices.copy()
    c = vertex[hull.vertices].mean(axis=0)
    for k, f in enumerate(face):  # orient outwards
      a, b, d = vertex[f]
      if np.dot(np.cross(b - a, d - a), a - c) < 0:
        face[k] = f[::-1]
  a, b, c = vertex[face[:, 0]], vertex[face[:, 1]], vertex[face[:, 2]]
  vol6 = np.einsum("ij,ij->i", a, np.cross(b, c))
  V = vol6.sum() / 6.0
  if abs(V) < 1e-18:
    return 0.0, np.zeros(3), np.zeros((3, 3))
  com = ((a + b + c) * vol6[:, None]).sum(axis=0) / (24.0 * V)
  # second moments: integral of x x^T over a tetrahedron (0, a, b, c) = vol/20 * (sum_i p_i p_i^T + s s^T), s = a+b+c
  ssum = a + b + c
  C = (np.einsum("i,ij,ik->jk", vol6, a, a) + np.einsum("i,ij,ik->jk", vol6, b, b) + np.einsum("i,ij,ik->jk", vol6, c, c)
       + np.einsum("i,ij,ik->jk", vol6, ssum, ssum)) / 120.0
  if V < 0:
    V, C = -V, -C
  C = C - V * np.outer(com, com)
  inertia = np.trace(C) * np.eye(3) - C
  return float(V), com, inertia




def _geom_volume_inertia(g: S.Geom):
  """(volume, diagonal unit-density inertia in the geom frame)."""
  t, s = g.type, g.size
  if t == S.GEOM_SPHERE:
    r = s[0]
    v = 4.0 / 3.0 * math.pi * r**3
    return v, np.full(3, 0.4 * v * r * r)
  if t == S.GEOM_BOX:
    v = 8 * s[0] * s[1] * s[2]
    return v, v / 3.0 * np.array(
      [s[1] ** 2 + s[2] ** 2, s[0] ** 2 + s[2] ** 2, s[0] ** 2 + s[1] ** 2]
    )
  if t == S.GEOM_CYLINDER:
    r, h = s[0], s[1]
    v = math.pi * r * r * 2 * h
    ixy = v * (3 * r * r + 4 * h * h) / 12.0
    return v, np.array([ixy, ixy, v * r * r / 2])
  if t == S.GEOM_ELLIPSOID:
    v = 4.0 / 3.0 * math.pi * s[0] * s[1] * s[2]
    return v, v / 5.0 * np.array(
      [s[1] ** 2 + s[2] ** 2, s[0] ** 2 + s[2] ** 2, s[0] ** 2 + s[1] ** 2]
    )
  if t == S.GEOM_CAPSULE:
    r, h = s[0], s[1]
    vc = math.pi * r * r * 2 * h
    vs = 4.0 / 3.0 * math.pi * r**3
    v = vc + vs
    iz = vc * r * r / 2 + vs * 0.4 * r * r
    # hemispheres displaced by h (+ 3r/8 centroid offset inside each hemisphere)
    ixy = vc * (3 * r * r + 4 * h * h) / 12.0 + vs * (0.4 * r * r + h * h + 0.75 * r * h)
    return v, np.array([ixy, ixy, iz])
  return 0.0, np.zeros(3)  # plane / mesh / hfield carry no mass here


def _body_inertial_from_geoms(b: S.Body, meshes: dict | None = None):
  tot_m, com = 0.0, np.zeros(3)
  parts = []
  for g in b.geoms:
    if g.type == S.GEOM_MESH and meshes and g.mesh in meshes and (g.mass is not None or g.density > 0):
      mesh = meshes[g.mesh]
      try:
        vol, mc, mi = mesh_volume_inertia(mesh.load(), mesh.face)
      except (OSError, ValueError):
        continue  # asset not readable here: the geom carries no mass (bodies of the zoo robots have <inertial>)
      if vol <= 0:
        continue
      m = g.mass if g.mass is not None else g.density * vol
      if m <= 0:
        continue
      R = quat_to_mat(g.quat)
      w, v = np.linalg.eigh(mi * (m / vol))
      parts.append((m, g.pos + R @ mc, R @ v, w))
      tot_m += m
      com += m * (g.pos + R @ mc)
      continue
    vol, inert = _geom_volume_inertia(g)
    if vol <= 0:
      continue
    m = g.mass if g.mass is not None else g.density * vol
    if m <= 0:
      continue
    parts.append((m, g.pos, quat_to_mat(g.quat), inert * (m / vol)))
    tot_m += m
    com += m * g.pos
  if tot_m <= 0:
    return np.zeros(3), np.array([1.0, 0, 0, 0]), 0.0, np.zeros(3)
  com /= tot_m
  full = np.zeros((3, 3))
  for m, p, R, inert in parts:
    d = p - com
    full += R @ np.diag(inert) @ R.T + m * (np.dot(d, d) * np.eye(3) - np.outer(d, d))
  w, v = np.linalg.eigh(full)
  order = np.argsort(-w)  # MuJoCo sorts principal inertias in decreasing order
  w, v = w[order], v[:, order]
  if np.linalg.det(v) < 0:
    v[:, 2] *= -1
  return com, mat_to_quat(v), tot_m, w


# ---------------------------------------------------------------------------------------
# compile
# ---------------------------------------------------------------------------------------


def _rbound(t, s):
  if t == S.GEOM_SPHERE:
    return s[0]
  if t == S.GEOM_CAPSULE:
    return s[0] + s[1]
  if t == S.GEOM_CYLINDER:
    return math.hypot(s[0], s[1])
  if t in (S.GEOM_BOX, S.GEOM_ELLIPSOID):
    return float(np.linalg.norm(s)) if t == S.GEOM_BOX else float(max(s))
  return 0.0  # plane, mesh (non-colliding here)


_SUPPORTED_PAIRS = {
  (S.GEOM_PLANE, S.GEOM_SPHERE), (S.GEOM_PLANE, S.GEOM_CAPSULE), (S.GEOM_PLANE, S.GEOM_BOX),
  (S.GEOM_SPHERE, S.GEOM_SPHERE), (S.GEOM_SPHERE, S.GEOM_CAPSULE),
  (S.GEOM_CAPSULE, S.GEOM_CAPSULE),
  (S.GEOM_SPHERE, S.GEOM_BOX), (S.GEOM_CAPSULE, S.GEOM_BOX), (S.GEOM_BOX, S.GEOM_BOX),
  # convex routines (csrc/b2_convex.h): meshes through their convex hull, height fields prism by prism
  (S.GEOM_PLANE, S.GEOM_MESH), (S.GEOM_SPHERE, S.GEOM_MESH), (S.GEOM_CAPSULE, S.GEOM_MESH),
  (S.GEOM_BOX, S.GEOM_MESH), (S.GEOM_MESH, S.GEOM_MESH),
  (S.GEOM_HFIELD, S.GEOM_SPHERE), (S.GEOM_HFIELD, S.GEOM_CAPSULE), (S.GEOM_HFIELD, S.GEOM_BOX),
  (S.GEOM_HFIELD, S.GEOM_MESH),
}
# cylinders and ellipsoids: smooth convex cores with closed-form support points (GJK / EPA against every convex
# shape, prisms of a height field included; MuJoCo's plane primitives against a plane)
for _t in (S.GEOM_ELLIPSOID, S.GEOM_CYLINDER):
  _SUPPORTED_PAIRS |= {(S.GEOM_PLANE, _t), (S.GEOM_HFIELD, _t)}
  for _u in (S.GEOM_SPHERE, S.GEOM_CAPSULE, S.GEOM_ELLIPSOID, S.GEOM_CYLINDER, S.GEOM_BOX, S.GEOM_MESH):
    _SUPPORTED_PAIRS.add((min(_t, _u), max(_t, _u)))
STATIC_GRID_THRESHOLD = 16  # more static box/sphere/capsule geoms than this -> grid broadphase


def _build_static_grid(A, static, weld, gbody, gtype, ngeom, cell: float = 1.0) -> None:
  """Uniform xy grid over the static geoms' world AABBs (their bodies never move, so world pose = the
  composition of the welded chain; only world-body children are supported, which is what the terrain is).
  grid_params = [x0, y0, cell, nx, ny]; cell (ix, iy) -> index ix*ny + iy; grid_items lists positions in
  ``static_geom``; static_cell0 holds each static geom's minimal cell (ix0, iy0) for duplicate rejection."""
  A["static_geom"] = list(static)
  A["dyn_cgeom"] = []
  A["static_cell0"], A["grid_start"], A["grid_items"] = [], [0], []
  A["grid_params"] = [0.0, 0.0, cell, 0.0, 0.0]
  if not static:
    return
  lo, hi = [], []
  for g in static:
    b = gbody[g]
    if A["body_parentid"][b] != 0:
      raise NotImplementedError("static collision geoms must sit on a direct child of the world body")
    Rb = quat_to_mat(np.array(A["body_quat"][b]))
    pb = np.array(A["body_pos"][b])
    R = Rb @ quat_to_mat(np.array(A["geom_quat"][g]))
    c = pb + Rb @ np.array(A["geom_pos"][g])
    sz = np.array(A["geom_size"][g], dtype=float)
    if gtype[g] == S.GEOM_BOX:
      ext = np.abs(R) @ sz
    elif gtype[g] == S.GEOM_SPHERE:
      ext = np.full(3, sz[0])
    elif gtype[g] == S.GEOM_CAPSULE:
      ext = np.abs(R[:, 2]) * sz[1] + sz[0]
    else:
      raise NotImplementedError("static grid supports box / sphere / capsule geoms")
    lo.append(c - ext)
    hi.append(c + ext)
  lo, hi = np.array(lo), np.array(hi)
  x0, y0 = lo[:, 0].min(), lo[:, 1].min()
  # big outer borders would blow up the cell count: cap at 256 x 256 cells by growing the cell size
  span = max(hi[:, 0].max() - x0, hi[:, 1].max() - y0)
  cell = max(cell, span / 256.0)
  nx = int(np.floor((hi[:, 0].max() - x0) / cell)) + 1
  ny = int(np.floor((hi[:, 1].max() - y0) / cell)) + 1
  cells = [[] for _ in range(nx * ny)]
  for k in range(len(static)):
    ix0, ix1 = int((lo[k, 0] - x0) // cell), int((hi[k, 0] - x0) // cell)
    iy0, iy1 = int((lo[k, 1] - y0) // cell), int((hi[k, 1] - y0) // cell)
    A["static_cell0"].append([ix0, iy0])
    for ix in range(ix0, min(ix1, nx - 1) + 1):
      for iy in range(iy0, min(iy1, ny - 1) + 1):
        cells[ix * ny + iy].append(k)
  for c in cells:
    A["grid_items"].extend(c)
    A["grid_start"].append(len(A["grid_items"]))
  A["grid_params"] = [float(x0), float(y0), float(cell), float(nx), float(ny)]
  inset = set(static)
  # dynamic collision geoms that can touch the static set (bit masks are re-checked per candidate)
  smask_t = 0
  smask_a = 0
  for g in static:
    smask_t |= A["geom_contype"][g]
    smask_a |= A["geom_conaffinity"][g]
  A["dyn_cgeom"] = [g for g in range(ngeom)
                    if g not in inset and weld[gbody[g]] != 0
                    and ((A["geom_contype"][g] & smask_a) or (A["geom_conaffinity"][g] & smask_t))]
  for g in A["dyn_cgeom"]:
    if gtype[g] not in (S.GEOM_SPHERE, S.GEOM_CAPSULE, S.GEOM_ELLIPSOID, S.GEOM_CYLINDER, S.GEOM_BOX, S.GEOM_MESH):
      raise NotImplementedError("only sphere / capsule / ellipsoid / cylinder / box / mesh geoms can collide with grid-static geoms")


def compile_spec(spec: S.Spec) -> Model:
  """The compile stages in order: they fill ``A`` (a list per MODEL_ARRAYS row) and ``names``; ``_pack`` makes the Model."""
  A: dict[str, list] = {a.name: [] for a in MODEL_ARRAYS}
  names = {k: [] for k in ("body", "joint", "geom", "site", "actuator", "sensor")}
  mesh_ids, hfield_ids = {}, {}  # asset name -> mesh / height-field id
  # one depth-first pass: the ids of each element kind, and the first refusal among them, follow body order
  for b in spec.bodies:
    _body(spec, b, A, names)
    _joints(spec, b, A, names)
    _geoms(spec, b, A, names, mesh_ids, hfield_ids)
    _sites(b, A, names)
  _weld_and_root(A)
  _actuators(spec, A, names)
  _contact_sensors(spec, A, names)
  _collision_pairs(spec, A, names)
  _refuse_unsupported(A, names)
  m = _pack(spec, A, names)
  _set_const(m)
  _keyframes(spec, m)
  return m


def _body(spec: S.Spec, b: S.Body, A: dict, names: dict) -> None:
  """Frame and inertial of body ``b`` (from its geoms when it has no ``<inertial>``)."""
  b.id = len(names["body"])
  names["body"].append(b.name)
  A["body_parentid"].append(b.parent.id if b.parent is not None else 0)
  A["body_pos"].append(b.pos)
  A["body_quat"].append(b.quat / np.linalg.norm(b.quat))
  if b.mass is not None:
    ipos, iquat, mass, inertia = b.ipos, b.iquat, b.mass, b.inertia
  else:
    ipos, iquat, mass, inertia = _body_inertial_from_geoms(b, spec.meshes)
  A["body_ipos"].append(ipos)
  A["body_iquat"].append(iquat / np.linalg.norm(iquat))
  A["body_mass"].append(mass)
  A["body_inertia"].append(inertia)


def _joints(spec: S.Spec, b: S.Body, A: dict, names: dict) -> None:
  """Joints and dofs of body ``b``."""
  qpos0, nv0 = A["qpos0"], len(A["dof_bodyid"])
  # dof chain parent: last dof of the nearest ancestor that has dofs
  anc = b.parent
  while anc is not None and not A["body_dofnum"][anc.id]:
    anc = anc.parent
  par_dof = -1 if anc is None else A["body_dofadr"][anc.id] + A["body_dofnum"][anc.id] - 1
  A["body_jntadr"].append(len(names["joint"]) if b.joints else -1)
  A["body_jntnum"].append(len(b.joints))
  A["body_dofadr"].append(nv0 if b.joints else -1)
  for j in b.joints:
    j.id = len(names["joint"])
    names["joint"].append(j.name)
    A["jnt_type"].append(j.type)
    A["jnt_qposadr"].append(len(qpos0))
    A["jnt_dofadr"].append(len(A["dof_bodyid"]))
    A["jnt_bodyid"].append(b.id)
    A["jnt_pos"].append(j.pos)
    A["jnt_axis"].append(j.axis)
    limited = j.limited
    if limited == 2:
      limited = int(spec.autolimits and j.range[0] < j.range[1])
    if j.type == S.JNT_FREE:
      limited = 0
    if limited and j.range[1] - j.range[0] < 2.0 * j.margin:
      # both limit rows of the joint could be active at once; the engine keeps one row per joint
      raise NotImplementedError(
        f"joint '{j.name}': range narrower than twice its margin (both limits active at once) is not supported")
    A["jnt_limited"].append(limited)
    A["jnt_range"].append(j.range)
    A["jnt_solref"].append(j.solref_limit)
    A["jnt_solimp"].append(j.solimp_limit)
    A["jnt_margin"].append(j.margin)
    A["jnt_stiffness"].append(j.stiffness)
    if j.type == S.JNT_BALL:
      raise NotImplementedError("ball joints are outside the hot-path feature subset")
    qpos0.extend([*b.pos, *(b.quat / np.linalg.norm(b.quat))] if j.type == S.JNT_FREE else [j.ref])
    for _ in range(JOINT_WIDTH[j.type][1]):
      A["dof_parentid"].append(par_dof)
      par_dof = len(A["dof_bodyid"])
      A["dof_bodyid"].append(b.id)
      A["dof_jntid"].append(j.id)
      A["dof_armature"].append(j.armature)
      A["dof_damping"].append(j.damping)
      A["dof_frictionloss"].append(j.frictionloss)
  A["body_dofnum"].append(len(A["dof_bodyid"]) - nv0)


def _geoms(spec: S.Spec, b: S.Body, A: dict, names: dict, mesh_ids: dict, hfield_ids: dict) -> None:
  """Geoms of body ``b``; the first geom to use a mesh or height field adds the asset's data."""
  for g in b.geoms:
    g.id = len(names["geom"])
    names["geom"].append(g.name)
    A["geom_type"].append(g.type)
    A["geom_bodyid"].append(b.id)
    dataid, size, rbound = -1, g.size, _rbound(g.type, g.size)
    colliding = True
    if g.type == S.GEOM_MESH:
      # A mesh collides (through its convex hull) when it has collision bits and vertex data; a mesh whose
      # file cannot be read stays what it always was here: a visual.
      colliding = False
      mesh = spec.meshes.get(g.mesh) if g.mesh else None
      if mesh is not None and (g.contype or g.conaffinity):
        try:
          v = mesh.load()
        except OSError as e:
          raise FileNotFoundError(f"geom '{g.name}': mesh '{g.mesh}' has collision bits but its file is unreadable ({e})") from None
        if g.mesh not in mesh_ids:
          mesh_ids[g.mesh] = len(mesh_ids)
          A["mesh_vertadr"].append(sum(A["mesh_vertnum"]))
          A["mesh_vertnum"].append(len(v))
          A["mesh_vert"].extend(v.tolist())
        dataid, colliding = mesh_ids[g.mesh], True
        size = np.abs(v).max(axis=0)
        rbound = float(np.linalg.norm(v, axis=1).max())
    elif g.type == S.GEOM_HFIELD:
      hf = spec.hfields.get(g.hfield) if g.hfield else None
      if hf is None:
        raise ValueError(f"geom '{g.name}': hfield asset '{g.hfield}' not found")
      if g.hfield not in hfield_ids:
        hfield_ids[g.hfield] = len(hfield_ids)
        A["hfield_adr"].append(len(A["hfield_data"]))
        A["hfield_nrow"].append(hf.nrow)
        A["hfield_ncol"].append(hf.ncol)
        A["hfield_size"].append(hf.size)
        A["hfield_data"].extend(np.asarray(hf.userdata, dtype=float).reshape(-1).tolist())
      dataid = hfield_ids[g.hfield]
      size = np.array(hf.size[:3], dtype=float)
      rbound = float(np.sqrt(hf.size[0] ** 2 + hf.size[1] ** 2 + max(hf.size[2], hf.size[3]) ** 2))
    A["geom_dataid"].append(dataid)
    A["geom_contype"].append(g.contype if colliding else 0)
    A["geom_conaffinity"].append(g.conaffinity if colliding else 0)
    A["geom_condim"].append(g.condim)
    A["geom_priority"].append(g.priority)
    A["geom_size"].append(size)
    A["geom_pos"].append(g.pos)
    A["geom_quat"].append(g.quat / np.linalg.norm(g.quat))
    A["geom_friction"].append(g.friction)
    A["geom_solref"].append(g.solref)
    A["geom_solimp"].append(g.solimp)
    A["geom_solmix"].append(g.solmix)
    A["geom_margin"].append(g.margin)
    A["geom_gap"].append(g.gap)
    A["geom_rbound"].append(rbound)
    A["geom_rgba"].append(g.rgba)


def _sites(b: S.Body, A: dict, names: dict) -> None:
  for s in b.sites:
    s.id = len(names["site"])
    names["site"].append(s.name)
    A["site_bodyid"].append(b.id)
    A["site_pos"].append(s.pos)
    A["site_quat"].append(s.quat / np.linalg.norm(s.quat))


def _weld_and_root(A: dict) -> None:
  """``body_weldid``: the nearest body at or above each body that has dofs (0: welded to the world);
  ``body_rootid``: the child of the world body it hangs from."""
  parent, dofnum = A["body_parentid"], A["body_dofnum"]
  weld = np.zeros(len(parent), dtype=np.int32)
  root = np.zeros(len(parent), dtype=np.int32)
  for i in range(1, len(parent)):
    weld[i] = i if dofnum[i] > 0 else weld[parent[i]]
    root[i] = i if parent[i] == 0 else root[parent[i]]
  A["body_weldid"], A["body_rootid"] = weld, root


def _actuators(spec: S.Spec, A: dict, names: dict) -> None:
  for k, a in enumerate(spec.actuators):
    a.id = k
    names["actuator"].append(a.name)
    j = names["joint"].index(a.target)
    if A["jnt_type"][j] not in (S.JNT_HINGE, S.JNT_SLIDE):
      raise ValueError(f"actuator '{a.name}': only hinge/slide joint transmission is supported")
    A["actuator_trnid"].append(j)
    ctrlrange = np.array(a.ctrlrange, dtype=float)
    if a.inheritrange > 0:
      # position actuators inherit the joint range (spec_config.py:447 sets inheritrange=1.0)
      lo, hi = A["jnt_range"][j]
      mid, half = 0.5 * (lo + hi), 0.5 * (hi - lo) * a.inheritrange
      ctrlrange = np.array([mid - half, mid + half])
    cl = a.ctrllimited
    if cl == 2:
      cl = int(spec.autolimits and ctrlrange[0] < ctrlrange[1])
    fl = a.forcelimited
    if fl == 2:
      fl = int(spec.autolimits and a.forcerange[0] < a.forcerange[1])
    A["actuator_ctrllimited"].append(cl)
    A["actuator_forcelimited"].append(fl)
    A["actuator_ctrlrange"].append(ctrlrange)
    A["actuator_forcerange"].append(np.array(a.forcerange, dtype=float))
    A["actuator_gainprm"].append(np.array(a.gainprm, dtype=float))
    A["actuator_biasprm"].append(np.array(a.biasprm, dtype=float))
    A["actuator_gear"].append(a.gear)


def _contact_sensors(spec: S.Spec, A: dict, names: dict) -> None:
  adr = 0
  kind_of = {S.OBJ_BODY: "body", S.OBJ_XBODY: "body", S.OBJ_GEOM: "geom", S.OBJ_SITE: "site"}
  for k, sn in enumerate(spec.sensors):
    # contact sensors arrive through add_sensor: ContactSensorCfg's default type, or MuJoCo's mjSENS_CONTACT from
    # the reference's ContactSensorCfg on the MjSpec stand-in; anything else (an MJCF declaration, or add_sensor
    # with another mjtSensor type) is refused rather than evaluated as a contact sensor
    if sn.type not in (S.SENS_CONTACT, S.MJ_SENS_CONTACT):
      what = f"<{sn.tag or 'sensor'}>" if sn.type == S.SENS_MJCF else f"type {sn.type}"
      raise NotImplementedError(
        f"sensor '{sn.name}' ({what}): the engine evaluates contact sensors only (SURVEY.md §8a P9)")
    sn.id = k
    names["sensor"].append(sn.name)
    A["sensor_type"].append(S.SENS_CONTACT)  # (one id, whichever way the sensor was added)
    A["sensor_objtype"].append(sn.objtype)
    A["sensor_objid"].append(names[kind_of[sn.objtype]].index(sn.objname))
    A["sensor_reftype"].append(sn.reftype)
    A["sensor_refid"].append(
      names[kind_of[sn.reftype]].index(sn.refname) if sn.reftype >= 0 else -1
    )
    dataspec, reduce_, num = sn.intprm
    A["sensor_intprm"].append([dataspec, reduce_, num])
    slot = sum(d for b, d in enumerate(S.CONTACT_DATA_DIM) if dataspec >> b & 1)
    dim = slot * num
    A["sensor_adr"].append(adr)
    A["sensor_dim"].append(dim)
    adr += dim


def _collision_pairs(spec: S.Spec, A: dict, names: dict) -> None:
  """Candidate collision pairs (mj_collision's static filters), and the static grid that replaces the pairs of
  static geoms when there are more than STATIC_GRID_THRESHOLD of them."""
  excl = set()
  for b1, b2 in spec.excludes:
    i1, i2 = names["body"].index(b1), names["body"].index(b2)
    excl.add((min(i1, i2), max(i1, i2)))
  gtype, gbody, weld, parent = A["geom_type"], A["geom_bodyid"], A["body_weldid"], A["body_parentid"]
  ngeom = len(gtype)
  # static collision geoms: on a body welded to the world, not a plane, with any collision bit
  static = [g for g in range(ngeom)
            if weld[gbody[g]] == 0 and gtype[g] not in (S.GEOM_PLANE, S.GEOM_MESH, S.GEOM_HFIELD)
            and (A["geom_contype"][g] or A["geom_conaffinity"][g])]
  use_grid = len(static) > STATIC_GRID_THRESHOLD
  in_grid = set(static) if use_grid else set()
  pairs = []
  for g1 in range(ngeom):
    if g1 in in_grid:
      continue
    for g2 in range(g1 + 1, ngeom):
      if g2 in in_grid:
        continue
      ct1, ca1 = A["geom_contype"][g1], A["geom_conaffinity"][g1]
      ct2, ca2 = A["geom_contype"][g2], A["geom_conaffinity"][g2]
      if not ((ct1 & ca2) or (ct2 & ca1)):
        continue
      b1, b2 = gbody[g1], gbody[g2]
      w1, w2 = weld[b1], weld[b2]
      if w1 == w2:
        continue
      wp1, wp2 = weld[parent[w1]], weld[parent[w2]]
      if w1 != 0 and w2 != 0 and (w1 == wp2 or w2 == wp1):
        continue
      if (min(b1, b2), max(b1, b2)) in excl:
        continue
      a, b = (g1, g2) if gtype[g1] <= gtype[g2] else (g2, g1)
      if (gtype[a], gtype[b]) not in _SUPPORTED_PAIRS:
        if gtype[a] in (S.GEOM_PLANE, S.GEOM_HFIELD) and gtype[b] in (S.GEOM_PLANE, S.GEOM_HFIELD):
          continue
        raise NotImplementedError(
          f"collision pair {names['geom'][a]}({gtype[a]}) - {names['geom'][b]}({gtype[b]}) "
          "is outside the primitive set of the hot path"
        )
      pairs.append((a, b))
  # contacts of one (unordered) body pair are kept contiguous: the solver accumulates one 6x6
  # block per body pair (DESIGN.md "solver").  Order inside a body pair: geom ids.
  pairs.sort(key=lambda p: (min(gbody[p[0]], gbody[p[1]]), max(gbody[p[0]], gbody[p[1]]), p))
  A["pair_geom1"] = [p[0] for p in pairs]
  A["pair_geom2"] = [p[1] for p in pairs]
  _build_static_grid(A, static if use_grid else [], weld, gbody, gtype, ngeom)


def _refuse_unsupported(A: dict, names: dict) -> None:
  """Features the engine does not implement must fail here, not silently change the physics."""
  used = {g for p in zip(A["pair_geom1"], A["pair_geom2"]) for g in p}
  for g in used:
    if A["geom_condim"][g] not in (1, 3):
      raise NotImplementedError(
        f"geom '{names['geom'][g]}': condim {A['geom_condim'][g]} (torsional/rolling friction) is not implemented")
  if any(f != 0 for f in A["dof_frictionloss"]):
    raise NotImplementedError("joint frictionloss (dry-friction constraint rows) is not implemented")
  if len(A["dof_bodyid"]) > 64 or len(names["body"]) > 64:
    raise NotImplementedError("hot path supports nv <= 64 and nbody <= 64 (dof/body bitmasks)")


def _pack(spec: S.Spec, A: dict, names: dict) -> Model:
  """The arrays of MODEL_ARRAYS that the stages built, the sizes and the options, as a Model."""
  o = spec.option
  m = Model(names=names, opt_gravity=np.array(o.gravity, dtype=float))
  for a in MODEL_ARRAYS:
    if not a.set_const:
      arr = np.array(A[a.name], dtype=a.dtype)
      m.arrays[a.name] = np.ascontiguousarray(arr if a.width is None else arr.reshape(-1, a.width))
  scal = dict(
    nq=len(A["qpos0"]), nv=len(A["dof_bodyid"]), nu=len(names["actuator"]), nbody=len(names["body"]),
    njnt=len(names["joint"]), ngeom=len(names["geom"]), nsite=len(names["site"]), nsensor=len(names["sensor"]),
    nsensordata=sum(A["sensor_dim"]), npair=len(A["pair_geom1"]), nstatic=len(A["static_geom"]),
    opt_integrator=o.integrator, opt_cone=o.cone, opt_solver=o.solver,
    opt_iterations=o.iterations, opt_ls_iterations=o.ls_iterations,
    opt_timestep=o.timestep, opt_tolerance=o.tolerance, opt_ls_tolerance=o.ls_tolerance,
    opt_impratio=o.impratio,
  )
  for k, v in scal.items():
    m.arrays[k] = np.array(v, dtype=np.int32 if k in MODEL_SCALARS_I else np.float64)
  return m


def _keyframes(spec: S.Spec, m: Model) -> None:
  nq, nv, nu = int(m.nq), int(m.nv), int(m.nu)
  for k in spec.keys:
    qp = k.qpos if k.qpos is not None else m.qpos0
    qv, ct = k.qvel, k.ctrl
    if k.scope is not None and len(qp) != nq:
      # a key of an attached child: its values sit at the child's joints / actuators, defaults elsewhere
      jn, an = m.names["joint"], m.names["actuator"]
      full_q, full_v, full_c = np.array(m.qpos0, dtype=float), np.zeros(nv), np.zeros(nu)
      iq = iv = 0
      for name in k.scope[0]:
        j = jn.index(name)
        wq, wv = JOINT_WIDTH[int(m.jnt_type[j])]
        qa, va = int(m.jnt_qposadr[j]), int(m.jnt_dofadr[j])
        if iq + wq <= len(qp):
          full_q[qa:qa + wq] = np.asarray(qp, dtype=float)[iq:iq + wq]
        if qv is not None and iv + wv <= len(qv):
          full_v[va:va + wv] = np.asarray(qv, dtype=float)[iv:iv + wv]
        iq, iv = iq + wq, iv + wv
      if ct is not None:
        for i, name in enumerate(k.scope[1]):
          if i < len(ct):
            full_c[an.index(name)] = float(ct[i])
      qp, qv, ct = full_q, full_v, full_c
    if len(qp) != nq:
      raise ValueError(f"key '{k.name}': qpos has {len(qp)} entries, model nq={nq}")
    m.keys[k.name] = dict(
      qpos=np.array(qp, dtype=float),
      qvel=np.zeros(nv) if qv is None else np.array(qv, dtype=float),
      ctrl=np.zeros(nu) if ct is None or len(ct) != nu else np.array(ct, float),
    )


# ---------------------------------------------------------------------------------------
# mj_setConst subset: quantities evaluated at qpos0
# ---------------------------------------------------------------------------------------


def kinematics_qpos0(m: Model, qpos=None):
  """Numpy forward kinematics (used only for compile-time constants and host utilities)."""
  nb = int(m.nbody)
  qpos = m.qpos0 if qpos is None else qpos
  xpos = np.zeros((nb, 3))
  xquat = np.zeros((nb, 4))
  xquat[0, 0] = 1
  xanchor = np.zeros((int(m.njnt), 3))
  xaxis = np.zeros((int(m.njnt), 3))
  for i in range(1, nb):
    p = m.body_parentid[i]
    jn, ja = m.body_jntnum[i], m.body_jntadr[i]
    if jn == 1 and m.jnt_type[ja] == S.JNT_FREE:
      a = m.jnt_qposadr[ja]
      pos = qpos[a : a + 3].copy()
      quat = qpos[a + 3 : a + 7] / np.linalg.norm(qpos[a + 3 : a + 7])
      xanchor[ja] = pos
      xaxis[ja] = quat_to_mat(quat) @ m.jnt_axis[ja]
    else:
      R = quat_to_mat(xquat[p])
      pos = xpos[p] + R @ m.body_pos[i]
      quat = quat_mul(xquat[p], m.body_quat[i])
      for j in range(ja, ja + jn):
        Rq = quat_to_mat(quat)
        xanchor[j] = pos + Rq @ m.jnt_pos[j]
        xaxis[j] = Rq @ m.jnt_axis[j]
        d = qpos[m.jnt_qposadr[j]] - m.qpos0[m.jnt_qposadr[j]]
        if m.jnt_type[j] == S.JNT_SLIDE:
          pos = pos + xaxis[j] * d
        else:
          ql = np.concatenate([[math.cos(d / 2)], m.jnt_axis[j] * math.sin(d / 2)])
          quat = quat_mul(quat, ql)
          pos = xanchor[j] - quat_to_mat(quat) @ m.jnt_pos[j]
    xpos[i] = pos
    xquat[i] = quat / np.linalg.norm(quat)
  return xpos, xquat, xanchor, xaxis


def mass_matrix_qpos0(m: Model):
  """Dense joint-space inertia at qpos0 plus what the invweight computation needs."""
  nb, nv = int(m.nbody), int(m.nv)
  xpos, xquat, xanchor, xaxis = kinematics_qpos0(m)
  xipos = np.zeros((nb, 3))
  ximat = np.zeros((nb, 3, 3))
  for i in range(nb):
    R = quat_to_mat(xquat[i])
    xipos[i] = xpos[i] + R @ m.body_ipos[i]
    ximat[i] = quat_to_mat(quat_mul(xquat[i], m.body_iquat[i]))
  # 6D motion vectors [ang; lin] of each dof expressed at the world origin
  Sdof = np.zeros((nv, 6))
  for j in range(int(m.njnt)):
    d, b = m.jnt_dofadr[j], m.jnt_bodyid[j]
    t = m.jnt_type[j]
    if t == S.JNT_FREE:
      R = quat_to_mat(xquat[b])
      for k in range(3):
        Sdof[d + k, 3 + k] = 1.0
        ax = R[:, k]
        Sdof[d + 3 + k, :3] = ax
        Sdof[d + 3 + k, 3:] = np.cross(ax, -xpos[b])
    elif t == S.JNT_HINGE:
      Sdof[d, :3] = xaxis[j]
      Sdof[d, 3:] = np.cross(xaxis[j], -xanchor[j])
    else:
      Sdof[d, 3:] = xaxis[j]
  # chain membership
  chain = np.zeros((nb, nv), dtype=bool)
  for i in range(1, nb):
    chain[i] = chain[m.body_parentid[i]]
    if m.body_dofnum[i] > 0:
      chain[i, m.body_dofadr[i] : m.body_dofadr[i] + m.body_dofnum[i]] = True
  M = np.diag(np.array(m.dof_armature, dtype=float)) if nv else np.zeros((0, 0))
  for i in range(1, nb):
    mass = m.body_mass[i]
    if mass <= 0:
      continue
    Ic = ximat[i] @ np.diag(m.body_inertia[i]) @ ximat[i].T
    c = xipos[i]
    cx = np.array([[0, -c[2], c[1]], [c[2], 0, -c[0]], [-c[1], c[0], 0]])
    I6 = np.zeros((6, 6))
    I6[:3, :3] = Ic + mass * (cx @ cx.T)
    I6[:3, 3:] = mass * cx
    I6[3:, :3] = mass * cx.T
    I6[3:, 3:] = mass * np.eye(3)
    J = Sdof * chain[i][:, None]
    M += J @ I6 @ J.T
  return M, Sdof, chain, xipos


def _set_const(m: Model) -> None:
  nb, nv = int(m.nbody), int(m.nv)
  sub = np.array(m.body_mass, dtype=float).copy()
  for i in range(nb - 1, 0, -1):
    sub[m.body_parentid[i]] += sub[i]
  m.arrays["body_subtreemass"] = sub
  inv_b = np.zeros((nb, 2))
  inv_d = np.zeros(nv)
  mean = 1.0
  if nv:
    M, Sdof, chain, xipos = mass_matrix_qpos0(m)
    Minv = np.linalg.inv(M)
    mean = float(np.mean(np.diag(M)))
    for i in range(1, nb):
      if not chain[i].any():
        continue
      c = xipos[i]
      # 6 x nv Jacobian of body i at its com: rows [lin(3); ang(3)] in MuJoCo's jacp/jacr order
      J = np.zeros((6, nv))
      for d in np.nonzero(chain[i])[0]:
        ang, lin0 = Sdof[d, :3], Sdof[d, 3:]
        J[:3, d] = lin0 + np.cross(ang, c)
        J[3:, d] = ang
      Ainv = J @ Minv @ J.T
      inv_b[i, 0] = max(MINVAL, np.trace(Ainv[:3, :3]) / 3.0)
      inv_b[i, 1] = max(MINVAL, np.trace(Ainv[3:, 3:]) / 3.0)
    dinv = np.diag(Minv).copy()
    for j in range(int(m.njnt)):
      d = m.jnt_dofadr[j]
      if m.jnt_type[j] == S.JNT_FREE:
        dinv[d : d + 3] = dinv[d : d + 3].mean()
        dinv[d + 3 : d + 6] = dinv[d + 3 : d + 6].mean()
    inv_d = dinv
  m.arrays["body_invweight0"] = inv_b
  m.arrays["dof_invweight0"] = inv_d
  m.arrays["stat_meaninertia"] = np.array(mean, dtype=np.float64)

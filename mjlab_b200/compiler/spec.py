"""Minimal model *spec* (editable scene description) and MJCF reader.

The image has no ``mujoco`` wheel, so the part of ``mujoco.MjSpec`` that mjlab's
scene/entity layer touches (SURVEY.md Appendix D; reference call sites
``src/mjlab/scene/scene.py:32-39,133-147``, ``src/mjlab/entity/entity.py:114-161``,
``src/mjlab/utils/spec_config.py:245-276,400-453,514-629``) is provided here:
parse the MJCF subset used by the asset zoo (``g1.xml`` / ``go1.xml`` and the inline
test models of ``tests/test_entity.py``), expose editable element lists, attach one
spec under another with a name prefix, and hand the result to
:func:`mjlab_b200.compiler.compile.compile_spec`.

Supported MJCF: ``compiler(angle, autolimits)``, nested ``default`` classes for
geom/joint/site, ``body/inertial/joint/freejoint/geom/site`` (``pos quat euler axisangle
fromto``), ``contact/exclude``, ``option``, ``actuator/position|motor|general`` (joint
transmission), ``keyframe/key``.  Lights, cameras, materials, textures and mesh assets are
parsed only far enough to keep element ids stable (mesh geoms are kept as non-colliding
geoms; their pose is the XML pose, not the mesh-inertia-aligned pose C MuJoCo produces).
"""

from __future__ import annotations

import copy
import math
import xml.etree.ElementTree as ET
from dataclasses import dataclass, field
from pathlib import Path
from typing import Iterable

import numpy as np

# Enumerations follow MuJoCo's integer values (mjtJoint, mjtGeom, ...), which leak into
# compiled-model arrays that callers index (``typings/mujoco/_enums.pyi`` in the reference).
JNT_FREE, JNT_BALL, JNT_SLIDE, JNT_HINGE = 0, 1, 2, 3
GEOM_PLANE, GEOM_HFIELD, GEOM_SPHERE, GEOM_CAPSULE = 0, 1, 2, 3
GEOM_ELLIPSOID, GEOM_CYLINDER, GEOM_BOX, GEOM_MESH = 4, 5, 6, 7
GEOM_TYPES = {
  "plane": GEOM_PLANE,
  "hfield": GEOM_HFIELD,
  "sphere": GEOM_SPHERE,
  "capsule": GEOM_CAPSULE,
  "ellipsoid": GEOM_ELLIPSOID,
  "cylinder": GEOM_CYLINDER,
  "box": GEOM_BOX,
  "mesh": GEOM_MESH,
}
JNT_TYPES = {"free": JNT_FREE, "ball": JNT_BALL, "slide": JNT_SLIDE, "hinge": JNT_HINGE}
OBJ_BODY, OBJ_XBODY, OBJ_GEOM, OBJ_SITE = 1, 2, 5, 6
SENS_CONTACT = 100  # private id; only contact sensors are evaluated by the engine
MJ_SENS_CONTACT = 42  # mjtSensor.mjSENS_CONTACT, as the reference's ContactSensorCfg passes it to add_sensor
SENS_MJCF = 101     # any sensor declared in MJCF (<sensor><jointpos .../> ...): listed by name, refused by compile()
OBJ_UNKNOWN = 0
INT_EULER, INT_IMPLICITFAST = 0, 3
CONE_PYRAMIDAL, CONE_ELLIPTIC = 0, 1
SOL_PGS, SOL_CG, SOL_NEWTON = 0, 1, 2

CONTACT_DATA = ("found", "force", "torque", "dist", "pos", "normal", "tangent")
CONTACT_DATA_DIM = (1, 3, 3, 1, 3, 3, 3)
CONTACT_REDUCE = ("none", "mindist", "maxforce", "netforce")


def _vec(s, n=None, default=None):
  if s is None:
    return None if default is None else np.array(default, dtype=float)
  if isinstance(s, str):
    v = np.array([float(x) for x in s.split()], dtype=float)
  else:
    v = np.array(s, dtype=float).reshape(-1)
  if n is not None and v.size != n:
    raise ValueError(f"expected {n} numbers, got {v.size}: {s!r}")
  return v


def quat_mul(a, b):
  aw, ax, ay, az = a
  bw, bx, by, bz = b
  return np.array(
    [
      aw * bw - ax * bx - ay * by - az * bz,
      aw * bx + ax * bw + ay * bz - az * by,
      aw * by - ax * bz + ay * bw + az * bx,
      aw * bz + ax * by - ay * bx + az * bw,
    ]
  )


def quat_to_mat(q):
  w, x, y, z = q
  return np.array(
    [
      [w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
      [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
      [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z],
    ]
  )


def mat_to_quat(m):
  """Rotation matrix -> unit quaternion (w,x,y,z)."""
  t = np.trace(m)
  if t > 0:
    s = math.sqrt(t + 1.0) * 2
    q = [0.25 * s, (m[2, 1] - m[1, 2]) / s, (m[0, 2] - m[2, 0]) / s, (m[1, 0] - m[0, 1]) / s]
  elif m[0, 0] > m[1, 1] and m[0, 0] > m[2, 2]:
    s = math.sqrt(1.0 + m[0, 0] - m[1, 1] - m[2, 2]) * 2
    q = [(m[2, 1] - m[1, 2]) / s, 0.25 * s, (m[0, 1] + m[1, 0]) / s, (m[0, 2] + m[2, 0]) / s]
  elif m[1, 1] > m[2, 2]:
    s = math.sqrt(1.0 + m[1, 1] - m[0, 0] - m[2, 2]) * 2
    q = [(m[0, 2] - m[2, 0]) / s, (m[0, 1] + m[1, 0]) / s, 0.25 * s, (m[1, 2] + m[2, 1]) / s]
  else:
    s = math.sqrt(1.0 + m[2, 2] - m[0, 0] - m[1, 1]) * 2
    q = [(m[1, 0] - m[0, 1]) / s, (m[0, 2] + m[2, 0]) / s, (m[1, 2] + m[2, 1]) / s, 0.25 * s]
  q = np.array(q)
  return q / np.linalg.norm(q)


def z_to_quat(vec):
  """Quaternion rotating the z axis onto ``vec`` (MuJoCo's fromto convention)."""
  v = np.array(vec, dtype=float)
  v = v / np.linalg.norm(v)
  axis = np.cross([0.0, 0.0, 1.0], v)
  s = np.linalg.norm(axis)
  if s < 1e-10:
    axis = np.array([1.0, 0.0, 0.0])
  else:
    axis = axis / s
  ang = math.atan2(s, v[2])
  return np.concatenate([[math.cos(ang / 2)], axis * math.sin(ang / 2)])


def euler_to_quat(e):
  """Intrinsic xyz euler (MuJoCo default eulerseq='xyz')."""
  q = np.array([1.0, 0, 0, 0])
  for i, a in enumerate(e):
    ax = np.zeros(3)
    ax[i] = 1
    qi = np.concatenate([[math.cos(a / 2)], ax * math.sin(a / 2)])
    q = quat_mul(q, qi)
  return q


@dataclass
class Geom:
  name: str = ""
  type: int = GEOM_SPHERE
  size: np.ndarray = field(default_factory=lambda: np.zeros(3))
  pos: np.ndarray = field(default_factory=lambda: np.zeros(3))
  quat: np.ndarray = field(default_factory=lambda: np.array([1.0, 0, 0, 0]))
  contype: int = 1
  conaffinity: int = 1
  condim: int = 3
  priority: int = 0
  friction: np.ndarray = field(default_factory=lambda: np.array([1.0, 0.005, 0.0001]))
  solref: np.ndarray = field(default_factory=lambda: np.array([0.02, 1.0]))
  solimp: np.ndarray = field(default_factory=lambda: np.array([0.9, 0.95, 0.001, 0.5, 2.0]))
  solmix: float = 1.0
  margin: float = 0.0
  gap: float = 0.0
  group: int = 0
  rgba: np.ndarray = field(default_factory=lambda: np.array([0.5, 0.5, 0.5, 1.0]))
  mass: float | None = None
  density: float = 1000.0
  mesh: str | None = None
  hfield: str | None = None
  material: str | None = None  # visual only (terrains/terrain_generator.py:215 recolours geoms that have one)
  id: int = -1


@dataclass
class Joint:
  name: str = ""
  type: int = JNT_HINGE
  pos: np.ndarray = field(default_factory=lambda: np.zeros(3))
  axis: np.ndarray = field(default_factory=lambda: np.array([0.0, 0, 1]))
  range: np.ndarray = field(default_factory=lambda: np.zeros(2))
  limited: int = 2  # 0 false, 1 true, 2 auto (mjtLimited)
  armature: float = 0.0
  damping: float = 0.0
  frictionloss: float = 0.0
  stiffness: float = 0.0
  ref: float = 0.0
  margin: float = 0.0
  solref_limit: np.ndarray = field(default_factory=lambda: np.array([0.02, 1.0]))
  solimp_limit: np.ndarray = field(
    default_factory=lambda: np.array([0.9, 0.95, 0.001, 0.5, 2.0])
  )
  id: int = -1


@dataclass
class Site:
  name: str = ""
  pos: np.ndarray = field(default_factory=lambda: np.zeros(3))
  quat: np.ndarray = field(default_factory=lambda: np.array([1.0, 0, 0, 0]))
  size: np.ndarray = field(default_factory=lambda: np.array([0.005, 0.005, 0.005]))
  group: int = 0
  id: int = -1


@dataclass
class Frame:
  body: "Body"
  pos: np.ndarray
  quat: np.ndarray


class Visual:
  """A visual element of the spec (texture, material, light, camera): a named bag of attributes."""

  def __init__(self, name: str = "", **kw):
    self.name = name
    self.__dict__.update(kw)

  def __repr__(self):
    return f"Visual({self.name!r})"


@dataclass
class Body:
  name: str = ""
  pos: np.ndarray = field(default_factory=lambda: np.zeros(3))
  quat: np.ndarray = field(default_factory=lambda: np.array([1.0, 0, 0, 0]))
  # explicit <inertial>; None -> derived from geoms at compile time
  ipos: np.ndarray | None = None
  iquat: np.ndarray | None = None
  mass: float | None = None
  inertia: np.ndarray | None = None
  joints: list = field(default_factory=list)
  geoms: list = field(default_factory=list)
  sites: list = field(default_factory=list)
  children: list = field(default_factory=list)
  lights: list = field(default_factory=list)   # visual only (see Spec.light)
  cameras: list = field(default_factory=list)
  parent: "Body | None" = None
  id: int = -1

  def add_frame(self, pos=None, quat=None, **_) -> "Frame":
    """``MjsBody.add_frame``: a pose under this body that ``Spec.attach(child, frame=...)`` grafts onto
    (``scene/scene.py:137-147`` adds one identity frame per entity and for the terrain)."""
    return Frame(body=self, pos=np.zeros(3) if pos is None else np.asarray(pos, dtype=float),
                 quat=np.array([1.0, 0, 0, 0]) if quat is None else np.asarray(quat, dtype=float))

  def add_light(self, **kw) -> "Visual":
    v = Visual(**kw)
    self.lights.append(v)
    return v

  def add_camera(self, **kw) -> "Visual":
    v = Visual(**kw)
    self.cameras.append(v)
    return v

  def add_body(self, **kw) -> "Body":
    b = Body(**_np_kw(kw))
    b.parent = self
    self.children.append(b)
    return b

  def add_geom(self, **kw) -> Geom:
    kw = _np_kw(kw)
    if isinstance(kw.get("type"), str):
      kw["type"] = GEOM_TYPES[kw["type"]]
    if "size" in kw:
      s = np.zeros(3)
      v = np.array(kw["size"], dtype=float).reshape(-1)
      s[: v.size] = v
      kw["size"] = s
    kw.pop("material", None)
    for api, attr in (("hfieldname", "hfield"), ("meshname", "mesh")):  # MjsGeom attribute names
      if api in kw:
        kw[attr] = kw.pop(api)
    g = Geom(**kw)
    self.geoms.append(g)
    return g

  def add_site(self, **kw) -> Site:
    kw = _np_kw(kw)
    kw.pop("type", None)
    kw.pop("rgba", None)
    s = Site(**kw)
    self.sites.append(s)
    return s

  def add_joint(self, **kw) -> Joint:
    kw = _np_kw(kw)
    if isinstance(kw.get("type"), str):
      kw["type"] = JNT_TYPES[kw["type"]]
    j = Joint(**kw)
    self.joints.append(j)
    return j

  def add_freejoint(self, name: str = "") -> Joint:
    return self.add_joint(name=name, type=JNT_FREE)


def _np_kw(kw):
  out = {}
  for k, v in kw.items():
    if isinstance(v, (tuple, list)):
      v = np.array(v, dtype=float)
    out[k] = v
  return out


@dataclass
class Mesh:
  """``<asset><mesh>``: vertices in the mesh frame (after ``scale``).  Collision uses the convex hull of the
  vertex set (support mapping over all vertices, ``csrc/b2_convex.h``); faces are only needed to derive an
  inertia for bodies without ``<inertial>``.  ``file`` (STL binary/ASCII or OBJ) is read lazily."""

  name: str = ""
  vertex: np.ndarray | None = None  # (n, 3)
  face: np.ndarray | None = None    # (m, 3) int
  file: str | None = None
  scale: np.ndarray = field(default_factory=lambda: np.ones(3))

  def load(self) -> np.ndarray:
    if self.vertex is None:
      if self.file is None:
        raise ValueError(f"mesh '{self.name}' has neither vertex data nor a file")
      v, f = read_mesh_file(self.file)
      self.vertex, self.face = v * self.scale, f
    return self.vertex


@dataclass
class HField:
  """``<asset><hfield>`` / ``spec.add_hfield`` (``terrains/heightfield_terrains.py:213-225``): ``nrow x ncol``
  samples in [0, 1] (row index along y), ``size = (radius_x, radius_y, elevation_z, base_z)``."""

  name: str = ""
  nrow: int = 0
  ncol: int = 0
  size: np.ndarray = field(default_factory=lambda: np.array([1.0, 1.0, 1.0, 0.1]))
  userdata: np.ndarray | None = None


def read_mesh_file(path) -> tuple[np.ndarray, np.ndarray | None]:
  """Vertices (n, 3) and triangles (m, 3) of an STL (binary or ASCII) or OBJ file."""
  path = Path(path)
  raw = path.read_bytes()
  if path.suffix.lower() == ".obj":
    vs, fs = [], []
    for ln in raw.decode(errors="replace").splitlines():
      t = ln.split()
      if not t:
        continue
      if t[0] == "v":
        vs.append([float(x) for x in t[1:4]])
      elif t[0] == "f":
        idx = [int(x.split("/")[0]) for x in t[1:]]
        idx = [i - 1 if i > 0 else len(vs) + i for i in idx]
        fs.extend([idx[0], idx[k], idx[k + 1]] for k in range(1, len(idx) - 1))
    return np.array(vs, dtype=float).reshape(-1, 3), (np.array(fs, dtype=np.int64) if fs else None)
  if raw[:5].lower() == b"solid" and b"facet" in raw[:1000]:
    pts = [[float(x) for x in ln.split()[1:4]] for ln in raw.decode(errors="replace").splitlines()
           if ln.strip().startswith("vertex")]
    tri = np.array(pts, dtype=float).reshape(-1, 3, 3)
  else:
    n = int(np.frombuffer(raw[80:84], dtype="<u4")[0])
    rec = np.frombuffer(raw[84:84 + 50 * n], dtype=np.dtype([("n", "<f4", 3), ("v", "<f4", (3, 3)), ("a", "<u2")]))
    tri = rec["v"].astype(float)
  v, inv = np.unique(tri.reshape(-1, 3), axis=0, return_inverse=True)
  return v, inv.reshape(-1, 3)


@dataclass
class Actuator:
  """General actuator with joint transmission: force = gain*ctrl + bias (fixed gain,
  affine bias).  This is the only family mjlab creates (``spec_config.py:436-453``)."""

  name: str = ""
  target: str = ""
  gainprm: np.ndarray = field(default_factory=lambda: np.array([1.0] + [0.0] * 9))
  biasprm: np.ndarray = field(default_factory=lambda: np.zeros(10))
  gear: float = 1.0
  ctrllimited: int = 2
  ctrlrange: np.ndarray = field(default_factory=lambda: np.zeros(2))
  forcelimited: int = 2
  forcerange: np.ndarray = field(default_factory=lambda: np.zeros(2))
  inheritrange: float = 0.0
  id: int = -1


@dataclass
class Sensor:
  name: str = ""
  type: int = SENS_CONTACT
  objtype: int = OBJ_BODY
  objname: str = ""
  reftype: int = -1
  refname: str = ""
  intprm: tuple = (1, 0, 1)
  tag: str = ""  # MJCF element name of a declared (non-contact) sensor
  id: int = -1


@dataclass
class Key:
  name: str = ""
  qpos: np.ndarray | None = None
  qvel: np.ndarray | None = None
  ctrl: np.ndarray | None = None
  scope: tuple | None = None  # (joint names, actuator names) the values refer to: set when the key came in by attach


@dataclass
class Option:
  """Physics options (``MujocoCfg.edit_spec`` writes these, reference ``sim/sim.py:65-82``)."""

  timestep: float = 0.002
  gravity: tuple = (0.0, 0.0, -9.81)
  integrator: int = INT_EULER
  cone: int = CONE_PYRAMIDAL
  solver: int = SOL_NEWTON
  jacobian: int = 2
  iterations: int = 100
  tolerance: float = 1e-8
  ls_iterations: int = 50
  ls_tolerance: float = 0.01
  impratio: float = 1.0


class Spec:
  """Editable scene description (the subset of ``mujoco.MjSpec`` that mjlab uses)."""

  def __init__(self) -> None:
    self.modelname = "scene"
    self.worldbody = Body(name="world")
    self.option = Option()
    self.actuators: list[Actuator] = []
    self.sensors: list[Sensor] = []
    self.keys: list[Key] = []
    self.excludes: list[tuple[str, str]] = []
    self.meshes: dict[str, Mesh] = {}
    self.hfields: dict[str, HField] = {}
    self.textures: list[Visual] = []
    self.materials: list[Visual] = []
    self.stat = Visual(extent=None, center=None, meansize=None)  # <statistic>: visual scale hints (scene.py:33-34), unused by physics
    self.meshdir = ""  # <compiler meshdir>; mesh files are resolved against it when the MJCF is parsed
    self.assets: dict = {}  # MjSpec.assets (file name -> bytes): accepted; files are read from disk (Mesh.load)
    self.autolimits = True
    self.angle_scale = 1.0  # radians

  # -- traversal -------------------------------------------------------------------------
  def _walk(self, b: Body | None = None) -> Iterable[Body]:
    b = self.worldbody if b is None else b
    yield b
    for c in b.children:
      yield from self._walk(c)

  @property
  def bodies(self) -> list[Body]:
    return list(self._walk())

  @property
  def geoms(self) -> list[Geom]:
    return [g for b in self._walk() for g in b.geoms]

  @property
  def joints(self) -> list[Joint]:
    return [j for b in self._walk() for j in b.joints]

  @property
  def sites(self) -> list[Site]:
    return [s for b in self._walk() for s in b.sites]

  @property
  def tendons(self) -> list:
    return []

  def _find(self, items, name, kind):
    for it in items:
      if it.name == name:
        return it
    raise KeyError(f"{kind} '{name}' not found in spec")

  def body(self, name: str) -> Body:
    return self._find(self.bodies, name, "body")

  def geom(self, name: str) -> Geom:
    return self._find(self.geoms, name, "geom")

  def joint(self, name: str) -> Joint:
    return self._find(self.joints, name, "joint")

  def site(self, name: str) -> Site:
    return self._find(self.sites, name, "site")

  def actuator(self, name: str) -> Actuator:
    return self._find(self.actuators, name, "actuator")

  def sensor(self, name: str) -> Sensor:
    return self._find(self.sensors, name, "sensor")

  # visual elements (textures, materials, lights, cameras): kept so that the spec editors of
  # utils/spec_config.py (TextureCfg / MaterialCfg / LightCfg / CameraCfg .edit_spec) run and find what they
  # added; the physics compiler ignores them
  def texture(self, name: str) -> "Visual":
    return self._find(self.textures, name, "texture")

  def material(self, name: str) -> "Visual":
    return self._find(self.materials, name, "material")

  def light(self, name: str) -> "Visual":
    return self._find([v for b in self._walk() for v in b.lights], name, "light")

  def camera(self, name: str) -> "Visual":
    return self._find([v for b in self._walk() for v in b.cameras], name, "camera")

  def add_texture(self, **kw) -> "Visual":
    t = Visual(**kw)
    self.textures.append(t)
    return t

  def add_material(self, **kw) -> "Visual":
    m = Visual(textures=[""] * 10, **kw)
    self.materials.append(m)
    return m

  # -- element creation -------------------------------------------------------------------
  def add_actuator(self, **kw) -> Actuator:
    kw = _np_kw(kw)
    for drop in ("trntype", "gaintype", "biastype", "dyntype"):
      kw.pop(drop, None)
    a = Actuator(**kw)
    self.actuators.append(a)
    return a

  def add_sensor(self, **kw) -> Sensor:
    s = Sensor(**kw)
    self.sensors.append(s)
    return s

  def add_key(self, **kw) -> Key:
    k = Key(**_np_kw(kw))
    self.keys.append(k)
    return k

  def add_exclude(self, body1: str, body2: str) -> None:
    self.excludes.append((body1, body2))

  # -- composition ------------------------------------------------------------------------
  def add_mesh(self, name: str, vertex=None, face=None, file=None, scale=(1.0, 1.0, 1.0)) -> Mesh:
    m = Mesh(name=name, vertex=None if vertex is None else np.array(vertex, dtype=float).reshape(-1, 3),
             face=None if face is None else np.array(face, dtype=np.int64).reshape(-1, 3), file=file,
             scale=np.array(scale, dtype=float))
    if m.vertex is not None:
      m.vertex = m.vertex * m.scale
    self.meshes[name] = m
    return m

  def add_hfield(self, name: str, size, nrow: int, ncol: int, userdata) -> HField:
    h = HField(name=name, nrow=int(nrow), ncol=int(ncol), size=np.array(size, dtype=float).reshape(4),
               userdata=np.array(userdata, dtype=float).reshape(int(nrow), int(ncol)))
    self.hfields[name] = h
    return h

  def attach(self, child: "Spec", prefix: str = "", parent: Body | None = None, frame: "Frame | None" = None) -> None:
    """Graft a deep copy of ``child``'s world-body children under ``parent`` (default: the
    world body), prefixing every name.  Mirrors ``spec.attach(child, prefix=, frame=)`` as used by
    ``scene/scene.py:133-147``: the terrain is attached un-prefixed and before the entities,
    entities with ``"<name>/"``."""
    if frame is not None:
      parent = frame.body
    parent = self.worldbody if parent is None else parent
    # (no copy: as with MjSpec.attach the child's elements MOVE into this spec and are renamed in place, so an
    # entity that keeps its own spec sees the prefixed names the compiled model uses - entity/entity.py:594-624)
    if frame is not None and (np.any(frame.pos != 0) or np.any(frame.quat != np.array([1.0, 0, 0, 0]))):
      R = quat_to_mat(frame.quat)  # (poses of the child's top level move into the frame)
      for e in (*child.worldbody.children, *child.worldbody.geoms, *child.worldbody.sites):
        e.pos = frame.pos + R @ np.asarray(e.pos, dtype=float)
        e.quat = quat_mul(frame.quat, np.asarray(e.quat, dtype=float))
    child_names = {n.name for n in _all_names(child)}

    def ren(n):
      return prefix + n if n else n

    for b in child._walk():
      for g in b.geoms:  # asset references follow the prefixed asset names
        if g.mesh:
          g.mesh = ren(g.mesh)
        if g.hfield:
          g.hfield = ren(g.hfield)
      if b is child.worldbody:
        continue
      b.name = ren(b.name)
      for e in (*b.joints, *b.geoms, *b.sites):
        e.name = ren(e.name)
    for k, v in child.meshes.items():
      v.name = ren(k)
      self.meshes[v.name] = v
    for k, v in child.hfields.items():
      v.name = ren(k)
      self.hfields[v.name] = v
    # world-level geoms / sites of the child land on the parent body
    for g in child.worldbody.geoms:
      g.name = ren(g.name)
      parent.geoms.append(g)
    for s in child.worldbody.sites:
      s.name = ren(s.name)
      parent.sites.append(s)
    for c in child.worldbody.children:
      c.parent = parent
      parent.children.append(c)
    for a in child.actuators:
      a.name, a.target = ren(a.name), ren(a.target)
      self.actuators.append(a)
    for s in child.sensors:
      s.name, s.objname = ren(s.name), ren(s.objname)
      # a reference that does not exist in the child (e.g. "terrain") stays global
      if s.refname and s.refname in child_names:
        s.refname = ren(s.refname)
      self.sensors.append(s)
    # keyframes of the child keep their values for the child's own joints / actuators; the compiler pads the rest
    # of the parent model with the defaults (qpos0, zero velocity, zero control), as MuJoCo's attach does
    cj = [j.name for b in child._walk() for j in b.joints]
    ca = [a.name for a in child.actuators]
    for k in child.keys:
      k.name = ren(k.name)
      if getattr(k, "scope", None) is None:
        k.scope = (cj, ca)
      self.keys.append(k)
    for b1, b2 in child.excludes:
      self.excludes.append((ren(b1), ren(b2)))

  # -- io ---------------------------------------------------------------------------------
  @staticmethod
  def from_file(path: str | Path) -> "Spec":
    return _parse_mjcf(Path(path).read_text(), Path(path).parent)

  @staticmethod
  def from_string(xml: str, asset_dir: str | Path | None = None) -> "Spec":
    return _parse_mjcf(xml, None if asset_dir is None else Path(asset_dir))

  @staticmethod
  def to_zip(spec: "Spec", file) -> None:
    """``MjSpec.to_zip`` (``scene/scene.py:41-54``).  MuJoCo writes the MJCF and its assets; this compiler has no MJCF
    writer, so the archive holds what reloads here: the compiled model blob (``model.npz``, ``Model.load``)."""
    import io
    import zipfile

    buf = io.BytesIO()
    spec.compile().save(buf)
    with zipfile.ZipFile(file, "w", zipfile.ZIP_DEFLATED) as z:
      z.writestr("model.npz", buf.getvalue())

  def compile(self):
    from mjlab_b200.compiler.compile import compile_spec

    return compile_spec(self)


class _Named:
  def __init__(self, name):
    self.name = name


def _all_names(spec: Spec):
  out = []
  for b in spec._walk():
    out.append(_Named(b.name))
    out.extend(_Named(e.name) for e in (*b.geoms, *b.sites))
  return out


# ---------------------------------------------------------------------------------------
# MJCF reader
# ---------------------------------------------------------------------------------------


class _Defaults:
  """Nested default classes: class name -> {element tag -> attrib dict}."""

  def __init__(self):
    self.cls: dict[str, dict[str, dict[str, str]]] = {"main": {}}
    self.parent: dict[str, str | None] = {"main": None}

  def load(self, node: ET.Element, parent: str | None):
    name = node.get("class", "main" if parent is None else None)
    if name is None:
      raise ValueError("nested <default> needs a class name")
    base = copy.deepcopy(self.cls[parent]) if parent is not None and name != parent else {}
    if name in self.cls and parent is None:
      base = self.cls[name]
    for ch in node:
      if ch.tag == "default":
        continue
      base.setdefault(ch.tag, {}).update(ch.attrib)
    self.cls[name] = base
    self.parent[name] = parent
    for ch in node:
      if ch.tag == "default":
        self.load(ch, name)

  def attrs(self, tag: str, cls: str | None, own: dict[str, str]) -> dict[str, str]:
    out = dict(self.cls.get(cls or "main", {}).get(tag, {}))
    out.update(own)
    return out


def _orientation(a: dict[str, str], scale: float):
  if "quat" in a:
    q = _vec(a["quat"], 4)
    return q / np.linalg.norm(q)
  if "euler" in a:
    return euler_to_quat(_vec(a["euler"], 3) * scale)
  if "axisangle" in a:
    v = _vec(a["axisangle"], 4)
    ax = v[:3] / np.linalg.norm(v[:3])
    ang = v[3] * scale
    return np.concatenate([[math.cos(ang / 2)], ax * math.sin(ang / 2)])
  if "zaxis" in a:
    return z_to_quat(_vec(a["zaxis"], 3))
  if "xyaxes" in a:
    v = _vec(a["xyaxes"], 6)
    x = v[:3] / np.linalg.norm(v[:3])
    y = v[3:] - x * np.dot(x, v[3:])
    y /= np.linalg.norm(y)
    return mat_to_quat(np.stack([x, y, np.cross(x, y)], axis=1))
  return np.array([1.0, 0, 0, 0])


def _parse_geom(a: dict[str, str], scale: float) -> Geom:
  g = Geom(name=a.get("name", ""))
  g.type = GEOM_TYPES[a.get("type", "sphere")]
  size = _vec(a.get("size"), default=[0, 0, 0])
  g.size = np.zeros(3)
  g.size[: size.size] = size
  g.pos = _vec(a.get("pos"), 3, [0, 0, 0])
  g.quat = _orientation(a, scale)
  if "fromto" in a:
    ft = _vec(a["fromto"], 6)
    # MuJoCo: vec = from - to; z axis of the geom frame points along it.
    vec = ft[:3] - ft[3:]
    g.pos = 0.5 * (ft[:3] + ft[3:])
    g.quat = z_to_quat(vec)
    half = 0.5 * np.linalg.norm(vec)
    if g.type in (GEOM_CAPSULE, GEOM_CYLINDER):
      g.size[1] = half
    elif g.type in (GEOM_BOX, GEOM_ELLIPSOID):
      g.size[2] = half
  for k in ("contype", "conaffinity", "condim", "priority", "group"):
    if k in a:
      setattr(g, k, int(a[k]))
  for k in ("solmix", "margin", "gap", "density"):
    if k in a:
      setattr(g, k, float(a[k]))
  if "mass" in a:
    g.mass = float(a["mass"])
  if "friction" in a:
    f = _vec(a["friction"])
    g.friction = g.friction.copy()
    g.friction[: f.size] = f
  if "solref" in a:
    g.solref = _vec(a["solref"], 2)
  if "solimp" in a:
    s = _vec(a["solimp"])
    g.solimp = g.solimp.copy()
    g.solimp[: s.size] = s
  if "rgba" in a:
    g.rgba = _vec(a["rgba"], 4)
  g.mesh = a.get("mesh")
  g.hfield = a.get("hfield")
  return g


def _parse_joint(a: dict[str, str], scale: float) -> Joint:
  j = Joint(name=a.get("name", ""))
  j.type = JNT_TYPES[a.get("type", "hinge")]
  j.pos = _vec(a.get("pos"), 3, [0, 0, 0])
  ax = _vec(a.get("axis"), 3, [0, 0, 1])
  j.axis = ax / np.linalg.norm(ax)
  if "range" in a:
    j.range = _vec(a["range"], 2)
    if j.type == JNT_HINGE:
      j.range = j.range * scale
  if "limited" in a:
    j.limited = {"false": 0, "true": 1, "auto": 2}[a["limited"]]
  for k in ("armature", "damping", "frictionloss", "stiffness", "margin"):
    if k in a:
      setattr(j, k, float(a[k]))
  if "ref" in a:
    j.ref = float(a["ref"]) * (scale if j.type == JNT_HINGE else 1.0)
  if "solreflimit" in a:
    j.solref_limit = _vec(a["solreflimit"], 2)
  if "solimplimit" in a:
    s = _vec(a["solimplimit"])
    j.solimp_limit = j.solimp_limit.copy()
    j.solimp_limit[: s.size] = s
  return j


def _parse_body(node: ET.Element, parent: Body, dfl: _Defaults, childclass, scale):
  for ch in node:
    cls = ch.get("class", childclass)
    if ch.tag == "body":
      b = Body(name=ch.get("name", ""))
      b.pos = _vec(ch.get("pos"), 3, [0, 0, 0])
      b.quat = _orientation(ch.attrib, scale)
      b.parent = parent
      parent.children.append(b)
      _parse_body(ch, b, dfl, ch.get("childclass", childclass), scale)
    elif ch.tag == "inertial":
      parent.ipos = _vec(ch.get("pos"), 3, [0, 0, 0])
      parent.iquat = _orientation(ch.attrib, scale)
      parent.mass = float(ch.get("mass"))
      if ch.get("diaginertia") is not None:
        parent.inertia = _vec(ch.get("diaginertia"), 3)
      else:
        f = _vec(ch.get("fullinertia"), 6)
        full = np.array([[f[0], f[3], f[4]], [f[3], f[1], f[5]], [f[4], f[5], f[2]]])
        w, v = np.linalg.eigh(full)
        if np.linalg.det(v) < 0:
          v[:, 2] *= -1
        parent.inertia = w
        parent.iquat = quat_mul(parent.iquat, mat_to_quat(v))
    elif ch.tag == "freejoint":
      parent.joints.append(Joint(name=ch.get("name", ""), type=JNT_FREE))
    elif ch.tag == "joint":
      parent.joints.append(_parse_joint(dfl.attrs("joint", cls, ch.attrib), scale))
    elif ch.tag == "geom":
      parent.geoms.append(_parse_geom(dfl.attrs("geom", cls, ch.attrib), scale))
    elif ch.tag == "site":
      a = dfl.attrs("site", cls, ch.attrib)
      s = Site(name=a.get("name", ""))
      s.pos = _vec(a.get("pos"), 3, [0, 0, 0])
      s.quat = _orientation(a, scale)
      if "group" in a:
        s.group = int(a["group"])
      parent.sites.append(s)
    elif ch.tag in ("light", "camera"):
      pass  # visual only
    else:
      raise NotImplementedError(
        f"<{ch.tag}> inside <body> is outside the MJCF subset of the hot path "
        "(supported: body, inertial, joint, freejoint, geom, site, light, camera)")


def _parse_mjcf(xml: str, asset_dir: Path | None = None) -> Spec:
  root = ET.fromstring(xml)
  if root.tag != "mujoco":
    raise ValueError("root element must be <mujoco>")
  spec = Spec()
  spec.modelname = root.get("model", "scene")
  comp = root.find("compiler")
  scale = math.pi / 180.0  # MJCF default angle unit is degree
  if comp is not None:
    if comp.get("angle", "degree") == "radian":
      scale = 1.0
    spec.autolimits = comp.get("autolimits", "true") == "true"
  spec.angle_scale = scale
  dfl = _Defaults()
  for d in root.findall("default"):
    dfl.load(d, None)
  opt = root.find("option")
  if opt is not None:
    o = spec.option
    for k in ("timestep", "tolerance", "ls_tolerance", "impratio"):
      if opt.get(k) is not None:
        setattr(o, k, float(opt.get(k)))
    for k in ("iterations", "ls_iterations"):
      if opt.get(k) is not None:
        setattr(o, k, int(opt.get(k)))
    if opt.get("gravity") is not None:
      o.gravity = tuple(_vec(opt.get("gravity"), 3))
    if opt.get("integrator") is not None:
      o.integrator = {"Euler": INT_EULER, "implicitfast": INT_IMPLICITFAST}[
        opt.get("integrator")
      ]
    if opt.get("cone") is not None:
      o.cone = {"pyramidal": CONE_PYRAMIDAL, "elliptic": CONE_ELLIPTIC}[opt.get("cone")]
    if opt.get("solver") is not None:
      o.solver = {"PGS": SOL_PGS, "CG": SOL_CG, "Newton": SOL_NEWTON}[opt.get("solver")]
  for ch in root:
    if ch.tag not in ("compiler", "default", "option", "asset", "worldbody", "contact", "actuator",
                      "keyframe", "visual", "statistic", "size", "sensor"):
      raise NotImplementedError(
        f"<{ch.tag}> is outside the MJCF subset of the hot path (no tendons, equalities, ...)")
  # <sensor>: declarations are kept (an entity lists and finds its sensors by name, entity/entity.py); the engine
  # evaluates contact sensors only, so compile() refuses a model that still carries any other type
  for sen in root.findall("sensor"):
    for e in sen:
      target = next((e.get(k) for k in ("joint", "body", "site", "geom", "objname", "actuator", "tendon") if e.get(k)), "")
      objtype = {"body": OBJ_BODY, "site": OBJ_SITE, "geom": OBJ_GEOM}.get(
        next((k for k in ("body", "site", "geom") if e.get(k)), ""), OBJ_UNKNOWN)
      spec.sensors.append(Sensor(name=e.get("name", ""), type=SENS_MJCF, objtype=objtype, objname=target, tag=e.tag))
  meshdir = comp.get("meshdir", comp.get("assetdir", "")) if comp is not None else ""
  spec.meshdir = meshdir
  for asset in root.findall("asset"):
    for a in asset:
      if a.tag == "mesh":
        at = dfl.attrs("mesh", a.get("class"), a.attrib)
        f = at.get("file")
        name = at.get("name") or (Path(f).stem if f else "")
        if f is not None:
          f = str((asset_dir if asset_dir is not None else Path(".")) / meshdir / f)
        spec.add_mesh(name, vertex=_vec(at["vertex"]) if "vertex" in at else None,
                      face=_vec(at["face"]) if "face" in at else None, file=f, scale=_vec(at.get("scale"), 3, [1, 1, 1]))
      elif a.tag == "hfield":
        if a.get("file") is not None:
          raise NotImplementedError("<hfield file=...> (PNG / custom binary) is not supported: give nrow, ncol and elevation")
        nrow, ncol = int(a.get("nrow")), int(a.get("ncol"))
        elev = _vec(a.get("elevation"), nrow * ncol) if a.get("elevation") is not None else np.zeros(nrow * ncol)
        # MJCF lists the elevation rows top to bottom (image convention); mjModel.hfield_data stores row 0 at -y
        elev = elev.reshape(nrow, ncol)[::-1]
        lo, hi = float(elev.min()), float(elev.max())
        elev = (elev - lo) / (hi - lo) if hi > lo else np.zeros_like(elev)
        spec.add_hfield(a.get("name", ""), _vec(a.get("size"), 4), nrow, ncol, elev)
  wb = root.find("worldbody")
  if wb is not None:
    _parse_body(wb, spec.worldbody, dfl, None, scale)
  con = root.find("contact")
  if con is not None:
    for ex in con:
      if ex.tag != "exclude":
        raise NotImplementedError(f"<contact><{ex.tag}> (explicit contact pairs) is not supported")
      spec.excludes.append((ex.get("body1"), ex.get("body2")))
  act = root.find("actuator")
  if act is not None:
    for ch in act:
      a = dfl.attrs(ch.tag, ch.get("class"), ch.attrib)
      A = Actuator(name=a.get("name", ""), target=a.get("joint", ""))
      if "gear" in a:
        A.gear = _vec(a["gear"])[0]
      if "ctrlrange" in a:
        A.ctrlrange = _vec(a["ctrlrange"], 2)
      if "forcerange" in a:
        A.forcerange = _vec(a["forcerange"], 2)
      if "ctrllimited" in a:
        A.ctrllimited = {"false": 0, "true": 1, "auto": 2}[a["ctrllimited"]]
      if "forcelimited" in a:
        A.forcelimited = {"false": 0, "true": 1, "auto": 2}[a["forcelimited"]]
      if ch.tag == "position":
        kp = float(a.get("kp", 1.0))
        kv = float(a.get("kv", 0.0))
        A.gainprm[0] = kp
        A.biasprm[1] = -kp
        A.biasprm[2] = -kv
      elif ch.tag == "velocity":
        kv = float(a.get("kv", 1.0))
        A.gainprm[0] = kv
        A.biasprm[2] = -kv
      elif ch.tag == "general":
        if "gainprm" in a:
          v = _vec(a["gainprm"])
          A.gainprm[: v.size] = v
        if "biasprm" in a:
          v = _vec(a["biasprm"])
          A.biasprm[: v.size] = v
      elif ch.tag != "motor":
        raise ValueError(f"unsupported actuator <{ch.tag}>")
      spec.actuators.append(A)
  kf = root.find("keyframe")
  if kf is not None:
    for k in kf.findall("key"):
      spec.keys.append(
        Key(
          name=k.get("name", ""),
          qpos=_vec(k.get("qpos")),
          qvel=_vec(k.get("qvel")),
          ctrl=_vec(k.get("ctrl")),
        )
      )
  return spec

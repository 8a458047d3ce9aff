"""Offscreen frames (b2_render, csrc/b2_render.cuh; mjlab_b200/render.py) against an independent fp64 ray caster.

The caster below reads the same geom poses and model values as the kernel (Data geom_xpos / geom_xmat, Model geom_size
/ geom_rgba, the height fields' samples) and applies the shading model of DESIGN.md §4 in fp64.  A pixel whose
reference id (world, geom, the checker square of a plane, whether the point is in shadow) changes among rays offset by
±0.01 pixel is an edge pixel and is not compared, nor is one where two items are entered within the depth tolerance.  The file runs on the host-emulated library (CPU suite, small
images) and on the GPU (`-m gpu`); the env tests need the GPU.
"""

import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from mjlab_b200.render import MAX_ENVS, OffscreenRenderer, ViewerConfig, tracked_body
from mjlab_b200.sim import native

sys.path.insert(0, str(Path(__file__).parent / "emul"))

BACKENDS = [pytest.param("cuda", marks=pytest.mark.gpu), "emul"]
O = ViewerConfig.OriginType
PLANE, HFIELD, SPHERE, CAPSULE, ELLIPSOID, CYLINDER, BOX, MESH = range(8)
LIGHT = np.array([0.36, 0.48, 0.80])
AMBIENT, DIFFUSE, HEAD, CHECKER, CHECKER_DARK, SHADOW_EPS = 0.1, 0.6, 0.3, 0.5, 0.8, 1e-3
BG = np.array([153, 178, 204])

_emul = None


class Sim:
  """What OffscreenRenderer needs of a Simulation, on either backend, with the Data / Model fields as tensors."""

  def __init__(self, backend, model, n):
    self.mj_model, self.num_envs = model, n
    if backend == "emul":
      global _emul
      from engine import host_tensor, load_emul_library

      if _emul is None:
        _emul = load_emul_library()
      self.e, self.device, self._wrap, self.sim = native.Engine(_emul, model, n), "cpu", host_tensor, None
    else:
      from mjlab_b200.sim import Simulation, SimulationCfg
      from mjlab_b200.sim.sim_data import tensor_from_b2

      self.sim = Simulation(n, SimulationCfg(), model, "cuda:0")
      self.e, self.device = self.sim._engine, "cuda:0"
      self._wrap = lambda t: tensor_from_b2(t, self.sim)
    self._lib, self._h = self.e.lib, self.e.h

  def _stream(self):
    return ctypes.c_void_p(0 if self.sim is None else torch.cuda.current_stream().cuda_stream)

  def t(self, name, which=0):
    return self._wrap(self.e.get_field(which, name))

  def a(self, name, which=0):
    return self.t(name, which).cpu().numpy().astype(np.float64)

  def forward(self):
    self.e.check(self._lib.b2_forward(self._h, self._stream()))

  def step(self, k=1):
    self.e.check(self._lib.b2_step_n(self._h, k, self._stream()))


# ---- the fp64 reference ------------------------------------------------------------------------------------------

def camera(cfg, target, w, h):
  az, el = np.radians(cfg.azimuth), np.radians(cfg.elevation)
  f = np.array([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)])
  r = np.array([np.sin(az), -np.cos(az), 0.0])
  u = np.cross(r, f)
  ty = np.tan(np.radians(22.5))
  return np.asarray(target, float) - cfg.distance * f, f, r, u, ty, ty * w / h


def rays(cam, w, h, dx=0.0, dy=0.0):
  eye, f, r, u, ty, tx = cam
  jj, ii = np.meshgrid(np.arange(w) + 0.5 + dx, np.arange(h) + 0.5 + dy)
  a, b = (2 * jj / w - 1) * tx, (1 - 2 * ii / h) * ty
  d = f + a[..., None] * r + b[..., None] * u
  return d / np.linalg.norm(d, axis=-1, keepdims=True)


def items(sim, env_idx, noverlay=MAX_ENVS):
  """(world, geom, pos, mat) of everything drawn: geoms welded to the world from world 0, then the other geoms of
  worlds 0..noverlay-1 and env_idx.  Mesh geoms and alpha-0 geoms are left out."""
  m = sim.mj_model
  parent, dofnum = np.asarray(m.arrays["body_parentid"]), np.asarray(m.arrays["body_dofnum"])
  welded = [True] * len(parent)
  for b in range(1, len(parent)):
    welded[b] = dofnum[b] == 0 and welded[parent[b]]
  gt, gb = np.asarray(m.geom_type), np.asarray(m.geom_bodyid)
  xpos, xmat, rgba = sim.a("geom_xpos"), sim.a("geom_xmat"), sim.a("geom_rgba", 1)
  rgba = np.broadcast_to(rgba, (sim.num_envs,) + rgba.shape[1:])
  worlds = sorted(set(range(min(noverlay, sim.num_envs))) | {env_idx})
  out = []
  for g in range(len(gt)):
    if gt[g] == MESH:
      continue
    for w in ([0] if welded[gb[g]] else worlds):
      if rgba[w, g, 3] != 0:
        out.append((w, g, xpos[w, g], xmat[w, g].reshape(3, 3)))
  return out


def hfield_of(m, g):
  k = int(np.asarray(m.arrays["geom_dataid"])[g])
  size = np.asarray(m.arrays["hfield_size"]).reshape(-1, 4)[k]
  nrow, ncol = int(np.asarray(m.arrays["hfield_nrow"])[k]), int(np.asarray(m.arrays["hfield_ncol"])[k])
  adr = int(np.asarray(m.arrays["hfield_adr"])[k])
  return size, np.asarray(m.arrays["hfield_data"])[adr:adr + nrow * ncol].reshape(nrow, ncol)


def _tris(size, z, cells):
  """Top triangles (t = 0: (r,c) (r,c+1) (r+1,c+1); t = 1: (r,c) (r+1,c+1) (r+1,c)) of the given cells."""
  nrow, ncol = z.shape
  dx, dy = 2 * size[0] / (ncol - 1), 2 * size[1] / (nrow - 1)
  r, c = cells[:, 0], cells[:, 1]
  def v(rr, cc):
    return np.stack([-size[0] + dx * cc, -size[1] + dy * rr, z[rr, cc] * size[2]], -1)
  a, b1, d1, b2 = v(r, c), v(r, c + 1), v(r + 1, c + 1), v(r + 1, c)
  return np.concatenate([np.stack([a, b1, d1], 1), np.stack([a, d1, b2], 1)])


def _hit_tris(o, d, T):
  e1, e2 = T[:, 1] - T[:, 0], T[:, 2] - T[:, 0]
  p = np.cross(d, e2)
  det = np.einsum("ij,ij->i", e1, p)
  with np.errstate(divide="ignore", invalid="ignore"):
    tv = o - T[:, 0]
    u = np.einsum("ij,ij->i", tv, p) / det
    q = np.cross(tv, e1)
    v = q @ d / det
    t = np.einsum("ij,ij->i", e2, q) / det
  ok = (det != 0) & (u >= 0) & (v >= 0) & (u + v <= 1) & (t > 0)
  if not ok.any():
    return np.inf, None
  k = np.argmin(np.where(ok, t, np.inf))
  return t[k], np.cross(e1[k], e2[k])


def hit_hfield(size, z, o, d):
  """Per ray: the cells whose footprint the ray's xy path crosses inside the box (sampled finely, widened by one
  cell), all their triangles tested."""
  nrow, ncol = z.shape
  dx, dy = 2 * size[0] / (ncol - 1), 2 * size[1] / (nrow - 1)
  t = np.full(len(o), np.inf)
  n = np.zeros((len(o), 3))
  for i in range(len(o)):
    lo, hi = 0.0, np.inf
    for k, (a, b) in enumerate(((-size[0], size[0]), (-size[1], size[1]), (0.0, size[2]))):
      if d[i, k] == 0:
        if not a <= o[i, k] <= b:
          lo = np.inf
        continue
      t1, t2 = sorted(((a - o[i, k]) / d[i, k], (b - o[i, k]) / d[i, k]))
      lo, hi = max(lo, t1), min(hi, t2)
    if not lo <= hi:
      continue
    span = np.hypot(*(d[i, :2] * (hi - lo)))
    ts = np.linspace(lo, hi, int(span / (0.25 * min(dx, dy))) + 2)
    p = o[i] + ts[:, None] * d[i]
    c = np.clip(np.floor((p[:, 0] + size[0]) / dx).astype(int), 0, ncol - 2)
    r = np.clip(np.floor((p[:, 1] + size[1]) / dy).astype(int), 0, nrow - 2)
    cells = {(rr + a, cc + b) for rr, cc in zip(r, c) for a in (-1, 0, 1) for b in (-1, 0, 1)}
    cells = np.array([x for x in cells if 0 <= x[0] <= nrow - 2 and 0 <= x[1] <= ncol - 2])
    t[i], nn = _hit_tris(o[i], d[i], _tris(size, z, cells))
    if nn is not None:
      n[i] = nn
  return t, n


def _ball(o, d, cz, r):
  oc = o - np.array([0, 0, cz])
  a = np.einsum("ij,ij->i", d, d)
  tc = -np.einsum("ij,ij->i", oc, d) / a
  q = oc + tc[:, None] * d
  h = r * r - np.einsum("ij,ij->i", q, q)
  with np.errstate(invalid="ignore"):
    return np.where(h >= 0, tc - np.sqrt(np.maximum(h, 0) / a), np.inf)


def hit(m, g, pos, R, o, d):
  """Entry t (> 0) of the rays o + t d into geom g at (pos, R), the world normal there, and the checker parity."""
  t_ = int(np.asarray(m.geom_type)[g])
  s = np.asarray(m.geom_size)[g]
  ol, dl = (o - pos) @ R, d @ R
  nl = np.zeros_like(ol)
  par = np.zeros(len(o), int)
  with np.errstate(divide="ignore", invalid="ignore"):
    if t_ == PLANE:
      t = np.where(dl[:, 2] != 0, -ol[:, 2] / dl[:, 2], np.inf)
      x, y = ol[:, 0] + t * dl[:, 0], ol[:, 1] + t * dl[:, 1]
      if s[0] > 0 and s[1] > 0:
        t = np.where((np.abs(x) <= s[0]) & (np.abs(y) <= s[1]), t, np.inf)
      nl[:, 2] = 1
      par = (np.floor(np.nan_to_num(x) / CHECKER) + np.floor(np.nan_to_num(y) / CHECKER)).astype(np.int64) & 1
    elif t_ == HFIELD:
      size, z = hfield_of(m, g)
      t, nl = hit_hfield(size, z, ol, dl)
    elif t_ == SPHERE:
      t = _ball(ol, dl, 0, s[0])
      nl = ol + t[:, None] * dl
    elif t_ == ELLIPSOID:
      t = _ball(ol / s, dl / s, 0, 1.0)
      nl = (ol + t[:, None] * dl) / s ** 2
    elif t_ == CAPSULE:
      cands = []
      a = dl[:, 0] ** 2 + dl[:, 1] ** 2
      tc = -(ol[:, 0] * dl[:, 0] + ol[:, 1] * dl[:, 1]) / a
      q = ol[:, :2] + tc[:, None] * dl[:, :2]
      h = s[0] ** 2 - (q ** 2).sum(1)
      tt = np.where(h >= 0, tc - np.sqrt(np.maximum(h, 0) / a), np.inf)
      zz = ol[:, 2] + tt * dl[:, 2]
      tt = np.where(np.abs(zz) <= s[1], tt, np.inf)
      cands.append((tt, np.concatenate([ol[:, :2] + tt[:, None] * dl[:, :2], np.zeros((len(o), 1))], 1)))
      for e in (-1, 1):
        tb = _ball(ol, dl, e * s[1], s[0])
        cands.append((tb, ol + tb[:, None] * dl - np.array([0, 0, e * s[1]])))
      t = np.min([c[0] for c in cands], 0)
      k = np.argmin([c[0] for c in cands], 0)
      nl = np.stack([c[1] for c in cands])[k, np.arange(len(o))]
    elif t_ in (CYLINDER, BOX):
      los, his, axes = [], [], []
      if t_ == CYLINDER:
        a = dl[:, 0] ** 2 + dl[:, 1] ** 2
        tc = -(ol[:, 0] * dl[:, 0] + ol[:, 1] * dl[:, 1]) / a
        q = ol[:, :2] + tc[:, None] * dl[:, :2]
        h = s[0] ** 2 - (q ** 2).sum(1)
        dt = np.sqrt(np.maximum(h, 0) / a)
        los.append(np.where(h >= 0, tc - dt, np.inf)); his.append(np.where(h >= 0, tc + dt, -np.inf))
        slabs = [(2, s[1])]
      else:
        slabs = [(k, s[k]) for k in range(3)]
      for k, hk in slabs:
        a1, a2 = (-hk - ol[:, k]) / dl[:, k], (hk - ol[:, k]) / dl[:, k]
        inside = np.abs(ol[:, k]) <= hk
        los.append(np.where(dl[:, k] != 0, np.minimum(a1, a2), np.where(inside, -np.inf, np.inf)))
        his.append(np.where(dl[:, k] != 0, np.maximum(a1, a2), np.where(inside, np.inf, -np.inf)))
      L, H = np.array(los), np.array(his)
      t = L.max(0)
      t = np.where(t <= H.min(0), t, np.inf)
      k = L.argmax(0)
      if t_ == CYLINDER:
        side = k == 0
        nl[side, :2] = ol[side, :2] + t[side, None] * dl[side, :2]
        nl[~side, 2] = -np.sign(dl[~side, 2])
      else:
        nl[np.arange(len(o)), k] = -np.sign(dl[np.arange(len(o)), k])
  t = np.where(np.isfinite(t) & (t > 0), t, np.inf)
  return t, np.nan_to_num(nl, posinf=0.0, neginf=0.0) @ R.T, par


def reference(sim, cfg, target, w, h, dx=0.0, dy=0.0):
  """fp64 frame: rgb (float, before rounding), depth, seg and the shading id (seg, checker parity, shadow)."""
  m = sim.mj_model
  cam = camera(cfg, target, w, h)
  d = rays(cam, w, h, dx, dy).reshape(-1, 3)
  o = np.broadcast_to(cam[0], d.shape)
  it = items(sim, cfg.env_idx)
  rgba = np.broadcast_to(sim.a("geom_rgba", 1), (sim.num_envs, int(m.ngeom), 4))
  best, who, n, par = np.full(len(d), np.inf), np.full(len(d), -1), np.zeros_like(d), np.zeros(len(d), int)
  second = np.full(len(d), np.inf)  # the entry of the next-nearest item
  for k, (wd, g, pos, R) in enumerate(it):
    t, nn, pp = hit(m, g, pos, R, o, d)
    b = t < best
    second = np.where(b, best, np.minimum(second, t))
    best[b], who[b], n[b], par[b] = t[b], k, nn[b], pp[b]
  hitm = who >= 0
  n /= np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-300)
  n *= np.where(np.einsum("ij,ij->i", n, d) > 0, -1.0, 1.0)[:, None]
  diff = np.maximum(0.0, n @ LIGHT)
  shadow = np.zeros(len(d), bool)
  if cfg.enable_shadows:
    lit = hitm & (diff > 0)
    p = o[lit] + best[lit, None] * d[lit] + SHADOW_EPS * n[lit]
    L = np.broadcast_to(LIGHT, p.shape)
    sh = np.zeros(len(p), bool)
    for (wd, g, pos, R) in it:
      sh |= np.isfinite(hit(m, g, pos, R, p, L)[0])
    shadow[lit] = sh
  diff = np.where(shadow, 0.0, diff)
  light = AMBIENT + DIFFUSE * diff + HEAD * np.maximum(0.0, -np.einsum("ij,ij->i", n, d))
  seg = np.array([(it[k][0], it[k][1]) if k >= 0 else (-1, -1) for k in who])
  gt = np.asarray(m.geom_type)
  plane = np.array([k >= 0 and gt[it[k][1]] == PLANE for k in who])
  light = np.where(plane & (par == 1), light * CHECKER_DARK, light)
  col = np.array([rgba[it[k][0], it[k][1], :3] if k >= 0 else np.zeros(3) for k in who])
  rgb = np.where(hitm[:, None], np.clip(col * light[:, None], 0, 1) * 255, BG)
  depth = np.where(hitm, best * (d @ cam[1]), np.inf)
  sid = np.stack([seg[:, 0], seg[:, 1], np.where(plane, par, 0), shadow], 1)
  tie = hitm & (second - best <= 1e-4 * best)
  return rgb.reshape(h, w, 3), depth.reshape(h, w), seg.reshape(h, w, 2), sid.reshape(h, w, 4), tie.reshape(h, w)


def edge_mask(sim, cfg, target, w, h, sid):
  edge = np.zeros((h, w), bool)
  for dx, dy in ((0.01, 0), (-0.01, 0), (0, 0.01), (0, -0.01)):
    edge |= (reference(sim, cfg, target, w, h, dx, dy)[3] != sid).any(-1)
  return edge


def target_of(sim, cfg):
  b = tracked_body(sim.mj_model, cfg)
  return cfg.lookat if b < 0 else sim.a("subtree_com")[cfg.env_idx, b]


def compare(sim, cfg, min_geoms=3):
  r = OffscreenRenderer(sim, cfg, extra_outputs=True)
  r.update()
  rgb, depth, seg = r.render(), r.depth(), r.segmentation()
  target = target_of(sim, cfg)
  rgb_ref, depth_ref, seg_ref, sid, tie = reference(sim, cfg, target, cfg.width, cfg.height)
  # (a tie: two items entered within the depth tolerance, e.g. overlapping capsules of one leg; either id is right)
  edge = edge_mask(sim, cfg, target, cfg.width, cfg.height, sid) | tie
  ok = ~edge
  assert ok.mean() > 0.7, ok.mean()
  assert len({tuple(x) for x in seg_ref[ok].tolist()}) >= min_geoms  # the view is not empty
  bad = (seg != seg_ref).any(-1) & ok
  assert not bad.any(), (np.argwhere(bad)[:5], seg[bad][:5], seg_ref[bad][:5])
  fin = ok & np.isfinite(depth_ref)
  assert np.array_equal(np.isinf(depth[ok]), np.isinf(depth_ref[ok]))
  rel = np.abs(depth[fin] - depth_ref[fin]) / depth_ref[fin]
  assert rel.max() < 1e-4, rel.max()
  diff = np.abs(rgb.astype(int) - np.round(rgb_ref).astype(int))[ok]
  assert diff.max() <= 2, diff.max()
  return rgb, seg


# ---- scenes ------------------------------------------------------------------------------------------------------

def synthetic_scene(rng):
  """A finite plane, a random 8 x 6 height field, a welded box, and free bodies with every drawable primitive (and a
  mesh and an alpha-0 sphere, which are not drawn)."""
  from mjlab_b200.compiler.spec import Spec

  spec = Spec()
  spec.add_mesh("poly", vertex=rng.normal(size=(12, 3)) * 0.1)
  spec.add_hfield("bumps", size=[1.0, 0.8, 0.3, 0.1], nrow=6, ncol=8, userdata=rng.uniform(0, 1, (6, 8)))
  wb = spec.worldbody
  wb.add_geom(name="floor", type="plane", size=[3.0, 2.5, 0.05], rgba=[0.6, 0.6, 0.6, 1])
  wb.add_geom(name="terrain", type="hfield", hfieldname="bumps", pos=[0.8, 1.0, 0.0], rgba=[0.4, 0.7, 0.3, 1])
  wb.add_geom(name="block", type="box", size=[0.2, 0.3, 0.25], pos=[-1.0, 0.5, 0.25], quat=[0.9, 0, 0, 0.44],
              rgba=[0.8, 0.3, 0.3, 1])
  shapes = [("sphere", [0.18]), ("capsule", [0.1, 0.2]), ("ellipsoid", [0.25, 0.15, 0.1]), ("cylinder", [0.15, 0.2]),
            ("box", [0.2, 0.12, 0.1]), ("mesh", None), ("sphere", [0.3])]
  for k, (t, size) in enumerate(shapes):
    b = wb.add_body(name=f"b{k}", pos=[0, 0, 1])
    b.add_freejoint(name=f"j{k}")
    kw = dict(meshname="poly") if t == "mesh" else dict(size=size)
    alpha = 0.0 if k == len(shapes) - 1 else rng.uniform(0.2, 1.0)
    b.add_geom(name=f"g{k}", type=t, rgba=[*rng.uniform(0.2, 1.0, 3), alpha], **kw)
  return spec.compile()


def pose_free_bodies(sim, rng, spread=1.2):
  q = sim.t("qpos")
  n, nq = q.shape[0], q.shape[1]
  qp = np.zeros((n, nq), np.float32)
  for k in range(nq // 7):
    qp[:, 7 * k:7 * k + 3] = rng.uniform([-spread, -spread, 0.1], [spread, spread, 0.8], (n, 3))
    qq = rng.normal(size=(n, 4))
    qp[:, 7 * k + 3:7 * k + 7] = qq / np.linalg.norm(qq, axis=1, keepdims=True)
  q[...] = torch.as_tensor(qp, device=q.device)
  sim.forward()


def rollout(sim, model, steps, seed):
  """Random controls around the init keyframe, `steps` sub-steps."""
  rng = np.random.default_rng(seed)
  key = model.keys["robot/init_state"]
  sim.t("qpos")[...] = torch.as_tensor(np.tile(key["qpos"], (sim.num_envs, 1)), dtype=torch.float32, device=sim.device)
  sim.forward()
  for _ in range(steps):
    ctrl = np.tile(key["ctrl"], (sim.num_envs, 1)) + rng.uniform(-0.3, 0.3, (sim.num_envs, int(model.nu)))
    sim.t("ctrl")[...] = torch.as_tensor(ctrl, dtype=torch.float32, device=sim.device)
    sim.step()


def size(backend, w, h):
  return (w, h) if backend == "emul" else (4 * w, 4 * h)


# ---- 1. geometry against fp64 ------------------------------------------------------------------------------------

@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("shadows", [True, False])
def test_synthetic_scene(backend, shadows):
  rng = np.random.default_rng(5)
  m = synthetic_scene(rng)
  sim = Sim(backend, m, 3)
  pose_free_bodies(sim, rng)
  w, h = size(backend, 48, 36)
  cfg = ViewerConfig(lookat=(0.0, 0.3, 0.3), distance=4.0, elevation=-35.0, azimuth=60.0, env_idx=2, width=w,
                     height=h, enable_shadows=shadows)
  _, seg = compare(sim, cfg, min_geoms=8)
  drawn = {int(g) for g in np.unique(seg[..., 1])}
  names = m.names["geom"]
  assert names.index("g5") not in drawn and names.index("g6") not in drawn  # the mesh and the alpha-0 sphere


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("name,body,distance,elevation", [("g1_flat", "torso_link", 3.0, -20.0),
                                                           ("go1_rough_hf", "trunk", 2.5, -30.0)])
def test_shipped_scenes(backend, name, body, distance, elevation):
  from mjlab_b200.asset_zoo import load_compiled

  m = load_compiled(name)
  sim = Sim(backend, m, 2)
  rollout(sim, m, 20, seed=3)
  w, h = size(backend, 40, 30)
  cfg = ViewerConfig(origin_type=O.ASSET_BODY, asset_name="robot", body_name=body, distance=distance,
                     elevation=elevation, azimuth=130.0, env_idx=1, width=w, height=h)
  compare(sim, cfg)


# ---- 2. camera ---------------------------------------------------------------------------------------------------

def marker_scene():
  from mjlab_b200.compiler.spec import Spec

  spec = Spec()
  for name in ("robot/base", "offset"):
    b = spec.worldbody.add_body(name=name, pos=[0, 0, 1])
    b.add_freejoint(name=name + "_j")
    b.add_geom(name=name + "_g", type="sphere", size=[0.2])
  return spec.compile()


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("origin", [O.WORLD, O.ASSET_ROOT, O.ASSET_BODY])
def test_camera(backend, origin):
  m = marker_scene()
  sim = Sim(backend, m, 2)
  target = np.array([0.7, -0.4, 1.3])
  cfg = ViewerConfig(lookat=tuple(target) if origin == O.WORLD else (5.0, 5.0, 5.0), origin_type=origin,
                     asset_name="robot" if origin == O.ASSET_BODY else None,
                     body_name="base" if origin == O.ASSET_BODY else None, distance=6.0, elevation=-25.0,
                     azimuth=35.0, env_idx=1, width=96, height=72, enable_shadows=False)
  eye, f, r, u, ty, tx = camera(cfg, target, cfg.width, cfg.height)
  off = target + 0.9 * r - 0.6 * u + 0.5 * f
  qp = np.zeros((2, 14), np.float32)
  qp[:, 3] = qp[:, 10] = 1
  qp[1, 0:3], qp[1, 7:10] = target, off  # the tracked body of world 1 at the target
  qp[0, 0:3], qp[0, 7:10] = [50, 50, 50], [60, 60, 60]  # world 0's markers out of view
  sim.t("qpos")[...] = torch.as_tensor(qp, device=sim.device)
  sim.forward()
  assert np.allclose(target_of(sim, cfg), target, atol=1e-5)
  r_ = OffscreenRenderer(sim, cfg, extra_outputs=True)
  r_.update()
  seg = r_.segmentation()
  for g, p in ((0, target), (1, off)):
    ii, jj = np.nonzero((seg[..., 0] == 1) & (seg[..., 1] == g))
    assert len(ii) > 20
    v = p - eye
    x = (v @ r / (v @ f) / tx + 1) * cfg.width / 2 - 0.5
    y = (1 - v @ u / (v @ f) / ty) * cfg.height / 2 - 0.5
    assert abs(jj.mean() - x) < 0.5 and abs(ii.mean() - y) < 0.5, (g, jj.mean(), x, ii.mean(), y)
  assert abs(np.nonzero(seg[..., 1] == 0)[1].mean() - (cfg.width - 1) / 2) < 0.5


# ---- 3. overlay set ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("backend", BACKENDS)
def test_overlay_worlds(backend):
  from mjlab_b200.compiler.spec import Spec

  spec = Spec()
  b = spec.worldbody.add_body(name="ball", pos=[0, 0, 0])
  b.add_freejoint(name="ball_j")
  b.add_geom(name="ball_g", type="sphere", size=[0.3], rgba=[0.5, 0.5, 0.5, 1])
  m = spec.compile()
  n, env_idx = MAX_ENVS + 2, MAX_ENVS + 1
  sim = Sim(backend, m, n)
  qp = np.zeros((n, 7), np.float32)
  qp[:, 3] = 1
  qp[:, 0], qp[:, 1] = np.arange(n) % 6 - 2.5, np.arange(n) // 6 - 2.5
  sim.t("qpos")[...] = torch.as_tensor(qp, device=sim.device)
  sim.forward()
  cfg = ViewerConfig(lookat=(0, 0, 0), distance=16.0, elevation=-90.0, azimuth=90.0, env_idx=env_idx, width=64,
                     height=64, enable_shadows=False)
  r = OffscreenRenderer(sim, cfg, extra_outputs=True)
  r.update()
  rgb0, seg = r.render(), r.segmentation()
  assert set(np.unique(seg[..., 0]).tolist()) == set(range(MAX_ENVS)) | {env_idx, -1}
  sim.e.check(sim._lib.b2_expand_model_field(sim._h, b"geom_rgba", sim._stream(), None))
  sim.t("geom_rgba", 1)[5, 0] = torch.tensor([1.0, 0.0, 0.0, 1.0], device=sim.device)
  r.update()
  changed = (r.render() != rgb0).any(-1)
  assert changed.any() and np.array_equal(changed, seg[..., 0] == 5)


# ---- refusals ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("backend", BACKENDS)
def test_refusals(backend):
  m = marker_scene()
  sim = Sim(backend, m, 2)
  for kw in (dict(width=0), dict(height=4097), dict(env_idx=2), dict(env_idx=-1)):
    with pytest.raises(ValueError):
      OffscreenRenderer(sim, ViewerConfig(**kw))
  with pytest.raises(ValueError, match="asset_name/body_name required"):
    OffscreenRenderer(sim, ViewerConfig(origin_type=O.ASSET_BODY, asset_name="robot"))
  with pytest.raises(ValueError, match="Body 'hand' not found in asset 'robot'"):
    OffscreenRenderer(sim, ViewerConfig(origin_type=O.ASSET_BODY, asset_name="robot", body_name="hand"))
  with pytest.raises(KeyError):
    OffscreenRenderer(sim, ViewerConfig(origin_type=O.ASSET_ROOT, asset_name="arm"))
  # the library's own checks
  r = OffscreenRenderer(sim, ViewerConfig(width=8, height=8))
  for field, value in (("width", 5000), ("env_idx", 7), ("track_body", 99), ("rgb", None)):
    old = getattr(r._args, field)
    setattr(r._args, field, value)
    with pytest.raises(RuntimeError):
      r.update()
    setattr(r._args, field, old)
  r.update()


# ---- 4-5. environments (GPU) -------------------------------------------------------------------------------------

def _env(kind, render_mode, n=64):
  from mjlab_b200.envs import TrackingFlatEnv, VelocityFlatEnv, tracking_task_cfg, velocity_task_cfg

  if kind == "velocity":
    return VelocityFlatEnv(velocity_task_cfg("Mjlab-Velocity-Flat-Unitree-G1", num_envs=n), render_mode=render_mode)
  return TrackingFlatEnv(tracking_task_cfg("Mjlab-Tracking-Flat-Unitree-G1", num_envs=n), render_mode=render_mode)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["velocity", "tracking"])
def test_render_is_read_only(kind):
  outs = []
  for mode in ("rgb_array", None):
    env = _env(kind, mode)
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for _ in range(50):
      obs, rew, term, trunc, _ = env.step(torch.randn(env.num_envs, env.nu, device="cuda", generator=g) * 0.5)
      frame = env.render()
      assert (frame is None) == (mode is None)
      if frame is not None:
        assert frame.shape == (240, 320, 3) and frame.dtype == np.uint8
      d = env.sim.data
      rows.append([t.clone().cpu() for t in (d.qpos, d.qvel, obs, rew, term, trunc)])
    if mode is None:
      assert env._offline_renderer is None
      before = env.sim.launch_count()
      env.step(torch.zeros(env.num_envs, env.nu, device="cuda"))
      per_step = env.sim.launch_count() - before
    else:
      before = env.sim.launch_count()
      env.step(torch.zeros(env.num_envs, env.nu, device="cuda"))
      per_step_r = env.sim.launch_count() - before
    assert env.metadata["render_fps"] == pytest.approx(1.0 / env.step_dt)
    env.close()
    outs.append(rows)
  assert per_step == per_step_r  # a step launches nothing for rendering
  for a, b in zip(*outs):
    for x, y in zip(a, b):
      assert torch.equal(x, y)


def test_task_presets():
  from mjlab_b200.envs import tracking_task_cfg, velocity_task_cfg

  base = dict(origin_type=O.ASSET_BODY, asset_name="robot", azimuth=90.0, lookat=(0.0, 0.0, 0.0), height=240,
              width=320, env_idx=0, enable_shadows=True, enable_reflections=True)
  want = {"Mjlab-Velocity-Flat-Unitree-G1": dict(body_name="torso_link", distance=3.0, elevation=-5.0),
          "Mjlab-Velocity-Flat-Unitree-Go1": dict(body_name="trunk", distance=1.5, elevation=-10.0),
          "Mjlab-Velocity-Rough-Unitree-Go1": dict(body_name="trunk", distance=1.5, elevation=-10.0),
          "Mjlab-Tracking-Flat-Unitree-G1": dict(body_name="torso_link", distance=3.0, elevation=-5.0)}
  for name, w in want.items():
    cfg = (velocity_task_cfg if "Velocity" in name else tracking_task_cfg)(name).viewer
    assert cfg == ViewerConfig(**base, **w), name
  from mjlab_b200.envs import VelocityFlatEnv

  with pytest.raises(ValueError, match=r"Render mode human is not supported. Please use: \[None, 'rgb_array'\]."):
    VelocityFlatEnv(velocity_task_cfg("Mjlab-Velocity-Flat-Unitree-G1"), render_mode="human")


@pytest.mark.gpu
@pytest.mark.parametrize("task", ["Mjlab-Velocity-Flat-Unitree-G1", "Mjlab-Velocity-Flat-Unitree-Go1",
                                  "Mjlab-Velocity-Rough-Unitree-Go1", "Mjlab-Tracking-Flat-Unitree-G1"])
def test_preset_frames_show_the_robot(task):
  from mjlab_b200.envs import TrackingFlatEnv, VelocityFlatEnv, tracking_task_cfg, velocity_task_cfg

  velocity = "Velocity" in task
  cfg = (velocity_task_cfg if velocity else tracking_task_cfg)(task, num_envs=48)
  cfg.viewer.env_idx = 40
  env = (VelocityFlatEnv if velocity else TrackingFlatEnv)(cfg, render_mode="rgb_array")
  env.step(torch.zeros(env.num_envs, env.nu, device="cuda"))
  frame = env.render()
  assert frame.shape == (240, 320, 3)
  r = OffscreenRenderer(env.sim, cfg.viewer, extra_outputs=True)
  r.update()
  block = r.segmentation()[112:128, 152:168].reshape(-1, 2)
  robot = {i for i, n in enumerate(env.model.names["geom"]) if n.startswith("robot/")}
  assert any(w == 40 and g in robot for w, g in block.tolist())
  env.close()

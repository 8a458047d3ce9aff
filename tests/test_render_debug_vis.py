"""Debug visualisation in offscreen frames (csrc/b2_render.cuh's decoration items, mjlab_b200/render.py's
DebugVisualizer, the envs' update_visualizers) against an fp64 reproduction of DESIGN.md §4.4.

The scene part reuses tests/test_render.py's fp64 ray caster; on top of it, the nearest arrow (cylinder shaft, cone
head) or ghost geom entered before the opaque hit is shaded without shadows and blended, byte =
floor(255 (a c_d + (1 - a) c_o) + 1/2).  Pixels whose scene or decoration id (item, and the arrow part) changes among
rays offset by ±0.01 pixel are edge pixels and are not compared.  Kernel tests run on the host-emulated library and on
the GPU (`-m gpu`); the env tests need the GPU.
"""

import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

sys.path.insert(0, str(Path(__file__).parent))
sys.path.insert(0, str(Path(__file__).parents[1] / "tools"))

from test_render import (AMBIENT, BACKENDS, DIFFUSE, HEAD, LIGHT, MESH, Sim, camera, edge_mask, hit,  # noqa: E402
                         pose_free_bodies, rays, reference, synthetic_scene)

from mjlab_b200.render import OffscreenRenderer, ViewerConfig, _engine_tensor  # noqa: E402
from mjlab_b200.sim import native  # noqa: E402


def size(backend, w, h):
  return (w, h) if backend == "emul" else (4 * w, 4 * h)


# ---- the fp64 reference ------------------------------------------------------------------------------------------

def arrow_hit(rec, o, d):
  """Entry t (> 0) of the rays into the arrow record, the world normal there and the part hit (1 shaft side, 2 shaft
  cap, 3 cone side, 4 cone base)."""
  rec = np.asarray(rec, float)
  a, b, w, alpha = rec[:3], rec[3:6], rec[6], rec[10]
  n = len(o)
  t, nrm, part = np.full(n, np.inf), np.zeros((n, 3)), np.zeros(n, int)
  L = np.linalg.norm(b - a)
  if L < 1e-6 or alpha == 0:
    return t, nrm, part
  ez = (b - a) / L
  h = min(L / 2, 4 * w)
  ex = np.cross(ez, [0.0, 0.0, 1.0] if abs(ez[2]) < 0.9 else [1.0, 0.0, 0.0])
  ex /= np.linalg.norm(ex)
  R = np.stack([ex, np.cross(ez, ex), ez], 1)  # columns: the arrow's axes
  ol, dl = (o - a) @ R, d @ R

  def slab(z0, z1):
    with np.errstate(divide="ignore", invalid="ignore"):
      p, q = (z0 - ol[:, 2]) / dl[:, 2], (z1 - ol[:, 2]) / dl[:, 2]
    inside = (ol[:, 2] >= z0) & (ol[:, 2] <= z1)
    flat = dl[:, 2] == 0
    lo = np.where(flat, np.where(inside, -np.inf, np.inf), np.minimum(p, q))
    hi = np.where(flat, np.where(inside, np.inf, -np.inf), np.maximum(p, q))
    return lo, hi

  with np.errstate(divide="ignore", invalid="ignore"):
    # shaft
    A = dl[:, 0] ** 2 + dl[:, 1] ** 2
    tc = -(ol[:, 0] * dl[:, 0] + ol[:, 1] * dl[:, 1]) / A
    q2 = (ol[:, 0] + tc * dl[:, 0]) ** 2 + (ol[:, 1] + tc * dl[:, 1]) ** 2
    disc = w * w - q2
    lo = np.where(disc >= 0, tc - np.sqrt(np.maximum(disc, 0) / A), np.inf)
    hi = np.where(disc >= 0, tc + np.sqrt(np.maximum(disc, 0) / A), -np.inf)
    zl, zh = slab(0.0, L - h)
    e = np.maximum(lo, zl)
    ok = (e <= np.minimum(hi, zh)) & (e > 0)
    t = np.where(ok, e, np.inf)
    side = lo >= zl
    part = np.where(ok, np.where(side, 1, 2), 0)
    p = ol + t[:, None] * dl
    nl = np.where(side[:, None], p * [1, 1, 0], np.stack([0 * A, 0 * A, -np.sign(dl[:, 2])], 1))
    # head: cone x^2 + y^2 = k^2 (z - L)^2 on z <= L, clipped to z >= L - h
    k2 = (2 * w / h) ** 2
    qz = ol[:, 2] - L
    A = dl[:, 0] ** 2 + dl[:, 1] ** 2 - k2 * dl[:, 2] ** 2
    B = ol[:, 0] * dl[:, 0] + ol[:, 1] * dl[:, 1] - k2 * qz * dl[:, 2]
    C = ol[:, 0] ** 2 + ol[:, 1] ** 2 - k2 * qz ** 2
    disc = B * B - A * C
    sq = np.sqrt(np.maximum(disc, 0))
    r1, r2 = np.minimum((-B - sq) / A, (-B + sq) / A), np.maximum((-B - sq) / A, (-B + sq) / A)
    real = disc >= 0
    v1, v2 = real & (qz + r1 * dl[:, 2] <= 0), real & (qz + r2 * dl[:, 2] <= 0)
    one = np.where(v1, r1, r2)
    down = dl[:, 2] < 0
    clo = np.where(v1 & v2, r1, np.where(v1 | v2, np.where(down, one, -np.inf), np.inf))
    chi = np.where(v1 & v2, r2, np.where(v1 | v2, np.where(down, np.inf, one), -np.inf))
    zl, zh = slab(L - h, L)
    e = np.maximum(clo, zl)
    ok = (e <= np.minimum(chi, zh)) & (e > 0) & (e < t)
    t = np.where(ok, e, t)
    cside = clo >= zl
    part = np.where(ok, np.where(cside, 3, 4), part)
    p = ol + e[:, None] * dl
    cn = np.where(cside[:, None], np.stack([p[:, 0], p[:, 1], -k2 * (p[:, 2] - L)], 1),
                  np.stack([0 * A, 0 * A, -np.sign(dl[:, 2])], 1))
    nl = np.where(ok[:, None], cn, nl)
  return t, np.nan_to_num(nl) @ R.T, part


def ghost_items(sim, xpos, xmat):
  """(geom, pos, R) of the ghost: every non-mesh geom of a body not welded to the world, in geom order."""
  m = sim.mj_model
  parent, dofnum = np.asarray(m.arrays["body_parentid"]), np.asarray(m.arrays["body_dofnum"])
  welded = [True] * len(parent)
  for b in range(1, len(parent)):
    welded[b] = dofnum[b] == 0 and welded[parent[b]]
  gt, gb = np.asarray(m.geom_type), np.asarray(m.geom_bodyid)
  return [(g, xpos[g], xmat[g].reshape(3, 3)) for g in range(len(gt)) if gt[g] != MESH and not welded[gb[g]]]


def decorated(sim, cfg, target, w, h, arrows=(), ghost=None, ghost_rgba=None, dx=0.0, dy=0.0):
  """fp64 frame with decoration: rgb (float before rounding), the scene's sid and tie mask, the decoration id (item,
  part; -1 none)."""
  rgb, depth, seg, sid, tie = reference(sim, cfg, target, w, h, dx, dy)
  cam = camera(cfg, target, w, h)
  d = rays(cam, w, h, dx, dy).reshape(-1, 3)
  o = np.broadcast_to(cam[0], d.shape)
  best = (depth.reshape(-1) / (d @ cam[1])).copy()
  who, part, n = np.full(len(d), -1), np.zeros(len(d), int), np.zeros_like(d)
  cols = []
  k = 0
  for g, pos, R in (ghost or []):
    t, nn, _ = hit(sim.mj_model, g, pos, R, o, d)
    b = t < best
    best[b], who[b], part[b], n[b] = t[b], k, 0, nn[b]
    cols.append(ghost_rgba)
    k += 1
  for rec in arrows:
    t, nn, pp = arrow_hit(rec, o, d)
    b = t < best
    best[b], who[b], part[b], n[b] = t[b], k, pp[b], nn[b]
    cols.append(rec[7:11])
    k += 1
  n /= np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-300)
  n *= np.where(np.einsum("ij,ij->i", n, d) > 0, -1.0, 1.0)[:, None]
  light = AMBIENT + DIFFUSE * np.maximum(0.0, n @ LIGHT) + HEAD * np.maximum(0.0, -np.einsum("ij,ij->i", n, d))
  col = np.array([cols[i] if i >= 0 else (0, 0, 0, 0) for i in who], float).reshape(-1, 4)
  cd = np.clip(col[:, :3] * light[:, None], 0, 1)
  co = rgb.reshape(-1, 3) / 255
  blend = np.floor(255 * (col[:, 3:] * cd + (1 - col[:, 3:]) * co) + 0.5)
  out = np.where(who[:, None] >= 0, blend, rgb.reshape(-1, 3))
  did = np.stack([who, part], 1)
  return out.reshape(h, w, 3), sid, tie, did.reshape(h, w, 2)


def compare_decorated(sim, cfg, target, rgb, arrows=(), ghost=None, ghost_rgba=None, min_deco=50):
  w, h = cfg.width, cfg.height
  ref, sid, tie, did = decorated(sim, cfg, target, w, h, arrows, ghost, ghost_rgba)
  edge = edge_mask(sim, cfg, target, w, h, sid) | tie
  for dx, dy in ((0.01, 0), (-0.01, 0), (0, 0.01), (0, -0.01)):
    edge |= (decorated(sim, cfg, target, w, h, arrows, ghost, ghost_rgba, dx, dy)[3] != did).any(-1)
  ok = ~edge
  covered = ok & (did[..., 0] >= 0)
  assert covered.sum() >= min_deco, covered.sum()
  diff = np.abs(rgb.astype(int) - np.round(ref).astype(int))[ok]
  assert diff.max() <= 2, (diff.max(), np.argwhere((np.abs(rgb.astype(int) - np.round(ref).astype(int)).max(-1) > 2) & ok)[:5])
  return did, edge


def launch(r):
  """b2_render with the renderer's arguments as they stand (no reset of the decoration fields)."""
  s = r._sim
  if s._lib.b2_render(s._h, ctypes.byref(r._args), s._stream()) != 0:
    raise RuntimeError(s._lib.b2_last_error().decode())


def outputs(r):
  return r.render(), r.depth(), r.segmentation()


# ---- scenes ------------------------------------------------------------------------------------------------------

# (from, to, width, rgba): long and short shafts, one shorter than 4w (head = L/2), a vertical one, one of length 0 and
# one with alpha 0 (neither drawn)
ARROWS = [((-1.2, -0.6, 0.9), (0.4, -0.2, 1.1), 0.05, (0.9, 0.2, 0.2, 0.6)),
          ((0.3, 0.8, 0.3), (0.3, 0.8, 1.3), 0.06, (0.2, 0.3, 0.9, 0.8)),
          ((-0.3, 0.2, 1.4), (-0.18, 0.32, 1.42), 0.05, (0.1, 0.9, 0.3, 0.5)),
          ((0.9, -0.8, 0.4), (0.2, 0.1, 0.2), 0.03, (1.0, 1.0, 0.2, 1.0)),
          ((0.0, 0.0, 1.0), (0.0, 0.0, 1.0), 0.05, (0.5, 0.5, 0.5, 0.7)),
          ((-1.0, 1.0, 0.5), (0.0, 1.2, 0.5), 0.05, (0.5, 0.5, 0.5, 0.0))]


def records(arrows):
  return [np.array([*a, *b, w, *c, 0.0]) for a, b, w, c in arrows]


def arrows_cb(arrows):
  def cb(vis):
    for a, b, w, c in arrows:
      vis.add_arrow(a, b, c, width=w)
  return cb


def synthetic(backend, shadows, n=3):
  rng = np.random.default_rng(5)
  m = synthetic_scene(rng)
  sim = Sim(backend, m, n)
  pose_free_bodies(sim, rng)
  w, h = size(backend, 48, 36)
  cfg = ViewerConfig(lookat=(0.0, 0.3, 0.3), distance=4.0, elevation=-35.0, azimuth=60.0, env_idx=2, width=w,
                     height=h, enable_shadows=shadows)
  return sim, cfg


# ---- 1. arrows against fp64 --------------------------------------------------------------------------------------

@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("shadows", [True, False])
def test_arrows(backend, shadows):
  sim, cfg = synthetic(backend, shadows)
  r = OffscreenRenderer(sim, cfg, extra_outputs=True)
  r.update(debug_vis_callback=arrows_cb(ARROWS))
  assert r._args.ndecor == len(ARROWS)
  rgb = r.render()
  did, _ = compare_decorated(sim, cfg, np.array(cfg.lookat), rgb, records(ARROWS))
  seen = {int(k) for k in np.unique(did[..., 0]) if k >= 0}
  assert seen == {0, 1, 2, 3}  # every drawn arrow shows; the zero-length and alpha-0 ones do not
  parts = {int(p) for p in np.unique(did[..., 1])}
  assert {1, 3} <= parts


# ---- 2. ghost against fp64 ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("backend", BACKENDS)
def test_ghost(backend):
  sim, cfg = synthetic(backend, True)
  rng = np.random.default_rng(11)
  nq = int(sim.mj_model.nq)
  q = np.zeros(nq, np.float32)
  for k in range(nq // 7):
    q[7 * k:7 * k + 3] = rng.uniform([-1, -1, 0.3], [1, 1, 1.0])
    qq = rng.normal(size=4)
    q[7 * k + 3:7 * k + 7] = qq / np.linalg.norm(qq)
  color = (0.9, 0.4, 0.8, 0.5)
  r = OffscreenRenderer(sim, cfg, extra_outputs=True)
  qt = torch.as_tensor(q, device=sim.device)
  r.update(debug_vis_callback=lambda vis: vis.add_ghost_mesh(qt, color))
  rgb = r.render()
  dev = torch.device(sim.device)
  gx = _engine_tensor(r._ghost, "geom_xpos", dev)[0].cpu().numpy().astype(np.float64)
  gm = _engine_tensor(r._ghost, "geom_xmat", dev)[0].cpu().numpy().astype(np.float64)
  # the ghost's poses are the engine's own forward kinematics: those of a main world forwarded at the same qpos
  qpos = sim.t("qpos")
  old = qpos.clone()
  qpos[0] = qt
  sim.forward()
  assert np.allclose(gx, sim.a("geom_xpos")[0], atol=2e-5)
  assert np.allclose(gm, sim.a("geom_xmat")[0], atol=2e-5)
  qpos[...] = old
  sim.forward()
  did, _ = compare_decorated(sim, cfg, np.array(cfg.lookat), rgb, ghost=ghost_items(sim, gx, gm), ghost_rgba=color)
  assert len({int(k) for k in np.unique(did[..., 0]) if k >= 0}) >= 3


# ---- 3. invariance -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("backend", BACKENDS)
def test_invariance(backend):
  sim, cfg = synthetic(backend, True)
  r = OffscreenRenderer(sim, cfg, extra_outputs=True)
  # the renderer without decoration launches b2_render with the decoration fields zeroed
  r.update()
  a = r._args
  assert (a.decor, a.ndecor, a.ghost_xpos, a.ghost_xmat, list(a.ghost_rgba)) == (None, 0, None, None, [0.0] * 4)
  plain = outputs(r)
  for cb in (None, lambda vis: None):
    r.update(debug_vis_callback=cb)
    for x, y in zip(plain, outputs(r)):
      assert np.array_equal(x, y)
  # with decoration: depth and seg unchanged; every pixel no decoration item reaches is byte-equal
  q = sim.t("qpos")[1].clone()
  q[0:3] += torch.tensor([0.3, -0.2, 0.1], device=q.device)
  cb = arrows_cb(ARROWS)

  def both(vis):
    cb(vis)
    vis.add_ghost_mesh(q, (0.5, 0.7, 0.5, 0.5))

  r.update(debug_vis_callback=both)
  rgb, depth, seg = outputs(r)
  assert np.array_equal(depth, plain[1]) and np.array_equal(seg, plain[2])
  dev = torch.device(sim.device)
  gx = _engine_tensor(r._ghost, "geom_xpos", dev)[0].cpu().numpy().astype(np.float64)
  gm = _engine_tensor(r._ghost, "geom_xmat", dev)[0].cpu().numpy().astype(np.float64)
  target = np.array(cfg.lookat)
  reach = np.zeros((cfg.height, cfg.width), bool)
  for dx, dy in ((0, 0), (0.01, 0), (-0.01, 0), (0, 0.01), (0, -0.01)):
    did = decorated(sim, cfg, target, cfg.width, cfg.height, records(ARROWS), ghost_items(sim, gx, gm),
                    (0.5, 0.7, 0.5, 0.5), dx, dy)[3]
    reach |= did[..., 0] >= 0
  assert reach.any() and (~reach).sum() > 0.3 * reach.size
  assert np.array_equal(rgb[~reach], plain[0][~reach])
  assert (rgb[reach] != plain[0][reach]).any(-1).mean() > 0.5
  # decoration is cleared at every update
  r.update()
  for x, y in zip(plain, outputs(r)):
    assert np.array_equal(x, y)


# ---- 3b. frames without decoration against the kernel before decoration existed -----------------------------------

GOLDEN = Path(__file__).parent / "golden" / "render_scene_only.json"


def scene_only_digests(backend):
  """sha256 of the rgb, depth and seg buffers of frames without decoration: the synthetic scene (shadows on and off)
  and, on the GPU, the shipped G1 and Go1 height-field scenes after a random-control rollout."""
  import hashlib

  from test_render import O, rollout

  out = {}

  def add(sim, cfg, name):
    r = OffscreenRenderer(sim, cfg, extra_outputs=True)
    r.update()
    out[name] = [hashlib.sha256(np.ascontiguousarray(x).tobytes()).hexdigest() for x in outputs(r)]

  for shadows in (True, False):
    sim, cfg = synthetic(backend, shadows)
    add(sim, cfg, f"synthetic_shadows_{shadows}")
  if backend == "cuda":
    from mjlab_b200.asset_zoo import load_compiled

    for name, body in (("g1_flat", "torso_link"), ("go1_rough_hf", "trunk")):
      mm = load_compiled(name)
      sim = Sim(backend, mm, 40)
      rollout(sim, mm, 20, seed=3)
      add(sim, ViewerConfig(origin_type=O.ASSET_BODY, asset_name="robot", body_name=body, distance=2.5,
                            elevation=-25.0, azimuth=130.0, env_idx=35, width=640, height=360), name)
  return out


@pytest.mark.parametrize("backend", BACKENDS)
def test_scene_only_frames_are_unchanged(backend):
  """Frames without decoration are byte-identical to those of the kernel before decoration was added: the digests in
  tests/golden/render_scene_only.json were written by tools/render_scene_digests.py with that kernel's library (the
  CUDA build on an H100, and its host emulation)."""
  import json

  assert scene_only_digests(backend) == json.loads(GOLDEN.read_text())[backend]


# ---- 4. tile cull and brute force --------------------------------------------------------------------------------

def crowd_scene(nsph):
  """An infinite floor and one free body carrying `nsph` small spheres."""
  from mjlab_b200.compiler.spec import Spec

  spec = Spec()
  spec.worldbody.add_geom(name="floor", type="plane", size=[0, 0, 0.05], rgba=[0.6, 0.6, 0.6, 1])
  b = spec.worldbody.add_body(name="crowd", pos=[0, 0, 0.5])
  b.add_freejoint(name="crowd_j")
  for k in range(nsph):
    b.add_geom(name=f"s{k}", type="sphere", size=[0.03], pos=[0.01 * (k % 8), 0.01 * (k // 8), 0],
               rgba=[0.9, 0.3, 0.3, 1])
  return spec.compile()


LIST = 2048  # B2R_LIST, the tile list's capacity


@pytest.mark.parametrize("backend", BACKENDS)
@pytest.mark.parametrize("nsph", [64, 62])
def test_cull_paths(backend, nsph):
  """Tile cull against brute force with decoration, where the centre tile's list overflows: with 64 spheres the scene
  alone overflows it, with 62 the scene fits (1 + 33 x 62 = 2047 items in all) and the decoration pushes it over."""
  m = crowd_scene(nsph)
  n = 34
  sim = Sim(backend, m, n)
  qp = np.zeros((n, 7), np.float32)
  qp[:, 2], qp[:, 3] = 0.5, 1
  sim.t("qpos")[...] = torch.as_tensor(qp, device=sim.device)
  sim.forward()
  arrows = [((-0.4, -0.3, 0.6), (0.3, 0.2, 0.5), 0.02, (0.2, 0.3, 0.9, 0.6)),
            ((0.0, 0.0, 0.5), (0.0, 0.0, 0.6), 0.03, (0.9, 0.9, 0.2, 0.7))]
  q = qp[0] + np.array([0.05, 0.02, 0, 0, 0, 0, 0], np.float32)
  cfg = ViewerConfig(lookat=(0.0, 0.0, 0.5), distance=1.5, elevation=-30.0, azimuth=70.0, env_idx=n - 1, width=48,
                     height=48, enable_shadows=True)

  def cb(vis):
    arrows_cb(arrows)(vis)
    vis.add_ghost_mesh(torch.as_tensor(q, device=sim.device), (0.3, 0.8, 0.3, 0.5))

  frames = []
  for brute in (0, 1):
    r = OffscreenRenderer(sim, cfg, extra_outputs=True)
    r._args.brute = brute
    r.update(debug_vis_callback=cb)
    frames.append(outputs(r))
    assert r._args.ndecor == 2 and r._args.ghost_xpos
    dev = torch.device(sim.device)
    ghost_pos = _engine_tensor(r._ghost, "geom_xpos", dev)[0].cpu().numpy().astype(np.float64)
    r.close()
  for x, y in zip(*frames):
    assert np.array_equal(x, y)
  # What the centre tile (pixels 16..31 both ways) keeps: the floor (infinite, always kept), every sphere of the 33
  # drawn worlds and of the ghost, and the second arrow: each projects at least 4 pixels inside the tile, further than
  # its bounding sphere reaches (under 2 pixels), so the bounding-sphere cull keeps it.
  eye, f, rr, u, ty, tx = camera(cfg, np.array(cfg.lookat), cfg.width, cfg.height)
  pts = np.concatenate([sim.a("geom_xpos")[:, 1:].reshape(-1, 3), ghost_pos[1:],
                        [np.mean([arrows[1][0], arrows[1][1]], 0)]])
  v = pts - eye
  x = (v @ rr / (v @ f) / tx + 1) * cfg.width / 2
  y = (1 - v @ u / (v @ f) / ty) * cfg.height / 2
  assert ((x > 20) & (x < 28) & (y > 20) & (y < 28)).all(), (x.min(), x.max(), y.min(), y.max())
  scene = 1 + 33 * nsph
  kept = scene + nsph + 1
  if nsph == 64:
    assert scene > LIST
  else:
    assert scene <= LIST < kept  # only the decoration overflows the list
  seg = frames[0][2]
  assert (seg[16:32, 16:32, 1] >= 1).any()


# ---- 5. refusals -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("backend", BACKENDS)
def test_refusals(backend):
  sim, cfg = synthetic(backend, False)
  cfg.width, cfg.height = 16, 16
  r = OffscreenRenderer(sim, cfg)
  nq = int(sim.mj_model.nq)
  # the library's checks
  r.update(debug_vis_callback=arrows_cb(ARROWS[:1]))
  for field, value, msg in (("ndecor", native.RENDER_MAXDECOR + 1, "ndecor 65 outside"), ("ndecor", -1, "ndecor"),
                            ("decor", None, "decor is null")):
    old = getattr(r._args, field)
    setattr(r._args, field, value)
    with pytest.raises(RuntimeError, match=msg):
      launch(r)
    setattr(r._args, field, old)
  launch(r)
  r.update(debug_vis_callback=lambda vis: vis.add_ghost_mesh([0.0] * nq, (0.5, 0.5, 0.5, 0.5)))
  for k, value in ((3, 1.5), (0, float("nan")), (1, -0.1)):
    old = r._args.ghost_rgba[k]
    r._args.ghost_rgba[k] = value
    with pytest.raises(RuntimeError, match="ghost_rgba must lie in"):
      launch(r)
    r._args.ghost_rgba[k] = old
  r._args.ghost_xmat = None
  with pytest.raises(RuntimeError, match="ghost_xpos and ghost_xmat"):
    launch(r)
  # the visualiser's checks
  with pytest.raises(ValueError, match="at most 64 arrows"):
    r.update(debug_vis_callback=lambda vis: [vis.add_arrow((0, 0, 0), (1, 0, 0), (1, 0, 0, 1)) for _ in range(65)])
  for color in ((1.2, 0, 0, 1), (0, 0, float("nan"), 1), (0, 0, 0), (0, 0, 0, -0.5)):
    with pytest.raises(ValueError, match="color must be four finite values"):
      r.update(debug_vis_callback=lambda vis: vis.add_arrow((0, 0, 0), (1, 0, 0), color))
    with pytest.raises(ValueError, match="color must be four finite values"):
      r.update(debug_vis_callback=lambda vis: vis.add_ghost_mesh([0.0] * nq, color))
  with pytest.raises(ValueError, match=f"qpos has {nq - 1} values, the model has nq = {nq}"):
    r.update(debug_vis_callback=lambda vis: vis.add_ghost_mesh([0.0] * (nq - 1), (0.5, 0.5, 0.5, 0.5)))
  with pytest.raises(ValueError, match="width must be positive"):
    r.update(debug_vis_callback=lambda vis: vis.add_arrow((0, 0, 0), (1, 0, 0), (1, 0, 0, 1), width=0.0))
  with pytest.raises(ValueError, match="end must have 3 values"):
    r.update(debug_vis_callback=lambda vis: vis.add_arrow((0, 0, 0), (1, 0), (1, 0, 0, 1)))
  r.update()


# ---- 6. environments (GPU) ---------------------------------------------------------------------------------------

def _env(kind, render_mode, debug_vis, n=64, **kw):
  from mjlab_b200.envs import (TrackingFlatEnv, VelocityCommandCfg, VelocityFlatEnv, tracking_task_cfg,
                               velocity_task_cfg)

  if kind == "velocity":
    cfg = velocity_task_cfg("Mjlab-Velocity-Flat-Unitree-G1", num_envs=n, command=VelocityCommandCfg(debug_vis=debug_vis))
    return VelocityFlatEnv(cfg, render_mode=render_mode)
  cfg = tracking_task_cfg("Mjlab-Tracking-Flat-Unitree-G1", num_envs=n, debug_vis=debug_vis, **kw)
  return TrackingFlatEnv(cfg, render_mode=render_mode)


def test_presets_keep_debug_vis_off():
  from mjlab_b200.envs.tracking_env import TRACKING_TASKS, tracking_task_cfg
  from mjlab_b200.envs.velocity_env import VELOCITY_TASKS, velocity_task_cfg

  for name in VELOCITY_TASKS:
    assert velocity_task_cfg(name).command.debug_vis is False
  for name in TRACKING_TASKS:
    c = tracking_task_cfg(name)
    assert c.debug_vis is False and c.ghost_color == (0.5, 0.7, 0.5, 0.5)
  from mjlab_b200.envs import VelocityCommandCfg

  v = VelocityCommandCfg().viz
  assert (v.z_offset, v.scale) == (0.2, 0.75)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["velocity", "tracking"])
def test_debug_vis_is_read_only(kind):
  outs, per_step = [], []
  for debug_vis in (True, False):
    env = _env(kind, "rgb_array", debug_vis)
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for _ in range(50):
      obs, rew, term, trunc, _ = env.step(torch.randn(env.num_envs, env.nu, device="cuda", generator=g) * 0.5)
      assert env.render().shape == (240, 320, 3)
      d = env.sim.data
      rows.append([t.clone().cpu() for t in (d.qpos, d.qvel, obs, rew, term, trunc)])
    r = env._offline_renderer
    assert (r._args.ndecor == 4) == (debug_vis and kind == "velocity")
    assert bool(r._args.ghost_xpos) == (debug_vis and kind == "tracking")
    before = env.sim.launch_count()
    env.step(torch.zeros(env.num_envs, env.nu, device="cuda"))
    per_step.append(env.sim.launch_count() - before)
    env.close()
    outs.append(rows)
  assert per_step[0] == per_step[1]
  for a, b in zip(*outs):
    for x, y in zip(a, b):
      assert torch.equal(x, y)


def _quat_mat(q):
  w, x, y, z = q
  return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                   [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                   [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


@pytest.mark.gpu
def test_velocity_arrows():
  from mjlab_b200.entity_data import EntityData, EntityIndexing

  env = _env("velocity", "rgb_array", True, n=48)
  env.cfg.viewer.env_idx = env._offline_renderer._cfg.env_idx = env._offline_renderer._args.env_idx = 40
  g = torch.Generator(device="cuda").manual_seed(1)
  for _ in range(30):
    env.step(torch.randn(env.num_envs, env.nu, device="cuda", generator=g) * 0.5)
  env.render()
  dec = env._offline_renderer._decor[:4].cpu().numpy().astype(np.float64)
  ed = EntityData(EntityIndexing.from_model(env.model, "robot", "cuda:0"), env.sim.data, env.sim.model, "cuda:0",
                  env.num_envs)
  e = 40
  pos = ed.root_link_pos_w[e].cpu().numpy().astype(np.float64)
  R = _quat_mat(ed.root_link_quat_w[e].cpu().numpy().astype(np.float64))
  cmd = env.command[e].cpu().numpy().astype(np.float64)
  lin = ed.root_link_lin_vel_b[e].cpu().numpy().astype(np.float64)
  ang = ed.root_link_ang_vel_b[e].cpu().numpy().astype(np.float64)
  s, zo = 0.75, np.array([0, 0, 0.2])
  w2 = lambda v: pos + R @ v  # noqa: E731
  want = [(w2(zo * s), w2((zo + [cmd[0], cmd[1], 0]) * s), (0.2, 0.2, 0.6, 0.6)),
          (w2(zo * s), w2((zo + [0, 0, cmd[2]]) * s), (0.2, 0.6, 0.2, 0.6)),
          (w2(zo * s), w2((zo + [lin[0], lin[1], 0]) * s), (0.0, 0.6, 1.0, 0.7)),
          (w2(zo * s), w2((zo + [0, 0, ang[2]]) * s), (0.0, 1.0, 0.4, 0.7))]
  assert np.abs(cmd).max() > 0 and np.abs(lin[:2]).max() > 1e-3
  for row, (a, b, c) in zip(dec, want):
    assert np.allclose(row[0:3], a, atol=1e-5) and np.allclose(row[3:6], b, atol=1e-5), (row, a, b)
    assert row[6] == np.float32(0.015) and np.allclose(row[7:11], c)
  # a robot at the world origin draws no arrows (alpha 0)
  q = env.sim.data.qpos
  q[e, 0:3] = 0.0
  env.sim.forward()
  plain = OffscreenRenderer(env.sim, env.cfg.viewer)
  plain.update()
  frame = env.render()
  assert np.all(env._offline_renderer._decor[:4, 10].cpu().numpy() == 0)
  assert np.array_equal(frame, plain.render())
  env.close()


def _ghost_reference(env, e, t):
  """commands.py:410-414 in numpy: the first tracked body's position (plus the env origin) and orientation as the free
  joint, the clip's joint positions."""
  ix = env.robot.indexing
  q = np.zeros(env.nq)
  free, jadr = ix.free_joint_q_adr.cpu().numpy(), ix.joint_q_adr.cpu().numpy()
  q[free[:3]] = env.motion["body_pos_w"][t, 0].cpu().numpy() + env.env_origins[e].cpu().numpy()
  q[free[3:7]] = env.motion["body_quat_w"][t, 0].cpu().numpy()
  q[jadr] = env.motion["joint_pos"][t].cpu().numpy()
  return q


@pytest.mark.gpu
@pytest.mark.parametrize("clip", ["synthetic", "file"])
def test_tracking_ghost_qpos(clip, tmp_path):
  kw = {}
  if clip == "file":
    from make_motion_clip import make_clip

    kw["motion_file"] = str(make_clip(tmp_path / "clip.npz", frames=300, device="cuda:0"))
  env = _env("tracking", "rgb_array", True, n=16, **kw)
  from mjlab_b200.envs.tracking_env import BODY_NAMES

  assert BODY_NAMES[0] == "pelvis"
  T = env.motion["joint_pos"].shape[0]
  r = env._offline_renderer
  e = env.cfg.viewer.env_idx = r._args.env_idx = r._cfg.env_idx = 5
  body_ids = env.robot.indexing.body_ids[env.body_idx].cpu().numpy()
  origin = env.env_origins[e].cpu().numpy()
  for t in (0, 1, T // 3, T - 1):
    env.time_steps[e] = t
    assert np.allclose(env.ghost_qpos(e).cpu().numpy(), _ghost_reference(env, e, t), atol=1e-6)
    env.render()
    assert np.allclose(r._ghost_qpos.cpu().numpy(), _ghost_reference(env, e, t), atol=1e-6)
    # independently of how the qpos is built: the ghost's forward kinematics puts the tracked bodies where the clip
    # has them at frame t, shifted to the env's origin.  A recorded clip's body poses are the kinematics of its joint
    # positions, so every body must match; the synthetic clip's are the robot's starting poses, held, so only the
    # pelvis (the free joint) is checked there.
    xpos = _engine_tensor(r._ghost, "xpos", torch.device("cuda:0"))[0].cpu().numpy()[body_ids]
    want = env.motion["body_pos_w"][t].cpu().numpy() + origin
    k = len(body_ids) if clip == "file" else 1
    assert np.abs(xpos[:k] - want[:k]).max() < 2e-3, (t, np.abs(xpos[:k] - want[:k]).max())
  if clip == "file":  # the recorded clip moves, so a wrong frame would show
    a, b = env.motion["body_pos_w"][0].cpu().numpy(), env.motion["body_pos_w"][T // 3].cpu().numpy()
    assert np.abs(a - b).max() > 0.05
  assert list(env._offline_renderer._args.ghost_rgba) == pytest.approx([0.5, 0.7, 0.5, 0.5])
  env.close()

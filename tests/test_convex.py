"""Independent pin of the convex narrowphase (mjlab_b200/csrc/b2_convex.h: GJK distance, EPA depth, plane-mesh,
height-field prisms).  The routines are single-source (fp32 in the kernel, fp64/fp32 in the oracle), so these tests
do NOT compare oracle with kernel: they compare the routines (through the oracle's primitive entry points) with
exact values computed another way — the convex hull of the Minkowski difference (scipy.spatial.ConvexHull): the
origin's depth inside it is the penetration depth, its distance to it the separation — and with brute-force
point/triangle geometry for height fields."""

import ctypes

import numpy as np
import pytest
from scipy.spatial import ConvexHull

from oracle.oracle import load_library

G_SPHERE, G_CAPSULE, G_BOX, G_MESH = 2, 3, 6, 7


def _lib(prec):
  L = load_library(f"f{prec}")
  return L, (np.float64 if prec == 64 else np.float32), (ctypes.c_double if prec == 64 else ctypes.c_float)


def _p(a):
  return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _rot(rng):
  q = rng.normal(size=4)
  q /= np.linalg.norm(q)
  w, x, y, z = q
  return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                   [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                   [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _shape_points(t, pos, R, size, verts):
  """World-frame vertex set of the shape's convex CORE, and its inflation radius."""
  if t == G_SPHERE:
    return pos[None, :], size[0]
  if t == G_CAPSULE:
    return np.stack([pos + R[:, 2] * size[1], pos - R[:, 2] * size[1]]), size[0]
  if t == G_BOX:
    c = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]) * size
    return pos + c @ R.T, 0.0
  return pos + verts @ R.T, 0.0


def _closest_on_tri(a, b, c):
  """Closest point of triangle abc to the origin (projection, then edges)."""
  n = np.cross(b - a, c - a)
  best = None
  if np.dot(n, n) > 1e-30:
    p = n * (np.dot(a, n) / np.dot(n, n))
    M = np.stack([b - a, c - a], axis=1)
    uv, *_ = np.linalg.lstsq(M, p - a, rcond=None)
    if uv[0] >= 0 and uv[1] >= 0 and uv.sum() <= 1:
      best = p
  if best is None:
    cands = []
    for u, v in ((a, b), (b, c), (c, a)):
      e = v - u
      t = np.clip(-np.dot(u, e) / max(np.dot(e, e), 1e-300), 0, 1)
      cands.append(u + t * e)
    best = min(cands, key=lambda x: np.dot(x, x))
  return best


def _exact(ptsA, ptsB):
  """(signed core distance, normal A->B or None when not unique) from the hull of the Minkowski difference."""
  D = (ptsA[:, None, :] - ptsB[None, :, :]).reshape(-1, 3)
  hull = ConvexHull(D, qhull_options="QJ Pp" if len(D) < 5 else "Pp")
  eq = hull.equations  # n.x + off <= 0 inside
  off = eq[:, 3]
  if np.all(off <= 0):  # origin inside: depth = distance to the nearest facet plane
    d = -off
    k = int(np.argmin(d))
    planes = np.unique(np.round(eq, 9), axis=0)
    dd = np.sort(-planes[:, 3])
    unique = len(dd) < 2 or dd[1] - dd[0] > 1e-3
    return -d[k], (eq[k, :3] if unique else None)
  best = None
  for s in hull.simplices:
    p = _closest_on_tri(D[s[0]], D[s[1]], D[s[2]])
    if best is None or np.dot(p, p) < np.dot(best, best):
      best = p
  dist = np.linalg.norm(best)
  return dist, -best / dist


def _inside(pts, p, tol):
  if len(pts) < 4:
    if len(pts) == 1:
      return np.linalg.norm(p - pts[0]) <= tol
    e = pts[1] - pts[0]
    t = np.clip(np.dot(p - pts[0], e) / np.dot(e, e), 0, 1)
    return np.linalg.norm(p - pts[0] - t * e) <= tol
  h = ConvexHull(pts)
  return np.max(h.equations[:, :3] @ p + h.equations[:, 3]) <= tol


def _call_pair(L, dt, ct, t1, p1, R1, s1, v1, t2, p2, R2, s2, v2, margin, scale):
  out = np.zeros(7, dtype=dt)
  a = lambda x: None if x is None else np.ascontiguousarray(x, dtype=dt)  # noqa: E731
  A = [a(p1), a(R1.reshape(-1)), a(s1), a(v1), a(p2), a(R2.reshape(-1)), a(s2), a(v2)]
  n = L.b2o_prim_convex(ctypes.c_int(t1), _p(A[0]), _p(A[1]), _p(A[2]), _p(A[3]), ctypes.c_int(0 if v1 is None else len(v1)),
                        ctypes.c_int(t2), _p(A[4]), _p(A[5]), _p(A[6]), _p(A[7]), ctypes.c_int(0 if v2 is None else len(v2)),
                        ct(margin), ct(scale), _p(out))
  return n, out


def _random_shape(rng, t):
  size = rng.uniform(0.1, 0.4, size=3)
  verts = None
  if t == G_MESH:
    verts = rng.normal(size=(int(rng.integers(6, 24)), 3)) * rng.uniform(0.1, 0.35, size=3)
  return size, verts


@pytest.mark.parametrize("prec", [64, 32])
def test_pair_matches_minkowski_hull(prec):
  L, dt, ct = _lib(prec)
  rng = np.random.default_rng(5)
  tol = 2e-7 if prec == 64 else 2e-4
  types = [(G_MESH, G_MESH), (G_BOX, G_MESH), (G_SPHERE, G_MESH), (G_CAPSULE, G_MESH), (G_BOX, G_BOX)]
  nsep = npen = nnormal = 0
  for it in range(400):
    t1, t2 = types[it % len(types)]
    s1, v1 = _random_shape(rng, t1)
    s2, v2 = _random_shape(rng, t2)
    R1, R2 = _rot(rng), _rot(rng)
    p1 = rng.normal(size=3) * 0.05
    p2 = p1 + rng.normal(size=3) * rng.choice([0.08, 0.25, 0.5])
    A, ra = _shape_points(t1, p1, R1, s1, v1)
    B, rb = _shape_points(t2, p2, R2, s2, v2)
    core, nrm = _exact(A, B)
    want = core - ra - rb
    margin = 0.3
    n, out = _call_pair(L, dt, ct, t1, p1, R1, s1, v1, t2, p2, R2, s2, v2, margin, 1.0)
    if want > margin + 1e-3:
      assert n == 0, (it, want)
      continue
    if want > margin - 1e-3:
      continue
    assert n == 1, (it, want)
    dist, pos, nn = out[0], out[1:4].astype(float), out[4:7].astype(float)
    assert abs(dist - want) <= tol, (it, t1, t2, dist, want)
    assert abs(np.linalg.norm(nn) - 1) < 1e-4
    if core > 0:
      nsep += 1
    else:
      npen += 1
    if nrm is not None and abs(core) > 1e-3:
      nnormal += 1
      assert np.dot(nn, nrm) > 1 - (1e-6 if prec == 64 else 2e-3), (it, t1, t2, nn, nrm, core)
    # the two surface points (pos -+ n dist/2, pulled back by the radii) lie on the cores
    pa = pos - nn * (0.5 * dist) - nn * ra
    pb = pos + nn * (0.5 * dist) + nn * rb
    ptol = 5e-6 if prec == 64 else 2e-3
    assert _inside(A, pa, ptol), (it, t1, t2)
    assert _inside(B, pb, ptol), (it, t1, t2)
  assert nsep > 60 and npen > 60 and nnormal > 100, (nsep, npen, nnormal)


@pytest.mark.parametrize("prec", [64, 32])
def test_deep_and_touching_cases(prec):
  """Concentric shapes (deep penetration, GJK starts at the origin) and exact face contact."""
  L, dt, ct = _lib(prec)
  I = np.eye(3)
  h = np.array([0.2, 0.3, 0.4])
  cube = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]) * 0.25
  # box inside mesh cube, same centre: depth = min over axes of (h_k + 0.25)
  n, out = _call_pair(L, dt, ct, G_BOX, np.zeros(3), I, h, None, G_MESH, np.zeros(3), I, h, cube, 0.0, 1.0)
  assert n == 1 and abs(out[0] + 0.45) < 1e-5
  # sphere centre inside the cube, 0.05 from the +x face: dist = -(0.05 + r)
  n, out = _call_pair(L, dt, ct, G_SPHERE, np.array([0.2, 0.01, -0.02]), I, np.array([0.1, 0, 0]), None,
                      G_MESH, np.zeros(3), I, h, cube, 0.0, 1.0)
  assert n == 1 and abs(out[0] + 0.15) < 1e-5
  assert out[4] < -0.999  # normal from the sphere to the cube: the sphere leaves through +x, so the cube is pushed -x
  # separated by exactly the margin boundary
  n, out = _call_pair(L, dt, ct, G_SPHERE, np.array([0.5, 0.0, 0.0]), I, np.array([0.1, 0, 0]), None,
                      G_MESH, np.zeros(3), I, h, cube, 0.2, 1.0)
  assert n == 1 and abs(out[0] - 0.15) < 1e-6 and out[4] < -0.9999
  n, out = _call_pair(L, dt, ct, G_SPHERE, np.array([0.5, 0.0, 0.0]), I, np.array([0.1, 0, 0]), None,
                      G_MESH, np.zeros(3), I, h, cube, 0.1, 1.0)
  assert n == 0


@pytest.mark.parametrize("prec", [64, 32])
def test_plane_mesh(prec):
  L, dt, ct = _lib(prec)
  cube = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], dtype=float) * 0.25
  out = np.zeros(28, dtype=dt)

  def call(pos, R, margin):
    a = [np.zeros(3, dtype=dt), np.array([0, 0, 1], dtype=dt), np.ascontiguousarray(pos, dtype=dt),
         np.ascontiguousarray(R.reshape(-1), dtype=dt), np.ascontiguousarray(cube, dtype=dt)]
    n = L.b2o_prim_plane_mesh(_p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), _p(a[4]), ctypes.c_int(8), ct(margin), _p(out))
    return n, out[: 7 * n].reshape(n, 7).astype(float)

  # flat on the plane, sunk by 1 cm: the four bottom corners
  n, c = call(np.array([0.3, -0.2, 0.24]), np.eye(3), 0.0)
  assert n == 4
  assert np.allclose(c[:, 0], -0.01, atol=1e-6)
  corners = {(round(x - 0.3, 3), round(y + 0.2, 3)) for x, y in c[:, 1:3]}
  assert corners == {(-0.25, -0.25), (-0.25, 0.25), (0.25, -0.25), (0.25, 0.25)}
  assert np.allclose(c[:, 3], -0.005, atol=1e-6) and np.allclose(c[:, 4:7], [0, 0, 1])
  # tilted: a single lowest corner
  rng = np.random.default_rng(2)
  R = _rot(rng)
  W = cube @ R.T
  z = 0.3
  n, c = call(np.array([0.0, 0.0, z]), R, 0.0)
  low = np.sort(W[:, 2] + z)
  want = int(np.sum((low <= 0) & (low <= low[0] + 1e-3)))
  assert n == max(want, 0) if low[0] <= 0 else n == 0
  if n:
    assert abs(c[0, 0] - low[0]) < 1e-6
  # above the margin: nothing
  n, _ = call(np.array([0.0, 0.0, 2.0]), R, 0.01)
  assert n == 0


def _pt_tri_dist(p, a, b, c):
  q = _closest_on_tri(a - p, b - p, c - p)
  return np.linalg.norm(q), q + p


@pytest.mark.parametrize("prec", [64, 32])
def test_hfield_sphere_matches_triangle_geometry(prec):
  L, dt, ct = _lib(prec)
  rng = np.random.default_rng(11)
  nrow, ncol = 9, 12
  hsize = np.array([1.1, 0.8, 0.3, 0.2])
  ii, jj = np.meshgrid(np.arange(nrow), np.arange(ncol), indexing="ij")
  data = 0.5 + 0.25 * np.sin(0.9 * ii) * np.cos(0.7 * jj) + rng.uniform(-0.03, 0.03, size=(nrow, ncol))  # gentle slopes
  hp = np.array([0.2, -0.1, 0.05])
  R = np.eye(3)
  dx, dy = 2 * hsize[0] / (ncol - 1), 2 * hsize[1] / (nrow - 1)
  out = np.zeros(56, dtype=dt)
  tol = 1e-7 if prec == 64 else 2e-5
  checked = 0
  for it in range(60):
    r = rng.uniform(0.03, 0.08)
    c = np.array([rng.uniform(-0.9, 0.9), rng.uniform(-0.6, 0.6), 0.0])
    # height above the local surface: sometimes touching, sometimes clear
    col, row = int((c[0] + hsize[0]) / dx), int((c[1] + hsize[1]) / dy)
    c[2] = data[row:row + 2, col:col + 2].max() * hsize[2] + r + rng.uniform(-0.01, 0.02)
    margin = 0.01
    gp = hp + c
    a = [np.ascontiguousarray(x, dtype=dt) for x in (hp, R.reshape(-1), hsize, data.reshape(-1), gp, np.eye(3).reshape(-1),
                                                       np.array([r, 0, 0]))]
    n = L.b2o_prim_hfield(_p(a[0]), _p(a[1]), _p(a[2]), ctypes.c_int(nrow), ctypes.c_int(ncol), _p(a[3]),
                          ctypes.c_int(G_SPHERE), _p(a[4]), _p(a[5]), _p(a[6]), None, ctypes.c_int(0), ct(r), ct(margin), _p(out))
    got = np.sort(out[: 7 * n].reshape(n, 7)[:, 0].astype(float))
    # brute force: every top triangle near the sphere (the sphere centre stays above the surface here, so the closest
    # point of a prism is on its top face or the rim of it)
    want = []
    for rr in range(nrow - 1):
      for cc in range(ncol - 1):
        P = lambda i, j: np.array([-hsize[0] + dx * j, -hsize[1] + dy * i, data[i, j] * hsize[2]])  # noqa: E731
        for tri in ((P(rr, cc), P(rr, cc + 1), P(rr + 1, cc + 1)), (P(rr, cc), P(rr + 1, cc + 1), P(rr + 1, cc))):
          d, _ = _pt_tri_dist(c, *tri)
          # side walls of the prism can be closer than the top face only when the centre is beside it and below the
          # rim; skip configurations where that could matter
          if d - r <= margin:
            want.append(d - r)
    want = np.sort(np.array(want))
    if len(want) > 8:
      continue
    # a prism's side wall may be nearer than its top face: the routine's distances are then smaller or equal
    assert len(got) >= len(want), (it, got, want)
    if len(got) == len(want):
      assert np.all(got <= want + tol), (it, got, want)
      if len(want) and np.allclose(got, want, atol=tol):
        checked += 1
  assert checked > 8, checked


def test_hfield_flat_box_rest_contacts():
  """A box lying on a flat height field: every prism under it reports the box's penetration depth."""
  L, dt, ct = _lib(64)
  nrow = ncol = 5
  hsize = np.array([1.0, 1.0, 0.5, 0.1])
  data = np.full((nrow, ncol), 0.4)  # surface at z = 0.2
  out = np.zeros(56, dtype=dt)
  half = np.array([0.2, 0.2, 0.1])
  gp = np.array([0.13, -0.07, 0.2 + 0.1 - 0.004])
  Rz = np.array([[np.cos(0.3), -np.sin(0.3), 0], [np.sin(0.3), np.cos(0.3), 0], [0, 0, 1]])
  a = [np.ascontiguousarray(x, dtype=dt) for x in (np.zeros(3), np.eye(3).reshape(-1), hsize, data.reshape(-1), gp, Rz.reshape(-1), half)]
  n = L.b2o_prim_hfield(_p(a[0]), _p(a[1]), _p(a[2]), ctypes.c_int(nrow), ctypes.c_int(ncol), _p(a[3]),
                        ctypes.c_int(G_BOX), _p(a[4]), _p(a[5]), _p(a[6]), None, ctypes.c_int(0), ct(float(np.linalg.norm(half))),
                        ct(0.0), _p(out))
  c = out[: 7 * n].reshape(n, 7)
  assert n >= 2
  assert np.allclose(c[:, 0], -0.004, atol=1e-9)
  assert np.allclose(c[:, 4:7], [0, 0, 1], atol=1e-9)  # from the field up into the box
  assert np.allclose(c[:, 3], 0.2 - 0.002, atol=1e-9)


@pytest.mark.parametrize("prec", [64, 32])
def test_box_primitives_match_minkowski_hull(prec):
  """The primitive box routines (oracle/b2_oracle.c box_box / sphere_box, restated in the kernel) are own definitions;
  their DEEPEST contact must still carry the exact penetration depth of the two boxes — the origin's depth inside the
  hull of the Minkowski difference — and, when separated within the margin, the exact distance."""
  L, dt, ct = _lib(prec)
  rng = np.random.default_rng(17)
  tol = 1e-6 if prec == 64 else 2e-4
  npen = nsep = exact = 0
  out = np.zeros(7 * 8, dtype=dt)
  for it in range(300):
    h1, h2 = rng.uniform(0.08, 0.35, size=3), rng.uniform(0.08, 0.35, size=3)
    R1, R2 = _rot(rng), _rot(rng)
    p1 = rng.normal(size=3) * 0.05
    p2 = p1 + rng.normal(size=3) * rng.choice([0.15, 0.3, 0.5])
    A, _ = _shape_points(G_BOX, p1, R1, h1, None)
    B, _ = _shape_points(G_BOX, p2, R2, h2, None)
    core, nrm = _exact(A, B)
    margin = 0.05
    a = [np.ascontiguousarray(x, dtype=dt) for x in (p1, R1.reshape(-1), h1, p2, R2.reshape(-1), h2)]
    n = L.b2o_prim_box_box(_p(a[0]), _p(a[1]), _p(a[2]), _p(a[3]), _p(a[4]), _p(a[5]), ct(margin), _p(out))
    c = out[: 7 * n].reshape(n, 7).astype(float)
    if core > margin + 1e-3:
      assert n == 0, (it, core)
      continue
    if core > margin - 1e-3 or abs(core) < 1e-3:
      continue
    assert 1 <= n <= 8, (it, core, n)
    if core < 0:
      npen += 1
      # exact depth, or a face axis within the routine's 5 % preference of faces over a marginally shallower edge axis
      cmin = c[:, 0].min()
      assert 1.05 * core - 1e-5 - tol <= cmin <= core + tol, (it, cmin, core)
      exact += abs(cmin - core) <= tol
      if nrm is not None and abs(cmin - core) <= tol:
        k = int(np.argmin(c[:, 0]))
        assert np.dot(c[k, 4:7], nrm) > 1 - 2e-3, (it, c[k, 4:7], nrm)
    else:
      nsep += 1
      # separated boxes inside the margin: the routine reports the gap along its separating axis, a lower bound of
      # the closest-point distance (equal to it for face-vertex and edge-edge configurations)
      assert 0 < c[:, 0].min() <= core + tol, (it, c[:, 0].min(), core)
  assert npen > 80 and nsep > 5 and exact > 0.6 * npen, (npen, nsep, exact)

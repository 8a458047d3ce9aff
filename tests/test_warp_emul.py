"""Warp-level device helpers of b2_kernel.cuh executed on the host (tests/emul: 32 threads in lock step):
the blocked bottom-up L^T D L with its dof-tree / dense schedules, the triangular solves, symv and the
butterfly sum are checked against numpy without a GPU.  The schedules come from the same header
(b2_tables.h) that b2_create uses."""

import ctypes
import subprocess
from pathlib import Path

import numpy as np
import pytest

EMUL = Path(__file__).parent / "emul"


@pytest.fixture(scope="module")
def lib():
  so = EMUL / "libb2emul.so"
  srcs = [EMUL / "emul.cpp", EMUL / "warp_emul.h", EMUL.parents[1] / "mjlab_b200" / "csrc" / "b2_kernel.cuh",
          EMUL.parents[1] / "mjlab_b200" / "csrc" / "b2_tables.h"]
  if not so.exists() or so.stat().st_mtime < max(s.stat().st_mtime for s in srcs):
    subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-pthread", f"-I{EMUL}", "-o", str(so),
                    str(EMUL / "emul.cpp")], check=True)
  L = ctypes.CDLL(str(so))
  L.emul_wsum.restype = ctypes.c_float
  return L


def tri(i):
  return i * (i + 1) // 2


def ptr(a, t):
  return a.ctypes.data_as(ctypes.POINTER(t))


def random_tree(n, rng, branch=0.25):
  par = [-1]
  for k in range(1, n):
    par.append(k - 1 if rng.uniform() > branch else int(rng.integers(0, k)))
  return np.array(par, dtype=np.int32)


def model_trees():
  from mjlab_b200.asset_zoo import load_compiled

  return {n: np.asarray(load_compiled(n).dof_parentid, dtype=np.int32) for n in ("g1_flat", "go1_flat")}


def tree_spd(par, rng):
  n = len(par)
  M = np.zeros((n, n))
  for k in range(n):
    idx, p = [k], par[k]
    while p >= 0:
      idx.append(p)
      p = par[p]
    v = np.zeros(n)
    v[idx] = rng.normal(size=len(idx))
    M += np.outer(v, v)
  return M + np.diag(rng.uniform(0.5, 1.5, n))


def pack(M):
  n = len(M)
  return np.array([M[i, j] for i in range(n) for j in range(i + 1)], dtype=np.float32)


def py_schedules(par):
  n = len(par)
  anc = []
  for k in range(n):
    a, p = set(), par[k]
    while p >= 0:
      a.add(int(p))
      p = par[p]
    anc.append(a)
  word = lambda i, j: (tri(i) + j) | (i << 12) | (j << 18)
  dense = [word(i, j) for i in range(n) for j in range(i + 1)]
  sparse, start, kt = [], [], n - 1
  while kt >= 0:
    nb = min(4, kt + 1)
    lead = kt - nb + 1
    start.append(len(sparse))
    sparse += [word(i, j) for i in range(lead) for j in range(i + 1)
               if any(i in anc[kt - t] and j in anc[kt - t] for t in range(nb))]
    kt -= 4
  start += [len(sparse)] * (18 - len(start))
  return dense, sparse, start


def test_schedules_match_python_restatement(lib):
  rng = np.random.default_rng(0)
  trees = list(model_trees().values()) + [random_tree(n, rng) for n in (1, 4, 5, 33, 47, 64)]
  for par in trees:
    n = len(par)
    dense = np.zeros(tri(n), dtype=np.uint32)
    sparse = np.zeros(max(8 * tri(n), 1), dtype=np.uint32)
    start = np.zeros(18, dtype=np.int32)
    ns = lib.emul_schedules(n, ptr(par, ctypes.c_int), ptr(dense, ctypes.c_uint), ptr(sparse, ctypes.c_uint), ptr(start, ctypes.c_int))
    d, s, st = py_schedules(par)
    assert dense.tolist() == d and sparse[:ns].tolist() == s and start.tolist() == st
  # G1: the tree keeps 437 of the 1560 dense pair-visits (DESIGN.md 4.1)
  g1 = model_trees()["g1_flat"]
  assert len(py_schedules(g1)[1]) == 437


def _solve(lib, par, M, b, sparse):
  n = len(par)
  A = pack(M)
  inv = np.zeros(n, dtype=np.float32)
  x = b.astype(np.float32).copy()
  lib.emul_ldl(n, ptr(par, ctypes.c_int), ptr(A, ctypes.c_float), ptr(inv, ctypes.c_float), ptr(x, ctypes.c_float), int(sparse))
  return x, A, inv


@pytest.mark.parametrize("case", ["g1_flat", "go1_flat", "chain5", "tree33", "tree47", "tree64", "single"])
def test_ldl_factor_and_solve_on_tree_matrices(lib, case):
  rng = np.random.default_rng(3)
  par = model_trees()[case] if case in ("g1_flat", "go1_flat") else {
    "chain5": np.arange(-1, 4, dtype=np.int32), "tree33": random_tree(33, rng), "tree47": random_tree(47, rng),
    "tree64": random_tree(64, rng), "single": np.array([-1], dtype=np.int32)}[case]
  n = len(par)
  M = tree_spd(par, rng)
  b = rng.normal(size=n)
  ref = np.linalg.solve(M, b)
  for sparse in (True, False):  # tree schedule and dense schedule must both be exact on a tree matrix
    x, A, inv = _solve(lib, par, M, b, sparse)
    assert np.abs(x - ref).max() < 2e-4 * max(1.0, np.abs(ref).max()), (case, sparse)
    # D of L^T D L: pivots are positive and 1/d is what the solve uses
    d = np.array([A[tri(k) + k] for k in range(n)])
    assert (d > 0).all() and np.allclose(inv * d, 1.0, rtol=1e-5)
  # the tree schedule never touches entries outside the tree pattern: they stay exactly zero
  x, A, _ = _solve(lib, par, M, b, True)
  Mz = pack(M)
  assert (A[Mz == 0] == 0).all()


def test_dense_schedule_handles_branch_coupling(lib):
  """A contact between two branches fills the Hessian outside the tree pattern: the dense schedule must be exact."""
  rng = np.random.default_rng(5)
  par = model_trees()["g1_flat"]
  n = len(par)
  Q = rng.normal(size=(n, n))
  M = Q @ Q.T + n * np.eye(n)
  b = rng.normal(size=n)
  x, _, _ = _solve(lib, par, M, b, False)
  ref = np.linalg.solve(M, b)
  assert np.abs(x - ref).max() < 2e-4 * np.abs(ref).max()
  x_bad, _, _ = _solve(lib, par, M, b, True)  # the tree schedule is *not* valid here (the kernel's treeok guard)
  assert np.abs(x_bad - ref).max() > 1e-2 * np.abs(ref).max()


@pytest.mark.parametrize("n", [1, 5, 18, 35, 47, 64])
def test_symv_and_wsum(lib, n):
  rng = np.random.default_rng(n)
  Q = rng.normal(size=(n, n))
  M = Q + Q.T
  x = rng.normal(size=n).astype(np.float32)
  y = np.zeros(n, dtype=np.float32)
  Mp = pack(M)
  lib.emul_symv(n, ptr(Mp, ctypes.c_float), ptr(x, ctypes.c_float), ptr(y, ctypes.c_float))
  assert np.abs(y - M @ x).max() < 1e-4 * max(1.0, np.abs(M @ x).max())
  v = rng.normal(size=32).astype(np.float32)
  s = lib.emul_wsum(ptr(v, ctypes.c_float))
  assert s == pytest.approx(float(v.astype(np.float64).sum()), abs=1e-5)


def _rot(rng):
  q = rng.normal(size=4)
  q /= np.linalg.norm(q)
  w, x, y, z = q
  return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                   [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                   [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def test_box_primitives_device_code_matches_oracle(lib):
  """sphere-box, capsule-box and box-box: the CUDA device routines (compiled for the host) against the
  oracle's C routines on random configurations, including far-from-origin placements (fp32 vs fp64)."""
  from oracle.oracle import load_library

  orc = load_library("f64")
  dp, fp = ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_float)
  rng = np.random.default_rng(11)
  counts = {"sphere": 0, "capsule": 0, "capsule2": 0, "box": 0}
  for trial in range(600):
    off = rng.uniform(-1, 1, 3) * (60.0 if trial % 3 == 0 else 0.0)  # a third of the cases ~60 m from the origin
    tol = 3e-5 if trial % 3 == 0 else 3e-6
    bp = off + rng.uniform(-0.2, 0.2, 3)
    bm = _rot(rng)
    h = rng.uniform(0.1, 0.6, 3)
    box32 = np.concatenate([bp, bm.ravel()]).astype(np.float32)
    h32 = h.astype(np.float32)
    o64, o32 = np.zeros(56), np.zeros(56, dtype=np.float32)
    # sphere
    r = rng.uniform(0.03, 0.2)
    sp = bp + bm @ (rng.uniform(-1.2, 1.2, 3) * (h + r))
    n64 = orc.b2o_prim_sphere_box(ptr(sp, ctypes.c_double), ctypes.c_double(r), ptr(bp, ctypes.c_double), ptr(np.ascontiguousarray(bm.ravel()), ctypes.c_double),
                                  ptr(h, ctypes.c_double), ctypes.c_double(0.0), ptr(o64, ctypes.c_double))
    sp32 = sp.astype(np.float32)
    n32 = lib.emul_sphere_box(ptr(sp32, ctypes.c_float), ctypes.c_float(r), ptr(box32, ctypes.c_float), ptr(h32, ctypes.c_float),
                              ctypes.c_float(0.0), ptr(o32, ctypes.c_float))
    if abs(o64[0]) > 10 * tol or n64 == n32:  # (contact / no contact may flip within rounding of the surface)
      assert n64 == n32
      if n64:
        assert np.abs(o32[:4] - o64[:4]).max() < tol, (trial, o32[:7], o64[:7])
        # an edge / corner normal is a normalised difference of nearby points: rounding is amplified by 1/distance
        assert np.abs(o32[4:7] - o64[4:7]).max() < 100 * tol, (trial, o32[:7], o64[:7])
        counts["sphere"] += 1
    # capsule
    cm = _rot(rng)
    cs = np.array([rng.uniform(0.03, 0.1), rng.uniform(0.1, 0.4), 0.0])
    cp = bp + bm @ (rng.uniform(-1.1, 1.1, 3) * (h + cs[0] + 0.5 * cs[1]))
    n64 = orc.b2o_prim_capsule_box(ptr(cp, ctypes.c_double), ptr(np.ascontiguousarray(cm.ravel()), ctypes.c_double), ptr(cs, ctypes.c_double),
                                   ptr(bp, ctypes.c_double), ptr(np.ascontiguousarray(bm.ravel()), ctypes.c_double), ptr(h, ctypes.c_double),
                                   ctypes.c_double(0.0), ptr(o64, ctypes.c_double))
    cap32 = np.concatenate([cp, cm.ravel()]).astype(np.float32)
    cs32 = cs.astype(np.float32)
    n32 = lib.emul_capsule_box(ptr(cap32, ctypes.c_float), ptr(cs32, ctypes.c_float), ptr(box32, ctypes.c_float), ptr(h32, ctypes.c_float),
                               ctypes.c_float(0.0), ptr(o32, ctypes.c_float))
    if n64 == n32 and n64:
      # distances agree to rounding; the contact point may slide along a flat distance profile (see DESIGN.md 2)
      assert np.abs(o32[0 : 7 * n64 : 7] - o64[0 : 7 * n64 : 7]).max() < 10 * tol, (trial, o32[:14], o64[:14])
      counts["capsule2" if n64 == 2 else "capsule"] += 1
    # box
    p2 = bp + bm @ (rng.uniform(-1.0, 1.0, 3) * (h + 0.15))
    m2 = _rot(rng)
    h2 = rng.uniform(0.05, 0.3, 3)
    n64 = orc.b2o_prim_box_box(ptr(bp, ctypes.c_double), ptr(np.ascontiguousarray(bm.ravel()), ctypes.c_double), ptr(h, ctypes.c_double),
                               ptr(p2, ctypes.c_double), ptr(np.ascontiguousarray(m2.ravel()), ctypes.c_double), ptr(h2, ctypes.c_double),
                               ctypes.c_double(0.0), ptr(o64, ctypes.c_double))
    b232 = np.concatenate([p2, m2.ravel()]).astype(np.float32)
    h232 = h2.astype(np.float32)
    n32 = lib.emul_box_box(ptr(box32, ctypes.c_float), ptr(h32, ctypes.c_float), ptr(b232, ctypes.c_float), ptr(h232, ctypes.c_float),
                           ptr(o32, ctypes.c_float))
    if n64 == n32 and n64:
      assert np.abs(o32[: 7 * n64] - o64[: 7 * n64]).max() < 10 * tol, (trial, n64)
      counts["box"] += 1
  assert counts["sphere"] > 150 and counts["capsule"] > 50 and counts["capsule2"] > 3 and counts["box"] > 100, counts


def test_matrix_free_jacobian_product(lib):
  """mulJ (J x without ever forming J: per body-pair group a relative spatial velocity from the chain dofs,
  then S_m . V per contact direction, pyramid rows a0 +- mu a_t) against an explicit Jacobian built in numpy."""
  lay = np.zeros(9, dtype=np.int32)
  lib.emul_layout(ptr(lay, ctypes.c_int))
  CS0, CMU, CINFO, CJV0, CN, LINFO, LJV, LN, SD = lay.tolist()
  rng = np.random.default_rng(8)
  nv, nbody, MC, NLC = 35, 12, 24, 8
  # bodies 1..11 with random chain dof sets (nested along a random tree)
  bpar = [0] + [int(rng.integers(0, b)) for b in range(1, nbody)]
  masks = [0] * nbody
  nxt = 0
  for b in range(1, nbody):
    k = int(rng.integers(1, 4))
    own = sum(1 << d for d in range(nxt, min(nxt + k, nv)))
    nxt = min(nxt + k, nv)
    masks[b] = masks[bpar[b]] | own
  dofmask = np.array(masks, dtype=np.uint64)
  cdof = np.zeros((nv, SD), dtype=np.float32)
  cdof[:, :6] = rng.normal(size=(nv, 6))
  # contacts grouped by body pair (contiguous groups), mixed condim 1 / 3 and one excluded contact (dim 0)
  pairs = [(0, 3), (2, 7), (5, 9), (4, 4 if False else 11)]
  con = np.zeros((CN, MC), dtype=np.float32)
  coni = con.view(np.int32)
  gstart, c = [], 0
  dims = []
  for g, (b1, b2) in enumerate(pairs):
    gstart.append(c)
    for _ in range(int(rng.integers(1, 5))):
      dim = [3, 3, 1, 0][int(rng.integers(0, 4))]
      con[CS0 : CS0 + 18, c] = rng.normal(size=18)
      con[CMU, c] = rng.uniform(0.3, 1.2)
      coni[CINFO, c] = b1 | (b2 << 8) | (dim << 16) | (g << 24)  # body pair, condim, body-pair group
      dims.append(dim)
      c += 1
  ncon = c
  gstart.append(ncon)
  gstart = np.array(gstart, dtype=np.int32)
  lim = np.zeros((LN, NLC), dtype=np.float32)
  limi = lim.view(np.int32)
  nlim = 5
  ldof = rng.integers(0, nv, nlim)
  lside = rng.integers(0, 2, nlim)
  limi[LINFO, :nlim] = ldof | (lside << 16)
  x = rng.normal(size=nv).astype(np.float32)
  lib.emul_mulJ(ptr(x, ctypes.c_float), ptr(con, ctypes.c_float), ptr(lim, ctypes.c_float), ptr(gstart, ctypes.c_int),
                ptr(cdof, ctypes.c_float), dofmask.ctypes.data_as(ctypes.POINTER(ctypes.c_ulonglong)), ncon, nlim, len(pairs), MC, NLC)
  for ci in range(ncon):
    b1, b2 = coni[CINFO, ci] & 0xff, (coni[CINFO, ci] >> 8) & 0xff
    m1, m2 = int(dofmask[b1]), int(dofmask[b2])
    V = np.zeros(6)
    for d in range(nv):
      if (m1 ^ m2) >> d & 1:
        V += (1.0 if m2 >> d & 1 else -1.0) * cdof[d, :6] * x[d]
    a = [con[CS0 + 6 * mm : CS0 + 6 * mm + 6, ci] @ V for mm in range(3)]
    mu = con[CMU, ci]
    want = {3: [a[0] + mu * a[1], a[0] - mu * a[1], a[0] + mu * a[2], a[0] - mu * a[2]], 1: [a[0], 0, 0, 0], 0: [0, 0, 0, 0]}[dims[ci]]
    assert con[CJV0 : CJV0 + 4, ci] == pytest.approx(want, rel=1e-4, abs=1e-4), (ci, dims[ci])
  assert lim[LJV, :nlim] == pytest.approx(np.where(lside == 1, -1.0, 1.0) * x[ldof], rel=1e-6)

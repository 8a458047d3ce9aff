"""The field surface of the C ABI is pinned: for a few models, every Data and Model field the library registers, in
`b2_field_name` order, with its dtype, shape and strides, and the sizes the library derives (contact capacity,
shared memory per environment, reduced-solver block).  Runs on the host-emulated library (tests/emul).

Regenerate tests/golden/field_surface.json with `python tests/test_field_surface.py` only when a change to the
surface is intended."""

import ctypes
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
GOLDEN = HERE / "golden" / "field_surface.json"
MODELS = ("g1_flat", "go1_stairs_small", "go1_rough_hf", "convex_scene")
OPTIONS = ("maxcon", "smem_bytes_per_env", "reduced_block_cap")


def _model(name):
  if name == "convex_scene":
    from util import convex_scene

    return convex_scene()[0]
  from mjlab_b200.asset_zoo import load_compiled

  return load_compiled(name)


def surface(name):
  sys.path.insert(0, str(HERE / "emul"))
  from engine import EmulEngine

  from mjlab_b200.sim import native

  eng = EmulEngine(_model(name), 2, None, None)
  out = {}
  for which, side in ((0, "data"), (1, "model")):
    rows = []
    for f in eng.names(which):
      t = native.B2Tensor()
      assert eng.lib.b2_get_field(eng.h, which, f.encode(), ctypes.byref(t)) == 0, f
      rows.append([f, int(t.dtype), [int(t.shape[k]) for k in range(t.ndim)], [int(t.stride[k]) for k in range(t.ndim)]])
    out[side] = rows
  opts = {}
  for k in OPTIONS:
    v = ctypes.c_double()
    assert eng.lib.b2_get_option(eng.h, k.encode(), ctypes.byref(v)) == 0, k
    opts[k] = v.value
  out["options"] = opts
  return out


def test_field_surface_matches_golden():
  golden = json.loads(GOLDEN.read_text())
  assert sorted(golden) == sorted(MODELS)
  for name in MODELS:
    got = surface(name)
    for side in ("data", "model"):
      assert [r[0] for r in got[side]] == [r[0] for r in golden[name][side]], (name, side)
      for a, b in zip(got[side], golden[name][side]):
        assert a == b, (name, side, a, b)
    assert got["options"] == golden[name]["options"], name


def _dump(surfaces):
  """JSON with one field per line, so that a change to the surface reads as a short diff."""
  models = []
  for name, s in surfaces.items():
    parts = [f'  "{side}": [\n' + ",\n".join("   " + json.dumps(r) for r in s[side]) + "\n  ]" for side in ("data", "model")]
    parts.append(f'  "options": {json.dumps(s["options"])}')
    models.append(f' "{name}": {{\n' + ",\n".join(parts) + "\n }")
  return "{\n" + ",\n".join(models) + "\n}\n"


if __name__ == "__main__":
  sys.path[:0] = [str(HERE.parent), str(HERE)]
  GOLDEN.write_text(_dump({n: surface(n) for n in MODELS}))
  print(GOLDEN)

"""Digests (sha256) of offscreen frames without decoration, for tests/golden/render_scene_only.json: the scenes of
tests/test_render_debug_vis.py::scene_only_digests rendered by one library, the CUDA build (B2SIM_LIB selects it; run
on the GPU) or its host emulation (--emul LIB).  Prints one JSON object {backend: {scene: [rgb, depth, seg]}}.
  python tools/render_scene_digests.py cuda
  python tools/render_scene_digests.py emul [--emul path/to/libb2sim_emul.so]"""

from __future__ import annotations

import argparse
import ctypes
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import test_render  # noqa: E402
from test_render_debug_vis import scene_only_digests  # noqa: E402

from mjlab_b200.sim import native  # noqa: E402


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("backend", choices=["cuda", "emul"])
  ap.add_argument("--emul", help="a host-emulated library to use instead of building tests/emul's")
  a = ap.parse_args()
  if a.emul:
    test_render._emul = native.bind(ctypes.CDLL(a.emul))
  print(json.dumps({a.backend: scene_only_digests(a.backend)}))


if __name__ == "__main__":
  main()

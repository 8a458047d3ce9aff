"""Compile the reference's G1 / Go1 MJCF into the flat model blobs shipped in
``mjlab_b200/asset_zoo/compiled``.  The MJCF is read from $MJLAB_ASSET_ZOO, by default from the reference package
that oracle/install_reference.py installed under oracle/_ref.

Task sim options: dt 0.005, Newton 10 iterations, 20 line-search iterations, implicitfast,
pyramidal (reference ``tasks/velocity/velocity_env_cfg.py:248-256``).
"""

import os
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
os.environ.setdefault("MJLAB_ASSET_ZOO", str(Path(__file__).resolve().parents[1] / "oracle" / "_ref" / "mjlab" / "asset_zoo" / "robots"))

from mjlab_b200.asset_zoo import COMPILED_DIR, g1, go1, reference_xml  # noqa: E402
from mjlab_b200.asset_zoo.scene import compile_scene  # noqa: E402
from mjlab_b200.sim.sim import MujocoCfg  # noqa: E402
from mjlab_b200.terrains import FULL_SUB_TERRAINS, RoughTerrainCfg  # noqa: E402

TASK = MujocoCfg(timestep=0.005, iterations=10, ls_iterations=20)
_STAIRS = dict(step_height_range=(0.05, 0.15), step_width=0.3, platform_width=2.0, border_width=0.5)
# small stairs scene for parity tests (2 x 4 patches) and the full BASELINE config E terrain (10 x 20)
SMALL_STAIRS = RoughTerrainCfg(num_rows=2, num_cols=4, border_width=2.0, seed=3, sub_terrains=(
  ("flat", 0.25, {}), ("pyramid_stairs", 0.5, _STAIRS), ("pyramid_stairs_inv", 0.25, _STAIRS)))

# height-field scenes: a 2 x 4 patch terrain made of the four height-field sub-terrains (parity tests) and the
# 10 x 20 terrain with all seven sub-terrain types of the reference's (partly commented-out) ROUGH_TERRAINS_CFG
SMALL_HF = RoughTerrainCfg(num_rows=2, num_cols=4, border_width=2.0, seed=5, difficulty_range=(0.3, 0.9),
                           sub_terrains=tuple((k, 0.25, kw) for k, _, kw in FULL_SUB_TERRAINS[3:]))
FULL_HF = RoughTerrainCfg(seed=0, sub_terrains=FULL_SUB_TERRAINS)


def compile_all(g1_xml, go1_xml) -> dict:
  """Every shipped blob's model, by blob name."""
  return {
    "g1_flat": compile_scene(g1.robot_cfg(g1_xml, g1.velocity_sensors()), TASK),
    "g1_tracking_flat": compile_scene(g1.robot_cfg(g1_xml, g1.tracking_sensors()), TASK),
    "go1_flat": compile_scene(go1.robot_cfg(go1_xml, go1.velocity_sensors()), TASK),
    "go1_stairs_small": compile_scene(go1.robot_cfg(go1_xml, go1.velocity_sensors()), TASK, SMALL_STAIRS),
    "go1_rough": compile_scene(go1.robot_cfg(go1_xml, go1.velocity_sensors()), TASK, RoughTerrainCfg()),
    "go1_hf_small": compile_scene(go1.robot_cfg(go1_xml, go1.velocity_sensors()), TASK, SMALL_HF),
    "go1_rough_hf": compile_scene(go1.robot_cfg(go1_xml, go1.velocity_sensors()), TASK, FULL_HF),
  }


def main():
  COMPILED_DIR.mkdir(exist_ok=True)
  for name, m in compile_all(reference_xml("g1"), reference_xml("go1")).items():
    m.save(COMPILED_DIR / f"{name}.npz")
    print(
      f"{name}: nq={int(m.nq)} nv={int(m.nv)} nu={int(m.nu)} nbody={int(m.nbody)} "
      f"njnt={int(m.njnt)} ngeom={int(m.ngeom)} nsite={int(m.nsite)} npair={int(m.npair)} "
      f"nstatic={int(m.nstatic)} nsensordata={int(m.nsensordata)} meaninertia={float(m.stat_meaninertia):.5f}"
    )


if __name__ == "__main__":
  main()

"""Register budget of the step kernel, read from the ptxas report of the library build (csrc/build.log).

The primitive-only instantiations of `b2_step_kernel` (<0> forward, <1> step) run at 16 warps per SM, which leaves
128 registers per thread.  A kernel that needs more is cut to the budget by ptxas with spills to local memory,
and the occupancy only pays without that traffic (DESIGN.md §4.1).  This test keeps the budget from quietly
growing back: any spill, or more registers than the launch bound allows, fails it."""

import re
from pathlib import Path

import pytest

CSRC = Path(__file__).resolve().parents[1] / "mjlab_b200" / "csrc"
LOG = CSRC / "build.log"
LIB = CSRC / "libb2sim.so"
SOURCES = ["b2sim.cu", "b2_kernel.cuh", "b2_env.cuh", "b2_trackenv.cuh", "b2_convex.h", "b2_types.h", "b2_tables.h"]


def _launch_bound():
  """Threads per CTA and co-resident CTAs per SM of the primitive-only instantiations (b2_types.h defaults)."""
  text = (CSRC / "b2_types.h").read_text()
  warps = int(re.search(r"#define B2_WARPS_PER_CTA (\d+)", text).group(1))
  m = re.search(r"#define B2_MIN_CTAS \((\d+) / B2_WARPS_PER_CTA\)", text)
  return 32 * warps, int(m.group(1)) // warps


def _ptxas_report():
  if not LOG.exists() or not LIB.exists():
    pytest.skip("the CUDA library was not built in this tree (make -C mjlab_b200/csrc)")
  if any((CSRC / f).stat().st_mtime > LOG.stat().st_mtime for f in SOURCES):
    pytest.skip("csrc/build.log is older than the sources: rebuild the library")
  report, name = {}, None
  for line in LOG.read_text().splitlines():
    m = re.search(r"Compiling entry function '(\w+)'", line)
    if m:
      name = m.group(1)
      continue
    if name is None:
      continue
    m = re.search(r"Function properties for (\w+)", line)
    if m and m.group(1) != name:
      name = None  # a callee's report
      continue
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
    if m:
      report.setdefault(name, {}).update(stores=int(m.group(1)), loads=int(m.group(2)))
    m = re.search(r"Used (\d+) registers", line)
    if m:
      report.setdefault(name, {})["regs"] = int(m.group(1))
      name = None
  return report


@pytest.mark.parametrize("mode", [0, 1])
def test_step_kernel_fits_its_register_budget(mode):
  report = _ptxas_report()
  name = f"_Z14b2_step_kernelILi{mode}EEv8DevModel7DevData"
  assert name in report, f"no ptxas report for b2_step_kernel<{mode}> in {LOG}"
  r = report[name]
  threads, ctas = _launch_bound()
  budget = 65536 // (threads * ctas) // 8 * 8  # registers are allocated per thread in multiples of 8
  assert r["regs"] <= budget, f"b2_step_kernel<{mode}>: {r['regs']} registers, the launch bound allows {budget}"
  assert r["stores"] == 0 and r["loads"] == 0, (
      f"b2_step_kernel<{mode}> spills: {r['stores']} B of stores, {r['loads']} B of loads per thread")

"""The step kernel's phase marks (b2_kernel.cuh, PHASE_MARK) and their labels.

Under -DB2_PHASE_TIMING each mark adds the cycles since the previous one to g_phase_cycles[id], and
tools/phase_breakdown.py and tools/ncu_by_phase.py label each mark by the comment on its line.  Two marks with one id
would merge two phases into one row, an id past the array would write outside it, and a mark without a label would
drop out of both tools' tables."""

import re
from pathlib import Path

SRC = (Path(__file__).resolve().parents[1] / "mjlab_b200" / "csrc" / "b2_kernel.cuh").read_text()
MARK = re.compile(r"^[ \t]*PHASE_MARK\((\d+)\);[ \t]*//[ \t]*(.*\S)", re.M)  # the tools' regex


def test_phase_marks_are_unique_in_range_and_labelled():
  calls = re.findall(r"\bPHASE_MARK\((\d+)\)", SRC)
  assert calls, "no PHASE_MARK in b2_kernel.cuh"
  assert len(calls) == len(set(calls)), f"PHASE_MARK ids used twice: {sorted(calls, key=int)}"
  # g_phase_cycles[32], as b2_phase_cycles copies it out
  assert all(int(k) < 32 for k in calls), f"PHASE_MARK ids past the end of g_phase_cycles: {calls}"
  labelled = {k for k, _ in MARK.findall(SRC)}
  assert labelled == set(calls), f"PHASE_MARK calls without a `// label` on their line: {sorted(set(calls) - labelled)}"

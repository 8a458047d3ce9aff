"""Aggregate tools/ncu_by_line.py output by kernel phase / helper function.

  python tools/ncu_by_phase.py <report.ncu-rep> [kernel-substring]
Ranges come from the *current* b2_kernel.cuh, so the library and source must be the ones the report was captured
with.  A line belongs to the next PHASE_MARK after it (the mark's comment labels the code that ends there), unless an
out-of-line helper or the kernel itself starts in between; lines of a helper after its last mark count as the helper,
and lines of the kernel after its last mark as the kernel's tail."""
import os
import re
import subprocess
import sys

root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
src = open(os.path.join(root, "mjlab_b200", "csrc", "b2_kernel.cuh")).read().splitlines()
owner = {}  # source line -> label
region, pending = "?", []
for i, ln in enumerate(src, 1):
  start = None
  m = re.match(r"__device__ __noinline__ \w[\w ]*?(\w+)\(", ln)
  if m:
    start = "fn " + m.group(1)
  if re.match(r"__device__ __forceinline__ \w[\w ]*?(\w+)\(", ln):
    start = "inline helpers"
  if ln.startswith("template <int MODE>"):
    start = "kernel tail (after the last mark)"
  if start:
    owner.update((l, region) for l in pending)
    region, pending = start, []
  pending.append(i)
  m = re.match(r"^[ \t]*PHASE_MARK\((\d+)\);[ \t]*//[ \t]*(.*\S)", ln)
  if m:
    owner.update((l, m.group(1) + " " + m.group(2)) for l in pending)
    pending = []
owner.update((l, region) for l in pending)
out = subprocess.run([sys.executable, os.path.join(root, "tools", "ncu_by_line.py"), sys.argv[1],
                      sys.argv[2] if len(sys.argv) > 2 else "b2_step_kernelILi1", "100000"],
                     capture_output=True, text=True).stdout
tot = {}
for line in out.splitlines():
  m = re.match(r"\('([^']+)', (\d+)\)\s+samp\s+([\d.]+)%\s+inst\s+([\d.]+)%", line)
  if not m:
    if line.startswith("total"):
      print(line)
    continue
  f, l, sp, ip = m.group(1), int(m.group(2)), float(m.group(3)), float(m.group(4))
  key = owner.get(l, "?") if f == "b2_kernel.cuh" else "cuda intrinsics headers (shfl, ...)"
  t = tot.setdefault(key, [0.0, 0.0])
  t[0] += sp
  t[1] += ip
print(f"{'phase / function':44s} samples%  inst%")
for k, v in sorted(tot.items(), key=lambda x: -x[1][0]):
  print(f"{k:44s} {v[0]:7.1f} {v[1]:7.1f}")

"""Per-phase cycle breakdown of the step kernel on one of bench.py's workloads (needs the -DB2_PHASE_TIMING variant):
  B2SIM_LIB=mjlab_b200/csrc/variants/libb2sim_timing.so python tools/phase_breakdown.py [envs] [preroll] [opt=val ...]
B2_WORKLOAD (B, C, E or F, default B) picks the workload.
Each row is the code that ends at one PHASE_MARK of b2_kernel.cuh, labelled by the comment on that mark."""
import ctypes, os, re, sys
from pathlib import Path
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import torch
import bench
n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
env = bench.make_env(os.environ.get("B2_WORKLOAD", "B"), n, 42, "cuda:0")
g = torch.Generator(device="cuda:0"); g.manual_seed(0)
for _ in range(int(sys.argv[2]) if len(sys.argv) > 2 else 100):
  env.step(torch.rand((n, env.nu), generator=g, device="cuda:0") * 2 - 1)
sim = env.sim
for kv in sys.argv[3:]:
  k, v = kv.split("=")
  sim.set_option(k, float(v))
buf = (ctypes.c_ulonglong * 32)()
sim._lib.b2_phase_cycles(buf)  # reset
K = 20
for _ in range(K): sim.step()
torch.cuda.synchronize()
assert sim._lib.b2_phase_cycles(buf) == 0, "library built without -DB2_PHASE_TIMING"
src = (ROOT / "mjlab_b200" / "csrc" / "b2_kernel.cuh").read_text()
labels = {int(k): lab for k, lab in re.findall(r"^[ \t]*PHASE_MARK\((\d+)\);[ \t]*//[ \t]*(.*\S)", src, re.M)}
# marks 21-23 run inside the height-field routine and split the time of mark 20, so the total is marks 0-20
tot = sum(buf[i] for i in range(21))
st = sim.stats()
print(f"mean newton iters {st.niter_mean:.2f}, mean ncon {st.ncon_mean:.1f}; cycles per env-step (warp-serial): {tot / (K * n):.0f}")
for i in sorted(labels):
  print(f"{i:2d} {labels[i]:34s} {buf[i] / (K * n):10.0f} cyc/env  {100.0 * buf[i] / tot:5.1f}%")

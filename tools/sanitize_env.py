"""Small run of the fused MDP kernels (velocity and tracking tasks) for compute-sanitizer:
  compute-sanitizer --tool memcheck python tools/sanitize_env.py"""
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch  # noqa: E402

from mjlab_b200.envs import VelocityEnvCfg, VelocityFlatEnv  # noqa: E402
from mjlab_b200.envs.tracking_env import TrackingEnvCfg, TrackingFlatEnv  # noqa: E402

n = 64
g = torch.Generator(device="cuda:0")
g.manual_seed(0)
env = VelocityFlatEnv(VelocityEnvCfg(num_envs=n, episode_length_s=0.2), device="cuda:0")
for _ in range(12):  # (episodes of 10 steps: resets and masked forwards are exercised)
  env.step(torch.rand((n, env.nu), generator=g, device="cuda:0") * 2 - 1)
torch.cuda.synchronize()
print("velocity env ok", float(env.episode_length_buf.float().mean()))
trk = TrackingFlatEnv(TrackingEnvCfg(num_envs=n), device="cuda:0")
for _ in range(12):
  trk.step(torch.rand((n, trk.nu), generator=g, device="cuda:0") * 2 - 1)
torch.cuda.synchronize()
print("tracking env ok")
# a moving clip with the adaptive start-frame sampler (b2_trackenv_bins), falls forced so that failures are binned
sys.path.insert(0, str(Path(__file__).resolve().parent))
import tempfile  # noqa: E402

from make_motion_clip import make_clip  # noqa: E402

with tempfile.TemporaryDirectory() as tmp:
  clip = make_clip(Path(tmp) / "clip.npz", frames=960, device="cuda:0")
  ad = TrackingFlatEnv(TrackingEnvCfg(num_envs=n, motion_file=clip, adaptive_kernel_size=3), device="cuda:0")
  for k in range(12):
    if k % 3 == 0:
      ad.sim.data.qpos[: n // 4, 2] -= 0.4
    ad.step(torch.rand((n, ad.nu), generator=g, device="cuda:0") * 2 - 1)
  torch.cuda.synchronize()
  assert float(ad.bin_failed_count.sum()) > 0
  print("adaptive tracking env ok")

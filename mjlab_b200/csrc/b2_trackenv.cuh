// b2_trackenv.cuh — fused MDP glue of the motion-tracking task (BASELINE config C) around the physics step: the
// caller-side work of ManagerBasedRlEnv.step (reference src/mjlab/envs/manager_based_rl_env.py:106-147) with the
// terms of tasks/tracking/tracking_env_cfg.py as two kernels, one warp per environment (lane = tracked body or
// joint), instead of ~150 tiny torch launches (1.8 ms of a 3.7 ms env step at 4096 envs):
//   post1 (after the sub-steps): episode counter, terminations (time_out, anchor height / orientation, end-effector
//          height: tracking_env_cfg.py:253-278), rewards (:200-250), log row, RSI reset of finished envs onto the
//          clip (mdp/commands.py:283-352), clip time step + restart of envs that ran off its end -> mask for
//          b2_forward_masked;
//   post2 (after the masked forward): anchor-relative body targets (commands.py:354-388), interval push
//          (events.py:127-143), policy observation with noise and critic observation (:88-150);
//   bins (one CTA, between post1 and the forward, motion files only): the adaptive start-frame sampler's EMA and
//          the CDF post1 inverts (commands.py:256-297, 394-398).
// The torch implementation in mjlab_b200/envs/tracking_env.py is the reference; both consume the same per-step
// uniforms U[n][B2_TRACKENV_NU(nu)] (layout in include/b2sim.h), compared in tests.
#pragma once
#include "../../include/b2sim.h"
#include "b2_types.h"

namespace b2t {
struct Q { float w, x, y, z; };
struct V3 { float x, y, z; };
__device__ __forceinline__ Q qmul(Q a, Q b) {
  return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
          a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x, a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w};
}
__device__ __forceinline__ Q qinv(Q q) { return {q.w, -q.x, -q.y, -q.z}; }
__device__ __forceinline__ V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
__device__ __forceinline__ V3 qapply(Q q, V3 v) {  // R(q) v
  V3 u = {q.x, q.y, q.z}, t = cross(u, v);
  t = {2.f * t.x, 2.f * t.y, 2.f * t.z};
  V3 c = cross(u, t);
  return {v.x + q.w * t.x + c.x, v.y + q.w * t.y + c.y, v.z + q.w * t.z + c.z};
}
__device__ __forceinline__ V3 qapply_inv(Q q, V3 v) {  // R(q)^T v
  V3 u = {q.x, q.y, q.z}, t = cross(u, v);
  t = {2.f * t.x, 2.f * t.y, 2.f * t.z};
  V3 c = cross(u, t);
  return {v.x - q.w * t.x + c.x, v.y - q.w * t.y + c.y, v.z - q.w * t.z + c.z};
}
__device__ __forceinline__ Q yaw_quat(Q q) {
  float yaw = atan2f(2.f * (q.w * q.z + q.x * q.y), 1.f - 2.f * (q.y * q.y + q.z * q.z));
  return {cosf(0.5f * yaw), 0.f, 0.f, sinf(0.5f * yaw)};
}
__device__ __forceinline__ Q quat_from_euler(float r, float p, float y) {
  float cy = cosf(0.5f * y), sy = sinf(0.5f * y), cr = cosf(0.5f * r), sr = sinf(0.5f * r), cp = cosf(0.5f * p), sp = sinf(0.5f * p);
  return {cy * cr * cp + sy * sr * sp, cy * sr * cp - sy * cr * sp, cy * cr * sp + sy * sr * cp, sy * cr * cp - cy * sr * sp};
}
__device__ __forceinline__ float qerr(Q a, Q b) {  // rotation angle between two orientations
  Q d = qmul(a, qinv(b));
  return 2.f * atan2f(sqrtf(d.x * d.x + d.y * d.y + d.z * d.z), fabsf(d.w));
}
__device__ __forceinline__ void rot6(Q q, float* o) {  // first two columns of R(q), row-major over (3, 2)
  o[0] = 1.f - 2.f * (q.y * q.y + q.z * q.z); o[1] = 2.f * (q.x * q.y - q.w * q.z);
  o[2] = 2.f * (q.x * q.y + q.w * q.z);       o[3] = 1.f - 2.f * (q.x * q.x + q.z * q.z);
  o[4] = 2.f * (q.x * q.z - q.w * q.y);       o[5] = 2.f * (q.y * q.z + q.w * q.x);
}
__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ Q ldq(const float* p) { return {p[0], p[1], p[2], p[3]}; }
__device__ __forceinline__ V3 ldv(const float* p) { return {p[0], p[1], p[2]}; }
__device__ __forceinline__ float bcast(float v, int src) { return __shfl_sync(0xffffffffu, v, src); }
__device__ __forceinline__ Q bcastq(Q q, int s) { return {bcast(q.w, s), bcast(q.x, s), bcast(q.y, s), bcast(q.z, s)}; }
__device__ __forceinline__ V3 bcastv(V3 v, int s) { return {bcast(v.x, s), bcast(v.y, s), bcast(v.z, s)}; }

// RSI resample of one environment onto clip frame `ts` (commands.py:283-352): qpos / qvel / ctrl / xfrc_applied
__device__ __forceinline__ void resample(const DevData& dd, const B2TrackEnvArgs& A, int w, int lane, int nu, int nbody,
                                         long long ts, const float* Ub) {
  float* qpos = dd.qpos.p + (size_t)w * dd.qpos.stride;
  float* qvel = dd.qvel.p + (size_t)w * dd.qvel.stride;
  float* ctrl = dd.ctrl.p + (size_t)w * dd.ctrl.stride;
  float* xfrc = dd.xfrc_applied.p + (size_t)w * dd.xfrc_applied.stride;
  const size_t fb = (size_t)ts * A.nb;
  float pn[6], vn[6];
#pragma unroll
  for (int k = 0; k < 6; k++) {
    pn[k] = Ub[1 + k] * (A.pose_range[2 * k + 1] - A.pose_range[2 * k]) + A.pose_range[2 * k];
    vn[k] = Ub[7 + k] * (A.vel_range[2 * k + 1] - A.vel_range[2 * k]) + A.vel_range[2 * k];
  }
  Q ori = qmul(quat_from_euler(pn[3], pn[4], pn[5]), ldq(A.m_body_quat + 4 * fb));
  if (lane == 0) {
    const float* org = A.env_origins + 3 * (size_t)w;
    const float* bp = A.m_body_pos + 3 * fb; const float* bl = A.m_body_lin + 3 * fb; const float* ba = A.m_body_ang + 3 * fb;
    qpos[0] = bp[0] + org[0] + pn[0]; qpos[1] = bp[1] + org[1] + pn[1]; qpos[2] = bp[2] + org[2] + pn[2];
    qpos[3] = ori.w; qpos[4] = ori.x; qpos[5] = ori.y; qpos[6] = ori.z;
    qvel[0] = bl[0] + vn[0]; qvel[1] = bl[1] + vn[1]; qvel[2] = bl[2] + vn[2];
    V3 ab = qapply_inv(ori, {ba[0] + vn[3], ba[1] + vn[4], ba[2] + vn[5]});
    qvel[3] = ab.x; qvel[4] = ab.y; qvel[5] = ab.z;
  }
  for (int a = lane; a < nu; a += 32) {
    float jp = A.m_joint_pos[(size_t)ts * nu + a] + Ub[13 + a] * (A.jp_hi - A.jp_lo) + A.jp_lo;
    qpos[7 + a] = fminf(fmaxf(jp, A.soft_lo[a]), A.soft_hi[a]);
    qvel[6 + a] = A.m_joint_vel[(size_t)ts * nu + a];
    ctrl[a] = 0.f;
  }
  for (int i = lane; i < 6 * nbody; i += 32) xfrc[i] = 0.f;
}

// IEEE-rounded division: the library builds with --use_fast_math, but a sampled frame must round as torch's does
__device__ __forceinline__ float div_rn(float a, float b) {
#ifdef B2_HOST_EMULATION
  return a / b;
#else
  return __fdiv_rn(a, b);
#endif
}

// start frame of a reset or clip restart from its uniform u (B2_START_*, include/b2sim.h)
__device__ __forceinline__ long long start_frame(const B2TrackEnvArgs& A, float u) {
  if (A.adaptive == B2_START_FIRST) return 0;
  if (A.adaptive != B2_START_ADAPTIVE) return (long long)(u * (float)(A.T - 1));
  int lo = 0, hi = A.nbins - 1;  // first bin with cdf > u (cdf[nbins - 1] = 1 > u)
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (A.cdf[mid] > u) hi = mid; else lo = mid + 1;
  }
  const float c0 = lo > 0 ? A.cdf[lo - 1] : 0.f;
  const float frac = div_rn(u - c0, A.cdf[lo] - c0);
  const long long ts = (long long)(div_rn((float)lo + frac, (float)A.nbins) * (float)(A.T - 1));
  return ts < A.T - 1 ? ts : A.T - 1;
}

// unnormalised start-bin weight: replicate-padded correlation of (EMA + ratio / nbins) with the kernel
__device__ __forceinline__ float bin_weight(const B2TrackEnvArgs& A, int b, float floor_) {
  float s = 0.f;
  for (int i = 0; i < A.adaptive_kernel_size; i++) s += A.adaptive_kernel[i] * (A.bin_fail_ema[min(b + i, A.nbins - 1)] + floor_);
  return s;
}

__device__ __forceinline__ float norm3(V3 a, V3 b) {
  const float x = a.x - b.x, y = a.y - b.y, z = a.z - b.z;
  return sqrtf(x * x + y * y + z * z);
}

// the ten motion errors of one env against clip frame fr (MotionCommand._update_metrics, commands.py:221-255), from
// the lane's tracked body; lane 0 writes them to out[B2_TRACKENV_NMETRIC]
__device__ __forceinline__ void motion_errors(const B2TrackEnvArgs& A, int lane, bool hasb, int b, long long fr, V3 org,
                                              V3 pos, Q quat, V3 lin, V3 ang, V3 rel_p, Q rel_q, const float* qpos,
                                              const float* qvel, int nu, float* out) {
  const size_t fb = (size_t)fr * A.nb;
  // the anchor's errors first: its clip and robot poses are not held across the per-body errors
  const V3 cpa = ldv(A.m_body_pos + 3 * (fb + A.anchor));
  const float anchor_pos = norm3({cpa.x + org.x, cpa.y + org.y, cpa.z + org.z}, bcastv(pos, A.anchor));
  const float anchor_rot = qerr(ldq(A.m_body_quat + 4 * (fb + A.anchor)), bcastq(quat, A.anchor));
  float ep = 0.f, eq = 0.f, el = 0.f, ea = 0.f;
  if (hasb) {
    ep = norm3(rel_p, pos);
    eq = qerr(rel_q, quat);
    el = norm3(ldv(A.m_body_lin + 3 * (fb + b)), lin);
    ea = norm3(ldv(A.m_body_ang + 3 * (fb + b)), ang);
  }
  const float anchor_lin = bcast(el, A.anchor), anchor_ang = bcast(ea, A.anchor), inb = 1.f / (float)A.nb;
  ep = wsum(ep) * inb; eq = wsum(eq) * inb; el = wsum(el) * inb; ea = wsum(ea) * inb;
  float sj = 0.f, sv = 0.f;
  for (int a = lane; a < nu; a += 32) {
    const float dj = A.m_joint_pos[(size_t)fr * nu + a] - qpos[7 + a], dv = A.m_joint_vel[(size_t)fr * nu + a] - qvel[6 + a];
    sj += dj * dj;
    sv += dv * dv;
  }
  sj = sqrtf(wsum(sj));
  sv = sqrtf(wsum(sv));
  if (lane == 0) {
    out[0] = anchor_pos; out[1] = anchor_rot; out[2] = anchor_lin; out[3] = anchor_ang;
    out[4] = ep; out[5] = eq; out[6] = el; out[7] = ea; out[8] = sj; out[9] = sv;
  }
}

constexpr int kBinThreads = 256;

// sum over the CTA in a fixed order (every thread gets it)
__device__ __forceinline__ float cta_sum(float v, float* red) {
  v = wsum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  for (int k = 0; k < kBinThreads / 32; k++) t += red[k];
  __syncthreads();
  return t;
}

// sum of the bin weights over all bins, block-strided, in a fixed order
__device__ __forceinline__ float weight_total(const B2TrackEnvArgs& A, float floor_, float* red) {
  float t = 0.f;
  for (int b = threadIdx.x; b < A.nbins; b += kBinThreads) t += bin_weight(A, b, floor_);
  return cta_sum(t, red);
}
}  // namespace b2t

__global__ void b2_trackenv_post1_kernel(DevData dd, int nu, int nbody, B2TrackEnvArgs A) {
  using namespace b2t;
  const int lane = threadIdx.x & 31;
  const int w = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (w >= dd.nworld) return;
  const int S = 13 + nu;
  const float* U = A.U + (size_t)w * B2_TRACKENV_NU(nu);
  const float* qpos = dd.qpos.p + (size_t)w * dd.qpos.stride;
  const float* act = A.action + (size_t)w * nu;
  float* last = A.last_action + (size_t)w * nu;
  long long ts = A.time_steps[w];
  int ep = A.episode_length[w] + 1;
  // the joint terms' sums first: the body state below is not held across this loop
  float rate = 0.f, lim = 0.f;
  for (int a = lane; a < nu; a += 32) {
    float da = act[a] - last[a];
    rate += da * da;
    float jp = qpos[7 + a];
    lim += fmaxf(A.soft_lo[a] - jp, 0.f) + fmaxf(jp - A.soft_hi[a], 0.f);
  }
  const bool hasb = lane < A.nb;
  const int b = hasb ? lane : 0;
  const int bid = A.body_idx[b];
  const size_t fb = (size_t)ts * A.nb;
  // robot state of the lane's tracked body, clip state of the same body
  const V3 pos = ldv(dd.xpos.p + (size_t)w * dd.xpos.stride + 3 * bid);
  const Q quat = ldq(dd.xquat.p + (size_t)w * dd.xquat.stride + 4 * bid);
  const float* lv = dd.link_vel_w.p + (size_t)w * dd.link_vel_w.stride + 6 * bid;
  const V3 lin = {lv[0], lv[1], lv[2]}, ang = {lv[3], lv[4], lv[5]};
  const V3 org = ldv(A.env_origins + 3 * (size_t)w);
  const V3 cpa = ldv(A.m_body_pos + 3 * (fb + A.anchor));
  const V3 a_pos = {cpa.x + org.x, cpa.y + org.y, cpa.z + org.z};
  const Q a_quat = ldq(A.m_body_quat + 4 * (fb + A.anchor));
  const V3 r_pos = bcastv(pos, A.anchor);
  const Q r_quat = bcastq(quat, A.anchor);
  const V3 rel_p = ldv(A.body_pos_rel + 3 * ((size_t)w * A.nb + b));
  const Q rel_q = ldq(A.body_quat_rel + 4 * ((size_t)w * A.nb + b));
  // terminations (tracking_env_cfg.py:253-278)
  const bool trunc = ep >= A.max_episode_length;
  const V3 g = {0.f, 0.f, -1.f};
  const float ori_err = fabsf(qapply_inv(a_quat, g).z - qapply_inv(r_quat, g).z);
  const float* W = A.weight;
  const bool bad_z = A.term_on[0] && fabsf(a_pos.z - r_pos.z) > A.term_threshold[0];
  const bool bad_ori = A.term_on[1] && ori_err > A.term_threshold[1];
  bool ee_bad = false;
  for (int k = 0; k < A.nee; k++) ee_bad |= hasb && lane == A.ee_idx[k] && fabsf(rel_p.z - pos.z) > A.term_threshold[2];
  const bool bad_ee = A.term_on[2] && __any_sync(0xffffffffu, ee_bad);
  const bool term = bad_z || bad_ori || bad_ee;
  // rewards (:200-250): each term weighted, or 0 at weight 0 (not evaluated); the weights are uniform over the warp
  const float inb = 1.f / (float)A.nb;
  float v[B2_TRACKENV_NREW];
  float ep_ = 0.f, eq_ = 0.f, el_ = 0.f, ea_ = 0.f;
  if (hasb) {
    float dx = rel_p.x - pos.x, dy = rel_p.y - pos.y, dz = rel_p.z - pos.z;
    ep_ = dx * dx + dy * dy + dz * dz;
    float qe = qerr(rel_q, quat);
    eq_ = qe * qe;
    const V3 cl = ldv(A.m_body_lin + 3 * (fb + b)), ca = ldv(A.m_body_ang + 3 * (fb + b));
    el_ = (cl.x - lin.x) * (cl.x - lin.x) + (cl.y - lin.y) * (cl.y - lin.y) + (cl.z - lin.z) * (cl.z - lin.z);
    ea_ = (ca.x - ang.x) * (ca.x - ang.x) + (ca.y - ang.y) * (ca.y - ang.y) + (ca.z - ang.z) * (ca.z - ang.z);
  }
  const float dpx = a_pos.x - r_pos.x, dpy = a_pos.y - r_pos.y, dpz = a_pos.z - r_pos.z;
  const float e = qerr(a_quat, r_quat);
  v[0] = W[0] != 0.f ? W[0] * expf(-div_rn(dpx * dpx + dpy * dpy + dpz * dpz, A.std2[0])) : 0.f;
  v[1] = W[1] != 0.f ? W[1] * expf(-div_rn(e * e, A.std2[1])) : 0.f;
  v[2] = W[2] != 0.f ? W[2] * expf(-div_rn(wsum(ep_) * inb, A.std2[2])) : 0.f;
  v[3] = W[3] != 0.f ? W[3] * expf(-div_rn(wsum(eq_) * inb, A.std2[3])) : 0.f;
  v[4] = W[4] != 0.f ? W[4] * expf(-div_rn(wsum(el_) * inb, A.std2[4])) : 0.f;
  v[5] = W[5] != 0.f ? W[5] * expf(-div_rn(wsum(ea_) * inb, A.std2[5])) : 0.f;
  v[6] = W[6] != 0.f ? W[6] * wsum(rate) : 0.f;
  v[7] = W[7] != 0.f ? W[7] * wsum(lim) : 0.f;
  v[8] = W[8] != 0.f ? W[8] * dd.sensordata.p[(size_t)w * dd.sensordata.stride + A.self_collision_adr] : 0.f;
  float r = 0.f;
#pragma unroll
  for (int k = 0; k < B2_TRACKENV_NREW; k++) r += v[k];
  const float reward = r * A.step_dt;
  const bool done = term || trunc;
  if (A.episode_sums) {  // the episode logs and the motion errors
    const size_t row = (size_t)w * B2_TRACKENV_NREW;
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < B2_TRACKENV_NREW; k++) {
        const float s = A.episode_sums[row + k] + v[k] * A.step_dt;
        if (done) A.finished_sums[row + k] = s;
        A.episode_sums[row + k] = done ? 0.f : s;
      }
      float* f = A.term_flags + (size_t)w * B2_TRACKENV_NTERM;
      f[0] = trunc ? 1.f : 0.f; f[1] = bad_z ? 1.f : 0.f; f[2] = bad_ori ? 1.f : 0.f; f[3] = bad_ee ? 1.f : 0.f;
    }
    // motion errors: a done env hands over those of the last step's compute and takes new ones in post2, after the
    // forward; every other env takes them here, at its frame before the clip steps
    float* mm = A.motion_metrics + (size_t)w * B2_TRACKENV_NMETRIC;
    if (done) {
      if (lane < B2_TRACKENV_NMETRIC) A.finished_metrics[(size_t)w * B2_TRACKENV_NMETRIC + lane] = mm[lane];
    } else {
      const float* qvel = dd.qvel.p + (size_t)w * dd.qvel.stride;
      motion_errors(A, lane, hasb, b, ts, org, pos, quat, lin, ang, rel_p, rel_q, qpos, qvel, nu, mm);
    }
  }
  __syncwarp();  // every lane has read the pre-reset state
  if (lane == 0) {
    A.reward[w] = reward; A.terminated[w] = term; A.truncated[w] = trunc;
    A.log_row[3 * (size_t)w] = reward; A.log_row[3 * (size_t)w + 1] = term ? 1.f : 0.f;
    A.log_row[3 * (size_t)w + 2] = trunc ? 1.f : 0.f;
  }
  for (int a = lane; a < nu; a += 32) last[a] = done ? 0.f : act[a];
  // a failure counts in the bin of the frame the env reached (commands.py:257-265); time-outs and restarts do not
  if (A.adaptive == B2_START_ADAPTIVE && term && lane == 0) {
    const long long bin = ts * A.nbins / A.T;
    atomicAdd(A.bin_fail_cur + (bin < A.nbins - 1 ? bin : A.nbins - 1), 1.f);
  }
  // reset onto the clip (RSI), then the clip's time step; envs that ran off its end restart on it
  if (done) {
    ts = start_frame(A, U[0]);
    resample(dd, A, w, lane, nu, nbody, ts, U);
    ep = 0;
  }
  ts += 1;
  const bool ended = ts >= A.T;
  if (ended) {
    __syncwarp();
    ts = start_frame(A, U[S]);
    resample(dd, A, w, lane, nu, nbody, ts, U + S);
  }
  if (lane == 0) {
    A.time_steps[w] = ts;
    A.episode_length[w] = ep;
    A.mask[w] = done || ended;
  }
}

__global__ void b2_trackenv_post2_kernel(DevData dd, int nu, int nbody, B2TrackEnvArgs A) {
  using namespace b2t;
  const int lane = threadIdx.x & 31;
  const int w = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (w >= dd.nworld) return;
  const int S = 13 + nu;
  const float* U = A.U + (size_t)w * B2_TRACKENV_NU(nu);
  const float* P = U + 2 * S;       // push draws: 6 velocity + 1 timer
  const float* Z = U + 2 * S + 7;   // observation noise: anchor pos 3, anchor ori 6, base lin 3, base ang 3, jp nu, jv nu
  const float* qpos = dd.qpos.p + (size_t)w * dd.qpos.stride;
  float* qvel = dd.qvel.p + (size_t)w * dd.qvel.stride;
  const float* last = A.last_action + (size_t)w * nu;
  const long long ts = A.time_steps[w];
  const bool hasb = lane < A.nb;
  const int b = hasb ? lane : 0;
  const int bid = A.body_idx[b];
  const size_t fb = (size_t)ts * A.nb;
  const V3 pos = ldv(dd.xpos.p + (size_t)w * dd.xpos.stride + 3 * bid);
  const Q quat = ldq(dd.xquat.p + (size_t)w * dd.xquat.stride + 4 * bid);
  const V3 org = ldv(A.env_origins + 3 * (size_t)w);
  const V3 cpa = ldv(A.m_body_pos + 3 * (fb + A.anchor));
  const V3 a_pos = {cpa.x + org.x, cpa.y + org.y, cpa.z + org.z};
  const Q a_quat = ldq(A.m_body_quat + 4 * (fb + A.anchor));
  const V3 r_pos = bcastv(pos, A.anchor);
  const Q r_quat = bcastq(quat, A.anchor);
  // motion errors of a done env against its reset state, at the frame before the clip stepped and the targets of the
  // last command update (the reference's compute runs _update_metrics before _update_command)
  if (A.episode_sums && (A.terminated[w] || A.truncated[w])) {
    const float* lv = dd.link_vel_w.p + (size_t)w * dd.link_vel_w.stride + 6 * bid;
    const V3 rel_p = ldv(A.body_pos_rel + 3 * ((size_t)w * A.nb + b));
    const Q rel_q = ldq(A.body_quat_rel + 4 * ((size_t)w * A.nb + b));
    motion_errors(A, lane, hasb, b, ts > 0 ? ts - 1 : 0, org, pos, quat, {lv[0], lv[1], lv[2]}, {lv[3], lv[4], lv[5]},
                  rel_p, rel_q, qpos, qvel, nu, A.motion_metrics + (size_t)w * B2_TRACKENV_NMETRIC);
  }
  // command update: anchor-relative targets, yaw-aligned, height from the clip (commands.py:354-388)
  const Q dori = yaw_quat(qmul(r_quat, qinv(a_quat)));
  if (hasb) {
    const V3 cp = ldv(A.m_body_pos + 3 * (fb + b));
    const Q cq = ldq(A.m_body_quat + 4 * (fb + b));
    const Q rq = qmul(dori, cq);
    const V3 off = qapply(dori, {cp.x + org.x - a_pos.x, cp.y + org.y - a_pos.y, cp.z + org.z - a_pos.z});
    float* bp = A.body_pos_rel + 3 * ((size_t)w * A.nb + b);
    float* bq = A.body_quat_rel + 4 * ((size_t)w * A.nb + b);
    bp[0] = r_pos.x + off.x; bp[1] = r_pos.y + off.y; bp[2] = a_pos.z + off.z;
    bq[0] = rq.w; bq[1] = rq.x; bq[2] = rq.y; bq[3] = rq.z;
  }
  // interval push (push_by_setting_velocity, events.py:127-143) from the root's link velocity and orientation
  const float* pr = A.push_range;
  float tl = A.push_time_left[w] - A.step_dt;
  const bool push = A.push_on && tl <= 0.f;
  if (push) tl = P[6] * (A.push_hi - A.push_lo) + A.push_lo;
  if (lane == 0 && A.push_on) {
    if (push) {
      const float* rv = dd.link_vel_w.p + (size_t)w * dd.link_vel_w.stride + 6 * A.root_body;
      float v[6];
#pragma unroll
      for (int k = 0; k < 6; k++) v[k] = rv[k] + P[k] * (pr[2 * k + 1] - pr[2 * k]) + pr[2 * k];
      const Q rq = ldq(dd.xquat.p + (size_t)w * dd.xquat.stride + 4 * A.root_body);
      V3 ab = qapply_inv(rq, {v[3], v[4], v[5]});
      qvel[0] = v[0]; qvel[1] = v[1]; qvel[2] = v[2]; qvel[3] = ab.x; qvel[4] = ab.y; qvel[5] = ab.z;
    }
    A.push_time_left[w] = tl;
  }
  // observations (tracking_env_cfg.py:88-150): policy group with uniform noise, critic group privileged; without
  // state estimation the policy group has no anchor position and no base linear velocity
  const bool se = A.policy_state_estimation, noisy = A.policy_corruption;
  const int NP = se ? 5 * nu + 15 : 5 * nu + 9, NC = 5 * nu + 15 + 9 * A.nb;
  const int pj = NP - 3 * nu;            // policy: joint pos, joint vel, last action
  float* o = A.obs + (size_t)w * NP;
  float* cr = A.critic + (size_t)w * NC;
  const int cb = 2 * nu + 9;             // critic: body_pos_b / body_ori_b follow the anchor terms
  const int ct = cb + 9 * A.nb;          // critic: base_lin ... last_action
  for (int a = lane; a < nu; a += 32) {
    float cjp = A.m_joint_pos[(size_t)ts * nu + a], cjv = A.m_joint_vel[(size_t)ts * nu + a];
    o[a] = cjp; o[nu + a] = cjv; cr[a] = cjp; cr[nu + a] = cjv;
    float jp = qpos[7 + a] - A.default_joint_pos[a], jv = qvel[6 + a], la = last[a];
    o[pj + a] = noisy ? jp + (Z[15 + a] * 2.f - 1.f) * 0.01f : jp;
    o[pj + nu + a] = noisy ? jv + (Z[15 + nu + a] * 2.f - 1.f) * 0.5f : jv;
    o[pj + 2 * nu + a] = la;
    cr[ct + 6 + a] = jp; cr[ct + 6 + nu + a] = jv; cr[ct + 6 + 2 * nu + a] = la;
  }
  const V3 apb = qapply_inv(r_quat, {a_pos.x - r_pos.x, a_pos.y - r_pos.y, a_pos.z - r_pos.z});
  float aob[6];
  rot6(qmul(qinv(r_quat), a_quat), aob);
  const float* sb = dd.link_state_b.p + (size_t)w * dd.link_state_b.stride + 10 * A.root_body;
  if (lane == 0) {
    const float ap[3] = {apb.x, apb.y, apb.z};
    const int po = se ? 2 * nu + 3 : 2 * nu, pa = se ? 2 * nu + 12 : 2 * nu + 6;  // anchor ori, base ang
    for (int k = 0; k < 3; k++) {
      if (se) o[2 * nu + k] = noisy ? ap[k] + (Z[k] * 2.f - 1.f) * 0.25f : ap[k];
      cr[2 * nu + k] = ap[k];
    }
    for (int k = 0; k < 6; k++) { o[po + k] = noisy ? aob[k] + (Z[3 + k] * 2.f - 1.f) * 0.05f : aob[k]; cr[2 * nu + 3 + k] = aob[k]; }
    for (int k = 0; k < 3; k++) {
      if (se) o[2 * nu + 9 + k] = noisy ? sb[k] + (Z[9 + k] * 2.f - 1.f) * 0.5f : sb[k];
      o[pa + k] = noisy ? sb[3 + k] + (Z[12 + k] * 2.f - 1.f) * 0.2f : sb[3 + k];
      cr[ct + k] = sb[k]; cr[ct + 3 + k] = sb[3 + k];
    }
  }
  if (hasb) {
    const V3 pb = qapply_inv(r_quat, {pos.x - r_pos.x, pos.y - r_pos.y, pos.z - r_pos.z});
    float ob[6];
    rot6(qmul(qinv(r_quat), quat), ob);
    cr[cb + 3 * b] = pb.x; cr[cb + 3 * b + 1] = pb.y; cr[cb + 3 * b + 2] = pb.z;
    for (int k = 0; k < 6; k++) cr[cb + 3 * A.nb + 6 * b + k] = ob[k];
  }
}

// Adaptive start-frame sampler (commands.py:256-297, EMA :394-398), one CTA of kBinThreads between post1 and the
// masked forward: (1) metrics of the distribution post1 drew from, i.e. the one of the EMA before this step's
// update; (2) EMA update, this step's counts cleared; (3) CDF of the next step's distribution.  Any nbins: every
// pass loops over the bins, and the prefix sum walks contiguous per-thread chunks in a fixed order.
__global__ void __launch_bounds__(b2t::kBinThreads) b2_trackenv_bins_kernel(B2TrackEnvArgs A) {
  using namespace b2t;
  __shared__ float red[kBinThreads / 32];
  __shared__ int redi[kBinThreads / 32];
  const int t = threadIdx.x, lane = t & 31, nbins = A.nbins;
  const float floor_ = A.adaptive_uniform_ratio / (float)nbins;
  // (1) normalised entropy and top-1 bin (first index among equal maxima, as torch.max)
  float tot = weight_total(A, floor_, red);
  float h = 0.f, best = -1.f;
  int besti = 0;
  for (int b = t; b < nbins; b += kBinThreads) {
    const float p = div_rn(bin_weight(A, b, floor_), tot);
    h -= p * (float)log((double)(p + 1e-12f));  // (double: logf is approximate under --use_fast_math)
    if (p > best) { best = p; besti = b; }
  }
  h = cta_sum(h, red);
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
    if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
  }
  if (lane == 0) { red[t >> 5] = best; redi[t >> 5] = besti; }
  __syncthreads();
  if (t == 0) {
    for (int k = 1; k < kBinThreads / 32; k++)
      if (red[k] > best || (red[k] == best && redi[k] < besti)) { best = red[k]; besti = redi[k]; }
    A.metrics[0] = nbins > 1 ? h / logf((float)nbins) : 1.f;  // one bin: the uniform distribution over the clip
    A.metrics[1] = best;
    A.metrics[2] = (float)besti / (float)nbins;
  }
  __syncthreads();
  // (2) EMA of the failure counts
  for (int b = t; b < nbins; b += kBinThreads) {
    A.bin_fail_ema[b] = A.adaptive_alpha * A.bin_fail_cur[b] + (1.f - A.adaptive_alpha) * A.bin_fail_ema[b];
    A.bin_fail_cur[b] = 0.f;
  }
  __syncthreads();
  // (3) CDF: exclusive scan of the per-thread chunk sums, then each chunk in order
  tot = weight_total(A, floor_, red);
  const int chunk = (nbins + kBinThreads - 1) / kBinThreads, b0 = min(t * chunk, nbins), b1 = min(b0 + chunk, nbins);
  float own = 0.f;
  for (int b = b0; b < b1; b++) own += div_rn(bin_weight(A, b, floor_), tot);
  float inc = own;
  for (int o = 1; o < 32; o <<= 1) {
    const float v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) red[t >> 5] = inc;
  __syncthreads();
  float run = inc - own;
  for (int k = 0; k < (t >> 5); k++) run += red[k];
  for (int b = b0; b < b1; b++) {
    run += div_rn(bin_weight(A, b, floor_), tot);
    A.cdf[b] = b == nbins - 1 ? 1.f : run;  // the last step ends at 1 exactly: every u < 1 finds a bin
  }
}

// b2_env.cuh — fused MDP glue of the velocity-tracking task around the physics step (SURVEY.md §8f items
// 1-3): the caller-side work of ManagerBasedRlEnv.step (reference src/mjlab/envs/manager_based_rl_env.py:106-147
// with the terms of tasks/velocity/velocity_env_cfg.py) as two kernels instead of ~90 tiny torch launches:
//   pre  : ctrl = default_joint_pos + action_scale * action                     (joint_actions.py:85-103)
//   post : episode counter, terminations (bad_orientation, time_out), rewards (the five fixed terms, the opt-in terms
//          of B2VelEnvArgs.weight and their episode sums), the terrain-level curriculum of
//          the reset envs (opt-in, curriculums.py:18-52), masked reset (events.py:43-124), interval push
//          (events.py:127-143), command resample (configurable ranges, the opt-in command-velocity curriculum and
//          the command's metrics), observations.
// The torch implementation in mjlab_b200/envs/velocity_env.py is the reference; both consume the same
// per-step uniform numbers U[n][B2_VELENV_NU(nu)] (layout in include/b2sim.h) so they can be compared on one state
// (tests/test_mdp_kernels.py).
#pragma once
#include "../../include/b2sim.h"
#include "b2_types.h"

// B2VelEnvArgs is declared in include/b2sim.h (it is part of the C ABI).

__device__ __forceinline__ void b2e_rot_inv(const float* q, const float* v, float* r) {
  // r = R(q)^T v
  float t0 = 2.f * (q[2] * v[2] - q[3] * v[1]);
  float t1 = 2.f * (q[3] * v[0] - q[1] * v[2]);
  float t2 = 2.f * (q[1] * v[1] - q[2] * v[0]);
  r[0] = v[0] - q[0] * t0 + (q[2] * t2 - q[3] * t1);
  r[1] = v[1] - q[0] * t1 + (q[3] * t0 - q[1] * t2);
  r[2] = v[2] - q[0] * t2 + (q[1] * t1 - q[2] * t0);
}

__global__ void b2_velenv_pre_kernel(DevData dd, int nu, const float* __restrict__ action,
                                     const float* __restrict__ default_joint_pos,
                                     const float* __restrict__ action_scale) {
  long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= (long long)dd.nworld * nu) return;
  int w = (int)(tid / nu), a = (int)(tid % nu);
  dd.ctrl.p[(size_t)w * dd.ctrl.stride + a] = default_joint_pos[a] + action_scale[a] * action[tid];
}

__device__ __forceinline__ float b2e_wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// IEEE-rounded products, sums and square roots: the library builds with --use_fast_math (approximate sqrt, FMA
// contraction), but a terrain level must move exactly as on the torch path
#ifdef B2_HOST_EMULATION
__device__ __forceinline__ float b2e_mul_rn(float a, float b) { return a * b; }
__device__ __forceinline__ float b2e_add_rn(float a, float b) { return a + b; }
__device__ __forceinline__ float b2e_norm2_rn(float x, float y) { return sqrtf(x * x + y * y); }
#else
__device__ __forceinline__ float b2e_mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float b2e_add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float b2e_norm2_rn(float x, float y) {
  return __fsqrt_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
}
#endif

// Terrain-level curriculum of a reset env (B2VelEnvArgs, terrain_levels_vel + update_env_origins), on one lane: from
// the root position (x, y) and the command (c0, c1) of the episode that just ended, move the env's level and write
// the origin the reset spawns at.
__device__ __forceinline__ void b2e_terrain_level(const B2VelEnvArgs& A, int w, float x, float y, float c0, float c1,
                                                  float u) {
  float* org = A.env_origins + 3 * (size_t)w;
  const float dist = b2e_norm2_rn(x - org[0], y - org[1]);
  const bool up = dist > A.move_up_dist;
  const bool down = !up && dist < b2e_mul_rn(b2e_norm2_rn(c0, c1), A.episode_length_s) * 0.5f;
  int level = A.terrain_levels[w] + (up ? 1 : 0) - (down ? 1 : 0);
  level = level >= A.rows ? min((int)floorf(b2e_mul_rn(u, (float)A.rows)), A.rows - 1) : max(level, 0);
  A.terrain_levels[w] = level;
  const float* src = A.terrain_origins + 3 * ((size_t)level * A.cols + A.terrain_types[w]);
  org[0] = src[0]; org[1] = src[1]; org[2] = src[2];
}

// World-frame linear velocity (x, y) and height of geom g on body b (EntityData.geom_vel_w, entity/data.py:20-31,
// 282-288): cvel[3:6] - cvel[0:3] x (subtree_com[root] - geom_xpos).
__device__ __forceinline__ void b2e_geom_vel(const DevData& dd, int w, int g, int b, int root, float& vx, float& vy,
                                             float& z) {
  const float* p = dd.geom_xpos.p + (size_t)w * dd.geom_xpos.stride + 3 * g;
  const float* s = dd.subtree_com.p + (size_t)w * dd.subtree_com.stride + 3 * root;
  const float* c = dd.cvel.p + (size_t)w * dd.cvel.stride + 6 * b;
  const float o0 = s[0] - p[0], o1 = s[1] - p[1], o2 = s[2] - p[2];
  vx = c[3] - (c[1] * o2 - c[2] * o1);
  vy = c[4] - (c[2] * o0 - c[0] * o2);
  z = p[2];
}

// The reset state terms of a reset env (B2VelEnvArgs.reset_term), after the built-in reset has written the env's rows
__device__ __forceinline__ void b2e_reset_terms(const B2VelEnvArgs& A, float* qpos, float* qvel, int w, int lane) {
  const float* V = A.ev_V + (size_t)w * A.ev_v_width;
  for (int t = 0; t < A.n_reset; t++) {
    const int col = A.reset_term[t].col, count = A.reset_term[t].count;
    if (A.reset_term[t].kind == B2_RESET_ROOT) {
      if (lane == 0) {
        float d[12];
#pragma unroll
        for (int k = 0; k < 12; k++) d[k] = b2e_add_rn(b2e_mul_rn(V[col + k], A.reset_term[t].span[k]), A.reset_term[t].lo[k]);
        const float* org = A.env_origins + 3 * (size_t)w;
#pragma unroll
        for (int k = 0; k < 3; k++) qpos[k] = b2e_add_rn(b2e_add_rn(A.default_qpos[k], d[k]), org[k]);
        const float cr = cosf(d[3] * 0.5f), sr = sinf(d[3] * 0.5f), cp = cosf(d[4] * 0.5f), sp = sinf(d[4] * 0.5f);
        const float cy = cosf(d[5] * 0.5f), sy = sinf(d[5] * 0.5f);
        const float e[4] = {cy * cr * cp + sy * sr * sp, cy * sr * cp - sy * cr * sp, cy * cr * sp + sy * sr * cp,
                            sy * cr * cp - cy * sr * sp};
        const float* a = A.default_qpos + 3;
        float q[4] = {a[0] * e[0] - a[1] * e[1] - a[2] * e[2] - a[3] * e[3], a[0] * e[1] + a[1] * e[0] + a[2] * e[3] - a[3] * e[2],
                      a[0] * e[2] - a[1] * e[3] + a[2] * e[0] + a[3] * e[1], a[0] * e[3] + a[1] * e[2] - a[2] * e[1] + a[3] * e[0]};
        const float ang[3] = {d[9], d[10], d[11]};
        float ab[3];
        b2e_rot_inv(q, ang, ab);
        qpos[3] = q[0]; qpos[4] = q[1]; qpos[5] = q[2]; qpos[6] = q[3];
        qvel[0] = d[6]; qvel[1] = d[7]; qvel[2] = d[8]; qvel[3] = ab[0]; qvel[4] = ab[1]; qvel[5] = ab[2];
      }
    } else {
      const float plo = A.reset_term[t].lo[0], pspan = A.reset_term[t].span[0];
      const float vlo = A.reset_term[t].lo[1], vspan = A.reset_term[t].span[1];
      for (int j = lane; j < count; j += 32) {
        const int a = A.reset_term[t].joint[j];
        const float jp = b2e_mul_rn(A.default_joint_pos[a], b2e_add_rn(b2e_mul_rn(V[col + j], pspan), plo));
        qpos[7 + a] = fminf(fmaxf(jp, A.soft_lo[a]), A.soft_hi[a]);
        qvel[6 + a] = b2e_mul_rn(0.f, b2e_add_rn(b2e_mul_rn(V[col + count + j], vspan), vlo));
      }
    }
    __syncwarp();
  }
}

// feet_air_time (tasks/velocity/mdp/rewards.py:52-146) on one lane per foot: advances the foot's state (zeroed when
// the env is done, as reset(env_ids) does) and returns the warp's reward before the command scale.
__device__ __forceinline__ float b2e_air_time(const B2VelEnvArgs& A, const float* sd, int w, int lane, bool done) {
  float r = 0.f;
  if (lane < A.n_air) {
    const size_t k = (size_t)w * A.n_air + lane;
    const bool contact = sd[A.air_sensor_adr[lane]] > 0.f;
    float air = A.air_time[k], ct = A.contact_time[k], last = A.last_air_time[k];
    const bool first = air > 0.f && contact;  // landing: from the air time before this step's update
    if (first) last = air;
    air = contact ? 0.f : b2e_add_rn(air, A.step_dt);
    ct = contact ? b2e_add_rn(ct, A.step_dt) : 0.f;
    if (A.air_continuous)
      r = !contact && air > A.air_threshold_min && air <= A.air_threshold_max ? 1.f : 0.f;
    else if (first)
      r = fminf(fmaxf(last - A.air_threshold_min, 0.f), A.air_threshold_max - A.air_threshold_min);
    A.air_time[k] = done ? 0.f : air;
    A.contact_time[k] = done ? 0.f : ct;
    A.last_air_time[k] = done ? 0.f : last;
  }
  r = b2e_wsum(r);
  return A.air_continuous ? r : r / A.step_dt;
}

// One warp per environment (a thread per environment left 4096 threads = 128 warps on 132 SMs walking ~400
// dependent loads each: pure latency on the critical path of every env step).  Scalar terms are computed
// redundantly by every lane from values read before any lane writes; per-joint terms are spread over the lanes.
__global__ void b2_velenv_post_kernel(DevData dd, int nq, int nv, int nu, B2VelEnvArgs A) {
  const int lane = threadIdx.x & 31;
  const int w = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (w >= dd.nworld) return;
  float* qpos = dd.qpos.p + (size_t)w * dd.qpos.stride;
  float* qvel = dd.qvel.p + (size_t)w * dd.qvel.stride;
  float* ctrl = dd.ctrl.p + (size_t)w * dd.ctrl.stride;
  const float* act = A.action + (size_t)w * nu;
  const int NUU = B2_VELENV_NU(nu);
  const float* U = A.U + (size_t)w * NUU;
  float* last = A.last_action + (size_t)w * nu;
  float* cmd = A.command + 3 * (size_t)w;
  int ep = A.episode_length[w] + 1;
  const float down[3] = {0.f, 0.f, -1.f};
  float q[4] = {qpos[3], qpos[4], qpos[5], qpos[6]}, gb[3], lb[3];
  float c0 = cmd[0], c1 = cmd[1], c2 = cmd[2];
  float ctl = A.cmd_time_left[w] - A.step_dt, tl = A.push_time_left[w] - (A.push_off ? 0.f : A.step_dt);
  float htarget = A.heading_target[w];
  bool standing = A.is_standing[w] != 0;
  const float v0 = qvel[0], v1 = qvel[1], v2 = qvel[2], wz = qvel[5];
  // ranges of lin_vel_x and ang_vel_z in this step: the cfg's, or the last curriculum stage the counter has passed
  float xm = A.cmd_mid[0], xh = A.cmd_half[0], zm = A.cmd_mid[2], zh = A.cmd_half[2], zlo = A.ang_lo, zhi = A.ang_hi;
  if (A.n_stage > 0) {
    const int counter = *A.step_counter + 1;
#pragma unroll
    for (int s = 0; s < B2_VELENV_NSTAGE; s++)
      if (s < A.n_stage && counter > A.stage_step[s]) {
        xm = zm = A.stage_mid[s]; xh = zh = A.stage_half[s]; zlo = A.stage_lo[s]; zhi = A.stage_hi[s];
      }
  }
  b2e_rot_inv(q, down, gb);
  bool term = acosf(fminf(fmaxf(-gb[2], -1.f), 1.f)) > A.fall_angle;  // bad_orientation
  bool trunc = ep >= A.max_episode_length;                              // time_out
  // rewards (velocity_env_cfg.py:183-214)
  float lin[3] = {v0, v1, v2};
  b2e_rot_inv(q, lin, lb);
  float e0 = c0 - lb[0], e1 = c1 - lb[1], e2 = c2 - wz;
  float r_lin = expf(-(e0 * e0 + e1 * e1) / 0.25f), r_ang = expf(-(e2 * e2) / 0.25f);
  float pose = 0.f, lim = 0.f, rate = 0.f;
  for (int a = lane; a < nu; a += 32) {
    float jp = qpos[7 + a], dj = jp - A.default_joint_pos[a];
    pose += dj * dj * A.posture_inv_std2[a];
    lim += fmaxf(A.soft_lo[a] - jp, 0.f) + fmaxf(jp - A.soft_hi[a], 0.f);
    float da = act[a] - last[a];
    rate += da * da;
  }
  pose = b2e_wsum(pose); lim = b2e_wsum(lim); rate = b2e_wsum(rate);
  bool done = term || trunc;
  // opt-in terms: r[i] is term 5 + i unweighted, evaluated only at a non-zero weight
  float r[B2_VELENV_NTERM - 5] = {}, extra = 0.f;
  const float* W = A.weight;
  const float* sd = dd.sensordata.p + (size_t)w * dd.sensordata.stride;
  if (W[0] != 0.f) {  // air_time, scaled by the command (smooth or hard)
    const float cn = b2e_norm2_rn(c0, c1);
    const float s = A.air_hard_scale ? (cn > A.air_command_threshold ? 1.f : 0.f)
                                     : 0.5f * (1.f + tanhf((cn - A.air_command_threshold) / A.air_command_scale_width));
    r[0] = b2e_air_time(A, sd, w, lane, done) * s;
  }
  if (W[1] != 0.f) {  // feet_slide
    float v = 0.f;
    if (lane < A.n_slide && sd[A.slide_sensor_adr[lane]] > 0.f) {
      float vx, vy, z;
      b2e_geom_vel(dd, w, A.slide_geom[lane], A.slide_body[lane], A.root_body, vx, vy, z);
      v = sqrtf(vx * vx + vy * vy);
    }
    r[1] = b2e_wsum(v);
  }
  if (W[2] != 0.f) {  // foot_clearance_reward
    float v = 0.f;
    if (lane < A.n_clear) {
      float vx, vy, z;
      b2e_geom_vel(dd, w, A.clear_geom[lane], A.clear_body[lane], A.root_body, vx, vy, z);
      const float e = z - A.clearance_target_height;
      v = e * e * tanhf(A.clearance_tanh_mult * sqrtf(vx * vx + vy * vy));
    }
    r[2] = expf(-b2e_wsum(v) / A.clearance_std);
  }
  r[3] = term ? 0.f : 1.f;  // is_alive
  r[4] = term ? 1.f : 0.f;  // is_terminated
  if (W[5] != 0.f || W[6] != 0.f || W[7] != 0.f) {  // joint_torques_l2, joint_acc_l2, electrical_power_cost
    const float* af = dd.actuator_force.p + (size_t)w * dd.actuator_force.stride;
    const float* qa = dd.qacc.p + (size_t)w * dd.qacc.stride;
    float tau = 0.f, acc = 0.f, pw = 0.f;
    for (int a = lane; a < nu; a += 32) {
      const float f = af[a], j = qa[6 + a];
      tau += f * f;
      acc += j * j;
      pw += fmaxf(f * qvel[6 + a], 0.f);
    }
    r[5] = b2e_wsum(tau); r[6] = b2e_wsum(acc); r[7] = b2e_wsum(pw);
  }
  r[8] = gb[0] * gb[0] + gb[1] * gb[1];  // flat_orientation_l2
#pragma unroll
  for (int i = 0; i < B2_VELENV_NTERM - 5; i++) {
    r[i] = W[i] != 0.f ? r[i] * W[i] : 0.f;  // (a term at weight 0 adds nothing, not 0 * its value)
    extra += r[i];
  }
  __syncwarp();  // every lane holds the pre-reset state it needs; writes may start
  float r_pose = expf(-(pose / (float)nu));
  const float fixed = r_lin + r_ang + r_pose - lim - 0.1f * rate;
  const float reward = (fixed + extra) * A.step_dt;
  if (lane == 0) {
    A.reward[w] = reward;
    A.terminated[w] = term; A.truncated[w] = trunc; A.done[w] = done;
    A.log_row[3 * (size_t)w] = reward; A.log_row[3 * (size_t)w + 1] = term ? 1.f : 0.f;
    A.log_row[3 * (size_t)w + 2] = trunc ? 1.f : 0.f;
  }
  // episode sums (RewardManager.compute / reset): column k on lane k
  if (lane < B2_VELENV_NTERM) {
    float v = lane == 0 ? r_lin : lane == 1 ? r_ang : lane == 2 ? r_pose : lane == 3 ? -lim : lane == 4 ? -0.1f * rate : 0.f;
#pragma unroll
    for (int i = 0; i < B2_VELENV_NTERM - 5; i++)
      if (lane == 5 + i) v = r[i];
    const size_t k = (size_t)w * B2_VELENV_NTERM + lane;
    const float s = A.episode_sums[k] + v * A.step_dt;
    if (done) A.finished_sums[k] = s;
    A.episode_sums[k] = done ? 0.f : s;
  }
  // masked reset (reset_root_state_uniform + reset_joints_by_scale), command resample
  if (done) {
    if (A.curriculum) {  // before the reset events (manager_based_rl_env.py:205-208), from the pre-reset state
      if (lane == 0) b2e_terrain_level(A, w, qpos[0], qpos[1], c0, c1, U[12]);
      __syncwarp();  // every lane spawns at the new origin
    }
    for (int i = lane; i < nq; i += 32) {
      float v = A.default_qpos[i];
      if (i == 0) v += (U[0] - 0.5f) + A.env_origins[3 * (size_t)w];
      if (i == 1) v += (U[1] - 0.5f) + A.env_origins[3 * (size_t)w + 1];
      if (i == 2) v += A.env_origins[3 * (size_t)w + 2];  // terrain spawn height (0 on the flat scene)
      if (i == 3 || i == 6) {
        float yaw = (U[2] * 2.f - 1.f) * 3.14f;
        v = i == 3 ? cosf(0.5f * yaw) : sinf(0.5f * yaw);
      }
      if (i >= 7) v = fminf(fmaxf(v, A.soft_lo[i - 7]), A.soft_hi[i - 7]);
      qpos[i] = v;
    }
    for (int a = lane; a < nu; a += 32) { ctrl[a] = A.default_joint_pos[a]; last[a] = 0.f; }
    for (int i = lane; i < nv; i += 32) qvel[i] = 0.f;
    if (A.n_reset > 0) {
      __syncwarp();  // the built-in rows are written; the terms replace theirs
      b2e_reset_terms(A, qpos, qvel, w, lane);
    }
    ep = 0;
  } else {
    for (int a = lane; a < nu; a += 32) last[a] = act[a];
  }
  // command term (CommandTerm.compute + UniformVelocityCommand, velocity_command.py:64-110): resample on
  // reset and when the timer runs out, then heading control and standing envs every step.  mid + (2u - 1) half
  // is rounded as written (no contraction), so that at the default ranges it is bit-identical to 2u - 1, u - 0.5 and
  // (2u - 1) pi (scaling by 2 is exact)
  const float o0 = c0, o1 = c1, o2 = c2;  // the command before this step's resample (metrics)
  if (done || ctl <= 0.f) {
    c0 = b2e_add_rn(xm, b2e_mul_rn(U[3] * 2.f - 1.f, xh));
    c1 = b2e_add_rn(A.cmd_mid[1], b2e_mul_rn(U[4] * 2.f - 1.f, A.cmd_half[1]));
    c2 = b2e_add_rn(zm, b2e_mul_rn(U[5] * 2.f - 1.f, zh));
    htarget = b2e_add_rn(A.cmd_mid[3], b2e_mul_rn(U[6] * 2.f - 1.f, A.cmd_half[3]));
    standing = U[7] <= A.rel_standing;
    ctl = A.resample_lo + A.resample_span * U[8];
  }
  __syncwarp();  // the reset state is visible to every lane
  {
    // heading_w = atan2 of the body x axis in the world (entity/data.py:480-484), from the post-reset pose
    float qw = qpos[3], qx = qpos[4], qy = qpos[5], qz = qpos[6];
    if (lane == 0) {
      // metrics (CommandTerm.reset, then _update_metrics in compute): a done env hands its sums over and restarts;
      // the increment takes the fresh draw of a done env and every other env's command from before the resample,
      // with the velocity of the post-reset state (before the push)
      float qq[4] = {qw, qx, qy, qz}, vw[3] = {qvel[0], qvel[1], qvel[2]}, vb[3];
      b2e_rot_inv(qq, vw, vb);
      const float ex = (done ? c0 : o0) - vb[0], ey = (done ? c1 : o1) - vb[1];
      const float exy = sqrtf(ex * ex + ey * ey) / A.metric_steps;
      const float eyaw = fabsf((done ? c2 : o2) - qvel[5]) / A.metric_steps;
      const float mxy = A.metric_xy[w], myaw = A.metric_yaw[w];
      if (done) { A.finished_metrics[2 * (size_t)w] = mxy; A.finished_metrics[2 * (size_t)w + 1] = myaw; }
      A.metric_xy[w] = (done ? 0.f : mxy) + exy;
      A.metric_yaw[w] = (done ? 0.f : myaw) + eyaw;
    }
    float fx = 1.f - 2.f * (qy * qy + qz * qz), fy = 2.f * (qx * qy + qw * qz);
    float err = htarget - atan2f(fy, fx);
    err -= 6.28318530717959f * floorf((err + 3.14159265358979f) / 6.28318530717959f);  // wrap_to_pi
    c2 = fminf(fmaxf(A.heading_stiffness * err, zlo), zhi);
    if (standing) { c0 = 0.f; c1 = 0.f; c2 = 0.f; }
  }
  // interval event: push_by_setting_velocity
  float pv0 = qvel[0], pv1 = qvel[1];
  const bool push = !A.push_off && tl <= 0.f;
  if (push) {
    pv0 = (U[9] * 2.f - 1.f) * A.push_vel;
    pv1 = (U[10] * 2.f - 1.f) * A.push_vel;
    tl = U[11] * (A.push_hi - A.push_lo) + A.push_lo;
  }
  __syncwarp();
  if (lane == 0) {
    A.episode_length[w] = ep;
    cmd[0] = c0; cmd[1] = c1; cmd[2] = c2;
    A.heading_target[w] = htarget; A.is_standing[w] = standing; A.cmd_time_left[w] = ctl;
    A.push_time_left[w] = tl;
    if (push) { qvel[0] = pv0; qvel[1] = pv1; }
  }
  // observations from the (possibly reset / pushed) state
  // policy group with uniform noise (velocity_env_cfg.py:86-118), critic group without (:120-125)
  float* o = A.obs + (size_t)w * (9 + 3 * nu + 3);
  float* cr = A.critic + (size_t)w * (9 + 3 * nu + 3);
  const float* Z = U + 16;  // noise draws
  float q2[4] = {qpos[3], qpos[4], qpos[5], qpos[6]}, lin2[3] = {pv0, pv1, qvel[2]};
  b2e_rot_inv(q2, lin2, lb);
  b2e_rot_inv(q2, down, gb);
  if (lane < 3) {
    const int k = lane;
    const float av = qvel[3 + k];
    // (selects, not lb[k]: an array indexed by the lane would be placed in local memory)
    const float lk = k == 0 ? lb[0] : (k == 1 ? lb[1] : lb[2]), gk = k == 0 ? gb[0] : (k == 1 ? gb[1] : gb[2]);
    cr[k] = lk; cr[3 + k] = av; cr[6 + k] = gk;
    o[k] = lk + (Z[k] * 2.f - 1.f) * 0.1f;
    o[3 + k] = av + (Z[3 + k] * 2.f - 1.f) * 0.2f;
    o[6 + k] = gk + (Z[6 + k] * 2.f - 1.f) * 0.05f;
    const float ck = k == 0 ? c0 : (k == 1 ? c1 : c2);
    o[9 + 3 * nu + k] = ck; cr[9 + 3 * nu + k] = ck;
  }
  for (int a = lane; a < nu; a += 32) {
    float jp = qpos[7 + a] - A.default_joint_pos[a], jv = qvel[6 + a], la = last[a];
    cr[9 + a] = jp; cr[9 + nu + a] = jv; cr[9 + 2 * nu + a] = la;
    o[9 + a] = jp + (Z[9 + a] * 2.f - 1.f) * 0.01f;
    o[9 + nu + a] = jv + (Z[9 + nu + a] * 2.f - 1.f) * 1.5f;
    o[9 + 2 * nu + a] = la;
  }
}

// common_step_counter += 1 after the post kernel, launched only with the command-velocity curriculum on: the post
// kernel's warps all read the counter, so none of them can advance it.
__global__ void b2_velenv_counter_kernel(int32_t* __restrict__ counter) { *counter += 1; }

// Mean terrain level after the post kernel's curriculum update, the value terrain_levels_vel returns for logging: one
// CTA, launched only when the curriculum is on.  The sum of integer levels is exact in any order, so no accumulator
// has to be zeroed before the post kernel and the value is the same from run to run.
constexpr int kLevelMeanThreads = 256;
__global__ void __launch_bounds__(kLevelMeanThreads) b2_velenv_level_mean_kernel(int n, const int32_t* __restrict__ levels,
                                                                                float* __restrict__ mean) {
  __shared__ int part[kLevelMeanThreads / 32];
  int s = 0;
  for (int i = threadIdx.x; i < n; i += kLevelMeanThreads) s += levels[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    s = 0;
    for (int k = 0; k < kLevelMeanThreads / 32; k++) s += part[k];
#ifdef B2_HOST_EMULATION
    *mean = (float)s / (float)n;
#else
    *mean = __fdiv_rn((float)s, (float)n);
#endif
  }
}

// b2_events.cuh — the reset and interval randomize_field events of the fused environments (the reference's
// EventManager.apply("reset") / apply("interval") / reset, managers/event_manager.py:76-167, with randomize_field,
// envs/mdp/events.py:212-397), one launch per env step inside the captured step.  The torch implementation in
// mjlab_b200/envs/events.py is the reference (tests/test_events.py).
//
// One warp per env.  The terms run in table order; lane 0 owns an interval term's timer and hands its decision to the
// warp, the lanes share a firing term's (element, axis) entries.  A __syncwarp after each term orders two terms that
// write the same element, so the result does not depend on which lane held it.  No atomics: each env's rows belong to
// its warp.
#pragma once
#include "../../include/b2sim.h"

// The fields a term writes, resolved by b2_events from the model-field table.
struct B2EventFields {
  float* row[B2_EVENTS_NTERM];    // world 0's row
  int stride[B2_EVENTS_NTERM];    // floats from one world's row to the next
  // the state the state terms read and write (DevData rows, world 0)
  float *qpos, *qvel, *xfrc;
  const float *xpos, *xquat, *subtree_com, *cvel;
  int qpos_s, qvel_s, xfrc_s, xpos_s, xquat_s, subtree_com_s, cvel_s;
};

// One IEEE fp32 product / sum: the library builds with --use_fast_math, and the draws must be the ones torch computes
// (lo + u span: one product, then one sum; no contraction into an FMA, no flushed subnormals).
__device__ __forceinline__ float b2e_mul(float a, float b) {
#ifdef B2_HOST_EMULATION
  return a * b;
#else
  return __fmul_rn(a, b);
#endif
}
__device__ __forceinline__ float b2e_add(float a, float b) {
#ifdef B2_HOST_EMULATION
  return a + b;
#else
  return __fadd_rn(a, b);
#endif
}

// v + R(q) a (sign +1) or R(q)^T a (sign -1), q = (w, x, y, z) of unit norm
__device__ __forceinline__ void b2e_qrot(const float* q, const float* a, float sign, float* r) {
  const float x = sign * q[1], y = sign * q[2], z = sign * q[3];
  const float t0 = 2.f * (y * a[2] - z * a[1]), t1 = 2.f * (z * a[0] - x * a[2]), t2 = 2.f * (x * a[1] - y * a[0]);
  r[0] = a[0] + q[0] * t0 + (y * t2 - z * t1);
  r[1] = a[1] + q[0] * t1 + (z * t0 - x * t2);
  r[2] = a[2] + q[0] * t2 + (x * t1 - y * t0);
}

// push_by_setting_velocity of env w on one lane (B2EventArgs.state, PUSH)
__device__ __forceinline__ void b2e_push(const B2EventArgs& A, const B2EventFields& F, int t, const float* v, int w) {
  float* qv = F.qvel + (size_t)w * F.qvel_s;
  float q[4], lin[3], ang[3];
  if (A.refreshed[w]) {  // the state this step wrote; the masked forward after this launch has not seen it yet
    const float* qp = F.qpos + (size_t)w * F.qpos_s;
    const float s = rsqrtf(qp[3] * qp[3] + qp[4] * qp[4] + qp[5] * qp[5] + qp[6] * qp[6]);
    q[0] = qp[3] * s; q[1] = qp[4] * s; q[2] = qp[5] * s; q[3] = qp[6] * s;
    const float wb[3] = {qv[3], qv[4], qv[5]};
    lin[0] = qv[0]; lin[1] = qv[1]; lin[2] = qv[2];
    b2e_qrot(q, wb, 1.f, ang);
  } else {  // compute_velocity_from_cvel (entity/data.py:20-31) at the root link
    const int b = A.root_body;
    const float* c = F.cvel + (size_t)w * F.cvel_s + 6 * b;
    const float* p = F.xpos + (size_t)w * F.xpos_s + 3 * b;
    const float* sc = F.subtree_com + (size_t)w * F.subtree_com_s + 3 * b;
    const float* xq = F.xquat + (size_t)w * F.xquat_s + 4 * b;
    const float o0 = sc[0] - p[0], o1 = sc[1] - p[1], o2 = sc[2] - p[2];
    lin[0] = c[3] - (c[1] * o2 - c[2] * o1);
    lin[1] = c[4] - (c[2] * o0 - c[0] * o2);
    lin[2] = c[5] - (c[0] * o1 - c[1] * o0);
    ang[0] = c[0]; ang[1] = c[1]; ang[2] = c[2];
    q[0] = xq[0]; q[1] = xq[1]; q[2] = xq[2]; q[3] = xq[3];
  }
  float d[6];
#pragma unroll
  for (int k = 0; k < 6; k++) d[k] = b2e_add(b2e_mul(v[A.state[t].col + k], A.state[t].span6[k]), A.state[t].lo6[k]);
  const float aw[3] = {b2e_add(ang[0], d[3]), b2e_add(ang[1], d[4]), b2e_add(ang[2], d[5])};
  float ab[3];
  b2e_qrot(q, aw, -1.f, ab);
  qv[0] = b2e_add(lin[0], d[0]); qv[1] = b2e_add(lin[1], d[1]); qv[2] = b2e_add(lin[2], d[2]);
  qv[3] = ab[0]; qv[4] = ab[1]; qv[5] = ab[2];
}

__global__ void b2_events_kernel(int n, B2EventArgs A, B2EventFields F) {
  const int w = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= n) return;  // (whole warps: blockDim is a multiple of 32)
  const bool reset = A.terminated[w] || A.truncated[w];
  const float* v = A.V + (size_t)w * A.v_width;
  int first = 0, k = 0;
  for (int t = 0; t < A.nterm; t++) {
    const B2EventTerm T = A.term[t];
    bool fire = reset;
    if (T.mode == B2_EVENT_INTERVAL) {
      int f = 0;
      if (lane == 0) {
        float* tl = A.timers + (size_t)k * n + w;
        float x = b2e_add(*tl, -A.step_dt);
        f = x < 1e-6f;
        if (f) x = b2e_add(b2e_mul(v[T.col + T.count], T.interval_span), T.interval_lo);
        *tl = x;
      }
      fire = __shfl_sync(0xffffffffu, f, 0) != 0;
      k++;
    }
    if (fire) {
      float* row = F.row[t] + (size_t)w * F.stride[t];
      for (int j = lane; j < T.count; j += 32) {
        const B2EventElem E = A.elem[first + j];
        float x = b2e_add(b2e_mul(v[T.col + j], E.span), E.lo);
        if (T.distribution == B2_EVENT_LOG_UNIFORM) x = expf(x);
        const float old = row[E.offset];
        row[E.offset] = T.operation == B2_EVENT_ADD ? b2e_add(old, x) : T.operation == B2_EVENT_SCALE ? b2e_mul(old, x) : x;
      }
    }
    __syncwarp();
    first += T.count;
  }
  if (A.nstate == 0) return;
  // state terms: a reset env's wrenches are cleared first, then each term writes its own xfrc_applied / qvel entries
  float* xfrc = F.xfrc + (size_t)w * F.xfrc_s;
  if (A.clear_xfrc && reset)
    for (int j = lane; j < F.xfrc_s; j += 32) xfrc[j] = 0.f;
  __syncwarp();
  for (int t = 0; t < A.nstate; t++) {
    const int kind = A.state[t].kind, col = A.state[t].col, count = A.state[t].count;
    bool fire = reset;
    if (A.state[t].mode == B2_EVENT_INTERVAL) {
      int f = 0;
      if (lane == 0) {
        float* tl = A.timers + (size_t)A.state[t].timer * n + w;
        float x = b2e_add(*tl, -A.step_dt);
        f = x < 1e-6f;
        if (f) x = b2e_add(b2e_mul(v[col + (kind == B2_EVENT_PUSH ? 6 : 6 * count)], A.state[t].interval_span),
                            A.state[t].interval_lo);
        *tl = x;
      }
      fire = __shfl_sync(0xffffffffu, f, 0) != 0;
    }
    if (fire) {
      if (kind == B2_EVENT_WRENCH) {
        const int b0 = A.state[t].first;
        const float flo = A.state[t].lo[0], fspan = A.state[t].span[0], tlo = A.state[t].lo[1], tspan = A.state[t].span[1];
        for (int j = lane; j < 6 * count; j += 32) {
          const bool torque = j >= 3 * count;
          const int e = torque ? j - 3 * count : j;
          const float x = b2e_add(b2e_mul(v[col + j], torque ? tspan : fspan), torque ? tlo : flo);
          xfrc[6 * A.bodies[b0 + e / 3] + (torque ? 3 : 0) + e % 3] = x;
        }
      } else if (lane == 0) {
        b2e_push(A, F, t, v, w);
      }
    }
    __syncwarp();
  }
}

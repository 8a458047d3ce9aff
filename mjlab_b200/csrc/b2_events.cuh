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
}

// b2_nanguard.cuh — the NaN guard on the device (the reference's NanGuard, utils/nan_guard.py, run as stream work
// around the step kernel so that a captured CUDA graph carries it).  While armed (b2_nan_guard), every sub-step of
// b2_step / b2_step_n records the pre-step qpos / qvel of worlds 0..ncapture-1 into a ring and, after the sub-step,
// checks qpos, qvel, qacc and qacc_warmstart of every world for a non-finite value.  The first sub-step that finds one
// is the detection sub-step; from then on nothing is recorded or flagged, so what the host reads does not depend on
// when it looks.
//
// Launches: one start kernel per call (one CTA: records the pre-step state of the call's first sub-step for every
// captured world and reserves the call's sub-step numbers), then after each sub-step one check kernel per partition
// (one warp per world: checks the sub-step just run and records the pre-step state of the next one).  The check
// kernels take their sub-step as base + i, base being what the start kernel reserved, so no kernel both reads and
// writes the counter and a replayed graph numbers its sub-steps from the device.
//
// Partitions: b2_step_n may run two halves of the worlds on two streams, one ahead of the other by up to a chunk
// (B2_GUARD_CHUNK sub-steps; the streams join after each chunk while the guard is armed).  The detection sub-step is
// the minimum over both (atomicMin), but a partition that has run ahead may record past it before it sees the other's
// detection.  The ring therefore has buffer_size + B2_GUARD_CHUNK - 1 slots, entry k in slot k mod slots: a record of
// at most detection + B2_GUARD_CHUNK - 1 never overwrites one of the buffer_size entries up to the detection.
#pragma once
#include "b2_types.h"

#define B2_GUARD_CHUNK 8
#define B2_GUARD_NONE 0x7fffffffffffffffLL  // detection sub-step / first-bad sub-step of a world: none yet

struct B2Guard {
  float* ring;             // [slots][ncapture][nq + nv]: pre-step qpos then qvel of the captured worlds
  long long* ctl;          // [0] sub-steps reserved since arming, [1] first sub-step of the running call, [2] detection
  long long* first_bad;    // [nworld] first sub-step at which the world was seen non-finite (B2_GUARD_NONE: never)
  volatile int* word;      // device alias of the host-visible word: 1 once a non-finite state was found
  int slots, ncapture;
};

#ifdef B2_HOST_EMULATION
inline void b2g_atomic_min(long long* p, long long v) {
  long long old = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (v < old && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {
  }
}
inline void b2g_fence_system() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
#else
__device__ __forceinline__ void b2g_atomic_min(long long* p, long long v) { atomicMin(p, v); }
__device__ __forceinline__ void b2g_fence_system() { __threadfence_system(); }
#endif

// The host-visible word: mapped pinned memory, which the device writes and the host reads without a copy (`host`: its
// host address, `dev`: the device's).  Under host emulation "device" memory is host memory, so a plain allocation is
// both.
static inline cudaError_t b2g_word_alloc(void** host, void** dev) {
#ifdef B2_HOST_EMULATION
  cudaError_t e = cudaMalloc(host, sizeof(int));
  *dev = *host;
  return e;
#else
  cudaError_t e = cudaHostAlloc(host, sizeof(int), cudaHostAllocMapped);
  return e != cudaSuccess ? e : cudaHostGetDevicePointer(dev, *host, 0);
#endif
}
static inline void b2g_word_free(void* host) {
#ifdef B2_HOST_EMULATION
  cudaFree(host);
#else
  cudaFreeHost(host);
#endif
}

__device__ __forceinline__ bool b2g_finite(float x) { return (__float_as_int(x) & 0x7f800000) != 0x7f800000; }

// Pre-step state of world w (< ncapture) as entry k of the ring; `lane` of `nlanes` threads share the row.
__device__ __forceinline__ void b2g_record(const B2Guard& g, const DevData& d, int nq, int nv, int w, long long k,
                                          int lane, int nlanes) {
  float* row = g.ring + ((size_t)(k % g.slots) * g.ncapture + w) * (size_t)(nq + nv);
  const float* qpos = d.qpos.p + (size_t)w * d.qpos.stride;
  const float* qvel = d.qvel.p + (size_t)w * d.qvel.stride;
  for (int i = lane; i < nq; i += nlanes) row[i] = qpos[i];
  for (int i = lane; i < nv; i += nlanes) row[nq + i] = qvel[i];
}

// Before the call's first sub-step, on the caller's stream: reserve the call's n sub-step numbers and record the
// pre-step state of the first one.  One CTA.
__global__ void b2_guard_start_kernel(B2Guard g, DevData d, int nq, int nv, int n) {
  const long long k = g.ctl[0];
  if (k <= g.ctl[2])
    for (int w = threadIdx.x / 32; w < g.ncapture; w += blockDim.x / 32) b2g_record(g, d, nq, nv, w, k, threadIdx.x % 32, 32);
  __syncthreads();  // every thread has read ctl[0]
  if (threadIdx.x == 0) {
    g.ctl[1] = k;
    g.ctl[0] = k + n;
  }
}

// After sub-step i of the call, for the worlds [base, base + count): check them and, when `record`, record the
// captured ones among them as the next sub-step's pre-step state.  One warp per world.
__global__ void b2_guard_check_kernel(B2Guard g, DevData d, int nq, int nv, int base, int count, int i, int record) {
  const int lane = threadIdx.x % 32;
  const int j = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) / 32);
  if (j >= count) return;
  // (lane 0's reading of the detection for the whole warp: the other partition may lower it meanwhile)
  const long long k = g.ctl[1] + i, det = __shfl_sync(0xffffffffu, g.ctl[2], 0);
  if (k > det) return;  // frozen
  const int w = base + j;
  bool bad = false;
  const float* rows[4] = {d.qpos.p + (size_t)w * d.qpos.stride, d.qvel.p + (size_t)w * d.qvel.stride,
                          d.qacc.p + (size_t)w * d.qacc.stride, d.qacc_warmstart.p + (size_t)w * d.qacc_warmstart.stride};
  for (int a = 0; a < 4; a++)
    for (int c = lane; c < (a == 0 ? nq : nv); c += 32) bad |= !b2g_finite(rows[a][c]);
  if (__any_sync(0xffffffffu, bad) && lane == 0) {
    if (g.first_bad[w] == B2_GUARD_NONE) g.first_bad[w] = k;
    b2g_atomic_min(&g.ctl[2], k);
    *g.word = 1;
    b2g_fence_system();
  }
  if (record && w < g.ncapture && k < det) b2g_record(g, d, nq, nv, w, k + 1, lane, 32);
}

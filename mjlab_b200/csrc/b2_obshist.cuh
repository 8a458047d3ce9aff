// b2_obshist.cuh — clip, scale and history of the fused environments' observation groups (the reference's
// ObservationManager.compute_group, managers/observation_manager.py:153-188, with its CircularBuffer,
// utils/buffers/circular_buffer.py), one launch after the env's post kernel for every configured group.
// The torch implementation in mjlab_b200/envs/obs_history.py is the reference (tests/test_obs_history.py).  A group with
// a noise source first adds its terms' noise and bias to the noise-free values (envs/noise.py; tests/test_obs_noise.py).
//
// One thread per (group, env, element of the group's frame).  The output row is the history itself, laid out as the
// env returns it: each thread shifts its own column one frame older and writes its new value into the newest slot (a
// reset env gets it in every slot), so no ring pointer is kept and no thread waits on another.  Consecutive threads
// handle consecutive elements of a term, so the loads and stores of a warp are contiguous.  A term's bias is kept per
// element, a shared one replicated into every element's slot: each thread updates only its own slot, from the same
// draw, so the copies stay equal without atomics or a second launch.
#pragma once
#include "../../include/b2sim.h"

// One IEEE fp32 product without flushing subnormals: the library builds with --use_fast_math (-ftz=true), and the
// scaled value must be the one torch computes.
__device__ __forceinline__ float b2o_mul(float a, float b) {
#ifdef B2_HOST_EMULATION
  return a * b;
#else
  float r;
  asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
#endif
}
// One IEEE fp32 sum, likewise (and never contracted with a product into an FMA).
__device__ __forceinline__ float b2o_add(float a, float b) {
#ifdef B2_HOST_EMULATION
  return a + b;
#else
  float r;
  asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
#endif
}

// A noise class of include/b2sim.h applied to v: x = p0 (CONSTANT) or r p1 + p0, then v + x, v x or x.
__device__ __forceinline__ float b2o_noise(int cls, int op, float v, float p0, float p1, float r) {
  const float x = cls == B2_NOISE_CONSTANT ? p0 : b2o_add(b2o_mul(r, p1), p0);
  if (op == B2_NOISE_ADD) return b2o_add(v, x);
  if (op == B2_NOISE_SCALE) return b2o_mul(v, x);
  return cls == B2_NOISE_CONSTANT ? b2o_add(0.0f, x) : x;  // (torch.zeros_like(v) + bias)
}

// Draw c of env w for a class: W for UNIFORM, N for GAUSSIAN, none for CONSTANT.
__device__ __forceinline__ float b2o_draw(const B2ObsHistArgs& A, int cls, int w, int c) {
  if (cls == B2_NOISE_UNIFORM) return A.W[(size_t)w * A.nW + c];
  if (cls == B2_NOISE_GAUSSIAN) return A.N[(size_t)w * A.nN + c];
  return 0.0f;
}

// Element e of env w's frame in group G.  (A device function called with a fixed group, so that the term table is
// read from the parameter block at constant offsets.)
__device__ __forceinline__ void b2o_element(const B2ObsHistGroup& G, const B2ObsNoiseGroup& Z, const B2ObsHistArgs& A,
                                            int w, int e) {
  B2ObsHistTerm T = G.term[0];
  int k = 0;
#pragma unroll
  for (int t = 1; t < B2_OBSHIST_NTERM; t++)
    if (t < G.nterm && e >= G.term[t].src) T = G.term[t], k = t;
  const int j = e - T.src;
  const bool reset = A.terminated[w] || A.truncated[w];
  float v;
  if (Z.source) {
    const B2ObsNoiseTerm& M = Z.term[k];  // (read field by field: a dynamic index into the parameter block)
    v = Z.source[(size_t)w * Z.source_width + M.col + j];
    const int cls = M.noise, bcls = M.bias;
    if (cls != B2_NOISE_NONE) {
      const float p1 = cls == B2_NOISE_CONSTANT ? 0.0f : A.param[M.noise_p1 + j];
      v = b2o_noise(cls, M.noise_op, v, A.param[M.noise_p0 + j], p1, b2o_draw(A, cls, w, M.noise_draw + j));
    }
    if (bcls != B2_NOISE_NONE) {  // the bias after the noise; a reset env first redraws its own copy of it
      float* bp = Z.bias + (size_t)w * G.frame_width + e;
      float b = *bp;
      if (reset) {
        const float p1 = bcls == B2_NOISE_CONSTANT ? 0.0f : A.param[M.bias_p1 + j];
        b = b2o_noise(bcls, M.bias_op, b, A.param[M.bias_p0 + j], p1,
                      b2o_draw(A, bcls, w, M.bias_draw + (M.bias_shared ? 0 : j)));
        *bp = b;
      }
      v = b2o_add(v, b);
    }
  } else {
    v = G.frame[(size_t)w * G.frame_width + e];
  }
  if (T.clip) v = v < T.lo ? T.lo : (v > T.hi ? T.hi : v);  // (torch.clamp: NaN stays NaN)
  if (T.scale >= 0) v = b2o_mul(v, A.scale[T.scale + j]);
  float* o = G.out + (size_t)w * G.out_width + T.dst + j;
  const int H = T.frames > 1 ? T.frames : 1;
  // four older frames are loaded before any of them is overwritten: a store may alias the next load, so one frame at
  // a time would wait a memory round trip per frame
  for (int k = 0; k + 1 < H; k += 4) {
    float x[4];
#pragma unroll
    for (int i = 0; i < 4; i++) x[i] = reset || k + i + 1 >= H ? v : o[(size_t)(k + i + 1) * T.stride];
#pragma unroll
    for (int i = 0; i < 4; i++)
      if (k + i + 1 < H) o[(size_t)(k + i) * T.stride] = x[i];
  }
  o[(size_t)(H - 1) * T.stride] = v;
}

// Threads [0, n frame_width of group 0) serve group 0, the next n frame_width of group 1 serve group 1.
__global__ void b2_obs_history_kernel(int n, B2ObsHistArgs A) {
  long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n0 = (long long)n * A.group[0].frame_width;
  if (tid < n0) {
    b2o_element(A.group[0], A.noise[0], A, (int)(tid / A.group[0].frame_width), (int)(tid % A.group[0].frame_width));
    return;
  }
  tid -= n0;
  if (A.ngroup < 2 || tid >= (long long)n * A.group[1].frame_width) return;
  b2o_element(A.group[1], A.noise[1], A, (int)(tid / A.group[1].frame_width), (int)(tid % A.group[1].frame_width));
}

// b2sim.cu — libb2sim.so: C ABI (include/b2sim.h) around the fused sm_90a step kernel.
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/b2sim.h"
#include "b2_kernel.cuh"
#include "b2_tables.h"
#include "b2_env.cuh"
#include "b2_trackenv.cuh"
#include "b2_obshist.cuh"
#include "b2_events.cuh"
#include "b2_nanguard.cuh"
#include "b2_render.cuh"

static thread_local std::string g_err;
static int fail(const std::string& msg) {
  g_err = msg;
  return 1;
}
#define CUDA_OK(expr)                                                                     \
  do {                                                                                    \
    cudaError_t e_ = (expr);                                                              \
    if (e_ != cudaSuccess)                                                                \
      return fail(std::string(#expr) + ": " + cudaGetErrorString(e_));                    \
  } while (0)

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceGuard() {
    int cur;
    cudaGetDevice(&cur);
    if (prev >= 0 && cur != prev) cudaSetDevice(prev);
  }
};

struct Field {
  std::string name;
  void* ptr = nullptr;
  int dtype = B2_F32;
  int ndim = 1;
  int64_t shape[4] = {1, 1, 1, 1};
  int64_t stride[4] = {0, 0, 0, 1};
  FArr* farr = nullptr;  // model float arrays: where the kernel reads the pointer from
  int64_t n = 0;         // elements per world
};

struct b2_sim {
  int device = 0;
  int nworld = 0;
  DevModel hm;
  DevData hd;
  std::vector<Field> data_fields, model_fields;
  std::vector<void*> allocs;
  int64_t launches = 0;
  int* order = nullptr;       // heavy-first dispatch order (device)
  int sorted_dispatch = 1;
  int has_convex = 0;          // the model has mesh / height-field collision pairs: kernels with the convex routines
  int resident_ctas = 0;       // co-resident CTAs of the step kernel on this device
  cudaStream_t side[2] = {nullptr, nullptr};  // b2_step_n's two env partitions
  cudaEvent_t ev_fork = nullptr, ev_join[2] = {nullptr, nullptr};
  size_t smem_bytes = 0;
  std::vector<long long> events_checked;  // b2_events: the entry table last checked (address, size, fields, counts)
  // NaN guard (b2_nan_guard): the buffers of the last arming; those of earlier armings stay allocated until
  // b2_destroy, so that a graph captured while they were armed never writes freed memory
  int guard_on = 0, guard_buffer = 0;
  B2Guard guard = {};
  std::vector<void*> host_allocs;
  // b2_render: the drawable geoms, listed at the first call
  bool render_planned = false;
  B2RenderPlan render_plan = {};
};

static int pad4(int n) { return (n + 3) & ~3; }

template <typename T>
static int dev_upload(b2_sim* s, const std::vector<T>& h, const T** out) {
  void* p = nullptr;
  size_t bytes = sizeof(T) * std::max<size_t>(h.size(), 1);
  CUDA_OK(cudaMalloc(&p, bytes));
  s->allocs.push_back(p);
  if (!h.empty()) CUDA_OK(cudaMemcpy(p, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice));
  *out = (const T*)p;
  return 0;
}

__global__ void b2_tile_kernel(const float* __restrict__ src, float* __restrict__ dst, int n,
                               long long total) {
  long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid < total) dst[tid] = src[tid % n];
}
__global__ void b2_init_rows_kernel(float* dst, int stride, const float* __restrict__ src, int n,
                                    int nworld) {
  long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid < (long long)nworld * n) dst[(tid / n) * stride + (tid % n)] = src[tid % n];
}

// World poses of the grid-static geoms are constant: written into every world's geom_xpos / geom_xmat once.
__global__ void b2_static_rows_kernel(float* xpos, int xpos_stride, float* xmat, int xmat_stride,
                                      const float* __restrict__ pose, const int* __restrict__ static_geom,
                                      int nstatic, int nworld) {
  long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= (long long)nworld * nstatic) return;
  int k = (int)(tid % nstatic), g = static_geom[k];
  size_t w = (size_t)(tid / nstatic);
  const float* p = pose + 16 * (size_t)k;
  for (int i = 0; i < 3; i++) xpos[w * xpos_stride + 3 * g + i] = p[i];
  for (int i = 0; i < 9; i++) xmat[w * xmat_stride + 9 * g + i] = p[3 + i];
}

// The float part of the compact kinematic records (kinematic_tables), rebuilt from the shared rows of body_pos,
// body_quat, jnt_pos, jnt_axis and qpos0, so that a caller's write to one of them reaches the fast kinematics.  Only
// launched while the records are in use (fastkin: none of the five fields is expanded); the int words stay as built.
// (The joint and qpos address come from the records' own int words: two dependent loads per body, not four.)
__global__ void b2_kinrec_kernel(DevModel m) {
  float* rec = (float*)m.kinrec;
  for (int b = threadIdx.x; b < m.nbody; b += blockDim.x) {
    float* r = rec + 16 * b;
    const int tj = __float_as_int(r[11]), qa = __float_as_int(r[15]);
    for (int k = 0; k < 3; k++) r[k] = m.body_pos.p[3 * b + k];
    for (int k = 0; k < 4; k++) r[4 + k] = m.body_quat.p[4 * b + k];
    if ((tj & 0xff) != 0xff) {
      const int j = tj >> 8;
      for (int k = 0; k < 3; k++) { r[8 + k] = m.jnt_pos.p[3 * j + k]; r[12 + k] = m.jnt_axis.p[3 * j + k]; }
      r[3] = m.qpos0.p[qa];
    }
  }
}

// Heavy-first dispatch: order worlds by the previous step's (Newton iterations, contacts),
// descending, with a one-CTA counting sort (128 buckets).  Only scheduling changes, not results.
// Key = (Newton iterations, solver block class, contacts / 8): under phase-synchronous execution the warps of a
// CTA wait for each other at every phase boundary, so a CTA should hold environments of equal cost.
__device__ __forceinline__ int b2_order_key(int niter, int nd, int ncon, int nd_small) {
  return min(niter, 15) * 8 + (nd > nd_small ? 4 : 0) + min(ncon >> 3, 3);
}
__global__ void b2_order_kernel(const int* __restrict__ niter, int niter_stride, const int* __restrict__ ncon,
                                int ncon_stride, const int* __restrict__ nd, int nd_stride, int nd_small,
                                int base_world, int count, int* __restrict__ order) {
  __shared__ int hist[128];
  __shared__ int base[128];
  for (int i = threadIdx.x; i < 128; i += blockDim.x) hist[i] = 0;
  __syncthreads();
  // (keys stay in registers between the two passes: up to 4 worlds per thread, the common case; more are re-read)
  int keys[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    int k = threadIdx.x + j * blockDim.x;
    keys[j] = -1;
    if (k < count) {
      int w = base_world + k;
      keys[j] = 127 - b2_order_key(niter[(size_t)w * niter_stride], nd[(size_t)w * nd_stride], ncon[(size_t)w * ncon_stride], nd_small);
      atomicAdd(&hist[keys[j]], 1);
    }
  }
  for (int k = threadIdx.x + 4 * blockDim.x; k < count; k += blockDim.x) {
    int w = base_world + k;
    atomicAdd(&hist[127 - b2_order_key(niter[(size_t)w * niter_stride], nd[(size_t)w * nd_stride], ncon[(size_t)w * ncon_stride], nd_small)], 1);
  }
  __syncthreads();
  if (threadIdx.x < 32) {  // exclusive prefix over the 128 buckets: 4 per lane + a warp scan
    int h0 = hist[4 * threadIdx.x], h1 = hist[4 * threadIdx.x + 1], h2 = hist[4 * threadIdx.x + 2], h3 = hist[4 * threadIdx.x + 3];
    int sum = h0 + h1 + h2 + h3, incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, incl, o);
      if ((int)threadIdx.x >= o) incl += t;
    }
    int ex = incl - sum;
    base[4 * threadIdx.x] = ex; base[4 * threadIdx.x + 1] = ex + h0;
    base[4 * threadIdx.x + 2] = ex + h0 + h1; base[4 * threadIdx.x + 3] = ex + h0 + h1 + h2;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 4; j++) {
    int k = threadIdx.x + j * blockDim.x;
    if (k < count) order[base_world + atomicAdd(&base[keys[j]], 1)] = base_world + k;
  }
  for (int k = threadIdx.x + 4 * blockDim.x; k < count; k += blockDim.x) {
    int w = base_world + k;
    int key = 127 - b2_order_key(niter[(size_t)w * niter_stride], nd[(size_t)w * nd_stride], ncon[(size_t)w * ncon_stride], nd_small);
    order[base_world + atomicAdd(&base[key], 1)] = w;
  }
}

// ---- model and data tables ---------------------------------------------------------------------------------------
// Every array of the model descriptor and every Data field is named once, in one of the tables below; validation,
// upload, field registration and lookup all read them.

// Model sizes the descriptor's arrays scale with (D_ZERO: none).
enum Dim { D_NQ, D_NV, D_NU, D_NBODY, D_NJNT, D_NGEOM, D_NSITE, D_NSENSOR, D_NPAIR, D_NSTATIC, D_ZERO, D_NDIM };

// Float model arrays: `count` x max(width, 1) fp64 values in the descriptor, fp32 on the device, shared by all worlds
// (stride 0) until b2_expand_model_field gives one a per-world copy.  Model fields of shape (nworld, count[, width]).
struct FloatArray { const char* name; FArr DevModel::*dev; Dim count; int width; };
static const FloatArray kFloatArrays[] = {
    {"body_pos", &DevModel::body_pos, D_NBODY, 3}, {"body_quat", &DevModel::body_quat, D_NBODY, 4},
    {"body_ipos", &DevModel::body_ipos, D_NBODY, 3}, {"body_iquat", &DevModel::body_iquat, D_NBODY, 4},
    {"body_mass", &DevModel::body_mass, D_NBODY, 0}, {"body_subtreemass", &DevModel::body_subtreemass, D_NBODY, 0},
    {"body_inertia", &DevModel::body_inertia, D_NBODY, 3}, {"body_invweight0", &DevModel::body_invweight0, D_NBODY, 2},
    {"jnt_pos", &DevModel::jnt_pos, D_NJNT, 3}, {"jnt_axis", &DevModel::jnt_axis, D_NJNT, 3},
    {"jnt_range", &DevModel::jnt_range, D_NJNT, 2}, {"jnt_solref", &DevModel::jnt_solref, D_NJNT, 2},
    {"jnt_solimp", &DevModel::jnt_solimp, D_NJNT, 5}, {"jnt_margin", &DevModel::jnt_margin, D_NJNT, 0},
    {"jnt_stiffness", &DevModel::jnt_stiffness, D_NJNT, 0}, {"dof_armature", &DevModel::dof_armature, D_NV, 0},
    {"dof_damping", &DevModel::dof_damping, D_NV, 0}, {"dof_frictionloss", &DevModel::dof_frictionloss, D_NV, 0},
    {"dof_invweight0", &DevModel::dof_invweight0, D_NV, 0}, {"geom_size", &DevModel::geom_size, D_NGEOM, 3},
    {"geom_pos", &DevModel::geom_pos, D_NGEOM, 3}, {"geom_quat", &DevModel::geom_quat, D_NGEOM, 4},
    {"geom_friction", &DevModel::geom_friction, D_NGEOM, 3}, {"geom_solref", &DevModel::geom_solref, D_NGEOM, 2},
    {"geom_solimp", &DevModel::geom_solimp, D_NGEOM, 5}, {"geom_solmix", &DevModel::geom_solmix, D_NGEOM, 0},
    {"geom_margin", &DevModel::geom_margin, D_NGEOM, 0}, {"geom_gap", &DevModel::geom_gap, D_NGEOM, 0},
    {"geom_rbound", &DevModel::geom_rbound, D_NGEOM, 0}, {"geom_rgba", &DevModel::geom_rgba, D_NGEOM, 4},
    {"site_pos", &DevModel::site_pos, D_NSITE, 3}, {"site_quat", &DevModel::site_quat, D_NSITE, 4},
    {"actuator_gainprm", &DevModel::actuator_gainprm, D_NU, 10},
    {"actuator_biasprm", &DevModel::actuator_biasprm, D_NU, 10},
    {"actuator_ctrlrange", &DevModel::actuator_ctrlrange, D_NU, 2},
    {"actuator_forcerange", &DevModel::actuator_forcerange, D_NU, 2},
    {"actuator_gear", &DevModel::actuator_gear, D_NU, 0}, {"qpos0", &DevModel::qpos0, D_NQ, 0}};

// Integer model arrays.  The descriptor holds exactly mult x count of them (always, or only with a static grid,
// nstatic > 0, when `with_grid`), or any number when count is D_ZERO.  Values lie in [lo, size(hi) + hi_add), unchecked
// when lo is kAny.  `field`: callers can read the array as a Model field (1-D, shared by all worlds), in table order.
static const long long kAny = -(1ll << 40);
struct IntArray {
  const char* name; const int* DevModel::*dev; Dim count = D_ZERO; bool field = false;
  long long lo = kAny; Dim hi = D_ZERO; int hi_add = 0; int mult = 1; bool with_grid = false;
};
static const IntArray kIntArrays[] = {
    {"geom_bodyid", &DevModel::geom_bodyid, D_NGEOM, true, 0, D_NBODY},
    {"site_bodyid", &DevModel::site_bodyid, D_NSITE, true, 0, D_NBODY},
    {"body_parentid", &DevModel::body_parentid, D_NBODY, true, 0, D_NBODY},
    {"body_rootid", &DevModel::body_rootid, D_NBODY, true, 0, D_NBODY},
    {"body_jntadr", &DevModel::body_jntadr, D_NBODY, false, -1, D_NJNT},
    {"body_jntnum", &DevModel::body_jntnum, D_NBODY, false, 0, D_NJNT, 1},
    {"body_dofadr", &DevModel::body_dofadr, D_NBODY, false, -1, D_NV},
    {"body_dofnum", &DevModel::body_dofnum, D_NBODY, false, 0, D_NV, 1},
    {"jnt_type", &DevModel::jnt_type, D_NJNT, true, 0, D_ZERO, 4},
    {"jnt_qposadr", &DevModel::jnt_qposadr, D_NJNT, true, 0, D_NQ},
    {"jnt_dofadr", &DevModel::jnt_dofadr, D_NJNT, true, 0, D_NV},
    {"jnt_bodyid", &DevModel::jnt_bodyid, D_NJNT, false, 0, D_NBODY},
    {"jnt_limited", &DevModel::jnt_limited, D_NJNT, false, 0, D_ZERO, 2},
    {"dof_bodyid", &DevModel::dof_bodyid, D_NV, true, 0, D_NBODY},
    {"dof_jntid", &DevModel::dof_jntid, D_NV, false, 0, D_NJNT},
    {"dof_parentid", &DevModel::dof_parentid, D_NV, false, -1, D_NV},
    {"geom_type", &DevModel::geom_type, D_NGEOM, true, 0, D_ZERO, 9},
    {"geom_condim", &DevModel::geom_condim, D_NGEOM, true, 1, D_ZERO, 7},
    {"geom_priority", &DevModel::geom_priority, D_NGEOM, true},
    {"actuator_trnid", &DevModel::actuator_trnid, D_NU, true, 0, D_NJNT},
    {"actuator_ctrllimited", &DevModel::actuator_ctrllimited, D_NU, false, 0, D_ZERO, 2},
    {"actuator_forcelimited", &DevModel::actuator_forcelimited, D_NU, false, 0, D_ZERO, 2},
    {"pair_geom1", &DevModel::pair_geom1, D_NPAIR, false, 0, D_NGEOM},
    {"pair_geom2", &DevModel::pair_geom2, D_NPAIR, false, 0, D_NGEOM},
    {"sensor_objtype", &DevModel::sensor_objtype, D_NSENSOR}, {"sensor_objid", &DevModel::sensor_objid, D_NSENSOR},
    {"sensor_reftype", &DevModel::sensor_reftype, D_NSENSOR}, {"sensor_refid", &DevModel::sensor_refid, D_NSENSOR},
    {"sensor_intprm", &DevModel::sensor_intprm, D_NSENSOR, false, kAny, D_ZERO, 0, 3},
    {"sensor_adr", &DevModel::sensor_adr, D_NSENSOR, false, 0, D_ZERO, 1 << 20},
    {"sensor_dim", &DevModel::sensor_dim, D_NSENSOR, false, 0, D_ZERO, 1 << 20},
    {"geom_contype", &DevModel::geom_contype, D_NGEOM, false, kAny, D_ZERO, 0, 1, true},
    {"geom_conaffinity", &DevModel::geom_conaffinity, D_NGEOM, false, kAny, D_ZERO, 0, 1, true},
    {"static_geom", &DevModel::static_geom, D_NSTATIC, false, 0, D_NGEOM, 0, 1, true},
    {"static_cell0", &DevModel::static_cell0, D_NSTATIC, false, 0, D_ZERO, 1 << 20, 2, true},
    {"dyn_cgeom", &DevModel::dyn_cgeom, D_ZERO, false, 0, D_NGEOM},
    {"grid_items", &DevModel::grid_items, D_ZERO, false, 0, D_NSTATIC}, {"grid_start", &DevModel::grid_start},
    {"geom_dataid", &DevModel::geom_dataid}, {"mesh_vertadr", &DevModel::mesh_vertadr}, {"mesh_vertnum", &DevModel::mesh_vertnum},
    {"hfield_adr", &DevModel::hfield_adr}, {"hfield_nrow", &DevModel::hfield_nrow}, {"hfield_ncol", &DevModel::hfield_ncol}};

// Mesh and height-field assets: fp64 in the descriptor, fp32 on the device, shared by all worlds; not fields.
struct AssetArray { const char* name; const float* DevModel::*dev; };
static const AssetArray kAssetArrays[] = {
    {"mesh_vert", &DevModel::mesh_vert}, {"hfield_size", &DevModel::hfield_size}, {"hfield_data", &DevModel::hfield_data}};

// The descriptor's arrays, copied by b2_create and used only while it runs; the tables' arrays are looked up by
// their DevModel member (absent arrays read as empty).
struct HostModel {
  std::map<std::string, std::vector<int>> i;
  std::map<std::string, std::vector<double>> f;

  template <class T> static const std::vector<T>& find(const std::map<std::string, std::vector<T>>& m, const char* k) {
    static const std::vector<T> none;
    auto it = m.find(k);
    return it == m.end() ? none : it->second;
  }
  template <class Row, size_t N, class Member>
  static const char* name_of(const Row (&rows)[N], Member dev) {
    for (const Row& r : rows) if (r.dev == dev) return r.name;
    return "";
  }
  const std::vector<int>& at(const int* DevModel::*a) const { return find(i, name_of(kIntArrays, a)); }
  const std::vector<double>& at(FArr DevModel::*a) const { return find(f, name_of(kFloatArrays, a)); }
  const std::vector<double>& at(const float* DevModel::*a) const { return find(f, name_of(kAssetArrays, a)); }
  double scalar(const char* k) const {  // a size or option scalar, given as int32 or float64 (0 when absent)
    const std::vector<int>& vi = find(i, k); const std::vector<double>& vf = find(f, k);
    return !vi.empty() ? vi[0] : vf.empty() ? 0.0 : vf[0];
  }
};

// A field of `n` values per world, `wstride` elements apart (0: shared by all worlds).  `width` > 0 splits a world's
// values into (n / width, width), 9 into (n / 9, 3, 3) like mjwarp's mat33 arrays; `per_world`: one value per world,
// shape (nworld,).
static Field make_field(const char* name, void* p, int dtype, int nworld, int64_t wstride, int64_t n, int width,
                        bool per_world) {
  Field f;
  f.name = name; f.ptr = p; f.dtype = dtype; f.n = n;
  f.shape[0] = nworld; f.stride[0] = wstride;
  if (per_world) f.ndim = 1;
  else if (width == 9) {
    f.ndim = 4; f.shape[1] = n / 9; f.shape[2] = 3; f.shape[3] = 3;
    f.stride[1] = 9; f.stride[2] = 3; f.stride[3] = 1;
  } else if (width > 0) {
    f.ndim = 3; f.shape[1] = n / width; f.shape[2] = width; f.stride[1] = width; f.stride[2] = 1;
  } else { f.ndim = 2; f.shape[1] = n; f.stride[1] = 1; }
  return f;
}

// A per-world Data array (DArr: float, IArr: int) of `n` values per world; see make_field for `width`, `per_world`.
template <class A>
struct DataArray { const char* name; A DevData::*dev; int n; int width = 0; bool per_world = false; };

template <class A>
static int add_data(b2_sim* s, const DataArray<A>& r) {
  using T = typename std::remove_pointer<decltype(A::p)>::type;
  const int stride = r.n > 0 ? pad4(r.n) : 4;  // rows padded to 16 B
  void* p = nullptr;
  size_t bytes = sizeof(T) * (size_t)s->nworld * stride;
  CUDA_OK(cudaMalloc(&p, bytes));
  s->allocs.push_back(p);
  CUDA_OK(cudaMemset(p, 0, bytes));
  A& a = s->hd.*r.dev;
  a.p = (T*)p; a.stride = stride; a.n = r.n;
  s->data_fields.push_back(make_field(r.name, p, std::is_same<T, int>::value ? B2_I32 : B2_F32, s->nworld, stride, r.n,
                                      r.width, r.per_world));
  return 0;
}

// Every entry that launches the step kernel calls this first, on the caller's stream (before any partition fork, so
// that a captured graph holds it).
static int refresh_kinrec(b2_sim* s, cudaStream_t st) {
  if (!s->hm.fastkin) return 0;
  b2_kinrec_kernel<<<1, 64, 0, st>>>(s->hm);
  s->launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

static int launch(b2_sim* s, bool step, cudaStream_t st, int base = 0, int count = -1, int emit = 1) {
  if (count < 0) count = s->nworld;
  s->hd.emit = emit;
  s->hd.world_base = base;
  s->hd.world_count = count;
  const int grid = (count + B2_WARPS_PER_CTA - 1) / B2_WARPS_PER_CTA;
  if (step && s->sorted_dispatch && s->order && count >= 512 && s->hd.world_mask == nullptr) {
    b2_order_kernel<<<1, 1024, 0, st>>>(s->hd.solver_niter.p, s->hd.solver_niter.stride, s->hd.ncon.p,
                                        s->hd.ncon.stride, s->hd.solver_nd.p, s->hd.solver_nd.stride,
                                        s->hm.lay.ndcap, base, count, s->order);
    s->launches++;
    s->hd.world_order = s->order;
  } else {
    s->hd.world_order = nullptr;
  }
  // phase-synchronous warps need every warp of every CTA to own an environment (no early exits, no mask)
  s->hd.phase_sync = s->hd.world_mask == nullptr && count % B2_WARPS_PER_CTA == 0;
  if (step)
    if (s->has_convex) b2_step_kernel<3><<<grid, 32 * B2_WARPS_PER_CTA, s->smem_bytes, st>>>(s->hm, s->hd);
    else b2_step_kernel<1><<<grid, 32 * B2_WARPS_PER_CTA, s->smem_bytes, st>>>(s->hm, s->hd);
  else
    if (s->has_convex) b2_step_kernel<2><<<grid, 32 * B2_WARPS_PER_CTA, s->smem_bytes, st>>>(s->hm, s->hd);
    else b2_step_kernel<0><<<grid, 32 * B2_WARPS_PER_CTA, s->smem_bytes, st>>>(s->hm, s->hd);
  s->launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

// The NaN guard's work around the sub-steps of one call (b2_nanguard.cuh); nothing while the guard is disarmed.
static int guard_start(b2_sim* s, cudaStream_t st, int n) {
  if (!s->guard_on) return 0;
  b2_guard_start_kernel<<<1, 128, 0, st>>>(s->guard, s->hd, s->hm.nq, s->hm.nv, n);
  s->launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}
static int guard_check(b2_sim* s, cudaStream_t st, int base, int count, int i, int record) {
  if (!s->guard_on) return 0;
  b2_guard_check_kernel<<<(count + 3) / 4, 128, 0, st>>>(s->guard, s->hd, s->hm.nq, s->hm.nv, base, count, i, record);
  s->launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" {

const char* b2_last_error(void) { return g_err.c_str(); }
const char* b2_version(void) { return "b2sim 0.1.0 (sm_90a)"; }

// Debug builds (-DB2_PHASE_TIMING): cumulative per-phase cycles (sum over warps); reset on read.
int b2_phase_cycles(unsigned long long* out32) {
#ifdef B2_PHASE_TIMING
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(out32, b2::g_phase_cycles, sizeof(unsigned long long) * 32);
  unsigned long long z[32] = {0};
  cudaMemcpyToSymbol(b2::g_phase_cycles, z, sizeof(z));
  return 0;
#else
  (void)out32;
  return 1;
#endif
}

// Copies the descriptor's arrays into `h` and checks their sizes and index ranges (mjModel field names), so that a
// malformed table never reaches the index loops.  Returns "" when consistent.
static std::string read_desc(const B2ModelDesc* desc, HostModel& h) {
  for (int i = 0; i < desc->narray; i++) {
    const B2Array& a = desc->arrays[i];
    if (!a.name || a.n < 0 || (a.n > 0 && !a.data)) return "array without name or data";
    if (a.dtype == B2_I32) h.i[a.name].assign((const int32_t*)a.data, (const int32_t*)a.data + a.n);
    else if (a.dtype == B2_F64) h.f[a.name].assign((const double*)a.data, (const double*)a.data + a.n);
    else return std::string("array '") + a.name + "': dtype must be int32 or float64";
  }
  static const char* const kSizes[D_ZERO] = {"nq", "nv", "nu", "nbody", "njnt", "ngeom", "nsite", "nsensor", "npair", "nstatic"};
  long long size[D_NDIM] = {};
  for (int k = 0; k < D_ZERO; k++) {
    if (k != D_NSTATIC && HostModel::find(h.i, kSizes[k]).empty() && HostModel::find(h.f, kSizes[k]).empty())
      return "missing size scalar (nq nv nu nbody njnt ngeom nsite nsensor npair)";
    size[k] = (long long)h.scalar(kSizes[k]);
    if (size[k] < (k == D_NQ || k == D_NV || k == D_NBODY ? 1 : 0)) return "negative or zero model size";
  }
  // an array of exactly n values of `dtype`, with int values in [lo, hi) unless lo is kAny ("" when it is)
  auto require = [&](const char* name, int dtype, long long n, long long lo, long long hi) -> std::string {
    const bool is_int = h.i.count(name) > 0;
    long long have = is_int ? h.i.at(name).size() : HostModel::find(h.f, name).size();
    if (have != n) return std::string("array '") + name + "' has " + std::to_string(have) + " elements, expected " + std::to_string(n);
    if (n == 0) return "";
    if (is_int != (dtype == B2_I32)) return std::string("array '") + name + "' has the wrong dtype";
    if (is_int && lo != kAny)
      for (int v : h.i.at(name))
        if (v < lo || v >= hi) return std::string("array '") + name + "' holds an index out of range";
    return "";
  };
  std::string why;
  auto require_int = [&](const IntArray& r) { return require(r.name, B2_I32, r.mult * size[r.count], r.lo, size[r.hi] + r.hi_add); };
  for (const IntArray& r : kIntArrays)
    if (r.count != D_ZERO && !r.with_grid && !(why = require_int(r)).empty()) return why;
  for (const FloatArray& r : kFloatArrays)
    if (!(why = require(r.name, B2_F64, std::max(r.width, 1) * size[r.count], kAny, 0)).empty()) return why;
  if (size[D_NSTATIC] > 0) {
    for (const IntArray& r : kIntArrays)
      if (r.with_grid && !(why = require_int(r)).empty()) return why;
    if (!(why = require("grid_params", B2_F64, 5, kAny, 0)).empty()) return why;
  }
  for (const IntArray& r : kIntArrays) {  // optional index arrays: checked when present
    if (r.count != D_ZERO || r.lo == kAny || (!h.i.count(r.name) && !h.f.count(r.name))) continue;
    if (!h.i.count(r.name)) return std::string("array '") + r.name + "' has the wrong dtype";
    if (!(why = require(r.name, B2_I32, h.i.at(r.name).size(), r.lo, size[r.hi] + r.hi_add)).empty()) return why;
  }
  // parents precede children (the kinematic walks and the factorisation schedule rely on it)
  const std::vector<int>& bp = h.at(&DevModel::body_parentid);
  for (size_t b = 1; b < bp.size(); b++) if (bp[b] >= (int)b) return "body_parentid: parents must precede children";
  const std::vector<int>& dp = h.at(&DevModel::dof_parentid);
  for (size_t d = 0; d < dp.size(); d++) if (dp[d] >= (int)d) return "dof_parentid: parents must precede children";
  return "";
}

// ---- b2_create, stage by stage: each stage returns non-zero (message set) to refuse the model -------------------

// Sizes, solver options and capacities of the model.
static int read_model(const B2ModelDesc* desc, int ncon_per_world, int njmax, const HostModel& h, DevModel& m) {
  auto geti = [&](const char* k) { return (int)h.scalar(k); };
  memset(&m, 0, sizeof(m));
  m.nq = geti("nq"); m.nv = geti("nv"); m.nu = geti("nu"); m.nbody = geti("nbody");
  m.njnt = geti("njnt"); m.ngeom = geti("ngeom"); m.nsite = geti("nsite");
  m.nsensor = geti("nsensor"); m.nsensordata = geti("nsensordata"); m.npair = geti("npair");
  m.ntri = m.nv * (m.nv + 1) / 2;
  if (m.nv > 64 || m.nbody > 64) return fail("b2_create: nv and nbody must be <= 64");
  if (m.nv < 1) return fail("b2_create: model has no degrees of freedom");
  m.integrator = geti("opt_integrator"); m.iterations = geti("opt_iterations");
  m.ls_iterations = geti("opt_ls_iterations");
  m.timestep = (float)h.scalar("opt_timestep"); m.tolerance = (float)h.scalar("opt_tolerance");
  m.ls_tolerance = (float)h.scalar("opt_ls_tolerance"); m.impratio = (float)h.scalar("opt_impratio");
  m.meaninertia = (float)h.scalar("stat_meaninertia");
  for (int k = 0; k < 3; k++) m.gravity[k] = (float)desc->gravity[k];
  if (geti("opt_cone") != 0) return fail("b2_create: only pyramidal cones are supported");
  m.solver = geti("opt_solver");
  if (m.solver != SOL_NEWTON_ && m.solver != SOL_CG_)
    return fail("b2_create: solver must be Newton or CG (PGS works on the dual problem and is not implemented)");
  m.maxcon = ncon_per_world > 0 ? std::min(ncon_per_world, 255) : 48;
  m.njmax = njmax > 0 ? njmax : 300;
  // supported sensor set: contact sensors with data in {found,force,dist,pos,normal}, reduce none/netforce
  const std::vector<int>& intprm = h.at(&DevModel::sensor_intprm);
  for (int i = 0; i < m.nsensor; i++) {
    int ds = intprm[3 * i], rd = intprm[3 * i + 1];
    if ((ds & ~(1 | 2 | 8 | 16 | 32)) || (rd != 0 && rd != 3))
      return fail("b2_create: contact sensor data/reduce combination not implemented");
  }
  return 0;
}

// Tables derived from the body tree: depths, ancestor chains, dof / ancestor / subtree masks, and the compact
// kinematic records of the fast path (every body has at most one joint).
static int kinematic_tables(b2_sim* s, const HostModel& h) {
  DevModel& m = s->hm;
  const std::vector<int>& parent = h.at(&DevModel::body_parentid);
  const std::vector<int>& dofadr = h.at(&DevModel::body_dofadr);
  const std::vector<int>& dofnum = h.at(&DevModel::body_dofnum);
  int nb = m.nbody;
  std::vector<int> depth(nb, 0);
  std::vector<unsigned long long> dofmask(nb, 0ull), ancmask(nb, 0ull);
  int maxdepth = 1;
  ancmask[0] = 1ull;
  for (int b = 1; b < nb; b++) {
    depth[b] = depth[parent[b]] + 1;
    maxdepth = std::max(maxdepth, depth[b]);
    dofmask[b] = dofmask[parent[b]];
    for (int k = 0; k < dofnum[b]; k++) dofmask[b] |= 1ull << (dofadr[b] + k);
    ancmask[b] = ancmask[parent[b]] | (1ull << b);
  }
  std::vector<int> chain((size_t)nb * maxdepth, 0);
  for (int b = 1; b < nb; b++) {
    int c = b;
    for (int k = depth[b] - 1; k >= 0; k--) { chain[(size_t)b * maxdepth + k] = c; c = parent[c]; }
  }
  m.maxdepth = maxdepth;
  std::vector<unsigned long long> submask(nb, 0ull), dofbody(std::max(m.nv, 1), 0ull);
  for (int d = 0; d < nb; d++)
    for (int a = 0; a < nb; a++)
      if (ancmask[d] >> a & 1ull) submask[a] |= 1ull << d;
  for (int b = 1; b < nb; b++)
    for (int i = 0; i < m.nv; i++)
      if (dofmask[b] >> i & 1ull) dofbody[i] |= 1ull << b;
  std::vector<float> kinrec((size_t)nb * 16, 0.f);
  int fastkin = 1;
  const std::vector<int>& jn = h.at(&DevModel::body_jntnum); const std::vector<int>& ja = h.at(&DevModel::body_jntadr);
  const std::vector<int>& jt = h.at(&DevModel::jnt_type); const std::vector<int>& jq = h.at(&DevModel::jnt_qposadr);
  const std::vector<double>& bp = h.at(&DevModel::body_pos); const std::vector<double>& bq = h.at(&DevModel::body_quat);
  const std::vector<double>& jp = h.at(&DevModel::jnt_pos); const std::vector<double>& jax = h.at(&DevModel::jnt_axis);
  const std::vector<double>& q0 = h.at(&DevModel::qpos0);
  for (int b = 0; b < nb; b++) {
    if (jn[b] > 1) { fastkin = 0; break; }
    float* r = kinrec.data() + 16 * b;
    for (int k = 0; k < 3; k++) r[k] = (float)bp[3 * b + k];
    for (int k = 0; k < 4; k++) r[4 + k] = (float)bq[4 * b + k];
    int type = 0xff, j = 0, qa = 0;
    if (jn[b] == 1) {
      j = ja[b]; type = jt[j]; qa = jq[j];
      for (int k = 0; k < 3; k++) { r[8 + k] = (float)jp[3 * j + k]; r[12 + k] = (float)jax[3 * j + k]; }
      r[3] = (float)q0[qa];
    }
    int tj = type | (j << 8);
    memcpy(&r[11], &tj, 4);
    memcpy(&r[15], &qa, 4);
  }
  m.fastkin = fastkin;
  const float* kr = nullptr;
  int rc = dev_upload<int>(s, depth, &m.body_depth) || dev_upload<int>(s, chain, &m.body_chain) ||
           dev_upload<unsigned long long>(s, dofmask, &m.body_dofmask) || dev_upload<unsigned long long>(s, ancmask, &m.body_ancmask) ||
           dev_upload<unsigned long long>(s, submask, &m.body_submask) || dev_upload<unsigned long long>(s, dofbody, &m.dof_bodymask) ||
           dev_upload<float>(s, kinrec, &kr);
  m.kinrec = (const float4*)kr;
  return rc;
}

// World pose (pos[3], mat[9], rbound) of a geom on a jointless child of the world body, in double from world 0's
// model values: such geoms never move, so they are posed here once and shared by all worlds.
static void world_pose(const HostModel& h, int g, float* o) {
  const std::vector<double>& bp = h.at(&DevModel::body_pos); const std::vector<double>& bq = h.at(&DevModel::body_quat);
  const std::vector<double>& gp = h.at(&DevModel::geom_pos); const std::vector<double>& gq = h.at(&DevModel::geom_quat);
  auto qmul = [](const double* a, const double* b, double* r) {
    r[0] = a[0]*b[0] - a[1]*b[1] - a[2]*b[2] - a[3]*b[3];
    r[1] = a[0]*b[1] + a[1]*b[0] + a[2]*b[3] - a[3]*b[2];
    r[2] = a[0]*b[2] - a[1]*b[3] + a[2]*b[0] + a[3]*b[1];
    r[3] = a[0]*b[3] + a[1]*b[2] - a[2]*b[1] + a[3]*b[0];
  };
  auto q2m = [](const double* q, double* R) {
    R[0] = q[0]*q[0] + q[1]*q[1] - q[2]*q[2] - q[3]*q[3]; R[1] = 2*(q[1]*q[2] - q[0]*q[3]); R[2] = 2*(q[1]*q[3] + q[0]*q[2]);
    R[3] = 2*(q[1]*q[2] + q[0]*q[3]); R[4] = q[0]*q[0] - q[1]*q[1] + q[2]*q[2] - q[3]*q[3]; R[5] = 2*(q[2]*q[3] - q[0]*q[1]);
    R[6] = 2*(q[1]*q[3] - q[0]*q[2]); R[7] = 2*(q[2]*q[3] + q[0]*q[1]); R[8] = q[0]*q[0] - q[1]*q[1] - q[2]*q[2] + q[3]*q[3];
  };
  const int b = h.at(&DevModel::geom_bodyid)[g];
  double Rb[9], q[4], R[9];
  q2m(&bq[4 * b], Rb);
  qmul(&bq[4 * b], &gq[4 * g], q);
  double nq = std::sqrt(q[0]*q[0] + q[1]*q[1] + q[2]*q[2] + q[3]*q[3]);
  for (double& x : q) x /= nq;
  q2m(q, R);
  for (int i = 0; i < 3; i++)
    o[i] = (float)(bp[3 * b + i] + Rb[3 * i] * gp[3 * g] + Rb[3 * i + 1] * gp[3 * g + 1] + Rb[3 * i + 2] * gp[3 * g + 2]);
  for (int i = 0; i < 9; i++) o[3 + i] = (float)R[i];
  o[12] = (float)h.at(&DevModel::geom_rbound)[g];
}

// Collision plan: pose slots of the collision geoms, the grid-static set, a narrowphase routine for every pair, the
// broadphase pair words and the height-field pairs grouped by field.
static int collision_plan(b2_sim* s, const HostModel& h) {
  DevModel& m = s->hm;
  const std::vector<int>& parent = h.at(&DevModel::body_parentid); const std::vector<int>& dofnum = h.at(&DevModel::body_dofnum);
  const std::vector<int>& bodyid = h.at(&DevModel::geom_bodyid); const std::vector<int>& gt = h.at(&DevModel::geom_type);
  const std::vector<int>& pg1 = h.at(&DevModel::pair_geom1); const std::vector<int>& pg2 = h.at(&DevModel::pair_geom2);
  const std::vector<int>& sg = h.at(&DevModel::static_geom); const std::vector<int>& dyn = h.at(&DevModel::dyn_cgeom);
  const std::vector<int>& did = h.at(&DevModel::geom_dataid);
  std::vector<int> cslot(m.ngeom, -1), cgeom, fixed_geom, posegeom;  // (cslot: pose slot, or -2 - index into fixed_pose)
  auto welded = [&](int g) { int b = bodyid[g]; return b == 0 || (parent[b] == 0 && dofnum[b] == 0); };
  // Height fields welded to the world (a terrain has tens of them) get no slot: their pose records live in global
  // memory (fixed_pose, slot code -2 - index) - 56 bytes of shared memory per field and per environment otherwise,
  // and a pose computation per step.
  {
    std::vector<char> second(m.ngeom, 0);
    for (int p = 0; p < m.npair; p++) second[pg2[p]] = 1;
    for (int p = 0; p < m.npair; p++) {
      for (int g : {pg1[p], pg2[p]}) {
        if (cslot[g] != -1) continue;
        if (gt[g] == G_HFIELD && !second[g] && welded(g)) { cslot[g] = -2 - (int)fixed_geom.size(); fixed_geom.push_back(g); }
        else { cslot[g] = (int)cgeom.size(); cgeom.push_back(g); }
      }
    }
  }
  m.nfixed = (int)fixed_geom.size();
  std::vector<float> fixed_pose((size_t)std::max(m.nfixed, 1) * 16, 0.f);
  for (int f = 0; f < m.nfixed; f++) world_pose(h, fixed_geom[f], fixed_pose.data() + 16 * (size_t)f);
  // grid-static collision set: static geoms never move, so their world poses are computed here once (in
  // double, from world 0's model values) and shared by all worlds; only the other geoms are posed per step
  m.nstatic = (int)h.scalar("nstatic");
  m.ndyn = (int)dyn.size();
  std::vector<float> static_pose((size_t)std::max(m.nstatic, 1) * 16, 0.f);
  std::vector<char> is_static(m.ngeom, 0);
  if ((int)sg.size() != m.nstatic) return fail("b2_create: static_geom / nstatic mismatch");
  if (m.nstatic >= (1 << 20) || m.ndyn >= (1 << 11)) return fail("b2_create: static grid too large");
  for (int k = 0; k < m.nstatic; k++) {
    int g = sg[k], b = bodyid[g];
    if (g < 0 || g >= m.ngeom || parent[b] != 0 || dofnum[b] != 0)
      return fail("b2_create: grid-static geoms must sit on a jointless child of the world body");
    is_static[g] = 1;
    world_pose(h, g, static_pose.data() + 16 * (size_t)k);
  }
  for (int g : fixed_geom) is_static[g] = 1;
  for (int g = 0; g < m.ngeom; g++) if (!is_static[g]) posegeom.push_back(g);
  m.nposegeom = (int)posegeom.size();
  for (int g : dyn) {
    if (g < 0 || g >= m.ngeom || is_static[g]) return fail("b2_create: bad dyn_cgeom entry");
    if (cslot[g] < 0) { cslot[g] = (int)cgeom.size(); cgeom.push_back(g); }
  }
  if (m.nstatic > 0) {
    const std::vector<double>& gpar = HostModel::find(h.f, "grid_params");
    if (gpar.size() != 5) return fail("b2_create: grid_params must hold [x0, y0, cell, nx, ny]");
    m.grid_x0 = (float)gpar[0]; m.grid_y0 = (float)gpar[1]; m.grid_cell = (float)gpar[2];
    m.grid_nx = (int)gpar[3]; m.grid_ny = (int)gpar[4];
    if ((int)h.at(&DevModel::grid_start).size() != m.grid_nx * m.grid_ny + 1 || (int)h.at(&DevModel::static_cell0).size() != 2 * m.nstatic)
      return fail("b2_create: static grid tables have inconsistent sizes");
  }
  m.ncg = (int)cgeom.size();
  // every collision pair must have a narrowphase routine (primitives, or the convex routines of b2_convex.h)
  auto prim = [](int t) { return t == G_SPHERE || t == G_CAPSULE || t == G_BOX; };
  auto smooth = [](int t) { return t == G_ELLIPSOID || t == G_CYLINDER; };
  auto conv = [&](int t) { return prim(t) || t == G_MESH || smooth(t); };  // shapes the GJK/EPA routine takes (b2_convex.h)
  const std::vector<int>& vadr = h.at(&DevModel::mesh_vertadr); const std::vector<int>& vnum = h.at(&DevModel::mesh_vertnum);
  const std::vector<int>& hadr = h.at(&DevModel::hfield_adr); const std::vector<int>& hrow = h.at(&DevModel::hfield_nrow);
  const std::vector<int>& hcol = h.at(&DevModel::hfield_ncol); const std::vector<double>& hsize = h.at(&DevModel::hfield_size);
  const size_t nvert = h.at(&DevModel::mesh_vert).size(), nhdata = h.at(&DevModel::hfield_data).size();
  const int nmesh = (int)vnum.size(), nhf = (int)hrow.size();
  for (int p = 0; p < m.npair; p++) {
    int g1 = pg1[p], g2 = pg2[p];
    int t1 = gt[g1], t2 = gt[g2];
    bool ok = (t1 == G_PLANE && conv(t2)) || (t1 == G_HFIELD && conv(t2)) || (conv(t1) && conv(t2) && t1 <= t2);
    if (t2 == G_MESH || t1 == G_HFIELD || smooth(t1) || smooth(t2)) s->has_convex = 1;
    if (!ok) return fail("b2_create: collision pair with an unsupported geom type combination");
    for (int g : {g1, g2}) {
      int t = gt[g];
      if (t != G_MESH && t != G_HFIELD) continue;
      int id = g < (int)did.size() ? did[g] : -1;
      if (id < 0 || id >= (t == G_MESH ? nmesh : nhf)) return fail("b2_create: colliding mesh / hfield geom without asset data (geom_dataid)");
      if (t == G_MESH && (vnum[id] < 1 || (size_t)3 * (vadr[id] + vnum[id]) > nvert))
        return fail("b2_create: mesh vertex range outside mesh_vert");
      if (t == G_HFIELD && (hrow[id] < 2 || hcol[id] < 2 || (size_t)4 * (id + 1) > hsize.size() ||
                            (size_t)hadr[id] + (size_t)hrow[id] * hcol[id] > nhdata))
        return fail("b2_create: hfield sample range outside hfield_data");
    }
  }
  for (int g : dyn) {
    if (!conv(gt[g])) return fail("b2_create: unsupported dynamic geom type for the static grid");
    if (gt[g] == G_MESH || smooth(gt[g])) s->has_convex = 1;
  }
  for (int g : sg) if (!prim(gt[g])) return fail("b2_create: unsupported grid-static geom type");
  if (m.ncg >= 4096) return fail("b2_create: too many collision geoms");
  int rc = 0;
  std::vector<unsigned> pw(std::max(m.npair, 1), 0u);
  for (int p = 0; p < m.npair; p++) {
    int g1 = pg1[p], g2 = pg2[p];
    pw[p] = (unsigned)std::max(cslot[g1], 0) | ((unsigned)std::max(cslot[g2], 0) << 12) | (gt[g1] == G_PLANE ? 0x80000000u : 0u) |
            (gt[g1] == G_HFIELD ? 0x40000000u : 0u);
  }
  rc |= dev_upload<unsigned>(s, pw, &m.pair_word);
  // height-field pairs grouped by field: the kernel first finds the fields under the robot, then tests only
  // their pairs (a terrain is a grid of fields; the flat pair table would test every one of them)
  std::vector<int> hf_geom, hf_slot, hf_start, hf_pairs, hfd, nh;  // (hf_slot: pose slot, or -2 - index into fixed_pose)
  std::vector<std::vector<int>> per;
  std::vector<float> box;
  for (int p = 0; p < m.npair; p++) {
    int g1 = pg1[p], g2 = pg2[p];
    if (gt[g1] != G_HFIELD) { nh.push_back(p); continue; }
    size_t k = std::find(hf_geom.begin(), hf_geom.end(), g1) - hf_geom.begin();
    if (k == hf_geom.size()) {
      hf_geom.push_back(g1); hf_slot.push_back(cslot[g1]); per.emplace_back();
      for (int j = 0; j < 4; j++) box.push_back((float)hsize[4 * (size_t)did[g1] + j]);
    }
    per[k].push_back(p);
    if (std::find(hfd.begin(), hfd.end(), cslot[g2]) == hfd.end()) hfd.push_back(cslot[g2]);
  }
  m.nhf = (int)hf_geom.size(); m.nhfd = (int)hfd.size(); m.n_nhpair = m.npair;
  m.hfl_slot = m.hfl_geom = m.hfl_start = m.hfl_pairs = m.hfd_slot = m.nh_pairs = nullptr; m.hfl_box = nullptr;
  if (m.nhf > 0) {
    for (auto& v : per) { hf_start.push_back((int)hf_pairs.size()); hf_pairs.insert(hf_pairs.end(), v.begin(), v.end()); }
    hf_start.push_back((int)hf_pairs.size());
    m.n_nhpair = (int)nh.size();
    if (nh.empty()) nh.push_back(0);
    const float* bp = nullptr;
    rc |= dev_upload<int>(s, hf_slot, &m.hfl_slot); rc |= dev_upload<int>(s, hf_start, &m.hfl_start);
    rc |= dev_upload<int>(s, hf_geom, &m.hfl_geom);
    rc |= dev_upload<int>(s, hf_pairs, &m.hfl_pairs); rc |= dev_upload<int>(s, hfd, &m.hfd_slot);
    rc |= dev_upload<int>(s, nh, &m.nh_pairs); rc |= dev_upload<float>(s, box, &bp);
    m.hfl_box = (const float4*)bp;
  }
  rc |= dev_upload<int>(s, posegeom, &m.posegeom);
  rc |= dev_upload<float>(s, static_pose, &m.static_pose);
  rc |= dev_upload<int>(s, cslot, &m.geom_cslot);
  rc |= dev_upload<float>(s, fixed_pose, &m.fixed_pose);
  if (fixed_geom.empty()) fixed_geom.push_back(0);
  rc |= dev_upload<int>(s, fixed_geom, &m.fixed_geom);
  rc |= dev_upload<int>(s, cgeom, &m.cgeom);
  return rc;
}

// The model's arrays on the device (fp32 floats, shared by all worlds), its Model fields, and the schedules of the
// bottom-up blocked factorisation (b2_kernel.cuh: ldl_factor).
static int upload_model(b2_sim* s, const HostModel& h) {
  DevModel& m = s->hm;
  for (const IntArray& r : kIntArrays) {
    if (dev_upload<int>(s, h.at(r.dev), &(m.*r.dev))) return 1;
    if (r.field) {  // 1-D, shared by all worlds
      Field f; f.name = r.name; f.ptr = (void*)(m.*r.dev); f.dtype = B2_I32; f.ndim = 1;
      f.n = f.shape[0] = (int64_t)h.at(r.dev).size(); f.stride[0] = 1;
      s->model_fields.push_back(f);
    }
  }
  for (const AssetArray& r : kAssetArrays) {
    const std::vector<double>& v = h.at(r.dev);
    if (dev_upload<float>(s, std::vector<float>(v.begin(), v.end()), &(m.*r.dev))) return 1;
  }
  for (const FloatArray& r : kFloatArrays) {
    const std::vector<double>& v = h.at(r.dev);
    const float* p = nullptr;
    if (dev_upload<float>(s, std::vector<float>(v.begin(), v.end()), &p)) return 1;
    FArr& fa = m.*r.dev;
    fa.p = p; fa.stride = 0; fa.n = (int)v.size();
    Field f = make_field(r.name, (void*)p, B2_F32, s->nworld, 0, (int64_t)v.size(), r.width, false);
    f.farr = &fa;
    s->model_fields.push_back(f);
  }
  std::vector<unsigned> dense, sparse;
  b2_build_ldl_schedules(m.nv, h.at(&DevModel::dof_parentid).data(), dense, sparse, m.ldl_start);
  m.ldl_nsparse = (int)sparse.size();
  return dev_upload<unsigned>(s, dense, &m.ldl_dense) || dev_upload<unsigned>(s, sparse, &m.ldl_sparse);
}

// Per-world Data arrays (zeroed), registered as Data fields in this order.
static int alloc_data(b2_sim* s) {
  const DevModel& m = s->hm;
  DevData& d = s->hd;
  memset(&d, 0, sizeof(d));
  d.nworld = s->nworld;
  const int nq = m.nq, nv = m.nv, nu = m.nu, nb = m.nbody, ng = m.ngeom, ns = m.nsite, mc = m.maxcon;
  const DataArray<DArr> floats[] = {
      {"qpos", &DevData::qpos, nq}, {"qvel", &DevData::qvel, nv}, {"ctrl", &DevData::ctrl, nu},
      {"qacc_warmstart", &DevData::qacc_warmstart, nv}, {"qfrc_applied", &DevData::qfrc_applied, nv},
      {"xfrc_applied", &DevData::xfrc_applied, 6 * nb, 6}, {"act", &DevData::act, 0}, {"qacc", &DevData::qacc, nv},
      {"xpos", &DevData::xpos, 3 * nb, 3}, {"xquat", &DevData::xquat, 4 * nb, 4}, {"xmat", &DevData::xmat, 9 * nb, 9},
      {"xipos", &DevData::xipos, 3 * nb, 3}, {"subtree_com", &DevData::subtree_com, 3 * nb, 3},
      {"cvel", &DevData::cvel, 6 * nb, 6}, {"geom_xpos", &DevData::geom_xpos, 3 * ng, 3},
      {"geom_xmat", &DevData::geom_xmat, 9 * ng, 9}, {"site_xpos", &DevData::site_xpos, 3 * ns, 3},
      {"site_xmat", &DevData::site_xmat, 9 * ns, 9}, {"link_vel_w", &DevData::link_vel_w, 6 * nb, 6},
      {"com_vel_w", &DevData::com_vel_w, 6 * nb, 6}, {"link_state_b", &DevData::link_state_b, 10 * nb, 10},
      {"sensordata", &DevData::sensordata, m.nsensordata}, {"actuator_force", &DevData::actuator_force, nu},
      {"time", &DevData::time, 1, 0, true}, {"qfrc_bias", &DevData::qfrc_bias, nv},
      {"qfrc_smooth", &DevData::qfrc_smooth, nv}, {"qacc_smooth", &DevData::qacc_smooth, nv},
      {"qfrc_constraint", &DevData::qfrc_constraint, nv}, {"qM", &DevData::qM, nv * nv, nv},
      {"qM_packed", &DevData::qM_packed, m.ntri}, {"qacc_smooth_prev", &DevData::qacc_smooth_prev, nv},
      {"ctrl_prev", &DevData::ctrl_prev, nu}, {"contact_dist", &DevData::contact_dist, mc},
      {"contact_pos", &DevData::contact_pos, 3 * mc, 3}, {"contact_frame", &DevData::contact_frame, 9 * mc, 9},
      {"contact_force", &DevData::contact_force, 3 * mc, 3}, {"solver_cost", &DevData::solver_cost, 1, 0, true}};
  const DataArray<IArr> ints[] = {
      {"ncon", &DevData::ncon, 1, 0, true}, {"nefc", &DevData::nefc, 1, 0, true},
      {"solver_niter", &DevData::solver_niter, 1, 0, true}, {"contact_geom", &DevData::contact_geom, 2 * mc, 2},
      {"overflow", &DevData::overflow, 1, 0, true}, {"solver_nd", &DevData::solver_nd, 1, 0, true},
      {"solver_nls", &DevData::solver_nls, 1, 0, true}};  // (solver_nls: line-search derivative evaluations of the last step)
  for (const auto& r : floats) if (add_data(s, r)) return 1;
  for (const auto& r : ints) if (add_data(s, r)) return 1;
  return 0;
}

// Offsets of every region of one environment's shared-memory block (floats per environment), and the kernels'
// dynamic shared-memory limit.
static int shared_memory_layout(b2_sim* s, const HostModel& h) {
  DevModel& m = s->hm;
  const DevData& d = s->hd;
  const int nv = m.nv, nu = m.nu, nb = m.nbody, mc = m.maxcon;
  Layout& L = m.lay;
  int off = 0;
  auto alloc = [&](int n) { int o = off; off += pad4(std::max(n, 1)); return o; };
  L.maxcon = mc;
  L.nlimcap = pad4(std::max(m.njnt, 1));
  L.maxpair = m.nstatic > 0 ? 256 : 128;
  L.qpos = alloc(d.qpos.stride); L.qvel = alloc(d.qvel.stride); L.qacc_ws = alloc(d.qacc_warmstart.stride);
  L.cdof = alloc(7 * nv);
  int hsize = std::max(m.ntri, pad4(GP * m.ncg) + L.maxpair);
  L.H = alloc(hsize); L.gpose = L.H; L.pairlist = L.H + pad4(GP * m.ncg);
  L.invdiag = alloc(nv);
  L.qfrc_smooth = alloc(nv); L.qacc_smooth = alloc(nv); L.qacc = alloc(nv); L.Ma = alloc(nv);
  L.grad = alloc(nv); L.search = L.grad;  // search = -grad is formed in place
  L.Mv = alloc(nv); L.qfrc_c = alloc(nv); L.tmpv = alloc(nv);
  L.actf = alloc(nu);
  int ubase = off;
  // union A: regions that are dead once the smooth dynamics (phases 1-4) are done
  L.xpos = alloc(3 * nb); L.xquat = alloc(4 * nb); L.xipos = alloc(3 * nb); L.scom = alloc(3 * nb);
  L.cinert = alloc(11 * nb); L.crb = alloc(11 * nb);
  // joint anchors / axes are dead once the motion vectors exist (phase 2); cdofdot is first written in phase 4
  L.cdofdot = alloc(std::max(7 * nv, 2 * pad4(3 * m.njnt))); L.xanchor = L.cdofdot; L.xaxis = L.cdofdot + pad4(3 * m.njnt);
  L.cvel = alloc(7 * nb);
  L.cacc = alloc(7 * nb);
  int endA = off;
  off = ubase;
  // union B: constraint / solver regions
  L.contacts = alloc(C_NFIELD * mc); L.limits = alloc(L_NFIELD * L.nlimcap); L.gstart = alloc(mc + 1);
  // gV (group velocities / wrenches: J x, J^T f) and gu (Hessian projection) are never live together
  L.gV = alloc(std::max(6 * mc, 6 * nv)); L.gu = L.gV; L.glist = alloc(nv + 1); L.gA = alloc(36);
  L.gW = alloc(std::max(5 * mc, 4 * pad4(nv))); L.sens = off;  // (the CG variant keeps its four vectors here)
  // reduced Newton problem: room for the Schur complement on the largest leading block nv - 4k (k >= 1) whose
  // packed size fits 200 floats (G1: 19 x 19 = both legs + the first waist dof, 82 % of the bench workload's
  // environments; torso / arm contacts fall back to the full problem)
  L.ndcap = 0;
  for (int k = 1; nv - 4 * k >= 6; k++) {
    int cand = nv - 4 * k;
    if (cand * (cand + 1) / 2 <= 200) { L.ndcap = cand; break; }
  }
  L.Mred = alloc(L.ndcap * (L.ndcap + 1) / 2);
  int endB = off;
  // the lane-distributed height-field narrowphase keeps its owner records and its queue in the (then unused)
  // solver regions from gV on
  if (!h.at(&DevModel::hfield_data).empty()) endB = std::max(endB, L.gV + HF_SCRATCH);
  L.total = pad4(std::max(endA, endB));
  if (L.ndcap == 0) L.Mred = L.H;  // never used
  s->smem_bytes = sizeof(float) * ((size_t)L.total * B2_WARPS_PER_CTA + pad4(m.ldl_nsparse + 18));
  if (s->smem_bytes > 227 * 1024) return fail("b2_create: model too large for the per-environment shared-memory block");
  // The attribute is per function and per device, not per sim: only ever raise it, so that an earlier,
  // larger sim in the same process keeps launching after a smaller one is created.
  static size_t dev_max[64] = {0};
  if (s->smem_bytes > dev_max[s->device & 63]) {
    cudaError_t e1 = cudaFuncSetAttribute(b2_step_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s->smem_bytes);
    cudaError_t e2 = cudaFuncSetAttribute(b2_step_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s->smem_bytes);
    if (e1 == cudaSuccess) e1 = cudaFuncSetAttribute(b2_step_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s->smem_bytes);
    if (e2 == cudaSuccess) e2 = cudaFuncSetAttribute(b2_step_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s->smem_bytes);
    if (e1 != cudaSuccess || e2 != cudaSuccess)
      return fail(std::string("cudaFuncSetAttribute(max dynamic smem): ") + cudaGetErrorString(e1 != cudaSuccess ? e1 : e2));
    dev_max[s->device & 63] = s->smem_bytes;
  }
  return 0;
}

// Heavy-first order, the step kernel's co-resident CTAs, and the streams of b2_step_n.
static int launch_resources(b2_sim* s) {
  void* p = nullptr;
  if (cudaMalloc(&p, sizeof(int) * (size_t)s->nworld) != cudaSuccess) return fail("cudaMalloc(order)");
  s->allocs.push_back(p);
  s->order = (int*)p;
  int per_sm = 0, sms = 0;
  // (of the instantiation that steps this model: the convex one has a larger register budget)
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, s->has_convex ? b2_step_kernel<3> : b2_step_kernel<1>,
                                                32 * B2_WARPS_PER_CTA, s->smem_bytes);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, s->device);
  s->resident_ctas = per_sm * sms;
  for (int h = 0; h < 2; h++)
    if (cudaStreamCreateWithFlags(&s->side[h], cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&s->ev_join[h], cudaEventDisableTiming) != cudaSuccess)
      return fail("b2_create: stream/event creation failed");
  if (cudaEventCreateWithFlags(&s->ev_fork, cudaEventDisableTiming) != cudaSuccess) return fail("event");
  return 0;
}

// qpos <- qpos0 in every world, the constant poses of the static geoms, then one forward pass so all derived
// fields are valid.
static int first_forward(b2_sim* s) {
  const DevModel& m = s->hm;
  const DevData& d = s->hd;
  const int nworld = s->nworld;
  long long total = (long long)nworld * m.nq;
  b2_init_rows_kernel<<<(unsigned)((total + 255) / 256), 256>>>(d.qpos.p, d.qpos.stride, m.qpos0.p, m.nq, nworld);
  s->launches++;
  struct { int n; const float* pose; const int* geom; } posed[] = {{m.nstatic, m.static_pose, m.static_geom},
                                                                   {m.nfixed, m.fixed_pose, m.fixed_geom}};
  for (const auto& p : posed) {
    if (p.n == 0) continue;
    long long tot = (long long)nworld * p.n;
    b2_static_rows_kernel<<<(unsigned)((tot + 255) / 256), 256>>>(d.geom_xpos.p, d.geom_xpos.stride, d.geom_xmat.p,
                                                                   d.geom_xmat.stride, p.pose, p.geom, p.n, nworld);
    s->launches++;
  }
  if (launch(s, false, 0)) return 1;
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return fail(std::string("b2_create: initial forward failed: ") + cudaGetErrorString(e));
  return 0;
}

int b2_create(const B2ModelDesc* desc, int nworld, int ncon_per_world, int njmax, int cuda_device,
              b2_sim** out) {
  if (!desc || !out || nworld <= 0) return fail("b2_create: bad arguments");
  HostModel h;
  std::string why = read_desc(desc, h);
  if (!why.empty()) return fail("b2_create: " + why);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("b2_create: no CUDA device available (this library has no CPU path)");
  if (cuda_device < 0 || cuda_device >= ndev) return fail("b2_create: bad cuda_device");
  DeviceGuard guard(cuda_device);
  // the sim and everything allocated for it are released on every refusal below; handed out only on success
  std::unique_ptr<b2_sim, int (*)(b2_sim*)> s(new b2_sim(), b2_destroy);
  s->device = cuda_device;
  s->nworld = nworld;
  if (read_model(desc, ncon_per_world, njmax, h, s->hm) || kinematic_tables(s.get(), h) || collision_plan(s.get(), h) ||
      upload_model(s.get(), h) || alloc_data(s.get()) || shared_memory_layout(s.get(), h) || launch_resources(s.get()) ||
      first_forward(s.get()))
    return 1;
  *out = s.release();
  return 0;
}

int b2_destroy(b2_sim* s) {
  if (!s) return 0;
  DeviceGuard guard(s->device);
  for (void* p : s->allocs) cudaFree(p);
  for (void* p : s->host_allocs) b2g_word_free(p);
  for (int h = 0; h < 2; h++) {
    if (s->side[h]) cudaStreamDestroy(s->side[h]);
    if (s->ev_join[h]) cudaEventDestroy(s->ev_join[h]);
  }
  if (s->ev_fork) cudaEventDestroy(s->ev_fork);
  delete s;
  return 0;
}

static Field* find_field(b2_sim* s, int which, const char* name) {
  std::vector<Field>& v = which == B2_DATA ? s->data_fields : s->model_fields;
  for (Field& f : v)
    if (f.name == name) return &f;
  return nullptr;
}
static void fill_tensor(b2_sim* s, const Field& f, B2Tensor* out) {
  out->ptr = f.ptr; out->dtype = f.dtype; out->ndim = f.ndim; out->device = s->device;
  for (int k = 0; k < 4; k++) { out->shape[k] = f.shape[k]; out->stride[k] = f.stride[k]; }
}

int b2_get_field(b2_sim* s, int which, const char* name, B2Tensor* out) {
  if (!s || !name || !out) return fail("b2_get_field: bad arguments");
  Field* f = find_field(s, which, name);
  if (!f) return fail(std::string("b2_get_field: unknown field '") + name + "'");
  fill_tensor(s, *f, out);
  return 0;
}
int b2_num_fields(b2_sim* s, int which) {
  return (int)(which == B2_DATA ? s->data_fields.size() : s->model_fields.size());
}
const char* b2_field_name(b2_sim* s, int which, int index) {
  std::vector<Field>& v = which == B2_DATA ? s->data_fields : s->model_fields;
  if (index < 0 || index >= (int)v.size()) return nullptr;
  return v[index].name.c_str();
}

int b2_expand_model_field(b2_sim* s, const char* name, void* stream, B2Tensor* out) {
  if (!s || !name) return fail("b2_expand_model_field: bad arguments");
  Field* f = find_field(s, B2_MODEL, name);
  if (!f || !f->farr) return fail(std::string("b2_expand_model_field: '") + name + "' is not an expandable model field");
  DeviceGuard guard(s->device);
  if (f->farr->stride == 0 && s->nworld > 1) {
    int n = f->farr->n;
    void* p = nullptr;
    long long total = (long long)s->nworld * n;
    CUDA_OK(cudaMalloc(&p, sizeof(float) * (size_t)total));
    s->allocs.push_back(p);
    b2_tile_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(f->farr->p, (float*)p, n, total);
    s->launches++;
    CUDA_OK(cudaGetLastError());
    f->farr->p = (const float*)p; f->farr->stride = n;
    const DevModel& m = s->hm;
    if (f->farr == &m.body_pos || f->farr == &m.body_quat || f->farr == &m.jnt_pos || f->farr == &m.jnt_axis ||
        f->farr == &m.qpos0)
      s->hm.fastkin = 0;  // the compact kinematic records hold one row: per-world frames take the generic walk
    f->ptr = p; f->stride[0] = n;
  }
  if (out) fill_tensor(s, *f, out);
  return 0;
}

// Options of b2_set_option / b2_get_option.  A value lives in an int or a float of the sim or its model, or in a
// bit of DevModel::debug; read-only ones report what b2_create derived.  Setting an int or a bit takes (int)value,
// a bit is set by any non-zero value.
struct OptionRef { int* i; float* f = nullptr; int bit = 0; double scale = 1.0; };  // *f, bit `bit` of *i, or scale * *i
struct Option {
  const char* name;
  OptionRef (*ref)(b2_sim*);
  bool read_only = false;
  const char* (*refuse)(double) = nullptr;  // optional: why a value is not taken (nullptr when it is)
};
static const Option kOptions[] = {
    {"iterations", [](b2_sim* s) { return OptionRef{&s->hm.iterations}; }},
    {"ls_iterations", [](b2_sim* s) { return OptionRef{&s->hm.ls_iterations}; }},
    {"tolerance", [](b2_sim* s) { return OptionRef{nullptr, &s->hm.tolerance}; }},
    {"ls_tolerance", [](b2_sim* s) { return OptionRef{nullptr, &s->hm.ls_tolerance}; }},
    {"timestep", [](b2_sim* s) { return OptionRef{nullptr, &s->hm.timestep}; }},
    {"integrator", [](b2_sim* s) { return OptionRef{&s->hm.integrator}; }},
    {"solver", [](b2_sim* s) { return OptionRef{&s->hm.solver}; }, false, [](double v) -> const char* {
       return (int)v == SOL_NEWTON_ || (int)v == SOL_CG_ ? nullptr : "b2_set_option: solver must be 1 (CG) or 2 (Newton)"; }},
    {"debug_outputs", [](b2_sim* s) { return OptionRef{&s->hm.debug, nullptr, 1}; }},
    {"dense_factor", [](b2_sim* s) { return OptionRef{&s->hm.debug, nullptr, 2}; }},  // force the dense LDL schedule (tests)
    {"full_solver", [](b2_sim* s) { return OptionRef{&s->hm.debug, nullptr, 4}; }},  // Newton on all dofs even when a leading block suffices (tests, A/B)
    {"sorted_dispatch", [](b2_sim* s) { return OptionRef{&s->sorted_dispatch}; }},
    {"smem_bytes_per_env", [](b2_sim* s) { return OptionRef{&s->hm.lay.total, nullptr, 0, 4.0}; }, true},
    {"maxcon", [](b2_sim* s) { return OptionRef{&s->hm.maxcon}; }, true},
    {"resident_ctas", [](b2_sim* s) { return OptionRef{&s->resident_ctas}; }, true},
    {"reduced_block_cap", [](b2_sim* s) { return OptionRef{&s->hm.lay.ndcap}; }, true}};

static const Option* find_option(const char* key) {
  for (const Option& o : kOptions)
    if (!strcmp(o.name, key)) return &o;
  return nullptr;
}

int b2_set_option(b2_sim* s, const char* key, double v) {
  if (!s || !key) return fail("b2_set_option: bad arguments");
  const Option* o = find_option(key);
  if (!o || o->read_only) return fail(std::string("b2_set_option: unknown option '") + key + "'");
  if (o->refuse && o->refuse(v)) return fail(o->refuse(v));
  OptionRef r = o->ref(s);
  if (r.f) *r.f = (float)v;
  else if (r.bit) *r.i = (*r.i & ~r.bit) | ((int)v ? r.bit : 0);
  else *r.i = (int)v;
  return 0;
}
int b2_get_option(b2_sim* s, const char* key, double* v) {
  if (!s || !key || !v) return fail("b2_get_option: bad arguments");
  const Option* o = find_option(key);
  if (!o) return fail(std::string("b2_get_option: unknown option '") + key + "'");
  OptionRef r = o->ref(s);
  *v = r.f ? (double)*r.f : r.bit ? (double)((*r.i & r.bit) != 0) : r.scale * *r.i;
  return 0;
}

int b2_step(b2_sim* s, void* stream) {
  if (!s) return fail("b2_step: null sim");
  DeviceGuard guard(s->device);
  cudaStream_t st = (cudaStream_t)stream;
  return refresh_kinrec(s, st) || guard_start(s, st, 1) || launch(s, true, st) || guard_check(s, st, 0, s->nworld, 0, 0);
}
int b2_forward(b2_sim* s, void* stream) {
  if (!s) return fail("b2_forward: null sim");
  DeviceGuard guard(s->device);
  return refresh_kinrec(s, (cudaStream_t)stream) || launch(s, false, (cudaStream_t)stream);
}
int b2_forward_masked(b2_sim* s, const unsigned char* world_mask_dev, void* stream) {
  if (!s) return fail("b2_forward_masked: null sim");
  DeviceGuard guard(s->device);
  if (refresh_kinrec(s, (cudaStream_t)stream)) return 1;
  s->hd.world_mask = world_mask_dev;
  int rc = launch(s, false, (cudaStream_t)stream);
  s->hd.world_mask = nullptr;
  return rc;
}
int b2_step_n(b2_sim* s, int n, void* stream) {
  if (!s) return fail("b2_step_n: null sim");
  DeviceGuard guard(s->device);
  if (n <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (refresh_kinrec(s, st)) return 1;
  if (n > 1 && s->nworld >= 2048) {
    // Environments are independent, so the sub-steps of one half need not wait for the other: fork two
    // partitions onto internal streams (event fork/join, CUDA-graph capturable). Each partition keeps
    // per-sub-step launches (phase-aligned warps, fresh heavy-first order) while its launch tails overlap the
    // other partition's work.  (1, 3 and 4 partitions measured slower on the H100; DESIGN.md §9.)
    // While the NaN guard is armed the partitions join every B2_GUARD_CHUNK sub-steps, which bounds how far one can
    // run ahead of the other's detection (b2_nanguard.cuh).
    int per = (((s->nworld + 1) / 2 + B2_WARPS_PER_CTA - 1) / B2_WARPS_PER_CTA) * B2_WARPS_PER_CTA;
    const int chunk = s->guard_on ? B2_GUARD_CHUNK : n;
    for (int c0 = 0; c0 < n; c0 += chunk) {
      const int m = std::min(chunk, n - c0);
      if (guard_start(s, st, m)) return 1;
      CUDA_OK(cudaEventRecord(s->ev_fork, st));
      for (int h = 0; h < 2; h++) {
        int base = h * per, count = std::min(per, s->nworld - base);
        CUDA_OK(cudaStreamWaitEvent(s->side[h], s->ev_fork, 0));
        for (int i = 0; i < m; i++)
          if (launch(s, true, s->side[h], base, count, c0 + i == n - 1) ||
              guard_check(s, s->side[h], base, count, i, i < m - 1))
            return 1;
        CUDA_OK(cudaEventRecord(s->ev_join[h], s->side[h]));
        CUDA_OK(cudaStreamWaitEvent(st, s->ev_join[h], 0));
      }
    }
    return 0;
  }
  if (guard_start(s, st, n)) return 1;
  for (int i = 0; i < n; i++)
    if (launch(s, true, st, 0, -1, i == n - 1) || guard_check(s, st, 0, s->nworld, i, i < n - 1)) return 1;
  return 0;
}

int b2_nan_guard(b2_sim* s, int ncapture, int buffer_size, int flags) {
  if (!s) return fail("b2_nan_guard: null sim");
  if (flags != 0 && flags != B2_NAN_GUARD_ON) return fail("b2_nan_guard: flags must be 0 or B2_NAN_GUARD_ON");
  if (flags == 0) {
    s->guard_on = 0;
    return 0;
  }
  if (ncapture < 1 || ncapture > s->nworld || buffer_size < 1)
    return fail("b2_nan_guard: needs 1 <= ncapture <= nworld (" + std::to_string(s->nworld) + ") and buffer_size >= 1");
  const long long row = s->hm.nq + s->hm.nv, slots = (long long)buffer_size + B2_GUARD_CHUNK - 1;
  if (slots * ncapture > (1LL << 36) / row) return fail("b2_nan_guard: the ring of buffer_size x ncapture states is too large");
  DeviceGuard guard(s->device);
  CUDA_OK(cudaDeviceSynchronize());  // (work in flight keeps the last arming's buffers, which stay allocated)
  B2Guard g = {};
  g.slots = (int)slots;
  g.ncapture = ncapture;
  void* p = nullptr;
  const size_t ring_bytes = sizeof(float) * (size_t)(slots * ncapture * row);
  CUDA_OK(cudaMalloc(&p, ring_bytes));
  s->allocs.push_back(p);
  CUDA_OK(cudaMemset(p, 0, ring_bytes));
  g.ring = (float*)p;
  const long long ctl[3] = {0, 0, B2_GUARD_NONE};
  CUDA_OK(cudaMalloc(&p, sizeof(ctl)));
  s->allocs.push_back(p);
  CUDA_OK(cudaMemcpy(p, ctl, sizeof(ctl), cudaMemcpyHostToDevice));
  g.ctl = (long long*)p;
  const std::vector<long long> none(s->nworld, B2_GUARD_NONE);
  CUDA_OK(cudaMalloc(&p, sizeof(long long) * none.size()));
  s->allocs.push_back(p);
  CUDA_OK(cudaMemcpy(p, none.data(), sizeof(long long) * none.size(), cudaMemcpyHostToDevice));
  g.first_bad = (long long*)p;
  void* dp = nullptr;
  CUDA_OK(b2g_word_alloc(&p, &dp));
  s->host_allocs.push_back(p);
  *(volatile int*)p = 0;
  g.word = (volatile int*)dp;
  CUDA_OK(cudaDeviceSynchronize());
  s->guard = g;
  s->guard_buffer = buffer_size;
  s->guard_on = 1;
  return 0;
}

const volatile int32_t* b2_nan_guard_word(b2_sim* s) {
  return s && s->guard_on ? (const volatile int32_t*)s->host_allocs.back() : nullptr;
}

int b2_nan_guard_read(b2_sim* s, void* stream, int64_t* detected, float* states, unsigned char* flags) {
  if (!s || !detected) return fail("b2_nan_guard_read: bad arguments");
  if (!s->guard_on) return fail("b2_nan_guard_read: the NaN guard is not armed");
  DeviceGuard guard(s->device);
  CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
  const B2Guard& g = s->guard;
  long long ctl[3];
  CUDA_OK(cudaMemcpy(ctl, g.ctl, sizeof(ctl), cudaMemcpyDeviceToHost));
  *detected = ctl[2] == B2_GUARD_NONE ? -1 : ctl[2];
  if (*detected < 0) return 0;
  const long long d = ctl[2], first = std::max(0LL, d - s->guard_buffer + 1);
  const size_t entry = (size_t)g.ncapture * (s->hm.nq + s->hm.nv);
  if (states) {
    std::vector<float> ring((size_t)g.slots * entry);
    CUDA_OK(cudaMemcpy(ring.data(), g.ring, sizeof(float) * ring.size(), cudaMemcpyDeviceToHost));
    for (long long k = first; k <= d; k++)
      memcpy(states + (size_t)(k - first) * entry, ring.data() + (size_t)(k % g.slots) * entry, sizeof(float) * entry);
  }
  if (flags) {
    std::vector<long long> fb(s->nworld);
    CUDA_OK(cudaMemcpy(fb.data(), g.first_bad, sizeof(long long) * fb.size(), cudaMemcpyDeviceToHost));
    for (int w = 0; w < s->nworld; w++) flags[w] = fb[w] == d;
  }
  return 0;
}

int b2_velenv_pre(b2_sim* s, const float* action, const float* default_joint_pos,
                  const float* action_scale, void* stream) {
  if (!s || !action) return fail("b2_velenv_pre: bad arguments");
  DeviceGuard guard(s->device);
  long long total = (long long)s->nworld * s->hm.nu;
  if (total == 0) return 0;
  b2_velenv_pre_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      s->hd, s->hm.nu, action, default_joint_pos, action_scale);
  s->launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}
int b2_velenv_post(b2_sim* s, const B2VelEnvArgs* args, void* stream) {
  if (!s || !args) return fail("b2_velenv_post: bad arguments");
  if (s->hm.nq != s->hm.nu + 7 || s->hm.nv != s->hm.nu + 6)
    return fail("b2_velenv_post: expects one floating base plus nu actuated hinge joints");
  if (args->curriculum &&
      (!args->env_origins || !args->terrain_origins || !args->terrain_levels || !args->terrain_types ||
       !args->terrain_level_mean || args->rows < 1 || args->cols < 1))
    return fail("b2_velenv_post: the terrain curriculum needs env_origins, terrain_origins, terrain_levels, "
                "terrain_types, terrain_level_mean and rows, cols >= 1");
  const B2VelEnvArgs& a = *args;
  const float* W = a.weight;
  const bool feet_ok = a.n_air >= 0 && a.n_air <= 32 && a.n_slide >= 0 && a.n_slide <= 32 && a.n_clear >= 0 &&
                       a.n_clear <= 32 && a.root_body >= 0 && a.root_body < s->hm.nbody;
  if (!feet_ok || (W[0] != 0.f && (!a.air_sensor_adr || !a.air_time || !a.contact_time || !a.last_air_time)) ||
      (W[1] != 0.f && (!a.slide_sensor_adr || !a.slide_geom || !a.slide_body)) ||
      (W[2] != 0.f && (!a.clear_geom || !a.clear_body)))
    return fail("b2_velenv_post: the reward terms need at most 32 feet each, a valid root_body and the arrays of "
                "every term with a non-zero weight");
  if (!(a.resample_lo > 0.f && a.resample_span >= 0.f && a.ang_lo <= a.ang_hi))
    return fail("b2_velenv_post: the command needs resample_lo > 0, resample_span >= 0 and ang_lo <= ang_hi");
  if (a.n_stage < 0 || a.n_stage > B2_VELENV_NSTAGE || (a.n_stage > 0 && !a.step_counter))
    return fail("b2_velenv_post: the command curriculum needs 0 <= n_stage <= B2_VELENV_NSTAGE and a step_counter");
  if (!a.episode_sums || !a.finished_sums || !a.posture_inv_std2 || !a.metric_xy || !a.metric_yaw ||
      !a.finished_metrics || !(a.metric_steps > 0.f))
    return fail("b2_velenv_post: needs episode_sums, finished_sums, posture_inv_std2, metric_xy, metric_yaw, "
                "finished_metrics and metric_steps > 0");
  if (a.n_reset < 0 || a.n_reset > B2_VELENV_NRESET || (a.n_reset > 0 && (!a.ev_V || a.ev_v_width < 1)))
    return fail("b2_velenv_post: the reset state terms need 0 <= n_reset <= B2_VELENV_NRESET and the events' V");
  for (int t = 0; t < a.n_reset; t++) {
    const B2VelResetTerm& T = a.reset_term[t];
    const std::string which = "b2_velenv_post: reset term " + std::to_string(t);
    if (T.kind != B2_RESET_ROOT && T.kind != B2_RESET_JOINTS) return fail(which + " has an unknown kind code");
    const int draws = T.kind == B2_RESET_ROOT ? 12 : 2 * T.count;
    if ((T.kind == B2_RESET_ROOT ? T.count != 12 : (T.count < 1 || T.count > 32)) || T.col < 0 ||
        (long long)T.col + draws > a.ev_v_width)
      return fail(which + " reads V columns outside the row or has a bad count");
    for (int j = 0; T.kind == B2_RESET_JOINTS && j < T.count; j++)
      if (T.joint[j] < 0 || T.joint[j] >= s->hm.nu)
        return fail(which + " names joint " + std::to_string(T.joint[j]) + ", outside 0..nu-1");
  }
  DeviceGuard guard(s->device);
  b2_velenv_post_kernel<<<(s->nworld + 3) / 4, 128, 0, (cudaStream_t)stream>>>(  // one warp per environment
      s->hd, s->hm.nq, s->hm.nv, s->hm.nu, a);
  s->launches++;
  CUDA_OK(cudaGetLastError());
  if (a.n_stage > 0) {
    b2_velenv_counter_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(a.step_counter);
    s->launches++;
    CUDA_OK(cudaGetLastError());
  }
  if (args->curriculum) {
    b2_velenv_level_mean_kernel<<<1, kLevelMeanThreads, 0, (cudaStream_t)stream>>>(
        s->nworld, args->terrain_levels, args->terrain_level_mean);
    s->launches++;
    CUDA_OK(cudaGetLastError());
  }
  return 0;
}

// `settings`: also the task settings and the episode logs, which post1 and post2 read and bins does not
static int trackenv_check(b2_sim* s, const B2TrackEnvArgs* a, bool settings) {
  if (!s || !a) return fail("b2_trackenv: bad arguments");
  if (s->hm.nq != s->hm.nu + 7 || s->hm.nv != s->hm.nu + 6)
    return fail("b2_trackenv: expects one floating base plus nu actuated hinge joints");
  if (a->nb < 1 || a->nb > 32 || a->anchor < 0 || a->anchor >= a->nb || a->T < 2 || a->nee < 0 ||
      a->root_body < 0 || a->root_body >= s->hm.nbody || a->self_collision_adr < 0 ||
      a->self_collision_adr >= s->hm.nsensordata)
    return fail("b2_trackenv: bad sizes (1 <= nb <= 32 tracked bodies, anchor among them, T >= 2 clip frames)");
  if (a->adaptive < B2_START_UNIFORM || a->adaptive > B2_START_FIRST)
    return fail("b2_trackenv: unknown start-frame sampler (adaptive must be one of B2_START_*)");
  if (a->adaptive == B2_START_ADAPTIVE &&
      (a->nbins < 1 || a->adaptive_kernel_size < 1 || !a->adaptive_kernel || !a->cdf || !a->bin_fail_ema ||
       !a->bin_fail_cur || !a->metrics))
    return fail("b2_trackenv: the adaptive sampler needs nbins >= 1, a kernel of size >= 1 and its five arrays");
  if (!settings) return 0;
  const int logs = !!a->episode_sums + !!a->finished_sums + !!a->term_flags + !!a->motion_metrics + !!a->finished_metrics;
  bool ok = logs == 0 || logs == 5;
  for (int k = 0; k < 6; k++) ok = ok && a->std2[k] > 0.f && a->std2[k] < INFINITY;
  for (int k = 0; k < 3; k++)
    ok = ok && (a->term_on[k] == 0 || (a->term_on[k] == 1 && a->term_threshold[k] > 0.f && a->term_threshold[k] < INFINITY));
  for (int k = 0; k < 6; k++)
    ok = ok && a->pose_range[2 * k] <= a->pose_range[2 * k + 1] && a->vel_range[2 * k] <= a->vel_range[2 * k + 1] &&
         (!a->push_on || a->push_range[2 * k] <= a->push_range[2 * k + 1]);
  if (!ok)
    return fail("b2_trackenv: needs the five log arrays all set or all null, finite stds^2 > 0, finite thresholds > 0 "
                "on the terms that are on, and lo <= hi in every range");
  return 0;
}
int b2_trackenv_post1(b2_sim* s, const B2TrackEnvArgs* args, void* stream) {
  if (trackenv_check(s, args, true)) return 1;
  DeviceGuard guard(s->device);
  b2_trackenv_post1_kernel<<<(s->nworld + 3) / 4, 128, 0, (cudaStream_t)stream>>>(s->hd, s->hm.nu, s->hm.nbody, *args);
  s->launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}
int b2_trackenv_post2(b2_sim* s, const B2TrackEnvArgs* args, void* stream) {
  if (trackenv_check(s, args, true)) return 1;
  DeviceGuard guard(s->device);
  b2_trackenv_post2_kernel<<<(s->nworld + 3) / 4, 128, 0, (cudaStream_t)stream>>>(s->hd, s->hm.nu, s->hm.nbody, *args);
  s->launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}
int b2_trackenv_bins(b2_sim* s, const B2TrackEnvArgs* args, void* stream) {
  if (trackenv_check(s, args, false)) return 1;
  if (args->adaptive != B2_START_ADAPTIVE) return fail("b2_trackenv_bins: the args do not select the adaptive sampler");
  DeviceGuard guard(s->device);
  b2_trackenv_bins_kernel<<<1, b2t::kBinThreads, 0, (cudaStream_t)stream>>>(*args);
  s->launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

// The noise block of group g (include/b2sim.h): known codes, and every column, parameter and draw a term reads inside
// its row.
static int obsnoise_check(const B2ObsHistArgs* a, int g) {
  const B2ObsHistGroup& G = a->group[g];
  const B2ObsNoiseGroup& Z = a->noise[g];
  if (a->nW < 0 || a->nN < 0 || a->nparam < 0)
    return fail("b2_obs_history: nW, nN and nparam must be >= 0");
  // one noise class: its parameter rows inside param, its `count` draws from column `draw` inside W or N
  auto noise_ok = [&](int cls, int op, int p0, int p1, int draw, int dim, int count, const char** why) {
    if (cls < B2_NOISE_NONE || cls > B2_NOISE_GAUSSIAN || op < B2_NOISE_ADD || op > B2_NOISE_ABS)
      return *why = "an unknown noise class or operation", false;
    if (cls == B2_NOISE_NONE) return true;
    auto in_param = [&](int p) { return a->param && p >= 0 && (long long)p + dim <= a->nparam; };
    if (!in_param(p0) || (cls != B2_NOISE_CONSTANT && !in_param(p1)))
      return *why = "a parameter row outside param (or no param)", false;
    if (cls == B2_NOISE_CONSTANT) return true;
    const float* row = cls == B2_NOISE_UNIFORM ? a->W : a->N;
    const int width = cls == B2_NOISE_UNIFORM ? a->nW : a->nN;
    if (!row || draw < 0 || (long long)draw + count > width)
      return *why = "draws outside W or N (or no W or N)", false;
    return true;
  };
  for (int t = 0; t < G.nterm; t++) {
    const B2ObsNoiseTerm& M = Z.term[t];
    const int dim = G.term[t].dim;
    const char* why = nullptr;
    if (!noise_ok(M.noise, M.noise_op, M.noise_p0, M.noise_p1, M.noise_draw, dim, dim, &why) ||
        (M.bias_shared != 0 && M.bias_shared != 1 && (why = "bias_shared must be 0 or 1")) ||
        !noise_ok(M.bias, M.bias_op, M.bias_p0, M.bias_p1, M.bias_draw, dim, M.bias_shared ? 1 : dim, &why))
      return fail(std::string("b2_obs_history: noise of a term: ") + why);
    if (M.noise == B2_NOISE_NONE && M.bias == B2_NOISE_NONE) {
      if (Z.source && (M.col < 0 || (long long)M.col + dim > Z.source_width))
        return fail("b2_obs_history: noise of a term: its source columns lie outside the source row");
      continue;
    }
    if (!Z.source) return fail("b2_obs_history: noise of a term: the group has no source row");
    if (M.col < 0 || (long long)M.col + dim > Z.source_width)
      return fail("b2_obs_history: noise of a term: its source columns lie outside the source row");
    if (M.bias != B2_NOISE_NONE && !Z.bias) return fail("b2_obs_history: noise of a term: a bias needs the bias row");
  }
  if (Z.source && Z.source_width < 1) return fail("b2_obs_history: a source row needs source_width >= 1");
  return 0;
}

static int obshist_check(b2_sim* s, const B2ObsHistArgs* a) {
  if (!s || !a) return fail("b2_obs_history: bad arguments");
  if (!a->terminated || !a->truncated || a->ngroup < 1 || a->ngroup > B2_OBSHIST_NGROUP || a->nscale < 0 ||
      (a->nscale > 0 && !a->scale))
    return fail("b2_obs_history: needs terminated, truncated, 1 <= ngroup <= B2_OBSHIST_NGROUP and the scale row");
  for (int g = 0; g < a->ngroup; g++) {
    const B2ObsHistGroup& G = a->group[g];
    if (!G.frame || !G.out || G.frame_width < 1 || G.out_width < 1 || G.nterm < 1 || G.nterm > B2_OBSHIST_NTERM)
      return fail("b2_obs_history: a group needs its frame and out rows, widths >= 1 and 1 <= nterm <= B2_OBSHIST_NTERM");
    std::vector<char> seen(G.out_width, 0);
    long long next = 0, covered = 0;
    for (int t = 0; t < G.nterm; t++) {
      const B2ObsHistTerm& T = G.term[t];
      if (T.src != next || T.dim < 1 || T.frames < 0 || T.stride < 0 || T.scale < -1 ||
          (T.scale >= 0 && (long long)T.scale + T.dim > a->nscale) || (T.clip != 0 && T.clip != 1) ||
          (T.clip && !(T.lo <= T.hi && T.lo > -INFINITY && T.hi < INFINITY)))
        return fail("b2_obs_history: a term needs dim >= 1, frames >= 0, its scale factors inside the scale row and a "
                    "finite clip with lo <= hi, and the terms must follow each other through the frame row");
      next += T.dim;
      const int H = T.frames > 1 ? T.frames : 1;
      for (int k = 0; k < H; k++)
        for (int j = 0; j < T.dim; j++) {
          const long long c = (long long)T.dst + (long long)k * T.stride + j;
          if (c < 0 || c >= G.out_width || seen[c])
            return fail("b2_obs_history: the terms' frames must tile the out row (a column outside it or written twice)");
          seen[c] = 1;
          covered++;
        }
    }
    if (next != G.frame_width || covered != G.out_width)
      return fail("b2_obs_history: the terms' sizes do not add up to frame_width and out_width");
    if (obsnoise_check(a, g)) return 1;
  }
  return 0;
}
int b2_obs_history(b2_sim* s, const B2ObsHistArgs* args, void* stream) {
  if (obshist_check(s, args)) return 1;
  long long total = 0;
  for (int g = 0; g < args->ngroup; g++) total += (long long)s->nworld * args->group[g].frame_width;
  DeviceGuard guard(s->device);
  b2_obs_history_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(s->nworld, *args);
  s->launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

static int events_check(b2_sim* s, const B2EventArgs* a, B2EventFields* F) {
  if (!s || !a) return fail("b2_events: bad arguments");
  if (!a->terminated || !a->truncated || !a->V || (a->nterm > 0 && !a->elem) || a->v_width < 1 || a->nterm < 0 ||
      a->nterm > B2_EVENTS_NTERM || a->nstate < 0 || a->nstate > B2_EVENTS_NSTATE || a->nterm + a->nstate < 1 ||
      a->ninterval < 0 || a->nelem < 0 || !(a->step_dt > 0.0f))
    return fail("b2_events: needs terminated, truncated, V (v_width >= 1), the entry table, "
                "0 <= nterm <= B2_EVENTS_NTERM, 0 <= nstate <= B2_EVENTS_NSTATE, a term and step_dt > 0");
  long long first = 0;
  int ninterval = 0;
  for (int t = 0; t < a->nterm; t++) {
    const B2EventTerm& T = a->term[t];
    if ((T.mode != B2_EVENT_RESET && T.mode != B2_EVENT_INTERVAL) ||
        (T.operation != B2_EVENT_ADD && T.operation != B2_EVENT_SCALE && T.operation != B2_EVENT_ABS) ||
        (T.distribution != B2_EVENT_UNIFORM && T.distribution != B2_EVENT_LOG_UNIFORM))
      return fail("b2_events: term " + std::to_string(t) + " has an unknown mode, operation or distribution code");
    if (T.field < 0 || T.field >= (int)s->model_fields.size() || !s->model_fields[T.field].farr)
      return fail("b2_events: term " + std::to_string(t) + "'s field is not a float model field");
    const Field& f = s->model_fields[T.field];
    if (f.farr->stride == 0 && s->nworld > 1)
      return fail("b2_events: field '" + f.name + "' is shared by every world; b2_expand_model_field it first");
    const bool interval = T.mode == B2_EVENT_INTERVAL;
    if (T.count < 1 || T.col < 0 || (long long)T.col + T.count + (interval ? 1 : 0) > a->v_width ||
        first + T.count > a->nelem)
      return fail("b2_events: term " + std::to_string(t) + " reads V columns outside the block or entries outside "
                  "the table");
    if (interval && !(T.interval_lo >= 0.0f && T.interval_span >= 0.0f && T.interval_lo + T.interval_span < INFINITY))
      return fail("b2_events: term " + std::to_string(t) + " needs a finite interval with 0 <= lo and span >= 0");
    F->row[t] = const_cast<float*>(f.farr->p);
    F->stride[t] = f.farr->stride;
    first += T.count;
    ninterval += interval;
  }
  if (first != a->nelem) return fail("b2_events: the terms' counts do not add up to nelem");
  long long nbodies = 0;
  int last_timer = ninterval - 1;  // the state terms' rows follow the field terms', in table order
  for (int t = 0; t < a->nstate; t++) {
    const B2EventStateTerm& S = a->state[t];
    const std::string which = "b2_events: state term " + std::to_string(t);
    if ((S.kind != B2_EVENT_PUSH && S.kind != B2_EVENT_WRENCH) ||
        (S.mode != B2_EVENT_RESET && S.mode != B2_EVENT_INTERVAL) || (S.kind == B2_EVENT_PUSH && S.mode != B2_EVENT_INTERVAL))
      return fail(which + " has an unknown kind or mode code (a push is an interval term)");
    const bool interval = S.mode == B2_EVENT_INTERVAL;
    const long long draws = S.kind == B2_EVENT_PUSH ? 6 : 6LL * S.count;
    if ((S.kind == B2_EVENT_PUSH ? S.count != 6 : S.count < 1) || S.col < 0 ||
        (long long)S.col + draws + (interval ? 1 : 0) > a->v_width)
      return fail(which + " reads V columns outside the block or has a bad count");
    if (S.kind == B2_EVENT_WRENCH) {
      if (S.first != nbodies) return fail(which + "'s bodies do not follow the previous term's in the body table");
      nbodies += S.count;
    }
    if (interval) {
      if (S.timer <= last_timer || S.timer >= a->ninterval || !a->timers)
        return fail(which + " needs a timer row of its own, after the previous interval term's and below ninterval");
      last_timer = S.timer;
      if (!(S.interval_lo >= 0.0f && S.interval_span >= 0.0f && S.interval_lo + S.interval_span < INFINITY))
        return fail(which + " needs a finite interval with 0 <= lo and span >= 0");
      ninterval++;
    }
    if (S.kind == B2_EVENT_PUSH && (!a->refreshed || a->root_body < 1 || a->root_body >= s->hm.nbody))
      return fail(which + ": a push needs the refreshed mask and a root_body of the model");
  }
  if (nbodies != a->nbodies || (nbodies > 0 && !a->bodies))
    return fail("b2_events: the wrench terms' counts do not add up to nbodies");
  if ((a->clear_xfrc || nbodies > 0) && (!s->hd.xfrc_applied.p || s->hd.xfrc_applied.stride < 6 * s->hm.nbody))
    return fail("b2_events: the wrench terms need a per-world xfrc_applied");
  if (ninterval > a->ninterval || (ninterval > 0 && !a->timers))
    return fail("b2_events: the interval terms need their timers ([ninterval][n])");
  const DevData& d = s->hd;
  F->qpos = d.qpos.p; F->qvel = d.qvel.p; F->xfrc = d.xfrc_applied.p; F->xpos = d.xpos.p; F->xquat = d.xquat.p;
  F->subtree_com = d.subtree_com.p; F->cvel = d.cvel.p;
  F->qpos_s = d.qpos.stride; F->qvel_s = d.qvel.stride; F->xfrc_s = d.xfrc_applied.stride; F->xpos_s = d.xpos.stride;
  F->xquat_s = d.xquat.stride; F->subtree_com_s = d.subtree_com.stride; F->cvel_s = d.cvel.stride;
  // The entry table is device memory: it is read back and checked the first time this sim sees it with these fields
  // and counts (a synchronising copy, so outside a stream capture), and taken as unchanged after that, so that the
  // calls an env step captures read nothing back.
  std::vector<long long> key = {(long long)(uintptr_t)a->elem, a->nelem, (long long)(uintptr_t)a->bodies, a->nbodies};
  for (int t = 0; t < a->nterm; t++) key.insert(key.end(), {a->term[t].field, a->term[t].count});
  if (key == s->events_checked) return 0;
  std::vector<B2EventElem> elem(a->nelem);
  if (a->nelem)
    CUDA_OK(cudaMemcpy(elem.data(), a->elem, sizeof(B2EventElem) * elem.size(), cudaMemcpyDeviceToHost));
  std::vector<int32_t> bodies(a->nbodies);
  if (a->nbodies)
    CUDA_OK(cudaMemcpy(bodies.data(), a->bodies, sizeof(int32_t) * bodies.size(), cudaMemcpyDeviceToHost));
  for (int32_t b : bodies)
    if (b < 1 || b >= s->hm.nbody)
      return fail("b2_events: a wrench term names body " + std::to_string(b) + ", outside the model's bodies 1.." +
                  std::to_string(s->hm.nbody - 1));
  first = 0;
  for (int t = 0; t < a->nterm; t++) {
    const Field& f = s->model_fields[a->term[t].field];
    for (int j = 0; j < a->term[t].count; j++) {
      const B2EventElem& E = elem[first + j];
      if (E.offset < 0 || E.offset >= f.farr->n)
        return fail("b2_events: term " + std::to_string(t) + " writes element " + std::to_string(E.offset) +
                    ", outside the row of '" + f.name + "' (" + std::to_string(f.farr->n) + " floats)");
    }
    first += a->term[t].count;
  }
  s->events_checked = key;
  return 0;
}
int b2_events(b2_sim* s, const B2EventArgs* args, void* stream) {
  B2EventFields F = {};
  DeviceGuard guard(s ? s->device : 0);
  if (events_check(s, args, &F)) return 1;
  const long long threads = 32LL * s->nworld;
  b2_events_kernel<<<(unsigned)((threads + 127) / 128), 128, 0, (cudaStream_t)stream>>>(s->nworld, *args, F);
  s->launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int b2_step_host(b2_sim* s, const float* ctrl_host, int nsteps, float* qpos_host, float* qvel_host,
                 void* stream) {
  if (!s) return fail("b2_step_host: null sim");
  DeviceGuard guard(s->device);
  cudaStream_t st = (cudaStream_t)stream;
  const DevModel& m = s->hm; const DevData& d = s->hd;
  if (ctrl_host && m.nu > 0)
    CUDA_OK(cudaMemcpy2DAsync(d.ctrl.p, sizeof(float) * d.ctrl.stride, ctrl_host, sizeof(float) * m.nu,
                              sizeof(float) * m.nu, s->nworld, cudaMemcpyHostToDevice, st));
  if (nsteps > 0 && b2_step_n(s, nsteps, stream)) return 1;
  if (qpos_host)
    CUDA_OK(cudaMemcpy2DAsync(qpos_host, sizeof(float) * m.nq, d.qpos.p, sizeof(float) * d.qpos.stride,
                              sizeof(float) * m.nq, s->nworld, cudaMemcpyDeviceToHost, st));
  if (qvel_host)
    CUDA_OK(cudaMemcpy2DAsync(qvel_host, sizeof(float) * m.nv, d.qvel.p, sizeof(float) * d.qvel.stride,
                              sizeof(float) * m.nv, s->nworld, cudaMemcpyDeviceToHost, st));
  return 0;
}

// The drawable geoms (b2_render.cuh: B2RenderPlan), from the model's tables on the device.
static int render_plan(b2_sim* s) {
  const DevModel& m = s->hm;
  auto fetch = [](const int* p, int n) {
    std::vector<int> v((size_t)std::max(n, 0));
    if (n > 0 && cudaMemcpy(v.data(), p, sizeof(int) * n, cudaMemcpyDeviceToHost) != cudaSuccess) v.clear();
    return v;
  };
  const std::vector<int> type = fetch(m.geom_type, m.ngeom), body = fetch(m.geom_bodyid, m.ngeom);
  const std::vector<int> parent = fetch(m.body_parentid, m.nbody), dofnum = fetch(m.body_dofnum, m.nbody);
  const std::vector<int> sgeom = fetch(m.static_geom, m.nstatic), fgeom = fetch(m.fixed_geom, m.nfixed);
  if ((int)type.size() != m.ngeom || (int)body.size() != m.ngeom || (int)parent.size() != m.nbody ||
      (int)dofnum.size() != m.nbody || (int)sgeom.size() != m.nstatic || (int)fgeom.size() != m.nfixed)
    return fail("b2_render: reading the model's tables failed");
  std::vector<char> welded(m.nbody, 1);  // bodies are numbered parents first
  for (int b = 1; b < m.nbody; b++) welded[b] = dofnum[b] == 0 && welded[parent[b]];
  std::vector<int> pose(m.ngeom, -1), stat, dyn;
  for (int k = 0; k < m.nstatic; k++) pose[sgeom[k]] = k;
  for (int f = 0; f < m.nfixed; f++) pose[fgeom[f]] = -2 - f;
  for (int g = 0; g < m.ngeom; g++) {
    if (type[g] == G_MESH) continue;
    if (welded[body[g]]) { stat.push_back(g); stat.push_back(pose[g]); }
    else dyn.push_back(g);
  }
  B2RenderPlan& P = s->render_plan;
  P.nstat = (int)stat.size() / 2;
  P.ndyn = (int)dyn.size();
  if (dev_upload<int>(s, stat, &P.stat) || dev_upload<int>(s, dyn, &P.dyn)) return 1;
  s->render_planned = true;
  return 0;
}

int b2_render(b2_sim* s, const B2RenderArgs* a, void* stream) {
  if (!s || !a) return fail("b2_render: bad arguments");
  if (a->width < 1 || a->width > 4096 || a->height < 1 || a->height > 4096)
    return fail("b2_render: width and height must lie in 1..4096");
  if (a->env_idx < 0 || a->env_idx >= s->nworld) return fail("b2_render: env_idx outside [0, nworld)");
  if (a->noverlay < 0) return fail("b2_render: noverlay must be >= 0");
  if (a->track_body < -1 || a->track_body >= s->hm.nbody) return fail("b2_render: track_body outside [-1, nbody)");
  if (!a->rgb) return fail("b2_render: rgb is null");
  if (a->ndecor < 0 || a->ndecor > B2R_MAXDECOR)
    return fail("b2_render: ndecor " + std::to_string(a->ndecor) + " outside [0, " + std::to_string(B2R_MAXDECOR) + "]");
  if (a->ndecor > 0 && !a->decor) return fail("b2_render: decor is null with ndecor > 0");
  if (!a->ghost_xpos != !a->ghost_xmat) return fail("b2_render: ghost_xpos and ghost_xmat must both be set or both null");
  if (a->ghost_xpos)
    for (int k = 0; k < 4; k++)
      if (!(a->ghost_rgba[k] >= 0.f && a->ghost_rgba[k] <= 1.f))
        return fail("b2_render: ghost_rgba must lie in [0, 1]");
  DeviceGuard guard(s->device);
  if (!s->render_planned && render_plan(s)) return 1;
  const B2RenderPlan& P = s->render_plan;
  B2RenderFrame F = {};
  F.width = a->width; F.height = a->height;
  F.ntx = (a->width + B2R_TILE - 1) / B2R_TILE;
  const int nty = (a->height + B2R_TILE - 1) / B2R_TILE;
  F.env_idx = a->env_idx;
  F.noverlay = std::min(a->noverlay, s->nworld);
  const int nworlds = F.noverlay + (a->env_idx >= F.noverlay ? 1 : 0);
  F.nitem = P.nstat + nworlds * P.ndyn;
  F.track_body = a->track_body;
  F.shadows = a->shadows != 0; F.brute = a->brute != 0;
  for (int k = 0; k < 3; k++) F.lookat[k] = a->lookat[k];
  F.distance = a->distance;
  const double deg = 3.14159265358979323846 / 180.0, az = a->azimuth * deg, el = a->elevation * deg;
  const double f[3] = {std::cos(el) * std::cos(az), std::cos(el) * std::sin(az), std::sin(el)};
  const double r[3] = {std::sin(az), -std::cos(az), 0.0};  // f x z, normalised
  const double u[3] = {r[1] * f[2] - r[2] * f[1], r[2] * f[0] - r[0] * f[2], r[0] * f[1] - r[1] * f[0]};
  for (int k = 0; k < 3; k++) { F.fwd[k] = (float)f[k]; F.right[k] = (float)r[k]; F.up[k] = (float)u[k]; }
  F.tan_y = (float)std::tan(22.5 * deg);
  F.tan_x = (float)(std::tan(22.5 * deg) * a->width / a->height);
  F.rgb = a->rgb; F.depth = a->depth; F.seg = a->seg;
  F.nghost = a->ghost_xpos ? P.ndyn : 0;
  F.ndeco = F.nghost + a->ndecor;
  F.decor = a->decor; F.ghost_xpos = a->ghost_xpos; F.ghost_xmat = a->ghost_xmat;
  for (int k = 0; k < 4; k++) F.ghost_rgba[k] = a->ghost_rgba[k];
  // the scene, then (with decoration) the decoration over it: b2_render.cuh, b2_render_kernel
  b2_render_kernel<false><<<F.ntx * nty, B2R_TILE * B2R_TILE, 0, (cudaStream_t)stream>>>(s->hm, s->hd, P, F);
  s->launches++;
  if (F.ndeco > 0) {
    b2_render_kernel<true><<<F.ntx * nty, B2R_TILE * B2R_TILE, 0, (cudaStream_t)stream>>>(s->hm, s->hd, P, F);
    s->launches++;
  }
  CUDA_OK(cudaGetLastError());
  return 0;
}

int b2_stats(b2_sim* s, void* stream, B2Stats* out) {
  if (!s || !out) return fail("b2_stats: bad arguments");
  DeviceGuard guard(s->device);
  cudaStream_t st = (cudaStream_t)stream;
  const DevData& d = s->hd;
  size_t n = (size_t)s->nworld;
  std::vector<int> ncon(n * d.ncon.stride), nefc(n * d.nefc.stride), nit(n * d.solver_niter.stride), ovf(n * d.overflow.stride);
  CUDA_OK(cudaStreamSynchronize(st));
  CUDA_OK(cudaMemcpy(ncon.data(), d.ncon.p, sizeof(int) * ncon.size(), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(nefc.data(), d.nefc.p, sizeof(int) * nefc.size(), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(nit.data(), d.solver_niter.p, sizeof(int) * nit.size(), cudaMemcpyDeviceToHost));
  CUDA_OK(cudaMemcpy(ovf.data(), d.overflow.p, sizeof(int) * ovf.size(), cudaMemcpyDeviceToHost));
  memset(out, 0, sizeof(*out));
  out->ncon_cap = s->hm.maxcon; out->nefc_cap = s->hm.njmax;
  double sc = 0, se = 0, si = 0;
  for (size_t w = 0; w < n; w++) {
    int c = ncon[w * d.ncon.stride], e = nefc[w * d.nefc.stride], it = nit[w * d.solver_niter.stride];
    out->ncon_max = std::max(out->ncon_max, c); out->nefc_max = std::max(out->nefc_max, e);
    out->niter_max = std::max(out->niter_max, it);
    out->overflow_worlds += ovf[w * d.overflow.stride] ? 1 : 0;
    sc += c; se += e; si += it;
  }
  out->ncon_mean = sc / n; out->nefc_mean = se / n; out->niter_mean = si / n;
  return 0;
}

int64_t b2_launch_count(b2_sim* s) { return s ? s->launches : 0; }

int b2_algorithmic_bytes(b2_sim* s, void* stream, double* solver_bytes, double* step_bytes) {
  B2Stats st;
  if (b2_stats(s, stream, &st)) return 1;
  const DevModel& m = s->hm;
  double nv = m.nv, nefc = st.nefc_mean;
  // BASELINE.md §4 / SURVEY.md §8d: solver stage with J resident in HBM (the reference formulation)
  double solver = 4.0 * (nefc * nv + 3.0 * nefc + nv * nv + 5.0 * nv);
  // whole step: state in/out + consumer-visible kinematics (what this kernel actually moves)
  double in = m.nq + m.nv + m.nu + m.nv + m.nv + 6.0 * m.nbody;
  double outb = m.nq + 3.0 * m.nv + m.nu + m.nsensordata + (3 + 4 + 9 + 3 + 3 + 6) * (double)m.nbody +
                12.0 * m.nposegeom + 12.0 * m.nsite;  // geoms welded to the world are posed once at create, not per step
  if (solver_bytes) *solver_bytes = solver * s->nworld;
  if (step_bytes) *step_bytes = 4.0 * (in + outb) * s->nworld;
  return 0;
}

}  // extern "C"

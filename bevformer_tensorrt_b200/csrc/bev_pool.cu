// bev_pool.cu — BEVPoolV2 (plugins BEVPoolV2TRT / BEVPoolV2TRT2) on sm_90a: forward in FP32 / FP16 / BF16 / INT8 and
// the depth / feature gradients in FP32 / FP16 / BF16, and FP32 depth with FP16 / BF16 features (what torch.autocast
// hands the op: a softmax depth and conv features), forward and both gradients.
//
// For every interval k (s = interval_starts[k], len = interval_lengths[k], cell = ranks_bev[s]):
//   out[cell, c] = sum_{i = s}^{s + len - 1} feat[ranks_feat[i], c] * depth[ranks_depth[i]]
// (reference: TensorRT/plugin/bev_pool_v2/bevPoolKernel.cu; backward third_party/bev_mmdet3d/ops/bev_pool_v2/src/
// bev_pool_cuda.cu). Input contract, as voxel_pooling_prepare_v2 builds the ranks: points sorted by ranks_bev, one
// interval per distinct cell, each depth cell referenced by at most one point.
//
// Index safety (beyond the reference, which checks no index): [s, s + len) is clipped to [0, P); an interval whose
// cell is outside [0, out_h * out_w) is dropped; a point whose ranks_depth or ranks_feat is outside its tensor is
// dropped. No input forms an address outside a tensor.
//
// Kernel shape: a lane group of G = pow2(ceil(C / VEC)) <= 32 lanes owns one interval and one tile of G * VEC channels;
// a lane owns VEC consecutive channels (a 16-byte vector where C and the pointers allow). The group loads G point indices
// at a time, coalesced and evict-first, and hands them out by shuffle; four feat rows are in flight per lane. Each lane
// keeps one accumulator per channel and adds the points in their order: FP32 is the reference kernel's FFMA chain bit
// for bit, FP16 accumulates in FP32 and rounds once, INT8 sums exactly in int32 and requantises as the reference does.
// BF16 is FP16's arithmetic on bf16 storage (each element widened exactly, `u << 16`). FP32 depth (depth element type TD
// = float, features T = FP16 / BF16) changes three things only: the per-point depth load of the forward and of the
// feature gradient, and the depth-gradient store, which is not rounded. Those instantiations have __global__ wrappers
// of their own (bev_pool*_f32_depth_kernel) around the same __device__ body, so the same-dtype kernels keep their
// names and templates <T, VEC>.
#include <type_traits>

#include "common.cuh"

namespace b200 {

namespace {

constexpr int kBevThreads = 256;
// feat_dtype of the FP32-depth entries: nvinfer1::DataType's codes, as the MSDA / DCN workspace queries take them
constexpr int kFeatF16 = 1, kFeatBF16 = 7;

struct BevPoolArgs {
  const int32_t *ranks_depth, *ranks_feat, *ranks_bev, *starts, *lengths;
  long long depth_size, feat_rows, cells;
  int C, P, I;
};

template <typename T, int VEC>
struct alignas(sizeof(T) * VEC) Pack {
  T v[VEC];
};

template <typename T>
using AccT = typename std::conditional<std::is_same<T, int8_t>::value, int, float>::type;

template <typename T>
__device__ __forceinline__ AccT<T> widen(T x) {
  if constexpr (std::is_same<T, __half>::value) return __half2float(x);
  else if constexpr (std::is_same<T, __nv_bfloat16>::value) return bf16_to_f(x);
  else return static_cast<AccT<T>>(x);
}

template <typename T>
__device__ __forceinline__ T narrow(float x) {
  if constexpr (std::is_same<T, __half>::value) return __float2half_rn(x);
  else if constexpr (std::is_same<T, __nv_bfloat16>::value) return __float2bfloat16_rn(x);
  else return x;
}

// acc + f * d: one FFMA for FP32, FP16 and BF16 (the product of two 2-byte values is exact in FP32), an exact int32 MAD
// for INT8
template <typename T>
__device__ __forceinline__ AccT<T> mad(T f, AccT<T> d, AccT<T> acc) {
  if constexpr (std::is_same<T, int8_t>::value) return acc + static_cast<int>(f) * d;
  else return __fmaf_rn(widen(f), d, acc);
}

// The interval's point range clipped to [0, P) and its cell; false when the interval is dropped.
__device__ __forceinline__ bool interval_of(const BevPoolArgs &a, int k, int &s, int &e, int &cell) {
  const long long s0 = __ldcs(a.starts + k), len = __ldcs(a.lengths + k);
  const long long lo = s0 > 0 ? s0 : 0, hi = s0 + len < a.P ? s0 + len : a.P;
  if (lo >= hi) return false;
  cell = __ldg(a.ranks_bev + lo);
  if (cell < 0 || cell >= a.cells) return false;
  s = static_cast<int>(lo), e = static_cast<int>(hi);
  return true;
}

// The thread's lane group in the whole grid, in 64 bits: items * G passes 2^32 long before items passes INT_MAX.
__device__ __forceinline__ long long group_index(int G) {
  return (static_cast<long long>(blockIdx.x) * kBevThreads + threadIdx.x) / G;
}

__device__ __forceinline__ unsigned group_mask(int G) {
  return G == 32 ? kFullMask : ((1u << G) - 1) << ((threadIdx.x & 31) & ~(G - 1));
}

template <typename T, typename TD, int VEC>
__device__ __forceinline__ void bev_pool_body(const BevPoolArgs a, const TD *__restrict__ depth,
                                              const T *__restrict__ feat, T *__restrict__ out, float scale_io, int G) {
  using Acc = AccT<T>;
  using P = Pack<T, VEC>;
  const int gl = threadIdx.x & (G - 1);
  const long long k = group_index(G);
  int s, e, cell;
  if (k >= a.I || !interval_of(a, static_cast<int>(k), s, e, cell)) return;  // uniform within the group
  const unsigned mask = group_mask(G);
  const int c0 = (blockIdx.y * G + gl) * VEC;
  const bool active = c0 < a.C;
  Acc acc[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) acc[v] = 0;
  for (int base = s; base < e; base += G) {
    const int i = base + gl;
    int rf = -1;
    Acc dv = 0;
    if (i < e) {
      const int rd = __ldcs(a.ranks_depth + i), r = __ldcs(a.ranks_feat + i);
      if (rd >= 0 && rd < a.depth_size && r >= 0 && r < a.feat_rows) rf = r, dv = widen(__ldg(depth + rd));
    }
    const int n = min(G, e - base);
    for (int j = 0; j < n; j += 4) {
      int rfs[4];
      Acc dvs[4];
      P rows[4] = {};
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        rfs[u] = __shfl_sync(mask, rf, j + u, G);
        dvs[u] = __shfl_sync(mask, dv, j + u, G);
        if (j + u >= n) rfs[u] = -1;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (active && rfs[u] >= 0) rows[u] = *reinterpret_cast<const P *>(feat + static_cast<size_t>(rfs[u]) * a.C + c0);
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (active && rfs[u] >= 0) {
#pragma unroll
          for (int v = 0; v < VEC; ++v) acc[v] = mad(rows[u].v[v], dvs[u], acc[v]);
        }
    }
  }
  if (!active) return;
  P o;
#pragma unroll
  for (int v = 0; v < VEC; ++v) {
    if constexpr (std::is_same<T, int8_t>::value)
      o.v[v] = static_cast<int8_t>(to_int8_sat(__fmul_rn(__int2float_rn(acc[v]), scale_io)));
    else
      o.v[v] = narrow<T>(acc[v]);
  }
  *reinterpret_cast<P *>(out + static_cast<size_t>(cell) * a.C + c0) = o;
}

template <typename T, int VEC>
__global__ void __launch_bounds__(kBevThreads) bev_pool_kernel(const BevPoolArgs a, const T *__restrict__ depth,
                                                               const T *__restrict__ feat, T *__restrict__ out,
                                                               float scale_io, int G) {
  bev_pool_body<T, T, VEC>(a, depth, feat, out, scale_io, G);
}

template <typename T, int VEC>
__global__ void __launch_bounds__(kBevThreads) bev_pool_f32_depth_kernel(const BevPoolArgs a,
                                                                         const float *__restrict__ depth,
                                                                         const T *__restrict__ feat,
                                                                         T *__restrict__ out, int G) {
  bev_pool_body<T, float, VEC>(a, depth, feat, out, 0.f, G);
}

// Backward, step 1 (one group per interval): depth_grad[rd] = sum_c out_grad[cell, c] * feat[rf, c] for every kept point
// (a fixed-order lane-partial FFMA chain and butterfly sum), and point_cell[i] = the cell point i pooled into, -1 when it
// pooled into none. With depth_grad == NULL only point_cell is written.
template <typename T, typename TD, int VEC>
__device__ __forceinline__ void bev_pool_depth_grad_body(const BevPoolArgs a, const T *__restrict__ out_grad,
                                                         const T *__restrict__ feat, TD *__restrict__ depth_grad,
                                                         int *__restrict__ point_cell, int G) {
  using P = Pack<T, VEC>;
  const int gl = threadIdx.x & (G - 1);
  const long long k = group_index(G);
  int s, e, cell;
  if (k >= a.I || !interval_of(a, static_cast<int>(k), s, e, cell)) return;
  const unsigned mask = group_mask(G);
  const T *og = out_grad + static_cast<size_t>(cell) * a.C;
  for (int base = s; base < e; base += G) {
    const int i = base + gl;
    int rf = -1, rd = -1;
    if (i < e) {
      const int d = __ldcs(a.ranks_depth + i), r = __ldcs(a.ranks_feat + i);
      const bool kept = d >= 0 && d < a.depth_size && r >= 0 && r < a.feat_rows;
      if (kept) rf = r, rd = d;
      point_cell[i] = kept ? cell : -1;
    }
    if (!depth_grad) continue;
    const int n = min(G, e - base);
    for (int j = 0; j < n; ++j) {
      const int rfj = __shfl_sync(mask, rf, j, G), rdj = __shfl_sync(mask, rd, j, G);
      if (rfj < 0) continue;  // uniform within the group
      const T *f = feat + static_cast<size_t>(rfj) * a.C;
      float part = 0.f;
      for (int c0 = gl * VEC; c0 < a.C; c0 += G * VEC) {
        const P g = *reinterpret_cast<const P *>(og + c0), x = *reinterpret_cast<const P *>(f + c0);
#pragma unroll
        for (int v = 0; v < VEC; ++v) part = __fmaf_rn(widen(g.v[v]), widen(x.v[v]), part);
      }
      for (int o = G / 2; o > 0; o >>= 1) part = __fadd_rn(part, __shfl_xor_sync(mask, part, o, G));
      if (gl == 0) depth_grad[rdj] = narrow<TD>(part);
    }
  }
}

template <typename T, int VEC>
__global__ void __launch_bounds__(kBevThreads) bev_pool_depth_grad_kernel(const BevPoolArgs a, const T *__restrict__ out_grad,
                                                                          const T *__restrict__ feat,
                                                                          T *__restrict__ depth_grad,
                                                                          int *__restrict__ point_cell, int G) {
  bev_pool_depth_grad_body<T, T, VEC>(a, out_grad, feat, depth_grad, point_cell, G);
}

template <typename T, int VEC>
__global__ void __launch_bounds__(kBevThreads) bev_pool_depth_grad_f32_depth_kernel(const BevPoolArgs a,
                                                                                    const T *__restrict__ out_grad,
                                                                                    const T *__restrict__ feat,
                                                                                    float *__restrict__ depth_grad,
                                                                                    int *__restrict__ point_cell, int G) {
  bev_pool_depth_grad_body<T, float, VEC>(a, out_grad, feat, depth_grad, point_cell, G);
}

// Backward, step 2 (one group per run of equal ranks_feat in `order`, the points sorted by ranks_feat):
// feat_grad[rf, c] = sum over the run's pooled points of out_grad[cell, c] * depth[rd], in run order.
template <typename T, typename TD, int VEC>
__device__ __forceinline__ void bev_pool_feat_grad_body(const BevPoolArgs a, const int32_t *__restrict__ order,
                                                        const T *__restrict__ out_grad, const TD *__restrict__ depth,
                                                        const int *__restrict__ point_cell, T *__restrict__ feat_grad,
                                                        int G) {
  using P = Pack<T, VEC>;
  const int gl = threadIdx.x & (G - 1);
  const long long jl = group_index(G);
  if (jl >= a.P) return;
  const int j = static_cast<int>(jl);
  const int head = __ldg(order + j);
  if (head < 0 || head >= a.P) return;
  const int rf = __ldg(a.ranks_feat + head);
  if (rf < 0 || rf >= a.feat_rows) return;
  if (j > 0) {
    const int prev = __ldg(order + j - 1);
    if (prev >= 0 && prev < a.P && __ldg(a.ranks_feat + prev) == rf) return;  // not the first point of its run
  }
  const int c0 = (blockIdx.y * G + gl) * VEC;
  if (c0 >= a.C) return;
  float acc[VEC];
#pragma unroll
  for (int v = 0; v < VEC; ++v) acc[v] = 0.f;
  for (int jj = j; jj < a.P; ++jj) {
    const int i = __ldg(order + jj);
    if (i < 0 || i >= a.P || __ldg(a.ranks_feat + i) != rf) break;
    const int cell = point_cell[i];
    if (cell < 0) continue;
    const float dv = widen(__ldg(depth + __ldg(a.ranks_depth + i)));
    const P g = *reinterpret_cast<const P *>(out_grad + static_cast<size_t>(cell) * a.C + c0);
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = __fmaf_rn(widen(g.v[v]), dv, acc[v]);
  }
  P o;
#pragma unroll
  for (int v = 0; v < VEC; ++v) o.v[v] = narrow<T>(acc[v]);
  *reinterpret_cast<P *>(feat_grad + static_cast<size_t>(rf) * a.C + c0) = o;
}

template <typename T, int VEC>
__global__ void __launch_bounds__(kBevThreads) bev_pool_feat_grad_kernel(const BevPoolArgs a, const int32_t *__restrict__ order,
                                                                         const T *__restrict__ out_grad,
                                                                         const T *__restrict__ depth,
                                                                         const int *__restrict__ point_cell,
                                                                         T *__restrict__ feat_grad, int G) {
  bev_pool_feat_grad_body<T, T, VEC>(a, order, out_grad, depth, point_cell, feat_grad, G);
}

template <typename T, int VEC>
__global__ void __launch_bounds__(kBevThreads) bev_pool_feat_grad_f32_depth_kernel(const BevPoolArgs a,
                                                                                   const int32_t *__restrict__ order,
                                                                                   const T *__restrict__ out_grad,
                                                                                   const float *__restrict__ depth,
                                                                                   const int *__restrict__ point_cell,
                                                                                   T *__restrict__ feat_grad, int G) {
  bev_pool_feat_grad_body<T, float, VEC>(a, order, out_grad, depth, point_cell, feat_grad, G);
}

// Widest vector (elements) that divides C and keeps every row of every listed tensor aligned.
template <typename T>
int pick_vec(int C, std::initializer_list<const void *> ptrs) {
  for (int v = 16 / static_cast<int>(sizeof(T)); v > 1; v /= 2) {
    bool ok = C % v == 0;
    for (const void *p : ptrs) ok = ok && reinterpret_cast<uintptr_t>(p) % (v * sizeof(T)) == 0;
    if (ok) return v;
  }
  return 1;
}

int group_size(int C, int vec) {
  const int lanes = (C + vec - 1) / vec;
  int G = 1;
  while (G < lanes && G < 32) G *= 2;
  return G;
}

dim3 grid_of(long long items, int C, int vec, int G, bool tiled) {
  const long long per_block = kBevThreads / G;
  const unsigned tiles = tiled ? static_cast<unsigned>((C + G * vec - 1) / (G * vec)) : 1u;
  return dim3(static_cast<unsigned>((items + per_block - 1) / per_block), tiles);
}

bool aligned(const void *p, size_t bytes) { return reinterpret_cast<uintptr_t>(p) % bytes == 0; }

// depth_elem: the byte size of a depth element (and of the depth gradient's); elem: that of a feat / out element (and
// of out_grad's and the feature gradient's). Every pointer must be aligned to its element.
int check_args(const void *depth, const void *feat, const void *out, const int32_t *rd, const int32_t *rf,
               const int32_t *rb, const int32_t *st, const int32_t *ln, int C, int P, int I, long long depth_size,
               long long feat_rows, int out_h, int out_w, size_t depth_elem, size_t elem) {
  if (C <= 0 || P < 0 || I < 0 || depth_size < 0 || feat_rows < 0 || out_h <= 0 || out_w <= 0) return B200_ERR_BAD_PARAM;
  if (!out || (P > 0 && (!rd || !rf || !rb)) || (I > 0 && (!st || !ln))) return B200_ERR_BAD_PARAM;
  if ((depth_size > 0 && !depth) || (feat_rows > 0 && !feat)) return B200_ERR_BAD_PARAM;
  if (feat_rows > (1ll << 62) / C) return B200_ERR_BAD_PARAM;
  if (!aligned(depth, depth_elem)) return B200_ERR_BAD_PARAM;
  for (const void *p : {feat, out})
    if (!aligned(p, elem)) return B200_ERR_BAD_PARAM;
  for (const int32_t *p : {rd, rf, rb, st, ln})
    if (!aligned(p, sizeof(int32_t))) return B200_ERR_BAD_PARAM;
  return B200_OK;
}

template <typename T, typename TD, int VEC>
void launch_fwd(const BevPoolArgs &a, const TD *depth, const T *feat, T *out, float scale_io, cudaStream_t s) {
  const int G = group_size(a.C, VEC);
  const dim3 grid = grid_of(a.I, a.C, VEC, G, true);
  if constexpr (std::is_same<T, TD>::value)
    bev_pool_kernel<T, VEC><<<grid, kBevThreads, 0, s>>>(a, depth, feat, out, scale_io, G);
  else
    bev_pool_f32_depth_kernel<T, VEC><<<grid, kBevThreads, 0, s>>>(a, depth, feat, out, G);
}

template <typename T, typename TD = T>
int bev_pool_forward(const BevPoolArgs &a, const TD *depth, const T *feat, T *out, float scale_io, void *stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (cudaMemsetAsync(out, 0, static_cast<size_t>(a.cells) * a.C * sizeof(T), s) != cudaSuccess) return B200_ERR_LAUNCH;
  if (a.I == 0) return B200_OK;
  switch (pick_vec<T>(a.C, {feat, out})) {
    case 16: if constexpr (sizeof(T) == 1) launch_fwd<T, TD, 16>(a, depth, feat, out, scale_io, s); break;
    case 8: if constexpr (sizeof(T) <= 2) launch_fwd<T, TD, 8>(a, depth, feat, out, scale_io, s); break;
    case 4: launch_fwd<T, TD, 4>(a, depth, feat, out, scale_io, s); break;
    case 2: launch_fwd<T, TD, 2>(a, depth, feat, out, scale_io, s); break;
    default: launch_fwd<T, TD, 1>(a, depth, feat, out, scale_io, s); break;
  }
  return check_launch();
}

template <typename T, typename TD, int VEC>
void launch_depth_grad(const BevPoolArgs &a, const T *out_grad, const T *feat, TD *depth_grad, int *point_cell,
                       cudaStream_t s) {
  const int G = group_size(a.C, VEC);
  const dim3 grid = grid_of(a.I, a.C, VEC, G, false);
  if constexpr (std::is_same<T, TD>::value)
    bev_pool_depth_grad_kernel<T, VEC><<<grid, kBevThreads, 0, s>>>(a, out_grad, feat, depth_grad, point_cell, G);
  else
    bev_pool_depth_grad_f32_depth_kernel<T, VEC><<<grid, kBevThreads, 0, s>>>(a, out_grad, feat, depth_grad,
                                                                              point_cell, G);
}

template <typename T, typename TD, int VEC>
void launch_feat_grad(const BevPoolArgs &a, const int32_t *order, const T *out_grad, const TD *depth,
                      const int *point_cell, T *feat_grad, cudaStream_t s) {
  const int G = group_size(a.C, VEC);
  const dim3 grid = grid_of(a.P, a.C, VEC, G, true);
  if constexpr (std::is_same<T, TD>::value)
    bev_pool_feat_grad_kernel<T, VEC><<<grid, kBevThreads, 0, s>>>(a, order, out_grad, depth, point_cell, feat_grad, G);
  else
    bev_pool_feat_grad_f32_depth_kernel<T, VEC><<<grid, kBevThreads, 0, s>>>(a, order, out_grad, depth, point_cell,
                                                                             feat_grad, G);
}

// Each kernel takes its vector width from the tensors it reads and writes alone, so the depth gradient's lane partition,
// and with it its bits, does not depend on whether or where a feature gradient is asked for. The depth tensors (TD)
// are read or written one element per point and never set the width.
template <typename T, typename TD = T>
int bev_pool_backward(const BevPoolArgs &a, const int32_t *order, const T *out_grad, const TD *depth, const T *feat,
                      TD *depth_grad, T *feat_grad, void *workspace, size_t workspace_size, void *stream) {
  if (!out_grad || (!depth_grad && !feat_grad)) return B200_ERR_BAD_PARAM;
  if (feat_grad && a.P > 0 && !order) return B200_ERR_BAD_PARAM;
  if (!aligned(depth_grad, sizeof(TD)) || !aligned(feat_grad, sizeof(T)) || !aligned(order, sizeof(int32_t)) ||
      !aligned(workspace, sizeof(int)))
    return B200_ERR_BAD_PARAM;
  const size_t ws = b200_bev_pool_backward_workspace_size(a.P);
  if (ws && (!workspace || workspace_size < ws)) return B200_ERR_BAD_PARAM;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int *point_cell = static_cast<int *>(workspace);
  if (depth_grad && cudaMemsetAsync(depth_grad, 0, static_cast<size_t>(a.depth_size) * sizeof(TD), s) != cudaSuccess)
    return B200_ERR_LAUNCH;
  if (feat_grad && cudaMemsetAsync(feat_grad, 0, static_cast<size_t>(a.feat_rows) * a.C * sizeof(T), s) != cudaSuccess)
    return B200_ERR_LAUNCH;
  if (ws && cudaMemsetAsync(point_cell, 0xff, ws, s) != cudaSuccess) return B200_ERR_LAUNCH;
  if (a.I > 0) {
    switch (pick_vec<T>(a.C, {out_grad, feat})) {
      case 8: if constexpr (sizeof(T) <= 2) launch_depth_grad<T, TD, 8>(a, out_grad, feat, depth_grad, point_cell, s); break;
      case 4: launch_depth_grad<T, TD, 4>(a, out_grad, feat, depth_grad, point_cell, s); break;
      case 2: launch_depth_grad<T, TD, 2>(a, out_grad, feat, depth_grad, point_cell, s); break;
      default: launch_depth_grad<T, TD, 1>(a, out_grad, feat, depth_grad, point_cell, s); break;
    }
    const int st = check_launch();
    if (st != B200_OK) return st;
  }
  if (!feat_grad || a.P == 0) return B200_OK;
  switch (pick_vec<T>(a.C, {out_grad, feat_grad})) {
    case 8: if constexpr (sizeof(T) <= 2) launch_feat_grad<T, TD, 8>(a, order, out_grad, depth, point_cell, feat_grad, s); break;
    case 4: launch_feat_grad<T, TD, 4>(a, order, out_grad, depth, point_cell, feat_grad, s); break;
    case 2: launch_feat_grad<T, TD, 2>(a, order, out_grad, depth, point_cell, feat_grad, s); break;
    default: launch_feat_grad<T, TD, 1>(a, order, out_grad, depth, point_cell, feat_grad, s); break;
  }
  return check_launch();
}

}  // namespace

}  // namespace b200

using namespace b200;

#define B200_BEV_POOL_ARGS                                                                                      \
  BevPoolArgs a{ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths, depth_size, feat_rows,  \
                static_cast<long long>(out_height) * out_width, channels, num_points, num_intervals}

extern "C" {

int b200_bev_pool_f32(const float *depth, const float *feat, const int32_t *ranks_depth, const int32_t *ranks_feat,
                      const int32_t *ranks_bev, const int32_t *interval_starts, const int32_t *interval_lengths,
                      int channels, int num_points, int num_intervals, int64_t depth_size, int64_t feat_rows,
                      int out_height, int out_width, float *out, void *stream) {
  const int st = check_args(depth, feat, out, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths,
                            channels, num_points, num_intervals, depth_size, feat_rows, out_height, out_width,
                            sizeof(float), sizeof(float));
  if (st != B200_OK) return st;
  B200_BEV_POOL_ARGS;
  return bev_pool_forward<float>(a, depth, feat, out, 0.f, stream);
}

int b200_bev_pool_f16(const void *depth, const void *feat, const int32_t *ranks_depth, const int32_t *ranks_feat,
                      const int32_t *ranks_bev, const int32_t *interval_starts, const int32_t *interval_lengths,
                      int channels, int num_points, int num_intervals, int64_t depth_size, int64_t feat_rows,
                      int out_height, int out_width, void *out, void *stream) {
  const int st = check_args(depth, feat, out, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths,
                            channels, num_points, num_intervals, depth_size, feat_rows, out_height, out_width,
                            sizeof(__half), sizeof(__half));
  if (st != B200_OK) return st;
  B200_BEV_POOL_ARGS;
  return bev_pool_forward<__half>(a, static_cast<const __half *>(depth), static_cast<const __half *>(feat),
                                  static_cast<__half *>(out), 0.f, stream);
}

int b200_bev_pool_bf16(const void *depth, const void *feat, const int32_t *ranks_depth, const int32_t *ranks_feat,
                       const int32_t *ranks_bev, const int32_t *interval_starts, const int32_t *interval_lengths,
                       int channels, int num_points, int num_intervals, int64_t depth_size, int64_t feat_rows,
                       int out_height, int out_width, void *out, void *stream) {
  const int st = check_args(depth, feat, out, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths,
                            channels, num_points, num_intervals, depth_size, feat_rows, out_height, out_width,
                            sizeof(__nv_bfloat16), sizeof(__nv_bfloat16));
  if (st != B200_OK) return st;
  B200_BEV_POOL_ARGS;
  return bev_pool_forward<__nv_bfloat16>(a, static_cast<const __nv_bfloat16 *>(depth),
                                         static_cast<const __nv_bfloat16 *>(feat), static_cast<__nv_bfloat16 *>(out),
                                         0.f, stream);
}

int b200_bev_pool_f32_depth(int feat_dtype, const float *depth, const void *feat, const int32_t *ranks_depth,
                            const int32_t *ranks_feat, const int32_t *ranks_bev, const int32_t *interval_starts,
                            const int32_t *interval_lengths, int channels, int num_points, int num_intervals,
                            int64_t depth_size, int64_t feat_rows, int out_height, int out_width, void *out,
                            void *stream) {
  if (feat_dtype != kFeatF16 && feat_dtype != kFeatBF16) return B200_ERR_UNSUPPORTED;
  const int st = check_args(depth, feat, out, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths,
                            channels, num_points, num_intervals, depth_size, feat_rows, out_height, out_width,
                            sizeof(float), 2);
  if (st != B200_OK) return st;
  B200_BEV_POOL_ARGS;
  if (feat_dtype == kFeatF16)
    return bev_pool_forward<__half, float>(a, depth, static_cast<const __half *>(feat), static_cast<__half *>(out), 0.f,
                                           stream);
  return bev_pool_forward<__nv_bfloat16, float>(a, depth, static_cast<const __nv_bfloat16 *>(feat),
                                                static_cast<__nv_bfloat16 *>(out), 0.f, stream);
}

int b200_bev_pool_i8(const int8_t *depth, float scale_depth, const int8_t *feat, float scale_feat,
                     const int32_t *ranks_depth, const int32_t *ranks_feat, const int32_t *ranks_bev,
                     const int32_t *interval_starts, const int32_t *interval_lengths, int channels, int num_points,
                     int num_intervals, int64_t depth_size, int64_t feat_rows, int out_height, int out_width,
                     int8_t *out, float scale_out, void *stream) {
  const int st = check_args(depth, feat, out, ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths,
                            channels, num_points, num_intervals, depth_size, feat_rows, out_height, out_width,
                            sizeof(int8_t), sizeof(int8_t));
  if (st != B200_OK) return st;
  if (channels % 4 != 0) return B200_ERR_UNSUPPORTED;
  B200_BEV_POOL_ARGS;
  const float scale_io = scale_depth * scale_feat / scale_out;  // on the host, as bevPoolKernel.cu's launcher
  return bev_pool_forward<int8_t>(a, depth, feat, out, scale_io, stream);
}

size_t b200_bev_pool_backward_workspace_size(int num_points) {
  return num_points > 0 ? static_cast<size_t>(num_points) * sizeof(int) : 0;
}

int b200_bev_pool_backward_f32(const float *out_grad, const float *depth, const float *feat, const int32_t *ranks_depth,
                               const int32_t *ranks_feat, const int32_t *ranks_bev, const int32_t *interval_starts,
                               const int32_t *interval_lengths, const int32_t *feat_order, int channels, int num_points,
                               int num_intervals, int64_t depth_size, int64_t feat_rows, int out_height, int out_width,
                               float *depth_grad, float *feat_grad, void *workspace, size_t workspace_size,
                               void *stream) {
  const int st = check_args(depth, feat, out_grad, ranks_depth, ranks_feat, ranks_bev, interval_starts,
                            interval_lengths, channels, num_points, num_intervals, depth_size, feat_rows, out_height,
                            out_width, sizeof(float), sizeof(float));
  if (st != B200_OK) return st;
  B200_BEV_POOL_ARGS;
  return bev_pool_backward<float>(a, feat_order, out_grad, depth, feat, depth_grad, feat_grad, workspace,
                                  workspace_size, stream);
}

int b200_bev_pool_backward_f16(const void *out_grad, const void *depth, const void *feat, const int32_t *ranks_depth,
                               const int32_t *ranks_feat, const int32_t *ranks_bev, const int32_t *interval_starts,
                               const int32_t *interval_lengths, const int32_t *feat_order, int channels, int num_points,
                               int num_intervals, int64_t depth_size, int64_t feat_rows, int out_height, int out_width,
                               void *depth_grad, void *feat_grad, void *workspace, size_t workspace_size,
                               void *stream) {
  const int st = check_args(depth, feat, out_grad, ranks_depth, ranks_feat, ranks_bev, interval_starts,
                            interval_lengths, channels, num_points, num_intervals, depth_size, feat_rows, out_height,
                            out_width, sizeof(__half), sizeof(__half));
  if (st != B200_OK) return st;
  B200_BEV_POOL_ARGS;
  return bev_pool_backward<__half>(a, feat_order, static_cast<const __half *>(out_grad),
                                   static_cast<const __half *>(depth), static_cast<const __half *>(feat),
                                   static_cast<__half *>(depth_grad), static_cast<__half *>(feat_grad), workspace,
                                   workspace_size, stream);
}

int b200_bev_pool_backward_bf16(const void *out_grad, const void *depth, const void *feat, const int32_t *ranks_depth,
                                const int32_t *ranks_feat, const int32_t *ranks_bev, const int32_t *interval_starts,
                                const int32_t *interval_lengths, const int32_t *feat_order, int channels,
                                int num_points, int num_intervals, int64_t depth_size, int64_t feat_rows,
                                int out_height, int out_width, void *depth_grad, void *feat_grad, void *workspace,
                                size_t workspace_size, void *stream) {
  const int st = check_args(depth, feat, out_grad, ranks_depth, ranks_feat, ranks_bev, interval_starts,
                            interval_lengths, channels, num_points, num_intervals, depth_size, feat_rows, out_height,
                            out_width, sizeof(__nv_bfloat16), sizeof(__nv_bfloat16));
  if (st != B200_OK) return st;
  B200_BEV_POOL_ARGS;
  using B = __nv_bfloat16;
  return bev_pool_backward<B>(a, feat_order, static_cast<const B *>(out_grad), static_cast<const B *>(depth),
                              static_cast<const B *>(feat), static_cast<B *>(depth_grad), static_cast<B *>(feat_grad),
                              workspace, workspace_size, stream);
}

int b200_bev_pool_backward_f32_depth(int feat_dtype, const void *out_grad, const float *depth, const void *feat,
                                     const int32_t *ranks_depth, const int32_t *ranks_feat, const int32_t *ranks_bev,
                                     const int32_t *interval_starts, const int32_t *interval_lengths,
                                     const int32_t *feat_order, int channels, int num_points, int num_intervals,
                                     int64_t depth_size, int64_t feat_rows, int out_height, int out_width,
                                     float *depth_grad, void *feat_grad, void *workspace, size_t workspace_size,
                                     void *stream) {
  if (feat_dtype != kFeatF16 && feat_dtype != kFeatBF16) return B200_ERR_UNSUPPORTED;
  const int st = check_args(depth, feat, out_grad, ranks_depth, ranks_feat, ranks_bev, interval_starts,
                            interval_lengths, channels, num_points, num_intervals, depth_size, feat_rows, out_height,
                            out_width, sizeof(float), 2);
  if (st != B200_OK) return st;
  B200_BEV_POOL_ARGS;
  if (feat_dtype == kFeatF16)
    return bev_pool_backward<__half, float>(a, feat_order, static_cast<const __half *>(out_grad), depth,
                                            static_cast<const __half *>(feat), depth_grad,
                                            static_cast<__half *>(feat_grad), workspace, workspace_size, stream);
  using B = __nv_bfloat16;
  return bev_pool_backward<B, float>(a, feat_order, static_cast<const B *>(out_grad), depth,
                                     static_cast<const B *>(feat), depth_grad, static_cast<B *>(feat_grad), workspace,
                                     workspace_size, stream);
}

}  // extern "C"

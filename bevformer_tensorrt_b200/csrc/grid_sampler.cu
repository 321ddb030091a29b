// grid_sampler.cu — GridSampler2DTRT / GridSampler3DTRT for H100 (sm_90a).
//
// Replaces the reference launchers grid_sample<float|__half|__half2> and grid_sample_int8
// (TensorRT/plugin/grid_sampler/gridSamplerKernel.cu:1933-2043) and their kernels (:666-1923).
// Semantics = the reference FP32 kernel = ATen grid_sample with two twists (SURVEY Appendix B): the grid is
// channel-first [N, 2|3, ...] and spans [-10, 10] (gridSamplerKernel.cu:82-92, :694-698).
//
// The reference runs one thread per output pixel that walks all C channels with a read-modify-write on the output
// per tap (:725-739). Here a thread owns (pixel, slice of channel packets): the source index, tap offsets, weights and
// validity are computed once in fp32 registers, then each packet costs 4 independent loads + 4 FMAs + one store;
// consecutive threads are consecutive output pixels of the same channel, so loads are as coalesced as the sampling
// grid is smooth and stores are fully coalesced. FP16 and INT8 inputs are converted in registers (fp32 math), INT8
// output is requantised once (T2int8). The reference's __half kernels compute coordinates in half precision and its
// INT8 kernel leaves out-of-image taps uninitialised (:1140-1176); neither is reproduced.
#include <climits>

#include <cuda.h>  // CUtensorMap (types only; the encoder is fetched through cudaGetDriverEntryPoint)

#include "common.cuh"
#include "packets.cuh"

namespace b200 {

struct GsParams {
  const void *in;
  const void *grid;
  void *out;
  int N, C, CP;       // CP = channel packets (C, ceil(C/2), ceil(C/4))
  int Di, Hi, Wi;     // input spatial (Di = 1 for 2-D)
  int Do, Ho, Wo;     // output spatial
  int interp, padding, align;
  int slices, cps;    // channel slices per pixel, packets per slice
  float scale_i, scale_g, scale_o;
};

// ---- coordinate helpers: fp32, op-for-op the reference's (and ATen's) formulas -----------------------------------
__device__ __forceinline__ float gs_unnormalize(float coord, int size, bool align) {
  // no FMA contraction: the reference forms (coord+10)/2, size/10 and the product as separately rounded fp32 ops
  const float half = __fmul_rn(__fadd_rn(coord, 10.f), 0.5f);
  if (align) return __fmul_rn(half, __fdiv_rn(static_cast<float>(size - 1), 10.f));
  return __fadd_rn(__fmul_rn(half, __fdiv_rn(static_cast<float>(size), 10.f)), -0.5f);
}
__device__ __forceinline__ float gs_clip(float in, int limit) {
  return fminf(static_cast<float>(limit - 1), fmaxf(in, 0.f));
}
__device__ __forceinline__ float gs_reflect(float in, int twice_low, int twice_high) {
  if (twice_low == twice_high) return 0.f;
  const float mn = __fmul_rn(static_cast<float>(twice_low), 0.5f);
  const float span = __fmul_rn(static_cast<float>(twice_high - twice_low), 0.5f);
  in = fabsf(__fsub_rn(in, mn));
  const float extra = fmodf(in, span);
  const int flips = static_cast<int>(floorf(__fdiv_rn(in, span)));
  return (flips % 2 == 0) ? __fadd_rn(extra, mn) : __fadd_rn(__fsub_rn(span, extra), mn);
}
__device__ __forceinline__ float gs_safe(float x) {
  if (x > static_cast<float>(INT_MAX - 1) || x < static_cast<float>(INT_MIN) || !isfinite(x)) return -100.f;
  return x;
}
__device__ __forceinline__ float gs_compute_coordinates(float coord, int size, int padding, bool align) {
  if (padding == 1) {
    coord = gs_clip(coord, size);
  } else if (padding == 2) {
    coord = align ? gs_reflect(coord, 0, 2 * (size - 1)) : gs_reflect(coord, -1, 2 * size - 1);
    coord = gs_clip(coord, size);
  }
  return gs_safe(coord);
}
__device__ __forceinline__ float gs_source_index(float coord, int size, int padding, bool align) {
  return gs_compute_coordinates(gs_unnormalize(coord, size, align), size, padding, align);
}
__device__ __forceinline__ float cubic1(float x, float A) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic2(float x, float A) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }
__device__ __forceinline__ void cubic_coeffs(float (&c)[4], float t) {
  const float A = -0.75f;
  c[0] = cubic2(t + 1.f, A);
  c[1] = cubic1(t, A);
  const float x2 = 1.f - t;
  c[2] = cubic1(x2, A);
  c[3] = cubic2(x2 + 1.f, A);
}

// ---- 2-D kernel -----------------------------------------------------------------------------------------------------
// INTERP is a template parameter so that the bilinear kernel (the one BEVFormer uses) does not carry the bicubic
// path's registers: 64 registers -> 4 CTAs of 256 threads per SM.
template <int K, int INTERP>
__global__ void __launch_bounds__(256, INTERP == 2 ? 2 : 4) grid_sample_2d_kernel(const GsParams p) {
  using P = Pk<K>;
  using T = typename P::T;
  constexpr int W = P::W;
  const long long plane_o = static_cast<long long>(p.Ho) * p.Wo;
  const long long plane_i = static_cast<long long>(p.Hi) * p.Wi;
  const long long total = static_cast<long long>(p.N) * p.slices * plane_o;
  const bool align = p.align != 0;
  // INT8 output requantisation is a true division in the reference's fp32 oracle form; one reciprocal here differs by
  // at most an ulp before rounding to int8.
  const float so = K == kI8x4 ? 1.f / p.scale_o : 1.f;

  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long pix = idx % plane_o;
    const int s = static_cast<int>((idx / plane_o) % p.slices);
    const long long n = idx / (plane_o * p.slices);
    float gx, gy, gz;
    P::grid_xy(p.grid, plane_o, pix, n, p.scale_g, gx, gy, gz, false);

    const int cp0 = s * p.cps, cp1 = min(p.CP, cp0 + p.cps);
    const T *in_n = static_cast<const T *>(p.in) + (n * p.CP + cp0) * plane_i;
    T *out_p = static_cast<T *>(p.out) + (n * p.CP + cp0) * plane_o + pix;

    if (INTERP == 0) {  // bilinear (:700-740)
      const float ix = gs_source_index(gx, p.Wi, p.padding, align);
      const float iy = gs_source_index(gy, p.Hi, p.padding, align);
      const int ix_nw = static_cast<int>(floorf(ix)), iy_nw = static_cast<int>(floorf(iy));
      const int ix_se = ix_nw + 1, iy_se = iy_nw + 1;
      const float fx1 = __fsub_rn(static_cast<float>(ix_se), ix), fx0 = __fsub_rn(ix, static_cast<float>(ix_nw));
      const float fy1 = __fsub_rn(static_cast<float>(iy_se), iy), fy0 = __fsub_rn(iy, static_cast<float>(iy_nw));
      const bool x0 = ix_nw >= 0 && ix_nw < p.Wi, x1 = ix_se >= 0 && ix_se < p.Wi;
      const bool y0 = iy_nw >= 0 && iy_nw < p.Hi, y1 = iy_se >= 0 && iy_se < p.Hi;
      const float w_nw = (x0 && y0) ? fx1 * fy1 : 0.f, w_ne = (x1 && y0) ? fx0 * fy1 : 0.f;
      const float w_sw = (x0 && y1) ? fx1 * fy0 : 0.f, w_se = (x1 && y1) ? fx0 * fy0 : 0.f;
      // out-of-image taps alias an in-image address (clamped), so loads are unconditional; what they load is dropped
      // (pk_load_if), not multiplied by their zero weight
      const bool v_nw = x0 && y0, v_ne = x1 && y0, v_sw = x0 && y1, v_se = x1 && y1;
      const int cx0 = min(max(ix_nw, 0), p.Wi - 1), cx1 = min(max(ix_se, 0), p.Wi - 1);
      const int cy0 = min(max(iy_nw, 0), p.Hi - 1), cy1 = min(max(iy_se, 0), p.Hi - 1);
      const int o_nw = cy0 * p.Wi + cx0, o_ne = cy0 * p.Wi + cx1, o_sw = cy1 * p.Wi + cx0, o_se = cy1 * p.Wi + cx1;
      const T *ip = in_n;
      T *op = out_p;
#pragma unroll 8
      for (int cp = cp0; cp < cp1; ++cp, ip += plane_i, op += plane_o) {
        float a[W], b[W], c[W], d[W], o[W];
        pk_load_if<K>(ip + o_nw, v_nw, a, p.scale_i), pk_load_if<K>(ip + o_ne, v_ne, b, p.scale_i);
        pk_load_if<K>(ip + o_sw, v_sw, c, p.scale_i), pk_load_if<K>(ip + o_se, v_se, d, p.scale_i);
#pragma unroll
        for (int i = 0; i < W; ++i) o[i] = fmaf(d[i], w_se, fmaf(c[i], w_sw, fmaf(b[i], w_ne, a[i] * w_nw)));
        P::store(op, o, so);
      }
    } else if (INTERP == 1) {  // nearest (:741-756): ::round, half away from zero
      const float ix = gs_source_index(gx, p.Wi, p.padding, align);
      const float iy = gs_source_index(gy, p.Hi, p.padding, align);
      const int ixn = static_cast<int>(roundf(ix)), iyn = static_cast<int>(roundf(iy));
      const bool ok = ixn >= 0 && ixn < p.Wi && iyn >= 0 && iyn < p.Hi;
      const int o_n = ok ? iyn * p.Wi + ixn : 0;
      const T *ip = in_n;
      T *op = out_p;
      for (int cp = cp0; cp < cp1; ++cp, ip += plane_i, op += plane_o) {
        float a[W];
        P::load(ip + o_n, a, p.scale_i);
#pragma unroll
        for (int i = 0; i < W; ++i) a[i] = ok ? a[i] : 0.f;
        P::store(op, a, so);
      }
    } else {  // bicubic (:757-792)
      const float ix = gs_unnormalize(gx, p.Wi, align), iy = gs_unnormalize(gy, p.Hi, align);
      const float ix_nw = floorf(ix), iy_nw = floorf(iy);
      float cx[4], cy[4];
      cubic_coeffs(cx, ix - ix_nw);
      cubic_coeffs(cy, iy - iy_nw);
      int xo[4], yo[4];  // column / row offsets, -1 when outside (get_value_bounded :615-629)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int xi = static_cast<int>(gs_compute_coordinates(ix_nw - 1.f + i, p.Wi, p.padding, align));
        const int yi = static_cast<int>(gs_compute_coordinates(iy_nw - 1.f + i, p.Hi, p.padding, align));
        xo[i] = (xi >= 0 && xi < p.Wi) ? xi : -1;
        yo[i] = (yi >= 0 && yi < p.Hi) ? yi * p.Wi : -1;
      }
      const T *ip = in_n;
      T *op = out_p;
      for (int cp = cp0; cp < cp1; ++cp, ip += plane_i, op += plane_o) {
        float o[W];
#pragma unroll
        for (int i = 0; i < W; ++i) o[i] = 0.f;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          float row[W];
#pragma unroll
          for (int i = 0; i < W; ++i) row[i] = 0.f;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float v[W];
            const bool ok = xo[q] >= 0 && yo[r] >= 0;
            P::load(ip + (ok ? yo[r] + xo[q] : 0), v, p.scale_i);
#pragma unroll
            for (int i = 0; i < W; ++i) row[i] = fmaf(ok ? v[i] : 0.f, cx[q], row[i]);
          }
#pragma unroll
          for (int i = 0; i < W; ++i) o[i] = fmaf(row[i], cy[r], o[i]);
        }
        P::store(op, o, so);
      }
    }
  }
}

// ---- 2-D bilinear tile kernel (opt-in: b200_grid_sample_set_tile_path): source window staged in shared memory by TMA ------
// For a smooth sampling grid (the prev-BEV warp is a small rotation, onnx_ops.py:226-232) the source pixels of an 8 x 32
// output tile form a compact window. One CTA = one output tile x one block of channel packets:
//   1. every thread evaluates the index arithmetic of its pixel (the same device functions as the generic kernel: the
//      sampled pixel is bit-identical), and the CTA reduces the bounding box of the clamped tap coordinates;
//   2. if the box fits kBH rows x kRowBytes, warp 0 stages it: mode 2 = one 2-D tensor copy per channel packet
//      (cp.async.bulk.tensor.2d over the [N*CP*Hi, Wi] view, SASS UTMALDG.2D), mode 1 = one bulk copy per (packet, row)
//      (cp.async.bulk, SASS UBLKCP); completion counted on one mbarrier; otherwise the CTA runs the per-tap global loads;
//   3. each packet is then 4 shared-memory loads at compile-time channel offsets + 4 FMAs + one coalesced store.
// Where it was timed, mode 2 equalled the generic kernel and mode 1 was slower (small bulk copies per row serialise) —
// the op is bound by the latency chain grid load -> index arithmetic -> first loads, not by the tap loads, so the generic
// kernel stays the default. Two TMA facts learnt on the way: a tensor copy whose innermost origin
// coordinate x element size is not a multiple of 16 bytes raises "illegal instruction" on this part (3-D and 2-D boxes
// alike), so the window origin is rounded down to 16 bytes; rounding costs up to 7 halves / 3 words of row slack.
constexpr int kTW = 32, kTH = 8;  // output tile (a warp = 32 consecutive x)
constexpr int kBH = 16;           // source window rows held in shared memory

template <int K>
struct TileCfg {
  using T = typename Pk<K>::T;
  static constexpr int kEB = static_cast<int>(sizeof(T));
  static constexpr int kCB = kEB == 2 ? 32 : 16;                   // packets per CTA
  static constexpr int kRowBytes = kEB == 2 ? 96 : 176;            // 48 halves / 44 words per window row (incl. alignment slack)
  static constexpr int kRowElems = kRowBytes / kEB;
  static constexpr int kSmem = kCB * kBH * kRowBytes;              // 48 KB / 44 KB
};

template <int K, bool TENSOR>
__global__ void __launch_bounds__(256, 4) grid_sample_2d_tile_kernel(const GsParams p, const __grid_constant__ CUtensorMap tmap,
                                                                     int tiles_x) {
  using P = Pk<K>;
  using T = typename P::T;
  using Cfg = TileCfg<K>;
  constexpr int W = P::W;
  constexpr int CB = Cfg::kCB, EB = Cfg::kEB, RE = Cfg::kRowElems;
  extern __shared__ __align__(128) unsigned char gs_smem[];
  __shared__ int red[8][4];
  __shared__ int fin[4];
  __shared__ __align__(8) unsigned long long bar;
  const T *win = reinterpret_cast<const T *>(gs_smem);

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int ty = blockIdx.x / tiles_x, tx = blockIdx.x - ty * tiles_x;
  const int ox = tx * kTW + lane, oy = ty * kTH + warp;
  const int n = blockIdx.z, cp0 = blockIdx.y * CB, cp1 = min(p.CP, cp0 + CB);
  const bool valid = ox < p.Wo && oy < p.Ho;
  const long long plane_o = static_cast<long long>(p.Ho) * p.Wo, plane_i = static_cast<long long>(p.Hi) * p.Wi;
  const long long pix = static_cast<long long>(oy) * p.Wo + ox;
  const bool align = p.align != 0;
  const float so = K == kI8x4 ? 1.f / p.scale_o : 1.f;

  float w_nw = 0.f, w_ne = 0.f, w_sw = 0.f, w_se = 0.f;
  bool v_nw = false, v_ne = false, v_sw = false, v_se = false;  // tap inside the image
  int cx0 = INT_MAX, cx1 = INT_MIN, cy0 = INT_MAX, cy1 = INT_MIN;
  if (valid) {
    float gx, gy, gz;
    P::grid_xy(p.grid, plane_o, pix, n, p.scale_g, gx, gy, gz, false);
    const float ix = gs_source_index(gx, p.Wi, p.padding, align);
    const float iy = gs_source_index(gy, p.Hi, p.padding, align);
    const int ix_nw = static_cast<int>(floorf(ix)), iy_nw = static_cast<int>(floorf(iy));
    const int ix_se = ix_nw + 1, iy_se = iy_nw + 1;
    const float fx1 = __fsub_rn(static_cast<float>(ix_se), ix), fx0 = __fsub_rn(ix, static_cast<float>(ix_nw));
    const float fy1 = __fsub_rn(static_cast<float>(iy_se), iy), fy0 = __fsub_rn(iy, static_cast<float>(iy_nw));
    const bool x0 = ix_nw >= 0 && ix_nw < p.Wi, x1 = ix_se >= 0 && ix_se < p.Wi;
    const bool y0 = iy_nw >= 0 && iy_nw < p.Hi, y1 = iy_se >= 0 && iy_se < p.Hi;
    w_nw = (x0 && y0) ? fx1 * fy1 : 0.f, w_ne = (x1 && y0) ? fx0 * fy1 : 0.f;
    w_sw = (x0 && y1) ? fx1 * fy0 : 0.f, w_se = (x1 && y1) ? fx0 * fy0 : 0.f;
    // out-of-image taps alias an in-image pixel (clamped), so loads are unconditional; what they load is dropped
    v_nw = x0 && y0, v_ne = x1 && y0, v_sw = x0 && y1, v_se = x1 && y1;
    cx0 = min(max(ix_nw, 0), p.Wi - 1), cx1 = min(max(ix_se, 0), p.Wi - 1);
    cy0 = min(max(iy_nw, 0), p.Hi - 1), cy1 = min(max(iy_se, 0), p.Hi - 1);
  }
  // ---- bounding box of the tile's taps
  int bx0 = min(cx0, cx1), bx1 = max(cx0, cx1), by0 = min(cy0, cy1), by1 = max(cy0, cy1);
  if (!valid) bx0 = by0 = INT_MAX, bx1 = by1 = INT_MIN;
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) {
    bx0 = min(bx0, __shfl_xor_sync(kFullMask, bx0, d)), bx1 = max(bx1, __shfl_xor_sync(kFullMask, bx1, d));
    by0 = min(by0, __shfl_xor_sync(kFullMask, by0, d)), by1 = max(by1, __shfl_xor_sync(kFullMask, by1, d));
  }
  if (lane == 0) red[warp][0] = bx0, red[warp][1] = bx1, red[warp][2] = by0, red[warp][3] = by1;
  const uint32_t barr = static_cast<uint32_t>(__cvta_generic_to_shared(&bar));
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(barr) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // warp 0 finishes the reduction and, if the window fits, issues the row copies (segment start rounded down to 16 bytes)
  if (warp == 0) {
    const int w8 = lane & 7;
    bx0 = __reduce_min_sync(kFullMask, red[w8][0]), bx1 = __reduce_max_sync(kFullMask, red[w8][1]);
    by0 = __reduce_min_sync(kFullMask, red[w8][2]), by1 = __reduce_max_sync(kFullMask, red[w8][3]);
    const int xs = bx0 & ~(16 / EB - 1);
    const int len = ((bx1 - xs + 1) * EB + 15) & ~15, nrows = by1 - by0 + 1, ncp = cp1 - cp0;
    const bool fits0 = bx1 >= bx0 && len <= Cfg::kRowBytes && nrows <= kBH;
    if (lane == 0) fin[0] = xs, fin[1] = by0, fin[2] = fits0 ? 1 : 0;
    if (fits0 && TENSOR) {
      // one 2-D tensor copy per channel packet: box = kRowElems columns x kBH rows of the [N*CP*Hi, Wi] view, origin
      // (xs, plane row + by0) with xs * EB a multiple of 16 bytes; columns past the image are zero-filled, rows past the
      // plane belong to the next plane (never read: the window is inside the image)
      if (lane == 0) {
        const uint32_t dst0 = static_cast<uint32_t>(__cvta_generic_to_shared(gs_smem));
        const int row0 = (n * p.CP + cp0) * p.Hi + by0;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(barr), "r"(ncp * kBH * Cfg::kRowBytes) : "memory");
#pragma unroll 1
        for (int c = 0; c < ncp; ++c)
          asm volatile(
              "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                  dst0 + c * (kBH * Cfg::kRowBytes)),
              "l"(&tmap), "r"(xs), "r"(row0 + c * p.Hi), "r"(barr)
              : "memory");
      }
    } else if (fits0) {
      if (lane == 0)
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(barr), "r"(ncp * nrows * len) : "memory");
      __syncwarp();
      const unsigned char *src0 = static_cast<const unsigned char *>(p.in) +
                                  ((static_cast<long long>(n) * p.CP + cp0) * plane_i + static_cast<long long>(by0) * p.Wi + xs) * EB;
      const uint32_t dst0 = static_cast<uint32_t>(__cvta_generic_to_shared(gs_smem));
      for (int i = lane; i < ncp * nrows; i += 32) {
        const int c = i / nrows, r = i - c * nrows;
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                         dst0 + (c * kBH + r) * Cfg::kRowBytes),
                     "l"(src0 + (c * plane_i + static_cast<long long>(r) * p.Wi) * EB), "r"(len), "r"(barr)
                     : "memory");
      }
    }
  }
  __syncthreads();
  const int xs = fin[0];
  by0 = fin[1];
  const bool fits = fin[2] != 0;  // CTA-uniform
  T *out_p = static_cast<T *>(p.out) + (static_cast<long long>(n) * p.CP + cp0) * plane_o + pix;

  if (fits) {
    uint32_t done = 0;
    while (!done)
      asm volatile("{ .reg .pred q; mbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2; selp.u32 %0, 1, 0, q; }"
                   : "=r"(done) : "r"(barr), "r"(0u) : "memory");
    if (valid) {
      const int o_nw = (cy0 - by0) * RE + (cx0 - xs), o_ne = (cy0 - by0) * RE + (cx1 - xs);
      const int o_sw = (cy1 - by0) * RE + (cx0 - xs), o_se = (cy1 - by0) * RE + (cx1 - xs);
      const int ncp = cp1 - cp0;
#pragma unroll 8
      for (int c = 0; c < CB; ++c) {
        if (c >= ncp) break;
        const T *wc = win + c * (kBH * RE);
        float a[W], b[W], cc[W], d[W], o[W];
        pk_unpack_if<K>(wc[o_nw], v_nw, a, p.scale_i), pk_unpack_if<K>(wc[o_ne], v_ne, b, p.scale_i);
        pk_unpack_if<K>(wc[o_sw], v_sw, cc, p.scale_i), pk_unpack_if<K>(wc[o_se], v_se, d, p.scale_i);
#pragma unroll
        for (int i = 0; i < W; ++i) o[i] = fmaf(d[i], w_se, fmaf(cc[i], w_sw, fmaf(b[i], w_ne, a[i] * w_nw)));
        P::store(out_p + c * plane_o, o, so);
      }
    }
  } else if (valid) {  // window too large for shared memory (a strongly distorted grid): per-tap global loads
    const T *ip = static_cast<const T *>(p.in) + (static_cast<long long>(n) * p.CP + cp0) * plane_i;
    const int o_nw = cy0 * p.Wi + cx0, o_ne = cy0 * p.Wi + cx1, o_sw = cy1 * p.Wi + cx0, o_se = cy1 * p.Wi + cx1;
    T *op = out_p;
#pragma unroll 4
    for (int cp = cp0; cp < cp1; ++cp, ip += plane_i, op += plane_o) {
      float a[W], b[W], cc[W], d[W], o[W];
      pk_load_if<K>(ip + o_nw, v_nw, a, p.scale_i), pk_load_if<K>(ip + o_ne, v_ne, b, p.scale_i);
      pk_load_if<K>(ip + o_sw, v_sw, cc, p.scale_i), pk_load_if<K>(ip + o_se, v_se, d, p.scale_i);
#pragma unroll
      for (int i = 0; i < W; ++i) o[i] = fmaf(d[i], w_se, fmaf(cc[i], w_sw, fmaf(b[i], w_ne, a[i] * w_nw)));
      P::store(op, o, so);
    }
  }
}

// ---- 3-D kernel (GridSampler3DTRT, :1271-1923): trilinear / nearest, fp32 / fp16 kLINEAR ----------------------------
template <int K>
__global__ void __launch_bounds__(256) grid_sample_3d_kernel(const GsParams p) {
  using P = Pk<K>;
  using T = typename P::T;
  const long long plane_o = static_cast<long long>(p.Do) * p.Ho * p.Wo;
  const long long plane_i = static_cast<long long>(p.Di) * p.Hi * p.Wi;
  const long long total = static_cast<long long>(p.N) * p.slices * plane_o;
  const bool align = p.align != 0;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long pix = idx % plane_o;
    const int s = static_cast<int>((idx / plane_o) % p.slices);
    const long long n = idx / (plane_o * p.slices);
    float gx, gy, gz;
    P::grid_xy(p.grid, plane_o, pix, n, 1.f, gx, gy, gz, true);
    const float ix = gs_source_index(gx, p.Wi, p.padding, align);
    const float iy = gs_source_index(gy, p.Hi, p.padding, align);
    const float iz = gs_source_index(gz, p.Di, p.padding, align);
    const int cp0 = s * p.cps, cp1 = min(p.CP, cp0 + p.cps);
    const T *ip = static_cast<const T *>(p.in) + (n * p.CP + cp0) * plane_i;
    T *op = static_cast<T *>(p.out) + (n * p.CP + cp0) * plane_o + pix;
    if (p.interp == 0) {
      const int x0 = static_cast<int>(floorf(ix)), y0 = static_cast<int>(floorf(iy)), z0 = static_cast<int>(floorf(iz));
      const float fx = ix - x0, fy = iy - y0, fz = iz - z0;
      int off[8];
      float wt[8];
      unsigned inside = 0;  // bit t: corner t is inside the volume
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const int dx = t & 1, dy = (t >> 1) & 1, dz = t >> 2;
        const int x = x0 + dx, y = y0 + dy, z = z0 + dz;
        const bool ok = x >= 0 && x < p.Wi && y >= 0 && y < p.Hi && z >= 0 && z < p.Di;
        // weight of a corner = product over axes of (1 - f) for the low side and f for the high side, written as the
        // reference does: (x_high - ix) etc. (:1330-1337)
        const float wx = dx ? fx : (static_cast<float>(x0 + 1) - ix);
        const float wy = dy ? fy : (static_cast<float>(y0 + 1) - iy);
        const float wz = dz ? fz : (static_cast<float>(z0 + 1) - iz);
        wt[t] = ok ? wx * wy * wz : 0.f;
        off[t] = ok ? (z * p.Hi + y) * p.Wi + x : 0;
        inside |= ok ? 1u << t : 0u;
      }
      for (int cp = cp0; cp < cp1; ++cp, ip += plane_i, op += plane_o) {
        float o[1] = {0.f};
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          float v[1];
          pk_load_if<K>(ip + off[t], (inside >> t) & 1u, v, 1.f);  // an outside corner reads element 0 and drops it
          o[0] = fmaf(v[0], wt[t], o[0]);
        }
        P::store(op, o, 1.f);
      }
    } else {
      const int x = static_cast<int>(roundf(ix)), y = static_cast<int>(roundf(iy)), z = static_cast<int>(roundf(iz));
      const bool ok = x >= 0 && x < p.Wi && y >= 0 && y < p.Hi && z >= 0 && z < p.Di;
      const int o_n = ok ? (z * p.Hi + y) * p.Wi + x : 0;
      for (int cp = cp0; cp < cp1; ++cp, ip += plane_i, op += plane_o) {
        float v[1];
        P::load(ip + o_n, v, 1.f);
        v[0] = ok ? v[0] : 0.f;
        P::store(op, v, 1.f);
      }
    }
  }
}

// ---- host -----------------------------------------------------------------------------------------------------------
static std::atomic<int> g_gs_tile{0};  // 1: shared-memory tile path for 2-D bilinear where it applies (b200_grid_sample_set_tile_path)

typedef CUresult (*GsEncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// B200_ERR_UNSUPPORTED = the layout does not meet the copies' 16-byte rules (the caller takes the generic kernel).
// mode 1: one bulk copy per (packet, row); mode 2: one 2-D tensor copy per packet.
template <int K>
static int launch_gs_tile(const GsParams &p, int mode, cudaStream_t s) {
  using Cfg = TileCfg<K>;
  if (reinterpret_cast<uintptr_t>(p.in) % 16 || (static_cast<long long>(p.Wi) * Cfg::kEB) % 16) return B200_ERR_UNSUPPORTED;
  if (p.N > 65535 || static_cast<long long>(p.N) * p.CP * p.Hi >= (1ll << 31)) return B200_ERR_UNSUPPORTED;
  const int tiles_x = (p.Wo + kTW - 1) / kTW, tiles_y = (p.Ho + kTH - 1) / kTH;
  const long long tiles = static_cast<long long>(tiles_x) * tiles_y;
  const int cblocks = (p.CP + Cfg::kCB - 1) / Cfg::kCB;
  if (tiles > 0x7fffffffll || cblocks > 65535) return B200_ERR_UNSUPPORTED;
  CUtensorMap tm{};
  if (mode == 2) {
    static std::atomic<GsEncodeTiledFn> cached{nullptr};
    GsEncodeTiledFn encode = cached.load(std::memory_order_acquire);
    if (!encode) {
      void *fn = nullptr;
      cudaDriverEntryPointQueryResult qres;
      if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn)
        return B200_ERR_UNSUPPORTED;
      encode = reinterpret_cast<GsEncodeTiledFn>(fn);
      cached.store(encode, std::memory_order_release);
    }
    const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(p.Wi), static_cast<cuuint64_t>(p.N) * p.CP * p.Hi};
    const cuuint64_t gstr[1] = {static_cast<cuuint64_t>(p.Wi) * Cfg::kEB};
    const cuuint32_t box[2] = {static_cast<cuuint32_t>(Cfg::kRowElems), kBH};
    const cuuint32_t estr[2] = {1, 1};
    const CUtensorMapDataType dt = Cfg::kEB == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    if (encode(&tm, dt, 2, const_cast<void *>(p.in), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return B200_ERR_UNSUPPORTED;
  }
  auto launch = [&](auto kern) -> int {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem) != cudaSuccess) return B200_ERR_LAUNCH;
    kern<<<dim3(static_cast<unsigned>(tiles), cblocks, p.N), 256, Cfg::kSmem, s>>>(p, tm, tiles_x);
    return check_launch();
  };
  return mode == 2 ? launch(grid_sample_2d_tile_kernel<K, true>) : launch(grid_sample_2d_tile_kernel<K, false>);
}

// The one check of a call's dims, which fills p's geometry: N, C and the input extents from input_dims, the output
// extents from grid_dims (Di = Do = 1 in 2-D), CP = packets of `width` channels. planar3d: the layout has a 3-D kernel.
// The output dims must be [N, C, grid spatial]: the kernels write that extent whatever output_dims says.
static int gs_geom(GsParams &p, const int *od, const int *id, const int *gd, int nb, int width, bool planar3d, int interp,
                   int padding) {
  // rank 4, or 5 for the linear layouts: the reference printf()s and returns (:1959-1961, :2040-2042)
  if (nb != 4 && (nb != 5 || !planar3d)) return B200_ERR_UNSUPPORTED;
  if (interp < 0 || interp > 2 || padding < 0 || padding > 2) return B200_ERR_BAD_PARAM;
  for (int i = 0; i < nb; ++i)
    if (id[i] <= 0 || gd[i] <= 0 || od[i] <= 0) return B200_ERR_BAD_PARAM;
  if (gd[0] != id[0] || gd[1] != nb - 2) return B200_ERR_BAD_PARAM;
  for (int i = 0; i < nb; ++i)
    if (od[i] != (i < 2 ? id[i] : gd[i])) return B200_ERR_BAD_PARAM;
  if (nb == 5 && interp == 2) return B200_ERR_UNSUPPORTED;  // no 3-D bicubic
  const int s = nb - 4;  // 1 where there is a depth axis
  p.N = id[0], p.C = id[1], p.CP = (id[1] + width - 1) / width, p.interp = interp, p.padding = padding;
  p.Di = s ? id[2] : 1, p.Hi = id[2 + s], p.Wi = id[3 + s], p.Do = s ? gd[2] : 1, p.Ho = gd[2 + s], p.Wo = gd[3 + s];
  const long long plane_i = static_cast<long long>(p.Di) * p.Hi * p.Wi;
  const long long plane_o = static_cast<long long>(p.Do) * p.Ho * p.Wo;
  return plane_i >= (1ll << 31) || plane_o >= (1ll << 31) ? B200_ERR_BAD_PARAM : B200_OK;
}

template <int K>
static int launch_gs(void *out, const void *in, const void *grid, const int *od, const int *id, const int *gd, int nb,
                     int interp, int padding, int align, float si, float sg, float so, cudaStream_t s) {
  if (!out || !in || !grid || !od || !id || !gd) return B200_ERR_BAD_PARAM;
  GsParams p{};
  const int st = gs_geom(p, od, id, gd, nb, Pk<K>::W, K == kF32 || K == kF16, interp, padding);
  if (st != B200_OK) return st;
  p.in = in, p.grid = grid, p.out = out, p.align = align, p.scale_i = si, p.scale_g = sg, p.scale_o = so;
  if (nb == 4 && interp == 0 && g_gs_tile.load(std::memory_order_relaxed)) {
    const int tst = launch_gs_tile<K>(p, g_gs_tile.load(std::memory_order_relaxed), s);
    if (tst != B200_ERR_UNSUPPORTED) return tst;
  }
  // about two resident waves of the 132 SMs (4 CTAs x 256 threads each) so that the index arithmetic of a pixel (~150
  // instructions) is amortised over as many channel packets as possible, at most 64 per thread
  const unsigned blocks = plan_slices(static_cast<long long>(p.N) * p.Do * p.Ho * p.Wo, p.CP, 132ll * 1024 * 2, 64,
                                      p.slices, p.cps);
  const auto kern = nb == 5      ? grid_sample_3d_kernel<(K == kF16 ? kF16 : kF32)>
                    : interp == 0 ? grid_sample_2d_kernel<K, 0>
                    : interp == 1 ? grid_sample_2d_kernel<K, 1>
                                  : grid_sample_2d_kernel<K, 2>;
  kern<<<blocks, 256, 0, s>>>(p);
  return check_launch();
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_grid_sample_set_tile_path(int mode) { return g_gs_tile.exchange(mode < 0 || mode > 2 ? 0 : mode); }

int b200_grid_sample_f32(float *output, const float *input, const float *grid, const int *output_dims,
                         const int *input_dims, const int *grid_dims, int nb_dims, int interp, int padding,
                         int align_corners, void *stream) {
  return launch_gs<kF32>(output, input, grid, output_dims, input_dims, grid_dims, nb_dims, interp, padding,
                         align_corners, 1.f, 1.f, 1.f, static_cast<cudaStream_t>(stream));
}

int b200_grid_sample_f16(void *output, const void *input, const void *grid, const int *output_dims,
                         const int *input_dims, const int *grid_dims, int nb_dims, int interp, int padding,
                         int align_corners, void *stream) {
  return launch_gs<kF16>(output, input, grid, output_dims, input_dims, grid_dims, nb_dims, interp, padding,
                         align_corners, 1.f, 1.f, 1.f, static_cast<cudaStream_t>(stream));
}

int b200_grid_sample_f16_chw2(void *output, const void *input, const void *grid, const int *output_dims,
                              const int *input_dims, const int *grid_dims, int nb_dims, int interp, int padding,
                              int align_corners, void *stream) {
  return launch_gs<kF16x2>(output, input, grid, output_dims, input_dims, grid_dims, nb_dims, interp, padding,
                           align_corners, 1.f, 1.f, 1.f, static_cast<cudaStream_t>(stream));
}

int b200_grid_sample_i8_chw4(int8_t *output, float scale_o, const int8_t *input, float scale_i, const int8_t *grid,
                             float scale_g, const int *output_dims, const int *input_dims, const int *grid_dims,
                             int nb_dims, int interp, int padding, int align_corners, void *stream) {
  if (!(scale_o > 0.f)) return B200_ERR_BAD_PARAM;
  return launch_gs<kI8x4>(output, input, grid, output_dims, input_dims, grid_dims, nb_dims, interp, padding,
                          align_corners, scale_i, scale_g, scale_o, static_cast<cudaStream_t>(stream));
}

}  // extern "C"

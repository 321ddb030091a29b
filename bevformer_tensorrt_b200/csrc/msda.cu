// msda.cu — multi-scale deformable attention for H100 (sm_90a).
//
// Replaces the reference launchers ms_deformable_im2col_cuda<float|__half>, …_h2 and …_int8<float|__half2>
// (TensorRT/plugin/multi_scale_deformable_attn/multiScaleDeformableAttnKernel.cu:1106-1218) and their kernels
// (:611-1104). Semantics follow the FP32 kernel (:611-688 with the tap rule :133-178); see include/b200_bev_ops.h.
//
// Work decomposition (the reference uses one thread per output scalar, re-reading all logits/offsets per channel):
//   item            = one (batch, query, head): NP = L*P sampling points, C channels.
//   lane group      = LPI = C/VEC lanes own one item (VEC = 4 fp32, 8 fp16, 8 int8 channels per lane), so each
//                     bilinear tap of an item is ONE vector load per lane (128-bit; 64-bit for int8) and a warp covers 32/LPI items.
//   point ownership = offsets/logits are read exactly once with vector loads: chunk c (4 consecutive points) of an
//                     item belongs to lane c % LPI of its group. The owner evaluates the index arithmetic once
//                     (fp32, bit-exact with the reference), folds softmax numerator x bilinear weight x tap validity
//                     into four tap weights, and broadcasts {packed address code, 4 weights} to its group with warp
//                     shuffles. Softmax max / sum are shuffle reductions inside the lane group.
//   gather          = all lanes of the group then issue the four 128-bit taps of that point for their channel slice
//                     and accumulate in fp32 registers; points that are out of range in every item of the warp are
//                     skipped with one ballot (the common case for cameras that do not see the BEV query).
// Memory: value taps go through the read-only path and are meant to hit L1/L2 (the 95 MB value stack of the base
// config fits the 126 MB L2); offsets/logits/out are streamed with L1::no_allocate so they do not evict taps.
#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "msda_geometry.cuh"
#include "msda_index.cuh"

namespace b200 {

constexpr int kMaxLevels = kMsdaMaxLevels;
constexpr int kThreads = 256;
#ifndef B200_MSDA_MIN_BLOCKS
#define B200_MSDA_MIN_BLOCKS 3
#endif
constexpr int kMinBlocks = B200_MSDA_MIN_BLOCKS;  // 3: registers capped at 85, 24 resident warps per SM

// exact by default; 1 = mixed FHFMA (opt-in, see Io<__half, 1>). Atomic: enqueue may be called from several host
// threads (SURVEY §8(b) threading), the setter from another.
static std::atomic<int> g_f16_mode{0};
// FP16 kernel selection: 0 (default) = this file's round-1 gather kernel everywhere, 1 (opt-in, measured slower) =
// resident-tail kernel (msda_res.cu) where its envelope holds.
static std::atomic<int> g_f16_path{0};
static std::atomic<int> g_res_cap_bytes{128 * 1024};
// Launch shape of the FP32 / FP16 plugin op, encoded as units | strided << 8. units: 1 = one block of items per CTA
// (round-1 grid), 2 / 4 = batched launch with the visibility scan (see msda_gather_kernel); strided: where the units of
// a CTA lie. -1 = not decided yet: the first launch reads the environment variable B200_MSDA_BATCH ("1", "2", "4",
// "2s", "4s"), else kDefaultBatch. b200_msda_set_batch_units overrides.
constexpr int kDefaultBatch = 1;
// Gather-depth variant of the same launch (one-unit grid only): 0 = default (3 CTAs per SM, one point = 4 tap loads in
// flight per warp), 1 = 2 CTAs per SM (128-register budget, same source: the compiler keeps a chunk's 16 tap loads in
// flight), 2 = the same with the 16 loads written before the FMAs in the source, 3 = 128-thread CTAs, 5 per SM (20 warps,
// 96 registers: the point in between). Initial value: environment variable B200_MSDA_VARIANT ("0" .. "3"), else 0.
static std::atomic<int> g_gather_variant{-1};
static int msda_gather_variant() {
  int v = g_gather_variant.load(std::memory_order_relaxed);
  if (v < 0) {
    const char *e = getenv("B200_MSDA_VARIANT");
    v = (e != nullptr && e[0] >= '0' && e[0] <= '3' && e[1] == '\0') ? e[0] - '0' : 0;
    g_gather_variant.store(v, std::memory_order_relaxed);
  }
  return v;
}
static std::atomic<int> g_batch_units{-1};
static int msda_batch_units() {
  int v = g_batch_units.load(std::memory_order_relaxed);
  if (v < 0) {
    const char *e = getenv("B200_MSDA_BATCH");
    v = kDefaultBatch;
    if (e != nullptr && (e[0] == '1' || e[0] == '2' || e[0] == '4')) {
      if (e[1] == '\0') v = e[0] - '0';
      else if (e[1] == 's' && e[2] == '\0' && e[0] != '1') v = (e[0] - '0') | 0x100;
    }
    g_batch_units.store(v, std::memory_order_relaxed);
  }
  return v;
}

struct MsdaParams {
  const void *value;
  const int32_t *shapes;
  const void *ref;
  const void *off;
  const void *logits;
  void *out;
  int B, S, M, C, L, Q, P, G;
  long long items;
  int ref_is_half;  // int8 path: dtype of reference_points
  // fused spatial-cross-attention epilogue (EPI = 1): accum[q, m*C + c] += bev_mask[b, q] * out[b, q, m, c]
  // camera-loop form (EPI = 2): items are (q, head); offsets / logits are [Q, M, ...] shared by all B cameras (the
  // reference repeats the query per camera, spatial_cross_attention.py:254); accum[q, m*C + c] = sum_b ... (plain store)
  const float *mask;
  float *accum;
  float scale_value, scale_offset, scale_weight, scale_out;
  int4 *trace;  // DBG instantiations: per (item, point) sampling-index record {in_range, h_low, w_low, tap_mask}
  int unit_stride;  // batched launch (UPW > 1): 0 = a CTA's units are consecutive blocks, 1 = a grid apart
};

// ---------------------------------------------------------------------------------------------------------------
// Per-dtype I/O. A lane moves one vector of channels per tap: 4 floats / 8 halves (16 B) or 8 int8 (8 B).
//   Wt  = number of 32-bit registers that carry the four tap weights of a point from the owner lane:
//         4 (fp32 weights) or 2 (fp16 pairs, for the FHFMA paths).
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 ffma2(float2 a, float w, float2 c) {
  // two IEEE fp32 FMAs (the pairwise form of the accumulation; each lane rounds once)
  return make_float2(fmaf(a.x, w, c.x), fmaf(a.y, w, c.y));
}

template <typename T, int MODE>
struct Io;

template <int MODE>
struct Io<float, MODE> {
  static constexpr int kVec = 4, kWt = 4;
  using Tap = uint4;
  __device__ static Tap ld(const char *p) { return ldg128(p); }
  __device__ static void store_zero(float *p) { stg128_stream(p, make_uint4(0u, 0u, 0u, 0u)); }
  __device__ static void load_off4(const float *p, float, float (&ox)[4], float (&oy)[4]) {
    const uint4 a = ldg128_stream(p), b = ldg128_stream(p + 4);
    ox[0] = __uint_as_float(a.x), oy[0] = __uint_as_float(a.y), ox[1] = __uint_as_float(a.z),
    oy[1] = __uint_as_float(a.w);
    ox[2] = __uint_as_float(b.x), oy[2] = __uint_as_float(b.y), ox[3] = __uint_as_float(b.z),
    oy[3] = __uint_as_float(b.w);
  }
  // visibility scan (UPW > 1): the same two loads as load_off4, issued for several units before any is decoded
  struct OffRaw {
    uint4 a, b;
  };
  __device__ static OffRaw ld_off_raw(const float *p) { return OffRaw{ldg128_stream(p), ldg128_stream(p + 4)}; }
  __device__ static void decode_off(const OffRaw &w, float, float (&ox)[4], float (&oy)[4]) {
    ox[0] = __uint_as_float(w.a.x), oy[0] = __uint_as_float(w.a.y), ox[1] = __uint_as_float(w.a.z),
    oy[1] = __uint_as_float(w.a.w);
    ox[2] = __uint_as_float(w.b.x), oy[2] = __uint_as_float(w.b.y), ox[3] = __uint_as_float(w.b.z),
    oy[3] = __uint_as_float(w.b.w);
  }
  __device__ static void load_lg4(const float *p, float, float (&lg)[4]) {
    const uint4 a = ldg128_stream(p);
    lg[0] = __uint_as_float(a.x), lg[1] = __uint_as_float(a.y), lg[2] = __uint_as_float(a.z),
    lg[3] = __uint_as_float(a.w);
  }
  __device__ static void pack_w(float (&o)[4], float w00, float w01, float w10, float w11) {
    o[0] = w00, o[1] = w01, o[2] = w10, o[3] = w11;
  }
  __device__ static void fma_point(float (&acc)[4], const Tap (&t)[4], const float (&w)[4]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float2 *a2 = reinterpret_cast<float2 *>(acc);
      a2[0] = ffma2(make_float2(__uint_as_float(t[k].x), __uint_as_float(t[k].y)), w[k], a2[0]);
      a2[1] = ffma2(make_float2(__uint_as_float(t[k].z), __uint_as_float(t[k].w)), w[k], a2[1]);
    }
  }
  __device__ static void store(float *p, const float (&acc)[4], float inv_sum, const MsdaParams &) {
    stg128_stream(p, make_uint4(__float_as_uint(acc[0] * inv_sum), __float_as_uint(acc[1] * inv_sum),
                                __float_as_uint(acc[2] * inv_sum), __float_as_uint(acc[3] * inv_sum)));
  }
};

// MODE 0: exact — taps widened to fp32 (HADD2.F32), fp32 weights, FFMA2.
// MODE 1: mixed — fp16 weights, FHFMA (fp16 x fp16 + fp32 -> fp32, one rounding). Faster, but the 2^-11 relative
//         rounding of the weights costs up to ~3e-4 absolute on O(1) outputs: opt-in only (b200_msda_set_f16_mode).
template <int MODE>
struct Io<__half, MODE> {
  static constexpr int kVec = 8, kWt = MODE == 1 ? 2 : 4;
  using Tap = uint4;
  __device__ static Tap ld(const char *p) { return ldg128(p); }
  __device__ static void store_zero(__half *p) { stg128_stream(p, make_uint4(0u, 0u, 0u, 0u)); }
  __device__ static void load_off4(const __half *p, float, float (&ox)[4], float (&oy)[4]) {
    const uint4 a = ldg128_stream(p);
    const float2 p0 = h2_to_f2(a.x), p1 = h2_to_f2(a.y), p2 = h2_to_f2(a.z), p3 = h2_to_f2(a.w);
    ox[0] = p0.x, oy[0] = p0.y, ox[1] = p1.x, oy[1] = p1.y, ox[2] = p2.x, oy[2] = p2.y, ox[3] = p3.x, oy[3] = p3.y;
  }
  using OffRaw = uint4;
  __device__ static OffRaw ld_off_raw(const __half *p) { return ldg128_stream(p); }
  __device__ static void decode_off(const OffRaw &a, float, float (&ox)[4], float (&oy)[4]) {
    const float2 p0 = h2_to_f2(a.x), p1 = h2_to_f2(a.y), p2 = h2_to_f2(a.z), p3 = h2_to_f2(a.w);
    ox[0] = p0.x, oy[0] = p0.y, ox[1] = p1.x, oy[1] = p1.y, ox[2] = p2.x, oy[2] = p2.y, ox[3] = p3.x, oy[3] = p3.y;
  }
  __device__ static void load_lg4(const __half *p, float, float (&lg)[4]) {
    const uint2 a = ldg64_stream(p);
    const float2 p0 = h2_to_f2(a.x), p1 = h2_to_f2(a.y);
    lg[0] = p0.x, lg[1] = p0.y, lg[2] = p1.x, lg[3] = p1.y;
  }
  __device__ static void pack_w(float (&o)[kWt], float w00, float w01, float w10, float w11) {
    if (MODE == 1) {
      o[0] = __uint_as_float(f2_to_h2(w00, w01)), o[1] = __uint_as_float(f2_to_h2(w10, w11));
    } else {
      o[0] = w00, o[1] = w01, o[kWt - 2] = w10, o[kWt - 1] = w11;
    }
  }
  __device__ static void fma_point(float (&acc)[8], const Tap (&t)[4], const float (&w)[kWt]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t u[4] = {t[k].x, t[k].y, t[k].z, t[k].w};
      if (MODE == 1) {
        const uint32_t wp = __float_as_uint(w[k >> 1]);
        const unsigned short wh = static_cast<unsigned short>((k & 1) ? (wp >> 16) : (wp & 0xffffu));
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          acc[2 * i] = fma_f32_f16(static_cast<unsigned short>(u[i] & 0xffffu), wh, acc[2 * i]);
          acc[2 * i + 1] = fma_f32_f16(static_cast<unsigned short>(u[i] >> 16), wh, acc[2 * i + 1]);
        }
      } else {
        float2 *a2 = reinterpret_cast<float2 *>(acc);
#pragma unroll
        for (int i = 0; i < 4; ++i) a2[i] = ffma2(h2_to_f2(u[i]), w[k < kWt ? k : 0], a2[i]);
      }
    }
  }
  __device__ static void store(__half *p, const float (&acc)[8], float inv_sum, const MsdaParams &) {
    stg128_stream(p, make_uint4(f2_to_h2(acc[0] * inv_sum, acc[1] * inv_sum), f2_to_h2(acc[2] * inv_sum, acc[3] * inv_sum),
                                f2_to_h2(acc[4] * inv_sum, acc[5] * inv_sum),
                                f2_to_h2(acc[6] * inv_sum, acc[7] * inv_sum)));
  }
};

// BF16: FP16's lane layout (8 channels = 16 B per lane) and FP16's exact MODE 0 arithmetic: every bf16 word is widened
// to fp32 exactly (bf2_to_f2: a shift and a mask), fp32 weights, FFMA2, one rounding of the result. No mixed mode.
template <int MODE>
struct Io<__nv_bfloat16, MODE> {
  static_assert(MODE == 0, "BF16 has the exact mode only");
  static constexpr int kVec = 8, kWt = 4;
  using Tap = uint4;
  __device__ static Tap ld(const char *p) { return ldg128(p); }
  __device__ static void store_zero(__nv_bfloat16 *p) { stg128_stream(p, make_uint4(0u, 0u, 0u, 0u)); }
  using OffRaw = uint4;
  __device__ static OffRaw ld_off_raw(const __nv_bfloat16 *p) { return ldg128_stream(p); }
  __device__ static void decode_off(const OffRaw &a, float, float (&ox)[4], float (&oy)[4]) {
    const float2 p0 = bf2_to_f2(a.x), p1 = bf2_to_f2(a.y), p2 = bf2_to_f2(a.z), p3 = bf2_to_f2(a.w);
    ox[0] = p0.x, oy[0] = p0.y, ox[1] = p1.x, oy[1] = p1.y, ox[2] = p2.x, oy[2] = p2.y, ox[3] = p3.x, oy[3] = p3.y;
  }
  __device__ static void load_off4(const __nv_bfloat16 *p, float s, float (&ox)[4], float (&oy)[4]) {
    decode_off(ldg128_stream(p), s, ox, oy);
  }
  __device__ static void load_lg4(const __nv_bfloat16 *p, float, float (&lg)[4]) {
    const uint2 a = ldg64_stream(p);
    const float2 p0 = bf2_to_f2(a.x), p1 = bf2_to_f2(a.y);
    lg[0] = p0.x, lg[1] = p0.y, lg[2] = p1.x, lg[3] = p1.y;
  }
  __device__ static void pack_w(float (&o)[4], float w00, float w01, float w10, float w11) {
    o[0] = w00, o[1] = w01, o[2] = w10, o[3] = w11;
  }
  __device__ static void fma_point(float (&acc)[8], const Tap (&t)[4], const float (&w)[4]) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t u[4] = {t[k].x, t[k].y, t[k].z, t[k].w};
      float2 *a2 = reinterpret_cast<float2 *>(acc);
#pragma unroll
      for (int i = 0; i < 4; ++i) a2[i] = ffma2(bf2_to_f2(u[i]), w[k], a2[i]);
    }
  }
  __device__ static void store(__nv_bfloat16 *p, const float (&acc)[8], float inv_sum, const MsdaParams &) {
    stg128_stream(p, make_uint4(f2_to_bf2(acc[0] * inv_sum, acc[1] * inv_sum), f2_to_bf2(acc[2] * inv_sum, acc[3] * inv_sum),
                                f2_to_bf2(acc[4] * inv_sum, acc[5] * inv_sum),
                                f2_to_bf2(acc[6] * inv_sum, acc[7] * inv_sum)));
  }
};

// INT8: 8 channels (8 bytes) per lane, 4 lanes per item like FP16 — same ownership structure, half the tap bytes.
// Taps are dequantised in registers. int8 -> fp16 is exact (|q| <= 128): flip the sign bit, splice each byte under the
// exponent byte 0x64 (= 1024 + byte as fp16) with PRMT, subtract 1152 with one packed HADD2 per pair. The product with
// the fp16 tap weight is accumulated in fp32 by FHFMA; the fp16 weight rounding (2^-11 relative) is two orders of
// magnitude below the INT8 output step. scale_value is applied once, at the requantisation.
template <int MODE>
struct Io<int8_t, MODE> {
  static constexpr int kVec = 8, kWt = 2;
  using Tap = uint2;
  __device__ static Tap ld(const char *p) { return ldg64(p); }
  __device__ static void store_zero(int8_t *p) {
    asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(0u), "r"(0u) : "memory");
  }
  __device__ static float deq(uint32_t word, int byte, float s) {
    return static_cast<float>(static_cast<int8_t>(word >> (8 * byte))) * s;
  }
  // off*scale is rounded to fp32 first, then fused with ref*size — as in the reference INT8 kernel (…Kernel.cu:916-921)
  __device__ static void load_off4(const int8_t *p, float s, float (&ox)[4], float (&oy)[4]) {
    const uint2 a = ldg64_stream(p);
    ox[0] = deq(a.x, 0, s), oy[0] = deq(a.x, 1, s), ox[1] = deq(a.x, 2, s), oy[1] = deq(a.x, 3, s);
    ox[2] = deq(a.y, 0, s), oy[2] = deq(a.y, 1, s), ox[3] = deq(a.y, 2, s), oy[3] = deq(a.y, 3, s);
  }
  __device__ static void load_lg4(const int8_t *p, float s, float (&lg)[4]) {
    const uint32_t a = ldg32_stream(p);
    lg[0] = deq(a, 0, s), lg[1] = deq(a, 1, s), lg[2] = deq(a, 2, s), lg[3] = deq(a, 3, s);
  }
  __device__ static void pack_w(float (&o)[2], float w00, float w01, float w10, float w11) {
    o[0] = __uint_as_float(f2_to_h2(w00, w01)), o[1] = __uint_as_float(f2_to_h2(w10, w11));
  }
  __device__ static void fma_point(float (&acc)[8], const Tap (&t)[4], const float (&w)[2]) {
    const __half2 bias = __floats2half2_rn(1152.f, 1152.f);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t wp = __float_as_uint(w[k >> 1]);
      const unsigned short wh = static_cast<unsigned short>((k & 1) ? (wp >> 16) : (wp & 0xffffu));
      const uint32_t u[2] = {t[k].x, t[k].y};
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const uint32_t x = u[i] ^ 0x80808080u;
        uint32_t lo = __byte_perm(x, 0x64646464u, 0x4140), hi = __byte_perm(x, 0x64646464u, 0x4342);
        const __half2 a = __hsub2(*reinterpret_cast<__half2 *>(&lo), bias);
        const __half2 b = __hsub2(*reinterpret_cast<__half2 *>(&hi), bias);
        const uint32_t ua = *reinterpret_cast<const uint32_t *>(&a), ub = *reinterpret_cast<const uint32_t *>(&b);
        acc[4 * i + 0] = fma_f32_f16(static_cast<unsigned short>(ua & 0xffffu), wh, acc[4 * i + 0]);
        acc[4 * i + 1] = fma_f32_f16(static_cast<unsigned short>(ua >> 16), wh, acc[4 * i + 1]);
        acc[4 * i + 2] = fma_f32_f16(static_cast<unsigned short>(ub & 0xffffu), wh, acc[4 * i + 2]);
        acc[4 * i + 3] = fma_f32_f16(static_cast<unsigned short>(ub >> 16), wh, acc[4 * i + 3]);
      }
    }
  }
  __device__ static void store(int8_t *p, const float (&acc)[8], float inv_sum, const MsdaParams &prm) {
    // real = acc * scale_value / sum ; q = T2int8(real / scale_out)
    const float mul = prm.scale_value * inv_sum / prm.scale_out;
    uint32_t o[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      uint32_t word = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        word |= (static_cast<uint32_t>(to_int8_sat(acc[4 * i + j] * mul)) & 0xffu) << (8 * j);
      o[i] = word;
    }
    asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(o[0]), "r"(o[1]) : "memory");
  }
};

template <typename R>
__device__ __forceinline__ float ref_to_float(const R *p, long long i);
template <>
__device__ __forceinline__ float ref_to_float<float>(const float *p, long long i) {
  return __ldg(p + i);
}
template <>
__device__ __forceinline__ float ref_to_float<__half>(const __half *p, long long i) {
  return __half2float(__ldg(p + i));
}

// Reference points of one (batch, query) for the four points of a chunk: point k of a chunk uses group k % G
// (G in {1,2,4}; P % 4 == 0), so px[k], py[k] are filled once and indexed with compile-time k (no local memory).
template <typename R>
__device__ __forceinline__ void load_ref(const R *p, int G, float (&px)[4], float (&py)[4]);
template <>
__device__ __forceinline__ void load_ref<__half>(const __half *p, int G, float (&px)[4], float (&py)[4]) {
  if (G == 4) {
    const uint4 a = ldg128(p);
    const float2 f0 = h2_to_f2(a.x), f1 = h2_to_f2(a.y), f2 = h2_to_f2(a.z), f3 = h2_to_f2(a.w);
    px[0] = f0.x, py[0] = f0.y, px[1] = f1.x, py[1] = f1.y, px[2] = f2.x, py[2] = f2.y, px[3] = f3.x, py[3] = f3.y;
  } else if (G == 2) {
    const uint2 a = ldg64(p);
    const float2 f0 = h2_to_f2(a.x), f1 = h2_to_f2(a.y);
    px[0] = px[2] = f0.x, py[0] = py[2] = f0.y, px[1] = px[3] = f1.x, py[1] = py[3] = f1.y;
  } else {
    const float2 f0 = h2_to_f2(ldg32(p));
    px[0] = px[1] = px[2] = px[3] = f0.x, py[0] = py[1] = py[2] = py[3] = f0.y;
  }
}
template <>
__device__ __forceinline__ void load_ref<float>(const float *p, int G, float (&px)[4], float (&py)[4]) {
  if (G == 4) {
    const uint4 a = ldg128(p), b = ldg128(p + 4);
    px[0] = __uint_as_float(a.x), py[0] = __uint_as_float(a.y), px[1] = __uint_as_float(a.z), py[1] = __uint_as_float(a.w);
    px[2] = __uint_as_float(b.x), py[2] = __uint_as_float(b.y), px[3] = __uint_as_float(b.z), py[3] = __uint_as_float(b.w);
  } else if (G == 2) {
    const uint4 a = ldg128(p);
    px[0] = px[2] = __uint_as_float(a.x), py[0] = py[2] = __uint_as_float(a.y);
    px[1] = px[3] = __uint_as_float(a.z), py[1] = py[3] = __uint_as_float(a.w);
  } else {
    const uint2 a = ldg64(p);
    px[0] = px[1] = px[2] = px[3] = __uint_as_float(a.x), py[0] = py[1] = py[2] = py[3] = __uint_as_float(a.y);
  }
}

// The same reference-point words as load_ref, split into "issue the load" and "decode" so that the visibility scan of a
// batched launch (UPW > 1) can put the loads of several units in flight before the first one is consumed. The raw
// words are replicated so that decode is the G == 4 pattern whatever G is (G = 2: {p0, p1, p0, p1}; G = 1: p0 four times).
template <typename R>
struct RefRaw;
template <>
struct RefRaw<__half> {
  uint4 a;
  __device__ __forceinline__ void load4(const __half *p) { a = ldg128(p); }
  __device__ __forceinline__ void load2(const __half *p) {
    const uint2 t = ldg64(p);
    a = make_uint4(t.x, t.y, t.x, t.y);
  }
  __device__ __forceinline__ void load1(const __half *p) {
    const uint32_t t = ldg32(p);
    a = make_uint4(t, t, t, t);
  }
  __device__ __forceinline__ void decode(float (&px)[4], float (&py)[4]) const {
    const float2 f0 = h2_to_f2(a.x), f1 = h2_to_f2(a.y), f2 = h2_to_f2(a.z), f3 = h2_to_f2(a.w);
    px[0] = f0.x, py[0] = f0.y, px[1] = f1.x, py[1] = f1.y, px[2] = f2.x, py[2] = f2.y, px[3] = f3.x, py[3] = f3.y;
  }
};
template <>
struct RefRaw<float> {
  uint4 a, b;
  __device__ __forceinline__ void load4(const float *p) { a = ldg128(p), b = ldg128(p + 4); }
  __device__ __forceinline__ void load2(const float *p) { a = ldg128(p), b = a; }
  __device__ __forceinline__ void load1(const float *p) {
    const uint2 t = ldg64(p);
    a = make_uint4(t.x, t.y, t.x, t.y), b = a;
  }
  __device__ __forceinline__ void decode(float (&px)[4], float (&py)[4]) const {
    px[0] = __uint_as_float(a.x), py[0] = __uint_as_float(a.y), px[1] = __uint_as_float(a.z), py[1] = __uint_as_float(a.w);
    px[2] = __uint_as_float(b.x), py[2] = __uint_as_float(b.y), px[3] = __uint_as_float(b.z), py[3] = __uint_as_float(b.w);
  }
};

// ---------------------------------------------------------------------------------------------------------------
// Main kernel. T = storage type of value/offsets/logits/out, R = storage type of reference points.
// Requirements checked on the host: LPI = C*sizeof(T)/16 in {1,2,4,8,16,32}, P % 4 == 0, G in {1,2,4},
// ceil(NP/4 / LPI) <= ROUNDS, NP/4 <= kMaxChunks, (S + 1) * M * C * sizeof(T) < 2^31, 16-byte aligned tensors.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kMaxChunks = 64;

// What a sampling point outside every image loads in the gather kernel (one tap vector of zeros, never written).
__device__ const uint4 g_msda_zero_tap = {0u, 0u, 0u, 0u};

//
// UPW ("units per warp", plugin-op form EPI = 0 only) > 1 is the batched launch: a CTA covers UPW consecutive blocks of
// IPB items and each warp walks UPW units (unit u of warp w = the 32/LPI items at item0 + u*IPB + w*IPW, the same item
// groups as the UPW = 1 grid, so results are bit-identical). Before the walk the warp runs a VISIBILITY SCAN: the
// offsets and reference points of all its UPW units are loaded back to back (raw words, nothing decoded until every
// load is issued) and phase A's range test is evaluated per unit. Units no point of which lands in an image — 4 of 5 on
// a camera ring — are answered with zeros straight away; their memory latencies overlap instead of each costing a
// CTA slot one full DRAM round trip (the UPW = 1 grid spends ~4 k cycles of a CTA slot per invisible block). Visible
// units run the unchanged body below (which re-reads its 2 offset vectors per lane from L2).
//
// MINB / PIF ("points in flight") are the gather-depth variants (b200_msda_set_gather_variant). At the default register
// cap (85: 3 CTAs = 24 warps per SM) the compiler rotates four 16-byte tap buffers, i.e. ONE point = 4 tap loads are in
// flight per warp (SASS: each LDG.E.128 is consumed ~70 instructions after it issues). On camera-ring inputs the kernel
// is latency-bound (ncu: issue 57 %, L1 58 %, long-scoreboard stalls dominant), so the variants trade warps for loads
// per warp: MINB = 2 lifts the cap to 128 registers (16 warps per SM) and ptxas then hoists all 16 tap loads of a 4-point
// chunk above the first FMA by itself (126 registers, no spills; PIF = 2 compiles to the same code and is not
// instantiated); PIF = 4 states that order in the source. 16 warps x 16 loads against 24 x 4 in flight per SM. The FMA
// order is unchanged, so every variant returns the same bits.
// NT = threads per CTA: warps never synchronise with each other and there is no shared memory, so a CTA is only a
// scheduling and register-allocation unit; NT = 128 with MINB = 5 is the middle point (20 warps per SM, 96 registers).
template <typename T, typename R, int C, int ROUNDS, int MODE, int EPI, bool DBG = false, int UPW = 1, int MINB = kMinBlocks,
          int PIF = 1, int NT = kThreads>
__global__ void __launch_bounds__(NT, MINB) msda_gather_kernel(const MsdaParams prm) {
  static_assert(NT % 32 == 0 && NT >= 32 && NT <= 1024, "whole warps");
  static_assert(UPW == 1 || EPI == 0, "the batched launch exists for the plugin-op form only");
  static_assert(PIF == 1 || PIF == 2 || PIF == 4, "points in flight: 1, 2 or 4 of a chunk's 4 points");
  static_assert(UPW >= 1 && UPW <= 8, "visibility bits live in one register");
  using IO = Io<T, MODE>;
  constexpr int VEC = IO::kVec;
  constexpr int LPI = C / VEC;
  constexpr int IPW = 32 / LPI;
  constexpr int IPB = IPW * (NT / 32);
  constexpr int NW = IO::kWt;
  // lanes whose sub-index is 0 (one per item of the warp); shifted by j it selects the owner lanes j
  constexpr unsigned OWNER0 = LPI == 1 ? 0xffffffffu
                              : LPI == 2 ? 0x55555555u
                              : LPI == 4 ? 0x11111111u
                              : LPI == 8 ? 0x01010101u
                              : LPI == 16 ? 0x00010001u
                                          : 0x00000001u;

  const int M = prm.M, Q = prm.Q, P = prm.P, G = prm.G, L = prm.L;
  const int NP = L * P, NCH = NP >> 2, CPL = P >> 2;  // chunks (4 points) in total / per level
  constexpr int IPB_ = IPB;
  // Block of IPB items a unit stands for: unit u of CTA x is block x*UPW + u (consecutive: a CTA covers UPW*IPB
  // neighbouring items) or block x + u*gridDim.x (prm.unit_stride: the units of a CTA are a grid apart, so visible and
  // invisible units mix inside every CTA and CTA run times even out). The host only takes UPW > 1 when IPB % M == 0,
  // so unit u's (batch, query) is bq0 + u * ustep * (IPB / M) and the head index m is the same for every unit.
  long long blk0 = blockIdx.x, ustep = 1;
  if constexpr (UPW > 1) {
    if (prm.unit_stride) ustep = gridDim.x;
    else blk0 *= UPW;
  }
  const long long item0 = blk0 * IPB_;

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int sub = lane % LPI;
  // unit 0 of this warp; the unit loop below re-derives these for u > 0 (UPW > 1 only)
  const long long it_raw = item0 + warp * IPW + lane / LPI;
  bool active = it_raw < prm.items;
  long long it = active ? it_raw : prm.items - 1;  // inactive lanes shadow the last item, never store
  long long bq0 = it / M;  // EPI < 2: b * Q + q; EPI == 2: q
  const int m = static_cast<int>(it - bq0 * M);
  const T *off_item = static_cast<const T *>(prm.off) + it * NP * 2;
  const T *lg_item = static_cast<const T *>(prm.logits) + it * NP;
  T *out_item = static_cast<T *>(prm.out) + it * C + sub * VEC;

  if (EPI == 1) {
    // Fused SCA epilogue: a (camera, query) pair with bev_mask == 0 contributes exactly nothing, whatever it samples.
    // When that holds for every item of the warp (one query x 8 heads share the mask value) nothing is read at all —
    // for a camera ring about 4 of 5 warps leave here.
    const float mk0 = __ldg(prm.mask + bq0);
    if (__ballot_sync(kFullMask, active && mk0 != 0.f) == 0u) return;
  }

  // Level table, per warp and without any block barrier: lane l < L holds (H_l, W_l) and the exclusive prefix sum of
  // H*W (the level's first pixel); consumers fetch their level's entry with shuffles. All global loads of the prologue
  // (shapes, reference points, offsets) are independent, so a warp pays one memory latency before it can decide whether
  // anything it owns is visible at all.
  int lvH = 1, lvW = 1;
  if (lane < L) {
    const int2 hw = __ldg(reinterpret_cast<const int2 *>(prm.shapes) + lane);
    lvH = hw.x, lvW = hw.y;
  }
  int lvStart;
  {
    const int area = lane < L ? lvH * lvW : 0;
    int incl = area;
#pragma unroll
    for (int d = 1; d < kMaxLevels; d <<= 1) {
      const int t = __shfl_up_sync(kFullMask, incl, d);
      if (lane >= d) incl += t;
    }
    lvStart = incl - area;
  }

  // ---- visibility scan (batched launch): bit u of vis = some point of some ACTIVE item of unit u is in range
  unsigned vis = 1u;
  if constexpr (UPW > 1) {
    typename IO::OffRaw oraw[UPW][ROUNDS];
    RefRaw<R> rraw[UPW];
    bool act[UPW];
#pragma unroll
    for (int u = 0; u < UPW; ++u) {
      const long long itr = it_raw + u * ustep * IPB_;
      act[u] = itr < prm.items;
      const long long itu = act[u] ? itr : it;  // units past the end shadow unit 0's item (valid address; act[] gates them)
      const T *offu = static_cast<const T *>(prm.off) + itu * NP * 2;
#pragma unroll
      for (int r = 0; r < ROUNDS; ++r) {
        const int c = r * LPI + sub;
        oraw[u][r] = IO::ld_off_raw(offu + (c < NCH ? c : 0) * 8);
      }
    }
    long long bqu[UPW];
#pragma unroll
    for (int u = 0; u < UPW; ++u) bqu[u] = act[u] ? bq0 + u * ustep * (IPB_ / M) : bq0;
    const R *refp = static_cast<const R *>(prm.ref);
    if (G == 4) {
#pragma unroll
      for (int u = 0; u < UPW; ++u) rraw[u].load4(refp + bqu[u] * 8);
    } else if (G == 2) {
#pragma unroll
      for (int u = 0; u < UPW; ++u) rraw[u].load2(refp + bqu[u] * 4);
    } else {
#pragma unroll
      for (int u = 0; u < UPW; ++u) rraw[u].load1(refp + bqu[u] * 2);
    }
    vis = 0u;
#pragma unroll
    for (int u = 0; u < UPW; ++u) {
      float spx[4], spy[4];
      rraw[u].decode(spx, spy);
      bool any = false;
#pragma unroll
      for (int r = 0; r < ROUNDS; ++r) {
        const int c = r * LPI + sub;
        const bool have = c < NCH;
        const int lv = (have ? c : 0) / CPL;
        const int H = __shfl_sync(kFullMask, lvH, lv), W = __shfl_sync(kFullMask, lvW, lv);
        float ox[4], oy[4];
        IO::decode_off(oraw[u][r], prm.scale_offset, ox, oy);
#pragma unroll
        for (int k = 0; k < 4; ++k) {  // the statement of phase A below, word for word
          const float w_im = __fadd_rn(__fmaf_rn(spx[k], static_cast<float>(W), ox[k]), -0.5f);
          const float h_im = __fadd_rn(__fmaf_rn(spy[k], static_cast<float>(H), oy[k]), -0.5f);
          any |= have && h_im > -1.f && w_im > -1.f && h_im < static_cast<float>(H) && w_im < static_cast<float>(W);
        }
      }
      if (__ballot_sync(kFullMask, act[u] && any) != 0u) vis |= 1u << u;
    }
  }

  const long long it_first = it, bq_first = bq0;  // unit 0 (clamped), the base the later units derive from
#pragma unroll 1
  for (int u = 0; u < UPW; ++u) {
  if constexpr (UPW > 1) {
    if (u > 0) {
      const long long itr = it_raw + u * ustep * IPB_;
      active = itr < prm.items;
      it = active ? itr : it_first;  // lane groups past the end shadow unit 0's item, never store
      out_item = static_cast<T *>(prm.out) + it * C + sub * VEC;
    }
    if (((vis >> u) & 1u) == 0u) {  // warp-uniform
      if (active) IO::store_zero(out_item);
      continue;
    }
    if (u > 0) {
      bq0 = active ? bq_first + u * ustep * (IPB_ / M) : bq_first;
      off_item = static_cast<const T *>(prm.off) + it * NP * 2;
      lg_item = static_cast<const T *>(prm.logits) + it * NP;
    }
  }
  bool zero_stored = false;  // batched launch: phase A's own early-out fired (it cannot after a positive scan, but stays correct)
  float lg[ROUNDS][4];
  float sum = 0.f;
  bool have_sm = false;  // warp-uniform
  unsigned inr = 0;      // bit r*4+k: point in range (…Kernel.cu:674)
  float acc[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) acc[i] = 0.f;

  const int num_b = EPI == 2 ? prm.B : 1;
  for (int bi = 0; bi < num_b; ++bi) {
  const int b = EPI == 2 ? bi : static_cast<int>(bq0 / Q);
  const long long bq = EPI == 2 ? static_cast<long long>(bi) * Q + bq0 : bq0;
  float mk = 1.f;
  if (EPI == 2) {
    mk = __ldg(prm.mask + bq);
    if (__ballot_sync(kFullMask, active && mk != 0.f) == 0u) continue;  // this camera sees none of the warp's queries
  }
  // Reference points of this item's (batch, query): 2G values, the same for every head (and every lane group that
  // shares the query) — a broadcast load.
  float rpx[4], rpy[4];
  load_ref<R>(static_cast<const R *>(prm.ref) + bq * 2 * G, G, rpx, rpy);

  // ---- phase A: sampling positions of the points this lane owns (chunk c = r*LPI + sub), the bit-exact part
  float him[ROUNDS][4], wim[ROUNDS][4];
  inr = 0;
#pragma unroll
  for (int r = 0; r < ROUNDS; ++r) {
    const int c = r * LPI + sub;
    const bool have = c < NCH && (EPI != 2 || mk != 0.f);
    const int cc = have ? c : 0;
    const int lv = cc / CPL;
    const int H = __shfl_sync(kFullMask, lvH, lv), W = __shfl_sync(kFullMask, lvW, lv);
    float ox[4], oy[4];
    IO::load_off4(off_item + cc * 8, prm.scale_offset, ox, oy);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      wim[r][k] = __fadd_rn(__fmaf_rn(rpx[k], static_cast<float>(W), ox[k]), -0.5f);
      him[r][k] = __fadd_rn(__fmaf_rn(rpy[k], static_cast<float>(H), oy[k]), -0.5f);
      const bool ok = have && him[r][k] > -1.f && wim[r][k] > -1.f && him[r][k] < static_cast<float>(H) &&
                      wim[r][k] < static_cast<float>(W);
      inr |= ok ? (1u << (r * 4 + k)) : 0u;
    }
  }
  // Nothing of this warp's items lands inside any image (a camera that does not see these BEV queries): the result
  // is exactly 0 (= 0 / sum), and logits are never read.
  if (__ballot_sync(kFullMask, inr != 0u) == 0u) {
    if (EPI == 2) continue;                            // next camera
    if (EPI == 0 && active) IO::store_zero(out_item);  // the fused epilogue adds nothing for invisible items
    if constexpr (UPW == 1) {
      return;
    } else {
      zero_stored = true;
      break;
    }
  }

  // ---- phase B: softmax statistics over the item's NP logits (…Kernel.cu:642-648, :667-669); camera-independent,
  // so the camera-loop form computes them when the first camera that sees the warp's queries turns up
  if (EPI != 2 || !have_sm) {
  have_sm = true;
  float mx = -INFINITY;
#pragma unroll
  for (int r = 0; r < ROUNDS; ++r) {
    const int c = r * LPI + sub;
    if (c < NCH) {
      IO::load_lg4(lg_item + c * 4, prm.scale_weight, lg[r]);
    } else {
      lg[r][0] = lg[r][1] = lg[r][2] = lg[r][3] = -INFINITY;
    }
    mx = fmaxf(mx, fmaxf(fmaxf(lg[r][0], lg[r][1]), fmaxf(lg[r][2], lg[r][3])));
  }
#pragma unroll
  for (int d = 1; d < LPI; d <<= 1) mx = fmaxf(mx, __shfl_xor_sync(kFullMask, mx, d));
  sum = 0.f;
#pragma unroll
  for (int r = 0; r < ROUNDS; ++r) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      lg[r][k] = expf(lg[r][k] - mx);  // exp(-inf) = 0 for the padding slots
      sum += lg[r][k];
    }
  }
#pragma unroll
  for (int d = 1; d < LPI; d <<= 1) sum += __shfl_xor_sync(kFullMask, sum, d);
  }

  // ---- phase C: gather
  const char *zeros = reinterpret_cast<const char *>(&g_msda_zero_tap);
  const unsigned step_b = static_cast<unsigned>(M * C) * sizeof(T);  // bytes between horizontally adjacent pixels
  const char *vbase = reinterpret_cast<const char *>(static_cast<const T *>(prm.value) +
                                                     (static_cast<long long>(b) * prm.S * M + m) * C + sub * VEC);

#pragma unroll
  for (int r = 0; r < ROUNDS; ++r) {
    if (r * LPI >= NCH) break;  // uniform
    // owner: per point, the byte offset of the top-left tap (bit 0 = "column step usable"), the byte offset of the
    // bottom-left tap, and the four tap weights = bilinear weight x softmax numerator x tap validity.
    unsigned otop[4], obot[4];
    float tw[4][NW];
    {
      const int c = r * LPI + sub;
      const int cc = c < NCH ? c : 0;
      const int lv = cc / CPL;
      const int H = __shfl_sync(kFullMask, lvH, lv), W = __shfl_sync(kFullMask, lvW, lv);
      const int start = __shfl_sync(kFullMask, lvStart, lv);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const bool ok = (inr >> (r * 4 + k)) & 1u;
        const float hf = floorf(him[r][k]), wf = floorf(wim[r][k]);
        const int h_low = ok ? static_cast<int>(hf) : 0, w_low = ok ? static_cast<int>(wf) : 0;
        const float lh = __fsub_rn(him[r][k], hf), lw = __fsub_rn(wim[r][k], wf);
        const int h0 = max(h_low, 0), w0 = max(w_low, 0);
        const bool t = h_low >= 0, bt = h_low + 1 <= H - 1, lf = w_low >= 0, rt = w_low + 1 <= W - 1;
        const unsigned top = ok ? static_cast<unsigned>(start + h0 * W + w0) * step_b : 0u;
        otop[k] = top | ((ok && lf && rt) ? 1u : 0u) | (ok ? 2u : 0u);  // tap offsets are multiples of 16 bytes
        obot[k] = top + ((ok && t && bt) ? static_cast<unsigned>(W) * step_b : 0u);
        const float hh = 1.f - lh, hw = 1.f - lw;
        const float e = EPI == 2 ? lg[r][k] * mk : lg[r][k];  // bev_mask folded into the tap weights
        IO::pack_w(tw[k], (ok && t && lf) ? hh * hw * e : 0.f, (ok && t && rt) ? hh * lw * e : 0.f,
                   (ok && bt && lf) ? lh * hw * e : 0.f, (ok && bt && rt) ? lh * lw * e : 0.f);
        if (DBG && active && c < NCH) {
          // the index record of THIS kernel's own arithmetic (parity tests compare it bit for bit with the oracle);
          // points the early-outs above never reach are out of range = the all-zero record the host pre-fills
          const int tm = ((t && lf) ? 1 : 0) | ((t && rt) ? 2 : 0) | ((bt && lf) ? 4 : 0) | ((bt && rt) ? 8 : 0);
          prm.trace[it * NP + c * 4 + k] = ok ? make_int4(1, h_low, w_low, tm) : make_int4(0, 0, 0, 0);
        }
      }
    }
    const unsigned vm = __ballot_sync(kFullMask, ((inr >> (r * 4)) & 0xfu) != 0u);

#pragma unroll
    for (int j = 0; j < LPI; ++j) {
      if (r * LPI + j >= NCH) break;             // uniform
      if ((vm & (OWNER0 << j)) == 0u) continue;  // uniform: chunk out of range for every item of the warp
      const int src = (lane & ~(LPI - 1)) | j;
      if constexpr (PIF > 1) {
#pragma unroll
        for (int k0 = 0; k0 < 4; k0 += PIF) {
          typename IO::Tap tp[PIF][4];
          float wp[PIF][NW];
#pragma unroll
          for (int i = 0; i < PIF; ++i) {  // addresses, weights and the 4 tap loads of PIF points first ...
            const unsigned ot = __shfl_sync(kFullMask, otop[k0 + i], src);
            const unsigned ob = __shfl_sync(kFullMask, obot[k0 + i], src);
#pragma unroll
            for (int n = 0; n < NW; ++n) wp[i][n] = __shfl_sync(kFullMask, tw[k0 + i][n], src);
            const unsigned dx = (ot & 1u) ? step_b : 0u;
            const char *base = (ot & 2u) ? vbase : zeros;  // see the note at the one-point form below
            const char *p0 = base + (ot & ~3u);
            const char *p1 = base + ob;
            tp[i][0] = IO::ld(p0), tp[i][1] = IO::ld(p0 + dx), tp[i][2] = IO::ld(p1), tp[i][3] = IO::ld(p1 + dx);
          }
#pragma unroll
          for (int i = 0; i < PIF; ++i) IO::fma_point(acc, tp[i], wp[i]);  // ... then the FMAs, in the default order
        }
        continue;
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const unsigned ot = __shfl_sync(kFullMask, otop[k], src);
        const unsigned ob = __shfl_sync(kFullMask, obot[k], src);
        float w[NW];
#pragma unroll
        for (int i = 0; i < NW; ++i) w[i] = __shfl_sync(kFullMask, tw[k][i], src);
        // A point in range whose neighbour is outside the image: the missing taps carry weight 0 and alias one of the
        // point's own in-image taps, so they add nothing that tap does not add already. A point out of range altogether
        // (bit 1 of ot clear; its offsets and weights are all 0) has no tap of its own to alias, and no element of value
        // may be assumed finite (0 * Inf is NaN): it reads 16 bytes of zeros instead, so it adds an exact 0 and the loop
        // stays free of branches.
        const unsigned dx = (ot & 1u) ? step_b : 0u;
        const char *base = (ot & 2u) ? vbase : zeros;
        const char *p0 = base + (ot & ~3u);
        const char *p1 = base + ob;
        const typename IO::Tap t[4] = {IO::ld(p0), IO::ld(p0 + dx), IO::ld(p1), IO::ld(p1 + dx)};
        IO::fma_point(acc, t, w);
      }
    }
  }

  }  // cameras

  if (EPI == 0) {
    if (active && !zero_stored) IO::store(out_item, acc, 1.f / sum, prm);
  } else if (EPI == 2) {
    // one plain store per (query, head): the camera sum happened in registers, queries no camera sees get zeros
    if (active) {
      const float sc = have_sm ? 1.f / sum : 0.f;
      float *dst = prm.accum + it * C + sub * VEC;
#pragma unroll
      for (int i = 0; i < VEC; i += 4)
        *reinterpret_cast<float4 *>(dst + i) = make_float4(acc[i] * sc, acc[i + 1] * sc, acc[i + 2] * sc, acc[i + 3] * sc);
    }
  } else {
    // Fused SCA epilogue (reference: slots = (queries * bev_mask).sum(0), spatial_cross_attention.py:270): the
    // per-camera output never goes to memory; visible items add their bev_mask-weighted result into the fp32 BEV
    // accumulator with vector reductions (at most one add per camera that sees the query).
    unsigned any = inr;
#pragma unroll
    for (int d = 1; d < LPI; d <<= 1) any |= __shfl_xor_sync(kFullMask, any, d);
    const float mk1 = __ldg(prm.mask + bq0);
    if (active && any != 0u && mk1 != 0.f) {
      const float sc = mk1 / sum;
      float *dst = prm.accum + ((bq0 - (bq0 / Q) * Q) * M + m) * C + sub * VEC;
#pragma unroll
      for (int i = 0; i < VEC; i += 4)
        asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(dst + i), "f"(acc[i] * sc),
                     "f"(acc[i + 1] * sc), "f"(acc[i + 2] * sc), "f"(acc[i + 3] * sc)
                     : "memory");
    }
  }
  }  // units
}

// ---------------------------------------------------------------------------------------------------------------
// Generic fallback: any C / P / G (one thread per output scalar, fp32 math). Correctness path for odd shapes.
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float load_as_float(const T *p, long long i, float s);
template <>
__device__ __forceinline__ float load_as_float<float>(const float *p, long long i, float) {
  return __ldg(p + i);
}
template <>
__device__ __forceinline__ float load_as_float<__half>(const __half *p, long long i, float) {
  return __half2float(__ldg(p + i));
}
template <>
__device__ __forceinline__ float load_as_float<__nv_bfloat16>(const __nv_bfloat16 *p, long long i, float) {
  return bf16_to_f(__ldg(p + i));
}
template <>
__device__ __forceinline__ float load_as_float<int8_t>(const int8_t *p, long long i, float s) {
  return static_cast<float>(__ldg(p + i)) * s;
}
template <typename T>
__device__ __forceinline__ void store_from_float(T *p, long long i, float v, const MsdaParams &prm);
template <>
__device__ __forceinline__ void store_from_float<float>(float *p, long long i, float v, const MsdaParams &) {
  p[i] = v;
}
template <>
__device__ __forceinline__ void store_from_float<__half>(__half *p, long long i, float v, const MsdaParams &) {
  p[i] = __float2half_rn(v);
}
template <>
__device__ __forceinline__ void store_from_float<__nv_bfloat16>(__nv_bfloat16 *p, long long i, float v, const MsdaParams &) {
  p[i] = __float2bfloat16_rn(v);
}
template <>
__device__ __forceinline__ void store_from_float<int8_t>(int8_t *p, long long i, float v, const MsdaParams &prm) {
  p[i] = static_cast<int8_t>(to_int8_sat(v * prm.scale_value / prm.scale_out));
}

template <typename T, typename R>
__global__ void __launch_bounds__(kThreads) msda_generic_kernel(const MsdaParams prm) {
  const int M = prm.M, C = prm.C, Q = prm.Q, P = prm.P, G = prm.G, L = prm.L, NP = L * P;
  const long long n = prm.items * C;
  const T *value = static_cast<const T *>(prm.value);
  const T *off = static_cast<const T *>(prm.off);
  const T *logits = static_cast<const T *>(prm.logits);
  const R *ref = static_cast<const R *>(prm.ref);
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < n;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % C);
    const long long it = idx / C;
    const long long bq = it / M;
    const int m = static_cast<int>(it - bq * M);
    const int b = static_cast<int>(bq / Q);
    float mx = -INFINITY;
    for (int i = 0; i < NP; ++i) mx = fmaxf(mx, load_as_float<T>(logits, it * NP + i, prm.scale_weight));
    float acc = 0.f, sum = 0.f;
    long long start = 0;
    int k = 0;
    for (int l = 0; l < L; ++l) {
      const int H = prm.shapes[2 * l], W = prm.shapes[2 * l + 1];
      const T *vl = value + ((static_cast<long long>(b) * prm.S + start) * M + m) * C + c;
      for (int p = 0; p < P; ++p, ++k) {
        const int g = p % G;
        const float rx = ref_to_float<R>(ref, bq * 2 * G + 2 * g), ry = ref_to_float<R>(ref, bq * 2 * G + 2 * g + 1);
        const float ox = load_as_float<T>(off, (it * NP + k) * 2, prm.scale_offset);
        const float oy = load_as_float<T>(off, (it * NP + k) * 2 + 1, prm.scale_offset);
        const float e = expf(load_as_float<T>(logits, it * NP + k, prm.scale_weight) - mx);
        sum += e;
        const PointRec pr = point_record(rx, ry, ox, oy, H, W);
        if (prm.trace != nullptr && c == 0)
          prm.trace[it * NP + k] = pr.in_range ? make_int4(1, pr.h_low, pr.w_low, tap_mask_of(pr, H, W)) : make_int4(0, 0, 0, 0);
        if (!pr.in_range) continue;
        const int tm = tap_mask_of(pr, H, W);
        const long long stp = static_cast<long long>(M) * C;
        const T *t0 = vl + (static_cast<long long>(pr.h_low) * W + pr.w_low) * stp;
        const float v1 = (tm & 1) ? load_as_float<T>(t0, 0, 1.f) : 0.f;
        const float v2 = (tm & 2) ? load_as_float<T>(t0, stp, 1.f) : 0.f;
        const float v3 = (tm & 4) ? load_as_float<T>(t0, W * stp, 1.f) : 0.f;
        const float v4 = (tm & 8) ? load_as_float<T>(t0, W * stp + stp, 1.f) : 0.f;
        const float hh = 1.f - pr.lh, hw = 1.f - pr.lw;
        acc += (hh * hw * v1 + hh * pr.lw * v2 + pr.lh * hw * v3 + pr.lh * pr.lw * v4) * e;
      }
      start += static_cast<long long>(H) * W;
    }
    store_from_float<T>(static_cast<T *>(prm.out), idx, acc / sum, prm);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Diagnostic kernel: sampling-index records (same device function as the product kernels).
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void msda_index_kernel(const int32_t *shapes, const T *ref, const T *off, int B, int M, int L, int Q, int P,
                                  int G, int4 *rec) {
  const int NP = L * P;
  const long long n = static_cast<long long>(B) * Q * M * NP;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < n;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(idx % NP);
    const long long it = idx / NP;
    const long long bq = it / M;
    const int l = k / P, g = (k % P) % G;
    const int H = shapes[2 * l], W = shapes[2 * l + 1];
    const PointRec pr = point_record(load_as_float<T>(ref, bq * 2 * G + 2 * g, 1.f),
                                     load_as_float<T>(ref, bq * 2 * G + 2 * g + 1, 1.f),
                                     load_as_float<T>(off, idx * 2, 1.f), load_as_float<T>(off, idx * 2 + 1, 1.f), H, W);
    rec[idx] = pr.in_range ? make_int4(1, pr.h_low, pr.w_low, tap_mask_of(pr, H, W)) : make_int4(0, 0, 0, 0);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------------------------
template <typename T, typename R, int C, int ROUNDS, int MODE, int EPI>
static int launch_gather(const MsdaParams &p, cudaStream_t s) {
  constexpr int LPI = C / Io<T, 0>::kVec;
  constexpr int IPB = (32 / LPI) * (kThreads / 32);
  const long long blocks = (p.items + IPB - 1) / IPB;
  if (blocks > 0x7fffffffll) return B200_ERR_BAD_PARAM;
  auto launch = [s](void (*kernel)(const MsdaParams), long long grid, int threads, const MsdaParams &prm) {
    kernel<<<static_cast<unsigned>(grid), threads, 0, s>>>(prm);
    return check_launch();
  };
  // Batched launch (visibility scan over UPW units per warp): the FP32 / FP16 plugin op at <= 2 rounds, which covers
  // every BEVFormer shape (NP = 32 points: 2 rounds FP16, 1 round FP32). The traced instantiation follows the same
  // switch, so the index records the parity tests read come out of whichever kernel the plugin op runs.
  if constexpr (EPI == 0 && MODE == 0 && ROUNDS <= 2 && !std::is_same<T, int8_t>::value) {
    const int cfg = msda_batch_units(), upw = cfg & 0xff;
    if ((upw == 4 || upw == 2) && IPB % p.M == 0) {
      const long long bb = (blocks + upw - 1) / upw;
      MsdaParams q = p;
      q.unit_stride = (cfg >> 8) & 1;
      if (p.trace != nullptr)
        return launch(upw == 4 ? msda_gather_kernel<T, R, C, ROUNDS, 0, 0, true, 4>
                               : msda_gather_kernel<T, R, C, ROUNDS, 0, 0, true, 2>, bb, kThreads, q);
      if (msda_gather_variant() == 1)  // batched scan AND 2 CTAs per SM (128-register budget)
        return launch(upw == 4 ? msda_gather_kernel<T, R, C, ROUNDS, 0, 0, false, 4, 2>
                               : msda_gather_kernel<T, R, C, ROUNDS, 0, 0, false, 2, 2>, bb, kThreads, q);
      return launch(upw == 4 ? msda_gather_kernel<T, R, C, ROUNDS, 0, 0, false, 4>
                             : msda_gather_kernel<T, R, C, ROUNDS, 0, 0, false, 2>, bb, kThreads, q);
    }
  }
  if constexpr (EPI == 0 && MODE == 0) {
    if (p.trace != nullptr) return launch(msda_gather_kernel<T, R, C, ROUNDS, MODE, 0, true>, blocks, kThreads, p);
  }
  // Gather-depth variants of the same plugin op (one-unit grid, untraced launches): see the kernel's header comment.
  if constexpr (EPI == 0 && MODE == 0 && ROUNDS <= 2 && !std::is_same<T, int8_t>::value) {
    switch (msda_gather_variant()) {
      case 1: return launch(msda_gather_kernel<T, R, C, ROUNDS, 0, 0, false, 1, 2, 1>, blocks, kThreads, p);
      case 2: return launch(msda_gather_kernel<T, R, C, ROUNDS, 0, 0, false, 1, 2, 4>, blocks, kThreads, p);
      case 3: {  // 128-thread CTAs, 5 per SM
        constexpr int IPB128 = (32 / LPI) * (128 / 32);
        const long long b128 = (p.items + IPB128 - 1) / IPB128;
        if (b128 > 0x7fffffffll) break;
        return launch(msda_gather_kernel<T, R, C, ROUNDS, 0, 0, false, 1, 5, 2, 128>, b128, 128, p);
      }
      default: break;
    }
  }
  // The fused spatial-cross-attention forms follow the same switch with one alternative: any non-zero gather variant runs
  // them at 2 CTAs per SM (same source, 128-register budget: a chunk's 16 tap loads in flight per warp).
  if constexpr (EPI != 0 && MODE == 0 && ROUNDS <= 2) {
    if (msda_gather_variant() != 0)
      return launch(msda_gather_kernel<T, R, C, ROUNDS, 0, EPI, false, 1, 2, 1>, blocks, kThreads, p);
  }
  return launch(msda_gather_kernel<T, R, C, ROUNDS, MODE, EPI>, blocks, kThreads, p);
}

template <typename T, typename R>
static int launch_generic(const MsdaParams &p, cudaStream_t s) {
  msda_generic_kernel<T, R><<<msda_grid_for(p.items * p.C), kThreads, 0, s>>>(p);
  return check_launch();
}

template <typename T, typename R, int C, int MODE, int EPI>
static int dispatch_rounds(const MsdaParams &p, cudaStream_t s) {
  constexpr int LPI = C / Io<T, 0>::kVec;
  const int nch = p.L * p.P / 4;
  const int rounds = (nch + LPI - 1) / LPI;
  if (rounds <= 1) return launch_gather<T, R, C, 1, MODE, EPI>(p, s);
  if (rounds <= 2) return launch_gather<T, R, C, 2, MODE, EPI>(p, s);
  if (EPI == 0 && rounds <= 4) return launch_gather<T, R, C, 4, MODE, 0>(p, s);
  return EPI == 0 ? launch_generic<T, R>(p, s) : B200_ERR_UNSUPPORTED;
}

template <typename T, typename R, int MODE, int EPI = 0>
static int dispatch(const MsdaParams &p, const MsdaGeom &g, cudaStream_t s) {
  // every BEVFormer variant has embed_dims / num_heads = 256 / 8 = 32 channels per head
  if (msda_aligned({p.value, p.off, p.logits, p.out, p.accum, p.ref}, 16) && msda_aligned({p.shapes}, 8) &&
      msda_lane_group_shape(g, kMaxChunks * 4))
    return dispatch_rounds<T, R, 32, MODE, EPI>(p, s);
  return EPI == 0 ? launch_generic<T, R>(p, s) : B200_ERR_UNSUPPORTED;
}

static MsdaParams make_params(const void *value, const int32_t *shapes, const void *ref, const void *off,
                              const void *logits, void *out, const MsdaGeom &g) {
  MsdaParams p{};
  p.value = value, p.shapes = shapes, p.ref = ref, p.off = off, p.logits = logits, p.out = out;
  msda_set_dims(p, g);
  p.items = static_cast<long long>(g.B) * g.Q * g.M;
  p.scale_value = p.scale_offset = p.scale_weight = p.scale_out = 1.f;
  return p;
}

// Argument checks of every forward entry, and the zero-fill of a traced launch's records. Each plugin op checks, selects
// its kernel and launches in one place, untraced (records == nullptr) or traced, so a trace entry runs the kernel its
// plugin op runs.
static int op_prologue(MsdaParams &p, const MsdaGeom &g, int32_t *records, cudaStream_t s) {
  if (!p.value || !p.shapes || !p.ref || !p.off || !p.logits || !(p.out || (p.accum && p.mask)))
    return B200_ERR_BAD_PARAM;
  const int st = msda_check_dims(g);
  if (st != B200_OK || !records) return st;
  if (cudaMemsetAsync(records, 0, static_cast<size_t>(p.items) * g.L * g.P * 16, s) != cudaSuccess) return B200_ERR_LAUNCH;
  p.trace = reinterpret_cast<int4 *>(records);
  return B200_OK;
}

// FP32, and BF16 value / offsets / logits / out with FP32 reference points (a bf16 reference point would move the
// sampling position by up to 2^-9 of the level's extent; BF16 takes FP16's kernel selection, without the FP16 mode and
// path switches).
template <typename T, typename R>
static int msda_exact_op(MsdaParams p, const MsdaGeom &g, int32_t *records, cudaStream_t s) {
  const int st = op_prologue(p, g, records, s);
  return st != B200_OK ? st : dispatch<T, R, 0>(p, g, s);
}

// Resident-tail kernel only with exact arithmetic; a traced launch is always exact (the gather kernel's DBG
// instantiation exists for MODE 0 only).
static int msda_f16_op(MsdaParams p, const MsdaGeom &g, int32_t *records, cudaStream_t s) {
  int st = op_prologue(p, g, records, s);
  if (st != B200_OK) return st;
  const bool mixed = g_f16_mode.load(std::memory_order_relaxed) != 0;
  if (g_f16_path.load(std::memory_order_relaxed) && !mixed) {
    st = msda_res_f16(p.value, p.shapes, p.ref, p.off, p.logits, p.out, p.trace, g,
                      g_res_cap_bytes.load(std::memory_order_relaxed), s);
    if (st != B200_ERR_UNSUPPORTED) return st;
  }
  return mixed && !records ? dispatch<__half, __half, 1>(p, g, s) : dispatch<__half, __half, 0>(p, g, s);
}

// The C-ABI entries of each family: the plugin ops and their trace twins, which require `records`.
using MsdaOp = int (*)(MsdaParams, const MsdaGeom &, int32_t *, cudaStream_t);

template <MsdaOp OP, bool TRACE = false>
static int plugin_entry(const void *value, const int32_t *shapes, const void *ref, const void *off, const void *logits,
                        void *out, int32_t *records, const MsdaGeom &g, void *stream) {
  if (TRACE && !records) return B200_ERR_BAD_PARAM;
  return OP(make_params(value, shapes, ref, off, logits, out, g), g, records, static_cast<cudaStream_t>(stream));
}

template <bool TRACE = false>
static int i8_entry(const int8_t *value, float scale_value, const int32_t *shapes, const void *ref, int ref_is_half,
                    const int8_t *off, float scale_offset, const int8_t *logits, float scale_weight, int8_t *out,
                    float scale_out, int32_t *records, const MsdaGeom &g, void *stream) {
  if (TRACE && !records) return B200_ERR_BAD_PARAM;
  if (g.C % 4 != 0 || g.P % 4 != 0) return B200_ERR_UNSUPPORTED;  // …Plugin.cpp:151-156
  if (!(scale_out > 0.f)) return B200_ERR_BAD_PARAM;
  MsdaParams p = make_params(value, shapes, ref, off, logits, out, g);
  p.scale_value = scale_value, p.scale_offset = scale_offset, p.scale_weight = scale_weight, p.scale_out = scale_out;
  p.ref_is_half = ref_is_half;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int st = op_prologue(p, g, records, s);
  if (st != B200_OK) return st;
  return ref_is_half ? dispatch<int8_t, __half, 0>(p, g, s) : dispatch<int8_t, float, 0>(p, g, s);
}

// The fused spatial-cross-attention forms: EPI 1 camera-summed (accum), EPI 2 camera-shared (slots).
template <typename T, typename R, int EPI>
static int sca_entry(const void *value, const int32_t *shapes, const void *ref, const void *off, const void *logits,
                     const float *bev_mask, float *accum, const MsdaGeom &g, void *stream) {
  MsdaParams p = make_params(value, shapes, ref, off, logits, nullptr, g);
  p.mask = bev_mask, p.accum = accum;
  if (EPI == 2) p.items = static_cast<long long>(g.Q) * g.M;  // one item per (query, head); cameras are looped inside
  const int st = op_prologue(p, g, nullptr, static_cast<cudaStream_t>(stream));
  return st != B200_OK ? st : dispatch<T, R, 0, EPI>(p, g, static_cast<cudaStream_t>(stream));
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_msda_set_f16_mode(int mode) { return g_f16_mode.exchange(mode ? 1 : 0); }
int b200_msda_set_f16_path(int path) { return g_f16_path.exchange(path ? 1 : 0); }
int b200_msda_set_gather_variant(int variant) {
  const int before = msda_gather_variant();
  if (variant >= 0 && variant <= 3) g_gather_variant.store(variant, std::memory_order_relaxed);
  return before;  // any other value (e.g. -1) only queries
}

int b200_msda_set_batch_units(int units, int strided) {
  const int before = msda_batch_units();
  if (units == 1) g_batch_units.store(1, std::memory_order_relaxed);
  else if (units == 2 || units == 4) g_batch_units.store(units | (strided ? 0x100 : 0), std::memory_order_relaxed);
  return before;  // any other `units` (e.g. 0) only queries
}
int b200_msda_set_resident_bytes(int bytes) { return g_res_cap_bytes.exchange(bytes < 8192 ? 8192 : (bytes > 200 * 1024 ? 200 * 1024 : bytes)); }

int b200_msda_f32(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                  const float *sampling_offsets, const float *attn_weight, int batch, int spatial_size, int num_heads,
                  int channels, int num_levels, int num_query, int num_point, int points_per_group, float *out,
                  void *stream) {
  return plugin_entry<msda_exact_op<float, float>>(value, spatial_shapes, reference_points, sampling_offsets,
      attn_weight, out, nullptr,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_f16(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                  const void *sampling_offsets, const void *attn_weight, int batch, int spatial_size, int num_heads,
                  int channels, int num_levels, int num_query, int num_point, int points_per_group, void *out,
                  void *stream) {
  return plugin_entry<msda_f16_op>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight, out, nullptr,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_f16_h2(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                     const void *sampling_offsets, const void *attn_weight, int batch, int spatial_size,
                     int num_heads, int channels, int num_levels, int num_query, int num_point, int points_per_group,
                     void *out, void *stream) {
  if (channels % 2 != 0) return B200_ERR_UNSUPPORTED;  // …Plugin.cpp:240-245
  return b200_msda_f16(value, spatial_shapes, reference_points, sampling_offsets, attn_weight, batch, spatial_size,
                       num_heads, channels, num_levels, num_query, num_point, points_per_group, out, stream);
}

int b200_msda_bf16(const void *value, const int32_t *spatial_shapes, const float *reference_points,
                   const void *sampling_offsets, const void *attn_weight, int batch, int spatial_size, int num_heads,
                   int channels, int num_levels, int num_query, int num_point, int points_per_group, void *out,
                   void *stream) {
  return plugin_entry<msda_exact_op<__nv_bfloat16, float>>(value, spatial_shapes, reference_points, sampling_offsets,
      attn_weight, out, nullptr,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_i8(const int8_t *value, float scale_value, const int32_t *spatial_shapes, const void *reference_points,
                 int ref_is_half, const int8_t *sampling_offsets, float scale_offset, const int8_t *attn_weight,
                 float scale_weight, int batch, int spatial_size, int num_heads, int channels, int num_levels,
                 int num_query, int num_point, int points_per_group, int8_t *out, float scale_out, void *stream) {
  return i8_entry(value, scale_value, spatial_shapes, reference_points, ref_is_half, sampling_offsets, scale_offset,
      attn_weight, scale_weight, out, scale_out, nullptr,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_sca_f32(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                      const float *sampling_offsets, const float *attn_weight, const float *bev_mask, int batch,
                      int spatial_size, int num_heads, int channels, int num_levels, int num_query, int num_point,
                      int points_per_group, float *accum, void *stream) {
  return sca_entry<float, float, 1>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight, bev_mask,
      accum, msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group),
      stream);
}

int b200_msda_sca_f16(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                      const void *sampling_offsets, const void *attn_weight, const float *bev_mask, int batch,
                      int spatial_size, int num_heads, int channels, int num_levels, int num_query, int num_point,
                      int points_per_group, float *accum, void *stream) {
  return sca_entry<__half, __half, 1>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight, bev_mask,
      accum, msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group),
      stream);
}

int b200_msda_sca_bf16(const void *value, const int32_t *spatial_shapes, const float *reference_points,
                       const void *sampling_offsets, const void *attn_weight, const float *bev_mask, int batch,
                       int spatial_size, int num_heads, int channels, int num_levels, int num_query, int num_point,
                       int points_per_group, float *accum, void *stream) {
  return sca_entry<__nv_bfloat16, float, 1>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight,
      bev_mask, accum,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_sca_shared_f32(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                             const float *sampling_offsets, const float *attn_weight, const float *bev_mask,
                             int batch, int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                             int num_point, int points_per_group, float *slots, void *stream) {
  return sca_entry<float, float, 2>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight, bev_mask,
      slots, msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group),
      stream);
}

int b200_msda_sca_shared_f16(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                             const void *sampling_offsets, const void *attn_weight, const float *bev_mask, int batch,
                             int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                             int num_point, int points_per_group, float *slots, void *stream) {
  return sca_entry<__half, __half, 2>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight, bev_mask,
      slots, msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group),
      stream);
}

int b200_msda_sca_shared_bf16(const void *value, const int32_t *spatial_shapes, const float *reference_points,
                              const void *sampling_offsets, const void *attn_weight, const float *bev_mask, int batch,
                              int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                              int num_point, int points_per_group, float *slots, void *stream) {
  return sca_entry<__nv_bfloat16, float, 2>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight,
      bev_mask, slots,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

// The plugin ops with the trace switch on: same kernel selection, plus one record per point.
int b200_msda_f32_trace(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                        const float *sampling_offsets, const float *attn_weight, int batch, int spatial_size,
                        int num_heads, int channels, int num_levels, int num_query, int num_point,
                        int points_per_group, float *out, int32_t *records, void *stream) {
  return plugin_entry<msda_exact_op<float, float>, true>(value, spatial_shapes, reference_points, sampling_offsets,
      attn_weight, out, records,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_f16_trace(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                        const void *sampling_offsets, const void *attn_weight, int batch, int spatial_size,
                        int num_heads, int channels, int num_levels, int num_query, int num_point,
                        int points_per_group, void *out, int32_t *records, void *stream) {
  return plugin_entry<msda_f16_op, true>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight, out,
      records, msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group),
      stream);
}

int b200_msda_bf16_trace(const void *value, const int32_t *spatial_shapes, const float *reference_points,
                         const void *sampling_offsets, const void *attn_weight, int batch, int spatial_size,
                         int num_heads, int channels, int num_levels, int num_query, int num_point,
                         int points_per_group, void *out, int32_t *records, void *stream) {
  return plugin_entry<msda_exact_op<__nv_bfloat16, float>, true>(value, spatial_shapes, reference_points,
      sampling_offsets, attn_weight, out, records,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_i8_trace(const int8_t *value, float scale_value, const int32_t *spatial_shapes,
                       const void *reference_points, int ref_is_half, const int8_t *sampling_offsets,
                       float scale_offset, const int8_t *attn_weight, float scale_weight, int batch, int spatial_size,
                       int num_heads, int channels, int num_levels, int num_query, int num_point, int points_per_group,
                       int8_t *out, float scale_out, int32_t *records, void *stream) {
  return i8_entry<true>(value, scale_value, spatial_shapes, reference_points, ref_is_half, sampling_offsets,
      scale_offset, attn_weight, scale_weight, out, scale_out, records,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_debug_indices(int dtype, const int32_t *spatial_shapes, const void *reference_points,
                            const void *sampling_offsets, int batch, int num_heads, int num_levels, int num_query,
                            int num_point, int points_per_group, int32_t *records, void *stream) {
  if (!spatial_shapes || !reference_points || !sampling_offsets || !records) return B200_ERR_BAD_PARAM;
  const long long n = static_cast<long long>(batch) * num_query * num_heads * num_levels * num_point;
  if (n <= 0) return B200_ERR_BAD_PARAM;
  const unsigned blocks = msda_grid_for(n);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dtype == 0)
    msda_index_kernel<float><<<blocks, 256, 0, s>>>(spatial_shapes, static_cast<const float *>(reference_points),
                                                    static_cast<const float *>(sampling_offsets), batch, num_heads,
                                                    num_levels, num_query, num_point, points_per_group,
                                                    reinterpret_cast<int4 *>(records));
  else if (dtype == 1)
    msda_index_kernel<__half><<<blocks, 256, 0, s>>>(spatial_shapes, static_cast<const __half *>(reference_points),
                                                     static_cast<const __half *>(sampling_offsets), batch, num_heads,
                                                     num_levels, num_query, num_point, points_per_group,
                                                     reinterpret_cast<int4 *>(records));
  else
    return B200_ERR_UNSUPPORTED;
  return check_launch();
}

}  // extern "C"

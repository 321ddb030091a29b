// msda_backward.cu — backward of the plugin-signature multi-scale deformable attention op (b200_msda_f32 / _f16):
// gradients for value, reference points, sampling offsets and the PRE-softmax attention logits. The training graph of the
// reference reaches mmcv's ms_deform_attn_backward for this (bev_mmdet3d/.../multi_scale_deformable_attn_function.py);
// here softmax and the location arithmetic live inside the op, so their derivatives do too.
//
// Per item (b, q, head m) and point k = (level l, point p), group g = p % G, with the forward's position rule
// (point_record, msda_index.cuh): a_k = softmax(logits)_k, s_k[c] = bilinear sample, go[c] = grad_out[b, q, m, c],
//   d_k            = sum_c go[c] * s_k[c]
//   grad_logits_k  = a_k * (d_k - sum_j a_j d_j)
//   grad_value[b, pixel(tap), m, c] += a_k * w_tap * go[c]           every in-image tap of every in-range point
//   grad_off_x,k   = a_k * sum_c go[c] * ((1-lh)(v2-v1) + lh(v4-v3))  offsets are in pixels: no W / H factor
//   grad_off_y,k   = a_k * sum_c go[c] * ((1-lw)(v3-v1) + lw(v4-v2))  (taps outside the image count as 0)
//   grad_ref_x[b, q, g] = sum_{m, l, p: p % G == g} W_l * grad_off_x,k   (grad_ref_y with H_l)
// A point outside the range gate contributes nothing except its share of the softmax denominator.
//
// Two kernels; msda_bw_takes_c32() is the one place that chooses between them:
//   * msda_bw_c32_kernel — C = 32. A lane group of C/VEC lanes (VEC = 4 fp32 / 8 fp16 channels) owns one item and walks
//     its points together. Every lane of the group evaluates the point's position itself (the loads are broadcasts), so
//     each lane holds lh, lw and a_k and can fold its four partial tap dots into partial (d, grad_off_x, grad_off_y)
//     BEFORE the group reduction: three shuffle trees per point instead of four, and no owner-to-group broadcast. d and
//     the two offset gradients of a point are parked in shared memory until sum_j a_j d_j is known, then written once.
//     grad_value is scattered with red.global.add.v4.f32 into an fp32 accumulator. A warp none of whose items has a
//     point in range writes zeros and reads nothing else (exact: every d_k is 0).
//   * msda_bw_generic_kernel — any C / P / G, unaligned tensors: one thread per item, scalar loads and atomics.
// grad_reference_points: both kernels write one fp32 partial per (item, group) in a fixed order; a second kernel sums
// the heads in head order. FP16 / BF16 grad_value: the fp32 accumulator is the workspace, rounded once by a final kernel.
// BF16 reads fp32 reference points and writes an fp32 grad_reference_points (BwRef below); FP32 and FP16 use T.
//
// The fused SCA forms (msda.cu, b200_msda_sca_* and b200_msda_sca_shared_*) are differentiated by the same lane-group
// kernel with an epilogue parameter EPI, as in the forward; grad_slots is fp32 [Q, M*C] for both dtypes:
//   * EPI 1, camera-summed: items (b, q, m) as above with go[c] = bev_mask[b, q] * grad_slots[q, m*C + c]. A pair with
//     bev_mask == 0 contributes nothing to the forward whatever it samples, so it reads nothing here and gets exact
//     zeros (the composition mask * grad_slots into the plugin backward would give 0 * NaN on a non-finite pixel).
//   * EPI 2, camera-shared: one item per (q, m), offsets and logits shared by the B cameras, cameras looped inside. With
//     D_k = sum_{b: mask_b != 0} mask_b * sum_c gs[c] s_{b,k}[c] (camera order): grad_logits_k = a_k (D_k - sum_j a_j D_j),
//     grad_off_k = a_k sum_b mask_b (...), grad_value[b] += mask_b a_k w_tap gs; the per-point parking slots accumulate
//     across cameras and each offset / logit gradient is written once. grad_reference_points[b, q] gets one partial per
//     (b, q, m, g) as above. Cameras with mask 0 and cameras in which no point of the warp is in range are skipped; the
//     softmax is evaluated when the first camera that sees the warp's queries turns up (the forward's have_sm), and a
//     query no camera sees gets zero offset and logit gradients without its logits being used.
//
// Determinism: grad_sampling_offsets, grad_attention_weights and grad_reference_points are ordered sums (fixed shuffle
// trees, fixed loops): the same bits on every run and for every subset of requested gradients. grad_value is summed
// with float atomics and is not (as in mmcv).
#include "common.cuh"
#include "msda_geometry.cuh"
#include "msda_index.cuh"

namespace b200 {
namespace {

constexpr int kBwMaxLevels = kMsdaMaxLevels;
constexpr int kBwThreads = 256;
constexpr int kBwC32MaxPoints = 64;  // the C = 32 kernel parks 3 floats per (item, point) in shared memory

struct MsdaBwParams {
  const void *value, *ref, *off, *logits, *gout;  // gout: grad_out in T; EPI 1 / 2: grad_slots, fp32 [Q, M*C]
  const int32_t *shapes;
  float *gv_acc;    // fp32 [B, S, M, C] accumulator (zeroed by the entry), or null
  void *goff;       // [items, NP, 2] in T, or null
  void *glog;       // [items, NP] in T, or null
  float *ref_part;  // fp32 [items, G, 2] partials of grad_reference_points (EPI 2: [B, items, G, 2]), or null
  int B, S, M, C, L, Q, P, G;
  long long items;     // EPI 0 / 1: B * Q * M; EPI 2: Q * M
  const float *mask;   // EPI 1 / 2: bev_mask [B, Q] (last, so that the EPI 0 kernels read their fields where they did)
};

template <typename T>
struct BwIo;
template <>
struct BwIo<float> {
  static constexpr int kVec = 4;
  __device__ static float ld(const float *p) { return __ldg(p); }
  __device__ static void st(float *p, float v) { *p = v; }
  __device__ static void st2(float *p, float a, float b) { *reinterpret_cast<float2 *>(p) = make_float2(a, b); }
  __device__ static float2 ld2(const float *p) { return __ldg(reinterpret_cast<const float2 *>(p)); }
  __device__ static void unpack(const uint4 &u, float (&v)[4]) {
    v[0] = __uint_as_float(u.x), v[1] = __uint_as_float(u.y), v[2] = __uint_as_float(u.z), v[3] = __uint_as_float(u.w);
  }
};
template <>
struct BwIo<__nv_bfloat16> {
  static constexpr int kVec = 8;
  __device__ static float ld(const __nv_bfloat16 *p) { return bf16_to_f(__ldg(p)); }
  __device__ static void st(__nv_bfloat16 *p, float v) { *p = __float2bfloat16_rn(v); }
  __device__ static void st2(__nv_bfloat16 *p, float a, float b) {
    *reinterpret_cast<uint32_t *>(p) = f2_to_bf2(a, b);
  }
  __device__ static float2 ld2(const __nv_bfloat16 *p) { return bf2_to_f2(ldg32(p)); }
  __device__ static void unpack(const uint4 &u, float (&v)[8]) {
    const float2 a = bf2_to_f2(u.x), b = bf2_to_f2(u.y), c = bf2_to_f2(u.z), d = bf2_to_f2(u.w);
    v[0] = a.x, v[1] = a.y, v[2] = b.x, v[3] = b.y, v[4] = c.x, v[5] = c.y, v[6] = d.x, v[7] = d.y;
  }
};
template <>
struct BwIo<__half> {
  static constexpr int kVec = 8;
  __device__ static float ld(const __half *p) { return __half2float(__ldg(p)); }
  __device__ static void st(__half *p, float v) { *p = __float2half_rn(v); }
  __device__ static void st2(__half *p, float a, float b) { *reinterpret_cast<__half2 *>(p) = __floats2half2_rn(a, b); }
  __device__ static float2 ld2(const __half *p) { return h2_to_f2(ldg32(p)); }
  __device__ static void unpack(const uint4 &u, float (&v)[8]) {
    const float2 a = h2_to_f2(u.x), b = h2_to_f2(u.y), c = h2_to_f2(u.z), d = h2_to_f2(u.w);
    v[0] = a.x, v[1] = a.y, v[2] = b.x, v[3] = b.y, v[4] = c.x, v[5] = c.y, v[6] = d.x, v[7] = d.y;
  }
};

// Storage type of the reference points and of their gradient: T, except BF16, which reads and writes them in fp32 (a
// bf16 reference point would move the sample by up to 2^-9 of the level's extent).
template <typename T>
struct BwRef {
  using type = T;
};
template <>
struct BwRef<__nv_bfloat16> {
  using type = float;
};

__device__ __forceinline__ void red_add_v4(float *p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// ---- C = 32 --------------------------------------------------------------------------------------------------------
// Requirements (msda_bw_takes_c32): P % 4 == 0, G in {1, 2, 4}, L * P <= kBwC32MaxPoints, 16-byte aligned tensors.

// the reference-point partials of one item, summed over the points of each group in a fixed order
__device__ __forceinline__ void store_ref_partial(float *ref_item, const float (&rx)[4], const float (&ry)[4], int G) {
  if (G == 4) {
#pragma unroll
    for (int j = 0; j < 4; ++j) ref_item[2 * j] = rx[j], ref_item[2 * j + 1] = ry[j];
  } else if (G == 2) {
    ref_item[0] = rx[0] + rx[2], ref_item[1] = ry[0] + ry[2];
    ref_item[2] = rx[1] + rx[3], ref_item[3] = ry[1] + ry[3];
  } else {
    ref_item[0] = (rx[0] + rx[1]) + (rx[2] + rx[3]), ref_item[1] = (ry[0] + ry[1]) + (ry[2] + ry[3]);
  }
}

// EPI: 0 = plugin op, 1 = camera-summed SCA, 2 = camera-shared SCA (see the top of the file). For EPI 0 / 1 the camera
// loop below runs once, for the item's own camera.
template <typename T, int EPI>
__global__ void __launch_bounds__(kBwThreads, 2) msda_bw_c32_kernel(const MsdaBwParams prm) {
  using IO = BwIo<T>;
  using R = typename BwRef<T>::type;
  constexpr int C = 32, VEC = IO::kVec, LPI = C / VEC, IPW = 32 / LPI, IPB = IPW * (kBwThreads / 32);
  extern __shared__ float bw_park[];  // [IPB][NP][3]: d, grad_off_x, grad_off_y of every point of the CTA's items
  __shared__ int sH[kBwMaxLevels], sW[kBwMaxLevels], sStart[kBwMaxLevels];

  const int M = prm.M, Q = prm.Q, P = prm.P, G = prm.G, L = prm.L, NP = L * P;
  if (threadIdx.x == 0) {
    int start = 0;
    for (int l = 0; l < L; ++l) {
      sH[l] = prm.shapes[2 * l], sW[l] = prm.shapes[2 * l + 1], sStart[l] = start;
      start += sH[l] * sW[l];
    }
  }
  __syncthreads();  // the only block-wide barrier: warps are independent from here on

  const int lane = threadIdx.x & 31, sub = lane % LPI;
  const long long it_raw = static_cast<long long>(blockIdx.x) * IPB + threadIdx.x / LPI;
  const bool active = it_raw < prm.items;
  const long long it = active ? it_raw : prm.items - 1;  // lane groups past the end shadow the last item, never store
  const long long bq = it / M;  // EPI 2: q
  const int m = static_cast<int>(it - bq * M);
  const T *off_item = static_cast<const T *>(prm.off) + it * NP * 2;
  const T *lg_item = static_cast<const T *>(prm.logits) + it * NP;
  T *goff_item = prm.goff ? static_cast<T *>(prm.goff) + it * NP * 2 : nullptr;
  T *glog_item = prm.glog ? static_cast<T *>(prm.glog) + it * NP : nullptr;
  float *ref_first = prm.ref_part ? prm.ref_part + it * G * 2 : nullptr;
  float *park = bw_park + static_cast<size_t>(threadIdx.x / LPI) * NP * 3;
  if (EPI == 2 && active)  // the parking slots accumulate over the cameras
    for (int k = sub; k < NP; k += LPI) park[3 * k] = park[3 * k + 1] = park[3 * k + 2] = 0.f;

  float mx, inv, go[VEC];
  bool have_sm = false;    // EPI 2: the softmax statistics and grad_slots are loaded (warp-uniform)
  bool seen = EPI == 0;    // EPI 1: bev_mask != 0; EPI 2: some point is in range in a camera with a non-zero mask
  float sad = 0.f;  // sum_j a_j d_j, the same ordered sum in every lane of the group
  float rx[4] = {0.f, 0.f, 0.f, 0.f}, ry[4] = {0.f, 0.f, 0.f, 0.f};
  const int num_b = EPI == 2 ? prm.B : 1;
  for (int bi = 0; bi < num_b; ++bi) {
  const long long bqc = EPI == 2 ? static_cast<long long>(bi) * Q + bq : bq;  // (camera, query) of ref and mask
  const int b = EPI == 2 ? bi : static_cast<int>(bq / Q);
  const R *ref_bq = static_cast<const R *>(prm.ref) + bqc * 2 * G;
  float *ref_item = EPI == 2 && ref_first ? ref_first + bi * prm.items * G * 2 : ref_first;
  float mk = 1.f;
  bool live = active;  // EPI 1 / 2: and this (camera, query) pair has bev_mask != 0; nothing else of the pair is read
  if constexpr (EPI != 0) {
    mk = active ? __ldg(prm.mask + bqc) : 0.f;
    live = active && mk != 0.f;
    if (EPI == 1) seen = live;
  }

  // point j of a 4-point chunk reads group j % G (P % 4 == 0 and G divides 4)
  float rpx[4], rpy[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 r = EPI == 0 || live ? BwIo<R>::ld2(ref_bq + 2 * (j % G)) : make_float2(0.f, 0.f);
    rpx[j] = r.x, rpy[j] = r.y;
  }

  // ---- is any point of any item of this warp in range? (points dealt round-robin to the lanes of the group)
  bool any = false;
  if (EPI == 0 || live)
    for (int k = sub; k < NP; k += LPI) {
      const int l = k / P, g = (k - l * P) % G;
      const float2 r = BwIo<R>::ld2(ref_bq + 2 * g), o = IO::ld2(off_item + 2 * k);
      any |= point_record(r.x, r.y, o.x, o.y, sH[l], sW[l]).in_range;
    }
  if (__ballot_sync(kFullMask, any && live) == 0u) {
    if constexpr (EPI == 2) {
      // this camera adds nothing to any item of the warp: its reference-point partials are 0
      if (active && ref_item && sub == 0)
        for (int i = 0; i < 2 * G; ++i) ref_item[i] = 0.f;
      continue;
    }
    // a camera that sees none of these queries (or, EPI 1, a zero mask): every gradient of these items is exactly 0
    if (active) {
      for (int k = sub; k < NP; k += LPI) {
        if (goff_item) IO::st2(goff_item + 2 * k, 0.f, 0.f);
        if (glog_item) IO::st(glog_item + k, 0.f);
      }
      if (ref_item && sub == 0)
        for (int i = 0; i < 2 * G; ++i) ref_item[i] = 0.f;
    }
    return;
  }

  if (EPI != 2 || !have_sm) {
  have_sm = true;
  // ---- softmax statistics (EPI 1: a pair with a zero mask in a live warp does not read its logits)
  mx = -INFINITY;
  for (int k = sub; k < NP; k += LPI) mx = fmaxf(mx, EPI != 1 || live ? IO::ld(lg_item + k) : 0.f);
#pragma unroll
  for (int d = 1; d < LPI; d <<= 1) mx = fmaxf(mx, __shfl_xor_sync(kFullMask, mx, d));
  float sum = 0.f;
  for (int k = sub; k < NP; k += LPI) sum += expf((EPI != 1 || live ? IO::ld(lg_item + k) : 0.f) - mx);
#pragma unroll
  for (int d = 1; d < LPI; d <<= 1) sum += __shfl_xor_sync(kFullMask, sum, d);
  inv = 1.f / sum;

  if constexpr (EPI == 0) {
    IO::unpack(ldg128_stream(static_cast<const T *>(prm.gout) + it * C + sub * VEC), go);
  } else {
    // EPI 1: go = bev_mask * grad_slots, formed at the load; EPI 2: grad_slots (the mask weighs each camera below)
    const float *gs = static_cast<const float *>(prm.gout) + ((EPI == 2 ? bq : bq % Q) * M + m) * C + sub * VEC;
#pragma unroll
    for (int i = 0; i < VEC; i += 4) {
      const float4 v = EPI == 2 || live ? __ldg(reinterpret_cast<const float4 *>(gs + i)) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float s = EPI == 2 ? 1.f : mk;
      go[i] = s * v.x, go[i + 1] = s * v.y, go[i + 2] = s * v.z, go[i + 3] = s * v.w;
    }
  }
  }

  const long long stp = static_cast<long long>(M) * C;  // elements between horizontally adjacent pixels
  const long long vb = (static_cast<long long>(b) * prm.S * M + m) * C + sub * VEC;
  const T *value = static_cast<const T *>(prm.value);
  const bool scatter = prm.gv_acc != nullptr && active;

  for (int k0 = 0; k0 < NP; k0 += 4) {
    const int l = k0 / P, H = sH[l], W = sW[l];
    const long long lvl = vb + static_cast<long long>(sStart[l]) * stp;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + j;
      const float2 o = EPI == 0 || live ? IO::ld2(off_item + 2 * k) : make_float2(0.f, 0.f);
      PointRec rec = point_record(rpx[j], rpy[j], o.x, o.y, H, W);
      if (EPI != 0) rec.in_range = rec.in_range && live;
      float pd = 0.f, pgx = 0.f, pgy = 0.f, a = 0.f;
      if (__ballot_sync(kFullMask, rec.in_range) != 0u) {  // else: out of range in every item of the warp
        if (rec.in_range) {
          const int tm = tap_mask_of(rec, H, W);
          a = expf(IO::ld(lg_item + k) - mx) * inv;
          const float am = EPI == 2 ? a * mk : a;  // the grad_value weight of a unit tap
          const long long e0 = lvl + (static_cast<long long>(rec.h_low) * W + rec.w_low) * stp;
          const long long eo[4] = {e0, e0 + stp, e0 + W * stp, e0 + W * stp + stp};
          const float hh = 1.f - rec.lh, hw = 1.f - rec.lw;
          const float cw[4] = {hh * hw, hh * rec.lw, rec.lh * hw, rec.lh * rec.lw};
          float dot[4];
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            // a tap outside the image is never read: it is 0 whatever lies at the address it would alias
            dot[t] = 0.f;
            if (tm & (1 << t)) {
              float v[VEC];
              IO::unpack(ldg128(value + eo[t]), v);
#pragma unroll
              for (int i = 0; i < VEC; ++i) dot[t] = fmaf(go[i], v[i], dot[t]);
              if (scatter) {
                const float w = am * cw[t];
#pragma unroll
                for (int i = 0; i < VEC; i += 4)
                  red_add_v4(prm.gv_acc + eo[t] + i, w * go[i], w * go[i + 1], w * go[i + 2], w * go[i + 3]);
              }
            }
          }
          pd = cw[0] * dot[0] + cw[1] * dot[1] + cw[2] * dot[2] + cw[3] * dot[3];
          pgx = hh * (dot[1] - dot[0]) + rec.lh * (dot[3] - dot[2]);
          pgy = hw * (dot[2] - dot[0]) + rec.lw * (dot[3] - dot[1]);
        }
#pragma unroll
        for (int d = 1; d < LPI; d <<= 1) {
          pd += __shfl_xor_sync(kFullMask, pd, d);
          pgx += __shfl_xor_sync(kFullMask, pgx, d);
          pgy += __shfl_xor_sync(kFullMask, pgy, d);
        }
      }
      if constexpr (EPI == 2) {
        // pd, pgx, pgy are the same in every lane of the group, and so is rec: seen needs no reduction
        seen = seen || rec.in_range;
        pd *= mk, pgx *= mk, pgy *= mk;
        const float gx = a * pgx, gy = a * pgy;
        sad += a * pd;
        rx[j] += static_cast<float>(W) * gx, ry[j] += static_cast<float>(H) * gy;
        if (sub == k % LPI) park[3 * k] += pd, park[3 * k + 1] += pgx, park[3 * k + 2] += pgy;
      } else {
        const float gx = a * pgx, gy = a * pgy;
        sad += a * pd;
        rx[j] += static_cast<float>(W) * gx, ry[j] += static_cast<float>(H) * gy;
        if (sub == k % LPI) park[3 * k] = pd, park[3 * k + 1] = gx, park[3 * k + 2] = gy;
      }
    }
  }
  if constexpr (EPI == 2) {
    if (active && ref_item && sub == 0) store_ref_partial(ref_item, rx, ry, G);
#pragma unroll
    for (int j = 0; j < 4; ++j) rx[j] = ry[j] = 0.f;
  }
  }  // cameras

  if (!active) return;
  if (!seen) {
    // EPI 1: a pair with a zero mask in a warp with live pairs; EPI 2: a query no camera sees (its logits are not used)
    for (int k = sub; k < NP; k += LPI) {
      if (goff_item) IO::st2(goff_item + 2 * k, 0.f, 0.f);
      if (glog_item) IO::st(glog_item + k, 0.f);
    }
    if (EPI == 1 && ref_first && sub == 0)
      for (int i = 0; i < 2 * G; ++i) ref_first[i] = 0.f;
    return;
  }
  // every lane writes the points it parked itself (k % LPI == sub), so no barrier is needed
  for (int k = sub; k < NP; k += LPI) {
    if constexpr (EPI == 2) {
      // the offset gradients were parked without their a_k, which is camera-independent
      const float a = expf(IO::ld(lg_item + k) - mx) * inv;
      if (glog_item) IO::st(glog_item + k, a * (park[3 * k] - sad));
      if (goff_item) IO::st2(goff_item + 2 * k, a * park[3 * k + 1], a * park[3 * k + 2]);
    } else {
      if (glog_item) {
        const float a = expf(IO::ld(lg_item + k) - mx) * inv;
        IO::st(glog_item + k, a * (park[3 * k] - sad));
      }
      if (goff_item) IO::st2(goff_item + 2 * k, park[3 * k + 1], park[3 * k + 2]);
    }
  }
  if (EPI != 2 && ref_first && sub == 0) store_ref_partial(ref_first, rx, ry, G);
}

// ---- generic: one thread per item ------------------------------------------------------------------------------------
// d, grad_off_x / a, grad_off_y / a of one in-range point; with `acc`, also its grad_value contributions. Not inlined:
// the logits pass below evaluates d a second time and must get the bits of the first.
template <typename T>
__device__ __noinline__ void bw_point_generic(const T *vl, float *acc, const T *go, const PointRec rec, int H, int W,
                                               int C, long long stp, float a, float *res) {
  using IO = BwIo<T>;
  const int tm = tap_mask_of(rec, H, W);
  const long long e0 = (static_cast<long long>(rec.h_low) * W + rec.w_low) * stp;
  const long long eo[4] = {e0, e0 + stp, e0 + W * stp, e0 + W * stp + stp};
  const float hh = 1.f - rec.lh, hw = 1.f - rec.lw;
  const float cw[4] = {hh * hw, hh * rec.lw, rec.lh * hw, rec.lh * rec.lw};
  float d = 0.f, gx = 0.f, gy = 0.f;
  for (int c = 0; c < C; ++c) {
    const float g = IO::ld(go + c);
    float v[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      v[t] = (tm & (1 << t)) ? IO::ld(vl + eo[t] + c) : 0.f;
      if (acc != nullptr && (tm & (1 << t))) atomicAdd(acc + eo[t] + c, a * cw[t] * g);
    }
    d += g * (cw[0] * v[0] + cw[1] * v[1] + cw[2] * v[2] + cw[3] * v[3]);
    gx += g * (hh * (v[1] - v[0]) + rec.lh * (v[3] - v[2]));
    gy += g * (hw * (v[2] - v[0]) + rec.lw * (v[3] - v[1]));
  }
  res[0] = d, res[1] = gx, res[2] = gy;
}

template <typename T>
__global__ void __launch_bounds__(kBwThreads) msda_bw_generic_kernel(const MsdaBwParams prm) {
  using IO = BwIo<T>;
  using R = typename BwRef<T>::type;
  const int M = prm.M, C = prm.C, Q = prm.Q, P = prm.P, G = prm.G, L = prm.L, NP = L * P;
  const T *value = static_cast<const T *>(prm.value), *off = static_cast<const T *>(prm.off);
  const T *logits = static_cast<const T *>(prm.logits);
  const R *ref = static_cast<const R *>(prm.ref);
  const long long stp = static_cast<long long>(M) * C;
  for (long long it = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; it < prm.items;
       it += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long bq = it / M;
    const int m = static_cast<int>(it - bq * M), b = static_cast<int>(bq / Q);
    const T *go = static_cast<const T *>(prm.gout) + it * C;
    float mx = -INFINITY, sum = 0.f;
    for (int k = 0; k < NP; ++k) mx = fmaxf(mx, IO::ld(logits + it * NP + k));
    for (int k = 0; k < NP; ++k) sum += expf(IO::ld(logits + it * NP + k) - mx);
    const float inv = 1.f / sum;
    float *rp = prm.ref_part ? prm.ref_part + it * G * 2 : nullptr;
    if (rp)
      for (int i = 0; i < 2 * G; ++i) rp[i] = 0.f;
    float sad = 0.f;                        // sum_j a_j d_j, complete after pass 0
    for (int pass = 0; pass < 2; ++pass) {  // 0: everything but the logits gradient; 1: the logits gradient
      if (pass == 1 && prm.glog == nullptr) break;
      long long start = 0;
      for (int l = 0, k = 0; l < L; ++l) {
        const int H = prm.shapes[2 * l], W = prm.shapes[2 * l + 1];
        const long long lvl = ((static_cast<long long>(b) * prm.S + start) * M + m) * C;
        for (int p = 0; p < P; ++p, ++k) {
          const int g = p % G;
          const PointRec rec = point_record(BwIo<R>::ld(ref + bq * 2 * G + 2 * g), BwIo<R>::ld(ref + bq * 2 * G + 2 * g + 1),
                                            IO::ld(off + (it * NP + k) * 2), IO::ld(off + (it * NP + k) * 2 + 1), H, W);
          const float a = expf(IO::ld(logits + it * NP + k) - mx) * inv;
          float res[3] = {0.f, 0.f, 0.f};
          if (rec.in_range)
            bw_point_generic<T>(value + lvl, pass == 0 && prm.gv_acc ? prm.gv_acc + lvl : nullptr, go, rec, H, W, C, stp,
                                a, res);
          if (pass == 0) {
            const float gx = a * res[1], gy = a * res[2];
            sad += a * res[0];
            if (prm.goff) {
              IO::st(static_cast<T *>(prm.goff) + (it * NP + k) * 2, gx);
              IO::st(static_cast<T *>(prm.goff) + (it * NP + k) * 2 + 1, gy);
            }
            if (rp) rp[2 * g] += static_cast<float>(W) * gx, rp[2 * g + 1] += static_cast<float>(H) * gy;
          } else {
            IO::st(static_cast<T *>(prm.glog) + it * NP + k, a * (res[0] - sad));
          }
        }
        start += static_cast<long long>(H) * W;
      }
    }
  }
}

// ---- finalisation ----------------------------------------------------------------------------------------------------
// grad_reference_points[bq, g, xy] = the items' partials summed in head order
template <typename T>
__global__ void msda_bw_ref_kernel(const float *part, T *gref, long long nbq, int M, int G2) {
  const long long n = nbq * G2;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long bq = i / G2;
    const int e = static_cast<int>(i - bq * G2);
    float s = 0.f;
    for (int m = 0; m < M; ++m) s += part[(bq * M + m) * G2 + e];
    BwIo<T>::st(gref + i, s);
  }
}

// the fp32 grad_value accumulator rounded once to the 2-byte storage type (FP16 or BF16)
template <typename T>
__global__ void msda_bw_f32_round_kernel(const float *in, T *out, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    BwIo<T>::st(out + i, in[i]);
}

// ---- host ------------------------------------------------------------------------------------------------------------
// Workspace: [fp32 grad_value accumulator, FP16 only][fp32 grad_reference_points partials, one per (item, group, xy)]
struct BwPlan {
  size_t gv, ref, total;
};
BwPlan bw_plan(bool f16, const MsdaGeom &g) {
  BwPlan pl{};
  pl.gv = 0;
  pl.ref = f16 ? align256(static_cast<size_t>(g.B) * g.S * g.M * g.C * 4) : 0;
  pl.total = pl.ref + align256(static_cast<size_t>(g.B) * g.Q * g.M * g.G * 2 * 4);
  return pl;
}

// The kernel selection rule, in one place: the lane-group kernel takes the lane-group shape with at most 64 points per
// item when every tensor it moves as 128-bit words is 16-byte aligned; everything else runs the one-thread-per-item
// kernel.
bool msda_bw_takes_c32(const MsdaBwParams &p, const MsdaGeom &g) {
  return msda_aligned({p.value, p.ref, p.off, p.logits, p.gout, p.gv_acc, p.goff, p.glog}, 16) &&
         msda_lane_group_shape(g, kBwC32MaxPoints);
}

// EPI 0: the plugin op (mask null, gout = grad_out in T). EPI 1 / 2: the fused SCA forms (gout = grad_slots, fp32
// [Q, M*C]; mask = bev_mask [B, Q]), lane-group kernel only: shapes outside its envelope return B200_ERR_UNSUPPORTED.
// T: storage type of value, offsets, logits and their gradients; R: of the reference points and their gradient.
template <typename T, int EPI, typename R = typename BwRef<T>::type>
int msda_backward(const void *value, const int32_t *shapes, const void *ref, const void *off, const void *logits,
                  const float *mask, const void *gout, void *gvalue, void *gref, void *goff, void *glog,
                  void *workspace, const MsdaGeom &g, void *stream) {
  constexpr bool kF16 = sizeof(T) == 2;  // FP16 or BF16: grad_value is accumulated in the fp32 workspace
  if (!value || !shapes || !ref || !off || !logits || !gout || !workspace) return B200_ERR_BAD_PARAM;
  if (EPI != 0 && !mask) return B200_ERR_BAD_PARAM;
  int st = msda_check_dims(g);
  if (st != B200_OK) return st;
  if (!msda_aligned({value, off, logits, gvalue, goff, glog}, sizeof(T)) || !msda_aligned({ref, gref}, sizeof(R)) ||
      !msda_aligned({gout}, EPI == 0 ? sizeof(T) : sizeof(float)) || !msda_aligned({mask, shapes}, 4) ||
      !msda_aligned({workspace}, 256))
    return B200_ERR_BAD_PARAM;
  if (!gvalue && !gref && !goff && !glog) return B200_OK;

  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const BwPlan pl = bw_plan(kF16, g);
  char *ws = static_cast<char *>(workspace);
  const long long nv = static_cast<long long>(g.B) * g.S * g.M * g.C;
  MsdaBwParams p{};
  p.value = value, p.shapes = shapes, p.ref = ref, p.off = off, p.logits = logits, p.gout = gout, p.mask = mask;
  msda_set_dims(p, g);
  p.items = static_cast<long long>(EPI == 2 ? 1 : g.B) * g.Q * g.M;
  p.gv_acc = gvalue ? (kF16 ? reinterpret_cast<float *>(ws + pl.gv) : static_cast<float *>(gvalue)) : nullptr;
  p.goff = goff, p.glog = glog;
  p.ref_part = gref ? reinterpret_cast<float *>(ws + pl.ref) : nullptr;
  const bool c32 = msda_bw_takes_c32(p, g);
  if (EPI != 0 && !c32) return B200_ERR_UNSUPPORTED;
  if (p.gv_acc && cudaMemsetAsync(p.gv_acc, 0, static_cast<size_t>(nv) * 4, s) != cudaSuccess) return B200_ERR_LAUNCH;

  if (c32) {
    constexpr int IPB = (32 / (32 / BwIo<T>::kVec)) * (kBwThreads / 32);
    const long long blocks = (p.items + IPB - 1) / IPB;
    if (blocks > 0x7fffffffll) return B200_ERR_BAD_PARAM;
    const size_t smem = static_cast<size_t>(IPB) * g.L * g.P * 3 * sizeof(float);
    if (cudaFuncSetAttribute(msda_bw_c32_kernel<T, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             IPB * kBwC32MaxPoints * 3 * static_cast<int>(sizeof(float))) != cudaSuccess)
      return B200_ERR_LAUNCH;
    msda_bw_c32_kernel<T, EPI><<<static_cast<unsigned>(blocks), kBwThreads, smem, s>>>(p);
  } else if constexpr (EPI == 0) {
    msda_bw_generic_kernel<T><<<msda_grid_for(p.items), kBwThreads, 0, s>>>(p);
  }
  if ((st = check_launch()) != B200_OK) return st;
  if constexpr (kF16) {
    if (gvalue) {
      msda_bw_f32_round_kernel<T><<<msda_grid_for(nv), kBwThreads, 0, s>>>(p.gv_acc, static_cast<T *>(gvalue), nv);
      if ((st = check_launch()) != B200_OK) return st;
    }
  }
  if (gref) {
    const long long nbq = static_cast<long long>(g.B) * g.Q;
    msda_bw_ref_kernel<R><<<msda_grid_for(nbq * 2 * g.G), kBwThreads, 0, s>>>(p.ref_part, static_cast<R *>(gref), nbq, g.M,
                                                                        2 * g.G);
    if ((st = check_launch()) != B200_OK) return st;
  }
  return B200_OK;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_msda_backward_workspace_size(int dtype, int batch, int spatial_size, int num_heads, int channels,
                                         int num_levels, int num_query, int num_point, int points_per_group) {
  const MsdaGeom g =
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group);
  if ((dtype != 0 && dtype != 1 && dtype != 7) || msda_check_dims(g) != B200_OK) return 0;
  return bw_plan(dtype != 0, g).total;
}


int b200_msda_backward_f32(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                           const float *sampling_offsets, const float *attn_weight, const float *grad_output,
                           float *grad_value, float *grad_reference_points, float *grad_sampling_offsets,
                           float *grad_attn_weight, void *workspace, int batch, int spatial_size, int num_heads,
                           int channels, int num_levels, int num_query, int num_point, int points_per_group,
                           void *stream) {
  return msda_backward<float, 0>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight, nullptr,
      grad_output, grad_value, grad_reference_points, grad_sampling_offsets, grad_attn_weight, workspace,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_backward_f16(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                           const void *sampling_offsets, const void *attn_weight, const void *grad_output,
                           void *grad_value, void *grad_reference_points, void *grad_sampling_offsets,
                           void *grad_attn_weight, void *workspace, int batch, int spatial_size, int num_heads,
                           int channels, int num_levels, int num_query, int num_point, int points_per_group,
                           void *stream) {
  return msda_backward<__half, 0>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight, nullptr,
      grad_output, grad_value, grad_reference_points, grad_sampling_offsets, grad_attn_weight, workspace,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_sca_backward_f32(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                               const float *sampling_offsets, const float *attn_weight, const float *bev_mask,
                               const float *grad_slots, float *grad_value, float *grad_reference_points,
                               float *grad_sampling_offsets, float *grad_attn_weight, void *workspace, int batch,
                               int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                               int num_point, int points_per_group, void *stream) {
  return msda_backward<float, 1>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight, bev_mask,
      grad_slots, grad_value, grad_reference_points, grad_sampling_offsets, grad_attn_weight, workspace,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_sca_backward_f16(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                               const void *sampling_offsets, const void *attn_weight, const float *bev_mask,
                               const float *grad_slots, void *grad_value, void *grad_reference_points,
                               void *grad_sampling_offsets, void *grad_attn_weight, void *workspace, int batch,
                               int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                               int num_point, int points_per_group, void *stream) {
  return msda_backward<__half, 1>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight, bev_mask,
      grad_slots, grad_value, grad_reference_points, grad_sampling_offsets, grad_attn_weight, workspace,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_sca_shared_backward_f32(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                                      const float *sampling_offsets, const float *attn_weight, const float *bev_mask,
                                      const float *grad_slots, float *grad_value, float *grad_reference_points,
                                      float *grad_sampling_offsets, float *grad_attn_weight, void *workspace,
                                      int batch, int spatial_size, int num_heads, int channels, int num_levels,
                                      int num_query, int num_point, int points_per_group, void *stream) {
  return msda_backward<float, 2>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight, bev_mask,
      grad_slots, grad_value, grad_reference_points, grad_sampling_offsets, grad_attn_weight, workspace,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_sca_shared_backward_f16(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                                      const void *sampling_offsets, const void *attn_weight, const float *bev_mask,
                                      const float *grad_slots, void *grad_value, void *grad_reference_points,
                                      void *grad_sampling_offsets, void *grad_attn_weight, void *workspace, int batch,
                                      int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                                      int num_point, int points_per_group, void *stream) {
  return msda_backward<__half, 2>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight, bev_mask,
      grad_slots, grad_value, grad_reference_points, grad_sampling_offsets, grad_attn_weight, workspace,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

// BF16: value, offsets, logits, grad_output and their gradients in bf16; reference points and their gradient in fp32.
int b200_msda_backward_bf16(const void *value, const int32_t *spatial_shapes, const float *reference_points,
                            const void *sampling_offsets, const void *attn_weight, const void *grad_output,
                            void *grad_value, float *grad_reference_points, void *grad_sampling_offsets,
                            void *grad_attn_weight, void *workspace, int batch, int spatial_size, int num_heads,
                            int channels, int num_levels, int num_query, int num_point, int points_per_group,
                            void *stream) {
  return msda_backward<__nv_bfloat16, 0>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight,
      nullptr, grad_output, grad_value, grad_reference_points, grad_sampling_offsets, grad_attn_weight, workspace,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_sca_backward_bf16(const void *value, const int32_t *spatial_shapes, const float *reference_points,
                                const void *sampling_offsets, const void *attn_weight, const float *bev_mask,
                                const float *grad_slots, void *grad_value, float *grad_reference_points,
                                void *grad_sampling_offsets, void *grad_attn_weight, void *workspace, int batch,
                                int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                                int num_point, int points_per_group, void *stream) {
  return msda_backward<__nv_bfloat16, 1>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight,
      bev_mask, grad_slots, grad_value, grad_reference_points, grad_sampling_offsets, grad_attn_weight, workspace,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

int b200_msda_sca_shared_backward_bf16(const void *value, const int32_t *spatial_shapes,
                                       const float *reference_points, const void *sampling_offsets,
                                       const void *attn_weight, const float *bev_mask, const float *grad_slots,
                                       void *grad_value, float *grad_reference_points, void *grad_sampling_offsets,
                                       void *grad_attn_weight, void *workspace, int batch, int spatial_size,
                                       int num_heads, int channels, int num_levels, int num_query, int num_point,
                                       int points_per_group, void *stream) {
  return msda_backward<__nv_bfloat16, 2>(value, spatial_shapes, reference_points, sampling_offsets, attn_weight,
      bev_mask, grad_slots, grad_value, grad_reference_points, grad_sampling_offsets, grad_attn_weight, workspace,
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group), stream);
}

}  // extern "C"

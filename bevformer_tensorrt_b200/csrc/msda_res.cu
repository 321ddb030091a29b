// msda_res.cu — FP16 multi-scale deformable attention with the coarse pyramid levels RESIDENT IN SHARED MEMORY
// (channels == 32, levels*points <= 32, points % 4 == 0): the third-generation path of the FP16 plugin op.
//
// Why: the round-1 kernel (msda.cu) is bound by the SM's L1/LSU data path — one
// 128-byte line (tag lookup) per clock — and, for inputs whose taps miss L1, by the L2 -> L1 return path: every
// bilinear tap of a head is its own 64-byte piece of a 512-byte pixel record, four line lookups per sample. Half of the samples of a BEVFormer pyramid land in its two coarsest
// levels, which are tiny per (camera, head): 1825 pixels x 64 B = 117 KB at base shapes.
//
//   * A CTA is bound to ONE (camera, head) pair (persistent, one CTA per SM, `cpp` CTAs share a pair and interleave
//     its query blocks). It stages the TAIL of the pair's value slice — the maximal run of whole levels, counted from
//     the coarsest, that fits its shared memory — with TMA tensor loads (cp.async.bulk.tensor.2d over value viewed as
//     [B*S rows, M*32 channels], box = 128 rows x the head's 32 channels: the 64-byte slices of 128 consecutive pixels
//     land densely, [row][64 B]; SASS UTMALDG), once, and then serves every tap of those levels from shared memory.
//   * 8 lanes per item (camera, query, head), 4 items per warp. Lane = (column c, 8 channels): the two horizontally
//     adjacent taps of a sample are ONE 128-byte shared-memory wavefront (consecutive pixels are consecutive 64-byte
//     rows: conflict-free), so a sample costs 2 data-path cycles instead of 4 line lookups, and nothing crosses the
//     L2 -> L1 path. Levels outside the tail are gathered from global memory exactly like the round-1 kernel does
//     (64-byte pieces through L1), with an 8x smaller L1 footprint per CTA (one head instead of eight).
//   * Index arithmetic, softmax and tap weights are the round-1 kernel's (bit-exact index math in fp32, the owner
//     lane of a 4-point chunk folds softmax numerator x bilinear weight x validity into four fp32 tap weights and
//     hands them to its group by warp shuffles); accumulation in fp32 (HADD2.F32 widening + FFMA2).
//
// Replaces ms_deformable_im2col_cuda<__half> / _h2
// (TensorRT/plugin/multi_scale_deformable_attn/multiScaleDeformableAttnKernel.cu:1130-1169, kernels :691-846).
#include <cuda.h>  // CUtensorMap (types only; the encoder is fetched through cudaGetDriverEntryPoint)

#include "common.cuh"
#include "msda_geometry.cuh"

namespace b200 {

constexpr int kResMaxLevels = kMsdaMaxLevels;
constexpr int kBoxRows = 128;  // pixels per TMA box
#ifndef B200_RES_WARPS
#define B200_RES_WARPS 24
#endif
constexpr int kResWarps = B200_RES_WARPS;
constexpr int kResThreads = kResWarps * 32;
constexpr int kResItemsPerBlock = kResWarps * 4;

struct ResParams {
  const char *value;
  const int32_t *shapes;
  const void *ref, *off, *logits;
  void *out;
  int B, S, M, Q, P, G, L;
  int cpp;       // CTAs per (camera, head) pair
  int cap_rows;  // shared-memory capacity in pixels (multiple of kBoxRows)
  int4 *trace;
};

__device__ __forceinline__ uint32_t res_smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
  return r;
}

__device__ __forceinline__ float2 res_ffma2(float2 a, float w, float2 c) {
  return make_float2(fmaf(a.x, w, c.x), fmaf(a.y, w, c.y));
}

// acc[0..7] += w * (8 halves of v)
__device__ __forceinline__ void fma8(float (&acc)[8], const uint4 v, float w) {
  float2 *a2 = reinterpret_cast<float2 *>(acc);
  a2[0] = res_ffma2(h2_to_f2(v.x), w, a2[0]);
  a2[1] = res_ffma2(h2_to_f2(v.y), w, a2[1]);
  a2[2] = res_ffma2(h2_to_f2(v.z), w, a2[2]);
  a2[3] = res_ffma2(h2_to_f2(v.w), w, a2[3]);
}

// reference points of one (camera, query): point k of a chunk uses group k % G (G in {1, 2, 4}; P % 4 == 0)
__device__ __forceinline__ void res_load_ref(const __half *p, int G, float (&px)[4], float (&py)[4]) {
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

template <bool DBG>
__global__ void __launch_bounds__(kResThreads, 1) msda_res_kernel(const ResParams prm, const __grid_constant__ CUtensorMap tmap) {
  extern __shared__ __align__(128) char tail[];  // [cap_rows][64 B]: pixels [T0, S) of this CTA's (camera, head)
  __shared__ __align__(8) unsigned long long bar;

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 3, sub = lane & 7, col = sub >> 2, cj = sub & 3;
  const int M = prm.M, Q = prm.Q, P = prm.P, G = prm.G, L = prm.L, S = prm.S;
  const int NP = L * P, NCH = NP >> 2, CPL = P >> 2;

  // ---- level table in registers (lane l < L): H, W, first pixel; the tail boundary T0 = first pixel of the finest
  // level such that everything from there to the end of the slice fits the shared-memory rows
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
    for (int d = 1; d < kResMaxLevels; d <<= 1) {
      const int t = __shfl_up_sync(kFullMask, incl, d);
      if (lane >= d) incl += t;
    }
    lvStart = incl - area;
  }
  int T0 = (lane < L && S - lvStart <= prm.cap_rows) ? lvStart : S;
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) T0 = min(T0, __shfl_xor_sync(kFullMask, T0, d));

  const uint32_t barr = res_smem_u32(&bar), tail_s = res_smem_u32(tail);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(barr) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int pairs = prm.B * M;
  const int groups = gridDim.x / prm.cpp;  // pairs in flight
  const int j = blockIdx.x % prm.cpp;
  uint32_t phase = 0;
  for (int pair = blockIdx.x / prm.cpp; pair < pairs; pair += groups) {
    const int b = pair / M, m = pair - b * M;
    // ---- stage the tail: rows b*S + T0 ... of the [B*S, M*32] view, columns of head m
    const int boxes = (S - T0 + kBoxRows - 1) / kBoxRows;
    if (boxes > 0) {
      if (threadIdx.x == 0) {
        // the buffer was last read through the generic proxy (previous pair): order those reads before the async writes
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(barr), "r"(boxes * kBoxRows * 64) : "memory");
        for (int i = 0; i < boxes; ++i)
          asm volatile(
              "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                  tail_s + i * kBoxRows * 64),
              "l"(&tmap), "r"(m * 32), "r"(b * S + T0 + i * kBoxRows), "r"(barr)
              : "memory");
      }
      uint32_t done = 0;
      while (!done)
        asm volatile("{ .reg .pred q; mbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2; selp.u32 %0, 1, 0, q; }"
                     : "=r"(done) : "r"(barr), "r"(phase) : "memory");
      phase ^= 1u;
    }

    const char *vbase = prm.value + (static_cast<long long>(b) * S * M + m) * 64 + cj * 16;
    const uint32_t tbase = tail_s + cj * 16;
    const unsigned step_b = static_cast<unsigned>(M) * 64u;  // bytes between horizontally adjacent pixels

    for (long long qb = static_cast<long long>(j) * kResItemsPerBlock; qb < Q; qb += static_cast<long long>(prm.cpp) * kResItemsPerBlock) {
      const long long q_raw = qb + warp * 4 + g;
      const bool active = q_raw < Q;
      const long long bq = static_cast<long long>(b) * Q + (active ? q_raw : Q - 1);
      const long long it = bq * M + m;
      const __half *off_item = static_cast<const __half *>(prm.off) + it * NP * 2;
      const __half *lg_item = static_cast<const __half *>(prm.logits) + it * NP;
      __half *out_item = static_cast<__half *>(prm.out) + it * 32 + cj * 8;

      // ---- phase A (bit-exact): lane `sub` owns chunk `sub` (4 consecutive points of one level)
      const bool have = sub < NCH;
      const int cc = have ? sub : 0;
      const int lv = cc / CPL;
      const int H = __shfl_sync(kFullMask, lvH, lv), W = __shfl_sync(kFullMask, lvW, lv);
      const int start = __shfl_sync(kFullMask, lvStart, lv);
      float rpx[4], rpy[4];
      res_load_ref(static_cast<const __half *>(prm.ref) + bq * 2 * G, G, rpx, rpy);
      float him[4], wim[4];
      unsigned inr = 0;
      {
        const uint4 a = ldg128_stream(off_item + cc * 8);
        const float2 p0 = h2_to_f2(a.x), p1 = h2_to_f2(a.y), p2 = h2_to_f2(a.z), p3 = h2_to_f2(a.w);
        const float ox[4] = {p0.x, p1.x, p2.x, p3.x}, oy[4] = {p0.y, p1.y, p2.y, p3.y};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wim[k] = __fadd_rn(__fmaf_rn(rpx[k], static_cast<float>(W), ox[k]), -0.5f);
          him[k] = __fadd_rn(__fmaf_rn(rpy[k], static_cast<float>(H), oy[k]), -0.5f);
          const bool ok = have && him[k] > -1.f && wim[k] > -1.f && him[k] < static_cast<float>(H) && wim[k] < static_cast<float>(W);
          inr |= ok ? (1u << k) : 0u;
        }
      }
      const unsigned vm = __ballot_sync(kFullMask, inr != 0u);
      if (vm == 0u) {  // nothing of the warp's items is in range: exact zeros, logits are never read
        if (active && col == 0) stg128_stream(out_item, make_uint4(0u, 0u, 0u, 0u));
        continue;
      }
      // ---- phase B: softmax statistics over the item's NP logits (8 lanes)
      float lg[4];
      if (have) {
        const uint2 a = ldg64_stream(lg_item + cc * 4);
        const float2 p0 = h2_to_f2(a.x), p1 = h2_to_f2(a.y);
        lg[0] = p0.x, lg[1] = p0.y, lg[2] = p1.x, lg[3] = p1.y;
      } else {
        lg[0] = lg[1] = lg[2] = lg[3] = -INFINITY;
      }
      float mx = fmaxf(fmaxf(lg[0], lg[1]), fmaxf(lg[2], lg[3]));
#pragma unroll
      for (int d = 1; d < 8; d <<= 1) mx = fmaxf(mx, __shfl_xor_sync(kFullMask, mx, d));
      float sum = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) lg[k] = expf(lg[k] - mx), sum += lg[k];
#pragma unroll
      for (int d = 1; d < 8; d <<= 1) sum += __shfl_xor_sync(kFullMask, sum, d);

      // ---- phase C (owner): per point, the pixel of the top-left tap (bit 0: column step usable, bit 1: row step usable)
      // and the four tap weights = bilinear weight x softmax numerator x tap validity
      unsigned code[4];
      float tw[4][4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const bool ok = (inr >> k) & 1u;
        const float hf = floorf(him[k]), wf = floorf(wim[k]);
        const int h_low = ok ? static_cast<int>(hf) : 0, w_low = ok ? static_cast<int>(wf) : 0;
        const float lh = __fsub_rn(him[k], hf), lw = __fsub_rn(wim[k], wf), hh = 1.f - lh, hw = 1.f - lw;
        const bool t = h_low >= 0, bt = h_low + 1 <= H - 1, lf = w_low >= 0, rt = w_low + 1 <= W - 1;
        const unsigned pix = static_cast<unsigned>(start + (ok ? max(h_low, 0) * W + max(w_low, 0) : 0));
        code[k] = (pix << 2) | ((ok && lf && rt) ? 1u : 0u) | ((ok && t && bt) ? 2u : 0u);
        const float e = lg[k];
        tw[k][0] = (ok && t && lf) ? hh * hw * e : 0.f, tw[k][1] = (ok && t && rt) ? hh * lw * e : 0.f;
        tw[k][2] = (ok && bt && lf) ? lh * hw * e : 0.f, tw[k][3] = (ok && bt && rt) ? lh * lw * e : 0.f;
        if (DBG && active && have) {
          const int tm = ((t && lf) ? 1 : 0) | ((t && rt) ? 2 : 0) | ((bt && lf) ? 4 : 0) | ((bt && rt) ? 8 : 0);
          prm.trace[it * NP + cc * 4 + k] = ok ? make_int4(1, h_low, w_low, tm) : make_int4(0, 0, 0, 0);
        }
      }

      // ---- gather: lane = (column col, channels 8*cj .. 8*cj+7)
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll 1
      for (int ch = 0; ch < NCH; ++ch) {
        if ((vm & (0x01010101u << ch)) == 0u) continue;  // warp-uniform: chunk out of range for every item
        const int src = (lane & 24) | ch;
        const int lvc = ch / CPL;
        const int Wc = __shfl_sync(kFullMask, lvW, lvc);
        const int startc = __shfl_sync(kFullMask, lvStart, lvc);
        unsigned pa[4], pb[4];
        const unsigned inp = __shfl_sync(kFullMask, inr, src);  // the owner's range bits of this chunk's four points
        float wt[4], wb[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const unsigned cd = __shfl_sync(kFullMask, code[k], src);
          const float w0 = __shfl_sync(kFullMask, tw[k][0], src), w1 = __shfl_sync(kFullMask, tw[k][1], src);
          const float w2 = __shfl_sync(kFullMask, tw[k][2], src), w3 = __shfl_sync(kFullMask, tw[k][3], src);
          wt[k] = col ? w1 : w0, wb[k] = col ? w3 : w2;
          // a neighbour outside the image carries weight 0 and aliases one of the point's own in-image taps; a point
          // out of range altogether (bit k of inp clear) aliases the level's first pixel and is left out of the sum
          pa[k] = (cd >> 2) + (static_cast<unsigned>(col) & cd & 1u);
          pb[k] = pa[k] + ((cd & 2u) ? static_cast<unsigned>(Wc) : 0u);
        }
        uint4 va[4], vb[4];
        if (startc >= T0) {  // warp-uniform: this level lives in shared memory
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            va[k] = lds128(tbase + (pa[k] - static_cast<unsigned>(T0)) * 64u);
            vb[k] = lds128(tbase + (pb[k] - static_cast<unsigned>(T0)) * 64u);
          }
        } else {
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            va[k] = ldg128(vbase + static_cast<unsigned long long>(pa[k]) * step_b);
            vb[k] = ldg128(vbase + static_cast<unsigned long long>(pb[k]) * step_b);
          }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (!((inp >> k) & 1u)) continue;
          fma8(acc, va[k], wt[k]);
          fma8(acc, vb[k], wb[k]);
        }
      }
      // the two columns of a sample live in lanes sub and sub ^ 4
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += __shfl_xor_sync(kFullMask, acc[i], 4);
      if (active && col == 0) {
        const float inv = 1.f / sum;
        stg128_stream(out_item, make_uint4(f2_to_h2(acc[0] * inv, acc[1] * inv), f2_to_h2(acc[2] * inv, acc[3] * inv),
                                           f2_to_h2(acc[4] * inv, acc[5] * inv), f2_to_h2(acc[6] * inv, acc[7] * inv)));
      }
    }
    __syncthreads();  // every warp is done with the tail before the next pair's copies overwrite it
  }
}

// ---- host -----------------------------------------------------------------------------------------------------------
typedef CUresult (*ResEncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                     const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static ResEncodeTiledFn res_encoder() {
  static std::atomic<ResEncodeTiledFn> cached{nullptr};
  ResEncodeTiledFn fn = cached.load(std::memory_order_acquire);
  if (!fn) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || !p) return nullptr;
    fn = reinterpret_cast<ResEncodeTiledFn>(p);
    cached.store(fn, std::memory_order_release);
  }
  return fn;
}

int msda_res_f16(const void *value, const int32_t *shapes, const void *ref, const void *off, const void *logits,
                 void *out, int4 *trace, const MsdaGeom &g, int cap_bytes, cudaStream_t s) {
  // msda_check_dims has bounded L by kResMaxLevels and (S + 1) * M * 64 by 2^30
  if (!msda_lane_group_shape(g, 32)) return B200_ERR_UNSUPPORTED;
  if (!msda_aligned({value, off, logits, out, ref}, 16) || !msda_aligned({shapes}, 8)) return B200_ERR_UNSUPPORTED;
  if (static_cast<long long>(g.B) * g.S >= (1ll << 31)) return B200_ERR_UNSUPPORTED;
  ResEncodeTiledFn encode = res_encoder();
  if (!encode) return B200_ERR_LAUNCH;
  // value viewed as [B*S rows][M*32 halves]; box = the 32 channels of one head x 128 rows, dense in shared memory
  CUtensorMap tm;
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(g.M) * 32, static_cast<cuuint64_t>(g.B) * g.S};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(g.M) * 64};
  const cuuint32_t box[2] = {32, kBoxRows};
  const cuuint32_t estr[2] = {1, 1};
  if (encode(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(value), gdim, gstride, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return B200_ERR_LAUNCH;

  ResParams p{};
  p.value = static_cast<const char *>(value), p.shapes = shapes, p.ref = ref, p.off = off, p.logits = logits, p.out = out;
  p.B = g.B, p.S = g.S, p.M = g.M, p.Q = g.Q, p.P = g.P, p.G = g.G, p.L = g.L, p.trace = trace;
  const MsdaSlabGrid sg = msda_slab_grid(g, msda_sm_count(), kResItemsPerBlock);
  p.cpp = sg.cpp;
  // never more rows than the slice has (small shapes), always whole boxes
  int cap_rows = cap_bytes / 64 / kBoxRows * kBoxRows;
  const int need = (g.S + kBoxRows - 1) / kBoxRows * kBoxRows;
  if (cap_rows > need) cap_rows = need;
  if (cap_rows < kBoxRows) cap_rows = kBoxRows;
  p.cap_rows = cap_rows;
  const int smem = cap_rows * 64;
  auto launch = [&](auto kernel) -> int {
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return B200_ERR_LAUNCH;
    kernel<<<sg.grid, kResThreads, smem, s>>>(p, tm);
    return check_launch();
  };
  return trace ? launch(msda_res_kernel<true>) : launch(msda_res_kernel<false>);
}

}  // namespace b200

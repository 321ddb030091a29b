// dcn_fused.cu — DCNv2 as ONE fused implicit GEMM on the Hopper tensor cores (wgmma), FP16.
//
// out[b, co, p] = bias[co] + sum_{t, c} W[co, c, t] * mask[b,t,p] * bilinear(x[b, c], p, t)     (reference:
// modulatedDeformableConv2dKernel.cu:259-318 im2col + :735-759 cuBLAS GEMM + bias kernel, with a 26.7 MB column buffer
// per image in between). Here the column tile never exists in global memory:
//
//   GEMM view   D[M = Co, N = output pixels of one image] += A[M, K] * B[N, K]^T,  K = kh*kw*C ordered
//               (64-channel chunk, tap, channel)
//   A (weights) : pre-permuted once per call to [Co][C/64][tap][64] (K-major rows); thread 0 copies each k-block slice
//                 by TMA, one k-block ahead, into shared memory in the canonical K-major SWIZZLE_128B layout (128-byte
//                 rows, 16-byte chunks XOR row&7), completion counted in bytes on the stage's mbarrier.
//   B (columns) : GATHERED by the 16 compute warps straight into the same canonical layout: the input is first brought to
//                 NHWC so that the 64 channels of a k-block are 128 contiguous bytes per bilinear corner; a thread
//                 does 4 x LDG.128, blends 8 channels with the (mask-folded) corner weights, packs to fp16 and
//                 issues one swizzled STS.128. Sampling positions / corner weights of the tile's pixels x kh*kw taps
//                 are computed once per tile into a shared-memory table (fp32, op-for-op the reference's index math).
//   MMA         : the same 16 warps form 4 warpgroups; each issues wgmma.mma_async m64nNk16 (f16 in, fp32 accumulators
//                 in registers) on its share of the Co x pixels tile, straight from the shared-memory stage. The
//                 wgmma of k-block kb runs while the warps gather k-block kb+1; a stage is released on its "empty"
//                 mbarrier once wgmma.wait_group shows the MMAs that read it have completed.
//   epilogue    : accumulators -> +bias -> fp16 (or requantised int8) -> NCHW rows.
// Persistent CTAs (one per SM) loop over (image, pixel tile) work items.
//
// Requirements of this path (otherwise dcn.cu's v1 path runs): FP16, groups == 1, deformable_groups == 1,
// C % 64 == 0, Co in {128, 256, 512}, kh*kw <= 9.
#include <cuda.h>  // CUtensorMap (types only; the encoder is fetched through cudaGetDriverEntryPoint)

#include "dcn_geometry.cuh"

namespace b200 {

constexpr int kBK = 64;           // channels per k-block: 64 fp16 = one 128-byte swizzle row
constexpr int kGatherWarps = 16;  // 4 warpgroups: 512 gather threads (the kernel is latency-bound on the corner loads)
constexpr int kWarpGroups = kGatherWarps / 4;
constexpr int kFusedThreads = kGatherWarps * 32;  // thread 0 also issues the weight TMA
constexpr int kMaxTaps = 9;

struct DcnFusedParams {
  const __half *x_nhwc, *w_r;
  const void *bias, *offset, *mask;  // FP16 path: __half; INT8 path: offset/mask int8, bias float (converted by the host)
  void *out;                         // FP16 path: __half; INT8 path: int8
  float scale_off, scale_mask, out_mul, out_div;  // INT8 path: dequant scales; out = T2int8((acc*out_mul + bias)/out_div)
  float out_inv;                                  // 1 / out_div, rounded once on the host
  int B, C, H, W, Co, kh, kw, pad_h, pad_w, stride_h, stride_w, dil_h, dil_w, Ho, Wo;
  int tiles_per_img, num_tiles, kb_per_tap, num_kb;
};

// What a sample outside the image loads in the gather (eight fp16 zeros, never written).
__device__ const uint4 g_dcn_zero_tap = {0u, 0u, 0u, 0u};

struct __align__(16) TapEntry {  // 16 bytes: one LDS.128 / STS.128
  int pix;       // (h0*W + w0) of the top-left corner, clamped into the image
  int step;      // bit0: column neighbour usable, bit1: row neighbour usable, bit2: the sample is inside the image
  uint32_t w12;  // fp16 pair: corner weights (top-left, top-right), mask folded in
  uint32_t w34;  // fp16 pair: (bottom-left, bottom-right)
};

// ---- PTX wrappers ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// K-major, SWIZZLE_128B shared-memory matrix descriptor (sm_90 GMMA): start>>4 | LBO(=1, unused when swizzled) |
// SBO = 1024 B (8 rows x 128 B) | layout SWIZZLE_128B (1 << 62). Advancing K by 16 fp16 adds 32 bytes to the start.
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
  return static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | (static_cast<uint64_t>(1024 >> 4) << 32) |
         (1ull << 62);
}
// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, both operands K-major in shared memory; acc == 0 overwrites D.
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t acc);
template <>
__device__ __forceinline__ void wgmma_f16<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(acc));
}
template <>
__device__ __forceinline__ void wgmma_f16<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(acc));
}

// ---- pre-passes -----------------------------------------------------------------------------------------------------
// NCHW -> NHWC (fp16): 64 channels x 64 pixels per block through shared memory; 128-bit global accesses on both sides
// when HW % 8 == 0 (rows of the NCHW planes are then 16-byte aligned), scalar loads otherwise.
__global__ void __launch_bounds__(512) dcn_nchw_to_nhwc_kernel(const __half *__restrict__ in, __half *__restrict__ out,
                                                               int C, int HW) {
  __shared__ __half tile[64][66];  // row stride 33 words: column reads are conflict-free
  const int b = blockIdx.z, p0 = blockIdx.x * 64, c0 = blockIdx.y * 64;
  const int t = threadIdx.x;
  {
    const int c = t >> 3, pj = (t & 7) * 8;  // 64 channel rows x 8 chunks of 8 pixels
    const __half *src = in + (static_cast<long long>(b) * C + c0 + c) * HW + p0 + pj;
    if ((HW & 7) == 0 && p0 + pj + 8 <= HW) {
      const uint4 v = ldg128(src);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) *reinterpret_cast<uint32_t *>(&tile[c][pj + 2 * i]) = w[i];
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) tile[c][pj + i] = (p0 + pj + i < HW) ? src[i] : __float2half(0.f);
    }
  }
  __syncthreads();
  {
    const int pp = t >> 3, cj = (t & 7) * 8;  // 64 pixels x 8 chunks of 8 channels
    if (p0 + pp < HW) {
      uint32_t w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const __half2 h = __halves2half2(tile[cj + 2 * i][pp], tile[cj + 2 * i + 1][pp]);
        w[i] = *reinterpret_cast<const uint32_t *>(&h);
      }
      *reinterpret_cast<uint4 *>(out + (static_cast<long long>(b) * HW + p0 + pp) * C + c0 + cj) =
          make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
}

// W[co][c][t] -> Wr[co][k],  k = (c / 64) * (kk * 64) + t * 64 + (c % 64): K is ordered (channel chunk, tap, channel).
// Consecutive k-blocks are then the kh*kw taps of ONE 64-channel chunk, whose bilinear corners overlap spatially, so the
// gather of tap t+1 mostly hits in L1 what tap t brought in.
__global__ void dcn_weight_reorder_kernel(const __half *__restrict__ w, __half *__restrict__ wr, int Co, int C, int kk) {
  const long long n = static_cast<long long>(Co) * C * kk;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % kBK);
    const int t = static_cast<int>((i / kBK) % kk);
    const int cc = static_cast<int>((i / (static_cast<long long>(kBK) * kk)) % (C / kBK));
    const long long co = i / (static_cast<long long>(C) * kk);
    wr[i] = w[(co * C + cc * kBK + ci) * kk + t];
  }
}

// T2int8(real / div) of the INT8 epilogue (…Conv2dKernel.cu:578-579, T2int8 :51-55) without the generic division
// sequence (reciprocal, fix-ups, slow-path check: ~10 issue slots on each of 65 k outputs per tile, on the warps that
// also feed the tensor core): quotient from the host-rounded reciprocal plus one Newton step on the exact remainder
// (two FMAs) — the correctly rounded quotient except for isolated last-bit cases, which move a result only when it sits
// within 2^-24 of a rounding boundary. Saturation and round-half-away-from-zero in one conversion: trunc(q + copysign(0.5, q))
// with cvt.sat clamps to [-128, 127] exactly like the clamp-then-round of to_int8_sat (NaN -> 0 in both).
__device__ __forceinline__ int requant_i8(float real, float div, float inv) {
  float q = real * inv;
  q = fmaf(fmaf(-q, div, real), inv, q);
  const float h = __uint_as_float((__float_as_uint(q) & 0x80000000u) | 0x3f000000u);
  int r;
  asm("cvt.rzi.sat.s8.f32 %0, %1;" : "=r"(r) : "f"(q + h));
  return r;
}

// ---- the fused kernel -----------------------------------------------------------------------------------------------
template <int MH>
struct FusedCfg {
  // The fp32 accumulators live in the registers of the 4 warpgroups: Co x kBN floats over 512 threads. Co = 128 and 256
  // take 128-pixel tiles, Co = 512 64-pixel tiles (64 accumulator registers a thread at most, beside the gather's 32).
  static constexpr int kMB = 2 * MH;                              // 64-row blocks of Co (wgmma M = 64)
  static constexpr int kBN = MH <= 2 ? 128 : 64;                  // output pixels per tile
  static constexpr int kMPW = MH <= 2 ? 1 : 2;                    // row blocks per warpgroup
  static constexpr int kNSplit = kWarpGroups * kMPW / kMB;        // warpgroups sharing a row block split the pixels
  static constexpr int kWN = kBN / kNSplit;                       // wgmma N
  static_assert(kMB / kMPW * kNSplit == kWarpGroups && (kWN == 64 || kWN == 128), "warpgroup split");
  static constexpr int kABytes = MH * 128 * 128;  // Co rows x 128 B
  static constexpr int kBBytes = kBN * 128;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kTableBytes = kMaxTaps * kBN * static_cast<int>(sizeof(TapEntry));
  static constexpr int kStages = (220 * 1024 - kTableBytes) / kStageBytes >= 4 ? 4 : (220 * 1024 - kTableBytes) / kStageBytes;
  static constexpr int kSmemBytes = 1024 /*align slack*/ + kStages * kStageBytes + kTableBytes + 256 /*barriers*/;
  static_assert(kStages >= 2 && kSmemBytes <= 227 * 1024, "tile does not fit shared memory");
};

// I8 = true: the INT8 plugin flavour computed by in-register dequantisation — the pre-passes hand this kernel the int8
// activations / weights as (exact) fp16 integers, offsets and masks are dequantised while the sampling table is built,
// the fp32 accumulators are rescaled by scale_in*scale_w, biased and requantised once (T2int8) in the epilogue.
template <int MH, bool I8>
__global__ void __launch_bounds__(kFusedThreads, 1) dcn_fused_kernel(const DcnFusedParams p,
                                                                     const __grid_constant__ CUtensorMap tmap_w) {
  using Cfg = FusedCfg<MH>;
  constexpr int S = Cfg::kStages;
  constexpr int kBN = Cfg::kBN, kWN = Cfg::kWN, kMPW = Cfg::kMPW;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t *stage_base = smem;
  TapEntry *table = reinterpret_cast<TapEntry *>(smem + S * Cfg::kStageBytes);
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem + S * Cfg::kStageBytes + Cfg::kTableBytes);  // [0..S) full, [S..2S) empty

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + S);

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full0 + 8 * s, kGatherWarps + 1);  // 16 gather warps + thread 0's expect_tx arrive
      mbar_init(empty0 + 8 * s, kGatherWarps);     // every warp, once its warpgroup's MMAs on the stage completed
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int HoWo = p.Ho * p.Wo, HW = p.H * p.W, kk = p.kh * p.kw;
  const int my_tiles = (p.num_tiles - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / gridDim.x;

  // weight slice (A) of the kbt-th k-block of this CTA into its stage: cp.async.bulk.tensor writes each [128 rows x 64 k]
  // box in the same 128-byte-swizzled layout the GMMA descriptor expects (issued by thread 0 only)
  const auto issue_weights = [&](uint32_t q) {
    const int s = q % S;
    mbar_wait(empty0 + 8 * s, ((q / S) & 1) ^ 1);
    const uint32_t bar = full0 + 8 * s;
    const uint32_t dst = smem_u32(stage_base + s * Cfg::kStageBytes);
    const int kb = static_cast<int>(q % static_cast<uint32_t>(p.num_kb));
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(Cfg::kABytes) : "memory");
#pragma unroll
    for (int mh = 0; mh < MH; ++mh)
      asm volatile(
          "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
          ::"r"(dst + mh * 16384), "l"(&tmap_w), "r"(kb * kBK), "r"(mh * 128), "r"(bar)
          : "memory");
  };
  const uint32_t total_kb = static_cast<uint32_t>(my_tiles) * static_cast<uint32_t>(p.num_kb);
  if (threadIdx.x == 0 && total_kb > 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_w) : "memory");
    issue_weights(0);
  }
  {
    // =================================== gather + MMA + epilogue ===================================
    const int pt = threadIdx.x;  // 0..kGatherWarps*32-1
    // this warpgroup's share of the tile: kMPW 64-row blocks of Co from mb0, kWN pixels from n0
    const int wg = warp >> 2;
    const int mb0 = (wg % (Cfg::kMB / kMPW)) * kMPW, n0 = (wg / (Cfg::kMB / kMPW)) * kWN;
    float acc[kMPW][kWN / 2];
#pragma unroll
    for (int m = 0; m < kMPW; ++m)
#pragma unroll
      for (int i = 0; i < kWN / 2; ++i) acc[m][i] = 0.f;
    uint32_t kbt = 0;
    for (int it = 0; it < my_tiles; ++it) {
      const int tile = blockIdx.x + it * gridDim.x;
      const int b = tile / p.tiles_per_img;
      const int p0 = (tile - b * p.tiles_per_img) * kBN;

      // ---- sampling table of this tile: (tap, pixel) -> clamped corner + mask-folded bilinear weights. Every warp has
      // passed the full barrier of the previous tile's last k-block, so nobody still reads the previous table.
      for (int e = pt; e < kk * kBN; e += kGatherWarps * 32) {
        const int n = e % kBN, t = e / kBN;
        const int pix = p0 + n;
        TapEntry te{0, 0, 0u, 0u};
        if (pix < HoWo) {
          const int h_col = pix / p.Wo, w_col = pix - h_col * p.Wo;
          const int i = t / p.kw, j = t - i * p.kw;
          const long long oi = (static_cast<long long>(b) * 2 * kk + 2 * t) * HoWo + pix;
          const long long mi = (static_cast<long long>(b) * kk + t) * HoWo + pix;
          float oh, ow, m;
          if (I8) {  // off*scale rounded to fp32 first, like the reference INT8 im2col (…Conv2dKernel.cu:509-514)
            oh = static_cast<float>(__ldg(static_cast<const int8_t *>(p.offset) + oi)) * p.scale_off;
            ow = static_cast<float>(__ldg(static_cast<const int8_t *>(p.offset) + oi + HoWo)) * p.scale_off;
            m = static_cast<float>(__ldg(static_cast<const int8_t *>(p.mask) + mi)) * p.scale_mask;
          } else {
            oh = __half2float(__ldg(static_cast<const __half *>(p.offset) + oi));
            ow = __half2float(__ldg(static_cast<const __half *>(p.offset) + oi + HoWo));
            m = __half2float(__ldg(static_cast<const __half *>(p.mask) + mi));
          }
          const float h_im = __fadd_rn(static_cast<float>(h_col * p.stride_h - p.pad_h + i * p.dil_h), oh);
          const float w_im = __fadd_rn(static_cast<float>(w_col * p.stride_w - p.pad_w + j * p.dil_w), ow);
          if (h_im > -1.f && w_im > -1.f && h_im < static_cast<float>(p.H) && w_im < static_cast<float>(p.W)) {
            const float hf = floorf(h_im), wf = floorf(w_im);
            const int h_low = static_cast<int>(hf), w_low = static_cast<int>(wf);
            const float lh = __fsub_rn(h_im, hf), lw = __fsub_rn(w_im, wf), hh = 1.f - lh, hw = 1.f - lw;
            const bool tp = h_low >= 0, bt = h_low + 1 <= p.H - 1, lf = w_low >= 0, rt = w_low + 1 <= p.W - 1;
            te.pix = max(h_low, 0) * p.W + max(w_low, 0);
            te.step = ((lf && rt) ? 1 : 0) | ((tp && bt) ? 2 : 0) | 4;
            te.w12 = f2_to_h2((tp && lf) ? hh * hw * m : 0.f, (tp && rt) ? hh * lw * m : 0.f);
            te.w34 = f2_to_h2((bt && lf) ? lh * hw * m : 0.f, (bt && rt) ? lh * lw * m : 0.f);
          } else {
            // a sample outside the image is the reference's `0 * mask` whatever the image holds (0 * Inf is NaN): bit 2
            // of step stays clear and the gather reads a vector of zeros for it, not pixel 0; the first weight keeps the
            // sign / NaN of the mask
            te.w12 = f2_to_h2(0.f * m, 0.f);
          }
        }
        table[e] = te;
      }
      asm volatile("bar.sync 1, %0;" ::"n"(kGatherWarps * 32) : "memory");

      // ---- k-blocks: gather the column tile (B) of k-block kb into stage s, then multiply the stage
      constexpr int kRowsPerPass = kGatherWarps * 32 / 8;
      const int j8 = pt & 7, rowp = pt >> 3;  // 16-byte chunk within the 128-byte row; row within a pass
      const __half *xb = p.x_nhwc + static_cast<long long>(b) * HW * p.C;
      constexpr int kPasses = kBN / kRowsPerPass;
      for (int kb = 0; kb < p.num_kb; ++kb, ++kbt) {
        const int s = kbt % S;
        uint8_t *a_st = stage_base + s * Cfg::kStageBytes;
        uint8_t *b_st = a_st + Cfg::kABytes;
        const int cc = kb / kk, t = kb - cc * kk;  // K order: (channel chunk, tap, channel)
        // Issue every corner load of this k-block first and only then wait for the stage to be free: the loads fly
        // while the tensor cores still read the stage's previous contents. (The weight slice A arrives by TMA.)
        TapEntry te[kPasses];
        uint4 v[kPasses][4];
#pragma unroll
        for (int pass = 0; pass < kPasses; ++pass) te[pass] = table[t * kBN + pass * kRowsPerPass + rowp];
#pragma unroll
        for (int pass = 0; pass < kPasses; ++pass) {
          const __half *c00 = (te[pass].step & 4) ? xb + static_cast<long long>(te[pass].pix) * p.C + cc * kBK + j8 * 8
                                                  : reinterpret_cast<const __half *>(&g_dcn_zero_tap);
          const int dx = (te[pass].step & 1) ? p.C : 0, dy = (te[pass].step & 2) ? p.W * p.C : 0;
          v[pass][0] = ldg128(c00), v[pass][1] = ldg128(c00 + dx), v[pass][2] = ldg128(c00 + dy),
          v[pass][3] = ldg128(c00 + dy + dx);
        }
        mbar_wait(empty0 + 8 * s, ((kbt / S) & 1) ^ 1);
#pragma unroll
        for (int pass = 0; pass < kPasses; ++pass) {
          const int n = pass * kRowsPerPass + rowp;
          // The column operand is FP16 in any case (tensor-core input); blending the four corners with packed HFMA2
          // (fp16 weights = mask x bilinear, <= 1) instead of fp32 costs two extra 2^-11 roundings on values that are
          // then summed over K = kh*kw*C with fp32 accumulation — far below the FP16 output rounding — and removes all
          // conversions from the gather's inner loop (the reference's FP16 im2col is fp16 arithmetic too, :321-388).
          const __half2 w12 = *reinterpret_cast<const __half2 *>(&te[pass].w12);
          const __half2 w34 = *reinterpret_cast<const __half2 *>(&te[pass].w34);
          const __half2 w1 = __low2half2(w12), w2 = __high2half2(w12), w3 = __low2half2(w34), w4 = __high2half2(w34);
          const uint32_t a[4] = {v[pass][0].x, v[pass][0].y, v[pass][0].z, v[pass][0].w};
          const uint32_t bq[4] = {v[pass][1].x, v[pass][1].y, v[pass][1].z, v[pass][1].w};
          const uint32_t c[4] = {v[pass][2].x, v[pass][2].y, v[pass][2].z, v[pass][2].w};
          const uint32_t d[4] = {v[pass][3].x, v[pass][3].y, v[pass][3].z, v[pass][3].w};
          uint32_t o[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            __half2 r = __hmul2(w1, *reinterpret_cast<const __half2 *>(&a[q]));
            r = __hfma2(w2, *reinterpret_cast<const __half2 *>(&bq[q]), r);
            r = __hfma2(w3, *reinterpret_cast<const __half2 *>(&c[q]), r);
            r = __hfma2(w4, *reinterpret_cast<const __half2 *>(&d[q]), r);
            o[q] = *reinterpret_cast<const uint32_t *>(&r);
          }
          *reinterpret_cast<uint4 *>(b_st + n * 128 + ((j8 ^ (n & 7)) << 4)) = make_uint4(o[0], o[1], o[2], o[3]);
        }
        fence_proxy_async();  // make the generic-proxy stores visible to the tensor-core (async) proxy
        __syncwarp();
        if (lane == 0) mbar_arrive(full0 + 8 * s);

        // ---- MMA on stage s once every warp's columns and the TMA's weights have landed
        mbar_wait(full0 + 8 * s, (kbt / S) & 1);
        const uint32_t a_addr = smem_u32(a_st), b_addr = smem_u32(b_st) + n0 * 128;
        wgmma_fence();
#pragma unroll
        for (int k4 = 0; k4 < kBK / 16; ++k4) {
#pragma unroll
          for (int m = 0; m < kMPW; ++m)
            wgmma_f16<kWN>(acc[m], make_sw128_desc(a_addr + (mb0 + m) * 8192 + k4 * 32), make_sw128_desc(b_addr + k4 * 32),
                           (kb | k4) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the MMAs of the previous k-block have completed: release its stage
        __syncwarp();
        if (kb > 0 && lane == 0) mbar_arrive(empty0 + 8 * ((kbt - 1) % S));
        // next k-block's weights: its stage was last read by k-block kbt+1-S, which every warp has released by now
        // when S >= 3 (they passed this k-block's full barrier); with S == 2 this waits for the slowest warpgroup
        if (threadIdx.x == 0 && kbt + 1 < total_kb) issue_weights(kbt + 1);
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(empty0 + 8 * ((kbt - 1) % S));

      // ---- epilogue: registers -> +bias -> fp16 / int8 -> NCHW. Accumulator fragment of m64nN: warp w of the
      // warpgroup holds rows 16w + lane/4 (+8); register 4j + {0,1} (+{2,3} for the +8 row) holds the pixel pair
      // 8j + 2*(lane%4) + {0,1}.
      const int wr = (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int m = 0; m < kMPW; ++m) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int co = (mb0 + m) * 64 + wr + 8 * h;
          if (I8) {
            const float bias = __ldg(static_cast<const float *>(p.bias) + co);
            int8_t *orow = static_cast<int8_t *>(p.out) + (static_cast<long long>(b) * p.Co + co) * HoWo;
#pragma unroll
            for (int j = 0; j < kWN / 8; ++j) {
              const int pix = p0 + n0 + 8 * j + 2 * (lane & 3);
              // out = T2int8((acc * scale_i*scale_w + bias) / scale_o)   (…Conv2dKernel.cu:578-579)
              const int q0 = requant_i8(fmaf(acc[m][4 * j + 2 * h], p.out_mul, bias), p.out_div, p.out_inv);
              const int q1 = requant_i8(fmaf(acc[m][4 * j + 2 * h + 1], p.out_mul, bias), p.out_div, p.out_inv);
              // An INT8 row is Ho*Wo BYTES long: a pixel pair is 2-byte aligned only when the row start is.
              if (pix + 1 < HoWo && (reinterpret_cast<uintptr_t>(orow + pix) & 1) == 0) {
                *reinterpret_cast<unsigned short *>(orow + pix) =
                    static_cast<unsigned short>((q0 & 0xff) | ((q1 & 0xff) << 8));
              } else {
                if (pix < HoWo) orow[pix] = static_cast<int8_t>(q0);
                if (pix + 1 < HoWo) orow[pix + 1] = static_cast<int8_t>(q1);
              }
            }
          } else {
            const float bias = __half2float(__ldg(static_cast<const __half *>(p.bias) + co));
            __half *orow = static_cast<__half *>(p.out) + (static_cast<long long>(b) * p.Co + co) * HoWo;
#pragma unroll
            for (int j = 0; j < kWN / 8; ++j) {
              const int pix = p0 + n0 + 8 * j + 2 * (lane & 3);
              const uint32_t hw = f2_to_h2(acc[m][4 * j + 2 * h] + bias, acc[m][4 * j + 2 * h + 1] + bias);
              // Rows are Ho*Wo halves long: a pixel pair is 4-byte aligned unless Ho*Wo and co are both odd.
              if (pix + 1 < HoWo && (reinterpret_cast<uintptr_t>(orow + pix) & 3) == 0) {
                *reinterpret_cast<uint32_t *>(orow + pix) = hw;
              } else {
                unsigned short *o16 = reinterpret_cast<unsigned short *>(orow);
                if (pix < HoWo) o16[pix] = static_cast<unsigned short>(hw);
                if (pix + 1 < HoWo) o16[pix + 1] = static_cast<unsigned short>(hw >> 16);
              }
            }
          }
        }
      }
    }
  }
}

// ---- host -----------------------------------------------------------------------------------------------------------
bool dcn_fused_supported(const DcnGeom &g) {
  return g.groups == 1 && g.dg == 1 && g.C % kBK == 0 && (g.Co == 128 || g.Co == 256 || g.Co == 512) &&
         g.kh * g.kw <= kMaxTaps;
}

// Byte offsets of the workspace sections: the NHWC copy of the input, the permuted weights, and the bias vector the
// epilogue reads (FP16 zeros when there is no bias, or the INT8 flavour's fp32 bias), with room for 512 fp32 values:
// the largest Co the kernel takes.
struct DcnFusedLayout {
  size_t x, w, bias, total;
};
static DcnFusedLayout dcn_fused_layout(const DcnGeom &g) {
  DcnFusedLayout l{};
  size_t o = 0;
  l.x = o, o += align256(static_cast<size_t>(g.B) * g.H * g.W * g.C * 2);
  l.w = o, o += align256(static_cast<size_t>(g.Co) * g.C * (g.kh * g.kw) * 2);
  l.bias = o, o += 512 * sizeof(float);
  l.total = o;
  return l;
}
size_t dcn_fused_workspace_bytes(const DcnGeom &g) { return dcn_fused_layout(g).total; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 2-D tensor map over the permuted weights Wr[Co][K] (fp16): box = 64 k x 128 rows, 128-byte swizzle.
static int make_weight_tmap(CUtensorMap *tm, const __half *w_r, int Co, int K) {
  static EncodeTiledFn encode = nullptr;
  if (!encode) {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn)
      return B200_ERR_LAUNCH;
    encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(Co)};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(K) * 2};
  const cuuint32_t box[2] = {kBK, 128};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = encode(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half *>(w_r), gdim, gstride, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? B200_OK : B200_ERR_LAUNCH;
}

template <int MH, bool I8>
static int launch_fused_mh(const DcnFusedParams &p, cudaStream_t stream) {
  using Cfg = FusedCfg<MH>;
  // per launch: the attribute is per device (and this may run on several devices / host threads); the call is cheap
  if (cudaFuncSetAttribute(dcn_fused_kernel<MH, I8>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes) !=
      cudaSuccess)
    return B200_ERR_LAUNCH;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int grid = p.num_tiles < sms ? p.num_tiles : sms;
  CUtensorMap tmap;
  const int ts = make_weight_tmap(&tmap, p.w_r, p.Co, p.kh * p.kw * p.C);
  if (ts != B200_OK) return ts;
  dcn_fused_kernel<MH, I8><<<grid, kFusedThreads, Cfg::kSmemBytes, stream>>>(p, tmap);
  return check_launch();
}

// The layer, its k-block and tile counts into `p` (whose tensors are set), then the launch for Co = 128 * MH.
template <bool I8>
static int launch_fused(DcnFusedParams &p, const DcnGeom &g, cudaStream_t stream) {
  dcn_set_layer(p, g);
  p.kb_per_tap = g.C / kBK;
  p.num_kb = g.kh * g.kw * p.kb_per_tap;
  const int mh = g.Co / 128;
  const int bn = mh == 1 ? FusedCfg<1>::kBN : (mh == 2 ? FusedCfg<2>::kBN : FusedCfg<4>::kBN);
  p.tiles_per_img = (g.Ho * g.Wo + bn - 1) / bn;
  p.num_tiles = p.tiles_per_img * g.B;
  switch (mh) {
    case 1: return launch_fused_mh<1, I8>(p, stream);
    case 2: return launch_fused_mh<2, I8>(p, stream);
    case 4: return launch_fused_mh<4, I8>(p, stream);
    default: return B200_ERR_UNSUPPORTED;
  }
}

int dcn_fused_f16(const __half *input, const __half *weight, const __half *bias, const __half *offset,
                  const __half *mask, __half *output, void *workspace, const DcnGeom &g, int flags, cudaStream_t stream) {
  // flags: bit 0 = `input` is already NHWC (channels-last), bit 1 = `weight` is already permuted (b200_dcn_pack_weights_f16)
  const int kk = g.kh * g.kw, HW = g.H * g.W;
  const DcnFusedLayout l = dcn_fused_layout(g);
  uint8_t *ws = static_cast<uint8_t *>(workspace);
  __half *x_nhwc = reinterpret_cast<__half *>(ws + l.x), *w_r = reinterpret_cast<__half *>(ws + l.w);
  if (!bias) {  // the kernel always reads a bias vector (no per-thread null test in the epilogue): use zeros
    __half *zb = reinterpret_cast<__half *>(ws + l.bias);
    if (cudaMemsetAsync(zb, 0, static_cast<size_t>(g.Co) * 2, stream) != cudaSuccess) return B200_ERR_LAUNCH;
    bias = zb;
  }
  int st = B200_OK;
  if (flags & 1) {
    x_nhwc = const_cast<__half *>(input);
  } else {
    dcn_nchw_to_nhwc_kernel<<<dim3((HW + 63) / 64, g.C / 64, g.B), 512, 0, stream>>>(input, x_nhwc, g.C, HW);
    st = check_launch();
    if (st != B200_OK) return st;
  }
  if (flags & 2) {
    w_r = const_cast<__half *>(weight);
  } else {
    const long long wn = static_cast<long long>(g.Co) * g.C * kk;
    dcn_weight_reorder_kernel<<<static_cast<unsigned>((wn + 255) / 256), 256, 0, stream>>>(weight, w_r, g.Co, g.C, kk);
    st = check_launch();
    if (st != B200_OK) return st;
  }

  DcnFusedParams p{};
  p.x_nhwc = x_nhwc, p.w_r = w_r, p.bias = bias, p.offset = offset, p.mask = mask, p.out = output;
  return launch_fused<false>(p, g, stream);
}

int dcn_pack_weights_f16(const __half *weight, __half *packed, const DcnGeom &g, cudaStream_t stream) {
  const int kk = g.kh * g.kw;
  const long long wn = static_cast<long long>(g.Co) * g.C * kk;
  dcn_weight_reorder_kernel<<<static_cast<unsigned>((wn + 255) / 256), 256, 0, stream>>>(weight, packed, g.Co, g.C, kk);
  return check_launch();
}

// ---- INT8 flavour: pre-passes + launch ---------------------------------------------------------------------------------
// input kCHW4 int8 [B, C/4, H, W, 4] -> NHWC fp16 (the int8 values as exact fp16 integers): 64 pixels x 64 channels per
// block through shared memory, so that both sides are coalesced (reads: 64 consecutive pixels of a channel quad = 256
// contiguous bytes; writes: the 64 channels of a pixel = one 128-byte row)
__global__ void __launch_bounds__(256) dcn_chw4_to_nhwc_f16_kernel(const int8_t *__restrict__ in, __half *__restrict__ out,
                                                                   int C, int HW) {
  __shared__ uint32_t tile[16][65];  // [channel quad][pixel], 65: the transposed reads below are conflict-free
  const int b = blockIdx.z, p0 = blockIdx.x * 64, q0 = blockIdx.y * 16;
  const int t = threadIdx.x;
  {
    const int quad = t >> 4, pj = (t & 15) * 4;  // 16 quads x 16 groups of 4 pixels
    const uint32_t *src = reinterpret_cast<const uint32_t *>(in) + (static_cast<long long>(b) * (C / 4) + q0 + quad) * HW + p0 + pj;
#pragma unroll
    for (int i = 0; i < 4; ++i) tile[quad][pj + i] = (p0 + pj + i < HW) ? __ldg(src + i) : 0u;
  }
  __syncthreads();
  {
    const int pp = t >> 2, cj = t & 3;  // 64 pixels x 4 chunks of 16 channels
    if (p0 + pp < HW) {
      uint32_t o[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t u = tile[cj * 4 + i][pp];
        o[2 * i] = f2_to_h2(static_cast<float>(static_cast<int8_t>(u)), static_cast<float>(static_cast<int8_t>(u >> 8)));
        o[2 * i + 1] = f2_to_h2(static_cast<float>(static_cast<int8_t>(u >> 16)), static_cast<float>(static_cast<int8_t>(u >> 24)));
      }
      uint4 *dst = reinterpret_cast<uint4 *>(out + (static_cast<long long>(b) * HW + p0 + pp) * C + q0 * 4 + cj * 16);
      dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
      dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
    }
  }
}

// weight kCHW4 int8 [Co, C/4, kh, kw, 4] -> Wr fp16 [Co][C/64][t][64]
__global__ void dcn_weight_reorder_i8_kernel(const int8_t *__restrict__ w, __half *__restrict__ wr, int Co, int C, int kk) {
  const long long n = static_cast<long long>(Co) * C * kk;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ci = static_cast<int>(i % kBK);
    const int t = static_cast<int>((i / kBK) % kk);
    const int cc = static_cast<int>((i / (static_cast<long long>(kBK) * kk)) % (C / kBK));
    const long long co = i / (static_cast<long long>(C) * kk);
    const int c = cc * kBK + ci;
    wr[i] = __float2half_rn(static_cast<float>(w[((co * (C / 4) + c / 4) * kk + t) * 4 + (c & 3)]));
  }
}

// bias (float or half, may be null) -> float vector
__global__ void dcn_bias_to_f32_kernel(const void *bias, int is_half, float *out, int Co) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Co) out[i] = !bias ? 0.f : (is_half ? __half2float(static_cast<const __half *>(bias)[i]) : static_cast<const float *>(bias)[i]);
}

int dcn_fused_i8(const int8_t *input, float scale_i, const int8_t *weight, float scale_w, const void *bias, int bias_is_half,
                 const int8_t *offset, float scale_off, const int8_t *mask, float scale_mask, int8_t *output, float scale_o,
                 void *workspace, const DcnGeom &g, cudaStream_t stream) {
  const int kk = g.kh * g.kw, HW = g.H * g.W;
  const DcnFusedLayout l = dcn_fused_layout(g);
  uint8_t *ws = static_cast<uint8_t *>(workspace);
  __half *x_nhwc = reinterpret_cast<__half *>(ws + l.x), *w_r = reinterpret_cast<__half *>(ws + l.w);
  float *bias_f = reinterpret_cast<float *>(ws + l.bias);

  dcn_chw4_to_nhwc_f16_kernel<<<dim3((HW + 63) / 64, g.C / 64, g.B), 256, 0, stream>>>(input, x_nhwc, g.C, HW);
  int st = check_launch();
  if (st != B200_OK) return st;
  const long long wn = static_cast<long long>(g.Co) * g.C * kk;
  dcn_weight_reorder_i8_kernel<<<static_cast<unsigned>((wn + 255) / 256), 256, 0, stream>>>(weight, w_r, g.Co, g.C, kk);
  st = check_launch();
  if (st != B200_OK) return st;
  dcn_bias_to_f32_kernel<<<(g.Co + 255) / 256, 256, 0, stream>>>(bias, bias_is_half, bias_f, g.Co);
  st = check_launch();
  if (st != B200_OK) return st;

  DcnFusedParams p{};
  p.x_nhwc = x_nhwc, p.w_r = w_r, p.bias = bias_f, p.offset = offset, p.mask = mask, p.out = output;
  p.scale_off = scale_off, p.scale_mask = scale_mask, p.out_mul = scale_i * scale_w, p.out_div = scale_o, p.out_inv = 1.f / scale_o;
  return launch_fused<true>(p, g, stream);
}

}  // namespace b200

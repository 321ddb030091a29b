// msda_v2.cu — packed-layout INT8 multi-scale deformable attention (channels == 32, 16 <= levels*points <= 32,
// points % 4 == 0): the second-generation path of the INT8 plugin op.
//
// Why: the round-1 kernel (msda.cu) gathers each bilinear tap of a head as its own 32-byte piece out of the reference's
// value layout [S, heads, 32]. An SM's L1/LSU path retires about ONE distinct 128-byte line per clock whatever the piece
// size (so INT8 runs no faster than FP16 in that layout), and the SIMT accumulate pays 13 convert / FMA slots per 8 bytes. Both are properties of the LAYOUT, so this path changes the layout first:
//
//   1. PACK pre-pass (msda_pack_kernel): `value` is re-laid per (camera, head) as COLUMN-PAIR ENTRIES
//          entry(level, parity, r, x) = { pixel(y0, x), pixel(y0 + 1, x) },  y0 = 2r - parity,   64 bytes,
//      with the two rows interleaved per channel: [ch0:y0, ch0:y1, ch1:y0, ch1:y1, ...]; rows outside the image are
//      zeros; both parities of every level are stored (2 x the INT8 value bytes: 97 MB at base shapes, L2-resident).
//      A bilinear sample (h_low, w_low) is then exactly the two adjacent entries (r, w_low), (r, w_low + 1) of parity
//      h_low & 1: ONE 128-byte run (1.5 lines on average instead of 4 requests): 0.51-0.54 samples/clk/SM from L2 in a
//      B200 microbenchmark against 0.25 for four 32-byte taps. Value tiles enter shared memory by TMA bulk copies
//      (cp.async.bulk, SASS UBLKCP: the pixels of a row chunk are contiguous in [S, heads*32]), are interleaved by the
//      threads (conflict-free: a warp reads 256 contiguous bytes) and leave as 16-byte stores.
//   2. GATHER (msda_i8p_kernel): persistent CTAs bound to one (camera, head) slab; the slab's coarsest levels (both
//      parity copies) stay resident in shared memory after one TMA bulk-copy staging; 8 lanes per item, 4 items per warp;
//      a sample is ONE 16-byte load per lane (8 lanes x 16 B = the 128-byte run: a conflict-free shared-memory
//      wavefront for resident levels, 1.5 L1 lines otherwise) and 8 dp2a against 16-bit fixed-point tap-weight pairs
//      (details at the kernel). Weight quantisation to 16 bits: |error| <= 2^-17 per tap weight, <= 0.13 value-quanta
//      worst case over 128 taps (typically 0.006) before the division by sum(exp) >= 1 — two orders of magnitude below
//      the INT8 output step. A warp walks one block of 4 items per step; the gather has one launch shape and reads no
//      launch-shape setting of the FP32 / FP16 op.
//
// Replaces (same as msda.cu) ms_deformable_im2col_cuda_int8<float|__half2>
// (TensorRT/plugin/multi_scale_deformable_attn/multiScaleDeformableAttnKernel.cu:1172-1218, kernels :849-1104).
// The FP16 op keeps the reference layout (msda.cu's gather kernel, or the opt-in resident-tail kernel of msda_res.cu):
// for 64-byte taps the re-layout only helps where taps hit L1 (the L2 -> L1 path tops out at 70 B/clk/SM either way),
// and a tensor-core variant (mma.sync with the interleaved entry as A fragment, built and measured on B200: 3.3 ms
// against 1.03 ms) loses to fragment-order loads that touch 4 lines per quarter warp.
#include "common.cuh"
#include "msda_geometry.cuh"

namespace b200 {

constexpr int kV2MaxLevels = 8;
constexpr int kPackCols = 64;  // pixels per pack tile row
constexpr int kEB = 64;        // entry bytes

// The packed-stack plan is a pure function of spatial_shapes and is evaluated ON THE DEVICE from the same device-resident
// tensor the reference plugin receives (TensorRT hands the plugin device pointers only).
struct LevelInfo {
  int H, W;
  int pix0;    // first pixel of the level inside S
  int e0, e1;  // first entry of the parity-0 / parity-1 block inside a (camera, head) slab
  int tiles0;  // pack tiles (row pair x 64-column chunk x parity) before this level
  int tiles;   // ... and of this level
};

__device__ __forceinline__ int level_block(int H, int W) { return (H / 2 + 1) * W; }

// level `want` (want == L: totals in .e0 (entries per slab) and .tiles0)
__device__ LevelInfo plan_level(const int32_t *shapes, int L, int want) {
  LevelInfo r{};
  int e = 0, pix = 0, tiles = 0;
  for (int l = 0; l < L; ++l) {
    const int H = __ldg(shapes + 2 * l), W = __ldg(shapes + 2 * l + 1);
    const int blk = level_block(H, W);
    const int nt = (H / 2 + 1) * ((W + kPackCols - 1) / kPackCols) * 2;
    if (l == want) r.H = H, r.W = W, r.pix0 = pix, r.e0 = e, r.e1 = e + blk, r.tiles0 = tiles, r.tiles = nt;
    e += 2 * blk, pix += H * W, tiles += nt;
  }
  if (want >= L) r.e0 = e, r.tiles0 = tiles;
  return r;
}

__device__ __forceinline__ uint32_t smem_addr(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// ---------------------------------------------------------------------------------------------------------------
// 1. pack pre-pass
// ---------------------------------------------------------------------------------------------------------------
struct PackParams {
  const char *value;  // int8 [B, S, M*32]
  char *packed;       // [B, M, entries, 64]
  const int32_t *shapes;
  int B, S, M, L;
};

// One tile = one (level, parity, row pair r, 64-column chunk) of one camera: two rows x 64 pixels x (M*32) bytes arrive in
// shared memory by two TMA bulk copies, then the threads build 16-byte pieces of the interleaved entries.
// Persistent CTAs loop over the tiles (their number is known on the device only).
__global__ void __launch_bounds__(256) msda_pack_kernel(const PackParams p) {
  extern __shared__ __align__(128) char tile[];  // [2][kPackCols][M*32]
  __shared__ __align__(8) unsigned long long bar;
  __shared__ LevelInfo lvs[kV2MaxLevels + 1];
  const int b = blockIdx.y;
  if (threadIdx.x <= p.L) lvs[threadIdx.x] = plan_level(p.shapes, p.L, threadIdx.x);
  const uint32_t barr = smem_addr(&bar);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(barr) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int tiles_total = lvs[p.L].tiles0, entries = lvs[p.L].e0;
  const int pix_bytes = p.M * 32;
  const long long slab = static_cast<long long>(entries) * kEB;
  const unsigned per_x = static_cast<unsigned>(p.M * 4);  // 16-byte pieces per pixel column (all heads)
  uint32_t phase = 0;
  for (int tidx = blockIdx.x; tidx < tiles_total; tidx += gridDim.x) {
    int l = 0;
    while (l + 1 < p.L && tidx >= lvs[l].tiles0 + lvs[l].tiles) ++l;
    const LevelInfo lv = lvs[l];
    const int t = tidx - lv.tiles0;
    const int chunks = (lv.W + kPackCols - 1) / kPackCols, per_par = (lv.H / 2 + 1) * chunks;
    const int par = t / per_par, r = (t % per_par) / chunks, chunk = t % chunks;
    const int x0 = chunk * kPackCols, ncol = min(kPackCols, lv.W - x0);
    const int row_bytes = ncol * pix_bytes;
    const int y0 = 2 * r - par;
    bool valid[2];
#pragma unroll
    for (int rho = 0; rho < 2; ++rho) valid[rho] = (y0 + rho >= 0) && (y0 + rho < lv.H);
    if (threadIdx.x == 0) {
      // the tile buffer was last touched through the generic proxy (zero fill / reads of the previous tile): order
      // those accesses before the async-proxy writes of the bulk copies
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      const uint32_t tx = (valid[0] ? row_bytes : 0) + (valid[1] ? row_bytes : 0);
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(barr), "r"(tx) : "memory");
#pragma unroll
      for (int rho = 0; rho < 2; ++rho) {
        if (!valid[rho]) continue;
        const char *src = p.value + (static_cast<long long>(b) * p.S + lv.pix0 + static_cast<long long>(y0 + rho) * lv.W + x0) * pix_bytes;
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                         smem_addr(tile + rho * kPackCols * pix_bytes)),
                     "l"(src), "r"(row_bytes), "r"(barr)
                     : "memory");
      }
    }
    // rows outside the image are zeros (the gather gives them weight 0, but they must be finite)
#pragma unroll
    for (int rho = 0; rho < 2; ++rho)
      if (!valid[rho])
        for (int i = threadIdx.x; i < row_bytes / 16; i += blockDim.x)
          reinterpret_cast<uint4 *>(tile + rho * kPackCols * pix_bytes)[i] = make_uint4(0u, 0u, 0u, 0u);
    {
      uint32_t done = 0;
      while (!done)
        asm volatile("{ .reg .pred q; mbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2; selp.u32 %0, 1, 0, q; }"
                     : "=r"(done) : "r"(barr), "r"(phase) : "memory");
      phase ^= 1u;
    }
    __syncthreads();

    // piece i = (x, m, j): consecutive threads walk (m, j) first = 256 contiguous bytes of one pixel in shared memory
    // (conflict-free), 16 output bytes each: channels 8j..8j+7 of head m as (y0, y1) byte pairs
    const long long ent = static_cast<long long>(par ? lv.e1 : lv.e0) + static_cast<long long>(r) * lv.W + x0;
    const unsigned pieces = static_cast<unsigned>(ncol) * per_x;
    for (unsigned i = threadIdx.x; i < pieces; i += blockDim.x) {
      const unsigned x = i / per_x, mj = i - x * per_x, m = mj >> 2, j = mj & 3u;
      const char *s0 = tile + x * pix_bytes + m * 32 + j * 8;
      const uint2 a = *reinterpret_cast<const uint2 *>(s0);                          // row y0
      const uint2 c = *reinterpret_cast<const uint2 *>(s0 + kPackCols * pix_bytes);  // row y0 + 1, same channels
      uint4 o;  // bytes (a0 c0 a1 c1)(a2 c2 a3 c3)...
      o.x = __byte_perm(a.x, c.x, 0x5140), o.y = __byte_perm(a.x, c.x, 0x7362);
      o.z = __byte_perm(a.y, c.y, 0x5140), o.w = __byte_perm(a.y, c.y, 0x7362);
      char *dst = p.packed + (static_cast<long long>(b) * p.M + m) * slab + (ent + x) * kEB + j * 16;
      *reinterpret_cast<uint4 *>(dst) = o;
    }
    __syncthreads();  // the tile buffer is reused by the next bulk copies
  }
}

// ---------------------------------------------------------------------------------------------------------------
// 2. gather: persistent CTAs bound to one (camera, head) slab, coarse levels resident in shared memory
// ---------------------------------------------------------------------------------------------------------------
struct I8PParams {
  const char *packed;
  const void *ref;
  const int8_t *off, *logits;
  int8_t *out;
  const int32_t *shapes;
  int B, M, Q, P, G, NP, L;
  int cpp;          // CTAs per (camera, head) pair
  int cap_entries;  // shared-memory capacity in 64-byte entries
  float scale_value, scale_offset, scale_weight, scale_out;
  int4 *trace;
};

__device__ __forceinline__ int dp2a_lo(uint32_t a, uint32_t b, int c) {
  int d;
  asm("dp2a.lo.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
__device__ __forceinline__ int dp2a_hi(uint32_t a, uint32_t b, int c) {
  int d;
  asm("dp2a.hi.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
// two tap weights in [0, 1] as 16-bit fixed point, (w_y0 | w_y1 << 16)
__device__ __forceinline__ uint32_t fixed_pair(float w0, float w1) {
  uint32_t r;  // round to nearest, saturate at 65535 (w = 1.0), pack
  asm("{ .reg .u16 a, b; .reg .f32 x, y;\n\t"
      "mul.f32 x, %1, 0f47800000; mul.f32 y, %2, 0f47800000;\n\t"
      "cvt.rni.sat.u16.f32 a, x; cvt.rni.sat.u16.f32 b, y; mov.b32 %0, {a, b}; }"
      : "=r"(r) : "f"(w0), "f"(w1));
  return r;
}
__device__ __forceinline__ float deq8(uint32_t word, int byte, float s) {
  return static_cast<float>(static_cast<int8_t>(word >> (8 * byte))) * s;
}
__device__ __forceinline__ uint4 lds128_v2(uint32_t addr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
  return r;
}

#ifndef B200_I8_WARPS
#define B200_I8_WARPS 32
#endif
constexpr int kI8Warps = B200_I8_WARPS;
constexpr int kI8Threads = kI8Warps * 32;
constexpr int kI8ItemsPerWarp = 4;
constexpr int kI8ItemsPerBlock = kI8ItemsPerWarp * kI8Warps;
constexpr int kI8CopyBytes = 16384;  // one bulk copy of the tail staging

// R: reference-point storage (__half or float).
//   * CTA <-> one (camera, head) slab of the packed stack, `cpp` CTAs per slab interleaving its query blocks; the TAIL of
//     the slab — the maximal run of whole levels (both parity copies), counted from the coarsest, that fits shared memory —
//     is staged once by TMA bulk copies (the slab is contiguous; SASS UBLKCP) and every sample of those levels is ONE
//     conflict-free 128-byte shared-memory wavefront (two adjacent 64-byte entries over 8 lanes).
//   * 8 lanes per item (camera, query, head), 4 items per warp; chunk c (4 points of one level) of an item is owned by lane
//     c, which evaluates the bit-exact index arithmetic (…Kernel.cu:657-674 / :138-172: fp32, loc = fma(ref, size, off)
//     - 0.5) and the softmax numerators once and hands {entry | right-column flag, (w_y0, w_y1) of the left column, of
//     the right column as 16-bit fixed point} to its group with three shuffles per point;
//   * a sample is one 16-byte load per lane (lane = (column, 8 channels x (y0, y1))) and 8 dp2a: b = {ch_i:y0, ch_i:y1,
//     ch_j:y0, ch_j:y1}, a = (w_y0, w_y1) as u16; int32 accumulators (exact), the two columns are added by one shuffle
//     round, scale_value / (65536 * sum(exp)) / scale_out applied at the single requantisation.
template <typename R, bool DBG>
__global__ void __launch_bounds__(kI8Threads, 1) msda_i8p_kernel(const I8PParams prm) {
  extern __shared__ __align__(128) char tail[];  // entries [E0, entries) of this CTA's slab, then the per-warp records
  __shared__ __align__(8) unsigned long long bar;

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int sub = lane & 7, grp_i = lane >> 3, col = sub >> 2, cj = sub & 3;
  // per-warp sample records: [item][point k of the chunk][chunk] x {address col 0, weights col 0, address col 1, weights
  // col 1}; 33 slots per item so that the four items of a warp sit in different banks
  const uint32_t rec_s = smem_addr(tail) + static_cast<uint32_t>(prm.cap_entries) * kEB + (warp * kI8ItemsPerWarp + grp_i) * (33 * 16);
  const int M = prm.M, Q = prm.Q, P = prm.P, G = prm.G, NP = prm.NP, L = prm.L;
  const int NCH = NP >> 2, CPL = P >> 2;

  // ---- level table in registers (lane l < L): H, W, first entry of the parity-0 block (parity 1 follows at + blk)
  int lvH = 1, lvW = 1;
  if (lane < L) {
    lvH = __ldg(prm.shapes + 2 * lane), lvW = __ldg(prm.shapes + 2 * lane + 1);
  }
  const int lvBlk = lane < L ? level_block(lvH, lvW) : 0;
  int lvE0;
  {
    int incl = 2 * lvBlk;
#pragma unroll
    for (int d = 1; d < kV2MaxLevels; d <<= 1) {
      const int t = __shfl_up_sync(kFullMask, incl, d);
      if (lane >= d) incl += t;
    }
    lvE0 = incl - 2 * lvBlk;
  }
  const int entries = __shfl_sync(kFullMask, lvE0 + 2 * lvBlk, L - 1);
  int E0 = (lane < L && entries - lvE0 <= prm.cap_entries) ? lvE0 : entries;
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) E0 = min(E0, __shfl_xor_sync(kFullMask, E0, d));

  const uint32_t barr = smem_addr(&bar), tail_s = smem_addr(tail);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(barr) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // lane `sub` owns chunk `sub` (4 consecutive points of one level) of its item: the level's constants, once
  const bool have = sub < NCH;
  const int c = have ? sub : 0, lvl = c / CPL;
  const int H = __shfl_sync(kFullMask, lvH, lvl), W = __shfl_sync(kFullMask, lvW, lvl);
  const int e0 = __shfl_sync(kFullMask, lvE0, lvl), blk = __shfl_sync(kFullMask, lvBlk, lvl);
  const float Hf = static_cast<float>(H), Wf = static_cast<float>(W);
  const bool own_tail = e0 >= E0;
  const int gmask = G - 1;  // G in {1, 2, 4}: point k of a chunk uses reference group k & (G - 1)
  unsigned tailmask = 0;    // bit ch: chunk ch belongs to a level that lives in shared memory (warp-uniform)
  for (int ch = 0; ch < NCH; ++ch) tailmask |= (__shfl_sync(kFullMask, lvE0, ch / CPL) >= E0) ? (1u << ch) : 0u;

  const int pairs = prm.B * M;
  const int groups = gridDim.x / prm.cpp;
  const int j = blockIdx.x % prm.cpp;
  const long long slab = static_cast<long long>(entries) * kEB;
  uint32_t phase = 0;
  for (int pair = blockIdx.x / prm.cpp; pair < pairs; pair += groups) {
    const int b = pair / M, m = pair - b * M;
    const char *vl = prm.packed + static_cast<long long>(pair) * slab;
    const int tail_bytes = (entries - E0) * kEB;
    if (tail_bytes > 0) {
      if (threadIdx.x == 0) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(barr), "r"(tail_bytes) : "memory");
        for (int o = 0; o < tail_bytes; o += kI8CopyBytes) {
          const int n = min(kI8CopyBytes, tail_bytes - o);
          asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(tail_s + o),
                       "l"(vl + static_cast<long long>(E0) * kEB + o), "r"(n), "r"(barr)
                       : "memory");
        }
      }
      uint32_t done = 0;
      while (!done)
        asm volatile("{ .reg .pred q; mbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2; selp.u32 %0, 1, 0, q; }"
                     : "=r"(done) : "r"(barr), "r"(phase) : "memory");
      phase ^= 1u;
    }
    const char *gbase = vl + cj * 16;

    const long long qstep = static_cast<long long>(prm.cpp) * kI8ItemsPerBlock;
    for (long long qb = static_cast<long long>(j) * kI8ItemsPerBlock; qb < Q; qb += qstep) {
      const long long q_raw = qb + warp * kI8ItemsPerWarp + grp_i;
      const bool active = q_raw < Q;
      const long long bq = static_cast<long long>(b) * Q + (active ? q_raw : Q - 1);
      const long long it = bq * M + m;

      float rpx[4], rpy[4];
      if (sizeof(R) == 2) {
        const uint32_t *rp = reinterpret_cast<const uint32_t *>(prm.ref) + bq * G;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = h2_to_f2(__ldg(rp + (k & gmask)));
          rpx[k] = f.x, rpy[k] = f.y;
        }
      } else {
        const float2 *rp = reinterpret_cast<const float2 *>(prm.ref) + bq * G;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float2 f = __ldg(rp + (k & gmask));
          rpx[k] = f.x, rpy[k] = f.y;
        }
      }
      // ---- phase A (bit-exact): loc = fma(ref, size, off) - 0.5; off * scale is rounded to fp32 first (…Kernel.cu:916-921)
      const uint2 o8 = ldg64_stream(prm.off + it * NP * 2 + c * 8);
      float wim[4], him[4];
      unsigned inr = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t w2 = k < 2 ? o8.x : o8.y;
        const float ox = deq8(w2, (k & 1) * 2, prm.scale_offset), oy = deq8(w2, (k & 1) * 2 + 1, prm.scale_offset);
        wim[k] = __fadd_rn(__fmaf_rn(rpx[k], Wf, ox), -0.5f);
        him[k] = __fadd_rn(__fmaf_rn(rpy[k], Hf, oy), -0.5f);
        const bool ok = have && him[k] > -1.f && wim[k] > -1.f && him[k] < Hf && wim[k] < Wf;
        inr |= ok ? (1u << k) : 0u;
      }
      int8_t *out_item = prm.out + it * 32;
      const unsigned vm = __ballot_sync(kFullMask, inr != 0u);  // bit (8*item + chunk): the chunk has a point in range
      if (vm == 0u) {  // nothing of the warp's items is in range: exact zeros, logits are never read
        if (active) reinterpret_cast<uint32_t *>(out_item)[sub] = 0u;
        continue;
      }
      // ---- phase B: softmax statistics over the item's NP logits (group of 8 lanes)
      float lg[4];
      if (have) {
        const uint32_t l4 = ldg32_stream(prm.logits + it * NP + c * 4);
#pragma unroll
        for (int k = 0; k < 4; ++k) lg[k] = deq8(l4, k, prm.scale_weight);
      } else {
        lg[0] = lg[1] = lg[2] = lg[3] = -INFINITY;
      }
      float mx = fmaxf(fmaxf(lg[0], lg[1]), fmaxf(lg[2], lg[3]));
#pragma unroll
      for (int d = 1; d < 8; d <<= 1) mx = fmaxf(mx, __shfl_xor_sync(kFullMask, mx, d));
      float sum = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) lg[k] = __expf(lg[k] - mx), sum += lg[k];  // ex2.approx: 2 ulp, far below the INT8 steps
#pragma unroll
      for (int d = 1; d < 8; d <<= 1) sum += __shfl_xor_sync(kFullMask, sum, d);

      // ---- phase C (owner): one 16-byte record per point {load address and (w_y0, w_y1) of the left column, of the
      // right column}: a shared-memory address for resident levels, a byte offset into the slab otherwise
      __syncwarp();  // the previous iteration's records have been consumed
      if (have) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const bool ok = (inr >> k) & 1u;
          const float hf = floorf(him[k]), wf = floorf(wim[k]);
          const int h_low = ok ? static_cast<int>(hf) : 0, w_low = ok ? static_cast<int>(wf) : 0;
          const float lh = __fsub_rn(him[k], hf), lw = __fsub_rn(wim[k], wf), hh = 1.f - lh, hw = 1.f - lw;
          const bool t = h_low >= 0, bt = h_low + 1 <= H - 1, lf = w_low >= 0, rt = w_low + 1 <= W - 1;
          const float e = lg[k];
          const float w00 = (ok && t && lf) ? hh * hw * e : 0.f, w01 = (ok && t && rt) ? hh * lw * e : 0.f;
          const float w10 = (ok && bt && lf) ? lh * hw * e : 0.f, w11 = (ok && bt && rt) ? lh * lw * e : 0.f;
          const int par = h_low & 1, r = (h_low + 1) >> 1;
          const int xl = max(w_low, 0), xr = min(w_low + 1, W - 1);
          const unsigned ent = static_cast<unsigned>(e0 + (par ? blk : 0) + r * W + xl);
          // the right column is the next entry; without a right neighbour it aliases the left one and carries weight 0
          const unsigned a0 = own_tail ? tail_s + (ent - static_cast<unsigned>(E0)) * kEB : ent * kEB;
          const unsigned a1 = a0 + (xr > xl ? kEB : 0);
          asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(rec_s + (k * 8 + sub) * 16), "r"(a0), "r"(fixed_pair(w00, w10)),
                       "r"(a1), "r"(fixed_pair(w01, w11))
                       : "memory");
          if (DBG && active)
            prm.trace[it * NP + c * 4 + k] = ok ? make_int4(1, h_low, w_low, ((t && lf) ? 1 : 0) | ((t && rt) ? 2 : 0) |
                                                                                 ((bt && lf) ? 4 : 0) | ((bt && rt) ? 8 : 0))
                                                : make_int4(0, 0, 0, 0);
        }
      }
      __syncwarp();

      // ---- gather: lane = (column col, channels 8*cj .. +7 as (y0, y1) byte pairs): one 8-byte record read, one 16-byte
      // load and 8 dp2a per sample
      int acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      const uint32_t my_rec = rec_s + col * 8;
#pragma unroll 1
      for (int ch = 0; ch < NCH; ++ch) {
        if ((vm & (0x01010101u << ch)) == 0u) continue;  // warp-uniform: chunk out of range for every item
        uint2 rr[4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
          asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(rr[k].x), "=r"(rr[k].y) : "r"(my_rec + (k * 8 + ch) * 16));
        uint4 v[4];
        if ((tailmask >> ch) & 1u) {  // warp-uniform
#pragma unroll
          for (int k = 0; k < 4; ++k) v[k] = lds128_v2(rr[k].x + cj * 16);
        } else {
#pragma unroll
          for (int k = 0; k < 4; ++k) v[k] = ldg128(gbase + rr[k].x);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const unsigned wq = rr[k].y;
          acc[0] = dp2a_lo(wq, v[k].x, acc[0]), acc[1] = dp2a_hi(wq, v[k].x, acc[1]);
          acc[2] = dp2a_lo(wq, v[k].y, acc[2]), acc[3] = dp2a_hi(wq, v[k].y, acc[3]);
          acc[4] = dp2a_lo(wq, v[k].z, acc[4]), acc[5] = dp2a_hi(wq, v[k].z, acc[5]);
          acc[6] = dp2a_lo(wq, v[k].w, acc[6]), acc[7] = dp2a_hi(wq, v[k].w, acc[7]);
        }
      }
      // the two columns of a sample live in lanes sub and sub ^ 4
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] += __shfl_xor_sync(kFullMask, acc[i], 4);
      if (active && col == 0) {
        // real = acc / 65536 * scale_value / sum ; q = T2int8(real / scale_out)
        const float mul = __fdividef(prm.scale_value, 65536.f * sum * prm.scale_out);
        uint32_t o[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          uint32_t word = 0;
#pragma unroll
          for (int jj = 0; jj < 4; ++jj)
            word |= (static_cast<uint32_t>(to_int8_sat(static_cast<float>(acc[4 * i + jj]) * mul)) & 0xffu) << (8 * jj);
          o[i] = word;
        }
        asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(out_item + 8 * cj), "r"(o[0]), "r"(o[1]) : "memory");
      }
    }
    __syncthreads();  // every warp is done with the tail before the next slab's copies overwrite it
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
static std::atomic<int> g_i8_tail_bytes{128 * 1024};  // shared memory of the gather kernel's resident tail

// The packed kernel's shape: at most kV2MaxLevels levels and 16 to 32 points per item.
static bool i8p_shape_ok(const MsdaGeom &g) {
  return g.L >= 1 && g.L <= kV2MaxLevels && g.L * g.P >= 16 && msda_lane_group_shape(g, 32);
}

// Upper bound of the packed stack from the tensor DIMENSIONS only (what getWorkspaceSize sees): both parity copies of
// every level, sum_l 2 * (H_l/2 + 1) * W_l <= S + 2 * sum_l W_l <= 3 * S entries per (camera, head).
static size_t i8p_workspace_bound(const MsdaGeom &g) { return static_cast<size_t>(3) * g.S * kEB * g.B * g.M; }

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_msda_i8_workspace_size(int batch, int spatial_size, int num_heads, int channels, int num_levels, int num_point,
                                   int points_per_group) {
  // no query count: the packed stack does not depend on it
  const MsdaGeom g = msda_geom(batch, spatial_size, num_heads, channels, num_levels, 0, num_point, points_per_group);
  if (g.B <= 0 || g.M <= 0 || g.S <= 0) return 0;
  if (!i8p_shape_ok(g)) return 0;
  return i8p_workspace_bound(g);
}

int b200_msda_i8_ws(const int8_t *value, float scale_value, const int32_t *spatial_shapes, const void *reference_points,
                    int ref_is_half, const int8_t *sampling_offsets, float scale_offset, const int8_t *attn_weight,
                    float scale_weight, int batch, int spatial_size, int num_heads, int channels, int num_levels,
                    int num_query, int num_point, int points_per_group, int8_t *out, float scale_out, void *workspace,
                    size_t workspace_bytes, int32_t *trace_records, void *stream) {
  const MsdaGeom g =
      msda_geom(batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group);
  if (!(scale_out > 0.f)) return B200_ERR_BAD_PARAM;
  if (!value || !spatial_shapes || !reference_points || !sampling_offsets || !attn_weight || !out || !workspace)
    return B200_ERR_BAD_PARAM;
  if (g.B <= 0 || g.S <= 0 || g.M <= 0 || g.Q <= 0) return B200_ERR_BAD_PARAM;
  if (!i8p_shape_ok(g)) return B200_ERR_UNSUPPORTED;
  if (workspace_bytes < i8p_workspace_bound(g)) return B200_ERR_BAD_PARAM;
  if (static_cast<long long>(3) * g.S * kEB >= (1ll << 31)) return B200_ERR_UNSUPPORTED;  // 32-bit slab offsets
  const long long items = static_cast<long long>(g.B) * g.Q * g.M;
  const long long blocks = (items + kI8ItemsPerBlock - 1) / kI8ItemsPerBlock;
  if (blocks > 0x7fffffffll) return B200_ERR_UNSUPPORTED;
  if (!msda_aligned({value, workspace, sampling_offsets, attn_weight, out, reference_points}, 16) ||
      !msda_aligned({spatial_shapes}, 4))
    return B200_ERR_UNSUPPORTED;
  cudaStream_t s = static_cast<cudaStream_t>(stream);

  // 1. pack: persistent CTAs, 2 rows x 64 pixels x (M*32) bytes of shared memory each
  PackParams pp{};
  pp.value = reinterpret_cast<const char *>(value), pp.packed = static_cast<char *>(workspace), pp.shapes = spatial_shapes;
  pp.B = g.B, pp.S = g.S, pp.M = g.M, pp.L = g.L;
  const int smem = 2 * kPackCols * g.M * 32;
  if (smem > 200 * 1024) return B200_ERR_UNSUPPORTED;
  const int sms = msda_sm_count();
  int per_sm = (200 * 1024) / (smem + 2048);
  per_sm = per_sm < 1 ? 1 : (per_sm > 6 ? 6 : per_sm);
  const unsigned gx = static_cast<unsigned>((sms * per_sm + g.B - 1) / g.B);
  if (cudaFuncSetAttribute(msda_pack_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
    return B200_ERR_LAUNCH;
  msda_pack_kernel<<<dim3(gx < 1 ? 1 : gx, static_cast<unsigned>(g.B)), 256, smem, s>>>(pp);
  int st = check_launch();
  if (st != B200_OK) return st;

  // 2. gather: one persistent CTA per SM, `cpp` CTAs per (camera, head) slab
  I8PParams gp{};
  gp.packed = static_cast<const char *>(workspace), gp.ref = reference_points, gp.off = sampling_offsets;
  gp.logits = attn_weight, gp.out = out, gp.shapes = spatial_shapes;
  gp.B = g.B, gp.M = g.M, gp.Q = g.Q, gp.P = g.P, gp.G = g.G, gp.NP = g.L * g.P, gp.L = g.L;
  gp.scale_value = scale_value, gp.scale_offset = scale_offset, gp.scale_weight = scale_weight, gp.scale_out = scale_out;
  const MsdaSlabGrid sg = msda_slab_grid(g, sms, kI8ItemsPerBlock);
  gp.cpp = sg.cpp;
  long long cap = g_i8_tail_bytes.load(std::memory_order_relaxed);
  const long long need = static_cast<long long>(3) * g.S * kEB;  // never more than a whole slab
  if (cap > need) cap = (need + 127) / 128 * 128;
  gp.cap_entries = static_cast<int>(cap / kEB);
  const int gsmem = gp.cap_entries * kEB + kI8Warps * kI8ItemsPerWarp * 33 * 16;  // tail + per-warp sample records
  auto launch = [&](auto kern) -> int {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, gsmem) != cudaSuccess) return B200_ERR_LAUNCH;
    kern<<<sg.grid, kI8Threads, gsmem, s>>>(gp);
    return check_launch();
  };
  if (trace_records) {
    if (cudaMemsetAsync(trace_records, 0, static_cast<size_t>(items) * gp.NP * 16, s) != cudaSuccess) return B200_ERR_LAUNCH;
    gp.trace = reinterpret_cast<int4 *>(trace_records);
    return ref_is_half ? launch(msda_i8p_kernel<__half, true>) : launch(msda_i8p_kernel<float, true>);
  }
  return ref_is_half ? launch(msda_i8p_kernel<__half, false>) : launch(msda_i8p_kernel<float, false>);
}

int b200_msda_set_i8_resident_bytes(int bytes) {
  return g_i8_tail_bytes.exchange(bytes < 4096 ? 4096 : (bytes > 200 * 1024 ? 200 * 1024 : bytes));
}

}  // extern "C"

// dcn_backward.cu — the DCNv2 backward pass (mmcv's modulated_deform_conv_backward, which the reference binding calls in
// det2trt/models/functions/modulated_deformable_conv2d.py:107-157): gradients for input, offset, mask, weight and bias.
//
// Notation per (image b, group g): col[(c,t), p] = mask[t,p] * bilinear(x[c], pos(t,p)) (the forward's sampled column),
// gc[(c,t), p] = sum_m W[m, (c,t)] * grad_out[m, p]. Then
//   grad_input [c, y, x]  = sum over samples whose valid corner is (y, x) of gc * mask * corner_weight     (float atomics)
//   grad_offset[2t (+1), p] = sum over the deformable group's channels of gc * mask * d bilinear / dh (dw)
//   grad_mask  [t, p]     = sum over the deformable group's channels of gc * bilinear(x)
//   grad_weight[m, (c,t)] = sum_{b,p} grad_out[m, p] * col[(c,t), p]
//   grad_bias  [m]        = sum_{b,p} grad_out[m, p]
// with mmcv's coordinate weights and the forward's index rule (h > -1 && w > -1 && h < H && w < W, floor corners, each
// corner valid on its own). Everything accumulates in fp32; FP16 / BF16 storage is converted at load and rounded once
// at the end. Three hand-written kernels on the FP32 pipe, modelled on dcn_generic.cu (64-pixel tiles, a per-tile sampling
// table, K blocks of KC input channels x the taps), no library GEMM:
//   * data kernel   — CTA = (image, deformable group, 64-pixel tile, split of the group's channel chunks). Per chunk it
//                     computes the gc tile from W and grad_out in shared memory, scatters grad_input with atomics, and
//                     sums the offset / mask terms over the chunk's channels in a fixed order into per-CTA fp32
//                     accumulators, which it writes as one partial per split;
//   * weight kernel — CTA = (64 output channels, K block, split of the (image, pixel tile) items): samples the column
//                     tile exactly as the forward does and accumulates grad_out x col^T into one partial per split;
//   * finalisation  — sums the partials in split order (grad_offset / grad_mask / grad_weight), reduces grad_bias with
//                     a fixed tree, converts the fp32 grad_input accumulator to FP16.
// So grad_weight, grad_bias, grad_offset and grad_mask are bit-reproducible and do not depend on which other gradients
// are requested; grad_input is not (float atomics, as in mmcv and torchvision).
#include <algorithm>
#include <type_traits>

#include "dcn_geometry.cuh"

namespace b200 {
namespace {

constexpr int kBT = 64;      // pixels per tile
constexpr int kRB = 48;      // rows (channel, tap) of a K block at most
constexpr int kMC = 32;      // output channels per step of the data kernel's reduction
constexpr int kThreads = 256;
constexpr int kTargetCtas = 512;  // splits are chosen from the geometry (never the device), so results never depend on it

struct BwTap {
  float lh, lw, m;
  int o1;     // top-left corner inside the channel plane, clamped into the image
  int flags;  // bits 0-3: corner (tl, tr, bl, br) valid; bit 4: +1 column usable; bit 5: +1 row usable
};

struct DcnBwParams {
  const void *im, *weight, *offset, *mask, *gout;
  float *gin;      // fp32 NCHW accumulator of grad_input, or null
  float *om_part;  // [B][dg][nsplit][3][kk][P] (offset-h, offset-w, mask), or null
  float *w_part;   // [wsplit][Co][Kg]
  int B, C, H, W, Co, kh, kw, pad_h, pad_w, stride_h, stride_w, dil_h, dil_w, groups, dg, Ho, Wo;
  int KC, npass, nsplit, wsplit;
  int nhwc;    // input is [B][H][W][C] (flags bit 0)
  int packed;  // weight is packed [Co][C/64][kk][64] by b200_dcn_pack_weights_f16 (flags bit 1; groups == 1)
};

template <typename T>
__device__ __forceinline__ float bw_ld(const T *p);
template <>
__device__ __forceinline__ float bw_ld<float>(const float *p) {
  return __ldg(p);
}
template <>
__device__ __forceinline__ float bw_ld<__half>(const __half *p) {
  return __half2float(__ldg(p));
}
template <>
__device__ __forceinline__ float bw_ld<__nv_bfloat16>(const __nv_bfloat16 *p) {
  return bf16_to_f(__ldg(p));
}
template <typename T>
__device__ __forceinline__ void bw_st(T *p, float v);
template <>
__device__ __forceinline__ void bw_st<float>(float *p, float v) {
  *p = v;
}
template <>
__device__ __forceinline__ void bw_st<__half>(__half *p, float v) {
  *p = __float2half_rn(v);
}
template <>
__device__ __forceinline__ void bw_st<__nv_bfloat16>(__nv_bfloat16 *p, float v) {
  *p = __float2bfloat16_rn(v);
}

// Sampling position of tap t at output pixel pix; `off` / `msk` point at the (image, deformable group) planes.
// The index arithmetic is the forward's (dcn_generic.cu), op for op.
template <typename T>
__device__ BwTap bw_tap(const DcnBwParams &p, const T *off, const T *msk, int t, int pix) {
  BwTap tp{0.f, 0.f, 0.f, 0, 0};
  const int HoWo = p.Ho * p.Wo;
  const int h_col = pix / p.Wo, w_col = pix - h_col * p.Wo;
  const int i = t / p.kw, j = t - i * p.kw;
  const float oh = bw_ld(off + static_cast<long long>(2 * t) * HoWo + pix);
  const float ow = bw_ld(off + static_cast<long long>(2 * t + 1) * HoWo + pix);
  tp.m = bw_ld(msk + static_cast<long long>(t) * HoWo + pix);
  const float h_im = __fadd_rn(static_cast<float>(h_col * p.stride_h - p.pad_h + i * p.dil_h), oh);
  const float w_im = __fadd_rn(static_cast<float>(w_col * p.stride_w - p.pad_w + j * p.dil_w), ow);
  if (h_im > -1.f && w_im > -1.f && h_im < static_cast<float>(p.H) && w_im < static_cast<float>(p.W)) {
    const float hf = floorf(h_im), wf = floorf(w_im);
    const int h_low = static_cast<int>(hf), w_low = static_cast<int>(wf);
    tp.lh = __fsub_rn(h_im, hf), tp.lw = __fsub_rn(w_im, wf);
    const bool tpv = h_low >= 0, bt = h_low + 1 <= p.H - 1, lf = w_low >= 0, rt = w_low + 1 <= p.W - 1;
    tp.o1 = max(h_low, 0) * p.W + max(w_low, 0);
    tp.flags = (tpv && lf ? 1 : 0) | (tpv && rt ? 2 : 0) | (bt && lf ? 4 : 0) | (bt && rt ? 8 : 0) |
               (lf && rt ? 16 : 0) | (tpv && bt ? 32 : 0);
  }
  return tp;
}

// the four corner values of a sample (0 for invalid corners) and their pixel indices inside the image
struct Corners {
  float v[4];
  int a[4];
};
// channel c of image `im` (either layout): element of pixel a at chan[a * pix_stride]
template <typename T>
__device__ __forceinline__ const T *bw_channel(const DcnBwParams &p, const T *im, int c) {
  return im + (p.nhwc ? static_cast<long long>(c) : static_cast<long long>(c) * p.H * p.W);
}
template <typename T>
__device__ __forceinline__ Corners bw_corners(const DcnBwParams &p, const BwTap &tp, const T *chan) {
  Corners c;
  const int dx = (tp.flags & 16) ? 1 : 0, dy = (tp.flags & 32) ? p.W : 0, ps = p.nhwc ? p.C : 1;
  c.a[0] = tp.o1, c.a[1] = tp.o1 + dx, c.a[2] = tp.o1 + dy, c.a[3] = tp.o1 + dy + dx;
#pragma unroll
  for (int q = 0; q < 4; ++q) c.v[q] = (tp.flags & (1 << q)) ? bw_ld(chan + static_cast<long long>(c.a[q]) * ps) : 0.f;
  return c;
}
// W[m][cl][t] (m global output channel, cl channel inside the group), plain or packed
__device__ __forceinline__ long long bw_widx(const DcnBwParams &p, int m, int cl, int t) {
  const int kk = p.kh * p.kw;
  const long long row = static_cast<long long>(m) * (p.C / p.groups) * kk;
  return p.packed ? row + (cl / 64) * 64 * kk + t * 64 + cl % 64 : row + static_cast<long long>(cl) * kk + t;
}

// K block y of the (group's) channel chunks: chunk q = KC channels, pass over taps when kh*kw > kRB (then KC == 1)
struct KBlock {
  int t0, nt, rows;
};
__device__ __forceinline__ KBlock kblock(const DcnBwParams &p, int pass) {
  const int kk = p.kh * p.kw;
  KBlock k;
  k.t0 = pass * kRB;
  k.nt = min(kRB, kk - k.t0);
  k.rows = p.KC * k.nt;
  return k;
}

// ---- data gradient: grad_input (atomics) and the offset / mask partials --------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads) dcn_bw_data_kernel(const DcnBwParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int kk = p.kh * p.kw, P = p.Ho * p.Wo, HW = p.H * p.W;
  const int Cg = p.C / p.groups, Mg = p.Co / p.groups, cpd = p.C / p.dg;
  float *Bs = reinterpret_cast<float *>(smem_raw);  // [kMC][kBT]   grad_out
  float *As = Bs + kMC * kBT;                       // [kMC][kRB]   W^T
  float *red = As + kMC * kRB;                      // [3][kRB][kBT] per-row offset / mask terms
  float *acc_om = red + 3 * kRB * kBT;              // [3][kk][kBT]
  BwTap *tab = reinterpret_cast<BwTap *>(acc_om + 3 * kk * kBT);  // [kk][kBT]

  const int n0 = blockIdx.x * kBT, b = blockIdx.z;
  const int dgi = blockIdx.y / p.nsplit, s = blockIdx.y % p.nsplit;
  const int nch = cpd / p.KC, cps = (nch + p.nsplit - 1) / p.nsplit;
  const int q_beg = s * cps, q_end = min(nch, q_beg + cps);
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const bool want_om = p.om_part != nullptr;

  const T *im = static_cast<const T *>(p.im) + static_cast<long long>(b) * p.C * HW;
  const T *go = static_cast<const T *>(p.gout) + static_cast<long long>(b) * p.Co * P;
  const T *off = static_cast<const T *>(p.offset) + (static_cast<long long>(b) * p.dg + dgi) * 2 * kk * P;
  const T *msk = static_cast<const T *>(p.mask) + (static_cast<long long>(b) * p.dg + dgi) * kk * P;
  for (int e = tid; e < kk * kBT; e += kThreads) {
    const int t = e / kBT, n = e - t * kBT;
    tab[e] = n0 + n < P ? bw_tap(p, off, msk, t, n0 + n) : BwTap{0.f, 0.f, 0.f, 0, 0};
    if (want_om) acc_om[e] = 0.f, acc_om[kk * kBT + e] = 0.f, acc_om[2 * kk * kBT + e] = 0.f;
  }

  for (int q = q_beg; q < q_end; ++q) {
    const int c0 = dgi * cpd + q * p.KC;  // first (global) channel of the chunk
    const int g = c0 / Cg, cl0 = c0 - g * Cg;
    const T *wt = static_cast<const T *>(p.weight);
    for (int pass = 0; pass < p.npass; ++pass) {
      const KBlock kb = kblock(p, pass);
      float acc[3][4];
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
      for (int m0 = 0; m0 < Mg; m0 += kMC) {
        __syncthreads();  // previous users of As / Bs / red (and the table, on the first pass) are done
        for (int e = tid; e < kMC * kRB; e += kThreads) {  // rows beyond kb.rows are zero-filled
          const int mm = e / kRB, r = e - mm * kRB;
          As[e] = (m0 + mm < Mg && r < kb.rows)
                      ? bw_ld(wt + bw_widx(p, g * Mg + m0 + mm, cl0 + r / kb.nt, kb.t0 + r % kb.nt))
                      : 0.f;
        }
        for (int e = tid; e < kMC * kBT; e += kThreads) {
          const int mm = e / kBT, n = e - mm * kBT;
          Bs[e] = (m0 + mm < Mg && n0 + n < P) ? bw_ld(go + static_cast<long long>(g * Mg + m0 + mm) * P + n0 + n) : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int mm = 0; mm < kMC; ++mm) {
          const float4 bv = *reinterpret_cast<const float4 *>(Bs + mm * kBT + tx * 4);
#pragma unroll
          for (int i = 0; i < 3; ++i) {
            const float a = As[mm * kRB + ty + 16 * i];
            acc[i][0] = fmaf(a, bv.x, acc[i][0]), acc[i][1] = fmaf(a, bv.y, acc[i][1]);
            acc[i][2] = fmaf(a, bv.z, acc[i][2]), acc[i][3] = fmaf(a, bv.w, acc[i][3]);
          }
        }
      }
      // epilogue: gc of (row, pixel) -> grad_input corners, offset / mask terms
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const int r = ty + 16 * i;
        if (r >= kb.rows) continue;
        const int c = c0 + r / kb.nt, t = kb.t0 + r % kb.nt;
        const T *chan = bw_channel(p, im, c);
        float *gplane = p.gin ? p.gin + (static_cast<long long>(b) * p.C + c) * HW : nullptr;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int n = tx * 4 + j;
          const BwTap tp = tab[t * kBT + n];
          const float gcv = acc[i][j];
          float goh = 0.f, gow = 0.f, gm = 0.f;
          if (tp.flags) {
            const Corners cn = bw_corners(p, tp, chan);
            const float lh = tp.lh, lw = tp.lw, hh = 1.f - lh, hw = 1.f - lw;
            const float cw[4] = {hh * hw, hh * lw, lh * hw, lh * lw};
            if (gplane) {
              const float gmv = gcv * tp.m;
#pragma unroll
              for (int k = 0; k < 4; ++k)
                if (tp.flags & (1 << k)) atomicAdd(gplane + cn.a[k], gmv * cw[k]);
            }
            if (want_om) {
              gm = gcv * (cw[0] * cn.v[0] + cw[1] * cn.v[1] + cw[2] * cn.v[2] + cw[3] * cn.v[3]);
              const float gmv = gcv * tp.m;
              goh = gmv * (-hw * cn.v[0] - lw * cn.v[1] + hw * cn.v[2] + lw * cn.v[3]);
              gow = gmv * (-hh * cn.v[0] + hh * cn.v[1] - lh * cn.v[2] + lh * cn.v[3]);
            }
          }
          if (want_om) {
            red[r * kBT + n] = goh;
            red[(kRB + r) * kBT + n] = gow;
            red[(2 * kRB + r) * kBT + n] = gm;
          }
        }
      }
      if (want_om) {
        __syncthreads();
        // the chunk's channels, summed in channel order, into the CTA's accumulators
        for (int e = tid; e < kb.nt * kBT; e += kThreads) {
          const int tl = e / kBT, n = e - tl * kBT;
          float s0 = 0.f, s1 = 0.f, s2 = 0.f;
          for (int cl = 0; cl < p.KC; ++cl) {
            const int r = cl * kb.nt + tl;
            s0 += red[r * kBT + n], s1 += red[(kRB + r) * kBT + n], s2 += red[(2 * kRB + r) * kBT + n];
          }
          const int a = (kb.t0 + tl) * kBT + n;
          acc_om[a] += s0, acc_om[kk * kBT + a] += s1, acc_om[2 * kk * kBT + a] += s2;
        }
      }
    }
  }
  if (!want_om) return;
  __syncthreads();
  float *part = p.om_part + ((static_cast<long long>(b) * p.dg + dgi) * p.nsplit + s) * 3 * kk * P;
  for (int e = tid; e < 3 * kk * kBT; e += kThreads) {
    const int row = e / kBT, n = e - row * kBT;  // row = component * kk + tap
    if (n0 + n < P) part[static_cast<long long>(row) * P + n0 + n] = acc_om[e];
  }
}

// ---- weight gradient: per-split partials of grad_out x col^T ---------------------------------------------------------
constexpr int kLdA = kBT + 1;  // [pixel][64 output channels], padded
constexpr int kLdB = kRB + 1;  // [pixel][rows], padded

template <typename T>
__global__ void __launch_bounds__(kThreads) dcn_bw_weight_kernel(const DcnBwParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int kk = p.kh * p.kw, P = p.Ho * p.Wo, HW = p.H * p.W;
  const int Cg = p.C / p.groups, Mg = p.Co / p.groups, cpd = p.C / p.dg, Kg = Cg * kk;
  float *At = reinterpret_cast<float *>(smem_raw);  // [kBT][kLdA]  grad_out^T
  float *Bt = At + kBT * kLdA;                      // [kBT][kLdB]  col^T
  BwTap *tab = reinterpret_cast<BwTap *>(Bt + kBT * kLdB);  // [nt][kBT]

  const int nrb = (Cg / p.KC) * p.npass;
  const int m0 = blockIdx.x * 64, g = blockIdx.y / nrb, rb = blockIdx.y % nrb;
  const int q = rb / p.npass, pass = rb % p.npass;
  const int cl0 = q * p.KC, c0 = g * Cg + cl0, dgi = c0 / cpd;
  const KBlock kb = kblock(p, pass);
  const int ptiles = (P + kBT - 1) / kBT, items = p.B * ptiles, ipw = (items + p.wsplit - 1) / p.wsplit;
  const int it_beg = blockIdx.z * ipw, it_end = min(items, it_beg + ipw);
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;

  float acc[4][3];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) acc[i][j] = 0.f;

  for (int e = tid; e < kBT * kLdB; e += kThreads)  // rows beyond kb.rows stay zero (the item loop never writes them)
    Bt[e] = 0.f;
  for (int it = it_beg; it < it_end; ++it) {
    const int b = it / ptiles, n0 = (it - b * ptiles) * kBT;
    const T *off = static_cast<const T *>(p.offset) + (static_cast<long long>(b) * p.dg + dgi) * 2 * kk * P;
    const T *msk = static_cast<const T *>(p.mask) + (static_cast<long long>(b) * p.dg + dgi) * kk * P;
    const T *go = static_cast<const T *>(p.gout) + (static_cast<long long>(b) * p.Co + g * Mg + m0) * P;
    const T *im = static_cast<const T *>(p.im) + static_cast<long long>(b) * p.C * HW;
    __syncthreads();  // the previous item's FMAs are done with At / Bt / tab
    for (int e = tid; e < kb.nt * kBT; e += kThreads) {
      const int tl = e / kBT, n = e - tl * kBT;
      tab[e] = n0 + n < P ? bw_tap(p, off, msk, kb.t0 + tl, n0 + n) : BwTap{0.f, 0.f, 0.f, 0, 0};
    }
    for (int e = tid; e < 64 * kBT; e += kThreads) {
      const int mm = e / kBT, n = e - mm * kBT;
      At[n * kLdA + mm] = (m0 + mm < Mg && n0 + n < P) ? bw_ld(go + static_cast<long long>(mm) * P + n0 + n) : 0.f;
    }
    __syncthreads();
    // column tile: col[(c, t), pixel] = mask * bilinear, the forward's sampled value (in fp32)
    for (int e = tid; e < kb.rows * kBT; e += kThreads) {
      const int r = e / kBT, n = e - r * kBT;
      const BwTap tp = tab[(r % kb.nt) * kBT + n];
      float v = 0.f;
      if (tp.flags) {
        const Corners cn = bw_corners(p, tp, bw_channel(p, im, c0 + r / kb.nt));
        const float lh = tp.lh, lw = tp.lw, hh = 1.f - lh, hw = 1.f - lw;
        v = tp.m * (hh * hw * cn.v[0] + hh * lw * cn.v[1] + lh * hw * cn.v[2] + lh * lw * cn.v[3]);
      }
      Bt[n * kLdB + r] = v;
    }
    __syncthreads();
#pragma unroll 4
    for (int n = 0; n < kBT; ++n) {
      float a[4], c[3];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = At[n * kLdA + ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 3; ++j) c[j] = Bt[n * kLdB + tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) acc[i][j] = fmaf(a[i], c[j], acc[i][j]);
    }
  }
  float *part = p.w_part + (static_cast<long long>(blockIdx.z) * p.Co + g * Mg) * Kg;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= Mg) continue;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const int r = tx + 16 * j;
      if (r < kb.rows) part[static_cast<long long>(m) * Kg + (cl0 + r / kb.nt) * kk + kb.t0 + r % kb.nt] = acc[i][j];
    }
  }
}

// ---- finalisation ----------------------------------------------------------------------------------------------------
template <typename T>
__global__ void dcn_bw_sum_weight_kernel(const float *part, T *grad_weight, long long n, int splits) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float s = 0.f;
    for (int z = 0; z < splits; ++z) s += part[z * n + i];
    bw_st(grad_weight + i, s);
  }
}

// (b, dg, t, pixel) -> grad_offset[b][dg*2kk + 2t (+1)][pixel], grad_mask[b][dg*kk + t][pixel]
template <typename T>
__global__ void dcn_bw_sum_offset_mask_kernel(const float *part, T *grad_offset, T *grad_mask, int BD, int kk, int P,
                                              int splits) {
  const long long n = static_cast<long long>(BD) * kk * P;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long bd = i / (static_cast<long long>(kk) * P), tp = i - bd * kk * P;  // tp = t * P + pixel
    const float *pp = part + bd * splits * 3 * kk * P + tp;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int z = 0; z < splits; ++z, pp += 3ll * kk * P) s0 += pp[0], s1 += pp[static_cast<long long>(kk) * P], s2 += pp[2ll * kk * P];
    const long long t = tp / P, pix = tp - t * P;
    if (grad_offset) {
      bw_st(grad_offset + (bd * 2 * kk + 2 * t) * P + pix, s0);
      bw_st(grad_offset + (bd * 2 * kk + 2 * t + 1) * P + pix, s1);
    }
    if (grad_mask) bw_st(grad_mask + i, s2);
  }
}

// one CTA per output channel: fixed per-thread strides and a fixed tree, so the sum is the same on every run
template <typename T>
__global__ void __launch_bounds__(kThreads) dcn_bw_bias_kernel(const T *gout, T *grad_bias, int B, int Co, int P) {
  __shared__ float sh[kThreads];
  const int co = blockIdx.x;
  float s = 0.f;
  for (int b = 0; b < B; ++b) {
    const T *row = gout + (static_cast<long long>(b) * Co + co) * P;
    for (int i = threadIdx.x; i < P; i += kThreads) s += bw_ld(row + i);
  }
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int w = kThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) bw_st(grad_bias + co, sh[0]);
}

// the fp32 grad_input accumulator rounded once to the 2-byte storage type (FP16 or BF16)
template <typename T>
__global__ void dcn_bw_f32_round_kernel(const float *in, T *out, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    bw_st(out + i, in[i]);
}

// Everything the launches need that follows from the geometry alone (also what the workspace query returns).
struct BwPlan {
  int KC, npass, nsplit, wsplit;
  size_t gin, om, w, total;  // byte offsets of the workspace sections
  size_t smem_data, smem_weight;
};

int pick_kc_bw(int Cg, int cpd, int kk) {
  int kc = 16;
  while (kc > 1 && (kc * kk > kRB || Cg % kc || cpd % kc)) kc >>= 1;
  return kc;
}

// 0 on success, else the status to return
int bw_plan(BwPlan &pl, bool f16, const DcnGeom &g) {
  if (!dcn_positive(g) || g.pad_h < 0 || g.pad_w < 0 || !dcn_groups_divide(g) || g.Ho <= 0 || g.Wo <= 0)
    return B200_ERR_BAD_PARAM;
  const long long P = static_cast<long long>(g.Ho) * g.Wo, kk = static_cast<long long>(g.kh) * g.kw;
  // 32-bit offsets inside planes and tiles; every tensor below 2^31 elements
  if (static_cast<long long>(g.C) * kk * P >= (1ll << 31) || static_cast<long long>(g.B) * g.C * g.H * g.W >= (1ll << 31) ||
      static_cast<long long>(g.B) * g.Co * P >= (1ll << 31) || static_cast<long long>(g.B) * g.dg * 2 * kk * P >= (1ll << 31))
    return B200_ERR_BAD_PARAM;
  const int Cg = g.C / g.groups, cpd = g.C / g.dg, Mg = g.Co / g.groups;
  pl.KC = pick_kc_bw(Cg, cpd, static_cast<int>(kk));
  pl.npass = pl.KC > 1 ? 1 : (static_cast<int>(kk) + kRB - 1) / kRB;
  const int ptiles = static_cast<int>((P + kBT - 1) / kBT);
  const int nch = cpd / pl.KC;
  pl.nsplit = std::min(nch, std::max(1, (kTargetCtas + g.dg * ptiles - 1) / (g.dg * ptiles)));
  const long long wbase = static_cast<long long>((Mg + 63) / 64) * g.groups * (Cg / pl.KC) * pl.npass;
  const long long items = static_cast<long long>(g.B) * ptiles;
  pl.wsplit = static_cast<int>(std::min<long long>(items, std::max<long long>(1, (4 * kTargetCtas + wbase - 1) / wbase)));
  if (wbase > 65535) return B200_ERR_UNSUPPORTED;
  size_t o = 0;
  pl.gin = o, o += f16 ? align256(static_cast<size_t>(g.B) * g.C * g.H * g.W * 4) : 0;
  pl.om = o, o += align256(static_cast<size_t>(g.B) * g.dg * pl.nsplit * 3 * kk * P * 4);
  pl.w = o, o += align256(static_cast<size_t>(pl.wsplit) * g.Co * Cg * kk * 4);
  pl.total = o;
  pl.smem_data = (kMC * kBT + kMC * kRB + 3 * kRB * kBT + 3 * kk * kBT) * 4 + kk * kBT * sizeof(BwTap);
  pl.smem_weight = (kBT * kLdA + kBT * kLdB) * 4 + std::min<long long>(kk, kRB) * kBT * sizeof(BwTap);
  if (pl.smem_data > 200 * 1024) return B200_ERR_UNSUPPORTED;  // kernel_h * kernel_w > 75
  return B200_OK;
}

template <typename T>
int dcn_backward(const T *input, const T *weight, const T *offset, const T *mask, const T *grad_output, T *grad_input,
                 T *grad_weight, T *grad_bias, T *grad_offset, T *grad_mask, void *workspace, const DcnGeom &g, int flags,
                 cudaStream_t s) {
  constexpr bool kF16 = sizeof(T) == 2;  // FP16 or BF16: grad_input is accumulated in the fp32 workspace
  if (!input || !weight || !offset || !mask || !grad_output || !workspace) return B200_ERR_BAD_PARAM;
  if (flags & ~3) return B200_ERR_BAD_PARAM;
  BwPlan pl{};
  int st = bw_plan(pl, kF16, g);
  if (st != B200_OK) return st;
  const void *ptrs[] = {input, weight, offset, mask, grad_output, grad_input, grad_weight, grad_bias, grad_offset, grad_mask};
  for (const void *q : ptrs)
    if (reinterpret_cast<uintptr_t>(q) % sizeof(T)) return B200_ERR_BAD_PARAM;
  if (reinterpret_cast<uintptr_t>(workspace) % 256) return B200_ERR_BAD_PARAM;
  if (flags) {  // the layouts of b200_dcn_f16_ex: its envelope and alignment
    if (reinterpret_cast<uintptr_t>(input) % 16 || reinterpret_cast<uintptr_t>(weight) % 16) return B200_ERR_BAD_PARAM;
    if (!std::is_same<T, __half>::value || !dcn_fused_supported(g)) return B200_ERR_UNSUPPORTED;
  }
  if (!grad_input && !grad_weight && !grad_bias && !grad_offset && !grad_mask) return B200_OK;

  char *ws = static_cast<char *>(workspace);
  const int kk = g.kh * g.kw;
  const long long HW = static_cast<long long>(g.H) * g.W, P = static_cast<long long>(g.Ho) * g.Wo;
  const long long nx = static_cast<long long>(g.B) * g.C * HW;

  DcnBwParams p{};
  p.im = input, p.weight = weight, p.offset = offset, p.mask = mask, p.gout = grad_output;
  dcn_set_layer(p, g);
  p.groups = g.groups, p.dg = g.dg;
  p.KC = pl.KC, p.npass = pl.npass, p.nsplit = pl.nsplit, p.wsplit = pl.wsplit;
  p.nhwc = flags & 1, p.packed = (flags >> 1) & 1;
  const unsigned ptiles = static_cast<unsigned>((P + kBT - 1) / kBT);

  if (grad_input || grad_offset || grad_mask) {
    p.gin = grad_input ? (kF16 ? reinterpret_cast<float *>(ws + pl.gin) : reinterpret_cast<float *>(grad_input)) : nullptr;
    p.om_part = (grad_offset || grad_mask) ? reinterpret_cast<float *>(ws + pl.om) : nullptr;
    if (p.gin && cudaMemsetAsync(p.gin, 0, static_cast<size_t>(nx) * 4, s) != cudaSuccess) return B200_ERR_LAUNCH;
    if (cudaFuncSetAttribute(dcn_bw_data_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             static_cast<int>(pl.smem_data)) != cudaSuccess)
      return B200_ERR_LAUNCH;
    if (static_cast<long long>(g.dg) * pl.nsplit > 65535 || g.B > 65535) return B200_ERR_UNSUPPORTED;
    dcn_bw_data_kernel<T><<<dim3(ptiles, g.dg * pl.nsplit, g.B), kThreads, pl.smem_data, s>>>(p);
    if ((st = check_launch()) != B200_OK) return st;
    if constexpr (kF16) {
      if (grad_input) {
        dcn_bw_f32_round_kernel<T><<<grid_for(nx), 256, 0, s>>>(p.gin, grad_input, nx);
        if ((st = check_launch()) != B200_OK) return st;
      }
    }
    if (p.om_part) {
      const long long n = static_cast<long long>(g.B) * g.dg * kk * P;
      dcn_bw_sum_offset_mask_kernel<T><<<grid_for(n), 256, 0, s>>>(p.om_part, grad_offset, grad_mask, g.B * g.dg, kk,
                                                                  static_cast<int>(P), pl.nsplit);
      if ((st = check_launch()) != B200_OK) return st;
    }
  }
  if (grad_weight) {
    p.gin = nullptr, p.om_part = nullptr, p.w_part = reinterpret_cast<float *>(ws + pl.w);
    const int Cg = g.C / g.groups, Mg = g.Co / g.groups;
    const dim3 grid((Mg + 63) / 64, g.groups * (Cg / pl.KC) * pl.npass, pl.wsplit);
    if (grid.y > 65535u || grid.z > 65535u) return B200_ERR_UNSUPPORTED;
    if (cudaFuncSetAttribute(dcn_bw_weight_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             static_cast<int>(pl.smem_weight)) != cudaSuccess)
      return B200_ERR_LAUNCH;
    dcn_bw_weight_kernel<T><<<grid, kThreads, pl.smem_weight, s>>>(p);
    if ((st = check_launch()) != B200_OK) return st;
    const long long n = static_cast<long long>(g.Co) * Cg * kk;
    dcn_bw_sum_weight_kernel<T><<<grid_for(n), 256, 0, s>>>(p.w_part, grad_weight, n, pl.wsplit);
    if ((st = check_launch()) != B200_OK) return st;
  }
  if (grad_bias) {
    dcn_bw_bias_kernel<T><<<g.Co, kThreads, 0, s>>>(grad_output, grad_bias, g.B, g.Co, static_cast<int>(P));
    if ((st = check_launch()) != B200_OK) return st;
  }
  return B200_OK;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_dcn_backward_workspace_size(int dtype, int batch, int channels, int height, int width, int channels_out,
                                        int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h,
                                        int dilation_w, int dilation_h, int group, int deformable_group) {
  BwPlan pl{};
  if (bw_plan(pl, dtype != 0, dcn_geom(batch, channels, height, width, channels_out, kernel_w, kernel_h, stride_w,
                                       stride_h, pad_w, pad_h, dilation_w, dilation_h, group, deformable_group)) != B200_OK)
    return 0;
  return pl.total;
}

int b200_dcn_backward_f32(const float *input, const float *weight, const float *offset, const float *mask,
                          const float *grad_output, float *grad_input, float *grad_weight, float *grad_bias,
                          float *grad_offset, float *grad_mask, void *workspace, int batch, int channels, int height,
                          int width, int channels_out, int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w,
                          int pad_h, int dilation_w, int dilation_h, int group, int deformable_group, void *stream) {
  return dcn_backward<float>(input, weight, offset, mask, grad_output, grad_input, grad_weight, grad_bias, grad_offset,
                             grad_mask, workspace,
                             dcn_geom(batch, channels, height, width, channels_out, kernel_w, kernel_h, stride_w,
                                      stride_h, pad_w, pad_h, dilation_w, dilation_h, group, deformable_group),
                             0, static_cast<cudaStream_t>(stream));
}

int b200_dcn_backward_f16(const void *input, const void *weight, const void *offset, const void *mask,
                          const void *grad_output, void *grad_input, void *grad_weight, void *grad_bias,
                          void *grad_offset, void *grad_mask, void *workspace, int batch, int channels, int height,
                          int width, int channels_out, int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w,
                          int pad_h, int dilation_w, int dilation_h, int group, int deformable_group, int flags,
                          void *stream) {
  using H = __half;
  return dcn_backward<H>(static_cast<const H *>(input), static_cast<const H *>(weight), static_cast<const H *>(offset),
                         static_cast<const H *>(mask), static_cast<const H *>(grad_output), static_cast<H *>(grad_input),
                         static_cast<H *>(grad_weight), static_cast<H *>(grad_bias), static_cast<H *>(grad_offset),
                         static_cast<H *>(grad_mask), workspace,
                         dcn_geom(batch, channels, height, width, channels_out, kernel_w, kernel_h, stride_w, stride_h,
                                  pad_w, pad_h, dilation_w, dilation_h, group, deformable_group),
                         flags, static_cast<cudaStream_t>(stream));
}

// BF16: every tensor and gradient in bf16, fp32 accumulation; no flags (there is no BF16 fused forward whose layouts
// it would read).
int b200_dcn_backward_bf16(const void *input, const void *weight, const void *offset, const void *mask,
                           const void *grad_output, void *grad_input, void *grad_weight, void *grad_bias,
                           void *grad_offset, void *grad_mask, void *workspace, int batch, int channels, int height,
                           int width, int channels_out, int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w,
                           int pad_h, int dilation_w, int dilation_h, int group, int deformable_group, void *stream) {
  using B = __nv_bfloat16;
  return dcn_backward<B>(static_cast<const B *>(input), static_cast<const B *>(weight), static_cast<const B *>(offset),
                         static_cast<const B *>(mask), static_cast<const B *>(grad_output), static_cast<B *>(grad_input),
                         static_cast<B *>(grad_weight), static_cast<B *>(grad_bias), static_cast<B *>(grad_offset),
                         static_cast<B *>(grad_mask), workspace,
                         dcn_geom(batch, channels, height, width, channels_out, kernel_w, kernel_h, stride_w, stride_h,
                                  pad_w, pad_h, dilation_w, dilation_h, group, deformable_group),
                         0, static_cast<cudaStream_t>(stream));
}

}  // extern "C"

// dcn_generic.cu — modulated deformable convolution for EVERY shape the fused wgmma kernel (dcn_fused.cu) does not take:
// FP32, groups > 1, deformable groups > 1, channel counts that are not multiples of 64, any kernel size / stride /
// dilation. A hand-written fused implicit GEMM on the FP32 pipe: no column buffer in global memory, no library GEMM.
//
// Replaces, for those shapes, ModulatedDeformConvForwardCUDAKernel<float|__half> — deformable im2col into a workspace
// (TensorRT/plugin/modulated_deformable_conv2d/modulatedDeformableConv2dKernel.cu:259-388), one cublasGemmEx per image and
// group (:735-754) and a bias kernel (:550-568) — including the reference op test's own shape (groups = 2,
// deform_groups = 2, det2trt/models/utils/test_trt_ops/test_modulated_deformable_conv2d.py:6-11,37).
//
// GEMM view per (image, group):  out[co, pix] = bias[co] + sum_k W[co, k] * col[k, pix],  k = (channel, tap) in the
// weight tensor's own order [Co][C/groups][kh][kw]. CTA tile 64 output channels x 64 output pixels, 256 threads x (4 x 4)
// accumulators, K walked in blocks of KC input channels x all kh*kw taps:
//   * a per-tile SAMPLING TABLE in shared memory holds, for every (tap, pixel) of the tile and the current deformable
//     group, the four corner weights (bilinear x mask, fp32, the reference's index arithmetic op for op: h_im =
//     (h_in + i*dil) + offset, :306-307; zero weights for corners outside the image, :85-116) and the corner offsets.
//     It is rebuilt only when the K walk enters the next deformable group;
//   * the B tile (KC*kk x 64 pixels) is sampled straight into shared memory through that table (consecutive threads =
//     consecutive pixels), the A tile (64 x KC*kk weights) is read k-contiguous and stored transposed;
//   * fp32 FMAs from shared memory, bias added in the epilogue, FP16 / BF16 storage converted at load / store only.
#include "dcn_geometry.cuh"

namespace b200 {

struct DcnGParams {
  const void *im, *weight, *bias, *offset, *mask;
  void *out;
  int B, C, H, W, Co, kh, kw, pad_h, pad_w, stride_h, stride_w, dil_h, dil_w, groups, dg, Ho, Wo;
  int KC;  // input channels per K block (divides C/groups and C/dg)
};

struct DcnTap {
  float w[4];
  int o1;    // offset of the top-left corner inside a channel plane
  int step;  // bit 0: +1 column usable, bit 1: +1 row usable (W added), bit 2: the sample is inside the image
};

constexpr int kGT = 64;  // tile edge (output channels and pixels)

template <typename T>
__device__ __forceinline__ float g_ld(const T *p);
template <>
__device__ __forceinline__ float g_ld<float>(const float *p) {
  return __ldg(p);
}
template <>
__device__ __forceinline__ float g_ld<__half>(const __half *p) {
  return __half2float(__ldg(p));
}
template <>
__device__ __forceinline__ float g_ld<__nv_bfloat16>(const __nv_bfloat16 *p) {
  return bf16_to_f(__ldg(p));
}
template <typename T>
__device__ __forceinline__ void g_st(T *p, float v);
template <>
__device__ __forceinline__ void g_st<float>(float *p, float v) {
  *p = v;
}
template <>
__device__ __forceinline__ void g_st<__half>(__half *p, float v) {
  *p = __float2half_rn(v);
}
template <>
__device__ __forceinline__ void g_st<__nv_bfloat16>(__nv_bfloat16 *p, float v) {
  *p = __float2bfloat16_rn(v);
}

template <typename T>
__global__ void __launch_bounds__(256) dcn_generic_kernel(const DcnGParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int kk = p.kh * p.kw, KB = p.KC * kk;  // K block length
  float *As = reinterpret_cast<float *>(smem_raw);             // [KB][kGT + 1]  (transposed weights)
  float *Bs = As + KB * (kGT + 1);                             // [KB][kGT]      (sampled columns)
  Bs = reinterpret_cast<float *>((reinterpret_cast<uintptr_t>(Bs) + 15) & ~static_cast<uintptr_t>(15));
  DcnTap *tab = reinterpret_cast<DcnTap *>(Bs + KB * kGT);     // [kk][kGT]

  const int HoWo = p.Ho * p.Wo, HW = p.H * p.W;
  const int Cg = p.C / p.groups, Mg = p.Co / p.groups, cpd = p.C / p.dg, Kg = Cg * kk;
  const int n0 = blockIdx.x * kGT, m0 = blockIdx.y * kGT;
  const int b = blockIdx.z / p.groups, g = blockIdx.z % p.groups;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const T *im = static_cast<const T *>(p.im) + static_cast<long long>(b) * p.C * HW;
  const T *wt = static_cast<const T *>(p.weight) + static_cast<long long>(g) * Mg * Kg;
  const T *off = static_cast<const T *>(p.offset) + static_cast<long long>(b) * p.dg * 2 * kk * HoWo;
  const T *msk = static_cast<const T *>(p.mask) + static_cast<long long>(b) * p.dg * kk * HoWo;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  int cur_dg = -1;
  for (int c0 = 0; c0 < Cg; c0 += p.KC) {
    const int cglob = g * Cg + c0;  // first input channel of this K block
    const int dgi = cglob / cpd;
    __syncthreads();  // the previous block's FMAs are done with As / Bs / tab
    if (dgi != cur_dg) {
      cur_dg = dgi;
      for (int e = tid; e < kk * kGT; e += 256) {
        const int t = e / kGT, n = e - t * kGT, pix = n0 + n;
        DcnTap tp{};
        if (pix < HoWo) {
          const int h_col = pix / p.Wo, w_col = pix - h_col * p.Wo;
          const int i = t / p.kw, j = t - i * p.kw;
          const float oh = g_ld(off + (static_cast<long long>(dgi) * 2 * kk + 2 * t) * HoWo + pix);
          const float ow = g_ld(off + (static_cast<long long>(dgi) * 2 * kk + 2 * t + 1) * HoWo + pix);
          const float m = g_ld(msk + (static_cast<long long>(dgi) * kk + t) * HoWo + pix);
          const float h_im = __fadd_rn(static_cast<float>(h_col * p.stride_h - p.pad_h + i * p.dil_h), oh);
          const float w_im = __fadd_rn(static_cast<float>(w_col * p.stride_w - p.pad_w + j * p.dil_w), ow);
          const bool ok = h_im > -1.f && w_im > -1.f && h_im < static_cast<float>(p.H) && w_im < static_cast<float>(p.W);
          const float hf = floorf(h_im), wf = floorf(w_im);
          const int h_low = ok ? static_cast<int>(hf) : 0, w_low = ok ? static_cast<int>(wf) : 0;
          const float lh = __fsub_rn(h_im, hf), lw = __fsub_rn(w_im, wf), hh = 1.f - lh, hw = 1.f - lw;
          const bool tpv = h_low >= 0, bt = h_low + 1 <= p.H - 1, lf = w_low >= 0, rt = w_low + 1 <= p.W - 1;
          tp.w[0] = (ok && tpv && lf) ? hh * hw * m : 0.f, tp.w[1] = (ok && tpv && rt) ? hh * lw * m : 0.f;
          tp.w[2] = (ok && bt && lf) ? lh * hw * m : 0.f, tp.w[3] = (ok && bt && rt) ? lh * lw * m : 0.f;
          tp.o1 = max(h_low, 0) * p.W + max(w_low, 0);
          tp.step = ((lf && rt) ? 1 : 0) | ((tpv && bt) ? 2 : 0) | (ok ? 4 : 0);
          // a sample outside the image is the reference's `0 * mask`, whatever the image holds: kept in w[0] and
          // stored as the column value without touching the image
          if (!ok) tp.w[0] = 0.f * m;
        }
        tab[e] = tp;
      }
      __syncthreads();
    }
    // A tile: weights [m0 + m][c0*kk + k], k contiguous in memory -> As[k][m]
    for (int e = tid; e < KB * kGT; e += 256) {
      const int k = e % KB, m = e / KB;
      As[k * (kGT + 1) + m] = (m0 + m < Mg) ? g_ld(wt + static_cast<long long>(m0 + m) * Kg + c0 * kk + k) : 0.f;
    }
    // B tile: col[(c, t)][pix] sampled through the table
    for (int e = tid; e < KB * kGT; e += 256) {
      const int n = e % kGT, k = e / kGT;
      const int c = k / kk, t = k - c * kk;
      const DcnTap tp = tab[t * kGT + n];
      const T *ip = im + static_cast<long long>(cglob + c) * HW + tp.o1;
      const int dx = tp.step & 1, dy = (tp.step & 2) ? p.W : 0;
      // A missing corner of a sample inside the image has weight 0 and aliases one of that sample's own in-image corners
      // (never out of the plane). A sample outside the image reads nothing: its column value is w[0] = 0 * mask.
      float v = tp.w[0];
      if (tp.step & 4)
        v = fmaf(tp.w[3], g_ld(ip + dy + dx), fmaf(tp.w[2], g_ld(ip + dy), fmaf(tp.w[1], g_ld(ip + dx), tp.w[0] * g_ld(ip))));
      Bs[k * kGT + n] = v;
    }
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < KB; ++k) {
      const float4 bv = *reinterpret_cast<const float4 *>(Bs + k * kGT + tx * 4);
      const float *ap = As + k * (kGT + 1) + ty * 4;
      const float a0 = ap[0], a1 = ap[1], a2 = ap[2], a3 = ap[3];
      acc[0][0] = fmaf(a0, bv.x, acc[0][0]), acc[0][1] = fmaf(a0, bv.y, acc[0][1]);
      acc[0][2] = fmaf(a0, bv.z, acc[0][2]), acc[0][3] = fmaf(a0, bv.w, acc[0][3]);
      acc[1][0] = fmaf(a1, bv.x, acc[1][0]), acc[1][1] = fmaf(a1, bv.y, acc[1][1]);
      acc[1][2] = fmaf(a1, bv.z, acc[1][2]), acc[1][3] = fmaf(a1, bv.w, acc[1][3]);
      acc[2][0] = fmaf(a2, bv.x, acc[2][0]), acc[2][1] = fmaf(a2, bv.y, acc[2][1]);
      acc[2][2] = fmaf(a2, bv.z, acc[2][2]), acc[2][3] = fmaf(a2, bv.w, acc[2][3]);
      acc[3][0] = fmaf(a3, bv.x, acc[3][0]), acc[3][1] = fmaf(a3, bv.y, acc[3][1]);
      acc[3][2] = fmaf(a3, bv.z, acc[3][2]), acc[3][3] = fmaf(a3, bv.w, acc[3][3]);
    }
  }
  // epilogue: + bias, store NCHW
  T *out = static_cast<T *>(p.out) + (static_cast<long long>(b) * p.Co + static_cast<long long>(g) * Mg) * HoWo;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= Mg) continue;
    const float bv = p.bias ? g_ld(static_cast<const T *>(p.bias) + g * Mg + m) : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int pix = n0 + tx * 4 + j;
      if (pix < HoWo) g_st(out + static_cast<long long>(m) * HoWo + pix, acc[i][j] + bv);
    }
  }
}

static int pick_kc(int Cg, int cpd, int kk) {
  int kc = 16;
  while (kc > 1 && (kc * kk > 48 || Cg % kc || cpd % kc)) kc >>= 1;
  return kc;
}

template <typename T>
int dcn_generic_launch(const T *input, const T *weight, const T *bias, const T *offset, const T *mask, T *output,
                       const DcnGeom &g, cudaStream_t stream) {
  DcnGParams p{};
  p.im = input, p.weight = weight, p.bias = bias, p.offset = offset, p.mask = mask, p.out = output;
  dcn_set_layer(p, g);
  p.groups = g.groups, p.dg = g.dg;
  const int kk = g.kh * g.kw, Cg = g.C / g.groups, cpd = g.C / g.dg;
  p.KC = pick_kc(Cg, cpd, kk);
  const int KB = p.KC * kk;
  const size_t smem = static_cast<size_t>(KB) * (kGT + 1) * 4 + 16 + static_cast<size_t>(KB) * kGT * 4 +
                      static_cast<size_t>(kk) * kGT * sizeof(DcnTap);
  if (smem > 200 * 1024) return B200_ERR_UNSUPPORTED;  // kernels beyond ~12x12 taps
  const long long HoWo = static_cast<long long>(g.Ho) * g.Wo;
  const dim3 grid(static_cast<unsigned>((HoWo + kGT - 1) / kGT), static_cast<unsigned>((g.Co / g.groups + kGT - 1) / kGT),
                  static_cast<unsigned>(g.B * g.groups));
  if (grid.y > 65535u || grid.z > 65535u) return B200_ERR_UNSUPPORTED;
  if (cudaFuncSetAttribute(dcn_generic_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)) !=
      cudaSuccess)
    return B200_ERR_LAUNCH;
  dcn_generic_kernel<T><<<grid, 256, smem, stream>>>(p);
  return check_launch();
}

template int dcn_generic_launch(const float *, const float *, const float *, const float *, const float *, float *, const DcnGeom &, cudaStream_t);
template int dcn_generic_launch(const __half *, const __half *, const __half *, const __half *, const __half *, __half *, const DcnGeom &, cudaStream_t);
template int dcn_generic_launch(const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, const __nv_bfloat16 *, __nv_bfloat16 *, const DcnGeom &, cudaStream_t);

}  // namespace b200

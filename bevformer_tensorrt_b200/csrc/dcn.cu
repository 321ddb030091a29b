// dcn.cu — modulated deformable convolution (DCNv2, plugin ModulatedDeformableConv2dTRT / …TRT2) for H100 (sm_90a):
// entry points and dispatch.
//
// Replaces ModulatedDeformConvForwardCUDAKernel<float|__half|__half2> and …_int8<T>
// (TensorRT/plugin/modulated_deformable_conv2d/modulatedDeformableConv2dKernel.cu:695-978) and its kernels
// (deformable im2col :259-548, cuBLAS GEMM per image and group :735-754, bias / requantisation epilogues :550-607).
//
// Two hand-written kernels, no library GEMM anywhere on this path:
//   * dcn_fused.cu   — wgmma implicit GEMM for the backbone shapes (FP16 and INT8, groups = deformable groups = 1,
//                      C % 64 == 0, Co in {128, 256, 512}): the column tile is sampled straight into the GMMA operand
//                      layout in shared memory, weights arrive by TMA, accumulators live in registers;
//   * dcn_generic.cu — fused implicit GEMM on the FP32 pipe for every other shape (FP32, groups / deformable groups > 1,
//                      small or odd channel counts, any kernel size).
// The reference's `cublas_handle` argument is kept in the C ABI for signature compatibility and ignored.
#include <cstdlib>
#include <type_traits>

#include "dcn_geometry.cuh"

namespace b200 {

// -1: read B200_DCN_FUSED once (default on). Atomic: enqueue may run on several host threads (SURVEY §8(b)).
static std::atomic<int> g_dcn_fused{-1};
static bool dcn_fused_enabled() {
  int v = g_dcn_fused.load(std::memory_order_relaxed);
  if (v < 0) {
    const char *e = getenv("B200_DCN_FUSED");
    v = (e && e[0] == '0') ? 0 : 1;
    g_dcn_fused.store(v, std::memory_order_relaxed);
  }
  return v == 1;
}

template <typename T>
static int dcn_forward(const T *input, const T *weight, const T *bias, const T *offset, const T *mask, T *output,
                       void *workspace, const DcnGeom &g, cudaStream_t stream) {
  if (!input || !weight || !offset || !mask || !output) return B200_ERR_BAD_PARAM;
  if (!dcn_positive(g)) return B200_ERR_BAD_PARAM;
  // the reference exit(1)s on these (…Conv2dPlugin.cpp:300-336); here they are a status
  if (!dcn_groups_divide(g)) return B200_ERR_UNSUPPORTED;
  if (g.Ho <= 0 || g.Wo <= 0) return B200_ERR_BAD_PARAM;
  if (static_cast<long long>(g.C) * (g.kh * g.kw) * (static_cast<long long>(g.Ho) * g.Wo) >= (1ll << 31))
    return B200_ERR_BAD_PARAM;

  // the fused pre-passes use 128-bit accesses: unaligned views (storage offsets) take the generic kernel instead
  const bool aligned = workspace && reinterpret_cast<uintptr_t>(workspace) % 256 == 0 &&
                       reinterpret_cast<uintptr_t>(input) % 16 == 0 && reinterpret_cast<uintptr_t>(weight) % 16 == 0 &&
                       reinterpret_cast<uintptr_t>(output) % 16 == 0;
  // the wgmma kernel reads FP16 bits: BF16 (also 2 bytes) takes the generic kernel
  if (std::is_same<T, __half>::value && aligned && dcn_fused_enabled() && dcn_fused_supported(g))
    return dcn_fused_f16(reinterpret_cast<const __half *>(input), reinterpret_cast<const __half *>(weight),
                         reinterpret_cast<const __half *>(bias), reinterpret_cast<const __half *>(offset),
                         reinterpret_cast<const __half *>(mask), reinterpret_cast<__half *>(output), workspace, g, 0,
                         stream);
  return dcn_generic_launch<T>(input, weight, bias, offset, mask, output, g, stream);
}

// ---- INT8 for the shapes the fused tensor-core kernel does not take (groups / deformable groups > 1, other channel
// counts): dequantise into the workspace, run the generic fused kernel (fp32 accumulation), requantise once.
// A correctness path: every DCN of the BEVFormer backbones goes through dcn_fused_i8 instead.
__global__ void dcn_i8_chw4_to_nchw_f16_kernel(const int8_t *in, float scale, __half *out, int C, long long plane,
                                               long long total) {  // [N, C/4, plane, 4] -> [N, C, plane]
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long pix = idx % plane, nc4 = idx / plane;
    const long long n = nc4 / (C / 4), c4 = nc4 % (C / 4);
    const uint32_t u = ldg32(in + idx * 4);
#pragma unroll
    for (int i = 0; i < 4; ++i)
      out[(n * C + c4 * 4 + i) * plane + pix] = __float2half_rn(static_cast<float>(static_cast<int8_t>(u >> (8 * i))) * scale);
  }
}
__global__ void dcn_i8_to_f16_kernel(const int8_t *in, float scale, __half *out, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    out[i] = __float2half_rn(static_cast<float>(in[i]) * scale);
}
__global__ void dcn_bias_to_f16_kernel(const void *bias, int is_half, __half *out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = is_half ? static_cast<const __half *>(bias)[i] : __float2half_rn(static_cast<const float *>(bias)[i]);
}
__global__ void dcn_f16_to_i8_kernel(const __half *in, float inv_scale, int8_t *out, long long n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    out[i] = static_cast<int8_t>(to_int8_sat(__half2float(in[i]) * inv_scale));
}

struct DcnI8Plan {  // byte offsets into the workspace
  size_t x, w, off, mask, bias, out, total;
};
static DcnI8Plan dcn_i8_plan(const DcnGeom &g) {
  DcnI8Plan p{};
  size_t o = 0;
  p.x = o, o += align256(static_cast<size_t>(g.B) * g.C * g.H * g.W * 2);
  p.w = o, o += align256(static_cast<size_t>(g.Co) * (g.C / g.groups) * g.kh * g.kw * 2);
  p.off = o, o += align256(static_cast<size_t>(g.B) * g.dg * 2 * g.kh * g.kw * g.Ho * g.Wo * 2);
  p.mask = o, o += align256(static_cast<size_t>(g.B) * g.dg * g.kh * g.kw * g.Ho * g.Wo * 2);
  p.bias = o, o += align256(static_cast<size_t>(g.Co) * 2);
  p.out = o, o += align256(static_cast<size_t>(g.B) * g.Co * g.Ho * g.Wo * 2);
  p.total = o;  // (no column buffer: the generic kernel samples straight into shared memory)
  return p;
}

static int dcn_i8_unfused(const int8_t *input, float scale_i, const int8_t *weight, float scale_w, const void *bias,
                          int bias_is_half, const int8_t *offset, float scale_off, const int8_t *mask, float scale_mask,
                          int8_t *output, float scale_o, void *workspace, const DcnGeom &g, cudaStream_t s) {
  if (g.groups <= 0 || g.dg <= 0) return B200_ERR_BAD_PARAM;
  if (g.C % 4 || (g.C / g.groups) % 4 || !dcn_groups_divide(g))
    return B200_ERR_UNSUPPORTED;  // kCHW4 packs 4 channels; the reference exit(1)s on the group mismatches
  const DcnI8Plan pl = dcn_i8_plan(g);
  char *ws = static_cast<char *>(workspace);
  __half *x = reinterpret_cast<__half *>(ws + pl.x), *w = reinterpret_cast<__half *>(ws + pl.w);
  __half *off = reinterpret_cast<__half *>(ws + pl.off), *msk = reinterpret_cast<__half *>(ws + pl.mask);
  __half *b = reinterpret_cast<__half *>(ws + pl.bias), *out = reinterpret_cast<__half *>(ws + pl.out);
  const long long plane = static_cast<long long>(g.H) * g.W, kk = static_cast<long long>(g.kh) * g.kw;
  const long long nx = static_cast<long long>(g.B) * (g.C / 4) * plane;
  const long long nw = static_cast<long long>(g.Co) * (g.C / g.groups / 4) * kk;
  const long long noff = static_cast<long long>(g.B) * g.dg * 2 * kk * g.Ho * g.Wo;
  const long long nout = static_cast<long long>(g.B) * g.Co * g.Ho * g.Wo;
  dcn_i8_chw4_to_nchw_f16_kernel<<<grid_for(nx), 256, 0, s>>>(input, scale_i, x, g.C, plane, nx);
  dcn_i8_chw4_to_nchw_f16_kernel<<<grid_for(nw), 256, 0, s>>>(weight, scale_w, w, g.C / g.groups, kk, nw);
  dcn_i8_to_f16_kernel<<<grid_for(noff), 256, 0, s>>>(offset, scale_off, off, noff);
  dcn_i8_to_f16_kernel<<<grid_for(noff / 2), 256, 0, s>>>(mask, scale_mask, msk, noff / 2);
  if (bias) dcn_bias_to_f16_kernel<<<(g.Co + 255) / 256, 256, 0, s>>>(bias, bias_is_half, b, g.Co);
  g_launch_count.fetch_add(bias ? 4 : 3, std::memory_order_relaxed);
  int st = check_launch();
  if (st != B200_OK) return st;
  st = dcn_forward<__half>(x, w, bias ? b : nullptr, off, msk, out, nullptr, g, s);
  if (st != B200_OK) return st;
  dcn_f16_to_i8_kernel<<<grid_for(nout), 256, 0, s>>>(out, 1.f / scale_o, output, nout);
  return check_launch();
}

// ---- FP16 kCHW2 (what the …TRT2 plugin negotiates for input, offset and weight, …Conv2dPlugin.cpp:222-250): TensorRT's
// [N, ceil(C/2), H, W, 2] packets are unpacked into plain NCHW in the workspace, then the normal FP16 path runs.
__global__ void dcn_chw2_to_nchw_kernel(const __half2 *in, __half *out, int C, long long plane, long long total) {
  // total = N * ceil(C/2) * plane packets
  const int C2 = (C + 1) / 2;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long pix = idx % plane, nc2 = idx / plane;
    const long long n = nc2 / C2, c2 = nc2 % C2;
    const __half2 v = in[idx];
    out[(n * C + 2 * c2) * plane + pix] = __low2half(v);
    if (2 * c2 + 1 < C) out[(n * C + 2 * c2 + 1) * plane + pix] = __high2half(v);
  }
}

struct DcnChw2Plan {
  size_t x, off, w, rest, total;
};
static DcnChw2Plan dcn_chw2_plan(const DcnGeom &g, size_t inner) {
  DcnChw2Plan p{};
  size_t o = 0;
  p.x = o, o += align256(static_cast<size_t>(g.B) * g.C * g.H * g.W * 2);
  p.off = o, o += align256(static_cast<size_t>(g.B) * g.dg * 2 * g.kh * g.kw * g.Ho * g.Wo * 2);
  p.w = o, o += align256(static_cast<size_t>(g.Co) * (g.C / g.groups) * g.kh * g.kw * 2);
  p.rest = o, o += inner;
  p.total = o;
  return p;
}

// The layers a workspace query sizes (it returns 0 for any other). Looser than the launchers' check: the kernel size,
// the dilation and the input's height and width are looked at only through Ho and Wo.
static bool dcn_query_ok(const DcnGeom &g) {
  return g.stride_h > 0 && g.stride_w > 0 && g.groups > 0 && g.dg > 0 && g.Ho > 0 && g.Wo > 0 && g.B > 0 && g.C > 0 &&
         g.Co > 0;
}

// b200_dcn_workspace_size(1, ...): the fused FP16 kernel's workspace for the largest channels_out it takes (the query
// has no channels_out argument, nor has the reference's formula). The generic kernel needs none (the reference sizes a
// column buffer here, …Conv2dPlugin.cpp:73-115). Never 0: hosts pass a real pointer.
static size_t dcn_f16_workspace_bytes(DcnGeom g) {
  g.Co = 512;
  const size_t fused = dcn_fused_workspace_bytes(g);
  return fused > 256 ? fused : 256;
}

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_dcn_workspace_size(int dtype, int batch, int channels, int height, int width, int kernel_w, int kernel_h,
                               int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w, int dilation_h) {
  const DcnGeom g = dcn_geom(batch, channels, height, width, 512, kernel_w, kernel_h, stride_w, stride_h, pad_w, pad_h,
                             dilation_w, dilation_h, 1, 1);
  if (!dcn_query_ok(g)) return 0;
  return dtype == 0 || dtype == 7 ? 256 : dcn_f16_workspace_bytes(g);  // FP32 and BF16 run the generic kernel only
}

size_t b200_dcn_i8_workspace_size(int batch, int channels, int height, int width, int channels_out, int kernel_w,
                                  int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                                  int dilation_h, int group, int deformable_group) {
  const DcnGeom g = dcn_geom(batch, channels, height, width, channels_out, kernel_w, kernel_h, stride_w, stride_h, pad_w,
                             pad_h, dilation_w, dilation_h, group, deformable_group);
  if (!dcn_query_ok(g)) return 0;
  const size_t fused = dcn_f16_workspace_bytes(g), unfused = dcn_i8_plan(g).total;
  return fused > unfused ? fused : unfused;
}

int b200_dcn_set_fused(int enabled) {  // enabled < 0: query only
  const int prev = dcn_fused_enabled() ? 1 : 0;
  if (enabled >= 0) g_dcn_fused.store(enabled ? 1 : 0, std::memory_order_relaxed);
  return prev;
}

int b200_dcn_pack_weights_f16(const void *weight, void *packed, int channels_out, int channels, int kernel_h, int kernel_w,
                              void *stream) {
  if (!weight || !packed || channels_out <= 0 || channels <= 0 || kernel_h <= 0 || kernel_w <= 0) return B200_ERR_BAD_PARAM;
  DcnGeom g{};  // packing depends on the weight's shape alone
  g.C = channels, g.Co = channels_out, g.kh = kernel_h, g.kw = kernel_w, g.groups = g.dg = 1;
  if (!dcn_fused_supported(g)) return B200_ERR_UNSUPPORTED;
  return dcn_pack_weights_f16(static_cast<const __half *>(weight), static_cast<__half *>(packed), g,
                              static_cast<cudaStream_t>(stream));
}

int b200_dcn_f16_ex(const void *input, const void *weight, const void *bias, const void *offset, const void *mask,
                    void *output, void *workspace, int batch, int channels, int height, int width, int channels_out,
                    int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                    int dilation_h, int group, int deformable_group, int flags, void *stream) {
  const DcnGeom g = dcn_geom(batch, channels, height, width, channels_out, kernel_w, kernel_h, stride_w, stride_h, pad_w,
                             pad_h, dilation_w, dilation_h, group, deformable_group);
  if (!input || !weight || !offset || !mask || !output || !workspace) return B200_ERR_BAD_PARAM;
  if (!dcn_positive(g) || g.Ho <= 0 || g.Wo <= 0) return B200_ERR_BAD_PARAM;
  if (!dcn_fused_supported(g) || reinterpret_cast<uintptr_t>(workspace) % 256 != 0 ||
      reinterpret_cast<uintptr_t>(input) % 16 != 0 || reinterpret_cast<uintptr_t>(weight) % 16 != 0)
    return B200_ERR_UNSUPPORTED;
  return dcn_fused_f16(static_cast<const __half *>(input), static_cast<const __half *>(weight),
                       static_cast<const __half *>(bias), static_cast<const __half *>(offset),
                       static_cast<const __half *>(mask), static_cast<__half *>(output), workspace, g, flags,
                       static_cast<cudaStream_t>(stream));
}

int b200_dcn_i8(const int8_t *input, float scale_i, const int8_t *weight, float scale_w, const void *bias, int bias_is_half,
                const int8_t *offset, float scale_off, const int8_t *mask, float scale_mask, int8_t *output, float scale_o,
                void *workspace, int batch, int channels, int height, int width, int channels_out, int kernel_w,
                int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w, int dilation_h, int group,
                int deformable_group, int /*im2col_step*/, void * /*cublas_handle*/, void *stream) {
  const DcnGeom g = dcn_geom(batch, channels, height, width, channels_out, kernel_w, kernel_h, stride_w, stride_h, pad_w,
                             pad_h, dilation_w, dilation_h, group, deformable_group);
  if (!input || !weight || !offset || !mask || !output || !workspace) return B200_ERR_BAD_PARAM;
  // the group counts are checked on the unfused path, after the alignment checks
  if (!dcn_extents_positive(g) || !(scale_o > 0.f) || g.Ho <= 0 || g.Wo <= 0) return B200_ERR_BAD_PARAM;
  if (reinterpret_cast<uintptr_t>(workspace) % 256 != 0) return B200_ERR_UNSUPPORTED;
  // both pre-passes read the kCHW4 input (and the unfused one the weight) as 32-bit packets
  if (reinterpret_cast<uintptr_t>(input) % 4 != 0 || reinterpret_cast<uintptr_t>(weight) % 4 != 0)
    return B200_ERR_UNSUPPORTED;
  // every DCN of the BEVFormer backbones takes the fused tensor-core path; other shapes dequantise into the workspace
  // (sized by b200_dcn_i8_workspace_size) and run the generic fused kernel
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!dcn_fused_enabled() || !dcn_fused_supported(g))
    return dcn_i8_unfused(input, scale_i, weight, scale_w, bias, bias_is_half, offset, scale_off, mask, scale_mask,
                          output, scale_o, workspace, g, s);
  return dcn_fused_i8(input, scale_i, weight, scale_w, bias, bias_is_half, offset, scale_off, mask, scale_mask, output,
                      scale_o, workspace, g, s);
}

// im2col_step is ignored: the reference computes it but loops per image anyway (…Kernel.cu:711-735).
int b200_dcn_f32(const float *input, const float *weight, const float *bias, const float *offset, const float *mask,
                 float *output, void *workspace, int batch, int channels, int height, int width, int channels_out,
                 int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                 int dilation_h, int group, int deformable_group, int /*im2col_step*/, void * /*cublas_handle*/,
                 void *stream) {
  return dcn_forward<float>(input, weight, bias, offset, mask, output, workspace,
                            dcn_geom(batch, channels, height, width, channels_out, kernel_w, kernel_h, stride_w, stride_h,
                                     pad_w, pad_h, dilation_w, dilation_h, group, deformable_group),
                            static_cast<cudaStream_t>(stream));
}

int b200_dcn_f16(const void *input, const void *weight, const void *bias, const void *offset, const void *mask,
                 void *output, void *workspace, int batch, int channels, int height, int width, int channels_out,
                 int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                 int dilation_h, int group, int deformable_group, int /*im2col_step*/, void * /*cublas_handle*/,
                 void *stream) {
  using H = __half;
  return dcn_forward<H>(static_cast<const H *>(input), static_cast<const H *>(weight), static_cast<const H *>(bias),
                        static_cast<const H *>(offset), static_cast<const H *>(mask), static_cast<H *>(output),
                        workspace,
                        dcn_geom(batch, channels, height, width, channels_out, kernel_w, kernel_h, stride_w, stride_h,
                                 pad_w, pad_h, dilation_w, dilation_h, group, deformable_group),
                        static_cast<cudaStream_t>(stream));
}

// BF16: the generic kernel (fp32 accumulation, one rounding per output); there is no BF16 tensor-core path.
int b200_dcn_bf16(const void *input, const void *weight, const void *bias, const void *offset, const void *mask,
                  void *output, void *workspace, int batch, int channels, int height, int width, int channels_out,
                  int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                  int dilation_h, int group, int deformable_group, int /*im2col_step*/, void * /*cublas_handle*/,
                  void *stream) {
  using B = __nv_bfloat16;
  return dcn_forward<B>(static_cast<const B *>(input), static_cast<const B *>(weight), static_cast<const B *>(bias),
                        static_cast<const B *>(offset), static_cast<const B *>(mask), static_cast<B *>(output),
                        workspace,
                        dcn_geom(batch, channels, height, width, channels_out, kernel_w, kernel_h, stride_w, stride_h,
                                 pad_w, pad_h, dilation_w, dilation_h, group, deformable_group),
                        static_cast<cudaStream_t>(stream));
}

size_t b200_dcn_f16_chw2_workspace_size(int batch, int channels, int height, int width, int channels_out, int kernel_w,
                                        int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                                        int dilation_h, int group, int deformable_group) {
  const DcnGeom g = dcn_geom(batch, channels, height, width, channels_out, kernel_w, kernel_h, stride_w, stride_h, pad_w,
                             pad_h, dilation_w, dilation_h, group, deformable_group);
  if (!dcn_query_ok(g)) return 0;
  return dcn_chw2_plan(g, dcn_f16_workspace_bytes(g)).total;
}

int b200_dcn_f16_chw2(const void *input, const void *weight, const void *bias, const void *offset, const void *mask,
                      void *output, void *workspace, int batch, int channels, int height, int width, int channels_out,
                      int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                      int dilation_h, int group, int deformable_group, int /*im2col_step*/, void * /*cublas_handle*/,
                      void *stream) {
  const DcnGeom g = dcn_geom(batch, channels, height, width, channels_out, kernel_w, kernel_h, stride_w, stride_h, pad_w,
                             pad_h, dilation_w, dilation_h, group, deformable_group);
  if (!input || !weight || !offset || !mask || !output || !workspace) return B200_ERR_BAD_PARAM;
  if (!dcn_positive(g)) return B200_ERR_BAD_PARAM;
  if (!dcn_groups_divide(g)) return B200_ERR_UNSUPPORTED;
  if (reinterpret_cast<uintptr_t>(workspace) % 256 != 0) return B200_ERR_UNSUPPORTED;
  if (g.Ho <= 0 || g.Wo <= 0) return B200_ERR_BAD_PARAM;
  const DcnChw2Plan pl = dcn_chw2_plan(g, dcn_f16_workspace_bytes(g));
  char *ws = static_cast<char *>(workspace);
  __half *x = reinterpret_cast<__half *>(ws + pl.x), *off = reinterpret_cast<__half *>(ws + pl.off);
  __half *w = reinterpret_cast<__half *>(ws + pl.w);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long plane = static_cast<long long>(g.H) * g.W, kk = static_cast<long long>(g.kh) * g.kw;
  const int coff = g.dg * 2 * static_cast<int>(kk), cw = g.C / g.groups;
  const long long nx = static_cast<long long>(g.B) * ((g.C + 1) / 2) * plane;
  const long long no = static_cast<long long>(g.B) * ((coff + 1) / 2) * g.Ho * g.Wo;
  const long long nw = static_cast<long long>(g.Co) * ((cw + 1) / 2) * kk;
  dcn_chw2_to_nchw_kernel<<<grid_for(nx), 256, 0, s>>>(static_cast<const __half2 *>(input), x, g.C, plane, nx);
  dcn_chw2_to_nchw_kernel<<<grid_for(no), 256, 0, s>>>(static_cast<const __half2 *>(offset), off, coff,
                                                      static_cast<long long>(g.Ho) * g.Wo, no);
  dcn_chw2_to_nchw_kernel<<<grid_for(nw), 256, 0, s>>>(static_cast<const __half2 *>(weight), w, cw, kk, nw);
  g_launch_count.fetch_add(2, std::memory_order_relaxed);
  const int st = check_launch();
  if (st != B200_OK) return st;
  return dcn_forward<__half>(x, w, static_cast<const __half *>(bias), off, static_cast<const __half *>(mask),
                             static_cast<__half *>(output), ws + pl.rest, g, s);
}

}  // extern "C"

// rotate.cu — RotateTRT / RotateTRT2 for H100 (sm_90a).
//
// Replaces the reference launchers rotate<float|__half>, rotate_h2 and rotate_int8<float|__half>
// (TensorRT/plugin/rotate/rotateKernel.cu:708-748) and their kernels (:128-705). BEVFormer calls it once per frame to
// align prev_bev with the ego motion (det2trt/models/modules/transformer.py:296-304): img [C, H, W], angle [1] in
// degrees, center [2] in pixels; out[c, h, w] = img sampled at the pixel the inverse rotation maps (h, w) to,
// zero-padded, bilinear or nearest.
//
// Semantics = the reference FP32 kernel (:128-210), including where its SASS contracts to FFMA (the index arithmetic
// decides which pixel "nearest" picks, so the contraction pattern is reproduced with explicit __f*_rn intrinsics; see
// rot_matrix / rot_source_index). The reference's __half kernels compute the matrix and the coordinates in half
// precision (:213-260, 0.25-pixel resolution at x = 500) and its INT8 kernel quantises the four tap weights to 7 bits
// and leaves out-of-image taps uninitialised (:470-520); neither is reproduced: FP16 and INT8 images are converted in
// registers, coordinates and blending are fp32, INT8 output is requantised once (T2int8).
//
// The reference runs one thread per pixel that walks all C channels with a read-modify-write on the output per tap and
// recomputes cos/sin six times per thread. Here the matrix is computed once per CTA, a thread owns (pixel, slice of
// channel packets) for the planar layouts, and for the channels-last entry (b200_rotate_hwc: prev_bev is [H*W, C] in
// memory at the call site, the reference permutes it twice around the plugin) a thread owns one 16-byte channel
// vector of one pixel, so every tap is a fully coalesced 128-bit load.
#include <climits>
#include <cmath>

#include "common.cuh"
#include "packets.cuh"

namespace b200 {

struct RotParams {
  const void *in;
  void *out;
  const void *angle, *center;
  float *debug;    // rotate_index_kernel only: [H*W*2] source indices (ix, iy)
  int C, CP, H, W;
  int interp;      // 0 bilinear, 1 nearest (RotateInterpolation, rotateKernel.h:12)
  int ac_half;     // angle / center are __half
  int slices, cps;
  float scale_i, scale_o;
};

// ---- index arithmetic: op-for-op the reference FP32 kernel as compiled (fmad contraction included) -----------------
// m = {cos, sin, m2, m5}: matrix[0] = matrix[4] = cos, matrix[1] = -matrix[3] = sin (:138-143).
__device__ __forceinline__ void rot_matrix(const RotParams &p, float (&m)[4]) {
  float a, c0, c1;
  if (p.ac_half) {
    a = __half2float(__ldg(static_cast<const __half *>(p.angle)));
    c0 = __half2float(__ldg(static_cast<const __half *>(p.center)));
    c1 = __half2float(__ldg(static_cast<const __half *>(p.center) + 1));
  } else {
    a = __ldg(static_cast<const float *>(p.angle));
    c0 = __ldg(static_cast<const float *>(p.center));
    c1 = __ldg(static_cast<const float *>(p.center) + 1);
  }
  // -(*angle) * M_PI / 180.f : float * double / float -> evaluated in double, rounded once (:137)
  const float ang = static_cast<float>(static_cast<double>(-a) * M_PI / 180.0);
  const float c = cosf(ang), s = sinf(ang);
  const float cx = __fsub_rn(c0, __fmul_rn(0.5f, static_cast<float>(p.W)));
  const float cy = __fsub_rn(c1, __fmul_rn(0.5f, static_cast<float>(p.H)));
  m[0] = c, m[1] = s;
  m[2] = __fadd_rn(cx, __fmaf_rn(-cx, c, -__fmul_rn(cy, s)));  // -cx*cos - cy*sin + cx
  m[3] = __fadd_rn(cy, __fmaf_rn(-cy, c, __fmul_rn(cx, s)));   //  cx*sin - cy*cos + cy
}

__device__ __forceinline__ float rot_safe(float x) {  // safe_downgrade_to_int_range (:73-78)
  if (x > static_cast<float>(INT_MAX - 1) || x < static_cast<float>(INT_MIN) || !isfinite(x)) return -100.f;
  return x;
}

__device__ __forceinline__ void rot_source_index(const float (&m)[4], int w, int h, int W, int H, float &ix,
                                                 float &iy) {
  const float x = (0.5f - 0.5f * W) + w, y = (0.5f - 0.5f * H) + h;  // exact in fp32 (:148)
  const float nx = __fadd_rn(m[2], __fmaf_rn(m[0], x, __fmul_rn(m[1], y)));
  const float ny = __fadd_rn(m[3], __fmaf_rn(m[0], y, -__fmul_rn(m[1], x)));
  const float gx = __fdiv_rn(nx, __fmul_rn(0.5f, static_cast<float>(W)));
  const float gy = __fdiv_rn(ny, __fmul_rn(0.5f, static_cast<float>(H)));
  // grid_sampler_compute_source_index: ((coord + 1) * size - 1) / 2 (:103-109)
  ix = rot_safe(__fmul_rn(__fmaf_rn(static_cast<float>(W), __fadd_rn(gx, 1.f), -1.f), 0.5f));
  iy = rot_safe(__fmul_rn(__fmaf_rn(static_cast<float>(H), __fadd_rn(gy, 1.f), -1.f), 0.5f));
}

// Four taps of one output pixel: clamped offsets (in pixels), weights and validity (bit i of `in`: tap i is inside the
// image). An out-of-image tap aliases an in-image pixel; what it loads is dropped, not multiplied by its zero weight
// (0 * Inf is NaN, and the reference never loads such a tap). Nearest = one tap.
struct RotTaps {
  int o[4];
  float w[4];
  unsigned in;
};
template <int INTERP>
__device__ __forceinline__ RotTaps rot_taps(float ix, float iy, int W, int H) {
  RotTaps t;
  if (INTERP == 0) {
    const int x0 = static_cast<int>(floorf(ix)), y0 = static_cast<int>(floorf(iy));
    const int x1 = x0 + 1, y1 = y0 + 1;
    const float fx1 = __fsub_rn(static_cast<float>(x1), ix), fx0 = __fsub_rn(ix, static_cast<float>(x0));
    const float fy1 = __fsub_rn(static_cast<float>(y1), iy), fy0 = __fsub_rn(iy, static_cast<float>(y0));
    const bool vx0 = x0 >= 0 && x0 < W, vx1 = x1 >= 0 && x1 < W, vy0 = y0 >= 0 && y0 < H, vy1 = y1 >= 0 && y1 < H;
    t.w[0] = (vx0 && vy0) ? __fmul_rn(fx1, fy1) : 0.f, t.w[1] = (vx1 && vy0) ? __fmul_rn(fx0, fy1) : 0.f;
    t.w[2] = (vx0 && vy1) ? __fmul_rn(fx1, fy0) : 0.f, t.w[3] = (vx1 && vy1) ? __fmul_rn(fx0, fy0) : 0.f;
    const int cx0 = min(max(x0, 0), W - 1), cx1 = min(max(x1, 0), W - 1);
    const int cy0 = min(max(y0, 0), H - 1), cy1 = min(max(y1, 0), H - 1);
    t.o[0] = cy0 * W + cx0, t.o[1] = cy0 * W + cx1, t.o[2] = cy1 * W + cx0, t.o[3] = cy1 * W + cx1;
    t.in = ((vx0 && vy0) ? 1u : 0u) | ((vx1 && vy0) ? 2u : 0u) | ((vx0 && vy1) ? 4u : 0u) | ((vx1 && vy1) ? 8u : 0u);
  } else {
    const int xn = static_cast<int>(roundf(ix)), yn = static_cast<int>(roundf(iy));  // ::round (:190-191)
    const bool ok = xn >= 0 && xn < W && yn >= 0 && yn < H;
    t.o[0] = ok ? yn * W + xn : 0, t.w[0] = ok ? 1.f : 0.f;
    t.o[1] = t.o[2] = t.o[3] = 0, t.w[1] = t.w[2] = t.w[3] = 0.f;
    t.in = ok ? 1u : 0u;
  }
  return t;
}

// ---- planar layouts: [CP, H, W] packets (kLINEAR fp32/fp16, kCHW2, kCHW4) -----------------------------------------
template <int K, int INTERP>
__global__ void __launch_bounds__(256, 4) rotate_planar_kernel(const RotParams p) {
  using P = Pk<K>;
  using T = typename P::T;
  constexpr int PW = P::W;
  __shared__ float sm[4];
  if (threadIdx.x == 0) {
    float m[4];
    rot_matrix(p, m);
    sm[0] = m[0], sm[1] = m[1], sm[2] = m[2], sm[3] = m[3];
  }
  __syncthreads();
  const float m[4] = {sm[0], sm[1], sm[2], sm[3]};
  const int plane = p.H * p.W;
  const long long total = static_cast<long long>(p.slices) * plane;
  const float so = K == kI8x4 ? 1.f / p.scale_o : 1.f;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int pix = static_cast<int>(idx % plane), s = static_cast<int>(idx / plane);
    const int w = pix % p.W, h = pix / p.W;
    float ix, iy;
    rot_source_index(m, w, h, p.W, p.H, ix, iy);
    const RotTaps t = rot_taps<INTERP>(ix, iy, p.W, p.H);
    const int cp0 = s * p.cps, cp1 = min(p.CP, cp0 + p.cps);
    const T *ip = static_cast<const T *>(p.in) + static_cast<long long>(cp0) * plane;
    T *op = static_cast<T *>(p.out) + static_cast<long long>(cp0) * plane + pix;
    if (INTERP == 0) {
#pragma unroll 4
      for (int cp = cp0; cp < cp1; ++cp, ip += plane, op += plane) {
        float a[PW], b[PW], c[PW], d[PW], o[PW];
        pk_load_if<K>(ip + t.o[0], t.in & 1u, a, p.scale_i), pk_load_if<K>(ip + t.o[1], t.in & 2u, b, p.scale_i);
        pk_load_if<K>(ip + t.o[2], t.in & 4u, c, p.scale_i), pk_load_if<K>(ip + t.o[3], t.in & 8u, d, p.scale_i);
#pragma unroll
        for (int i = 0; i < PW; ++i)
          o[i] = fmaf(d[i], t.w[3], fmaf(c[i], t.w[2], fmaf(b[i], t.w[1], a[i] * t.w[0])));
        P::store(op, o, so);
      }
    } else {
#pragma unroll 4
      for (int cp = cp0; cp < cp1; ++cp, ip += plane, op += plane) {
        float a[PW];
        P::load(ip + t.o[0], a, p.scale_i);
#pragma unroll
        for (int i = 0; i < PW; ++i) a[i] = t.w[0] != 0.f ? a[i] : 0.f;
        P::store(op, a, so);
      }
    }
  }
}

// ---- channels-last: [H, W, C], 16-byte channel vectors ----------------------------------------------------------------
template <int K>
struct Vec16;
template <>
struct Vec16<kF32> {
  static constexpr int N = 4;
  __device__ static void load(const void *p, bool valid, float (&v)[4]) {
    uint4 u = ldg128(p);
    if (!valid) u = make_uint4(0u, 0u, 0u, 0u);
    v[0] = __uint_as_float(u.x), v[1] = __uint_as_float(u.y), v[2] = __uint_as_float(u.z), v[3] = __uint_as_float(u.w);
  }
  __device__ static void store(void *p, const float (&v)[4]) {
    stg128_stream(p, make_uint4(__float_as_uint(v[0]), __float_as_uint(v[1]), __float_as_uint(v[2]),
                                __float_as_uint(v[3])));
  }
};
template <>
struct Vec16<kF16> {
  static constexpr int N = 8;
  __device__ static void load(const void *p, bool valid, float (&v)[8]) {
    uint4 u = ldg128(p);
    if (!valid) u = make_uint4(0u, 0u, 0u, 0u);
    const uint32_t r[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = h2_to_f2(r[i]);
      v[2 * i] = f.x, v[2 * i + 1] = f.y;
    }
  }
  __device__ static void store(void *p, const float (&v)[8]) {
    stg128_stream(p, make_uint4(f2_to_h2(v[0], v[1]), f2_to_h2(v[2], v[3]), f2_to_h2(v[4], v[5]),
                                f2_to_h2(v[6], v[7])));
  }
};

// LP lanes share one pixel: lane j blends the 16-byte vectors j, j + LP, ... of its four taps, so the index arithmetic
// (two IEEE divisions) is paid once per LP-th of a pixel and each group of 8 lanes reads whole 128-byte lines.
template <int K, int INTERP>
__global__ void __launch_bounds__(256, 3) rotate_hwc_kernel(const RotParams p) {
  using V = Vec16<K>;
  constexpr int N = V::N;
  __shared__ float sm[4];
  if (threadIdx.x == 0) {
    float m[4];
    rot_matrix(p, m);
    sm[0] = m[0], sm[1] = m[1], sm[2] = m[2], sm[3] = m[3];
  }
  __syncthreads();
  const float m[4] = {sm[0], sm[1], sm[2], sm[3]};
  const int nvec = p.C / N, lp = p.slices;  // lanes per pixel (power of two <= 8)
  const long long total = static_cast<long long>(p.H) * p.W * lp;
  constexpr size_t esz = K == kF32 ? 4 : 2;
  const size_t row = static_cast<size_t>(p.C) * esz;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(idx % lp), pix = static_cast<int>(idx / lp);
    const int w = pix % p.W, h = pix / p.W;
    float ix, iy;
    rot_source_index(m, w, h, p.W, p.H, ix, iy);
    const RotTaps t = rot_taps<INTERP>(ix, iy, p.W, p.H);
    const char *i0 = static_cast<const char *>(p.in) + t.o[0] * row, *i1 = static_cast<const char *>(p.in) + t.o[1] * row;
    const char *i2 = static_cast<const char *>(p.in) + t.o[2] * row, *i3 = static_cast<const char *>(p.in) + t.o[3] * row;
    char *op = static_cast<char *>(p.out) + static_cast<size_t>(pix) * row;
#pragma unroll 2
    for (int v = j; v < nvec; v += lp) {
      const size_t off = static_cast<size_t>(v) * N * esz;
      float o[N];
      if (INTERP == 0) {
        float a[N], b[N], c[N], d[N];
        V::load(i0 + off, t.in & 1u, a), V::load(i1 + off, t.in & 2u, b), V::load(i2 + off, t.in & 4u, c);
        V::load(i3 + off, t.in & 8u, d);
#pragma unroll
        for (int i = 0; i < N; ++i) o[i] = fmaf(d[i], t.w[3], fmaf(c[i], t.w[2], fmaf(b[i], t.w[1], a[i] * t.w[0])));
      } else {
        V::load(i0 + off, t.in & 1u, o);
      }
      V::store(op + off, o);
    }
  }
}

// Source indices only (tests: the part of the op that must match the reference bit for bit).
__global__ void rotate_index_kernel(const RotParams p) {
  float m[4];
  rot_matrix(p, m);
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= p.H * p.W) return;
  float ix, iy;
  rot_source_index(m, pix % p.W, pix / p.W, p.W, p.H, ix, iy);
  p.debug[2 * pix] = ix, p.debug[2 * pix + 1] = iy;
}

// ---- host -----------------------------------------------------------------------------------------------------------
// The one check of an image's dims {C, H, W}, which fills p's C, CP (packets of `width` channels), H and W: every extent
// positive and a plane below 2^31 pixels (the kernels index a plane in int).
static int rot_geom(RotParams &p, const int *dims, int width) {
  if (!dims || dims[0] <= 0 || dims[1] <= 0 || dims[2] <= 0) return B200_ERR_BAD_PARAM;
  if (static_cast<long long>(dims[1]) * dims[2] >= (1ll << 31)) return B200_ERR_BAD_PARAM;
  p.C = dims[0], p.CP = (dims[0] + width - 1) / width, p.H = dims[1], p.W = dims[2];
  return B200_OK;
}

// The checks both image launchers share; fills the parameters both take.
static int rot_params(RotParams &p, void *out, const void *in, const void *angle, const void *center, const int *dims,
                      int width, int interp) {
  if (!out || !in || !angle || !center || interp < 0 || interp > 1) return B200_ERR_BAD_PARAM;
  p = RotParams{};
  p.in = in, p.out = out, p.angle = angle, p.center = center, p.interp = interp;
  return rot_geom(p, dims, width);
}

template <int K>
static int launch_rotate(void *out, const void *in, const void *angle, const void *center, int ac_half,
                         const int *dims, int interp, float si, float so, void *stream) {
  RotParams p;
  const int st = rot_params(p, out, in, angle, center, dims, Pk<K>::W, interp);
  if (st != B200_OK) return st;
  p.ac_half = ac_half, p.scale_i = si, p.scale_o = so;
  // enough (pixel, slice) threads to fill 132 SMs a few times over, at most 16 packets per thread
  const unsigned blocks = plan_slices(static_cast<long long>(p.H) * p.W, p.CP, 132ll * 2048 * 4, 16, p.slices, p.cps);
  (interp == 0 ? rotate_planar_kernel<K, 0> : rotate_planar_kernel<K, 1>)<<<blocks, 256, 0,
                                                                          static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch();
}

template <int K>
static int launch_rotate_hwc(void *out, const void *in, const void *angle, const void *center, const int *dims,
                             int interp, void *stream) {
  RotParams p;
  const int st = rot_params(p, out, in, angle, center, dims, 1, interp);
  if (st != B200_OK) return st;
  if (p.C % Vec16<K>::N) return B200_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) return B200_ERR_UNSUPPORTED;
  p.ac_half = K == kF16;
  const int nvec = p.C / Vec16<K>::N;
  p.slices = nvec >= 8 ? 8 : nvec >= 4 ? 4 : nvec >= 2 ? 2 : 1;
  const unsigned blocks = capped_blocks(static_cast<long long>(p.H) * p.W * p.slices);
  (interp == 0 ? rotate_hwc_kernel<K, 0> : rotate_hwc_kernel<K, 1>)<<<blocks, 256, 0,
                                                                    static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch();
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_rotate_f32(float *output, const float *input, const float *angle, const float *center,
                    const int *input_dims, int interp, void *stream) {
  return launch_rotate<kF32>(output, input, angle, center, 0, input_dims, interp, 1.f, 1.f, stream);
}

int b200_rotate_f16(void *output, const void *input, const void *angle, const void *center, const int *input_dims,
                    int interp, void *stream) {
  return launch_rotate<kF16>(output, input, angle, center, 1, input_dims, interp, 1.f, 1.f, stream);
}

int b200_rotate_f16_h2(void *output, const void *input, const void *angle, const void *center, const int *input_dims,
                       int interp, void *stream) {
  return launch_rotate<kF16x2>(output, input, angle, center, 1, input_dims, interp, 1.f, 1.f, stream);
}

int b200_rotate_i8(int8_t *output, float scale_o, const int8_t *input, float scale_i, const void *angle,
                   const void *center, int angle_is_half, const int *input_dims, int interp, void *stream) {
  if (!(scale_o > 0.f)) return B200_ERR_BAD_PARAM;
  return launch_rotate<kI8x4>(output, input, angle, center, angle_is_half != 0, input_dims, interp, scale_i, scale_o,
                              stream);
}

int b200_rotate_hwc(void *output, const void *input, const void *angle, const void *center, int dtype,
                    const int *input_dims, int interp, void *stream) {
  if (dtype == 0) return launch_rotate_hwc<kF32>(output, input, angle, center, input_dims, interp, stream);
  if (dtype == 1) return launch_rotate_hwc<kF16>(output, input, angle, center, input_dims, interp, stream);
  return B200_ERR_UNSUPPORTED;
}

int b200_rotate_debug_indices(const float *angle, const float *center, const int *input_dims, float *source_xy,
                              void *stream) {
  if (!angle || !center || !source_xy) return B200_ERR_BAD_PARAM;
  RotParams p{};
  const int st = rot_geom(p, input_dims, 1);
  if (st != B200_OK) return st;
  const long long total = static_cast<long long>(p.H) * p.W;
  if (2 * total >= (1ll << 31)) return B200_ERR_BAD_PARAM;  // the kernel indexes source_xy in int
  p.angle = angle, p.center = center, p.debug = source_xy;
  rotate_index_kernel<<<static_cast<unsigned>(total / 256 + 1), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  return check_launch();
}

}  // extern "C"

// packets.cuh — per-layout packet I/O shared by the samplers (grid_sampler.cu, rotate.cu).
//
// A packet is the unit stored per (channel group, pixel) by the TensorRT tensor formats the reference plugins accept
// (gridSamplerPlugin.cpp:184-232, rotatePlugin.cpp:122-153): float / __half (kLINEAR), __half2 (kCHW2), 4 x int8
// (kCHW4). Values are converted to fp32 registers on load and back on store; INT8 requantises once (T2int8).
#pragma once
#include "common.cuh"

namespace b200 {

enum { kF32 = 0, kF16 = 1, kF16x2 = 2, kI8x4 = 3 };

// Pk<K>::zero() is the packet whose every channel unpacks to +0. A bilinear tap outside the image is loaded from a
// clamped (in-image) address and then replaced by it (pk_load_if), so that it contributes exactly 0 whatever the
// aliased pixel holds: 0 * Inf and 0 * NaN are NaN, and the reference never loads such a tap at all.

template <int K>
struct Pk;
template <>
struct Pk<kF32> {
  using T = float;
  static constexpr int W = 1;
  __device__ static void unpack(T raw, float (&v)[1], float) { v[0] = raw; }
  __device__ static void load(const T *p, float (&v)[1], float) { v[0] = __ldg(p); }
  __device__ static T zero() { return 0.f; }
  __device__ static void store(T *p, const float (&v)[1], float) { *p = v[0]; }
  __device__ static void grid_xy(const void *g, long long plane, long long pix, long long n, float, float &x, float &y,
                                 float &z, bool has_z) {
    const T *gp = static_cast<const T *>(g) + n * (has_z ? 3 : 2) * plane + pix;
    x = __ldg(gp), y = __ldg(gp + plane), z = has_z ? __ldg(gp + 2 * plane) : 0.f;
  }
};
template <>
struct Pk<kF16> {
  using T = __half;
  static constexpr int W = 1;
  __device__ static void unpack(T raw, float (&v)[1], float) { v[0] = __half2float(raw); }
  __device__ static void load(const T *p, float (&v)[1], float) { v[0] = __half2float(__ldg(p)); }
  __device__ static T zero() { return __ushort_as_half(0); }
  __device__ static void store(T *p, const float (&v)[1], float) { *p = __float2half_rn(v[0]); }
  __device__ static void grid_xy(const void *g, long long plane, long long pix, long long n, float, float &x, float &y,
                                 float &z, bool has_z) {
    const T *gp = static_cast<const T *>(g) + n * (has_z ? 3 : 2) * plane + pix;
    x = __half2float(__ldg(gp)), y = __half2float(__ldg(gp + plane));
    z = has_z ? __half2float(__ldg(gp + 2 * plane)) : 0.f;
  }
};
template <>
struct Pk<kF16x2> {  // kCHW2: [N, ceil(C/2), H, W, 2]; the 2-channel grid is one (x, y) pair per pixel (:946-961)
  using T = uint32_t;
  static constexpr int W = 2;
  __device__ static void unpack(T raw, float (&v)[2], float) {
    const float2 f = h2_to_f2(raw);
    v[0] = f.x, v[1] = f.y;
  }
  __device__ static void load(const T *p, float (&v)[2], float) {
    const float2 f = h2_to_f2(__ldg(p));
    v[0] = f.x, v[1] = f.y;
  }
  __device__ static T zero() { return 0u; }
  __device__ static void store(T *p, const float (&v)[2], float) { *p = f2_to_h2(v[0], v[1]); }
  __device__ static void grid_xy(const void *g, long long plane, long long pix, long long n, float, float &x, float &y,
                                 float &z, bool) {
    const float2 f = h2_to_f2(__ldg(static_cast<const T *>(g) + n * plane + pix));
    x = f.x, y = f.y, z = 0.f;
  }
};
template <>
struct Pk<kI8x4> {  // kCHW4: [N, ceil(C/4), H, W, 4]; grid = (x, y, pad, pad) int8 per pixel (:1088-1103)
  using T = uint32_t;
  static constexpr int W = 4;
  __device__ static void unpack(T raw, float (&v)[4], float s) {
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = static_cast<float>(static_cast<int8_t>(raw >> (8 * i))) * s;
  }
  __device__ static void load(const T *p, float (&v)[4], float s) {
    const uint32_t u = __ldg(p);
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = static_cast<float>(static_cast<int8_t>(u >> (8 * i))) * s;
  }
  __device__ static T zero() { return 0u; }
  __device__ static void store(T *p, const float (&v)[4], float inv_so) {
    uint32_t u = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) u |= (static_cast<uint32_t>(to_int8_sat(v[i] * inv_so)) & 0xffu) << (8 * i);
    *p = u;
  }
  __device__ static void grid_xy(const void *g, long long plane, long long pix, long long n, float sg, float &x,
                                 float &y, float &z, bool) {
    const uint32_t u = __ldg(static_cast<const T *>(g) + n * plane + pix);
    x = static_cast<float>(static_cast<int8_t>(u)) * sg, y = static_cast<float>(static_cast<int8_t>(u >> 8)) * sg;
    z = 0.f;
  }
};

template <int K>
__device__ __forceinline__ void pk_unpack_if(typename Pk<K>::T raw, bool valid, float (&v)[Pk<K>::W], float s) {
  Pk<K>::unpack(valid ? raw : Pk<K>::zero(), v, s);  // one select on the raw word, before any conversion
}
template <int K>
__device__ __forceinline__ void pk_load_if(const typename Pk<K>::T *p, bool valid, float (&v)[Pk<K>::W], float s) {
  pk_unpack_if<K>(__ldg(p), valid, v, s);
}

}  // namespace b200

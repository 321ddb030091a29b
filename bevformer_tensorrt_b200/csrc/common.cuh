// common.cuh — shared device/host helpers for libb200_bev_ops (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "b200_bev_ops.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libb200_bev_ops is written for sm_90a (H100) only"
#endif

namespace b200 {

extern std::atomic<unsigned long long> g_launch_count;

inline int check_launch() {
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  return cudaGetLastError() == cudaSuccess ? B200_OK : B200_ERR_LAUNCH;
}

// workspace carve-outs start on 256-byte boundaries
inline size_t align256(size_t b) { return (b + 255) / 256 * 256; }

// Blocks of 256 threads for a grid-stride loop over `threads` items, capped at 2^22.
inline unsigned capped_blocks(long long threads) {
  return static_cast<unsigned>(threads / 256 + 1 < (1 << 22) ? threads / 256 + 1 : (1 << 22));
}

// (pixel, slice) threads: a pixel's channel packets are split into `slices` runs of `cps` packets. Slices double until
// there are at least min_threads threads and at most max_cps packets per thread, or every packet has its own slice.
// Returns the blocks of 256 threads.
inline unsigned plan_slices(long long pixels, int packets, long long min_threads, int max_cps, int &slices, int &cps) {
  int n = 1;
  while (n < packets && (pixels * n < min_threads || (packets + n - 1) / n > max_cps)) n <<= 1;
  cps = (packets + n - 1) / n;
  slices = (packets + cps - 1) / cps;
  return capped_blocks(pixels * slices);
}

constexpr unsigned kFullMask = 0xffffffffu;

// ---- 128-bit read-only loads -------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ldg128(const void *p) { return __ldg(reinterpret_cast<const uint4 *>(p)); }
__device__ __forceinline__ uint2 ldg64(const void *p) { return __ldg(reinterpret_cast<const uint2 *>(p)); }
__device__ __forceinline__ uint32_t ldg32(const void *p) { return __ldg(reinterpret_cast<const uint32_t *>(p)); }

// streaming (read-once) variants: do not allocate in L1, evict-first in L2 is left to the default policy
__device__ __forceinline__ uint4 ldg128_stream(const void *p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint2 ldg64_stream(const void *p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ uint32_t ldg32_stream(const void *p) {
  uint32_t r;
  asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ void stg128_stream(void *p, uint4 v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

__device__ __forceinline__ float2 h2_to_f2(uint32_t u) {
  return __half22float2(*reinterpret_cast<const __half2 *>(&u));
}
__device__ __forceinline__ uint32_t f2_to_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t *>(&h);
}

// BF16 is the upper half of an fp32 word, so a packed pair widens exactly with a shift and a mask (no conversion
// instruction); the store rounds to nearest even once.
__device__ __forceinline__ float2 bf2_to_f2(uint32_t u) {
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
__device__ __forceinline__ uint32_t f2_to_bf2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t *>(&h);
}
__device__ __forceinline__ float bf16_to_f(__nv_bfloat16 v) {
  return __uint_as_float(static_cast<uint32_t>(__bfloat16_as_ushort(v)) << 16);
}

// d = a(f16) * b(f16) + c(f32) with one rounding: the product of two fp16 values (11-bit significands) is exact in fp32,
// so widening both factors and issuing one fp32 FMA rounds exactly once.
__device__ __forceinline__ float fma_f32_f16(unsigned short a, unsigned short b, float c) {
  return fmaf(__half2float(__ushort_as_half(a)), __half2float(__ushort_as_half(b)), c);
}

// T2int8<float> of the reference (multiScaleDeformableAttnKernel.cu:51-55): saturate, round half away from zero.
__device__ __forceinline__ int to_int8_sat(float a) {
  a = a > 127.f ? 127.f : a;
  a = a < -128.f ? -128.f : a;
  return static_cast<int>(a + (a > 0.f ? 0.5f : -0.5f));
}

}  // namespace b200

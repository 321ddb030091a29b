// msda_geometry.cuh — the geometry of one multi-scale deformable attention call, as the msda*.cu host code passes it
// around: every C-ABI entry builds it once from its scalar arguments (msda_geom) and hands it on by reference.
#pragma once
#include <initializer_list>

#include "common.cuh"

namespace b200 {

struct MsdaGeom {
  int B, S, M, C, L, Q, P, G;
};

// Arguments in the C ABI's order.
inline MsdaGeom msda_geom(int batch, int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                          int num_point, int points_per_group) {
  return MsdaGeom{batch, spatial_size, num_heads, channels, num_levels, num_query, num_point, points_per_group};
}

// The kernels keep one lane (gather) or one shared-memory slot (backward) per level.
constexpr int kMsdaMaxLevels = 16;

// The envelope of every forward and backward entry: every dimension positive, at most kMsdaMaxLevels levels, and value
// element offsets (at 4 bytes per element, one row past the end) below 2^31.
inline int msda_check_dims(const MsdaGeom &g) {
  if (g.B <= 0 || g.S <= 0 || g.M <= 0 || g.C <= 0 || g.L <= 0 || g.Q <= 0 || g.P <= 0 || g.G <= 0)
    return B200_ERR_BAD_PARAM;
  if (g.L > kMsdaMaxLevels) return B200_ERR_UNSUPPORTED;
  if ((static_cast<long long>(g.S) + 1) * g.M * g.C * 4 >= (1ll << 31)) return B200_ERR_BAD_PARAM;
  return B200_OK;
}

// The shape every lane-group kernel takes: 32 channels per head (every BEVFormer call site), points in chunks of 4,
// 1 / 2 / 4 reference points per query, and at most `max_points` points (L * P) per item, the caller's own bound.
inline bool msda_lane_group_shape(const MsdaGeom &g, int max_points) {
  return g.C == 32 && g.P % 4 == 0 && (g.G == 1 || g.G == 2 || g.G == 4) && g.L * g.P <= max_points;
}

// Every pointer of `ptrs` is a multiple of `align` bytes (a null pointer is).
inline bool msda_aligned(std::initializer_list<const void *> ptrs, uintptr_t align) {
  for (const void *q : ptrs)
    if (reinterpret_cast<uintptr_t>(q) % align) return false;
  return true;
}

// The geometry of a kernel's parameter struct (MsdaParams, MsdaBwParams); ResParams, PackParams and I8PParams carry a
// subset, which their launchers set.
template <typename Prm>
inline void msda_set_dims(Prm &p, const MsdaGeom &g) {
  p.B = g.B, p.S = g.S, p.M = g.M, p.C = g.C, p.L = g.L, p.Q = g.Q, p.P = g.P, p.G = g.G;
}

// Grid of a grid-stride kernel over n elements at 256 threads per CTA: ceil(n / 256) CTAs, at least 1, at most 2^20.
inline unsigned msda_grid_for(long long n) {
  const long long b = (n + 255) / 256;
  return static_cast<unsigned>(b < (1 << 20) ? (b > 0 ? b : 1) : (1 << 20));
}

// Streaming multiprocessors of the current device, for the persistent launches (132 if the query fails).
inline int msda_sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

// Grid of the persistent resident-tail (msda_res.cu) and packed INT8 (msda_v2.cu) kernels: a CTA is bound to one
// (camera, head) pair, `cpp` CTAs share a pair and interleave its blocks of `items_per_block` queries, and there are
// never more CTAs than SMs or than a pair has query blocks.
struct MsdaSlabGrid {
  int cpp, grid;
};
inline MsdaSlabGrid msda_slab_grid(const MsdaGeom &g, int sms, int items_per_block) {
  const int pairs = g.B * g.M;
  int cpp = pairs >= sms ? 1 : sms / pairs;
  const int blocks_q = (g.Q + items_per_block - 1) / items_per_block;
  if (cpp > blocks_q) cpp = blocks_q;
  return MsdaSlabGrid{cpp, pairs >= sms ? sms : pairs * cpp};
}

// msda_res.cu: the FP16 resident-tail kernel; cap_bytes is its shared memory for the tail. `g` has passed
// msda_check_dims. Returns B200_ERR_UNSUPPORTED for a shape or alignment outside its envelope.
int msda_res_f16(const void *value, const int32_t *shapes, const void *ref, const void *off, const void *logits,
                 void *out, int4 *trace, const MsdaGeom &g, int cap_bytes, cudaStream_t s);

}  // namespace b200

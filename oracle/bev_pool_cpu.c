/* oracle/bev_pool_cpu.c — TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
 *
 * Plain-C restatement of BEVPoolV2 (reference TensorRT/plugin/bev_pool_v2/bevPoolKernel.cu and the backward of
 * third_party/bev_mmdet3d/ops/bev_pool_v2/src/bev_pool_cuda.cu) with the index-safety rules of
 * include/b200_bev_ops.h: [s, s + len) clipped to [0, P), an interval whose cell ranks_bev[max(s, 0)] lies outside
 * [0, cells) dropped, a point whose ranks_depth / ranks_feat lies outside its tensor dropped.
 *   bev_pool_f64          float64 forward
 *   bev_pool_f32_fma      float32 forward as an explicit fmaf chain in point order (the reference kernel's FFMA chain)
 *   bev_pool_i8           INT8 forward: exact int32 sum, one float multiply by scale_io, saturate, round half away
 *   bev_pool_backward_f64 float64 depth / feature gradients
 *   bev_pool_backward_f32_lanes  float32 depth / feature gradients in the device kernels' lane partition and order
 * Built with -ffp-contract=off so every operation rounds where it is written. */
#include <math.h>
#include <stdint.h>
#include <string.h>

static int interval_of(const int32_t *rb, const int32_t *st, const int32_t *ln, int k, int P, long long cells,
                       long long *s, long long *e, long long *cell) {
  long long s0 = st[k], hi = s0 + (long long)ln[k];
  long long lo = s0 > 0 ? s0 : 0;
  if (hi > P) hi = P;
  if (lo >= hi) return 0;
  if (rb[lo] < 0 || rb[lo] >= cells) return 0;
  *s = lo, *e = hi, *cell = rb[lo];
  return 1;
}

static int kept(const int32_t *rd, const int32_t *rf, long long i, long long depth_size, long long feat_rows) {
  return rd[i] >= 0 && rd[i] < depth_size && rf[i] >= 0 && rf[i] < feat_rows;
}

void bev_pool_f64(const double *depth, const double *feat, const int32_t *rd, const int32_t *rf, const int32_t *rb,
                  const int32_t *st, const int32_t *ln, int C, int P, int I, long long depth_size,
                  long long feat_rows, long long cells, double *out) {
  memset(out, 0, sizeof(double) * (size_t)cells * C);
  for (int k = 0; k < I; ++k) {
    long long s, e, cell;
    if (!interval_of(rb, st, ln, k, P, cells, &s, &e, &cell)) continue;
    for (int c = 0; c < C; ++c) {
      double acc = 0.0;
      for (long long i = s; i < e; ++i)
        if (kept(rd, rf, i, depth_size, feat_rows)) acc += feat[(long long)rf[i] * C + c] * depth[rd[i]];
      out[cell * C + c] = acc;
    }
  }
}

void bev_pool_f32_fma(const float *depth, const float *feat, const int32_t *rd, const int32_t *rf, const int32_t *rb,
                      const int32_t *st, const int32_t *ln, int C, int P, int I, long long depth_size,
                      long long feat_rows, long long cells, float *out) {
  memset(out, 0, sizeof(float) * (size_t)cells * C);
  for (int k = 0; k < I; ++k) {
    long long s, e, cell;
    if (!interval_of(rb, st, ln, k, P, cells, &s, &e, &cell)) continue;
    for (int c = 0; c < C; ++c) {
      float acc = 0.0f;
      for (long long i = s; i < e; ++i)
        if (kept(rd, rf, i, depth_size, feat_rows)) acc = fmaf(feat[(long long)rf[i] * C + c], depth[rd[i]], acc);
      out[cell * C + c] = acc;
    }
  }
}

/* T2int8<float> of bevPoolKernel.cu: saturate to [-128, 127], add +-0.5 in float, truncate. */
static int8_t t2int8(float a) {
  a = a > 127.0f ? 127.0f : a;
  a = a < -128.0f ? -128.0f : a;
  return (int8_t)(a + (a > 0.0f ? 0.5f : -0.5f));
}

void bev_pool_i8(const int8_t *depth, const int8_t *feat, const int32_t *rd, const int32_t *rf, const int32_t *rb,
                 const int32_t *st, const int32_t *ln, int C, int P, int I, long long depth_size, long long feat_rows,
                 long long cells, float scale_d, float scale_f, float scale_o, int8_t *out) {
  const float scale_io = scale_d * scale_f / scale_o;
  memset(out, 0, (size_t)cells * C);
  for (int k = 0; k < I; ++k) {
    long long s, e, cell;
    if (!interval_of(rb, st, ln, k, P, cells, &s, &e, &cell)) continue;
    for (int c = 0; c < C; ++c) {
      uint32_t acc = 0; /* int32 arithmetic wraps as the device's does */
      for (long long i = s; i < e; ++i)
        if (kept(rd, rf, i, depth_size, feat_rows))
          acc += (uint32_t)((int32_t)feat[(long long)rf[i] * C + c] * (int32_t)depth[rd[i]]);
      out[cell * C + c] = t2int8((float)(int32_t)acc * scale_io);
    }
  }
}

void bev_pool_backward_f64(const double *out_grad, const double *depth, const double *feat, const int32_t *rd,
                           const int32_t *rf, const int32_t *rb, const int32_t *st, const int32_t *ln, int C, int P,
                           int I, long long depth_size, long long feat_rows, long long cells, double *depth_grad,
                           double *feat_grad) {
  memset(depth_grad, 0, sizeof(double) * (size_t)depth_size);
  memset(feat_grad, 0, sizeof(double) * (size_t)feat_rows * C);
  for (int k = 0; k < I; ++k) {
    long long s, e, cell;
    if (!interval_of(rb, st, ln, k, P, cells, &s, &e, &cell)) continue;
    const double *og = out_grad + cell * C;
    for (long long i = s; i < e; ++i) {
      if (!kept(rd, rf, i, depth_size, feat_rows)) continue;
      const double *f = feat + (long long)rf[i] * C;
      double *fg = feat_grad + (long long)rf[i] * C;
      double dot = 0.0;
      for (int c = 0; c < C; ++c) {
        dot += og[c] * f[c];
        fg[c] += og[c] * depth[rd[i]];
      }
      depth_grad[rd[i]] = dot;
    }
  }
}

/* float32 depth / feature gradients in the device kernels' exact order of operations, for a lane group of G lanes
 * (a power of two, <= 32) that each own VEC consecutive channels (VEC divides C):
 *   depth_grad[rd[i]]: lane l runs an fmaf chain over its channel chunks l, l + G, l + 2G, ... (VEC channels each,
 *     in channel order); then G/2, G/4, ..., 1: every lane adds (one rounding) the partial of lane l ^ o; lane 0's sum.
 *   feat_grad[f, c]: an fmaf chain over the pooled points with ranks_feat = f in point order (the stable sort).
 * point_cell[i] = the cell of the interval that pooled point i, -1 when none did (within the contract one interval
 * covers a point). Either output may be NULL. point_cell: scratch of P entries. */
void bev_pool_backward_f32_lanes(const float *out_grad, const float *depth, const float *feat, const int32_t *rd,
                                 const int32_t *rf, const int32_t *rb, const int32_t *st, const int32_t *ln, int C,
                                 int P, int I, long long depth_size, long long feat_rows, long long cells, int G,
                                 int VEC, float *depth_grad, float *feat_grad, long long *point_cell) {
  for (long long i = 0; i < P; ++i) point_cell[i] = -1;
  if (depth_grad) memset(depth_grad, 0, sizeof(float) * (size_t)depth_size);
  if (feat_grad) memset(feat_grad, 0, sizeof(float) * (size_t)feat_rows * C);
  for (int k = 0; k < I; ++k) {
    long long s, e, cell;
    if (!interval_of(rb, st, ln, k, P, cells, &s, &e, &cell)) continue;
    for (long long i = s; i < e; ++i) {
      if (!kept(rd, rf, i, depth_size, feat_rows)) continue;
      point_cell[i] = cell;
      if (!depth_grad) continue;
      const float *og = out_grad + cell * C, *f = feat + (long long)rf[i] * C;
      float part[32];
      for (int l = 0; l < G; ++l) {
        part[l] = 0.0f;
        for (long long c0 = (long long)l * VEC; c0 < C; c0 += (long long)G * VEC)
          for (int v = 0; v < VEC; ++v) part[l] = fmaf(og[c0 + v], f[c0 + v], part[l]);
      }
      for (int o = G / 2; o > 0; o >>= 1) {
        float next[32];
        for (int l = 0; l < G; ++l) next[l] = part[l] + part[l ^ o];
        memcpy(part, next, sizeof(float) * (size_t)G);
      }
      depth_grad[rd[i]] = part[0];
    }
  }
  if (!feat_grad) return;
  for (long long i = 0; i < P; ++i) {
    if (point_cell[i] < 0) continue;
    const float *og = out_grad + point_cell[i] * C, d = depth[rd[i]];
    float *fg = feat_grad + (long long)rf[i] * C;
    for (int c = 0; c < C; ++c) fg[c] = fmaf(og[c], d, fg[c]);
  }
}

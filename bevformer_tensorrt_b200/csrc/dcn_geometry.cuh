// dcn_geometry.cuh — the geometry of one DCNv2 layer, as the dcn*.cu host code passes it around: every C-ABI entry
// builds it once from its scalar arguments (dcn_geom) and hands it on by reference.
#pragma once
#include "common.cuh"

namespace b200 {

struct DcnGeom {
  int B, C, H, W, Co, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, groups, dg;
  int Ho, Wo;  // 0 when a stride is not positive
};

// Where the last window starts, counted from the first: negative when the dilated kernel does not fit the padded input.
template <typename I>
inline I dcn_extent_numerator(I in, I k, I pad, I dil) {
  return in + 2 * pad - (dil * (k - 1) + 1);
}
// Output extent of one axis with C's truncating division, as the launchers compute it (a numerator in (-stride, 0)
// still gives 1).
template <typename I>
inline I dcn_out_extent(I in, I k, I stride, I pad, I dil) {
  return dcn_extent_numerator(in, k, pad, dil) / stride + 1;
}

// Arguments in the C ABI's order (every *_w before its *_h).
inline DcnGeom dcn_geom(int batch, int channels, int height, int width, int channels_out, int kernel_w, int kernel_h,
                        int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w, int dilation_h, int group,
                        int deformable_group) {
  DcnGeom g{batch,  channels, height,     width,      channels_out, kernel_h, kernel_w, stride_h, stride_w,
            pad_h,  pad_w,    dilation_h, dilation_w, group,        deformable_group, 0, 0};
  if (stride_h > 0 && stride_w > 0) {
    g.Ho = dcn_out_extent(height, kernel_h, stride_h, pad_h, dilation_h);
    g.Wo = dcn_out_extent(width, kernel_w, stride_w, pad_w, dilation_w);
  }
  return g;
}

// Every extent, kernel size, stride and dilation is positive. Padding may be negative here; the group counts are
// checked by dcn_positive, or by the caller where a launcher rejects them later than the other dimensions.
inline bool dcn_extents_positive(const DcnGeom &g) {
  return g.B > 0 && g.C > 0 && g.H > 0 && g.W > 0 && g.Co > 0 && g.kh > 0 && g.kw > 0 && g.stride_h > 0 &&
         g.stride_w > 0 && g.dil_h > 0 && g.dil_w > 0;
}
inline bool dcn_positive(const DcnGeom &g) { return dcn_extents_positive(g) && g.groups > 0 && g.dg > 0; }

// The groups split the input and output channels, the deformable groups the input channels.
inline bool dcn_groups_divide(const DcnGeom &g) { return g.C % g.groups == 0 && g.Co % g.groups == 0 && g.C % g.dg == 0; }

// The layer fields of a kernel's parameter struct (DcnGParams, DcnFusedParams, DcnBwParams); the group counts, which
// DcnFusedParams does not have, are set by the launchers that use them.
template <typename P>
inline void dcn_set_layer(P &p, const DcnGeom &g) {
  p.B = g.B, p.C = g.C, p.H = g.H, p.W = g.W, p.Co = g.Co, p.kh = g.kh, p.kw = g.kw;
  p.pad_h = g.pad_h, p.pad_w = g.pad_w, p.stride_h = g.stride_h, p.stride_w = g.stride_w, p.dil_h = g.dil_h,
  p.dil_w = g.dil_w, p.Ho = g.Ho, p.Wo = g.Wo;
}

inline unsigned grid_for(long long n) { return static_cast<unsigned>(n / 256 + 1 < (1 << 20) ? n / 256 + 1 : (1 << 20)); }

// dcn_fused.cu
bool dcn_fused_supported(const DcnGeom &g);
size_t dcn_fused_workspace_bytes(const DcnGeom &g);
int dcn_fused_f16(const __half *input, const __half *weight, const __half *bias, const __half *offset,
                  const __half *mask, __half *output, void *workspace, const DcnGeom &g, int flags, cudaStream_t stream);
int dcn_fused_i8(const int8_t *input, float scale_i, const int8_t *weight, float scale_w, const void *bias, int bias_is_half,
                 const int8_t *offset, float scale_off, const int8_t *mask, float scale_mask, int8_t *output, float scale_o,
                 void *workspace, const DcnGeom &g, cudaStream_t stream);
int dcn_pack_weights_f16(const __half *weight, __half *packed, const DcnGeom &g, cudaStream_t stream);

// dcn_generic.cu
template <typename T>
int dcn_generic_launch(const T *input, const T *weight, const T *bias, const T *offset, const T *mask, T *output,
                       const DcnGeom &g, cudaStream_t stream);

}  // namespace b200

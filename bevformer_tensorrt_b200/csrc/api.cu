// api.cu — library-level C ABI: identification, status strings, launch counter, and the plugin-shaped
// enqueue / supportsFormatCombination mirrors of every plugin (reference: the …Plugin.cpp files named below).
#include "common.cuh"
#include "dcn_geometry.cuh"
#include "msda_geometry.cuh"

namespace b200 {
std::atomic<unsigned long long> g_launch_count{0};

// Shape unpacking of the reference's MSDA plugin (…Plugin.cpp:75-88): batch / spatial / heads / channels from value's
// dims, L = `levels` (shapes.d[0]), G from ref.d[3] / 2, Q from offsets.d[1], P from weights.d[3] / L.
static MsdaGeom msda_desc_geom(const b200_tensor_desc *in, int levels) {
  const int32_t *v = in[0].dims.d;
  return msda_geom(v[0], v[1], v[2], v[3], levels, in[3].dims.d[1], in[4].dims.d[3] / levels, in[2].dims.d[3] / 2);
}

// The image input of the grid sampler, rotate and DCN plugins: fp32 linear, fp16 linear (kCHW2 for the …TRT2 flavour)
// or int8 kCHW4 (gridSamplerPlugin.cpp:171-186, rotatePlugin.cpp:122-153, …Conv2dPlugin.cpp:213-250).
static bool image_format_ok(const b200_tensor_desc &d, int use_h2) {
  if (d.type == 2) return d.format == 3;
  if (d.type == 1) return d.format == (use_h2 ? 1 : 0);
  return d.type == 0 && d.format == 0;
}

static long long desc_numel(const b200_dims &d) {
  if (d.nbDims < 0 || d.nbDims > 8) return -1;
  long long n = 1;
  for (int i = 0; i < d.nbDims; ++i) {
    if (d.d[i] < 0) return -1;
    n *= d.d[i];
  }
  return n;
}
}  // namespace b200

using namespace b200;

extern "C" {

const char *b200_bev_ops_version(void) { return "b200_bev_ops 0.1.2 sm_90a"; }

const char *b200_status_string(int status) {
  switch (status) {
    case B200_OK: return "ok";
    case B200_ERR_UNSUPPORTED: return "unsupported dtype/format/shape";
    case B200_ERR_BAD_PARAM: return "bad parameter";
    case B200_ERR_LAUNCH: return "CUDA launch error";
    default: return "unknown status";
  }
}

unsigned long long b200_launch_count(void) { return g_launch_count.load(std::memory_order_relaxed); }

// IPluginV2DynamicExt::enqueue of the reference, argument for argument (…Plugin.cpp:71-140), with msda_desc_geom's
// shapes and the scales of the tensor descriptors.
int b200_msda_enqueue(const b200_tensor_desc *in, const b200_tensor_desc *out, const void *const *inputs,
                      void *const *outputs, void *workspace, void *stream, int use_h2) {
  // The reference asks for 0 workspace bytes (…Plugin.cpp:64-69). A host that lends b200_msda_enqueue_workspace_size()
  // bytes gets the second-generation INT8 kernels (msda_v2.cu); workspace == NULL keeps the round-1 kernels.
  if (!in || !out || !inputs || !outputs) return B200_ERR_BAD_PARAM;
  if (in[1].dims.d[0] <= 0) return B200_ERR_BAD_PARAM;
  const MsdaGeom g = msda_desc_geom(in, in[1].dims.d[0]);
  const int32_t *shapes = static_cast<const int32_t *>(inputs[1]);
  switch (in[0].type) {
    case 0:  // kFLOAT
      return b200_msda_f32(static_cast<const float *>(inputs[0]), shapes, static_cast<const float *>(inputs[2]),
                           static_cast<const float *>(inputs[3]), static_cast<const float *>(inputs[4]), g.B, g.S, g.M,
                           g.C, g.L, g.Q, g.P, g.G, static_cast<float *>(outputs[0]), stream);
    case 1:  // kHALF
      if (use_h2 && g.C % 2 == 0)
        return b200_msda_f16_h2(inputs[0], shapes, inputs[2], inputs[3], inputs[4], g.B, g.S, g.M, g.C, g.L, g.Q, g.P,
                                g.G, outputs[0], stream);
      return b200_msda_f16(inputs[0], shapes, inputs[2], inputs[3], inputs[4], g.B, g.S, g.M, g.C, g.L, g.Q, g.P, g.G,
                           outputs[0], stream);
    case 2: {  // kINT8; reference points stay fp16 or fp32 (…Plugin.cpp:168-176)
      if (in[2].type != 0 && in[2].type != 1) return B200_ERR_UNSUPPORTED;
      const size_t ws = workspace ? b200_msda_i8_workspace_size(g.B, g.S, g.M, g.C, g.L, g.P, g.G) : 0;
      if (ws) {
        const int st = b200_msda_i8_ws(static_cast<const int8_t *>(inputs[0]), in[0].scale, shapes, inputs[2],
                                       in[2].type == 1, static_cast<const int8_t *>(inputs[3]), in[3].scale,
                                       static_cast<const int8_t *>(inputs[4]), in[4].scale, g.B, g.S, g.M, g.C, g.L,
                                       g.Q, g.P, g.G, static_cast<int8_t *>(outputs[0]), out[0].scale, workspace, ws,
                                       nullptr, stream);
        if (st != B200_ERR_UNSUPPORTED) return st;
      }
      return b200_msda_i8(static_cast<const int8_t *>(inputs[0]), in[0].scale, shapes, inputs[2], in[2].type == 1,
                          static_cast<const int8_t *>(inputs[3]), in[3].scale, static_cast<const int8_t *>(inputs[4]),
                          in[4].scale, g.B, g.S, g.M, g.C, g.L, g.Q, g.P, g.G, static_cast<int8_t *>(outputs[0]),
                          out[0].scale, stream);
    }
    default:
      return B200_ERR_UNSUPPORTED;
  }
}

// getWorkspaceSize mirror for the MSDA plugin shell: dimensions only, like the TensorRT call.
size_t b200_msda_enqueue_workspace_size(const b200_tensor_desc *in) {
  if (!in) return 0;
  if (in[1].dims.d[0] <= 0) return 0;
  if (in[0].type != 2) return 0;  // kINT8 only
  const MsdaGeom g = msda_desc_geom(in, in[1].dims.d[0]);
  return b200_msda_i8_workspace_size(g.B, g.S, g.M, g.C, g.L, g.P, g.G);
}

int b200_msda_supports_format(int pos, const b200_tensor_desc *io, int nb_inputs, int nb_outputs) {
  if (!io || nb_inputs != 5 || nb_outputs != 1) return 0;
  const MsdaGeom g = msda_desc_geom(io, io[1].dims.d[0] > 0 ? io[1].dims.d[0] : 1);
  const bool int8_ok = (g.C % 4 == 0) && (g.P % 4 == 0);
  const bool linear = io[pos].format == 0;
  switch (pos) {
    case 0: return linear && (io[0].type == 0 || io[0].type == 1 || (io[0].type == 2 && int8_ok));
    case 1: return linear && io[1].type == 3;
    case 2:
      if (io[0].type == 0 || io[0].type == 1) return linear && io[2].type == io[0].type;
      return linear && (io[2].type == 0 || io[2].type == 1);
    case 3:
    case 4: return linear && io[pos].type == io[0].type;
    case 5: return io[5].type == io[0].type && io[5].format == io[0].format;
    default: return 0;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// GridSampler{2D,3D}TRT[2]: IPluginV2DynamicExt::enqueue / supportsFormatCombination of the reference, argument for
// argument (gridSamplerPlugin.cpp:110-155, :168-194). inputs: input, grid; attributes: interpolation_mode, padding_mode,
// align_corners (:277-288). Dispatch: fp32 / fp16 linear, fp16 kCHW2 (…TRT2), int8 kCHW4 with the descriptors' scales.
int b200_grid_sampler_enqueue(const b200_tensor_desc *in, const b200_tensor_desc *out, const void *const *inputs,
                              void *const *outputs, void *workspace, void *stream, int interpolation_mode,
                              int padding_mode, int align_corners) {
  (void)workspace;  // 0 bytes (gridSamplerPlugin.cpp:102-108)
  if (!in || !out || !inputs || !outputs) return B200_ERR_BAD_PARAM;
  const int nb = in[0].dims.nbDims;
  if ((nb != 4 && nb != 5) || in[1].dims.nbDims != nb || out[0].dims.nbDims != nb) return B200_ERR_BAD_PARAM;
  const int *id = in[0].dims.d, *gd = in[1].dims.d, *od = out[0].dims.d;
  if (in[0].type == 0)
    return b200_grid_sample_f32(static_cast<float *>(outputs[0]), static_cast<const float *>(inputs[0]),
                                static_cast<const float *>(inputs[1]), od, id, gd, nb, interpolation_mode, padding_mode,
                                align_corners, stream);
  if (in[0].type == 1)
    return (in[0].format == 1 /* kCHW2 */ ? b200_grid_sample_f16_chw2 : b200_grid_sample_f16)(
        outputs[0], inputs[0], inputs[1], od, id, gd, nb, interpolation_mode, padding_mode, align_corners, stream);
  if (in[0].type == 2)
    return b200_grid_sample_i8_chw4(static_cast<int8_t *>(outputs[0]), out[0].scale, static_cast<const int8_t *>(inputs[0]),
                                    in[0].scale, static_cast<const int8_t *>(inputs[1]), in[1].scale, od, id, gd, nb,
                                    interpolation_mode, padding_mode, align_corners, stream);
  return B200_ERR_UNSUPPORTED;
}

// io[0] input, io[1] grid, io[2] output. use_h2 = the …TRT2 flavour (FP16 as kCHW2 packets).
int b200_grid_sampler_supports_format(int pos, const b200_tensor_desc *io, int nb_inputs, int nb_outputs, int use_h2) {
  if (!io || nb_inputs != 2 || nb_outputs != 1 || pos < 0 || pos > 2) return 0;
  const b200_tensor_desc &d = io[pos], &x = io[0];
  if (pos != 0) return d.type == x.type && d.format == x.format;
  if (x.dims.nbDims == 5) return (d.type == 0 || d.type == 1) && d.format == 0;  // 5-D: fp32 / fp16 linear (:187-189)
  return image_format_ok(d, use_h2);
}

// ------------------------------------------------------------------------------------------------------------------
// RotateTRT[2]: enqueue / supportsFormatCombination of the reference (rotatePlugin.cpp:75-113, :122-153). inputs: img
// [C, H, W], angle [1], center [2]; attribute interpolation. Dispatch: fp32, fp16 linear (kCHW2 for …TRT2), int8 kCHW4
// with the descriptors' scales and angle / center in the type of the angle descriptor.
int b200_rotate_enqueue(const b200_tensor_desc *in, const b200_tensor_desc *out, const void *const *inputs,
                        void *const *outputs, void *workspace, void *stream, int interp, int use_h2) {
  if (!in || !out || !inputs || !outputs) return B200_ERR_BAD_PARAM;
  // the kernels read angle[0], center[0..1] and write an image of the input's extent
  const b200_dims &img = in[0].dims, &o = out[0].dims;
  if (img.nbDims != 3 || o.nbDims != 3 || o.d[0] != img.d[0] || o.d[1] != img.d[1] || o.d[2] != img.d[2])
    return B200_ERR_BAD_PARAM;
  if (desc_numel(in[1].dims) != 1 || desc_numel(in[2].dims) != 2) return B200_ERR_BAD_PARAM;
  if (in[0].type == 0)
    return b200_rotate_f32(static_cast<float *>(outputs[0]), static_cast<const float *>(inputs[0]),
                           static_cast<const float *>(inputs[1]), static_cast<const float *>(inputs[2]), img.d, interp, stream);
  if (in[0].type == 1)
    return (use_h2 ? b200_rotate_f16_h2 : b200_rotate_f16)(outputs[0], inputs[0], inputs[1], inputs[2], img.d, interp, stream);
  if (in[0].type == 2)
    return b200_rotate_i8(static_cast<int8_t *>(outputs[0]), out[0].scale, static_cast<const int8_t *>(inputs[0]),
                          in[0].scale, inputs[1], inputs[2], in[1].type == 1, img.d, interp, stream);
  return B200_ERR_UNSUPPORTED;
}

// io[0] img, io[1] angle, io[2] center, io[3] output. angle and center are linear in the image's type, or fp32 / fp16
// of one type for an int8 image.
int b200_rotate_supports_format(int pos, const b200_tensor_desc *io, int nb_inputs, int nb_outputs, int use_h2) {
  if (!io || nb_inputs != 3 || nb_outputs != 1 || pos < 0 || pos > 3) return 0;
  const b200_tensor_desc &d = io[pos], &img = io[0];
  if (pos == 0) return image_format_ok(d, use_h2);
  if (pos == 3) return d.type == img.type && d.format == img.format;
  if (d.format != 0) return 0;
  if (img.type == 2) return (d.type == 0 || d.type == 1) && d.type == io[1].type;
  return d.type == img.type;
}

// ------------------------------------------------------------------------------------------------------------------
// ModulatedDeformableConv2dTRT[2]: enqueue of the reference (…Conv2dPlugin.cpp:117-199). inputs: x, offset, mask,
// weight[, bias]. stride / padding / dilation are the plugin attributes' int[2] in ONNX order (h, w), as the exporter
// writes them (stride_i=_pair(stride), functions/modulated_deformable_conv2d.py): element [0] goes to the launcher's
// *_h slot and [1] to *_w. (The reference's call hands [0] to *_w, which disagrees with its own getOutputDimensions for
// asymmetric layers.) workspace: b200_dcn_enqueue_workspace_size.
size_t b200_dcn_enqueue_workspace_size(const b200_tensor_desc *in, const int32_t *stride, const int32_t *padding,
                                       const int32_t *dilation, int groups, int deform_groups) {
  if (!in || !stride || !padding || !dilation) return 0;
  const int32_t *x = in[0].dims.d, *w = in[3].dims.d;
  if (in[0].type == 2)
    return b200_dcn_i8_workspace_size(x[0], x[1], x[2], x[3], w[0], w[3], w[2], stride[1], stride[0], padding[1], padding[0],
                                      dilation[1], dilation[0], groups, deform_groups);
  if (in[0].type == 1 && in[0].format == 1)
    return b200_dcn_f16_chw2_workspace_size(x[0], x[1], x[2], x[3], w[0], w[3], w[2], stride[1], stride[0], padding[1],
                                            padding[0], dilation[1], dilation[0], groups, deform_groups);
  return b200_dcn_workspace_size(in[0].type == 1, x[0], x[1], x[2], x[3], w[3], w[2], stride[1], stride[0], padding[1],
                                 padding[0], dilation[1], dilation[0]);
}

// …TRT: fp32 / fp16 linear everywhere. …TRT2 (use_h2): FP16 input, offset and weight as kCHW2 packets, mask / bias /
// output linear. INT8 (both, when C and Co / groups are multiples of 4): input and weight kCHW4, offset / mask / output
// int8 linear, bias fp32 or fp16 linear.
int b200_dcn_supports_format(int pos, const b200_tensor_desc *io, int nb_inputs, int nb_outputs, int groups, int use_h2) {
  if (!io || (nb_inputs != 4 && nb_inputs != 5) || nb_outputs != 1 || pos < 0 || pos > nb_inputs) return 0;
  const b200_tensor_desc &d = io[pos], &x = io[0];
  const bool int8_ok = groups > 0 && x.dims.d[1] % 4 == 0 && (io[nb_inputs].dims.d[1] / groups) % 4 == 0;
  if (pos == 0) return image_format_ok(d, use_h2) && (d.type != 2 || int8_ok);
  const bool bias = nb_inputs == 5 && pos == 4;
  if (x.type == 2) {
    if (bias) return (d.type == 0 || d.type == 1) && d.format == 0;
    return d.type == 2 && d.format == (pos == 3 ? 3 : 0);  // weight kCHW4; offset, mask, output linear
  }
  if (bias || pos == nb_inputs || pos == 2) return d.type == x.type && d.format == 0;
  return d.type == x.type && d.format == x.format;  // offset, weight follow the input's format (…Conv2dPlugin.cpp:246-249)
}

static bool dims_are(const b200_dims &d, long long d0, long long d1, long long d2, long long d3) {
  return d.nbDims == 4 && d.d[0] == d0 && d.d[1] == d1 && d.d[2] == d2 && d.d[3] == d3;
}

// The descriptors TensorRT passes must describe the layer the attributes define: TensorRT sizes the output from the
// offset tensor, the launcher from the attributes, and a disagreement would read or write outside a tensor.
static bool dcn_geometry_ok(const b200_tensor_desc *in, const b200_tensor_desc *out, int nb_inputs, int sh, int sw, int ph,
                            int pw, int dh, int dw, int groups, int deform_groups) {
  const b200_dims &x = in[0].dims, &w = in[3].dims;
  if (x.nbDims != 4 || w.nbDims != 4 || groups <= 0 || deform_groups <= 0) return false;
  const long long n = x.d[0], c = x.d[1], h = x.d[2], wd = x.d[3], co = w.d[0], kh = w.d[2], kw = w.d[3], taps = kh * kw;
  if (n <= 0 || h <= 0 || wd <= 0 || kh <= 0 || kw <= 0 || sh <= 0 || sw <= 0 || dh <= 0 || dw <= 0) return false;
  // Beyond the launchers' rule: TensorRT floors the output extent, so the dilated kernel must fit the padded input (a
  // numerator in (-stride, 0) truncates to a 1-pixel output), and padding is never negative.
  if (ph < 0 || pw < 0 || dcn_extent_numerator<long long>(h, kh, ph, dh) < 0 ||
      dcn_extent_numerator<long long>(wd, kw, pw, dw) < 0)
    return false;
  const long long ho = dcn_out_extent<long long>(h, kh, sh, ph, dh), wo = dcn_out_extent<long long>(wd, kw, sw, pw, dw);
  if (static_cast<long long>(w.d[1]) * groups != c) return false;
  if (nb_inputs == 5 && !(in[4].dims.nbDims == 1 && in[4].dims.d[0] == co)) return false;
  return dims_are(in[1].dims, n, deform_groups * 2 * taps, ho, wo) && dims_are(in[2].dims, n, deform_groups * taps, ho, wo) &&
         dims_are(out[0].dims, n, co, ho, wo);
}

int b200_dcn_enqueue(const b200_tensor_desc *in, const b200_tensor_desc *out, const void *const *inputs,
                     void *const *outputs, void *workspace, void *stream, int nb_inputs, const int32_t *stride,
                     const int32_t *padding, const int32_t *dilation, int groups, int deform_groups) {
  if (!in || !out || !inputs || !outputs || !stride || !padding || !dilation) return B200_ERR_BAD_PARAM;
  if (nb_inputs != 4 && nb_inputs != 5) return B200_ERR_BAD_PARAM;
  // the geometry that is checked is the geometry that is launched (launcher order: *_w before *_h)
  const int sh = stride[0], sw = stride[1], ph = padding[0], pw = padding[1], dh = dilation[0], dw = dilation[1];
  if (!dcn_geometry_ok(in, out, nb_inputs, sh, sw, ph, pw, dh, dw, groups, deform_groups)) return B200_ERR_BAD_PARAM;
  const int32_t *x = in[0].dims.d, *w = in[3].dims.d;
  const void *bias = nb_inputs == 5 ? inputs[4] : nullptr;
  switch (in[0].type) {
    case 0:
      return b200_dcn_f32(static_cast<const float *>(inputs[0]), static_cast<const float *>(inputs[3]),
                          static_cast<const float *>(bias), static_cast<const float *>(inputs[1]),
                          static_cast<const float *>(inputs[2]), static_cast<float *>(outputs[0]), workspace, x[0], x[1],
                          x[2], x[3], w[0], w[3], w[2], sw, sh, pw, ph, dw, dh, groups, deform_groups, x[0], nullptr, stream);
    case 1:
      if (in[0].format == 1)
        return b200_dcn_f16_chw2(inputs[0], inputs[3], bias, inputs[1], inputs[2], outputs[0], workspace, x[0], x[1], x[2],
                                 x[3], w[0], w[3], w[2], sw, sh, pw, ph, dw, dh, groups, deform_groups, x[0], nullptr, stream);
      return b200_dcn_f16(inputs[0], inputs[3], bias, inputs[1], inputs[2], outputs[0], workspace, x[0], x[1], x[2], x[3],
                          w[0], w[3], w[2], sw, sh, pw, ph, dw, dh, groups, deform_groups, x[0], nullptr, stream);
    case 2:
      return b200_dcn_i8(static_cast<const int8_t *>(inputs[0]), in[0].scale, static_cast<const int8_t *>(inputs[3]),
                         in[3].scale, bias, nb_inputs == 5 && in[4].type == 1, static_cast<const int8_t *>(inputs[1]),
                         in[1].scale, static_cast<const int8_t *>(inputs[2]), in[2].scale,
                         static_cast<int8_t *>(outputs[0]), out[0].scale, workspace, x[0], x[1], x[2], x[3], w[0], w[3],
                         w[2], sw, sh, pw, ph, dw, dh, groups, deform_groups, x[0], nullptr, stream);
    default:
      return B200_ERR_UNSUPPORTED;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// BEVPoolV2TRT[2]: enqueue / supportsFormatCombination of the reference (bevPoolPlugin.cpp:71-117, :128-143). The
// reference takes C from feat.d[3], the interval count from interval_starts.d[0] and the output size from the output
// descriptor, and checks nothing; here every extent the index checks use comes from the descriptors and must agree.
int b200_bev_pool_enqueue(const b200_tensor_desc *in, const b200_tensor_desc *out, const void *const *inputs,
                          void *const *outputs, void *workspace, void *stream, int out_height, int out_width) {
  (void)workspace;
  if (!in || !out || !inputs || !outputs) return B200_ERR_BAD_PARAM;
  const b200_dims &fd = in[1].dims;
  if (fd.nbDims < 1 || fd.nbDims > 8) return B200_ERR_BAD_PARAM;
  const int C = fd.d[fd.nbDims - 1];
  const long long depth_size = desc_numel(in[0].dims), feat_size = desc_numel(fd);
  if (C <= 0 || depth_size < 0 || feat_size < 0) return B200_ERR_BAD_PARAM;
  for (int i = 2; i < 7; ++i)
    if (in[i].dims.nbDims != 1) return B200_ERR_BAD_PARAM;
  const int P = in[2].dims.d[0], I = in[5].dims.d[0];
  if (in[3].dims.d[0] != P || in[4].dims.d[0] != P || in[6].dims.d[0] != I) return B200_ERR_BAD_PARAM;
  if (!dims_are(out[0].dims, 1, out_height, out_width, C)) return B200_ERR_BAD_PARAM;
  const int32_t *idx[5];
  for (int i = 0; i < 5; ++i) idx[i] = static_cast<const int32_t *>(inputs[2 + i]);
  const long long rows = feat_size / C;
  switch (in[0].type) {
    case 0:
      return b200_bev_pool_f32(static_cast<const float *>(inputs[0]), static_cast<const float *>(inputs[1]), idx[0],
                               idx[1], idx[2], idx[3], idx[4], C, P, I, depth_size, rows, out_height, out_width,
                               static_cast<float *>(outputs[0]), stream);
    case 1:
      return b200_bev_pool_f16(inputs[0], inputs[1], idx[0], idx[1], idx[2], idx[3], idx[4], C, P, I, depth_size, rows,
                               out_height, out_width, outputs[0], stream);
    case 2:
      return b200_bev_pool_i8(static_cast<const int8_t *>(inputs[0]), in[0].scale,
                              static_cast<const int8_t *>(inputs[1]), in[1].scale, idx[0], idx[1], idx[2], idx[3],
                              idx[4], C, P, I, depth_size, rows, out_height, out_width,
                              static_cast<int8_t *>(outputs[0]), out[0].scale, stream);
    default:
      return B200_ERR_UNSUPPORTED;
  }
}

int b200_bev_pool_supports_format(int pos, const b200_tensor_desc *io, int nb_inputs, int nb_outputs) {
  if (!io || nb_inputs != 7 || nb_outputs != 1 || pos < 0 || pos > 7) return 0;
  const b200_tensor_desc &d = io[pos];
  if (d.format != 0) return 0;
  if (pos == 0) {
    const b200_dims &fd = io[1].dims;
    const bool int8_ok = fd.nbDims >= 1 && fd.nbDims <= 8 && fd.d[fd.nbDims - 1] > 0 && fd.d[fd.nbDims - 1] % 4 == 0;
    return d.type == 0 || d.type == 1 || (d.type == 2 && int8_ok);
  }
  if (pos == 1 || pos == 7) return d.type == io[0].type;
  return d.type == 3;
}

}  // extern "C"

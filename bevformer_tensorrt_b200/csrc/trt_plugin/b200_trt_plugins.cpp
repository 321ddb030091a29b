// b200_trt_plugins.cpp — TensorRT plugin shells over libb200_bev_ops (compiled only where TensorRT's NvInfer.h exists;
// this image has no TensorRT, so the build in bevformer_tensorrt_b200/build.py skips it and tests/test_host_logic.py
// compiles it against tests/mock_trt/NvInfer.h, a declaration-only stand-in, to keep it honest;
// tests/test_trt_plugins_gpu.py runs it the same way on device data).
//
// Same plugin names / versions / input orders / attributes as the reference, so an ONNX graph exported by the
// reference's symbolic() functions resolves to these plugins unchanged:
//   MultiScaleDeformableAttnTRT, MultiScaleDeformableAttnTRT2   (multiScaleDeformableAttnPlugin.cpp:19-23, :345-346)
//   GridSampler2DTRT, GridSampler2DTRT2, GridSampler3DTRT, GridSampler3DTRT2   (gridSamplerPlugin.cpp:20-26, :558-561)
//   ModulatedDeformableConv2dTRT, ModulatedDeformableConv2dTRT2   (modulatedDeformableConv2dPlugin.cpp:19-23, :515-516)
//   RotateTRT, RotateTRT2                                         (rotatePlugin.cpp:19-21, :216-330)
//   BEVPoolV2TRT, BEVPoolV2TRT2                                   (bevPoolPlugin.cpp:17-21, :225-383)
// enqueue() forwards to the C ABI (include/b200_bev_ops.h); nothing is computed here.
#if __has_include(<NvInfer.h>)
#include <NvInfer.h>

#include <cstring>
#include <string>
#include <vector>

#include "b200_bev_ops.h"

namespace b200_trt {
using namespace nvinfer1;

static_assert(sizeof(b200_tensor_desc) == sizeof(PluginTensorDesc), "b200_tensor_desc must mirror PluginTensorDesc");

enum class Op { kMSDA, kGridSampler2D, kGridSampler3D, kDCN, kRotate, kBEVPool };

struct Attrs {  // serialised verbatim (the reference serialises the same fields: gridSamplerPlugin.cpp:157-166,
                // modulatedDeformableConv2dPlugin.cpp:200-211; MSDA serialises nothing, …Plugin.cpp:142-146)
  int32_t interp = 0, padding = 0, align = 0;                           // grid sampler; rotate uses interp only
  int32_t stride[2] = {1, 1}, pad[2] = {0, 0}, dil[2] = {1, 1}, groups = 1, deform_groups = 1;  // DCN
};

// BEVPool's attributes live outside Attrs, so the serialisation of every other plugin keeps its size; BEVPool serialises
// them as the reference does (bevPoolPlugin.cpp:112-119): int32 out_width, then int32 out_height.
struct BevAttrs {
  int32_t out_height = 128, out_width = 128;
};

// A constant dimension expression. The declaration-only mock of the TensorRT API has no IExprBuilder definition; there
// the overload below, which yields no expression, is chosen, and the shell still compiles.
template <class B>
auto dim_constant(B &b, int32_t v, int) -> decltype(b.constant(v)) {
  return b.constant(v);
}
template <class B>
const IDimensionExpr *dim_constant(B &, int32_t, long) {
  return nullptr;
}

class Plugin final : public IPluginV2DynamicExt {
 public:
  Plugin(Op op, bool v2, const Attrs &a, const BevAttrs &bev = BevAttrs{}) : op_(op), v2_(v2), a_(a), bev_(bev) {}

  // ---- IPluginV2DynamicExt
  IPluginV2DynamicExt *clone() const noexcept override {
    auto *p = new (std::nothrow) Plugin(op_, v2_, a_, bev_);
    if (p) p->setPluginNamespace(ns_.c_str());
    return p;
  }
  DimsExprs getOutputDimensions(int32_t, const DimsExprs *in, int32_t nb, IExprBuilder &b) noexcept override {
    DimsExprs o{};
    o.nbDims = 4;
    if (op_ == Op::kBEVPool) {  // [1, out_height, out_width, feat.d3] (bevPoolPlugin.cpp:41-52)
      o.d[0] = dim_constant(b, 1, 0), o.d[1] = dim_constant(b, bev_.out_height, 0);
      o.d[2] = dim_constant(b, bev_.out_width, 0), o.d[3] = in[1].d[3];
    } else if (op_ == Op::kRotate) {  // output = img dims [C, H, W] (rotatePlugin.cpp:52-62)
      o.nbDims = 3;
      o.d[0] = in[0].d[0], o.d[1] = in[0].d[1], o.d[2] = in[0].d[2];
    } else if (op_ == Op::kMSDA) {  // [value.d0, offsets.d1, value.d2, value.d3] (…Plugin.cpp:48-58)
      o.d[0] = in[0].d[0], o.d[1] = in[3].d[1], o.d[2] = in[0].d[2], o.d[3] = in[0].d[3];
    } else if (op_ == Op::kGridSampler2D) {  // [in.d0, in.d1, grid.d2, grid.d3] (gridSamplerPlugin.cpp:85-96)
      o.d[0] = in[0].d[0], o.d[1] = in[0].d[1], o.d[2] = in[1].d[2], o.d[3] = in[1].d[3];
    } else if (op_ == Op::kGridSampler3D) {  // [in.d0, in.d1, grid.d2, grid.d3, grid.d4]
      o.nbDims = 5;
      o.d[0] = in[0].d[0], o.d[1] = in[0].d[1], o.d[2] = in[1].d[2], o.d[3] = in[1].d[3], o.d[4] = in[1].d[4];
    } else {  // [in.d0, weight.d0, offset.d2, offset.d3] (…Conv2dPlugin.cpp:60-66)
      o.d[0] = in[0].d[0], o.d[1] = in[3].d[0], o.d[2] = in[1].d[2], o.d[3] = in[1].d[3];
    }
    (void)nb;
    return o;
  }
  bool supportsFormatCombination(int32_t pos, const PluginTensorDesc *io, int32_t nbIn, int32_t nbOut) noexcept override {
    const auto *d = reinterpret_cast<const b200_tensor_desc *>(io);
    switch (op_) {
      case Op::kMSDA: return b200_msda_supports_format(pos, d, nbIn, nbOut) != 0;
      case Op::kBEVPool: return b200_bev_pool_supports_format(pos, d, nbIn, nbOut) != 0;
      case Op::kRotate: return b200_rotate_supports_format(pos, d, nbIn, nbOut, v2_) != 0;
      case Op::kDCN: return b200_dcn_supports_format(pos, d, nbIn, nbOut, a_.groups, v2_) != 0;
      default: return b200_grid_sampler_supports_format(pos, d, nbIn, nbOut, v2_) != 0;
    }
  }
  void configurePlugin(const DynamicPluginTensorDesc *, int32_t nbIn, const DynamicPluginTensorDesc *, int32_t) noexcept override {
    nb_inputs_ = nbIn;  // DCN: 4 inputs without bias, 5 with (…Conv2dPlugin.cpp:297-299)
  }
  size_t getWorkspaceSize(const PluginTensorDesc *in, int32_t, const PluginTensorDesc *, int32_t) const noexcept override {
    if (op_ == Op::kMSDA)  // the reference asks for 0 (…Plugin.cpp:64-69); the v2 kernels want room for the packed value stack
      return b200_msda_enqueue_workspace_size(reinterpret_cast<const b200_tensor_desc *>(in));
    if (op_ != Op::kDCN) return 0;  // grid sampler / rotate need none
    return b200_dcn_enqueue_workspace_size(reinterpret_cast<const b200_tensor_desc *>(in), a_.stride, a_.pad, a_.dil,
                                           a_.groups, a_.deform_groups);
  }
  int32_t enqueue(const PluginTensorDesc *in, const PluginTensorDesc *out, const void *const *inputs, void *const *outputs,
                  void *workspace, cudaStream_t stream) noexcept override {
    const auto *i = reinterpret_cast<const b200_tensor_desc *>(in);
    const auto *o = reinterpret_cast<const b200_tensor_desc *>(out);
    switch (op_) {
      case Op::kMSDA: return b200_msda_enqueue(i, o, inputs, outputs, workspace, stream, v2_);
      case Op::kBEVPool:  // both names run the same kernels
        return b200_bev_pool_enqueue(i, o, inputs, outputs, workspace, stream, bev_.out_height, bev_.out_width);
      case Op::kRotate: return b200_rotate_enqueue(i, o, inputs, outputs, workspace, stream, a_.interp, v2_);
      case Op::kDCN:  // inputs x, offset, mask, weight[, bias]; attributes are ONNX (h, w) pairs, checked against the descriptors
        return b200_dcn_enqueue(i, o, inputs, outputs, workspace, stream, nb_inputs_, a_.stride, a_.pad, a_.dil, a_.groups,
                                a_.deform_groups);
      default: return b200_grid_sampler_enqueue(i, o, inputs, outputs, workspace, stream, a_.interp, a_.padding, a_.align);
    }
  }
  // ---- IPluginV2Ext / IPluginV2
  DataType getOutputDataType(int32_t, const DataType *types, int32_t) const noexcept override { return types[0]; }
  const char *getPluginType() const noexcept override {
    switch (op_) {
      case Op::kMSDA: return v2_ ? "MultiScaleDeformableAttnTRT2" : "MultiScaleDeformableAttnTRT";
      case Op::kGridSampler2D: return v2_ ? "GridSampler2DTRT2" : "GridSampler2DTRT";
      case Op::kGridSampler3D: return v2_ ? "GridSampler3DTRT2" : "GridSampler3DTRT";
      case Op::kRotate: return v2_ ? "RotateTRT2" : "RotateTRT";
      case Op::kBEVPool: return v2_ ? "BEVPoolV2TRT2" : "BEVPoolV2TRT";
      default: return v2_ ? "ModulatedDeformableConv2dTRT2" : "ModulatedDeformableConv2dTRT";
    }
  }
  const char *getPluginVersion() const noexcept override { return "1"; }
  int32_t getNbOutputs() const noexcept override { return 1; }
  int32_t initialize() noexcept override { return 0; }
  void terminate() noexcept override {}
  size_t getSerializationSize() const noexcept override {
    if (op_ == Op::kBEVPool) return 2 * sizeof(int32_t);
    return op_ == Op::kMSDA ? 0 : sizeof(Attrs) + sizeof(int32_t);
  }
  void serialize(void *buf) const noexcept override {
    if (op_ == Op::kMSDA) return;
    if (op_ == Op::kBEVPool) {
      std::memcpy(buf, &bev_.out_width, sizeof(int32_t));
      std::memcpy(static_cast<char *>(buf) + sizeof(int32_t), &bev_.out_height, sizeof(int32_t));
      return;
    }
    std::memcpy(buf, &a_, sizeof(Attrs));
    std::memcpy(static_cast<char *>(buf) + sizeof(Attrs), &nb_inputs_, sizeof(int32_t));
  }
  void destroy() noexcept override { delete this; }
  void setPluginNamespace(const char *ns) noexcept override { ns_ = ns ? ns : ""; }
  const char *getPluginNamespace() const noexcept override { return ns_.c_str(); }
  void set_nb_inputs(int32_t n) { nb_inputs_ = n; }

 private:
  Op op_;
  bool v2_;
  Attrs a_;
  BevAttrs bev_;
  int32_t nb_inputs_ = 5;
  std::string ns_;
};

class Creator final : public IPluginCreator {
 public:
  Creator(Op op, bool v2) : op_(op), v2_(v2) {
    if (op == Op::kGridSampler2D || op == Op::kGridSampler3D) {
      fields_ = {{"interpolation_mode", nullptr, PluginFieldType::kINT32, 1},
                 {"padding_mode", nullptr, PluginFieldType::kINT32, 1},
                 {"align_corners", nullptr, PluginFieldType::kINT32, 1}};
    } else if (op == Op::kRotate) {
      fields_ = {{"interpolation", nullptr, PluginFieldType::kINT32, 1}};
    } else if (op == Op::kBEVPool) {
      fields_ = {{"out_height", nullptr, PluginFieldType::kINT32, 1}, {"out_width", nullptr, PluginFieldType::kINT32, 1}};
    } else if (op == Op::kDCN) {
      fields_ = {{"stride", nullptr, PluginFieldType::kINT32, 2},   {"padding", nullptr, PluginFieldType::kINT32, 2},
                 {"dilation", nullptr, PluginFieldType::kINT32, 2}, {"groups", nullptr, PluginFieldType::kINT32, 1},
                 {"deform_groups", nullptr, PluginFieldType::kINT32, 1}};
    }
    fc_.nbFields = static_cast<int32_t>(fields_.size());
    fc_.fields = fields_.data();
  }
  const char *getPluginName() const noexcept override { return Plugin(op_, v2_, Attrs{}).getPluginType(); }
  const char *getPluginVersion() const noexcept override { return "1"; }
  const PluginFieldCollection *getFieldNames() noexcept override { return &fc_; }
  IPluginV2 *createPlugin(const char *, const PluginFieldCollection *fc) noexcept override {
    Attrs a;
    BevAttrs bev;
    for (int32_t i = 0; fc && i < fc->nbFields; ++i) {
      const PluginField &f = fc->fields[i];
      const auto *v = static_cast<const int32_t *>(f.data);
      if (!v || !f.name) continue;
      const std::string n = f.name;
      if (n == "interpolation_mode" || n == "interpolation") a.interp = v[0];
      else if (n == "padding_mode") a.padding = v[0];
      else if (n == "align_corners") a.align = v[0];
      else if (n == "stride") a.stride[0] = v[0], a.stride[1] = f.length > 1 ? v[1] : v[0];
      else if (n == "padding") a.pad[0] = v[0], a.pad[1] = f.length > 1 ? v[1] : v[0];
      else if (n == "dilation") a.dil[0] = v[0], a.dil[1] = f.length > 1 ? v[1] : v[0];
      else if (n == "groups") a.groups = v[0];
      else if (n == "deform_groups") a.deform_groups = v[0];
      else if (n == "out_height") bev.out_height = v[0];
      else if (n == "out_width") bev.out_width = v[0];
    }
    return new (std::nothrow) Plugin(op_, v2_, a, bev);
  }
  IPluginV2 *deserializePlugin(const char *, const void *data, size_t len) noexcept override {
    Attrs a;
    int32_t nb = 5;
    if (op_ == Op::kBEVPool) {
      BevAttrs bev;
      if (len >= 2 * sizeof(int32_t)) {
        std::memcpy(&bev.out_width, data, sizeof(int32_t));
        std::memcpy(&bev.out_height, static_cast<const char *>(data) + sizeof(int32_t), sizeof(int32_t));
      }
      return new (std::nothrow) Plugin(op_, v2_, a, bev);
    }
    if (op_ != Op::kMSDA && len >= sizeof(Attrs) + sizeof(int32_t)) {
      std::memcpy(&a, data, sizeof(Attrs));
      std::memcpy(&nb, static_cast<const char *>(data) + sizeof(Attrs), sizeof(int32_t));
    }
    auto *p = new (std::nothrow) Plugin(op_, v2_, a);
    if (p) p->set_nb_inputs(nb);
    return p;
  }
  void setPluginNamespace(const char *ns) noexcept override { ns_ = ns ? ns : ""; }
  const char *getPluginNamespace() const noexcept override { return ns_.c_str(); }

 private:
  Op op_;
  bool v2_;
  std::vector<PluginField> fields_;
  PluginFieldCollection fc_{};
  std::string ns_;
};

#define B200_REGISTER(cls_name, op, v2)                  \
  class cls_name final : public IPluginCreator {         \
   public:                                               \
    cls_name() : c_(op, v2) {}                           \
    const char *getPluginName() const noexcept override { return c_.getPluginName(); }                          \
    const char *getPluginVersion() const noexcept override { return c_.getPluginVersion(); }                    \
    const PluginFieldCollection *getFieldNames() noexcept override { return c_.getFieldNames(); }               \
    IPluginV2 *createPlugin(const char *n, const PluginFieldCollection *f) noexcept override { return c_.createPlugin(n, f); } \
    IPluginV2 *deserializePlugin(const char *n, const void *d, size_t l) noexcept override { return c_.deserializePlugin(n, d, l); } \
    void setPluginNamespace(const char *ns) noexcept override { c_.setPluginNamespace(ns); }                    \
    const char *getPluginNamespace() const noexcept override { return c_.getPluginNamespace(); }                \
   private:                                              \
    Creator c_;                                          \
  };                                                     \
  REGISTER_TENSORRT_PLUGIN(cls_name)

B200_REGISTER(MsdaCreator, Op::kMSDA, false);
B200_REGISTER(MsdaCreator2, Op::kMSDA, true);
B200_REGISTER(GridSampler2DCreator, Op::kGridSampler2D, false);
B200_REGISTER(GridSampler2DCreator2, Op::kGridSampler2D, true);
B200_REGISTER(GridSampler3DCreator, Op::kGridSampler3D, false);
B200_REGISTER(GridSampler3DCreator2, Op::kGridSampler3D, true);
B200_REGISTER(DcnCreator, Op::kDCN, false);
B200_REGISTER(DcnCreator2, Op::kDCN, true);
B200_REGISTER(RotateCreator, Op::kRotate, false);
B200_REGISTER(RotateCreator2, Op::kRotate, true);
B200_REGISTER(BEVPoolCreator, Op::kBEVPool, false);
B200_REGISTER(BEVPoolCreator2, Op::kBEVPool, true);

}  // namespace b200_trt
#endif  // __has_include(<NvInfer.h>)

// tests/mock_trt/bev_pool_capi.cpp — TEST-ONLY. A C face for the TensorRT plugin shells
// (csrc/trt_plugin/b200_trt_plugins.cpp, compiled against the mock NvInfer.h next to this file) with the calls
// tests/test_bev_pool_cpu.py and tests/test_bev_pool_plugin_gpu.py make: creator fields -> createPlugin, serialize ->
// deserializePlugin, getOutputDimensions, supportsFormatCombination, enqueue, destroy. The mock declares IExprBuilder
// without defining it; this file defines a minimal one first, so the BEVPool shells' constant output dimensions can be
// read back. Every function only turns one virtual call into a C call.
#include <NvInfer.h>

#include <cstdio>
#include <deque>
#include <string>
#include <vector>

namespace nvinfer1 {
class IDimensionExpr {
 public:
  explicit IDimensionExpr(int32_t v) : value(v) {}
  int32_t value;
};
class IExprBuilder {
 public:
  const IDimensionExpr *constant(int32_t v) noexcept {
    exprs_.emplace_back(v);
    return &exprs_.back();
  }

 private:
  std::deque<IDimensionExpr> exprs_;
};
}  // namespace nvinfer1

#include "../../bevformer_tensorrt_b200/csrc/trt_plugin/b200_trt_plugins.cpp"

using namespace nvinfer1;
using b200_trt::Creator;
using b200_trt::Op;

namespace {
Creator *find_creator(const char *name) {
  static Creator creators[] = {{Op::kBEVPool, false}, {Op::kBEVPool, true}, {Op::kRotate, false}, {Op::kRotate, true},
                               {Op::kDCN, false},     {Op::kGridSampler2D, false}};
  for (Creator &c : creators)
    if (std::string(c.getPluginName()) == name) return &c;
  return nullptr;
}
IPluginV2DynamicExt *dyn(void *p) { return static_cast<IPluginV2DynamicExt *>(static_cast<IPluginV2 *>(p)); }
}  // namespace

extern "C" {

// Creator::createPlugin with INT32 fields: field i is names[i] with lengths[i] values, stored one after another.
void *bcapi_create(const char *plugin_name, int nb_fields, const char *const *names, const int32_t *values,
                   const int32_t *lengths) {
  Creator *c = find_creator(plugin_name);
  if (!c) return nullptr;
  std::vector<PluginField> fields;
  for (int i = 0, at = 0; i < nb_fields; at += lengths[i], ++i)
    fields.push_back({names[i], values + at, PluginFieldType::kINT32, lengths[i]});
  PluginFieldCollection fc{nb_fields, fields.data()};
  return c->createPlugin("layer", &fc);
}

// The creator's field names, comma separated, into buf.
void bcapi_field_names(const char *plugin_name, char *buf, int len) {
  std::string s;
  if (Creator *c = find_creator(plugin_name)) {
    const PluginFieldCollection *fc = c->getFieldNames();
    for (int i = 0; i < fc->nbFields; ++i) s += (i ? "," : "") + std::string(fc->fields[i].name);
  }
  snprintf(buf, len, "%s", s.c_str());
}

const char *bcapi_plugin_type(void *plugin) { return static_cast<IPluginV2 *>(plugin)->getPluginType(); }
const char *bcapi_plugin_version(void *plugin) { return static_cast<IPluginV2 *>(plugin)->getPluginVersion(); }

size_t bcapi_serialization_size(void *plugin) { return static_cast<IPluginV2 *>(plugin)->getSerializationSize(); }
void bcapi_serialize(void *plugin, void *buf) { static_cast<IPluginV2 *>(plugin)->serialize(buf); }

void *bcapi_deserialize(const char *plugin_name, const void *blob, size_t len) {
  Creator *c = find_creator(plugin_name);
  return c ? c->deserializePlugin("layer", blob, len) : nullptr;
}

// getOutputDimensions for 7 inputs whose feat (input 1) has last dimension feat_c; dims[0..3] receive the result.
int bcapi_output_dims(void *plugin, int32_t feat_c, int32_t *dims) {
  IExprBuilder b;
  const IDimensionExpr c(feat_c);
  DimsExprs in[7]{};
  in[1].nbDims = 4, in[1].d[3] = &c;
  const DimsExprs o = dyn(plugin)->getOutputDimensions(0, in, 7, b);
  for (int i = 0; i < o.nbDims; ++i) dims[i] = o.d[i] ? o.d[i]->value : -1;
  return o.nbDims;
}

int bcapi_supports(void *plugin, int pos, const PluginTensorDesc *in_out, int nb_inputs, int nb_outputs) {
  return dyn(plugin)->supportsFormatCombination(pos, in_out, nb_inputs, nb_outputs) ? 1 : 0;
}

int bcapi_enqueue(void *plugin, const PluginTensorDesc *in, const PluginTensorDesc *out, const void *const *inputs,
                  void *const *outputs, void *stream) {
  return dyn(plugin)->enqueue(in, out, inputs, outputs, nullptr, static_cast<cudaStream_t>(stream));
}

void bcapi_destroy(void *plugin) { static_cast<IPluginV2 *>(plugin)->destroy(); }

}  // extern "C"

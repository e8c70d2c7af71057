// host_capi.cc -- extern "C" face of the graph host for language bindings (the
// Python front-end and the tests drive it through ctypes). Mirrors the calls a
// C++ user of the reference makes in examples/lce_minimal.cc:31-53:
//   resolver + RegisterLCECustomOps -> build graph -> AllocateTensors -> Invoke.
#include <cuda_runtime.h>

#include <cstring>
#include <string>
#include <vector>

#include "flexbuffer_map.h"
#include "host_graph.h"
#include "lce_b200_tflite.h"

using lce_b200::Graph;
using lce_b200::OpResolver;

namespace lce_b200 {
void RegisterBuiltinOps(OpResolver* resolver);  // builtin_ops.cc
bool BuildGraphFromTflite(const uint8_t* data, size_t size, const OpResolver& resolver,
                          Graph* graph);        // tflite_model.cc
// One resolver per selector of RegisterLCECustomOps (lce_ops_register.h:25-53):
// 0 = default, 1 = use_reference_bconv, 2 = use_indirect_bgemm.
OpResolver* Resolver(int which) {
  static OpResolver* r[3] = {nullptr, nullptr, nullptr};
  if (which < 0 || which > 2) which = 0;
  if (!r[which]) {
    auto* res = new OpResolver();
    compute_engine::tflite::RegisterLCECustomOps(res, which == 1, which == 2);
    // the reference's other registrations stay reachable under explicit names
    res->AddCustom("LceBconv2d:REF", compute_engine::tflite::Register_BCONV_2D_REF());
    res->AddCustom("LceBconv2d:OPT_BGEMM", compute_engine::tflite::Register_BCONV_2D_OPT_BGEMM());
    res->AddCustom("LceBconv2d:OPT_INDIRECT_BGEMM",
                   compute_engine::tflite::Register_BCONV_2D_OPT_INDIRECT_BGEMM());
    RegisterBuiltinOps(res);
    r[which] = res;
  }
  return r[which];
}
OpResolver* DefaultResolver() { return Resolver(0); }
}  // namespace lce_b200

extern "C" {

void* lce_host_graph_create(int device_arena) { return new Graph(device_arena != 0); }
void lce_host_graph_destroy(void* g) { delete static_cast<Graph*>(g); }
const char* lce_host_last_error(void* g) { return static_cast<Graph*>(g)->last_error().c_str(); }

// FlatBufferModel::BuildFromBuffer + InterpreterBuilder in one call
// (examples/lce_minimal.cc:31-45). Returns nullptr on failure; *error gets a message
// valid until the next call on this thread.
void* lce_host_graph_from_tflite(const uint8_t* data, size_t size, int device_arena,
                                 const char** error) {
  static thread_local std::string msg;
  auto* g = new Graph(device_arena != 0);
  if (!lce_b200::BuildGraphFromTflite(data, size, *lce_b200::DefaultResolver(), g)) {
    msg = g->last_error();
    if (error) *error = msg.c_str();
    delete g;
    return nullptr;
  }
  return g;
}

// The same with the selectors of RegisterLCECustomOps / the reference's Interpreter
// (LCE/tflite/python/interpreter.py:40-58): use_reference_bconv resolves LceBconv2d to
// Register_BCONV_2D_REF, use_indirect_bgemm to Register_BCONV_2D_OPT_INDIRECT_BGEMM.
void* lce_host_graph_from_tflite_ex(const uint8_t* data, size_t size, int device_arena,
                                    int use_reference_bconv, int use_indirect_bgemm,
                                    const char** error) {
  static thread_local std::string msg;
  auto* g = new Graph(device_arena != 0);
  const int which = use_reference_bconv ? 1 : (use_indirect_bgemm ? 2 : 0);
  if (!lce_b200::BuildGraphFromTflite(data, size, *lce_b200::Resolver(which), g)) {
    msg = g->last_error();
    if (error) *error = msg.c_str();
    delete g;
    return nullptr;
  }
  return g;
}

// Device selection for processes that drive several GPUs (one graph per device).
int lce_host_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}
int lce_host_set_device(int index) { return cudaSetDevice(index) == cudaSuccess ? 0 : 1; }
int lce_host_get_device(void) {
  int d = -1;
  if (cudaGetDevice(&d) != cudaSuccess) cudaGetLastError();
  return d;
}

// Make an external registration (e.g. the oracle-backed CPU ops used by the CPU
// tests) available under `name`.
void lce_host_register_custom(const char* name, const TfLiteRegistration* registration) {
  for (int w = 0; w < 3; ++w) lce_b200::Resolver(w)->AddCustom(name, registration);
}
int lce_host_has_custom(const char* name) {
  return lce_b200::DefaultResolver()->FindCustom(name) != nullptr;
}

int lce_host_add_tensor(void* g, int type, const int* dims, int ndims, const void* const_data,
                        size_t const_bytes, int has_quant, float scale, int zero_point,
                        const char* name) {
  return static_cast<Graph*>(g)->AddTensor(static_cast<TfLiteType>(type),
                                           std::vector<int>(dims, dims + ndims), const_data,
                                           const_bytes, has_quant != 0, scale, zero_point,
                                           name ? name : "");
}

int lce_host_add_custom_node(void* gv, const char* op_name, const int* inputs, int n_in,
                             const int* outputs, int n_out, const uint8_t* options,
                             size_t options_len) {
  auto* g = static_cast<Graph*>(gv);
  const TfLiteRegistration* reg = lce_b200::DefaultResolver()->FindCustom(op_name);
  if (!reg) {
    g->set_error(std::string("custom op not registered: ") + op_name);
    return -1;
  }
  return g->AddNode(reg, std::vector<int>(inputs, inputs + n_in),
                    std::vector<int>(outputs, outputs + n_out), options, options_len, nullptr, 0,
                    op_name);
}

void lce_host_set_io(void* g, const int* inputs, int n_in, const int* outputs, int n_out) {
  static_cast<Graph*>(g)->SetInputs(std::vector<int>(inputs, inputs + n_in));
  static_cast<Graph*>(g)->SetOutputs(std::vector<int>(outputs, outputs + n_out));
}
int lce_host_allocate_tensors(void* g) { return static_cast<Graph*>(g)->AllocateTensors(); }
int lce_host_resize_input(void* g, int tensor, const int* dims, int ndims) {
  return static_cast<Graph*>(g)->ResizeInputTensor(tensor, std::vector<int>(dims, dims + ndims));
}
int lce_host_invoke(void* g) { return static_cast<Graph*>(g)->Invoke(); }
int lce_host_enable_cuda_graph(void* g, int on) {
  return static_cast<Graph*>(g)->EnableCudaGraph(on != 0);
}
int lce_host_fuse_residual_blocks(void* g) { return static_cast<Graph*>(g)->FuseResidualBlocks(); }
int lce_host_fuse_float_glue(void* g) { return static_cast<Graph*>(g)->FuseFloatGlue(); }
int lce_host_fuse_channel_gates(void* g) { return static_cast<Graph*>(g)->FuseChannelGates(); }
int lce_host_fuse_spatial_scales(void* g) { return static_cast<Graph*>(g)->FuseSpatialScales(); }
int lce_host_fuse_binary_bases(void* g) { return static_cast<Graph*>(g)->FuseBinaryBases(); }
int lce_host_fuse_pooled_signs(void* g) { return static_cast<Graph*>(g)->FusePooledSigns(); }
int lce_host_fuse_quantized_activations(void* g) {
  return static_cast<Graph*>(g)->FuseQuantizedActivations();
}
int lce_host_fuse_grouped_conv_affine(void* g) { return static_cast<Graph*>(g)->FuseGroupedConvAffine(); }
int lce_host_fuse_dense_blocks(void* g) { return static_cast<Graph*>(g)->FuseDenseBlocks(); }
int lce_host_fuse_activation_chains(void* g) { return static_cast<Graph*>(g)->FuseActivationChains(); }
int lce_host_fuse_upsample_merges(void* g) { return static_cast<Graph*>(g)->FuseUpsampleMerges(); }
int lce_host_fuse_resize_argmax(void* g) { return static_cast<Graph*>(g)->FuseResizeArgmax(); }
int lce_host_fuse_subpixel_convs(void* g) { return static_cast<Graph*>(g)->FuseSubpixelConvs(); }
int lce_host_fuse_binary_transpose_convs(void* g) { return static_cast<Graph*>(g)->FuseBinaryTransposeConvs(); }
int lce_host_fuse_binary_fully_connected(void* g) { return static_cast<Graph*>(g)->FuseBinaryFullyConnected(); }
int lce_host_fuse_binary_fc_max(void* g) { return static_cast<Graph*>(g)->FuseBinaryFcMax(); }
int lce_host_fuse_residual_pairs(void* g) { return static_cast<Graph*>(g)->FuseResidualPairs(); }
void lce_host_enable_profiling(void* g, int on) { static_cast<Graph*>(g)->EnableProfiling(on != 0); }
void lce_host_reset_profile(void* g) { static_cast<Graph*>(g)->ResetProfile(); }
double lce_host_node_time_ms(void* g, int node) { return static_cast<Graph*>(g)->NodeTimeMs(node); }
const char* lce_host_node_name(void* g, int node) {
  return static_cast<Graph*>(g)->node(node).name.c_str();
}
int lce_host_node_num_inputs(void* g, int node) {
  return static_cast<Graph*>(g)->node(node).node.inputs->size;
}
int lce_host_node_input(void* g, int node, int k) {
  return static_cast<Graph*>(g)->node(node).node.inputs->data[k];
}
int lce_host_node_num_outputs(void* g, int node) {
  return static_cast<Graph*>(g)->node(node).node.outputs->size;
}
int lce_host_node_output(void* g, int node, int k) {
  return static_cast<Graph*>(g)->node(node).node.outputs->data[k];
}
int lce_host_synchronize(void* g) { return static_cast<Graph*>(g)->Synchronize(); }
int lce_host_tensor_read_async(void* g, int i, void* dst, size_t bytes) {
  return static_cast<Graph*>(g)->ReadTensorAsync(i, dst, bytes);
}
void lce_host_preserve_all_tensors(void* g, int on) {
  static_cast<Graph*>(g)->set_preserve_all_tensors(on != 0);
}
int lce_host_num_tensors(void* g) { return static_cast<int>(static_cast<Graph*>(g)->num_tensors()); }
int lce_host_num_nodes(void* g) { return static_cast<int>(static_cast<Graph*>(g)->num_nodes()); }
int lce_host_tensor_type(void* g, int i) { return static_cast<Graph*>(g)->tensor(i)->type; }
int lce_host_tensor_ndims(void* g, int i) { return static_cast<Graph*>(g)->tensor(i)->dims->size; }
int lce_host_tensor_dim(void* g, int i, int d) {
  return static_cast<Graph*>(g)->tensor(i)->dims->data[d];
}
size_t lce_host_tensor_bytes(void* g, int i) { return static_cast<Graph*>(g)->tensor(i)->bytes; }
void* lce_host_tensor_data(void* g, int i) { return static_cast<Graph*>(g)->tensor(i)->data.raw; }
int lce_host_tensor_in_arena(void* g, int i) {
  return static_cast<Graph*>(g)->tensor(i)->allocation_type == kTfLiteArenaRw;
}
const char* lce_host_tensor_name(void* g, int i) { return static_cast<Graph*>(g)->tensor(i)->name; }
float lce_host_tensor_scale(void* g, int i) { return static_cast<Graph*>(g)->tensor(i)->params.scale; }
int lce_host_tensor_zero_point(void* g, int i) {
  return static_cast<Graph*>(g)->tensor(i)->params.zero_point;
}
int lce_host_tensor_write(void* g, int i, const void* src, size_t bytes) {
  return static_cast<Graph*>(g)->WriteTensor(i, src, bytes);
}
int lce_host_tensor_read(void* g, int i, void* dst, size_t bytes) {
  return static_cast<Graph*>(g)->ReadTensor(i, dst, bytes);
}
size_t lce_host_arena_bytes(void* g) { return static_cast<Graph*>(g)->arena_bytes(); }
void* lce_host_stream(void* g) { return static_cast<Graph*>(g)->stream(); }
int lce_host_num_inputs(void* g) { return static_cast<int>(static_cast<Graph*>(g)->inputs().size()); }
int lce_host_num_outputs(void* g) { return static_cast<int>(static_cast<Graph*>(g)->outputs().size()); }
int lce_host_input(void* g, int k) { return static_cast<Graph*>(g)->inputs()[k]; }
int lce_host_output(void* g, int k) { return static_cast<Graph*>(g)->outputs()[k]; }

// FlexBuffers helpers for bindings: parse a map of ints / write one.
int lce_host_flex_get_int(const uint8_t* buf, size_t len, const char* key, int* found) {
  lce_b200::FlexMap m(buf, len);
  *found = m.Has(key) ? 1 : 0;
  return m.AsInt32(key);
}
float lce_host_flex_get_float(const uint8_t* buf, size_t len, const char* key, float default_value) {
  return lce_b200::FlexMap(buf, len).AsFloat(key, default_value);
}
int lce_host_flex_get_bool(const uint8_t* buf, size_t len, const char* key, int default_value) {
  return lce_b200::FlexMap(buf, len).AsBool(key, default_value != 0) ? 1 : 0;
}
int lce_host_flex_map_size(const uint8_t* buf, size_t len) {
  lce_b200::FlexMap m(buf, len);
  return m.ok() ? static_cast<int>(m.size()) : -1;
}
// keys: '\0'-separated list; returns the number of bytes written (<= cap) or -1.
int lce_host_flex_write_int_map(const char* keys, const int64_t* values, int n, uint8_t* out,
                                size_t cap) {
  std::vector<std::pair<std::string, int64_t>> items;
  const char* k = keys;
  for (int i = 0; i < n; ++i) {
    items.emplace_back(std::string(k), values[i]);
    k += strlen(k) + 1;
  }
  auto bytes = lce_b200::WriteFlexIntMap(std::move(items));
  if (bytes.empty() || bytes.size() > cap) return -1;
  memcpy(out, bytes.data(), bytes.size());
  return static_cast<int>(bytes.size());
}

}  // extern "C"

#include "host_graph.h"

#include "builtin_params.h"
#include "flexbuffer_map.h"
#include "lce_b200.h"
#include "lce_b200_types.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace lce_b200 {

namespace {
size_t TypeSize(TfLiteType t) {
  switch (t) {
    case kTfLiteFloat32: return 4;
    case kTfLiteInt32: return 4;
    case kTfLiteInt64: return 8;
    case kTfLiteUInt8:
    case kTfLiteInt8:
    case kTfLiteBool: return 1;
    default: return 0;
  }
}
TfLiteIntArray* MakeDims(const std::vector<int>& d) {
  TfLiteIntArray* a = LceB200IntArrayCreate(static_cast<int>(d.size()));
  for (size_t i = 0; i < d.size(); ++i) a->data[i] = d[i];
  return a;
}
size_t BytesOf(const TfLiteTensor& t) {
  size_t n = TypeSize(t.type);
  for (int i = 0; i < t.dims->size; ++i) n *= static_cast<size_t>(std::max(t.dims->data[i], 0));
  return n;
}
constexpr size_t kAlign = 256;
size_t AlignUp(size_t x) { return (x + kAlign - 1) / kAlign * kAlign; }
}  // namespace

// ------------------------------ OpResolver ------------------------------- //
void OpResolver::AddCustom(const char* name, const TfLiteRegistration* r) { custom_[name] = r; }
void OpResolver::AddBuiltin(int code, const TfLiteRegistration* r) { builtin_[code] = r; }
const TfLiteRegistration* OpResolver::FindCustom(const std::string& name) const {
  auto it = custom_.find(name);
  return it == custom_.end() ? nullptr : it->second;
}
const TfLiteRegistration* OpResolver::FindBuiltin(int code) const {
  auto it = builtin_.find(code);
  return it == builtin_.end() ? nullptr : it->second;
}

// --------------------------------- Graph --------------------------------- //
Graph::Graph(bool device_arena) : device_arena_(device_arena) {
  memset(&ctx_, 0, sizeof(ctx_));
  ctx_.impl_ = this;
  ctx_.ResizeTensor = &Graph::ResizeTensorCb;
  ctx_.ReportError = &Graph::ReportErrorCb;
  ctx_.AddTensors = &Graph::AddTensorsCb;
  ctx_.GetTensor = &Graph::GetTensorCb;
  ctx_.GetExternalContext = &Graph::GetExternalContextCb;
  ctx_.SetExternalContext = &Graph::SetExternalContextCb;
  ctx_.recommended_num_threads = 1;
  if (device_arena_) {
    cudaStream_t s = nullptr;
    if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess) stream_ = s;
    else cudaGetLastError();
  }
}

Graph::~Graph() {
  for (auto& n : nodes_) {
    if (n->initialized && n->registration->free) n->registration->free(&ctx_, n->node.user_data);
    LceB200IntArrayFree(n->node.inputs);
    LceB200IntArrayFree(n->node.outputs);
    LceB200IntArrayFree(n->node.temporaries);
    LceB200IntArrayFree(n->node.intermediates);
  }
  if (graph_exec_) cudaGraphExecDestroy(static_cast<cudaGraphExec_t>(graph_exec_));
  FreeArena();
  for (void* p : const_dev_)
    if (p) cudaFree(p);
  for (auto& t : tensors_) {
    LceB200IntArrayFree(t.dims);
    if (t.quantization.params) {
      auto* q = static_cast<TfLiteAffineQuantization*>(t.quantization.params);
      free(q->scale);
      LceB200IntArrayFree(q->zero_point);
      free(q);
    }
  }
  if (stream_) cudaStreamDestroy(static_cast<cudaStream_t>(stream_));
}

void Graph::RefreshContext() {
  ctx_.tensors = tensors_.data();
  ctx_.tensors_size = tensors_.size();
}

int Graph::AddTensor(TfLiteType type, const std::vector<int>& dims, const void* const_data,
                     size_t const_bytes, bool has_quant, float scale, int zero_point,
                     const std::string& name, bool const_on_device) {
  TfLiteTensor t;
  memset(&t, 0, sizeof(t));
  t.type = type;
  t.dims = MakeDims(dims);
  t.params.scale = scale;
  t.params.zero_point = zero_point;
  if (has_quant) {
    auto* q = static_cast<TfLiteAffineQuantization*>(malloc(sizeof(TfLiteAffineQuantization)));
    q->scale = static_cast<TfLiteFloatArray*>(malloc(sizeof(TfLiteFloatArray) + sizeof(float)));
    q->scale->size = 1;
    q->scale->data[0] = scale;
    q->zero_point = LceB200IntArrayCreate(1);
    q->zero_point->data[0] = zero_point;
    q->quantized_dimension = 0;
    t.quantization.type = kTfLiteAffineQuantization;
    t.quantization.params = q;
  }
  t.bytes = BytesOf(t);
  names_.push_back(name);
  const_host_.emplace_back();
  const_dev_.push_back(nullptr);
  const int idx = static_cast<int>(tensors_.size());
  if (const_data) {
    auto& h = const_host_.back();
    h.assign(static_cast<const uint8_t*>(const_data),
             static_cast<const uint8_t*>(const_data) + const_bytes);
    h.resize(const_bytes + 64, 0);  // slack: kernels may read whole vectors
    t.allocation_type = kTfLiteMmapRo;
    t.data.raw = reinterpret_cast<char*>(h.data());
    t.bytes = const_bytes;
    if (const_on_device && device_arena_) {
      void* d = nullptr;
      if (cudaMalloc(&d, const_bytes + 64) == cudaSuccess &&
          cudaMemcpy(d, h.data(), const_bytes + 64, cudaMemcpyHostToDevice) == cudaSuccess) {
        const_dev_.back() = d;
        t.data.raw = static_cast<char*>(d);
      } else {
        cudaGetLastError();
      }
    }
  } else {
    t.allocation_type = kTfLiteArenaRw;
  }
  tensors_.push_back(t);
  tensors_.back().name = names_.back().c_str();
  for (size_t i = 0; i < tensors_.size(); ++i) tensors_[i].name = names_[i].c_str();
  RefreshContext();
  allocated_ = false;
  return idx;
}

int Graph::AddNode(const TfLiteRegistration* registration, const std::vector<int>& inputs,
                   const std::vector<int>& outputs, const uint8_t* custom_options,
                   size_t options_len, const void* builtin_data, size_t builtin_bytes,
                   const std::string& name) {
  auto rec = std::make_unique<NodeRecord>();
  rec->registration = registration;
  rec->name = name;
  if (custom_options) rec->custom_options.assign(custom_options, custom_options + options_len);
  if (builtin_data)
    rec->builtin_blob.assign(static_cast<const uint8_t*>(builtin_data),
                             static_cast<const uint8_t*>(builtin_data) + builtin_bytes);
  rec->node.inputs = MakeDims(inputs);
  rec->node.outputs = MakeDims(outputs);
  rec->node.temporaries = LceB200IntArrayCreate(0);
  rec->node.intermediates = LceB200IntArrayCreate(0);
  rec->node.custom_initial_data = rec->custom_options.data();
  rec->node.custom_initial_data_size = static_cast<int>(rec->custom_options.size());
  rec->node.builtin_data = rec->builtin_blob.empty() ? nullptr : rec->builtin_blob.data();
  nodes_.push_back(std::move(rec));
  allocated_ = false;
  return static_cast<int>(nodes_.size()) - 1;
}

TfLiteStatus Graph::ResizeTensorCb(TfLiteContext* c, TfLiteTensor* t, TfLiteIntArray* new_size) {
  // Takes ownership of new_size (common.h: ResizeTensor contract).
  auto* g = static_cast<Graph*>(c->impl_);
  if (t->allocation_type == kTfLiteMmapRo) {
    LceB200IntArrayFree(new_size);
    g->error_ = "ResizeTensor called on a constant tensor";
    return kTfLiteError;
  }
  LceB200IntArrayFree(t->dims);
  t->dims = new_size;
  t->bytes = BytesOf(*t);
  g->allocated_ = false;
  return kTfLiteOk;
}

void Graph::ReportErrorCb(TfLiteContext* c, const char* msg, ...) {
  auto* g = static_cast<Graph*>(c->impl_);
  char buf[1024];
  va_list ap;
  va_start(ap, msg);
  vsnprintf(buf, sizeof(buf), msg, ap);
  va_end(ap);
  g->error_ = buf;
}

TfLiteStatus Graph::AddTensorsCb(TfLiteContext* c, int n, int* first) {
  auto* g = static_cast<Graph*>(c->impl_);
  if (first) *first = static_cast<int>(g->tensors_.size());
  for (int i = 0; i < n; ++i)
    g->AddTensor(kTfLiteNoType, {0}, nullptr, 0, false, 0.f, 0, "temporary");
  return kTfLiteOk;
}

TfLiteTensor* Graph::GetTensorCb(const TfLiteContext* c, int i) {
  auto* g = static_cast<Graph*>(c->impl_);
  if (i < 0 || i >= static_cast<int>(g->tensors_.size())) return nullptr;
  return &g->tensors_[i];
}

TfLiteExternalContext* Graph::GetExternalContextCb(TfLiteContext* c, TfLiteExternalContextType t) {
  auto* g = static_cast<Graph*>(c->impl_);
  return (t >= 0 && t < kTfLiteMaxExternalContexts) ? g->external_[t] : nullptr;
}
void Graph::SetExternalContextCb(TfLiteContext* c, TfLiteExternalContextType t,
                                 TfLiteExternalContext* e) {
  auto* g = static_cast<Graph*>(c->impl_);
  if (t >= 0 && t < kTfLiteMaxExternalContexts) g->external_[t] = e;
}

void Graph::FreeArena() {
  if (!arena_) return;
  if (device_arena_) cudaFree(arena_);
  else free(arena_);
  arena_ = nullptr;
  arena_bytes_ = 0;
}

// Greedy-by-size offset assignment over tensor lifetimes (the idea of TFLite's
// arena planner): tensors whose [first_use, last_use] node ranges are disjoint may
// share bytes. Graph inputs live from -1, graph outputs until the end.
TfLiteStatus Graph::PlanArena() {
  const int n_nodes = static_cast<int>(nodes_.size());
  const int n_t = static_cast<int>(tensors_.size());
  std::vector<int> first(n_t, n_nodes + 1), last(n_t, -2);
  auto touch = [&](int t, int when) {
    if (t < 0 || t >= n_t) return;
    first[t] = std::min(first[t], when);
    last[t] = std::max(last[t], when);
  };
  for (int t : inputs_) touch(t, -1);
  for (int i = 0; i < n_nodes; ++i) {
    const TfLiteNode& nd = nodes_[i]->node;
    for (int k = 0; k < nd.inputs->size; ++k) touch(nd.inputs->data[k], i);
    for (int k = 0; k < nd.outputs->size; ++k) touch(nd.outputs->data[k], i);
    for (int k = 0; k < nd.temporaries->size; ++k) touch(nd.temporaries->data[k], i);
  }
  for (int t : outputs_) touch(t, n_nodes);
  if (preserve_all_)
    for (int t = 0; t < n_t; ++t)
      if (last[t] >= -1) { first[t] = -1; last[t] = n_nodes; }
  struct Item { int t; size_t bytes; size_t off; };
  std::vector<Item> items;
  for (int t = 0; t < n_t; ++t) {
    if (tensors_[t].allocation_type != kTfLiteArenaRw || last[t] < -1) continue;
    items.push_back({t, AlignUp(std::max<size_t>(tensors_[t].bytes, 1) + 64), 0});
  }
  std::sort(items.begin(), items.end(),
            [](const Item& a, const Item& b) { return a.bytes > b.bytes; });
  std::vector<Item> placed;
  size_t total = 0;
  for (auto& it : items) {
    std::vector<std::pair<size_t, size_t>> busy;
    for (auto& p : placed)
      if (!(last[p.t] < first[it.t] || last[it.t] < first[p.t]))
        busy.emplace_back(p.off, p.off + p.bytes);
    std::sort(busy.begin(), busy.end());
    size_t off = 0;
    for (auto& b : busy) {
      if (off + it.bytes <= b.first) break;
      off = std::max(off, b.second);
    }
    it.off = off;
    placed.push_back(it);
    total = std::max(total, off + it.bytes);
  }
  if (total > arena_bytes_) {
    FreeArena();
    if (device_arena_) {
      if (cudaMalloc(&arena_, total) != cudaSuccess) {
        error_ = std::string("cudaMalloc of the tensor arena failed: ") +
                 cudaGetErrorString(cudaGetLastError());
        return kTfLiteError;
      }
    } else {
      arena_ = malloc(total);
      if (!arena_) return kTfLiteError;
    }
    arena_bytes_ = total;
  }
  for (auto& p : placed) tensors_[p.t].data.raw = static_cast<char*>(arena_) + p.off;
  return kTfLiteOk;
}

// ------------------------------ graph fusion ------------------------------ //
namespace {
// The names of the builtin nodes the passes match: "builtin:<BuiltinOperator code>", as
// BuildGraphFromTflite gives them (tflite_model.cc:323). Custom nodes carry their op's name.
constexpr const char* kAdd = "builtin:0";
constexpr const char* kConcatenation = "builtin:2";
constexpr const char* kConv2d = "builtin:3";
constexpr const char* kDepthwiseConv2d = "builtin:4";
constexpr const char* kDequantize = "builtin:6";
constexpr const char* kFullyConnected = "builtin:9";
constexpr const char* kMaxPool2d = "builtin:17";
constexpr const char* kResizeNearest = "builtin:97";
constexpr const char* kResizeBilinear = "builtin:23";
constexpr const char* kArgMax = "builtin:56";
constexpr const char* kDepthToSpace = "builtin:5";
constexpr const char* kTransposeConv = "builtin:67";
constexpr const char* kMul = "builtin:18";
constexpr const char* kReshape = "builtin:22";
constexpr const char* kReduceMax = "builtin:82";
constexpr const char* kRelu = "builtin:19";
constexpr const char* kMean = "builtin:40";
constexpr const char* kDiv = "builtin:42";
constexpr const char* kStridedSlice = "builtin:45";
constexpr const char* kPrelu = "builtin:54";
constexpr const char* kMaximum = "builtin:55";
constexpr const char* kMinimum = "builtin:57";
constexpr const char* kRound = "builtin:116";

std::vector<int> Ints(const TfLiteIntArray* a) { return std::vector<int>(a->data, a->data + a->size); }
}  // namespace

bool Graph::IsGraphOutput(int t) const {
  return std::find(outputs_.begin(), outputs_.end(), t) != outputs_.end();
}

std::vector<size_t> Graph::Consumers(int t) const {
  std::vector<size_t> c;
  for (size_t k = 0; k < nodes_.size(); ++k)
    for (int q = 0; q < nodes_[k]->node.inputs->size; ++q)
      if (nodes_[k]->node.inputs->data[q] == t) { c.push_back(k); break; }
  return c;
}

size_t Graph::SoleConsumer(int t) const {
  if (IsGraphOutput(t)) return kNoNode;
  const std::vector<size_t> c = Consumers(t);
  return c.size() == 1 ? c[0] : kNoNode;
}

size_t Graph::SoleReaderAsFirstInput(int t) const {
  if (IsGraphOutput(t)) return kNoNode;
  size_t found = kNoNode;
  int slots = 0;
  for (size_t k = 0; k < nodes_.size(); ++k)
    for (int q = 0; q < nodes_[k]->node.inputs->size; ++q)
      if (nodes_[k]->node.inputs->data[q] == t) { ++slots; found = k; }
  return slots == 1 && nodes_[found]->node.inputs->data[0] == t ? found : kNoNode;
}

bool Graph::ReadyBefore(int t, size_t i) const {
  if (std::find(inputs_.begin(), inputs_.end(), t) != inputs_.end()) return true;
  for (size_t k = 0; k < i; ++k)
    for (int q = 0; q < nodes_[k]->node.outputs->size; ++q)
      if (nodes_[k]->node.outputs->data[q] == t) return true;
  return false;
}

bool Graph::SameDims(const TfLiteIntArray* a, const TfLiteIntArray* b) {
  if (!a || !b || a->size != b->size) return false;
  for (int k = 0; k < a->size; ++k)
    if (a->data[k] != b->data[k]) return false;
  return true;
}

const BuiltinParams* Graph::Params(const NodeRecord& n) {
  return n.builtin_blob.size() >= sizeof(BuiltinParams)
             ? reinterpret_cast<const BuiltinParams*>(n.builtin_blob.data())
             : nullptr;
}

int32_t Graph::Activation(const NodeRecord& n) { return Params(n) ? Params(n)->activation : 0; }

int Graph::PerChannelConstOp(size_t k, const char* op, int x, int C, bool any_activation) const {
  if (k >= nodes_.size()) return -1;
  const NodeRecord& n = *nodes_[k];
  if (n.name != op || n.initialized || n.node.inputs->size != 2 || n.node.outputs->size != 1 ||
      n.node.inputs->data[0] != x || tensors_[n.node.outputs->data[0]].type != kTfLiteFloat32 ||
      !Params(n) || (!any_activation && Params(n)->activation != 0))
    return -1;
  const int v = n.node.inputs->data[1];
  if (v < 0) return -1;
  const TfLiteTensor& t = tensors_[v];
  if (t.type != kTfLiteFloat32 || t.allocation_type != kTfLiteMmapRo || t.dims->size < 1 ||
      t.dims->data[t.dims->size - 1] != C)
    return -1;
  for (int d = 0; d + 1 < t.dims->size; ++d)
    if (t.dims->data[d] != 1) return -1;
  return v;
}

bool Graph::IsQuantize(size_t k) const {
  if (k >= nodes_.size()) return false;
  const NodeRecord& n = *nodes_[k];
  return n.name == "LceQuantize" && !n.initialized && n.node.inputs->size == 1 &&
         n.node.outputs->size == 1 && tensors_[n.node.outputs->data[0]].type == kTfLiteInt32;
}

void Graph::EraseNode(size_t k) {
  TfLiteNode& n = nodes_[k]->node;
  LceB200IntArrayFree(n.inputs);
  LceB200IntArrayFree(n.outputs);
  LceB200IntArrayFree(n.temporaries);
  LceB200IntArrayFree(n.intermediates);
  nodes_.erase(nodes_.begin() + k);
  allocated_ = false;
}

void Graph::EraseNodes(std::vector<size_t> ks) {
  std::sort(ks.begin(), ks.end());
  for (auto it = ks.rbegin(); it != ks.rend(); ++it) EraseNode(*it);   // the highest index first
}

void Graph::SetNodeIO(NodeRecord& n, const std::vector<int>& inputs, const std::vector<int>& outputs,
                      const std::vector<int>& temporaries) {
  LceB200IntArrayFree(n.node.inputs);
  LceB200IntArrayFree(n.node.outputs);
  LceB200IntArrayFree(n.node.temporaries);
  n.node.inputs = MakeDims(inputs);
  n.node.outputs = MakeDims(outputs);
  n.node.temporaries = MakeDims(temporaries);
  allocated_ = false;
}

void Graph::SetBuiltinBlob(NodeRecord& n, const void* bytes, size_t len) {
  const uint8_t* b = static_cast<const uint8_t*>(bytes);
  n.builtin_blob.assign(b, b + len);
  n.node.builtin_data = n.builtin_blob.empty() ? nullptr : n.builtin_blob.data();
  allocated_ = false;
}

void Graph::SetCustomOptions(NodeRecord& n, std::vector<uint8_t> options) {
  n.custom_options = std::move(options);
  n.node.custom_initial_data = n.custom_options.data();
  n.node.custom_initial_data_size = static_cast<int>(n.custom_options.size());
  allocated_ = false;
}

extern "C" TfLiteRegistration* lce_b200_internal_Register_BCONV_2D_FUSED(const TfLiteRegistration* original);
extern "C" int lce_b200_internal_grouped_packs(const lce_bconv2d_desc* d);   // lce_b200.cu

int Graph::FuseResidualBlocks() {
  if (!device_arena_) return 0;
  int removed = 0;
  for (size_t i = 0; i < nodes_.size(); ++i) {
    NodeRecord& b = *nodes_[i];
    if (b.name != "LceBconv2d" || b.initialized || b.node.inputs->size != 5) continue;
    TfLiteRegistration* fused_reg = lce_b200_internal_Register_BCONV_2D_FUSED(b.registration);
    if (fused_reg == nullptr) continue;   // a foreign "LceBconv2d" (e.g. the CPU test double)
    const int y = b.node.outputs->data[0];
    if (tensors_[y].type != kTfLiteFloat32) continue;
    const size_t ai = SoleConsumer(y);
    if (ai == kNoNode) continue;
    NodeRecord& a = *nodes_[ai];
    if (a.name != kAdd || a.node.inputs->size != 2 || ai <= i) continue;
    const int in0 = a.node.inputs->data[0], in1 = a.node.inputs->data[1];
    if (in0 == in1) continue;
    const int r = in0 == y ? in1 : in0;
    if (tensors_[r].type != kTfLiteFloat32 || tensors_[r].allocation_type == kTfLiteMmapRo) continue;
    // Preconditions of the fused kernel, checked before the graph is rewritten (both graphs below
    // run correctly unfused): the shortcut has exactly the convolution's shape (ADD would also
    // accept a broadcast over the last dimension), and the convolution is ungrouped (filter words
    // per pixel == input words per pixel) or grouped such that the fused sign-pack takes it. Of the
    // grouped layers only those with channels_in == channels_out are fused: binary MobileNets'
    // layers in place of depthwise convolutions, the case this fusion is measured on; other
    // grouped layers run unfused.
    if (!SameDims(tensors_[y].dims, tensors_[r].dims)) continue;
    const TfLiteIntArray* xs = tensors_[b.node.inputs->data[0]].dims;
    const TfLiteIntArray* fs = tensors_[b.node.inputs->data[1]].dims;
    if (!xs || !fs || xs->size != 4 || fs->size != 4 || fs->data[3] < 1 || xs->data[3] % fs->data[3] != 0)
      continue;
    if (xs->data[3] != fs->data[3]) {
      lce_bconv2d_desc d{};
      d.channels_in = FlexMap(b.custom_options.data(), b.custom_options.size()).AsInt32("channels_in");
      d.channels_out = fs->data[0];
      d.groups = xs->data[3] / fs->data[3];
      d.out_type = LCE_OUT_FLOAT;
      if (d.channels_in != d.channels_out || !lce_b200_internal_grouped_packs(&d)) continue;
    }
    // the shortcut must already exist when the bconv runs
    if (!ReadyBefore(r, i)) continue;
    const int o = a.node.outputs->data[0];
    const int32_t add_act = Activation(a);
    std::vector<size_t> absorbed{ai};
    // optional: the LceQuantize that consumes the sum
    int packed = -1;
    for (size_t c : Consumers(o)) {
      NodeRecord& q = *nodes_[c];
      if (q.name == "LceQuantize" && c > ai && tensors_[o].type == kTfLiteFloat32) {
        packed = q.node.outputs->data[0];
        absorbed.push_back(c);
        break;
      }
    }
    std::vector<int> ins = Ints(b.node.inputs);
    ins.push_back(r);
    std::vector<int> outs{o};
    if (packed >= 0) outs.push_back(packed);
    SetNodeIO(b, ins, outs);
    b.registration = fused_reg;
    SetBuiltinBlob(b, &add_act, sizeof(add_act));
    b.name = packed >= 0 ? "LceBconv2d+ADD+LceQuantize" : "LceBconv2d+ADD";
    removed += static_cast<int>(absorbed.size());
    EraseNodes(absorbed);
  }
  allocated_ = false;
  return removed;
}

extern "C" TfLiteRegistration* lce_b200_internal_Register_BCONV_2D_PAIR(const TfLiteRegistration* fused);
extern "C" int lce_b200_internal_pair_pays_off(const lce_bconv2d_desc* d);   // lce_b200.cu

int Graph::FuseResidualPairs() {
  if (!device_arena_) return 0;
  // the channel count of a fused residual block (no chain) whose layer the pair kernel takes and
  // runs faster than two blocks at the input's current spatial size, or 0
  auto pair_channels = [&](const NodeRecord& n) {
    if (n.initialized || n.node.inputs->size != 6) return 0;
    const TfLiteIntArray* xd = tensors_[n.node.inputs->data[0]].dims;
    const TfLiteIntArray* fd = tensors_[n.node.inputs->data[1]].dims;
    if (xd->size != 4 || fd->size != 4) return 0;
    FlexMap m(n.custom_options.data(), n.custom_options.size());
    lce_bconv2d_desc d{};
    d.batch = xd->data[0]; d.in_h = xd->data[1]; d.in_w = xd->data[2];
    d.channels_in = m.AsInt32("channels_in");
    d.channels_out = fd->data[0]; d.filter_h = fd->data[1]; d.filter_w = fd->data[2];
    d.groups = fd->data[3] == (d.channels_in + 31) / 32 && xd->data[3] == fd->data[3] ? 1 : 0;
    d.stride_h = m.AsInt32("stride_height"); d.stride_w = m.AsInt32("stride_width");
    d.dilation_h = m.AsInt32("dilation_height_factor");
    d.dilation_w = m.AsInt32("dilation_width_factor");
    d.padding = m.AsInt32("padding"); d.pad_value = m.AsInt32("pad_values");
    d.out_type = tensors_[n.node.outputs->data[0]].type == kTfLiteFloat32 ? LCE_OUT_FLOAT : -1;
    return lce_b200_internal_pair_pays_off(&d) ? d.channels_out : 0;
  };
  int removed = 0;
  for (size_t i = 0; i < nodes_.size(); ++i) {
    NodeRecord& a = *nodes_[i];
    if (a.name != "LceBconv2d+ADD+LceQuantize" || a.node.outputs->size != 2) continue;
    TfLiteRegistration* pair_reg = lce_b200_internal_Register_BCONV_2D_PAIR(a.registration);
    if (pair_reg == nullptr) continue;
    // x1 and its signs feed the next block alone
    const int x1 = a.node.outputs->data[0], p1 = a.node.outputs->data[1];
    const size_t bi = SoleConsumer(x1);
    if (bi == kNoNode || SoleConsumer(p1) != bi || bi <= i) continue;
    NodeRecord& b = *nodes_[bi];
    if ((b.name != "LceBconv2d+ADD" && b.name != "LceBconv2d+ADD+LceQuantize") ||
        b.registration != a.registration || b.node.inputs->data[0] != p1 ||
        b.node.inputs->data[5] != x1)
      continue;
    const int C = pair_channels(a);
    if (C == 0 || pair_channels(b) != C) continue;
    std::vector<int> ins = Ints(a.node.inputs);
    ins.insert(ins.end(), b.node.inputs->data + 1, b.node.inputs->data + 5);
    // each block's blob is its ADD's activation
    const int32_t acts[2] = {*reinterpret_cast<const int32_t*>(a.builtin_blob.data()),
                             *reinterpret_cast<const int32_t*>(b.builtin_blob.data())};
    const uint32_t n = static_cast<uint32_t>(a.custom_options.size());
    std::vector<uint8_t> opts(reinterpret_cast<const uint8_t*>(&n), reinterpret_cast<const uint8_t*>(&n) + 4);
    opts.insert(opts.end(), a.custom_options.begin(), a.custom_options.end());
    opts.insert(opts.end(), b.custom_options.begin(), b.custom_options.end());
    SetNodeIO(a, ins, Ints(b.node.outputs));
    SetCustomOptions(a, opts);
    SetBuiltinBlob(a, acts, sizeof(acts));
    a.registration = pair_reg;
    a.name = "LceBconv2d+ADD+" + b.name;
    EraseNode(bi);
    ++removed;
  }
  allocated_ = false;
  return removed;
}

extern "C" TfLiteRegistration* lce_b200_internal_Register_BCONV_2D_GATE(const TfLiteRegistration* original);

int Graph::FuseChannelGates() {
  if (!device_arena_) return 0;
  int removed = 0;
  for (size_t i = 0; i < nodes_.size(); ++i) {
    NodeRecord& b = *nodes_[i];
    if (b.name != "LceBconv2d" || b.initialized || b.node.inputs->size != 5 || b.node.outputs->size != 1)
      continue;
    TfLiteRegistration* gate_reg = lce_b200_internal_Register_BCONV_2D_GATE(b.registration);
    if (gate_reg == nullptr) continue;
    const int y = b.node.outputs->data[0];
    const TfLiteIntArray* yd = tensors_[y].dims;
    if (tensors_[y].type != kTfLiteFloat32 || !yd || yd->size != 4) continue;
    const int C = yd->data[3];
    // MUL(y, g): g a computed float [B, 1, 1, C]
    const size_t km = SoleConsumer(y);
    if (km == kNoNode) continue;
    const NodeRecord& m = *nodes_[km];
    if (m.name != kMul || m.initialized || m.node.inputs->size != 2 || m.node.outputs->size != 1 ||
        m.node.inputs->data[0] != y || tensors_[m.node.outputs->data[0]].type != kTfLiteFloat32 ||
        Activation(m) != 0)
      continue;
    const int g = m.node.inputs->data[1];
    if (g < 0 || g == y) continue;
    const TfLiteTensor& gt = tensors_[g];
    if (gt.type != kTfLiteFloat32 || gt.allocation_type == kTfLiteMmapRo || !gt.dims || gt.dims->size != 4 ||
        gt.dims->data[0] != yd->data[0] || gt.dims->data[1] != 1 || gt.dims->data[2] != 1 ||
        gt.dims->data[3] != C || !ReadyBefore(g, i))
      continue;
    // PRELU(t, alpha [1, ..., 1, C])
    const int t1 = m.node.outputs->data[0];
    const size_t kp = SoleConsumer(t1);
    const int alpha = PerChannelConstOp(kp, kPrelu, t1, C);
    if (alpha < 0) continue;
    // ADD(u, shortcut), the shortcut a computed float tensor of y's shape; its activation applies
    const int t2 = nodes_[kp]->node.outputs->data[0];
    const size_t ka = SoleConsumer(t2);
    if (ka == kNoNode) continue;
    const NodeRecord& a = *nodes_[ka];
    if (a.name != kAdd || a.initialized || a.node.inputs->size != 2 || a.node.outputs->size != 1)
      continue;
    const int in0 = a.node.inputs->data[0], in1 = a.node.inputs->data[1];
    if (in0 == in1 || (in0 != t2 && in1 != t2)) continue;
    const int r = in0 == t2 ? in1 : in0;
    if (r < 0 || tensors_[r].type != kTfLiteFloat32 || tensors_[r].allocation_type == kTfLiteMmapRo ||
        !SameDims(tensors_[r].dims, yd) || !ReadyBefore(r, i))
      continue;
    const int o = a.node.outputs->data[0];
    if (tensors_[o].type != kTfLiteFloat32) continue;
    const int32_t add_act = Activation(a);
    std::vector<size_t> absorbed{km, kp, ka};
    // the next block's BatchNorm and sign: MUL(o, scale) -> ADD(shift) -> LceQuantize, when the
    // convolution is ungrouped (the fused sign-pack needs groups == 1)
    int sc = -1, sh = -1, packed = -1;
    const TfLiteIntArray* xs = tensors_[b.node.inputs->data[0]].dims;
    const TfLiteIntArray* fs = tensors_[b.node.inputs->data[1]].dims;
    const bool ungrouped = xs && fs && xs->size == 4 && fs->size == 4 && xs->data[3] == fs->data[3];
    for (size_t c : Consumers(o)) {
      if (!ungrouped) break;
      const int v1 = PerChannelConstOp(c, kMul, o, C);
      if (v1 < 0) continue;
      const int t3 = nodes_[c]->node.outputs->data[0];
      const size_t k2 = SoleConsumer(t3);
      const int v2 = PerChannelConstOp(k2, kAdd, t3, C);
      if (v2 < 0) continue;
      const size_t kq = SoleConsumer(nodes_[k2]->node.outputs->data[0]);
      if (!IsQuantize(kq)) continue;
      sc = v1; sh = v2; packed = nodes_[kq]->node.outputs->data[0];
      absorbed.insert(absorbed.end(), {c, k2, kq});
      break;
    }
    std::vector<int> ins = Ints(b.node.inputs);
    ins.insert(ins.end(), {r, g, alpha, sc, sh});
    std::vector<int> outs{o};
    if (packed >= 0) outs.push_back(packed);
    SetNodeIO(b, ins, outs);
    b.registration = gate_reg;
    SetBuiltinBlob(b, &add_act, sizeof(add_act));
    b.name = packed >= 0 ? "LceBconv2d+MUL+PRELU+ADD+MUL+ADD+LceQuantize" : "LceBconv2d+MUL+PRELU+ADD";
    removed += static_cast<int>(absorbed.size());
    EraseNodes(absorbed);   // all after node i
  }
  allocated_ = false;
  return removed;
}

extern "C" TfLiteRegistration* lce_b200_internal_Register_BCONV_2D_SCALE(const TfLiteRegistration* original);

int Graph::FuseSpatialScales() {
  if (!device_arena_) return 0;
  int removed = 0;
  for (size_t i = 0; i < nodes_.size(); ++i) {
    NodeRecord& b = *nodes_[i];
    if (b.name != "LceBconv2d" || b.initialized || b.node.inputs->size != 5 || b.node.outputs->size != 1)
      continue;
    TfLiteRegistration* scale_reg = lce_b200_internal_Register_BCONV_2D_SCALE(b.registration);
    if (scale_reg == nullptr) continue;
    const int y = b.node.outputs->data[0];
    const TfLiteIntArray* yd = tensors_[y].dims;
    if (tensors_[y].type != kTfLiteFloat32 || !yd || yd->size != 4) continue;
    const int C = yd->data[3];
    // MUL(y, gamma): gamma a float constant [1, OH, OW, C] or [OH, OW, C], no fused activation
    const size_t km = SoleConsumer(y);
    if (km == kNoNode) continue;
    const NodeRecord& m = *nodes_[km];
    if (m.name != kMul || m.initialized || m.node.inputs->size != 2 || m.node.outputs->size != 1 ||
        m.node.inputs->data[0] != y || tensors_[m.node.outputs->data[0]].type != kTfLiteFloat32 ||
        !Params(m) || Activation(m) != 0)
      continue;
    const int gamma = m.node.inputs->data[1];
    if (gamma < 0 || gamma == y) continue;
    const TfLiteTensor& gt = tensors_[gamma];
    const TfLiteIntArray* gd = gt.dims;
    if (gt.type != kTfLiteFloat32 || gt.allocation_type != kTfLiteMmapRo || !gd ||
        !(gd->size == 3 || (gd->size == 4 && gd->data[0] == 1)))
      continue;
    const int lead = gd->size - 3;
    if (gd->data[lead] != yd->data[1] || gd->data[lead + 1] != yd->data[2] || gd->data[lead + 2] != C)
      continue;
    // ADD(t, shortcut), the shortcut a computed float tensor of y's shape; its activation applies
    const int t1 = m.node.outputs->data[0];
    const size_t ka = SoleConsumer(t1);
    if (ka == kNoNode) continue;
    const NodeRecord& a = *nodes_[ka];
    if (a.name != kAdd || a.initialized || a.node.inputs->size != 2 || a.node.outputs->size != 1)
      continue;
    const int in0 = a.node.inputs->data[0], in1 = a.node.inputs->data[1];
    if (in0 == in1 || (in0 != t1 && in1 != t1)) continue;
    const int r = in0 == t1 ? in1 : in0;
    if (r < 0 || tensors_[r].type != kTfLiteFloat32 || tensors_[r].allocation_type == kTfLiteMmapRo ||
        !SameDims(tensors_[r].dims, yd) || !ReadyBefore(r, i))
      continue;
    const int o = a.node.outputs->data[0];
    if (tensors_[o].type != kTfLiteFloat32) continue;
    const int32_t add_act = Activation(a);
    std::vector<size_t> absorbed{km, ka};
    // the next block's BatchNorm and sign: MUL(o, scale) -> ADD(shift) -> LceQuantize, when the
    // convolution is ungrouped (the fused sign-pack needs groups == 1); o may have other readers
    int sc = -1, sh = -1, packed = -1;
    const TfLiteIntArray* xs = tensors_[b.node.inputs->data[0]].dims;
    const TfLiteIntArray* fs = tensors_[b.node.inputs->data[1]].dims;
    const bool ungrouped = xs && fs && xs->size == 4 && fs->size == 4 && xs->data[3] == fs->data[3];
    for (size_t c : Consumers(o)) {
      if (!ungrouped) break;
      const int v1 = PerChannelConstOp(c, kMul, o, C);
      if (v1 < 0) continue;
      const int t3 = nodes_[c]->node.outputs->data[0];
      const size_t k2 = SoleConsumer(t3);
      const int v2 = PerChannelConstOp(k2, kAdd, t3, C);
      if (v2 < 0) continue;
      const size_t kq = SoleConsumer(nodes_[k2]->node.outputs->data[0]);
      if (!IsQuantize(kq)) continue;
      sc = v1; sh = v2; packed = nodes_[kq]->node.outputs->data[0];
      absorbed.insert(absorbed.end(), {c, k2, kq});
      break;
    }
    std::vector<int> ins = Ints(b.node.inputs);
    ins.insert(ins.end(), {r, gamma, sc, sh});
    std::vector<int> outs{o};
    if (packed >= 0) outs.push_back(packed);
    SetNodeIO(b, ins, outs);
    b.registration = scale_reg;
    SetBuiltinBlob(b, &add_act, sizeof(add_act));
    b.name = packed >= 0 ? "LceBconv2d+MUL+ADD+MUL+ADD+LceQuantize" : "LceBconv2d+MUL+ADD";
    removed += static_cast<int>(absorbed.size());
    EraseNodes(absorbed);   // all after node i
  }
  allocated_ = false;
  return removed;
}

extern "C" TfLiteRegistration* lce_b200_internal_Register_BCONV_2D_DENSE(const TfLiteRegistration* original);
extern "C" int lce_b200_internal_slice_takes(const lce_bconv2d_desc* d);   // lce_b200.cu

int Graph::FuseDenseBlocks() {
  if (!device_arena_) return 0;
  auto dims4 = [&](int t) {
    const TfLiteIntArray* d = tensors_[t].dims;
    return d && d->size == 4 ? d : nullptr;
  };
  auto producer = [&](int t) {
    for (size_t k = 0; k < nodes_.size(); ++k)
      for (int q = 0; q < nodes_[k]->node.outputs->size; ++q)
        if (nodes_[k]->node.outputs->data[q] == t) return k;
    return kNoNode;
  };
  // node k is a STRIDED_SLICE of x [B,H,W,C] (through the builtin's own normalisation) to the
  // channels [lo, hi), the other axes whole, with a float output read once and not a graph output
  auto channel_slice = [&](size_t k, int x, const TfLiteIntArray* xd, int lo, int hi) {
    if (k >= nodes_.size()) return false;
    const NodeRecord& n = *nodes_[k];
    if (n.name != kStridedSlice || n.initialized || !Params(n) || n.node.inputs->size != 4 ||
        n.node.outputs->size != 1 || n.node.inputs->data[0] != x)
      return false;
    const int32_t* v[3];
    for (int q = 0; q < 3; ++q) {
      const int t = n.node.inputs->data[1 + q];
      if (t < 0 || tensors_[t].type != kTfLiteInt32 || tensors_[t].allocation_type != kTfLiteMmapRo ||
          !tensors_[t].data.raw || tensors_[t].dims->size != 1 ||
          tensors_[t].dims->data[0] != tensors_[n.node.inputs->data[1]].dims->data[0])
        return false;
      v[q] = tensors_[t].data.i32;
    }
    SliceBounds sb;
    if (StridedSliceBounds(xd->data, 4, v[0], v[1], v[2], tensors_[n.node.inputs->data[1]].dims->data[0],
                           *Params(n), &sb) != nullptr)
      return false;
    for (int d = 0; d < 3; ++d)
      if (sb.begin[d] != 0 || sb.end[d] != xd->data[d]) return false;
    const int out = n.node.outputs->data[0];
    return sb.begin[3] == lo && sb.end[3] == hi && tensors_[out].type == kTfLiteFloat32 &&
           SoleConsumer(out) != kNoNode;
  };
  // One layer read from the MUL at node i: x -> MUL(scale) -> ADD(shift) -> LceQuantize ->
  // LceBconv2d (float y, one that run_slice takes, same image size), then either
  //   dense: CONCATENATION([x, y], last axis) = out, or
  //   improvement: ADD(b, y) or ADD(y, b) with no activation = sum and CONCATENATION([a, sum], last
  //   axis) = out, a and b the STRIDED_SLICEs x[..., :C - C_out] and x[..., C - C_out:],
  // every intermediate read once and not a graph output.
  struct Layer {
    int kind;   // DensePrepare's layer kind: 0 dense, 1 improvement
    size_t mul, add, quant, conv, cat, sum, slice_a, slice_b;
    int x, scale, shift, packed, out, c_out;
    const TfLiteRegistration* reg;
    std::vector<size_t> x_readers;   // the layer's nodes that read x, in graph order
  };
  auto match = [&](size_t i, Layer* L) {
    const NodeRecord& m = *nodes_[i];
    if (m.name != kMul || m.node.inputs->size != 2) return false;
    const int x = m.node.inputs->data[0];
    const TfLiteIntArray* xd = x >= 0 && tensors_[x].type == kTfLiteFloat32 ? dims4(x) : nullptr;
    if (!xd || xd->data[3] % 4 != 0) return false;
    const int C = xd->data[3];
    L->mul = i; L->x = x;
    L->scale = PerChannelConstOp(i, kMul, x, C);
    if (L->scale < 0) return false;
    const int t1 = m.node.outputs->data[0];
    L->add = SoleConsumer(t1);
    L->shift = PerChannelConstOp(L->add, kAdd, t1, C);
    if (L->shift < 0) return false;
    L->quant = SoleConsumer(nodes_[L->add]->node.outputs->data[0]);
    if (!IsQuantize(L->quant)) return false;
    L->packed = nodes_[L->quant]->node.outputs->data[0];
    L->conv = SoleConsumer(L->packed);
    if (L->conv == kNoNode) return false;
    const NodeRecord& b = *nodes_[L->conv];
    if (b.name != "LceBconv2d" || b.initialized || b.node.inputs->size != 5 || b.node.outputs->size != 1 ||
        b.node.inputs->data[0] != L->packed)
      return false;
    L->reg = lce_b200_internal_Register_BCONV_2D_DENSE(b.registration);
    if (L->reg == nullptr) return false;   // a foreign "LceBconv2d" (e.g. the CPU test double)
    const int y = b.node.outputs->data[0];
    const TfLiteIntArray* yd = tensors_[y].type == kTfLiteFloat32 ? dims4(y) : nullptr;
    const TfLiteIntArray* pd = dims4(L->packed);
    const TfLiteIntArray* fd = dims4(b.node.inputs->data[1]);
    if (!yd || !pd || !fd || yd->data[0] != xd->data[0] || yd->data[1] != xd->data[1] ||
        yd->data[2] != xd->data[2])
      return false;
    FlexMap opts(b.custom_options.data(), b.custom_options.size());
    lce_bconv2d_desc d{};
    d.batch = xd->data[0]; d.in_h = xd->data[1]; d.in_w = xd->data[2];
    d.channels_in = opts.AsInt32("channels_in");
    d.channels_out = fd->data[0];
    d.groups = fd->data[3] == (d.channels_in + 31) / 32 && pd->data[3] == fd->data[3] ? 1 : 0;
    d.out_type = LCE_OUT_FLOAT;
    if (d.channels_in != C || d.groups != 1 || yd->data[3] != d.channels_out ||
        !lce_b200_internal_slice_takes(&d))
      return false;
    L->c_out = d.channels_out;
    const size_t next = SoleConsumer(y);
    if (next == kNoNode) return false;
    std::vector<int> cat_ins{x, y};
    int c_cat = C + d.channels_out;
    L->kind = nodes_[next]->name == kConcatenation ? 0 : 1;
    if (L->kind == 0) {
      L->cat = next;
      L->x_readers = {L->mul, L->cat};
    } else {
      // the improvement layer's tail
      L->sum = next;
      const NodeRecord& a = *nodes_[L->sum];
      if (a.name != kAdd || a.initialized || a.node.inputs->size != 2 || a.node.outputs->size != 1 ||
          !Params(a) || Params(a)->activation != 0 || d.channels_out > C)
        return false;
      const int bt = a.node.inputs->data[a.node.inputs->data[0] == y ? 1 : 0];
      const int sum = a.node.outputs->data[0];
      const TfLiteIntArray* sd = tensors_[sum].type == kTfLiteFloat32 ? dims4(sum) : nullptr;
      if (bt < 0 || bt == y || !sd || sd->data[3] != d.channels_out) return false;
      L->slice_b = producer(bt);
      if (!channel_slice(L->slice_b, x, xd, C - d.channels_out, C)) return false;
      L->cat = SoleConsumer(sum);
      if (L->cat == kNoNode || nodes_[L->cat]->node.inputs->size != 2) return false;
      const int at = nodes_[L->cat]->node.inputs->data[0];
      L->slice_a = at >= 0 ? producer(at) : kNoNode;
      if (!channel_slice(L->slice_a, x, xd, 0, C - d.channels_out) || L->slice_b >= L->sum ||
          L->slice_a >= L->cat || L->conv >= L->sum || L->sum >= L->cat)
        return false;
      cat_ins = {at, sum};
      c_cat = C;
      L->x_readers = {L->mul, L->slice_a, L->slice_b};
      std::sort(L->x_readers.begin(), L->x_readers.end());
    }
    const NodeRecord& c = *nodes_[L->cat];
    if (c.name != kConcatenation || c.initialized || c.node.inputs->size != 2 || c.node.outputs->size != 1 ||
        c.node.inputs->data[0] != cat_ins[0] || c.node.inputs->data[1] != cat_ins[1] || !Params(c) ||
        Params(c)->activation != 0 || (Params(c)->axis != 3 && Params(c)->axis != -1))
      return false;
    L->out = c.node.outputs->data[0];
    const TfLiteIntArray* od = tensors_[L->out].type == kTfLiteFloat32 ? dims4(L->out) : nullptr;
    return od && od->data[0] == xd->data[0] && od->data[1] == xd->data[1] && od->data[2] == xd->data[2] &&
           od->data[3] == c_cat && i < L->add && L->add < L->quant && L->quant < L->conv &&
           L->conv < L->cat;
  };
  int removed = 0;
  for (size_t i = 0; i < nodes_.size(); ++i) {
    Layer first;
    if (nodes_[i]->initialized || !match(i, &first)) continue;
    // the block: each map x_j (j >= 1) read only by the next layer's nodes (a dense layer's MUL and
    // CONCATENATION, an improvement layer's MUL and two STRIDED_SLICEs)
    std::vector<Layer> block{first};
    for (;;) {
      const int xj = block.back().out;
      if (IsGraphOutput(xj)) break;
      const std::vector<size_t> readers = Consumers(xj);
      Layer next;
      bool found = false;
      for (size_t r : readers)
        if (match(r, &next) && next.x == xj && next.x_readers == readers) {
          found = true;
          break;
        }
      if (!found) break;
      block.push_back(next);
    }
    const int X = block.back().out;
    const int c_total = tensors_[X].dims->data[3];
    std::vector<size_t> absorbed;
    for (size_t j = 0; j < block.size(); ++j) {
      const Layer& L = block[j];
      const TfLiteIntArray* pd = tensors_[L.packed].dims;
      const std::string tmp_name = names_[L.packed];   // AddTensor appends to names_
      std::vector<int> tmps{AddTensor(kTfLiteInt32, std::vector<int>(pd->data, pd->data + 4), nullptr, 0,
                                      false, 0.f, 0, tmp_name)};
      if (L.kind == 1) {
        // the convolution's own output when a CORRECTION plan needs it (DensePrepare sizes it)
        const TfLiteIntArray* xd = tensors_[L.x].dims;
        const std::string y_name = names_[nodes_[L.conv]->node.outputs->data[0]];
        tmps.push_back(AddTensor(kTfLiteFloat32, {xd->data[0], xd->data[1], xd->data[2], L.c_out}, nullptr,
                                 0, false, 0.f, 0, y_name));
      }
      NodeRecord& conv = *nodes_[L.conv];
      NodeRecord& n = *nodes_[L.mul];
      std::vector<int> ins{j == 0 ? L.x : X, L.scale, L.shift};
      ins.insert(ins.end(), conv.node.inputs->data + 1, conv.node.inputs->data + 5);
      SetNodeIO(n, ins, {X}, tmps);
      SetCustomOptions(n, conv.custom_options);
      const int32_t blob[2] = {c_total, L.kind};   // DensePrepare
      SetBuiltinBlob(n, blob, sizeof(blob));
      n.registration = L.reg;
      if (L.kind == 0) {
        n.name = "MUL+ADD+LceQuantize+LceBconv2d+CONCATENATION";
        absorbed.insert(absorbed.end(), {L.add, L.quant, L.conv, L.cat});
      } else {
        n.name = "MUL+ADD+LceQuantize+LceBconv2d+STRIDED_SLICE+ADD+CONCATENATION";
        absorbed.insert(absorbed.end(), {L.add, L.quant, L.conv, L.slice_a, L.slice_b, L.sum, L.cat});
      }
    }
    // a first improvement layer's slices may precede its MUL, and node i moves back by their number
    const size_t before_i = std::count_if(absorbed.begin(), absorbed.end(), [&](size_t k) { return k < i; });
    removed += static_cast<int>(absorbed.size());
    EraseNodes(absorbed);
    i -= before_i;
  }
  allocated_ = false;
  return removed;
}

const TfLiteRegistration* FusedPoolDepthwiseRegistration();  // builtin_ops.cc
const TfLiteRegistration* FusedStemRegistration();
const TfLiteRegistration* ActivationChainRegistration();
const TfLiteRegistration* PooledSignRegistration();
const TfLiteRegistration* Quant2Registration();
const TfLiteRegistration* GroupedConvAffineRegistration();

int Graph::FuseActivationChains() {
  if (!device_arena_) return 0;
  int removed = 0;
  for (size_t i = 0; i < nodes_.size(); ++i) {
    NodeRecord& a = *nodes_[i];
    if (a.initialized) continue;
    // after a fused residual block the chain starts on the sum; elsewhere node i is its first op
    const bool after_bconv = a.name == "LceBconv2d+ADD" && a.node.inputs->size == 6 &&
                             a.node.outputs->size == 1;
    if (!after_bconv && a.name != kAdd && a.name != kPrelu) continue;
    int cur = after_bconv ? a.node.outputs->data[0] : a.node.inputs->data[0];
    if (cur < 0 || tensors_[cur].type != kTfLiteFloat32 || tensors_[cur].dims->size < 1) continue;
    const int C = tensors_[cur].dims->data[tensors_[cur].dims->size - 1];
    std::vector<size_t> absorbed;
    int vec[4] = {-1, -1, -1, -1};   // shift_in, alpha, shift_out, sign_shift
    size_t k = after_bconv ? SoleConsumer(cur) : i;
    // RPReLU: ADD? -> PRELU? -> ADD?; an ADD read only by an LceQuantize is the RSign's instead
    const char* steps[3] = {kAdd, kPrelu, kAdd};
    for (int s = 0; s < 3 && k < nodes_.size(); ++s) {
      const int v = PerChannelConstOp(k, steps[s], cur, C);
      if (v < 0 || (s != 1 && IsQuantize(SoleConsumer(nodes_[k]->node.outputs->data[0])))) continue;
      vec[s] = v;
      absorbed.push_back(k);
      cur = nodes_[k]->node.outputs->data[0];
      k = SoleConsumer(cur);
    }
    const bool any_float = !absorbed.empty();
    // RSign of the next binary layer: [ADD(sign_shift) ->] LceQuantize of the chain's result
    int packed = -1;
    for (size_t c : Consumers(cur)) {
      if (!any_float && !after_bconv && c != i) continue;   // stand-alone: node i must start it
      if (IsQuantize(c)) {
        packed = nodes_[c]->node.outputs->data[0];
        absorbed.push_back(c);
        break;
      }
      const int v = PerChannelConstOp(c, kAdd, cur, C);
      const size_t q = v >= 0 ? SoleConsumer(nodes_[c]->node.outputs->data[0]) : kNoNode;
      if (IsQuantize(q)) {
        vec[3] = v;
        packed = nodes_[q]->node.outputs->data[0];
        absorbed.push_back(c);
        absorbed.push_back(q);
        break;
      }
    }
    // a stand-alone chain must replace at least two nodes (node i is one of them)
    if (absorbed.size() < (after_bconv ? 1u : 2u)) continue;
    std::string name;
    if (vec[0] >= 0 && vec[1] >= 0 && vec[2] >= 0) {
      name = "+RPReLU";
    } else {
      if (vec[0] >= 0) name += "+ADD";
      if (vec[1] >= 0) name += "+PRELU";
      if (vec[2] >= 0) name += "+ADD";
    }
    if (packed >= 0) name += vec[3] >= 0 ? "+ADD+LceQuantize" : "+LceQuantize";
    // the float result stays a tensor when something else reads it; a stand-alone chain without
    // float steps would only copy its input
    const std::vector<size_t> readers = Consumers(cur);
    const bool keep_out = after_bconv || (any_float && (IsGraphOutput(cur) ||
                                                        readers.size() > (packed >= 0 ? 1u : 0u)));
    std::vector<int> ins, outs{keep_out ? cur : -1};
    if (packed >= 0) outs.push_back(packed);
    if (after_bconv) {
      ins = Ints(a.node.inputs);
      a.name += name;
    } else {
      ins.push_back(a.node.inputs->data[0]);
      a.registration = ActivationChainRegistration();
      a.name = name.substr(1);
    }
    ins.insert(ins.end(), vec, vec + 4);
    SetNodeIO(a, ins, outs);
    // node i, when the chain starts on it, is the node just rewritten; the others are all after it
    absorbed.erase(std::remove(absorbed.begin(), absorbed.end(), i), absorbed.end());
    removed += static_cast<int>(absorbed.size());
    EraseNodes(absorbed);
  }
  allocated_ = false;
  return removed;
}

int Graph::FusePooledSigns() {
  if (!device_arena_) return 0;
  int removed = 0;
  for (size_t i = 0; i < nodes_.size(); ++i) {
    NodeRecord& p = *nodes_[i];
    if (p.name != kMaxPool2d || p.initialized || p.node.inputs->size != 1 || p.node.outputs->size != 1 ||
        !Params(p))
      continue;
    const int x = p.node.inputs->data[0], y = p.node.outputs->data[0];
    const TfLiteIntArray* xd = tensors_[x].dims;
    if (tensors_[x].type != kTfLiteFloat32 || tensors_[y].type != kTfLiteFloat32 || !xd || xd->size != 4)
      continue;
    const int C = xd->data[3];
    const size_t km = SoleConsumer(y);
    const int scale = PerChannelConstOp(km, kMul, y, C);
    if (scale < 0 || km <= i) continue;
    const int t1 = nodes_[km]->node.outputs->data[0];
    const size_t ka = SoleConsumer(t1);
    const int shift = PerChannelConstOp(ka, kAdd, t1, C);
    if (shift < 0 || ka <= km) continue;
    // larq's Flatten -> QuantDense: ADD -> RESHAPE [B, OH * OW * C] -> LceQuantize. With C % 32 == 0 the
    // flattened map packs to the map's own words, so the node writes them as [B, OH * OW * C / 32].
    const int t2 = nodes_[ka]->node.outputs->data[0];
    size_t kq = SoleConsumer(t2), kr = kNoNode;
    if (kq != kNoNode && nodes_[kq]->name == kReshape && !nodes_[kq]->initialized && C % 32 == 0 &&
        nodes_[kq]->node.inputs->size >= 1 && nodes_[kq]->node.inputs->data[0] == t2 &&
        nodes_[kq]->node.outputs->size == 1) {
      const int r = nodes_[kq]->node.outputs->data[0];
      const TfLiteIntArray* yd = tensors_[y].dims;
      const TfLiteIntArray* rd = tensors_[r].dims;
      if (tensors_[r].type == kTfLiteFloat32 && yd && yd->size == 4 && rd && rd->size == 2 &&
          rd->data[0] == yd->data[0] &&
          static_cast<int64_t>(rd->data[1]) == static_cast<int64_t>(yd->data[1]) * yd->data[2] * yd->data[3]) {
        kr = kq;
        kq = SoleConsumer(r);
      }
    }
    if (!IsQuantize(kq) || kq <= (kr != kNoNode ? kr : ka)) continue;
    SetNodeIO(p, {x, scale, shift}, {nodes_[kq]->node.outputs->data[0]});
    p.registration = PooledSignRegistration();   // builtin_data stays the pool's parameters
    p.name = kr != kNoNode ? "MAX_POOL_2D+MUL+ADD+RESHAPE+LceQuantize" : "MAX_POOL_2D+MUL+ADD+LceQuantize";
    std::vector<size_t> gone{km, ka, kq};
    if (kr != kNoNode) gone.push_back(kr);
    EraseNodes(gone);
    removed += static_cast<int>(gone.size());
  }
  allocated_ = false;
  return removed;
}

extern "C" TfLiteRegistration* lce_b200_internal_Register_BCONV_2D_BASES(const TfLiteRegistration* original);
extern "C" TfLiteRegistration* lce_b200_internal_Register_SHIFT_SIGN_PLANES(void);
extern "C" int lce_b200_internal_bases_takes(const lce_bconv2d_desc* d, int m_bases, int n_planes);   // lce_b200.cu

int Graph::FuseBinaryBases() {
  if (!device_arena_) return 0;
  constexpr int kMax = 8;   // bases, planes and next planes per node (lce::kMaxBases)
  auto producer = [&](int t) -> size_t {
    for (size_t k = 0; k < nodes_.size(); ++k)
      for (int q = 0; q < nodes_[k]->node.outputs->size; ++q)
        if (nodes_[k]->node.outputs->data[q] == t) return k;
    return kNoNode;
  };
  auto is_const = [&](int t, TfLiteType type) {
    return t >= 0 && tensors_[t].type == type && tensors_[t].allocation_type == kTfLiteMmapRo;
  };
  // node k = ADD(x, u), u a one-element float constant, no fused activation, whose output only an
  // LceQuantize reads: that LceQuantize (and *shift = u), else kNoNode
  auto shift_sign = [&](size_t k, int x, float* shift) -> size_t {
    if (k >= nodes_.size()) return kNoNode;
    const NodeRecord& a = *nodes_[k];
    if (a.name != kAdd || a.initialized || a.node.inputs->size != 2 || a.node.outputs->size != 1 ||
        a.node.inputs->data[0] != x || !Params(a) || Activation(a) != 0)
      return kNoNode;
    const int u = a.node.inputs->data[1];
    if (!is_const(u, kTfLiteFloat32) || tensors_[u].bytes != sizeof(float)) return kNoNode;
    const size_t q = SoleConsumer(a.node.outputs->data[0]);
    if (!IsQuantize(q)) return kNoNode;
    memcpy(shift, const_host_[u].data(), sizeof(float));
    return q;
  };
  // an unprepared plain LceBconv2d of this library with float output and constant inputs
  auto plain_term = [&](size_t k) {
    if (k >= nodes_.size()) return false;
    const NodeRecord& b = *nodes_[k];
    if (b.name != "LceBconv2d" || b.initialized || b.node.inputs->size != 5 || b.node.outputs->size != 1 ||
        tensors_[b.node.outputs->data[0]].type != kTfLiteFloat32 ||
        lce_b200_internal_Register_BCONV_2D_BASES(b.registration) == nullptr)
      return false;
    const int* in = b.node.inputs->data;
    return is_const(in[1], kTfLiteInt32) && is_const(in[2], kTfLiteFloat32) && is_const(in[3], kTfLiteFloat32);
  };
  int removed = 0;
  for (size_t i = 0; i < nodes_.size(); ++i) {
    if (!plain_term(i)) continue;
    // the sum ADD(...ADD(ADD(t_0, t_1), t_2)..., t_{K-1}), every intermediate read by the next ADD alone
    std::vector<size_t> terms{i}, absorbed;
    int cur = nodes_[i]->node.outputs->data[0];
    for (;;) {
      const size_t a = SoleConsumer(cur);
      if (a >= nodes_.size()) break;
      const NodeRecord& an = *nodes_[a];
      if (an.name != kAdd || an.initialized || an.node.inputs->size != 2 || an.node.outputs->size != 1 ||
          an.node.inputs->data[0] != cur || !Params(an) || Activation(an) != 0 ||
          tensors_[an.node.outputs->data[0]].type != kTfLiteFloat32)
        break;
      const int t = an.node.inputs->data[1];
      const size_t tk = producer(t);
      if (!plain_term(tk) || SoleConsumer(t) != a) break;
      terms.push_back(tk);
      absorbed.push_back(a);
      cur = an.node.outputs->data[0];
    }
    const int K = static_cast<int>(terms.size());
    if (K < 2) continue;   // a single LceBconv2d is never a bases layer
    const TfLiteIntArray* yd = tensors_[cur].dims;
    if (!yd || yd->size != 4) continue;
    const int C = yd->data[3];
    // the BatchNorm MUL(bn_scale) -> ADD(bn_shift, any activation)
    const size_t km = SoleConsumer(cur);
    const int bn_s = PerChannelConstOp(km, kMul, cur, C);
    if (bn_s < 0) continue;
    const int t1 = nodes_[km]->node.outputs->data[0];
    const size_t kb = SoleConsumer(t1);
    const int bn_t = PerChannelConstOp(kb, kAdd, t1, C, true);
    if (bn_t < 0) continue;
    // the planes: term k reads plane k / M, and each plane is read by its M terms alone
    std::vector<int> planes;
    for (size_t k : terms) {
      const int q = nodes_[k]->node.inputs->data[0];
      if (std::find(planes.begin(), planes.end(), q) == planes.end()) planes.push_back(q);
    }
    const int N = static_cast<int>(planes.size());
    if (K % N != 0 || N > kMax || K / N > kMax) continue;
    const int M = K / N;
    bool ok = true;
    for (int k = 0; k < K && ok; ++k) ok = nodes_[terms[k]]->node.inputs->data[0] == planes[k / M];
    for (int n = 0; n < N && ok; ++n)
      ok = !IsGraphOutput(planes[n]) && static_cast<int>(Consumers(planes[n]).size()) == M &&
           SameDims(tensors_[planes[n]].dims, tensors_[planes[0]].dims);
    // identical geometry (options and filter shape); term (n, m) convolves with base m's filter
    const NodeRecord& t0 = *nodes_[terms[0]];
    for (int k = 1; k < K && ok; ++k) {
      const NodeRecord& tk = *nodes_[terms[k]];
      const int fk = tk.node.inputs->data[1], fm = nodes_[terms[k % M]]->node.inputs->data[1];
      ok = tk.custom_options == t0.custom_options &&
           SameDims(tensors_[fk].dims, tensors_[t0.node.inputs->data[1]].dims) &&
           (fk == fm || const_host_[fk] == const_host_[fm]);
    }
    if (!ok) continue;
    const TfLiteIntArray* xd = tensors_[planes[0]].dims;
    const TfLiteIntArray* fd = tensors_[t0.node.inputs->data[1]].dims;
    if (!xd || !fd || xd->size != 4 || fd->size != 4) continue;
    FlexMap opts(t0.custom_options.data(), t0.custom_options.size());
    lce_bconv2d_desc d{};
    d.batch = xd->data[0]; d.in_h = xd->data[1]; d.in_w = xd->data[2];
    d.channels_in = opts.AsInt32("channels_in");
    d.channels_out = fd->data[0]; d.filter_h = fd->data[1]; d.filter_w = fd->data[2];
    d.groups = fd->data[3] == (d.channels_in + 31) / 32 && xd->data[3] == fd->data[3] ? 1 : 0;
    d.stride_h = opts.AsInt32("stride_height"); d.stride_w = opts.AsInt32("stride_width");
    d.dilation_h = opts.AsInt32("dilation_height_factor");
    d.dilation_w = opts.AsInt32("dilation_width_factor");
    d.padding = opts.AsInt32("padding"); d.pad_value = opts.AsInt32("pad_values");
    d.activation = opts.AsInt32("fused_activation_function");
    d.out_type = LCE_OUT_FLOAT;
    if (d.channels_out != C || !lce_b200_internal_bases_takes(&d, M, N)) continue;
    // where the planes come from: N pairs ADD(x, u_n) -> LceQuantize of one x, turned into one planes
    // node below, or the outputs of one earlier fused node that already writes them
    std::vector<size_t> pairs;   // shift ADD, LceQuantize of each plane
    std::vector<float> in_shifts;
    int x = -1;
    for (int n = 0; n < N && ok; ++n) {
      const size_t kq = producer(planes[n]);
      const size_t ks = kq < nodes_.size() && IsQuantize(kq) ? producer(nodes_[kq]->node.inputs->data[0]) : kNoNode;
      float u = 0.f;
      if (ks < nodes_.size() && nodes_[ks]->node.inputs->size == 2) {
        if (x < 0) x = nodes_[ks]->node.inputs->data[0];
        ok = shift_sign(ks, x, &u) == kq;
        pairs.insert(pairs.end(), {ks, kq});
        in_shifts.push_back(u);
      } else {
        ok = false;
      }
    }
    if (!ok) {
      // already fused: every plane is an output of the same earlier node that writes shifted signs
      const size_t kp = producer(planes[0]);
      ok = kp < nodes_.size() && (nodes_[kp]->name == "LceBconv2dBases+LceQuantize" ||
                                  nodes_[kp]->name == "ADD+LceQuantize");
      for (int n = 1; n < N && ok; ++n) ok = producer(planes[n]) == kp;
      if (!ok) continue;
      pairs.clear();
    } else {
      // the planes node reads x [.., channels_in]
      const TfLiteIntArray* xs = tensors_[x].dims;
      if (tensors_[x].type != kTfLiteFloat32 || !xs || xs->size != 4 || xs->data[3] != d.channels_in) continue;
    }
    // the optional shortcut ADD(o, r, any activation), r computed, of o's shape
    int o = nodes_[kb]->node.outputs->data[0];
    size_t last = kb;
    int r = -1;
    int32_t add_act = 0;
    const size_t ka = SoleConsumer(o);
    if (ka < nodes_.size()) {
      const NodeRecord& a = *nodes_[ka];
      if (a.name == kAdd && !a.initialized && a.node.inputs->size == 2 && a.node.outputs->size == 1 && Params(a) &&
          tensors_[a.node.outputs->data[0]].type == kTfLiteFloat32) {
        const int in0 = a.node.inputs->data[0], in1 = a.node.inputs->data[1];
        const int rr = in0 == o ? in1 : in0;
        if (in0 != in1 && rr >= 0 && tensors_[rr].type == kTfLiteFloat32 &&
            tensors_[rr].allocation_type != kTfLiteMmapRo && SameDims(tensors_[rr].dims, yd) && ReadyBefore(rr, i)) {
          r = rr;
          add_act = Activation(a);
          absorbed.push_back(kb);
          last = ka;
          o = a.node.outputs->data[0];
        }
      }
    }
    // the next layer's shifted signs among o's readers; o itself is stored when anything else reads it
    std::vector<int> next;
    std::vector<float> next_shifts;
    size_t others = 0;
    for (size_t c : Consumers(o)) {
      float u = 0.f;
      const size_t q = next.size() < kMax ? shift_sign(c, o, &u) : kNoNode;
      if (q == kNoNode) {
        ++others;
        continue;
      }
      next.push_back(nodes_[q]->node.outputs->data[0]);
      next_shifts.push_back(u);
      absorbed.insert(absorbed.end(), {c, q});
    }
    const int32_t store = IsGraphOutput(o) || others > 0 || next.empty();
    // rewrite: node `last` becomes the layer, the first shift ADD the planes node
    std::vector<int> ins(planes);
    for (size_t k : terms) {
      const int* in = nodes_[k]->node.inputs->data;
      ins.insert(ins.end(), {in[1], in[2], in[3]});
    }
    ins.insert(ins.end(), {bn_s, bn_t, r});
    std::vector<int> outs;
    if (store) outs.push_back(o);
    outs.insert(outs.end(), next.begin(), next.end());
    std::vector<uint8_t> blob(6 * sizeof(int32_t) + next_shifts.size() * sizeof(float));
    const int32_t head[6] = {M, N, static_cast<int32_t>(next.size()), Activation(*nodes_[kb]), add_act, store};
    memcpy(blob.data(), head, sizeof(head));
    if (!next_shifts.empty()) memcpy(blob.data() + sizeof(head), next_shifts.data(), next_shifts.size() * sizeof(float));
    std::vector<uint8_t> options = t0.custom_options;
    NodeRecord& f = *nodes_[last];
    f.registration = lce_b200_internal_Register_BCONV_2D_BASES(t0.registration);
    SetCustomOptions(f, std::move(options));
    SetNodeIO(f, ins, outs);
    SetBuiltinBlob(f, blob.data(), blob.size());
    f.name = next.empty() ? "LceBconv2dBases" : "LceBconv2dBases+LceQuantize";
    absorbed.insert(absorbed.end(), terms.begin(), terms.end());
    absorbed.push_back(km);
    if (!pairs.empty()) {
      NodeRecord& pn = *nodes_[pairs[0]];   // the first shift ADD: x exists there
      std::vector<uint8_t> pblob(sizeof(int32_t) + in_shifts.size() * sizeof(float));
      const int32_t n32 = N;
      memcpy(pblob.data(), &n32, sizeof(n32));
      memcpy(pblob.data() + sizeof(n32), in_shifts.data(), in_shifts.size() * sizeof(float));
      pn.registration = lce_b200_internal_Register_SHIFT_SIGN_PLANES();
      SetNodeIO(pn, {x}, planes);
      SetBuiltinBlob(pn, pblob.data(), pblob.size());
      pn.name = "ADD+LceQuantize";
      absorbed.insert(absorbed.end(), pairs.begin() + 1, pairs.end());
    }
    removed += static_cast<int>(absorbed.size());
    EraseNodes(absorbed);
    i = SIZE_MAX;   // indices moved: scan again from the start
  }
  allocated_ = false;
  return removed;
}

int Graph::FuseQuantizedActivations() {
  // the host copy of a float constant, else nullptr (data.raw may be its device copy)
  auto float_const = [&](int t) -> const float* {
    if (t < 0 || tensors_[t].type != kTfLiteFloat32 || tensors_[t].allocation_type != kTfLiteMmapRo)
      return nullptr;
    return reinterpret_cast<const float*>(const_host_[t].data());
  };
  auto count = [&](int t) {
    int64_t n = 1;
    for (int d = 0; d < tensors_[t].dims->size; ++d) n *= tensors_[t].dims->data[d];
    return n;
  };
  // node k (after node `after`) is the builtin `name` of x [and a one-element float constant equal to
  // `value`], with no fused activation and a float output: returns that output, else -1
  auto step = [&](size_t k, long long after, const char* name, int x, bool binary, float value) {
    if (k >= nodes_.size() || static_cast<long long>(k) <= after) return -1;
    const NodeRecord& n = *nodes_[k];
    if (n.name != name || n.initialized || n.node.inputs->size != (binary ? 2 : 1) ||
        n.node.outputs->size != 1 || n.node.inputs->data[0] != x || !Params(n) || Params(n)->activation != 0 ||
        tensors_[n.node.outputs->data[0]].type != kTfLiteFloat32)
      return -1;
    if (binary) {
      const int v = n.node.inputs->data[1];
      const float* c = float_const(v);
      if (!c || count(v) != 1 || memcmp(c, &value, sizeof(float)) != 0) return -1;
    }
    return n.node.outputs->data[0];
  };
  // One consumer of the quantised tensor: CONV_2D or FULLY_CONNECTED with constant +-alpha weights.
  struct Layer {
    size_t node;
    int N, kh, kw;
    BuiltinParams p;
    std::vector<int32_t> filter;
    std::vector<float> mul, bias;
  };
  // fills `l` when node k qualifies (see host_graph.h)
  auto layer = [&](size_t k, size_t after, int t, int C, Layer* l) {
    if (k >= nodes_.size() || k <= after) return false;
    const NodeRecord& n = *nodes_[k];
    const bool fc = n.name == kFullyConnected;
    if ((!fc && n.name != kConv2d) || n.initialized || !Params(n) || Params(n)->activation != 0 ||
        n.node.inputs->size < 2 || n.node.inputs->size > 3 || n.node.outputs->size != 1 ||
        n.node.inputs->data[0] != t || tensors_[n.node.outputs->data[0]].type != kTfLiteFloat32)
      return false;
    const int wt = n.node.inputs->data[1], bt = n.node.inputs->size > 2 ? n.node.inputs->data[2] : -1;
    const float* w = float_const(wt);
    const float* b = bt < 0 ? nullptr : float_const(bt);
    if (!w || (bt >= 0 && !b)) return false;
    const TfLiteIntArray* wd = tensors_[wt].dims;
    if (wd->size != (fc ? 2 : 4) || wd->data[wd->size - 1] != C) return false;
    // a FULLY_CONNECTED output becomes [rows,1,1,N]: the same bytes, but not the shape a caller reads
    if (fc && IsGraphOutput(n.node.outputs->data[0])) return false;
    l->node = k;
    l->N = wd->data[0];
    l->kh = fc ? 1 : wd->data[1];
    l->kw = fc ? 1 : wd->data[2];
    l->p = *Params(n);
    if (fc) {
      l->p.padding = LCE_PADDING_VALID;
      l->p.stride_h = l->p.stride_w = l->p.dilation_h = l->p.dilation_w = 1;
    }
    const int64_t taps = static_cast<int64_t>(l->kh) * l->kw, K = taps * C;
    if (l->N < 1 || taps < 1 || 3 * K >= (1 << 24) || (b && count(bt) != l->N)) return false;
    lce_bconv2d_desc d{};
    d.batch = d.in_h = d.in_w = 1;
    d.channels_in = 3 * C; d.channels_out = l->N; d.groups = 1;
    d.filter_h = l->kh; d.filter_w = l->kw;
    d.stride_h = l->p.stride_h; d.stride_w = l->p.stride_w;
    d.dilation_h = l->p.dilation_h; d.dilation_w = l->p.dilation_w;
    d.padding = l->p.padding; d.pad_value = 1; d.out_type = LCE_OUT_FLOAT;
    int oh, ow, ph, pw;
    if (lce_b200_bconv2d_out_shape(&d, &oh, &ow, &ph, &pw) != 0) return false;
    const int cw = C / 32;
    l->filter.assign(static_cast<size_t>(l->N) * taps * 3 * cw, 0);
    l->mul.resize(l->N);
    l->bias.resize(l->N);
    for (int o = 0; o < l->N; ++o) {
      const float* wo = w + static_cast<int64_t>(o) * K;
      uint32_t mag;
      memcpy(&mag, wo, 4);
      mag &= 0x7fffffffu;
      if (mag == 0 || mag >= 0x7f800000u) return false;
      int64_t sum = 0;   // W_o: the sum of the filter's signs
      for (int64_t tap = 0; tap < taps; ++tap)
        for (int c = 0; c < C; ++c) {
          uint32_t bits;
          memcpy(&bits, wo + tap * C + c, 4);
          if ((bits & 0x7fffffffu) != mag) return false;
          const bool neg = bits >> 31;
          sum += neg ? -1 : 1;
          if (neg)
            for (int plane = 0; plane < 3; ++plane)
              l->filter[((static_cast<size_t>(o) * taps + tap) * 3 + plane) * cw + c / 32] |=
                  static_cast<int32_t>(1u << (c % 32));
        }
      float alpha_f;
      memcpy(&alpha_f, &mag, 4);
      const double alpha = alpha_f;
      l->mul[o] = static_cast<float>(-alpha / 6.0);
      l->bias[o] = static_cast<float>(alpha * static_cast<double>(sum) / 2.0 + (b ? static_cast<double>(b[o]) : 0.0));
    }
    return true;
  };

  int removed = 0;
  for (size_t i = 0; i < nodes_.size(); ++i) {
    if (nodes_[i]->name != kMaximum || nodes_[i]->node.inputs->size != 2) continue;
    const int x = nodes_[i]->node.inputs->data[0];
    if (x < 0 || tensors_[x].type != kTfLiteFloat32 || !tensors_[x].dims || tensors_[x].dims->size < 1) continue;
    const int C = tensors_[x].dims->data[tensors_[x].dims->size - 1];
    if (C <= 0 || C % 32 != 0) continue;
    const int t1 = step(i, -1, kMaximum, x, true, 0.0f);
    if (t1 < 0) continue;
    const size_t kmin = SoleConsumer(t1);
    const int t2 = step(kmin, i, kMinimum, t1, true, 1.0f);
    if (t2 < 0) continue;
    const size_t kmul = SoleConsumer(t2);
    const int t3 = step(kmul, kmin, kMul, t2, true, 3.0f);
    if (t3 < 0) continue;
    const size_t kround = SoleConsumer(t3);
    const int t4 = step(kround, kmul, kRound, t3, false, 0.0f);
    if (t4 < 0) continue;
    const size_t kdiv = SoleConsumer(t4);
    const int t5 = step(kdiv, kround, kDiv, t4, true, 3.0f);
    if (t5 < 0 || IsGraphOutput(t5)) continue;
    const std::vector<size_t> users = Consumers(t5);
    if (users.empty()) continue;
    std::vector<Layer> layers(users.size());
    bool ok = true;
    for (size_t u = 0; u < users.size() && ok; ++u) ok = layer(users[u], kdiv, t5, C, &layers[u]);
    if (!ok) continue;
    // the optional pool in front: x is read by the quantiser only
    size_t head = i;
    int src = x;
    if (SoleConsumer(x) == i && tensors_[x].dims->size == 4)
      for (size_t k = 0; k < i; ++k) {
        const NodeRecord& p = *nodes_[k];
        if (p.name == kMaxPool2d && !p.initialized && Params(p) && p.node.inputs->size == 1 &&
            p.node.outputs->size == 1 && p.node.outputs->data[0] == x &&
            tensors_[p.node.inputs->data[0]].type == kTfLiteFloat32) {
          head = k;
          src = p.node.inputs->data[0];
        }
      }
    const std::vector<int> xdims = Ints(tensors_[x].dims);
    std::vector<int> pdims = xdims.size() == 4 ? xdims : std::vector<int>{static_cast<int>(count(x) / C), 1, 1, C};
    pdims[3] = 3 * (C / 32);
    const int planes = AddTensor(kTfLiteInt32, pdims, nullptr, 0, false, 0.0f, 0, names_[t5] + "_planes");
    NodeRecord& h = *nodes_[head];
    if (head == i) {   // no pool: filter_h == 0 tells the node so
      BuiltinParams bp;
      memset(&bp, 0, sizeof(bp));
      SetBuiltinBlob(h, &bp, sizeof(bp));
    }
    SetNodeIO(h, {src}, {planes});
    h.registration = Quant2Registration();
    h.name = head == i ? "Quant2" : "MAX_POOL_2D+Quant2";
    for (const Layer& l : layers) {
      const int f = AddTensor(kTfLiteInt32, {l.N, l.kh, l.kw, 3 * (C / 32)}, l.filter.data(),
                              l.filter.size() * sizeof(int32_t), false, 0.0f, 0, names_[t5] + "_bfilter");
      const int m = AddTensor(kTfLiteFloat32, {l.N}, l.mul.data(), l.mul.size() * sizeof(float), false, 0.0f, 0,
                              names_[t5] + "_pmul");
      const int b = AddTensor(kTfLiteFloat32, {l.N}, l.bias.data(), l.bias.size() * sizeof(float), false, 0.0f, 0,
                              names_[t5] + "_pbias");
      NodeRecord& n = *nodes_[l.node];
      SetNodeIO(n, {planes, f, m, b, -1}, {n.node.outputs->data[0]});
      SetCustomOptions(n, WriteFlexIntMap({{"channels_in", 3 * C},
                                           {"dilation_height_factor", l.p.dilation_h},
                                           {"dilation_width_factor", l.p.dilation_w},
                                           {"fused_activation_function", 0},
                                           {"pad_values", 1},
                                           {"padding", l.p.padding},
                                           {"stride_height", l.p.stride_h},
                                           {"stride_width", l.p.stride_w}}));
      SetBuiltinBlob(n, nullptr, 0);
      n.registration = lce_b200_Register_BCONV_2D();
      n.name = "LceBconv2d";
    }
    std::vector<size_t> gone{kmin, kmul, kround, kdiv};
    if (head != i) gone.push_back(i);
    removed += static_cast<int>(gone.size());
    EraseNodes(gone);
    i = head;
  }
  allocated_ = false;
  return removed;
}

int Graph::FuseGroupedConvAffine() {
  int removed = 0;
  for (size_t i = 0; i < nodes_.size(); ++i) {
    NodeRecord& conv = *nodes_[i];
    if (conv.name != kConv2d || conv.initialized || !Params(conv) || Params(conv)->activation != 0 ||
        conv.node.inputs->size < 2 || conv.node.inputs->size > 3 || conv.node.outputs->size != 1)
      continue;
    const int x = conv.node.inputs->data[0], w = conv.node.inputs->data[1];
    const int y = conv.node.outputs->data[0];
    if (x < 0 || w < 0 || tensors_[x].dims->size != 4 || tensors_[w].dims->size != 4 ||
        tensors_[x].type != kTfLiteFloat32 || tensors_[y].type != kTfLiteFloat32)
      continue;
    // grouped only: TFLite's groups = C_in / filter_in, exact, and dividing C_out
    const int cin = tensors_[x].dims->data[3], fin = tensors_[w].dims->data[3], C = tensors_[w].dims->data[0];
    if (fin < 1 || fin == cin || cin % fin != 0 || C % (cin / fin) != 0) continue;
    // the fused node takes over y and the MUL's output as the first operand alone
    const size_t km = SoleReaderAsFirstInput(y);
    const int scale = PerChannelConstOp(km, kMul, y, C);
    if (scale < 0 || km <= i) continue;
    const int u = nodes_[km]->node.outputs->data[0];
    const size_t ka = SoleReaderAsFirstInput(u);
    const int shift = PerChannelConstOp(ka, kAdd, u, C, /*any_activation=*/true);
    if (shift < 0 || ka <= km) continue;
    const BuiltinParams two[2] = {*Params(conv), *Params(*nodes_[ka])};
    SetNodeIO(conv, {x, w, conv.node.inputs->size > 2 ? conv.node.inputs->data[2] : -1, scale, shift},
              {nodes_[ka]->node.outputs->data[0]});
    SetBuiltinBlob(conv, two, sizeof(two));
    conv.registration = GroupedConvAffineRegistration();
    conv.name = "CONV_2D+MUL+ADD";
    EraseNodes({km, ka});
    removed += 2;
  }
  allocated_ = false;
  return removed;
}

// [DEQUANTIZE ->] CONV_2D(3x3, stride 2, 3 -> 16 or 8) -> DEPTHWISE_CONV_2D(3x3, stride 2,
// multiplier 1), each intermediate consumed once: one node (the stem of QuickNet and QuickNetLarge,
// 16, and of QuickNetSmall, 8). The image is read once, as the bytes the host shipped; the
// dequantised image and the first conv's map never reach HBM.
int Graph::FuseStem() {
  auto dims4 = [&](int t, int d) { return tensors_[t].dims->size == 4 ? tensors_[t].dims->data[d] : -1; };
  for (size_t i = 0; i < nodes_.size(); ++i) {
    NodeRecord& c1 = *nodes_[i];
    if (c1.name != kConv2d || c1.initialized || c1.node.inputs->size < 3 || !Params(c1)) continue;
    const BuiltinParams p1 = *Params(c1);
    const int w1 = c1.node.inputs->data[1];
    const int x = c1.node.inputs->data[0];
    const int c1_out = dims4(w1, 0);
    // dims4(x, 3) != 3: a grouped convolution's filter has fewer input channels than x
    if ((c1_out != 16 && c1_out != 8) || dims4(w1, 1) != 3 || dims4(w1, 2) != 3 || dims4(w1, 3) != 3 ||
        dims4(x, 3) != 3 || p1.stride_h != 2 || p1.stride_w != 2 || p1.dilation_h != 1 ||
        p1.dilation_w != 1 || tensors_[x].type != kTfLiteFloat32 ||
        tensors_[c1.node.outputs->data[0]].type != kTfLiteFloat32)
      continue;
    const size_t di = SoleReaderAsFirstInput(c1.node.outputs->data[0]);
    if (di == kNoNode || di <= i) continue;
    NodeRecord& dw = *nodes_[di];
    if (dw.name != kDepthwiseConv2d || dw.initialized || dw.node.inputs->size < 3 || !Params(dw)) continue;
    const BuiltinParams p2 = *Params(dw);
    const int w2 = dw.node.inputs->data[1];
    if (dims4(w2, 1) != 3 || dims4(w2, 2) != 3 || dims4(w2, 3) != c1_out || p2.stride_h != 2 ||
        p2.stride_w != 2 || p2.dilation_h != 1 || p2.dilation_w != 1 || p2.depth_multiplier != 1)
      continue;
    // the kernel takes the filters and biases by value: they must be constants
    bool consts = true;
    for (int t : {w1, c1.node.inputs->data[2], w2, dw.node.inputs->data[2]})
      if (t >= 0 && tensors_[t].allocation_type != kTfLiteMmapRo) consts = false;
    if (!consts) continue;
    // a DEQUANTIZE that feeds only this conv is folded in: the kernel reads the quantised image
    int src = x;
    size_t qi = kNoNode;
    for (size_t k = 0; k < i; ++k) {
      NodeRecord& dq = *nodes_[k];
      if (dq.name == kDequantize && !dq.initialized && dq.node.outputs->size == 1 &&
          dq.node.outputs->data[0] == x && dq.node.inputs->size == 1 && SoleReaderAsFirstInput(x) == i &&
          (tensors_[dq.node.inputs->data[0]].type == kTfLiteInt8 ||
           tensors_[dq.node.inputs->data[0]].type == kTfLiteUInt8)) {
        qi = k;
        src = dq.node.inputs->data[0];
      }
    }
    const BuiltinParams two[2] = {p1, p2};
    SetNodeIO(c1, {src, w1, c1.node.inputs->data[2], w2, dw.node.inputs->data[2]}, {dw.node.outputs->data[0]});
    SetBuiltinBlob(c1, two, sizeof(two));
    c1.registration = FusedStemRegistration();
    c1.name = qi != kNoNode ? "DEQUANTIZE+CONV_2D+DEPTHWISE_CONV_2D" : "CONV_2D+DEPTHWISE_CONV_2D";
    std::vector<size_t> absorbed{di};
    if (qi != kNoNode) absorbed.push_back(qi);
    EraseNodes(absorbed);
    return static_cast<int>(absorbed.size());
  }
  return 0;
}

extern "C" int lce_b200_internal_conv_packs_alike(int filter_h, int filter_w, int stride_h,
                                                  int stride_w, int in_c, int out_c);   // lce_b200_builtins.cu

// CONV_2D (float) whose output also feeds an LceQuantize: the conv emits the packed signs from its
// epilogue as a second output and the LceQuantize node disappears (first layer of every stage),
// where the signs leave the kernel that computes the floats unchanged.
int Graph::FuseConvQuantize() {
  int removed = 0;
  for (size_t i = 0; i < nodes_.size(); ++i) {
    NodeRecord& conv = *nodes_[i];
    if (conv.name != kConv2d || conv.initialized || conv.node.outputs->size != 1) continue;
    const int y = conv.node.outputs->data[0];
    if (tensors_[y].type != kTfLiteFloat32) continue;
    if (conv.node.inputs->size >= 2 && Params(conv)) {
      const TfLiteIntArray* fd = tensors_[conv.node.inputs->data[1]].dims;
      const TfLiteIntArray* xd = tensors_[conv.node.inputs->data[0]].dims;
      // a grouped convolution (filter_in != the input's channels) runs its own kernel, without signs
      if (fd && xd && fd->size == 4 && xd->size == 4 && fd->data[3] != xd->data[3]) continue;
      const BuiltinParams* bp = Params(conv);
      if (fd && fd->size == 4 &&
          !lce_b200_internal_conv_packs_alike(fd->data[1], fd->data[2], bp->stride_h, bp->stride_w,
                                              fd->data[3], fd->data[0]))
        continue;
    }
    for (size_t k = i + 1; k < nodes_.size(); ++k) {
      NodeRecord& q = *nodes_[k];
      if (q.name != "LceQuantize" || q.initialized || q.node.inputs->size != 1 ||
          q.node.inputs->data[0] != y || q.node.outputs->size != 1)
        continue;
      const int packed = q.node.outputs->data[0];
      if (tensors_[packed].type != kTfLiteInt32) break;
      SetNodeIO(conv, Ints(conv.node.inputs), {y, packed});
      conv.name = "CONV_2D+LceQuantize";
      EraseNode(k);
      ++removed;
      break;
    }
  }
  return removed;
}

int Graph::FuseFloatGlue() {
  if (!device_arena_) return 0;
  // LCE_B200_FUSE_STEM=0 / LCE_B200_FUSE_CONV_QUANT=0 switch the two fusions off (A/B runs)
  const char* stem_env = getenv("LCE_B200_FUSE_STEM");
  int removed = (stem_env && stem_env[0] == '0') ? 0 : FuseStem();
  // CONV_2D -> LceQuantize: the tensor-core pointwise kernel (lce_b200_pw.cuh) has the output row
  // in registers and emits the sign words for free; other shapes pack with the stand-alone kernel
  const char* cq_env = getenv("LCE_B200_FUSE_CONV_QUANT");
  if (!(cq_env && cq_env[0] == '0')) removed += FuseConvQuantize();
  // RELU -> MEAN (the model heads): the mean applies the activation as it reads
  for (size_t i = 0; i < nodes_.size(); ++i) {
    NodeRecord& relu = *nodes_[i];
    if (relu.name != kRelu || relu.initialized || relu.node.inputs->size != 1 || relu.node.outputs->size != 1)
      continue;
    const int y = relu.node.outputs->data[0];
    const size_t mi = SoleReaderAsFirstInput(y);
    if (mi == kNoNode || mi <= i) continue;
    NodeRecord& mean = *nodes_[mi];
    if (mean.name != kMean || mean.initialized || !Params(mean)) continue;
    BuiltinParams mp = *Params(mean);
    mp.activation = 1;   // kTfLiteActRelu
    SetBuiltinBlob(mean, &mp, sizeof(mp));
    mean.node.inputs->data[0] = relu.node.inputs->data[0];
    mean.name = "RELU+MEAN";
    EraseNode(i);
    ++removed;
    break;
  }
  for (size_t i = 0; i < nodes_.size(); ++i) {
    NodeRecord& pool = *nodes_[i];
    if (pool.name != kMaxPool2d || pool.initialized || !Params(pool)) continue;
    const BuiltinParams* pp = Params(pool);
    if (pp->filter_h != 2 || pp->filter_w != 2 || pp->stride_h != 1 || pp->stride_w != 1 ||
        pp->padding != 1 /* VALID */ || pp->activation != 0)
      continue;
    const int y = pool.node.outputs->data[0];
    const size_t di = SoleReaderAsFirstInput(y);
    if (di == kNoNode || di <= i) continue;
    NodeRecord& dw = *nodes_[di];
    if (dw.name != kDepthwiseConv2d || !Params(dw)) continue;
    const BuiltinParams* dp = Params(dw);
    const TfLiteTensor& f = tensors_[dw.node.inputs->data[1]];
    if (f.dims->size != 4 || f.dims->data[1] != 3 || f.dims->data[2] != 3 ||
        (f.dims->data[3] & 3) || dp->dilation_h != 1 || dp->dilation_w != 1 ||
        dp->depth_multiplier != 1 || tensors_[y].type != kTfLiteFloat32)
      continue;
    // rewrite the pool node into the fused node; it takes the depthwise node's constants / output
    const BuiltinParams two[2] = {*pp, *dp};
    SetNodeIO(pool, {pool.node.inputs->data[0], dw.node.inputs->data[1],
                     dw.node.inputs->size > 2 ? dw.node.inputs->data[2] : -1},
              {dw.node.outputs->data[0]});
    SetBuiltinBlob(pool, two, sizeof(two));
    pool.registration = FusedPoolDepthwiseRegistration();
    pool.name = "MAX_POOL_2D+DEPTHWISE_CONV_2D";
    EraseNode(di);
    ++removed;
  }
  allocated_ = false;
  return removed;
}

const TfLiteRegistration* UpsampleMergeRegistration();   // builtin_ops.cc

int Graph::FuseUpsampleMerges() {
  if (!device_arena_) return 0;
  auto fuse = [&](size_t i) -> int {   // nodes removed by fusing the resize at i, 0 when it stays
    NodeRecord& r = *nodes_[i];
    if (r.name != kResizeNearest || r.initialized || r.node.inputs->size != 2 || r.node.outputs->size != 1 ||
        !Params(r))
      return 0;
    const int u = r.node.inputs->data[0], size = r.node.inputs->data[1], v = r.node.outputs->data[0];
    if (u < 0 || size < 0 || tensors_[u].type != kTfLiteFloat32 || tensors_[v].type != kTfLiteFloat32) return 0;
    const TfLiteIntArray* vd = tensors_[v].dims;
    if (!vd || vd->size != 4) return 0;
    const size_t ai = SoleConsumer(v);
    if (ai == kNoNode || ai <= i) return 0;
    NodeRecord& a = *nodes_[ai];
    if (a.name != kAdd || a.initialized || a.node.inputs->size != 2 || a.node.outputs->size != 1 || !Params(a))
      return 0;
    const int in0 = a.node.inputs->data[0], in1 = a.node.inputs->data[1];
    if (in0 == in1) return 0;
    const int skip = in0 == v ? in1 : in0;
    if (skip < 0 || tensors_[skip].type != kTfLiteFloat32 || !SameDims(vd, tensors_[skip].dims)) return 0;
    const int s = a.node.outputs->data[0];
    if (tensors_[s].type != kTfLiteFloat32) return 0;
    // the sign tail: the sum's only LceQuantize reader, on whole 32-channel words
    const std::vector<size_t> readers = Consumers(s);
    size_t kq = kNoNode;
    int quantizers = 0;
    for (size_t k : readers)
      if (nodes_[k]->name == "LceQuantize") { ++quantizers; kq = k; }
    const bool tail = quantizers == 1 && IsQuantize(kq) && kq > ai && vd->data[3] % 32 == 0;
    const bool store = !tail || readers.size() > 1 || IsGraphOutput(s);
    std::vector<int> outs{store ? s : -1};
    if (tail) outs.push_back(nodes_[kq]->node.outputs->data[0]);
    const BuiltinParams two[2] = {*Params(r), *Params(a)};
    // the ADD's node becomes the merge: u and skip both exist where it runs
    SetNodeIO(a, {u, size, skip}, outs);
    SetBuiltinBlob(a, two, sizeof(two));
    a.registration = UpsampleMergeRegistration();
    a.name = tail ? "RESIZE_NEAREST_NEIGHBOR+ADD+LceQuantize" : "RESIZE_NEAREST_NEIGHBOR+ADD";
    if (tail) {
      EraseNodes({i, kq});
      return 2;
    }
    EraseNode(i);
    return 1;
  };
  int removed = 0;
  for (size_t i = 0; i < nodes_.size();) {
    const int k = fuse(i);
    removed += k;
    if (k == 0) ++i;   // else node i is erased and its successor moved up
  }
  allocated_ = false;
  return removed;
}

const TfLiteRegistration* ResizeArgmaxRegistration();   // builtin_ops.cc

int Graph::FuseResizeArgmax() {
  if (!device_arena_) return 0;
  auto fuse = [&](size_t i) -> bool {   // the resize at i is fused into its ARG_MAX and erased
    NodeRecord& r = *nodes_[i];
    if (r.name != kResizeBilinear || r.initialized || r.node.inputs->size != 2 || r.node.outputs->size != 1 ||
        !Params(r))
      return false;
    const int x = r.node.inputs->data[0], size = r.node.inputs->data[1], v = r.node.outputs->data[0];
    if (x < 0 || size < 0 || tensors_[x].type != kTfLiteFloat32 || tensors_[v].type != kTfLiteFloat32) return false;
    const TfLiteIntArray* xd = tensors_[x].dims;
    if (!xd || xd->size != 4 || !tensors_[v].dims || tensors_[v].dims->size != 4) return false;
    const size_t ai = SoleReaderAsFirstInput(v);
    if (ai == kNoNode || ai <= i) return false;
    NodeRecord& a = *nodes_[ai];
    if (a.name != kArgMax || a.initialized || a.node.inputs->size != 2 || a.node.outputs->size != 1 || !Params(a))
      return false;
    const int axis_t = a.node.inputs->data[1];
    int axis;
    if (axis_t < 0 || ArgMaxAxis(&tensors_[axis_t], 4, &axis) != nullptr || axis != 3) return false;
    if (static_cast<int64_t>(xd->data[2]) * xd->data[3] > lce_b200_resize_bilinear_argmax_max_row_floats())
      return false;
    const BuiltinParams two[2] = {*Params(r), *Params(a)};
    // the ARG_MAX's node becomes the fused one: x exists where it runs
    SetNodeIO(a, {x, size, axis_t}, Ints(a.node.outputs));
    SetBuiltinBlob(a, two, sizeof(two));
    a.registration = ResizeArgmaxRegistration();
    a.name = "RESIZE_BILINEAR+ARG_MAX";
    EraseNode(i);
    return true;
  };
  int removed = 0;
  for (size_t i = 0; i < nodes_.size();) {
    if (fuse(i)) ++removed;   // node i is erased and its successor moved up
    else ++i;
  }
  allocated_ = false;
  return removed;
}

const TfLiteRegistration* SubpixelConvRegistration();   // builtin_ops.cc
extern "C" int lce_b200_internal_conv_runs_igemm(int in_h, int in_w, int in_c, int filter_h, int filter_w,
                                                 int stride_h, int stride_w, int dilation_h, int dilation_w,
                                                 int out_c);   // lce_b200_builtins.cu

int Graph::FuseSubpixelConvs() {
  if (!device_arena_) return 0;
  auto is_const = [&](int t, TfLiteType type) {
    return t >= 0 && tensors_[t].type == type && tensors_[t].allocation_type == kTfLiteMmapRo;
  };
  auto Elements = [&](int t) {
    int64_t n = 1;
    for (int k = 0; tensors_[t].dims && k < tensors_[t].dims->size; ++k) n *= tensors_[t].dims->data[k];
    return n;
  };
  auto fuse = [&](size_t i) -> int {   // nodes removed by fusing the conv at i, 0 when it stays
    NodeRecord& cv = *nodes_[i];
    const BuiltinParams* cp = Params(cv);
    if (cv.name != kConv2d || cv.initialized || cv.node.inputs->size < 2 || cv.node.inputs->size > 3 ||
        cv.node.outputs->size != 1 || !cp)
      return 0;
    const int x = cv.node.inputs->data[0], f = cv.node.inputs->data[1], y = cv.node.outputs->data[0];
    const int bias = cv.node.inputs->size == 3 ? cv.node.inputs->data[2] : -1;
    if (x < 0 || tensors_[x].type != kTfLiteFloat32 || tensors_[y].type != kTfLiteFloat32) return 0;
    const TfLiteIntArray* xd = tensors_[x].dims;
    const TfLiteIntArray* fd = is_const(f, kTfLiteFloat32) ? tensors_[f].dims : nullptr;
    if (!xd || xd->size != 4 || !fd || fd->size != 4 || fd->data[1] != 3 || fd->data[2] != 3 ||
        fd->data[3] != xd->data[3])
      return 0;
    const int cin = xd->data[3], cout = fd->data[0];
    if (bias >= 0 && (!is_const(bias, kTfLiteFloat32) || Elements(bias) != cout)) return 0;
    if (cp->stride_h != 1 || cp->stride_w != 1 || cp->dilation_h != 1 || cp->dilation_w != 1 ||
        cp->padding != LCE_PADDING_SAME || cin % 4 != 0 || cout > lce_b200_subpixel_conv_max_out_channels() ||
        !lce_b200_internal_conv_runs_igemm(xd->data[1], xd->data[2], cin, 3, 3, 1, 1, 1, 1, cout))
      return 0;
    const size_t di = SoleReaderAsFirstInput(y);
    if (di == kNoNode || di <= i) return 0;
    NodeRecord& ds = *nodes_[di];
    if (ds.name != kDepthToSpace || ds.initialized || ds.node.inputs->size != 1 || ds.node.outputs->size != 1 ||
        !Params(ds))
      return 0;
    const int r = Params(ds)->block_size, s = ds.node.outputs->data[0];
    if (r < 2 || cout % (r * r) != 0 || tensors_[s].type != kTfLiteFloat32) return 0;
    BuiltinParams four[4] = {*cp, *Params(ds), {}, {}};
    // the residual: s's one reader an ADD whose other operand is a RESIZE_BILINEAR output of s's shape
    // that only the ADD reads, resized from a float32 4-D image by a constant size
    size_t ai = SoleConsumer(s), ri = kNoNode;
    int img = -1, size = -1;
    if (ai != kNoNode && ai > di) {
      NodeRecord& a = *nodes_[ai];
      const int in0 = a.node.inputs->size == 2 ? a.node.inputs->data[0] : -1;
      const int in1 = a.node.inputs->size == 2 ? a.node.inputs->data[1] : -1;
      const int v = in0 == s ? in1 : in0;
      if (a.name == kAdd && !a.initialized && a.node.outputs->size == 1 && Params(a) && in0 != in1 && v >= 0 &&
          tensors_[a.node.outputs->data[0]].type == kTfLiteFloat32 && tensors_[v].type == kTfLiteFloat32 &&
          SameDims(tensors_[v].dims, tensors_[s].dims) && tensors_[s].dims && tensors_[s].dims->size == 4 &&
          SoleConsumer(v) == ai) {
        for (size_t k = 0; k < ai && ri == kNoNode; ++k)
          if (nodes_[k]->node.outputs->size == 1 && nodes_[k]->node.outputs->data[0] == v) ri = k;
      }
      if (ri != kNoNode) {
        NodeRecord& rz = *nodes_[ri];
        img = rz.node.inputs->size == 2 ? rz.node.inputs->data[0] : -1;
        size = rz.node.inputs->size == 2 ? rz.node.inputs->data[1] : -1;
        if (rz.name != kResizeBilinear || rz.initialized || !Params(rz) || img < 0 ||
            tensors_[img].type != kTfLiteFloat32 || !tensors_[img].dims || tensors_[img].dims->size != 4 ||
            !is_const(size, kTfLiteInt32) || Elements(size) != 2)
          ri = kNoNode;
      }
    }
    std::vector<int> ins{x, f, bias};
    if (ri != kNoNode) {
      NodeRecord& a = *nodes_[ai];
      four[2] = *Params(*nodes_[ri]);
      four[3] = *Params(a);
      ins.push_back(img);
      ins.push_back(size);
      // the ADD's node becomes the fused one: x and img both exist where it runs
      SetNodeIO(a, ins, Ints(a.node.outputs));
      SetBuiltinBlob(a, four, sizeof(four));
      a.registration = SubpixelConvRegistration();
      a.name = "CONV_2D+DEPTH_TO_SPACE+RESIZE_BILINEAR+ADD";
      EraseNodes({i, di, ri});
      return 3;
    }
    SetNodeIO(ds, ins, {s});
    SetBuiltinBlob(ds, four, sizeof(four));
    ds.registration = SubpixelConvRegistration();
    ds.name = "CONV_2D+DEPTH_TO_SPACE";
    EraseNode(i);
    return 1;
  };
  int removed = 0;
  for (size_t i = 0; i < nodes_.size();) {
    const int k = fuse(i);
    removed += k;
    if (k == 0) ++i;   // else node i is erased and its successor moved up
  }
  allocated_ = false;
  return removed;
}

const TfLiteRegistration* BinaryTransposeConvRegistration();   // builtin_ops.cc
extern "C" int lce_b200_internal_shuffle_takes(const lce_bconv2d_desc* d, int s_h, int s_w);   // lce_b200.cu

int Graph::FuseBinaryTransposeConvs() {
  if (!device_arena_) return 0;
  auto fuse = [&](size_t i) -> int {   // nodes removed by fusing the TRANSPOSE_CONV at i, 0 when it stays
    NodeRecord& tc = *nodes_[i];
    const BuiltinParams* tp = Params(tc);
    if (tc.name != kTransposeConv || tc.initialized || !tp || tc.node.inputs->size < 3 || tc.node.inputs->size > 4 ||
        tc.node.outputs->size != 1)
      return 0;
    const int shape = tc.node.inputs->data[0], w = tc.node.inputs->data[1], x = tc.node.inputs->data[2];
    const int bias = tc.node.inputs->size == 4 ? tc.node.inputs->data[3] : -1, y = tc.node.outputs->data[0];
    const int sh = tp->stride_h, sw = tp->stride_w;
    if (shape < 0 || w < 0 || x < 0 || tensors_[shape].type != kTfLiteInt32 ||
        tensors_[shape].allocation_type != kTfLiteMmapRo || tensors_[w].type != kTfLiteFloat32 ||
        tensors_[w].allocation_type != kTfLiteMmapRo || tensors_[x].type != kTfLiteFloat32 ||
        tensors_[y].type != kTfLiteFloat32 || tp->activation < LCE_ACT_NONE || tp->activation > LCE_ACT_RELU6 ||
        sh <= 0 || sw <= 0 || sh * sw < 2)
      return 0;
    const TfLiteIntArray* wd = tensors_[w].dims;
    const TfLiteIntArray* xd = tensors_[x].dims;
    if (!wd || wd->size != 4 || !xd || xd->size != 4 || wd->data[1] != sh || wd->data[2] != sw ||
        wd->data[3] != xd->data[3] || const_host_[shape].size() < 4 * sizeof(int32_t) ||
        tensors_[shape].bytes != 4 * sizeof(int32_t))
      return 0;
    const int C = wd->data[0], cin = xd->data[3];
    // the output exactly in * s: no output_padding rows (which would hold the bias alone)
    int32_t os[4];
    memcpy(os, const_host_[shape].data(), sizeof(os));
    if (os[1] != static_cast<int64_t>(xd->data[1]) * sh || os[2] != static_cast<int64_t>(xd->data[2]) * sw ||
        os[3] != C)
      return 0;
    if (bias >= 0 && (tensors_[bias].type != kTfLiteFloat32 || tensors_[bias].allocation_type != kTfLiteMmapRo ||
                      !tensors_[bias].dims || tensors_[bias].dims->size != 1 || tensors_[bias].dims->data[0] != C))
      return 0;
    // every weight exactly +1.0f or -1.0f (not -0.0, not 0.5)
    const size_t nw = static_cast<size_t>(C) * sh * sw * cin;
    if (const_host_[w].size() < nw * sizeof(float)) return 0;
    std::vector<uint32_t> wb(nw);
    memcpy(wb.data(), const_host_[w].data(), nw * sizeof(float));
    for (uint32_t v : wb)
      if (v != 0x3f800000u && v != 0xbf800000u) return 0;
    lce_bconv2d_desc d;
    memset(&d, 0, sizeof(d));
    d.batch = xd->data[0]; d.in_h = xd->data[1]; d.in_w = xd->data[2]; d.channels_in = cin;
    d.filter_h = 1; d.filter_w = 1; d.channels_out = sh * sw * C; d.groups = 1;
    d.stride_h = 1; d.stride_w = 1; d.dilation_h = 1; d.dilation_w = 1;
    d.padding = LCE_PADDING_VALID; d.pad_value = 1; d.activation = LCE_ACT_NONE; d.out_type = LCE_OUT_FLOAT;
    if (!lce_b200_internal_shuffle_takes(&d, sh, sw)) return 0;   // C % 64 == 0, the b1 mma.sync kernel
    // x: an LceDequantize of packed signs q, read by the TRANSPOSE_CONV alone
    size_t di = kNoNode;
    for (size_t k = 0; k < i && di == kNoNode; ++k)
      if (nodes_[k]->node.outputs->size == 1 && nodes_[k]->node.outputs->data[0] == x) di = k;
    if (di == kNoNode || SoleConsumer(x) != i) return 0;
    const NodeRecord& dq = *nodes_[di];
    const int q = dq.node.inputs->size == 1 ? dq.node.inputs->data[0] : -1;
    if (dq.name != "LceDequantize" || dq.initialized || q < 0 || tensors_[q].type != kTfLiteInt32) return 0;
    // the ADD: y's one reader, the other operand of y's shape (no broadcast) and ready before it
    size_t ai = SoleConsumer(y);
    int skip = -1;
    if (ai != kNoNode) {
      const NodeRecord& a = *nodes_[ai];
      const int in0 = a.node.inputs->size == 2 ? a.node.inputs->data[0] : -1;
      const int in1 = a.node.inputs->size == 2 ? a.node.inputs->data[1] : -1;
      skip = in0 == y ? in1 : in0;
      if (ai <= i || a.name != kAdd || a.initialized || a.node.outputs->size != 1 || !Params(a) || in0 == in1 ||
          skip < 0 || tensors_[skip].type != kTfLiteFloat32 || tensors_[a.node.outputs->data[0]].type != kTfLiteFloat32 ||
          !SameDims(tensors_[skip].dims, tensors_[y].dims) || !ReadyBefore(skip, ai)) {
        ai = kNoNode;
        skip = -1;
      }
    }
    const int s = ai != kNoNode ? nodes_[ai]->node.outputs->data[0] : y;
    // the signs: the sum's only LceQuantize reader; the sum itself stays stored
    size_t kq = kNoNode;
    int quantizers = 0;
    for (size_t k : Consumers(s))
      if (nodes_[k]->name == "LceQuantize") { ++quantizers; kq = k; }
    const bool tail = quantizers == 1 && IsQuantize(kq) && kq > (ai != kNoNode ? ai : i);
    std::vector<int> outs{s};
    if (tail) outs.push_back(nodes_[kq]->node.outputs->data[0]);
    // the filter: each weight's sign bit, rows (i, j, c) of the 1x1 GEMM, ceil(Cin / 32) words per row
    const int cw = (cin + 31) / 32;
    std::vector<int32_t> filt(static_cast<size_t>(d.channels_out) * cw, 0);
    for (int c = 0; c < C; ++c)
      for (int fi = 0; fi < sh; ++fi)
        for (int fj = 0; fj < sw; ++fj) {
          const size_t src = ((static_cast<size_t>(c) * sh + fi) * sw + fj) * cin;
          int32_t* row = filt.data() + (static_cast<size_t>(fi * sw + fj) * C + c) * cw;
          for (int ci = 0; ci < cin; ++ci)
            if (wb[src + ci] >> 31) row[ci >> 5] |= static_cast<int32_t>(1u << (ci & 31));
        }
    const int ft = AddTensor(kTfLiteInt32, {d.channels_out, 1, 1, cw}, filt.data(), filt.size() * sizeof(int32_t),
                             false, 0.0f, 0, names_[w] + "_packed", /*const_on_device=*/true);
    struct {
      BuiltinParams tconv, add;
      int32_t channels_in;
    } params{*tp, ai != kNoNode ? *Params(*nodes_[ai]) : BuiltinParams{}, cin};
    // the ADD's node (or without it the TRANSPOSE_CONV's) becomes the fused one: q and the skip exist
    // where it runs, and every reader of the sum and of the signs comes after it
    NodeRecord& f = ai != kNoNode ? *nodes_[ai] : tc;
    SetNodeIO(f, {q, ft, bias, skip}, outs);
    SetBuiltinBlob(f, &params, sizeof(params));
    f.registration = BinaryTransposeConvRegistration();
    f.name = std::string("LceBconv2dTranspose") + (ai != kNoNode ? "+ADD" : "") + (tail ? "+LceQuantize" : "");
    std::vector<size_t> gone{di};
    if (ai != kNoNode) gone.push_back(i);
    if (tail) gone.push_back(kq);
    EraseNodes(gone);
    return static_cast<int>(gone.size());
  };
  int removed = 0;
  for (size_t i = 0; i < nodes_.size();) {
    const int k = fuse(i);
    removed += k;
    i = k > 0 ? 0 : i + 1;   // indices moved: scan again (a fused node no longer matches)
  }
  allocated_ = false;
  return removed;
}

const TfLiteRegistration* BinaryFullyConnectedRegistration();   // builtin_ops.cc
const TfLiteRegistration* BinaryFcMaxRegistration();            // builtin_ops.cc
extern "C" int lce_b200_internal_fc_takes(const lce_bconv2d_desc* d);   // lce_b200.cu
extern "C" int lce_b200_internal_fc_max_takes(const lce_bconv2d_desc* d, int points);   // lce_b200.cu

namespace {
lce_bconv2d_desc FcDesc(int64_t rows, int K, int N) {   // a binary dense layer's rows x 1 x 1 plan
  lce_bconv2d_desc d;
  memset(&d, 0, sizeof(d));
  d.batch = static_cast<int>(rows); d.in_h = 1; d.in_w = 1; d.channels_in = K;
  d.filter_h = 1; d.filter_w = 1; d.channels_out = N; d.groups = 1;
  d.stride_h = 1; d.stride_w = 1; d.dilation_h = 1; d.dilation_w = 1;
  d.padding = LCE_PADDING_VALID; d.pad_value = 1; d.activation = LCE_ACT_NONE; d.out_type = LCE_OUT_FLOAT;
  return d;
}
}  // namespace

bool Graph::MatchBinaryFc(size_t i, BinaryFcMatch* m) const {
  // a constant float32 [n] (exactly rank 1), or -1
  auto vec = [&](int t, int n) {
    return t >= 0 && tensors_[t].type == kTfLiteFloat32 && tensors_[t].allocation_type == kTfLiteMmapRo &&
                   tensors_[t].dims && tensors_[t].dims->size == 1 && tensors_[t].dims->data[0] == n
               ? t
               : -1;
  };
  if (i >= nodes_.size()) return false;
  const NodeRecord& fc = *nodes_[i];
  const BuiltinParams* fp = Params(fc);
  if (fc.name != kFullyConnected || fc.initialized || !fp || fc.node.inputs->size < 2 || fc.node.inputs->size > 3 ||
      fc.node.outputs->size != 1)
    return false;
  const int x = fc.node.inputs->data[0], w = fc.node.inputs->data[1], y = fc.node.outputs->data[0];
  const int bias_in = fc.node.inputs->size == 3 ? fc.node.inputs->data[2] : -1;
  if (x < 0 || w < 0 || tensors_[w].type != kTfLiteFloat32 || tensors_[w].allocation_type != kTfLiteMmapRo ||
      tensors_[x].type != kTfLiteFloat32 || tensors_[y].type != kTfLiteFloat32 || fp->activation < LCE_ACT_NONE ||
      fp->activation > LCE_ACT_RELU6)
    return false;
  const TfLiteIntArray* wd = tensors_[w].dims;
  const TfLiteIntArray* xd = tensors_[x].dims;
  if (!wd || wd->size != 2 || !xd || xd->size < 1 || wd->data[0] <= 0 || wd->data[1] <= 0) return false;
  const int N = wd->data[0], K = wd->data[1];
  const int bias = vec(bias_in, N);
  if (bias_in >= 0 && bias < 0) return false;
  // keep_num_dims keeps x's leading axes, so each row must be x's last axis
  if (fp->keep_dims != 0 && xd->data[xd->size - 1] != K) return false;
  // every row o exactly +-alpha_o: one positive, finite magnitude, bitwise, in the whole row (no 0.0 or
  // -0.0, no 0.5 among 1.0s)
  const size_t nw = static_cast<size_t>(N) * K;
  if (const_host_[w].size() < nw * sizeof(float)) return false;
  m->wb.resize(nw);
  memcpy(m->wb.data(), const_host_[w].data(), nw * sizeof(float));
  m->alpha.assign(N, 0.0f);
  m->unit = true;
  for (int o = 0; o < N; ++o) {
    const uint32_t mag = m->wb[static_cast<size_t>(o) * K] & 0x7fffffffu;
    if (mag == 0 || mag >= 0x7f800000u) return false;
    for (int k = 1; k < K; ++k)
      if ((m->wb[static_cast<size_t>(o) * K + k] & 0x7fffffffu) != mag) return false;
    memcpy(&m->alpha[o], &mag, sizeof(float));
    m->unit = m->unit && mag == 0x3f800000u;
  }
  // x: an LceDequantize of packed signs q, read by the FULLY_CONNECTED alone
  size_t di = kNoNode;
  for (size_t k = 0; k < i && di == kNoNode; ++k)
    if (nodes_[k]->node.outputs->size == 1 && nodes_[k]->node.outputs->data[0] == x) di = k;
  if (di == kNoNode || SoleConsumer(x) != i) return false;
  const NodeRecord& dq = *nodes_[di];
  const int q = dq.node.inputs->size == 1 ? dq.node.inputs->data[0] : -1;
  if (dq.name != "LceDequantize" || dq.initialized || q < 0 || tensors_[q].type != kTfLiteInt32) return false;
  // q's words are the rows' words: each row is x's last axis (any K), or whole words of a map whose
  // last axis packs without a padded word (C % 32 == 0, K % 32 == 0)
  const TfLiteIntArray* qd = tensors_[q].dims;
  const int last = xd->data[xd->size - 1];
  if (!qd || qd->size != xd->size || qd->data[qd->size - 1] != (last + 31) / 32) return false;
  for (int k = 0; k + 1 < xd->size; ++k)
    if (qd->data[k] != xd->data[k]) return false;
  if (last != K && (last % 32 != 0 || K % 32 != 0)) return false;
  int64_t elems = 1;
  for (int k = 0; k < xd->size; ++k) elems *= xd->data[k];
  if (elems % K != 0 || elems / K > INT32_MAX) return false;
  m->rows = elems / K;
  const lce_bconv2d_desc d = FcDesc(m->rows, K, N);
  if (!lce_b200_internal_fc_takes(&d)) return false;   // N % 64 == 0, the b1 mma.sync kernel
  // the BatchNorm: MUL(scale [N]) as y's one reader, then ADD(shift [N]) as the product's one reader
  size_t km = SoleConsumer(y), ka = kNoNode;
  int scale = vec(PerChannelConstOp(km, kMul, y, N), N), shift = -1;
  if (scale >= 0 && km > i) {
    const int t1 = nodes_[km]->node.outputs->data[0];
    ka = SoleConsumer(t1);
    shift = vec(PerChannelConstOp(ka, kAdd, t1, N, /*any_activation=*/true), N);
    if (shift < 0 || ka <= km || Activation(*nodes_[ka]) < LCE_ACT_NONE || Activation(*nodes_[ka]) > LCE_ACT_RELU6)
      ka = kNoNode;
  }
  if (ka == kNoNode) {
    km = kNoNode;
    scale = shift = -1;
  }
  m->fc = i; m->dq = di; m->km = km; m->ka = ka;
  m->q = q; m->w = w; m->K = K; m->N = N; m->bias = bias; m->scale = scale; m->shift = shift;
  m->result = ka != kNoNode ? nodes_[ka]->node.outputs->data[0] : y;
  return true;
}

void Graph::BinaryFcConstants(const BinaryFcMatch& m, int* filter, int* alpha) {
  // the filter: each weight's sign bit, ceil(K / 32) words per output row
  const int N = m.N, K = m.K, cw = (K + 31) / 32;
  std::vector<int32_t> filt(static_cast<size_t>(N) * cw, 0);
  for (int o = 0; o < N; ++o)
    for (int k = 0; k < K; ++k)
      if (m.wb[static_cast<size_t>(o) * K + k] >> 31) filt[static_cast<size_t>(o) * cw + (k >> 5)] |= static_cast<int32_t>(1u << (k & 31));
  const std::string name = names_[m.w];
  *filter = AddTensor(kTfLiteInt32, {N, 1, 1, cw}, filt.data(), filt.size() * sizeof(int32_t), false, 0.0f, 0,
                      name + "_packed", /*const_on_device=*/true);
  // alpha = 1.0 everywhere multiplies by nothing: the node reads no vector for it
  *alpha = m.unit ? -1
                  : AddTensor(kTfLiteFloat32, {N}, m.alpha.data(), m.alpha.size() * sizeof(float), false, 0.0f, 0,
                              name + "_alpha", /*const_on_device=*/true);
}

int Graph::FuseBinaryFullyConnected() {
  if (!device_arena_) return 0;
  auto fuse = [&](size_t i) -> int {   // nodes removed by fusing the FULLY_CONNECTED at i, 0 when it stays
    BinaryFcMatch m;
    if (!MatchBinaryFc(i, &m)) return 0;
    // the signs: the result's only LceQuantize reader; the result itself stays stored
    size_t kq = kNoNode;
    int quantizers = 0;
    for (size_t k : Consumers(m.result))
      if (nodes_[k]->name == "LceQuantize") { ++quantizers; kq = k; }
    const bool tail = quantizers == 1 && IsQuantize(kq) && kq > (m.ka != kNoNode ? m.ka : i);
    std::vector<int> outs{m.result};
    if (tail) outs.push_back(nodes_[kq]->node.outputs->data[0]);
    int ft, at;
    BinaryFcConstants(m, &ft, &at);
    struct {
      BuiltinParams fc, add;
      int32_t channels_in;
    } params{*Params(*nodes_[i]), m.ka != kNoNode ? *Params(*nodes_[m.ka]) : BuiltinParams{}, m.K};
    // the ADD's node (or without it the FULLY_CONNECTED's) becomes the fused one: q exists where it runs,
    // and every reader of the result and of the signs comes after it
    NodeRecord& f = m.ka != kNoNode ? *nodes_[m.ka] : *nodes_[i];
    SetNodeIO(f, {m.q, ft, at, m.bias, m.scale, m.shift}, outs);
    SetBuiltinBlob(f, &params, sizeof(params));
    f.registration = BinaryFullyConnectedRegistration();
    f.name = std::string("LceBfc") + (m.ka != kNoNode ? "+MUL+ADD" : "") + (tail ? "+LceQuantize" : "");
    std::vector<size_t> gone{m.dq};
    if (m.ka != kNoNode) {
      gone.push_back(i);
      gone.push_back(m.km);
    }
    if (tail) gone.push_back(kq);
    EraseNodes(gone);
    return static_cast<int>(gone.size());
  };
  int removed = 0;
  for (size_t i = 0; i < nodes_.size();) {
    const int k = fuse(i);
    removed += k;
    i = k > 0 ? 0 : i + 1;   // indices moved: scan again (a fused node no longer matches)
  }
  allocated_ = false;
  return removed;
}

int Graph::FuseBinaryFcMax() {
  if (!device_arena_) return 0;
  auto fuse = [&](size_t i) -> int {   // nodes removed by fusing the FULLY_CONNECTED at i, 0 when it stays
    BinaryFcMatch m;
    if (!MatchBinaryFc(i, &m)) return 0;
    // the layer's result: [B, P, N], read by a REDUCE_MAX over axis 1 alone and not a graph output
    const TfLiteIntArray* rd = tensors_[m.result].dims;
    const size_t kr = SoleConsumer(m.result);
    if (!rd || rd->size != 3 || rd->data[2] != m.N || rd->data[1] <= 0 || kr >= nodes_.size() ||
        kr <= (m.ka != kNoNode ? m.ka : i))
      return 0;
    const NodeRecord& r = *nodes_[kr];
    if (r.name != kReduceMax || r.initialized || !Params(r) || r.node.inputs->size != 2 || r.node.outputs->size != 1 ||
        r.node.inputs->data[0] != m.result)
      return 0;
    const int axes = r.node.inputs->data[1], mx = r.node.outputs->data[0];
    if (axes < 0 || tensors_[axes].type != kTfLiteInt32 || tensors_[axes].allocation_type != kTfLiteMmapRo ||
        tensors_[mx].type != kTfLiteFloat32)
      return 0;
    const TfLiteIntArray* ad = tensors_[axes].dims;
    int64_t na = 1;
    for (int k = 0; ad && k < ad->size; ++k) na *= ad->data[k];
    if (!ad || ad->size > 1 || const_host_[axes].size() < static_cast<size_t>(na) * sizeof(int32_t)) return 0;
    std::vector<int32_t> av(static_cast<size_t>(na));
    memcpy(av.data(), const_host_[axes].data(), av.size() * sizeof(int32_t));
    if (av.empty()) return 0;
    for (int32_t a : av)   // exactly the point axis (duplicates allowed)
      if (a != 1 && a != -2) return 0;
    const int points = rd->data[1];
    const lce_bconv2d_desc d = FcDesc(m.rows, m.K, m.N);
    if (m.rows != static_cast<int64_t>(rd->data[0]) * points || !lce_b200_internal_fc_max_takes(&d, points)) return 0;
    // the signs: the max's only LceQuantize reader; the floats are stored only when something else reads them
    size_t kq = kNoNode;
    int quantizers = 0;
    const std::vector<size_t> readers = Consumers(mx);
    for (size_t k : readers)
      if (nodes_[k]->name == "LceQuantize") { ++quantizers; kq = k; }
    const bool tail = quantizers == 1 && IsQuantize(kq) && kq > kr;
    const bool store = !tail || readers.size() > 1 || IsGraphOutput(mx);
    std::vector<int> outs;
    if (store) outs.push_back(mx);
    if (tail) outs.push_back(nodes_[kq]->node.outputs->data[0]);
    int ft, at;
    BinaryFcConstants(m, &ft, &at);
    BinaryFcMaxParams params{*Params(*nodes_[i]), m.ka != kNoNode ? *Params(*nodes_[m.ka]) : BuiltinParams{},
                             *Params(r), m.K, points, store ? 1 : 0, tail ? 1 : 0};
    // the REDUCE_MAX's node becomes the fused one: q exists where it runs, and every reader of the max
    // and of its signs comes after it
    NodeRecord& f = *nodes_[kr];
    SetNodeIO(f, {m.q, ft, at, m.bias, m.scale, m.shift}, outs);
    SetBuiltinBlob(f, &params, sizeof(params));
    f.registration = BinaryFcMaxRegistration();
    f.name = std::string("LceBfc") + (m.ka != kNoNode ? "+MUL+ADD" : "") + "+REDUCE_MAX" + (tail ? "+LceQuantize" : "");
    std::vector<size_t> gone{m.dq, i};
    if (m.ka != kNoNode) {
      gone.push_back(m.km);
      gone.push_back(m.ka);
    }
    if (tail) gone.push_back(kq);
    EraseNodes(gone);
    return static_cast<int>(gone.size());
  };
  int removed = 0;
  for (size_t i = 0; i < nodes_.size();) {
    const int k = fuse(i);
    removed += k;
    i = k > 0 ? 0 : i + 1;   // indices moved: scan again (a fused node no longer matches)
  }
  allocated_ = false;
  return removed;
}

TfLiteStatus Graph::AllocateTensors() {
  RefreshContext();
  if (graph_exec_) {
    cudaGraphExecDestroy(static_cast<cudaGraphExec_t>(graph_exec_));
    graph_exec_ = nullptr;
  }
  for (auto& n : nodes_) {
    if (!n->initialized) {
      if (n->registration->init) {
        // custom ops get their flexbuffer options, builtins this host's parameter blob
        const bool custom = !n->custom_options.empty() || !n->node.builtin_data;
        const char* buf = custom ? reinterpret_cast<const char*>(n->custom_options.data())
                                 : static_cast<const char*>(n->node.builtin_data);
        const size_t len = custom ? n->custom_options.size() : n->builtin_blob.size();
        n->node.user_data = n->registration->init(&ctx_, buf, len);
      }
      n->initialized = true;
    }
    if (n->registration->prepare) {
      if (n->registration->prepare(&ctx_, &n->node) != kTfLiteOk) {
        if (error_.empty()) error_ = "prepare failed for node " + n->name;
        return kTfLiteError;
      }
      RefreshContext();
    }
  }
  if (PlanArena() != kTfLiteOk) return kTfLiteError;
  allocated_ = true;
  warmed_ = false;
  return kTfLiteOk;
}

TfLiteStatus Graph::ResizeInputTensor(int t, const std::vector<int>& dims) {
  if (t < 0 || t >= static_cast<int>(tensors_.size())) return kTfLiteError;
  return ResizeTensorCb(&ctx_, &tensors_[t], MakeDims(dims));
}

TfLiteStatus Graph::EnableCudaGraph(bool on) {
  use_cuda_graph_ = on && device_arena_;
  if (!use_cuda_graph_ && graph_exec_) {
    cudaGraphExecDestroy(static_cast<cudaGraphExec_t>(graph_exec_));
    graph_exec_ = nullptr;
  }
  return kTfLiteOk;
}

TfLiteStatus Graph::Invoke() {
  if (!allocated_ && AllocateTensors() != kTfLiteOk) return kTfLiteError;
  lce_b200_set_stream(stream_);  // nullptr (legacy default stream) for a host arena
  const bool prof = profiling_ && device_arena_ && !use_cuda_graph_;
  if (prof && node_events_.size() != nodes_.size()) {
    node_events_.assign(nodes_.size(), {});
    node_ms_.assign(nodes_.size(), 0.0);
  }
  auto run_nodes = [&]() -> TfLiteStatus {
    for (size_t i = 0; i < nodes_.size(); ++i) {
      auto& n = nodes_[i];
      cudaEvent_t e0 = nullptr, e1 = nullptr;
      if (prof) {
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        cudaEventRecord(e0, static_cast<cudaStream_t>(stream_));
      }
      if (n->registration->invoke(&ctx_, &n->node) != kTfLiteOk) {
        if (error_.empty()) error_ = "invoke failed for node " + n->name;
        return kTfLiteError;
      }
      if (prof) {
        cudaEventRecord(e1, static_cast<cudaStream_t>(stream_));
        node_events_[i].emplace_back(e0, e1);
      }
    }
    return kTfLiteOk;
  };
  if (!use_cuda_graph_) return run_nodes();
  cudaStream_t s = static_cast<cudaStream_t>(stream_);
  if (!graph_exec_) {
    // First call runs eagerly (ops build their plans: allocations are not
    // capturable); the second call records the launch sequence.
    if (!warmed_) {
      warmed_ = true;
      return run_nodes();
    }
    cudaGraph_t graph = nullptr;
    if (cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
      cudaGetLastError();
      return run_nodes();
    }
    TfLiteStatus rc = run_nodes();
    if (cudaStreamEndCapture(s, &graph) != cudaSuccess || rc != kTfLiteOk || !graph) {
      cudaGetLastError();
      error_ = "CUDA graph capture failed";
      return kTfLiteError;
    }
    cudaGraphExec_t exec = nullptr;
    if (cudaGraphInstantiate(&exec, graph, 0) != cudaSuccess) {
      cudaGraphDestroy(graph);
      error_ = "cudaGraphInstantiate failed";
      return kTfLiteError;
    }
    cudaGraphDestroy(graph);
    graph_exec_ = exec;
  }
  if (cudaGraphLaunch(static_cast<cudaGraphExec_t>(graph_exec_), s) != cudaSuccess) {
    error_ = "cudaGraphLaunch failed";
    return kTfLiteError;
  }
  return kTfLiteOk;
}

void Graph::ResetProfile() {
  for (auto& v : node_events_)
    for (auto& p : v) {
      cudaEventDestroy(static_cast<cudaEvent_t>(p.first));
      cudaEventDestroy(static_cast<cudaEvent_t>(p.second));
    }
  node_events_.assign(nodes_.size(), {});
  node_ms_.assign(nodes_.size(), 0.0);
}

double Graph::NodeTimeMs(size_t node) {
  if (node >= node_events_.size()) return 0.0;
  if (stream_) cudaStreamSynchronize(static_cast<cudaStream_t>(stream_));
  for (auto& p : node_events_[node]) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, static_cast<cudaEvent_t>(p.first),
                             static_cast<cudaEvent_t>(p.second)) == cudaSuccess)
      node_ms_[node] += ms;
    cudaEventDestroy(static_cast<cudaEvent_t>(p.first));
    cudaEventDestroy(static_cast<cudaEvent_t>(p.second));
  }
  node_events_[node].clear();
  return node_ms_[node];
}

TfLiteStatus Graph::Synchronize() {
  if (device_arena_ && cudaStreamSynchronize(static_cast<cudaStream_t>(stream_)) != cudaSuccess) {
    error_ = std::string("stream synchronize failed: ") + cudaGetErrorString(cudaGetLastError());
    return kTfLiteError;
  }
  return kTfLiteOk;
}

TfLiteStatus Graph::ReadTensorAsync(int i, void* dst, size_t bytes) {
  TfLiteTensor& t = tensors_[i];
  if (bytes > t.bytes || !t.data.raw || !device_arena_) {
    error_ = "ReadTensorAsync: size mismatch, unallocated tensor or host arena";
    return kTfLiteError;
  }
  if (cudaMemcpyAsync(dst, t.data.raw, bytes, cudaMemcpyDefault,
                      static_cast<cudaStream_t>(stream_)) != cudaSuccess) {
    error_ = "ReadTensorAsync: copy failed";
    return kTfLiteError;
  }
  return kTfLiteOk;
}

TfLiteStatus Graph::WriteTensor(int i, const void* src, size_t bytes) {
  TfLiteTensor& t = tensors_[i];
  if (bytes > t.bytes || !t.data.raw) {
    error_ = "WriteTensor: size mismatch or unallocated tensor";
    return kTfLiteError;
  }
  if (device_arena_ && t.allocation_type == kTfLiteArenaRw) {
    cudaStream_t s = static_cast<cudaStream_t>(stream_);
    if (cudaMemcpyAsync(t.data.raw, src, bytes, cudaMemcpyDefault, s) != cudaSuccess) {
      error_ = "WriteTensor: H2D copy failed";
      return kTfLiteError;
    }
  } else {
    memcpy(t.data.raw, src, bytes);
  }
  return kTfLiteOk;
}

TfLiteStatus Graph::ReadTensor(int i, void* dst, size_t bytes) {
  TfLiteTensor& t = tensors_[i];
  if (bytes > t.bytes || !t.data.raw) {
    error_ = "ReadTensor: size mismatch or unallocated tensor";
    return kTfLiteError;
  }
  if (device_arena_ && t.allocation_type == kTfLiteArenaRw) {
    cudaStream_t s = static_cast<cudaStream_t>(stream_);
    if (cudaMemcpyAsync(dst, t.data.raw, bytes, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
        cudaStreamSynchronize(s) != cudaSuccess) {
      error_ = std::string("ReadTensor: D2H copy failed: ") +
               cudaGetErrorString(cudaGetLastError());
      return kTfLiteError;
    }
  } else {
    memcpy(dst, const_host_[i].empty() ? t.data.raw : reinterpret_cast<char*>(const_host_[i].data()),
           bytes);
  }
  return kTfLiteOk;
}

}  // namespace lce_b200

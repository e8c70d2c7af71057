// tflite_model.cc -- `.tflite` (FlatBuffers, schema v3 "TFL3") reader that builds a
// lce_b200::Graph through an OpResolver: the role FlatBufferModel +
// InterpreterBuilder play for the reference (examples/lce_minimal.cc:31-45,
// LCE/tflite/python/interpreter_wrapper_lite.cc:28-58). flatbuffers is not vendored,
// so table access is hand-written from the wire format: uint32 root
// offset, int32 back-offset from a table to its vtable, uint16 vtable slots, uint32
// forward offsets for strings / vectors / sub-tables. Every access is bounds-checked.
#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "host_graph.h"
#include "lce_b200_tflite.h"
#include "builtin_params.h"

namespace lce_b200 {

namespace {

struct Buf {
  const uint8_t* p;
  size_t n;
  bool ok(size_t off, size_t len) const { return off <= n && len <= n - off; }
  template <class T>
  bool rd(size_t off, T* v) const {
    if (!ok(off, sizeof(T))) return false;
    memcpy(v, p + off, sizeof(T));
    return true;
  }
};

struct Vec {
  const Buf* b = nullptr;
  size_t data = 0;  // offset of element 0
  uint32_t len = 0;
  template <class T>
  T at(uint32_t i) const {
    T v{};
    b->rd(data + sizeof(T) * i, &v);
    return v;
  }
};

struct Table {
  const Buf* b = nullptr;
  size_t pos = 0;  // 0 = null table
  size_t field(int id) const {
    if (!pos) return 0;
    int32_t soff;
    if (!b->rd(pos, &soff)) return 0;
    const int64_t vt = static_cast<int64_t>(pos) - soff;
    if (vt < 0) return 0;
    uint16_t vt_len;
    if (!b->rd(static_cast<size_t>(vt), &vt_len)) return 0;
    const size_t slot = 4 + 2 * static_cast<size_t>(id);
    if (slot + 2 > vt_len) return 0;
    uint16_t off;
    if (!b->rd(static_cast<size_t>(vt) + slot, &off) || off == 0) return 0;
    return pos + off;
  }
  template <class T>
  T scalar(int id, T def) const {
    const size_t f = field(id);
    T v = def;
    if (f) b->rd(f, &v);
    return v;
  }
  size_t indirect(int id) const {
    const size_t f = field(id);
    uint32_t off;
    if (!f || !b->rd(f, &off)) return 0;
    return b->ok(f + off, 4) ? f + off : 0;
  }
  Table table(int id) const { return Table{b, indirect(id)}; }
  Vec vec(int id, size_t elem) const {
    const size_t v = indirect(id);
    uint32_t len;
    if (!v || !b->rd(v, &len) || !b->ok(v + 4, static_cast<size_t>(len) * elem)) return Vec{};
    return Vec{b, v + 4, len};
  }
  std::string str(int id) const {
    Vec v = vec(id, 1);
    return v.b ? std::string(reinterpret_cast<const char*>(b->p + v.data), v.len) : std::string();
  }
  Table elem_table(const Vec& v, uint32_t i) const {
    uint32_t off;
    const size_t slot = v.data + 4 * static_cast<size_t>(i);
    if (!b->rd(slot, &off) || !b->ok(slot + off, 4)) return Table{b, 0};
    return Table{b, slot + off};
  }
};

TfLiteType FromSchemaType(int t) {
  switch (t) {  // schema.fbs:39
    case 0: return kTfLiteFloat32;
    case 2: return kTfLiteInt32;
    case 3: return kTfLiteUInt8;
    case 4: return kTfLiteInt64;
    case 6: return kTfLiteBool;
    case 9: return kTfLiteInt8;
    default: return kTfLiteNoType;
  }
}

}  // namespace

// Builds `graph` from the flatbuffer. Constants of float builtins are placed on the
// device when the graph has a device arena; LCE constants may stay on the host
// (the plan uploads them once). Returns false and sets graph->last_error on failure.
bool BuildGraphFromTflite(const uint8_t* data, size_t size, const OpResolver& resolver,
                          Graph* graph) {
  Buf b{data, size};
  uint32_t root;
  if (size < 8 || memcmp(data + 4, "TFL3", 4) != 0 || !b.rd(0, &root) || !b.ok(root, 4)) {
    graph->set_error("not a TFL3 flatbuffer");
    return false;
  }
  Table model{&b, root};
  Vec codes = model.vec(1, 4), subgraphs = model.vec(2, 4), buffers = model.vec(4, 4);
  if (!subgraphs.b || subgraphs.len < 1) {
    graph->set_error("model has no subgraph");
    return false;
  }
  Table sg = model.elem_table(subgraphs, 0);
  Vec tensors = sg.vec(0, 4), ops = sg.vec(3, 4);
  Vec inputs = sg.vec(1, 4), outputs = sg.vec(2, 4);
  // Every tensor index the file carries is checked HERE, once: the op shells and the fusion
  // passes index context->tensors with them without further checks. Operator inputs may be -1
  // (kTfLiteOptionalTensor); operator outputs and the graph's inputs / outputs may not.
  if (!tensors.b || !ops.b) {
    graph->set_error("subgraph without a tensors or operators vector");
    return false;
  }
  auto index_ok = [&](int32_t t, bool optional) {
    return (optional && t == -1) || (t >= 0 && static_cast<uint32_t>(t) < tensors.len);
  };
  for (uint32_t k = 0; k < inputs.len; ++k)
    if (!index_ok(inputs.at<int32_t>(k), false)) {
      graph->set_error("graph input refers to a missing tensor");
      return false;
    }
  for (uint32_t k = 0; k < outputs.len; ++k)
    if (!index_ok(outputs.at<int32_t>(k), false)) {
      graph->set_error("graph output refers to a missing tensor");
      return false;
    }
  for (uint32_t i = 0; i < ops.len; ++i) {
    Table op = sg.elem_table(ops, i);
    if (op.scalar<uint32_t>(0, 0) >= codes.len) {
      graph->set_error("operator refers to a missing operator code");
      return false;
    }
    Vec in = op.vec(1, 4), out = op.vec(2, 4);
    for (uint32_t k = 0; k < in.len; ++k)
      if (!index_ok(in.at<int32_t>(k), true)) {
        graph->set_error("operator " + std::to_string(i) + " input refers to a missing tensor");
        return false;
      }
    for (uint32_t k = 0; k < out.len; ++k)
      if (!index_ok(out.at<int32_t>(k), false)) {
        graph->set_error("operator " + std::to_string(i) + " output refers to a missing tensor");
        return false;
      }
  }

  // which tensors are constants of builtin ops (=> device copies)
  std::vector<char> builtin_const(tensors.len, 0);
  for (uint32_t i = 0; i < ops.len; ++i) {
    Table op = sg.elem_table(ops, i);
    const uint32_t ci = op.scalar<uint32_t>(0, 0);
    Table code = model.elem_table(codes, ci);
    int32_t bc = code.scalar<int32_t>(3, 0);
    if (bc == 0) bc = code.scalar<int8_t>(0, 0);
    if (bc == 32) continue;
    Vec in = op.vec(1, 4);
    for (uint32_t k = 0; k < in.len; ++k) {
      const int32_t t = in.at<int32_t>(k);
      if ((bc == 34 || bc == 60) && k >= 1) continue;  // PAD paddings / PADV2 value: read on host
      if (t >= 0 && static_cast<uint32_t>(t) < tensors.len) builtin_const[t] = 1;
    }
  }

  for (uint32_t i = 0; i < tensors.len; ++i) {
    Table t = sg.elem_table(tensors, i);
    Vec shape = t.vec(0, 4);
    std::vector<int> dims(shape.len);
    for (uint32_t k = 0; k < shape.len; ++k) dims[k] = shape.at<int32_t>(k);
    const TfLiteType type = FromSchemaType(t.scalar<int8_t>(1, 0));
    const uint32_t buf_idx = t.scalar<uint32_t>(2, 0);
    const void* cdata = nullptr;
    size_t cbytes = 0;
    if (buf_idx != 0 && buf_idx < buffers.len) {
      Table bt = model.elem_table(buffers, buf_idx);
      Vec d = bt.vec(0, 1);
      if (d.b && d.len > 0) {
        cdata = data + d.data;
        cbytes = d.len;
      }
    }
    Table q = t.table(4);
    bool has_q = false;
    float scale = 0.f;
    int zp = 0;
    if (q.pos) {
      Vec sc = q.vec(2, 4), z = q.vec(3, 8);
      if (sc.b && sc.len > 0) {
        has_q = true;
        scale = sc.at<float>(0);
        zp = z.b && z.len > 0 ? static_cast<int>(z.at<int64_t>(0)) : 0;
      }
    }
    graph->AddTensor(type, dims, cdata, cbytes, has_q, scale, zp, t.str(3),
                     /*const_on_device=*/cdata != nullptr && builtin_const[i] != 0 &&
                         type == kTfLiteFloat32);
  }

  for (uint32_t i = 0; i < ops.len; ++i) {
    Table op = sg.elem_table(ops, i);
    const uint32_t ci = op.scalar<uint32_t>(0, 0);
    if (ci >= codes.len) {
      graph->set_error("operator refers to a missing operator code");
      return false;
    }
    Table code = model.elem_table(codes, ci);
    int32_t bc = code.scalar<int32_t>(3, 0);
    if (bc == 0) bc = code.scalar<int8_t>(0, 0);  // models written before builtin_code:int32
    Vec in = op.vec(1, 4), out = op.vec(2, 4);
    std::vector<int> iv(in.len), ov(out.len);
    for (uint32_t k = 0; k < in.len; ++k) iv[k] = in.at<int32_t>(k);
    for (uint32_t k = 0; k < out.len; ++k) ov[k] = out.at<int32_t>(k);
    if (bc == 32) {  // CUSTOM (schema.fbs:294)
      const std::string name = code.str(1);
      const TfLiteRegistration* reg = resolver.FindCustom(name);
      if (!reg) {
        graph->set_error("Encountered unresolved custom op: " + name);
        return false;
      }
      Vec co = op.vec(5, 1);
      graph->AddNode(reg, iv, ov, co.b ? data + co.data : nullptr, co.b ? co.len : 0, nullptr, 0,
                     name);
      continue;
    }
    const TfLiteRegistration* reg = resolver.FindBuiltin(bc);
    if (!reg) {
      graph->set_error("builtin operator " + std::to_string(bc) + " is not supported");
      return false;
    }
    BuiltinParams bp;
    memset(&bp, 0, sizeof(bp));
    bp.builtin_code = bc;
    bp.dilation_h = bp.dilation_w = 1;
    bp.depth_multiplier = 1;
    bp.beta = 1.0f;
    Table o = op.table(4);
    switch (bc) {
      case 3:  // CONV_2D: Conv2DOptions (schema.fbs:806)
        bp.padding = o.scalar<int8_t>(0, 0);
        bp.stride_w = o.scalar<int32_t>(1, 0);
        bp.stride_h = o.scalar<int32_t>(2, 0);
        bp.activation = o.scalar<int8_t>(3, 0);
        bp.dilation_w = o.scalar<int32_t>(4, 1);
        bp.dilation_h = o.scalar<int32_t>(5, 1);
        break;
      case 4:  // DEPTHWISE_CONV_2D (schema.fbs:839)
        bp.padding = o.scalar<int8_t>(0, 0);
        bp.stride_w = o.scalar<int32_t>(1, 0);
        bp.stride_h = o.scalar<int32_t>(2, 0);
        bp.depth_multiplier = o.scalar<int32_t>(3, 0);
        bp.activation = o.scalar<int8_t>(4, 0);
        bp.dilation_w = o.scalar<int32_t>(5, 1);
        bp.dilation_h = o.scalar<int32_t>(6, 1);
        break;
      case 1:
      case 17:  // AVERAGE_POOL_2D / MAX_POOL_2D: Pool2DOptions (schema.fbs:830)
        bp.padding = o.scalar<int8_t>(0, 0);
        bp.stride_w = o.scalar<int32_t>(1, 0);
        bp.stride_h = o.scalar<int32_t>(2, 0);
        bp.filter_w = o.scalar<int32_t>(3, 0);
        bp.filter_h = o.scalar<int32_t>(4, 0);
        bp.activation = o.scalar<int8_t>(5, 0);
        break;
      case 9:  // FULLY_CONNECTED (schema.fbs:907)
        bp.activation = o.scalar<int8_t>(0, 0);
        bp.keep_dims = o.scalar<int8_t>(2, 0);
        break;
      case 25:  // SOFTMAX (schema.fbs:929)
        bp.beta = o.scalar<float>(0, 1.0f);
        break;
      case 0:
      case 18:
      case 42:  // ADD / MUL / DIV (schema.fbs:939,945; DivOptions)
        bp.activation = o.scalar<int8_t>(0, 0);
        break;
      case 2:  // CONCATENATION (schema.fbs:934)
        bp.axis = o.scalar<int32_t>(0, 0);
        bp.activation = o.scalar<int8_t>(1, 0);
        break;
      case 40:
      case 82:  // MEAN / REDUCE_MAX: ReducerOptions (schema.fbs:1106)
        bp.keep_dims = o.scalar<int8_t>(0, 0);
        break;
      case 22: {  // RESHAPE (schema.fbs:1044)
        Vec ns = o.vec(0, 4);
        bp.n_new_shape = ns.b ? static_cast<int>(std::min<uint32_t>(ns.len, 8)) : 0;
        for (int k = 0; k < bp.n_new_shape; ++k) bp.new_shape[k] = ns.at<int32_t>(k);
        break;
      }
      case 45:  // STRIDED_SLICE: StridedSliceOptions
        bp.begin_mask = o.scalar<int32_t>(0, 0);
        bp.end_mask = o.scalar<int32_t>(1, 0);
        bp.ellipsis_mask = o.scalar<int32_t>(2, 0);
        bp.new_axis_mask = o.scalar<int32_t>(3, 0);
        bp.shrink_axis_mask = o.scalar<int32_t>(4, 0);
        bp.offset = o.scalar<int8_t>(5, 0);
        break;
      case 49:  // SPLIT: SplitOptions
        bp.num_splits = o.scalar<int32_t>(0, 0);
        break;
      case 23:  // RESIZE_BILINEAR: ResizeBilinearOptions (fields 0 and 1 are the deprecated sizes)
        bp.align_corners = o.scalar<int8_t>(2, 0);
        bp.half_pixel_centers = o.scalar<int8_t>(3, 0);
        break;
      case 97:  // RESIZE_NEAREST_NEIGHBOR: ResizeNearestNeighborOptions
        bp.align_corners = o.scalar<int8_t>(0, 0);
        bp.half_pixel_centers = o.scalar<int8_t>(1, 0);
        break;
      case 56:  // ARG_MAX: ArgMaxOptions
        bp.output_type = o.scalar<int8_t>(0, 0);
        break;
      case 5:  // DEPTH_TO_SPACE: DepthToSpaceOptions
        bp.block_size = o.scalar<int32_t>(0, 0);
        break;
      case 67:  // TRANSPOSE_CONV: TransposeConvOptions
        bp.padding = o.scalar<int8_t>(0, 0);
        bp.stride_w = o.scalar<int32_t>(1, 0);
        bp.stride_h = o.scalar<int32_t>(2, 0);
        bp.activation = o.scalar<int8_t>(3, 0);
        break;
      default:
        break;
    }
    graph->AddNode(reg, iv, ov, nullptr, 0, &bp, sizeof(bp), "builtin:" + std::to_string(bc));
  }
  std::vector<int> gi(inputs.len), go(outputs.len);
  for (uint32_t k = 0; k < inputs.len; ++k) gi[k] = inputs.at<int32_t>(k);
  for (uint32_t k = 0; k < outputs.len; ++k) go[k] = outputs.at<int32_t>(k);
  graph->SetInputs(gi);
  graph->SetOutputs(go);
  return true;
}

}  // namespace lce_b200

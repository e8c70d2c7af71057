// lce_ops.cc -- the TFLite custom-op shell (init / free / prepare / invoke) for
// LceQuantize, LceDequantize, LceBconv2d and LceBMaxPool2d on top of the CUDA C-ABI
// (include/lce_b200.h). It mirrors, check for check and message for message, what
// the reference's op shell does around its CPU kernels:
//   LCE/tflite/kernels/bconv2d.cc       Init :85, Free :133, Prepare :138, Eval :551
//   LCE/tflite/kernels/quantization.cc  QuantizePrepare :19, DequantizePrepare :43,
//                                       QuantizeEval :76, DequantizeEval :116
//   LCE/tflite/kernels/bmaxpool.cc      Init :21, Prepare :40, Eval :75
// Tensor memory: `TfLiteTensor::data` of activations may be a DEVICE pointer (this
// repository's graph host keeps the arena in HBM) or a HOST pointer (a stock TFLite
// interpreter): host tensors are staged through the device inside invoke. Constant
// inputs (filter, multiplier, bias, thresholds) may live on either side.
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <vector>

#include "flexbuffer_map.h"
#include "lce_b200.h"
#include "lce_b200_tflite.h"

// lce_b200.cu: whether run_fused / run_fused_chain take packed output for a plan of *d
extern "C" int lce_b200_internal_grouped_packs(const lce_bconv2d_desc* d);

namespace {

// The stream the ops launch on: set by the graph host before it walks its nodes. Thread local:
// two graphs invoked from two threads (one Interpreter per device) do not see each other's.
thread_local void* g_stream = nullptr;

#define LCE_ENSURE(ctx, cond)                                                          \
  do {                                                                                 \
    if (!(cond)) {                                                                     \
      (ctx)->ReportError((ctx), "%s:%d %s was not true.", __FILE__, __LINE__, #cond);  \
      return kTfLiteError;                                                             \
    }                                                                                  \
  } while (0)
#define LCE_ENSURE_MSG(ctx, cond, msg)              \
  do {                                              \
    if (!(cond)) {                                  \
      (ctx)->ReportError((ctx), "%s", (msg));       \
      return kTfLiteError;                          \
    }                                               \
  } while (0)
#define LCE_ENSURE_CAPI(ctx, call)                                  \
  do {                                                              \
    if ((call) != 0) {                                              \
      (ctx)->ReportError((ctx), "%s", lce_b200_last_error());       \
      return kTfLiteError;                                          \
    }                                                               \
  } while (0)

// kernel_util.cc:78-116 -- optional inputs are index -1 and come back as nullptr.
const TfLiteTensor* GetInput(TfLiteContext* c, const TfLiteNode* n, int i) {
  if (i >= n->inputs->size) return nullptr;
  const int idx = n->inputs->data[i];
  if (idx == kTfLiteOptionalTensor) return nullptr;
  return c->GetTensor ? c->GetTensor(c, idx) : &c->tensors[idx];
}
TfLiteTensor* GetOutput(TfLiteContext* c, const TfLiteNode* n, int i) {
  const int idx = n->outputs->data[i];
  return c->GetTensor ? c->GetTensor(c, idx) : &c->tensors[idx];
}
int NumDims(const TfLiteTensor* t) { return t->dims->size; }
int Dim(const TfLiteTensor* t, int i) { return t->dims->data[i]; }
int BitpackedSize(int n) { return (n + 31) / 32; }
int64_t NumElements(const TfLiteTensor* t) {
  int64_t n = 1;
  for (int i = 0; i < t->dims->size; ++i) n *= t->dims->data[i];
  return n;
}

bool OnDevice(const void* p) {
  if (!p) return true;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// Staging for host-resident activation tensors (stock-TFLite arena).
struct Staging {
  void* in = nullptr;
  void* out = nullptr;
  size_t in_bytes = 0, out_bytes = 0;
  ~Staging() {
    cudaFree(in);
    cudaFree(out);
  }
  bool Reserve(size_t ib, size_t ob) {
    if (ib > in_bytes) {
      cudaFree(in);
      in = nullptr;
      if (cudaMalloc(&in, ib + 16) != cudaSuccess) return false;
      in_bytes = ib;
    }
    if (ob > out_bytes) {
      cudaFree(out);
      out = nullptr;
      if (cudaMalloc(&out, ob + 16) != cudaSuccess) return false;
      out_bytes = ob;
    }
    return true;
  }
};

// Runs `launch(in_dev, out_dev)` with device views of (input, output), staging
// host tensors through HBM when the interpreter's arena lives on the host.
template <class F>
TfLiteStatus WithDeviceIO(TfLiteContext* ctx, Staging* st, const TfLiteTensor* input,
                          TfLiteTensor* output, F launch) {
  const bool in_dev = OnDevice(input->data.raw_const);
  const bool out_dev = OnDevice(output->data.raw);
  if (in_dev && out_dev) return launch(input->data.raw_const, output->data.raw);
  cudaStream_t s = static_cast<cudaStream_t>(g_stream);
  if (!st->Reserve(in_dev ? 0 : input->bytes, out_dev ? 0 : output->bytes)) {
    ctx->ReportError(ctx, "lce_b200: cudaMalloc of staging buffers failed");
    return kTfLiteError;
  }
  const void* din = input->data.raw_const;
  void* dout = output->data.raw;
  if (!in_dev) {
    if (input->bytes &&
        cudaMemcpyAsync(st->in, input->data.raw_const, input->bytes, cudaMemcpyHostToDevice, s) !=
            cudaSuccess) {
      ctx->ReportError(ctx, "lce_b200: H2D staging copy failed: %s",
                       cudaGetErrorString(cudaGetLastError()));
      return kTfLiteError;
    }
    din = st->in;
  }
  if (!out_dev) dout = st->out;
  TfLiteStatus rc = launch(din, dout);
  if (rc != kTfLiteOk) return rc;
  if (!out_dev) {
    if ((output->bytes &&
         cudaMemcpyAsync(output->data.raw, st->out, output->bytes, cudaMemcpyDeviceToHost, s) !=
             cudaSuccess) ||
        cudaStreamSynchronize(s) != cudaSuccess) {
      ctx->ReportError(ctx, "lce_b200: D2H staging copy failed: %s",
                       cudaGetErrorString(cudaGetLastError()));
      return kTfLiteError;
    }
  }
  return kTfLiteOk;
}

// ------------------------------------------------------------------------- //
// LceBconv2d
// ------------------------------------------------------------------------- //
enum class KernelType { kReference, kOptimizedBGEMM, kOptimizedIndirectBGEMM, kCuda };

struct BconvOpData {
  lce_bconv2d_desc desc{};
  bool successfully_initialized = false;
  bool plan_stale = true;
  lce_b200_bconv2d* plan = nullptr;
  // what the plan was built from (constant inputs, output type / quantisation, activation)
  const void* plan_key[4] = {nullptr, nullptr, nullptr, nullptr};
  int plan_out_type = -1, plan_zero_point = 0, plan_activation = -1;
  float plan_scale = 0.0f;
  int zp_mode = LCE_ZERO_PADDING_REFERENCE;  // set by Prepare from the registration
  Staging staging;
  ~BconvOpData() { lce_b200_bconv2d_destroy(plan); }
};

#define LCE_ENSURE_PARAM(op_data, context, a)                                          \
  do {                                                                                 \
    if (!(a)) {                                                                        \
      (context)->ReportError((context), "%s:%d %s was not true.", __FILE__, __LINE__, #a); \
      return op_data;                                                                  \
    }                                                                                  \
  } while (0)

void* BconvInit(TfLiteContext* context, const char* buffer, size_t length) {
  auto* op = new BconvOpData();
  lce_b200::FlexMap m(reinterpret_cast<const uint8_t*>(buffer), length);
  LCE_ENSURE_PARAM(op, context, m.Has("stride_height"));
  LCE_ENSURE_PARAM(op, context, m.Has("stride_width"));
  LCE_ENSURE_PARAM(op, context, m.Has("dilation_height_factor"));
  LCE_ENSURE_PARAM(op, context, m.Has("dilation_width_factor"));
  LCE_ENSURE_PARAM(op, context, m.Has("padding"));
  LCE_ENSURE_PARAM(op, context, m.Has("pad_values"));
  LCE_ENSURE_PARAM(op, context, m.Has("channels_in"));
  LCE_ENSURE_PARAM(op, context, m.Has("fused_activation_function"));
  lce_bconv2d_desc& d = op->desc;
  d.stride_h = m.AsInt32("stride_height");
  d.stride_w = m.AsInt32("stride_width");
  d.dilation_h = m.AsInt32("dilation_height_factor");
  d.dilation_w = m.AsInt32("dilation_width_factor");
  d.padding = m.AsInt32("padding");  // schema Padding: SAME=0, VALID=1
  d.pad_value = m.AsInt32("pad_values");
  if (d.pad_value != 0 && d.pad_value != 1) {
    context->ReportError(context, "Attribute pad_values must be 0 or 1.");
    return op;
  }
  d.channels_in = m.AsInt32("channels_in");
  // ConvertActivation (LCE/tflite/kernels/utils.h:10-24): unknown values -> NONE
  const int act = m.AsInt32("fused_activation_function");
  d.activation = (act >= LCE_ACT_NONE && act <= LCE_ACT_RELU6) ? act : LCE_ACT_NONE;
  op->successfully_initialized = true;
  return op;
}

void BconvFree(TfLiteContext*, void* buffer) { delete static_cast<BconvOpData*>(buffer); }

template <KernelType kernel_type, bool FUSED = false>
TfLiteStatus BconvPrepare(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<BconvOpData*>(node->user_data);
  if (!op->successfully_initialized) return kTfLiteError;
  lce_bconv2d_desc& d = op->desc;

  // fused: 6 inputs, or 10 with the activation chain (inputs 6..9, Graph::FuseActivationChains)
  LCE_ENSURE(context, FUSED ? (node->inputs->size == 6 || node->inputs->size == 10)
                            : node->inputs->size == 5);
  const TfLiteTensor* input = GetInput(context, node, 0);
  const TfLiteTensor* filter = GetInput(context, node, 1);
  const TfLiteTensor* post_mul = GetInput(context, node, 2);
  const TfLiteTensor* post_bias = GetInput(context, node, 3);
  const TfLiteTensor* thresholds = GetInput(context, node, 4);
  TfLiteTensor* output = GetOutput(context, node, 0);
  LCE_ENSURE(context, input != nullptr && filter != nullptr);
  LCE_ENSURE(context, NumDims(input) == 4);
  LCE_ENSURE(context, NumDims(filter) == 4);
  LCE_ENSURE(context, input->type == kTfLiteInt32);
  LCE_ENSURE(context, filter->type == kTfLiteInt32);
  LCE_ENSURE_MSG(context,
                 output->type == kTfLiteInt32 || output->type == kTfLiteInt8 ||
                     output->type == kTfLiteFloat32,
                 "Supported output types are int8, int32, and float32.");

  d.channels_out = Dim(filter, 0);
  d.filter_h = Dim(filter, 1);
  d.filter_w = Dim(filter, 2);
  // groups: bconv2d.cc:169-186
  if (Dim(filter, 3) == BitpackedSize(d.channels_in)) {
    d.groups = 1;
  } else {
    LCE_ENSURE_MSG(context, kernel_type != KernelType::kOptimizedBGEMM,
                   "Grouped binary convolutions are not supported with this kernel.");
    LCE_ENSURE(context, Dim(filter, 3) > 0 && BitpackedSize(d.channels_in) % Dim(filter, 3) == 0);
    const int groups = BitpackedSize(d.channels_in) / Dim(filter, 3);
    LCE_ENSURE(context, d.channels_in % groups == 0);
    const int group_size = d.channels_in / groups;
    LCE_ENSURE(context, group_size % 32 == 0);
    LCE_ENSURE(context, d.channels_out % groups == 0);
    d.groups = groups;
  }
  LCE_ENSURE(context, Dim(input, 3) == BitpackedSize(d.channels_in));

  d.out_type = output->type == kTfLiteFloat32 ? LCE_OUT_FLOAT
               : output->type == kTfLiteInt8  ? LCE_OUT_INT8
                                              : LCE_OUT_BITPACKED;
  // Zero padding: legality as bconv2d.cc:188-200 and, with it, WHICH of the reference's two
  // results this node reproduces (LCE_ZERO_PADDING_*, include/lce_b200_types.h): the reference
  // registration computes the reference kernel's integers; the optimised registrations -- the
  // reference's default Register_BCONV_2D among them -- one-padding plus the float correction of
  // zero_padding_correction.h. The default registration accepts the union of both rules and
  // follows the optimised kernels wherever they are legal.
  op->zp_mode = LCE_ZERO_PADDING_REFERENCE;
  if (d.padding == LCE_PADDING_SAME && d.pad_value == 0) {
    const bool ref_rule = d.channels_in % 2 == 0;
    const bool opt_rule = output->type == kTfLiteFloat32 && d.activation == LCE_ACT_NONE;
    bool legal;
    if (kernel_type == KernelType::kReference) {
      legal = ref_rule;
    } else if (kernel_type == KernelType::kCuda) {
      legal = ref_rule || opt_rule;
      if (opt_rule) op->zp_mode = LCE_ZERO_PADDING_CORRECTION;
    } else {
      legal = opt_rule;
      op->zp_mode = LCE_ZERO_PADDING_CORRECTION;
    }
    LCE_ENSURE_MSG(context, legal,
                   "Zero-padding is only supported by the reference kernel with an even "
                   "number of input channels, or when using "
                   "float output with no fused activation function.");
  }

  d.batch = Dim(input, 0);
  d.in_h = Dim(input, 1);
  d.in_w = Dim(input, 2);
  int out_h, out_w, pad_h, pad_w;
  LCE_ENSURE_CAPI(context, lce_b200_bconv2d_out_shape(&d, &out_h, &out_w, &pad_h, &pad_w));

  if (output->type == kTfLiteInt32) {
    LCE_ENSURE(context, thresholds != nullptr);
    LCE_ENSURE(context, NumDims(thresholds) == 1);
    LCE_ENSURE(context, thresholds->type == kTfLiteInt32);
    LCE_ENSURE(context, Dim(thresholds, 0) == d.channels_out);
  } else {
    LCE_ENSURE(context, post_mul != nullptr && post_bias != nullptr);
    LCE_ENSURE(context, post_mul->type == kTfLiteFloat32);
    LCE_ENSURE(context, post_bias->type == kTfLiteFloat32);
    LCE_ENSURE(context, NumDims(post_mul) == 1);
    LCE_ENSURE(context, NumDims(post_bias) == 1);
    LCE_ENSURE(context, Dim(post_mul, 0) == d.channels_out);
    LCE_ENSURE(context, Dim(post_bias, 0) == d.channels_out);
  }
  if (output->type == kTfLiteInt8) {
    LCE_ENSURE(context, output->quantization.type == kTfLiteAffineQuantization);
    d.out_scale = output->params.scale;
    d.out_zero_point = output->params.zero_point;
  }
  if (kernel_type == KernelType::kOptimizedIndirectBGEMM) {
    LCE_ENSURE_MSG(context, input->allocation_type != kTfLiteDynamic,
                   "The input tensor must not have dynamic allocation type");
  }

  TfLiteIntArray* output_shape = LceB200IntArrayCreate(4);
  output_shape->data[0] = d.batch;
  output_shape->data[1] = out_h;
  output_shape->data[2] = out_w;
  output_shape->data[3] =
      output->type == kTfLiteInt32 ? BitpackedSize(d.channels_out) : d.channels_out;
  if (context->ResizeTensor(context, output, output_shape) != kTfLiteOk) return kTfLiteError;
  if (FUSED) {
    // graph-level fusion (host_graph.cc::FuseResidualBlocks): input 5 = the shortcut of the
    // ADD that followed, optional output 1 = the LceQuantize of the sum.
    const TfLiteTensor* residual = GetInput(context, node, 5);
    LCE_ENSURE(context, output->type == kTfLiteFloat32 && residual != nullptr);
    LCE_ENSURE(context, residual->type == kTfLiteFloat32 && NumDims(residual) == 4);
    LCE_ENSURE(context, Dim(residual, 0) == d.batch && Dim(residual, 1) == out_h &&
                            Dim(residual, 2) == out_w && Dim(residual, 3) == d.channels_out);
    // the chain's per-channel constants: shift_in, alpha, shift_out, sign_shift (absent = -1)
    for (int k = 6; k < node->inputs->size; ++k) {
      const TfLiteTensor* v = GetInput(context, node, k);
      LCE_ENSURE(context, v == nullptr || (v->type == kTfLiteFloat32 &&
                                           NumElements(v) == d.channels_out));
    }
    if (node->outputs->size > 1) {
      LCE_ENSURE(context, lce_b200_internal_grouped_packs(&d));
      TfLiteIntArray* packed_shape = LceB200IntArrayCreate(4);
      packed_shape->data[0] = d.batch;
      packed_shape->data[1] = out_h;
      packed_shape->data[2] = out_w;
      packed_shape->data[3] = BitpackedSize(d.channels_out);
      if (context->ResizeTensor(context, GetOutput(context, node, 1), packed_shape) != kTfLiteOk)
        return kTfLiteError;
    }
  }

  // "Prepare could be called multiple times; when the input tensor is resized, we
  // should always re-do the one-time setup" (bconv2d.cc:295-297).
  op->plan_stale = true;
  return kTfLiteOk;
}

TfLiteStatus BconvEnsurePlan(TfLiteContext* context, TfLiteNode* node);

// Fused node: [in, filter, mul, bias, thr, residual (, shift_in, alpha, shift_out, sign_shift)]
// -> [out, packed_out?]; device arena only.
TfLiteStatus BconvFusedEval(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<BconvOpData*>(node->user_data);
  if (BconvEnsurePlan(context, node) != kTfLiteOk) return kTfLiteError;
  const TfLiteTensor* input = GetInput(context, node, 0);
  const TfLiteTensor* residual = GetInput(context, node, 5);
  TfLiteTensor* output = GetOutput(context, node, 0);
  TfLiteTensor* packed = node->outputs->size > 1 ? GetOutput(context, node, 1) : nullptr;
  int add_act = LCE_ACT_NONE;
  if (node->builtin_data) add_act = *static_cast<const int32_t*>(node->builtin_data);
  LCE_ENSURE_MSG(context, OnDevice(input->data.raw) && OnDevice(output->data.raw) &&
                              OnDevice(residual->data.raw),
                 "fused LceBconv2d needs a device arena");
  if (node->inputs->size == 10) {
    auto vec = [&](int k) {
      const TfLiteTensor* v = GetInput(context, node, k);
      return v ? v->data.f : nullptr;
    };
    const lce_chain_desc chain{vec(6), vec(7), vec(8), vec(9)};
    LCE_ENSURE_CAPI(context, lce_b200_bconv2d_run_fused_chain(
                                 op->plan, input->data.i32, residual->data.f, add_act, &chain,
                                 output->data.f, packed ? packed->data.i32 : nullptr, g_stream));
    return kTfLiteOk;
  }
  LCE_ENSURE_CAPI(context,
                  lce_b200_bconv2d_run_fused(op->plan, input->data.i32, residual->data.f, add_act,
                                             output->data.f, packed ? packed->data.i32 : nullptr,
                                             g_stream));
  return kTfLiteOk;
}

TfLiteStatus BconvEval(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<BconvOpData*>(node->user_data);
  if (BconvEnsurePlan(context, node) != kTfLiteOk) return kTfLiteError;
  const TfLiteTensor* input = GetInput(context, node, 0);
  TfLiteTensor* output = GetOutput(context, node, 0);
  const TfLiteType ot = output->type;
  if (ot != kTfLiteFloat32 && ot != kTfLiteInt8 && ot != kTfLiteInt32) return kTfLiteError;
  return WithDeviceIO(context, &op->staging, input, output,
                      [&](const void* in_dev, void* out_dev) -> TfLiteStatus {
                        LCE_ENSURE_CAPI(context,
                                        lce_b200_bconv2d_run(op->plan,
                                                             static_cast<const int32_t*>(in_dev),
                                                             out_dev, g_stream));
                        return kTfLiteOk;
                      });
}

// OneTimeSetup (bconv2d.cc:324-392): build / refresh the plan after a (re)prepare.
TfLiteStatus BconvEnsurePlan(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<BconvOpData*>(node->user_data);
  const TfLiteTensor* input = GetInput(context, node, 0);
  const TfLiteTensor* filter = GetInput(context, node, 1);
  const TfLiteTensor* post_mul = GetInput(context, node, 2);
  const TfLiteTensor* post_bias = GetInput(context, node, 3);
  const TfLiteTensor* thresholds = GetInput(context, node, 4);
  TfLiteTensor* output = GetOutput(context, node, 0);
  const TfLiteType ot = output->type;
  if (ot != kTfLiteFloat32 && ot != kTfLiteInt8 && ot != kTfLiteInt32) return kTfLiteError;

  if (op->plan_stale) {
    // The re-tiled weights and folded epilogue vectors are reused only while every constant
    // input, the output type and its quantisation are what the plan was built from; the reference
    // redoes its OneTimeSetup on every Prepare (bconv2d.cc:295-297).
    const void* key[4] = {filter->data.raw_const, post_mul ? post_mul->data.raw_const : nullptr,
                          post_bias ? post_bias->data.raw_const : nullptr,
                          thresholds ? thresholds->data.raw_const : nullptr};
    const bool same = op->plan && op->plan_key[0] == key[0] && op->plan_key[1] == key[1] &&
                      op->plan_key[2] == key[2] && op->plan_key[3] == key[3] &&
                      op->plan_out_type == op->desc.out_type && op->plan_scale == op->desc.out_scale &&
                      op->plan_zero_point == op->desc.out_zero_point &&
                      op->plan_activation == op->desc.activation;
    if (same) {
      LCE_ENSURE_CAPI(context, lce_b200_bconv2d_set_input_shape(op->plan, op->desc.batch,
                                                                 op->desc.in_h, op->desc.in_w));
    } else {
      lce_b200_bconv2d_destroy(op->plan);
      op->plan = nullptr;
      LCE_ENSURE_CAPI(context,
                      lce_b200_bconv2d_create(
                          &op->desc, filter->data.i32, post_mul ? post_mul->data.f : nullptr,
                          post_bias ? post_bias->data.f : nullptr,
                          thresholds ? thresholds->data.i32 : nullptr, &op->plan));
      for (int i = 0; i < 4; ++i) op->plan_key[i] = key[i];
      op->plan_out_type = op->desc.out_type;
      op->plan_scale = op->desc.out_scale;
      op->plan_zero_point = op->desc.out_zero_point;
      op->plan_activation = op->desc.activation;
    }
    LCE_ENSURE_CAPI(context, lce_b200_bconv2d_set_zero_padding_mode(op->plan, op->zp_mode));
    op->plan_stale = false;
  }
  (void)input;
  return kTfLiteOk;
}

// ------------------------------------------------------------------------- //
// LceQuantize / LceDequantize
// ------------------------------------------------------------------------- //
struct IoOpData {
  Staging staging;
};
// The reference registers these with init = free = nullptr (quantization.cc:149-159)
// and keeps no per-node state; staging for host arenas is the only state here and
// lives in node->user_data when an init is provided. To keep init/free null like
// the reference, staging buffers are thread-local instead.
thread_local Staging tl_staging;

TfLiteStatus QuantizePrepare(TfLiteContext* context, TfLiteNode* node) {
  LCE_ENSURE(context, node->inputs->size == 1);
  LCE_ENSURE(context, node->outputs->size == 1);
  const TfLiteTensor* input = GetInput(context, node, 0);
  TfLiteTensor* output = GetOutput(context, node, 0);
  LCE_ENSURE(context, input->type == kTfLiteFloat32 || input->type == kTfLiteInt8 ||
                          input->type == kTfLiteBool);
  LCE_ENSURE(context, output->type == kTfLiteInt32);
  const int num_dims = NumDims(input);
  LCE_ENSURE(context, num_dims == NumDims(output));
  LCE_ENSURE(context, num_dims >= 1);
  TfLiteIntArray* output_dims = LceB200IntArrayCreate(num_dims);
  for (int i = 0; i < num_dims; ++i) output_dims->data[i] = Dim(input, i);
  output_dims->data[num_dims - 1] = BitpackedSize(Dim(input, num_dims - 1));
  return context->ResizeTensor(context, output, output_dims);
}

TfLiteStatus DequantizePrepare(TfLiteContext* context, TfLiteNode* node) {
  LCE_ENSURE(context, node->inputs->size == 1);
  LCE_ENSURE(context, node->outputs->size == 1);
  const TfLiteTensor* input = GetInput(context, node, 0);
  TfLiteTensor* output = GetOutput(context, node, 0);
  LCE_ENSURE(context, input->type == kTfLiteInt32);
  LCE_ENSURE(context, output->type == kTfLiteFloat32 || output->type == kTfLiteInt8 ||
                          output->type == kTfLiteBool);
  const int num_dims = NumDims(input);
  LCE_ENSURE(context, num_dims == NumDims(output));
  LCE_ENSURE(context, num_dims >= 1);
  for (int i = 0; i < num_dims - 1; ++i) LCE_ENSURE(context, Dim(output, i) == Dim(input, i));
  // The output channel count cannot be inferred from the packed count, so there is
  // no resize here (quantization.cc:61-71).
  LCE_ENSURE(context, Dim(input, num_dims - 1) == BitpackedSize(Dim(output, num_dims - 1)));
  return kTfLiteOk;
}

TfLiteStatus QuantizeEval(TfLiteContext* context, TfLiteNode* node) {
  const TfLiteTensor* input = GetInput(context, node, 0);
  TfLiteTensor* output = GetOutput(context, node, 0);
  int in_type;
  int32_t zero_point = 0;
  if (input->type == kTfLiteFloat32) {
    in_type = LCE_T_FLOAT;
  } else if (input->type == kTfLiteInt8) {
    in_type = LCE_T_INT8;
    zero_point = input->params.zero_point;
  } else if (input->type == kTfLiteBool) {
    in_type = LCE_T_BOOL;
  } else {
    return kTfLiteError;
  }
  const int nd = NumDims(input);
  const int64_t cols = Dim(input, nd - 1);
  const int64_t rows = cols ? NumElements(input) / cols : 0;
  return WithDeviceIO(context, &tl_staging, input, output,
                      [&](const void* in_dev, void* out_dev) -> TfLiteStatus {
                        LCE_ENSURE_CAPI(context,
                                        lce_b200_quantize(in_type, in_dev, rows, cols, zero_point,
                                                          static_cast<int32_t*>(out_dev),
                                                          g_stream));
                        return kTfLiteOk;
                      });
}

TfLiteStatus DequantizeEval(TfLiteContext* context, TfLiteNode* node) {
  const TfLiteTensor* input = GetInput(context, node, 0);
  TfLiteTensor* output = GetOutput(context, node, 0);
  int out_type;
  if (output->type == kTfLiteFloat32) out_type = LCE_T_FLOAT;
  else if (output->type == kTfLiteInt8) out_type = LCE_T_INT8;
  else if (output->type == kTfLiteBool) out_type = LCE_T_BOOL;
  else return kTfLiteError;
  const int nd = NumDims(output);
  const int64_t cols = Dim(output, nd - 1);
  const int64_t rows = cols ? NumElements(output) / cols : 0;
  return WithDeviceIO(context, &tl_staging, input, output,
                      [&](const void* in_dev, void* out_dev) -> TfLiteStatus {
                        LCE_ENSURE_CAPI(context,
                                        lce_b200_dequantize(out_type,
                                                            static_cast<const int32_t*>(in_dev),
                                                            rows, cols, output->params.scale,
                                                            output->params.zero_point, out_dev,
                                                            g_stream));
                        return kTfLiteOk;
                      });
}

// ------------------------------------------------------------------------- //
// LceBMaxPool2d
// ------------------------------------------------------------------------- //
struct BMaxPoolOpData {
  lce_bmaxpool_desc desc{};
  Staging staging;
};

void* BMaxPoolInit(TfLiteContext*, const char* buffer, size_t length) {
  auto* op = new BMaxPoolOpData();
  lce_b200::FlexMap m(reinterpret_cast<const uint8_t*>(buffer), length);
  op->desc.filter_h = m.AsInt32("filter_height");
  op->desc.filter_w = m.AsInt32("filter_width");
  op->desc.stride_h = m.AsInt32("stride_height");
  op->desc.stride_w = m.AsInt32("stride_width");
  op->desc.padding = m.AsInt32("padding");
  return op;
}
void BMaxPoolFree(TfLiteContext*, void* buffer) { delete static_cast<BMaxPoolOpData*>(buffer); }

TfLiteStatus BMaxPoolPrepare(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<BMaxPoolOpData*>(node->user_data);
  LCE_ENSURE(context, node->inputs->size == 1);
  LCE_ENSURE(context, node->outputs->size == 1);
  TfLiteTensor* output = GetOutput(context, node, 0);
  const TfLiteTensor* input = GetInput(context, node, 0);
  LCE_ENSURE(context, NumDims(input) == 4);
  LCE_ENSURE(context, input->type == kTfLiteInt32);
  LCE_ENSURE(context, output->type == kTfLiteInt32);
  LCE_ENSURE(context, op->desc.stride_h != 0);
  LCE_ENSURE(context, op->desc.stride_w != 0);
  LCE_ENSURE(context, op->desc.filter_h != 0);
  LCE_ENSURE(context, op->desc.filter_w != 0);
  op->desc.batch = Dim(input, 0);
  op->desc.in_h = Dim(input, 1);
  op->desc.in_w = Dim(input, 2);
  op->desc.channels_packed = Dim(input, 3);
  int out_h, out_w;
  LCE_ENSURE_CAPI(context, lce_b200_bmaxpool_out_shape(&op->desc, &out_h, &out_w));
  TfLiteIntArray* output_size = LceB200IntArrayCreate(4);
  output_size->data[0] = op->desc.batch;
  output_size->data[1] = out_h;
  output_size->data[2] = out_w;
  output_size->data[3] = op->desc.channels_packed;
  return context->ResizeTensor(context, output, output_size);
}

TfLiteStatus BMaxPoolEval(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<BMaxPoolOpData*>(node->user_data);
  TfLiteTensor* output = GetOutput(context, node, 0);
  const TfLiteTensor* input = GetInput(context, node, 0);
  return WithDeviceIO(context, &op->staging, input, output,
                      [&](const void* in_dev, void* out_dev) -> TfLiteStatus {
                        LCE_ENSURE_CAPI(context,
                                        lce_b200_bmaxpool(&op->desc,
                                                          static_cast<const int32_t*>(in_dev),
                                                          static_cast<int32_t*>(out_dev),
                                                          g_stream));
                        return kTfLiteOk;
                      });
}

// ------------------------------------------------------------------------- //
// Two residual blocks in one node (Graph::FuseResidualPairs):
// [x0 packed, f1, mul1, bias1, thr1, x0, f2, mul2, bias2, thr2] -> [x2, packed x2?].
// Options: [uint32 n][layer 1's n option bytes][layer 2's option bytes]; builtin_data: the two
// ADD activations (int32[2]). Each layer keeps the op data of a plain LceBconv2d.
// ------------------------------------------------------------------------- //
struct PairOpData {
  BconvOpData* layer[2] = {nullptr, nullptr};
  ~PairOpData() {
    delete layer[0];
    delete layer[1];
  }
};

void* PairInit(TfLiteContext* context, const char* buffer, size_t length) {
  auto* op = new PairOpData();
  uint32_t n = 0;
  if (length >= 4) memcpy(&n, buffer, 4);
  if (length < 4 || n > length - 4) {
    context->ReportError(context, "LceBconv2d pair: malformed options");
    op->layer[0] = new BconvOpData();
    op->layer[1] = new BconvOpData();
    return op;
  }
  op->layer[0] = static_cast<BconvOpData*>(BconvInit(context, buffer + 4, n));
  op->layer[1] = static_cast<BconvOpData*>(BconvInit(context, buffer + 4 + n, length - 4 - n));
  return op;
}
void PairFree(TfLiteContext*, void* buffer) { delete static_cast<PairOpData*>(buffer); }

// Layer k of a pair node seen as a plain LceBconv2d node [x0 packed, filter, mul, bias, thr] ->
// [x2]: x1 has x2's shape and x0's packed shape, so both layers check against the same tensors.
struct PairLayerView {
  TfLiteNode node{};
  PairLayerView(const TfLiteNode* pair, int k, void* user_data) {
    node.inputs = LceB200IntArrayCreate(5);
    node.inputs->data[0] = pair->inputs->data[0];
    for (int i = 1; i < 5; ++i) node.inputs->data[i] = pair->inputs->data[5 * k + i];
    node.outputs = LceB200IntArrayCreate(1);
    node.outputs->data[0] = pair->outputs->data[0];
    node.user_data = user_data;
  }
  ~PairLayerView() {
    LceB200IntArrayFree(node.inputs);
    LceB200IntArrayFree(node.outputs);
  }
};

template <KernelType kt>
TfLiteStatus PairPrepare(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<PairOpData*>(node->user_data);
  LCE_ENSURE(context, node->inputs->size == 10);
  LCE_ENSURE(context, node->outputs->size == 1 || node->outputs->size == 2);
  for (int k = 0; k < 2; ++k) {
    PairLayerView v(node, k, op->layer[k]);
    if (BconvPrepare<kt>(context, &v.node) != kTfLiteOk) return kTfLiteError;
  }
  const lce_bconv2d_desc& d = op->layer[1]->desc;
  const TfLiteTensor* residual = GetInput(context, node, 5);
  LCE_ENSURE(context, GetOutput(context, node, 0)->type == kTfLiteFloat32);
  LCE_ENSURE(context, residual != nullptr && residual->type == kTfLiteFloat32 && NumDims(residual) == 4);
  LCE_ENSURE(context, Dim(residual, 0) == d.batch && Dim(residual, 1) == d.in_h &&
                          Dim(residual, 2) == d.in_w && Dim(residual, 3) == d.channels_out);
  if (node->outputs->size > 1) {
    TfLiteIntArray* packed_shape = LceB200IntArrayCreate(4);
    packed_shape->data[0] = d.batch;
    packed_shape->data[1] = d.in_h;
    packed_shape->data[2] = d.in_w;
    packed_shape->data[3] = BitpackedSize(d.channels_out);
    if (context->ResizeTensor(context, GetOutput(context, node, 1), packed_shape) != kTfLiteOk)
      return kTfLiteError;
  }
  return kTfLiteOk;
}

TfLiteStatus PairEval(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<PairOpData*>(node->user_data);
  for (int k = 0; k < 2; ++k) {
    PairLayerView v(node, k, op->layer[k]);
    if (BconvEnsurePlan(context, &v.node) != kTfLiteOk) return kTfLiteError;
  }
  const TfLiteTensor* input = GetInput(context, node, 0);
  const TfLiteTensor* residual = GetInput(context, node, 5);
  TfLiteTensor* output = GetOutput(context, node, 0);
  TfLiteTensor* packed = node->outputs->size > 1 ? GetOutput(context, node, 1) : nullptr;
  const int32_t* act = static_cast<const int32_t*>(node->builtin_data);
  LCE_ENSURE(context, act != nullptr);
  LCE_ENSURE_MSG(context, OnDevice(input->data.raw) && OnDevice(output->data.raw) &&
                              OnDevice(residual->data.raw),
                 "fused LceBconv2d pair needs a device arena");
  LCE_ENSURE_CAPI(context, lce_b200_bconv2d_run_fused_pair(
                               op->layer[0]->plan, op->layer[1]->plan, input->data.i32,
                               residual->data.f, act[0], act[1], output->data.f,
                               packed ? packed->data.i32 : nullptr, g_stream));
  return kTfLiteOk;
}

// ------------------------------------------------------------------------- //
// Real-to-Binary's gated block in one node (Graph::FuseChannelGates):
// [in, filter, mul, bias, thr, residual, gate [B,1,1,C], alpha, sign_scale, sign_shift]
// -> [out, packed_out?]; absent vectors are -1; builtin_data: the shortcut ADD's activation.
// ------------------------------------------------------------------------- //
// The node seen as a fused residual block [in, filter, mul, bias, thr, residual] -> its outputs.
struct GateBlockView {
  TfLiteNode node{};
  explicit GateBlockView(const TfLiteNode* gated) {
    node.inputs = LceB200IntArrayCreate(6);
    for (int i = 0; i < 6; ++i) node.inputs->data[i] = gated->inputs->data[i];
    node.outputs = LceB200IntArrayCreate(gated->outputs->size);
    for (int i = 0; i < gated->outputs->size; ++i) node.outputs->data[i] = gated->outputs->data[i];
    node.user_data = gated->user_data;
  }
  ~GateBlockView() {
    LceB200IntArrayFree(node.inputs);
    LceB200IntArrayFree(node.outputs);
  }
};

template <KernelType kt>
TfLiteStatus GatePrepare(TfLiteContext* context, TfLiteNode* node) {
  LCE_ENSURE(context, node->inputs->size == 10);
  GateBlockView v(node);
  if (BconvPrepare<kt, true>(context, &v.node) != kTfLiteOk) return kTfLiteError;
  const lce_bconv2d_desc& d = static_cast<BconvOpData*>(node->user_data)->desc;
  const TfLiteTensor* gate = GetInput(context, node, 6);
  LCE_ENSURE_MSG(context,
                 gate != nullptr && gate->type == kTfLiteFloat32 && NumDims(gate) == 4 &&
                     Dim(gate, 0) == d.batch && Dim(gate, 1) == 1 && Dim(gate, 2) == 1 &&
                     Dim(gate, 3) == d.channels_out,
                 "gated LceBconv2d: the gate must be a float32 [batch, 1, 1, channels_out] tensor");
  for (int k = 7; k < 10; ++k) {
    const TfLiteTensor* t = GetInput(context, node, k);
    LCE_ENSURE(context, t == nullptr || (t->type == kTfLiteFloat32 && NumElements(t) == d.channels_out));
  }
  return kTfLiteOk;
}

TfLiteStatus GateEval(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<BconvOpData*>(node->user_data);
  if (BconvEnsurePlan(context, node) != kTfLiteOk) return kTfLiteError;
  const TfLiteTensor* input = GetInput(context, node, 0);
  const TfLiteTensor* residual = GetInput(context, node, 5);
  const TfLiteTensor* gate = GetInput(context, node, 6);
  TfLiteTensor* output = GetOutput(context, node, 0);
  TfLiteTensor* packed = node->outputs->size > 1 ? GetOutput(context, node, 1) : nullptr;
  int add_act = LCE_ACT_NONE;
  if (node->builtin_data) add_act = *static_cast<const int32_t*>(node->builtin_data);
  LCE_ENSURE_MSG(context, OnDevice(input->data.raw) && OnDevice(output->data.raw) &&
                              OnDevice(residual->data.raw) && OnDevice(gate->data.raw),
                 "gated LceBconv2d needs a device arena");
  auto vec = [&](int k) {
    const TfLiteTensor* v = GetInput(context, node, k);
    return v ? v->data.f : nullptr;
  };
  const lce_gate_desc gd{gate->data.f, vec(7), vec(8), vec(9)};
  LCE_ENSURE_CAPI(context, lce_b200_bconv2d_run_fused_gate(
                               op->plan, input->data.i32, &gd, residual->data.f, add_act,
                               output->data.f, packed ? packed->data.i32 : nullptr, g_stream));
  return kTfLiteOk;
}

// ------------------------------------------------------------------------- //
// XNOR-Net++'s scaled block in one node (Graph::FuseSpatialScales):
// [in, filter, mul, bias, thr, residual, scale [1,OH,OW,C] or [OH,OW,C], sign_scale, sign_shift]
// -> [out, packed_out?]; absent vectors are -1; builtin_data: the shortcut ADD's activation.
// ------------------------------------------------------------------------- //
template <KernelType kt>
TfLiteStatus ScalePrepare(TfLiteContext* context, TfLiteNode* node) {
  LCE_ENSURE(context, node->inputs->size == 9);
  GateBlockView v(node);
  if (BconvPrepare<kt, true>(context, &v.node) != kTfLiteOk) return kTfLiteError;
  const lce_bconv2d_desc& d = static_cast<BconvOpData*>(node->user_data)->desc;
  const TfLiteTensor* out = GetOutput(context, node, 0);
  const TfLiteTensor* scale = GetInput(context, node, 6);
  const int r = scale ? NumDims(scale) : 0;
  LCE_ENSURE_MSG(context,
                 scale != nullptr && scale->type == kTfLiteFloat32 && (r == 3 || (r == 4 && Dim(scale, 0) == 1)) &&
                     Dim(scale, r - 3) == Dim(out, 1) && Dim(scale, r - 2) == Dim(out, 2) &&
                     Dim(scale, r - 1) == d.channels_out,
                 "scaled LceBconv2d: the scale must be a float32 [1, out_h, out_w, channels_out] tensor");
  for (int k = 7; k < 9; ++k) {
    const TfLiteTensor* t = GetInput(context, node, k);
    LCE_ENSURE(context, t == nullptr || (t->type == kTfLiteFloat32 && NumElements(t) == d.channels_out));
  }
  return kTfLiteOk;
}

TfLiteStatus ScaleEval(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<BconvOpData*>(node->user_data);
  if (BconvEnsurePlan(context, node) != kTfLiteOk) return kTfLiteError;
  const TfLiteTensor* input = GetInput(context, node, 0);
  const TfLiteTensor* residual = GetInput(context, node, 5);
  const TfLiteTensor* scale = GetInput(context, node, 6);
  TfLiteTensor* output = GetOutput(context, node, 0);
  TfLiteTensor* packed = node->outputs->size > 1 ? GetOutput(context, node, 1) : nullptr;
  int add_act = LCE_ACT_NONE;
  if (node->builtin_data) add_act = *static_cast<const int32_t*>(node->builtin_data);
  LCE_ENSURE_MSG(context, OnDevice(input->data.raw) && OnDevice(output->data.raw) &&
                              OnDevice(residual->data.raw) && OnDevice(scale->data.raw),
                 "scaled LceBconv2d needs a device arena");
  auto vec = [&](int k) {
    const TfLiteTensor* v = GetInput(context, node, k);
    return v ? v->data.f : nullptr;
  };
  const lce_scale_desc sd{scale->data.f, vec(7), vec(8)};
  LCE_ENSURE_CAPI(context, lce_b200_bconv2d_run_fused_scale(
                               op->plan, input->data.i32, &sd, residual->data.f, add_act,
                               output->data.f, packed ? packed->data.i32 : nullptr, g_stream));
  return kTfLiteOk;
}

// ------------------------------------------------------------------------- //
// An ABC-Net layer in one node (Graph::FuseBinaryBases): [q_0..q_{N-1}, (filter, mul, bias) of each
// term n * M + m, bn_scale, bn_shift, shortcut] -> [out if stored, next planes...]; builtin_data
// int32 {M, N, next planes, bn activation, shortcut activation, out stored} then the next shifts as
// floats; options are the terms' LceBconv2d options.
// ------------------------------------------------------------------------- //
struct BasesOpData {
  BconvOpData* conv = nullptr;   // the terms' parameters (desc)
  lce_b200_bconv2d_bases* plan = nullptr;
  ~BasesOpData() {
    lce_b200_bconv2d_bases_destroy(plan);
    delete conv;
  }
};
struct BasesNodeParams {
  int32_t m, n, n_next, bn_act, add_act, store;
  float shift[8];
};

void* BasesInit(TfLiteContext* context, const char* buffer, size_t length) {
  auto* op = new BasesOpData();
  op->conv = static_cast<BconvOpData*>(BconvInit(context, buffer, length));
  return op;
}
void BasesFree(TfLiteContext*, void* buffer) { delete static_cast<BasesOpData*>(buffer); }

bool BasesParamsOf(const TfLiteNode* node, BasesNodeParams* b) {
  if (!node->builtin_data) return false;
  memset(b, 0, sizeof(*b));
  memcpy(b, node->builtin_data, 6 * sizeof(int32_t));
  if (b->m < 1 || b->n < 1 || b->m > 8 || b->n > 8 || b->n_next < 0 || b->n_next > 8) return false;
  memcpy(b->shift, static_cast<const char*>(node->builtin_data) + 6 * sizeof(int32_t), b->n_next * sizeof(float));
  return true;
}

TfLiteStatus BasesPrepare(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<BasesOpData*>(node->user_data);
  if (!op->conv->successfully_initialized) return kTfLiteError;
  BasesNodeParams bp;
  LCE_ENSURE(context, BasesParamsOf(node, &bp));
  const int T = bp.m * bp.n;
  LCE_ENSURE(context, node->inputs->size == bp.n + 3 * T + 3);
  LCE_ENSURE(context, node->outputs->size == bp.store + bp.n_next);
  lce_bconv2d_desc& d = op->conv->desc;
  const TfLiteTensor* input = GetInput(context, node, 0);
  const TfLiteTensor* filter = GetInput(context, node, bp.n);
  LCE_ENSURE(context, input != nullptr && filter != nullptr && NumDims(input) == 4 && NumDims(filter) == 4);
  LCE_ENSURE(context, input->type == kTfLiteInt32 && filter->type == kTfLiteInt32);
  for (int k = 1; k < bp.n; ++k) {
    const TfLiteTensor* q = GetInput(context, node, k);
    LCE_ENSURE(context, q != nullptr && q->type == kTfLiteInt32 && NumDims(q) == 4);
    for (int a = 0; a < 4; ++a) LCE_ENSURE(context, Dim(q, a) == Dim(input, a));
  }
  d.channels_out = Dim(filter, 0);
  d.filter_h = Dim(filter, 1);
  d.filter_w = Dim(filter, 2);
  d.groups = 1;
  LCE_ENSURE(context, Dim(filter, 3) == BitpackedSize(d.channels_in) && Dim(input, 3) == Dim(filter, 3));
  d.out_type = LCE_OUT_FLOAT;
  d.batch = Dim(input, 0);
  d.in_h = Dim(input, 1);
  d.in_w = Dim(input, 2);
  int out_h, out_w, pad_h, pad_w;
  LCE_ENSURE_CAPI(context, lce_b200_bconv2d_out_shape(&d, &out_h, &out_w, &pad_h, &pad_w));
  for (int t = 0; t < T; ++t) {
    const TfLiteTensor* f = GetInput(context, node, bp.n + 3 * t);
    const TfLiteTensor* mul = GetInput(context, node, bp.n + 3 * t + 1);
    const TfLiteTensor* bias = GetInput(context, node, bp.n + 3 * t + 2);
    LCE_ENSURE(context, f != nullptr && f->type == kTfLiteInt32 && NumElements(f) == NumElements(filter));
    LCE_ENSURE(context, mul != nullptr && mul->type == kTfLiteFloat32 && NumElements(mul) == d.channels_out);
    LCE_ENSURE(context, bias != nullptr && bias->type == kTfLiteFloat32 && NumElements(bias) == d.channels_out);
  }
  for (int k = 0; k < 2; ++k) {
    const TfLiteTensor* v = GetInput(context, node, bp.n + 3 * T + k);
    LCE_ENSURE(context, v != nullptr && v->type == kTfLiteFloat32 && NumElements(v) == d.channels_out);
  }
  const TfLiteTensor* residual = GetInput(context, node, bp.n + 3 * T + 2);
  if (residual != nullptr) {
    LCE_ENSURE(context, residual->type == kTfLiteFloat32 && NumDims(residual) == 4);
    LCE_ENSURE(context, Dim(residual, 0) == d.batch && Dim(residual, 1) == out_h && Dim(residual, 2) == out_w &&
                            Dim(residual, 3) == d.channels_out);
  }
  for (int k = 0; k < node->outputs->size; ++k) {
    TfLiteTensor* o = GetOutput(context, node, k);
    const bool is_out = bp.store && k == 0;
    LCE_ENSURE(context, o->type == (is_out ? kTfLiteFloat32 : kTfLiteInt32));
    TfLiteIntArray* shape = LceB200IntArrayCreate(4);
    shape->data[0] = d.batch;
    shape->data[1] = out_h;
    shape->data[2] = out_w;
    shape->data[3] = is_out ? d.channels_out : BitpackedSize(d.channels_out);
    if (context->ResizeTensor(context, o, shape) != kTfLiteOk) return kTfLiteError;
  }
  op->conv->plan_stale = true;
  return kTfLiteOk;
}

TfLiteStatus BasesEval(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<BasesOpData*>(node->user_data);
  BasesNodeParams bp;
  LCE_ENSURE(context, BasesParamsOf(node, &bp));
  const int T = bp.m * bp.n;
  const lce_bconv2d_desc& d = op->conv->desc;
  if (op->plan == nullptr) {
    // the constants are the graph's and do not change; later Prepares only resize the input
    std::vector<lce_bconv2d_desc> descs(T, d);
    std::vector<const int32_t*> filters(T);
    std::vector<const float*> muls(T), biases(T);
    for (int t = 0; t < T; ++t) {
      filters[t] = GetInput(context, node, bp.n + 3 * t)->data.i32;
      muls[t] = GetInput(context, node, bp.n + 3 * t + 1)->data.f;
      biases[t] = GetInput(context, node, bp.n + 3 * t + 2)->data.f;
    }
    LCE_ENSURE_CAPI(context, lce_b200_bconv2d_bases_create(bp.m, bp.n, descs.data(), filters.data(), muls.data(),
                                                           biases.data(), &op->plan));
    op->conv->plan_stale = true;
  }
  if (op->conv->plan_stale) {
    LCE_ENSURE_CAPI(context, lce_b200_bconv2d_bases_set_input_shape(op->plan, d.batch, d.in_h, d.in_w));
    op->conv->plan_stale = false;
  }
  const int32_t* planes[8];
  for (int n = 0; n < bp.n; ++n) {
    const TfLiteTensor* q = GetInput(context, node, n);
    LCE_ENSURE_MSG(context, OnDevice(q->data.raw), "LceBconv2dBases needs a device arena");
    planes[n] = q->data.i32;
  }
  const TfLiteTensor* residual = GetInput(context, node, bp.n + 3 * T + 2);
  float* out = bp.store ? GetOutput(context, node, 0)->data.f : nullptr;
  int32_t* next[8];
  for (int k = 0; k < bp.n_next; ++k) next[k] = GetOutput(context, node, bp.store + k)->data.i32;
  LCE_ENSURE_CAPI(context, lce_b200_bconv2d_bases_run(
                               op->plan, planes, GetInput(context, node, bp.n + 3 * T)->data.f,
                               GetInput(context, node, bp.n + 3 * T + 1)->data.f, bp.bn_act,
                               residual ? residual->data.f : nullptr, bp.add_act, out, bp.n_next, bp.shift,
                               next, g_stream));
  return kTfLiteOk;
}

// ABC-Net's shifted signs of a float map in one node (Graph::FuseBinaryBases): [x] -> [q_0..q_{N-1}];
// builtin_data int32 N then the N shifts as floats.
TfLiteStatus ShiftPlanesPrepare(TfLiteContext* context, TfLiteNode* node) {
  LCE_ENSURE(context, node->inputs->size == 1 && node->builtin_data != nullptr);
  int32_t n = 0;
  memcpy(&n, node->builtin_data, sizeof(n));
  LCE_ENSURE(context, n >= 1 && n <= 8 && node->outputs->size == n);
  const TfLiteTensor* x = GetInput(context, node, 0);
  LCE_ENSURE(context, x != nullptr && x->type == kTfLiteFloat32 && NumDims(x) >= 1);
  LCE_ENSURE(context, Dim(x, NumDims(x) - 1) % 32 == 0);
  for (int k = 0; k < n; ++k) {
    TfLiteTensor* q = GetOutput(context, node, k);
    LCE_ENSURE(context, q->type == kTfLiteInt32);
    TfLiteIntArray* shape = LceB200IntArrayCreate(NumDims(x));
    for (int a = 0; a < NumDims(x); ++a) shape->data[a] = Dim(x, a);
    shape->data[shape->size - 1] = BitpackedSize(Dim(x, NumDims(x) - 1));
    if (context->ResizeTensor(context, q, shape) != kTfLiteOk) return kTfLiteError;
  }
  return kTfLiteOk;
}

TfLiteStatus ShiftPlanesEval(TfLiteContext* context, TfLiteNode* node) {
  int32_t n = 0;
  memcpy(&n, node->builtin_data, sizeof(n));
  float shifts[8];
  memcpy(shifts, static_cast<const char*>(node->builtin_data) + sizeof(n), n * sizeof(float));
  const TfLiteTensor* x = GetInput(context, node, 0);
  int32_t* planes[8];
  for (int k = 0; k < n; ++k) planes[k] = GetOutput(context, node, k)->data.i32;
  LCE_ENSURE_MSG(context, OnDevice(x->data.raw) && OnDevice(planes[0]), "shifted signs need a device arena");
  const int c = Dim(x, NumDims(x) - 1);
  LCE_ENSURE_CAPI(context, lce_b200_f32_shift_sign_planes(x->data.f, NumElements(x) / c, c, n, shifts, planes,
                                                          g_stream));
  return kTfLiteOk;
}

// ------------------------------------------------------------------------- //
// A BinaryDenseNet dense layer or a MeliusNet improvement layer in one node
// (Graph::FuseDenseBlocks): [src, scale, shift, filter, mul, bias, thr] -> [X]. X is the block's
// final map [B, H, W, C_L]; builtin_data: int32 {C_L, the layer kind (kDenseLayer /
// kImprovementLayer)}; options are the layer's LceBconv2d options, so C_j = channels_in. The node
// packs the signs of src[..., :C_j] * scale + shift, then
//   dense layer, temporaries [packed signs]: writes the convolution's channels_out new channels to
//     X[..., C_j : C_j + channels_out];
//   improvement layer, temporaries [packed signs, scratch]: adds them to X[..., C_j - channels_out :
//     C_j] in place; the scratch is [B, H, W, channels_out] for a zero-padding CORRECTION plan
//     (lce_b200_bconv2d_run_slice_add) and empty otherwise.
// src is x_0 for a block's first layer, which also copies x_0 into X[..., :C_j] and sets X's
// shape, and X for the others.
// ------------------------------------------------------------------------- //
enum { kDenseLayer = 0, kImprovementLayer = 1 };

// The node seen as a plain LceBconv2d node [packed signs, filter, mul, bias, thr] -> [X].
struct DenseLayerView {
  TfLiteNode node{};
  explicit DenseLayerView(const TfLiteNode* dense) {
    node.inputs = LceB200IntArrayCreate(5);
    node.inputs->data[0] = dense->temporaries->data[0];
    for (int i = 1; i < 5; ++i) node.inputs->data[i] = dense->inputs->data[2 + i];
    node.outputs = LceB200IntArrayCreate(1);
    node.outputs->data[0] = dense->outputs->data[0];
    node.user_data = dense->user_data;
  }
  ~DenseLayerView() {
    LceB200IntArrayFree(node.inputs);
    LceB200IntArrayFree(node.outputs);
  }
};

TfLiteStatus ResizeTo(TfLiteContext* context, TfLiteTensor* t, int b, int h, int w, int c) {
  TfLiteIntArray* dims = LceB200IntArrayCreate(4);
  dims->data[0] = b;
  dims->data[1] = h;
  dims->data[2] = w;
  dims->data[3] = c;
  return context->ResizeTensor(context, t, dims);
}

TfLiteTensor* Temporary(TfLiteContext* context, TfLiteNode* node, int k) {
  return context->GetTensor ? context->GetTensor(context, node->temporaries->data[k])
                            : &context->tensors[node->temporaries->data[k]];
}

template <KernelType kt>
TfLiteStatus DensePrepare(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<BconvOpData*>(node->user_data);
  if (!op->successfully_initialized) return kTfLiteError;
  LCE_ENSURE(context, node->inputs->size == 7 && node->outputs->size == 1 && node->builtin_data != nullptr);
  const int c_total = static_cast<const int32_t*>(node->builtin_data)[0];
  const int kind = static_cast<const int32_t*>(node->builtin_data)[1];
  LCE_ENSURE(context, (kind == kDenseLayer && node->temporaries->size == 1) ||
                          (kind == kImprovementLayer && node->temporaries->size == 2));
  const int c_in = op->desc.channels_in;
  const TfLiteTensor* src = GetInput(context, node, 0);
  TfLiteTensor* x = GetOutput(context, node, 0);
  TfLiteTensor* packed = Temporary(context, node, 0);
  LCE_ENSURE(context, src != nullptr && src->type == kTfLiteFloat32 && NumDims(src) == 4);
  LCE_ENSURE(context, x->type == kTfLiteFloat32 && packed->type == kTfLiteInt32);
  const int b = Dim(src, 0), h = Dim(src, 1), w = Dim(src, 2);
  if (node->inputs->data[0] != node->outputs->data[0]) {
    // the block's first layer: X takes x_0's pixels
    LCE_ENSURE(context, Dim(src, 3) == c_in);
  } else {
    LCE_ENSURE_MSG(context, Dim(x, 3) == c_total, "dense layer: the block's map has another channel count");
  }
  for (int k = 1; k < 3; ++k) {
    const TfLiteTensor* v = GetInput(context, node, k);
    LCE_ENSURE(context, v == nullptr || (v->type == kTfLiteFloat32 && NumElements(v) == c_in));
  }
  if (ResizeTo(context, packed, b, h, w, BitpackedSize(c_in)) != kTfLiteOk) return kTfLiteError;
  DenseLayerView v(node);
  if (BconvPrepare<kt>(context, &v.node) != kTfLiteOk) return kTfLiteError;
  // BconvPrepare gave X the convolution's output shape: the layer keeps the image size and its new
  // channels fit X (a dense layer's after C_j, an improvement layer's before); then X takes the
  // block's shape again
  const int c_out = op->desc.channels_out;
  LCE_ENSURE(context, op->desc.out_type == LCE_OUT_FLOAT && Dim(x, 1) == h && Dim(x, 2) == w &&
                          (kind == kDenseLayer ? c_in + c_out <= c_total : c_out <= c_in && c_in <= c_total));
  if (kind == kImprovementLayer) {
    TfLiteTensor* scratch = Temporary(context, node, 1);
    LCE_ENSURE(context, scratch->type == kTfLiteFloat32);
    const bool corr = op->zp_mode == LCE_ZERO_PADDING_CORRECTION;
    if (ResizeTo(context, scratch, b, h, w, corr ? c_out : 0) != kTfLiteOk) return kTfLiteError;
  }
  return ResizeTo(context, x, b, h, w, c_total);
}

TfLiteStatus DenseEval(TfLiteContext* context, TfLiteNode* node) {
  auto* op = static_cast<BconvOpData*>(node->user_data);
  DenseLayerView v(node);
  if (BconvEnsurePlan(context, &v.node) != kTfLiteOk) return kTfLiteError;
  const TfLiteTensor* src = GetInput(context, node, 0);
  const TfLiteTensor* scale = GetInput(context, node, 1);
  const TfLiteTensor* shift = GetInput(context, node, 2);
  TfLiteTensor* x = GetOutput(context, node, 0);
  TfLiteTensor* packed = Temporary(context, node, 0);
  LCE_ENSURE_MSG(context, OnDevice(src->data.raw) && OnDevice(x->data.raw) && OnDevice(packed->data.raw),
                 "dense LceBconv2d needs a device arena");
  const int c_in = op->desc.channels_in, c_total = Dim(x, 3);
  const bool first = node->inputs->data[0] != node->outputs->data[0];
  const int64_t rows = static_cast<int64_t>(Dim(x, 0)) * Dim(x, 1) * Dim(x, 2);
  LCE_ENSURE_CAPI(context, lce_b200_f32_affine_sign(src->data.f, Dim(src, 3), rows, c_in,
                                                    scale ? scale->data.f : nullptr,
                                                    shift ? shift->data.f : nullptr, packed->data.i32,
                                                    first ? x->data.f : nullptr, c_total, g_stream));
  if (static_cast<const int32_t*>(node->builtin_data)[1] == kImprovementLayer) {
    TfLiteTensor* scratch = Temporary(context, node, 1);
    LCE_ENSURE_CAPI(context, lce_b200_bconv2d_run_slice_add(
                                 op->plan, packed->data.i32, x->data.f + c_in - op->desc.channels_out,
                                 c_total, scratch->bytes ? scratch->data.f : nullptr, g_stream));
    return kTfLiteOk;
  }
  LCE_ENSURE_CAPI(context, lce_b200_bconv2d_run_slice(op->plan, packed->data.i32, x->data.f + c_in,
                                                      c_total, g_stream));
  return kTfLiteOk;
}

template <KernelType kt>
TfLiteRegistration* BconvDenseRegistration() {
  static TfLiteRegistration r = {BconvInit, BconvFree, DensePrepare<kt>, DenseEval};
  return &r;
}

template <KernelType kt>
TfLiteRegistration* BconvGateRegistration() {
  static TfLiteRegistration r = {BconvInit, BconvFree, GatePrepare<kt>, GateEval};
  return &r;
}

template <KernelType kt>
TfLiteRegistration* BconvScaleRegistration() {
  static TfLiteRegistration r = {BconvInit, BconvFree, ScalePrepare<kt>, ScaleEval};
  return &r;
}

template <KernelType kt>
TfLiteRegistration* BconvPairRegistration() {
  static TfLiteRegistration r = {PairInit, PairFree, PairPrepare<kt>, PairEval};
  return &r;
}

template <KernelType kt>
TfLiteRegistration* BconvFusedRegistration() {
  static TfLiteRegistration r = {BconvInit, BconvFree, BconvPrepare<kt, true>, BconvFusedEval};
  return &r;
}

template <KernelType kt>
TfLiteRegistration* BconvRegistration() {
  static TfLiteRegistration r = {BconvInit, BconvFree, BconvPrepare<kt>, BconvEval};
  return &r;
}

}  // namespace

extern "C" {

#ifndef LCE_B200_USE_TFLITE_HEADERS
TfLiteIntArray* LceB200IntArrayCreate(int size) {
  auto* a = static_cast<TfLiteIntArray*>(
      malloc(sizeof(TfLiteIntArray) + sizeof(int) * (size > 0 ? size : 0)));
  if (a) a->size = size;
  return a;
}
void LceB200IntArrayFree(TfLiteIntArray* a) { free(a); }
#endif

// host-internal: the fused residual-block node created by Graph::FuseResidualBlocks
// The fused node keeps the validation rules and zero-padding result of the registration the
// LceBconv2d node was resolved to (nullptr: not one of this library's LceBconv2d registrations).
TfLiteRegistration* lce_b200_internal_Register_BCONV_2D_FUSED(const TfLiteRegistration* original) {
  if (original == BconvRegistration<KernelType::kCuda>()) return BconvFusedRegistration<KernelType::kCuda>();
  if (original == BconvRegistration<KernelType::kReference>())
    return BconvFusedRegistration<KernelType::kReference>();
  if (original == BconvRegistration<KernelType::kOptimizedBGEMM>())
    return BconvFusedRegistration<KernelType::kOptimizedBGEMM>();
  if (original == BconvRegistration<KernelType::kOptimizedIndirectBGEMM>())
    return BconvFusedRegistration<KernelType::kOptimizedIndirectBGEMM>();
  return nullptr;
}

// host-internal: the two-block node created by Graph::FuseResidualPairs from two fused nodes of
// this registration (nullptr: not one of this library's fused LceBconv2d registrations)
TfLiteRegistration* lce_b200_internal_Register_BCONV_2D_PAIR(const TfLiteRegistration* fused) {
  if (fused == BconvFusedRegistration<KernelType::kCuda>()) return BconvPairRegistration<KernelType::kCuda>();
  if (fused == BconvFusedRegistration<KernelType::kReference>())
    return BconvPairRegistration<KernelType::kReference>();
  if (fused == BconvFusedRegistration<KernelType::kOptimizedBGEMM>())
    return BconvPairRegistration<KernelType::kOptimizedBGEMM>();
  if (fused == BconvFusedRegistration<KernelType::kOptimizedIndirectBGEMM>())
    return BconvPairRegistration<KernelType::kOptimizedIndirectBGEMM>();
  return nullptr;
}

// host-internal: the gated-block node created by Graph::FuseChannelGates from a plain LceBconv2d
// node of this registration (nullptr: not one of this library's LceBconv2d registrations)
TfLiteRegistration* lce_b200_internal_Register_BCONV_2D_GATE(const TfLiteRegistration* original) {
  if (original == BconvRegistration<KernelType::kCuda>()) return BconvGateRegistration<KernelType::kCuda>();
  if (original == BconvRegistration<KernelType::kReference>())
    return BconvGateRegistration<KernelType::kReference>();
  if (original == BconvRegistration<KernelType::kOptimizedBGEMM>())
    return BconvGateRegistration<KernelType::kOptimizedBGEMM>();
  if (original == BconvRegistration<KernelType::kOptimizedIndirectBGEMM>())
    return BconvGateRegistration<KernelType::kOptimizedIndirectBGEMM>();
  return nullptr;
}

// host-internal: the scaled-block node created by Graph::FuseSpatialScales from a plain LceBconv2d
// node of this registration (nullptr: not one of this library's LceBconv2d registrations)
TfLiteRegistration* lce_b200_internal_Register_BCONV_2D_SCALE(const TfLiteRegistration* original) {
  if (original == BconvRegistration<KernelType::kCuda>()) return BconvScaleRegistration<KernelType::kCuda>();
  if (original == BconvRegistration<KernelType::kReference>())
    return BconvScaleRegistration<KernelType::kReference>();
  if (original == BconvRegistration<KernelType::kOptimizedBGEMM>())
    return BconvScaleRegistration<KernelType::kOptimizedBGEMM>();
  if (original == BconvRegistration<KernelType::kOptimizedIndirectBGEMM>())
    return BconvScaleRegistration<KernelType::kOptimizedIndirectBGEMM>();
  return nullptr;
}

// host-internal: the ABC-Net layer node created by Graph::FuseBinaryBases from plain LceBconv2d nodes
// of this registration (nullptr: not one of this library's LceBconv2d registrations). The terms are
// one-padded or VALID, where every registration computes the same integers, so one node serves all.
TfLiteRegistration* lce_b200_internal_Register_BCONV_2D_BASES(const TfLiteRegistration* original) {
  static TfLiteRegistration r = {BasesInit, BasesFree, BasesPrepare, BasesEval};
  if (original == BconvRegistration<KernelType::kCuda>() || original == BconvRegistration<KernelType::kReference>() ||
      original == BconvRegistration<KernelType::kOptimizedBGEMM>() ||
      original == BconvRegistration<KernelType::kOptimizedIndirectBGEMM>())
    return &r;
  return nullptr;
}

// host-internal: Graph::FuseBinaryBases's one-pass shifted signs
TfLiteRegistration* lce_b200_internal_Register_SHIFT_SIGN_PLANES(void) {
  static TfLiteRegistration r = {nullptr, nullptr, ShiftPlanesPrepare, ShiftPlanesEval};
  return &r;
}

// host-internal: the dense- or improvement-layer node created by Graph::FuseDenseBlocks from a plain
// LceBconv2d node of this registration (nullptr: not one of this library's LceBconv2d registrations)
TfLiteRegistration* lce_b200_internal_Register_BCONV_2D_DENSE(const TfLiteRegistration* original) {
  if (original == BconvRegistration<KernelType::kCuda>()) return BconvDenseRegistration<KernelType::kCuda>();
  if (original == BconvRegistration<KernelType::kReference>())
    return BconvDenseRegistration<KernelType::kReference>();
  if (original == BconvRegistration<KernelType::kOptimizedBGEMM>())
    return BconvDenseRegistration<KernelType::kOptimizedBGEMM>();
  if (original == BconvRegistration<KernelType::kOptimizedIndirectBGEMM>())
    return BconvDenseRegistration<KernelType::kOptimizedIndirectBGEMM>();
  return nullptr;
}

void lce_b200_set_stream(void* stream) { g_stream = stream; }
void* lce_b200_get_stream(void) { return g_stream; }

TfLiteRegistration* lce_b200_Register_QUANTIZE(void) {
  static TfLiteRegistration r = {nullptr, nullptr, QuantizePrepare, QuantizeEval};
  return &r;
}
TfLiteRegistration* lce_b200_Register_DEQUANTIZE(void) {
  static TfLiteRegistration r = {nullptr, nullptr, DequantizePrepare, DequantizeEval};
  return &r;
}
TfLiteRegistration* lce_b200_Register_BCONV_2D_REF(void) {
  return BconvRegistration<KernelType::kReference>();
}
TfLiteRegistration* lce_b200_Register_BCONV_2D_OPT_BGEMM(void) {
  return BconvRegistration<KernelType::kOptimizedBGEMM>();
}
TfLiteRegistration* lce_b200_Register_BCONV_2D_OPT_INDIRECT_BGEMM(void) {
  return BconvRegistration<KernelType::kOptimizedIndirectBGEMM>();
}
TfLiteRegistration* lce_b200_Register_BCONV_2D(void) {
  return BconvRegistration<KernelType::kCuda>();
}
TfLiteRegistration* lce_b200_Register_BMAXPOOL_2D(void) {
  static TfLiteRegistration r = {BMaxPoolInit, BMaxPoolFree, BMaxPoolPrepare, BMaxPoolEval};
  return &r;
}

}  // extern "C"

namespace compute_engine {
namespace tflite {
TfLiteRegistration* Register_QUANTIZE() { return lce_b200_Register_QUANTIZE(); }
TfLiteRegistration* Register_DEQUANTIZE() { return lce_b200_Register_DEQUANTIZE(); }
TfLiteRegistration* Register_BCONV_2D() { return lce_b200_Register_BCONV_2D(); }
TfLiteRegistration* Register_BCONV_2D_REF() { return lce_b200_Register_BCONV_2D_REF(); }
TfLiteRegistration* Register_BCONV_2D_OPT_BGEMM() { return lce_b200_Register_BCONV_2D_OPT_BGEMM(); }
TfLiteRegistration* Register_BCONV_2D_OPT_INDIRECT_BGEMM() {
  return lce_b200_Register_BCONV_2D_OPT_INDIRECT_BGEMM();
}
TfLiteRegistration* Register_BMAXPOOL_2D() { return lce_b200_Register_BMAXPOOL_2D(); }
}  // namespace tflite
}  // namespace compute_engine

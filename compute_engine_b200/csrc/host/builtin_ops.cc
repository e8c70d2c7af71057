// builtin_ops.cc -- TfLiteRegistrations for the float builtins QuickNet /
// QuickNetLarge / Bi-RealNet-18 / ReActNet-A / Real-to-Binary Net use around the binary path, backed by
// the fp32 CUDA kernels of lce_b200_builtins.cu. Shape inference follows TFLite's
// builtin kernels (tensorflow/lite/kernels/{conv,depthwise_conv,pooling,add,mul,
// fully_connected,softmax,reduce,reshape,activations,logistic}.cc). Device arena only.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>

#include "builtin_params.h"
#include "flexbuffer_map.h"
#include "host_graph.h"
#include "lce_b200.h"
#include "lce_b200_builtins.h"

namespace lce_b200 {
namespace {

#define B_ENSURE(ctx, cond, msg)                 \
  do {                                           \
    if (!(cond)) {                               \
      (ctx)->ReportError((ctx), "%s", (msg));    \
      return kTfLiteError;                       \
    }                                            \
  } while (0)
#define B_CAPI(ctx, call)                                     \
  do {                                                        \
    if ((call) != 0) {                                        \
      (ctx)->ReportError((ctx), "%s", lce_b200_last_error()); \
      return kTfLiteError;                                    \
    }                                                         \
  } while (0)

TfLiteTensor* T(TfLiteContext* c, const TfLiteIntArray* a, int i) {
  if (i >= a->size || a->data[i] < 0) return nullptr;
  return &c->tensors[a->data[i]];
}
int64_t Count(const TfLiteTensor* t) {
  int64_t n = 1;
  for (int i = 0; i < t->dims->size; ++i) n *= t->dims->data[i];
  return n;
}
TfLiteStatus Resize(TfLiteContext* c, TfLiteTensor* t, std::initializer_list<int> dims) {
  TfLiteIntArray* a = LceB200IntArrayCreate(static_cast<int>(dims.size()));
  int i = 0;
  for (int d : dims) a->data[i++] = d;
  return c->ResizeTensor(c, t, a);
}
TfLiteStatus ResizeTo(TfLiteContext* c, TfLiteTensor* t, const std::vector<int>& dims) {
  TfLiteIntArray* a = LceB200IntArrayCreate(static_cast<int>(dims.size()));
  for (size_t i = 0; i < dims.size(); ++i) a->data[i] = dims[i];
  return c->ResizeTensor(c, t, a);
}
bool OnDevice(const void* p) {
  cudaPointerAttributes a;
  if (!p || cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

void* Init(TfLiteContext*, const char* buffer, size_t length) {
  auto* p = new BuiltinParams();
  memset(p, 0, sizeof(*p));
  if (buffer && length >= sizeof(BuiltinParams)) memcpy(p, buffer, sizeof(BuiltinParams));
  return p;
}
void Free(TfLiteContext*, void* p) { delete static_cast<BuiltinParams*>(p); }
const BuiltinParams& P(TfLiteNode* n) { return *static_cast<BuiltinParams*>(n->user_data); }

// ---------------------------- CONV_2D / DEPTHWISE ---------------------------- //
// groups (CONV_2D only): TFLite's conv.cc infers groups = in_c / filter_in from a filter
// [out_c, fh, fw, filter_in]; ConvGroupChecks tells whether that division and out_c / groups are exact.
bool ConvDesc(TfLiteContext* c, TfLiteNode* n, bool depthwise, lce_f32_conv_desc* d, int* groups = nullptr) {
  const TfLiteTensor* in = T(c, n->inputs, 0);
  const TfLiteTensor* f = T(c, n->inputs, 1);
  if (!in || !f || in->dims->size != 4 || f->dims->size != 4) return false;
  if (groups) *groups = 1;
  const BuiltinParams& p = P(n);
  d->batch = in->dims->data[0];
  d->in_h = in->dims->data[1];
  d->in_w = in->dims->data[2];
  d->in_c = in->dims->data[3];
  d->filter_h = f->dims->data[1];
  d->filter_w = f->dims->data[2];
  d->out_c = depthwise ? f->dims->data[3] : f->dims->data[0];
  d->stride_h = p.stride_h;
  d->stride_w = p.stride_w;
  d->dilation_h = p.dilation_h;
  d->dilation_w = p.dilation_w;
  d->padding = p.padding;
  d->activation = p.activation;
  if (!depthwise && f->dims->data[3] != d->in_c) {
    if (!groups || f->dims->data[3] < 1) return false;
    *groups = d->in_c / f->dims->data[3];
  }
  return true;
}
TfLiteStatus ConvGroupChecks(TfLiteContext* c, TfLiteNode* n, const lce_f32_conv_desc& d) {
  const int filter_in = T(c, n->inputs, 1)->dims->data[3];
  if (filter_in == d.in_c) return kTfLiteOk;
  B_ENSURE(c, d.in_c % filter_in == 0,
           "CONV_2D: the input's channels must be a multiple of the filter's input channels");
  B_ENSURE(c, d.out_c % (d.in_c / filter_in) == 0,
           "CONV_2D: the filter count must be a multiple of the group count");
  return kTfLiteOk;
}
template <bool DW>
TfLiteStatus ConvPrepare(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_conv_desc d;
  int groups = 1;
  B_ENSURE(c, ConvDesc(c, n, DW, &d, DW ? nullptr : &groups), "CONV_2D: bad input / filter shapes");
  B_ENSURE(c, T(c, n->inputs, 0)->type == kTfLiteFloat32, "CONV_2D: only float32 is supported");
  if (DW) B_ENSURE(c, P(n).depth_multiplier == 1 && d.out_c == d.in_c,
                   "DEPTHWISE_CONV_2D: depth_multiplier must be 1");
  if (!DW && ConvGroupChecks(c, n, d) != kTfLiteOk) return kTfLiteError;
  int oh, ow;
  B_CAPI(c, lce_b200_f32_conv_out_shape(&d, &oh, &ow));
  if (!DW && n->outputs->size == 2) {
    B_ENSURE(c, groups == 1, "CONV_2D+LceQuantize: grouped convolutions are not supported");
    // fused LceQuantize (Graph::FuseFloatGlue): second output = bitpacked signs of the first
    TfLiteTensor* pk = T(c, n->outputs, 1);
    B_ENSURE(c, pk && pk->type == kTfLiteInt32, "CONV_2D+LceQuantize: packed output must be int32");
    if (Resize(c, pk, {d.batch, oh, ow, (d.out_c + 31) / 32}) != kTfLiteOk) return kTfLiteError;
  }
  return Resize(c, T(c, n->outputs, 0), {d.batch, oh, ow, d.out_c});
}
template <bool DW>
TfLiteStatus ConvInvoke(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_conv_desc d;
  int groups = 1;
  ConvDesc(c, n, DW, &d, DW ? nullptr : &groups);
  const TfLiteTensor* in = T(c, n->inputs, 0);
  const TfLiteTensor* f = T(c, n->inputs, 1);
  const TfLiteTensor* bias = T(c, n->inputs, 2);
  TfLiteTensor* out = T(c, n->outputs, 0);
  B_ENSURE(c, OnDevice(in->data.raw) && OnDevice(f->data.raw) && OnDevice(out->data.raw),
           "float builtins need a device arena (no CPU path)");
  if (groups != 1)
    B_CAPI(c, lce_b200_f32_grouped_conv2d(&d, groups, in->data.f, f->data.f, bias ? bias->data.f : nullptr,
                                          nullptr, nullptr, LCE_ACT_NONE, out->data.f, lce_b200_get_stream()));
  else if (DW)
    B_CAPI(c, lce_b200_f32_depthwise_conv2d(&d, in->data.f, f->data.f, bias ? bias->data.f : nullptr,
                                             out->data.f, lce_b200_get_stream()));
  else if (n->outputs->size == 2)
    B_CAPI(c, lce_b200_f32_conv2d_packed(&d, in->data.f, f->data.f, bias ? bias->data.f : nullptr,
                                         out->data.f, T(c, n->outputs, 1)->data.i32,
                                         lce_b200_get_stream()));
  else
    B_CAPI(c, lce_b200_f32_conv2d(&d, in->data.f, f->data.f, bias ? bias->data.f : nullptr,
                                  out->data.f, lce_b200_get_stream()));
  return kTfLiteOk;
}

// -------------- fused grouped CONV_2D -> MUL(scale) -> ADD(shift): a BatchNorm after the conv -------------- //
// Created by Graph::FuseGroupedConvAffine; builtin_data = { BuiltinParams conv, BuiltinParams add };
// inputs [x, filter, bias (-1 when absent), scale, shift], scale and shift constants of out_c floats.
// Runs lce_b200_f32_grouped_conv2d with the epilogue, the ADD's activation as the post activation.
struct ConvAffineParams {
  BuiltinParams conv, add;
};
void* ConvAffineInit(TfLiteContext*, const char* buffer, size_t length) {
  auto* p = new ConvAffineParams();
  memset(p, 0, sizeof(*p));
  if (buffer && length >= sizeof(ConvAffineParams)) memcpy(p, buffer, sizeof(ConvAffineParams));
  return p;
}
void ConvAffineFree(TfLiteContext*, void* p) { delete static_cast<ConvAffineParams*>(p); }
TfLiteStatus ConvAffinePrepare(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_conv_desc d;
  int groups = 1;
  B_ENSURE(c, n->inputs->size == 5 && n->outputs->size == 1 && ConvDesc(c, n, false, &d, &groups),
           "CONV_2D+MUL+ADD: bad input / filter shapes");
  B_ENSURE(c, T(c, n->inputs, 0)->type == kTfLiteFloat32, "CONV_2D: only float32 is supported");
  if (ConvGroupChecks(c, n, d) != kTfLiteOk) return kTfLiteError;
  for (int k = 3; k < 5; ++k) {
    const TfLiteTensor* v = T(c, n->inputs, k);
    B_ENSURE(c, v && v->type == kTfLiteFloat32 && Count(v) == d.out_c,
             "CONV_2D+MUL+ADD: scale and shift must be float32 with one value per output channel");
  }
  int oh, ow;
  B_CAPI(c, lce_b200_f32_conv_out_shape(&d, &oh, &ow));
  return Resize(c, T(c, n->outputs, 0), {d.batch, oh, ow, d.out_c});
}
TfLiteStatus ConvAffineInvoke(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_conv_desc d;
  int groups = 1;
  ConvDesc(c, n, false, &d, &groups);
  const TfLiteTensor* bias = T(c, n->inputs, 2);
  const TfLiteTensor* scale = T(c, n->inputs, 3);
  const TfLiteTensor* shift = T(c, n->inputs, 4);
  TfLiteTensor* out = T(c, n->outputs, 0);
  B_ENSURE(c, OnDevice(T(c, n->inputs, 0)->data.raw) && OnDevice(out->data.raw) && OnDevice(scale->data.raw) &&
                  OnDevice(shift->data.raw),
           "float builtins need a device arena (no CPU path)");
  B_CAPI(c, lce_b200_f32_grouped_conv2d(&d, groups, T(c, n->inputs, 0)->data.f, T(c, n->inputs, 1)->data.f,
                                        bias ? bias->data.f : nullptr, scale->data.f, shift->data.f,
                                        static_cast<const ConvAffineParams*>(n->user_data)->add.activation,
                                        out->data.f, lce_b200_get_stream()));
  return kTfLiteOk;
}

// ------------------------------ FULLY_CONNECTED ------------------------------ //
TfLiteStatus FcPrepare(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* in = T(c, n->inputs, 0);
  const TfLiteTensor* w = T(c, n->inputs, 1);
  B_ENSURE(c, in && w && w->dims->size == 2, "FULLY_CONNECTED: weights must be [out, in]");
  const int k = w->dims->data[1];
  B_ENSURE(c, k > 0 && Count(in) % k == 0, "FULLY_CONNECTED: input size mismatch");
  if (!P(n).keep_dims) return Resize(c, T(c, n->outputs, 0), {static_cast<int>(Count(in) / k), w->dims->data[0]});
  // keep_num_dims: the input's shape with its last axis, which must be the weights' input size, now N
  B_ENSURE(c, in->dims->size >= 1 && in->dims->data[in->dims->size - 1] == k,
           "FULLY_CONNECTED: keep_num_dims needs the input's last axis to be the weights' input size");
  TfLiteIntArray* dims = LceB200IntArrayCreate(in->dims->size);
  for (int i = 0; i < in->dims->size; ++i) dims->data[i] = in->dims->data[i];
  dims->data[dims->size - 1] = w->dims->data[0];
  return c->ResizeTensor(c, T(c, n->outputs, 0), dims);
}
TfLiteStatus FcInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* in = T(c, n->inputs, 0);
  const TfLiteTensor* w = T(c, n->inputs, 1);
  const TfLiteTensor* bias = T(c, n->inputs, 2);
  TfLiteTensor* out = T(c, n->outputs, 0);
  lce_f32_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.batch = static_cast<int>(Count(in) / w->dims->data[1]);
  d.in_h = d.in_w = d.filter_h = d.filter_w = d.stride_h = d.stride_w = d.dilation_h =
      d.dilation_w = 1;
  d.in_c = w->dims->data[1];
  d.out_c = w->dims->data[0];
  d.padding = LCE_PADDING_VALID;
  d.activation = P(n).activation;
  B_CAPI(c, lce_b200_f32_conv2d(&d, in->data.f, w->data.f, bias ? bias->data.f : nullptr,
                                out->data.f, lce_b200_get_stream()));
  return kTfLiteOk;
}

// ---------------------------------- pooling ---------------------------------- //
bool PoolDesc(TfLiteContext* c, TfLiteNode* n, lce_f32_pool_desc* d) {
  const TfLiteTensor* in = T(c, n->inputs, 0);
  if (!in || in->dims->size != 4) return false;
  const BuiltinParams& p = P(n);
  d->batch = in->dims->data[0]; d->in_h = in->dims->data[1]; d->in_w = in->dims->data[2];
  d->channels = in->dims->data[3];
  d->filter_h = p.filter_h; d->filter_w = p.filter_w;
  d->stride_h = p.stride_h; d->stride_w = p.stride_w;
  d->padding = p.padding; d->activation = p.activation;
  return true;
}
TfLiteStatus PoolPrepare(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_pool_desc d;
  B_ENSURE(c, PoolDesc(c, n, &d), "POOL_2D: input must be 4-D");
  int oh, ow;
  B_CAPI(c, lce_b200_f32_pool_out_shape(&d, &oh, &ow));
  return Resize(c, T(c, n->outputs, 0), {d.batch, oh, ow, d.channels});
}
template <bool MAX>
TfLiteStatus PoolInvoke(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_pool_desc d;
  PoolDesc(c, n, &d);
  const float* in = T(c, n->inputs, 0)->data.f;
  float* out = T(c, n->outputs, 0)->data.f;
  if (MAX) B_CAPI(c, lce_b200_f32_max_pool(&d, in, out, lce_b200_get_stream()));
  else B_CAPI(c, lce_b200_f32_avg_pool(&d, in, out, lce_b200_get_stream()));
  return kTfLiteOk;
}

// --------------- fused MAX_POOL_2D -> MUL(scale) -> ADD(shift) -> LceQuantize --------------- //
// Created by Graph::FusePooledSigns; builtin_data = the pool's BuiltinParams; inputs [x, scale,
// shift], each constant [C] (or [1, ..., 1, C]) for x [B,H,W,C]; output the packed signs
// [B,OH,OW,ceil(C/32)], or [B, OH*OW*C/32] when the pass looked through a flattening RESHAPE.
TfLiteStatus PooledSignPrepare(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_pool_desc d;
  B_ENSURE(c, n->inputs->size == 3 && PoolDesc(c, n, &d) && T(c, n->inputs, 0)->type == kTfLiteFloat32,
           "MAX_POOL_2D+MUL+ADD+LceQuantize: a 4-D float32 input and two constants expected");
  for (int k = 1; k < 3; ++k) {
    const TfLiteTensor* v = T(c, n->inputs, k);
    B_ENSURE(c, v && v->type == kTfLiteFloat32 && Count(v) == d.channels,
             "MAX_POOL_2D+MUL+ADD+LceQuantize: scale and shift must be float32 with one value per channel");
  }
  TfLiteTensor* pk = T(c, n->outputs, 0);
  B_ENSURE(c, pk && pk->type == kTfLiteInt32, "MAX_POOL_2D+MUL+ADD+LceQuantize: packed output must be int32");
  int oh, ow;
  B_CAPI(c, lce_b200_f32_pool_out_shape(&d, &oh, &ow));
  // through a flattening RESHAPE (C % 32 == 0): the same words as [B, OH * OW * C / 32]
  if (pk->dims->size == 2) return Resize(c, pk, {d.batch, oh * ow * (d.channels / 32)});
  return Resize(c, pk, {d.batch, oh, ow, (d.channels + 31) / 32});
}
TfLiteStatus PooledSignInvoke(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_pool_desc d;
  PoolDesc(c, n, &d);
  const TfLiteTensor* scale = T(c, n->inputs, 1);
  const TfLiteTensor* shift = T(c, n->inputs, 2);
  B_ENSURE(c, OnDevice(scale->data.raw) && OnDevice(shift->data.raw),
           "MAX_POOL_2D+MUL+ADD+LceQuantize: constants must be device-resident");
  B_CAPI(c, lce_b200_f32_maxpool_affine_sign(T(c, n->inputs, 0)->data.f, d.batch, d.in_h, d.in_w, d.channels,
                                             d.filter_h, d.filter_w, d.stride_h, d.stride_w, d.padding,
                                             d.activation, scale->data.f, shift->data.f,
                                             T(c, n->outputs, 0)->data.i32, lce_b200_get_stream()));
  return kTfLiteOk;
}

// ------------- fused MAX_POOL_2D(2x2 s1 VALID) + DEPTHWISE_CONV_2D(3x3) ------------- //
// Created by Graph::FuseFloatGlue; builtin_data = { BuiltinParams pool, BuiltinParams dw }.
struct PoolDwParams {
  BuiltinParams pool, dw;
};
void* PoolDwInit(TfLiteContext*, const char* buffer, size_t length) {
  auto* p = new PoolDwParams();
  memset(p, 0, sizeof(*p));
  if (buffer && length >= sizeof(PoolDwParams)) memcpy(p, buffer, sizeof(PoolDwParams));
  return p;
}
void PoolDwFree(TfLiteContext*, void* p) { delete static_cast<PoolDwParams*>(p); }
bool PoolDwDescs(TfLiteContext* c, TfLiteNode* n, lce_f32_pool_desc* pd, lce_f32_conv_desc* dd) {
  const auto& pp = *static_cast<PoolDwParams*>(n->user_data);
  const TfLiteTensor* in = T(c, n->inputs, 0);
  const TfLiteTensor* f = T(c, n->inputs, 1);
  if (!in || !f || in->dims->size != 4 || f->dims->size != 4) return false;
  pd->batch = in->dims->data[0]; pd->in_h = in->dims->data[1]; pd->in_w = in->dims->data[2];
  pd->channels = in->dims->data[3];
  pd->filter_h = pp.pool.filter_h; pd->filter_w = pp.pool.filter_w;
  pd->stride_h = pp.pool.stride_h; pd->stride_w = pp.pool.stride_w;
  pd->padding = pp.pool.padding; pd->activation = pp.pool.activation;
  int ph, pw;
  if (lce_b200_f32_pool_out_shape(pd, &ph, &pw)) return false;
  dd->batch = pd->batch; dd->in_h = ph; dd->in_w = pw; dd->in_c = pd->channels;
  dd->filter_h = f->dims->data[1]; dd->filter_w = f->dims->data[2]; dd->out_c = f->dims->data[3];
  dd->stride_h = pp.dw.stride_h; dd->stride_w = pp.dw.stride_w;
  dd->dilation_h = pp.dw.dilation_h; dd->dilation_w = pp.dw.dilation_w;
  dd->padding = pp.dw.padding; dd->activation = pp.dw.activation;
  return true;
}
TfLiteStatus PoolDwPrepare(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_pool_desc pd;
  lce_f32_conv_desc dd;
  B_ENSURE(c, PoolDwDescs(c, n, &pd, &dd), "MAX_POOL_2D+DEPTHWISE_CONV_2D: bad shapes");
  int oh, ow;
  B_CAPI(c, lce_b200_f32_conv_out_shape(&dd, &oh, &ow));
  return Resize(c, T(c, n->outputs, 0), {dd.batch, oh, ow, dd.out_c});
}
TfLiteStatus PoolDwInvoke(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_pool_desc pd;
  lce_f32_conv_desc dd;
  PoolDwDescs(c, n, &pd, &dd);
  const TfLiteTensor* bias = T(c, n->inputs, 2);
  B_CAPI(c, lce_b200_f32_maxpool2x2_depthwise3x3(&pd, &dd, T(c, n->inputs, 0)->data.f,
                                                   T(c, n->inputs, 1)->data.f,
                                                   bias ? bias->data.f : nullptr,
                                                   T(c, n->outputs, 0)->data.f,
                                                   lce_b200_get_stream()));
  return kTfLiteOk;
}

// ---- fused stem [DEQUANTIZE +] CONV_2D(3x3 s2, 3 -> 16 or 8) + DEPTHWISE_CONV_2D(3x3 s2) ---- //
// Created by Graph::FuseStem; builtin_data = { conv1, depthwise } BuiltinParams;
// inputs [x (float32, or the int8 / uint8 input of the removed DEQUANTIZE), w1, b1, w2, b2].
struct StemBlob {
  BuiltinParams c1, dw;
};
struct StemParams {
  BuiltinParams c1, dw;
  // host copies of the (constant) filters and biases: the kernel takes them by value
  std::vector<float> w1, b1, w2, b2;
};
void* StemInit(TfLiteContext*, const char* buffer, size_t length) {
  auto* p = new StemParams();
  memset(&p->c1, 0, sizeof(p->c1));
  memset(&p->dw, 0, sizeof(p->dw));
  if (buffer && length >= sizeof(StemBlob)) {
    memcpy(&p->c1, buffer, sizeof(BuiltinParams));
    memcpy(&p->dw, buffer + sizeof(BuiltinParams), sizeof(BuiltinParams));
  }
  return p;
}
// Copy a constant float tensor to the host (device constants: one synchronous copy, at Prepare).
bool HostCopy(const TfLiteTensor* t, std::vector<float>* out) {
  out->clear();
  if (!t) return true;   // optional bias
  if (t->type != kTfLiteFloat32 || t->allocation_type != kTfLiteMmapRo || !t->data.raw) return false;
  out->resize(t->bytes / sizeof(float));
  if (OnDevice(t->data.raw))
    return cudaMemcpy(out->data(), t->data.raw, out->size() * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess;
  memcpy(out->data(), t->data.raw, out->size() * sizeof(float));
  return true;
}
void StemFree(TfLiteContext*, void* p) { delete static_cast<StemParams*>(p); }
void FillConvDesc(lce_f32_conv_desc* d, const BuiltinParams& bp, int batch, int h, int w, int cin,
                  const TfLiteTensor* filter) {
  d->batch = batch; d->in_h = h; d->in_w = w; d->in_c = cin;
  d->filter_h = filter->dims->data[1]; d->filter_w = filter->dims->data[2];
  d->stride_h = bp.stride_h; d->stride_w = bp.stride_w;
  d->dilation_h = bp.dilation_h; d->dilation_w = bp.dilation_w;
  d->padding = bp.padding; d->activation = bp.activation;
}
bool StemDescs(TfLiteContext* c, TfLiteNode* n, lce_f32_conv_desc* d1, lce_f32_conv_desc* d2) {
  const auto& sp = *static_cast<StemParams*>(n->user_data);
  const TfLiteTensor* in = T(c, n->inputs, 0);
  const TfLiteTensor* w1 = T(c, n->inputs, 1);
  const TfLiteTensor* w2 = T(c, n->inputs, 3);
  if (!in || !w1 || !w2 || in->dims->size != 4 || w1->dims->size != 4 || w2->dims->size != 4)
    return false;
  int oh, ow;
  FillConvDesc(d1, sp.c1, in->dims->data[0], in->dims->data[1], in->dims->data[2],
               in->dims->data[3], w1);
  d1->out_c = w1->dims->data[0];
  if (lce_b200_f32_conv_out_shape(d1, &oh, &ow)) return false;
  FillConvDesc(d2, sp.dw, d1->batch, oh, ow, d1->out_c, w2);
  d2->out_c = w2->dims->data[3];
  return true;
}
TfLiteStatus StemPrepare(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_conv_desc d1, d2;
  B_ENSURE(c, StemDescs(c, n, &d1, &d2), "fused stem: bad shapes");
  const TfLiteTensor* in = T(c, n->inputs, 0);
  B_ENSURE(c, in->type == kTfLiteFloat32 || in->type == kTfLiteInt8 || in->type == kTfLiteUInt8,
           "fused stem: the input must be float32, int8 or uint8");
  B_ENSURE(c, d1.in_c == 3, "fused stem: three input channels expected");
  const size_t c1 = static_cast<size_t>(d1.out_c);
  B_ENSURE(c, (c1 == 16 || c1 == 8) && d2.out_c == d1.out_c, "fused stem: 16 or 8 first-conv channels expected");
  auto& sp = *static_cast<StemParams*>(n->user_data);
  if (sp.w1.empty()) {
    B_ENSURE(c, HostCopy(T(c, n->inputs, 1), &sp.w1) && HostCopy(T(c, n->inputs, 2), &sp.b1) &&
                    HostCopy(T(c, n->inputs, 3), &sp.w2) && HostCopy(T(c, n->inputs, 4), &sp.b2) &&
                    sp.w1.size() == c1 * 27 && sp.w2.size() == 9 * c1 && (sp.b1.empty() || sp.b1.size() == c1) &&
                    (sp.b2.empty() || sp.b2.size() == c1),
             "fused stem: the filters and biases must be constant float tensors");
  }
  int oh, ow;
  B_CAPI(c, lce_b200_f32_conv_out_shape(&d2, &oh, &ow));
  return Resize(c, T(c, n->outputs, 0), {d2.batch, oh, ow, d2.out_c});
}
TfLiteStatus StemInvoke(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_conv_desc d1, d2;
  StemDescs(c, n, &d1, &d2);
  const auto& sp = *static_cast<const StemParams*>(n->user_data);
  const TfLiteTensor* in = T(c, n->inputs, 0);
  const int in_type = in->type == kTfLiteFloat32 ? LCE_T_FLOAT : in->type == kTfLiteInt8 ? LCE_T_INT8 : LCE_T_BOOL;
  B_CAPI(c, lce_b200_f32_stem_conv_dw(&d1, &d2, in_type, in->data.raw, in->params.scale, in->params.zero_point,
                                      sp.w1.data(), sp.b1.empty() ? nullptr : sp.b1.data(), sp.w2.data(),
                                      sp.b2.empty() ? nullptr : sp.b2.data(), T(c, n->outputs, 0)->data.f,
                                      lce_b200_get_stream()));
  return kTfLiteOk;
}

// The size of `a` when its shape with leading 1s dropped is `x`'s trailing dimensions, else 0. A
// kernel that reads a[i % size] for element i of x then broadcasts `a` as TFLite does.
int64_t PreluAlphaCount(const TfLiteTensor* x, const TfLiteTensor* a) {
  int lead = 0;
  while (lead < a->dims->size && a->dims->data[lead] == 1) ++lead;
  const int r = a->dims->size - lead;
  if (r > x->dims->size) return 0;
  int64_t n = 1;
  for (int i = 0; i < r; ++i) {
    if (a->dims->data[lead + i] != x->dims->data[x->dims->size - r + i]) return 0;
    n *= a->dims->data[lead + i];
  }
  return n;
}

// ------------------------------ ADD / MUL / RELU ------------------------------ //
// The kernels compute out[i] = a[i] (op) b[i % Count(b)], which is TFLite's broadcast whenever b's
// shape with leading 1s dropped is a's trailing dimensions: a's own shape, [C] (a's last
// dimension), or a per-position [1,H,W,C], [H,W,C], [W,C] (XNOR-Net++'s scale). A b of higher rank
// would make the output's rank b's. A b of one element (a scalar, or all dimensions 1) is read as
// b[0] for every element. MAXIMUM, MINIMUM and DIV take only the first two and the one element.
// MUL's one further broadcast: a [B,H,W,C] tensor by a per-image, per-channel [B,1,1,C] one (the
// channel gate of Real-to-Binary Net); runs as lce_b200_f32_gate_sign with only the gate set.
bool ImageChannelBroadcast(const TfLiteTensor* a, const TfLiteTensor* b) {
  return a->dims->size == 4 && b->dims->size == 4 && b->dims->data[0] == a->dims->data[0] &&
         b->dims->data[1] == 1 && b->dims->data[2] == 1 && b->dims->data[3] == a->dims->data[3];
}
// b is a's own shape, [C] with any leading 1s, or one element: what out[i] = a[i] op b[i % Count(b)]
// computes as TFLite broadcasts it
bool PlainBroadcast(const TfLiteTensor* a, const TfLiteTensor* b) {
  const int64_t nb = PreluAlphaCount(a, b);
  return a->dims->size > 0 && b->dims->size <= a->dims->size && nb > 0 &&
         (nb == Count(a) || nb == a->dims->data[a->dims->size - 1] || nb == 1);
}
// b's shape with leading 1s dropped is a's trailing dimensions, of at most a's rank
bool TrailingBroadcast(const TfLiteTensor* a, const TfLiteTensor* b) {
  return a->dims->size > 0 && b->dims->size <= a->dims->size && PreluAlphaCount(a, b) > 0;
}
template <bool MUL>
TfLiteStatus EltPrepare(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* a = T(c, n->inputs, 0);
  const TfLiteTensor* b = T(c, n->inputs, 1);
  B_ENSURE(c, a && b, "ADD/MUL: two inputs required");
  const bool plain = TrailingBroadcast(a, b);
  if (MUL)
    B_ENSURE(c, plain || (Count(b) > 0 && ImageChannelBroadcast(a, b)),
             "MUL: only same-shape, last-dimension or [B,H,W,C] x [B,1,1,C] broadcast is supported");
  else
    B_ENSURE(c, plain, "ADD/MUL: only same-shape or last-dimension broadcast is supported");
  TfLiteIntArray* dims = LceB200IntArrayCreate(a->dims->size);
  for (int i = 0; i < a->dims->size; ++i) dims->data[i] = a->dims->data[i];
  return c->ResizeTensor(c, T(c, n->outputs, 0), dims);
}
template <bool MUL>
TfLiteStatus EltInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* a = T(c, n->inputs, 0);
  const TfLiteTensor* b = T(c, n->inputs, 1);
  TfLiteTensor* out = T(c, n->outputs, 0);
  B_ENSURE(c, OnDevice(b->data.raw), "float builtins need device-resident operands");
  const int64_t na = Count(a);
  if (MUL && TrailingBroadcast(a, b) && !PlainBroadcast(a, b)) {   // per position: [1,H,W,C], [W,C], ...
    const lce_scale_desc scale{b->data.f, nullptr, nullptr};
    const int ch = a->dims->data[a->dims->size - 1];
    const int64_t nb = Count(b);
    B_CAPI(c, lce_b200_f32_scale_sign(a->data.f, &scale, nullptr, P(n).activation, na / nb, nb / ch, ch,
                                      out->data.f, nullptr, lce_b200_get_stream()));
    return kTfLiteOk;
  }
  if (MUL && !TrailingBroadcast(a, b)) {   // [B,1,1,C] (EltPrepare)
    const lce_gate_desc gate{b->data.f, nullptr, nullptr, nullptr};
    const int ch = a->dims->data[3];
    B_CAPI(c, lce_b200_f32_gate_sign(a->data.f, &gate, nullptr, P(n).activation, a->dims->data[0],
                                     na / (static_cast<int64_t>(a->dims->data[0]) * ch), ch,
                                     out->data.f, nullptr, lce_b200_get_stream()));
    return kTfLiteOk;
  }
  if (MUL) B_CAPI(c, lce_b200_f32_mul(a->data.f, b->data.f, out->data.f, Count(a), Count(b),
                                      P(n).activation, lce_b200_get_stream()));
  else B_CAPI(c, lce_b200_f32_add(a->data.f, b->data.f, out->data.f, Count(a), Count(b),
                                  P(n).activation, lce_b200_get_stream()));
  return kTfLiteOk;
}
TfLiteStatus SameShapePrepare(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* a = T(c, n->inputs, 0);
  TfLiteIntArray* dims = LceB200IntArrayCreate(a->dims->size);
  for (int i = 0; i < a->dims->size; ++i) dims->data[i] = a->dims->data[i];
  return c->ResizeTensor(c, T(c, n->outputs, 0), dims);
}
TfLiteStatus ReluInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* a = T(c, n->inputs, 0);
  B_CAPI(c, lce_b200_f32_activation(a->data.f, T(c, n->outputs, 0)->data.f, Count(a), LCE_ACT_RELU,
                                    lce_b200_get_stream()));
  return kTfLiteOk;
}

// MAXIMUM (55), MINIMUM (57), DIV (42): float32, b of the shapes ADD takes
template <int CODE>
TfLiteStatus MinMaxDivPrepare(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* a = T(c, n->inputs, 0);
  const TfLiteTensor* b = T(c, n->inputs, 1);
  B_ENSURE(c, a && b && a->type == kTfLiteFloat32 && b->type == kTfLiteFloat32,
           "MAXIMUM/MINIMUM/DIV: two float32 inputs required");
  B_ENSURE(c, PlainBroadcast(a, b),
           "MAXIMUM/MINIMUM/DIV: only same-shape, last-dimension or single-element broadcast is supported");
  return SameShapePrepare(c, n);
}
template <int CODE>
TfLiteStatus MinMaxDivInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* a = T(c, n->inputs, 0);
  const TfLiteTensor* b = T(c, n->inputs, 1);
  float* out = T(c, n->outputs, 0)->data.f;
  B_ENSURE(c, OnDevice(b->data.raw), "float builtins need device-resident operands");
  if (CODE == 55)
    B_CAPI(c, lce_b200_f32_maximum(a->data.f, b->data.f, out, Count(a), Count(b), lce_b200_get_stream()));
  else if (CODE == 57)
    B_CAPI(c, lce_b200_f32_minimum(a->data.f, b->data.f, out, Count(a), Count(b), lce_b200_get_stream()));
  else
    B_CAPI(c, lce_b200_f32_div(a->data.f, b->data.f, out, Count(a), Count(b), P(n).activation,
                               lce_b200_get_stream()));
  return kTfLiteOk;
}
TfLiteStatus RoundPrepare(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  B_ENSURE(c, x && x->type == kTfLiteFloat32, "ROUND: only float32 is supported");
  return SameShapePrepare(c, n);
}
TfLiteStatus RoundInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  B_CAPI(c, lce_b200_f32_round(x->data.f, T(c, n->outputs, 0)->data.f, Count(x), lce_b200_get_stream()));
  return kTfLiteOk;
}

// ------------- fused [MAX_POOL_2D ->] MAXIMUM(0) -> MINIMUM(1) -> MUL(3) -> ROUND [-> DIV(3)] ------------- //
// Created by Graph::FuseQuantizedActivations; builtin_data = the pool's BuiltinParams, or with
// filter_h == 0 no pool; input x [B,H,W,C] (without a pool also [rows, C], taken as [rows,1,1,C]),
// C % 32 == 0; output the level's bit planes [B,OH,OW,3*C/32] (lce_b200_f32_quant2_planes).
bool Quant2Desc(TfLiteContext* c, TfLiteNode* n, lce_f32_pool_desc* d) {
  const TfLiteTensor* in = T(c, n->inputs, 0);
  if (!in || in->type != kTfLiteFloat32 || in->dims->size < 1) return false;
  const BuiltinParams& p = P(n);
  if (p.filter_h != 0) return PoolDesc(c, n, d);
  const int C = in->dims->data[in->dims->size - 1];
  if (C <= 0) return false;
  memset(d, 0, sizeof(*d));
  d->channels = C;
  if (in->dims->size == 4) {
    d->batch = in->dims->data[0]; d->in_h = in->dims->data[1]; d->in_w = in->dims->data[2];
  } else {
    d->batch = static_cast<int>(Count(in) / C); d->in_h = d->in_w = 1;
  }
  return true;
}
TfLiteStatus Quant2Prepare(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_pool_desc d;
  B_ENSURE(c, n->inputs->size == 1 && Quant2Desc(c, n, &d), "Quant2: a float32 input [..., C] expected");
  B_ENSURE(c, d.channels % 32 == 0, "Quant2: the channel count must be a multiple of 32");
  TfLiteTensor* pk = T(c, n->outputs, 0);
  B_ENSURE(c, pk && pk->type == kTfLiteInt32, "Quant2: the planes output must be int32");
  int oh = d.in_h, ow = d.in_w;
  if (d.filter_h != 0) B_CAPI(c, lce_b200_f32_pool_out_shape(&d, &oh, &ow));
  return Resize(c, pk, {d.batch, oh, ow, 3 * (d.channels / 32)});
}
TfLiteStatus Quant2Invoke(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_pool_desc d;
  Quant2Desc(c, n, &d);
  B_CAPI(c, lce_b200_f32_quant2_planes(T(c, n->inputs, 0)->data.f, d.batch, d.in_h, d.in_w, d.channels,
                                       d.filter_h, d.filter_w, d.stride_h, d.stride_w, d.padding,
                                       d.activation, T(c, n->outputs, 0)->data.i32, lce_b200_get_stream()));
  return kTfLiteOk;
}

TfLiteStatus LogisticPrepare(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  B_ENSURE(c, x && x->type == kTfLiteFloat32, "LOGISTIC: only float32 is supported");
  return SameShapePrepare(c, n);
}
TfLiteStatus LogisticInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  B_CAPI(c, lce_b200_f32_logistic(x->data.f, T(c, n->outputs, 0)->data.f, Count(x),
                                  lce_b200_get_stream()));
  return kTfLiteOk;
}

// ----------------------------------- PRELU ----------------------------------- //
// out = x >= 0 ? x : x * alpha (TF/lite/kernels/internal/reference/prelu.h). Alpha broadcasts by
// element index modulo its size (PreluAlphaCount), per-channel [1, 1, C] among the shapes.
TfLiteStatus PreluPrepare(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  const TfLiteTensor* a = T(c, n->inputs, 1);
  B_ENSURE(c, x && a && x->type == kTfLiteFloat32 && a->type == kTfLiteFloat32,
           "PRELU: float32 input and alpha expected");
  const int64_t na = PreluAlphaCount(x, a);
  B_ENSURE(c, na > 0 && na <= INT32_MAX,
           "PRELU: alpha must have the shape of the input's trailing dimensions (leading 1s "
           "allowed); other broadcasts are not supported");
  return SameShapePrepare(c, n);
}
TfLiteStatus PreluInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  const TfLiteTensor* a = T(c, n->inputs, 1);
  B_ENSURE(c, OnDevice(a->data.raw), "PRELU: alpha must be device-resident");
  const int64_t na = PreluAlphaCount(x, a);
  const lce_chain_desc chain{nullptr, a->data.f, nullptr, nullptr};
  B_CAPI(c, lce_b200_f32_chain_sign(x->data.f, &chain, Count(x) / na, static_cast<int>(na),
                                    T(c, n->outputs, 0)->data.f, nullptr, lce_b200_get_stream()));
  return kTfLiteOk;
}

// ------------------ ADD / PRELU / ADD [/ ADD -> LceQuantize] chain ------------------ //
// Created by Graph::FuseActivationChains where no binary convolution precedes the chain.
// inputs [x, shift_in, alpha, shift_out, sign_shift] (absent = -1), each constant [C] for
// x [..., C]; outputs [o (-1 when only the signs are read), packed signs?].
TfLiteStatus ChainPrepare(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  B_ENSURE(c, x && x->type == kTfLiteFloat32 && x->dims->size >= 1 && n->inputs->size == 5,
           "activation chain: float32 input and four optional constants expected");
  const int ch = x->dims->data[x->dims->size - 1];
  for (int k = 1; k < 5; ++k) {
    const TfLiteTensor* v = T(c, n->inputs, k);
    B_ENSURE(c, !v || (v->type == kTfLiteFloat32 && Count(v) == ch),
             "activation chain: the constants must be float32 with one value per channel");
  }
  TfLiteTensor* o = T(c, n->outputs, 0);
  if (o && SameShapePrepare(c, n) != kTfLiteOk) return kTfLiteError;
  if (n->outputs->size > 1) {
    TfLiteTensor* pk = T(c, n->outputs, 1);
    B_ENSURE(c, pk && pk->type == kTfLiteInt32, "activation chain: packed output must be int32");
    TfLiteIntArray* dims = LceB200IntArrayCreate(x->dims->size);
    for (int i = 0; i < x->dims->size; ++i) dims->data[i] = x->dims->data[i];
    dims->data[x->dims->size - 1] = (ch + 31) / 32;
    if (c->ResizeTensor(c, pk, dims) != kTfLiteOk) return kTfLiteError;
  }
  return kTfLiteOk;
}
TfLiteStatus ChainInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  const float* v[4];
  for (int k = 0; k < 4; ++k) {
    const TfLiteTensor* t = T(c, n->inputs, k + 1);
    v[k] = t ? t->data.f : nullptr;
    B_ENSURE(c, !t || OnDevice(t->data.raw), "activation chain: constants must be device-resident");
  }
  const lce_chain_desc chain{v[0], v[1], v[2], v[3]};
  const int ch = x->dims->data[x->dims->size - 1];
  TfLiteTensor* o = T(c, n->outputs, 0);
  TfLiteTensor* pk = n->outputs->size > 1 ? T(c, n->outputs, 1) : nullptr;
  B_CAPI(c, lce_b200_f32_chain_sign(x->data.f, &chain, ch ? Count(x) / ch : 0, ch,
                                    o ? o->data.f : nullptr, pk ? pk->data.i32 : nullptr,
                                    lce_b200_get_stream()));
  return kTfLiteOk;
}

// --------------------------------- DEQUANTIZE -------------------------------- //
// int8 / uint8 -> float32 with the input tensor's (scale, zero_point): TF/lite/kernels/dequantize.cc.
TfLiteStatus DequantPrepare(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* a = T(c, n->inputs, 0);
  TfLiteTensor* o = T(c, n->outputs, 0);
  B_ENSURE(c, a && o && (a->type == kTfLiteInt8 || a->type == kTfLiteUInt8) && o->type == kTfLiteFloat32,
           "DEQUANTIZE: only int8 / uint8 -> float32 is supported");
  return SameShapePrepare(c, n);
}
TfLiteStatus DequantInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* a = T(c, n->inputs, 0);
  B_CAPI(c, lce_b200_dequantize_affine(a->type == kTfLiteInt8 ? LCE_T_INT8 : LCE_T_BOOL, a->data.raw,
                                       T(c, n->outputs, 0)->data.f, Count(a), a->params.scale,
                                       a->params.zero_point, lce_b200_get_stream()));
  return kTfLiteOk;
}

// ----------------------------------- MEAN ----------------------------------- //
TfLiteStatus MeanPrepare(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* in = T(c, n->inputs, 0);
  const TfLiteTensor* axes = T(c, n->inputs, 1);
  B_ENSURE(c, in && in->dims->size == 4, "MEAN: input must be 4-D");
  // only the global-average-pool form (axes = {1, 2}) is needed by these models
  bool ok = axes && axes->type == kTfLiteInt32 && Count(axes) == 2 && !OnDevice(axes->data.raw);
  if (ok) {
    const int a0 = axes->data.i32[0], a1 = axes->data.i32[1];
    ok = (a0 == 1 && a1 == 2) || (a0 == 2 && a1 == 1);
  }
  B_ENSURE(c, ok, "MEAN: only reduction over axes {1,2} is supported");
  if (P(n).keep_dims)
    return Resize(c, T(c, n->outputs, 0), {in->dims->data[0], 1, 1, in->dims->data[3]});
  return Resize(c, T(c, n->outputs, 0), {in->dims->data[0], in->dims->data[3]});
}
TfLiteStatus MeanInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* in = T(c, n->inputs, 0);
  // P(n).activation: a RELU folded in front of the mean by Graph::FuseFloatGlue (0 = none)
  B_CAPI(c, lce_b200_f32_mean_hw_act(in->data.f, T(c, n->outputs, 0)->data.f, in->dims->data[0],
                                     in->dims->data[1], in->dims->data[2], in->dims->data[3],
                                     P(n).activation, lce_b200_get_stream()));
  return kTfLiteOk;
}

// ---------------------------------- SOFTMAX ---------------------------------- //
TfLiteStatus SoftmaxInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* in = T(c, n->inputs, 0);
  const int cols = in->dims->data[in->dims->size - 1];
  B_CAPI(c, lce_b200_f32_softmax(in->data.f, T(c, n->outputs, 0)->data.f,
                                 cols ? Count(in) / cols : 0, cols, P(n).beta,
                                 lce_b200_get_stream()));
  return kTfLiteOk;
}

// ---------------------------------- RESHAPE ---------------------------------- //
TfLiteStatus ReshapePrepare(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* in = T(c, n->inputs, 0);
  const BuiltinParams& p = P(n);
  std::vector<int> shape(p.new_shape, p.new_shape + p.n_new_shape);
  const TfLiteTensor* st = T(c, n->inputs, 1);
  if (shape.empty() && st && st->type == kTfLiteInt32 && !OnDevice(st->data.raw))
    shape.assign(st->data.i32, st->data.i32 + Count(st));
  int64_t known = 1;
  int wild = -1;
  for (size_t i = 0; i < shape.size(); ++i) {
    if (shape[i] == -1) wild = static_cast<int>(i);
    else known *= shape[i];
  }
  if (wild >= 0) shape[wild] = known ? static_cast<int>(Count(in) / known) : 0;
  int64_t total = 1;
  for (int d : shape) total *= d;
  B_ENSURE(c, total == Count(in), "RESHAPE: element count mismatch");
  TfLiteIntArray* dims = LceB200IntArrayCreate(static_cast<int>(shape.size()));
  for (size_t i = 0; i < shape.size(); ++i) dims->data[i] = shape[i];
  return c->ResizeTensor(c, T(c, n->outputs, 0), dims);
}
TfLiteStatus ReshapeInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* in = T(c, n->inputs, 0);
  TfLiteTensor* out = T(c, n->outputs, 0);
  if (in->bytes && cudaMemcpyAsync(out->data.raw, in->data.raw, in->bytes, cudaMemcpyDeviceToDevice,
                                   static_cast<cudaStream_t>(lce_b200_get_stream())) != cudaSuccess) {
    c->ReportError(c, "RESHAPE: device copy failed");
    return kTfLiteError;
  }
  return kTfLiteOk;
}

// ------------------------------- PAD / PADV2 ------------------------------- //
// inputs: [x, paddings int32 [rank,2] (host constant), (PADV2: constant value, host scalar)].
// float32 and int32 (bitpacked) tensors of rank <= 4 (TF/lite/kernels/pad.cc).
bool PadGeometry(TfLiteContext* c, TfLiteNode* n, int32_t in4[4], int32_t before[4],
                 int32_t after[4], int* rank) {
  const TfLiteTensor* in = T(c, n->inputs, 0);
  const TfLiteTensor* pads = T(c, n->inputs, 1);
  if (!in || !pads || pads->type != kTfLiteInt32 || OnDevice(pads->data.raw) || !pads->data.raw)
    return false;
  const int r = in->dims->size;
  if (r < 1 || r > 4 || Count(pads) != 2 * r) return false;
  for (int i = 0; i < 4; ++i) { in4[i] = 1; before[i] = after[i] = 0; }
  for (int i = 0; i < r; ++i) {
    in4[4 - r + i] = in->dims->data[i];
    before[4 - r + i] = pads->data.i32[2 * i];
    after[4 - r + i] = pads->data.i32[2 * i + 1];
    if (before[4 - r + i] < 0 || after[4 - r + i] < 0) return false;
  }
  *rank = r;
  return true;
}
TfLiteStatus PadPrepare(TfLiteContext* c, TfLiteNode* n) {
  int32_t in4[4], before[4], after[4];
  int r = 0;
  const TfLiteTensor* in = T(c, n->inputs, 0);
  B_ENSURE(c, in && (in->type == kTfLiteFloat32 || in->type == kTfLiteInt32),
           "PAD: only float32 / int32 tensors are supported");
  B_ENSURE(c, PadGeometry(c, n, in4, before, after, &r),
           "PAD: paddings must be a constant int32 [rank, 2] tensor with rank <= 4");
  TfLiteIntArray* dims = LceB200IntArrayCreate(r);
  for (int i = 0; i < r; ++i) dims->data[i] = in4[4 - r + i] + before[4 - r + i] + after[4 - r + i];
  return c->ResizeTensor(c, T(c, n->outputs, 0), dims);
}
TfLiteStatus PadInvoke(TfLiteContext* c, TfLiteNode* n) {
  int32_t in4[4], before[4], after[4];
  int r = 0;
  B_ENSURE(c, PadGeometry(c, n, in4, before, after, &r), "PAD: bad paddings");
  uint32_t fill = 0;  // 0.0f / bitpacked +1
  const TfLiteTensor* v = T(c, n->inputs, 2);
  if (v) {
    B_ENSURE(c, v->data.raw && !OnDevice(v->data.raw) && Count(v) == 1 && v->bytes == 4,
             "PADV2: constant_values must be a constant 32-bit scalar");
    memcpy(&fill, v->data.raw, 4);
  }
  B_CAPI(c, lce_b200_pad4d_32(T(c, n->inputs, 0)->data.raw, T(c, n->outputs, 0)->data.raw, in4,
                              before, after, fill, lce_b200_get_stream()));
  return kTfLiteOk;
}

// -------------------- RESIZE_BILINEAR / RESIZE_NEAREST_NEIGHBOR -------------------- //
// inputs [x (float32 [B,H,W,C]), size (constant int32 [2] = new_height, new_width, read on the host
// as PAD reads its paddings)]; output [B, new_height, new_width, C], so the batch follows x's
// (TF/lite/kernels/resize_bilinear.cc, resize_nearest_neighbor.cc).
const int32_t* HostInts(const TfLiteTensor* t);
const char* ResizeGeometry(TfLiteContext* c, TfLiteNode* n, bool bilinear, const BuiltinParams& p,
                           int32_t* out_h, int32_t* out_w) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  const TfLiteTensor* size = T(c, n->inputs, 1);
  if (!x || x->type != kTfLiteFloat32 || x->dims->size != 4)
    return bilinear ? "RESIZE_BILINEAR: the input must be a 4-D float32 tensor"
                    : "RESIZE_NEAREST_NEIGHBOR: the input must be a 4-D float32 tensor";
  if (!size || size->allocation_type != kTfLiteMmapRo || !HostInts(size) || Count(size) != 2)
    return bilinear ? "RESIZE_BILINEAR: the size must be a constant int32 tensor of 2 values"
                    : "RESIZE_NEAREST_NEIGHBOR: the size must be a constant int32 tensor of 2 values";
  if (size->data.i32[0] <= 0 || size->data.i32[1] <= 0)
    return bilinear ? "RESIZE_BILINEAR: the size must be positive"
                    : "RESIZE_NEAREST_NEIGHBOR: the size must be positive";
  if (bilinear && p.align_corners && p.half_pixel_centers)
    return "RESIZE_BILINEAR: align_corners and half_pixel_centers cannot both be set";
  *out_h = size->data.i32[0];
  *out_w = size->data.i32[1];
  return nullptr;
}
template <bool BILINEAR>
TfLiteStatus ResizePrepare(TfLiteContext* c, TfLiteNode* n) {
  int32_t oh, ow;
  const char* why = ResizeGeometry(c, n, BILINEAR, P(n), &oh, &ow);
  B_ENSURE(c, why == nullptr, why);
  const TfLiteIntArray* d = T(c, n->inputs, 0)->dims;
  return Resize(c, T(c, n->outputs, 0), {d->data[0], oh, ow, d->data[3]});
}
template <bool BILINEAR>
TfLiteStatus ResizeInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  const TfLiteTensor* o = T(c, n->outputs, 0);
  const BuiltinParams& p = P(n);
  const int* d = x->dims->data;
  if (BILINEAR)
    B_CAPI(c, lce_b200_f32_resize_bilinear(x->data.f, d[0], d[1], d[2], d[3], o->dims->data[1], o->dims->data[2],
                                           p.align_corners, p.half_pixel_centers, o->data.f,
                                           lce_b200_get_stream()));
  else
    B_CAPI(c, lce_b200_f32_resize_nearest(x->data.f, d[0], d[1], d[2], d[3], o->dims->data[1], o->dims->data[2],
                                          p.align_corners, p.half_pixel_centers, o->data.f,
                                          lce_b200_get_stream()));
  return kTfLiteOk;
}

// ------------- fused RESIZE_NEAREST_NEIGHBOR -> ADD [-> LceQuantize]: a decoder merge ------------- //
// Created by Graph::FuseUpsampleMerges; builtin_data = { BuiltinParams resize, BuiltinParams add };
// inputs [u, size, skip], outputs [sum (-1 when only the signs are read), packed signs?].
struct MergeParams {
  BuiltinParams resize, add;
};
void* MergeInit(TfLiteContext*, const char* buffer, size_t length) {
  auto* p = new MergeParams();
  memset(p, 0, sizeof(*p));
  if (buffer && length >= sizeof(MergeParams)) memcpy(p, buffer, sizeof(MergeParams));
  return p;
}
void MergeFree(TfLiteContext*, void* p) { delete static_cast<MergeParams*>(p); }
TfLiteStatus MergePrepare(TfLiteContext* c, TfLiteNode* n) {
  const auto& mp = *static_cast<const MergeParams*>(n->user_data);
  B_ENSURE(c, n->inputs->size == 3 && n->outputs->size >= 1 && n->outputs->size <= 2,
           "RESIZE_NEAREST_NEIGHBOR+ADD: inputs [u, size, skip] and one or two outputs expected");
  int32_t oh, ow;
  const char* why = ResizeGeometry(c, n, false, mp.resize, &oh, &ow);
  B_ENSURE(c, why == nullptr, why);
  const TfLiteIntArray* u = T(c, n->inputs, 0)->dims;
  const TfLiteTensor* skip = T(c, n->inputs, 2);
  B_ENSURE(c, skip && skip->type == kTfLiteFloat32 && skip->dims->size == 4 && skip->dims->data[0] == u->data[0] &&
                  skip->dims->data[1] == oh && skip->dims->data[2] == ow && skip->dims->data[3] == u->data[3],
           "RESIZE_NEAREST_NEIGHBOR+ADD: the skip map must have the resized map's shape");
  TfLiteTensor* o = T(c, n->outputs, 0);
  if (o && Resize(c, o, {u->data[0], oh, ow, u->data[3]}) != kTfLiteOk) return kTfLiteError;
  if (n->outputs->size == 2) {
    TfLiteTensor* pk = T(c, n->outputs, 1);
    B_ENSURE(c, pk && pk->type == kTfLiteInt32, "RESIZE_NEAREST_NEIGHBOR+ADD+LceQuantize: packed output must be int32");
    if (Resize(c, pk, {u->data[0], oh, ow, (u->data[3] + 31) / 32}) != kTfLiteOk) return kTfLiteError;
  }
  return kTfLiteOk;
}
TfLiteStatus MergeInvoke(TfLiteContext* c, TfLiteNode* n) {
  const auto& mp = *static_cast<const MergeParams*>(n->user_data);
  const TfLiteTensor* u = T(c, n->inputs, 0);
  const TfLiteTensor* skip = T(c, n->inputs, 2);
  TfLiteTensor* o = T(c, n->outputs, 0);
  TfLiteTensor* pk = n->outputs->size > 1 ? T(c, n->outputs, 1) : nullptr;
  const int* d = u->dims->data;
  B_CAPI(c, lce_b200_f32_upsample_add_sign(u->data.f, d[0], d[1], d[2], d[3], skip->dims->data[1],
                                           skip->dims->data[2], mp.resize.align_corners,
                                           mp.resize.half_pixel_centers, skip->data.f, mp.add.activation,
                                           o ? o->data.f : nullptr, pk ? pk->data.i32 : nullptr,
                                           lce_b200_get_stream()));
  return kTfLiteOk;
}

// --------------------------------- ARG_MAX --------------------------------- //
// inputs [x (float32, rank >= 1), axis (read on the host, as the resizes read their size)]; output x's
// shape without the axis, of ArgMaxOptions.output_type (int32 or int64) (TF/lite/kernels/arg_min_max.cc).
// Checks x = input 0, the axis at input `axis_input` and output 0; returns nullptr, or why they are refused.
const char* ArgMaxChecks(TfLiteContext* c, TfLiteNode* n, int axis_input, const BuiltinParams& p, int* axis) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  if (!x || x->type != kTfLiteFloat32 || x->dims->size < 1)
    return "ARG_MAX: the input must be a float32 tensor of rank 1 or more";
  const char* why = ArgMaxAxis(T(c, n->inputs, axis_input), x->dims->size, axis);
  if (why) return why;
  if (x->dims->data[*axis] <= 0) return "ARG_MAX: the reduced axis is empty";
  if (p.output_type != 2 && p.output_type != 4) return "ARG_MAX: output_type must be int32 or int64";
  const TfLiteTensor* o = T(c, n->outputs, 0);
  if (!o || o->type != (p.output_type == 4 ? kTfLiteInt64 : kTfLiteInt32))
    return "ARG_MAX: the output tensor's type differs from output_type";
  return nullptr;
}
TfLiteStatus ArgMaxPrepare(TfLiteContext* c, TfLiteNode* n) {
  B_ENSURE(c, n->inputs->size == 2 && n->outputs->size == 1, "ARG_MAX: inputs [x, axis] and one output expected");
  int axis;
  const char* why = ArgMaxChecks(c, n, 1, P(n), &axis);
  B_ENSURE(c, why == nullptr, why);
  const TfLiteIntArray* d = T(c, n->inputs, 0)->dims;
  TfLiteIntArray* dims = LceB200IntArrayCreate(d->size - 1);
  for (int k = 0, j = 0; k < d->size; ++k)
    if (k != axis) dims->data[j++] = d->data[k];
  return c->ResizeTensor(c, T(c, n->outputs, 0), dims);
}
TfLiteStatus ArgMaxInvoke(TfLiteContext* c, TfLiteNode* n) {
  int axis;
  const char* why = ArgMaxChecks(c, n, 1, P(n), &axis);
  B_ENSURE(c, why == nullptr, why);
  const TfLiteTensor* x = T(c, n->inputs, 0);
  TfLiteTensor* o = T(c, n->outputs, 0);
  int64_t outer = 1, inner = 1;
  for (int k = 0; k < axis; ++k) outer *= x->dims->data[k];
  for (int k = axis + 1; k < x->dims->size; ++k) inner *= x->dims->data[k];
  B_CAPI(c, lce_b200_f32_argmax(x->data.f, outer, x->dims->data[axis], inner, o->type == kTfLiteInt64,
                                o->data.raw, lce_b200_get_stream()));
  return kTfLiteOk;
}

// -------------------------------- REDUCE_MAX -------------------------------- //
// inputs [x (float32, rank 1-5), axes (a constant int32 tensor, 0-D or 1-D, read on the host)]; output
// x's shape with the reduced axes kept as 1 (ReducerOptions.keep_dims) or dropped. Negative axes count
// from the end and duplicates are allowed, as in TFLite; the reduced axes must be contiguous, so the
// op is [outer, n, inner] reduced over n. Returns nullptr, or why the node is refused.
const char* ReduceMaxChecks(TfLiteContext* c, TfLiteNode* n, int* first, int* last) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  const TfLiteTensor* axes = T(c, n->inputs, 1);
  const TfLiteTensor* o = T(c, n->outputs, 0);
  if (!x || x->type != kTfLiteFloat32) return "REDUCE_MAX: the input must be float32";
  if (!o || o->type != kTfLiteFloat32) return "REDUCE_MAX: the output must be float32";
  if (!axes || axes->allocation_type != kTfLiteMmapRo || !axes->data.raw || OnDevice(axes->data.raw))
    return "REDUCE_MAX: the axes must be a constant tensor";
  if (axes->type != kTfLiteInt32 || axes->dims->size > 1) return "REDUCE_MAX: the axes must be a 0-D or 1-D int32 tensor";
  const int rank = x->dims->size;
  if (rank < 1 || rank > 5) return "REDUCE_MAX: the input's rank must be 1 to 5";
  if (Count(axes) < 1) return "REDUCE_MAX: no axis to reduce";
  bool red[5] = {};
  for (int64_t k = 0; k < Count(axes); ++k) {
    const int a = axes->data.i32[k];
    if (a < -rank || a >= rank) return "REDUCE_MAX: an axis is out of range";
    red[a < 0 ? a + rank : a] = true;
  }
  *first = 0;
  while (!red[*first]) ++*first;
  *last = *first;
  while (*last + 1 < rank && red[*last + 1]) ++*last;
  for (int k = *last + 1; k < rank; ++k)
    if (red[k]) return "REDUCE_MAX: the reduced axes must be contiguous";
  return nullptr;
}
TfLiteStatus ReduceMaxPrepare(TfLiteContext* c, TfLiteNode* n) {
  B_ENSURE(c, n->inputs->size == 2 && n->outputs->size == 1, "REDUCE_MAX: inputs [x, axes] and one output expected");
  int first, last;
  const char* why = ReduceMaxChecks(c, n, &first, &last);
  B_ENSURE(c, why == nullptr, why);
  const TfLiteIntArray* d = T(c, n->inputs, 0)->dims;
  std::vector<int> dims;
  for (int k = 0; k < d->size; ++k)
    if (k < first || k > last) dims.push_back(d->data[k]);
    else if (P(n).keep_dims) dims.push_back(1);
  return ResizeTo(c, T(c, n->outputs, 0), dims);
}
TfLiteStatus ReduceMaxInvoke(TfLiteContext* c, TfLiteNode* n) {
  int first, last;
  const char* why = ReduceMaxChecks(c, n, &first, &last);
  B_ENSURE(c, why == nullptr, why);
  const TfLiteTensor* x = T(c, n->inputs, 0);
  int64_t outer = 1, r = 1, inner = 1;
  for (int k = 0; k < x->dims->size; ++k)
    (k < first ? outer : k > last ? inner : r) *= x->dims->data[k];
  B_CAPI(c, lce_b200_f32_reduce_max(x->data.f, outer, r, inner, T(c, n->outputs, 0)->data.f, lce_b200_get_stream()));
  return kTfLiteOk;
}

// ------------------ fused RESIZE_BILINEAR -> ARG_MAX: a segmentation head ------------------ //
// Created by Graph::FuseResizeArgmax; builtin_data = { BuiltinParams resize, BuiltinParams argmax };
// inputs [x, size, axis (the channel axis)], outputs [labels [B, new_height, new_width]].
struct ResizeArgmaxParams {
  BuiltinParams resize, argmax;
};
void* ResizeArgmaxInit(TfLiteContext*, const char* buffer, size_t length) {
  auto* p = new ResizeArgmaxParams();
  memset(p, 0, sizeof(*p));
  if (buffer && length >= sizeof(ResizeArgmaxParams)) memcpy(p, buffer, sizeof(ResizeArgmaxParams));
  return p;
}
void ResizeArgmaxFree(TfLiteContext*, void* p) { delete static_cast<ResizeArgmaxParams*>(p); }
TfLiteStatus ResizeArgmaxPrepare(TfLiteContext* c, TfLiteNode* n) {
  const auto& rp = *static_cast<const ResizeArgmaxParams*>(n->user_data);
  B_ENSURE(c, n->inputs->size == 3 && n->outputs->size == 1,
           "RESIZE_BILINEAR+ARG_MAX: inputs [x, size, axis] and one output expected");
  int32_t oh, ow;
  const char* why = ResizeGeometry(c, n, true, rp.resize, &oh, &ow);
  B_ENSURE(c, why == nullptr, why);
  int axis;
  why = ArgMaxChecks(c, n, 2, rp.argmax, &axis);
  B_ENSURE(c, why == nullptr, why);
  const TfLiteIntArray* d = T(c, n->inputs, 0)->dims;
  B_ENSURE(c, axis == 3, "RESIZE_BILINEAR+ARG_MAX: the axis must be the channel axis");
  B_ENSURE(c, static_cast<int64_t>(d->data[2]) * d->data[3] <= lce_b200_resize_bilinear_argmax_max_row_floats(),
           "RESIZE_BILINEAR+ARG_MAX: the source rows do not fit shared memory");
  return Resize(c, T(c, n->outputs, 0), {d->data[0], oh, ow});
}
TfLiteStatus ResizeArgmaxInvoke(TfLiteContext* c, TfLiteNode* n) {
  const auto& rp = *static_cast<const ResizeArgmaxParams*>(n->user_data);
  const TfLiteTensor* x = T(c, n->inputs, 0);
  TfLiteTensor* o = T(c, n->outputs, 0);
  const int* d = x->dims->data;
  B_CAPI(c, lce_b200_f32_resize_bilinear_argmax(x->data.f, d[0], d[1], d[2], d[3], o->dims->data[1],
                                                o->dims->data[2], rp.resize.align_corners,
                                                rp.resize.half_pixel_centers, o->type == kTfLiteInt64,
                                                o->data.raw, lce_b200_get_stream()));
  return kTfLiteOk;
}

// ------------------------------ DEPTH_TO_SPACE ------------------------------ //
// inputs [x (float32 [B, H, W, C])], output [B, H * r, W * r, C / r^2] (TF/lite/kernels/depth_to_space.cc:
// rank 4, block_size > 0, C % r^2 == 0, input and output of one type; float32 only here).
const char* DepthToSpaceChecks(const TfLiteTensor* x, const TfLiteTensor* o, int r) {
  if (!x || x->dims->size != 4) return "DEPTH_TO_SPACE: the input must be a 4-D tensor";
  if (x->type != kTfLiteFloat32) return "DEPTH_TO_SPACE: only float32 is supported";
  if (!o || o->type != x->type) return "DEPTH_TO_SPACE: the output's type differs from the input's";
  if (r <= 0) return "DEPTH_TO_SPACE: block_size must be positive";
  if (x->dims->data[3] % (static_cast<int64_t>(r) * r))
    return "DEPTH_TO_SPACE: the input's channels must be a multiple of block_size^2";
  return nullptr;
}
TfLiteStatus DepthToSpacePrepare(TfLiteContext* c, TfLiteNode* n) {
  B_ENSURE(c, n->inputs->size == 1 && n->outputs->size == 1, "DEPTH_TO_SPACE: one input and one output expected");
  const TfLiteTensor* x = T(c, n->inputs, 0);
  const int r = P(n).block_size;
  const char* why = DepthToSpaceChecks(x, T(c, n->outputs, 0), r);
  B_ENSURE(c, why == nullptr, why);
  const int* d = x->dims->data;
  B_ENSURE(c, static_cast<int64_t>(d[1]) * r <= INT32_MAX && static_cast<int64_t>(d[2]) * r <= INT32_MAX,
           "DEPTH_TO_SPACE: the output is too large");
  return Resize(c, T(c, n->outputs, 0), {d[0], d[1] * r, d[2] * r, d[3] / (r * r)});
}
TfLiteStatus DepthToSpaceInvoke(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  const int* d = x->dims->data;
  B_CAPI(c, lce_b200_f32_depth_to_space(x->data.f, d[0], d[1], d[2], d[3], P(n).block_size,
                                        T(c, n->outputs, 0)->data.f, lce_b200_get_stream()));
  return kTfLiteOk;
}

// ----- fused CONV_2D -> DEPTH_TO_SPACE [-> ADD(RESIZE_BILINEAR(img))]: a super-resolution tail ----- //
// Created by Graph::FuseSubpixelConvs; builtin_data = { BuiltinParams conv, depth_to_space, resize, add }
// (the last two zero without the residual); inputs [x, filter, bias (-1 when absent)] or [x, filter,
// bias, img, size], outputs [y [B, H * r, W * r, C']]. Runs lce_b200_f32_subpixel_conv.
struct SubpixelParams {
  BuiltinParams conv, d2s, resize, add;
};
void* SubpixelInit(TfLiteContext*, const char* buffer, size_t length) {
  auto* p = new SubpixelParams();
  memset(p, 0, sizeof(*p));
  if (buffer && length >= sizeof(SubpixelParams)) memcpy(p, buffer, sizeof(SubpixelParams));
  return p;
}
void SubpixelFree(TfLiteContext*, void* p) { delete static_cast<SubpixelParams*>(p); }
TfLiteStatus SubpixelPrepare(TfLiteContext* c, TfLiteNode* n) {
  const auto& sp = *static_cast<const SubpixelParams*>(n->user_data);
  B_ENSURE(c, (n->inputs->size == 3 || n->inputs->size == 5) && n->outputs->size == 1,
           "CONV_2D+DEPTH_TO_SPACE: inputs [x, filter, bias] or [x, filter, bias, img, size] and one output expected");
  lce_f32_conv_desc d;
  int groups = 1;
  B_ENSURE(c, ConvDesc(c, n, false, &d, &groups) && groups == 1,
           "CONV_2D+DEPTH_TO_SPACE: bad input / filter shapes");
  const TfLiteTensor* x = T(c, n->inputs, 0);
  B_ENSURE(c, x->type == kTfLiteFloat32, "CONV_2D+DEPTH_TO_SPACE: only float32 is supported");
  B_ENSURE(c, d.stride_h == 1 && d.stride_w == 1 && d.dilation_h == 1 && d.dilation_w == 1 &&
                  d.padding == LCE_PADDING_SAME,
           "CONV_2D+DEPTH_TO_SPACE: the convolution must have stride 1, dilation 1 and SAME padding");
  const int r = sp.d2s.block_size;
  B_ENSURE(c, r > 0 && d.out_c % (r * r) == 0,
           "CONV_2D+DEPTH_TO_SPACE: the conv's channels must be a multiple of block_size^2");
  B_ENSURE(c, d.out_c <= lce_b200_subpixel_conv_max_out_channels(),
           "CONV_2D+DEPTH_TO_SPACE: the conv has too many output channels");
  const int cp = d.out_c / (r * r);
  if (n->inputs->size == 5) {
    const TfLiteTensor* img = T(c, n->inputs, 3);
    const TfLiteTensor* size = T(c, n->inputs, 4);
    B_ENSURE(c, img && img->type == kTfLiteFloat32 && img->dims->size == 4 && img->dims->data[0] == d.batch &&
                    img->dims->data[3] == cp,
             "CONV_2D+DEPTH_TO_SPACE+RESIZE_BILINEAR+ADD: img must be float32 [B, h, w, C']");
    B_ENSURE(c, size && size->allocation_type == kTfLiteMmapRo && HostInts(size) && Count(size) == 2 &&
                    size->data.i32[0] == d.in_h * r && size->data.i32[1] == d.in_w * r,
             "CONV_2D+DEPTH_TO_SPACE+RESIZE_BILINEAR+ADD: the size must be the constant output size");
    B_ENSURE(c, !(sp.resize.align_corners && sp.resize.half_pixel_centers),
             "RESIZE_BILINEAR: align_corners and half_pixel_centers cannot both be set");
  }
  return Resize(c, T(c, n->outputs, 0), {d.batch, d.in_h * r, d.in_w * r, cp});
}
TfLiteStatus SubpixelInvoke(TfLiteContext* c, TfLiteNode* n) {
  const auto& sp = *static_cast<const SubpixelParams*>(n->user_data);
  lce_f32_conv_desc d;
  ConvDesc(c, n, false, &d);
  const TfLiteTensor* bias = T(c, n->inputs, 2);
  const TfLiteTensor* img = n->inputs->size == 5 ? T(c, n->inputs, 3) : nullptr;
  B_CAPI(c, lce_b200_f32_subpixel_conv(&d, T(c, n->inputs, 0)->data.f, T(c, n->inputs, 1)->data.f,
                                       bias ? bias->data.f : nullptr, sp.d2s.block_size, img ? img->data.f : nullptr,
                                       img ? img->dims->data[1] : 0, img ? img->dims->data[2] : 0,
                                       sp.resize.align_corners, sp.resize.half_pixel_centers, sp.add.activation,
                                       T(c, n->outputs, 0)->data.f, lce_b200_get_stream()));
  return kTfLiteOk;
}

// ------------------------------ TRANSPOSE_CONV ------------------------------ //
// inputs [output_shape (constant int32 [4], read on the host as the resizes read their size), weights
// [Cout, kh, kw, Cin], x [B, H, W, Cin], bias [Cout] (-1 when absent)], output [B, output_shape[1],
// output_shape[2], Cout]: the batch follows x's, as the resizes' does, so a batch resize keeps the
// model's output_shape (output_shape[0] is not read). Float32 only. The padding is TFLite's
// (TF/lite/kernels/transpose_conv.cc): ComputePaddingHeightWidth run on the output's size, the floor
// half of the total, and x's H and W must be what a convolution with this filter, stride and padding
// gives from the output's (TF's consistency condition; Keras' output_padding < stride meets it).
// Fills *d, or returns why the node is refused.
int TransposeConvInputSize(int padding, int out, int k, int s) {
  return padding == LCE_PADDING_SAME ? (out + s - 1) / s : (out + s - k) / s;
}
const char* TransposeConvChecks(TfLiteContext* c, TfLiteNode* n, const BuiltinParams& p,
                                lce_f32_transpose_conv_desc* d) {
  if ((n->inputs->size != 3 && n->inputs->size != 4) || n->outputs->size != 1)
    return "TRANSPOSE_CONV: inputs [output_shape, weights, input, bias] and one output expected";
  const TfLiteTensor* shape = T(c, n->inputs, 0);
  const TfLiteTensor* w = T(c, n->inputs, 1);
  const TfLiteTensor* x = T(c, n->inputs, 2);
  const TfLiteTensor* bias = n->inputs->size == 4 ? T(c, n->inputs, 3) : nullptr;
  const TfLiteTensor* o = T(c, n->outputs, 0);
  if (!shape || shape->allocation_type != kTfLiteMmapRo || !HostInts(shape) || Count(shape) != 4)
    return "TRANSPOSE_CONV: output_shape must be a constant int32 tensor of 4 elements";
  if (!w || !x || !o || w->type != kTfLiteFloat32 || x->type != kTfLiteFloat32 || o->type != kTfLiteFloat32 ||
      (bias && bias->type != kTfLiteFloat32))
    return "TRANSPOSE_CONV: only float32 is supported";
  if (w->dims->size != 4 || x->dims->size != 4) return "TRANSPOSE_CONV: the weights and the input must be 4-D";
  const int cout = w->dims->data[0], kh = w->dims->data[1], kw = w->dims->data[2];
  if (w->dims->data[3] != x->dims->data[3]) return "TRANSPOSE_CONV: the weights' input channels differ from the input's";
  if (bias && (bias->dims->size != 1 || bias->dims->data[0] != cout))
    return "TRANSPOSE_CONV: the bias must have shape [Cout]";
  const int32_t* os = shape->data.i32;
  if (os[3] != cout) return "TRANSPOSE_CONV: output_shape[3] differs from the weights' output channels";
  if (p.stride_h <= 0 || p.stride_w <= 0) return "TRANSPOSE_CONV: strides must be positive";
  if (p.activation < LCE_ACT_NONE || p.activation > LCE_ACT_RELU6)
    return "TRANSPOSE_CONV: the fused activation must be NONE, RELU, RELU_N1_TO_1 or RELU6";
  if (p.padding != LCE_PADDING_SAME && p.padding != LCE_PADDING_VALID) return "TRANSPOSE_CONV: unknown padding";
  if (os[1] <= 0 || os[2] <= 0 || kh <= 0 || kw <= 0 || cout <= 0)
    return "TRANSPOSE_CONV: the output and the filter must not be empty";
  if (x->dims->data[1] != TransposeConvInputSize(p.padding, os[1], kh, p.stride_h) ||
      x->dims->data[2] != TransposeConvInputSize(p.padding, os[2], kw, p.stride_w))
    return "TRANSPOSE_CONV: the input's height and width are not what a convolution with this filter, stride "
           "and padding gives from output_shape";
  auto pad = [](int in, int k, int s, int out) {   // ComputePaddingWithOffset(s, 1, out, k, in), floor half
    const int64_t total = static_cast<int64_t>(in - 1) * s + k - out;
    return static_cast<int>(total > 0 ? total / 2 : 0);
  };
  *d = {x->dims->data[0], x->dims->data[1], x->dims->data[2], x->dims->data[3], kh, kw, cout, os[1], os[2],
        p.stride_h, p.stride_w, pad(x->dims->data[1], kh, p.stride_h, os[1]),
        pad(x->dims->data[2], kw, p.stride_w, os[2]), p.activation};
  return nullptr;
}
TfLiteStatus TransposeConvPrepare(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_transpose_conv_desc d;
  const char* why = TransposeConvChecks(c, n, P(n), &d);
  B_ENSURE(c, why == nullptr, why);
  return Resize(c, T(c, n->outputs, 0), {d.batch, d.out_h, d.out_w, d.out_c});
}
TfLiteStatus TransposeConvInvoke(TfLiteContext* c, TfLiteNode* n) {
  lce_f32_transpose_conv_desc d;
  TransposeConvChecks(c, n, P(n), &d);
  const TfLiteTensor* bias = n->inputs->size == 4 ? T(c, n->inputs, 3) : nullptr;
  B_CAPI(c, lce_b200_f32_transpose_conv2d(&d, T(c, n->inputs, 2)->data.f, T(c, n->inputs, 1)->data.f,
                                          bias ? bias->data.f : nullptr, T(c, n->outputs, 0)->data.f,
                                          lce_b200_get_stream()));
  return kTfLiteOk;
}

// --- fused LceDequantize -> TRANSPOSE_CONV (+-1, k = s) [-> ADD(skip)] [-> LceQuantize]: a binary upsampler --- //
// Created by Graph::FuseBinaryTransposeConvs; builtin_data = BinaryTConvParams; inputs [q (packed signs
// [B, H, W, ceil(Cin / 32)]), filter (the weights' signs as a packed 1x1 LceBconv2d filter [s_h * s_w *
// C, 1, 1, ceil(Cin / 32)], rows in (i, j, c) order), bias ([C] or -1), skip ([B, H * s_h, W * s_w, C]
// or -1)], outputs [sum [B, H * s_h, W * s_w, C], packed signs?]. The node owns a 1x1 LceBconv2d plan
// and runs lce_b200_bconv2d_run_fused_shuffle, which takes the +-1 dot product from its accumulators.
struct BinaryTConvParams {
  BuiltinParams tconv, add;
  int32_t channels_in;
};
struct BinaryTConvOp {
  BinaryTConvParams p;
  lce_b200_bconv2d* plan = nullptr;
};
void* BinaryTConvInit(TfLiteContext*, const char* buffer, size_t length) {
  auto* op = new BinaryTConvOp();
  memset(&op->p, 0, sizeof(op->p));
  if (buffer && length >= sizeof(BinaryTConvParams)) memcpy(&op->p, buffer, sizeof(BinaryTConvParams));
  return op;
}
void BinaryTConvFree(TfLiteContext*, void* p) {
  auto* op = static_cast<BinaryTConvOp*>(p);
  lce_b200_bconv2d_destroy(op->plan);
  delete op;
}
TfLiteStatus BinaryTConvPrepare(TfLiteContext* c, TfLiteNode* n) {
  auto* op = static_cast<BinaryTConvOp*>(n->user_data);
  const BinaryTConvParams& bp = op->p;
  B_ENSURE(c, n->inputs->size == 4 && n->outputs->size >= 1 && n->outputs->size <= 2,
           "LceBconv2dTranspose: inputs [q, filter, bias, skip] and one or two outputs expected");
  const TfLiteTensor* q = T(c, n->inputs, 0);
  const TfLiteTensor* f = T(c, n->inputs, 1);
  const TfLiteTensor* bias = T(c, n->inputs, 2);
  const TfLiteTensor* skip = T(c, n->inputs, 3);
  const int sh = bp.tconv.stride_h, sw = bp.tconv.stride_w, cin = bp.channels_in;
  B_ENSURE(c, sh > 0 && sw > 0 && cin > 0, "LceBconv2dTranspose: bad strides or input channels");
  B_ENSURE(c, q && q->type == kTfLiteInt32 && q->dims->size == 4 && q->dims->data[3] == (cin + 31) / 32,
           "LceBconv2dTranspose: the input must be the packed signs [B, H, W, ceil(Cin / 32)]");
  B_ENSURE(c, f && f->type == kTfLiteInt32 && f->allocation_type == kTfLiteMmapRo && f->dims->size == 4 &&
                  f->dims->data[1] == 1 && f->dims->data[2] == 1 && f->dims->data[3] == (cin + 31) / 32 &&
                  f->dims->data[0] % (sh * sw) == 0,
           "LceBconv2dTranspose: the filter must be a constant packed [s_h * s_w * C, 1, 1, ceil(Cin / 32)]");
  const int C = f->dims->data[0] / (sh * sw);
  B_ENSURE(c, !bias || (bias->type == kTfLiteFloat32 && bias->allocation_type == kTfLiteMmapRo &&
                        Count(bias) == C),
           "LceBconv2dTranspose: the bias must be a constant float32 [C]");
  const int B = q->dims->data[0], H = q->dims->data[1], W = q->dims->data[2];
  B_ENSURE(c, static_cast<int64_t>(H) * sh <= INT32_MAX && static_cast<int64_t>(W) * sw <= INT32_MAX,
           "LceBconv2dTranspose: the output is too large");
  const int OH = H * sh, OW = W * sw;
  B_ENSURE(c, !skip || (skip->type == kTfLiteFloat32 && skip->dims->size == 4 && skip->dims->data[0] == B &&
                        skip->dims->data[1] == OH && skip->dims->data[2] == OW && skip->dims->data[3] == C),
           "LceBconv2dTranspose+ADD: the skip map must have the output's shape");
  if (Resize(c, T(c, n->outputs, 0), {B, OH, OW, C}) != kTfLiteOk) return kTfLiteError;
  if (n->outputs->size == 2) {
    TfLiteTensor* pk = T(c, n->outputs, 1);
    B_ENSURE(c, pk && pk->type == kTfLiteInt32, "LceBconv2dTranspose+LceQuantize: packed output must be int32");
    if (Resize(c, pk, {B, OH, OW, (C + 31) / 32}) != kTfLiteOk) return kTfLiteError;
  }
  if (op->plan) {
    B_CAPI(c, lce_b200_bconv2d_set_input_shape(op->plan, B, H, W));
    return kTfLiteOk;
  }
  lce_bconv2d_desc d;
  memset(&d, 0, sizeof(d));
  d.batch = B; d.in_h = H; d.in_w = W; d.channels_in = cin;
  d.filter_h = 1; d.filter_w = 1; d.channels_out = sh * sw * C; d.groups = 1;
  d.stride_h = 1; d.stride_w = 1; d.dilation_h = 1; d.dilation_w = 1;
  d.padding = LCE_PADDING_VALID; d.pad_value = 1; d.activation = LCE_ACT_NONE; d.out_type = LCE_OUT_FLOAT;
  const std::vector<float> ones(d.channels_out, 1.0f), zeros(d.channels_out, 0.0f);
  B_CAPI(c, lce_b200_bconv2d_create(&d, f->data.i32, ones.data(), zeros.data(), nullptr, &op->plan));
  return kTfLiteOk;
}
TfLiteStatus BinaryTConvInvoke(TfLiteContext* c, TfLiteNode* n) {
  const auto* op = static_cast<const BinaryTConvOp*>(n->user_data);
  const TfLiteTensor* bias = T(c, n->inputs, 2);
  const TfLiteTensor* skip = T(c, n->inputs, 3);
  TfLiteTensor* pk = n->outputs->size > 1 ? T(c, n->outputs, 1) : nullptr;
  B_CAPI(c, lce_b200_bconv2d_run_fused_shuffle(op->plan, T(c, n->inputs, 0)->data.i32, op->p.tconv.stride_h,
                                               op->p.tconv.stride_w, bias ? bias->data.f : nullptr,
                                               op->p.tconv.activation, skip ? skip->data.f : nullptr,
                                               op->p.add.activation, T(c, n->outputs, 0)->data.f,
                                               pk ? pk->data.i32 : nullptr, lce_b200_get_stream()));
  return kTfLiteOk;
}

// --- fused LceDequantize -> FULLY_CONNECTED (+-alpha) [-> MUL -> ADD] [-> LceQuantize]: a binary dense layer --- //
// Created by Graph::FuseBinaryFullyConnected; builtin_data = BinaryFcParams; inputs [q (packed signs whose
// words are the rows' words, ceil(K / 32) per row), filter (the weights' signs as a packed 1x1 LceBconv2d
// filter [N, 1, 1, ceil(K / 32)]), alpha ([N] or -1), bias, scale, shift ([N] or -1)], outputs [result
// [rows, N], packed signs [rows, N / 32]?]. rows follow q's size, so a batch resize re-plans them. The
// node owns a 1x1 LceBconv2d plan of rows x 1 x 1 and runs lce_b200_bconv2d_run_fused_fc.
struct BinaryFcParams {
  BuiltinParams fc, add;
  int32_t channels_in;
};
struct BinaryFcOp {
  BinaryFcParams p;
  lce_b200_bconv2d* plan = nullptr;
};
void* BinaryFcInit(TfLiteContext*, const char* buffer, size_t length) {
  auto* op = new BinaryFcOp();
  memset(&op->p, 0, sizeof(op->p));
  if (buffer && length >= sizeof(BinaryFcParams)) memcpy(&op->p, buffer, sizeof(BinaryFcParams));
  return op;
}
void BinaryFcFree(TfLiteContext*, void* p) {
  auto* op = static_cast<BinaryFcOp*>(p);
  lce_b200_bconv2d_destroy(op->plan);
  delete op;
}
TfLiteStatus BinaryFcPrepare(TfLiteContext* c, TfLiteNode* n) {
  auto* op = static_cast<BinaryFcOp*>(n->user_data);
  const int K = op->p.channels_in;
  B_ENSURE(c, n->inputs->size == 6 && n->outputs->size >= 1 && n->outputs->size <= 2 && K > 0,
           "LceBfc: inputs [q, filter, alpha, bias, scale, shift] and one or two outputs expected");
  const TfLiteTensor* q = T(c, n->inputs, 0);
  const TfLiteTensor* f = T(c, n->inputs, 1);
  const int cw = (K + 31) / 32;
  B_ENSURE(c, q && q->type == kTfLiteInt32 && q->dims->size >= 1 && Count(q) % cw == 0,
           "LceBfc: the input must be packed signs of whole rows of ceil(K / 32) words");
  B_ENSURE(c, f && f->type == kTfLiteInt32 && f->allocation_type == kTfLiteMmapRo && f->dims->size == 4 &&
                  f->dims->data[1] == 1 && f->dims->data[2] == 1 && f->dims->data[3] == cw,
           "LceBfc: the filter must be a constant packed [N, 1, 1, ceil(K / 32)]");
  const int N = f->dims->data[0];
  for (int k = 2; k < 6; ++k) {
    const TfLiteTensor* v = T(c, n->inputs, k);
    B_ENSURE(c, !v || (v->type == kTfLiteFloat32 && v->allocation_type == kTfLiteMmapRo && Count(v) == N),
             "LceBfc: alpha, bias, scale and shift must be constant float32 [N]");
  }
  const int64_t rows = Count(q) / cw;
  B_ENSURE(c, rows <= INT32_MAX, "LceBfc: too many rows");
  // FULLY_CONNECTED's keep_num_dims: q's leading axes (the input's), then N (the pass took it only when
  // the input's last axis is K, so q holds one row per leading index)
  auto shape = [&](int last) {
    std::vector<int> d{static_cast<int>(rows), last};
    if (op->p.fc.keep_dims) {
      d.assign(q->dims->data, q->dims->data + q->dims->size);
      d.back() = last;
    }
    return d;
  };
  if (ResizeTo(c, T(c, n->outputs, 0), shape(N)) != kTfLiteOk) return kTfLiteError;
  if (n->outputs->size == 2) {
    TfLiteTensor* pk = T(c, n->outputs, 1);
    B_ENSURE(c, pk && pk->type == kTfLiteInt32, "LceBfc+LceQuantize: packed output must be int32");
    if (ResizeTo(c, pk, shape((N + 31) / 32)) != kTfLiteOk) return kTfLiteError;
  }
  if (op->plan) {
    B_CAPI(c, lce_b200_bconv2d_set_input_shape(op->plan, static_cast<int>(rows), 1, 1));
    return kTfLiteOk;
  }
  lce_bconv2d_desc d;
  memset(&d, 0, sizeof(d));
  d.batch = static_cast<int>(rows); d.in_h = 1; d.in_w = 1; d.channels_in = K;
  d.filter_h = 1; d.filter_w = 1; d.channels_out = N; d.groups = 1;
  d.stride_h = 1; d.stride_w = 1; d.dilation_h = 1; d.dilation_w = 1;
  d.padding = LCE_PADDING_VALID; d.pad_value = 1; d.activation = LCE_ACT_NONE; d.out_type = LCE_OUT_FLOAT;
  const std::vector<float> ones(N, 1.0f), zeros(N, 0.0f);
  B_CAPI(c, lce_b200_bconv2d_create(&d, f->data.i32, ones.data(), zeros.data(), nullptr, &op->plan));
  return kTfLiteOk;
}
TfLiteStatus BinaryFcInvoke(TfLiteContext* c, TfLiteNode* n) {
  const auto* op = static_cast<const BinaryFcOp*>(n->user_data);
  auto vec = [&](int k) -> const float* {
    const TfLiteTensor* v = T(c, n->inputs, k);
    return v ? v->data.f : nullptr;
  };
  TfLiteTensor* pk = n->outputs->size > 1 ? T(c, n->outputs, 1) : nullptr;
  B_CAPI(c, lce_b200_bconv2d_run_fused_fc(op->plan, T(c, n->inputs, 0)->data.i32, vec(2), vec(3),
                                          op->p.fc.activation, vec(4), vec(5), op->p.add.activation,
                                          T(c, n->outputs, 0)->data.f, pk ? pk->data.i32 : nullptr,
                                          lce_b200_get_stream()));
  return kTfLiteOk;
}

// --- fused LceDequantize -> FULLY_CONNECTED [-> MUL -> ADD] -> REDUCE_MAX(points) [-> LceQuantize] --- //
// Created by Graph::FuseBinaryFcMax; builtin_data = BinaryFcMaxParams; inputs as LceBfc's, outputs [max
// [B, N] (or [B, 1, N] with keep_dims)?, packed signs [B, N / 32]?] as the params say, temporaries [keys:
// B * N 64-bit words]. The rows follow q's size (B * points), so a batch resize re-plans them. The node
// owns a 1x1 LceBconv2d plan of rows x 1 x 1 and runs lce_b200_bconv2d_run_fused_fc_max, which
// initialises the keys itself.
struct BinaryFcMaxOp {
  BinaryFcMaxParams p;
  lce_b200_bconv2d* plan = nullptr;
};
void* BinaryFcMaxInit(TfLiteContext*, const char* buffer, size_t length) {
  auto* op = new BinaryFcMaxOp();
  memset(&op->p, 0, sizeof(op->p));
  if (buffer && length >= sizeof(BinaryFcMaxParams)) memcpy(&op->p, buffer, sizeof(BinaryFcMaxParams));
  return op;
}
void BinaryFcMaxFree(TfLiteContext*, void* p) {
  auto* op = static_cast<BinaryFcMaxOp*>(p);
  lce_b200_bconv2d_destroy(op->plan);
  delete op;
}
TfLiteStatus BinaryFcMaxPrepare(TfLiteContext* c, TfLiteNode* n) {
  auto* op = static_cast<BinaryFcMaxOp*>(n->user_data);
  const BinaryFcMaxParams& p = op->p;
  const int K = p.channels_in, P = p.points;
  B_ENSURE(c, n->inputs->size == 6 && K > 0 && P > 0 && (p.store_max || p.store_signs) &&
                  n->outputs->size == p.store_max + p.store_signs,
           "LceBfc+REDUCE_MAX: inputs [q, filter, alpha, bias, scale, shift] and the max and/or its signs expected");
  const TfLiteTensor* q = T(c, n->inputs, 0);
  const TfLiteTensor* f = T(c, n->inputs, 1);
  const int cw = (K + 31) / 32;
  B_ENSURE(c, q && q->type == kTfLiteInt32 && q->dims->size == 3 && q->dims->data[1] == P && q->dims->data[2] == cw,
           "LceBfc+REDUCE_MAX: the input must be packed signs [B, points, ceil(K / 32)]");
  B_ENSURE(c, f && f->type == kTfLiteInt32 && f->allocation_type == kTfLiteMmapRo && f->dims->size == 4 &&
                  f->dims->data[1] == 1 && f->dims->data[2] == 1 && f->dims->data[3] == cw,
           "LceBfc+REDUCE_MAX: the filter must be a constant packed [N, 1, 1, ceil(K / 32)]");
  const int N = f->dims->data[0];
  B_ENSURE(c, N % 32 == 0, "LceBfc+REDUCE_MAX: N must be a multiple of 32");
  for (int k = 2; k < 6; ++k) {
    const TfLiteTensor* v = T(c, n->inputs, k);
    B_ENSURE(c, !v || (v->type == kTfLiteFloat32 && v->allocation_type == kTfLiteMmapRo && Count(v) == N),
             "LceBfc+REDUCE_MAX: alpha, bias, scale and shift must be constant float32 [N]");
  }
  const int B = q->dims->data[0];
  const int64_t rows = static_cast<int64_t>(B) * P;
  B_ENSURE(c, rows <= INT32_MAX, "LceBfc+REDUCE_MAX: too many rows");
  int o = 0;
  if (p.store_max) {
    TfLiteTensor* mx = T(c, n->outputs, o++);
    B_ENSURE(c, mx && mx->type == kTfLiteFloat32, "LceBfc+REDUCE_MAX: the max must be float32");
    if (ResizeTo(c, mx, p.reduce.keep_dims ? std::vector<int>{B, 1, N} : std::vector<int>{B, N}) != kTfLiteOk)
      return kTfLiteError;
  }
  if (p.store_signs) {
    TfLiteTensor* pk = T(c, n->outputs, o);
    B_ENSURE(c, pk && pk->type == kTfLiteInt32, "LceBfc+REDUCE_MAX+LceQuantize: packed output must be int32");
    if (ResizeTo(c, pk, p.reduce.keep_dims ? std::vector<int>{B, 1, N / 32} : std::vector<int>{B, N / 32}) !=
        kTfLiteOk)
      return kTfLiteError;
  }
  if (n->temporaries->size != 1) {
    int first = 0;
    if (c->AddTensors(c, 1, &first) != kTfLiteOk) return kTfLiteError;
    LceB200IntArrayFree(n->temporaries);
    n->temporaries = LceB200IntArrayCreate(1);
    n->temporaries->data[0] = first;
  }
  TfLiteTensor* keys = &c->tensors[n->temporaries->data[0]];   // c->tensors may have moved
  keys->type = kTfLiteInt64;
  if (Resize(c, keys, {std::max(B, 1) * N}) != kTfLiteOk) return kTfLiteError;
  if (op->plan) {
    B_CAPI(c, lce_b200_bconv2d_set_input_shape(op->plan, static_cast<int>(rows), 1, 1));
    return kTfLiteOk;
  }
  lce_bconv2d_desc d;
  memset(&d, 0, sizeof(d));
  d.batch = static_cast<int>(rows); d.in_h = 1; d.in_w = 1; d.channels_in = K;
  d.filter_h = 1; d.filter_w = 1; d.channels_out = N; d.groups = 1;
  d.stride_h = 1; d.stride_w = 1; d.dilation_h = 1; d.dilation_w = 1;
  d.padding = LCE_PADDING_VALID; d.pad_value = 1; d.activation = LCE_ACT_NONE; d.out_type = LCE_OUT_FLOAT;
  const std::vector<float> ones(N, 1.0f), zeros(N, 0.0f);
  B_CAPI(c, lce_b200_bconv2d_create(&d, f->data.i32, ones.data(), zeros.data(), nullptr, &op->plan));
  return kTfLiteOk;
}
TfLiteStatus BinaryFcMaxInvoke(TfLiteContext* c, TfLiteNode* n) {
  const auto* op = static_cast<const BinaryFcMaxOp*>(n->user_data);
  const BinaryFcMaxParams& p = op->p;
  auto vec = [&](int k) -> const float* {
    const TfLiteTensor* v = T(c, n->inputs, k);
    return v ? v->data.f : nullptr;
  };
  float* mx = p.store_max ? T(c, n->outputs, 0)->data.f : nullptr;
  int32_t* pk = p.store_signs ? T(c, n->outputs, p.store_max)->data.i32 : nullptr;
  B_CAPI(c, lce_b200_bconv2d_run_fused_fc_max(op->plan, T(c, n->inputs, 0)->data.i32, vec(2), vec(3), p.fc.activation,
                                              vec(4), vec(5), p.add.activation, p.points,
                                              c->tensors[n->temporaries->data[0]].data.raw, mx, pk,
                                              lce_b200_get_stream()));
  return kTfLiteOk;
}

// ------------------------------ CONCATENATION ------------------------------ //
// Strided device copies (one cudaMemcpy2DAsync per input): no kernel of ours.
TfLiteStatus ConcatPrepare(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* a = T(c, n->inputs, 0);
  B_ENSURE(c, a && n->inputs->size >= 1, "CONCATENATION: no inputs");
  const int r = a->dims->size;
  int axis = P(n).axis < 0 ? P(n).axis + r : P(n).axis;
  B_ENSURE(c, axis >= 0 && axis < r, "CONCATENATION: axis out of range");
  B_ENSURE(c, P(n).activation == 0, "CONCATENATION: fused activation is not supported");
  int sum = 0;
  for (int k = 0; k < n->inputs->size; ++k) {
    const TfLiteTensor* t = T(c, n->inputs, k);
    B_ENSURE(c, t && t->dims->size == r && t->type == a->type,
             "CONCATENATION: inputs must agree in rank and type");
    for (int i = 0; i < r; ++i)
      B_ENSURE(c, i == axis || t->dims->data[i] == a->dims->data[i],
               "CONCATENATION: inputs must agree outside the axis");
    sum += t->dims->data[axis];
  }
  TfLiteIntArray* dims = LceB200IntArrayCreate(r);
  for (int i = 0; i < r; ++i) dims->data[i] = i == axis ? sum : a->dims->data[i];
  return c->ResizeTensor(c, T(c, n->outputs, 0), dims);
}
TfLiteStatus ConcatInvoke(TfLiteContext* c, TfLiteNode* n) {
  TfLiteTensor* out = T(c, n->outputs, 0);
  const int r = out->dims->size;
  const int axis = P(n).axis < 0 ? P(n).axis + r : P(n).axis;
  size_t outer = 1, inner = out->bytes / std::max<int64_t>(Count(out), 1);  // element size
  for (int i = 0; i < axis; ++i) outer *= out->dims->data[i];
  for (int i = axis + 1; i < r; ++i) inner *= out->dims->data[i];
  const size_t out_pitch = inner * out->dims->data[axis];
  size_t off = 0;
  for (int k = 0; k < n->inputs->size; ++k) {
    const TfLiteTensor* t = T(c, n->inputs, k);
    const size_t w = inner * t->dims->data[axis];
    if (w && outer &&
        cudaMemcpy2DAsync(out->data.raw + off, out_pitch, t->data.raw, w, w, outer,
                          cudaMemcpyDefault,
                          static_cast<cudaStream_t>(lce_b200_get_stream())) != cudaSuccess) {
      c->ReportError(c, "CONCATENATION: device copy failed");
      return kTfLiteError;
    }
    off += w;
  }
  return kTfLiteOk;
}

// ----------------------------- STRIDED_SLICE / SPLIT ----------------------------- //
// One strided device copy per output, as CONCATENATION: no kernel of ours. Every index vector is a
// host constant. The copy of outer rows of `width` bytes, each `pitch` bytes apart in x.
TfLiteStatus CopyRows(TfLiteContext* c, void* dst, const void* src, size_t width, size_t pitch,
                      size_t rows, const char* what) {
  if (width && rows &&
      cudaMemcpy2DAsync(dst, width, src, pitch, width, rows, cudaMemcpyDeviceToDevice,
                        static_cast<cudaStream_t>(lce_b200_get_stream())) != cudaSuccess) {
    c->ReportError(c, "%s: device copy failed", what);
    return kTfLiteError;
  }
  return kTfLiteOk;
}
// A constant int32 tensor in host memory (the model's own buffer), or nullptr.
const int32_t* HostInts(const TfLiteTensor* t) {
  return t && t->type == kTfLiteInt32 && t->data.raw && !OnDevice(t->data.raw) ? t->data.i32 : nullptr;
}
// inputs [x (float32 / int32), begin, end, strides]
const char* SliceGeometry(TfLiteContext* c, TfLiteNode* n, SliceBounds* sb) {
  const TfLiteTensor* x = T(c, n->inputs, 0);
  if (n->inputs->size != 4 || !x || (x->type != kTfLiteFloat32 && x->type != kTfLiteInt32))
    return "STRIDED_SLICE: a float32 or int32 input, then begin, end and strides, expected";
  const TfLiteTensor* v[3] = {T(c, n->inputs, 1), T(c, n->inputs, 2), T(c, n->inputs, 3)};
  for (const TfLiteTensor* t : v)
    if (!HostInts(t) || t->dims->size != 1 || t->dims->data[0] != v[0]->dims->data[0])
      return "STRIDED_SLICE: begin, end and strides must be constant int32 vectors of one length";
  return StridedSliceBounds(x->dims->data, x->dims->size, v[0]->data.i32, v[1]->data.i32,
                            v[2]->data.i32, v[0]->dims->data[0], P(n), sb);
}
TfLiteStatus StridedSlicePrepare(TfLiteContext* c, TfLiteNode* n) {
  SliceBounds sb;
  const char* why = SliceGeometry(c, n, &sb);
  B_ENSURE(c, why == nullptr, why);
  TfLiteIntArray* dims = LceB200IntArrayCreate(sb.rank);
  for (int k = 0; k < sb.rank; ++k) dims->data[k] = sb.end[k] - sb.begin[k];
  return c->ResizeTensor(c, T(c, n->outputs, 0), dims);
}
TfLiteStatus StridedSliceInvoke(TfLiteContext* c, TfLiteNode* n) {
  SliceBounds sb;
  const char* why = SliceGeometry(c, n, &sb);
  B_ENSURE(c, why == nullptr, why);
  const TfLiteTensor* x = T(c, n->inputs, 0);
  int a = 0;   // the sliced axis (axis 0 when the slice is the whole of x)
  while (a + 1 < sb.rank && sb.begin[a] == 0 && sb.end[a] == x->dims->data[a]) ++a;
  size_t outer = 1, inner = 4;
  for (int k = 0; k < a; ++k) outer *= x->dims->data[k];
  for (int k = a + 1; k < sb.rank; ++k) inner *= x->dims->data[k];
  return CopyRows(c, T(c, n->outputs, 0)->data.raw, x->data.raw + sb.begin[a] * inner,
                  (sb.end[a] - sb.begin[a]) * inner, x->dims->data[a] * inner, outer, "STRIDED_SLICE");
}

// inputs [axis (constant int32 scalar, negative counts from the end), x (float32 / int32)];
// num_splits outputs of equal size along the axis
bool SplitGeometry(TfLiteContext* c, TfLiteNode* n, int* axis, size_t* outer, size_t* inner) {
  const TfLiteTensor* ax = T(c, n->inputs, 0);
  const TfLiteTensor* x = T(c, n->inputs, 1);
  if (n->inputs->size != 2 || !HostInts(ax) || Count(ax) != 1 || !x ||
      (x->type != kTfLiteFloat32 && x->type != kTfLiteInt32) || x->dims->size < 1 || x->dims->size > 4)
    return false;
  const int r = x->dims->size;
  *axis = ax->data.i32[0] < 0 ? ax->data.i32[0] + r : ax->data.i32[0];
  if (*axis < 0 || *axis >= r) return false;
  *outer = 1;
  *inner = 4;
  for (int k = 0; k < *axis; ++k) *outer *= x->dims->data[k];
  for (int k = *axis + 1; k < r; ++k) *inner *= x->dims->data[k];
  return true;
}
TfLiteStatus SplitPrepare(TfLiteContext* c, TfLiteNode* n) {
  int axis;
  size_t outer, inner;
  B_ENSURE(c, SplitGeometry(c, n, &axis, &outer, &inner),
           "SPLIT: a constant int32 axis within the input's rank, and a float32 or int32 input of "
           "rank 1 to 4, expected");
  const TfLiteTensor* x = T(c, n->inputs, 1);
  const int parts = P(n).num_splits;
  B_ENSURE(c, parts > 0 && n->outputs->size == parts, "SPLIT: num_splits must equal the output count");
  B_ENSURE(c, x->dims->data[axis] % parts == 0, "SPLIT: num_splits must divide the axis");
  for (int k = 0; k < parts; ++k) {
    TfLiteIntArray* dims = LceB200IntArrayCreate(x->dims->size);
    for (int i = 0; i < x->dims->size; ++i)
      dims->data[i] = i == axis ? x->dims->data[i] / parts : x->dims->data[i];
    if (c->ResizeTensor(c, T(c, n->outputs, k), dims) != kTfLiteOk) return kTfLiteError;
  }
  return kTfLiteOk;
}
TfLiteStatus SplitInvoke(TfLiteContext* c, TfLiteNode* n) {
  int axis;
  size_t outer, inner;
  B_ENSURE(c, SplitGeometry(c, n, &axis, &outer, &inner), "SPLIT: bad axis or input");
  const TfLiteTensor* x = T(c, n->inputs, 1);
  const size_t pitch = x->dims->data[axis] * inner, width = pitch / n->outputs->size;
  for (int k = 0; k < n->outputs->size; ++k)
    if (CopyRows(c, T(c, n->outputs, k)->data.raw, x->data.raw + k * width, width, pitch, outer,
                 "SPLIT") != kTfLiteOk)
      return kTfLiteError;
  return kTfLiteOk;
}


// -------------------------- TFLite_Detection_PostProcess -------------------------- //
// The custom op that ends a TF Object Detection API SSD (TF/lite/kernels/detection_postprocess.cc),
// float32 inputs only, over the whole batch. inputs [box encodings [B, N, K >= 4], class predictions
// [B, N, num_classes + label_offset], anchors (constant [N, 4])], outputs [boxes [B, D, 4], classes
// [B, D], scores [B, D], num_detections [B]] with D = max_detections * max_classes_per_detection, one
// temporary: lce_b200_f32_detection_postprocess's workspace. The anchors are a constant of a custom op,
// so the reader leaves them on the host; Prepare validates them there and copies them to device memory
// the op owns, once.
struct DetectionOp {
  lce_b200_detection_options o;
  float* anchors_dev = nullptr;
};
void* DetectionInit(TfLiteContext*, const char* buffer, size_t length) {
  auto* op = new DetectionOp();
  const FlexMap m(reinterpret_cast<const uint8_t*>(buffer), length);
  lce_b200_detection_options& o = op->o;
  o.max_detections = m.AsInt32("max_detections");
  o.max_classes_per_detection = m.AsInt32("max_classes_per_detection");
  o.detections_per_class = m.Has("detections_per_class") ? m.AsInt32("detections_per_class") : 100;
  o.num_classes = m.AsInt32("num_classes");
  o.use_regular_nms = m.AsBool("use_regular_nms", false) ? 1 : 0;
  o.nms_score_threshold = m.AsFloat("nms_score_threshold", 0.0f);
  o.nms_iou_threshold = m.AsFloat("nms_iou_threshold", 0.0f);
  o.y_scale = m.AsFloat("y_scale", 0.0f);
  o.x_scale = m.AsFloat("x_scale", 0.0f);
  o.h_scale = m.AsFloat("h_scale", 0.0f);
  o.w_scale = m.AsFloat("w_scale", 0.0f);
  return op;
}
void DetectionFree(TfLiteContext*, void* p) {
  auto* op = static_cast<DetectionOp*>(p);
  if (op->anchors_dev) cudaFree(op->anchors_dev);
  delete op;
}
TfLiteStatus DetectionPrepare(TfLiteContext* c, TfLiteNode* n) {
  auto* op = static_cast<DetectionOp*>(n->user_data);
  const lce_b200_detection_options& o = op->o;
  B_ENSURE(c, n->inputs->size == 3 && n->outputs->size == 4,
           "TFLite_Detection_PostProcess: three inputs and four outputs expected");
  const TfLiteTensor* boxes = T(c, n->inputs, 0);
  const TfLiteTensor* scores = T(c, n->inputs, 1);
  const TfLiteTensor* anchors = T(c, n->inputs, 2);
  B_ENSURE(c, boxes && scores && anchors && boxes->type == kTfLiteFloat32 && scores->type == kTfLiteFloat32 &&
                  anchors->type == kTfLiteFloat32,
           "TFLite_Detection_PostProcess: box encodings, class predictions and anchors must be float32 "
           "(quantized post-processing is not supported)");
  B_ENSURE(c, boxes->dims->size == 3 && scores->dims->size == 3 && anchors->dims->size == 2,
           "TFLite_Detection_PostProcess: box encodings and class predictions must be 3-D, anchors 2-D");
  const int B = boxes->dims->data[0], N = boxes->dims->data[1], K = boxes->dims->data[2];
  const int S = scores->dims->data[2];
  B_ENSURE(c, scores->dims->data[0] == B && scores->dims->data[1] == N && anchors->dims->data[0] == N &&
                  anchors->dims->data[1] == 4 && K >= 4 && N >= 1 && S >= 1,
           "TFLite_Detection_PostProcess: shapes must be box encodings [B, N, >= 4], class predictions "
           "[B, N, C] and anchors [N, 4]");
  B_ENSURE(c, o.num_classes >= 1 && o.num_classes <= S,
           "TFLite_Detection_PostProcess: num_classes must be in [1, the class predictions' last dimension]");
  B_ENSURE(c, o.max_detections >= 1, "TFLite_Detection_PostProcess: max_detections must be at least 1");
  B_ENSURE(c, o.max_classes_per_detection >= 1,
           "TFLite_Detection_PostProcess: max_classes_per_detection must be at least 1");
  B_ENSURE(c, !o.use_regular_nms || o.detections_per_class >= 1,
           "TFLite_Detection_PostProcess: detections_per_class must be at least 1");
  B_ENSURE(c, o.nms_iou_threshold > 0.0f && o.nms_iou_threshold <= 1.0f,
           "TFLite_Detection_PostProcess: nms_iou_threshold must be in (0, 1]");
  if (N > lce_b200_detection_max_anchors()) {
    c->ReportError(c, "TFLite_Detection_PostProcess: %d anchors are more than the %d one image's NMS holds in "
                   "shared memory", N, lce_b200_detection_max_anchors());
    return kTfLiteError;
  }
  B_ENSURE(c, anchors->allocation_type == kTfLiteMmapRo && anchors->data.raw && !OnDevice(anchors->data.raw),
           "TFLite_Detection_PostProcess: the anchors must be a constant tensor");
  for (int i = 0; i < N; ++i) {
    const float h = anchors->data.f[4 * i + 2], w = anchors->data.f[4 * i + 3];
    B_ENSURE(c, std::isfinite(h) && std::isfinite(w) && h >= 0.0f && w >= 0.0f,
             "TFLite_Detection_PostProcess: anchor heights and widths must be finite and non-negative");
  }
  if (!op->anchors_dev) {   // no device on a host-arena graph: Invoke then reports it
    void* d = nullptr;
    if (cudaMalloc(&d, sizeof(float) * 4 * N) == cudaSuccess &&
        cudaMemcpy(d, anchors->data.raw, sizeof(float) * 4 * N, cudaMemcpyHostToDevice) == cudaSuccess) {
      op->anchors_dev = static_cast<float*>(d);
    } else {
      if (d) cudaFree(d);
      cudaGetLastError();
    }
  }
  if (n->temporaries->size != 1) {
    int first = 0;
    if (c->AddTensors(c, 1, &first) != kTfLiteOk) return kTfLiteError;
    LceB200IntArrayFree(n->temporaries);
    n->temporaries = LceB200IntArrayCreate(1);
    n->temporaries->data[0] = first;
  }
  TfLiteTensor* ws = &c->tensors[n->temporaries->data[0]];   // c->tensors may have moved
  ws->type = kTfLiteUInt8;
  const size_t bytes = lce_b200_detection_workspace_bytes(std::max(B, 1), N, &o);
  B_ENSURE(c, bytes > 0 && bytes <= static_cast<size_t>(INT32_MAX),
           "TFLite_Detection_PostProcess: the batch needs too large a workspace");
  if (Resize(c, ws, {static_cast<int>(bytes)}) != kTfLiteOk) return kTfLiteError;
  const int D = o.max_detections * o.max_classes_per_detection;
  if (Resize(c, T(c, n->outputs, 0), {B, D, 4}) != kTfLiteOk || Resize(c, T(c, n->outputs, 1), {B, D}) != kTfLiteOk ||
      Resize(c, T(c, n->outputs, 2), {B, D}) != kTfLiteOk || Resize(c, T(c, n->outputs, 3), {B}) != kTfLiteOk)
    return kTfLiteError;
  for (int k = 0; k < 4; ++k)
    B_ENSURE(c, T(c, n->outputs, k)->type == kTfLiteFloat32, "TFLite_Detection_PostProcess: outputs must be float32");
  return kTfLiteOk;
}
TfLiteStatus DetectionInvoke(TfLiteContext* c, TfLiteNode* n) {
  const auto* op = static_cast<const DetectionOp*>(n->user_data);
  B_ENSURE(c, op->anchors_dev, "TFLite_Detection_PostProcess: the anchors could not be copied to the device");
  const TfLiteTensor* boxes = T(c, n->inputs, 0);
  const TfLiteTensor* scores = T(c, n->inputs, 1);
  const int* d = boxes->dims->data;
  B_CAPI(c, lce_b200_f32_detection_postprocess(
                boxes->data.f, scores->data.f, d[0], d[1], d[2], scores->dims->data[2], op->anchors_dev, &op->o,
                T(c, n->outputs, 0)->data.f, T(c, n->outputs, 1)->data.f, T(c, n->outputs, 2)->data.f,
                T(c, n->outputs, 3)->data.f, c->tensors[n->temporaries->data[0]].data.raw, lce_b200_get_stream()));
  return kTfLiteOk;
}
}  // namespace

const char* StridedSliceBounds(const int32_t* dims, int rank, const int32_t* begin, const int32_t* end,
                               const int32_t* strides, int n, const BuiltinParams& p, SliceBounds* out) {
  if (rank < 1 || rank > 4) return "STRIDED_SLICE: the input's rank must be 1 to 4";
  if (n < 1 || n > rank) return "STRIDED_SLICE: begin, end and strides need 1 to rank values";
  if (p.ellipsis_mask || p.new_axis_mask || p.shrink_axis_mask)
    return "STRIDED_SLICE: ellipsis_mask, new_axis_mask and shrink_axis_mask are not supported";
  if (p.offset) return "STRIDED_SLICE: offset is not supported";
  out->rank = rank;
  int sliced = 0;
  for (int k = 0; k < rank; ++k) {
    const int64_t size = dims[k];
    int64_t b = 0, e = size;
    if (k < n) {   // the axes beyond n are whole
      if (strides[k] != 1) return "STRIDED_SLICE: only unit strides are supported";
      // strided_slice_logic.h StartForAxis / EndForAxis at stride 1: a mask bit takes the whole
      // side, a negative index counts from the end, then both clamp to [0, size]
      b = (p.begin_mask >> k) & 1 ? 0 : begin[k];
      e = (p.end_mask >> k) & 1 ? size : end[k];
      if (b < 0) b += size;
      if (e < 0) e += size;
      b = std::min(std::max<int64_t>(b, 0), size);
      e = std::min(std::max(e, b), size);
    }
    out->begin[k] = static_cast<int>(b);
    out->end[k] = static_cast<int>(e);
    if (b != 0 || e != size) ++sliced;
  }
  if (sliced > 1) return "STRIDED_SLICE: at most one axis may be sliced";
  return nullptr;
}

const char* ArgMaxAxis(const TfLiteTensor* axis, int rank, int* out) {
  if (!axis || axis->allocation_type != kTfLiteMmapRo || !axis->data.raw || OnDevice(axis->data.raw))
    return "ARG_MAX: the axis must be a constant tensor";
  if (axis->type != kTfLiteInt32 && axis->type != kTfLiteInt64) return "ARG_MAX: the axis must be int32 or int64";
  if (axis->dims->size > 1 || Count(axis) != 1) return "ARG_MAX: the axis must have exactly one element";
  int64_t a;
  if (axis->type == kTfLiteInt32) {
    a = axis->data.i32[0];
  } else {
    memcpy(&a, axis->data.raw, sizeof(a));
  }
  if (a < -rank || a >= rank) return "ARG_MAX: the axis is out of range";
  *out = static_cast<int>(a < 0 ? a + rank : a);
  return nullptr;
}

const TfLiteRegistration* FusedStemRegistration() {
  static TfLiteRegistration r = {StemInit, StemFree, StemPrepare, StemInvoke};
  return &r;
}
const TfLiteRegistration* FusedPoolDepthwiseRegistration() {
  static TfLiteRegistration r = {PoolDwInit, PoolDwFree, PoolDwPrepare, PoolDwInvoke};
  return &r;
}
const TfLiteRegistration* ActivationChainRegistration() {
  static TfLiteRegistration r = {Init, Free, ChainPrepare, ChainInvoke};
  return &r;
}
const TfLiteRegistration* Quant2Registration() {
  static TfLiteRegistration r = {Init, Free, Quant2Prepare, Quant2Invoke};
  return &r;
}
const TfLiteRegistration* PooledSignRegistration() {
  static TfLiteRegistration r = {Init, Free, PooledSignPrepare, PooledSignInvoke};
  return &r;
}
const TfLiteRegistration* GroupedConvAffineRegistration() {
  static TfLiteRegistration r = {ConvAffineInit, ConvAffineFree, ConvAffinePrepare, ConvAffineInvoke};
  return &r;
}
const TfLiteRegistration* ResizeArgmaxRegistration() {
  static TfLiteRegistration r = {ResizeArgmaxInit, ResizeArgmaxFree, ResizeArgmaxPrepare, ResizeArgmaxInvoke};
  return &r;
}
const TfLiteRegistration* BinaryTransposeConvRegistration() {
  static TfLiteRegistration r = {BinaryTConvInit, BinaryTConvFree, BinaryTConvPrepare, BinaryTConvInvoke};
  return &r;
}
const TfLiteRegistration* BinaryFullyConnectedRegistration() {
  static TfLiteRegistration r = {BinaryFcInit, BinaryFcFree, BinaryFcPrepare, BinaryFcInvoke};
  return &r;
}
const TfLiteRegistration* BinaryFcMaxRegistration() {
  static TfLiteRegistration r = {BinaryFcMaxInit, BinaryFcMaxFree, BinaryFcMaxPrepare, BinaryFcMaxInvoke};
  return &r;
}
const TfLiteRegistration* SubpixelConvRegistration() {
  static TfLiteRegistration r = {SubpixelInit, SubpixelFree, SubpixelPrepare, SubpixelInvoke};
  return &r;
}
const TfLiteRegistration* UpsampleMergeRegistration() {
  static TfLiteRegistration r = {MergeInit, MergeFree, MergePrepare, MergeInvoke};
  return &r;
}

void RegisterBuiltinOps(OpResolver* r) {
  static TfLiteRegistration conv = {Init, Free, ConvPrepare<false>, ConvInvoke<false>};
  static TfLiteRegistration dw = {Init, Free, ConvPrepare<true>, ConvInvoke<true>};
  static TfLiteRegistration fc = {Init, Free, FcPrepare, FcInvoke};
  static TfLiteRegistration maxp = {Init, Free, PoolPrepare, PoolInvoke<true>};
  static TfLiteRegistration avgp = {Init, Free, PoolPrepare, PoolInvoke<false>};
  static TfLiteRegistration add = {Init, Free, EltPrepare<false>, EltInvoke<false>};
  static TfLiteRegistration mul = {Init, Free, EltPrepare<true>, EltInvoke<true>};
  static TfLiteRegistration relu = {Init, Free, SameShapePrepare, ReluInvoke};
  static TfLiteRegistration mean = {Init, Free, MeanPrepare, MeanInvoke};
  static TfLiteRegistration softmax = {Init, Free, SameShapePrepare, SoftmaxInvoke};
  static TfLiteRegistration reshape = {Init, Free, ReshapePrepare, ReshapeInvoke};
  // BuiltinOperator codes, schema.fbs:259-325
  r->AddBuiltin(3, &conv);
  r->AddBuiltin(4, &dw);
  r->AddBuiltin(9, &fc);
  r->AddBuiltin(17, &maxp);
  r->AddBuiltin(1, &avgp);
  r->AddBuiltin(0, &add);
  r->AddBuiltin(18, &mul);
  r->AddBuiltin(19, &relu);
  r->AddBuiltin(40, &mean);
  r->AddBuiltin(25, &softmax);
  r->AddBuiltin(22, &reshape);
  static TfLiteRegistration pad = {Init, Free, PadPrepare, PadInvoke};
  static TfLiteRegistration concat = {Init, Free, ConcatPrepare, ConcatInvoke};
  r->AddBuiltin(34, &pad);   // PAD
  r->AddBuiltin(60, &pad);   // PADV2
  r->AddBuiltin(2, &concat);  // CONCATENATION
  static TfLiteRegistration dequant = {Init, Free, DequantPrepare, DequantInvoke};
  r->AddBuiltin(6, &dequant);  // DEQUANTIZE
  static TfLiteRegistration prelu = {Init, Free, PreluPrepare, PreluInvoke};
  r->AddBuiltin(54, &prelu);   // PRELU
  static TfLiteRegistration logistic = {Init, Free, LogisticPrepare, LogisticInvoke};
  r->AddBuiltin(14, &logistic);  // LOGISTIC
  static TfLiteRegistration maximum = {Init, Free, MinMaxDivPrepare<55>, MinMaxDivInvoke<55>};
  static TfLiteRegistration minimum = {Init, Free, MinMaxDivPrepare<57>, MinMaxDivInvoke<57>};
  static TfLiteRegistration div = {Init, Free, MinMaxDivPrepare<42>, MinMaxDivInvoke<42>};
  static TfLiteRegistration round = {Init, Free, RoundPrepare, RoundInvoke};
  r->AddBuiltin(55, &maximum);   // MAXIMUM
  r->AddBuiltin(57, &minimum);   // MINIMUM
  r->AddBuiltin(42, &div);       // DIV
  r->AddBuiltin(116, &round);    // ROUND
  static TfLiteRegistration strided_slice = {Init, Free, StridedSlicePrepare, StridedSliceInvoke};
  r->AddBuiltin(45, &strided_slice);  // STRIDED_SLICE
  static TfLiteRegistration split = {Init, Free, SplitPrepare, SplitInvoke};
  r->AddBuiltin(49, &split);  // SPLIT
  static TfLiteRegistration resize_bilinear = {Init, Free, ResizePrepare<true>, ResizeInvoke<true>};
  static TfLiteRegistration resize_nearest = {Init, Free, ResizePrepare<false>, ResizeInvoke<false>};
  r->AddBuiltin(23, &resize_bilinear);  // RESIZE_BILINEAR
  r->AddBuiltin(97, &resize_nearest);   // RESIZE_NEAREST_NEIGHBOR
  static TfLiteRegistration arg_max = {Init, Free, ArgMaxPrepare, ArgMaxInvoke};
  r->AddBuiltin(56, &arg_max);   // ARG_MAX
  static TfLiteRegistration reduce_max = {Init, Free, ReduceMaxPrepare, ReduceMaxInvoke};
  r->AddBuiltin(82, &reduce_max);   // REDUCE_MAX
  static TfLiteRegistration depth_to_space = {Init, Free, DepthToSpacePrepare, DepthToSpaceInvoke};
  r->AddBuiltin(5, &depth_to_space);   // DEPTH_TO_SPACE
  static TfLiteRegistration transpose_conv = {Init, Free, TransposeConvPrepare, TransposeConvInvoke};
  r->AddBuiltin(67, &transpose_conv);   // TRANSPOSE_CONV
  static TfLiteRegistration detection = {DetectionInit, DetectionFree, DetectionPrepare, DetectionInvoke};
  r->AddCustom("TFLite_Detection_PostProcess", &detection);
}

}  // namespace lce_b200

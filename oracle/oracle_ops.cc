// oracle/oracle_ops.cc -- TEST INFRASTRUCTURE ONLY: the CPU oracle
// (oracle/lce_oracle.c) wrapped as TfLiteRegistrations, so that the graph host's
// plumbing (resolver, flexbuffer attributes, init -> prepare -> invoke, resize,
// arena) can be exercised WITHOUT a GPU: the "single
// LceBconv2d 56x56x256->256 k3 s1 on the CPU reference interpreter (bit-exact
// plumbing, no GPU)". Never linked into compute_engine_b200/.
#include <cstring>

#include "../compute_engine_b200/csrc/host/flexbuffer_map.h"
#include "../include/lce_b200_tflite.h"
#include "../include/lce_b200_types.h"

extern "C" {
int lce_oracle_bconv2d_out_shape(const lce_bconv2d_desc*, int*, int*, int*, int*);
int lce_oracle_bconv2d_mt(const lce_bconv2d_desc*, int, const int32_t*, const int32_t*,
                          const float*, const float*, const int32_t*, void*);
int lce_oracle_quantize(int, const void*, int64_t, int64_t, int32_t, int32_t*);
int lce_oracle_dequantize(int, const int32_t*, int64_t, int64_t, float, int32_t, void*);
int lce_oracle_bmaxpool_out_shape(const lce_bmaxpool_desc*, int*, int*);
int lce_oracle_bmaxpool(const lce_bmaxpool_desc*, const int32_t*, int32_t*);
}

namespace {
const TfLiteTensor* In(TfLiteContext* c, TfLiteNode* n, int i) {
  const int idx = n->inputs->data[i];
  return idx == kTfLiteOptionalTensor ? nullptr : &c->tensors[idx];
}
TfLiteTensor* Out(TfLiteContext* c, TfLiteNode* n, int i) { return &c->tensors[n->outputs->data[i]]; }
int64_t Count(const TfLiteTensor* t) {
  int64_t n = 1;
  for (int i = 0; i < t->dims->size; ++i) n *= t->dims->data[i];
  return n;
}

void* ConvInit(TfLiteContext*, const char* buffer, size_t length) {
  auto* d = new lce_bconv2d_desc();
  memset(d, 0, sizeof(*d));
  lce_b200::FlexMap m(reinterpret_cast<const uint8_t*>(buffer), length);
  d->stride_h = m.AsInt32("stride_height");
  d->stride_w = m.AsInt32("stride_width");
  d->dilation_h = m.AsInt32("dilation_height_factor");
  d->dilation_w = m.AsInt32("dilation_width_factor");
  d->padding = m.AsInt32("padding");
  d->pad_value = m.AsInt32("pad_values");
  d->channels_in = m.AsInt32("channels_in");
  d->activation = m.AsInt32("fused_activation_function");
  return d;
}
void ConvFree(TfLiteContext*, void* p) { delete static_cast<lce_bconv2d_desc*>(p); }
TfLiteStatus ConvPrepare(TfLiteContext* c, TfLiteNode* n) {
  auto* d = static_cast<lce_bconv2d_desc*>(n->user_data);
  const TfLiteTensor* in = In(c, n, 0);
  const TfLiteTensor* f = In(c, n, 1);
  TfLiteTensor* out = Out(c, n, 0);
  d->batch = in->dims->data[0];
  d->in_h = in->dims->data[1];
  d->in_w = in->dims->data[2];
  d->channels_out = f->dims->data[0];
  d->filter_h = f->dims->data[1];
  d->filter_w = f->dims->data[2];
  d->groups = ((d->channels_in + 31) / 32) / f->dims->data[3];
  d->out_type = out->type == kTfLiteFloat32 ? LCE_OUT_FLOAT
                : out->type == kTfLiteInt8  ? LCE_OUT_INT8
                                            : LCE_OUT_BITPACKED;
  d->out_scale = out->params.scale;
  d->out_zero_point = out->params.zero_point;
  int oh, ow, ph, pw;
  if (lce_oracle_bconv2d_out_shape(d, &oh, &ow, &ph, &pw)) return kTfLiteError;
  TfLiteIntArray* s = LceB200IntArrayCreate(4);
  s->data[0] = d->batch;
  s->data[1] = oh;
  s->data[2] = ow;
  s->data[3] = out->type == kTfLiteInt32 ? (d->channels_out + 31) / 32 : d->channels_out;
  return c->ResizeTensor(c, out, s);
}
TfLiteStatus ConvEval(TfLiteContext* c, TfLiteNode* n) {
  auto* d = static_cast<lce_bconv2d_desc*>(n->user_data);
  const TfLiteTensor* mul = In(c, n, 2);
  const TfLiteTensor* bias = In(c, n, 3);
  const TfLiteTensor* thr = In(c, n, 4);
  return lce_oracle_bconv2d_mt(d, c->recommended_num_threads, In(c, n, 0)->data.i32,
                               In(c, n, 1)->data.i32, mul ? mul->data.f : nullptr,
                               bias ? bias->data.f : nullptr, thr ? thr->data.i32 : nullptr,
                               Out(c, n, 0)->data.raw) == 0
             ? kTfLiteOk
             : kTfLiteError;
}

TfLiteStatus QPrepare(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* in = In(c, n, 0);
  TfLiteIntArray* s = LceB200IntArrayCreate(in->dims->size);
  for (int i = 0; i < in->dims->size; ++i) s->data[i] = in->dims->data[i];
  s->data[in->dims->size - 1] = (in->dims->data[in->dims->size - 1] + 31) / 32;
  return c->ResizeTensor(c, Out(c, n, 0), s);
}
TfLiteStatus QEval(TfLiteContext* c, TfLiteNode* n) {
  const TfLiteTensor* in = In(c, n, 0);
  const int t = in->type == kTfLiteFloat32 ? LCE_T_FLOAT : in->type == kTfLiteInt8 ? LCE_T_INT8 : LCE_T_BOOL;
  const int64_t cols = in->dims->data[in->dims->size - 1];
  return lce_oracle_quantize(t, in->data.raw, cols ? Count(in) / cols : 0, cols,
                             in->params.zero_point, Out(c, n, 0)->data.i32) == 0
             ? kTfLiteOk
             : kTfLiteError;
}
TfLiteStatus DQPrepare(TfLiteContext*, TfLiteNode*) { return kTfLiteOk; }
TfLiteStatus DQEval(TfLiteContext* c, TfLiteNode* n) {
  TfLiteTensor* out = Out(c, n, 0);
  const int t = out->type == kTfLiteFloat32 ? LCE_T_FLOAT : out->type == kTfLiteInt8 ? LCE_T_INT8 : LCE_T_BOOL;
  const int64_t cols = out->dims->data[out->dims->size - 1];
  return lce_oracle_dequantize(t, In(c, n, 0)->data.i32, cols ? Count(out) / cols : 0, cols,
                               out->params.scale, out->params.zero_point, out->data.raw) == 0
             ? kTfLiteOk
             : kTfLiteError;
}

void* PoolInit(TfLiteContext*, const char* buffer, size_t length) {
  auto* d = new lce_bmaxpool_desc();
  memset(d, 0, sizeof(*d));
  lce_b200::FlexMap m(reinterpret_cast<const uint8_t*>(buffer), length);
  d->filter_h = m.AsInt32("filter_height");
  d->filter_w = m.AsInt32("filter_width");
  d->stride_h = m.AsInt32("stride_height");
  d->stride_w = m.AsInt32("stride_width");
  d->padding = m.AsInt32("padding");
  return d;
}
void PoolFree(TfLiteContext*, void* p) { delete static_cast<lce_bmaxpool_desc*>(p); }
TfLiteStatus PoolPrepare(TfLiteContext* c, TfLiteNode* n) {
  auto* d = static_cast<lce_bmaxpool_desc*>(n->user_data);
  const TfLiteTensor* in = In(c, n, 0);
  d->batch = in->dims->data[0];
  d->in_h = in->dims->data[1];
  d->in_w = in->dims->data[2];
  d->channels_packed = in->dims->data[3];
  int oh, ow;
  if (lce_oracle_bmaxpool_out_shape(d, &oh, &ow)) return kTfLiteError;
  TfLiteIntArray* s = LceB200IntArrayCreate(4);
  s->data[0] = d->batch; s->data[1] = oh; s->data[2] = ow; s->data[3] = d->channels_packed;
  return c->ResizeTensor(c, Out(c, n, 0), s);
}
TfLiteStatus PoolEval(TfLiteContext* c, TfLiteNode* n) {
  return lce_oracle_bmaxpool(static_cast<lce_bmaxpool_desc*>(n->user_data), In(c, n, 0)->data.i32,
                             Out(c, n, 0)->data.i32) == 0
             ? kTfLiteOk
             : kTfLiteError;
}
}  // namespace

extern "C" {
TfLiteRegistration* lce_oracle_Register_BCONV_2D() {
  static TfLiteRegistration r = {ConvInit, ConvFree, ConvPrepare, ConvEval};
  return &r;
}
TfLiteRegistration* lce_oracle_Register_QUANTIZE() {
  static TfLiteRegistration r = {nullptr, nullptr, QPrepare, QEval};
  return &r;
}
TfLiteRegistration* lce_oracle_Register_DEQUANTIZE() {
  static TfLiteRegistration r = {nullptr, nullptr, DQPrepare, DQEval};
  return &r;
}
TfLiteRegistration* lce_oracle_Register_BMAXPOOL_2D() {
  static TfLiteRegistration r = {PoolInit, PoolFree, PoolPrepare, PoolEval};
  return &r;
}
}

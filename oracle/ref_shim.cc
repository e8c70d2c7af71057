// oracle/ref_shim.cc -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// Thin extern "C" wrapper that instantiates the reference's OWN header-only
// kernels from where they lie under /root/reference (nothing is copied):
//   bitpack_matrix / unpack_matrix      larq_compute_engine/core/bitpacking/bitpack.h:249,325
//   BConv2DReference                    larq_compute_engine/core/bconv2d/reference.h:35
//   indirect_bgemm::SelectRuntimeKernel larq_compute_engine/core/indirect_bgemm/select_kernel.h:30
//     -> Kernel4x2Portable (x86)        larq_compute_engine/core/indirect_bgemm/kernel_4x2_portable.h:23
//   zero_padding_correction::*          larq_compute_engine/core/bconv2d/zero_padding_correction.h:30-304
//   BMaxPool                            larq_compute_engine/core/bmaxpool.h:24
//   ComputePaddingHeightWidth           tensorflow/lite/kernels/padding.h:62
// The op shell (tflite/kernels/bconv2d.cc) needs flexbuffers + ruy, which are
// not vendored, so the two pieces of it that define results are restated here
// and cited: Prepare's shape inference (bconv2d.cc:169-248) and OneTimeSetup's
// double-precision multiplier/bias fold + clamp bounds (bconv2d.cc:324-392,
// CalculateActivationRange at tensorflow/lite/kernels/kernel_util.h:285-300).
//
// Built by oracle/Makefile into oracle/_ref/liblce_ref.so (git-ignored).
#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstring>
#include <limits>
#include <memory>
#include <thread>
#include <vector>

// Include order matters: utils.h / bmaxpool.h do `using namespace tflite`
// inside compute_engine::core, which reference.h silently relies on.
#include "larq_compute_engine/core/bitpacking/utils.h"
#include "larq_compute_engine/core/bmaxpool.h"
#include "larq_compute_engine/core/bconv2d/reference.h"
#include "larq_compute_engine/core/bconv2d/zero_padding_correction.h"
#include "larq_compute_engine/core/bconv2d/optimized_indirect_bgemm.h"
#include "larq_compute_engine/core/indirect_bgemm/select_kernel.h"
#include "tensorflow/lite/kernels/padding.h"

#include "../include/lce_b200_types.h"

namespace ce = compute_engine::core;
using ce::TBitpacked;
using tflite::RuntimeShape;

namespace {

struct Prepared {
  ce::bconv2d::BConv2DParams p;
  int out_h, out_w;
  int cw_in;       // packed words per input pixel
  int cw_in_pg;    // packed words per group
  int cw_out;      // packed words per output pixel (bitpacked output)
};

// Restates bconv2d.cc:169-248 (groups, padding, output dims).
bool prepare(const lce_bconv2d_desc* d, Prepared* q) {
  auto& p = q->p;
  std::memset(&p, 0, sizeof(p));
  p.filter_width = d->filter_w;
  p.filter_height = d->filter_h;
  p.channels_in = d->channels_in;
  p.channels_out = d->channels_out;
  p.groups = d->groups;
  p.stride_height = d->stride_h;
  p.stride_width = d->stride_w;
  p.dilation_height_factor = d->dilation_h;
  p.dilation_width_factor = d->dilation_w;
  p.padding_type =
      d->padding == LCE_PADDING_SAME ? kTfLitePaddingSame : kTfLitePaddingValid;
  p.pad_value = d->pad_value;
  if (d->groups < 1 || d->channels_in % d->groups || d->channels_out % d->groups)
    return false;
  if (d->groups > 1 && (d->channels_in / d->groups) % 32) return false;
  p.padding_values = tflite::ComputePaddingHeightWidth(
      p.stride_height, p.stride_width, p.dilation_height_factor,
      p.dilation_width_factor, d->in_h, d->in_w, p.filter_height,
      p.filter_width, p.padding_type, &q->out_h, &q->out_w);
  q->cw_in = ce::bitpacking::GetBitpackedSize(d->channels_in);
  q->cw_in_pg = ce::bitpacking::GetBitpackedSize(d->channels_in / d->groups);
  q->cw_out = ce::bitpacking::GetBitpackedSize(d->channels_out);
  return true;
}

// Restates OneTimeSetup, bconv2d.cc:353-389.
struct Folded {
  std::vector<float> mul, bias;
  std::int32_t clamp_min, clamp_max;
};

void fold(const lce_bconv2d_desc* d, const float* post_mul,
          const float* post_bias, Folded* f) {
  const int n = d->channels_out;
  f->mul.assign(n + LCE_EXTRA_BYTES / sizeof(float), 0.f);
  f->bias.assign(n + LCE_EXTRA_BYTES / sizeof(float), 0.f);
  const std::int32_t backtransform_add =
      d->filter_h * d->filter_w * (d->channels_in / d->groups);
  const double output_scale = d->out_type == LCE_OUT_INT8 ? d->out_scale : 1.0;
  const double output_zero_point =
      d->out_type == LCE_OUT_INT8 ? d->out_zero_point : 0.0;
  for (int i = 0; i < n; ++i) {
    const double m = post_mul[i];
    const double b = post_bias[i];
    f->mul[i] = -1 * m / output_scale;
    f->bias[i] = (b + static_cast<double>(backtransform_add) * m) / output_scale +
                 output_zero_point;
  }
  std::int32_t nominal_min, nominal_max;
  switch (d->activation) {  // kernel_util.h:285-300 (int32 instantiation)
    case LCE_ACT_RELU:
      nominal_min = 0;
      nominal_max = std::numeric_limits<std::int32_t>::max();
      break;
    case LCE_ACT_RELU6:
      nominal_min = 0;
      nominal_max = 6;
      break;
    case LCE_ACT_RELU_N1_TO_1:
      nominal_min = -1;
      nominal_max = 1;
      break;
    default:
      nominal_min = std::numeric_limits<std::int32_t>::lowest();
      nominal_max = std::numeric_limits<std::int32_t>::max();
  }
  nominal_min = std::max(nominal_min, -1 * backtransform_add);
  nominal_max = std::min(nominal_max, backtransform_add);
  f->clamp_min = -1 * nominal_max + backtransform_add;
  f->clamp_max = -1 * nominal_min + backtransform_add;
}

template <typename Dst>
void fill_transform(ce::bconv2d::OutputTransform<Dst>& t, const Folded& f,
                    const std::int32_t*) {
  t.clamp_min = f.clamp_min;
  t.clamp_max = f.clamp_max;
  t.multiplier = f.mul.data();
  t.bias = f.bias.data();
}
void fill_transform(ce::bconv2d::OutputTransform<TBitpacked>& t, const Folded&,
                    const std::int32_t* thresholds) {
  t.thresholds = thresholds;
}

// kind 0: kReference (bconv2d.cc:499-516). kind 1: kOptimizedIndirectBGEMM
// (bconv2d.cc:463-496).
template <typename Dst>
int run_typed(const lce_bconv2d_desc* d, const Prepared& q, int kind,
              const TBitpacked* input, const TBitpacked* filter,
              const float* post_mul, const float* post_bias,
              const std::int32_t* thresholds, Dst* output, int batch) {
  Folded f;
  constexpr bool bitpacked = std::is_same<Dst, TBitpacked>::value;
  if (!bitpacked) fold(d, post_mul, post_bias, &f);
  ce::bconv2d::OutputTransform<Dst> t;
  fill_transform(t, f, thresholds);

  const RuntimeShape in_shape({batch, d->in_h, d->in_w, q.cw_in});
  const RuntimeShape filt_shape(
      {d->channels_out, d->filter_h, d->filter_w, q.cw_in_pg});
  const RuntimeShape out_shape(
      {batch, q.out_h, q.out_w, bitpacked ? q.cw_out : d->channels_out});

  const bool zero_pad = d->padding == LCE_PADDING_SAME && d->pad_value == 0;
  if (kind == 0) {
    // Legality as in bconv2d.cc:188-200 (kReference branch).
    if (zero_pad && d->channels_in % 2 != 0) return 2;
    ce::bconv2d::BConv2DReference<std::int32_t, Dst>(
        &q.p, in_shape, input, filt_shape, filter, t, out_shape, output);
    return 0;
  }
  // Indirect BGEMM path. Legality bconv2d.cc:188-200 (optimised branch).
  if (zero_pad &&
      !(std::is_same<Dst, float>::value && d->activation == LCE_ACT_NONE))
    return 2;
  std::vector<float> padding_buffer;
  if (zero_pad) {
    padding_buffer.resize(ce::bconv2d::zero_padding_correction::GetCacheSize(
        d->filter_h, d->filter_w, d->channels_out, d->dilation_h,
        d->dilation_w));
    ce::bconv2d::zero_padding_correction::CacheCorrectionValues(
        filter, d->filter_h, d->filter_w, d->channels_out,
        d->channels_in / d->groups, d->dilation_h, d->dilation_w, post_mul,
        padding_buffer.data());
  }
  auto kernel = ce::indirect_bgemm::SelectRuntimeKernel<Dst>(&q.p, in_shape,
                                                             out_shape, t);
  kernel->PackWeights(filter);
  kernel->FillIndirectionBuffer(&q.p, in_shape, out_shape, input);
  ce::bconv2d::BConv2DOptimizedIndirectBGEMM<std::int32_t, Dst>(
      kernel.get(), &q.p, in_shape, out_shape, output, padding_buffer.data(),
      d->pad_value);
  return 0;
}

int run_any(const lce_bconv2d_desc* d, const Prepared& q, int kind,
            const TBitpacked* input, const TBitpacked* filter,
            const float* post_mul, const float* post_bias,
            const std::int32_t* thresholds, void* output, int batch) {
  switch (d->out_type) {
    case LCE_OUT_FLOAT:
      return run_typed<float>(d, q, kind, input, filter, post_mul, post_bias,
                              thresholds, static_cast<float*>(output), batch);
    case LCE_OUT_INT8:
      return run_typed<std::int8_t>(d, q, kind, input, filter, post_mul,
                                    post_bias, thresholds,
                                    static_cast<std::int8_t*>(output), batch);
    case LCE_OUT_BITPACKED:
      return run_typed<TBitpacked>(d, q, kind, input, filter, post_mul,
                                   post_bias, thresholds,
                                   static_cast<TBitpacked*>(output), batch);
  }
  return 1;
}

}  // namespace

extern "C" {

const char* lce_ref_version() {
  return "larq/compute-engine e6860fcf core headers, g++ "
#ifdef __VERSION__
      __VERSION__
#endif
      ;
}

int lce_ref_bconv2d_out_shape(const lce_bconv2d_desc* d, int* out_h, int* out_w,
                              int* pad_h, int* pad_w) {
  Prepared q;
  if (!prepare(d, &q)) return 1;
  *out_h = q.out_h;
  *out_w = q.out_w;
  *pad_h = q.p.padding_values.height;
  *pad_w = q.p.padding_values.width;
  return 0;
}

// Whole batch in one call on the calling thread (kind: 0 reference, 1 indirect).
int lce_ref_bconv2d(const lce_bconv2d_desc* d, int kind, const int32_t* input,
                    const int32_t* filter, const float* post_mul,
                    const float* post_bias, const int32_t* thresholds,
                    void* output) {
  Prepared q;
  if (!prepare(d, &q)) return 1;
  return run_any(d, q, kind, input, filter, post_mul, post_bias, thresholds,
                 output, d->batch);
}

// The reference's bconv kernels are single-threaded by construction
// (indirect_bgemm/kernel.h:180-183); a batch is run as independent per-image
// calls spread over `threads` host threads.
int lce_ref_bconv2d_mt(const lce_bconv2d_desc* d, int kind, int threads,
                       const int32_t* input, const int32_t* filter,
                       const float* post_mul, const float* post_bias,
                       const int32_t* thresholds, void* output) {
  Prepared q;
  if (!prepare(d, &q)) return 1;
  const size_t in_img = size_t(d->in_h) * d->in_w * q.cw_in;
  const size_t out_elems =
      size_t(q.out_h) * q.out_w *
      (d->out_type == LCE_OUT_BITPACKED ? q.cw_out : d->channels_out);
  const size_t out_bytes =
      out_elems * (d->out_type == LCE_OUT_INT8 ? 1 : 4);
  std::atomic<int> next{0};
  std::atomic<int> rc{0};
  auto work = [&]() {
    for (;;) {
      const int b = next.fetch_add(1);
      if (b >= d->batch) break;
      int r = run_any(d, q, kind, input + b * in_img, filter, post_mul,
                      post_bias, thresholds,
                      static_cast<char*>(output) + b * out_bytes, 1);
      if (r) rc.store(r);
    }
  };
  threads = std::max(1, std::min(threads, d->batch));
  std::vector<std::thread> pool;
  for (int i = 1; i < threads; ++i) pool.emplace_back(work);
  work();
  for (auto& t : pool) t.join();
  return rc.load();
}

// LceQuantize: quantization.cc:76-114 -> bitpack_tensor (utils.h:24-33).
int lce_ref_quantize(int in_type, const void* in, int64_t rows, int64_t cols,
                     int32_t zero_point, int32_t* out) {
  switch (in_type) {
    case LCE_T_FLOAT:
      ce::bitpacking::bitpack_matrix(static_cast<const float*>(in), rows, cols,
                                     out, 0);
      return 0;
    case LCE_T_INT8:
      ce::bitpacking::bitpack_matrix(static_cast<const std::int8_t*>(in), rows,
                                     cols, out, zero_point);
      return 0;
    case LCE_T_BOOL:
      // quantization.cc:88-108: bool viewed as uint8 with zero point 1.
      ce::bitpacking::bitpack_matrix(static_cast<const std::uint8_t*>(in), rows,
                                     cols, out, 1);
      return 0;
  }
  return 1;
}

// LceDequantize: quantization.cc:116-147 -> unpack_matrix (bitpack.h:325-346).
int lce_ref_dequantize(int out_type, const int32_t* in, int64_t rows,
                       int64_t cols, float scale, int32_t zero_point,
                       void* out) {
  switch (out_type) {
    case LCE_T_FLOAT:
      ce::bitpacking::unpack_matrix(in, rows, cols, static_cast<float*>(out));
      return 0;
    case LCE_T_INT8: {
      int offset = tflite::TfLiteRound(1.0f / scale);
      std::int8_t zero_bit = std::min(127, zero_point + offset);
      std::int8_t one_bit = std::max(-128, zero_point - offset);
      ce::bitpacking::unpack_matrix(in, rows, cols,
                                    static_cast<std::int8_t*>(out), zero_bit,
                                    one_bit);
      return 0;
    }
    case LCE_T_BOOL:
      ce::bitpacking::unpack_matrix(in, rows, cols, static_cast<bool*>(out),
                                    true, false);
      return 0;
  }
  return 1;
}

int lce_ref_bmaxpool_out_shape(const lce_bmaxpool_desc* d, int* out_h,
                               int* out_w) {
  tflite::ComputePaddingHeightWidth(
      d->stride_h, d->stride_w, 1, 1, d->in_h, d->in_w, d->filter_h,
      d->filter_w,
      d->padding == LCE_PADDING_SAME ? kTfLitePaddingSame : kTfLitePaddingValid,
      out_h, out_w);
  return 0;
}

// LceBMaxPool2d: bmaxpool.cc:40-88 -> BMaxPool (bmaxpool.h:24-88).
int lce_ref_bmaxpool(const lce_bmaxpool_desc* d, const int32_t* in,
                     int32_t* out) {
  ce::BMaxPoolParams p;
  p.filter_height = d->filter_h;
  p.filter_width = d->filter_w;
  p.stride_height = d->stride_h;
  p.stride_width = d->stride_w;
  p.padding_type =
      d->padding == LCE_PADDING_SAME ? kTfLitePaddingSame : kTfLitePaddingValid;
  int out_h, out_w;
  p.padding = tflite::ComputePaddingHeightWidth(
      p.stride_height, p.stride_width, 1, 1, d->in_h, d->in_w, p.filter_height,
      p.filter_width, p.padding_type, &out_h, &out_w);
  const RuntimeShape in_shape({d->batch, d->in_h, d->in_w, d->channels_packed});
  const RuntimeShape out_shape({d->batch, out_h, out_w, d->channels_packed});
  ce::BMaxPool(p, in_shape, in, out_shape, out);
  return 0;
}

}  // extern "C"

/*
 * lce_b200_types.h -- plain-C descriptors shared by the C-ABI CUDA layer
 * (include/lce_b200.h), the CPU oracle (oracle/lce_oracle.c) and the compiled
 * reference shim (oracle/ref_shim.cc). No torch / TFLite types here.
 *
 * Field meanings follow the reference's BConv2DParams
 * (larq_compute_engine/core/bconv2d/params.h:12-32) and BMaxPoolParams
 * (larq_compute_engine/core/bmaxpool.h:14-21); enum integers follow the TFLite
 * schema the converter writes into the op's flexbuffer
 * (larq_compute_engine/mlir/ir/lce_ops.cc:36-64).
 */
#ifndef LCE_B200_TYPES_H_
#define LCE_B200_TYPES_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* TFLite schema `Padding` (schema.fbs:792) */
enum { LCE_PADDING_SAME = 0, LCE_PADDING_VALID = 1 };
/* TFLite schema `ActivationFunctionType` (schema.fbs:796) */
enum {
  LCE_ACT_NONE = 0,
  LCE_ACT_RELU = 1,
  LCE_ACT_RELU_N1_TO_1 = 2,
  LCE_ACT_RELU6 = 3
};
/* Output element type of LceBconv2d: dispatch of bconv2d.cc:551-564 */
enum { LCE_OUT_FLOAT = 0, LCE_OUT_INT8 = 1, LCE_OUT_BITPACKED = 2 };
/* SAME padding with pad_values == 0 ("zero padding"), the two results the reference has:
 *  REFERENCE  : the reference kernel's integers (LCE/core/bconv2d/reference.h:76-77,100-103: an
 *               out-of-bounds tap adds channels_in_per_group / 2), any output type, needs an
 *               even channels_in (bconv2d.cc:188-200) -- Register_BCONV_2D_REF.
 *  CORRECTION : the optimised kernels' result -- one-padding, OutputTransform, then a FLOAT
 *               correction on the edge outputs (optimized_bgemm.h:153-177,
 *               zero_padding_correction.h:39-299); float output without fused activation only --
 *               Register_BCONV_2D (the reference's default) and ..._OPT_INDIRECT_BGEMM.
 * The two differ by float rounding (up to ~1e5 ULP near cancellation). */
enum { LCE_ZERO_PADDING_REFERENCE = 0, LCE_ZERO_PADDING_CORRECTION = 1 };
/* Input element type of LceQuantize / output of LceDequantize
 * (quantization.cc:76-147) */
enum { LCE_T_FLOAT = 0, LCE_T_INT8 = 1, LCE_T_BOOL = 2 };

/* One LceBconv2d invocation. Activations are NHWC with the channel axis
 * bitpacked into int32 words (bit i of word w = channel 32w+i, bit 1 <=> value
 * < 0; types.h:41-47, bitpack.h:159); filters are OHWI-packed
 * [channels_out, filter_h, filter_w, ceil(channels_in/groups/32)]. */
typedef struct lce_bconv2d_desc {
  int32_t batch, in_h, in_w;
  int32_t channels_in;  /* unpacked, whole tensor (attribute `channels_in`) */
  int32_t filter_h, filter_w;
  int32_t channels_out;
  int32_t groups;
  int32_t stride_h, stride_w;
  int32_t dilation_h, dilation_w;
  int32_t padding;    /* LCE_PADDING_* */
  int32_t pad_value;  /* 0 or 1 (attribute `pad_values`) */
  int32_t activation; /* LCE_ACT_* */
  int32_t out_type;   /* LCE_OUT_* */
  float out_scale;    /* int8 output only (TfLiteTensor::params.scale) */
  int32_t out_zero_point;
} lce_bconv2d_desc;

typedef struct lce_bmaxpool_desc {
  int32_t batch, in_h, in_w;
  int32_t channels_packed; /* int32 words per pixel */
  int32_t filter_h, filter_w;
  int32_t stride_h, stride_w;
  int32_t padding; /* LCE_PADDING_* */
} lce_bmaxpool_desc;

/* Epilogue of a plain BGEMM (config 5 sweep): what OutputTransform<Dst>
 * (output_transform.h:94-168) needs, already folded. */
typedef struct lce_bgemm_epilogue {
  int32_t out_type;  /* LCE_OUT_*; 3 = raw int32 accumulators */
  int32_t clamp_min, clamp_max;
  const float* multiplier; /* [N], folded (mul') */
  const float* bias;       /* [N], folded (bias') */
  const int32_t* thresholds; /* [N] */
} lce_bgemm_epilogue;
#define LCE_OUT_RAW_ACC 3

/* The per-channel float chain ReActNet puts behind a binary convolution: RPReLU
 * (ADD(shift_in) -> PRELU(alpha) -> ADD(shift_out)), then the next layer's RSign
 * (ADD(sign_shift) -> LceQuantize). Each pointer is a device vector with one float per channel;
 * NULL means the op is absent, which is not the same as adding zeros (-0 + 0 = +0). Per element,
 * in TFLite's order and rounding:
 *   t = s + shift_in;  u = t >= 0 ? t : t * alpha;  o = u + shift_out;  bit = (o + sign_shift) < 0 */
typedef struct lce_chain_desc {
  const float* shift_in;
  const float* alpha;
  const float* shift_out;
  const float* sign_shift;
} lce_chain_desc;

/* The gated block tail of Real-to-Binary Net behind a binary convolution: MUL by a per-image,
 * per-channel gate (the sigmoid of a squeeze-excitation branch), PRELU(alpha), the shortcut ADD,
 * then the next block's BatchNorm and sign (MUL(sign_scale) -> ADD(sign_shift) -> LceQuantize).
 * `gate` is a device tensor [batch][channels] and is required; the other pointers are device
 * vectors with one float per channel, NULL when the op is absent (as in lce_chain_desc). Per
 * element of image b, channel c, in TFLite's order and rounding:
 *   t = s * gate[b][c];  u = t >= 0 ? t : t * alpha;  o = act(u + residual);
 *   bit = (o * sign_scale + sign_shift) < 0 */
typedef struct lce_gate_desc {
  const float* gate;
  const float* alpha;
  const float* sign_scale;
  const float* sign_shift;
} lce_gate_desc;

/* XNOR-Net++'s learned output scale behind a binary convolution (Bulat & Tzimiropoulos, BMVC
 * 2019): MUL by a constant Gamma of one float per output position and channel (alpha[C] x beta[OH]
 * x gamma[OW], folded by the converter into one [1, OH, OW, C] tensor), the shortcut ADD, then the
 * next block's BatchNorm and sign (MUL(sign_scale) -> ADD(sign_shift) -> LceQuantize). `scale` is
 * a device tensor [OH * OW][channels] and is required; sign_scale / sign_shift are device vectors
 * with one float per channel, NULL when the op is absent. Per element of position p within its
 * image, channel c, in TFLite's order and rounding:
 *   o = act(s * scale[p][c] + residual);  bit = (o * sign_scale + sign_shift) < 0 */
typedef struct lce_scale_desc {
  const float* scale;
  const float* sign_scale;
  const float* sign_shift;
} lce_scale_desc;

/* One float TRANSPOSE_CONV (TF/lite/kernels/internal/reference/transpose_conv.h): input
 * [batch, in_h, in_w, in_c], filter [out_c, filter_h, filter_w, in_c], output [batch, out_h, out_w,
 * out_c]. Input pixel (iy, ix) and tap (fy, fx) reach output pixel (iy * stride_h - pad_h + fy,
 * ix * stride_w - pad_w + fx); pad_h / pad_w are the floor half of the total padding TFLite computes
 * for a convolution from the output's size back to the input's. */
typedef struct lce_f32_transpose_conv_desc {
  int32_t batch, in_h, in_w, in_c;
  int32_t filter_h, filter_w, out_c;
  int32_t out_h, out_w;
  int32_t stride_h, stride_w;
  int32_t pad_h, pad_w;
  int32_t activation; /* LCE_ACT_* */
} lce_f32_transpose_conv_desc;

#ifdef __cplusplus
}
#endif
#endif /* LCE_B200_TYPES_H_ */

/*
 * lce_b200.h -- the drop-in boundary: a C-ABI CUDA layer (sm_90a) for the one
 * hot path of larq/compute-engine: LceQuantize -> LceBconv2d (-> LceBMaxPool2d,
 * LceDequantize). Plain pointers and sizes only; no torch / TFLite types.
 *
 * Every entry point cites the reference interface it replaces (LCE =
 * /root/reference/larq_compute_engine). The TFLite custom-op shell that sits on
 * top of these calls (TfLiteRegistration {init, free, prepare, invoke}) is
 * declared in include/lce_b200_tflite.h; the binding a reference maintainer
 * would add is shown in INTEGRATION.md.
 *
 * Conventions
 *  - `*_dev` pointers are CUDA device pointers on the current device; `stream`
 *    is a cudaStream_t passed as void* (NULL = default stream). Calls are
 *    asynchronous on that stream unless the name ends in `_host`.
 *  - Return value: 0 = ok (kTfLiteOk), non-zero = error (kTfLiteError); the
 *    message is available from lce_b200_last_error() (thread local), mirroring
 *    context->ReportError in the reference (bconv2d.cc:76-83).
 *  - There is NO CPU fallback: without a CUDA device every compute call fails.
 */
#ifndef LCE_B200_H_
#define LCE_B200_H_

#include <stddef.h>
#include <stdint.h>

#include "lce_b200_types.h"

#ifdef __cplusplus
extern "C" {
#endif

#define LCE_B200_ABI_VERSION 1

int lce_b200_abi_version(void);
const char* lce_b200_last_error(void);
/* Number of visible CUDA devices (0 if none / driver missing). */
int lce_b200_device_count(void);

/* ---- LceQuantize --------------------------------------------------------
 * Replaces QuantizeEval (LCE/tflite/kernels/quantization.cc:76-114) ->
 * bitpack_tensor (LCE/core/bitpacking/utils.h:24-33) -> bitpack_matrix
 * (LCE/core/bitpacking/bitpack.h:249-308). in: [rows, cols] of in_type
 * (LCE_T_*); out: [rows, ceil(cols/32)] int32. */
int lce_b200_quantize(int in_type, const void* in_dev, int64_t rows,
                      int64_t cols, int32_t zero_point, int32_t* out_dev,
                      void* stream);

/* ---- LceDequantize ------------------------------------------------------
 * Replaces DequantizeEval (quantization.cc:116-147) -> unpack_matrix
 * (bitpack.h:325-346). `cols` is the unpacked channel count. */
int lce_b200_dequantize(int out_type, const int32_t* in_dev, int64_t rows,
                        int64_t cols, float scale, int32_t zero_point,
                        void* out_dev, void* stream);

/* ---- LceBMaxPool2d ------------------------------------------------------
 * Replaces bmaxpool::Prepare/Eval (LCE/tflite/kernels/bmaxpool.cc:40-88) ->
 * BMaxPool (LCE/core/bmaxpool.h:24-88). */
int lce_b200_bmaxpool_out_shape(const lce_bmaxpool_desc* d, int* out_h,
                                int* out_w);
int lce_b200_bmaxpool(const lce_bmaxpool_desc* d, const int32_t* in_dev,
                      int32_t* out_dev, void* stream);

/* ---- LceBconv2d ---------------------------------------------------------
 * A plan object carries what bconv2d::OpData carries (bconv2d.cc:44-74): the
 * parameters, the folded output transform, and device copies of the constant
 * inputs, re-laid-out once for the kernel ("LHS cached", optimized_bgemm.h:135).
 *
 * out_shape  : shape inference of Prepare (bconv2d.cc:169-248).
 * create     : Init + Prepare + OneTimeSetup (bconv2d.cc:85-131,138-300,324-392).
 *              `filter` is OHWI-packed [channels_out, filter_h, filter_w,
 *              ceil(channels_in/groups/32)]; `post_mul`/`post_bias` are the op's
 *              inputs 2/3 (float/int8 output), `thresholds` input 4 (bitpacked
 *              output); absent optional inputs are NULL (bconv2d.cc:145-152).
 *              These four may be host or device pointers. desc->batch/in_h/in_w
 *              give the initial input shape. Refuses what the reference refuses
 *              (bconv2d.cc:113-116,169-200), with the reference-kernel rule for
 *              zero padding (even channels_in).
 * set_input_shape : what a second Prepare after ResizeInputTensor does
 *              (bconv2d.cc:295-297).
 * run        : Eval (bconv2d.cc:551-564) on bitpacked NHWC input
 *              [batch, in_h, in_w, ceil(channels_in/32)] -> output NHWC float /
 *              int8 [.., channels_out] or int32 [.., ceil(channels_out/32)].
 * run_f32    : the same with LceQuantize fused into the prologue: input is the
 *              float NHWC tensor [batch, in_h, in_w, channels_in].
 * run_host   : run with HOST buffers (H2D, kernel, D2H, synchronised) -- the
 *              call a stock TFLite interpreter with a host arena makes. */
typedef struct lce_b200_bconv2d lce_b200_bconv2d;

int lce_b200_bconv2d_out_shape(const lce_bconv2d_desc* d, int* out_h,
                               int* out_w, int* pad_h, int* pad_w);
int lce_b200_bconv2d_create(const lce_bconv2d_desc* d, const int32_t* filter,
                            const float* post_mul, const float* post_bias,
                            const int32_t* thresholds, lce_b200_bconv2d** plan);
int lce_b200_bconv2d_set_input_shape(lce_b200_bconv2d* plan, int batch,
                                     int in_h, int in_w);
/* Which of the reference's two zero-padding results a plan reproduces (LCE_ZERO_PADDING_*,
 * lce_b200_types.h). create() picks REFERENCE when channels_in is even (what
 * Register_BCONV_2D_REF computes) and CORRECTION otherwise; the op shell sets it from the
 * registration it was built through. No effect unless padding == SAME and pad_value == 0. */
int lce_b200_bconv2d_set_zero_padding_mode(lce_b200_bconv2d* plan, int mode);
int lce_b200_bconv2d_get_desc(const lce_b200_bconv2d* plan,
                              lce_bconv2d_desc* d, int* out_h, int* out_w);
int lce_b200_bconv2d_run(lce_b200_bconv2d* plan, const int32_t* in_dev,
                         void* out_dev, void* stream);
int lce_b200_bconv2d_run_f32(lce_b200_bconv2d* plan, const float* in_dev,
                             void* out_dev, void* stream);
/* Fused residual-block tail (graph-level fusion of the converter pattern
 *   LceBconv2d(float out) -> ADD(shortcut) [-> LceQuantize of the sum]):
 *   out = act_add(OutputTransform(acc) + residual);  packed_out = bitpack(out) (optional).
 * Bit-identical to running the three ops one after the other. Float output plans only;
 * packed_out additionally needs groups == 1, or channels_out / groups a multiple of 32 on the b1
 * mma.sync kernel (LCE_B200_BCONV_IMMA and _B1 not 0 when the plan was created); the same holds
 * for run_fused_chain. residual / packed_out may be NULL. */
int lce_b200_bconv2d_run_fused(lce_b200_bconv2d* plan, const int32_t* in_dev,
                               const float* residual_dev, int add_activation,
                               float* out_dev, int32_t* packed_out_dev, void* stream);
/* run_fused followed by ReActNet's per-channel chain (lce_chain_desc, lce_b200_types.h) on every
 * output: out = o, packed_out = bitpack(o + sign_shift) (optional). Each chain vector holds
 * channels_out floats on the device; chain may be NULL (then this is run_fused). The mma.sync
 * kernel applies the chain in its epilogue; plans that run on another kernel, or that finish
 * zero padding with the float correction pass, run run_fused and then lce_b200_f32_chain_sign in
 * place. Bit-identical to the op sequence either way. */
int lce_b200_bconv2d_run_fused_chain(lce_b200_bconv2d* plan, const int32_t* in_dev,
                                     const float* residual_dev, int add_activation,
                                     const lce_chain_desc* chain, float* out_dev,
                                     int32_t* packed_out_dev, void* stream);
/* Two consecutive fused residual blocks in one kernel:
 *   x1 = act1(OutputTransform1(conv1(x0 packed)) + x0);  out = act2(OutputTransform2(conv2(bitpack(x1))) + x1);
 *   packed_out = bitpack(out) (optional, may be NULL).
 * Bit-identical to two run_fused calls, but x1 and its signs stay on chip. Both plans must be
 * ungrouped 3x3 / stride 1 / dilation 1 SAME layers with pad_values = 1, float output,
 * channels_in == channels_out == 32, 64 or 128, on the b1 mma.sync kernel (32-channel plans get
 * the pair kernel's fragments at creation and otherwise run on the wgmma kernel), and plan2 must
 * take plan1's output shape; anything else is refused with a message. out must not overlap
 * residual. */
int lce_b200_bconv2d_run_fused_pair(lce_b200_bconv2d* plan1, lce_b200_bconv2d* plan2,
                                    const int32_t* in_dev, const float* residual_dev,
                                    int act1, int act2, float* out_dev,
                                    int32_t* packed_out_dev, void* stream);
/* The same chain without a convolution, in one pass over a float [rows, channels] tensor
 * (ReActNet's chains after a CONCATENATION, a lone RSign; the PRELU builtin): element i takes
 * channel i % channels of every present vector. out = o (may be NULL when nothing else reads it;
 * may be x_dev), packed_out[row][ceil(channels/32)] = bitpack(o + sign_shift) (may be NULL). With
 * only `alpha` set this is PRELU (TF/lite/kernels/internal/reference/prelu.h),
 * out = x >= 0 ? x : x * alpha, and `channels` may be any alpha size dividing the element count. */
int lce_b200_f32_chain_sign(const float* x_dev, const lce_chain_desc* chain, int64_t rows,
                            int channels, float* out_dev, int32_t* packed_out_dev, void* stream);
/* Real-to-Binary Net's gated block tail (lce_gate_desc, lce_b200_types.h) behind the convolution:
 *   out = act(prelu(OutputTransform(acc) * gate[b][c], alpha) + residual),
 *   packed_out = bitpack(out * sign_scale + sign_shift) (optional),
 * with b the output pixel's image. residual may be NULL (then act applies to the PRELU result);
 * add_activation is an LCE_ACT_* code. gate_desc and gate_desc->gate are required. Float-output
 * plans only; packed_out needs groups == 1; out must not overlap residual or the gate. The mma.sync
 * kernel applies the tail in its epilogue; plans on another kernel, or that finish zero padding
 * with the float correction pass, run run_fused without a residual and then
 * lce_b200_f32_gate_sign in place. Bit-identical to the op sequence either way. */
int lce_b200_bconv2d_run_fused_gate(lce_b200_bconv2d* plan, const int32_t* in_dev,
                                    const lce_gate_desc* gate_desc, const float* residual_dev,
                                    int add_activation, float* out_dev, int32_t* packed_out_dev,
                                    void* stream);
/* The same tail without a convolution, in one pass over a float [batch, pixels, channels] tensor:
 * element (b, p, c) takes gate[b][c] and channel c of the other present vectors. residual (same
 * shape as x, may be NULL), out (may be NULL when only the signs are read; may be x_dev) and
 * packed_out[b][p][ceil(channels/32)] (may be NULL) as in run_fused_gate. With only `gate` set
 * this is the MUL builtin of a [B,H,W,C] tensor by a [B,1,1,C] one, out = act(x * gate). */
int lce_b200_f32_gate_sign(const float* x_dev, const lce_gate_desc* gate_desc,
                           const float* residual_dev, int activation, int64_t batch,
                           int64_t pixels, int channels, float* out_dev, int32_t* packed_out_dev,
                           void* stream);
/* XNOR-Net++'s scaled block tail (lce_scale_desc, lce_b200_types.h) behind the convolution:
 *   out = act(fl(fl(OutputTransform(acc) * scale[p][c]) + residual)),
 *   packed_out = bitpack(fl(fl(out * sign_scale) + sign_shift)) (optional),
 * with p = m mod (OH * OW) the output pixel's position within its image. residual may be NULL (then
 * act applies to the product); add_activation is an LCE_ACT_* code. scale_desc and
 * scale_desc->scale are required. Float-output plans only; packed_out needs groups == 1; out must
 * not overlap residual or the scale. The mma.sync kernel applies the tail in its epilogue; plans on
 * another kernel, or that finish zero padding with the float correction pass, run the convolution
 * and then lce_b200_f32_scale_sign in place. Bit-identical to the op sequence either way. */
int lce_b200_bconv2d_run_fused_scale(lce_b200_bconv2d* plan, const int32_t* in_dev,
                                     const lce_scale_desc* scale_desc, const float* residual_dev,
                                     int add_activation, float* out_dev, int32_t* packed_out_dev,
                                     void* stream);
/* The same tail without a convolution, in one pass over a float [batch, pixels, channels] tensor:
 * element (b, p, c) takes scale[p][c] and channel c of the other present vectors. residual, out and
 * packed_out as in lce_b200_f32_gate_sign. With only `scale` set this is the MUL builtin of a
 * [B,H,W,C] tensor by a [1,H,W,C] one (any b whose shape, leading 1s dropped, is x's trailing
 * dimensions), out = act(x * scale). */
int lce_b200_f32_scale_sign(const float* x_dev, const lce_scale_desc* scale_desc,
                            const float* residual_dev, int activation, int64_t batch,
                            int64_t pixels, int channels, float* out_dev, int32_t* packed_out_dev,
                            void* stream);
/* The sigmoid that ends Real-to-Binary Net's gate, TFLite's LOGISTIC
 * (TF/lite/kernels/internal/reference/logistic.h): out = 1 above 16.619047164916992188, exp(x)
 * below -9, else 1 / (1 + exp(-x)). CUDA's expf is not libm's: within 4 ulp of the formula, not
 * bit-identical to a CPU run. */
int lce_b200_f32_logistic(const float* in_dev, float* out_dev, int64_t n, void* stream);
/* BinaryDenseNet's dense layer writes its new channels into the block's map in place:
 * run, but output pixel m's channels_out floats go to out_dev + m * out_pixel_stride, and nothing
 * else is written. Float-output plans on the mma.sync kernel only (created with
 * LCE_B200_BCONV_IMMA not 0 and channels_out a multiple of 64); REFERENCE zero padding stays in
 * the kernel, CORRECTION plans finish with the float correction pass on the same strided rows.
 * Refuses, with a message, other plans, a stride below channels_out or not a multiple of 4, an
 * out_dev that is not 16-byte aligned, and an output span that overlaps the input. Bit-identical
 * to run followed by a copy of each pixel's row. */
int lce_b200_bconv2d_run_slice(lce_b200_bconv2d* plan, const int32_t* in_dev, float* out_dev,
                               int64_t out_pixel_stride, void* stream);
/* MeliusNet's improvement layer adds its new channels to a channel slice of the block's map in
 * place: for every output pixel m and c < channels_out,
 *   io_dev[m * io_pixel_stride + c] = io_dev[m * io_pixel_stride + c] + y[m][c]
 * (one __fadd_rn, TFLite's ADD), y being exactly what run computes; nothing else in io is written.
 * Takes the plans run_slice takes, with its stride, alignment and input-overlap refusals. One-
 * padding and REFERENCE zero-padding plans run it in one mma.sync launch. A CORRECTION plan (zero
 * padding with the float correction) writes y to scratch_dev ([pixels, channels_out] floats,
 * 16-byte aligned, overlapping neither io nor the input) and the correction pass adds it to io;
 * refuses such a plan without a scratch. Other plans ignore scratch_dev, which may be NULL. */
int lce_b200_bconv2d_run_slice_add(lce_b200_bconv2d* plan, const int32_t* in_dev, float* io_dev,
                                   int64_t io_pixel_stride, float* scratch_dev, void* stream);
/* A binary learned upsampler, LceDequantize -> TRANSPOSE_CONV (+-1 weights, kernel = stride s_h x s_w)
 * [-> ADD(skip)] [-> LceQuantize], as the 1x1 plan's GEMM to s_h * s_w * C columns in (i, j, c) order
 * followed by a pixel shuffle in the store: GEMM row (b, y, x), column (i * s_w + j) * C + c goes to
 * out[b, y * s_h + i, x * s_w + j, c], out [batch, in_h * s_h, in_w * s_w, C]. Per element:
 *   t = act(D + bias[c]);  out = add_act(t + skip) (skip NULL: out = t);  packed_out = bitpack(out),
 * D the +-1 dot product as an exact integer, one rounding for the bias (bias NULL: t = act(D)) and one
 * for the skip, which is TFLite's TRANSPOSE_CONV and ADD bit for bit. D = channels_in - 2 popcount(a ^ w)
 * comes from the accumulators: the plan's post_mul / post_bias are not applied. The plan must be an
 * ungrouped 1x1 / stride 1 plan with float output, no fused activation and no zero padding,
 * channels_out = s_h * s_w * C with C % 64 == 0, on the b1 mma.sync kernel
 * (lce_b200_internal_shuffle_takes); bias holds C device floats, skip and out are [batch, in_h * s_h,
 * in_w * s_w, C] and packed_out (may be NULL) [.., C / 32]. out must not overlap skip or the input. */
int lce_b200_bconv2d_run_fused_shuffle(lce_b200_bconv2d* plan, const int32_t* in_dev, int s_h, int s_w,
                                       const float* bias_dev, int activation, const float* skip_dev,
                                       int add_activation, float* out_dev, int32_t* packed_out_dev,
                                       void* stream);
/* A binary dense layer, LceDequantize -> FULLY_CONNECTED (weights +-alpha_c, [bias]) [-> MUL(scale) ->
 * ADD(shift)] [-> LceQuantize], as the plan's 1x1 GEMM of batch rows (in_h = in_w = 1) on the instance of
 * the b1 mma.sync kernel run_fused_shuffle uses, with s_h = s_w = 1. Per row m, column c < N =
 * channels_out:
 *   y = activation(fl(fl(alpha[c] * D) + bias[c]));
 *   y = bn_activation(fl(fl(y * scale[c]) + shift[c]));   out[m][c] = y;   packed_out = bitpack(y),
 * D the +-1 dot product channels_in - 2 popcount(a ^ w) as an exact integer, each step rounded on its
 * own as TFLite's FULLY_CONNECTED, MUL and ADD round the result (a NULL vector drops its step;
 * bn_activation applies either way). With every alpha a power of two that is TFLite's FULLY_CONNECTED
 * bit for bit; otherwise TFLite's loop rounds after each of its K terms and the results can differ by
 * about K * 2^-24 * K * alpha. The plan must be an ungrouped 1x1 / stride 1 plan of in_h = in_w = 1 with
 * float output, no fused activation and no zero padding, N % 64 == 0, on the b1 mma.sync kernel
 * (lce_b200_internal_fc_takes); the post_mul / post_bias are not applied. alpha, bias, scale and shift
 * hold N device floats each (8-byte aligned) or are NULL; out is [batch, N] (16-byte aligned) and
 * packed_out (may be NULL) [batch, N / 32]; out, packed_out and the input must not overlap. */
int lce_b200_bconv2d_run_fused_fc(lce_b200_bconv2d* plan, const int32_t* in_dev, const float* alpha_dev,
                                  const float* bias_dev, int activation, const float* scale_dev,
                                  const float* shift_dev, int bn_activation, float* out_dev,
                                  int32_t* packed_out_dev, void* stream);
/* lce_b200_bconv2d_run_fused_fc's binary dense layer followed by REDUCE_MAX over each image's rows, the
 * plan's batch rows being images of `points` consecutive rows: max_out[b][c] is TFLite's reference
 * reduction (cur = -FLT_MAX, then cur = y > cur ? y : cur in row order) of column c of rows b * points ..
 * b * points + points - 1, each y computed as run_fused_fc computes it, and packed_out[b] = bitpack of
 * max_out[b]. A NaN is never chosen, of equal values (-0.0, +0.0) the first row's wins, and an image
 * whose values are all NaN or -inf gives -FLT_MAX. The columns are never stored: each CTA merges its
 * rows into keys_dev, B * N 64-bit words (16-byte aligned) of workspace this call initialises, with
 * atomicMax, so the result does not depend on the CTAs' order. max_out [B, N] and packed_out [B, N / 32]
 * may each be NULL but not both; keys, max_out, packed_out and the input must not overlap. The plan is
 * run_fused_fc's, with batch a multiple of points. */
int lce_b200_bconv2d_run_fused_fc_max(lce_b200_bconv2d* plan, const int32_t* in_dev, const float* alpha_dev,
                                      const float* bias_dev, int activation, const float* scale_dev,
                                      const float* shift_dev, int bn_activation, int points, void* keys_dev,
                                      float* max_out_dev, int32_t* packed_out_dev, void* stream);
/* The signs of a dense layer's BatchNorm in one pass over a strided float [rows, channels] map
 * (row r starts at x_dev + r * x_pixel_stride):
 *   packed_out[r][ceil(channels/32)] = bitpack(x * scale[c] + shift[c]),
 * rounded after the multiply and again after the add, as TFLite's MUL then ADD. scale or shift
 * may be NULL (that op is absent). copy_out (may be NULL) receives x bit for bit, row r at
 * copy_out + r * copy_pixel_stride. */
int lce_b200_f32_affine_sign(const float* x_dev, int64_t x_pixel_stride, int64_t rows,
                             int channels, const float* scale, const float* shift,
                             int32_t* packed_out_dev, float* copy_out_dev,
                             int64_t copy_pixel_stride, void* stream);
/* BinaryAlexNet's and XNOR-Net's pooled BatchNorm and sign, MAX_POOL_2D -> MUL(scale) -> ADD(shift)
 * -> LceQuantize, in one pass over a float NHWC map [batch, in_h, in_w, channels]:
 *   packed_out[b][oy][ox][ceil(channels/32)] bit c =
 *     bitpack(act(max over the in-bounds window) * scale[c] + shift[c]),
 * the max taken as the MAX_POOL_2D builtin takes it (from -FLT_MAX with fmaxf, then the pool's
 * fused activation `activation`, an LCE_ACT_* code), the affine step rounded after the multiply and
 * again after the add, as TFLite's MUL then ADD. Tail bits are 0. padding is LCE_PADDING_SAME or
 * LCE_PADDING_VALID with the pool's output size; scale or shift may be NULL (that op is absent).
 * Bit-identical to the four ops one after the other. */
int lce_b200_f32_maxpool_affine_sign(const float* x_dev, int batch, int in_h, int in_w, int channels,
                                     int filter_h, int filter_w, int stride_h, int stride_w,
                                     int padding, int activation, const float* scale,
                                     const float* shift, int32_t* packed_out_dev, void* stream);
/* MAXIMUM / MINIMUM (TF/lite/kernels/internal/reference/maximum_minimum.h: a > b ? a : b and
 * a < b ? a : b), DIV (reference/div.h: one IEEE division, then the fused activation) and ROUND
 * (reference/round.h: halves to even), on device pointers: out[i] = a[i] (op) b[i % b_len], with b_len == n (same
 * shape), the last dimension, or 1. Bit-identical to numpy float32. */
int lce_b200_f32_maximum(const float* a_dev, const float* b_dev, float* out_dev, int64_t n,
                         int64_t b_len, void* stream);
int lce_b200_f32_minimum(const float* a_dev, const float* b_dev, float* out_dev, int64_t n,
                         int64_t b_len, void* stream);
int lce_b200_f32_div(const float* a_dev, const float* b_dev, float* out_dev, int64_t n, int64_t b_len,
                     int activation, void* stream);
int lce_b200_f32_round(const float* in_dev, float* out_dev, int64_t n, void* stream);
/* DoReFaNet's 2-bit activation quantiser, [MAX_POOL_2D ->] MAXIMUM(0) -> MINIMUM(1) -> MUL(3) ->
 * ROUND [-> DIV(3)], in one pass over a float NHWC map [batch, in_h, in_w, channels], written as the
 * bit planes of the level q = rint(min(max(v, 0), 1) * 3) in {0, 1, 2, 3}:
 *   planes_out[b][oy][ox][3 * channels/32] = [bit 0 of q | bit 1 of q | bit 1 of q],
 * each part channels/32 words packed as LceQuantize packs signs (bit c % 32 of word c / 32). A binary
 * convolution with channels_in = 3 * channels, one-padding and each tap's filter words repeated
 * three times then accumulates D = sum s * (3 - 2 q) over real taps (and sum 3 s over padded ones),
 * so sum s * q / 3 = (3 W - D) / 6 with W the sum of a filter's signs. v is x, or with filter_h and
 * filter_w not 0 the max over the in-bounds pool window taken as the MAX_POOL_2D builtin takes it
 * (from -FLT_MAX with fmaxf, then `activation`); with both 0 the pool arguments are ignored and
 * the output has the input's size. q uses the float operations of the MAXIMUM, MINIMUM, MUL and
 * ROUND builtins, so the levels are theirs bit for bit. channels must be a multiple of 32. */
int lce_b200_f32_quant2_planes(const float* x_dev, int batch, int in_h, int in_w, int channels,
                               int filter_h, int filter_w, int stride_h, int stride_w, int padding,
                               int activation, int32_t* planes_out_dev, void* stream);
/* ---- ABC-Net's multiple binary bases (Lin et al., NeurIPS 2017) ---------
 * One layer y = sum over n < N, m < M of t_nm, where t_nm is an LceBconv2d (float output) of input
 * plane A_n with base filter B_m, followed by the BatchNorm, an optional shortcut and the next
 * layer's shifted signs:
 *   y = (...((t_00 + t_01) + t_02) ... + t_{N-1,M-1})   (left to right, n outer, m inner)
 *   o = bn_act(fl(fl(y * bn_scale[c]) + bn_shift[c]));  out = residual ? add_act(fl(o + residual)) : o
 *   next_planes[k] = bitpack(fl(out + next_shifts[k]) < 0)
 * Each t_nm is exactly what lce_b200_bconv2d_run computes for term (n, m)'s own plan, and the sums and
 * the tail round as TFLite's ADD and MUL do, so the result is bit-identical to the M * N + N + 3 ops.
 * bases_create takes the M * N terms in that order (index n * M + m): their descriptors (all equal),
 * filters (term (n, m)'s filter must equal term (0, m)'s) and post_mul / post_bias (host or device).
 * It refuses, with a message: terms that are not float output without a fused activation; grouped
 * terms; channels_in % 32 != 0 or channels_out % 64 != 0; zero padding (SAME with pad_values 0,
 * whose optimised result needs a per-term float correction: run such terms unfused); more than 8
 * bases or planes; M bases whose b1 fragments for one 64-channel tile (M * ceil(k*k*channels_in/256)
 * * 2 KB) leave no room for two 4 KB input slices in one CTA's 227 KB of shared memory; and
 * LCE_B200_BCONV_IMMA or _B1 set to 0.
 * bases_run: planes_dev[N] are the packed inputs [batch, in_h, in_w, channels_in / 32]; bn_scale /
 * bn_shift are required device vectors [channels_out]; residual (may be NULL) and out (may be NULL:
 * not stored) are float [batch, out_h, out_w, channels_out]; next_shifts[n_next] (host floats) and
 * next_planes_dev[n_next] ([batch, out_h, out_w, channels_out / 32], 8-byte aligned) with n_next in
 * 0..8. Activations are LCE_ACT_* codes. The outputs must not overlap the input planes or the
 * residual. The M bases' fragments stay in shared memory for the whole CTA. */
typedef struct lce_b200_bconv2d_bases lce_b200_bconv2d_bases;
int lce_b200_bconv2d_bases_create(int m_bases, int n_planes, const lce_bconv2d_desc* terms,
                                  const int32_t* const* filters, const float* const* post_mul,
                                  const float* const* post_bias, lce_b200_bconv2d_bases** plan);
int lce_b200_bconv2d_bases_set_input_shape(lce_b200_bconv2d_bases* plan, int batch, int in_h,
                                           int in_w);
int lce_b200_bconv2d_bases_get_desc(const lce_b200_bconv2d_bases* plan, lce_bconv2d_desc* d,
                                    int* out_h, int* out_w);
int lce_b200_bconv2d_bases_run(lce_b200_bconv2d_bases* plan, const int32_t* const* planes_dev,
                               const float* bn_scale_dev, const float* bn_shift_dev,
                               int bn_activation, const float* residual_dev, int add_activation,
                               float* out_dev, int n_next, const float* next_shifts,
                               int32_t* const* next_planes_dev, void* stream);
void lce_b200_bconv2d_bases_destroy(lce_b200_bconv2d_bases* plan);
/* ABC-Net's shifted signs of a float map without a fused producer, N x (ADD(x, shifts[k]) ->
 * LceQuantize), in one pass over x [pixels, channels] (channels % 32 == 0):
 *   planes[k][pixel][channels / 32] = bitpack(fl(x + shifts[k]) < 0),  1 <= n_planes <= 8,
 * shifts on the host, planes device pointers. Bit-identical to the 2 N ops. */
int lce_b200_f32_shift_sign_planes(const float* x_dev, int64_t pixels, int channels, int n_planes,
                                   const float* shifts, int32_t* const* planes_dev, void* stream);
/* TFLite's RESIZE_NEAREST_NEIGHBOR and RESIZE_BILINEAR (TF/lite/kernels/internal/reference/
 * resize_nearest_neighbor.h, resize_bilinear.h) of a float NHWC map [batch, in_h, in_w, channels] to
 * [batch, out_h, out_w, channels]. Per axis, scale = in / (float)out, or with align_corners and
 * out > 1 (in - 1) / (float)(out - 1), computed in float on the host.
 * Nearest: source = min(align_corners ? roundf((o + off) * scale) : floorf((o + off) * scale), in - 1)
 * with off = half_pixel_centers ? 0.5 : 0, and with half_pixel_centers clamped below at 0 too.
 * Bilinear: v = half_pixel_centers ? (o + 0.5) * scale - 0.5 : o * scale, lo = max(floor(v), 0),
 * hi = min(ceil(v), in - 1) per axis, and out = x[lo_y,lo_x]*(1-dy)*(1-dx) + x[hi_y,lo_x]*dy*(1-dx)
 * + x[lo_y,hi_x]*(1-dy)*dx + x[hi_y,hi_x]*dy*dx with dy = v_y - lo_y, dx = v_x - lo_x, left to
 * right with every product and sum rounded; refuses align_corners with half_pixel_centers, as
 * TFLite's Prepare does. Every float step is one IEEE operation, so both are the reference kernels'
 * results bit for bit. */
int lce_b200_f32_resize_nearest(const float* in_dev, int batch, int in_h, int in_w, int channels, int out_h,
                                int out_w, int align_corners, int half_pixel_centers, float* out_dev,
                                void* stream);
int lce_b200_f32_resize_bilinear(const float* in_dev, int batch, int in_h, int in_w, int channels, int out_h,
                                 int out_w, int align_corners, int half_pixel_centers, float* out_dev,
                                 void* stream);
/* A decoder merge, RESIZE_NEAREST_NEIGHBOR(u) -> ADD(skip) [-> LceQuantize], in one pass that reads u
 * at each output pixel's nearest source pixel (u [batch, in_h, in_w, channels]; skip, out
 * [batch, out_h, out_w, channels]):
 *   out = act(fl(u[source] + skip)),  packed_out[pixel][ceil(channels/32)] = bitpack(out < 0),
 * the source as lce_b200_f32_resize_nearest finds it, act an LCE_ACT_* code, tail bits 0. out or
 * packed_out may be NULL (not written). Bit-identical to the three ops one after the other. */
int lce_b200_f32_upsample_add_sign(const float* u_dev, int batch, int in_h, int in_w, int channels, int out_h,
                                   int out_w, int align_corners, int half_pixel_centers, const float* skip_dev,
                                   int activation, float* out_dev, int32_t* packed_out_dev, void* stream);
/* TFLite's float ARG_MAX (TF/lite/kernels/internal/reference/arg_min_max.h with std::greater) of a float
 * tensor viewed as [outer, n, inner], reduced over n (n >= 1): out[o][i] = the reference's sequential
 * result, v = x[o][0][i], idx = 0, and for k = 1 .. n-1 take x[o][k][i] only when x[o][k][i] > v. Ties go
 * to the lowest index (-0.0 equals +0.0), a NaN at index 0 gives 0, a NaN elsewhere is never chosen.
 * out_dev is int64 [outer, inner] when out_int64 is set, else int32; every element is written. */
int lce_b200_f32_argmax(const float* in_dev, int64_t outer, int n, int64_t inner, int out_int64, void* out_dev,
                        void* stream);
/* TFLite's float REDUCE_MAX (TF/lite/kernels/internal/reference/reduce.h, from memory) of a float tensor
 * viewed as [outer, n, inner], reduced over n (n >= 0): out[o][i] = the sequential result of cur =
 * -FLT_MAX, then cur = x > cur ? x : cur for x = x[o][0][i] .. x[o][n-1][i]. A NaN is never chosen, of
 * equal values (-0.0, +0.0) the first wins, and an all-NaN, all--inf or empty slice gives -FLT_MAX.
 * Offsets are 64-bit. */
int lce_b200_f32_reduce_max(const float* in_dev, int64_t outer, int64_t n, int64_t inner, float* out_dev,
                            void* stream);
/* The largest in_w * channels lce_b200_f32_resize_bilinear_argmax takes: it stages two source rows of
 * that many floats in shared memory. */
int lce_b200_resize_bilinear_argmax_max_row_floats(void);
/* lce_b200_f32_resize_bilinear followed by lce_b200_f32_argmax over the channel axis, in one pass that
 * never writes the resized map: out [batch, out_h, out_w] (int64 when out_int64 is set, else int32)
 * is the index ARG_MAX picks from each output pixel's channels, each value computed as
 * lce_b200_f32_resize_bilinear computes it, so the labels equal the two ops' bit for bit. Refuses
 * in_w * channels above lce_b200_resize_bilinear_argmax_max_row_floats(). */
int lce_b200_f32_resize_bilinear_argmax(const float* in_dev, int batch, int in_h, int in_w, int channels,
                                        int out_h, int out_w, int align_corners, int half_pixel_centers,
                                        int out_int64, void* out_dev, void* stream);
/* TFLite's float DEPTH_TO_SPACE (TF/lite/kernels/internal/reference/depth_to_space.h): in [batch, in_h,
 * in_w, channels] to out [batch, in_h * block_size, in_w * block_size, channels / block_size^2] with
 * out[b, y*r + i, x*r + j, c] = in[b, y, x, (i*r + j) * C' + c] (r = block_size, C' = channels / r^2);
 * the values are moved, not computed. Refuses block_size <= 0 and channels % r^2 != 0. */
int lce_b200_f32_depth_to_space(const float* in_dev, int batch, int in_h, int in_w, int channels, int block_size,
                                float* out_dev, void* stream);
/* TFLite's float TRANSPOSE_CONV (TF/lite/kernels/internal/reference/transpose_conv.h) as a gather
 * (lce_f32_transpose_conv_desc, lce_b200_types.h): each output is one fmaf chain from 0 over its taps in
 * the reference's order, then the bias (may be NULL) added with one rounding, then the activation; no
 * atomics, so the result is the same every run. */
int lce_b200_f32_transpose_conv2d(const lce_f32_transpose_conv_desc* d, const float* in_dev,
                                  const float* filter_dev, const float* bias_dev, float* out_dev,
                                  void* stream);
/* The largest out_c lce_b200_f32_subpixel_conv takes: every CTA computes all the conv's channels. */
int lce_b200_subpixel_conv_max_out_channels(void);
/* A super-resolution network's sub-pixel tail in one pass: lce_b200_f32_conv2d(d) (stride 1, dilation 1,
 * SAME; out_c = C' * block_size^2 <= lce_b200_subpixel_conv_max_out_channels(); K = filter_h * filter_w *
 * in_c <= 4096), then lce_b200_f32_depth_to_space(block_size), then, when img_dev is set, an ADD (with
 * add_activation) of lce_b200_f32_resize_bilinear(img [batch, img_h, img_w, C'] to (in_h * block_size,
 * in_w * block_size), align_corners, half_pixel_centers). out [batch, in_h * r, in_w * r, C'] equals the
 * ops run one by one bit for bit where lce_b200_f32_conv2d runs the convolution on its implicit-GEMM
 * kernels; the conv output, the shuffled map and the resized image are never written. */
struct lce_f32_conv_desc; /* lce_b200_builtins.h */
int lce_b200_f32_subpixel_conv(const struct lce_f32_conv_desc* d, const float* in_dev, const float* filter_dev,
                               const float* bias_dev, int block_size, const float* img_dev, int img_h, int img_w,
                               int align_corners, int half_pixel_centers, int add_activation, float* out_dev,
                               void* stream);
/* TFLite_Detection_PostProcess (TF/lite/kernels/detection_postprocess.cc) with its float32 inputs,
 * applied to every image of a batch as TFLite applies it to its single image. */
typedef struct {
  int max_detections, max_classes_per_detection, detections_per_class, num_classes, use_regular_nms;
  float nms_score_threshold, nms_iou_threshold, y_scale, x_scale, h_scale, w_scale;
} lce_b200_detection_options;
/* The largest anchor count one image's (or one class's) NMS holds in shared memory. */
int lce_b200_detection_max_anchors(void);
/* Device workspace bytes lce_b200_f32_detection_postprocess needs (0 for invalid arguments). */
size_t lce_b200_detection_workspace_bytes(int batch, int num_anchors, const lce_b200_detection_options* opts);
/* boxes [batch, num_anchors, box_dim >= 4] (y, x, h, w encodings; the first 4 of each row are read),
 * scores [batch, num_anchors, score_dim] (class c at c + score_dim - num_classes), anchors
 * [num_anchors, 4] (y, x, h, w), all device float32. Outputs, D = max_detections *
 * max_classes_per_detection: det_boxes [batch, D, 4] (ymin, xmin, ymax, xmax; 16-byte aligned),
 * det_classes and det_scores [batch, D], num_detections [batch]; every element is written, the slots
 * TFLite leaves alone as 0. Decode: ycenter = y / y_scale * ha + ya, half_h = 0.5f * exp(h / h_scale) * ha
 * and so on, each step rounded in float, exp in double rounded once. A score is kept when
 * >= nms_score_threshold; candidates go by score descending (-0 as +0), ties to the lower anchor; a
 * candidate is dropped when its IoU with a selected box (TFLite's formula; 0 for a box of non-positive
 * area) is > nms_iou_threshold. Fast mode: NMS on each anchor's best score (ArgMaxVector for one class
 * per detection; several go by score descending, class ascending, NaN last). Regular mode: NMS per class
 * up to detections_per_class, then the stable top-max_detections of the class lists in class order.
 * Refuses more than lce_b200_detection_max_anchors() anchors. No allocation, no synchronisation. */
int lce_b200_f32_detection_postprocess(const float* boxes_dev, const float* scores_dev, int batch, int num_anchors,
                                       int box_dim, int score_dim, const float* anchors_dev,
                                       const lce_b200_detection_options* opts, float* det_boxes_dev,
                                       float* det_classes_dev, float* det_scores_dev, float* num_detections_dev,
                                       void* workspace_dev, void* stream);
/* Grouped CONV_2D (TF/lite/kernels/conv.cc with groups = in_c / filter_in): x NHWC [batch, in_h,
 * in_w, d->in_c], filter OHWI [d->out_c, filter_h, filter_w, d->in_c / groups]; output channel o reads
 * the input channels [(o / (out_c / groups)) * in_c / groups, ...). `groups` must divide in_c and
 * out_c; any stride, dilation and SAME / VALID padding. Each output is the fmaf chain of
 * lce_b200_f32_conv2d over its group's channels (acc = 0, then (fy, fx, ci) in order, padded taps as
 * fma(0, w, acc)), then
 *   y = act(acc [+ bias[o]]),  y = fl(y * scale[o]),  y = fl(y + shift[o]),  out = post_act(y)
 * with act = d->activation and post_activation an LCE_ACT_* code: a BatchNorm folded as MUL then ADD
 * behind the convolution, rounded as those ops round. bias, scale and shift may be NULL (that step is
 * absent). So the result equals one lce_b200_f32_conv2d per group on the channel slices, concatenated
 * (then MUL and ADD), bit for bit. 3x3 stride-1 convolutions of 8 -> 8 channels in 4 groups and 4 -> 8
 * in 8 groups on 16-byte aligned tensors run a tiled kernel; other shapes a direct one. */
struct lce_f32_conv_desc; /* lce_b200_builtins.h */
int lce_b200_f32_grouped_conv2d(const struct lce_f32_conv_desc* d, int groups, const float* in_dev,
                                const float* filter_dev, const float* bias_dev, const float* scale_dev,
                                const float* shift_dev, int post_activation, float* out_dev,
                                void* stream);
int lce_b200_bconv2d_run_host(lce_b200_bconv2d* plan, const int32_t* in_host,
                              void* out_host);
void lce_b200_bconv2d_destroy(lce_b200_bconv2d* plan);

/* ---- BGEMM --------------------------------------------------------------
 * Replaces bgemm::BGemm (LCE/core/bgemm/bgemm.h:25-84) with the orientation of
 * optimized_bgemm.h:126-151: A = activations [M, Kw] (row per output pixel),
 * W = filters [N, Kw]; out [M, N] row-major (raw int32 accumulators, float or
 * int8) or [M, ceil(N/32)] bitpacked. The epilogue is OutputTransform<Dst>
 * (LCE/core/bconv2d/output_transform.h:94-168), already folded. */
typedef struct lce_b200_bgemm lce_b200_bgemm;

int lce_b200_bgemm_create(int N, int Kw, const int32_t* W,
                          const lce_bgemm_epilogue* ep, lce_b200_bgemm** plan);
int lce_b200_bgemm_run(lce_b200_bgemm* plan, int64_t M, const int32_t* A_dev,
                       void* out_dev, void* stream);
void lce_b200_bgemm_destroy(lce_b200_bgemm* plan);

/* Number of kernels this library has launched in this process (bench.py's
 * `gpu_launches`). */
uint64_t lce_b200_launch_count(void);
/* Diagnostics. path_counts: inner-product launches so far by kernel family
 * {wgmma (lce_b200_tc.cuh), mma.sync b1 or int8 (lce_b200_imma.cuh), XOR + POPC
 * (lce_b200_kernels.cuh)} -- the tests use it to prove which kernel ran.
 * tc_debug: the wgmma kernel's deadlock-watchdog record; out[7] != 0 means a
 * wait timed out ({barrier tag, block, thread, parity, count} in out[0..4]);
 * reading clears the flag. */
void lce_b200_path_counts(uint64_t out[3]);
int lce_b200_tc_debug(int32_t out[8]);

#ifdef __cplusplus
}
#endif
#endif /* LCE_B200_H_ */

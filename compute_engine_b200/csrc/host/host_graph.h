// host_graph.h -- the caller of the hot path: a small graph host that plays the
// role TFLite's Subgraph plays for the reference (tensorflow/lite/core/subgraph.cc:
// OpInit :1271, OpPrepare :1302, OpInvoke :1368, ResizeInputTensor :1170,
// AllocateTensors) but keeps the tensor arena in HBM, so consecutive ops never
// round-trip through the host, and can replay the op sequence as one CUDA graph.
//
// It drives ANY TfLiteRegistration {init, free, prepare, invoke}: this library's
// CUDA ops (lce_ops.cc), the float builtins the three model families need
// (builtin_ops.cc), or -- in CPU tests -- the oracle-backed registrations built
// under oracle/ (arena then lives on the host; no CUDA call is made).
#ifndef LCE_B200_HOST_GRAPH_H_
#define LCE_B200_HOST_GRAPH_H_

#include <cstdint>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "lce_b200_tflite.h"

namespace lce_b200 {

struct BuiltinParams;   // builtin_params.h

// MutableOpResolver stand-in (tensorflow/lite/mutable_op_resolver.h:83): custom ops
// by name, builtins by schema BuiltinOperator code.
class OpResolver {
 public:
  void AddCustom(const char* name, const TfLiteRegistration* registration);
  void AddBuiltin(int builtin_code, const TfLiteRegistration* registration);
  const TfLiteRegistration* FindCustom(const std::string& name) const;
  const TfLiteRegistration* FindBuiltin(int builtin_code) const;

 private:
  std::map<std::string, const TfLiteRegistration*> custom_;
  std::map<int, const TfLiteRegistration*> builtin_;
};

struct NodeRecord {
  TfLiteNode node{};
  const TfLiteRegistration* registration = nullptr;
  std::vector<uint8_t> custom_options;
  std::vector<uint8_t> builtin_blob;  // builtin parameter struct (node.builtin_data)
  bool initialized = false;
  std::string name;
};

class Graph {
 public:
  // device_arena: activations in HBM (cudaMalloc) vs host memory (CPU tests).
  explicit Graph(bool device_arena);
  ~Graph();
  Graph(const Graph&) = delete;
  Graph& operator=(const Graph&) = delete;

  // const_data != nullptr makes a constant (kTfLiteMmapRo) tensor; its bytes are
  // copied (host copy always; device copy too when `const_on_device`).
  int AddTensor(TfLiteType type, const std::vector<int>& dims, const void* const_data,
                size_t const_bytes, bool has_quant, float scale, int zero_point,
                const std::string& name, bool const_on_device = false);
  int AddNode(const TfLiteRegistration* registration, const std::vector<int>& inputs,
              const std::vector<int>& outputs, const uint8_t* custom_options,
              size_t options_len, const void* builtin_data = nullptr,
              size_t builtin_bytes = 0, const std::string& name = "");
  void SetInputs(const std::vector<int>& t) { inputs_ = t; }
  void SetOutputs(const std::vector<int>& t) { outputs_ = t; }
  const std::vector<int>& inputs() const { return inputs_; }
  const std::vector<int>& outputs() const { return outputs_; }

  // Graph-level fusion of the converter's residual-block pattern
  //   LceBconv2d(float out y) -> ADD(y, shortcut) [-> LceQuantize of the sum]
  // into one node (the bconv epilogue adds the shortcut and emits the packed signs for
  // the next binary layer). Bit-identical results; y must have no other consumer.
  // Returns the number of (ADD, LceQuantize) nodes removed. Call before AllocateTensors.
  int FuseResidualBlocks();

  // ReActNet's per-channel chain: RPReLU (ADD(const) -> PRELU(const) -> ADD(const)) and the next
  // layer's RSign ([ADD(const) ->] LceQuantize), each step optional:
  //   after a "LceBconv2d+ADD" node (FuseResidualBlocks first) it moves into that node's epilogue
  //   (inputs 6..9 = shift_in, alpha, shift_out, sign_shift; lce_b200_bconv2d_run_fused_chain);
  //   elsewhere it becomes one node (lce_b200_f32_chain_sign) that replaces at least two.
  // Only float constants of shape [1, ..., 1, C] (kTfLiteMmapRo), ADDs without fused activation,
  // and intermediates with a single consumer that are not graph outputs are absorbed; otherwise
  // the graph is left as it is. Bit-identical. Returns the number of nodes removed.
  int FuseActivationChains();

  // Real-to-Binary Net's gated block tail
  //   LceBconv2d(float y) -> MUL(y, g [B,1,1,C]) -> PRELU(alpha) -> ADD(shortcut)
  //     [-> MUL(scale) -> ADD(shift) -> LceQuantize, the next block's BatchNorm and sign]
  // becomes one node "LceBconv2d+MUL+PRELU+ADD[+MUL+ADD+LceQuantize]"
  // (lce_b200_bconv2d_run_fused_gate): inputs [in, filter, mul, bias, thr, shortcut, g, alpha,
  // scale, shift (-1 when the sign tail is absent)], outputs [sum, packed signs?]. Only when g is
  // a computed float [B,1,1,C] tensor, alpha / scale / shift are float constants of shape
  // [1, ..., 1, C], the MULs and the BatchNorm ADD have no fused activation (the shortcut ADD's is
  // applied), every intermediate has a single consumer and is not a graph output, and g and the
  // shortcut exist before the convolution runs. Run before FuseActivationChains, which would
  // otherwise take the BatchNorm's ADD -> LceQuantize as a lone RSign. Bit-identical. Returns the
  // number of nodes removed.
  int FuseChannelGates();

  // XNOR-Net++'s scaled block tail
  //   LceBconv2d(float y) -> MUL(y, gamma) -> ADD(shortcut)
  //     [-> MUL(scale) -> ADD(shift) -> LceQuantize, the next block's BatchNorm and sign]
  // becomes one node "LceBconv2d+MUL+ADD[+MUL+ADD+LceQuantize]" (lce_b200_bconv2d_run_fused_scale):
  // inputs [in, filter, mul, bias, thr, shortcut, gamma, scale, shift (-1 when the sign tail is
  // absent)], outputs [sum, packed signs?]. Only when gamma is a float constant of shape
  // [1, OH, OW, C] or [OH, OW, C] (one value per output position and channel), scale / shift are
  // float constants of shape [C] or [1, ..., 1, C], the MULs and the BatchNorm ADD have no fused
  // activation (the shortcut ADD's, any, is applied), y, the MUL's output and the BatchNorm's
  // intermediates have a single consumer and are not graph outputs (the sum may have other
  // readers), and the shortcut exists before the convolution runs; otherwise the graph is left as
  // it is. Run before FuseFloatGlue and FuseActivationChains, which would otherwise take the
  // BatchNorm's ADD -> LceQuantize as a lone RSign. Bit-identical. Returns the number of nodes
  // removed.
  int FuseSpatialScales();

  // ABC-Net's multiple binary bases (Lin et al., NeurIPS 2017): a layer on a float map x with N
  // shifted signs q_n = LceQuantize(ADD(x, u_n)) and M weight bases,
  //   t_nm = LceBconv2d(q_n, B_m)  ->  ADD(...ADD(ADD(t_00, t_01), t_02)..., t_{N-1,M-1})  (n outer)
  //     -> MUL(bn_scale) -> ADD(bn_shift, any activation) [-> ADD(shortcut, any activation)]
  //     [-> the next layer's ADD(o, u'_k) -> LceQuantize pairs]
  // becomes one node "LceBconv2dBases[+LceQuantize]" (lce_b200_bconv2d_bases_run): inputs [q_0..q_{N-1},
  // then filter, mul, bias of each term in (n, m) order, bn_scale, bn_shift, shortcut (-1 when
  // absent)], outputs [o if anything other than the absorbed pairs reads it or it is a graph output,
  // then the next planes], builtin_data int32 {M, N, next planes, BatchNorm activation, shortcut
  // activation, o stored} and the next shifts as floats; options are term 0's. When the q_n come
  // from unfused pairs, they become one node "ADD+LceQuantize" (lce_b200_f32_shift_sign_planes): inputs
  // [x], outputs [q_0..q_{N-1}], builtin_data int32 N then the N shifts. Only when every u_n is a
  // one-element float constant and the ADDs have no fused activation; M * N >= 2 (a single
  // LceBconv2d never matches) with M, N <= 8; the terms are plain float LceBconv2d nodes with equal
  // options and filter shapes, constant inputs and term (n, m)'s filter equal to term (0, m)'s; term
  // k of the chain reads plane k / M, and each plane is read by its M terms alone; the chain's ADDs
  // take the running sum as their first operand and have no fused activation; bn_scale / bn_shift
  // are float constants [C] or [1, ..., 1, C]; every intermediate has one consumer and is not a graph
  // output; and lce_b200_bconv2d_bases_create takes the terms (one-padded or VALID, no fused
  // activation, channels_out % 64 == 0, the bases' weights within shared memory). Zero-padded layers
  // stay unfused. Run first: FuseResidualBlocks would take ADD(t_00, t_01) as a residual block.
  // Bit-identical. Returns the number of nodes removed.
  int FuseBinaryBases();

  // BinaryAlexNet's and XNOR-Net's pooled BatchNorm and sign
  //   MAX_POOL_2D(x) -> MUL(scale) -> ADD(shift) -> LceQuantize
  // becomes one node "MAX_POOL_2D+MUL+ADD+LceQuantize" (lce_b200_f32_maxpool_affine_sign): inputs
  // [x, scale, shift], output [packed signs], builtin_data the pool's parameters; the float map is
  // read once and only the signs are written. Only when scale and shift are float constants of shape
  // [C] or [1, ..., 1, C] and the second operand of their op, the MUL and ADD have no fused
  // activation (the pool's own is applied), and the pool, MUL and ADD outputs each have one consumer
  // and are not graph outputs; otherwise the graph is left as it is. Run before FuseChannelGates /
  // FuseActivationChains, which would otherwise take the ADD -> LceQuantize as a lone RSign.
  // Bit-identical. Returns the number of nodes removed (3 per pooled layer).
  int FusePooledSigns();

  // DoReFaNet's 2-bit activations: the quantiser a = round(clip(x, 0, 1) * 3) / 3 in front of a float
  // convolution or dense layer whose weights are +-alpha_o,
  //   [MAX_POOL_2D ->] MAXIMUM(0) -> MINIMUM(1) -> MUL(3) -> ROUND -> DIV(3) -> CONV_2D | FULLY_CONNECTED
  // becomes two nodes: "[MAX_POOL_2D+]Quant2" (lce_b200_f32_quant2_planes), which writes the level
  // q = 3 a as the int32 bit planes [plane 0 | plane 1 | plane 1], [B,H,W,3*C/32], and a plain
  // "LceBconv2d" over channels_in = 3 * C with pad_values 1 and the layer's stride, padding and
  // dilation, whose constants the pass synthesises: the filter's sign words (bit set = negative
  // weight) repeated three times per tap, post_mul[o] = fl(-alpha_o / 6) and post_bias[o] =
  // fl(alpha_o * W_o / 2 + bias_o), W_o the sum of filter o's signs, both computed in double. With
  // t = 1 - 2 bit the convolution's accumulator is D = sum s * (3 - 2 q), a padded tap counting as
  // q = 0, so y = alpha/3 * sum s * q + bias = -alpha/6 * D + alpha * W / 2 + bias: CONV_2D's zero
  // padding is one-padding here. FULLY_CONNECTED [rows,K] -> [rows,N] is the 1x1 VALID case; its output
  // tensor becomes [rows,1,1,N], the same bytes. Only when the four constants have one element and
  // are exactly 0, 1, 3 and 3; MUL and DIV have no fused activation; every layer that reads the
  // quantised tensor qualifies (several may): float constant weights whose magnitude is bitwise
  // one non-zero finite value per output channel, a float constant bias or none, no fused
  // activation (LCE clamps before the multiplier, TFLite after the bias), C % 32 == 0,
  // 3 * k * k * C < 2^24 (so float(D) is exact), parameters lce_b200_bconv2d_out_shape accepts, and for
  // FULLY_CONNECTED an output that is not a graph output; every intermediate has one consumer and
  // none is a graph output. The pool is absorbed when only the quantiser reads it. Otherwise the
  // graph is left as it is. The levels are the unfused ops' bit for bit and D is an exact integer,
  // so y is the real-valued result rounded twice; TFLite's float CONV_2D rounds after each of its
  // K = k * k * C terms, so the two differ by up to about K * 2^-24 * sum |a| |w|: NOT bit-identical
  // to the float ops, and a difference can flip a level of the next quantiser at a near-tie. Returns
  // the number of nodes removed (4, or 5 with the pool, per quantiser).
  int FuseQuantizedActivations();

  // A BatchNorm behind a grouped convolution (Keras Conv2D(groups=g), or MeliusNet's stem with each
  // group convolution as one op)
  //   CONV_2D(filter [C, kh, kw, C_in / g], no fused activation) -> MUL(scale) -> ADD(shift, any activation)
  // becomes one node "CONV_2D+MUL+ADD" (lce_b200_f32_grouped_conv2d with the epilogue): inputs [x,
  // filter, bias (-1 when absent), scale, shift], builtin_data { the conv's, the ADD's BuiltinParams }.
  // Only when g = C_in / filter_in is an exact division other than 1 and divides C, scale and shift
  // are float constants of shape [C] or [1, ..., 1, C] and the second operand of their op, the MUL
  // has no fused activation, and the conv and MUL outputs each have one consumer and are not graph
  // outputs; an ungrouped CONV_2D is never matched. Bit-identical. Returns the nodes removed (2 each).
  int FuseGroupedConvAffine();

  // BinaryDenseNet's dense layers
  //   x_j [B,H,W,C_j] -> MUL(scale) -> ADD(shift) -> LceQuantize -> LceBconv2d (float y_j)
  //   x_{j+1} = CONCATENATION([x_j, y_j], last axis)
  // and MeliusNet's improvement layers
  //   x_j -> MUL(scale) -> ADD(shift) -> LceQuantize -> LceBconv2d (float y_j, C_out channels)
  //   a = STRIDED_SLICE(x_j)[..., :C_j - C_out], b = STRIDED_SLICE(x_j)[..., C_j - C_out:]
  //   x_{j+1} = CONCATENATION([a, ADD(b, y_j)], last axis)
  // become one node each, "MUL+ADD+LceQuantize+LceBconv2d+CONCATENATION" or
  // "MUL+ADD+LceQuantize+LceBconv2d+STRIDED_SLICE+ADD+CONCATENATION": inputs [src, scale, shift,
  // filter, mul, bias, thr], outputs [X], temporaries [packed signs] or [packed signs, scratch]. A
  // chain of such layers shares one tensor X, the block's final map [B,H,W,C_L]; each layer reads
  // X's first C_j channels; a dense layer writes its new ones into X[..., C_j : C_j + C_out]
  // (lce_b200_f32_affine_sign, lce_b200_bconv2d_run_slice), an improvement layer adds its own to
  // X[..., C_j - C_out : C_j] (lce_b200_bconv2d_run_slice_add, through the scratch [B,H,W,C_out]
  // for a zero-padding CORRECTION plan), so no x_j and no slice or concatenation copy exists. src
  // is x_0 for the block's first layer, which also copies x_0 into X, and X for the others. Only
  // when scale and shift are float constants [C] or [1, ..., 1, C], the MUL and ADDs have no fused
  // activation, the LceBconv2d is a plain node with float output that run_slice takes (same image
  // size), the CONCATENATION is exactly [x_j, y_j] / [a, sum] on the last axis with no activation,
  // the slices cover exactly those channels with every other axis whole and unit strides (the
  // STRIDED_SLICE builtin's own normalisation decides), C_j and C_L are multiples of 4, every
  // intermediate has one consumer and is not a graph output, and each x_j with j >= 1 is read only
  // by the next layer's nodes (a dense layer's MUL and CONCATENATION, an improvement layer's MUL
  // and two STRIDED_SLICEs). Run first: FuseResidualBlocks would otherwise take an improvement
  // layer's LceBconv2d -> ADD(b), and FuseChannelGates / FuseActivationChains the ADD ->
  // LceQuantize as a lone RSign. Bit-identical. Returns the number of nodes removed.
  int FuseDenseBlocks();

  // Two consecutive residual blocks x1 = x0 + f1(sign x0), x2 = x1 + f2(sign x1) -- a
  // "LceBconv2d+ADD+LceQuantize" node whose two outputs only the next "LceBconv2d+ADD[+LceQuantize]"
  // node reads, as its packed input and its shortcut -- become one node
  // "LceBconv2d+ADD+LceBconv2d+ADD[+LceQuantize]" (lce_b200_bconv2d_run_fused_pair): x1 stays on
  // chip. Inputs [x0 packed, f1, mul1, bias1, thr1, x0, f2, mul2, bias2, thr2], outputs
  // [x2, packed x2?]. Both layers must be ones the pair kernel takes (3x3, stride 1, one-padding,
  // C -> C, C = 64 or 128), on an image its tiles cover at least half full at the tensors' shapes
  // when the pass runs (smaller images run faster unpaired); pairing is greedy in graph order. Call
  // after FuseResidualBlocks and FuseActivationChains. Bit-identical. Returns the nodes removed.
  int FuseResidualPairs();

  // Fusions among the float builtins around the binary path:
  //   MAX_POOL_2D(2x2, stride 1, VALID) -> DEPTHWISE_CONV_2D(3x3)  =>  one node
  //   CONV_2D(3x3 s2 -> 16) -> DEPTHWISE_CONV_2D(3x3 s2) -> CONV_2D(1x1 -> 64)  =>  one node (opt-in)
  //   CONV_2D -> LceQuantize  =>  the conv writes the packed signs as a second output
  // (QuickNet's anti-aliased down-sampling). Bit-identical. Returns the nodes removed.
  int FuseFloatGlue();
  int FuseConvQuantize();  // part of FuseFloatGlue: CONV_2D -> LceQuantize => conv with 2 outputs
  int FuseStem();  // part of FuseFloatGlue: [DEQUANTIZE +] stem conv + depthwise conv -> one node

  // A segmentation decoder's merge
  //   RESIZE_NEAREST_NEIGHBOR(u) -> ADD(v, skip) [-> LceQuantize]
  // becomes one node "RESIZE_NEAREST_NEIGHBOR+ADD[+LceQuantize]" (lce_b200_f32_upsample_add_sign),
  // which reads u at each output pixel's nearest source pixel, so the upsampled copy of u is never
  // written and the sum is read by nobody to make its signs: inputs [u, size, skip], outputs [sum (-1
  // when only the absorbed LceQuantize reads it and it is not a graph output), packed signs?],
  // builtin_data { the resize's, the ADD's BuiltinParams }; the ADD's activation is applied. v may be
  // either operand of the ADD. Only when v has one consumer, the ADD, and is not a graph output; u,
  // v and skip are float32 and v and skip have the same 4-D shape (no broadcast); otherwise the graph
  // is left as it is. The LceQuantize is absorbed only when C % 32 == 0 and it is the sum's only
  // LceQuantize reader. No other pass matches a RESIZE_NEAREST_NEIGHBOR, so the pass may run anywhere;
  // fuse_all runs it after FuseFloatGlue and before FuseChannelGates / FuseActivationChains, the
  // passes that look for a lone ADD -> LceQuantize sign tail, so that none of them can take the
  // merge's sign first. Bit-identical. Returns the number of nodes removed.
  int FuseUpsampleMerges();

  // A segmentation head that ends in a per-pixel label
  //   RESIZE_BILINEAR(x) -> ARG_MAX(v, axis = the channel axis)
  // becomes one node "RESIZE_BILINEAR+ARG_MAX" (lce_b200_f32_resize_bilinear_argmax), which computes
  // each output pixel's resized values from two source rows staged on chip and stores only their
  // label, so the resized map v is never written: inputs [x, size, axis], outputs [labels], builtin_data
  // { the resize's, the ARG_MAX's BuiltinParams }. Only when v is float32 and 4-D, has one consumer,
  // the ARG_MAX, which reads it as input 0, and is not a graph output; the axis is a constant that
  // normalises to 3; and x's rows (in_w * C floats) fit lce_b200_resize_bilinear_argmax_max_row_floats().
  // Otherwise the graph is left as it is. No other pass matches either op, so the pass may run
  // anywhere; fuse_all runs it after FuseUpsampleMerges. Bit-identical. Returns the nodes removed.
  int FuseResizeArgmax();

  // A super-resolution network's sub-pixel tail
  //   CONV_2D(x) -> DEPTH_TO_SPACE(y, r) [-> ADD(s, RESIZE_BILINEAR(img))]
  // becomes one node (lce_b200_f32_subpixel_conv) that computes each low-resolution pixel's conv
  // channels, stores them at their high-resolution addresses and adds the resized image there, so
  // y, s and the resized image are never written: "CONV_2D+DEPTH_TO_SPACE+RESIZE_BILINEAR+ADD", inputs
  // [x, filter, bias (-1 when absent), img, size], or without the ADD part "CONV_2D+DEPTH_TO_SPACE",
  // inputs [x, filter, bias]; builtin_data { the conv's, the DEPTH_TO_SPACE's, the resize's, the ADD's
  // BuiltinParams } (the last two zero without the ADD). Only when the conv is float32 and ungrouped,
  // with a constant [Cout, 3, 3, Cin] filter and a constant bias or none, stride 1, dilation 1, SAME,
  // Cin % 4 == 0, Cout <= lce_b200_subpixel_conv_max_out_channels(), and runs on the implicit-GEMM
  // kernels unfused (lce_b200_internal_conv_runs_igemm, the predicate conv2d_impl dispatches by), whose
  // chain the fused kernel repeats; y has one reader, the DEPTH_TO_SPACE, and is not a graph output;
  // r >= 2. The ADD part joins only when s's one reader is an ADD (either operand), the other operand
  // is a RESIZE_BILINEAR output of s's 4-D shape (no broadcast) read by the ADD alone, resized from a
  // float32 4-D img by a constant size, and neither s nor the resized map is a graph output; otherwise
  // the ADD and the resize stay as they are. Otherwise the graph is left as it is. No other pass
  // matches a DEPTH_TO_SPACE, so the pass may run anywhere; fuse_all runs it after FuseResizeArgmax.
  // Bit-identical. Returns the nodes removed.
  int FuseSubpixelConvs();

  // A binary learned upsampler, as a larq QuantConv2DTranspose(ste_sign, ste_sign) converts,
  //   LceDequantize(q) -> TRANSPOSE_CONV(+-1 weights, kernel = stride s_h x s_w, s_h * s_w >= 2, bias?,
  //   activation) [-> ADD(skip)] [-> LceQuantize]
  // becomes one node (lce_b200_bconv2d_run_fused_shuffle) that reads q's packed words, runs the layer as
  // a 1x1 binary convolution to s_h * s_w * C columns on the b1 mma.sync kernel and stores each column
  // at its pixel-shuffled address, adding the bias, the activation and the skip there and packing the
  // signs: "LceBconv2dTranspose[+ADD][+LceQuantize]", inputs [q, packed filter (a new constant), bias
  // (-1 when absent), skip (-1 when absent)], outputs [sum, signs?]. The sum is always stored (the
  // decoder's next shortcut reads it). Only when every weight is exactly +1.0f or -1.0f, the output is
  // exactly in * s (no output_padding), C % 64 == 0 and the plan lands on the b1 mma.sync kernel
  // (lce_b200_internal_shuffle_takes); the dequantized map is read by the TRANSPOSE_CONV alone and is
  // not a graph output. The ADD joins only when it is the TRANSPOSE_CONV output's one reader (not a graph
  // output), without broadcast, with the skip ready before it; the LceQuantize joins when it is the
  // sum's only sign reader. Otherwise the graph is left as it is. Bit-identical: every product is +-1,
  // so the dot product is exact in any order. fuse_all runs it before FuseResidualBlocks; no pass before
  // it matches a TRANSPOSE_CONV, its ADD or its LceQuantize. Returns the nodes removed.
  int FuseBinaryTransposeConvs();

  // A binary dense layer, as a larq QuantDense(ste_sign, ste_sign) converts (LCE has no binary dense op),
  //   LceDequantize(q) -> FULLY_CONNECTED(+-alpha_o weights, bias?, activation)
  //   [-> MUL(scale [N]) -> ADD(shift [N], activation)] [-> LceQuantize]
  // becomes one node (lce_b200_bconv2d_run_fused_fc) that reads q's packed words and runs the layer as
  // a 1x1 binary convolution of rows = the FULLY_CONNECTED's rows on the b1 mma.sync kernel, applying
  // alpha, the bias, the activation, the BatchNorm and its activation to the exact +-1 dot product D in
  // its store and packing the signs: "LceBfc[+MUL+ADD][+LceQuantize]", inputs [q, packed filter (a new
  // constant), alpha (a new constant [N], -1 when every alpha_o is 1.0), bias, scale, shift (-1 when
  // absent)], outputs [result, signs?]. The result is always stored. Only when every row o of the
  // constant [N, K] weights is exactly +-alpha_o with one positive finite magnitude bitwise (no 0.0 or
  // -0.0), the bias is a constant float32 [N], N % 64 == 0 and the plan lands on the b1 mma.sync kernel
  // (lce_b200_internal_fc_takes), the dequantized map is read by the FULLY_CONNECTED alone and is not a
  // graph output, and q's words are the rows' words (x's last axis is K, or it is a multiple of 32 and
  // so is K). The MUL and ADD join only as the sole readers of the previous result with constant
  // float32 [N] operands; the LceQuantize when it is the result's only sign reader. Otherwise the graph
  // is left as it is. Each step rounds as TFLite's ops do, so with every alpha_o a power of two (1.0
  // included) it is bit-identical; otherwise fl(fl(alpha * D) + b) is the real value rounded twice
  // where TFLite's loop rounds after each of its K terms: the two differ by up to about
  // K * 2^-24 * K * alpha_o, which can flip the next sign at a near-tie. fuse_all runs it right after
  // FuseBinaryTransposeConvs and FuseBinaryFcMax; no other pass before it matches a FULLY_CONNECTED.
  // With keep_num_dims (the layer's input's last axis then being K) the result keeps the input's
  // leading axes. Returns the nodes removed.
  int FuseBinaryFullyConnected();

  // A binary point-wise layer and the max over its points, as a BiPointNet's last shared MLP layer and
  // its global max-pool convert:
  //   LceDequantize(q) -> FULLY_CONNECTED(+-alpha_o weights, bias?, activation, keep_num_dims)
  //   [-> MUL(scale [N]) -> ADD(shift [N], activation)] -> REDUCE_MAX(axis 1 of [B, P, N]) [-> LceQuantize]
  // becomes one node (lce_b200_bconv2d_run_fused_fc_max), "LceBfc[+MUL+ADD]+REDUCE_MAX[+LceQuantize]",
  // inputs [q, packed filter, alpha, bias, scale, shift] as FuseBinaryFullyConnected's, outputs [max?,
  // signs?], one temporary (the per-(image, column) keys). The [B, P, N] map is never stored; the max
  // [B, N] only when a node other than the LceQuantize reads it or it is a graph output. Only under
  // FuseBinaryFullyConnected's conditions, when the layer's result is [B, P, N], read by the REDUCE_MAX
  // alone as its input and not a graph output, and the REDUCE_MAX's constant int32 axes are all the
  // point axis (1 or -2). The LceQuantize joins when it is the max's only sign reader. Otherwise the
  // graph is left as it is. Every value is the one FuseBinaryFullyConnected's node computes, and the
  // max is TFLite's reference rule over them (NaN never chosen, the first of equal values), so the
  // node's bits are the unfused pair's. fuse_all runs it right before FuseBinaryFullyConnected.
  // Returns the nodes removed.
  int FuseBinaryFcMax();

  // init (first time) + prepare of every node in order, then arena allocation.
  TfLiteStatus AllocateTensors();
  TfLiteStatus ResizeInputTensor(int tensor, const std::vector<int>& dims);
  TfLiteStatus Invoke();
  // Capture the node sequence into a CUDA graph and replay it on later Invokes.
  TfLiteStatus EnableCudaGraph(bool on);
  // Debug aid (TFLite's `preserve_all_tensors`): no arena reuse, so every intermediate
  // tensor can be read back after Invoke.
  void set_preserve_all_tensors(bool on) { preserve_all_ = on; allocated_ = false; }

  // Per-node device timing (eager mode only): CUDA events on the graph's stream
  // around every node's invoke; times accumulate until ResetProfile().
  void EnableProfiling(bool on) { profiling_ = on; }
  void ResetProfile();
  double NodeTimeMs(size_t node);   // synchronises the stream
  TfLiteStatus Synchronize();

  TfLiteTensor* tensor(int i) { return &tensors_[i]; }
  size_t num_tensors() const { return tensors_.size(); }
  size_t num_nodes() const { return nodes_.size(); }
  const NodeRecord& node(size_t i) const { return *nodes_[i]; }
  TfLiteStatus WriteTensor(int i, const void* host_src, size_t bytes);
  TfLiteStatus ReadTensor(int i, void* host_dst, size_t bytes);
  // async on the graph's stream; pinned host or device destinations; no synchronise
  TfLiteStatus ReadTensorAsync(int i, void* dst, size_t bytes);
  const std::string& last_error() const { return error_; }
  void set_error(const std::string& e) { error_ = e; }
  bool device_arena() const { return device_arena_; }
  size_t arena_bytes() const { return arena_bytes_; }
  void* stream() const { return stream_; }

 private:
  static TfLiteStatus ResizeTensorCb(TfLiteContext*, TfLiteTensor*, TfLiteIntArray*);
  static void ReportErrorCb(TfLiteContext*, const char* msg, ...);
  static TfLiteStatus AddTensorsCb(TfLiteContext*, int, int*);
  static TfLiteTensor* GetTensorCb(const TfLiteContext*, int);
  static TfLiteExternalContext* GetExternalContextCb(TfLiteContext*, TfLiteExternalContextType);
  static void SetExternalContextCb(TfLiteContext*, TfLiteExternalContextType,
                                   TfLiteExternalContext*);
  TfLiteStatus PlanArena();
  void FreeArena();
  void RefreshContext();

  // What the fusion passes ask of the graph. "No such node" is kNoNode, which no index equals and
  // every `k < nodes_.size()` test refuses, before and after nodes are erased.
  static constexpr size_t kNoNode = SIZE_MAX;
  bool IsGraphOutput(int t) const;
  std::vector<size_t> Consumers(int t) const;   // the nodes that read t, each once, in graph order
  // The one node that reads t (in any of its inputs, in several of them too), t not a graph output.
  size_t SoleConsumer(int t) const;
  // The node that reads t when t is read by exactly one input of one node, that node's first, and
  // is not a graph output: what a pass needs whose fused node takes over input 0 alone.
  size_t SoleReaderAsFirstInput(int t) const;
  bool ReadyBefore(int t, size_t i) const;      // t is a graph input or an output of a node before i
  static bool SameDims(const TfLiteIntArray* a, const TfLiteIntArray* b);
  static const BuiltinParams* Params(const NodeRecord& n);   // nullptr when the blob is too short
  static int32_t Activation(const NodeRecord& n);            // 0 for a node without parameters
  // Node k is the unprepared builtin `op`(x, v) with one float output, parameters, no fused
  // activation (unless any_activation) and v a float constant of shape [C] or [1, ..., 1, C]:
  // returns v, else -1 (also for k = kNoNode).
  int PerChannelConstOp(size_t k, const char* op, int x, int C, bool any_activation = false) const;
  // Node k is an unprepared LceQuantize with one input and one int32 output (false for kNoNode).
  bool IsQuantize(size_t k) const;
  // FuseBinaryFullyConnected's and FuseBinaryFcMax's match: the FULLY_CONNECTED at fc, the LceDequantize
  // dq of q before it, its BatchNorm's MUL km and ADD ka (kNoNode without them), the constants, and the
  // tensor the layer ends in (the ADD's output, or the FULLY_CONNECTED's).
  struct BinaryFcMatch {
    size_t fc, dq, km, ka;
    int q, w, K, N, bias, scale, shift, result;
    int64_t rows;
    bool unit;                  // every alpha_o is 1.0
    std::vector<uint32_t> wb;   // the [N, K] weights' bits
    std::vector<float> alpha;
  };
  bool MatchBinaryFc(size_t i, BinaryFcMatch* m) const;
  // The match's packed filter [N, 1, 1, ceil(K / 32)] and alpha [N] (-1 when unit) as new constants.
  void BinaryFcConstants(const BinaryFcMatch& m, int* filter, int* alpha);

  // How the passes rewrite it. Each clears allocated_. A node they rewrite has not been prepared,
  // so its temporaries are the ones its pass gives it.
  void EraseNode(size_t k);
  void EraseNodes(std::vector<size_t> ks);   // in any order, without duplicates
  void SetNodeIO(NodeRecord& n, const std::vector<int>& inputs, const std::vector<int>& outputs,
                 const std::vector<int>& temporaries = {});
  void SetBuiltinBlob(NodeRecord& n, const void* bytes, size_t len);   // and node.builtin_data
  void SetCustomOptions(NodeRecord& n, std::vector<uint8_t> options);  // and node.custom_initial_data

  bool device_arena_;
  std::vector<TfLiteTensor> tensors_;
  std::vector<std::string> names_;
  std::vector<std::vector<uint8_t>> const_host_;  // host copies of constants
  std::vector<void*> const_dev_;                   // device copies (or nullptr)
  std::vector<std::unique_ptr<NodeRecord>> nodes_;
  std::vector<int> inputs_, outputs_;
  TfLiteContext ctx_{};
  TfLiteExternalContext* external_[kTfLiteMaxExternalContexts] = {};
  std::string error_;
  void* arena_ = nullptr;
  size_t arena_bytes_ = 0;
  bool allocated_ = false;
  void* stream_ = nullptr;       // cudaStream_t
  bool use_cuda_graph_ = false;
  bool preserve_all_ = false;
  bool profiling_ = false;
  std::vector<std::vector<std::pair<void*, void*>>> node_events_;  // pending (start, stop)
  std::vector<double> node_ms_;
  bool warmed_ = false;          // one eager Invoke has run since the last allocation
  void* graph_exec_ = nullptr;   // cudaGraphExec_t
};

}  // namespace lce_b200
#endif

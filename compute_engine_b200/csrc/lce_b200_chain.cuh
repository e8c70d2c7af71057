// lce_b200_chain.cuh -- one element of ReActNet's per-channel chain (lce_chain_desc,
// include/lce_b200_types.h) and of Real-to-Binary Net's gated tail (lce_gate_desc), shared by the mma.sync convolution epilogue (lce_b200_imma.cuh) and
// the stand-alone pass lce_b200_f32_chain_sign (lce_b200_builtins.cu), so the two give the same
// bits. Each step rounds like the TFLite op it replaces: ADD (add.h) and PRELU (prelu.h) are one
// IEEE operation each. __fadd_rn / __fmul_rn keep nvcc from contracting t * alpha + shift_out into
// an FMA, which would round once where the op sequence rounds twice.
#ifndef LCE_B200_CHAIN_CUH_
#define LCE_B200_CHAIN_CUH_

namespace lce {

// RPReLU: o = prelu(s + shift_in, alpha) + shift_out; an absent step (has_* false) is skipped
__device__ __forceinline__ float chain_rprelu(float s, bool has_si, float si, bool has_a, float a,
                                              bool has_so, float so) {
  if (has_si) s = __fadd_rn(s, si);
  if (has_a) s = s >= 0.0f ? s : __fmul_rn(s, a);
  if (has_so) s = __fadd_rn(s, so);
  return s;
}

// RSign: LceQuantize's bit (bitpack.h:159) of o + sign_shift
__device__ __forceinline__ bool chain_sign(float o, bool has_ss, float ss) {
  return (has_ss ? __fadd_rn(o, ss) : o) < 0.0f;
}

// Real-to-Binary's gated tail (lce_gate_desc): u = prelu(s * g, alpha), MUL (mul.h) and PRELU one
// IEEE operation each; the shortcut ADD follows in the caller
__device__ __forceinline__ float gate_prelu(float s, float g, bool has_a, float a) {
  s = __fmul_rn(s, g);
  if (has_a) s = s >= 0.0f ? s : __fmul_rn(s, a);
  return s;
}

// the next block's BatchNorm and sign: LceQuantize's bit of (o * scale + shift), rounded twice
__device__ __forceinline__ bool affine_sign(float o, bool has_sc, float sc, bool has_sh, float sh) {
  if (has_sc) o = __fmul_rn(o, sc);
  if (has_sh) o = __fadd_rn(o, sh);
  return o < 0.0f;
}

}  // namespace lce
#endif

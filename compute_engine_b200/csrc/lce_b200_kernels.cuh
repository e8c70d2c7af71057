// lce_b200_kernels.cuh -- hand-written sm_90a kernels for the LCE binary-conv
// hot path. No tensor cores: the inner product is XOR + POPC on the integer pipes
// (the tensor-core inner products are lce_b200_imma.cuh and lce_b200_tc.cuh), operands staged
// in shared memory as 128-bit vectors, weights brought in by the TMA bulk-copy
// engine (cp.async.bulk -> UBLKCP) onto an mbarrier, activations gathered with
// zero-filling cp.async (LDGSTS), and the OutputTransform fused into the epilogue.
//
// Reference semantics (LCE = /root/reference/larq_compute_engine):
//   K1 bsign_pack      LCE/core/bitpacking/bitpack.h:114-308
//   K2/K3 bconv/bgemm  LCE/core/bconv2d/reference.h:35-148, optimized_bgemm.h:64-178,
//                      LCE/core/bgemm/kernels.h:22-134, output_transform.h:94-168
//   K4 bmaxpool        LCE/core/bmaxpool.h:24-88
//   K5 unpack          LCE/core/bitpacking/bitpack.h:312-346
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "lce_b200_types.h"

namespace lce {

// ------------------------------------------------------------------------- //
// Tile configuration of the binary implicit-GEMM kernel.
//   CTA tile  BM x BN = 64 output pixels x 64 output channels, 128 threads, 4 CTAs per SM
//   (measured 3-9 % faster on the QuickNet layers than 128 x 64 / 256 threads / 2 CTAs per SM:
//   four independent CTAs interleave their gather / compute / epilogue phases better).
//   Warp tile 16 x 64 (lanes: 4 along M x 8 along N), thread tile 4 x 8.
// ------------------------------------------------------------------------- //
#ifndef LCE_BM
#define LCE_BM 64
#endif
constexpr int kBM = LCE_BM;
constexpr int kBN = 64;
constexpr int kThreads = 2 * kBM;          // two gather threads per pixel; one warp per 16 pixels
#ifndef LCE_CTAS
#define LCE_CTAS (512 / (2 * LCE_BM))
#endif
constexpr int kCtasPerSm = LCE_CTAS;  // 2 CTAs of 256 threads or 4 of 128 (register bound)
constexpr int kTM = 4;
constexpr int kTN = 8;
// Upper bound on K words staged per chunk so that kCtasPerSm CTAs fit in 227 KB of shared
// memory: (BM+BN)*Kc*4 B <= 96 KiB (BM 128, 2 CTAs/SM) or 48 KiB (BM 64, 4 CTAs/SM).
constexpr int kMaxChunkWords = (kBM == 128) ? 128 : (kCtasPerSm <= 4 ? 96 : 72);

// Division by a launch-constant with one wide multiply and a shift (the index decompositions in
// the gather and the epilogue otherwise cost ~25 instructions each). Exact for 0 <= n < 2^31:
// mul = floor(2^(31+L)/d) + 1, L = ceil(log2 d), q = (n * mul) >> (31 + L).
struct FastDiv {
  uint32_t mul, shift;
};
inline FastDiv make_fastdiv(uint32_t d) {
  FastDiv f;
  uint32_t L = 0;
  while ((1ull << L) < d) ++L;
  f.mul = static_cast<uint32_t>(((1ull << (31 + L)) / (d ? d : 1)) + 1);
  f.shift = 31 + L;
  return f;
}
__device__ __forceinline__ uint32_t fdiv(uint32_t n, FastDiv d) {
  return static_cast<uint32_t>((static_cast<unsigned long long>(n) * d.mul) >> d.shift);
}

// REDUCE_MAX's rule (TFLite's reference reduction: cur = lowest(), then cur = in > cur ? in : cur in
// index order) as a 64-bit key that atomicMax can merge in any order. High word: the value's
// order-preserving key, -0.0 and +0.0 one key; low word: the complemented row index (rows < 2^31),
// so that the first of equal values wins, and below it the value's sign bit, which tells the zeros
// apart. A NaN is never chosen: its key is 0, below every value's.
__device__ __forceinline__ uint32_t max_key_hi(float v) {
  uint32_t b = __float_as_uint(v);
  if ((b & 0x7fffffffu) == 0) b = 0;
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ unsigned long long max_key(float v, uint32_t row) {
  if (v != v) return 0ull;
  return (static_cast<unsigned long long>(max_key_hi(v)) << 32) | ((0x7fffffffu - row) << 1) |
         (__float_as_uint(v) >> 31);
}
// The key's value: -FLT_MAX when no key beats the initial value's (no value, NaNs, -inf only).
__device__ __forceinline__ float max_key_value(unsigned long long key) {
  const uint32_t hi = static_cast<uint32_t>(key >> 32);
  if (hi <= max_key_hi(-3.402823466e38f)) return -3.402823466e38f;
  uint32_t b = (hi & 0x80000000u) ? (hi & 0x7fffffffu) : ~hi;
  if (b == 0 && (key & 1ull)) b = 0x80000000u;
  return __uint_as_float(b);
}

// Fused shortcut: each thread parks its own 4 x 8 residual values (8 x 16 B) in shared memory
// with cp.async at kernel start, so the epilogue never waits on L2 / HBM.
constexpr int kResStageBytes = kThreads * 8 * 16;

struct ConvKParams {
  const int32_t* in;        // bitpacked NHWC activations
  const int32_t* wt;        // tiled weights [n_tiles][Kv][BN][V]
  void* out;
  const float* mul;         // folded multiplier (padded to cout + BN)
  const float* bias;        // folded bias
  const int32_t* thr;       // thresholds
  const int32_t* tap_popc;  // [cout + BN][taps] popcounts, zero-padding correction; or nullptr
  // Fused residual-block tail (float output only): out = act(y + residual) -- the TFLite ADD
  // that follows LceBconv2d -- and packed_out = LceQuantize(out) for the next binary layer.
  const float* residual;    // [M][cout] or nullptr
  int32_t* packed_out;      // [M][cw_out] or nullptr
  int residual_act;         // fused activation of the ADD
  long long M;              // batch * out_h * out_w
  int H, W, Cw_total, Cw_pg, CwV;
  int KH, KW, sh, sw, dh, dw, ph, pw, OH, OW;
  int cout, cout_pg, tiles_per_group;
  int Kv, Kc_v, n_chunks;
  int clamp_min, clamp_max;
  int cw_out;        // words per output pixel (bitpacked output)
  int zp_half;       // channels_in_per_group / 2 (zero-padding correction)
  int vec_store;     // output rows are 16B-aligned for this thread's 8 channels
  int bp_fast;       // bitpacked output: tiles start on a 32-channel boundary
  int res_stage;     // residual rows are staged through shared memory (kResStageBytes extra)
  const int32_t* wpop;  // IMMA path: popcount of each channel's whole filter row
  int zp_float, cin_pg; // zero padding with the optimised kernels' float correction (host-side switch)
  FastDiv fd_ohw, fd_ow, fd_cwv, fd_kw, fd_tpg;  // / (OH*OW), / OW, / CwV, / KW, / tiles_per_group
  long long img_words;  // H * W * Cw_total (< 2^31, checked by the host)
  // mma.sync kernel, CHAIN instances only: ReActNet's per-channel chain on the fused sum
  // (lce_b200_chain.cuh); packed_out then holds the signs of o + sign_shift
  lce_chain_desc chain;
  // GATE instances only: Real-to-Binary's gated tail before the shortcut ADD; packed_out then
  // holds the signs of o * sign_scale + sign_shift
  lce_gate_desc gate;
  // SLICE instances only: output pixel m's cout floats start at out + m * out_stride, and so do
  // the residual's (lce_b200_bconv2d_run_slice, lce_b200_bconv2d_run_slice_add)
  long long out_stride;
  // mma.sync kernel, SHUFFLE instances only (lce_b200_bconv2d_run_fused_shuffle): a 1x1 GEMM to
  // shuf_sh * shuf_sw * shuf_c columns stored pixel-shuffled, out [B, OH * shuf_sh, OW * shuf_sw,
  // shuf_c]; the +-1 dot product shuf_k - 2 popc (shuf_k = channels_in), shuf_bias (shuf_c floats, or
  // nullptr) added and shuf_act applied before the shortcut ADD
  int shuf_sh, shuf_sw, shuf_c, shuf_act, shuf_k;
  const float* shuf_bias;
  // SHUFFLE instances, lce_b200_bconv2d_run_fused_fc (shuf_sh = shuf_sw = 1, OH = OW = 1, shuf_c =
  // cout): shuf_alpha multiplies the dot product before the bias, then after shuf_act a BatchNorm
  // shuf_scale, shuf_shift and shuf_act2 (each vector shuf_c floats or nullptr; run_fused_shuffle
  // passes none of them and shuf_act2 = NONE)
  const float* shuf_alpha;
  const float* shuf_scale;
  const float* shuf_shift;
  int shuf_act2;
  // FCMAX instances only (lce_b200_bconv2d_run_fused_fc_max): the same columns, never stored; each
  // one's max over the rows of each image (fd_pts: / points per image) goes into max_keys [B][cout]
  unsigned long long* max_keys;
  FastDiv fd_pts;
  // mma.sync kernel, group-window (GW) instances only: 8 % (2 * Cw_pg), a k-slice's step through
  // the window
  int win_step;
};

// --------------------------- PTX helpers ---------------------------------- //
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)
               : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
// TMA bulk copy global -> shared (1-D, no tensor map). SASS: UBLKCP.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(dst_smem)),
      "l"(static_cast<uint64_t>(__cvta_generic_to_global(src_gmem))), "r"(bytes),
      "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LCE_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra LCE_DONE;\n"
      "bra LCE_WAIT;\n"
      "LCE_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
template <int BYTES>
__device__ __forceinline__ void cp_async_zfill(void* dst_smem, const void* src, int src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2, %3;" ::"r"(smem_u32(dst_smem)),
               "l"(src), "n"(BYTES), "r"(src_bytes)
               : "memory");
}
template <int BYTES>
__device__ __forceinline__ void cp_async_zfill_u32(uint32_t dst_smem, const void* src,
                                                   int src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2, %3;" ::"r"(dst_smem), "l"(src),
               "n"(BYTES), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_cg16(void* dst_smem, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst_smem)), "l"(src),
               "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;" ::: "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.wait_all;" ::: "memory");
}

template <int V> struct VecT;
template <> struct VecT<1> { using T = uint32_t; };
template <> struct VecT<2> { using T = uint2; };
template <> struct VecT<4> { using T = uint4; };

__device__ __forceinline__ int xor_popc(uint32_t a, uint32_t b) { return __popc(a ^ b); }
__device__ __forceinline__ int xor_popc(const uint2& a, const uint2& b) {
  return __popc(a.x ^ b.x) + __popc(a.y ^ b.y);
}
__device__ __forceinline__ int xor_popc(const uint4& a, const uint4& b) {
  return __popc(a.x ^ b.x) + __popc(a.y ^ b.y) + __popc(a.z ^ b.z) + __popc(a.w ^ b.w);
}


template <int V>
__device__ __forceinline__ void load_words(const typename VecT<V>::T* p, uint32_t* dst);
template <>
__device__ __forceinline__ void load_words<1>(const uint32_t* p, uint32_t* dst) { dst[0] = *p; }
template <>
__device__ __forceinline__ void load_words<2>(const uint2* p, uint32_t* dst) {
  const uint2 v = *p;
  dst[0] = v.x; dst[1] = v.y;
}
template <>
__device__ __forceinline__ void load_words<4>(const uint4* p, uint32_t* dst) {
  const uint4 v = *p;
  dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
}

// Carry-save adder on bit-planes: a + b + c = s + 2*cy. Written as two explicit
// LOP3s (xor3 = 0x96, majority = 0xE8) so that exactly 2 ALU-pipe instructions are
// emitted per adder (left to the compiler the expression is re-associated into
// 3-4 LOP3s, and the ALU pipe -- not the POPC pipe -- becomes the limiter).
__device__ __forceinline__ void csa(uint32_t a, uint32_t b, uint32_t c, uint32_t& s,
                                    uint32_t& cy) {
  asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(s) : "r"(a), "r"(b), "r"(c));
  asm("lop3.b32 %0, %1, %2, %3, 0xE8;" : "=r"(cy) : "r"(a), "r"(b), "r"(c));
}
// sum_k popc(a[k] ^ w[k]) over 8 words with 4 POPCs:
//   x0+x1+x2 = s1+2c1, x3+x4+x5 = s2+2c2, s1+s2+x6 = s3+2c3, c1+c2+c3 = s4+2c4
//   => total = popc(s3) + popc(x7) + 2*popc(s4) + 4*popc(c4)      (exact integers)
// 8 XOR + 8 LOP3 on the ALU pipe, 4 POPC on the XU pipe, 1 IADD3 + 2 IMAD to accumulate
// (the multiply-adds run on the FMA pipe, which is otherwise idle here).
__device__ __forceinline__ int xor_popc8_acc(const uint32_t* a, const uint32_t* w, int acc) {
  uint32_t s1, c1, s2, c2, s3, c3, s4, c4;
  csa(a[0] ^ w[0], a[1] ^ w[1], a[2] ^ w[2], s1, c1);
  csa(a[3] ^ w[3], a[4] ^ w[4], a[5] ^ w[5], s2, c2);
  csa(s1, s2, a[6] ^ w[6], s3, c3);
  csa(c1, c2, c3, s4, c4);
  acc += __popc(s3) + __popc(a[7] ^ w[7]);
  int r;
  asm("mad.lo.s32 %0, %1, 2, %2;" : "=r"(r) : "r"(__popc(s4)), "r"(acc));
  asm("mad.lo.s32 %0, %1, 4, %2;" : "=r"(acc) : "r"(__popc(c4)), "r"(r));
  return acc;
}

// OutputTransform<float>::Run, output_transform.h:100-106: shift, int32 clamp,
// int->float, then an UNFUSED multiply and add (two roundings).
__device__ __forceinline__ float transform_float(int acc, int cmin, int cmax, float mul,
                                                 float bias) {
  int x = acc << 1;
  x = max(min(x, cmax), cmin);
  return __fadd_rn(__fmul_rn(static_cast<float>(x), mul), bias);
}
// the same with the doubled accumulator (acc << 1) already formed by the caller
__device__ __forceinline__ float transform_float_x2(int x, int cmin, int cmax, float mul,
                                                    float bias) {
  x = max(min(x, cmax), cmin);
  return __fadd_rn(__fmul_rn(static_cast<float>(x), mul), bias);
}
// core::round (std::round, ties away) + x86 cvttss2si semantics + saturate,
// types.h:50-94, output_transform.h:132-143.
__device__ __forceinline__ int round_saturate_i8(float y) {
  const float r = roundf(y);
  int q = (r >= -2147483648.0f && r < 2147483648.0f) ? static_cast<int>(r) : INT32_MIN;
  return max(-128, min(127, q));
}

// ------------------------------------------------------------------------- //
// K2/K3: binary implicit-GEMM convolution (a plain BGEMM is the 1x1 case).
//   acc[m][n] = sum_k popc(A[m][k] ^ W[n][k]),  k = (tap, channel word)
// One CTA computes a 64-pixel x 64-channel tile; K is staged chunk by chunk:
// weights by one bulk TMA copy from the pre-tiled layout, activation patches by
// zero-filling 4V-byte cp.async (out-of-bounds taps read as 0 bits = +1, the
// reference's one-padding: reference.h:106, optimized_bgemm.h:30-31).
// ------------------------------------------------------------------------- //
// ---- device functions of the implicit-GEMM kernel ----------------

// Decompose output pixel m into (batch image, oy, ox). 32-bit fast division when the pixel
// count allows it (always, in practice); a 64-bit divide otherwise.
__device__ __forceinline__ void split_pixel(const ConvKParams& p, long long m, long long* b,
                                            int* oy, int* ox) {
  uint32_t r;
  if (p.M < (1LL << 31)) {
    const uint32_t bb = fdiv(static_cast<uint32_t>(m), p.fd_ohw);
    r = static_cast<uint32_t>(m) - bb * static_cast<uint32_t>(p.OH * p.OW);
    *b = bb;
  } else {
    const int ohw = p.OH * p.OW;
    *b = m / ohw;
    r = static_cast<uint32_t>(m - *b * ohw);
  }
  const uint32_t y = fdiv(r, p.fd_ow);
  *oy = static_cast<int>(y);
  *ox = static_cast<int>(r - y * static_cast<uint32_t>(p.OW));
}

// Gather one K chunk of the im2col rows of tile `m0` into A_buf[kv - kv0][pixel] with
// zero-filling cp.async. Thread t handles pixel t % BM and every second k-vector.
// kSliceRows: the layout is A_buf[k-slice][pixel][8 words] instead (k = (kv - kv0) * V words into
// the chunk), and vectors at kv >= p.Kv -- the K tail padding -- are zero-filled.
// `in` (optional) replaces p.in as the packed input: one of several input planes.
template <int V, int BM_ = kBM, int NT_ = kThreads, bool kSliceRows = false>
__device__ __forceinline__ void gather_tile(const ConvKParams& p, typename VecT<V>::T* A_buf,
                                            long long m0, int g, int kv0, int kv1, int tid,
                                            const int32_t* in = nullptr) {
  using Vec = typename VecT<V>::T;
  constexpr int kStep = NT_ / BM_;  // threads per pixel: each takes every kStep-th k-vector
  const int lp = tid & (BM_ - 1);
  const int half = tid / BM_;
  const long long gm = m0 + lp;
  const bool pix_valid = gm < p.M;
  int iy0 = 0, ix0 = 0;
  const int32_t* src_in = in != nullptr ? in : p.in;
  const int32_t* img = src_in;
  if (pix_valid) {
    long long b;
    int oy, ox;
    split_pixel(p, gm, &b, &oy, &ox);
    iy0 = oy * p.sh - p.ph;
    ix0 = ox * p.sw - p.pw;
    img = src_in + b * p.img_words + g * p.Cw_pg;
  }
  int kv = kv0 + half;
  int tap = static_cast<int>(fdiv(static_cast<uint32_t>(kv), p.fd_cwv));
  int cv = kv - tap * p.CwV;
  int fy = static_cast<int>(fdiv(static_cast<uint32_t>(tap), p.fd_kw));
  int fx = tap - fy * p.KW;
  uint32_t dst = smem_u32(A_buf + half * BM_ + lp);
  for (; kv < kv1; kv += kStep, dst += kStep * BM_ * static_cast<uint32_t>(sizeof(Vec))) {
    const int iy = iy0 + fy * p.dh;
    const int ix = ix0 + fx * p.dw;
    const bool inside = pix_valid && (!kSliceRows || kv < p.Kv) &&
                        static_cast<unsigned>(iy) < static_cast<unsigned>(p.H) &&
                        static_cast<unsigned>(ix) < static_cast<unsigned>(p.W);
    // offsets inside one image fit 32 bits (img_words < 2^31)
    const int off = (iy * p.W + ix) * p.Cw_total + cv * V;
    const int32_t* src = inside ? img + off : src_in;
    uint32_t d = dst;
    if constexpr (kSliceRows) {
      const uint32_t k = static_cast<uint32_t>(kv - kv0) * V;
      d = smem_u32(A_buf) + (k >> 3) * (BM_ * 32) + lp * 32 + (k & 7) * 4;
    }
    cp_async_zfill_u32<V * 4>(d, src, inside ? V * 4 : 0);
    cv += kStep;
    while (cv >= p.CwV) {
      cv -= p.CwV;
      if (++fx == p.KW) {
        fx = 0;
        ++fy;
      }
    }
  }
}

template <int V>
__device__ __forceinline__ void compute_chunk(const typename VecT<V>::T* A_s,
                                              const typename VecT<V>::T* W_s, int nkv, int warp,
                                              int tm, int tn, int (&acc)[kTM][kTN]) {
  using Vec = typename VecT<V>::T;
    const Vec* a_ptr = A_s + warp * 16 + tm;
    const Vec* w_ptr = W_s + tn;
    // Main loop: 8 K-words at a time through a carry-save adder tree, so that 8
    // XOR words cost 4 POPCs (XU pipe, 16/clk/SM) + 16 LOP3s (ALU pipe, 64/clk/SM)
    // instead of 8 POPCs -- the two pipes issue side by side.
    constexpr int G = 8 / V;  // smem vectors per 8-word group
    int kv = 0;
#ifdef LCE_HALF_TILE
    // two pixels at a time: 16 instead of 32 live activation registers (the weight words are
    // re-read from shared memory for the second half), so more CTAs fit per SM
    for (; kv + G <= nkv; kv += G) {
#pragma unroll
      for (int h = 0; h < kTM / 2; ++h) {
        uint32_t a[2][8];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int gq = 0; gq < G; ++gq)
            load_words<V>(a_ptr + (kv + gq) * kBM + (h * 2 + i) * 4, &a[i][gq * V]);
#pragma unroll
        for (int j = 0; j < kTN; ++j) {
          uint32_t w[8];
#pragma unroll
          for (int gq = 0; gq < G; ++gq) load_words<V>(w_ptr + (kv + gq) * kBN + j * 8, &w[gq * V]);
#pragma unroll
          for (int i = 0; i < 2; ++i) acc[h * 2 + i][j] = xor_popc8_acc(a[i], w, acc[h * 2 + i][j]);
        }
        asm volatile("" ::: "memory");
      }
    }
#else
    for (; kv + G <= nkv; kv += G) {
      uint32_t a[kTM][8];
#pragma unroll
      for (int i = 0; i < kTM; ++i)
#pragma unroll
        for (int gq = 0; gq < G; ++gq) load_words<V>(a_ptr + (kv + gq) * kBM + i * 4, &a[i][gq * V]);
#pragma unroll
      for (int j = 0; j < kTN; ++j) {
        uint32_t w[8];
#pragma unroll
        for (int gq = 0; gq < G; ++gq) load_words<V>(w_ptr + (kv + gq) * kBN + j * 8, &w[gq * V]);
#pragma unroll
        for (int i = 0; i < kTM; ++i) acc[i][j] = xor_popc8_acc(a[i], w, acc[i][j]);
      }
    }
#endif
    for (; kv < nkv; ++kv) {  // K tail (< 8 words): plain XOR + POPC
      Vec a[kTM], w[kTN];
#pragma unroll
      for (int i = 0; i < kTM; ++i) a[i] = a_ptr[kv * kBM + i * 4];
#pragma unroll
      for (int j = 0; j < kTN; ++j) w[j] = w_ptr[kv * kBN + j * 8];
#pragma unroll
      for (int i = 0; i < kTM; ++i)
#pragma unroll
        for (int j = 0; j < kTN; ++j) acc[i][j] += xor_popc(a[i], w[j]);
    }
}

// SAME padding with pad value 0, in integers as the reference kernel does it
// (reference.h:76-77,100-103): an out-of-bounds tap contributes channels_in_per_group/2
// instead of popc(0 ^ w). Applied to the accumulators before the output transform.
__device__ __forceinline__ void zero_pad_correction(const ConvKParams& p, int (&acc)[kTM][kTN],
                                                    long long m0, int warp, int tm, int c0) {
  const int taps = p.KH * p.KW;
#pragma unroll
  for (int i = 0; i < kTM; ++i) {
    const long long m = m0 + warp * 16 + i * 4 + tm;
    if (m >= p.M) continue;
    long long b;
    int oy, ox;
    split_pixel(p, m, &b, &oy, &ox);
    // interior pixels (the vast majority) have no out-of-bounds tap
    const int iy_lo = oy * p.sh - p.ph, ix_lo = ox * p.sw - p.pw;
    if (iy_lo >= 0 && ix_lo >= 0 && iy_lo + (p.KH - 1) * p.dh < p.H &&
        ix_lo + (p.KW - 1) * p.dw < p.W)
      continue;
    for (int fy = 0; fy < p.KH; ++fy) {
      const int iy = iy_lo + fy * p.dh;
      const bool yin = static_cast<unsigned>(iy) < static_cast<unsigned>(p.H);
      for (int fx = 0; fx < p.KW; ++fx) {
        const int ix = ix_lo + fx * p.dw;
        if (yin && static_cast<unsigned>(ix) < static_cast<unsigned>(p.W)) continue;
        const int t = fy * p.KW + fx;
#pragma unroll
        for (int j = 0; j < kTN; ++j)
          acc[i][j] += p.zp_half - p.tap_popc[static_cast<size_t>(c0 + j) * taps + t];
      }
    }
  }
}

// Straight-line epilogues for the common case: the tile lies fully inside M and the group's
// channels, rows are 16-byte aligned. No per-element predicates, row pointers advance by a
// constant. `res_s`: this thread's staged shortcut values (or nullptr -> global loads).
__device__ __forceinline__ void epilogue_float_fast(const ConvKParams& p, int (&acc)[kTM][kTN],
                                                    long long m0, int c_tile, int warp, int tm,
                                                    int tn, const float* mulp, const float* biasp,
                                                    const float4* res_s) {
  const float4 mu0 = reinterpret_cast<const float4*>(mulp)[0];
  const float4 mu1 = reinterpret_cast<const float4*>(mulp)[1];
  const float4 bi0 = reinterpret_cast<const float4*>(biasp)[0];
  const float4 bi1 = reinterpret_cast<const float4*>(biasp)[1];
  const float mul_r[kTN] = {mu0.x, mu0.y, mu0.z, mu0.w, mu1.x, mu1.y, mu1.z, mu1.w};
  const float bias_r[kTN] = {bi0.x, bi0.y, bi0.z, bi0.w, bi1.x, bi1.y, bi1.z, bi1.w};
  const long long mrow = m0 + warp * 16 + tm;
  const size_t e0 = static_cast<size_t>(mrow) * p.cout + c_tile + tn * 8;
  const size_t estep = static_cast<size_t>(4) * p.cout;
  float* o = static_cast<float*>(p.out) + e0;
  const float* r = p.residual + e0;  // only dereferenced when residual != nullptr
  int32_t* pk = p.packed_out + static_cast<size_t>(mrow) * p.cw_out + (c_tile >> 5) + (tn >> 2);
  const bool has_res = p.residual != nullptr;
  const bool has_pk = p.packed_out != nullptr;
  const int ract = p.residual_act;
#pragma unroll
  for (int i = 0; i < kTM; ++i) {
    float y[kTN];
#pragma unroll
    for (int j = 0; j < kTN; ++j)
      y[j] = transform_float(acc[i][j], p.clamp_min, p.clamp_max, mul_r[j], bias_r[j]);
    if (has_res) {
      const float4 r0 = res_s ? res_s[(i * 2) * kThreads] : reinterpret_cast<const float4*>(r)[0];
      const float4 r1 =
          res_s ? res_s[(i * 2 + 1) * kThreads] : reinterpret_cast<const float4*>(r)[1];
      y[0] = __fadd_rn(y[0], r0.x); y[1] = __fadd_rn(y[1], r0.y);
      y[2] = __fadd_rn(y[2], r0.z); y[3] = __fadd_rn(y[3], r0.w);
      y[4] = __fadd_rn(y[4], r1.x); y[5] = __fadd_rn(y[5], r1.y);
      y[6] = __fadd_rn(y[6], r1.z); y[7] = __fadd_rn(y[7], r1.w);
      if (ract == LCE_ACT_RELU) {
#pragma unroll
        for (int j = 0; j < kTN; ++j) y[j] = fmaxf(y[j], 0.0f);
      } else if (ract == LCE_ACT_RELU6) {
#pragma unroll
        for (int j = 0; j < kTN; ++j) y[j] = fminf(fmaxf(y[j], 0.0f), 6.0f);
      } else if (ract == LCE_ACT_RELU_N1_TO_1) {
#pragma unroll
        for (int j = 0; j < kTN; ++j) y[j] = fminf(fmaxf(y[j], -1.0f), 1.0f);
      }
    }
    reinterpret_cast<float4*>(o)[0] = make_float4(y[0], y[1], y[2], y[3]);
    reinterpret_cast<float4*>(o)[1] = make_float4(y[4], y[5], y[6], y[7]);
    if (has_pk) {
      // LceQuantize of the value just written: bit = value < 0 (bitpack.h:159)
      uint32_t bits = 0;
#pragma unroll
      for (int j = 0; j < kTN; ++j) bits |= (y[j] < 0.0f) ? (1u << j) : 0u;
      uint32_t v = bits << (8 * (tn & 3));
      v |= __shfl_xor_sync(0xffffffffu, v, 1);
      v |= __shfl_xor_sync(0xffffffffu, v, 2);
      if ((tn & 3) == 0) *pk = static_cast<int32_t>(v);
      pk += static_cast<size_t>(4) * p.cw_out;
    }
    o += estep;
    r += estep;
  }
}

__device__ __forceinline__ void epilogue_raw_fast(const ConvKParams& p, int (&acc)[kTM][kTN],
                                                  long long m0, int c_tile, int warp, int tm,
                                                  int tn) {
  int* o = static_cast<int*>(p.out) +
           static_cast<size_t>(m0 + warp * 16 + tm) * p.cout + c_tile + tn * 8;
  const size_t estep = static_cast<size_t>(4) * p.cout;
#pragma unroll
  for (int i = 0; i < kTM; ++i) {
    reinterpret_cast<int4*>(o)[0] = make_int4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    reinterpret_cast<int4*>(o)[1] = make_int4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
    o += estep;
  }
}

// Position j*8+tn of the weight tile holds channel tn*8+j, so each thread owns 8 CONSECUTIVE
// output channels and stores them with 128-bit writes. mulp / biasp / thrp point at this
// thread's first channel.
template <int OUT>
__device__ __forceinline__ void epilogue_tile(const ConvKParams& p, int (&acc)[kTM][kTN],
                                              long long m0, int g, int tg, int warp, int tm,
                                              int tn, const float* mulp, const float* biasp,
                                              const int32_t* thrp,
                                              const float4* res_s = nullptr) {
  const int c_tile = g * p.cout_pg + tg * kBN;
  const int valid = min(kBN, p.cout_pg - tg * kBN);
  const int cofs = tn * 8;
  const int c0 = c_tile + cofs;
  if (p.tap_popc != nullptr) zero_pad_correction(p, acc, m0, warp, tm, c0);
  if (cofs + kTN <= valid && p.vec_store && m0 + kBM <= p.M) {
    if (OUT == LCE_OUT_FLOAT) {
      epilogue_float_fast(p, acc, m0, c_tile, warp, tm, tn, mulp, biasp, res_s);
      return;
    }
    if (OUT == LCE_OUT_RAW_ACC) {
      epilogue_raw_fast(p, acc, m0, c_tile, warp, tm, tn);
      return;
    }
  }
  float mul_r[kTN], bias_r[kTN];
  int thr_r[kTN];
  if (OUT == LCE_OUT_FLOAT || OUT == LCE_OUT_INT8) {
#pragma unroll
    for (int j = 0; j < kTN; ++j) {
      mul_r[j] = mulp[j];
      bias_r[j] = biasp[j];
    }
  } else if (OUT == LCE_OUT_BITPACKED) {
#pragma unroll
    for (int j = 0; j < kTN; ++j) thr_r[j] = thrp[j];
  }
  const bool full = cofs + kTN <= valid;

#pragma unroll
  for (int i = 0; i < kTM; ++i) {
    const long long m = m0 + warp * 16 + i * 4 + tm;
    const bool row_ok = m < p.M;

    if (OUT == LCE_OUT_RAW_ACC) {
      if (!row_ok) continue;
      int* o = static_cast<int*>(p.out) + m * p.cout + c0;
      if (full && p.vec_store) {
        reinterpret_cast<int4*>(o)[0] = make_int4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
        reinterpret_cast<int4*>(o)[1] = make_int4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
      } else {
#pragma unroll
        for (int j = 0; j < kTN; ++j)
          if (cofs + j < valid) o[j] = acc[i][j];
      }
    } else if (OUT == LCE_OUT_FLOAT) {
      float y[kTN];
#pragma unroll
      for (int j = 0; j < kTN; ++j)
        y[j] = transform_float(acc[i][j], p.clamp_min, p.clamp_max, mul_r[j], bias_r[j]);
      float* o = static_cast<float*>(p.out) + m * p.cout + c0;
      if (p.residual != nullptr && row_ok) {
        const float* r = p.residual + m * p.cout + c0;
        if (res_s != nullptr || (full && p.vec_store)) {
          const float4 r0 = res_s ? res_s[(i * 2) * kThreads] : reinterpret_cast<const float4*>(r)[0];
          const float4 r1 =
              res_s ? res_s[(i * 2 + 1) * kThreads] : reinterpret_cast<const float4*>(r)[1];
          y[0] = __fadd_rn(y[0], r0.x); y[1] = __fadd_rn(y[1], r0.y);
          y[2] = __fadd_rn(y[2], r0.z); y[3] = __fadd_rn(y[3], r0.w);
          y[4] = __fadd_rn(y[4], r1.x); y[5] = __fadd_rn(y[5], r1.y);
          y[6] = __fadd_rn(y[6], r1.z); y[7] = __fadd_rn(y[7], r1.w);
        } else {
#pragma unroll
          for (int j = 0; j < kTN; ++j)
            if (cofs + j < valid) y[j] = __fadd_rn(y[j], r[j]);
        }
        if (p.residual_act != LCE_ACT_NONE) {
#pragma unroll
          for (int j = 0; j < kTN; ++j) {
            if (p.residual_act == LCE_ACT_RELU) y[j] = fmaxf(y[j], 0.0f);
            else if (p.residual_act == LCE_ACT_RELU6) y[j] = fminf(fmaxf(y[j], 0.0f), 6.0f);
            else y[j] = fminf(fmaxf(y[j], -1.0f), 1.0f);
          }
        }
      }
      if (row_ok) {
        if (full && p.vec_store) {
          reinterpret_cast<float4*>(o)[0] = make_float4(y[0], y[1], y[2], y[3]);
          reinterpret_cast<float4*>(o)[1] = make_float4(y[4], y[5], y[6], y[7]);
        } else {
#pragma unroll
          for (int j = 0; j < kTN; ++j)
            if (cofs + j < valid) o[j] = y[j];
        }
      }
      if (p.packed_out != nullptr) {
        // LceQuantize of the value just written: bit = value < 0 (bitpack.h:159); the
        // four lanes holding one word's bytes combine with two shuffles (all lanes run them).
        uint32_t bits = 0;
#pragma unroll
        for (int j = 0; j < kTN; ++j)
          if (cofs + j < valid && y[j] < 0.0f) bits |= 1u << j;
        uint32_t v = bits << (8 * (tn & 3));
        v |= __shfl_xor_sync(0xffffffffu, v, 1);
        v |= __shfl_xor_sync(0xffffffffu, v, 2);
        const int q = tn >> 2;
        if (row_ok && (tn & 3) == 0 && q * 32 < valid)
          p.packed_out[m * p.cw_out + (c_tile >> 5) + q] = static_cast<int32_t>(v);
      }
    } else if (OUT == LCE_OUT_INT8) {
      if (!row_ok) continue;
      int q[kTN];
#pragma unroll
      for (int j = 0; j < kTN; ++j)
        q[j] = round_saturate_i8(
            transform_float(acc[i][j], p.clamp_min, p.clamp_max, mul_r[j], bias_r[j]));
      int8_t* o = static_cast<int8_t*>(p.out) + m * p.cout + c0;
      if (full && p.vec_store) {
        uint2 v;
        v.x = (q[0] & 0xFF) | ((q[1] & 0xFF) << 8) | ((q[2] & 0xFF) << 16) |
              (static_cast<uint32_t>(q[3] & 0xFF) << 24);
        v.y = (q[4] & 0xFF) | ((q[5] & 0xFF) << 8) | ((q[6] & 0xFF) << 16) |
              (static_cast<uint32_t>(q[7] & 0xFF) << 24);
        *reinterpret_cast<uint2*>(o) = v;
      } else {
#pragma unroll
        for (int j = 0; j < kTN; ++j)
          if (cofs + j < valid) o[j] = static_cast<int8_t>(q[j]);
      }
    } else {  // LCE_OUT_BITPACKED: bit = acc > threshold (output_transform.h:164-167)
      uint32_t bits = 0;
#pragma unroll
      for (int j = 0; j < kTN; ++j)
        if (cofs + j < valid && acc[i][j] > thr_r[j]) bits |= 1u << j;
      if (p.bp_fast) {
        // four neighbouring lanes hold the four bytes of one output word
        uint32_t v = bits << (8 * (tn & 3));
        v |= __shfl_xor_sync(0xffffffffu, v, 1);
        v |= __shfl_xor_sync(0xffffffffu, v, 2);
        const int q = tn >> 2;
        if (row_ok && (tn & 3) == 0 && q * 32 < valid)
          static_cast<int32_t*>(p.out)[m * p.cw_out + (c_tile >> 5) + q] =
              static_cast<int32_t>(v);
      } else if (row_ok && bits) {
        // groups whose channel count is not a multiple of 32: words are shared
        // between tiles; the host zero-fills the output first.
#pragma unroll
        for (int j = 0; j < kTN; ++j)
          if (bits & (1u << j)) {
            const int c = c0 + j;
            atomicOr(reinterpret_cast<unsigned int*>(p.out) + m * p.cw_out + (c >> 5),
                     1u << (c & 31));
          }
      }
    }
  }
}

// ------------------------------------------------------------------------- //
// One CTA = one 64 x 64 tile, K staged chunk by chunk (any K).
// ------------------------------------------------------------------------- //
template <int V, int OUT>
__global__ void __launch_bounds__(kThreads, kCtasPerSm) bconv_kernel(const ConvKParams p) {
  using Vec = typename VecT<V>::T;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  Vec* A_s = reinterpret_cast<Vec*>(smem_raw);     // [Kc_v][BM]
  Vec* W_s = A_s + static_cast<size_t>(p.Kc_v) * kBM;  // [Kc_v][BN]
  __shared__ __align__(8) uint64_t wbar;

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int tn = lane & 7, tm = lane >> 3;
  const int nt = blockIdx.y;
  const int g = static_cast<int>(fdiv(static_cast<uint32_t>(nt), p.fd_tpg));
  const int tg = nt - g * p.tiles_per_group;
  const long long m0 = static_cast<long long>(blockIdx.x) * kBM;

  if (tid == 0) {
    mbar_init(&wbar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  int acc[kTM][kTN];
#pragma unroll
  for (int i = 0; i < kTM; ++i)
#pragma unroll
    for (int j = 0; j < kTN; ++j) acc[i][j] = 0;

  // Fused shortcut: start pulling this thread's residual values towards L2 now, so the
  // DRAM latency of the epilogue's loads is covered by the gather + inner product.
  float4* R_s = nullptr;
  if (OUT == LCE_OUT_FLOAT && p.res_stage)
    R_s = reinterpret_cast<float4*>(W_s + static_cast<size_t>(p.Kc_v) * kBN) + tid;
  if (OUT == LCE_OUT_FLOAT && p.residual != nullptr && !p.res_stage) {
#pragma unroll
    for (int i = 0; i < kTM; ++i) {
      const long long m = m0 + warp * 16 + i * 4 + tm;
      if (m < p.M)
        asm volatile("prefetch.global.L2 [%0];" ::"l"(p.residual + m * p.cout + g * p.cout_pg +
                                                       tg * kBN + tn * 8));
    }
  }

  uint32_t phase = 0;
  for (int ch = 0; ch < p.n_chunks; ++ch) {
    const int kv0 = ch * p.Kc_v;
    const int kv1 = min(kv0 + p.Kc_v, p.Kv);
    if (tid == 0) {
      const uint32_t bytes = static_cast<uint32_t>(kv1 - kv0) * kBN * V * 4u;
      mbar_arrive_expect_tx(&wbar, bytes);
      bulk_g2s(W_s, p.wt + (static_cast<size_t>(nt) * p.Kv + kv0) * kBN * V, bytes, &wbar);
    }
    gather_tile<V>(p, A_s, m0, g, kv0, kv1, tid);
    if (OUT == LCE_OUT_FLOAT && p.res_stage && ch == 0) {
      // second cp.async group: the residual rows; only the gather group is waited for here
      cp_async_commit();
#pragma unroll
      for (int i = 0; i < kTM; ++i) {
        const long long m = m0 + warp * 16 + i * 4 + tm;
        const bool ok = m < p.M;
        const float* r = ok ? p.residual + m * p.cout + g * p.cout_pg + tg * kBN + tn * 8
                            : p.residual;
        cp_async_cg16(R_s + (i * 2) * kThreads, r, ok ? 16 : 0);
        cp_async_cg16(R_s + (i * 2 + 1) * kThreads, r + 4, ok ? 16 : 0);
      }
      cp_async_commit();
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      cp_async_wait_all();
    }
    mbar_wait(&wbar, phase);
    phase ^= 1u;
    __syncthreads();
    compute_chunk<V>(A_s, W_s, kv1 - kv0, warp, tm, tn, acc);
    __syncthreads();
  }
  const int c0 = g * p.cout_pg + tg * kBN + tn * 8;
  if (OUT == LCE_OUT_FLOAT && p.res_stage) cp_async_wait_all();  // own slots only: no barrier
  epilogue_tile<OUT>(p, acc, m0, g, tg, warp, tm, tn, p.mul + c0, p.bias + c0, p.thr + c0, R_s);
}

// Re-lay the OHWI-packed filter [cout][taps][Cw_pg] into the kernel's tiles:
// wt[n_tile][kv][pos][V], pos = j*8+tn <-> channel tn*8+j of the tile, zero for
// channels past the group's end. Runs once per plan ("weights are static").
__global__ void tile_weights_kernel(const int32_t* __restrict__ filter, int32_t* __restrict__ wt,
                                    int cout_pg, int tiles_per_group, int taps, int Cw_pg, int V,
                                    int Kv, long long total, int natural_order) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= total) return;
  const int v = static_cast<int>(idx % V);
  long long r = idx / V;
  const int pos = static_cast<int>(r % kBN);
  r /= kBN;
  const int kv = static_cast<int>(r % Kv);
  const int nt = static_cast<int>(r / Kv);
  const int g = nt / tiles_per_group, tg = nt - g * tiles_per_group;
  const int ch = tg * kBN + (natural_order ? pos : (pos & 7) * 8 + (pos >> 3));
  int32_t val = 0;
  if (ch < cout_pg) {
    const int CwV = Cw_pg / V;
    const int tap = kv / CwV, cv = kv - tap * CwV;
    const long long c = static_cast<long long>(g) * cout_pg + ch;
    val = filter[(c * taps + tap) * Cw_pg + cv * V + v];
  }
  wt[idx] = val;
}

// tap_popc[c][t] = sum over the packed channel words of popc(filter[c][t][:]).
__global__ void tap_popc_kernel(const int32_t* __restrict__ filter, int32_t* __restrict__ out,
                                int cout, int taps, int Cw_pg) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= cout * taps) return;
  const int32_t* f = filter + static_cast<size_t>(idx) * Cw_pg;
  int s = 0;
  for (int w = 0; w < Cw_pg; ++w) s += __popc(static_cast<uint32_t>(f[w]));
  out[idx] = s;
}

// ------------------------------------------------------------------------- //
// Zero padding with the optimised reference kernels' float correction, for the plans that do not
// run on the wgmma kernel (which has it in its epilogue): the convolution ran with one-padding
// and no fused tail; this pass adds the correction to the edge pixels
// (zero_padding_correction.h:178-299, the case analysis restated literally), then the fused ADD /
// activation / sign-pack tail if there is one. One warp per (pixel, 32 channels).
// ------------------------------------------------------------------------- //
struct ZpcTailParams {
  float* out;
  const float* src;          // the convolution's uncorrected output: out, or (with a residual) a
                             // separate buffer
  const float* mul;          // folded multiplier = -post_activation_multiplier
  const int32_t* tap_popc;   // [cout][taps]
  const float* residual;     // pixel m at residual + m * out_stride; may be out itself
  int32_t* packed_out;
  long long M;
  long long out_stride;      // floats from one output pixel to the next (cout unless strided)
  long long src_stride;      // the same for src
  int H, W, OH, OW, KH, KW, sh, sw, dh, dw;
  int cout, cin_pg, cw_out, residual_act;
};
__global__ void __launch_bounds__(256) zpc_tail_kernel(const ZpcTailParams p) {
  const int lane = threadIdx.x & 31;
  const int cw = (p.cout + 31) >> 5;
  const long long n_warps = p.M * cw;
  const long long stride = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const int eff_w = (p.KW - 1) * p.dw + 1, eff_h = (p.KH - 1) * p.dh + 1;
  const int left_off = ((p.OW - 1) * p.sw + eff_w - p.W) / 2;
  const int top_off = ((p.OH - 1) * p.sh + eff_h - p.H) / 2;
  const int taps = p.KH * p.KW;
  for (long long w = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5; w < n_warps; w += stride) {
    const long long m = w / cw;
    const int c = static_cast<int>(w - m * cw) * 32 + lane;
    const long long r = m % (static_cast<long long>(p.OH) * p.OW);
    const int oy = static_cast<int>(r / p.OW), ox = static_cast<int>(r % p.OW);
    const int o_top = top_off - oy * p.sh, o_bot = -o_top - p.H + eff_h;
    const int o_left = left_off - ox * p.sw, o_right = -o_left - p.W + eff_w;
    int cs = -1, X = 0, Y = 0;
    if (!(o_left <= 0 && o_right <= 0 && o_top <= 0 && o_bot <= 0)) {
      if (o_right <= 0 && o_top > 0 && o_bot < 0) { cs = 0; X = max(o_left, 0); Y = o_top; }
      else if (o_left < 0 && o_right > 0 && o_bot <= 0) { cs = 1; X = o_right; Y = max(o_top, 0); }
      else if (o_left > 0 && o_right < 0 && o_top <= 0) { cs = 2; X = o_left; Y = max(o_bot, 0); }
      else if (o_left <= 0 && o_top < 0 && o_bot > 0) { cs = 3; X = max(o_right, 0); Y = o_bot; }
    }
    if (cs < 0 && p.residual == nullptr && p.packed_out == nullptr) continue;   // interior, nothing fused
    float y = 0.0f;
    const bool ok = c < p.cout;
    if (ok) {
      y = p.src[m * p.src_stride + c];
      if (cs >= 0) {
        int corr = 0;
        for (int fy = 0; fy < p.KH; ++fy)
          for (int fx = 0; fx < p.KW; ++fx) {
            const int efx = p.dw * fx, efy = p.dh * fy;
            bool counted;
            if (cs == 0) counted = efy < Y || efx < X;
            else if (cs == 1) counted = efy < Y || (eff_w - efx) <= X;
            else if (cs == 2) counted = (eff_h - efy) <= Y || efx < X;
            else counted = (eff_h - efy) <= Y || (eff_w - efx) <= X;
            if (counted) corr += p.cin_pg - 2 * p.tap_popc[static_cast<size_t>(c) * taps + fy * p.KW + fx];
          }
        y = __fadd_rn(y, __fmul_rn(p.mul[c], static_cast<float>(corr)));
      }
      if (p.residual != nullptr) {
        y = __fadd_rn(y, p.residual[m * p.out_stride + c]);
        if (p.residual_act == LCE_ACT_RELU) y = fmaxf(y, 0.0f);
        else if (p.residual_act == LCE_ACT_RELU6) y = fminf(fmaxf(y, 0.0f), 6.0f);
        else if (p.residual_act == LCE_ACT_RELU_N1_TO_1) y = fminf(fmaxf(y, -1.0f), 1.0f);
      }
      p.out[m * p.out_stride + c] = y;
    }
    if (p.packed_out != nullptr) {
      const uint32_t word = __ballot_sync(0xffffffffu, ok && y < 0.0f);
      if (lane == 0) p.packed_out[m * p.cw_out + (c >> 5)] = static_cast<int32_t>(word);
    }
  }
}

// ------------------------------------------------------------------------- //
// K1: bsign_pack (LceQuantize). bit = value < zero_point (float: value < 0, so
// -0.0 and NaN pack as 0 and negative denormals as 1: compiled WITHOUT -ftz).
// Fast path (cols % 32 == 0, float): the tensor is one flat array; each thread
// converts 8 consecutive floats (two 128-bit loads) into one byte, four lanes
// assemble a word with two shuffles. HBM-bound: 4 B read + 1/8 B written / elem.
// ------------------------------------------------------------------------- //
__device__ __forceinline__ uint32_t sign_nibble(const float4& f) {
  return (f.x < 0.0f ? 1u : 0u) | (f.y < 0.0f ? 2u : 0u) | (f.z < 0.0f ? 4u : 0u) |
         (f.w < 0.0f ? 8u : 0u);
}

__global__ void __launch_bounds__(256) pack_f32_flat_kernel(const float4* __restrict__ in,
                                                            int32_t* __restrict__ out,
                                                            long long n_words) {
  // thread t handles floats [8t, 8t+8): lanes 4q..4q+3 form word q of the warp.
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long n_threads_needed = n_words * 4;
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
       t - (threadIdx.x & 31) < n_threads_needed; t += stride) {
    uint32_t byte = 0;
    if (t < n_threads_needed) {
      const float4 a = __ldcs(in + 2 * t);
      const float4 b = __ldcs(in + 2 * t + 1);
      byte = sign_nibble(a) | (sign_nibble(b) << 4);
    }
    uint32_t v = byte << (8 * (threadIdx.x & 3));
    v |= __shfl_xor_sync(0xffffffffu, v, 1);
    v |= __shfl_xor_sync(0xffffffffu, v, 2);
    if ((threadIdx.x & 3) == 0 && t < n_threads_needed) out[t >> 2] = static_cast<int32_t>(v);
  }
}

// General path: one warp per output word, lane i tests element 32w+i (ballot);
// elements past `cols` behave as zero_point (bit 0): bitpack.h:238-244.
template <typename T>
__device__ __forceinline__ bool below_zero_point(T x, int zp);
template <>
__device__ __forceinline__ bool below_zero_point<float>(float x, int) { return x < 0.0f; }
template <>
__device__ __forceinline__ bool below_zero_point<int8_t>(int8_t x, int zp) {
  return static_cast<int>(x) < zp;  // int32 compare: covers bitpack.h:259-288
}
template <>
__device__ __forceinline__ bool below_zero_point<uint8_t>(uint8_t x, int zp) {
  return static_cast<int>(x) < zp;  // bool viewed as uint8, zp = 1 (quantization.cc:88-108)
}

template <typename T>
__global__ void __launch_bounds__(256) pack_generic_kernel(const T* __restrict__ in,
                                                           int32_t* __restrict__ out,
                                                           long long rows, int cols, int cw,
                                                           int zero_point) {
  const long long n_words = rows * cw;
  const int lane = threadIdx.x & 31;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  for (long long w = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
       w < n_words; w += warps) {
    const long long r = w / cw;
    const int c = static_cast<int>(w - r * cw) * 32 + lane;
    bool bit = false;
    if (c < cols) bit = below_zero_point<T>(in[r * cols + c], zero_point);
    const uint32_t word = __ballot_sync(0xffffffffu, bit);
    if (lane == 0) out[w] = static_cast<int32_t>(word);
  }
}

// ------------------------------------------------------------------------- //
// K5: unpack (LceDequantize): bit 0 -> zero_bit_value, bit 1 -> one_bit_value.
// ------------------------------------------------------------------------- //
template <typename T>
__global__ void __launch_bounds__(256) unpack_kernel(const int32_t* __restrict__ in,
                                                     T* __restrict__ out, long long rows,
                                                     int cols, int cw, T zero_bit, T one_bit) {
  const long long n = rows * cols;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += stride) {
    const long long r = i / cols;
    const int c = static_cast<int>(i - r * cols);
    const uint32_t word = static_cast<uint32_t>(in[r * cw + (c >> 5)]);
    out[i] = ((word >> (c & 31)) & 1u) ? one_bit : zero_bit;
  }
}

// ------------------------------------------------------------------------- //
// K4: bmaxpool: AND over the in-bounds part of the window (bmaxpool.h:45-84).
// One thread per output word; the channel word is the fastest index (coalesced).
// ------------------------------------------------------------------------- //
__global__ void __launch_bounds__(256) bmaxpool_kernel(const int32_t* __restrict__ in,
                                                       int32_t* __restrict__ out, int B, int H,
                                                       int W, int C, int OH, int OW, int fh,
                                                       int fw, int sh, int sw, int ph, int pw) {
  const long long n = static_cast<long long>(B) * OH * OW * C;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += stride) {
    const int c = static_cast<int>(i % C);
    long long r = i / C;
    const int ox = static_cast<int>(r % OW);
    r /= OW;
    const int oy = static_cast<int>(r % OH);
    const int b = static_cast<int>(r / OH);
    const int y0 = oy * sh - ph, x0 = ox * sw - pw;
    const int ys = max(0, y0), ye = min(H, y0 + fh);
    const int xs = max(0, x0), xe = min(W, x0 + fw);
    int32_t m = ~0;
    for (int y = ys; y < ye; ++y)
      for (int x = xs; x < xe; ++x)
        m &= in[((static_cast<long long>(b) * H + y) * W + x) * C + c];
    out[i] = m;
  }
}

}  // namespace lce

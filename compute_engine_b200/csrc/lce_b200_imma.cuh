// lce_b200_imma.cuh -- the binary convolution's inner product on the mma.sync tensor pipe.
// The default for every plan with full 64-channel tiles and float, bitpacked or raw-accumulator
// output (the model families' LceBconv2d layers, the BGEMM sweep): on H100 it runs the QuickNet
// graph faster than the wgmma kernel of lce_b200_tc.cuh, which takes the other plans it is
// eligible for; the rest, and every plan when LCE_B200_BCONV_IMMA=0 and ..._TC=0, run the XOR + POPC
// kernel of lce_b200_kernels.cuh. All produce the reference's integers bit for bit
// (tests/test_gpu_parity.py runs the same cases through each); bench.py reports them side by side.
//
// Two inner products share the kernel's gather, TMA weight staging, zero-padding correction and
// epilogue (template parameter B1):
//  - b1 (default): the native binary instruction, mma.sync m16n8k256 b1 and.popc (SASS
//    BMMA.168256.AND.POPC; .xor.popc is lowered to two of them). Operands stay packed, so the
//    weights cost 256 B per K word per 64-channel tile in L2 and shared memory instead of 2048 B,
//    and one BMMA does the work of 8 IMMA.16832. Measured on an H100 80GB HBM3 at a 400 W power
//    limit (tools/microbench_mma.cu): 19.9 k binary MACs / clk / SM against IMMA's 2.5 k int8
//    MACs / clk / SM. See compute_chunk_b1 for the identity and fragment layout.
//  - int8 (LCE_B200_BCONV_B1=0), described below, kept for A/B runs.
//
// The int8 tensor pipe (mma.sync.m16n8k32, SASS IMMA.16832) does the XOR + POPC sum as a signed
// dot product. HBM, L2 and shared memory keep the reference's bitpacked words;
// only registers ever hold bytes. With activation bits a in {0,1} (u8) and weight bits mapped
// to w' = +1 / -1 (s8):
//     popc(a ^ w) = popc(w) + sum_k a_k * w'_k
// so the accumulators start at the per-channel popcount of the filter row and the tensor pipe
// adds the signed dot product -- the same integer the XOR+POPC kernel produces, bit for bit
// (out-of-bounds taps gather 0 words = "+1" padding exactly as before).
// To make the bits -> bytes expansion cheap, bit i of a nibble becomes the byte VALUE 2^i (one
// PRMT replicates the thread's byte into all four lanes of a register, one AND with 0x08040201
// isolates bit i in byte i) and the weight byte at that k position is +-(8 >> i): every product
// is +-8, the accumulators hold 8 * popc(a ^ w) exactly, and the epilogue's "<< 1" becomes ">> 2".
// Activations are expanded bits -> bytes in registers, per warp. The static weights are expanded
// once per plan into mma B-fragment order (8 bytes per lane, k-step and 8-channel sub-tile) and
// reach shared memory by TMA bulk copy, so a B fragment is one conflict-free 64-bit LDS.
//
// CTA = 128 pixels x 64 channels, 4 warps of 32 x 64 (2 x 8 m16n8 tiles, 64 accumulators per
// thread). Thread (gid = lane / 4, tig = lane % 4) expands byte `tig` of each 32-bit word: its
// low nibble feeds the k 0..15 half of the fragment, its high nibble the k 16..31 half -- any
// bit <-> k assignment is valid as long as A and B use the same one.
#ifndef LCE_B200_IMMA_CUH_
#define LCE_B200_IMMA_CUH_

#include "lce_b200_chain.cuh"
#include "lce_b200_kernels.cuh"

namespace lce {

constexpr int kIBM = 128;
constexpr int kIThreads = 128;
// resident CTAs per SM the kernel is compiled for (register cap 65536 / (128 * n))
#ifdef LCE_IMMA_ALL4
__host__ __device__ constexpr int imma_ctas_per_sm(int) { return 4; }
#else
__host__ __device__ constexpr int imma_ctas_per_sm(int V) { return V == 4 ? 3 : 4; }
#endif
constexpr int kIBytesPerWord = kIBM * 4 + 8 * 32 * 8;  // smem per K word: packed A column + B fragments
// K is staged in one chunk when it fits, else through a TWO-deep ring: chunk c+1 is gathered /
// TMA-copied while chunk c is multiplied. The host sizes the chunks (imma_smem_budget):
// 3 CTAs per SM for the uint4 instances (153 registers), 4 for the narrower ones (128).
// b1 inner product: smem per 8-word k-slice (A rows [128][8 words] + B fragments [8][32] x 8 B),
// 768 B per K word. The host stages K in one chunk when it fits kB1SmemCtas CTAs per SM, which
// holds for every QuickNet layer; the register cap allows kB1Ctas.
constexpr int kB1BytesPerSlice = kIBM * 32 + 8 * 32 * 8;
constexpr int kB1Ctas = 4;
// the bitpacked group-window instance needs more than 128 registers: 3 CTAs per SM (168)
__host__ __device__ constexpr int b1_ctas_per_sm(bool gw, int out) { return gw && out == LCE_OUT_BITPACKED ? 3 : kB1Ctas; }
constexpr int kB1SmemCtas = 2;
// K words padded up to the b1 instructions' granularity (4 words = m16n8k128), in vectors of V
__host__ __device__ constexpr int b1_padded_vectors(int Kv, int V) { return ((Kv * V + 3) & ~3) / V; }

// byte `tig` of w -> two registers of four u8 each: bit i of the low / high nibble -> byte i with
// value 2^i (sel = tig * 0x1111 replicates the byte; 4 ALU instructions, no multiplies)
__device__ __forceinline__ void expand01(uint32_t w, uint32_t sel, uint32_t& lo, uint32_t& hi) {
  const uint32_t t = __byte_perm(w, 0u, sel);
  lo = t & 0x08040201u;
  hi = (t >> 4) & 0x08040201u;
}
__device__ __forceinline__ void mma_u8s8(int (&c)[4], const uint32_t (&a)[4], uint32_t b0,
                                         uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// weight nibble -> four s8: byte i = +(8 >> i) for bit 0 (+1), -(8 >> i) for bit 1 (-1)
__host__ __device__ __forceinline__ uint32_t imma_weight_bytes(uint32_t nibble) {
  uint32_t r = 0;
  for (int i = 0; i < 4; ++i) {
    const int mag = 8 >> i;
    const int v = ((nibble >> i) & 1u) ? -mag : mag;
    r |= (static_cast<uint32_t>(v) & 0xFFu) << (8 * i);
  }
  return r;
}

// Plan-time: wtx[n_tile][k word][ns / 2][lane][ns & 1] = {b0, b1}, the B fragment (k-step = that
// word, channels ns*8 .. ns*8+7 of the tile) of `lane`; the fragments of two neighbouring
// sub-tiles sit side by side so one 128-bit LDS fetches both. Channels past the group's end read
// as 0 words.
__global__ void expand_weights_imma_kernel(const int32_t* __restrict__ filter,
                                           uint2* __restrict__ wtx, int cout_pg,
                                           int tiles_per_group, int taps, int Cw_pg,
                                           long long total) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= total) return;
  const int ns = static_cast<int>(((idx >> 6) & 3) * 2 + (idx & 1));   // idx = ((kw*4 + ns/2)*32 + lane)*2 + (ns&1)
  const int lane = static_cast<int>((idx >> 1) & 31);
  const int Kw = taps * Cw_pg;
  const long long r = idx >> 8;
  const int kw = static_cast<int>(r % Kw);
  const int nt = static_cast<int>(r / Kw);
  const int g = nt / tiles_per_group, tg = nt - g * tiles_per_group;
  const int ch = tg * kBN + ns * 8 + (lane >> 2);
  uint32_t w = 0;
  if (ch < cout_pg)
    w = static_cast<uint32_t>(filter[(static_cast<long long>(g) * cout_pg + ch) * Kw + kw]);
  const uint32_t byte = (w >> (8 * (lane & 3))) & 0xFFu;
  wtx[idx] = make_uint2(imma_weight_bytes(byte & 0xFu), imma_weight_bytes(byte >> 4));
}

template <int V>
__device__ __forceinline__ void compute_chunk_imma(const typename VecT<V>::T* A_s,
                                                   const uint2* B_s, int nkv, int warp, int gid,
                                                   int tig, int lane, int (&acc)[2][8][4]) {
  const uint4* b4_base = reinterpret_cast<const uint4*>(B_s) + lane;
  using Vec = typename VecT<V>::T;
  const uint32_t sel = 0x1111u * static_cast<uint32_t>(tig);
  const Vec* a_base = A_s + warp * 32 + gid;
#pragma unroll 1
  for (int kv = 0; kv < nkv; ++kv) {
    uint32_t r[2][2][V];   // [m sub-tile][row gid / gid + 8][word]
#pragma unroll
    for (int ms = 0; ms < 2; ++ms) {
      load_words<V>(a_base + kv * kIBM + ms * 16, r[ms][0]);
      load_words<V>(a_base + kv * kIBM + ms * 16 + 8, r[ms][1]);
    }
    // two k-steps at a time: 16 live fragment registers instead of 8 * V
    constexpr int H = V < 2 ? V : 2;
#pragma unroll
    for (int qh = 0; qh < V; qh += H) {
      uint32_t a[H][2][4];
#pragma unroll
      for (int q = 0; q < H; ++q)
#pragma unroll
        for (int ms = 0; ms < 2; ++ms) {
          expand01(r[ms][0][qh + q], sel, a[q][ms][0], a[q][ms][2]);
          expand01(r[ms][1][qh + q], sel, a[q][ms][1], a[q][ms][3]);
        }
#pragma unroll
      for (int q = 0; q < H; ++q) {
#pragma unroll
        for (int np = 0; np < 4; ++np) {
          const uint4 b = b4_base[((kv * V + qh + q) * 4 + np) * 32];
          mma_u8s8(acc[0][2 * np], a[q][0], b.x, b.y);
          mma_u8s8(acc[1][2 * np], a[q][1], b.x, b.y);
          mma_u8s8(acc[0][2 * np + 1], a[q][0], b.z, b.w);
          mma_u8s8(acc[1][2 * np + 1], a[q][1], b.z, b.w);
        }
      }
    }
  }
}

// ---- b1 inner product: popc(a ^ w) = popc(w) + popc(a) - 2 * popc(a & w) ----
// BMMA.168256.AND.POPC sums popc(a & w) over 256 k; one more per m16 tile against an all-ones B
// fragment gives popc(a) per pixel row. Operands stay packed: A rows [k-slice][pixel][8 words],
// thread (gid, tig) holds words 2*tig (a0 / a1, b0) and 2*tig + 1 (a2 / a3, b1) of its rows. A
// K tail of 4 words runs as m16n8k128, thread tig holding word tig. Padding words are 0 in A and
// B and add nothing.
__device__ __forceinline__ void bmma_k256(int (&c)[4], const uint32_t (&a)[4], uint32_t b0,
                                          uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, "
      "{%8,%9}, {%0,%1,%2,%3};"
      : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void bmma_k128(int (&c)[4], uint32_t a0, uint32_t a1, uint32_t b0) {
  asm volatile(
      "mma.sync.aligned.m16n8k128.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5}, {%6}, "
      "{%0,%1,%2,%3};"
      : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
      : "r"(a0), "r"(a1), "r"(b0));
}

// Plan-time: wtb[n_tile][k-slice][ns / 2][lane][ns & 1] = {b0, b1}, the packed filter words of
// channel ns*8 + lane/4 that `lane` feeds to the b1 mma (see above); two neighbouring sub-tiles
// side by side so one 128-bit LDS fetches both. A k128 tail slice has {word tig, 0}. Words past
// Kw and channels past the group's end are 0.
// win_cw > 0: a group-window plan (see bconv_imma_kernel's GW), Cw_pg = win_cw, `groups` groups;
// tiles run over all channels (tiles_per_group unused) and K = taps x [window group 0's win_cw
// words | window group 1's], Kw = taps * 2 * win_cw. Each channel's filter words sit in its own
// group's half of the window and the other half is 0: the fragments are block-diagonal.
__global__ void pack_weights_b1_kernel(const int32_t* __restrict__ filter, uint2* __restrict__ wtb,
                                       int cout_pg, int tiles_per_group, int Kw, int n_slices,
                                       long long total, int win_cw = 0, int groups = 1) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= total) return;
  const int ns = static_cast<int>(((idx >> 6) & 3) * 2 + (idx & 1));
  const int lane = static_cast<int>((idx >> 1) & 31);
  const long long r = idx >> 8;
  const int s = static_cast<int>(r % n_slices);
  const int nt = static_cast<int>(r / n_slices);
  const int tig = lane & 3;
  const bool tail = s * 8 + 4 >= ((Kw + 3) & ~3);
  const int k0 = s * 8 + (tail ? tig : 2 * tig);
  uint32_t w0, w1;
  if (win_cw > 0) {
    const int c = nt * kBN + ns * 8 + (lane >> 2);
    const int gb = min(nt * kBN / cout_pg, groups - 2), gc = c / cout_pg;
    auto word = [&](int k) -> uint32_t {
      const int tap = k / (2 * win_cw), wi = k - tap * 2 * win_cw;
      if (c >= cout_pg * groups || k >= Kw || gb + wi / win_cw != gc) return 0u;
      return static_cast<uint32_t>(filter[static_cast<long long>(c) * (Kw / 2) + tap * win_cw + wi % win_cw]);
    };
    w0 = word(k0);
    w1 = tail ? 0u : word(k0 + 1);
  } else {
    const int g = nt / tiles_per_group, tg = nt - g * tiles_per_group;
    const int ch = tg * kBN + ns * 8 + (lane >> 2);
    const int32_t* row = filter + (static_cast<long long>(g) * cout_pg + ch) * Kw;
    const bool ch_ok = ch < cout_pg;
    w0 = ch_ok && k0 < Kw ? static_cast<uint32_t>(row[k0]) : 0u;
    w1 = ch_ok && !tail && k0 + 1 < Kw ? static_cast<uint32_t>(row[k0 + 1]) : 0u;
  }
  wtb[idx] = make_uint2(w0, w1);
}

// acc += popc(a & w) and pa += popc(a) over `words` K words (a multiple of 4) of one chunk.
// GW (group window, K = taps x [window group 0's cw words | window group 1's], the chunk starting
// at window word k0): pa column n counts only window group (n & 1)'s bits. The popc BMMA's B
// fragment is that group's mask instead of all ones, so pa[ms][e] holds group e & 1's popcount.
template <bool GW = false>
__device__ __forceinline__ void compute_chunk_b1(const uint32_t* A_s, const uint2* B_s, int words,
                                                 int warp, int gid, int tig, int lane,
                                                 int (&acc)[2][8][4], int (&pa)[2][4], int k0 = 0,
                                                 int cw = 0, int step = 0) {
  const uint4* b4 = reinterpret_cast<const uint4*>(B_s) + lane;
  const uint2* a2 = reinterpret_cast<const uint2*>(A_s) + (warp * 32 + gid) * 4 + tig;
  const int full = words >> 3;
  // GW: r = the window position of this thread's word 2 * tig of the slice, advanced 8 (step =
  // 8 % cw2) per slice
  const int cw2 = 2 * cw;
  auto mask = [&](int q) { return (q >= cw) != (gid & 1) ? 0u : ~0u; };
  int r = 0;
  if constexpr (GW) r = (k0 + 2 * tig) % cw2;
#pragma unroll 2
  for (int s = 0; s < full; ++s) {
    uint32_t a[2][4];
#pragma unroll
    for (int ms = 0; ms < 2; ++ms) {
      const uint2 lo = a2[(s * kIBM + ms * 16) * 4];
      const uint2 hi = a2[(s * kIBM + ms * 16 + 8) * 4];
      a[ms][0] = lo.x; a[ms][1] = hi.x; a[ms][2] = lo.y; a[ms][3] = hi.y;
    }
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      const uint4 b = b4[(s * 4 + np) * 32];
      bmma_k256(acc[0][2 * np], a[0], b.x, b.y);
      bmma_k256(acc[1][2 * np], a[1], b.x, b.y);
      bmma_k256(acc[0][2 * np + 1], a[0], b.z, b.w);
      bmma_k256(acc[1][2 * np + 1], a[1], b.z, b.w);
    }
    uint32_t m0 = ~0u, m1 = ~0u;
    if constexpr (GW) {
      m0 = mask(r);
      m1 = mask(r + 1 == cw2 ? 0 : r + 1);
      r += step;
      if (r >= cw2) r -= cw2;
    }
    bmma_k256(pa[0], a[0], m0, m1);
    bmma_k256(pa[1], a[1], m0, m1);
  }
  if (words & 4) {
    const uint32_t* a1 = A_s + (full * kIBM + warp * 32 + gid) * 8 + tig;
    uint32_t lo[2], hi[2];
#pragma unroll
    for (int ms = 0; ms < 2; ++ms) {
      lo[ms] = a1[(ms * 16) * 8];
      hi[ms] = a1[(ms * 16 + 8) * 8];
    }
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      const uint4 b = b4[(full * 4 + np) * 32];
#pragma unroll
      for (int ms = 0; ms < 2; ++ms) {
        bmma_k128(acc[ms][2 * np], lo[ms], hi[ms], b.x);
        bmma_k128(acc[ms][2 * np + 1], lo[ms], hi[ms], b.z);
      }
    }
    uint32_t m = ~0u;
    if constexpr (GW) m = mask((k0 + full * 8 + tig) % cw2);
#pragma unroll
    for (int ms = 0; ms < 2; ++ms) bmma_k128(pa[ms], lo[ms], hi[ms], m);
  }
}

// SAME padding with pad value 0 (reference.h:100-103), for this kernel's accumulator layout:
// an out-of-bounds tap contributes channels_in_per_group / 2 instead of popc(0 ^ w) -- times
// 2^S, the accumulators' scale (8 for the int8 inner product, 1 for b1).
template <int S>
__device__ __forceinline__ void zero_pad_correction_imma(const ConvKParams& p,
                                                         int (&acc)[2][8][4], long long m0,
                                                         int c_tile, int warp, int gid, int tig) {
  const int taps = p.KH * p.KW;
#pragma unroll
  for (int ms = 0; ms < 2; ++ms) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long m = m0 + warp * 32 + ms * 16 + h * 8 + gid;
      if (m >= p.M) continue;
      long long b;
      int oy, ox;
      split_pixel(p, m, &b, &oy, &ox);
      const int iy_lo = oy * p.sh - p.ph, ix_lo = ox * p.sw - p.pw;
      if (iy_lo >= 0 && ix_lo >= 0 && iy_lo + (p.KH - 1) * p.dh < p.H &&
          ix_lo + (p.KW - 1) * p.dw < p.W)
        continue;  // interior pixel
      for (int fy = 0; fy < p.KH; ++fy) {
        const int iy = iy_lo + fy * p.dh;
        const bool yin = static_cast<unsigned>(iy) < static_cast<unsigned>(p.H);
        for (int fx = 0; fx < p.KW; ++fx) {
          const int ix = ix_lo + fx * p.dw;
          if (yin && static_cast<unsigned>(ix) < static_cast<unsigned>(p.W)) continue;
          const int t = fy * p.KW + fx;
#pragma unroll
          for (int ns = 0; ns < 8; ++ns) {
            const int c = c_tile + ns * 8 + tig * 2;
            acc[ms][ns][h * 2] +=
                (1 << S) * (p.zp_half - p.tap_popc[static_cast<size_t>(c) * taps + t]);
            acc[ms][ns][h * 2 + 1] +=
                (1 << S) * (p.zp_half - p.tap_popc[static_cast<size_t>(c + 1) * taps + t]);
          }
        }
      }
    }
  }
}

// Columns c and c + 1 of the SHUFFLE store, from the +-1 dot products y0, y1: FULLY_CONNECTED's alpha
// (run_fused_fc), one rounding; TRANSPOSE_CONV's or FULLY_CONNECTED's bias, one rounding, then its
// activation; then run_fused_fc's BatchNorm, MUL and ADD rounded apart as TFLite's ops round them, and
// the ADD's activation. Each vector is read here, per column pair, so none stays in registers.
__device__ __forceinline__ float act_clamp(float y, int act) {
  if (act == LCE_ACT_NONE) return y;
  const float lo = act == LCE_ACT_RELU_N1_TO_1 ? -1.0f : 0.0f;
  const float hi = act == LCE_ACT_RELU ? __int_as_float(0x7f800000) : (act == LCE_ACT_RELU6 ? 6.0f : 1.0f);
  return fminf(fmaxf(y, lo), hi);
}
__device__ __forceinline__ float2 fc_steps(const ConvKParams& p, int c, float y0, float y1) {
  if (p.shuf_alpha != nullptr) {
    const float2 a = __ldg(reinterpret_cast<const float2*>(p.shuf_alpha + c));
    y0 = __fmul_rn(y0, a.x);
    y1 = __fmul_rn(y1, a.y);
  }
  if (p.shuf_bias != nullptr) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(p.shuf_bias + c));
    y0 = __fadd_rn(y0, b.x);
    y1 = __fadd_rn(y1, b.y);
  }
  y0 = act_clamp(y0, p.shuf_act);
  y1 = act_clamp(y1, p.shuf_act);
  if (p.shuf_scale != nullptr) {
    const float2 a = __ldg(reinterpret_cast<const float2*>(p.shuf_scale + c));
    y0 = __fmul_rn(y0, a.x);
    y1 = __fmul_rn(y1, a.y);
  }
  if (p.shuf_shift != nullptr) {
    const float2 b = __ldg(reinterpret_cast<const float2*>(p.shuf_shift + c));
    y0 = __fadd_rn(y0, b.x);
    y1 = __fadd_rn(y1, b.y);
  }
  return make_float2(act_clamp(y0, p.shuf_act2), act_clamp(y1, p.shuf_act2));
}

// Accumulator (ms, ns, e) of thread (gid, tig): pixel m0 + warp*32 + ms*16 + (e/2)*8 + gid,
// channel c_tile + ns*8 + tig*2 + (e & 1), at scale 2^S. Full 64-channel tiles only
// (host-checked). CHAIN (float output): ReActNet's chain on the fused sum. Its four vectors and
// the output transform's multiplier and bias are read per row from chain_s = [shift_in | alpha |
// shift_out | sign_shift | mul | bias] x 64 channels in shared memory: holding them all in
// registers would exceed the b1 instances' 128-register cap. GATE (float output): Real-to-Binary's
// gated tail (p.gate) before the shortcut ADD, from chain_s = [- | alpha | sign_scale | sign_shift
// | mul | bias]; the gate row is each row's own image's (a tile can span several images). With
// SPATIAL it is the row's position within its image instead: XNOR-Net++'s scale Gamma[OH*OW][C]
// (lce_b200_bconv2d_run_fused_scale, alpha absent).
// SLICE (float output, no signs): row m goes to out + m * p.out_stride, a channel slice of a
// wider map; a shortcut is read at the same strided address, which may be the output itself.
// BITPACKED: the row's two output words, bit = acc > p.thr[c], packed like the float output's signs.
// GW (group-window plans): the last tile may hold only 32 channels (channels_out % 64 == 32); its
// upper half (ns 4..7, the second output word) is then neither read nor written.
// SHUFFLE (float output, 1x1 plan, lce_b200_bconv2d_run_fused_shuffle): column (i * sw + j) * C + c of
// row m = (b * OH + y) * OW + x goes to pixel ((b * OH + y) * sh + i) * OW * sw + x * sw + j of a
// [B, OH * sh, OW * sw, C] map, C = p.shuf_c a multiple of 64, so the tile's 64 columns are one phase
// (i, j)'s contiguous channels of that pixel; the shortcut and the signs are read and written there.
// The plan's output transform is not applied: y = D = p.shuf_k - 2 popc(a ^ w), the +-1 dot product,
// exact, then p.shuf_bias added with one rounding and p.shuf_act applied (TRANSPOSE_CONV's), then the
// shortcut. No per-channel vectors stay in registers, which keeps the instance within the b1 cap.
// The same instance runs lce_b200_bconv2d_run_fused_fc: with sh = sw = 1 and OH = OW = 1 the address
// is row-major [M, cout], and D is scaled by p.shuf_alpha before the bias and followed by the
// BatchNorm p.shuf_scale, p.shuf_shift and p.shuf_act2, each step rounded on its own.
template <int OUT, int S, bool CHAIN = false, bool GATE = false, bool SLICE = false, bool SPATIAL = false,
          bool GW = false, bool SHUFFLE = false>
__device__ __forceinline__ void epilogue_imma(const ConvKParams& p, int (&acc)[2][8][4],
                                              long long m0, int c_tile, int warp, int gid,
                                              int tig, const float* chain_s = nullptr) {
  static_assert(!(CHAIN && GATE), "one epilogue tail at a time");
  static_assert(!SPATIAL || GATE, "a spatial scale is the gate tail's");
  static_assert(!SLICE || (OUT == LCE_OUT_FLOAT && !CHAIN && !GATE), "a plain float slice");
  static_assert(!SHUFFLE || (OUT == LCE_OUT_FLOAT && !CHAIN && !GATE && !SLICE && !GW), "a plain float shuffle");
  static_assert(OUT != LCE_OUT_BITPACKED || !(CHAIN || GATE || SLICE), "float tails only");
  constexpr bool STAGED = CHAIN || GATE;
  const int cth = c_tile + tig * 2;
  // SHUFFLE: the tile's phase (si, sj) and first channel c_sh
  const int phase = SHUFFLE ? c_tile / p.shuf_c : 0;
  const int c_sh = SHUFFLE ? c_tile - phase * p.shuf_c : c_tile;
  const int si = SHUFFLE ? phase / p.shuf_sw : 0;
  const int sj = phase - si * p.shuf_sw;
  const bool hi = !GW || c_tile + 32 < p.cout;
  float2 mul_r[8], bias_r[8];
  int2 thr_r[8];
  if (OUT == LCE_OUT_FLOAT && !STAGED && !SHUFFLE) {
#pragma unroll
    for (int ns = 0; ns < 8; ++ns) {
      mul_r[ns] = *reinterpret_cast<const float2*>(p.mul + cth + ns * 8);
      bias_r[ns] = *reinterpret_cast<const float2*>(p.bias + cth + ns * 8);
    }
  }
  if (OUT == LCE_OUT_BITPACKED) {
#pragma unroll
    for (int ns = 0; ns < 8; ++ns) thr_r[ns] = __ldg(reinterpret_cast<const int2*>(p.thr + cth + ns * 8));
  }
  const bool has_res = OUT == LCE_OUT_FLOAT && p.residual != nullptr;
  const bool has_pk = OUT == LCE_OUT_BITPACKED || (OUT == LCE_OUT_FLOAT && !SLICE && p.packed_out != nullptr);
  // fused activation of the ADD as one clamp: y = min(max(y, lo), hi) (kernel_util.h:285-300)
  const int ract = p.residual_act;
  const float act_lo = ract == LCE_ACT_RELU_N1_TO_1 ? -1.0f : 0.0f;
  const float act_hi = ract == LCE_ACT_RELU ? __int_as_float(0x7f800000)
                                            : (ract == LCE_ACT_RELU6 ? 6.0f : 1.0f);
#pragma unroll
  for (int ms = 0; ms < 2; ++ms) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int lrow = warp * 32 + ms * 16 + h * 8 + gid;
      const long long m = m0 + lrow;
      const bool row_ok = m < p.M;
      // SHUFFLE: the output pixel of row m (M < 2^31, host-checked)
      long long opix = m;
      if constexpr (SHUFFLE) {
        const uint32_t yy = fdiv(static_cast<uint32_t>(m), p.fd_ow);   // b * OH + y
        const long long x = m - static_cast<long long>(yy) * p.OW;
        opix = (static_cast<long long>(yy) * p.shuf_sh + si) * (static_cast<long long>(p.OW) * p.shuf_sw) +
               x * p.shuf_sw + sj;
      }
      const size_t e0 = SLICE     ? static_cast<size_t>(m) * p.out_stride + cth
                        : SHUFFLE ? static_cast<size_t>(opix) * p.shuf_c + c_sh + tig * 2
                                  : static_cast<size_t>(m) * p.cout + cth;
      if (OUT == LCE_OUT_RAW_ACC) {
        if (row_ok) {
          int* o = static_cast<int*>(p.out) + e0;
#pragma unroll
          for (int ns = 0; ns < 8; ++ns)
            if (ns < 4 || hi)
              *reinterpret_cast<int2*>(o + ns * 8) =
                  make_int2(acc[ms][ns][h * 2] >> S, acc[ms][ns][h * 2 + 1] >> S);
        }
        continue;
      }
      uint32_t bits0 = 0, bits1 = 0;
      if (OUT == LCE_OUT_BITPACKED && row_ok) {
        // OutputTransform<TBitpacked>: bit = acc > threshold (output_transform.h:164-167)
#pragma unroll
        for (int ns = 0; ns < 4; ++ns) {
          bits0 |= (((acc[ms][ns][h * 2] >> S) > thr_r[ns].x ? 1u : 0u) |
                    ((acc[ms][ns][h * 2 + 1] >> S) > thr_r[ns].y ? 2u : 0u)) << (ns * 8);
          bits1 |= (((acc[ms][ns + 4][h * 2] >> S) > thr_r[ns + 4].x ? 1u : 0u) |
                    ((acc[ms][ns + 4][h * 2 + 1] >> S) > thr_r[ns + 4].y ? 2u : 0u)) << (ns * 8);
        }
        bits0 <<= tig * 2;
        bits1 <<= tig * 2;
      } else if (OUT != LCE_OUT_BITPACKED && row_ok) {
        float y[16];
#pragma unroll
        for (int ns = 0; ns < 8; ++ns) {
          // OutputTransform's (acc << 1); at scale 8 that is (acc8 >> 2), exactly
          int x0 = acc[ms][ns][h * 2], x1 = acc[ms][ns][h * 2 + 1];
          if constexpr (S > 0) {
            x0 >>= S - 1; x1 >>= S - 1;
          } else {
            x0 <<= 1; x1 <<= 1;
          }
          if constexpr (SHUFFLE) {
            y[2 * ns] = static_cast<float>(p.shuf_k - x0);
            y[2 * ns + 1] = static_cast<float>(p.shuf_k - x1);
          } else if constexpr (STAGED) {
            const float2 mu = *reinterpret_cast<const float2*>(chain_s + 4 * kBN + tig * 2 + ns * 8);
            const float2 bi = *reinterpret_cast<const float2*>(chain_s + 5 * kBN + tig * 2 + ns * 8);
            y[2 * ns] = transform_float_x2(x0, p.clamp_min, p.clamp_max, mu.x, bi.x);
            y[2 * ns + 1] = transform_float_x2(x1, p.clamp_min, p.clamp_max, mu.y, bi.y);
          } else {
            y[2 * ns] = transform_float_x2(x0, p.clamp_min, p.clamp_max, mul_r[ns].x, bias_r[ns].x);
            y[2 * ns + 1] =
                transform_float_x2(x1, p.clamp_min, p.clamp_max, mul_r[ns].y, bias_r[ns].y);
          }
        }
        if constexpr (SHUFFLE) {
          const int cv = c_sh + tig * 2;
#pragma unroll
          for (int ns = 0; ns < 8; ++ns) {
            const float2 r = fc_steps(p, cv + ns * 8, y[2 * ns], y[2 * ns + 1]);
            y[2 * ns] = r.x;
            y[2 * ns + 1] = r.y;
          }
        }
        if constexpr (GATE) {
          // MUL(gate) -> PRELU(alpha): gate row b = m / (OH * OW), or with SPATIAL the position
          // m - b * OH * OW (M < 2^31, host-checked)
          const uint32_t b = fdiv(static_cast<uint32_t>(m), p.fd_ohw);
          const uint32_t gi =
              SPATIAL ? static_cast<uint32_t>(m) - b * (static_cast<uint32_t>(p.OH) * p.OW) : b;
          const float* gr = p.gate.gate + static_cast<size_t>(gi) * p.cout + cth;
          const bool has_a = p.gate.alpha != nullptr;
#pragma unroll
          for (int ns = 0; ns < 8; ++ns) {
            const float2 gv = ns < 4 || hi ? __ldg(reinterpret_cast<const float2*>(gr + ns * 8))
                                           : make_float2(0.0f, 0.0f);
            const float2 al = *reinterpret_cast<const float2*>(chain_s + kBN + tig * 2 + ns * 8);
            y[2 * ns] = gate_prelu(y[2 * ns], gv.x, has_a, al.x);
            y[2 * ns + 1] = gate_prelu(y[2 * ns + 1], gv.y, has_a, al.y);
          }
        }
        if (has_res) {
          // (A TMA-staged copy of the shortcut tile was measured slower on every layer: the
          // extra 36 KB of shared memory cost a resident CTA. The rows are already in L2.)
          float2 rv[8];
          const float* r = p.residual + e0;
          // SLICE: the residual may be the output this kernel writes, so not the read-only
          // (non-coherent) path
#pragma unroll
          for (int ns = 0; ns < 8; ++ns)
            rv[ns] = !(ns < 4 || hi) ? make_float2(0.0f, 0.0f)
                     : SLICE         ? __ldcg(reinterpret_cast<const float2*>(r + ns * 8))
                                     : __ldg(reinterpret_cast<const float2*>(r + ns * 8));
#pragma unroll
          for (int ns = 0; ns < 8; ++ns) {
            y[2 * ns] = __fadd_rn(y[2 * ns], rv[ns].x);
            y[2 * ns + 1] = __fadd_rn(y[2 * ns + 1], rv[ns].y);
          }
          if (ract != LCE_ACT_NONE) {
#pragma unroll
            for (int j = 0; j < 16; ++j) y[j] = fminf(fmaxf(y[j], act_lo), act_hi);
          }
        }
        if constexpr (GATE) {
          // the gated tail applies the activation with or without a shortcut
          if (!has_res && ract != LCE_ACT_NONE) {
#pragma unroll
            for (int j = 0; j < 16; ++j) y[j] = fminf(fmaxf(y[j], act_lo), act_hi);
          }
        }
        if constexpr (CHAIN) {
          const bool has_si = p.chain.shift_in != nullptr, has_a = p.chain.alpha != nullptr;
          const bool has_so = p.chain.shift_out != nullptr;
#pragma unroll
          for (int ns = 0; ns < 8; ++ns) {
            const int k = tig * 2 + ns * 8;
            const float2 si = *reinterpret_cast<const float2*>(chain_s + k);
            const float2 al = *reinterpret_cast<const float2*>(chain_s + kBN + k);
            const float2 so = *reinterpret_cast<const float2*>(chain_s + 2 * kBN + k);
            y[2 * ns] = chain_rprelu(y[2 * ns], has_si, si.x, has_a, al.x, has_so, so.x);
            y[2 * ns + 1] = chain_rprelu(y[2 * ns + 1], has_si, si.y, has_a, al.y, has_so, so.y);
          }
        }
        float* o = static_cast<float*>(p.out) + e0;
#pragma unroll
        for (int ns = 0; ns < 8; ++ns)
          if (ns < 4 || hi) *reinterpret_cast<float2*>(o + ns * 8) = make_float2(y[2 * ns], y[2 * ns + 1]);
        if (has_pk) {
          if constexpr (CHAIN) {
            // RSign: LceQuantize of the value just written plus sign_shift
            const bool has_ss = p.chain.sign_shift != nullptr;
            const float* ss = chain_s + 3 * kBN + tig * 2;
#pragma unroll
            for (int ns = 0; ns < 4; ++ns) {
              const float2 s0 = *reinterpret_cast<const float2*>(ss + ns * 8);
              const float2 s1 = *reinterpret_cast<const float2*>(ss + ns * 8 + 32);
              bits0 |= ((chain_sign(y[2 * ns], has_ss, s0.x) ? 1u : 0u) |
                        (chain_sign(y[2 * ns + 1], has_ss, s0.y) ? 2u : 0u)) << (ns * 8);
              bits1 |= ((chain_sign(y[2 * ns + 8], has_ss, s1.x) ? 1u : 0u) |
                        (chain_sign(y[2 * ns + 9], has_ss, s1.y) ? 2u : 0u)) << (ns * 8);
            }
          } else if constexpr (GATE) {
            // the next block's BatchNorm and sign: bit of o * sign_scale + sign_shift
            const bool has_sc = p.gate.sign_scale != nullptr, has_sh = p.gate.sign_shift != nullptr;
            const float* sc = chain_s + 2 * kBN + tig * 2;
            const float* sh = chain_s + 3 * kBN + tig * 2;
#pragma unroll
            for (int ns = 0; ns < 4; ++ns) {
              const float2 c0 = *reinterpret_cast<const float2*>(sc + ns * 8);
              const float2 c1 = *reinterpret_cast<const float2*>(sc + ns * 8 + 32);
              const float2 h0 = *reinterpret_cast<const float2*>(sh + ns * 8);
              const float2 h1 = *reinterpret_cast<const float2*>(sh + ns * 8 + 32);
              bits0 |= ((affine_sign(y[2 * ns], has_sc, c0.x, has_sh, h0.x) ? 1u : 0u) |
                        (affine_sign(y[2 * ns + 1], has_sc, c0.y, has_sh, h0.y) ? 2u : 0u)) << (ns * 8);
              bits1 |= ((affine_sign(y[2 * ns + 8], has_sc, c1.x, has_sh, h1.x) ? 1u : 0u) |
                        (affine_sign(y[2 * ns + 9], has_sc, c1.y, has_sh, h1.y) ? 2u : 0u)) << (ns * 8);
            }
          } else {
            // LceQuantize of the value just written: bit = value < 0 (bitpack.h:159)
#pragma unroll
            for (int ns = 0; ns < 4; ++ns) {
              bits0 |= ((y[2 * ns] < 0.0f ? 1u : 0u) | (y[2 * ns + 1] < 0.0f ? 2u : 0u)) << (ns * 8);
              bits1 |= ((y[2 * ns + 8] < 0.0f ? 1u : 0u) | (y[2 * ns + 9] < 0.0f ? 2u : 0u)) << (ns * 8);
            }
          }
          bits0 <<= tig * 2;
          bits1 <<= tig * 2;
        }
      }
      if (has_pk) {  // uniform across the warp: every lane runs the shuffles
        bits0 |= __shfl_xor_sync(0xffffffffu, bits0, 1);
        bits1 |= __shfl_xor_sync(0xffffffffu, bits1, 1);
        bits0 |= __shfl_xor_sync(0xffffffffu, bits0, 2);
        bits1 |= __shfl_xor_sync(0xffffffffu, bits1, 2);
        if (row_ok && tig == 0) {
          int32_t* pk = (OUT == LCE_OUT_BITPACKED ? static_cast<int32_t*>(p.out) : p.packed_out) +
                        static_cast<size_t>(opix) * p.cw_out + (c_sh >> 5);
          pk[0] = static_cast<int32_t>(bits0);
          if (hi) pk[1] = static_cast<int32_t>(bits1);
        }
      }
    }
  }
}

// FCMAX (b1, lce_b200_bconv2d_run_fused_fc_max): the columns run_fused_fc stores (SHUFFLE with sh =
// sw = 1, fc_steps), but each column's max over the rows of each image instead of the rows. Row m
// belongs to image m / points (p.fd_pts); the thread's four rows m0 + warp * 32 + {0, 8, 16, 24} + gid
// come in row order, so it keeps one key (max_key) per image run and column and merges a run into
// p.max_keys[image][column] with atomicMax when its image ends. When the warp's 32 rows all belong to
// one image, its eight lanes of each column merge first and one of them writes. Column pair by column
// pair, so the accumulators of a pair die as it is done.
__device__ __forceinline__ void epilogue_fc_max(const ConvKParams& p, int (&acc)[2][8][4], long long m0,
                                                int c_tile, int warp, int gid, int tig) {
  const long long mw = m0 + warp * 32;   // the warp's first row (M < 2^31, host-checked)
  uint32_t img[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) img[r] = fdiv(static_cast<uint32_t>(mw + r * 8 + gid), p.fd_pts);
  const bool one = mw + 31 < p.M &&
                   fdiv(static_cast<uint32_t>(mw), p.fd_pts) == fdiv(static_cast<uint32_t>(mw + 31), p.fd_pts);
  auto merge = [&](uint32_t b, int c, unsigned long long k0, unsigned long long k1) {
    unsigned long long* kp = p.max_keys + static_cast<size_t>(b) * p.cout + c;
    if (k0) atomicMax(kp, k0);
    if (k1) atomicMax(kp + 1, k1);
  };
#pragma unroll
  for (int ns = 0; ns < 8; ++ns) {
    const int c = c_tile + ns * 8 + tig * 2;
    unsigned long long k0 = 0, k1 = 0;
    uint32_t cur = img[0];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const long long m = mw + r * 8 + gid;
      if (m >= p.M) break;
      if (img[r] != cur) {
        merge(cur, c, k0, k1);
        k0 = k1 = 0;
        cur = img[r];
      }
      // the +-1 dot product D = K - 2 popc(a ^ w), as the SHUFFLE store takes it
      const int x0 = acc[r >> 1][ns][(r & 1) * 2] << 1, x1 = acc[r >> 1][ns][(r & 1) * 2 + 1] << 1;
      const float2 y = fc_steps(p, c, static_cast<float>(p.shuf_k - x0), static_cast<float>(p.shuf_k - x1));
      k0 = max(k0, max_key(y.x, static_cast<uint32_t>(m)));
      k1 = max(k1, max_key(y.y, static_cast<uint32_t>(m)));
    }
    if (one) {   // uniform across the warp
#pragma unroll
      for (int off = 4; off < 32; off <<= 1) {
        k0 = max(k0, __shfl_xor_sync(0xffffffffu, k0, off));
        k1 = max(k1, __shfl_xor_sync(0xffffffffu, k1, off));
      }
      if (gid == 0) merge(cur, c, k0, k1);
    } else {
      merge(cur, c, k0, k1);
    }
  }
}

// B1 selects the inner product: packed b1 fragments (accumulators at scale 1) or int8 ones
// (scale 8). Both produce the same int32 accumulators. CHAIN (float output): the epilogue also
// applies p.chain (lce_b200_bconv2d_run_fused_chain); GATE (float output): p.gate
// (lce_b200_bconv2d_run_fused_gate), with SPATIAL p.gate indexed by position
// (lce_b200_bconv2d_run_fused_scale); SLICE (float output): the strided store of
// lce_b200_bconv2d_run_slice, and its read-add-write in lce_b200_bconv2d_run_slice_add; SHUFFLE (b1,
// float output): the pixel-shuffled store of lce_b200_bconv2d_run_fused_shuffle; FCMAX (b1): its
// run_fused_fc columns reduced to each image's max (epilogue_fc_max). The other instances compile as
// without them.
// GW (b1 only): a grouped plan whose groups hold 32 * odd output channels, so a 64-channel tile on
// 64-aligned channels may span two groups. Tile nt covers channels nt * 64 .. nt * 64 + 63 and
// gathers, per tap, the contiguous input words of two neighbouring groups (its window, from group
// gb = min(first channel's group, groups - 2)): p.Kv and p.CwV count the window's vectors, p.Cw_pg
// one group's words. The fragments are block-diagonal (pack_weights_b1_kernel) and pa counts each
// window group's bits apart (compute_chunk_b1), so every channel gets popc(a ^ w) over its own
// group alone: the XOR + POPC kernel's integers.
template <int V, int OUT, bool B1, bool CHAIN = false, bool GATE = false, bool SLICE = false,
          bool SPATIAL = false, bool GW = false, bool SHUFFLE = false, bool FCMAX = false>
__global__ void __launch_bounds__(kIThreads, B1 ? b1_ctas_per_sm(GW, OUT) : imma_ctas_per_sm(V))
bconv_imma_kernel(const ConvKParams p) {
  static_assert(!GW || (B1 && !SLICE), "group windows: b1, no slice store");
  static_assert(!SHUFFLE || B1, "the shuffle store: b1 only");
  static_assert(!FCMAX || (B1 && OUT == LCE_OUT_FLOAT && !CHAIN && !GATE && !SLICE && !GW && !SHUFFLE),
                "the max epilogue: b1, float columns, no other tail");
  using Vec = typename VecT<V>::T;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  // two buffers of { A: [Kc_v][128] packed vectors, B: [Kc_v*V][8][32] int8 fragments }, or for
  // B1 { A: [slices][128][8 words], B: [slices][8][32] b1 fragments }
  __shared__ __align__(8) uint64_t wbar[2];

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int gid = lane >> 2, tig = lane & 3;
  const int nt = blockIdx.y;
  // GW: g = the window's first group
  const int g = GW ? min(nt * kBN / p.cout_pg, p.cout / p.cout_pg - 2)
                   : static_cast<int>(fdiv(static_cast<uint32_t>(nt), p.fd_tpg));
  const int tg = GW ? 0 : nt - g * p.tiles_per_group;
  const long long m0 = static_cast<long long>(blockIdx.x) * kIBM;
  const int c_tile = GW ? nt * kBN : g * p.cout_pg + tg * kBN;
  // B1: K runs to the padded vector count, in 8-word slices (the last may be a 4-word one)
  const int Kv_end = B1 ? b1_padded_vectors(p.Kv, V) : p.Kv;
  const int n_slices = (Kv_end * V + 7) >> 3;
  const int chunk_slices = (p.Kc_v * V + 7) >> 3;

  if (tid == 0) {
    mbar_init(&wbar[0], 1);
    mbar_init(&wbar[1], 1);
    fence_barrier_init();
  }
  __syncthreads();

  // int8: accumulators start at 8 * popc(filter row): acc8 = 8 * (popc(w) + sum a * w').
  // B1: they sum popc(a & w), and pa sums popc(a) of each row.
  int acc[2][8][4];
  int pa[2][4] = {};
#pragma unroll
  for (int ns = 0; ns < 8; ++ns) {
    const int2 pw = B1 ? make_int2(0, 0)
                       : *reinterpret_cast<const int2*>(p.wpop + c_tile + ns * 8 + tig * 2);
#pragma unroll
    for (int ms = 0; ms < 2; ++ms) {
      acc[ms][ns][0] = pw.x * 8; acc[ms][ns][1] = pw.y * 8;
      acc[ms][ns][2] = pw.x * 8; acc[ms][ns][3] = pw.y * 8;
    }
  }
  if (OUT == LCE_OUT_FLOAT && !SLICE && !SHUFFLE && p.residual != nullptr) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const long long m = m0 + warp * 32 + i * 8 + gid;
      if (m < p.M && (!GW || c_tile + tig * 16 < p.cout))
        asm volatile("prefetch.global.L2 [%0];" ::"l"(p.residual + m * p.cout + c_tile + tig * 16));
    }
  }

  const size_t a_bytes = B1 ? static_cast<size_t>(chunk_slices) * kIBM * 32
                            : static_cast<size_t>(p.Kc_v) * kIBM * sizeof(Vec);
  const size_t chunk_bytes = B1 ? static_cast<size_t>(chunk_slices) * kB1BytesPerSlice
                                : static_cast<size_t>(p.Kc_v) * V * kIBytesPerWord;
  auto stage = [&](int ch) {
    unsigned char* base = smem_raw + (ch & 1) * chunk_bytes;
    Vec* A_b = reinterpret_cast<Vec*>(base);
    uint2* B_b = reinterpret_cast<uint2*>(base + a_bytes);
    const int kv0 = ch * p.Kc_v;
    const int kv1 = min(kv0 + p.Kc_v, Kv_end);
    if (tid == 0) {
      // B fragments: 8 * 32 uint2 per K word (int8) or per 8-word slice (b1)
      const size_t frag0 = B1 ? static_cast<size_t>(nt) * n_slices + (kv0 * V >> 3)
                              : (static_cast<size_t>(nt) * p.Kv + kv0) * V;
      const uint32_t nfrag = B1 ? static_cast<uint32_t>(((kv1 - kv0) * V + 7) >> 3)
                                : static_cast<uint32_t>(kv1 - kv0) * V;
      const uint32_t bytes = nfrag * (8 * 32 * 8);
      mbar_arrive_expect_tx(&wbar[ch & 1], bytes);
      bulk_g2s(B_b, reinterpret_cast<const uint2*>(p.wt) + frag0 * (8 * 32), bytes, &wbar[ch & 1]);
    }
    gather_tile<V, kIBM, kIThreads, B1>(p, A_b, m0, g, kv0, kv1, tid);
    cp_async_commit();
  };
  stage(0);
  for (int ch = 0; ch < p.n_chunks; ++ch) {
    const bool more = ch + 1 < p.n_chunks;
    if (more) stage(ch + 1);  // its buffer was released by the barrier that ended chunk ch - 1
    if (more) asm volatile("cp.async.wait_group 1;" ::: "memory");
    else asm volatile("cp.async.wait_group 0;" ::: "memory");
    mbar_wait(&wbar[ch & 1], (ch >> 1) & 1);
    __syncthreads();
    unsigned char* base = smem_raw + (ch & 1) * chunk_bytes;
    const uint2* B_b = reinterpret_cast<const uint2*>(base + a_bytes);
    const int kv0 = ch * p.Kc_v;
    const int nkv = min(kv0 + p.Kc_v, Kv_end) - kv0;
    if constexpr (B1)
      compute_chunk_b1<GW>(reinterpret_cast<const uint32_t*>(base), B_b, nkv * V, warp, gid, tig,
                           lane, acc, pa, kv0 * V, p.Cw_pg, p.win_step);
    else
      compute_chunk_imma<V>(reinterpret_cast<const Vec*>(base), B_b, nkv, warp, gid, tig, lane,
                            acc);
    __syncthreads();
  }
  constexpr int S = B1 ? 0 : 3;
  if constexpr (B1) {
    // popc(a ^ w) = popc(w) + popc(a) - 2 * popc(a & w); out-of-bounds taps (a = 0) give popc(w)
    // GW: wg0 / wg1 = the window group of the tile's channels 0-31 / 32-63
    const bool wg0 = GW && c_tile / p.cout_pg != g, wg1 = GW && (c_tile + 32) / p.cout_pg != g;
#pragma unroll
    for (int ns = 0; ns < 8; ++ns) {
      const int2 pw = *reinterpret_cast<const int2*>(p.wpop + c_tile + ns * 8 + tig * 2);
#pragma unroll
      for (int ms = 0; ms < 2; ++ms)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          // GW: the popcount of the channel's own window group (pa[ms][e] holds group e & 1's)
          const int a = !GW ? pa[ms][e] : (ns < 4 ? wg0 : wg1) ? pa[ms][e | 1] : pa[ms][e & 2];
          acc[ms][ns][e] = (e & 1 ? pw.y : pw.x) + a - 2 * acc[ms][ns][e];
        }
    }
  }
  if (p.tap_popc != nullptr) zero_pad_correction_imma<S>(p, acc, m0, c_tile, warp, gid, tig);
  if constexpr (CHAIN) {
    // the chain's four 64-channel slices and the tile's multiplier / bias go to the shared memory
    // the last K chunk released (the loop ended on a barrier)
    float* cs = reinterpret_cast<float*>(smem_raw);
    for (int i = tid; i < 6 * kBN; i += kIThreads) {
      const int k = i / kBN;
      const float* v = k == 0   ? p.chain.shift_in
                       : k == 1 ? p.chain.alpha
                       : k == 2 ? p.chain.shift_out
                       : k == 3 ? p.chain.sign_shift
                       : k == 4 ? p.mul
                                : p.bias;
      cs[i] = v != nullptr && (!GW || c_tile + (i & (kBN - 1)) < p.cout)
                  ? __ldg(v + c_tile + (i & (kBN - 1)))
                  : 0.0f;
    }
    __syncthreads();
    epilogue_imma<OUT, S, true, false, false, false, GW>(p, acc, m0, c_tile, warp, gid, tig, cs);
  } else if constexpr (GATE) {
    // likewise the gated tail's per-channel vectors (slot 0 unused); the gate itself is per image
    // and is read per row
    float* cs = reinterpret_cast<float*>(smem_raw);
    for (int i = tid; i < 6 * kBN; i += kIThreads) {
      const int k = i / kBN;
      const float* v = k == 1   ? p.gate.alpha
                       : k == 2 ? p.gate.sign_scale
                       : k == 3 ? p.gate.sign_shift
                       : k == 4 ? p.mul
                       : k == 5 ? p.bias
                                : nullptr;
      cs[i] = v != nullptr && (!GW || c_tile + (i & (kBN - 1)) < p.cout)
                  ? __ldg(v + c_tile + (i & (kBN - 1)))
                  : 0.0f;
    }
    __syncthreads();
    epilogue_imma<OUT, S, false, true, false, SPATIAL, GW>(p, acc, m0, c_tile, warp, gid, tig, cs);
  } else if constexpr (FCMAX) {
    epilogue_fc_max(p, acc, m0, c_tile, warp, gid, tig);
  } else {
    epilogue_imma<OUT, S, false, false, SLICE, false, GW, SHUFFLE>(p, acc, m0, c_tile, warp, gid, tig);
  }
}

// ---- ABC-Net's multiple binary bases (lce_b200_bconv2d_bases_run) ----
// One layer y = sum over n, m of t_nm, t_nm = OutputTransform_nm(bconv(A_n, B_m)), with N input
// planes A_n and M weight bases B_m, then the BatchNorm, the optional shortcut and the next
// layer's shifted signs. The M bases' b1 fragments for the CTA's 64-channel tile stay in shared
// memory for the whole CTA (one TMA copy); the input planes stream through a two-deep ring:
// with reuse, one whole-K plane per ring slot, multiplied by all M bases; otherwise one K chunk
// per slot, gathered again for every base. One accumulator set: each finished term is folded
// into a float running sum exactly as its own plan would output it (clamp, then the unfused
// multiply and add), the sum starting from t_00 and adding the terms left to right in (n, m)
// order, as the converter's ADD chain does.
constexpr int kMaxBases = 8;
struct BasesParams {
  ConvKParams p;   // geometry, ring sizes, clamp, wt = [tile][M][n_slices] fragments,
                   // residual / residual_act (the shortcut ADD), out (NULL: not stored), cw_out
  const int32_t* planes[kMaxBases];   // the N packed input planes
  const float* tmul;                  // [M * N][ldc] folded multipliers, term n * M + m
  const float* tbias;                 // [M * N][ldc] folded biases
  const int32_t* wpop;                // [M][ldc] popcount of each base's filter rows
  int ldc, n_bases, n_planes, reuse;
  const float* bn_scale;              // MUL(bn_scale) -> ADD(bn_shift, bn_act)
  const float* bn_shift;
  int bn_act;
  int n_next;                         // the next layer's planes: bit = fl(out + shift) < 0
  float next_shift[kMaxBases];
  int32_t* next_planes[kMaxBases];
  unsigned w_bytes;                   // one tile's fragments of all M bases
};

// TFLite's fused activation as the float builtins apply it
__device__ __forceinline__ float bases_act(float x, int act) {
  switch (act) {
    case LCE_ACT_RELU: return fmaxf(x, 0.0f);
    case LCE_ACT_RELU_N1_TO_1: return fminf(fmaxf(x, -1.0f), 1.0f);
    case LCE_ACT_RELU6: return fminf(fmaxf(x, 0.0f), 6.0f);
    default: return x;
  }
}

template <int V>
__global__ void __launch_bounds__(kIThreads, 1) bconv_bases_kernel(const __grid_constant__ BasesParams bp) {
  const ConvKParams& p = bp.p;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t wbar;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int gid = lane >> 2, tig = lane & 3;
  const int nt = blockIdx.y;
  const long long m0 = static_cast<long long>(blockIdx.x) * kIBM;
  const int c_tile = nt * kBN, cth = c_tile + tig * 2;
  const int Kv_end = b1_padded_vectors(p.Kv, V);
  const int n_slices = (Kv_end * V + 7) >> 3;
  const int chunk_slices = (p.Kc_v * V + 7) >> 3;
  const int M = bp.n_bases, nc = p.n_chunks;
  const uint2* W_s = reinterpret_cast<const uint2*>(smem_raw);
  unsigned char* A_base = smem_raw + bp.w_bytes;
  const size_t a_bytes = static_cast<size_t>(chunk_slices) * kIBM * 32;

  if (tid == 0) {
    mbar_init(&wbar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(&wbar, bp.w_bytes);
    bulk_g2s(smem_raw, reinterpret_cast<const unsigned char*>(p.wt) + static_cast<size_t>(nt) * bp.w_bytes,
             bp.w_bytes, &wbar);
  }
  // unit u of the ring: plane n, chunk ch (reuse: the whole K of plane u)
  const int per_plane = bp.reuse ? 1 : M * nc;
  const int U = bp.n_planes * per_plane;
  auto stage = [&](int u) {
    const int n = u / per_plane;
    const int ch = bp.reuse ? 0 : (u - n * per_plane) % nc;
    const int kv0 = ch * p.Kc_v;
    const int kv1 = min(kv0 + p.Kc_v, Kv_end);
    gather_tile<V, kIBM, kIThreads, true>(p, reinterpret_cast<typename VecT<V>::T*>(A_base + (u & 1) * a_bytes),
                                         m0, 0, kv0, kv1, tid, bp.planes[n]);
    cp_async_commit();
  };

  int acc[2][8][4];
  int pa[2][4];
  float sum[2][2][16];
  auto clear = [&]() {
#pragma unroll
    for (int ms = 0; ms < 2; ++ms) {
#pragma unroll
      for (int e = 0; e < 4; ++e) pa[ms][e] = 0;
#pragma unroll
      for (int ns = 0; ns < 8; ++ns)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[ms][ns][e] = 0;
    }
  };
  clear();
  stage(0);
  for (int u = 0; u < U; ++u) {
    const bool more = u + 1 < U;
    if (more) stage(u + 1);   // its slot was released by the barrier that ended unit u - 1
    if (more) asm volatile("cp.async.wait_group 1;" ::: "memory");
    else asm volatile("cp.async.wait_group 0;" ::: "memory");
    if (u == 0) mbar_wait(&wbar, 0);
    __syncthreads();
    const uint32_t* A_b = reinterpret_cast<const uint32_t*>(A_base + (u & 1) * a_bytes);
    const int n = u / per_plane;
    const int r = u - n * per_plane;
    const int m_lo = bp.reuse ? 0 : r / nc, m_hi = bp.reuse ? M : m_lo + 1;
    const int ch = bp.reuse ? 0 : r % nc;
    const int kv0 = ch * p.Kc_v;
    const int words = (min(kv0 + p.Kc_v, Kv_end) - kv0) * V;
    for (int m = m_lo; m < m_hi; ++m) {
      compute_chunk_b1(A_b, W_s + (static_cast<size_t>(m) * n_slices + ch * chunk_slices) * 256, words,
                       warp, gid, tig, lane, acc, pa);
      if (ch != nc - 1) continue;
      // the finished term t_nm: popc(a ^ w), OutputTransform, then into the running sum
      const int term = n * M + m;
      const float* tm = bp.tmul + static_cast<size_t>(term) * bp.ldc + cth;
      const float* tb = bp.tbias + static_cast<size_t>(term) * bp.ldc + cth;
      const int32_t* wp = bp.wpop + static_cast<size_t>(m) * bp.ldc + cth;
#pragma unroll
      for (int ns = 0; ns < 8; ++ns) {
        const int2 pw = __ldg(reinterpret_cast<const int2*>(wp + ns * 8));
        const float2 mu = __ldg(reinterpret_cast<const float2*>(tm + ns * 8));
        const float2 bi = __ldg(reinterpret_cast<const float2*>(tb + ns * 8));
#pragma unroll
        for (int ms = 0; ms < 2; ++ms)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int x0 = (pw.x + pa[ms][h * 2] - 2 * acc[ms][ns][h * 2]) << 1;
            const int x1 = (pw.y + pa[ms][h * 2 + 1] - 2 * acc[ms][ns][h * 2 + 1]) << 1;
            const float y0 = transform_float_x2(x0, p.clamp_min, p.clamp_max, mu.x, bi.x);
            const float y1 = transform_float_x2(x1, p.clamp_min, p.clamp_max, mu.y, bi.y);
            sum[ms][h][2 * ns] = term == 0 ? y0 : __fadd_rn(sum[ms][h][2 * ns], y0);
            sum[ms][h][2 * ns + 1] = term == 0 ? y1 : __fadd_rn(sum[ms][h][2 * ns + 1], y1);
          }
      }
      clear();
    }
    __syncthreads();
  }

  // MUL(bn_scale) -> ADD(bn_shift, bn_act) [-> ADD(shortcut, residual_act)], then the next planes
  const bool has_res = p.residual != nullptr;
  float* out = static_cast<float*>(p.out);
#pragma unroll
  for (int ms = 0; ms < 2; ++ms) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long m = m0 + warp * 32 + ms * 16 + h * 8 + gid;
      const bool row_ok = m < p.M;
      float* y = sum[ms][h];
      if (row_ok) {
        const size_t e0 = static_cast<size_t>(m) * p.cout + cth;
#pragma unroll
        for (int ns = 0; ns < 8; ++ns) {
          const float2 s = __ldg(reinterpret_cast<const float2*>(bp.bn_scale + cth + ns * 8));
          const float2 t = __ldg(reinterpret_cast<const float2*>(bp.bn_shift + cth + ns * 8));
          y[2 * ns] = bases_act(__fadd_rn(__fmul_rn(y[2 * ns], s.x), t.x), bp.bn_act);
          y[2 * ns + 1] = bases_act(__fadd_rn(__fmul_rn(y[2 * ns + 1], s.y), t.y), bp.bn_act);
        }
        if (has_res) {
#pragma unroll
          for (int ns = 0; ns < 8; ++ns) {
            const float2 rv = __ldg(reinterpret_cast<const float2*>(p.residual + e0 + ns * 8));
            y[2 * ns] = bases_act(__fadd_rn(y[2 * ns], rv.x), p.residual_act);
            y[2 * ns + 1] = bases_act(__fadd_rn(y[2 * ns + 1], rv.y), p.residual_act);
          }
        }
        if (out != nullptr) {
#pragma unroll
          for (int ns = 0; ns < 8; ++ns)
            *reinterpret_cast<float2*>(out + e0 + ns * 8) = make_float2(y[2 * ns], y[2 * ns + 1]);
        }
      }
      // LceQuantize(ADD(out, shift)): bit = fl(out + shift) < 0 (bitpack.h:159); the shuffles are
      // uniform across the warp
      for (int k = 0; k < bp.n_next; ++k) {
        const float sh = bp.next_shift[k];
        uint32_t bits0 = 0, bits1 = 0;
#pragma unroll
        for (int ns = 0; ns < 4; ++ns) {
          bits0 |= ((__fadd_rn(y[2 * ns], sh) < 0.0f ? 1u : 0u) |
                    (__fadd_rn(y[2 * ns + 1], sh) < 0.0f ? 2u : 0u)) << (ns * 8);
          bits1 |= ((__fadd_rn(y[2 * ns + 8], sh) < 0.0f ? 1u : 0u) |
                    (__fadd_rn(y[2 * ns + 9], sh) < 0.0f ? 2u : 0u)) << (ns * 8);
        }
        bits0 <<= tig * 2;
        bits1 <<= tig * 2;
        bits0 |= __shfl_xor_sync(0xffffffffu, bits0, 1);
        bits1 |= __shfl_xor_sync(0xffffffffu, bits1, 1);
        bits0 |= __shfl_xor_sync(0xffffffffu, bits0, 2);
        bits1 |= __shfl_xor_sync(0xffffffffu, bits1, 2);
        if (row_ok && tig == 0) {
          int32_t* pk = bp.next_planes[k] + static_cast<size_t>(m) * p.cw_out + (c_tile >> 5);
          pk[0] = static_cast<int32_t>(bits0);
          pk[1] = static_cast<int32_t>(bits1);
        }
      }
    }
  }
}

}  // namespace lce
#endif

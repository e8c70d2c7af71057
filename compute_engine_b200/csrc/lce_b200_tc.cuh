// lce_b200_tc.cuh -- the binary convolution / BGEMM on the Hopper tensor cores (wgmma).
//
//   acc[m][n] = sum_k popc(a[m][k] ^ w[n][k]) = popc(w[n]) + sum_k a_k * w'_k
//   a_k in {0,1},  w'_k = +1 if w_k = 0 else -1            (same identity as lce_b200_imma.cuh)
//
// so the reference's integers (LCE/core/bconv2d/reference.h:35-148, bgemm/kernels.h:22-134) come
// out of one int8 contraction, issued here as wgmma.mma_async .s32.s8.s8 (m64 x BN x k32). HBM, L2
// and the TMA-staged activation tiles keep the reference's BITPACKED words (types.h:41-47); bytes
// exist only in registers (activations) and in a plan-time expansion of the static weights.
//
// Persistent CTAs (two per SM where shared memory allows), 10 warps, warp-specialised:
//   w8        activation producer  TMA (cp.async.bulk.tensor) of the packed HALO of a 128-pixel
//                                  tile: the contiguous pixel range its taps touch, once per tile --
//                                  no im2col replication anywhere
//   w9        weight producer      cp.async.bulk of pre-expanded int8 stages (resident in shared
//                                  memory for the whole kernel when they fit, else a ring)
//   w0..w7    two math warpgroups  warpgroup g owns pixels 64g..64g+63 of the tile. Each thread
//                                  reads its two pixels' words from the halo (out-of-bounds taps
//                                  read as 0 = "+1" padding, reference.h:106) and expands them
//                                  straight into its wgmma A fragment: bit 8i+s of a word becomes
//                                  byte i of K column group s with VALUE 2^(s&3); the weight byte
//                                  there is +-(8 >> (s&3)), so every product is +-8 and D holds
//                                  8 * sum a*w'. The accumulators stay in registers through the
//                                  epilogue: OutputTransform (output_transform.h:94-168, unfused
//                                  fmul + fadd) [+ shortcut, activation, next layer's sign bits].
// Stage = 8 K-words = 256 bits of K = eight k32 MMAs.
#ifndef LCE_B200_TC_CUH_
#define LCE_B200_TC_CUH_

#include <cuda.h>

#include "lce_b200_kernels.cuh"

namespace lce {
namespace tc {

constexpr int kBM = 128;
constexpr int kNumMathWarps = 8;  // two warpgroups of four
constexpr int kWarpActProd = kNumMathWarps, kWarpWeightProd = kNumMathWarps + 1;
constexpr int kThreads = (kNumMathWarps + 2) * 32;
constexpr int kWS = 8;            // K words per stage
constexpr int kNR = 2;            // activation-halo stages
constexpr int kMaxNB = 32;        // weight stages in shared memory (barrier array size)
constexpr int kMaxRing = 4;       // weight ring slots when the weights do not stay resident
constexpr int kBarBytes = 1024;

struct TcParams {
  long long M;           // output pixels (< 2^31)
  long long total_px;    // input pixels batch * H * W
  int H, W, OH, OW, KH, KW, sh, sw, dh, dw, ph, pw;
  int taps;
  int Cw;                // channel words per pixel
  int CcB;               // words per pixel in a halo stage (box width; == Cw in flat mode)
  int n_chunks;          // channel chunks of CcB words
  int mode_flat;         // 1: 1-D word map, boxes of 256 words; 0: 2-D [pixel][word] map, boxes of CcB x 128
  int cout, BN, n_tiles, m_tiles;
  int S_full, S_last, S_t;   // weight stages per full / last chunk, per tile
  int nB, b_resident;    // ring: nB slots of kWS words
  int raw_stage_bytes;
  int off_raw, off_bar;  // byte offsets in dynamic shared memory (weights at 0)
  int Kw_total;          // taps * Cw: K words per output channel
  int clamp_min, clamp_max;
  int has_res, residual_act, cw_out, zp_half, ldc;   // ldc: padded channel count of the tables
  int zp_float, cin_pg;  // zero padding as the optimised reference kernels do it (float correction)
  const uint8_t* wt;       // [n_tiles][stage][BN x (32 * words) B core-matrix image], stages dense
  const float* mul;        // folded multiplier / bias, padded to n_tiles * BN
  const float* bias;
  const int32_t* wpop2;    // 2 * popcount of each channel's filter row
  const int32_t* thr;
  const int32_t* tap_popc_t;  // [taps][ldc] or nullptr (zero-padding correction)
  const float* zpc_cache;     // [4][eff_h][eff_w][ldc]: the optimised kernels' float corrections (zp_float)
  const float* residual;      // [M][cout] shortcut of a fused ADD (has_res)
  void* out;
  int32_t* packed_out;
  FastDiv fd_ohw, fd_ow, fd_kw, fd_mt;
};

// ------------------------------------------------------------------ PTX
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Deadlock watchdog (development aid, costs one counter per wait): a wait that does not complete
// within ~2 s records who was waiting on what in g_tc_dbg, raises g_tc_abort, and every later wait
// returns at once so the kernel terminates and the host can read the record (lce_b200_tc_debug).
__device__ int g_tc_abort = 0;
__device__ int g_tc_dbg[8] = {0, 0, 0, 0, 0, 0, 0, 0};
__device__ __forceinline__ bool mbar_try(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  // the suspend-time hint (ns) lets a waiting warp sleep in hardware instead of spinning through
  // the issue slots of the busy warps next to it; an arrival still wakes it at once
  asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\nselp.u32 %0, 1, 0, p;\n}\n"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity), "r"(20000u) : "memory");
  return ok != 0;
}
__device__ __noinline__ void tc_watchdog_fire(int tag, uint32_t parity, uint32_t cnt) {
  if (atomicCAS(&g_tc_abort, 0, 1) == 0) {
    g_tc_dbg[0] = tag; g_tc_dbg[1] = static_cast<int>(blockIdx.x); g_tc_dbg[2] = static_cast<int>(threadIdx.x);
    g_tc_dbg[3] = static_cast<int>(parity); g_tc_dbg[4] = static_cast<int>(cnt);
  }
}
__device__ __forceinline__ void mbar_wait_tc(uint64_t* bar, uint32_t parity, int tag = 0, uint32_t cnt = 0) {
  if (mbar_try(bar, parity)) return;
  const long long t0 = clock64();
  for (uint32_t i = 1;; ++i) {
    if (mbar_try(bar, parity)) return;
    if ((i & 255u) == 0) {
      if (*reinterpret_cast<volatile int*>(&g_tc_abort) != 0) return;
      if (clock64() - t0 > 4000000000LL) {
        tc_watchdog_fire(tag, parity, cnt);
        return;
      }
    }
  }
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n.reg .pred P;\nelect.sync _|P, 0xffffffff;\nselp.u32 %0, 1, 0, P;\n}\n" : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void tma_load_1d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0) {
  asm volatile("cp.async.bulk.tensor.1d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3}], [%2];" ::"r"(smem_u32(dst)),
               "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
               "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// TMA store of one box from shared memory; the issuing thread tracks it as a bulk async-group
// (elements outside the tensor are not written)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* tm, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(tm)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// this thread's bulk stores have finished reading shared memory (it may be overwritten)
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... and their writes are complete
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// wgmma: issued by all 128 threads of a warpgroup. A comes from registers, B from a shared-memory
// descriptor, D stays in registers. The fence orders this thread's register writes (A fragments,
// accumulators read by the previous epilogue) before the asynchronous reads; the empty asm
// statements keep the compiler from moving register accesses across the commit / wait.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void fence_regs(uint32_t (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(r[i])::"memory");
}
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
// Shared-memory matrix descriptor (sm_90): start address, leading / stride byte offsets >> 4,
// layout type in bits 62-63 (0 = no swizzle, 1 = 128-byte swizzle).
__device__ __forceinline__ uint64_t make_desc(uint32_t lo, uint32_t hi) {
  return (static_cast<uint64_t>(hi) << 32) | lo;
}
// B operand, K-major, no swizzle: 8 x 16 B core matrices, K-adjacent ones 128 B apart (LBO),
// 8-row groups `sbo` bytes apart.
__device__ __forceinline__ uint32_t bdesc_lo(uint32_t saddr) { return ((saddr & 0x3FFFFu) >> 4) | ((128u >> 4) << 16); }
__device__ __forceinline__ uint32_t bdesc_hi(uint32_t sbo) { return sbo >> 4; }

// ------------------------------------------------------------------ index helpers
struct Pixel { int b, oy, ox; };
__device__ __forceinline__ Pixel split_px(const TcParams& p, uint32_t m) {
  Pixel r;
  const uint32_t bb = fdiv(m, p.fd_ohw);
  const uint32_t rem = m - bb * static_cast<uint32_t>(p.OH * p.OW);
  const uint32_t y = fdiv(rem, p.fd_ow);
  r.b = static_cast<int>(bb);
  r.oy = static_cast<int>(y);
  r.ox = static_cast<int>(rem - y * static_cast<uint32_t>(p.OW));
  return r;
}
// The contiguous range of input pixels (flattened (b, y, x)) that the taps of tile m0 touch. The
// flattened index of (pixel m, tap) grows with m and with the tap, so the range runs from the first
// pixel's first tap to the last pixel's last tap, clipped to the tensor.
__device__ __forceinline__ void tile_halo(const TcParams& p, long long m0, long long* px_lo, int* px_cnt) {
  const long long m1 = min(m0 + kBM, p.M) - 1;
  const Pixel a = split_px(p, static_cast<uint32_t>(m0));
  const Pixel z = split_px(p, static_cast<uint32_t>(m1));
  long long lo = (static_cast<long long>(a.b) * p.H + (a.oy * p.sh - p.ph)) * p.W + (a.ox * p.sw - p.pw);
  long long hi = (static_cast<long long>(z.b) * p.H + (z.oy * p.sh - p.ph + (p.KH - 1) * p.dh)) * p.W +
                 (z.ox * p.sw - p.pw + (p.KW - 1) * p.dw) + 1;
  lo = max(lo, 0LL);
  hi = min(hi, p.total_px);
  if (lo > p.total_px - 1) lo = p.total_px - 1;
  *px_lo = lo;
  *px_cnt = static_cast<int>(max(hi - lo, 1LL));
}
// first word held by the halo stage (the TMA start coordinate must be 16-byte aligned)
__device__ __forceinline__ long long halo_word_base(const TcParams& p, long long px_lo) {
  return p.mode_flat ? ((px_lo * p.Cw) & ~3LL) : px_lo * p.CcB;
}

// Zero padding with the reference kernel's integers (zp_float == 0): the out-of-bounds taps of
// output pixel (oy, ox), each of which contributes cin_pg / 2 instead of popc(0 ^ w)
// (reference.h:100-103).
__device__ __forceinline__ unsigned long long zero_pad_tap_mask(const TcParams& p, int oy, int ox) {
  unsigned long long mask = 0;
  const int iy0 = oy * p.sh - p.ph, ix0 = ox * p.sw - p.pw;
  for (int fy = 0; fy < p.KH; ++fy)
    for (int fx = 0; fx < p.KW; ++fx) {
      const int iy = iy0 + fy * p.dh, ix = ix0 + fx * p.dw;
      if (!(static_cast<unsigned>(iy) < static_cast<unsigned>(p.H) && static_cast<unsigned>(ix) < static_cast<unsigned>(p.W)))
        mask |= 1ull << (fy * p.KW + fx);
    }
  return mask;
}
// Zero padding as the optimised kernels do it (zp_float == 1): the row of the correction cache
// that ApplyCorrection adds to output pixel (oy, ox), or -1 -- its case analysis restated
// literally (zero_padding_correction.h:189-285), "cannot happen" fall-through included.
__device__ __forceinline__ int zero_pad_cache_row(const TcParams& p, int oy, int ox) {
  const int eff_w = (p.KW - 1) * p.dw + 1, eff_h = (p.KH - 1) * p.dh + 1;
  const int left_off = ((p.OW - 1) * p.sw + eff_w - p.W) / 2;
  const int top_off = ((p.OH - 1) * p.sh + eff_h - p.H) / 2;
  const int o_top = top_off - oy * p.sh, o_bot = -o_top - p.H + eff_h;
  const int o_left = left_off - ox * p.sw, o_right = -o_left - p.W + eff_w;
  if (o_left <= 0 && o_right <= 0 && o_top <= 0 && o_bot <= 0) return -1;
  int cs, X, Y;
  if (o_right <= 0 && o_top > 0 && o_bot < 0) { cs = 0; X = max(o_left, 0); Y = o_top; }
  else if (o_left < 0 && o_right > 0 && o_bot <= 0) { cs = 1; X = o_right; Y = max(o_top, 0); }
  else if (o_left > 0 && o_right < 0 && o_top <= 0) { cs = 2; X = o_left; Y = max(o_bot, 0); }
  else if (o_left <= 0 && o_top < 0 && o_bot > 0) { cs = 3; X = max(o_right, 0); Y = o_bot; }
  else return -1;
  if (X >= eff_w || Y >= eff_h) return -1;   // outside the cache: images smaller than the filter
  return (cs * eff_h + Y) * eff_w + X;
}
// Plan time: CacheCorrectionValues (zero_padding_correction.h:39-176):
// cache[case][y][x][c] = (-post_mul[c]) * sum over the taps the case counts of (cin_pg - 2 popc(tap)).
// `mul` is the folded multiplier, which for float output IS -post_mul (bconv2d.cc:369-372).
__global__ void zpc_cache_kernel(const int32_t* __restrict__ tap_popc_t, const float* __restrict__ mul,
                                 float* __restrict__ cache, int cout, int ldc, int KH, int KW, int dh, int dw,
                                 int cin_pg) {
  const int eff_w = (KW - 1) * dw + 1, eff_h = (KH - 1) * dh + 1;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= 4 * eff_h * eff_w * cout) return;
  const int c = idx % cout;
  int r = idx / cout;
  const int x = r % eff_w;
  r /= eff_w;
  const int y = r % eff_h, cs = r / eff_h;
  float corr = 0.0f;
  for (int fy = 0; fy < KH; ++fy)
    for (int fx = 0; fx < KW; ++fx) {
      const int efx = dw * fx, efy = dh * fy;
      bool counted;
      if (cs == 0) counted = efy < y || efx < x;
      else if (cs == 1) counted = efy < y || (eff_w - efx) <= x;
      else if (cs == 2) counted = (eff_h - efy) <= y || efx < x;
      else counted = (eff_h - efy) <= y || (eff_w - efx) <= x;
      if (counted) corr = __fadd_rn(corr, static_cast<float>(cin_pg - 2 * tap_popc_t[static_cast<size_t>(fy * KW + fx) * ldc + c]));
    }
  cache[static_cast<size_t>((cs * eff_h + y) * eff_w + x) * ldc + c] = __fmul_rn(mul[c], corr);
}

// bit 8i+s of w -> byte i of v[s], value 2^(s&3): 9 ALU instructions
__device__ __forceinline__ void expand_word(uint32_t w, uint32_t* v) {
  v[0] = w & 0x01010101u; v[1] = w & 0x02020202u; v[2] = w & 0x04040404u; v[3] = w & 0x08080808u;
  const uint32_t h = w >> 4;
  v[4] = h & 0x01010101u; v[5] = h & 0x02020202u; v[6] = h & 0x04040404u; v[7] = h & 0x08080808u;
}

// Plan time: the weights as the exact shared-memory images the MMA reads. K words run in the
// order (channel chunk, tap, word); each chunk is cut into stages of kWS words; a stage of nw words
// is [BN / 8 row groups][2 * nw core matrices][8 rows][16 B] (no-swizzle K-major, row-group pitch
// nw * 256 B) and the stages of one n tile follow one another without padding.
// One thread per (n tile, K word, row) writes that word's 32 bytes.
__global__ void expand_weights_tc_kernel(const int32_t* __restrict__ filter, uint8_t* __restrict__ wt, int cout, int taps,
                                         int Cw, int CcB, int BN, long long total) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= total) return;
  const int Kw = taps * Cw;
  const int n = static_cast<int>(idx % BN);
  long long r = idx / BN;
  const int qg = static_cast<int>(r % Kw);
  const int nt = static_cast<int>(r / Kw);
  const int chunk_words = taps * CcB;
  const int chunk = qg / chunk_words;
  const int rem = qg - chunk * chunk_words;
  const int cc_this = min(CcB, Cw - chunk * CcB);
  const int st = rem / kWS, j = rem - st * kWS;
  const int nw = min(kWS, taps * cc_this - st * kWS);
  const int tap = rem / cc_this, cwi = rem - tap * cc_this;
  const int c = nt * BN + n;
  uint32_t bytes[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (c < cout) {
    const uint32_t w = static_cast<uint32_t>(filter[(static_cast<long long>(c) * taps + tap) * Cw + chunk * CcB + cwi]);
    for (int kk = 0; kk < 32; ++kk) {
      const int s = kk >> 2, i = kk & 3;
      const int mag = 8 >> (s & 3);
      const int v = ((w >> (8 * i + s)) & 1u) ? -mag : mag;
      bytes[kk >> 2] |= (static_cast<uint32_t>(v) & 0xFFu) << (8 * (kk & 3));
    }
  }
  uint8_t* dst = wt + (static_cast<long long>(nt) * Kw + chunk * chunk_words + st * kWS) * BN * 32 +
                 (n >> 3) * (nw * 256) + (2 * j) * 128 + (n & 7) * 16;
  *reinterpret_cast<uint4*>(dst) = make_uint4(bytes[0], bytes[1], bytes[2], bytes[3]);
  *reinterpret_cast<uint4*>(dst + 128) = make_uint4(bytes[4], bytes[5], bytes[6], bytes[7]);
}
// tap_popc_t[t][c] = popcount of filter[c][t][:] (transposed for the epilogue's per-pixel rows)
__global__ void tap_popc_t_kernel(const int32_t* __restrict__ filter, int32_t* __restrict__ out, int cout, int taps, int Cw,
                                  int ldc) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= cout * taps) return;
  const int c = idx / taps, t = idx - c * taps;
  const int32_t* f = filter + static_cast<size_t>(idx) * Cw;
  int s = 0;
  for (int w = 0; w < Cw; ++w) s += __popc(static_cast<uint32_t>(f[w]));
  out[static_cast<size_t>(t) * ldc + c] = s;
}
__global__ void wpop2_kernel(const int32_t* __restrict__ filter, int32_t* __restrict__ out, int cout, int Kw) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cout) return;
  const int32_t* f = filter + static_cast<size_t>(c) * Kw;
  int s = 0;
  for (int w = 0; w < Kw; ++w) s += __popc(static_cast<uint32_t>(f[w]));
  out[c] = 2 * s;
}

// ------------------------------------------------------------------ wgmma, A from registers
__device__ __forceinline__ void wgmma_s8_n32(uint32_t (&d)[16], const uint32_t (&a)[4], uint64_t desc, uint32_t scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, "
               "{%16,%17,%18,%19}, %20, p;\n}\n"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
                 "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_s8_n64(uint32_t (&d)[32], const uint32_t (&a)[4], uint64_t desc, uint32_t scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
               "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
               "{%32,%33,%34,%35}, %36, p;\n}\n"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
                 "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
                 "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
                 "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t desc, uint32_t scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
               "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
               "{%32,%33,%34,%35}, %36, p, 1, 1;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                 "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                 "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                 "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t desc, uint32_t scale_d) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
               "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
               "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
               "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
               "{%64,%65,%66,%67}, %68, p, 1, 1;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                 "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                 "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                 "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                 "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                 "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                 "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                 "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"(scale_d));
}

// ------------------------------------------------------------------ the kernel
template <int BN>
__device__ __forceinline__ void wgmma_s8(uint32_t (&d)[BN / 2], const uint32_t (&a)[4], uint64_t desc, uint32_t scale_d) {
  if constexpr (BN == 64) wgmma_s8_n64(d, a, desc, scale_d);
  else wgmma_s8_n32(d, a, desc, scale_d);
}

// the NW k32 MMAs of one stage (K word j of the stage image starts 256 B after word j - 1)
template <int BN, int NW>
__device__ __forceinline__ void wgmma_stage(uint32_t (&acc)[BN / 2], uint32_t (&a)[kWS][4], uint32_t lo, uint32_t hi,
                                            uint32_t scale_d) {
#pragma unroll
  for (int j = 0; j < NW; ++j) wgmma_s8<BN>(acc, a[j], make_desc(lo + j * 16, hi), j == 0 ? scale_d : 1u);
}

// OR of a 32-channel sign / threshold word over the four threads of a quad (each holds 8 channels)
__device__ __forceinline__ uint32_t quad_or(uint32_t v) {
  v |= __shfl_xor_sync(0xffffffffu, v, 1);
  v |= __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// Compiled for two CTAs per SM: one CTA's epilogue and halo waits overlap the other's MMAs.
template <int V, int OUT, int BN>
__global__ void __launch_bounds__(kThreads, 2)
bconv_tc_kernel(const __grid_constant__ CUtensorMap tm_in, const TcParams p) {
  extern __shared__ __align__(1024) unsigned char smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.off_bar);
  uint64_t* b_full = bars;                     // [kMaxNB]
  uint64_t* b_empty = b_full + kMaxNB;         // [kMaxNB]
  uint64_t* raw_full = b_empty + kMaxNB;       // [kNR]
  uint64_t* raw_empty = raw_full + kNR;        // [kNR]

  const int tid = threadIdx.x;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // provably warp-uniform
  const int lane = tid & 31;

  if (tid == 0) {
    for (int i = 0; i < kMaxNB; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], kNumMathWarps); }
    for (int i = 0; i < kNR; ++i) { mbar_init(&raw_full[i], 1); mbar_init(&raw_empty[i], kNumMathWarps); }
    fence_barrier_init();
  }
  __syncthreads();

  const int n_items = p.n_tiles * p.m_tiles;
  const int cc_last = p.Cw - (p.n_chunks - 1) * p.CcB;   // words per pixel in the last channel chunk
  const uint32_t row32 = static_cast<uint32_t>(BN) * 32u;   // bytes of one K word of a stage image

  if (warp == kWarpActProd) {
    // ===== activation producer =====
    if (lane == 0) {
      uint32_t cnt = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int nt = static_cast<int>(fdiv(static_cast<uint32_t>(item), p.fd_mt));
        const long long m0 = static_cast<long long>(item - nt * p.m_tiles) * kBM;
        long long px_lo;
        int px_cnt;
        tile_halo(p, m0, &px_lo, &px_cnt);
        const long long wbase = halo_word_base(p, px_lo);
        for (int ch = 0; ch < p.n_chunks; ++ch, ++cnt) {
          const int rs = cnt % kNR;
          mbar_wait_tc(&raw_empty[rs], ((cnt / kNR) & 1) ^ 1, 1);
          unsigned char* dst = smem + p.off_raw + rs * p.raw_stage_bytes;
          if (p.mode_flat) {
            const int nwords = static_cast<int>((px_lo + px_cnt) * p.Cw - wbase);
            const int nbox = (nwords + 255) >> 8;
            mbar_arrive_expect_tx(&raw_full[rs], nbox * 1024);
            for (int i = 0; i < nbox; ++i) tma_load_1d(dst + i * 1024, &tm_in, &raw_full[rs], static_cast<int>(wbase) + i * 256);
          } else {
            const int nbox = (px_cnt + 127) >> 7;
            const int box_bytes = 128 * p.CcB * 4;
            mbar_arrive_expect_tx(&raw_full[rs], nbox * box_bytes);
            for (int i = 0; i < nbox; ++i)
              tma_load_2d(dst + i * box_bytes, &tm_in, &raw_full[rs], ch * p.CcB, static_cast<int>(px_lo) + i * 128);
          }
        }
      }
    }
  } else if (warp == kWarpWeightProd) {
    // ===== weight producer =====
    if (lane == 0) {
      uint32_t bs = 0, slot = 0, par = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int nt = static_cast<int>(fdiv(static_cast<uint32_t>(item), p.fd_mt));
        const uint8_t* src = p.wt + static_cast<size_t>(nt) * p.Kw_total * row32;
        uint32_t wofs = 0;
        for (int ch = 0; ch < p.n_chunks; ++ch) {
          const int nq = p.taps * (ch == p.n_chunks - 1 ? cc_last : p.CcB);
          for (int q0 = 0; q0 < nq; q0 += kWS) {
            const int nw = min(kWS, nq - q0);
            const uint32_t bytes = static_cast<uint32_t>(nw) * row32;
            if (p.b_resident) {
              mbar_arrive_expect_tx(&b_full[bs], bytes);
              bulk_g2s(smem + wofs * row32, src + static_cast<size_t>(wofs) * row32, bytes, &b_full[bs]);
              ++bs;
            } else {
              mbar_wait_tc(&b_empty[slot], par ^ 1, 5);
              mbar_arrive_expect_tx(&b_full[slot], bytes);
              bulk_g2s(smem + slot * (row32 * kWS), src + static_cast<size_t>(wofs) * row32, bytes, &b_full[slot]);
              if (++slot == static_cast<uint32_t>(p.nB)) { slot = 0; par ^= 1; }
            }
            wofs += nw;
          }
        }
        if (p.b_resident) break;   // loaded once, kept for every tile of this CTA
      }
    }
  } else {
    // ===== math warpgroups: thread (g, t) of warp w holds pixels r0 = 64 * wg + 16 * (w & 3) + g
    // and r0 + 8, K bytes 4t..4t+3 and 16+4t..16+4t+3 of each k32 step, and channels
    // 8j + 2t, 8j + 2t + 1 of every 8-channel block j of the accumulator.
    const int wg = warp >> 2;
    const int g = lane >> 2, t = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + g;
    const int pitch = p.mode_flat ? p.Cw : p.CcB;
    const uint32_t tmask = 0x01010101u << t;
    const uint32_t smem_base = smem_u32(smem);
    constexpr int VPS = kWS / V;   // vectors per stage
    const float act_lo = p.residual_act == LCE_ACT_RELU_N1_TO_1 ? -1.0f : 0.0f;
    const float act_hi = p.residual_act == LCE_ACT_RELU ? __int_as_float(0x7f800000)
                                                        : (p.residual_act == LCE_ACT_RELU6 ? 6.0f : 1.0f);
    uint32_t cntR = 0, slot = 0, par = 0;
    bool first_item = true;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x, first_item = false) {
      const int nt = static_cast<int>(fdiv(static_cast<uint32_t>(item), p.fd_mt));
      const long long m0 = static_cast<long long>(item - nt * p.m_tiles) * kBM;
      long long px_lo;
      int px_cnt;
      tile_halo(p, m0, &px_lo, &px_cnt);
      const long long wbase = halo_word_base(p, px_lo);
      long long m[2];
      bool row_ok[2];
      int iy0[2], ix0[2], off0[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        m[i] = m0 + r0 + 8 * i;
        row_ok[i] = m[i] < p.M;
        iy0[i] = ix0[i] = off0[i] = 0;
        if (row_ok[i]) {
          const Pixel px = split_px(p, static_cast<uint32_t>(m[i]));
          iy0[i] = px.oy * p.sh - p.ph;
          ix0[i] = px.ox * p.sw - p.pw;
          // word offset of (this pixel's tap (0,0), channel word 0) inside the halo stage
          off0[i] = static_cast<int>(((static_cast<long long>(px.b) * p.H + iy0[i]) * p.W + ix0[i]) * pitch - wbase);
        }
      }
      uint32_t acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0;
      uint32_t scale_d = 0;
      uint32_t wofs = 0, bs = 0;   // K-word offset / stage index inside the tile's weights
      for (int ch = 0; ch < p.n_chunks; ++ch, ++cntR) {
        const int rs = cntR % kNR;
        const int cwv = (ch == p.n_chunks - 1 ? cc_last : p.CcB) / V;
        const int nvec = p.taps * cwv;
        const uint32_t* raw = reinterpret_cast<const uint32_t*>(smem + p.off_raw + rs * p.raw_stage_bytes);
        mbar_wait_tc(&raw_full[rs], (cntR / kNR) & 1, 7);
        int kv = 0, cv = 0, fy = 0, fx = 0;
        while (kv < nvec) {
          const int nw = min(kWS, (nvec - kv) * V);
          uint32_t b_addr;
          if (p.b_resident) {
            b_addr = smem_base + wofs * row32;
            if (first_item) mbar_wait_tc(&b_full[bs], 0, 3);
          } else {
            b_addr = smem_base + slot * (row32 * kWS);
            mbar_wait_tc(&b_full[slot], par, 4);
          }
          // the stage's A fragments: two pixels x kWS words, expanded in registers
          uint32_t a[kWS][4];
#pragma unroll
          for (int u = 0; u < VPS; ++u, ++kv) {
            uint32_t w[2][V];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
#pragma unroll
              for (int e = 0; e < V; ++e) w[i][e] = 0;
              const int iy = iy0[i] + fy * p.dh, ix = ix0[i] + fx * p.dw;
              if (row_ok[i] && kv < nvec && static_cast<unsigned>(iy) < static_cast<unsigned>(p.H) &&
                  static_cast<unsigned>(ix) < static_cast<unsigned>(p.W))
                load_words<V>(reinterpret_cast<const typename VecT<V>::T*>(raw + off0[i] + (fy * p.dh * p.W + fx * p.dw) * pitch + cv * V),
                              w[i]);
            }
#pragma unroll
            for (int e = 0; e < V; ++e) {
              uint32_t* f = a[u * V + e];
              f[0] = w[0][e] & tmask;
              f[1] = w[1][e] & tmask;
              f[2] = (w[0][e] >> 4) & tmask;
              f[3] = (w[1][e] >> 4) & tmask;
            }
            if (++cv == cwv) {
              cv = 0;
              if (++fx == p.KW) { fx = 0; ++fy; }
            }
          }
#pragma unroll
          for (int j = 0; j < kWS; ++j) fence_regs(a[j]);
          wgmma_fence();
          const uint32_t lo = bdesc_lo(b_addr);
          const uint32_t hi = bdesc_hi(static_cast<uint32_t>(nw) * 256u);
          // straight-line sequences: a predicated wgmma would make ptxas serialise the stage
          switch (nw) {
            case 8: wgmma_stage<BN, 8>(acc, a, lo, hi, scale_d); break;
            case 7: wgmma_stage<BN, 7>(acc, a, lo, hi, scale_d); break;
            case 6: wgmma_stage<BN, 6>(acc, a, lo, hi, scale_d); break;
            case 5: wgmma_stage<BN, 5>(acc, a, lo, hi, scale_d); break;
            case 4: wgmma_stage<BN, 4>(acc, a, lo, hi, scale_d); break;
            case 3: wgmma_stage<BN, 3>(acc, a, lo, hi, scale_d); break;
            case 2: wgmma_stage<BN, 2>(acc, a, lo, hi, scale_d); break;
            default: wgmma_stage<BN, 1>(acc, a, lo, hi, scale_d); break;
          }
          scale_d = 1;
          wgmma_commit();
          wgmma_wait_all();
          fence_regs(acc);
          if (!p.b_resident) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&b_empty[slot]);
            if (++slot == static_cast<uint32_t>(p.nB)) { slot = 0; par ^= 1; }
          }
          wofs += nw;
          ++bs;
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&raw_empty[rs]);
      }

      // ---- epilogue, from the accumulator registers
      const int c_tile = nt * BN;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        // zero padding: the reference kernel's out-of-bounds taps, or the optimised kernels' cache row
        unsigned long long oob = 0;
        int zrow = -1;
        if (p.tap_popc_t != nullptr && row_ok[i]) {
          const Pixel px = split_px(p, static_cast<uint32_t>(m[i]));
          if (p.zp_float) zrow = zero_pad_cache_row(p, px.oy, px.ox);
          else oob = zero_pad_tap_mask(p, px.oy, px.ox);
        }
        // x = 2 * acc = (acc8 >> 2) + 2 * popc(w)   (acc8 is a multiple of 8)
        int x[BN / 4];
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = c_tile + 8 * j + 2 * t;
          x[2 * j] = (static_cast<int>(acc[4 * j + 2 * i]) >> 2) + __ldg(p.wpop2 + c);
          x[2 * j + 1] = (static_cast<int>(acc[4 * j + 2 * i + 1]) >> 2) + __ldg(p.wpop2 + c + 1);
        }
        for (unsigned long long mk = oob; mk != 0; mk &= mk - 1) {
          const int tp = __ffsll(static_cast<long long>(mk)) - 1;
          const int32_t* tpc = p.tap_popc_t + static_cast<size_t>(tp) * p.ldc + c_tile + 2 * t;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            x[2 * j] += 2 * (p.zp_half - __ldg(tpc + 8 * j));
            x[2 * j + 1] += 2 * (p.zp_half - __ldg(tpc + 8 * j + 1));
          }
        }
#pragma unroll
        for (int cc = 0; cc < BN / 32; ++cc) {
          const int c0 = c_tile + cc * 32;
          if (c0 >= p.cout) break;   // warp-uniform
          uint32_t bits = 0;
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = 4 * cc + jj;
            const int c = c_tile + 8 * j + 2 * t;
            const bool c_ok = row_ok[i] && c < p.cout;
            const size_t o = static_cast<size_t>(m[i]) * p.cout + c;
            if (OUT == LCE_OUT_RAW_ACC) {
              if (c_ok) *reinterpret_cast<int2*>(static_cast<int32_t*>(p.out) + o) = make_int2(x[2 * j] >> 1, x[2 * j + 1] >> 1);
            } else if (OUT == LCE_OUT_FLOAT) {
              float y[2];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                y[e] = transform_float_x2(x[2 * j + e], p.clamp_min, p.clamp_max, __ldg(p.mul + c + e), __ldg(p.bias + c + e));
                // edge pixels: y += cache[row][c] (zero_padding_correction.h:289-291)
                if (zrow >= 0) y[e] = __fadd_rn(y[e], __ldg(p.zpc_cache + static_cast<size_t>(zrow) * p.ldc + c + e));
              }
              if (p.has_res && c_ok) {
                const float2 rv = __ldg(reinterpret_cast<const float2*>(p.residual + o));
                y[0] = __fadd_rn(y[0], rv.x);
                y[1] = __fadd_rn(y[1], rv.y);
                if (p.residual_act != LCE_ACT_NONE) {
                  y[0] = fminf(fmaxf(y[0], act_lo), act_hi);
                  y[1] = fminf(fmaxf(y[1], act_lo), act_hi);
                }
              }
              if (c_ok) *reinterpret_cast<float2*>(static_cast<float*>(p.out) + o) = make_float2(y[0], y[1]);
              // LceQuantize of the value just written: bit = value < 0 (bitpack.h:159)
              bits |= ((y[0] < 0.0f ? 1u : 0u) | (y[1] < 0.0f ? 2u : 0u)) << (8 * jj + 2 * t);
            } else if (OUT == LCE_OUT_INT8) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int q = round_saturate_i8(
                    transform_float_x2(x[2 * j + e], p.clamp_min, p.clamp_max, __ldg(p.mul + c + e), __ldg(p.bias + c + e)));
                if (row_ok[i] && c + e < p.cout) static_cast<int8_t*>(p.out)[o + e] = static_cast<int8_t>(q);
              }
            } else {  // LCE_OUT_BITPACKED: bit = acc > threshold (output_transform.h:164-167)
              bits |= (((x[2 * j] >> 1) > __ldg(p.thr + c) ? 1u : 0u) | ((x[2 * j + 1] >> 1) > __ldg(p.thr + c + 1) ? 2u : 0u))
                      << (8 * jj + 2 * t);
            }
          }
          if (OUT == LCE_OUT_BITPACKED) {
            bits = quad_or(bits);
            const int valid = p.cout - c0;
            if (valid < 32) bits &= (1u << valid) - 1u;
            if (t == 0 && row_ok[i]) static_cast<int32_t*>(p.out)[static_cast<size_t>(m[i]) * p.cw_out + (c0 >> 5)] = static_cast<int32_t>(bits);
          } else if (OUT == LCE_OUT_FLOAT && p.packed_out != nullptr) {
            bits = quad_or(bits);
            if (t == 0 && row_ok[i]) p.packed_out[static_cast<size_t>(m[i]) * p.cw_out + (c0 >> 5)] = static_cast<int32_t>(bits);
          }
        }
      }
    }
  }
}

}  // namespace tc
}  // namespace lce
#endif

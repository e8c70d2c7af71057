// lce_b200_pair.cuh -- two consecutive residual blocks in one kernel:
//     x1 = act1(T1(conv1(sign x0)) + x0),  x2 = act2(T2(conv2(sign x1)) + x1)
// with 3x3 / stride 1 / one-padding C -> C layers (QuickNet's blocks). x1 and its signs never
// leave the SM: per pair this saves the f32 write and read of x1 and the write and read of its
// packed signs, about half of what the two blocks move through HBM.
//
// One CTA owns a TH x TW output tile of one image:
//  1. Layer 1 runs over the tile plus a one-pixel ring, (TH + 2) x (TW + 2) pixels, from the
//     packed x0 words of the tile plus two, staged in shared memory (zero words outside the
//     image: one-padding in the b1 identity). Its epilogue is the one of lce_b200_imma.cuh:
//     transform_float_x2, __fadd_rn with x0, the ADD's clamp, sign = (< 0). The signs of the
//     whole region go to shared memory (0 words outside the image, i.e. the next layer's
//     padding); the f32 interior x1 stays in shared memory as well.
//  2. Layer 2 gathers its A operand from those signs and adds x1 from shared memory; it writes
//     x2 and, optionally, its packed signs.
// The inner product is lce_b200_imma.cuh's b1 one (BMMA.168256.AND.POPC plus the popc(a) row),
// on the same plan-time fragments (wt_nat), so the integers and then the floats are those of two
// run_fused calls bit for bit. Warp task = 32 pixels x 64 channels, as in bconv_imma_kernel (32
// pixels x 32 channels at C = 32).
//
// Tiles (8 warps, __launch_bounds__(256, 2): 128 registers, no spills with -Xptxas -v):
//   C = 32 : 14 x 14 (region 16 x 16 = 8 warp tasks), 42 KB of shared memory
//   C = 64 : 14 x 14 (region 16 x 16 = 8 warp tasks), 73 KB of shared memory
//   C = 128:  7 x 14 (region  9 x 16, 10 warp tasks), 99 KB
// At C = 32 (QuickNetSmall's 56 x 56 section) a tap is one word, so a 3 x 3 layer's K is 9 words:
// taps 0-7 fill one k256 slice (thread tig holds taps 2 tig and 2 tig + 1, two separate words of
// the packed tile) and tap 8 with three zero words is a k128 tail (thread 0 holds it). The plan's
// fragments are those of a 64-channel tile whose channels 32-63 are zero; only the first two
// 16-channel pairs are issued. Per 16 x 8 output fragment that is 2 BMMAs (one k256, one k128) for
// 288 bits of K, against 3 (two k256, one k128) for the 576 bits of C = 64.
// so two CTAs share an SM, and a 56 x 56 or 28 x 28 image splits into whole tiles. Larger C
// would need smaller tiles (more ring recompute and x0 ring re-reads) or a cluster; those stages
// stay on two run_fused calls. Measured on an H100 80GB HBM3 at a 400 W power limit, QuickNet
// batch 256, per profiled step: the 56 x 56 x 64 stage's four blocks 0.695 ms as four nodes,
// 0.449 ms as two pairs; the 28 x 28 x 128 stage's 0.393 ms, 0.300 ms. At a 700 W power limit,
// QuickNetSmall batch 256 (tools/quicknet_small_bench.py): the 56 x 56 x 32 stage's four blocks
// 0.686 ms as four nodes (on the wgmma kernel), 0.217 ms as two pairs.
#ifndef LCE_B200_PAIR_CUH_
#define LCE_B200_PAIR_CUH_

#include "lce_b200_imma.cuh"

namespace lce {

constexpr int kPThreads = 256;

struct PairParams {
  const int32_t* in;        // packed x0 [batch][H][W][CW]
  const float* residual;    // x0 [batch][H][W][C]
  float* out;               // x2
  int32_t* packed_out;      // packed x2 (may be null)
  const uint2* wt[2];       // each layer's b1 fragments [C / 64][n_slices][4][32][2]
  const int32_t* wpop[2];   // popc of each filter row
  const float* mul[2];
  const float* bias[2];
  int clamp_min[2], clamp_max[2];
  int act[2];               // the ADDs' fused activations
  int H, W, tiles_x, tiles_per_img;
};

template <int CW> struct PairShape {
  static_assert(CW == 1 || CW == 2 || CW == 4, "the pair kernel takes 32, 64 or 128 channels");
  static constexpr int C = 32 * CW;
  static constexpr int TH = CW == 4 ? 7 : 14, TW = 14;  // output tile
  static constexpr int RH = TH + 2, RW = TW + 2;        // layer 1's region: the tile plus a ring
  static constexpr int NW = C < kBN ? C : kBN;          // channels of a warp task
  static constexpr int NS = NW / 8;                     // its 8-channel n sub-tiles
  static constexpr int NT = C / NW;                     // warp tasks per pixel group
  static constexpr int Kw = 9 * CW;                     // K words of a 3x3 layer
  static constexpr int Kw4 = (Kw + 3) & ~3;             // padded to the k128 granularity
  static constexpr int n_full = Kw4 >> 3;               // 8-word slices
  static constexpr bool tail = (Kw4 & 4) != 0;          // a last 4-word slice
  static constexpr int n_slices = n_full + (tail ? 1 : 0);
  static constexpr int wt_bytes = NT * n_slices * 256 * 8;
  static constexpr int x1_stride = C + 8;               // floats; +8 keeps the float2 rows apart
  // weights of both layers | packed x0 over the region plus a ring | signs of x1 | x1 |
  // per layer [multiplier | bias | popc of the filter row] x C
  static constexpr int smem_bytes = 2 * wt_bytes + ((RH + 2) * (RW + 2) + RH * RW) * CW * 4 +
                                    TH * TW * x1_stride * 4 + 2 * 3 * C * 4;
};

// acc += popc(a & w), pa += popc(a) for the warp task's 32 output pixels [m0, m0 + 32) of an
// ow-wide grid of n_out pixels, whose 3x3 windows lie in the (ow + 2)-wide packed tile src
// (CW words per pixel). b4: this n-tile's fragments + lane. Rows past n_out compute garbage.
template <int CW>
__device__ __forceinline__ void pair_conv_b1(const uint32_t* src, int ow, int n_out, int m0,
                                             const uint4* b4, int gid, int tig,
                                             int (&acc)[2][8][4], int (&pa)[2][4]) {
  using S = PairShape<CW>;
  const int sw = ow + 2;
  int base[2][2];   // [ms][h]: the window's top-left pixel in src
#pragma unroll
  for (int ms = 0; ms < 2; ++ms)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int r = m0 + ms * 16 + h * 8 + gid;
      if (r >= n_out) r = 0;
      const int oy = r / ow;
      base[ms][h] = (oy * sw + (r - oy * ow)) * CW;
    }
#pragma unroll 1
  for (int s = 0; s < S::n_full; ++s) {
    const int kw = s * 8 + 2 * tig;
    uint32_t a[2][4];
    if constexpr (CW == 1) {
      // words 2 tig, 2 tig + 1 of the slice: taps kw and kw + 1 (both < 8 < Kw)
      const int off0 = (kw / 3) * sw + kw % 3, off1 = ((kw + 1) / 3) * sw + (kw + 1) % 3;
#pragma unroll
      for (int ms = 0; ms < 2; ++ms) {
        a[ms][0] = src[base[ms][0] + off0]; a[ms][1] = src[base[ms][1] + off0];
        a[ms][2] = src[base[ms][0] + off1]; a[ms][3] = src[base[ms][1] + off1];
      }
    } else {
      // words 2 tig, 2 tig + 1 of the slice: one tap (CW is even), channels word cw, cw + 1
      const int t = kw / CW;
      const int off = ((t / 3) * sw + t % 3) * CW + kw % CW;
      const bool live = kw < S::Kw;
#pragma unroll
      for (int ms = 0; ms < 2; ++ms) {
        const uint2 lo = live ? *reinterpret_cast<const uint2*>(src + base[ms][0] + off) : make_uint2(0, 0);
        const uint2 hi = live ? *reinterpret_cast<const uint2*>(src + base[ms][1] + off) : make_uint2(0, 0);
        a[ms][0] = lo.x; a[ms][1] = hi.x; a[ms][2] = lo.y; a[ms][3] = hi.y;
      }
    }
#pragma unroll
    for (int np = 0; np < S::NS / 2; ++np) {
      const uint4 b = b4[(s * 4 + np) * 32];
      bmma_k256(acc[0][2 * np], a[0], b.x, b.y);
      bmma_k256(acc[1][2 * np], a[1], b.x, b.y);
      bmma_k256(acc[0][2 * np + 1], a[0], b.z, b.w);
      bmma_k256(acc[1][2 * np + 1], a[1], b.z, b.w);
    }
    bmma_k256(pa[0], a[0], ~0u, ~0u);
    bmma_k256(pa[1], a[1], ~0u, ~0u);
  }
  if constexpr (S::tail) {
    // thread tig holds word 8 * n_full + tig
    const int kw = S::n_full * 8 + tig;
    const int t = kw / CW;
    const int off = ((t / 3) * sw + t % 3) * CW + kw % CW;
    const bool live = kw < S::Kw;
    uint32_t lo[2], hi[2];
#pragma unroll
    for (int ms = 0; ms < 2; ++ms) {
      lo[ms] = live ? src[base[ms][0] + off] : 0u;
      hi[ms] = live ? src[base[ms][1] + off] : 0u;
    }
#pragma unroll
    for (int np = 0; np < S::NS / 2; ++np) {
      const uint4 b = b4[(S::n_full * 4 + np) * 32];
#pragma unroll
      for (int ms = 0; ms < 2; ++ms) {
        bmma_k128(acc[ms][2 * np], lo[ms], hi[ms], b.x);
        bmma_k128(acc[ms][2 * np + 1], lo[ms], hi[ms], b.z);
      }
    }
#pragma unroll
    for (int ms = 0; ms < 2; ++ms) bmma_k128(pa[ms], lo[ms], hi[ms], ~0u);
  }
}

// One warp task of a layer: the accumulators of output pixels [m0, m0 + 32) x channels
// [c_tile, c_tile + NW), turned into popc(a ^ w) exactly as bconv_imma_kernel does.
// ch_s: the layer's [mul | bias | wpop] x C in shared memory.
template <int CW>
__device__ __forceinline__ void pair_task_acc(const float* ch_s, const uint32_t* src,
                                              const uint2* wt_s, int ow, int n_out, int m0,
                                              int nt, int lane, int (&acc)[2][8][4]) {
  using S = PairShape<CW>;
  const int gid = lane >> 2, tig = lane & 3;
  int pa[2][4] = {};
#pragma unroll
  for (int ms = 0; ms < 2; ++ms)
#pragma unroll
    for (int ns = 0; ns < S::NS; ++ns)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[ms][ns][e] = 0;
  const uint4* b4 = reinterpret_cast<const uint4*>(wt_s) + nt * S::n_slices * 128 + lane;
  pair_conv_b1<CW>(src, ow, n_out, m0, b4, gid, tig, acc, pa);
  const int c_tile = nt * S::NW;
#pragma unroll
  for (int ns = 0; ns < S::NS; ++ns) {
    const int2 pw = *reinterpret_cast<const int2*>(ch_s + 2 * S::C + c_tile + ns * 8 + tig * 2);
#pragma unroll
    for (int ms = 0; ms < 2; ++ms)
#pragma unroll
      for (int e = 0; e < 4; ++e)
        acc[ms][ns][e] = (e & 1 ? pw.y : pw.x) + pa[ms][e] - 2 * acc[ms][ns][e];
  }
}

// epilogue_imma's float path for one accumulator row: y = act(T(acc) + res), y[0, 2 NS)
template <int C, int NS>
__device__ __forceinline__ void pair_row(const PairParams& p, int L, const float* ch_s,
                                         const int (&acc)[2][8][4], int ms, int h,
                                         const float* res, int cth, float (&y)[16]) {
  const int ract = p.act[L];
  const float act_lo = ract == LCE_ACT_RELU_N1_TO_1 ? -1.0f : 0.0f;
  const float act_hi = ract == LCE_ACT_RELU ? __int_as_float(0x7f800000)
                                            : (ract == LCE_ACT_RELU6 ? 6.0f : 1.0f);
#pragma unroll
  for (int ns = 0; ns < NS; ++ns) {
    const float2 mu = *reinterpret_cast<const float2*>(ch_s + cth + ns * 8);
    const float2 bi = *reinterpret_cast<const float2*>(ch_s + C + cth + ns * 8);
    const float2 rv = *reinterpret_cast<const float2*>(res + ns * 8);
    const int x0 = acc[ms][ns][h * 2] << 1, x1 = acc[ms][ns][h * 2 + 1] << 1;
    y[2 * ns] = __fadd_rn(transform_float_x2(x0, p.clamp_min[L], p.clamp_max[L], mu.x, bi.x), rv.x);
    y[2 * ns + 1] =
        __fadd_rn(transform_float_x2(x1, p.clamp_min[L], p.clamp_max[L], mu.y, bi.y), rv.y);
  }
  if (ract != LCE_ACT_NONE) {
#pragma unroll
    for (int j = 0; j < 2 * NS; ++j) y[j] = fminf(fmaxf(y[j], act_lo), act_hi);
  }
}

// LceQuantize of the row's 2 NS values, gathered over the quad: words (c_tile >> 5) and, at
// NS = 8, + 1 (bits1 stays 0 at NS = 4)
template <int NS>
__device__ __forceinline__ void pair_signs(const float (&y)[16], bool ok, int tig, uint32_t& bits0,
                                           uint32_t& bits1) {
  bits0 = bits1 = 0;
  if (ok) {
#pragma unroll
    for (int ns = 0; ns < 4; ++ns) {
      bits0 |= ((y[2 * ns] < 0.0f ? 1u : 0u) | (y[2 * ns + 1] < 0.0f ? 2u : 0u)) << (ns * 8);
      if (NS == 8)
        bits1 |= ((y[2 * ns + 8] < 0.0f ? 1u : 0u) | (y[2 * ns + 9] < 0.0f ? 2u : 0u)) << (ns * 8);
    }
    bits0 <<= tig * 2;
    bits1 <<= tig * 2;
  }
  bits0 |= __shfl_xor_sync(0xffffffffu, bits0, 1);
  if (NS == 8) bits1 |= __shfl_xor_sync(0xffffffffu, bits1, 1);
  bits0 |= __shfl_xor_sync(0xffffffffu, bits0, 2);
  if (NS == 8) bits1 |= __shfl_xor_sync(0xffffffffu, bits1, 2);
}

template <int CW>
__global__ void __launch_bounds__(kPThreads, 2) bconv_pair_kernel(const PairParams p) {
  using S = PairShape<CW>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int gid = lane >> 2, tig = lane & 3;
  constexpr int TH = S::TH, TW = S::TW, RH = S::RH, RW = S::RW;
  const int img = blockIdx.x / p.tiles_per_img;
  const int t = blockIdx.x - img * p.tiles_per_img;
  const int ty = t / p.tiles_x;
  const int y0 = ty * TH, x0 = (t - ty * p.tiles_x) * TW;   // the tile's first output pixel

  uint2* wt_s = reinterpret_cast<uint2*>(smem_raw);                       // [2][wt_bytes]
  uint32_t* x0p_s = reinterpret_cast<uint32_t*>(smem_raw + 2 * S::wt_bytes);  // [RH+2][RW+2][CW]
  uint32_t* s1_s = x0p_s + (RH + 2) * (RW + 2) * CW;                       // [RH][RW][CW]
  float* x1_s = reinterpret_cast<float*>(s1_s + RH * RW * CW);             // [TH*TW][x1_stride]
  float* ch_s = x1_s + TH * TW * S::x1_stride;                             // [2][3][C]

  // weights of both layers and the packed x0 tile (zero-filled outside the image)
  {
    for (int i = tid; i < 2 * 3 * S::C; i += kPThreads) {
      const int L = i / (3 * S::C), k = i - L * 3 * S::C, v = k / S::C, c = k - v * S::C;
      ch_s[i] = v == 0 ? p.mul[L][c] : v == 1 ? p.bias[L][c] : __int_as_float(p.wpop[L][c]);
    }
    const uint4* w0 = reinterpret_cast<const uint4*>(p.wt[0]);
    const uint4* w1 = reinterpret_cast<const uint4*>(p.wt[1]);
    uint4* dst = reinterpret_cast<uint4*>(wt_s);
    constexpr int n16 = S::wt_bytes / 16;
    for (int i = tid; i < 2 * n16; i += kPThreads)
      cp_async_cg16(dst + i, i < n16 ? w0 + i : w1 + (i - n16), 16);
    const int pw = RW + 2, n_px = (RH + 2) * pw;
    for (int i = tid; i < n_px; i += kPThreads) {
      const int py = i / pw;
      const int gy = y0 - 2 + py, gx = x0 - 2 + (i - py * pw);
      const bool in = static_cast<unsigned>(gy) < static_cast<unsigned>(p.H) &&
                      static_cast<unsigned>(gx) < static_cast<unsigned>(p.W);
      const int32_t* g = in ? p.in + ((static_cast<long long>(img) * p.H + gy) * p.W + gx) * CW : p.in;
      cp_async_zfill<4 * CW>(x0p_s + i * CW, g, in ? 4 * CW : 0);
    }
    cp_async_commit();
    // the shortcut rows layer 1's epilogue reads, on their way to L2 meanwhile
    const int lines = RH * RW * (S::C / 32);
    for (int i = tid; i < lines; i += kPThreads) {
      const int r = i / (S::C / 32);
      const int ry = r / RW;
      const int gy = y0 - 1 + ry, gx = x0 - 1 + (r - ry * RW);
      if (static_cast<unsigned>(gy) < static_cast<unsigned>(p.H) &&
          static_cast<unsigned>(gx) < static_cast<unsigned>(p.W))
        asm volatile("prefetch.global.L2 [%0];" ::"l"(
            p.residual + ((static_cast<long long>(img) * p.H + gy) * p.W + gx) * S::C +
            (i - r * (S::C / 32)) * 32));
    }
    cp_async_wait_all();
    __syncthreads();
  }

  int acc[2][8][4];
  // ---- layer 1 over the region: signs of x1 -> s1_s, interior x1 -> x1_s
  {
    const int n_out = RH * RW;
    const int n_tasks = ((n_out + 31) >> 5) * S::NT;
#pragma unroll 1
    for (int task = warp; task < n_tasks; task += kPThreads / 32) {
      const int nt = task % S::NT, m0 = (task / S::NT) * 32;
      pair_task_acc<CW>(ch_s, x0p_s, wt_s, RW, n_out, m0, nt, lane, acc);
      const int cth = nt * S::NW + tig * 2;
#pragma unroll
      for (int ms = 0; ms < 2; ++ms)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = m0 + ms * 16 + h * 8 + gid;
          const int ry = r / RW, rx = r - (r / RW) * RW;
          const int gy = y0 - 1 + ry, gx = x0 - 1 + rx;
          const bool ok = r < n_out && static_cast<unsigned>(gy) < static_cast<unsigned>(p.H) &&
                          static_cast<unsigned>(gx) < static_cast<unsigned>(p.W);
          float y[16];
          if (ok) {
            const float* res = p.residual +
                ((static_cast<long long>(img) * p.H + gy) * p.W + gx) * S::C + cth;
            pair_row<S::C, S::NS>(p, 0, ch_s, acc, ms, h, res, cth, y);
            if (ry >= 1 && ry <= TH && rx >= 1 && rx <= TW) {
              float* o = x1_s + ((ry - 1) * TW + (rx - 1)) * S::x1_stride + cth;
#pragma unroll
              for (int ns = 0; ns < S::NS; ++ns)
                *reinterpret_cast<float2*>(o + ns * 8) = make_float2(y[2 * ns], y[2 * ns + 1]);
            }
          }
          uint32_t bits0, bits1;
          pair_signs<S::NS>(y, ok, tig, bits0, bits1);
          if (r < n_out && tig == 0) {
            uint32_t* w = s1_s + r * CW + (nt * S::NW >> 5);
            w[0] = bits0;
            if (S::NS == 8) w[1] = bits1;
          }
        }
    }
  }
  __syncthreads();
  // ---- layer 2 over the tile: x2 = act2(T2(conv2(s1)) + x1)
  {
    const int n_out = TH * TW;
    const int n_tasks = ((n_out + 31) >> 5) * S::NT;
    const uint2* wt2_s = wt_s + S::wt_bytes / 8;
    const float* ch2_s = ch_s + 3 * S::C;
#pragma unroll 1
    for (int task = warp; task < n_tasks; task += kPThreads / 32) {
      const int nt = task % S::NT, m0 = (task / S::NT) * 32;
      pair_task_acc<CW>(ch2_s, s1_s, wt2_s, TW, n_out, m0, nt, lane, acc);
      const int cth = nt * S::NW + tig * 2;
#pragma unroll
      for (int ms = 0; ms < 2; ++ms)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int i = m0 + ms * 16 + h * 8 + gid;
          const int iy = i / TW;
          const int gy = y0 + iy, gx = x0 + (i - iy * TW);
          const bool ok = i < n_out && gy < p.H && gx < p.W;
          float y[16];
          const long long px = (static_cast<long long>(img) * p.H + gy) * p.W + gx;
          if (ok) {
            pair_row<S::C, S::NS>(p, 1, ch2_s, acc, ms, h, x1_s + i * S::x1_stride + cth, cth, y);
            float* o = p.out + px * S::C + cth;
#pragma unroll
            for (int ns = 0; ns < S::NS; ++ns)
              *reinterpret_cast<float2*>(o + ns * 8) = make_float2(y[2 * ns], y[2 * ns + 1]);
          }
          if (p.packed_out != nullptr) {   // uniform across the CTA: every lane shuffles
            uint32_t bits0, bits1;
            pair_signs<S::NS>(y, ok, tig, bits0, bits1);
            if (ok && tig == 0) {
              int32_t* pk = p.packed_out + px * CW + (nt * S::NW >> 5);
              pk[0] = static_cast<int32_t>(bits0);
              if (S::NS == 8) pk[1] = static_cast<int32_t>(bits1);
            }
          }
        }
    }
  }
}

}  // namespace lce
#endif

// lce_b200_detect.cu -- TFLite_Detection_PostProcess (TF/lite/kernels/detection_postprocess.cc) over
// whole batches: each image's outputs are what TFLite's kernel gives for that image run alone.
//
//   1. detection_decode_kernel, one thread per (image, anchor): the center-size decode into the
//      workspace's [B, N, 4] corner boxes and, in fast mode, the anchor's best classes and max score.
//   2. detection_nms_kernel, one CTA per problem (an image in fast mode, an (image, class) pair in
//      regular mode): each kept score becomes a 64-bit key (score order << 32 | ~anchor) in shared
//      memory, so the largest live key is the next candidate of TFLite's stable descending sort. Greedy
//      NMS then alternates a block-wide arg-max with one pass that drops every live key whose box
//      overlaps the selected one. The arg-max takes the place of the sort: each selection reads the
//      live keys once in either form, and no sort has to finish before the first selection.
//      Fast mode writes the image's outputs here; regular mode stores each class's selections.
//   3. detection_merge_kernel (regular mode), one CTA per image: the stable top-max_detections of the
//      class lists in class order. Each entry's rank is its position in its own list plus, per other
//      class, a binary search for the entries ahead of it.
// Every float step of the decode and the IoU is one explicitly rounded operation, and exp runs in
// double and is rounded once, so the boxes are TFLite's with a correctly rounded expf.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>

#include "lce_b200.h"

namespace lce_b200_internal {
int fail(const char* fmt, ...);       // lce_b200.cu
int launch_check(const char* what);   // lce_b200.cu
}  // namespace lce_b200_internal
using lce_b200_internal::fail;
using lce_b200_internal::launch_check;

namespace {

// The opt-in shared memory of one sm_90 CTA, less the kernel's static arrays: the keys of
// kMaxAnchors anchors fill the rest.
constexpr int kSmemOptin = 227 * 1024;
constexpr int kStaticSmem = 1024;
constexpr int kMaxAnchors = (kSmemOptin - kStaticSmem) / 8;
constexpr int kFastThreads = 1024;    // B CTAs: many threads per image
constexpr int kRegularThreads = 256;  // B * C CTAs: several per SM

struct DetGeom {
  int B, N, K, S, label_offset, C, kc, mcpd, max_det, limit;
  float score_thr, iou_thr, ys, xs, hs, ws;
};

// Monotone in the score; -0.0 orders as +0.0. Never 0 for a number, so a key of 0 marks a dead entry.
__device__ __forceinline__ uint32_t score_order(float s) {
  const uint32_t u = __float_as_uint(s) == 0x80000000u ? 0u : __float_as_uint(s);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
// std::max<float> / std::min<float> as TFLite calls them, NaN operands included
__device__ __forceinline__ float tfl_max(float a, float b) { return a < b ? b : a; }
__device__ __forceinline__ float tfl_min(float a, float b) { return b < a ? b : a; }

__device__ __forceinline__ float box_area(const float4& b) {   // (ymin, xmin, ymax, xmax)
  return __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
}
// ComputeIntersectionOverUnion(boxes, i, j) with i the selected box
__device__ __forceinline__ float iou(const float4& i, float area_i, const float4& j) {
  const float area_j = box_area(j);
  if (area_i <= 0.0f || area_j <= 0.0f) return 0.0f;
  const float ymin = tfl_max(i.x, j.x), xmin = tfl_max(i.y, j.y);
  const float ymax = tfl_min(i.z, j.z), xmax = tfl_min(i.w, j.w);
  const float inter = __fmul_rn(tfl_max(__fsub_rn(ymax, ymin), 0.0f), tfl_max(__fsub_rn(xmax, xmin), 0.0f));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_i, area_j), inter));
}

__device__ __forceinline__ uint64_t block_max(uint64_t v, uint64_t* red) {
  for (int o = 16; o; o >>= 1) v = max(v, static_cast<uint64_t>(__shfl_xor_sync(~0u, v, o)));
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    v = l < static_cast<int>(blockDim.x >> 5) ? red[l] : 0;
    for (int o = 16; o; o >>= 1) v = max(v, static_cast<uint64_t>(__shfl_xor_sync(~0u, v, o)));
    if (l == 0) red[32] = v;
  }
  __syncthreads();
  return red[32];
}

__global__ void __launch_bounds__(256) detection_decode_kernel(const float* __restrict__ enc,
                                                               const float* __restrict__ scores,
                                                               const float* __restrict__ anchors, DetGeom g,
                                                               float4* __restrict__ dec, float* __restrict__ max_scores,
                                                               int* __restrict__ cls_idx) {
  const long long total = static_cast<long long>(g.B) * g.N;
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float* e = enc + t * g.K;
    const float* a = anchors + 4LL * (t % g.N);   // y, x, h, w
    const float yc = __fadd_rn(__fmul_rn(__fdiv_rn(e[0], g.ys), a[2]), a[0]);
    const float xc = __fadd_rn(__fmul_rn(__fdiv_rn(e[1], g.xs), a[3]), a[1]);
    const float hh = __fmul_rn(__fmul_rn(0.5f, static_cast<float>(exp(static_cast<double>(__fdiv_rn(e[2], g.hs))))), a[2]);
    const float hw = __fmul_rn(__fmul_rn(0.5f, static_cast<float>(exp(static_cast<double>(__fdiv_rn(e[3], g.ws))))), a[3]);
    dec[t] = make_float4(__fsub_rn(yc, hh), __fsub_rn(xc, hw), __fadd_rn(yc, hh), __fadd_rn(xc, hw));
    if (!max_scores) continue;
    // DecreasingPartialArgSort: one class is ArgMaxVector (the first of equal maxima; a NaN in class 0
    // stays the maximum). Several are picked by (score desc, class asc) with NaN below every number.
    const float* row = scores + t * g.S + g.label_offset;
    int* ci = cls_idx + t * g.kc;
    if (g.kc == 1) {
      int best = 0;
      float bv = row[0];
      for (int c = 1; c < g.C; ++c) {
        const float v = row[c];
        if (v > bv) { bv = v; best = c; }
      }
      ci[0] = best;
      max_scores[t] = bv;
      continue;
    }
    uint64_t prev = ~0ull;
    for (int r = 0; r < g.kc; ++r) {
      uint64_t bk = 0;
      for (int c = 0; c < g.C; ++c) {
        const float v = row[c];
        const uint64_t k = (static_cast<uint64_t>(v == v ? score_order(v) : 0u) << 32) | static_cast<uint32_t>(~c);
        if (k < prev && k > bk) bk = k;
      }
      ci[r] = static_cast<int>(~static_cast<uint32_t>(bk));
      prev = bk;
    }
    max_scores[t] = row[ci[0]];
  }
}

// NonMaxSuppressionSingleClassHelper for one problem; `limit` is its max_detections.
template <bool REGULAR>
__global__ void __launch_bounds__(1024) detection_nms_kernel(
    const float* __restrict__ scores, const float* __restrict__ max_scores, const float4* __restrict__ dec, DetGeom g,
    int* __restrict__ sel, float* __restrict__ sel_score, int* __restrict__ counts, const int* __restrict__ cls_idx,
    float4* __restrict__ out_boxes, float* __restrict__ out_classes, float* __restrict__ out_scores,
    float* __restrict__ out_num) {
  extern __shared__ uint64_t keys[];
  __shared__ uint64_t red[33];
  const int b = REGULAR ? blockIdx.x / g.C : blockIdx.x;
  const int cls = REGULAR ? blockIdx.x % g.C : 0;
  const long long base = static_cast<long long>(b) * g.N;
  uint64_t lm = 0;
  for (int n = threadIdx.x; n < g.N; n += blockDim.x) {
    const float s = REGULAR ? scores[(base + n) * g.S + g.label_offset + cls] : max_scores[base + n];
    const uint64_t k = s >= g.score_thr ? (static_cast<uint64_t>(score_order(s)) << 32) | static_cast<uint32_t>(~n) : 0;
    keys[n] = k;   // each thread only ever touches its own entries
    lm = max(lm, k);
  }
  uint64_t best = block_max(lm, red);
  const float4* d = dec + base;
  int* my_sel = sel + static_cast<long long>(blockIdx.x) * g.limit;
  int nsel = 0;
  while (best != 0) {
    const int i = static_cast<int>(~static_cast<uint32_t>(best));
    if (threadIdx.x == 0) {
      my_sel[nsel] = i;
      if (REGULAR) sel_score[static_cast<long long>(blockIdx.x) * g.limit + nsel] =
          scores[(base + i) * g.S + g.label_offset + cls];
    }
    if (++nsel == g.limit) break;
    const float4 bi = d[i];
    const float area_i = box_area(bi);
    lm = 0;
    for (int n = threadIdx.x; n < g.N; n += blockDim.x) {
      const uint64_t k = keys[n];
      if (!k) continue;
      if (n == i || iou(bi, area_i, d[n]) > g.iou_thr) keys[n] = 0;
      else lm = max(lm, k);
    }
    best = block_max(lm, red);
  }
  if (REGULAR) {
    if (threadIdx.x == 0) counts[blockIdx.x] = nsel;
    return;
  }
  __syncthreads();   // my_sel
  // DetectionPostprocessMultiClassFastHelper's outputs; every slot it leaves alone is zero
  const int D = g.max_det * g.mcpd;
  for (int s = threadIdx.x; s < D; s += blockDim.x) {
    const int r = s / g.mcpd, col = s - r * g.mcpd;
    float4 box = make_float4(0.f, 0.f, 0.f, 0.f);
    float c = 0.f, sc = 0.f;
    if (r < nsel && col < g.kc) {
      const int a = my_sel[r];
      const int k = cls_idx[(base + a) * g.kc + col];
      box = d[a];
      c = static_cast<float>(k);
      sc = scores[(base + a) * g.S + g.label_offset + k];
    }
    const long long o = static_cast<long long>(b) * D + s;
    out_boxes[o] = box;
    out_classes[o] = c;
    out_scores[o] = sc;
  }
  if (threadIdx.x == 0) out_num[b] = static_cast<float>(nsel);
}

// DetectionPostprocessMultiClassRegularHelper's merge and outputs for one image
__global__ void __launch_bounds__(256) detection_merge_kernel(const int* __restrict__ sel,
                                                              const float* __restrict__ sel_score,
                                                              const int* __restrict__ counts,
                                                              const float4* __restrict__ dec, DetGeom g,
                                                              float4* __restrict__ out_boxes,
                                                              float* __restrict__ out_classes,
                                                              float* __restrict__ out_scores,
                                                              float* __restrict__ out_num) {
  const int b = blockIdx.x;
  const int* cnt = counts + static_cast<long long>(b) * g.C;
  const int M = min(g.limit, g.max_det);   // an entry at position >= max_detections in its list is out
  const int D = g.max_det * g.mcpd;
  const long long ob = static_cast<long long>(b) * D;
  for (long long t = threadIdx.x; t < static_cast<long long>(g.C) * M; t += blockDim.x) {
    const int c = static_cast<int>(t / M), r = static_cast<int>(t % M);
    if (r >= cnt[c]) continue;
    const long long row = (static_cast<long long>(b) * g.C + c) * g.limit;
    const float s = sel_score[row + r];
    const uint32_t o = score_order(s);
    long long rank = r;
    for (int c2 = 0; c2 < g.C && rank < g.max_det; ++c2) {
      if (c2 == c) continue;
      // entries of class c2 ahead of this one: higher scores, and equal ones of a lower class
      const float* s2 = sel_score + (static_cast<long long>(b) * g.C + c2) * g.limit;
      int lo = 0, hi = min(cnt[c2], g.max_det);
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const uint32_t o2 = score_order(s2[mid]);
        if (c2 < c ? o2 >= o : o2 > o) lo = mid + 1;
        else hi = mid;
      }
      rank += lo;
    }
    if (rank < g.max_det) {
      out_boxes[ob + rank] = dec[static_cast<long long>(b) * g.N + sel[row + r]];
      out_classes[ob + rank] = static_cast<float>(c);
      out_scores[ob + rank] = s;
    }
  }
  long long total = 0;
  for (int c = 0; c < g.C; ++c) total += cnt[c];
  const int num = static_cast<int>(total < g.max_det ? total : g.max_det);
  for (int s = num + threadIdx.x; s < D; s += blockDim.x) {
    out_boxes[ob + s] = make_float4(0.f, 0.f, 0.f, 0.f);
    out_classes[ob + s] = 0.f;
    out_scores[ob + s] = 0.f;
  }
  if (threadIdx.x == 0) out_num[b] = static_cast<float>(num);
}

struct Workspace {
  size_t dec, max_scores, cls, sel, sel_score, counts, total;
};
size_t align16(size_t x) { return (x + 15) / 16 * 16; }
Workspace carve(int batch, int num_anchors, const lce_b200_detection_options& o) {
  const size_t bn = static_cast<size_t>(batch) * num_anchors;
  const int kc = std::min(o.max_classes_per_detection, o.num_classes);
  const size_t L = std::min(o.detections_per_class, num_anchors);
  Workspace w{};
  size_t at = 0;
  auto take = [&](size_t bytes) { const size_t p = at; at += align16(bytes); return p; };
  w.dec = take(bn * 16);
  if (o.use_regular_nms) {
    const size_t lists = static_cast<size_t>(batch) * o.num_classes;
    w.sel = take(lists * L * 4);
    w.sel_score = take(lists * L * 4);
    w.counts = take(lists * 4);
  } else {
    w.max_scores = take(bn * 4);
    w.cls = take(bn * kc * 4);
    w.sel = take(static_cast<size_t>(batch) * o.max_detections * 4);
  }
  w.total = at;
  return w;
}

const char* check_options(int num_anchors, int box_dim, int score_dim, const lce_b200_detection_options& o) {
  if (num_anchors < 1 || box_dim < 4 || score_dim < 1) return "bad box or score shapes";
  if (num_anchors > kMaxAnchors) return "too many anchors for one CTA's shared memory";
  if (o.num_classes < 1 || o.num_classes > score_dim) return "num_classes must be in [1, scores' last dimension]";
  if (o.max_detections < 1 || o.max_classes_per_detection < 1) return "max_detections and max_classes_per_detection must be positive";
  if (o.use_regular_nms && o.detections_per_class < 1) return "detections_per_class must be positive";
  if (!(o.nms_iou_threshold > 0.0f && o.nms_iou_threshold <= 1.0f)) return "nms_iou_threshold must be in (0, 1]";
  if (static_cast<long long>(o.max_detections) * o.max_classes_per_detection > (1LL << 30)) return "too many output slots";
  return nullptr;
}

bool g_smem_set[64] = {};

}  // namespace

extern "C" {

int lce_b200_detection_max_anchors(void) { return kMaxAnchors; }

size_t lce_b200_detection_workspace_bytes(int batch, int num_anchors, const lce_b200_detection_options* o) {
  if (!o || batch < 0 || num_anchors < 1 || o->num_classes < 1 || o->max_detections < 1 ||
      o->max_classes_per_detection < 1 || (o->use_regular_nms && o->detections_per_class < 1))
    return 0;
  return carve(batch, num_anchors, *o).total;
}

int lce_b200_f32_detection_postprocess(const float* boxes, const float* scores, int batch, int num_anchors,
                                       int box_dim, int score_dim, const float* anchors,
                                       const lce_b200_detection_options* o, float* det_boxes, float* det_classes,
                                       float* det_scores, float* num_detections, void* workspace, void* stream) {
  if (!o) return fail("detection_postprocess: no options");
  if (const char* why = check_options(num_anchors, box_dim, score_dim, *o))
    return fail("detection_postprocess: %s", why);
  if (batch < 0) return fail("detection_postprocess: negative batch");
  if (batch == 0) return 0;
  if (!boxes || !scores || !anchors || !det_boxes || !det_classes || !det_scores || !num_detections || !workspace)
    return fail("detection_postprocess: null tensor");
  if ((reinterpret_cast<uintptr_t>(det_boxes) | reinterpret_cast<uintptr_t>(workspace)) & 15)
    return fail("detection_postprocess: detection_boxes and the workspace must be 16-byte aligned");
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && !g_smem_set[dev]) {
    const int bytes = kMaxAnchors * 8;
    if (cudaFuncSetAttribute(detection_nms_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) !=
            cudaSuccess ||
        cudaFuncSetAttribute(detection_nms_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) !=
            cudaSuccess)
      return fail("detection_postprocess: shared memory attribute: %s", cudaGetErrorString(cudaGetLastError()));
    g_smem_set[dev] = true;
  }
  const Workspace w = carve(batch, num_anchors, *o);
  char* ws = static_cast<char*>(workspace);
  DetGeom g;
  g.B = batch;
  g.N = num_anchors;
  g.K = box_dim;
  g.S = score_dim;
  g.C = o->num_classes;
  g.label_offset = score_dim - o->num_classes;
  g.kc = std::min(o->max_classes_per_detection, o->num_classes);
  g.mcpd = o->max_classes_per_detection;
  g.max_det = o->max_detections;
  g.limit = o->use_regular_nms ? std::min(o->detections_per_class, num_anchors) : o->max_detections;
  g.score_thr = o->nms_score_threshold;
  g.iou_thr = o->nms_iou_threshold;
  g.ys = o->y_scale;
  g.xs = o->x_scale;
  g.hs = o->h_scale;
  g.ws = o->w_scale;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  float4* dec = reinterpret_cast<float4*>(ws + w.dec);
  float* max_scores = o->use_regular_nms ? nullptr : reinterpret_cast<float*>(ws + w.max_scores);
  int* cls = o->use_regular_nms ? nullptr : reinterpret_cast<int*>(ws + w.cls);
  const long long bn = static_cast<long long>(batch) * num_anchors;
  const int grid = static_cast<int>(std::min<long long>((bn + 255) / 256, 132 * 32));
  detection_decode_kernel<<<grid, 256, 0, s>>>(boxes, scores, anchors, g, dec, max_scores, cls);
  if (launch_check("detection_decode_kernel")) return 1;
  const size_t smem = static_cast<size_t>(num_anchors) * 8;
  int* sel = reinterpret_cast<int*>(ws + w.sel);
  float4* ob = reinterpret_cast<float4*>(det_boxes);
  if (!o->use_regular_nms) {
    detection_nms_kernel<false><<<batch, kFastThreads, smem, s>>>(scores, max_scores, dec, g, sel, nullptr, nullptr,
                                                                   cls, ob, det_classes, det_scores, num_detections);
    return launch_check("detection_nms_kernel");
  }
  float* sel_score = reinterpret_cast<float*>(ws + w.sel_score);
  int* counts = reinterpret_cast<int*>(ws + w.counts);
  const long long problems = static_cast<long long>(batch) * o->num_classes;
  if (problems > 0x7fffffffLL) return fail("detection_postprocess: too many (image, class) pairs");
  detection_nms_kernel<true><<<static_cast<unsigned>(problems), kRegularThreads, smem, s>>>(
      scores, nullptr, dec, g, sel, sel_score, counts, nullptr, nullptr, nullptr, nullptr, nullptr);
  if (launch_check("detection_nms_kernel")) return 1;
  detection_merge_kernel<<<batch, 256, 0, s>>>(sel, sel_score, counts, dec, g, ob, det_classes, det_scores,
                                               num_detections);
  return launch_check("detection_merge_kernel");
}

}  // extern "C"

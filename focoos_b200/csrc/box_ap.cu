// Box AP matching (trainer.BoxAPEvaluator.evaluate): the greedy assignment of detections to ground truths at every IoU threshold, per image on the
// device, so that evaluation keeps the instances where eval_postprocess left them and the host only accumulates precision / recall.
#include <algorithm>

#include "common.cuh"

namespace fb200 {

constexpr int BAM_MAX_K = 1024;   // detections per image
constexpr int BAM_MAX_G = 1024;   // ground truths per image
constexpr int BAM_MAX_T = 16;     // thresholds: one bit each in the uint16 output

struct BamThresholds {
  double t[BAM_MAX_T];
};

// numpy's maximum / minimum: a NaN operand propagates; otherwise the larger / smaller value
template <typename P>
__device__ __forceinline__ P np_max(P a, P b) { return (a >= b || a != a) ? a : b; }
template <typename P>
__device__ __forceinline__ P np_min(P a, P b) { return (a <= b || a != a) ? a : b; }

__device__ __forceinline__ float rn_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float rn_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float rn_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float rn_div(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double rn_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double rn_sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double rn_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double rn_div(double a, double b) { return __ddiv_rn(a, b); }

// candidate (v, j) beats (bv, bj) under numpy's first argmax: a NaN is the maximum, ties go to the lower index
__device__ __forceinline__ bool bam_better(double v, int j, double bv, int bj) {
  if (j < 0) return false;
  if (bj < 0) return true;
  const bool vn = v != v, bn = bv != bv;
  if (vn || bn) return vn && (!bn || j < bj);
  return v > bv || (v == bv && j < bj);
}

// ---------------------------------------------------------------------------------------------------------------------
// One CTA per image, one warp per threshold.  Setup (all threads): the image's detections and ground truths into shared memory with their areas,
// the stable descending-score rank of every detection, the per-class ground-truth counts.  Matching: warp t walks the detections in rank order; for
// each, the lanes scan the image's ground truths of the detection's class for cand = used ? -1 : IoU and reduce (value, lowest index) across the warp;
// lane 0 marks the winner used and sets bit t when cand >= threshold.  Matching only interacts inside one (image, class), so this is the evaluator's
// walk over the stable global sort by -score.  Integer results: every run is identical.
// ---------------------------------------------------------------------------------------------------------------------
template <typename P>
__global__ void box_ap_match_kernel(const float* __restrict__ scores, const int* __restrict__ classes, const float* __restrict__ boxes,
                                    const int* __restrict__ counts, int K, const P* __restrict__ gt_boxes, const int* __restrict__ gt_classes,
                                    const int* __restrict__ gt_offsets, BamThresholds thr, int T, int C, uint16_t* __restrict__ tp,
                                    unsigned long long* __restrict__ gt_count) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int b = blockIdx.x;
  const int n = min(max(counts[b], 0), K);
  const int g0 = gt_offsets[b], ng = gt_offsets[b + 1] - g0;
  // layout: P gbox[ng*4], P garea[ng], float dbox[K*4], float darea[K], float dscore[K], int dcls[K], int order[K], unsigned bits[K], int gcls[ng],
  //         unsigned char used[T*ng]
  P* gbox = reinterpret_cast<P*>(smem);
  P* garea = gbox + 4 * ng;
  float* dbox = reinterpret_cast<float*>(garea + ng);
  float* darea = dbox + 4 * K;
  float* dscore = darea + K;
  int* dcls = reinterpret_cast<int*>(dscore + K);
  int* order = dcls + K;
  unsigned* bits = reinterpret_cast<unsigned*>(order + K);
  int* gcls = reinterpret_cast<int*>(bits + K);
  unsigned char* used = reinterpret_cast<unsigned char*>(gcls + ng);

  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float* bx = boxes + ((int64_t)b * K + i) * 4;
    const float x0 = bx[0], y0 = bx[1], x1 = bx[2], y1 = bx[3];
    dbox[4 * i] = x0; dbox[4 * i + 1] = y0; dbox[4 * i + 2] = x1; dbox[4 * i + 3] = y1;
    darea[i] = rn_mul(rn_sub(x1, x0), rn_sub(y1, y0));
    dscore[i] = scores[(int64_t)b * K + i];
    dcls[i] = classes[(int64_t)b * K + i];
    bits[i] = 0u;
  }
  for (int j = threadIdx.x; j < ng; j += blockDim.x) {
    const P* gb = gt_boxes + (int64_t)(g0 + j) * 4;
    const P x0 = gb[0], y0 = gb[1], x1 = gb[2], y1 = gb[3];
    gbox[4 * j] = x0; gbox[4 * j + 1] = y0; gbox[4 * j + 2] = x1; gbox[4 * j + 3] = y1;
    garea[j] = rn_mul(rn_sub(x1, x0), rn_sub(y1, y0));
    const int c = gt_classes[g0 + j];
    gcls[j] = c;
    if (c >= 0 && c < C) atomicAdd(&gt_count[c], 1ull);
  }
  for (int j = threadIdx.x; j < T * ng; j += blockDim.x) used[j] = 0;
  __syncthreads();
  // rank = number of detections before i in (score descending, index ascending); a NaN score sorts last (a total order, so `order` is a permutation)
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float si = dscore[i] != dscore[i] ? -INFINITY : dscore[i];
    int r = 0;
    for (int j = 0; j < n; ++j) {
      const float sj = dscore[j] != dscore[j] ? -INFINITY : dscore[j];
      r += (sj > si || (sj == si && j < i)) ? 1 : 0;
    }
    order[r] = i;
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < T) {
    const double t = thr.t[warp];
    unsigned char* u = used + warp * ng;
    for (int r = 0; r < n; ++r) {
      const int i = order[r];
      const int c = dcls[i];
      if (c < 0 || c >= C) continue;  // the evaluator visits the classes 0..C-1 only
      const P dx0 = (P)dbox[4 * i], dy0 = (P)dbox[4 * i + 1], dx1 = (P)dbox[4 * i + 2], dy1 = (P)dbox[4 * i + 3];
      const P da = (P)darea[i];
      double bv = 0.0;
      int bj = -1;
      for (int j = lane; j < ng; j += 32) {
        if (gcls[j] != c) continue;
        double v;
        if (u[j]) {
          v = -1.0;
        } else {  // _iou_matrix: inter / max((aa + ab) - inter, 1e-12), inter = clip(rb - lt, 0).prod()
          const P ltx = np_max(dx0, gbox[4 * j]), lty = np_max(dy0, gbox[4 * j + 1]);
          const P rbx = np_min(dx1, gbox[4 * j + 2]), rby = np_min(dy1, gbox[4 * j + 3]);
          const P inter = rn_mul(np_max(rn_sub(rbx, ltx), (P)0), np_max(rn_sub(rby, lty), (P)0));
          const P den = np_max(rn_sub(rn_add(da, garea[j]), inter), (P)1e-12);
          v = (double)rn_div(inter, den);
        }
        if (bam_better(v, j, bv, bj)) { bv = v; bj = j; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
        if (bam_better(ov, oj, bv, bj)) { bv = ov; bj = oj; }
      }
      if (lane == 0 && bj >= 0 && bv >= t) {
        u[bj] = 1;
        atomicOr(&bits[i], 1u << warp);
      }
      __syncwarp();
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < K; i += blockDim.x) tp[(int64_t)b * K + i] = i < n ? (uint16_t)bits[i] : (uint16_t)0;
}

// bytes of the kernel's shared layout: per ground truth 5 P (box, area) + 1 int (class) + T flags; per detection 9 four-byte words (box, area, score,
// class, order, bits)
template <typename P>
size_t bam_smem(int K, int ng, int T) {
  return (size_t)ng * (5 * sizeof(P) + sizeof(int) + T) + (size_t)K * 9 * 4;
}

}  // namespace fb200

using namespace fb200;

extern "C" int fb200_box_ap_match(const float* scores, const int* classes, const float* boxes, const int* counts, int B, int K, const void* gt_boxes,
                                  int gt_fp64, const int* gt_classes, const int* gt_offsets, const int* gt_offsets_host, int G,
                                  const double* thresholds_host, int T, int C, uint16_t* tp, int64_t* gt_count, void* stream) {
  FB_CHECK_ARG(B >= 0 && K >= 0 && G >= 0 && C > 0 && gt_offsets_host && thresholds_host, "box_ap_match: bad arguments");
  FB_CHECK_ARG(K <= BAM_MAX_K, "box_ap_match: %d detections per image, the kernel holds at most %d", K, BAM_MAX_K);
  FB_CHECK_ARG(T >= 1 && T <= BAM_MAX_T, "box_ap_match: %d thresholds, the uint16 output holds 1 to %d", T, BAM_MAX_T);
  if (B == 0) return FB200_OK;
  FB_CHECK_ARG(scores && classes && boxes && counts && gt_offsets && tp && gt_count && (G == 0 || (gt_boxes && gt_classes)),
               "box_ap_match: null pointer");
  FB_CHECK_ARG(gt_offsets_host[0] == 0 && gt_offsets_host[B] == G, "box_ap_match: ground-truth offsets run from %d to %d, expected 0 to G = %d",
               gt_offsets_host[0], gt_offsets_host[B], G);
  int max_ng = 0;
  for (int b = 0; b < B; ++b) {
    const int ng = gt_offsets_host[b + 1] - gt_offsets_host[b];
    FB_CHECK_ARG(ng >= 0, "box_ap_match: ground-truth offsets are not monotonic at image %d (%d > %d)", b, gt_offsets_host[b], gt_offsets_host[b + 1]);
    FB_CHECK_ARG(ng <= BAM_MAX_G, "box_ap_match: image %d has %d ground truths, the kernel holds at most %d", b, ng, BAM_MAX_G);
    max_ng = std::max(max_ng, ng);
  }
  BamThresholds thr{};
  for (int t = 0; t < T; ++t) thr.t[t] = thresholds_host[t];
  const size_t smem = gt_fp64 ? bam_smem<double>(K, max_ng, T) : bam_smem<float>(K, max_ng, T);
  static bool configured = false;
  if (!configured) {  // the largest layout (fp64 ground truth at both limits) is under 100 KiB
    cudaFuncSetAttribute(box_ap_match_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bam_smem<double>(BAM_MAX_K, BAM_MAX_G, BAM_MAX_T));
    cudaFuncSetAttribute(box_ap_match_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bam_smem<double>(BAM_MAX_K, BAM_MAX_G, BAM_MAX_T));
    configured = true;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int threads = std::max(T * 32, 128);
  auto* gc = reinterpret_cast<unsigned long long*>(gt_count);
  if (gt_fp64)
    box_ap_match_kernel<double><<<B, threads, smem, st>>>(scores, classes, boxes, counts, K, (const double*)gt_boxes, gt_classes, gt_offsets, thr, T, C, tp, gc);
  else
    box_ap_match_kernel<float><<<B, threads, smem, st>>>(scores, classes, boxes, counts, K, (const float*)gt_boxes, gt_classes, gt_offsets, thr, T, C, tp, gc);
  FB_CHECK_LAUNCH("box_ap_match");
  return FB200_OK;
}

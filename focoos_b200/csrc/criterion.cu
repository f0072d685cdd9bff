// Training criterion of the DETR path (SURVEY §8 a20): matching cost, Hungarian assignment on the device, and the
// VFL / L1 / GIoU losses with their gradients w.r.t. the predictions, for all supervised layers in one launch each.
//
// Reference: BoxHungarianMatcher.forward  focoos/models/fai_detr/modelling.py:693-758  (cost; scipy LSA on the CPU)
//            SetCriterion.loss_labels_vfl :464-499, loss_boxes :513-531, forward :553-612
//            box_iou / generalized_box_iou  focoos/utils/box.py:27-64
//
// Layout: logits [L,B,Q,C] f32 (raw, pre-sigmoid), boxes [L,B,Q,4] f32 cxcywh in [0,1]; targets concatenated over
// the batch: labels [T] i32, boxes [T,4] f32 cxcywh, offsets [B+1] i32.  The cost matrix is stored target-major,
// cost[l][t][q], because the assignment runs with targets as rows (n_b <= Q, what scipy's transposition also does).
#include "common.cuh"

namespace fb200 {
namespace {

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }

struct BoxPair {
  float iou, giou, uni, enc;
  float x0, y0, x1, y1, tx0, ty0, tx1, ty1, iw, ih, ew, eh, inter;
};

__device__ __forceinline__ BoxPair box_pair(const float4 s, const float4 t) {
  BoxPair p;
  p.x0 = s.x - 0.5f * s.z; p.y0 = s.y - 0.5f * s.w; p.x1 = s.x + 0.5f * s.z; p.y1 = s.y + 0.5f * s.w;
  p.tx0 = t.x - 0.5f * t.z; p.ty0 = t.y - 0.5f * t.w; p.tx1 = t.x + 0.5f * t.z; p.ty1 = t.y + 0.5f * t.w;
  const float a1 = (p.x1 - p.x0) * (p.y1 - p.y0), a2 = (p.tx1 - p.tx0) * (p.ty1 - p.ty0);
  p.iw = fmaxf(fminf(p.x1, p.tx1) - fmaxf(p.x0, p.tx0), 0.f);
  p.ih = fmaxf(fminf(p.y1, p.ty1) - fmaxf(p.y0, p.ty0), 0.f);
  p.inter = p.iw * p.ih;
  p.uni = a1 + a2 - p.inter;
  p.iou = p.inter / p.uni;
  p.ew = fmaxf(fmaxf(p.x1, p.tx1) - fminf(p.x0, p.tx0), 0.f);
  p.eh = fmaxf(fmaxf(p.y1, p.ty1) - fminf(p.y0, p.ty0), 0.f);
  p.enc = p.ew * p.eh;
  p.giou = p.iou - (p.enc - p.uni) / (p.enc + 1e-5f);
  return p;
}

// ---------------------------------------------------------------------------------------------------------------
// cost[l][t][q] = w_bbox * L1 + w_class * (pos_focal - neg_focal) + w_giou * (-GIoU)        (modelling.py:722-741)
__global__ void match_cost_kernel(const float* __restrict__ logits, const float* __restrict__ boxes, const int* __restrict__ tl,
                                  const float* __restrict__ tb, const int* __restrict__ toff, int L, int B, int Q, int C, int T,
                                  float w_class, float w_bbox, float w_giou, float alpha, float gamma, float* __restrict__ cost) {
  const int64_t total = (int64_t)L * T * Q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int q = i % Q;
    const int t = (i / Q) % T;
    const int l = i / ((int64_t)Q * T);
    int b = 0;
    while (b + 1 < B && toff[b + 1] <= t) ++b;  // B is small (<= a few dozen)
    const int64_t row = ((int64_t)l * B + b) * Q + q;
    const float p = sigm(logits[row * C + tl[t]]);
    float neg, pos;
    if (gamma == 2.f) {
      neg = (1.f - alpha) * (p * p) * (-logf(1.f - p + 1e-8f));
      pos = alpha * ((1.f - p) * (1.f - p)) * (-logf(p + 1e-8f));
    } else {
      neg = (1.f - alpha) * powf(p, gamma) * (-logf(1.f - p + 1e-8f));
      pos = alpha * powf(1.f - p, gamma) * (-logf(p + 1e-8f));
    }
    const float4 s = reinterpret_cast<const float4*>(boxes)[row];
    const float4 g = reinterpret_cast<const float4*>(tb)[t];
    const float l1 = fabsf(s.x - g.x) + fabsf(s.y - g.y) + fabsf(s.z - g.z) + fabsf(s.w - g.w);
    const BoxPair bp = box_pair(s, g);
    cost[i] = w_bbox * l1 + w_class * (pos - neg) + w_giou * (-bp.giou);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Rectangular linear-sum assignment by shortest augmenting paths (Crouse 2016, the algorithm behind
// scipy.optimize.linear_sum_assignment which the reference calls at modelling.py:747), one CTA per (image, layer):
// rows = the image's n targets, columns = the Q queries; each Dijkstra step relaxes all columns in parallel and
// picks the next column with a block-wide arg-min.  Duals and path costs are kept in double like scipy.
constexpr int LSA_THREADS = 256;

__global__ void __launch_bounds__(LSA_THREADS) hungarian_kernel(const float* __restrict__ cost, const int* __restrict__ toff, int B, int Q, int T,
                                                                 int* __restrict__ match_q) {
  extern __shared__ __align__(16) unsigned char lsa_smem[];
  const int b = blockIdx.x, l = blockIdx.y;
  const int t0 = toff[b], n = toff[b + 1] - t0;
  if (n <= 0) return;
  double* v = reinterpret_cast<double*>(lsa_smem);       // [Q] column duals
  double* sp = v + Q;                                    // [Q] shortest path costs
  double* u = sp + Q;                                    // [n] row duals
  int* path = reinterpret_cast<int*>(u + n);             // [Q]
  int* row4col = path + Q;                               // [Q]
  int* col4row = row4col + Q;                            // [n]
  unsigned char* SC = reinterpret_cast<unsigned char*>(col4row + n);  // [Q]
  unsigned char* SR = SC + Q;                                         // [n]
  __shared__ double red_v[LSA_THREADS / 32];
  __shared__ int red_j[LSA_THREADS / 32];
  __shared__ double s_min;
  __shared__ int s_j, s_i, s_sink;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const float* cm = cost + ((int64_t)l * T + t0) * Q;
  for (int j = tid; j < Q; j += LSA_THREADS) { v[j] = 0.0; row4col[j] = -1; }
  for (int i = tid; i < n; i += LSA_THREADS) { u[i] = 0.0; col4row[i] = -1; }
  __syncthreads();
  for (int cur = 0; cur < n; ++cur) {
    for (int j = tid; j < Q; j += LSA_THREADS) { sp[j] = INFINITY; SC[j] = 0; path[j] = -1; }
    for (int i = tid; i < n; i += LSA_THREADS) SR[i] = 0;
    if (tid == 0) { s_min = 0.0; s_i = cur; s_sink = -1; }
    __syncthreads();
    while (true) {
      const int i = s_i;
      const double minv = s_min, ui = u[i];
      double best = INFINITY;
      int bj = -1, bfree = 0;
      for (int j = tid; j < Q; j += LSA_THREADS) {
        if (SC[j]) continue;
        const double r = minv + (double)cm[(int64_t)i * Q + j] - ui - v[j];
        if (r < sp[j]) { sp[j] = r; path[j] = i; }
        const double c = sp[j];
        const int fr = row4col[j] < 0;
        if (c < best || (c == best && (fr > bfree || (fr == bfree && j < bj)))) { best = c; bj = j; bfree = fr; }
      }
      // block arg-min; ties prefer an unassigned column, then the lower index
      for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_down_sync(0xffffffffu, best, o);
        const int oj = __shfl_down_sync(0xffffffffu, bj, o), of = __shfl_down_sync(0xffffffffu, bfree, o);
        if (oj >= 0 && (bj < 0 || ob < best || (ob == best && (of > bfree || (of == bfree && oj < bj))))) { best = ob; bj = oj; bfree = of; }
      }
      if (lane == 0) { red_v[wid] = best; red_j[wid] = bj; }
      __syncthreads();
      if (tid == 0) {
        double bb = INFINITY;
        int jj = -1, ff = 0;
        for (int w = 0; w < LSA_THREADS / 32; ++w) {
          const int oj = red_j[w];
          if (oj < 0) continue;
          const int of = row4col[oj] < 0;
          if (jj < 0 || red_v[w] < bb || (red_v[w] == bb && (of > ff || (of == ff && oj < jj)))) { bb = red_v[w]; jj = oj; ff = of; }
        }
        SR[i] = 1;
        s_min = bb;
        s_j = jj;
        if (jj < 0 || !(bb < INFINITY)) s_sink = -2;  // infeasible (NaN / inf costs)
        else {
          SC[jj] = 1;
          if (row4col[jj] < 0) s_sink = jj; else s_i = row4col[jj];
        }
      }
      __syncthreads();
      if (s_sink != -1) break;
    }
    if (s_sink == -2) {  // leave the remaining rows unmatched; the host wrapper reports it
      for (int i = tid; i < n; i += LSA_THREADS) match_q[(int64_t)l * T + t0 + i] = -1;
      return;
    }
    const double minv = s_min;
    // dual updates (u for visited rows, v for visited columns) - col4row still holds the pre-augmentation state
    for (int i = tid; i < n; i += LSA_THREADS) {
      if (i == cur) u[i] += minv;
      else if (SR[i]) u[i] += minv - sp[col4row[i]];
    }
    __syncthreads();
    for (int j = tid; j < Q; j += LSA_THREADS)
      if (SC[j]) v[j] -= minv - sp[j];
    __syncthreads();
    if (tid == 0) {  // augment along the alternating path back to `cur`
      int j = s_sink;
      while (true) {
        const int i = path[j];
        row4col[j] = i;
        const int pj = col4row[i];
        col4row[i] = j;
        j = pj;
        if (i == cur) break;
      }
    }
    __syncthreads();
  }
  for (int i = tid; i < n; i += LSA_THREADS) match_q[(int64_t)l * T + t0 + i] = col4row[i];
}

// ---------------------------------------------------------------------------------------------------------------
// Per matched pair: IoU (-> VFL target score), L1 and GIoU losses and their gradients w.r.t. the predicted box.
// One CTA per layer; targets are visited in a fixed order so the sums are reproducible.
__global__ void __launch_bounds__(256) loss_boxes_kernel(const float* __restrict__ boxes, const int* __restrict__ tl, const float* __restrict__ tb,
                                                          const int* __restrict__ toff, const int* __restrict__ match_q, int B, int Q, int T,
                                                          float inv_nb, float w_bbox, float w_giou, int* __restrict__ tclass, float* __restrict__ tscore,
                                                          float* __restrict__ g_l1, float* __restrict__ g_giou, float* __restrict__ sums) {
  const int l = blockIdx.x, tid = threadIdx.x;
  float s_l1 = 0.f, s_g = 0.f;
  for (int t = tid; t < T; t += blockDim.x) {
    const int q = match_q[(int64_t)l * T + t];
    if (q < 0) continue;
    int b = 0;
    while (b + 1 < B && toff[b + 1] <= t) ++b;
    const int64_t row = ((int64_t)l * B + b) * Q + q;
    const float4 s = reinterpret_cast<const float4*>(boxes)[row];
    const float4 g = reinterpret_cast<const float4*>(tb)[t];
    const BoxPair p = box_pair(s, g);
    tclass[row] = tl[t];
    tscore[row] = p.iou;
    s_l1 += fabsf(s.x - g.x) + fabsf(s.y - g.y) + fabsf(s.z - g.z) + fabsf(s.w - g.w);
    s_g += 1.f - p.giou;
    auto sgn = [](float d) { return d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f); };
    reinterpret_cast<float4*>(g_l1)[row] = make_float4(sgn(s.x - g.x) * inv_nb * w_bbox, sgn(s.y - g.y) * inv_nb * w_bbox, sgn(s.z - g.z) * inv_nb * w_bbox, sgn(s.w - g.w) * inv_nb * w_bbox);
    // d(1 - giou)/d(box), reverse mode through box.py:27-64
    const float dg = -inv_nb * w_giou;                // d (weighted loss) / d giou
    const float Ae = p.enc + 1e-5f;
    float dA = -dg * (p.uni + 1e-5f) / (Ae * Ae);      // giou = iou - (A-U)/(A+eps)
    float dU = dg / Ae;
    float dI = dg / p.uni;                             // iou = I/U
    dU += -dg * p.inter / (p.uni * p.uni);
    const float dArea1 = dU;                           // U = a1 + a2 - I
    dI += -dU;
    const float diw = dI * p.ih, dih = dI * p.iw;      // I = iw*ih
    const float dew = dA * p.eh, deh = dA * p.ew;      // A = ew*eh
    float dx0 = 0.f, dy0 = 0.f, dx1 = 0.f, dy1 = 0.f;
    auto tie = [](float a, float b2) { return a > b2 ? 1.f : (a == b2 ? 0.5f : 0.f); };  // torch splits max/min gradients on ties
    const float rawiw = fminf(p.x1, p.tx1) - fmaxf(p.x0, p.tx0), rawih = fminf(p.y1, p.ty1) - fmaxf(p.y0, p.ty0);
    if (rawiw >= 0.f) { dx1 += diw * tie(p.tx1, p.x1); dx0 += -diw * tie(p.x0, p.tx0); }
    if (rawih >= 0.f) { dy1 += dih * tie(p.ty1, p.y1); dy0 += -dih * tie(p.y0, p.ty0); }
    const float rawew = fmaxf(p.x1, p.tx1) - fminf(p.x0, p.tx0), raweh = fmaxf(p.y1, p.ty1) - fminf(p.y0, p.ty0);
    if (rawew >= 0.f) { dx1 += dew * tie(p.x1, p.tx1); dx0 += -dew * tie(p.tx0, p.x0); }
    if (raweh >= 0.f) { dy1 += deh * tie(p.y1, p.ty1); dy0 += -deh * tie(p.ty0, p.y0); }
    const float bw = p.x1 - p.x0, bh = p.y1 - p.y0;    // a1 = bw*bh
    dx1 += dArea1 * bh; dx0 -= dArea1 * bh; dy1 += dArea1 * bw; dy0 -= dArea1 * bw;
    reinterpret_cast<float4*>(g_giou)[row] = make_float4(dx0 + dx1, dy0 + dy1, 0.5f * (dx1 - dx0), 0.5f * (dy1 - dy0));
  }
  __shared__ float r1[256], r2[256];
  r1[tid] = s_l1; r2[tid] = s_g;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (tid < o) { r1[tid] += r1[tid + o]; r2[tid] += r2[tid + o]; }
    __syncthreads();
  }
  if (tid == 0) { sums[l * 3 + 1] = r1[0] * inv_nb; sums[l * 3 + 2] = r2[0] * inv_nb; }
}

// Varifocal loss over every (query, class) logit: weight * BCE-with-logits(x, iou * onehot), weight and target detached.
constexpr int VFL_BLOCKS = kNumSMs;
__global__ void __launch_bounds__(256) loss_vfl_kernel(const float* __restrict__ logits, const int* __restrict__ tclass, const float* __restrict__ tscore,
                                                        int64_t rows, int C, float alpha, float gamma, float inv_nb, float* __restrict__ grad,
                                                        float* __restrict__ partial) {
  const int l = blockIdx.y, tid = threadIdx.x;
  const int64_t total = rows * C, base = (int64_t)l * total;
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + tid; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / C;
    const int c = i - r * C;
    const float x = logits[base + i];
    const int tc = tclass[(int64_t)l * rows + r];
    const float t = (tc == c) ? 1.f : 0.f;
    const float ts = t * tscore[(int64_t)l * rows + r];
    const float p = sigm(x);
    const float w = alpha * (gamma == 2.f ? p * p : powf(p, gamma)) * (1.f - t) + ts;
    const float bce = (1.f - ts) * x - (fminf(x, 0.f) - log1pf(expf(-fabsf(x))));
    acc += w * bce;
    grad[base + i] = w * (p - ts) * inv_nb;
  }
  __shared__ float red[256];
  red[tid] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (tid < o) red[tid] += red[tid + o];
    __syncthreads();
  }
  if (tid == 0) partial[(int64_t)l * gridDim.x + blockIdx.x] = red[0];
}

__global__ void loss_finalize_kernel(const float* __restrict__ partial, int nblk, float inv_nb, float w_vfl, float w_bbox, float w_giou,
                                     float* __restrict__ sums) {
  const int l = blockIdx.x;
  if (threadIdx.x != 0) return;
  float s = 0.f;
  for (int i = 0; i < nblk; ++i) s += partial[(int64_t)l * nblk + i];
  sums[l * 3 + 0] = s * inv_nb * w_vfl;
  sums[l * 3 + 1] *= w_bbox;
  sums[l * 3 + 2] *= w_giou;
}

}  // namespace
}  // namespace fb200

using namespace fb200;

extern "C" int fb200_detr_match_cost(const float* logits, const float* boxes, const int* tgt_labels, const float* tgt_boxes, const int* tgt_offsets,
                                     int L, int B, int Q, int C, int T, float w_class, float w_bbox, float w_giou, float alpha, float gamma,
                                     float* cost, void* stream) {
  FB_CHECK_ARG(logits && boxes && tgt_labels && tgt_boxes && tgt_offsets && cost, "detr_match_cost: null pointer");
  FB_CHECK_ARG(L > 0 && B > 0 && Q > 0 && C > 0 && T > 0, "detr_match_cost: bad sizes L=%d B=%d Q=%d C=%d T=%d", L, B, Q, C, T);
  const int64_t total = (int64_t)L * T * Q;
  match_cost_kernel<<<(unsigned)std::min<int64_t>(cdiv(total, 256), kNumSMs * 8), 256, 0, (cudaStream_t)stream>>>(
      logits, boxes, tgt_labels, tgt_boxes, tgt_offsets, L, B, Q, C, T, w_class, w_bbox, w_giou, alpha, gamma, cost);
  FB_CHECK_LAUNCH("detr_match_cost");
  return FB200_OK;
}

extern "C" int fb200_hungarian(const float* cost, const int* tgt_offsets, int L, int B, int Q, int T, int max_targets, int* match_q, void* stream) {
  FB_CHECK_ARG(cost && tgt_offsets && match_q, "hungarian: null pointer");
  FB_CHECK_ARG(L > 0 && B > 0 && Q > 0 && T > 0, "hungarian: bad sizes");
  FB_CHECK_ARG(max_targets >= 1 && max_targets <= Q, "hungarian: an image has %d targets but only %d queries (the reference would match min(Q, n); not supported)", max_targets, Q);
  const size_t smem = (size_t)Q * (8 + 8 + 4 + 4 + 1) + (size_t)max_targets * (8 + 4 + 1) + 32;
  FB_CHECK_ARG(smem <= 200 * 1024, "hungarian: Q=%d too large for shared memory", Q);
  static bool attr_set = false;
  if (!attr_set) { cudaFuncSetAttribute(hungarian_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); attr_set = true; }
  hungarian_kernel<<<dim3(B, L), LSA_THREADS, smem, (cudaStream_t)stream>>>(cost, tgt_offsets, B, Q, T, match_q);
  FB_CHECK_LAUNCH("hungarian");
  return FB200_OK;
}

extern "C" int64_t fb200_detr_loss_workspace_bytes(int L, int B, int Q) {
  return (int64_t)L * B * Q * 8 + (int64_t)L * VFL_BLOCKS * 4 + 256;
}

extern "C" int fb200_detr_loss(const float* logits, const float* boxes, const int* tgt_labels, const float* tgt_boxes, const int* tgt_offsets,
                               const int* match_q, int L, int B, int Q, int C, int T, float num_boxes, float w_vfl, float w_bbox, float w_giou,
                               float alpha, float gamma, float* losses, float* grad_logits, float* grad_boxes_l1, float* grad_boxes_giou,
                               void* workspace, void* stream) {
  FB_CHECK_ARG(logits && boxes && tgt_offsets && losses && grad_logits && grad_boxes_l1 && grad_boxes_giou && workspace, "detr_loss: null pointer");
  FB_CHECK_ARG(L > 0 && B > 0 && Q > 0 && C > 0 && T >= 0 && num_boxes > 0.f, "detr_loss: bad sizes");
  FB_CHECK_ARG(T == 0 || (tgt_labels && tgt_boxes && match_q), "detr_loss: targets missing");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t rows = (int64_t)B * Q;
  int* tclass = reinterpret_cast<int*>(workspace);
  float* tscore = reinterpret_cast<float*>(tclass + L * rows);
  float* partial = tscore + L * rows;
  cudaMemsetAsync(tclass, 0xFF, (size_t)L * rows * 4, st);  // -1 = unmatched
  cudaMemsetAsync(tscore, 0, (size_t)L * rows * 4, st);
  cudaMemsetAsync(grad_boxes_l1, 0, (size_t)L * rows * 16, st);
  cudaMemsetAsync(grad_boxes_giou, 0, (size_t)L * rows * 16, st);
  cudaMemsetAsync(losses, 0, (size_t)L * 3 * 4, st);
  const float inv_nb = 1.f / num_boxes;
  if (T > 0) {
    loss_boxes_kernel<<<L, 256, 0, st>>>(boxes, tgt_labels, tgt_boxes, tgt_offsets, match_q, B, Q, T, inv_nb, w_bbox, w_giou, tclass, tscore, grad_boxes_l1, grad_boxes_giou, losses);
    FB_CHECK_LAUNCH("detr_loss(boxes)");
  }
  loss_vfl_kernel<<<dim3(VFL_BLOCKS, L), 256, 0, st>>>(logits, tclass, tscore, rows, C, alpha, gamma, inv_nb * w_vfl, grad_logits, partial);
  FB_CHECK_LAUNCH("detr_loss(vfl)");
  loss_finalize_kernel<<<L, 32, 0, st>>>(partial, VFL_BLOCKS, inv_nb, w_vfl, w_bbox, w_giou, losses);
  FB_CHECK_LAUNCH("detr_loss(finalize)");
  return FB200_OK;
}

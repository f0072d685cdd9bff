// Semantic-segmentation evaluation (trainer/evaluation/sem_seg_evaluation.py, models/fai_mf/processor.py:142-166): the NHWC mask probabilities the
// class x mask product reads, and the per-pixel class argmax folded into the (C+1) x (C+1) confusion-matrix histogram.
#include <algorithm>

#include "common.cuh"

namespace fb200 {

// ---------------------------------------------------------------------------------------------------------------------
// out[b,Y,X,q] = bilinear(sigmoid(x[b,:,:,q]))  for q < Q, 0 for Q <= q < Qo: the probabilities of fb200_mask_sigmoid_upsample (same source indices,
// same sigmoid and interpolation expressions) in the NHWC layout the per-image 1x1 conv reads, written as fp32, fp16 or the fp16 [hi | lo] pair.
// One thread per (pixel, 4 channels); the low-resolution taps are re-read from L1 / L2 (the input is ~1/16 of the output).
// ---------------------------------------------------------------------------------------------------------------------
template <typename T, int OUT>
__global__ void mask_sigmoid_upsample_nhwc_kernel(const T* __restrict__ x, int B, int h, int w, int Qp, int Q, void* __restrict__ out, int Qo, int H, int W,
                                                  float sh, float sw) {
  const int cv = Qo / 4;
  const int64_t total = (int64_t)B * H * W * cv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int q0 = (int)(i % cv) * 4;
    const int64_t pix = i / cv;
    const int X = pix % W, Y = (pix / W) % H, b = pix / ((int64_t)W * H);
    const float fy = fmaxf(((float)Y + 0.5f) * sh - 0.5f, 0.f), fx = fmaxf(((float)X + 0.5f) * sw - 0.5f, 0.f);
    const int y0 = min((int)fy, h - 1), y1 = min(y0 + 1, h - 1), x0 = min((int)fx, w - 1), x1 = min(x0 + 1, w - 1);
    const float lw1 = fx - (float)x0, lw0 = 1.f - lw1, lh1 = fy - (float)y0, lh0 = 1.f - lh1;
    const T* r0 = x + ((int64_t)b * h + y0) * w * Qp;
    const T* r1 = x + ((int64_t)b * h + y1) * w * Qp;
    float r[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int q = q0 + j;
      if (q >= Q) { r[j] = 0.f; continue; }
      const float v00 = 1.f / (1.f + expf(-to_f(r0[x0 * Qp + q]))), v01 = 1.f / (1.f + expf(-to_f(r0[x1 * Qp + q])));
      const float v10 = 1.f / (1.f + expf(-to_f(r1[x0 * Qp + q]))), v11 = 1.f / (1.f + expf(-to_f(r1[x1 * Qp + q])));
      r[j] = lh0 * (lw0 * v00 + lw1 * v01) + lh1 * (lw0 * v10 + lw1 * v11);
    }
    if (OUT == FB200_F32) {
      store4(static_cast<float*>(out) + pix * Qo + q0, r);
    } else if (OUT == FB200_F16) {
      store4(static_cast<__half*>(out) + pix * Qo + q0, r);
    } else {  // pair: hi = fp16(v), lo = fp16(v - hi)
      float hi[4], lo[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) { hi[j] = __half2float(__float2half_rn(r[j])); lo[j] = r[j] - hi[j]; }
      __half* o = static_cast<__half*>(out) + pix * 2 * Qo + q0;
      store4(o, hi);
      store4(o + Qo, lo);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// conf[(C+1) * pred + gt] += 1 over every pixel, pred = first argmax over c < C of scores[b,y,x,c] (a NaN is the maximum: the first NaN wins, as
// torch.argmax on the CPU), gt = labels[b,y,x] with ignore_label -> C.  One warp per pixel: the lanes read the channel row coalesced and reduce
// (value, index) pairs with an order-independent rule, so the label does not depend on the lane mapping.  SMEM: the CTA counts into a 32-bit
// shared histogram and flushes its non-zero bins with 64-bit atomics once; otherwise every pixel adds into the global matrix directly.
// Integer adds commute, so the matrix is exact and the same on every run.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int SS_THREADS = 512;

__device__ __forceinline__ bool ss_better(float v, int i, float bv, int bi) {
  const bool vn = v != v, bn = bv != bv;
  if (vn || bn) return vn && (!bn || i < bi);
  return v > bv || (v == bv && i < bi);
}

template <bool SMEM, typename L>
__global__ void __launch_bounds__(SS_THREADS) sem_seg_confusion_kernel(const float* __restrict__ scores, int64_t npix, int HW, int pitch, int64_t batch_stride,
                                                                        const L* __restrict__ labels, int C, int ignore_label,
                                                                        unsigned long long* __restrict__ conf, unsigned long long* __restrict__ invalid) {
  extern __shared__ unsigned int hist[];
  const int n = (C + 1) * (C + 1);
  if (SMEM) {
    for (int i = threadIdx.x; i < n; i += SS_THREADS) hist[i] = 0;
    __syncthreads();
  }
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (SS_THREADS / 32);
  unsigned int bad = 0;
  for (int64_t p = (int64_t)blockIdx.x * (SS_THREADS / 32) + (threadIdx.x >> 5); p < npix; p += warps) {
    const int64_t b = p / HW, r = p - b * HW;
    const float* row = scores + b * batch_stride + r * pitch;
    float bv = NAN;
    int bi = -1;
    for (int c = lane; c < C; c += 32) {
      const float v = row[c];
      if (bi < 0 || ss_better(v, c, bv, bi)) { bv = v; bi = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi >= 0 && (bi < 0 || ss_better(ov, oi, bv, bi))) { bv = ov; bi = oi; }
    }
    if (lane == 0) {
      const int g = (int)labels[p];
      const int gt = g == ignore_label ? C : g;
      if (gt < 0 || gt > C) {
        ++bad;
      } else if (SMEM) {
        atomicAdd(&hist[bi * (C + 1) + gt], 1u);
      } else {
        atomicAdd(&conf[bi * (C + 1) + gt], 1ull);
      }
    }
  }
  if (bad) atomicAdd(invalid, (unsigned long long)bad);
  if (SMEM) {
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += SS_THREADS)
      if (hist[i]) atomicAdd(&conf[i], (unsigned long long)hist[i]);
  }
}

}  // namespace fb200

using namespace fb200;

extern "C" int fb200_mask_sigmoid_upsample_nhwc(const void* x, int dtype, int B, int h, int w, int Qp, int Q, void* out, int out_dtype, int Qo, int H, int W,
                                                void* stream) {
  FB_CHECK_ARG(x && out && B > 0 && h > 0 && w > 0 && H > 0 && W > 0 && Q > 0 && Q <= Qp && Q <= Qo && Qo % 4 == 0,
               "mask_sigmoid_upsample_nhwc: bad arguments (Q <= Qp, Q <= Qo, Qo %% 4 == 0)");
  FB_CHECK_ARG(out_dtype == FB200_F32 || out_dtype == FB200_F16 || out_dtype == FB200_F16PAIR, "mask_sigmoid_upsample_nhwc: bad output dtype %d", out_dtype);
  const float sh = (float)h / (float)H, sw = (float)w / (float)W;
  const int64_t total = (int64_t)B * H * W * (Qo / 4);
  const unsigned grid = (unsigned)std::min<int64_t>(cdiv(total, 256), (int64_t)kNumSMs * 32);
  cudaStream_t st = (cudaStream_t)stream;
#define MSU_NHWC(OUT) FB_DISPATCH_DTYPE(dtype, T, (mask_sigmoid_upsample_nhwc_kernel<T, OUT><<<grid, 256, 0, st>>>((const T*)x, B, h, w, Qp, Q, out, Qo, H, W, sh, sw)))
  if (out_dtype == FB200_F32) MSU_NHWC(FB200_F32);
  else if (out_dtype == FB200_F16) MSU_NHWC(FB200_F16);
  else MSU_NHWC(FB200_F16PAIR);
#undef MSU_NHWC
  FB_CHECK_LAUNCH("mask_sigmoid_upsample_nhwc");
  return FB200_OK;
}

extern "C" int fb200_sem_seg_confusion(const float* scores, int B, int H, int W, int C, int pitch, int64_t batch_stride, const void* labels, int label_bytes,
                                       int ignore_label, int64_t* conf, int64_t* invalid, void* stream) {
  FB_CHECK_ARG(scores && labels && conf && invalid && B > 0 && H > 0 && W > 0 && C > 0 && pitch >= C && batch_stride >= (int64_t)H * W * pitch,
               "sem_seg_confusion: bad arguments");
  FB_CHECK_ARG(label_bytes == 1 || label_bytes == 4, "sem_seg_confusion: labels are uint8 or int32 (got %d bytes)", label_bytes);
  const int64_t npix = (int64_t)B * H * W;
  const size_t smem = (size_t)(C + 1) * (C + 1) * sizeof(unsigned int);
  constexpr size_t kSmemMax = 227 * 1024;
  const bool use_smem = smem <= kSmemMax;
  // shared histogram: 2 CTAs of 89 KiB per SM at C = 150, each flushing (C+1)^2 bins once; direct global adds: enough warps to cover the SMs
  const int64_t ctas = cdiv(npix, SS_THREADS / 32);
  const unsigned grid = (unsigned)std::min<int64_t>(ctas, (int64_t)kNumSMs * (use_smem ? (smem <= 113 * 1024 ? 2 : 1) : 4));
  cudaStream_t st = (cudaStream_t)stream;
  auto* cf = reinterpret_cast<unsigned long long*>(conf);
  auto* inv = reinterpret_cast<unsigned long long*>(invalid);
  const int HW = H * W;
  if (use_smem) {
    static bool configured = false;
    if (!configured) {
      cudaFuncSetAttribute(sem_seg_confusion_kernel<true, uint8_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemMax);
      cudaFuncSetAttribute(sem_seg_confusion_kernel<true, int>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemMax);
      configured = true;
    }
    if (label_bytes == 1)
      sem_seg_confusion_kernel<true, uint8_t><<<grid, SS_THREADS, smem, st>>>(scores, npix, HW, pitch, batch_stride, (const uint8_t*)labels, C, ignore_label, cf, inv);
    else
      sem_seg_confusion_kernel<true, int><<<grid, SS_THREADS, smem, st>>>(scores, npix, HW, pitch, batch_stride, (const int*)labels, C, ignore_label, cf, inv);
  } else {
    if (label_bytes == 1)
      sem_seg_confusion_kernel<false, uint8_t><<<grid, SS_THREADS, 0, st>>>(scores, npix, HW, pitch, batch_stride, (const uint8_t*)labels, C, ignore_label, cf, inv);
    else
      sem_seg_confusion_kernel<false, int><<<grid, SS_THREADS, 0, st>>>(scores, npix, HW, pitch, batch_stride, (const int*)labels, C, ignore_label, cf, inv);
  }
  FB_CHECK_LAUNCH("sem_seg_confusion");
  return FB200_OK;
}

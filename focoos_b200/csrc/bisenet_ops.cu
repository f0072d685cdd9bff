// BiSeNetFormer-family kernels (SURVEY §8 rows a18-a19): STDC depthwise 3x3/s2 conv + BN, 3x3/s2 average pool, global average
// pool, channel-gate multiply (ARM / FFM), and the semantic post-process (per-pixel argmax over score-weighted masks).
#include <algorithm>

#include "common.cuh"

namespace fb200 {

static inline unsigned grid_cap2(int64_t total, int threads) {
  int64_t g = cdiv(total, threads);
  const int64_t cap = (int64_t)kNumSMs * 32;
  return (unsigned)(g < cap ? (g > 0 ? g : 1) : cap);
}

// depthwise 3x3 stride 2 pad 1 + per-channel scale/bias (folded BN). w: fp32 [9][C] (tap-major). NHWC.
template <typename T>
__global__ void dwconv3x3s2_kernel(const T* __restrict__ x, const float* __restrict__ w, const float* __restrict__ scale,
                                   const float* __restrict__ bias, T* __restrict__ out, int B, int H, int W, int C, int Ho, int Wo) {
  const int cv = C / 4;
  const int64_t total = (int64_t)B * Ho * Wo * cv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (i % cv) * 4;
    const int64_t pix = i / cv;
    const int wo = pix % Wo, ho = (pix / Wo) % Ho, b = pix / ((int64_t)Wo * Ho);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hi = ho * 2 - 1 + kh;
      if (hi < 0 || hi >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int wi = wo * 2 - 1 + kw;
        if (wi < 0 || wi >= W) continue;
        float v[4], ww[4];
        load4(x + (((int64_t)b * H + hi) * W + wi) * C + c, v);
        load4(w + (kh * 3 + kw) * C + c, ww);
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] = fmaf(v[j], ww[j], acc[j]);
      }
    }
    float sc[4], bi[4];
    load4(scale + c, sc);
    load4(bias + c, bi);
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = acc[j] * sc[j] + bi[j];
    store4(out + pix * C + c, acc);
  }
}

// AvgPool2d(3, 2, 1), count_include_pad=True (divide by 9); output may be a channel slice (out_pitch)
template <typename T>
__global__ void avgpool3x3s2_kernel(const T* __restrict__ x, T* __restrict__ out, int B, int H, int W, int C, int Ho, int Wo, int out_pitch) {
  const int cv = C / 4;
  const int64_t total = (int64_t)B * Ho * Wo * cv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (i % cv) * 4;
    const int64_t pix = i / cv;
    const int wo = pix % Wo, ho = (pix / Wo) % Ho, b = pix / ((int64_t)Wo * Ho);
    float s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hi = ho * 2 - 1 + kh;
      if (hi < 0 || hi >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int wi = wo * 2 - 1 + kw;
        if (wi < 0 || wi >= W) continue;
        float v[4];
        load4(x + (((int64_t)b * H + hi) * W + wi) * C + c, v);
#pragma unroll
        for (int j = 0; j < 4; ++j) s[j] += v[j];
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) s[j] *= (1.f / 9.f);
    store4(out + pix * out_pitch + c, s);
  }
}

// mean over H*W per (b, c):  grid (C/64, B), block 256 = 16 channel-vec4 x 16 pixel lanes
template <typename T>
__global__ void __launch_bounds__(256) global_avgpool_kernel(const T* __restrict__ x, T* __restrict__ out, int HW, int C) {
  __shared__ float red[16][64 + 1];
  const int b = blockIdx.y, c0 = blockIdx.x * 64;
  const int cvec = threadIdx.x & 15, pl = threadIdx.x >> 4;
  const int c = c0 + cvec * 4;
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  if (c < C) {
    for (int p = pl; p < HW; p += 16) {
      float v[4];
      load4(x + ((int64_t)b * HW + p) * C + c, v);
#pragma unroll
      for (int j = 0; j < 4; ++j) s[j] += v[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) red[pl][cvec * 4 + j] = s[j];
  __syncthreads();
  if (threadIdx.x < 64 && c0 + threadIdx.x < C) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) t += red[i][threadIdx.x];
    out[(int64_t)b * C + c0 + threadIdx.x] = from_f<T>(t / (float)HW);
  }
}

// out = x * g[b,c] (+ addvec[b,c]) (+ addt[b,h,w,c]) (+ x)
template <typename T>
__global__ void channel_scale_kernel(const T* __restrict__ x, const T* __restrict__ g, const T* __restrict__ addvec, const T* __restrict__ addt,
                                     int self_add, T* __restrict__ out, int64_t HW, int C, int64_t total4) {
  const int cv = C / 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (i % cv) * 4;
    const int64_t pix = i / cv, b = pix / HW;
    float v[4], gg[4], o[4];
    load4(x + pix * C + c, v);
    load4(g + b * C + c, gg);
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = v[j] * gg[j];
    if (addvec) { float a[4]; load4(addvec + b * C + c, a);
#pragma unroll
      for (int j = 0; j < 4; ++j) o[j] += a[j]; }
    if (addt) { float a[4]; load4(addt + pix * C + c, a);
#pragma unroll
      for (int j = 0; j < 4; ++j) o[j] += a[j]; }
    if (self_add) {
#pragma unroll
      for (int j = 0; j < 4; ++j) o[j] += v[j]; }
    store4(out + pix * C + c, o);
  }
}

// labels[b,y,x] = argmax_q(scores[b,q] * masks[b,q,y,x]) (first maximum), counts[b,q] = pixels labelled q
__global__ void __launch_bounds__(256) mask_argmax_kernel(const float* __restrict__ masks, const float* __restrict__ scores, int Q, int64_t HW,
                                                          uint8_t* __restrict__ labels, int* __restrict__ counts) {
  extern __shared__ int hist[];  // [Q] ints then [Q] floats
  float* sc = reinterpret_cast<float*>(hist + Q);
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < Q; i += 256) { hist[i] = 0; sc[i] = scores[b * Q + i]; }
  __syncthreads();
  const float* mb = masks + (int64_t)b * Q * HW;
  if ((HW & 3) == 0) {  // 4 pixels per thread: 16-byte loads, 8 independent loads in flight per thread (HBM-bound: the masks are read exactly once)
    const int64_t HW4 = HW >> 2;
    for (int64_t p4 = (int64_t)blockIdx.x * 256 + threadIdx.x; p4 < HW4; p4 += (int64_t)gridDim.x * 256) {
      float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
      int bi[4] = {0, 0, 0, 0};
      const float4* col = reinterpret_cast<const float4*>(mb) + p4;
      int q = 0;
      for (; q + 8 <= Q; q += 8) {
        float4 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = __ldcs(col + (int64_t)(q + u) * HW4);
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const float s = sc[q + u];
          const float a0 = s * v[u].x, a1 = s * v[u].y, a2 = s * v[u].z, a3 = s * v[u].w;
          if (a0 > best[0]) { best[0] = a0; bi[0] = q + u; }
          if (a1 > best[1]) { best[1] = a1; bi[1] = q + u; }
          if (a2 > best[2]) { best[2] = a2; bi[2] = q + u; }
          if (a3 > best[3]) { best[3] = a3; bi[3] = q + u; }
        }
      }
      for (; q < Q; ++q) {
        const float4 v = __ldcs(col + (int64_t)q * HW4);
        const float s = sc[q];
        if (s * v.x > best[0]) { best[0] = s * v.x; bi[0] = q; }
        if (s * v.y > best[1]) { best[1] = s * v.y; bi[1] = q; }
        if (s * v.z > best[2]) { best[2] = s * v.z; bi[2] = q; }
        if (s * v.w > best[3]) { best[3] = s * v.w; bi[3] = q; }
      }
      *reinterpret_cast<uchar4*>(labels + (int64_t)b * HW + (p4 << 2)) = make_uchar4((unsigned char)bi[0], (unsigned char)bi[1], (unsigned char)bi[2], (unsigned char)bi[3]);
#pragma unroll
      for (int j = 0; j < 4; ++j) atomicAdd(&hist[bi[j]], 1);
    }
  } else {
    for (int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x; p < HW; p += (int64_t)gridDim.x * 256) {
      float best = -INFINITY;
      int bi = 0;
      for (int q = 0; q < Q; ++q) {
        const float v = sc[q] * mb[(int64_t)q * HW + p];
        if (v > best) { best = v; bi = q; }
      }
      labels[(int64_t)b * HW + p] = (uint8_t)bi;
      atomicAdd(&hist[bi], 1);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < Q; i += 256)
    if (hist[i]) atomicAdd(&counts[b * Q + i], hist[i]);
}

__global__ void bbox_init_kernel2(int* bbox, int n, int Wo, int Ho) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { bbox[i * 4 + 0] = Wo; bbox[i * 4 + 1] = Ho; bbox[i * 4 + 2] = -1; bbox[i * 4 + 3] = -1; }
}
__global__ void bbox_finish_kernel2(int* bbox, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && bbox[i * 4 + 2] < 0) { bbox[i * 4 + 0] = 0; bbox[i * 4 + 1] = 0; bbox[i * 4 + 2] = 0; bbox[i * 4 + 3] = 0; }
}
// kept (b,q): bin = (labels[b] == q) as float -> bilinear resize to (Ho,Wo) -> != 0 -> uint8 mask + bbox
__global__ void __launch_bounds__(256) label_resize_bbox_kernel(const uint8_t* __restrict__ labels, int H, int W, const int* __restrict__ bq, uint8_t* __restrict__ out,
                                                                int Ho, int Wo, float sh, float sw, int* __restrict__ bbox) {
  const int i = blockIdx.y;
  const uint8_t* p = labels + (int64_t)bq[i * 2] * H * W;
  const int q = bq[i * 2 + 1];
  int xmin = Wo, ymin = Ho, xmax = -1, ymax = -1;
  for (int64_t o = (int64_t)blockIdx.x * 256 + threadIdx.x; o < (int64_t)Ho * Wo; o += (int64_t)gridDim.x * 256) {
    const int X = o % Wo, Y = o / Wo;
    const float fy = fmaxf(((float)Y + 0.5f) * sh - 0.5f, 0.f), fx = fmaxf(((float)X + 0.5f) * sw - 0.5f, 0.f);
    const int y0 = min((int)fy, H - 1), x0 = min((int)fx, W - 1), y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
    const float ly = fy - (float)y0, lx = fx - (float)x0;
    const float b00 = p[(int64_t)y0 * W + x0] == q ? 1.f : 0.f, b01 = p[(int64_t)y0 * W + x1] == q ? 1.f : 0.f;
    const float b10 = p[(int64_t)y1 * W + x0] == q ? 1.f : 0.f, b11 = p[(int64_t)y1 * W + x1] == q ? 1.f : 0.f;
    const float r = (1.f - ly) * ((1.f - lx) * b00 + lx * b01) + ly * ((1.f - lx) * b10 + lx * b11);
    const bool on = r != 0.f;
    out[(int64_t)i * Ho * Wo + o] = on ? 1 : 0;
    if (on) { xmin = min(xmin, X); xmax = max(xmax, X); ymin = min(ymin, Y); ymax = max(ymax, Y); }
  }
  if (xmax >= 0) {
    atomicMin(&bbox[i * 4 + 0], xmin); atomicMin(&bbox[i * 4 + 1], ymin);
    atomicMax(&bbox[i * 4 + 2], xmax); atomicMax(&bbox[i * 4 + 3], ymax);
  }
}

}  // namespace fb200
using namespace fb200;

extern "C" int fb200_dwconv3x3s2_bn(const void* x, int dtype, int B, int H, int W, int C, const float* w9c, const float* scale, const float* bias, void* out,
                                    void* stream) {
  FB_CHECK_ARG(x && w9c && scale && bias && out && C % 4 == 0, "dwconv3x3s2: bad arguments");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const int64_t total = (int64_t)B * Ho * Wo * (C / 4);
  FB_DISPATCH_DTYPE(dtype, T, (dwconv3x3s2_kernel<T><<<grid_cap2(total, 256), 256, 0, (cudaStream_t)stream>>>((const T*)x, w9c, scale, bias, (T*)out, B, H, W, C, Ho, Wo)));
  FB_CHECK_LAUNCH("dwconv3x3s2");
  return FB200_OK;
}

extern "C" int fb200_avgpool3x3s2(const void* x, int dtype, int B, int H, int W, int C, void* out, int out_pitch, void* stream) {
  FB_CHECK_ARG(x && out && C % 4 == 0 && out_pitch % 4 == 0 && out_pitch >= C, "avgpool3x3s2: bad arguments");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const int64_t total = (int64_t)B * Ho * Wo * (C / 4);
  FB_DISPATCH_DTYPE(dtype, T, (avgpool3x3s2_kernel<T><<<grid_cap2(total, 256), 256, 0, (cudaStream_t)stream>>>((const T*)x, (T*)out, B, H, W, C, Ho, Wo, out_pitch)));
  FB_CHECK_LAUNCH("avgpool3x3s2");
  return FB200_OK;
}

extern "C" int fb200_global_avgpool(const void* x, int dtype, int B, int HW, int C, void* out, void* stream) {
  FB_CHECK_ARG(x && out && C % 4 == 0 && HW > 0, "global_avgpool: bad arguments");
  dim3 grid((unsigned)cdiv(C, 64), (unsigned)B);
  FB_DISPATCH_DTYPE(dtype, T, (global_avgpool_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>((const T*)x, (T*)out, HW, C)));
  FB_CHECK_LAUNCH("global_avgpool");
  return FB200_OK;
}

extern "C" int fb200_channel_scale(const void* x, const void* gate, const void* addvec, const void* addt, int self_add, void* out, int dtype, int B, int64_t HW,
                                   int C, void* stream) {
  FB_CHECK_ARG(x && gate && out && C % 4 == 0, "channel_scale: bad arguments");
  const int64_t total4 = (int64_t)B * HW * (C / 4);
  FB_DISPATCH_DTYPE(dtype, T, (channel_scale_kernel<T><<<grid_cap2(total4, 256), 256, 0, (cudaStream_t)stream>>>((const T*)x, (const T*)gate, (const T*)addvec, (const T*)addt, self_add, (T*)out, HW, C, total4)));
  FB_CHECK_LAUNCH("channel_scale");
  return FB200_OK;
}

extern "C" int fb200_mask_argmax(const float* masks, const float* scores, int B, int Q, int64_t HW, uint8_t* labels, int* counts, void* stream) {
  FB_CHECK_ARG(masks && scores && labels && counts && Q >= 1 && Q <= 255, "mask_argmax: bad arguments (Q <= 255)");
  dim3 grid((unsigned)std::min<int64_t>(cdiv((HW & 3) ? HW : HW / 4, 256), kNumSMs * 4), (unsigned)B);
  mask_argmax_kernel<<<grid, 256, Q * 8, (cudaStream_t)stream>>>(masks, scores, Q, HW, labels, counts);
  FB_CHECK_LAUNCH("mask_argmax");
  return FB200_OK;
}

extern "C" int fb200_label_resize_bbox(const uint8_t* labels, int H, int W, const int* bq, int n, uint8_t* out, int Ho, int Wo, int* bbox, void* stream) {
  FB_CHECK_ARG(labels && bq && out && bbox && n > 0, "label_resize_bbox: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  bbox_init_kernel2<<<(unsigned)cdiv(n, 128), 128, 0, st>>>(bbox, n, Wo, Ho);
  dim3 grid((unsigned)std::min<int64_t>(cdiv((int64_t)Ho * Wo, 256), 64), (unsigned)n);
  label_resize_bbox_kernel<<<grid, 256, 0, st>>>(labels, H, W, bq, out, Ho, Wo, (float)H / (float)Ho, (float)W / (float)Wo, bbox);
  bbox_finish_kernel2<<<(unsigned)cdiv(n, 128), 128, 0, st>>>(bbox, n);
  FB_CHECK_LAUNCH("label_resize_bbox");
  return FB200_OK;
}

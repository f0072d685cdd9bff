// Shared helpers for the focoos_b200 CUDA kernels (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "focoos_b200.h"

namespace fb200 {

void set_error(const char* fmt, ...);

#define FB_CHECK_ARG(cond, ...)                 \
  do {                                          \
    if (!(cond)) {                              \
      fb200::set_error(__VA_ARGS__);            \
      return FB200_ERR_INVALID;                 \
    }                                           \
  } while (0)

#define FB_CHECK_LAUNCH(name)                                                             \
  do {                                                                                    \
    cudaError_t _e = cudaGetLastError();                                                  \
    if (_e != cudaSuccess) {                                                              \
      fb200::set_error("%s: launch failed: %s", name, cudaGetErrorString(_e));            \
      return FB200_ERR_CUDA;                                                              \
    }                                                                                     \
  } while (0)

template <typename T> struct Vec4;  // 4 consecutive elements
template <> struct Vec4<float> { using type = float4; };
template <> struct Vec4<__half> { using type = uint2; };

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

// load / store 4 consecutive elements as fp32 (pointer must be 4-element aligned)
__device__ __forceinline__ void load4(const float* p, float (&v)[4]) {
  float4 t = *reinterpret_cast<const float4*>(p);
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void load4(const __half* p, float (&v)[4]) {
  uint2 t = *reinterpret_cast<const uint2*>(p);
  __half2 a = *reinterpret_cast<__half2*>(&t.x), b = *reinterpret_cast<__half2*>(&t.y);
  float2 fa = __half22float2(a), fb = __half22float2(b);
  v[0] = fa.x; v[1] = fa.y; v[2] = fb.x; v[3] = fb.y;
}
__device__ __forceinline__ void store4(float* p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void store4(__half* p, const float (&v)[4]) {
  __half2 a = __floats2half2_rn(v[0], v[1]), b = __floats2half2_rn(v[2], v[3]);
  uint2 t;
  t.x = *reinterpret_cast<uint32_t*>(&a);
  t.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = t;
}

__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act & 15) {
    case FB200_ACT_RELU: return fmaxf(v, 0.f);
    case FB200_ACT_SILU: return v / (1.f + expf(-v));
    case FB200_ACT_GELU: return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
    case FB200_ACT_SIGMOID: return 1.f / (1.f + expf(-v));
    default: return v;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// shared by conv_simt.cu (SIMT path) and conv_tc.cu (tensor-core path)
struct ConvParams {
  const void* x; const void* w; const float* scale; const float* bias; const void* res; void* out;
  int B, H, W, Cin, x_pitch, KH, KW, stride, pad, Ho, Wo, Cout, res_pitch, out_pitch, act;
  int64_t M; int K; int x_dtype, out_dtype, vec_ok; int split3; int64_t out_bs;  // out_bs: elements between images of `out`
  int64_t w_bs = 0;  // elements between the per-image weight sets (0 = one shared weight tensor)
  int64_t x_lo_off = 0;     // split3: elements from the hi plane of x to its lo plane
  int64_t out_lo_off = 0, res_lo_off = 0;  // out_dtype == FB200_F16PAIR: elements from the hi plane to the lo plane of out / residual
  float* rowmax = nullptr;  // not null: no output tensor, only max over the Cout columns of every row (atomic max into a buffer pre-filled with -inf)
};

static inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

// SMs of the target GPU (H100 SXM): sizes grid-stride caps and split counts; kernels stay correct on any SM count
constexpr int kNumSMs = 132;

// dispatch helper on activation dtype
#define FB_DISPATCH_DTYPE(dt, T, ...)                         \
  do {                                                        \
    if ((dt) == FB200_F32) { using T = float; __VA_ARGS__; }  \
    else if ((dt) == FB200_F16) { using T = __half; __VA_ARGS__; } \
    else { fb200::set_error("bad dtype %d", (int)(dt)); return FB200_ERR_INVALID; } \
  } while (0)

}  // namespace fb200

// LayerNorm(+residual) and small-sequence multi-head attention (head_dim 32, and head_dim 16 for the 128-wide MaskFormer pixel-decoder encoder).
#include "common.cuh"

namespace fb200 {

// one warp per row; C <= 1024, C % 4 == 0. Two-pass (mean, then centred variance) in registers.
template <typename T, int MAXV>
__global__ void __launch_bounds__(256) layernorm_kernel(const T* __restrict__ x, const T* __restrict__ res,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        T* __restrict__ out, int64_t M, int C, float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int nv = C / 4;  // vectors per row
  float v[MAXV][4];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nv) {
      load4(x + row * C + vi * 4, v[i]);
      if (res) {
        float r[4];
        load4(res + row * C + vi * 4, r);
#pragma unroll
        for (int j = 0; j < 4; ++j) v[i][j] += r[j];
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) s += v[i][j];
    }
  }
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nv) {
#pragma unroll
      for (int j = 0; j < 4; ++j) { const float d = v[i][j] - mean; q += d * d; }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nv) {
      float g[4], b[4], o[4];
      load4(gamma + vi * 4, g);
      load4(beta + vi * 4, b);
#pragma unroll
      for (int j = 0; j < 4; ++j) o[j] = (v[i][j] - mean) * rstd * g[j] + b[j];
      store4(out + row * C + vi * 4, o);
    }
  }
}

// grid: (B*heads, ceil(Lq/QT)); block 256 = 8 warps; each warp owns QT/8 queries.
// smem: Ks[Lk][33] + Vs[Lk][32] + per-warp probabilities P[8][Lk] + per-warp q[8][32]  (fp32)
constexpr int ATT_QT = 64;
template <typename T>
__global__ void __launch_bounds__(256) attention_kernel(const T* __restrict__ q, int q_pitch, const T* __restrict__ k,
                                                        int k_pitch, const T* __restrict__ v, int v_pitch, T* __restrict__ out,
                                                        int out_pitch, int Lq, int Lk, int heads, float scale) {
  extern __shared__ float sm[];
  float* Ks = sm;                   // [Lk][33]
  float* Vs = Ks + (size_t)Lk * 33; // [Lk][32]
  float* Ps = Vs + (size_t)Lk * 32; // [8][Lk]
  float* Qs = Ps + (size_t)8 * Lk;  // [8][32]
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // cooperative load of K,V for (b,h): Lk rows x 32 channels; 8 threads x 4 elements per row
  for (int i = threadIdx.x; i < Lk * 8; i += blockDim.x) {
    const int r = i >> 3, c = (i & 7) * 4;
    float kv[4], vv[4];
    load4(k + ((int64_t)b * Lk + r) * k_pitch + h * 32 + c, kv);
    load4(v + ((int64_t)b * Lk + r) * v_pitch + h * 32 + c, vv);
#pragma unroll
    for (int j = 0; j < 4; ++j) { Ks[r * 33 + c + j] = kv[j]; Vs[r * 32 + c + j] = vv[j]; }
  }
  __syncthreads();
  const int q0 = blockIdx.y * ATT_QT;
  float* P = Ps + (size_t)warp * Lk;
  float* Q = Qs + warp * 32;
  for (int qi = q0 + warp; qi < min(q0 + ATT_QT, Lq); qi += 8) {
    Q[lane] = to_f(q[((int64_t)b * Lq + qi) * q_pitch + h * 32 + lane]) * scale;  // torch scales q before QK^T
    __syncwarp();
    float mx = -INFINITY;
    for (int j = lane; j < Lk; j += 32) {
      float s = 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) s = fmaf(Q[d], Ks[j * 33 + d], s);
      P[j] = s;
      mx = fmaxf(mx, s);
    }
    mx = warp_max(mx);
    float sum = 0.f;
    for (int j = lane; j < Lk; j += 32) {
      const float e = expf(P[j] - mx);
      P[j] = e;
      sum += e;
    }
    sum = warp_sum(sum);
    __syncwarp();
    float o = 0.f;
    for (int j = 0; j < Lk; ++j) o = fmaf(P[j], Vs[j * 32 + lane], o);
    out[((int64_t)b * Lq + qi) * out_pitch + h * 32 + lane] = from_f<T>(o / sum);
    __syncwarp();
  }
}

int attention_mma_split(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch, float* out, int out_pitch, int B, int Lq, int Lk,
                        int heads, float scale, int out_pair, cudaStream_t st);
int attention_mma(const __half* q, int q_pitch, const __half* k, int k_pitch, const __half* v, int v_pitch, __half* out, int out_pitch, int B,
                  int Lq, int Lk, int heads, float scale, cudaStream_t st);
int attention_mma_split_stream(const float* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, int kv_pair, int kv_lo_off, const uint8_t* mask, int MP,
                               const int* allowed, float* out, int out_pitch, int B, int Lq, int Lk, int heads, float scale, cudaStream_t st);
int attention_mma_stream(const __half* q, int q_pitch, const __half* k, int k_pitch, const __half* v, int v_pitch, const uint8_t* mask, int LkP,
                         const int* allowed, __half* out, int out_pitch, int B, int Lq, int Lk, int heads, float scale, cudaStream_t st);
int attention_masked_simt(const void* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, const uint8_t* mask, int LkP, const int* allowed, void* out,
                          int out_pitch, int dtype, int B, int Lq, int Lk, int heads, float scale, cudaStream_t st);  // mf_ops.cu

// Shared memory of the resident kernels, which stage the whole K and V of a (batch, head): above 227 KiB per block the entry points take the streaming kernels instead.
constexpr size_t kAttnSmemMax = 227 * 1024;
constexpr int AM_PITCH = 40;  // halves per smem row of the tensor-core kernels (32 + 8 pad): conflict-free ldmatrix
inline size_t attention_simt_smem(int Lk) { return ((size_t)Lk * 33 + (size_t)Lk * 32 + (size_t)8 * Lk + 8 * 32) * sizeof(float); }  // attention_kernel: Lk <= 792
inline size_t attention_mma_smem(int Lk) { return ((size_t)2 * ((Lk + 63) & ~63) + 64) * AM_PITCH * sizeof(__half); }                 // attention_mma_kernel: Lk <= 1408
// attention_mma_split_kernel with NW warps (16 queries each) per CTA: L <= 640 for self-attention, Lk <= 704 for Lq <= 32
inline size_t attention_split_smem(int Lk, int NW) { return ((size_t)4 * ((Lk + 63) & ~63) + 2 * 16 * NW) * AM_PITCH * sizeof(__half); }
int attention_split_warps(int Lq);
// head_dim 16 (defined below): CUDA-core, fp16 tensor-core and split-precision tensor-core paths, each with a resident and a streaming kernel
int attention_hd16_simt(const void* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, void* out, int out_pitch, int dtype, int B, int Lq, int Lk,
                        int heads, float scale, cudaStream_t st);
int attention_hd16_mma(bool split, const void* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, void* out, int out_pitch, int B, int Lq, int Lk,
                       int heads, float scale, cudaStream_t st);
}  // namespace fb200
using namespace fb200;

extern "C" int fb200_layernorm(const void* x, const void* res, const float* gamma, const float* beta, void* out, int dtype,
                               int64_t M, int C, float eps, void* stream) {
  FB_CHECK_ARG(x && gamma && beta && out, "layernorm: null pointer");
  FB_CHECK_ARG(C % 4 == 0 && C <= 1024 && M > 0, "layernorm: C must be a multiple of 4 and <= 1024 (got %d)", C);
  const unsigned grid = (unsigned)cdiv(M, 8);
  cudaStream_t st = (cudaStream_t)stream;
  if (C <= 256) { FB_DISPATCH_DTYPE(dtype, T, (layernorm_kernel<T, 2><<<grid, 256, 0, st>>>((const T*)x, (const T*)res, gamma, beta, (T*)out, M, C, eps))); }
  else { FB_DISPATCH_DTYPE(dtype, T, (layernorm_kernel<T, 8><<<grid, 256, 0, st>>>((const T*)x, (const T*)res, gamma, beta, (T*)out, M, C, eps))); }
  FB_CHECK_LAUNCH("layernorm");
  return FB200_OK;
}

extern "C" int fb200_attention(const void* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, void* out,
                               int out_pitch, int dtype, int B, int Lq, int Lk, int heads, int head_dim, float scale,
                               void* stream) {
  FB_CHECK_ARG(q && k && v && out, "attention: null pointer");
  FB_CHECK_ARG(head_dim == 32 || head_dim == 16, "attention: head_dim must be 16 or 32 (got %d)", head_dim);
  FB_CHECK_ARG(B > 0 && Lq > 0 && Lk > 0 && heads > 0, "attention: B, Lq, Lk and heads must be positive (got %d, %d, %d, %d)", B, Lq, Lk, heads);
  FB_CHECK_ARG(q_pitch % 4 == 0 && k_pitch % 4 == 0 && v_pitch % 4 == 0, "attention: pitches must be multiples of 4");
  const int w = heads * head_dim;  // a pitch below the row width would make neighbouring rows overlap
  FB_CHECK_ARG(q_pitch >= w, "attention: q_pitch (%d) < heads*%d (%d)", q_pitch, head_dim, w);
  FB_CHECK_ARG(k_pitch >= w, "attention: k_pitch (%d) < heads*%d (%d)", k_pitch, head_dim, w);
  FB_CHECK_ARG(v_pitch >= w, "attention: v_pitch (%d) < heads*%d (%d)", v_pitch, head_dim, w);
  FB_CHECK_ARG(out_pitch >= w, "attention: out_pitch (%d) < heads*%d (%d)", out_pitch, head_dim, w);
  const bool mma_ok = dtype == FB200_F16 && q_pitch % 8 == 0 && k_pitch % 8 == 0 && v_pitch % 8 == 0 && out_pitch % 2 == 0 &&
                      (((uintptr_t)q | (uintptr_t)k | (uintptr_t)v) & 15) == 0 && ((uintptr_t)out & 3) == 0;
  if (head_dim == 16) {
    FB_CHECK_ARG(dtype == FB200_F32 || dtype == FB200_F16, "attention: bad dtype");
    if (mma_ok) return attention_hd16_mma(false, q, q_pitch, k, k_pitch, v, v_pitch, out, out_pitch, B, Lq, Lk, heads, scale, (cudaStream_t)stream);
    return attention_hd16_simt(q, q_pitch, k, k_pitch, v, v_pitch, out, out_pitch, dtype, B, Lq, Lk, heads, scale, (cudaStream_t)stream);
  }
  if (mma_ok) {
    if (attention_mma_smem(Lk) <= kAttnSmemMax)
      return attention_mma((const __half*)q, q_pitch, (const __half*)k, k_pitch, (const __half*)v, v_pitch, (__half*)out, out_pitch, B, Lq, Lk, heads, scale,
                           (cudaStream_t)stream);
    return attention_mma_stream((const __half*)q, q_pitch, (const __half*)k, k_pitch, (const __half*)v, v_pitch, nullptr, 0, nullptr, (__half*)out, out_pitch, B, Lq, Lk,
                                heads, scale, (cudaStream_t)stream);
  }
  if (attention_simt_smem(Lk) > kAttnSmemMax)  // keys streamed 128 at a time by the masked kernel, without a mask
    return attention_masked_simt(q, q_pitch, k, k_pitch, v, v_pitch, nullptr, 0, nullptr, out, out_pitch, dtype, B, Lq, Lk, heads, scale, (cudaStream_t)stream);
  const size_t smem = attention_simt_smem(Lk);
  FB_CHECK_ARG(smem <= kAttnSmemMax, "attention: Lk=%d does not fit shared memory", Lk);
  dim3 grid(B * heads, (unsigned)cdiv(Lq, ATT_QT));
  cudaStream_t st = (cudaStream_t)stream;
  static bool configured = false;
  if (!configured) {  // raise the dynamic-smem ceiling once (not inside a stream capture)
    cudaFuncSetAttribute(attention_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(attention_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    configured = true;
  }
  if (dtype == FB200_F32) {
    attention_kernel<float><<<grid, 256, smem, st>>>((const float*)q, q_pitch, (const float*)k, k_pitch, (const float*)v, v_pitch, (float*)out, out_pitch, Lq, Lk, heads, scale);
  } else if (dtype == FB200_F16) {
    attention_kernel<__half><<<grid, 256, smem, st>>>((const __half*)q, q_pitch, (const __half*)k, k_pitch, (const __half*)v, v_pitch, (__half*)out, out_pitch, Lq, Lk, heads, scale);
  } else { set_error("attention: bad dtype"); return FB200_ERR_INVALID; }
  FB_CHECK_LAUNCH("attention");
  return FB200_OK;
}

extern "C" int fb200_attention_masked_split(const float* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, int kv_dtype, int64_t kv_lo_off,
                                            const uint8_t* mask, int LkP, const int* allowed, float* out, int out_pitch, int B, int Lq, int Lk, int heads, int head_dim,
                                            float scale, void* stream) {
  FB_CHECK_ARG(q && k && v && out && head_dim == 32, "attention_masked_split: null pointer or head_dim != 32");
  FB_CHECK_ARG((mask == nullptr) == (allowed == nullptr), "attention_masked_split: mask and allowed go together");
  FB_CHECK_ARG(kv_dtype == FB200_F32 || kv_dtype == FB200_F16PAIR, "attention_masked_split: k / v are fp32 tensors or fp16 [hi|lo] pairs");
  FB_CHECK_ARG(B > 0 && Lq > 0 && Lk > 0 && heads > 0, "attention_masked_split: bad shape");
  FB_CHECK_ARG(q_pitch % 4 == 0 && out_pitch % 2 == 0 && ((uintptr_t)q & 15) == 0 && ((uintptr_t)out & 7) == 0, "attention_masked_split: q / out pitches / alignment");
  FB_CHECK_ARG(q_pitch >= heads * 32, "attention_masked_split: q_pitch (%d) < heads*32 (%d)", q_pitch, heads * 32);
  FB_CHECK_ARG(out_pitch >= heads * 32, "attention_masked_split: out_pitch (%d) < heads*32 (%d)", out_pitch, heads * 32);
  if (kv_dtype == FB200_F32) {
    FB_CHECK_ARG(k_pitch % 4 == 0 && v_pitch % 4 == 0 && (((uintptr_t)k | (uintptr_t)v) & 15) == 0, "attention_masked_split: k / v pitches / alignment");
    FB_CHECK_ARG(k_pitch >= heads * 32 && v_pitch >= heads * 32, "attention_masked_split: k_pitch (%d) / v_pitch (%d) < heads*32 (%d)", k_pitch, v_pitch, heads * 32);
  } else {  // pair rows: hi plane at the pointer, lo plane kv_lo_off halves further, 16-byte copies
    FB_CHECK_ARG(k_pitch % 8 == 0 && v_pitch % 8 == 0 && kv_lo_off % 8 == 0 && kv_lo_off >= heads * 32 && k_pitch >= kv_lo_off + heads * 32 && v_pitch >= kv_lo_off + heads * 32 &&
                     (((uintptr_t)k | (uintptr_t)v) & 15) == 0, "attention_masked_split: pair k / v need 16-byte aligned planes inside the row pitch");
  }
  FB_CHECK_ARG(mask == nullptr || (LkP % 4 == 0 && LkP >= ((Lk + 1) & ~1) && ((uintptr_t)mask & 3) == 0), "attention_masked_split: mask rows must be 4-byte aligned, pitch %% 4 == 0");
  return attention_mma_split_stream(q, q_pitch, k, k_pitch, v, v_pitch, kv_dtype == FB200_F16PAIR ? 1 : 0, (int)kv_lo_off, mask, LkP, allowed, out, out_pitch, B, Lq, Lk, heads,
                                    scale, (cudaStream_t)stream);
}

extern "C" int fb200_attention_split(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch, void* out, int out_dtype, int out_pitch, int B,
                                     int Lq, int Lk, int heads, int head_dim, float scale, void* stream) {
  FB_CHECK_ARG(q && k && v && out, "attention_split: null pointer");
  FB_CHECK_ARG(head_dim == 32 || head_dim == 16, "attention_split: head_dim must be 16 or 32 (got %d)", head_dim);
  FB_CHECK_ARG(B > 0 && Lq > 0 && Lk > 0 && heads > 0, "attention_split: B, Lq, Lk and heads must be positive (got %d, %d, %d, %d)", B, Lq, Lk, heads);
  FB_CHECK_ARG(q_pitch % 4 == 0 && k_pitch % 4 == 0 && v_pitch % 4 == 0 && out_pitch % 2 == 0 && (((uintptr_t)q | (uintptr_t)k | (uintptr_t)v) & 15) == 0 &&
                   ((uintptr_t)out & 7) == 0, "attention_split: pitches / alignment");
  FB_CHECK_ARG(out_dtype == FB200_F32 || out_dtype == FB200_F16PAIR, "attention_split: out_dtype must be F32 or F16PAIR");
  const int w = heads * head_dim;  // a pitch below the row width would make neighbouring rows overlap
  FB_CHECK_ARG(q_pitch >= w, "attention_split: q_pitch (%d) < heads*%d (%d)", q_pitch, head_dim, w);
  FB_CHECK_ARG(k_pitch >= w, "attention_split: k_pitch (%d) < heads*%d (%d)", k_pitch, head_dim, w);
  FB_CHECK_ARG(v_pitch >= w, "attention_split: v_pitch (%d) < heads*%d (%d)", v_pitch, head_dim, w);
  FB_CHECK_ARG(out_pitch >= w, "attention_split: out_pitch (%d) < heads*%d (%d)", out_pitch, head_dim, w);
  if (head_dim == 16) {
    FB_CHECK_ARG(out_dtype == FB200_F32, "attention_split: head_dim 16 writes fp32 rows only (out_dtype F32)");
    return attention_hd16_mma(true, q, q_pitch, k, k_pitch, v, v_pitch, out, out_pitch, B, Lq, Lk, heads, scale, (cudaStream_t)stream);
  }
  FB_CHECK_ARG(out_dtype != FB200_F16PAIR || out_pitch >= 2 * heads * 32, "attention_split: pair rows are [hi(heads*32) | lo(heads*32)]");
  // fp32 rows above the resident kernel's shared memory: the masked streaming kernel without a mask (keys staged 256 at a time); pair rows are refused there
  if (out_dtype == FB200_F32 && attention_split_smem(Lk, attention_split_warps(Lq)) > kAttnSmemMax)
    return attention_mma_split_stream(q, q_pitch, k, k_pitch, v, v_pitch, 0, 0, nullptr, 0, nullptr, (float*)out, out_pitch, B, Lq, Lk, heads, scale, (cudaStream_t)stream);
  return attention_mma_split(q, q_pitch, k, k_pitch, v, v_pitch, (float*)out, out_pitch, B, Lq, Lk, heads, scale, out_dtype == FB200_F16PAIR ? 1 : 0, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// fp16 tensor-core attention (head_dim 32): legacy mma.sync.m16n8k16 is the right tool here — per (batch, head) the
// problem is 300..400 x 32, far below one wgmma tile; the whole K and V of a head stay in shared memory and each
// warp runs a flash-style online softmax over 64-key blocks for 16 queries.  4 warps = 64 queries per CTA.
// ------------------------------------------------------------------------------------------------
namespace fb200 {

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const __half* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], const __half* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

__global__ void __launch_bounds__(128) attention_mma_kernel(const __half* __restrict__ q, int q_pitch, const __half* __restrict__ k, int k_pitch,
                                                            const __half* __restrict__ v, int v_pitch, __half* __restrict__ out, int out_pitch,
                                                            int Lq, int Lk, int heads, float scale_log2) {
  extern __shared__ __align__(16) __half smh[];
  const int LkP = (Lk + 63) & ~63;            // keys padded to whole 64-key blocks (zero rows)
  __half* Ks = smh;                           // [LkP][AM_PITCH]
  __half* Vs = Ks + (size_t)LkP * AM_PITCH;   // [LkP][AM_PITCH]
  __half* Qs = Vs + (size_t)LkP * AM_PITCH;   // [64][AM_PITCH]
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int q0 = blockIdx.y * 64;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // cooperative loads: 4 x 16-byte vectors per row
  for (int i = tid; i < LkP * 4; i += 128) {
    const int r = i >> 2, c = (i & 3) * 8;
    uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
    if (r < Lk) {
      kv = *reinterpret_cast<const uint4*>(k + ((int64_t)b * Lk + r) * k_pitch + h * 32 + c);
      vv = *reinterpret_cast<const uint4*>(v + ((int64_t)b * Lk + r) * v_pitch + h * 32 + c);
    }
    *reinterpret_cast<uint4*>(Ks + r * AM_PITCH + c) = kv;
    *reinterpret_cast<uint4*>(Vs + r * AM_PITCH + c) = vv;
  }
  for (int i = tid; i < 64 * 4; i += 128) {
    const int r = i >> 2, c = (i & 3) * 8;
    uint4 qv = make_uint4(0, 0, 0, 0);
    if (q0 + r < Lq) qv = *reinterpret_cast<const uint4*>(q + ((int64_t)b * Lq + q0 + r) * q_pitch + h * 32 + c);
    *reinterpret_cast<uint4*>(Qs + r * AM_PITCH + c) = qv;
  }
  __syncthreads();
  // Q fragments of this warp's 16 queries: 2 k-steps (d 0-15, 16-31)
  uint32_t qa[2][4];
  {
    const int r = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
    const int c = (lane >> 4) * 8;
    ldsm_x4(qa[0], Qs + r * AM_PITCH + c);
    ldsm_x4(qa[1], Qs + r * AM_PITCH + 16 + c);
  }
  float o[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // rows lane/4 and lane/4+8
  for (int kb = 0; kb < LkP; kb += 64) {
    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int j = 0; j < 4; ++j) s[nt][j] = 0.f;
      uint32_t kf[4];  // B fragments: (d 0-7, 8-15) = k-step 0, (d 16-23, 24-31) = k-step 1, for keys kb+nt*8..+7
      ldsm_x4(kf, Ks + (kb + nt * 8 + (lane & 7)) * AM_PITCH + (lane >> 3) * 8);
      mma16816(s[nt], qa[0], kf[0], kf[1]);
      mma16816(s[nt], qa[1], kf[2], kf[3]);
    }
    // mask padded keys, block row max
    float bm0 = -INFINITY, bm1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int key = kb + nt * 8 + (lane & 3) * 2;
      if (key >= Lk) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
      if (key + 1 >= Lk) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
      bm0 = fmaxf(bm0, fmaxf(s[nt][0], s[nt][1]));
      bm1 = fmaxf(bm1, fmaxf(s[nt][2], s[nt][3]));
    }
    bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 1)); bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 2));
    bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 1)); bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 2));
    const float nm0 = fmaxf(m0, bm0), nm1 = fmaxf(m1, bm1);  // finite: every block holds at least one real key
    const float a0 = exp2f((m0 - nm0) * scale_log2), a1 = exp2f((m1 - nm1) * scale_log2);
    m0 = nm0; m1 = nm1;
    l0 *= a0; l1 *= a1;
#pragma unroll
    for (int i = 0; i < 4; ++i) { o[i][0] *= a0; o[i][1] *= a0; o[i][2] *= a1; o[i][3] *= a1; }
    uint32_t pa[4][4];  // P as A fragments: 4 k-steps of 16 keys
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float p0 = exp2f((s[nt][0] - m0) * scale_log2), p1 = exp2f((s[nt][1] - m0) * scale_log2);
      const float p2 = exp2f((s[nt][2] - m1) * scale_log2), p3 = exp2f((s[nt][3] - m1) * scale_log2);
      l0 += p0 + p1; l1 += p2 + p3;
      pa[nt >> 1][(nt & 1) * 2 + 0] = pack_h2(p0, p1);
      pa[nt >> 1][(nt & 1) * 2 + 1] = pack_h2(p2, p3);
    }
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {  // 16 keys per step
      const int r = kb + ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
      uint32_t vf[4];
      ldsm_x4_trans(vf, Vs + r * AM_PITCH + (lane >> 4) * 8);        // d 0-7 (b0,b1), d 8-15 (b0,b1)
      mma16816(o[0], pa[ks], vf[0], vf[1]);
      mma16816(o[1], pa[ks], vf[2], vf[3]);
      ldsm_x4_trans(vf, Vs + r * AM_PITCH + 16 + (lane >> 4) * 8);   // d 16-23, 24-31
      mma16816(o[2], pa[ks], vf[0], vf[1]);
      mma16816(o[3], pa[ks], vf[2], vf[3]);
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  const int r0 = q0 + warp * 16 + (lane >> 2), r1 = r0 + 8;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const int c = h * 32 + nt * 8 + (lane & 3) * 2;
    if (r0 < Lq) *reinterpret_cast<uint32_t*>(out + ((int64_t)b * Lq + r0) * out_pitch + c) = pack_h2(o[nt][0] * i0, o[nt][1] * i0);
    if (r1 < Lq) *reinterpret_cast<uint32_t*>(out + ((int64_t)b * Lq + r1) * out_pitch + c) = pack_h2(o[nt][2] * i1, o[nt][3] * i1);
  }
}

// Split-precision variant for fp32 tensors (precision="fp32_tc"): Q, K, V are split into [hi | lo] fp16 halves while being staged in shared memory;
// S = Qh Kh^T + Qh Kl^T + Ql Kh^T and O += Ph Vh + Ph Vl + Pl Vh (P = softmax numerators, split in registers) reproduce the fp32 products to ~2^-21,
// with the same fragment algebra and online softmax as attention_mma_kernel.  fp32 in, fp32 out.
__device__ __forceinline__ void split_store4(__half* hi, __half* lo, const float4 v) {
  const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
  const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
  const __half2 l0 = __floats2half2_rn(v.x - f0.x, v.y - f0.y), l1 = __floats2half2_rn(v.z - f1.x, v.w - f1.y);
  *reinterpret_cast<__half2*>(hi) = h0; *reinterpret_cast<__half2*>(hi + 2) = h1;
  *reinterpret_cast<__half2*>(lo) = l0; *reinterpret_cast<__half2*>(lo + 2) = l1;
}

// blockDim.x = 32 * NW (NW <= 12 warps, 16 queries each): the K/V planes of a (batch, head) are staged once per 16*NW queries.  out_pair: the output is written as the
// fp16 [hi | lo] pair (row = [hi(heads*32) | lo(heads*32)], pitch out_pitch in halves) for the out_proj tensor-core linear that follows.
__global__ void __launch_bounds__(384) attention_mma_split_kernel(const float* __restrict__ q, int q_pitch, const float* __restrict__ k, int k_pitch,
                                                                  const float* __restrict__ v, int v_pitch, float* __restrict__ out, int out_pitch,
                                                                  int Lq, int Lk, int heads, float scale_log2, int out_pair) {
  extern __shared__ __align__(16) __half smh[];
  const int LkP = (Lk + 63) & ~63;
  const size_t kv = (size_t)LkP * AM_PITCH;
  __half* Kh = smh; __half* Kl = Kh + kv; __half* Vh = Kl + kv; __half* Vl = Vh + kv;
  const int QB = (int)(blockDim.x >> 5) * 16;  // queries per CTA
  __half* Qh = Vl + kv; __half* Ql = Qh + QB * AM_PITCH;
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int q0 = blockIdx.y * QB;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < LkP * 8; i += (int)blockDim.x) {  // 8 x float4 per 32-wide row
    const int r = i >> 3, c = (i & 7) * 4;
    float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
    if (r < Lk) {
      kk = *reinterpret_cast<const float4*>(k + ((int64_t)b * Lk + r) * k_pitch + h * 32 + c);
      vv = *reinterpret_cast<const float4*>(v + ((int64_t)b * Lk + r) * v_pitch + h * 32 + c);
    }
    split_store4(Kh + r * AM_PITCH + c, Kl + r * AM_PITCH + c, kk);
    split_store4(Vh + r * AM_PITCH + c, Vl + r * AM_PITCH + c, vv);
  }
  for (int i = tid; i < QB * 8; i += (int)blockDim.x) {
    const int r = i >> 3, c = (i & 7) * 4;
    float4 qq = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < Lq) qq = *reinterpret_cast<const float4*>(q + ((int64_t)b * Lq + q0 + r) * q_pitch + h * 32 + c);
    split_store4(Qh + r * AM_PITCH + c, Ql + r * AM_PITCH + c, qq);
  }
  __syncthreads();
  uint32_t qah[2][4], qal[2][4];
  {
    const int r = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
    const int c = (lane >> 4) * 8;
    ldsm_x4(qah[0], Qh + r * AM_PITCH + c); ldsm_x4(qah[1], Qh + r * AM_PITCH + 16 + c);
    ldsm_x4(qal[0], Ql + r * AM_PITCH + c); ldsm_x4(qal[1], Ql + r * AM_PITCH + 16 + c);
  }
  float o[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  for (int kb = 0; kb < LkP; kb += 64) {
    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int j = 0; j < 4; ++j) s[nt][j] = 0.f;
      uint32_t kh[4], kl[4];
      const int off = (kb + nt * 8 + (lane & 7)) * AM_PITCH + (lane >> 3) * 8;
      ldsm_x4(kh, Kh + off);
      ldsm_x4(kl, Kl + off);
      mma16816(s[nt], qal[0], kh[0], kh[1]); mma16816(s[nt], qal[1], kh[2], kh[3]);   // small terms first
      mma16816(s[nt], qah[0], kl[0], kl[1]); mma16816(s[nt], qah[1], kl[2], kl[3]);
      mma16816(s[nt], qah[0], kh[0], kh[1]); mma16816(s[nt], qah[1], kh[2], kh[3]);
    }
    float bm0 = -INFINITY, bm1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int key = kb + nt * 8 + (lane & 3) * 2;
      if (key >= Lk) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
      if (key + 1 >= Lk) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
      bm0 = fmaxf(bm0, fmaxf(s[nt][0], s[nt][1]));
      bm1 = fmaxf(bm1, fmaxf(s[nt][2], s[nt][3]));
    }
    bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 1)); bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 2));
    bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 1)); bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 2));
    const float nm0 = fmaxf(m0, bm0), nm1 = fmaxf(m1, bm1);
    const float a0 = exp2f((m0 - nm0) * scale_log2), a1 = exp2f((m1 - nm1) * scale_log2);
    m0 = nm0; m1 = nm1;
    l0 *= a0; l1 *= a1;
#pragma unroll
    for (int i = 0; i < 4; ++i) { o[i][0] *= a0; o[i][1] *= a0; o[i][2] *= a1; o[i][3] *= a1; }
    uint32_t pah[4][4], pal[4][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float p0 = exp2f((s[nt][0] - m0) * scale_log2), p1 = exp2f((s[nt][1] - m0) * scale_log2);
      const float p2 = exp2f((s[nt][2] - m1) * scale_log2), p3 = exp2f((s[nt][3] - m1) * scale_log2);
      l0 += p0 + p1; l1 += p2 + p3;
      const __half2 h01 = __floats2half2_rn(p0, p1), h23 = __floats2half2_rn(p2, p3);
      const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
      pah[nt >> 1][(nt & 1) * 2 + 0] = *reinterpret_cast<const uint32_t*>(&h01);
      pah[nt >> 1][(nt & 1) * 2 + 1] = *reinterpret_cast<const uint32_t*>(&h23);
      pal[nt >> 1][(nt & 1) * 2 + 0] = pack_h2(p0 - f01.x, p1 - f01.y);
      pal[nt >> 1][(nt & 1) * 2 + 1] = pack_h2(p2 - f23.x, p3 - f23.y);
    }
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const int r = kb + ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
      for (int half = 0; half < 2; ++half) {  // d 0-15, d 16-31
        uint32_t vh[4], vl[4];
        const int off = r * AM_PITCH + half * 16 + (lane >> 4) * 8;
        ldsm_x4_trans(vh, Vh + off);
        ldsm_x4_trans(vl, Vl + off);
        mma16816(o[half * 2 + 0], pal[ks], vh[0], vh[1]); mma16816(o[half * 2 + 1], pal[ks], vh[2], vh[3]);
        mma16816(o[half * 2 + 0], pah[ks], vl[0], vl[1]); mma16816(o[half * 2 + 1], pah[ks], vl[2], vl[3]);
        mma16816(o[half * 2 + 0], pah[ks], vh[0], vh[1]); mma16816(o[half * 2 + 1], pah[ks], vh[2], vh[3]);
      }
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  const int r0 = q0 + warp * 16 + (lane >> 2), r1 = r0 + 8;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const int c = h * 32 + nt * 8 + (lane & 3) * 2;
    if (out_pair) {
      __half* oh = reinterpret_cast<__half*>(out);
      const int lo_off = heads * 32;
      if (r0 < Lq) {
        const float a0 = o[nt][0] * i0, a1 = o[nt][1] * i0;
        const __half2 hh = __floats2half2_rn(a0, a1);
        const float2 hf = __half22float2(hh);
        __half* dst = oh + ((int64_t)b * Lq + r0) * out_pitch + c;
        *reinterpret_cast<__half2*>(dst) = hh;
        *reinterpret_cast<__half2*>(dst + lo_off) = __floats2half2_rn(a0 - hf.x, a1 - hf.y);
      }
      if (r1 < Lq) {
        const float a0 = o[nt][2] * i1, a1 = o[nt][3] * i1;
        const __half2 hh = __floats2half2_rn(a0, a1);
        const float2 hf = __half22float2(hh);
        __half* dst = oh + ((int64_t)b * Lq + r1) * out_pitch + c;
        *reinterpret_cast<__half2*>(dst) = hh;
        *reinterpret_cast<__half2*>(dst + lo_off) = __floats2half2_rn(a0 - hf.x, a1 - hf.y);
      }
      continue;
    }
    if (r0 < Lq) *reinterpret_cast<float2*>(out + ((int64_t)b * Lq + r0) * out_pitch + c) = make_float2(o[nt][0] * i0, o[nt][1] * i0);
    if (r1 < Lq) *reinterpret_cast<float2*>(out + ((int64_t)b * Lq + r1) * out_pitch + c) = make_float2(o[nt][2] * i1, o[nt][3] * i1);
  }
}

int attention_split_warps(int Lq) {
  // queries per CTA: as few CTAs per (batch, head) as 16 warps allow (each CTA stages the whole K and V of its head), warps rounded to what the last block needs
  constexpr int max_q = 192;  // upper bound of queries per CTA (multiple of 16)
  const int nblk = (int)cdiv(Lq, max_q);
  return (int)cdiv(cdiv(Lq, nblk), 16);
}

int attention_mma_split(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch, float* out, int out_pitch, int B, int Lq, int Lk,
                        int heads, float scale, int out_pair, cudaStream_t st) {
  const int NW = attention_split_warps(Lq);
  const size_t smem = attention_split_smem(Lk, NW);
  if (smem > kAttnSmemMax) { set_error("attention(split): Lk=%d does not fit shared memory", Lk); return FB200_ERR_UNSUPPORTED; }
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(attention_mma_split_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    configured = true;
  }
  dim3 grid(B * heads, (unsigned)cdiv(Lq, 16 * NW));
  attention_mma_split_kernel<<<grid, 32 * NW, smem, st>>>(q, q_pitch, k, k_pitch, v, v_pitch, out, out_pitch, Lq, Lk, heads, scale * 1.4426950408889634f, out_pair);
  FB_CHECK_LAUNCH("attention_mma_split");
  return FB200_OK;
}

// Streaming, masked variant of attention_mma_split_kernel for the masked cross-attention of the MaskFormer-family decoders in the fp32-accurate mode (100 queries x up to
// (H/8 * W/8) keys; fai_mf/modelling.py:510-513, nn/layers/transformer.py:206-238): K / V are staged (and split into fp16 hi / lo planes) ASK keys at a time, the online
// softmax carries across the chunks; mask[b,q,key] != 0 removes a key unless allowed[b,q] == 0 (a fully masked row attends everywhere).  Same three-product fragment
// algebra as above; fp32 in, fp32 out.  Replaces the CUDA-core attention_masked_kernel<float> (two shared-memory loads per FMA; 7.8 of 37.9 ms of the bs=16 800x800 step).
// KVP: K and V arrive already as fp16 [hi | lo] pairs (written by the epilogue of their projection, conv2d_pair with out_pair) - rows [hi(heads*32) | ... | lo(heads*32)] with
// the lo plane kv_lo_off halves behind the hi plane.  Staging is then a plain 16-byte cp.async copy, double buffered (chunk c+1 lands while chunk c is multiplied); with fp32
// K / V the chunk is converted while it is staged (synchronously, single buffer).
__device__ __forceinline__ void cp_async16_zfill(void* dst, const void* src, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst);
  const int sz = valid ? 16 : 0;  // src-size 0: the 16 destination bytes are zero-filled, the source is not read
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(sz) : "memory");
}
template <bool KVP> __host__ __device__ constexpr int ask_keys() { return KVP ? 128 : 256; }  // keys per staged chunk
template <bool KVP>
__global__ void __launch_bounds__(384) attention_mma_split_stream_kernel(const float* __restrict__ q, int q_pitch, const void* __restrict__ k_, int k_pitch,
                                                                         const void* __restrict__ v_, int v_pitch, int kv_lo_off, const uint8_t* __restrict__ mask, int MP,
                                                                         const int* __restrict__ allowed, float* __restrict__ out, int out_pitch, int Lq, int Lk,
                                                                         int heads, float scale_log2) {
  extern __shared__ __align__(16) __half smh[];
  constexpr int ASK = ask_keys<KVP>();
  constexpr int NBUF = KVP ? 2 : 1;
  constexpr size_t kv = (size_t)ASK * AM_PITCH;
  const float* k = reinterpret_cast<const float*>(k_);
  const float* v = reinterpret_cast<const float*>(v_);
  const int QB = (int)(blockDim.x >> 5) * 16;  // queries per CTA
  __half* Qh = smh + NBUF * 4 * kv; __half* Ql = Qh + QB * AM_PITCH;
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int q0 = blockIdx.y * QB;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < QB * 8; i += (int)blockDim.x) {
    const int r = i >> 3, c = (i & 7) * 4;
    float4 qq = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < Lq) qq = *reinterpret_cast<const float4*>(q + ((int64_t)b * Lq + q0 + r) * q_pitch + h * 32 + c);
    split_store4(Qh + r * AM_PITCH + c, Ql + r * AM_PITCH + c, qq);
  }
  __syncthreads();
  uint32_t qah[2][4], qal[2][4];
  {
    const int r = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
    const int c = (lane >> 4) * 8;
    ldsm_x4(qah[0], Qh + r * AM_PITCH + c); ldsm_x4(qah[1], Qh + r * AM_PITCH + 16 + c);
    ldsm_x4(qal[0], Ql + r * AM_PITCH + c); ldsm_x4(qal[1], Ql + r * AM_PITCH + 16 + c);
  }
  // the two query rows of this thread's accumulator fragments, and their mask rows
  const int r0 = q0 + warp * 16 + (lane >> 2), r1 = r0 + 8;
  const bool um0 = mask != nullptr && r0 < Lq && allowed[b * Lq + r0] > 0, um1 = mask != nullptr && r1 < Lq && allowed[b * Lq + r1] > 0;
  const uint8_t* mrow0 = um0 ? mask + ((int64_t)b * Lq + r0) * MP : nullptr;
  const uint8_t* mrow1 = um1 ? mask + ((int64_t)b * Lq + r1) * MP : nullptr;
  float o[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  // pair K / V: issue the 16-byte copies of chunk `ci` into buffer ci & 1 (planes Kh, Kl, Vh, Vl; 4 x 16 B per 32-half row and plane)
  auto issue_pair_chunk = [&](int ci) {
    if constexpr (KVP) {
      const __half* kp = reinterpret_cast<const __half*>(k_);
      const __half* vp = reinterpret_cast<const __half*>(v_);
      __half* base = smh + (size_t)(ci & 1) * 4 * kv;
      const int c0 = ci * ASK;
      for (int i = tid; i < ASK * 16; i += (int)blockDim.x) {
        const int r = i >> 4, plane = (i >> 2) & 3, c = (i & 3) * 8;   // plane 0 = Kh, 1 = Kl, 2 = Vh, 3 = Vl
        const bool ok = c0 + r < Lk;
        const int64_t row = (int64_t)b * Lk + (ok ? c0 + r : 0);
        const __half* src = (plane < 2 ? kp + row * k_pitch : vp + row * v_pitch) + (plane & 1) * kv_lo_off + h * 32 + c;
        cp_async16_zfill(base + plane * kv + r * AM_PITCH + c, src, ok);
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
  };
  const int nchunks = (Lk + ASK - 1) / ASK;
  if constexpr (KVP) issue_pair_chunk(0);
  for (int ci = 0; ci < nchunks; ++ci) {
    const int c0 = ci * ASK;
    __half* Kh = smh + (size_t)(KVP ? (ci & 1) : 0) * 4 * kv; __half* Kl = Kh + kv; __half* Vh = Kl + kv; __half* Vl = Vh + kv;
    if constexpr (KVP) {
      if (ci + 1 < nchunks) { issue_pair_chunk(ci + 1); asm volatile("cp.async.wait_group 1;" ::: "memory"); }
      else asm volatile("cp.async.wait_group 0;" ::: "memory");
      __syncthreads();  // chunk ci has landed for every thread's copies
    } else {
      __syncthreads();  // the previous chunk has been consumed by every warp
      for (int i = tid; i < ASK * 8; i += (int)blockDim.x) {  // 8 x float4 per 32-wide row
        const int r = i >> 3, c = (i & 7) * 4;
        float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
        if (c0 + r < Lk) {
          kk = *reinterpret_cast<const float4*>(k + ((int64_t)b * Lk + c0 + r) * k_pitch + h * 32 + c);
          vv = *reinterpret_cast<const float4*>(v + ((int64_t)b * Lk + c0 + r) * v_pitch + h * 32 + c);
        }
        split_store4(Kh + r * AM_PITCH + c, Kl + r * AM_PITCH + c, kk);
        split_store4(Vh + r * AM_PITCH + c, Vl + r * AM_PITCH + c, vv);
      }
      __syncthreads();
    }
    const int kend = min(ASK, (Lk - c0 + 63) & ~63);
    for (int kb = 0; kb < kend; kb += 64) {
      float s[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int j = 0; j < 4; ++j) s[nt][j] = 0.f;
        uint32_t kh[4], kl[4];
        const int off = (kb + nt * 8 + (lane & 7)) * AM_PITCH + (lane >> 3) * 8;
        ldsm_x4(kh, Kh + off);
        ldsm_x4(kl, Kl + off);
        mma16816(s[nt], qal[0], kh[0], kh[1]); mma16816(s[nt], qal[1], kh[2], kh[3]);   // small terms first
        mma16816(s[nt], qah[0], kl[0], kl[1]); mma16816(s[nt], qah[1], kl[2], kl[3]);
        mma16816(s[nt], qah[0], kh[0], kh[1]); mma16816(s[nt], qah[1], kh[2], kh[3]);
      }
      float bm0 = -INFINITY, bm1 = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int key = c0 + kb + nt * 8 + (lane & 3) * 2;
        bool d00 = key >= Lk, d01 = key + 1 >= Lk, d10 = d00, d11 = d01;
        // the two mask bytes of a row in one 16-bit load (key is even, rows are 4-byte aligned with a pitch that is a multiple of 4: byte key + 1 always exists)
        if (um0 && !d00) { const uint32_t mm = *reinterpret_cast<const uint16_t*>(mrow0 + key); d00 = (mm & 0xffu) != 0; d01 = d01 || (mm >> 8) != 0; }
        if (um1 && !d10) { const uint32_t mm = *reinterpret_cast<const uint16_t*>(mrow1 + key); d10 = (mm & 0xffu) != 0; d11 = d11 || (mm >> 8) != 0; }
        if (d00) s[nt][0] = -INFINITY;
        if (d01) s[nt][1] = -INFINITY;
        if (d10) s[nt][2] = -INFINITY;
        if (d11) s[nt][3] = -INFINITY;
        bm0 = fmaxf(bm0, fmaxf(s[nt][0], s[nt][1]));
        bm1 = fmaxf(bm1, fmaxf(s[nt][2], s[nt][3]));
      }
      bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 1)); bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 2));
      bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 1)); bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 2));
      const float nm0 = fmaxf(m0, bm0), nm1 = fmaxf(m1, bm1);
      // a row whose keys so far are all masked keeps m = -inf: its rescale factor and its numerators are zero (never exp2(-inf + inf))
      const float a0 = (m0 == -INFINITY) ? 0.f : exp2f((m0 - nm0) * scale_log2), a1 = (m1 == -INFINITY) ? 0.f : exp2f((m1 - nm1) * scale_log2);
      m0 = nm0; m1 = nm1;
      l0 *= a0; l1 *= a1;
#pragma unroll
      for (int i = 0; i < 4; ++i) { o[i][0] *= a0; o[i][1] *= a0; o[i][2] *= a1; o[i][3] *= a1; }
      uint32_t pah[4][4], pal[4][4];
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float p0 = (s[nt][0] == -INFINITY) ? 0.f : exp2f((s[nt][0] - m0) * scale_log2), p1 = (s[nt][1] == -INFINITY) ? 0.f : exp2f((s[nt][1] - m0) * scale_log2);
        const float p2 = (s[nt][2] == -INFINITY) ? 0.f : exp2f((s[nt][2] - m1) * scale_log2), p3 = (s[nt][3] == -INFINITY) ? 0.f : exp2f((s[nt][3] - m1) * scale_log2);
        l0 += p0 + p1; l1 += p2 + p3;
        const __half2 h01 = __floats2half2_rn(p0, p1), h23 = __floats2half2_rn(p2, p3);
        const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
        pah[nt >> 1][(nt & 1) * 2 + 0] = *reinterpret_cast<const uint32_t*>(&h01);
        pah[nt >> 1][(nt & 1) * 2 + 1] = *reinterpret_cast<const uint32_t*>(&h23);
        pal[nt >> 1][(nt & 1) * 2 + 0] = pack_h2(p0 - f01.x, p1 - f01.y);
        pal[nt >> 1][(nt & 1) * 2 + 1] = pack_h2(p2 - f23.x, p3 - f23.y);
      }
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const int r = kb + ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
        for (int half = 0; half < 2; ++half) {  // d 0-15, d 16-31
          uint32_t vh[4], vl[4];
          const int off = r * AM_PITCH + half * 16 + (lane >> 4) * 8;
          ldsm_x4_trans(vh, Vh + off);
          ldsm_x4_trans(vl, Vl + off);
          mma16816(o[half * 2 + 0], pal[ks], vh[0], vh[1]); mma16816(o[half * 2 + 1], pal[ks], vh[2], vh[3]);
          mma16816(o[half * 2 + 0], pah[ks], vl[0], vl[1]); mma16816(o[half * 2 + 1], pah[ks], vl[2], vl[3]);
          mma16816(o[half * 2 + 0], pah[ks], vh[0], vh[1]); mma16816(o[half * 2 + 1], pah[ks], vh[2], vh[3]);
        }
      }
    }
    if constexpr (KVP) __syncthreads();  // every warp is done with buffer ci & 1 before chunk ci + 2 is copied into it
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const int c = h * 32 + nt * 8 + (lane & 3) * 2;
    if (r0 < Lq) *reinterpret_cast<float2*>(out + ((int64_t)b * Lq + r0) * out_pitch + c) = make_float2(o[nt][0] * i0, o[nt][1] * i0);
    if (r1 < Lq) *reinterpret_cast<float2*>(out + ((int64_t)b * Lq + r1) * out_pitch + c) = make_float2(o[nt][2] * i1, o[nt][3] * i1);
  }
}

int attention_mma_split_stream(const float* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, int kv_pair, int kv_lo_off, const uint8_t* mask, int MP,
                               const int* allowed, float* out, int out_pitch, int B, int Lq, int Lk, int heads, float scale, cudaStream_t st) {
  // upper bound of queries per CTA (multiple of 16): one CTA per (batch, head) for the 100-query decoders, K / V staged once (trip 52: 3.12 ms vs 3.31 at 64, 7.15 at 32)
  constexpr int qb = 128;
  const int nblk = (int)cdiv(Lq, qb);
  const int NW = (int)cdiv(cdiv(Lq, nblk), 16);
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(attention_mma_split_stream_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(attention_mma_split_stream_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    configured = true;
  }
  dim3 grid(B * heads, (unsigned)cdiv(Lq, 16 * NW));
  if (kv_pair) {
    const size_t smem = ((size_t)2 * 4 * ask_keys<true>() + 2 * 16 * NW) * AM_PITCH * sizeof(__half);
    attention_mma_split_stream_kernel<true><<<grid, 32 * NW, smem, st>>>(q, q_pitch, k, k_pitch, v, v_pitch, kv_lo_off, mask, MP, allowed, out, out_pitch, Lq, Lk, heads,
                                                                           scale * 1.4426950408889634f);
  } else {
    const size_t smem = ((size_t)4 * ask_keys<false>() + 2 * 16 * NW) * AM_PITCH * sizeof(__half);
    attention_mma_split_stream_kernel<false><<<grid, 32 * NW, smem, st>>>(q, q_pitch, k, k_pitch, v, v_pitch, 0, mask, MP, allowed, out, out_pitch, Lq, Lk, heads,
                                                                            scale * 1.4426950408889634f);
  }
  FB_CHECK_LAUNCH("attention_mma_split_stream");
  return FB200_OK;
}

int attention_mma(const __half* q, int q_pitch, const __half* k, int k_pitch, const __half* v, int v_pitch, __half* out, int out_pitch, int B,
                  int Lq, int Lk, int heads, float scale, cudaStream_t st) {
  const size_t smem = attention_mma_smem(Lk);
  if (smem > kAttnSmemMax) { set_error("attention(mma): Lk=%d does not fit shared memory", Lk); return FB200_ERR_UNSUPPORTED; }
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(attention_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    configured = true;
  }
  dim3 grid(B * heads, (unsigned)cdiv(Lq, 64));
  attention_mma_kernel<<<grid, 128, smem, st>>>(q, q_pitch, k, k_pitch, v, v_pitch, out, out_pitch, Lq, Lk, heads, scale * 1.4426950408889634f);
  FB_CHECK_LAUNCH("attention_mma");
  return FB200_OK;
}

}  // namespace fb200

// ------------------------------------------------------------------------------------------------
// Streaming variant for long key sequences (MaskFormer masked cross-attention: 100 queries x up to (H/8 * W/8) keys):
// 64-key K/V blocks are double-buffered through shared memory; an optional per-(batch, query, key) uint8 mask (shared by all
// heads) is applied to the score fragments.  Same mma.sync m16n8k16 fragment algebra as attention_mma_kernel above.
// ------------------------------------------------------------------------------------------------
namespace fb200 {

__global__ void __launch_bounds__(128) attention_mma_stream_kernel(const __half* __restrict__ q, int q_pitch, const __half* __restrict__ k, int k_pitch,
                                                                   const __half* __restrict__ v, int v_pitch, const uint8_t* __restrict__ mask, int LkP,
                                                                   const int* __restrict__ allowed, __half* __restrict__ out, int out_pitch, int Lq,
                                                                   int Lk, int heads, float scale_log2) {
  __shared__ __align__(16) __half Ks[2][64 * AM_PITCH];
  __shared__ __align__(16) __half Vs[2][64 * AM_PITCH];
  __shared__ __align__(16) __half Qs[64 * AM_PITCH];
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int q0 = blockIdx.y * 64;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nblk = (Lk + 63) / 64;
  // this thread's slice of a 64x32 block: rows r_ld, r_ld + 32 ; 8 halves at column c_ld
  const int r_ld = tid >> 2, c_ld = (tid & 3) * 8;
  uint4 kreg[2], vreg[2];
  auto fetch = [&](int blk) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int key = blk * 64 + r_ld + i * 32;
      kreg[i] = make_uint4(0, 0, 0, 0); vreg[i] = make_uint4(0, 0, 0, 0);
      if (key < Lk) {
        kreg[i] = *reinterpret_cast<const uint4*>(k + ((int64_t)b * Lk + key) * k_pitch + h * 32 + c_ld);
        vreg[i] = *reinterpret_cast<const uint4*>(v + ((int64_t)b * Lk + key) * v_pitch + h * 32 + c_ld);
      }
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      *reinterpret_cast<uint4*>(&Ks[buf][(r_ld + i * 32) * AM_PITCH + c_ld]) = kreg[i];
      *reinterpret_cast<uint4*>(&Vs[buf][(r_ld + i * 32) * AM_PITCH + c_ld]) = vreg[i];
    }
  };
  for (int i = tid; i < 64 * 4; i += 128) {
    const int r = i >> 2, c = (i & 3) * 8;
    uint4 qv = make_uint4(0, 0, 0, 0);
    if (q0 + r < Lq) qv = *reinterpret_cast<const uint4*>(q + ((int64_t)b * Lq + q0 + r) * q_pitch + h * 32 + c);
    *reinterpret_cast<uint4*>(Qs + r * AM_PITCH + c) = qv;
  }
  fetch(0);
  stash(0);
  __syncthreads();
  uint32_t qa[2][4];
  {
    const int r = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
    const int c = (lane >> 4) * 8;
    ldsm_x4(qa[0], Qs + r * AM_PITCH + c);
    ldsm_x4(qa[1], Qs + r * AM_PITCH + 16 + c);
  }
  // the two query rows this thread holds score columns for
  const int qr0 = q0 + warp * 16 + (lane >> 2), qr1 = qr0 + 8;
  const bool use0 = mask && qr0 < Lq && allowed[b * Lq + qr0] > 0, use1 = mask && qr1 < Lq && allowed[b * Lq + qr1] > 0;
  const uint8_t* mr0 = mask ? mask + ((int64_t)b * Lq + min(qr0, Lq - 1)) * LkP : nullptr;
  const uint8_t* mr1 = mask ? mask + ((int64_t)b * Lq + min(qr1, Lq - 1)) * LkP : nullptr;
  float o[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  for (int blk = 0; blk < nblk; ++blk) {
    const int buf = blk & 1, kb = blk * 64;
    if (blk + 1 < nblk) fetch(blk + 1);
    const __half* Kb = Ks[buf];
    const __half* Vb = Vs[buf];
    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int j = 0; j < 4; ++j) s[nt][j] = 0.f;
      uint32_t kf[4];
      ldsm_x4(kf, Kb + (nt * 8 + (lane & 7)) * AM_PITCH + (lane >> 3) * 8);
      mma16816(s[nt], qa[0], kf[0], kf[1]);
      mma16816(s[nt], qa[1], kf[2], kf[3]);
    }
    float bm0 = -INFINITY, bm1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int key = kb + nt * 8 + (lane & 3) * 2;  // even; LkP % 4 == 0 keeps the 2-byte mask loads aligned
      bool d00 = key >= Lk, d01 = key + 1 >= Lk, d10 = d00, d11 = d01;
      if (use0 && key < LkP) { const uchar2 mm = *reinterpret_cast<const uchar2*>(mr0 + key); d00 |= mm.x != 0; d01 |= mm.y != 0; }
      if (use1 && key < LkP) { const uchar2 mm = *reinterpret_cast<const uchar2*>(mr1 + key); d10 |= mm.x != 0; d11 |= mm.y != 0; }
      if (d00) s[nt][0] = -INFINITY;
      if (d01) s[nt][1] = -INFINITY;
      if (d10) s[nt][2] = -INFINITY;
      if (d11) s[nt][3] = -INFINITY;
      bm0 = fmaxf(bm0, fmaxf(s[nt][0], s[nt][1]));
      bm1 = fmaxf(bm1, fmaxf(s[nt][2], s[nt][3]));
    }
    bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 1)); bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 2));
    bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 1)); bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 2));
    const float nm0 = fmaxf(m0, bm0), nm1 = fmaxf(m1, bm1);
    const float z0 = (nm0 == -INFINITY) ? 0.f : nm0, z1 = (nm1 == -INFINITY) ? 0.f : nm1;  // fully-masked-so-far rows stay at zero mass
    const float a0 = exp2f((m0 - z0) * scale_log2), a1 = exp2f((m1 - z1) * scale_log2);
    m0 = nm0; m1 = nm1;
    l0 *= a0; l1 *= a1;
#pragma unroll
    for (int i = 0; i < 4; ++i) { o[i][0] *= a0; o[i][1] *= a0; o[i][2] *= a1; o[i][3] *= a1; }
    uint32_t pa[4][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float p0 = exp2f((s[nt][0] - z0) * scale_log2), p1 = exp2f((s[nt][1] - z0) * scale_log2);
      const float p2 = exp2f((s[nt][2] - z1) * scale_log2), p3 = exp2f((s[nt][3] - z1) * scale_log2);
      l0 += p0 + p1; l1 += p2 + p3;
      pa[nt >> 1][(nt & 1) * 2 + 0] = pack_h2(p0, p1);
      pa[nt >> 1][(nt & 1) * 2 + 1] = pack_h2(p2, p3);
    }
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const int r = ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
      uint32_t vf[4];
      ldsm_x4_trans(vf, Vb + r * AM_PITCH + (lane >> 4) * 8);
      mma16816(o[0], pa[ks], vf[0], vf[1]);
      mma16816(o[1], pa[ks], vf[2], vf[3]);
      ldsm_x4_trans(vf, Vb + r * AM_PITCH + 16 + (lane >> 4) * 8);
      mma16816(o[2], pa[ks], vf[0], vf[1]);
      mma16816(o[3], pa[ks], vf[2], vf[3]);
    }
    if (blk + 1 < nblk) stash(buf ^ 1);  // the other buffer was last read in iteration blk-1, separated by the barrier below
    __syncthreads();
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const int c = h * 32 + nt * 8 + (lane & 3) * 2;
    if (qr0 < Lq) *reinterpret_cast<uint32_t*>(out + ((int64_t)b * Lq + qr0) * out_pitch + c) = pack_h2(o[nt][0] * i0, o[nt][1] * i0);
    if (qr1 < Lq) *reinterpret_cast<uint32_t*>(out + ((int64_t)b * Lq + qr1) * out_pitch + c) = pack_h2(o[nt][2] * i1, o[nt][3] * i1);
  }
}

int attention_mma_stream(const __half* q, int q_pitch, const __half* k, int k_pitch, const __half* v, int v_pitch, const uint8_t* mask, int LkP,
                         const int* allowed, __half* out, int out_pitch, int B, int Lq, int Lk, int heads, float scale, cudaStream_t st) {
  dim3 grid(B * heads, (unsigned)cdiv(Lq, 64));
  attention_mma_stream_kernel<<<grid, 128, 0, st>>>(q, q_pitch, k, k_pitch, v, v_pitch, mask, LkP, allowed, out, out_pitch, Lq, Lk, heads,
                                                    scale * 1.4426950408889634f);
  FB_CHECK_LAUNCH("attention_mma_stream");
  return FB200_OK;
}

}  // namespace fb200

// ------------------------------------------------------------------------------------------------
// head_dim 16: the encoder of the 128-wide MaskFormer pixel decoders (fai-mf-m / -s: 8 heads x 16 channels, unmasked self-attention over
// ceil(H/32) * ceil(W/32) tokens per image).  Three arithmetics, each with a kernel that keeps the whole K / V of a (batch, head) in shared memory
// (STREAM = false) and one that stages them CHUNK keys at a time with the online softmax carried across chunks (STREAM = true), taken above the
// resident kernel's shared-memory ceiling.  Both variants run the same code; the resident one has a single chunk.
// ------------------------------------------------------------------------------------------------
namespace fb200 {

// CUDA-core kernel (fp32 rows, and fp16 rows the tensor-core kernel cannot read): a warp runs two queries at once, one per half-warp, lane & 15 = channel;
// 8 warps x 4 query pairs = 64 queries per CTA.  grid (B*heads, ceil(Lq/64)), block 256.
// smem (floats): Ks[CH][17] + Vs[CH][16] + P[16][CH+1] (one row per half-warp) + Qs[64][16]
constexpr int ATT16_QT = 64, ATT16_PAIRS = 4, ATT16_CHUNK = 256;
inline size_t attention_hd16_simt_smem(int keys) { return ((size_t)keys * 17 + (size_t)keys * 16 + (size_t)16 * (keys + 1) + ATT16_QT * 16) * sizeof(float); }  // resident: Lk <= 1164

__device__ __forceinline__ float half_warp_max(float v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float half_warp_sum(float v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename T, bool STREAM>
__global__ void __launch_bounds__(256) attention_hd16_kernel(const T* __restrict__ q, int q_pitch, const T* __restrict__ k, int k_pitch, const T* __restrict__ v,
                                                             int v_pitch, T* __restrict__ out, int out_pitch, int Lq, int Lk, int heads, float scale) {
  extern __shared__ float sm[];
  const int CH = STREAM ? ATT16_CHUNK : Lk;  // keys staged at a time
  float* Ks = sm;                           // [CH][17]
  float* Vs = Ks + (size_t)CH * 17;         // [CH][16]
  float* Ps = Vs + (size_t)CH * 16;         // [16][CH + 1]
  float* Qs = Ps + (size_t)16 * (CH + 1);   // [64][16]
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, hq = lane >> 4, c = lane & 15;
  const int q0 = blockIdx.y * ATT16_QT;
  for (int i = threadIdx.x; i < ATT16_QT * 4; i += blockDim.x) {  // the CTA's queries, scaled (torch scales q before QK^T); rows past Lq are zero
    const int r = i >> 2, cc = (i & 3) * 4;
    float qv[4] = {0.f, 0.f, 0.f, 0.f};
    if (q0 + r < Lq) load4(q + ((int64_t)b * Lq + q0 + r) * q_pitch + h * 16 + cc, qv);
#pragma unroll
    for (int j = 0; j < 4; ++j) Qs[r * 16 + cc + j] = qv[j] * scale;
  }
  float* P = Ps + (size_t)(warp * 2 + hq) * (CH + 1);
  float o[ATT16_PAIRS], m[ATT16_PAIRS], l[ATT16_PAIRS];
#pragma unroll
  for (int p = 0; p < ATT16_PAIRS; ++p) { o[p] = 0.f; m[p] = -INFINITY; l[p] = 0.f; }
  for (int c0 = 0; c0 < Lk; c0 += CH) {
    const int n = min(CH, Lk - c0);
    __syncthreads();  // the previous chunk has been consumed by every warp
    for (int i = threadIdx.x; i < n * 4; i += blockDim.x) {
      const int r = i >> 2, cc = (i & 3) * 4;
      float kv[4], vv[4];
      load4(k + ((int64_t)b * Lk + c0 + r) * k_pitch + h * 16 + cc, kv);
      load4(v + ((int64_t)b * Lk + c0 + r) * v_pitch + h * 16 + cc, vv);
#pragma unroll
      for (int j = 0; j < 4; ++j) { Ks[r * 17 + cc + j] = kv[j]; Vs[r * 16 + cc + j] = vv[j]; }
    }
    __syncthreads();
#pragma unroll
    for (int p = 0; p < ATT16_PAIRS; ++p) {
      const float* Q = Qs + ((warp * ATT16_PAIRS + p) * 2 + hq) * 16;
      float mx = -INFINITY;
      for (int j = c; j < n; j += 16) {
        float s = 0.f;
#pragma unroll
        for (int d = 0; d < 16; ++d) s = fmaf(Q[d], Ks[j * 17 + d], s);
        P[j] = s;
        mx = fmaxf(mx, s);
      }
      const float nm = fmaxf(m[p], half_warp_max(mx));  // finite: every chunk holds at least one key
      const float a = expf(m[p] - nm);                  // 0 on the first chunk
      float sum = 0.f;
      for (int j = c; j < n; j += 16) {
        const float e = expf(P[j] - nm);
        P[j] = e;
        sum += e;
      }
      l[p] = l[p] * a + half_warp_sum(sum);
      m[p] = nm;
      __syncwarp();
      float acc = 0.f;
      for (int j = 0; j < n; ++j) acc = fmaf(P[j], Vs[j * 16 + c], acc);
      o[p] = o[p] * a + acc;
      __syncwarp();
    }
  }
#pragma unroll
  for (int p = 0; p < ATT16_PAIRS; ++p) {
    const int qi = q0 + (warp * ATT16_PAIRS + p) * 2 + hq;
    if (qi < Lq) out[((int64_t)b * Lq + qi) * out_pitch + h * 16 + c] = from_f<T>(o[p] / l[p]);
  }
}

int attention_hd16_simt(const void* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, void* out, int out_pitch, int dtype, int B, int Lq, int Lk,
                        int heads, float scale, cudaStream_t st) {
  const bool stream = attention_hd16_simt_smem(Lk) > kAttnSmemMax;
  const size_t smem = attention_hd16_simt_smem(stream ? ATT16_CHUNK : Lk);
  static bool configured = false;
  if (!configured) {  // raise the dynamic-smem ceiling once (not inside a stream capture)
    cudaFuncSetAttribute(attention_hd16_kernel<float, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(attention_hd16_kernel<__half, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(attention_hd16_kernel<float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);   // 53 KiB chunks
    cudaFuncSetAttribute(attention_hd16_kernel<__half, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    configured = true;
  }
  dim3 grid(B * heads, (unsigned)cdiv(Lq, ATT16_QT));
  if (stream) {
    FB_DISPATCH_DTYPE(dtype, T, (attention_hd16_kernel<T, true><<<grid, 256, smem, st>>>((const T*)q, q_pitch, (const T*)k, k_pitch, (const T*)v, v_pitch, (T*)out, out_pitch,
                                                                                         Lq, Lk, heads, scale)));
  } else {
    FB_DISPATCH_DTYPE(dtype, T, (attention_hd16_kernel<T, false><<<grid, 256, smem, st>>>((const T*)q, q_pitch, (const T*)k, k_pitch, (const T*)v, v_pitch, (T*)out, out_pitch,
                                                                                          Lq, Lk, heads, scale)));
  }
  FB_CHECK_LAUNCH("attention_hd16");
  return FB200_OK;
}

// Tensor-core kernels (mma.sync.m16n8k16, 16 queries per warp): QK^T is a single k-step per 8-key tile, PV two n8 tiles.  SPLIT = false: fp16 rows in and out
// (the "fp16" mode).  SPLIT = true: fp32 rows in and out (the "fp32_tc" mode), Q, K, V split into fp16 [hi | lo] planes while staged, three products per
// term (hi*hi + hi*lo + lo*hi) and the softmax in fp32, as attention_mma_split_kernel does for 32-channel heads.
// smem (halves): K / V planes [CH][AM16_PITCH] (2 fp16, 4 split) + Q planes [16*NW][AM16_PITCH] (1 fp16, 2 split); CH = keys rounded up to 64 (resident) or 256
constexpr int AM16_PITCH = 24;  // halves per smem row (16 + 8 pad): the 8 rows of an ldmatrix land in distinct banks
constexpr int AM16_CHUNK = 256;
inline size_t attention_hd16_mma_smem(bool split, int keys, int NW) {  // resident: Lk <= 2368 (fp16, 4 warps); self-attention L <= 1088 (split, NW from attention_split_warps)
  return ((size_t)(split ? 4 : 2) * ((keys + 63) & ~63) + (size_t)(split ? 2 : 1) * 16 * NW) * AM16_PITCH * sizeof(__half);
}

template <bool SPLIT, bool STREAM>
__global__ void __launch_bounds__(384) attention_hd16_mma_kernel(const void* __restrict__ q_, int q_pitch, const void* __restrict__ k_, int k_pitch,
                                                                 const void* __restrict__ v_, int v_pitch, void* __restrict__ out_, int out_pitch, int Lq, int Lk,
                                                                 int heads, float scale_log2) {
  extern __shared__ __align__(16) __half smh[];
  const int CH = STREAM ? AM16_CHUNK : ((Lk + 63) & ~63);  // keys staged at a time
  const size_t kv = (size_t)CH * AM16_PITCH;
  __half* Kh = smh; __half* Vh = Kh + kv;
  __half* Kl = Vh + kv; __half* Vl = Kl + kv;  // split only
  const int QB = (int)(blockDim.x >> 5) * 16;   // queries per CTA
  __half* Qh = smh + (SPLIT ? 4 : 2) * kv; __half* Ql = Qh + QB * AM16_PITCH;
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int q0 = blockIdx.y * QB;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if constexpr (SPLIT) {
    const float* q = reinterpret_cast<const float*>(q_);
    for (int i = tid; i < QB * 4; i += (int)blockDim.x) {  // 4 x float4 per 16-wide row
      const int r = i >> 2, c = (i & 3) * 4;
      float4 qq = make_float4(0.f, 0.f, 0.f, 0.f);
      if (q0 + r < Lq) qq = *reinterpret_cast<const float4*>(q + ((int64_t)b * Lq + q0 + r) * q_pitch + h * 16 + c);
      split_store4(Qh + r * AM16_PITCH + c, Ql + r * AM16_PITCH + c, qq);
    }
  } else {
    const __half* q = reinterpret_cast<const __half*>(q_);
    for (int i = tid; i < QB * 2; i += (int)blockDim.x) {  // 2 x 16 bytes per row
      const int r = i >> 1, c = (i & 1) * 8;
      uint4 qv = make_uint4(0, 0, 0, 0);
      if (q0 + r < Lq) qv = *reinterpret_cast<const uint4*>(q + ((int64_t)b * Lq + q0 + r) * q_pitch + h * 16 + c);
      *reinterpret_cast<uint4*>(Qh + r * AM16_PITCH + c) = qv;
    }
  }
  __syncthreads();
  uint32_t qah[4], qal[4];  // A fragments of this warp's 16 queries (one k-step: d 0-15)
  {
    const int r = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
    const int c = (lane >> 4) * 8;
    ldsm_x4(qah, Qh + r * AM16_PITCH + c);
    if constexpr (SPLIT) ldsm_x4(qal, Ql + r * AM16_PITCH + c);
  }
  float o[2][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;  // rows lane/4 and lane/4+8
  for (int c0 = 0; c0 < Lk; c0 += CH) {
    const int rows = min(CH, (Lk - c0 + 63) & ~63);  // staged rows: whole 64-key blocks, zero past Lk
    __syncthreads();  // the previous chunk has been consumed by every warp
    if constexpr (SPLIT) {
      const float* k = reinterpret_cast<const float*>(k_);
      const float* v = reinterpret_cast<const float*>(v_);
      for (int i = tid; i < rows * 4; i += (int)blockDim.x) {
        const int r = i >> 2, c = (i & 3) * 4;
        float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
        if (c0 + r < Lk) {
          kk = *reinterpret_cast<const float4*>(k + ((int64_t)b * Lk + c0 + r) * k_pitch + h * 16 + c);
          vv = *reinterpret_cast<const float4*>(v + ((int64_t)b * Lk + c0 + r) * v_pitch + h * 16 + c);
        }
        split_store4(Kh + r * AM16_PITCH + c, Kl + r * AM16_PITCH + c, kk);
        split_store4(Vh + r * AM16_PITCH + c, Vl + r * AM16_PITCH + c, vv);
      }
    } else {
      const __half* k = reinterpret_cast<const __half*>(k_);
      const __half* v = reinterpret_cast<const __half*>(v_);
      for (int i = tid; i < rows * 2; i += (int)blockDim.x) {
        const int r = i >> 1, c = (i & 1) * 8;
        uint4 kk = make_uint4(0, 0, 0, 0), vv = kk;
        if (c0 + r < Lk) {
          kk = *reinterpret_cast<const uint4*>(k + ((int64_t)b * Lk + c0 + r) * k_pitch + h * 16 + c);
          vv = *reinterpret_cast<const uint4*>(v + ((int64_t)b * Lk + c0 + r) * v_pitch + h * 16 + c);
        }
        *reinterpret_cast<uint4*>(Kh + r * AM16_PITCH + c) = kk;
        *reinterpret_cast<uint4*>(Vh + r * AM16_PITCH + c) = vv;
      }
    }
    __syncthreads();
    for (int kb = 0; kb < rows; kb += 64) {
      float s[8][4];
#pragma unroll
      for (int nt = 0; nt < 8; nt += 2) {
#pragma unroll
        for (int j = 0; j < 4; ++j) { s[nt][j] = 0.f; s[nt + 1][j] = 0.f; }
        // one x4 ldmatrix = the B fragments of two 8-key tiles: (keys nt*8.., d 0-7 | d 8-15), (keys nt*8+8.., d 0-7 | d 8-15)
        const int off = (kb + nt * 8 + (lane & 7) + (lane >> 4) * 8) * AM16_PITCH + ((lane >> 3) & 1) * 8;
        uint32_t kh[4];
        ldsm_x4(kh, Kh + off);
        if constexpr (SPLIT) {
          uint32_t kl[4];
          ldsm_x4(kl, Kl + off);
          mma16816(s[nt], qal, kh[0], kh[1]); mma16816(s[nt + 1], qal, kh[2], kh[3]);  // small terms first
          mma16816(s[nt], qah, kl[0], kl[1]); mma16816(s[nt + 1], qah, kl[2], kl[3]);
        }
        mma16816(s[nt], qah, kh[0], kh[1]); mma16816(s[nt + 1], qah, kh[2], kh[3]);
      }
      float bm0 = -INFINITY, bm1 = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int key = c0 + kb + nt * 8 + (lane & 3) * 2;
        if (key >= Lk) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
        if (key + 1 >= Lk) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
        bm0 = fmaxf(bm0, fmaxf(s[nt][0], s[nt][1]));
        bm1 = fmaxf(bm1, fmaxf(s[nt][2], s[nt][3]));
      }
      bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 1)); bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 2));
      bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 1)); bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 2));
      const float nm0 = fmaxf(m0, bm0), nm1 = fmaxf(m1, bm1);  // finite: every 64-key block holds at least one real key
      const float a0 = exp2f((m0 - nm0) * scale_log2), a1 = exp2f((m1 - nm1) * scale_log2);
      m0 = nm0; m1 = nm1;
      l0 *= a0; l1 *= a1;
#pragma unroll
      for (int i = 0; i < 2; ++i) { o[i][0] *= a0; o[i][1] *= a0; o[i][2] *= a1; o[i][3] *= a1; }
      uint32_t pah[4][4], pal[4][4];  // P as A fragments: 4 k-steps of 16 keys
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float p0 = exp2f((s[nt][0] - m0) * scale_log2), p1 = exp2f((s[nt][1] - m0) * scale_log2);
        const float p2 = exp2f((s[nt][2] - m1) * scale_log2), p3 = exp2f((s[nt][3] - m1) * scale_log2);
        l0 += p0 + p1; l1 += p2 + p3;
        const __half2 h01 = __floats2half2_rn(p0, p1), h23 = __floats2half2_rn(p2, p3);
        pah[nt >> 1][(nt & 1) * 2 + 0] = *reinterpret_cast<const uint32_t*>(&h01);
        pah[nt >> 1][(nt & 1) * 2 + 1] = *reinterpret_cast<const uint32_t*>(&h23);
        if constexpr (SPLIT) {
          const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
          pal[nt >> 1][(nt & 1) * 2 + 0] = pack_h2(p0 - f01.x, p1 - f01.y);
          pal[nt >> 1][(nt & 1) * 2 + 1] = pack_h2(p2 - f23.x, p3 - f23.y);
        }
      }
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {  // 16 keys per step; one x4.trans ldmatrix = (d 0-7, d 8-15) x (keys 0-7, 8-15)
        const int off = (kb + ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * AM16_PITCH + (lane >> 4) * 8;
        uint32_t vh[4];
        ldsm_x4_trans(vh, Vh + off);
        if constexpr (SPLIT) {
          uint32_t vl[4];
          ldsm_x4_trans(vl, Vl + off);
          mma16816(o[0], pal[ks], vh[0], vh[1]); mma16816(o[1], pal[ks], vh[2], vh[3]);
          mma16816(o[0], pah[ks], vl[0], vl[1]); mma16816(o[1], pah[ks], vl[2], vl[3]);
        }
        mma16816(o[0], pah[ks], vh[0], vh[1]); mma16816(o[1], pah[ks], vh[2], vh[3]);
      }
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
  const int r0 = q0 + warp * 16 + (lane >> 2), r1 = r0 + 8;
#pragma unroll
  for (int nt = 0; nt < 2; ++nt) {
    const int c = h * 16 + nt * 8 + (lane & 3) * 2;
    if constexpr (SPLIT) {
      float* out = reinterpret_cast<float*>(out_);
      if (r0 < Lq) *reinterpret_cast<float2*>(out + ((int64_t)b * Lq + r0) * out_pitch + c) = make_float2(o[nt][0] * i0, o[nt][1] * i0);
      if (r1 < Lq) *reinterpret_cast<float2*>(out + ((int64_t)b * Lq + r1) * out_pitch + c) = make_float2(o[nt][2] * i1, o[nt][3] * i1);
    } else {
      __half* out = reinterpret_cast<__half*>(out_);
      if (r0 < Lq) *reinterpret_cast<uint32_t*>(out + ((int64_t)b * Lq + r0) * out_pitch + c) = pack_h2(o[nt][0] * i0, o[nt][1] * i0);
      if (r1 < Lq) *reinterpret_cast<uint32_t*>(out + ((int64_t)b * Lq + r1) * out_pitch + c) = pack_h2(o[nt][2] * i1, o[nt][3] * i1);
    }
  }
}

int attention_hd16_mma(bool split, const void* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, void* out, int out_pitch, int B, int Lq, int Lk,
                       int heads, float scale, cudaStream_t st) {
  const int NW = split ? attention_split_warps(Lq) : 4;  // 16 queries per warp
  const bool stream = attention_hd16_mma_smem(split, Lk, NW) > kAttnSmemMax;
  const size_t smem = attention_hd16_mma_smem(split, stream ? AM16_CHUNK : Lk, NW);
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(attention_hd16_mma_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(attention_hd16_mma_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(attention_hd16_mma_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(attention_hd16_mma_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);   // up to 66 KiB
    configured = true;
  }
  dim3 grid(B * heads, (unsigned)cdiv(Lq, 16 * NW));
  const float sl2 = scale * 1.4426950408889634f;
  if (split && stream) attention_hd16_mma_kernel<true, true><<<grid, 32 * NW, smem, st>>>(q, q_pitch, k, k_pitch, v, v_pitch, out, out_pitch, Lq, Lk, heads, sl2);
  else if (split) attention_hd16_mma_kernel<true, false><<<grid, 32 * NW, smem, st>>>(q, q_pitch, k, k_pitch, v, v_pitch, out, out_pitch, Lq, Lk, heads, sl2);
  else if (stream) attention_hd16_mma_kernel<false, true><<<grid, 32 * NW, smem, st>>>(q, q_pitch, k, k_pitch, v, v_pitch, out, out_pitch, Lq, Lk, heads, sl2);
  else attention_hd16_mma_kernel<false, false><<<grid, 32 * NW, smem, st>>>(q, q_pitch, k, k_pitch, v, v_pitch, out, out_pitch, Lq, Lk, heads, sl2);
  FB_CHECK_LAUNCH("attention_hd16_mma");
  return FB200_OK;
}

}  // namespace fb200

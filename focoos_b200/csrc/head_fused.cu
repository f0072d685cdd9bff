// Row-wise glue of the query-selection / decoder / AIFI chain in the fp32-accurate mode (precision "fp32_tc"), fused so that every tensor-core linear reads its
// operand in the pair format straight from the kernel that produced it (no split_f32_pair / add / row_select / gather launches in between):
//   * layernorm_ex      LayerNorm over rows that may be gathered (top-k indices) and masked (valid_mask fill), written as fp32 and/or as the fp16 [hi|lo] pair,
//                       plus the pair of (y + pos) for the next q/k or sampling-offset projection
//   * split_pair_ex     pair(act(x)) and / or pair(x + pos) of an fp32 tensor in one pass
//   * box_refine_qpos   bbox refinement (inverse_sigmoid(ref) + delta -> sigmoid) and the first query_pos_head layer (4 -> 512, ReLU) of the NEXT decoder layer
//   * sigmoid_rows      sigmoid of a pitched [M, C] logits buffer into a dense one
// The arithmetic of each piece is the one of the kernel it replaces (same reduction order), so results are bit-identical to the unfused launches.
#include "common.cuh"

namespace fb200 {

__device__ __forceinline__ void pair_store4(__half* hi, __half* lo, const float (&v)[4]) {
  float h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) { h[j] = __half2float(__float2half_rn(v[j])); l[j] = v[j] - h[j]; }
  store4(hi, h);
  store4(lo, l);
}

struct LnExArgs {
  const float* x; int x_pitch;          // source rows
  const float* res;                     // optional residual [M, C] dense (added before the statistics)
  const int* gather; int gK; int S;     // gather != null: output row m reads source row (m / gK) * S + gather[m]
  const uint8_t* valid; const float* fill;  // valid != null: a source row r with !valid[r % S] is replaced by fill[C] (modelling.py:1202 memory * valid_mask behind enc_output.0)
  const float* gamma; const float* beta; float eps;
  int64_t M; int C;
  float* out_f32;                       // optional [M, C]
  __half* out_pair;                     // optional [M, 2C] = [hi | lo]
  const float* pos; int64_t pos_rows;   // optional positional term [pos_rows, C], broadcast when pos_rows < M
  __half* out_pair_pos;                 // optional pair of (y + pos)
};

// one warp per row; C <= 128 * MAXV, C % 4 == 0.  Same two-pass arithmetic (and lane mapping) as layernorm_kernel in norm_attn.cu.
template <int MAXV>
__global__ void __launch_bounds__(256) layernorm_ex_kernel(const LnExArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= a.M) return;
  const int C = a.C, nv = C / 4;
  int64_t src = row;
  if (a.gather) src = (row / a.gK) * (int64_t)a.S + a.gather[row];
  const bool filled = a.valid && !a.valid[src % a.S];
  const float* xr = filled ? a.fill : a.x + src * a.x_pitch;
  float v[MAXV][4];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nv) {
      load4(xr + vi * 4, v[i]);
      if (a.res) {
        float r[4];
        load4(a.res + row * C + vi * 4, r);
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
  const float rstd = rsqrtf(warp_sum(q) / (float)C + a.eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int vi = lane + i * 32;
    if (vi < nv) {
      float g[4], b[4], o[4];
      load4(a.gamma + vi * 4, g);
      load4(a.beta + vi * 4, b);
#pragma unroll
      for (int j = 0; j < 4; ++j) o[j] = (v[i][j] - mean) * rstd * g[j] + b[j];
      if (a.out_f32) store4(a.out_f32 + row * C + vi * 4, o);
      if (a.out_pair) pair_store4(a.out_pair + row * 2 * C + vi * 4, a.out_pair + row * 2 * C + C + vi * 4, o);
      if (a.out_pair_pos) {
        float p[4];
        load4(a.pos + (row % a.pos_rows) * C + vi * 4, p);
#pragma unroll
        for (int j = 0; j < 4; ++j) p[j] += o[j];
        pair_store4(a.out_pair_pos + row * 2 * C + vi * 4, a.out_pair_pos + row * 2 * C + C + vi * 4, p);
      }
    }
  }
}

// out_pair = pair(act(x)), out_pair_pos = pair(x + pos)   (x [rows, C] with pitch; 4 values per thread)
__global__ void split_pair_ex_kernel(const float* __restrict__ x, int64_t rows, int C, int x_pitch, int act, const float* __restrict__ pos, int64_t pos_rows,
                                     __half* __restrict__ out_pair, __half* __restrict__ out_pair_pos) {
  const int cv = C / 4;
  const int64_t total = rows * cv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / cv;
    const int c = (int)(i - r * cv) * 4;
    float v[4];
    load4(x + r * x_pitch + c, v);
    if (out_pair) {
      float w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) w[j] = apply_act(v[j], act);
      pair_store4(out_pair + r * 2 * C + c, out_pair + r * 2 * C + C + c, w);
    }
    if (out_pair_pos) {
      float p[4];
      load4(pos + (r % pos_rows) * C + c, p);
#pragma unroll
      for (int j = 0; j < 4; ++j) p[j] += v[j];
      pair_store4(out_pair_pos + r * 2 * C + c, out_pair_pos + r * 2 * C + C + c, p);
    }
  }
}

__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float inv_sigmoid_f(float x) {  // inverse_sigmoid (nn/layers/functional.py:4-6), eps 1e-5
  x = fminf(fmaxf(x, 0.f), 1.f);
  return logf(fmaxf(x, 1e-5f) / fmaxf(1.f - x, 1e-5f));
}

// block = 128 threads = 8 rows x 16 lanes; a lane computes N/16 outputs of the 4 -> N ReLU layer (N % 64 == 0) and writes them as the pair
__global__ void __launch_bounds__(128) box_refine_qpos_kernel(const float* __restrict__ delta, const float* __restrict__ ref_in, float* __restrict__ ref_out,
                                                              const float* __restrict__ w0, const float* __restrict__ b0, int N, __half* __restrict__ qpos_pair,
                                                              int64_t M) {
  extern __shared__ float sm[];  // w0 [N][4] + b0 [N]
  float* sw = sm;
  float* sb = sm + 4 * N;
  if (qpos_pair) {
    for (int i = threadIdx.x; i < 4 * N; i += blockDim.x) sw[i] = w0[i];
    for (int i = threadIdx.x; i < N; i += blockDim.x) sb[i] = b0[i];
  }
  __syncthreads();
  const int sub = threadIdx.x & 15;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 4);
  if (row >= M) return;
  float r[4];
  load4(ref_in + row * 4, r);
  if (delta) {
    float d[4];
    load4(delta + row * 4, d);
#pragma unroll
    for (int j = 0; j < 4; ++j) r[j] = sigmoid_f(d[j] + inv_sigmoid_f(r[j]));
    if (sub == 0) store4(ref_out + row * 4, r);
  }
  if (!qpos_pair) return;
  __half* hi = qpos_pair + row * 2 * N;
  __half* lo = hi + N;
  for (int n = sub * 4; n < N; n += 64) {
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float* w = sw + (n + j) * 4;
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) acc = fmaf(r[k], w[k], acc);   // k order and the trailing +bias of conv_igemm_simt (scale == 1)
      o[j] = fmaxf(fmaf(acc, 1.f, sb[n + j]), 0.f);
    }
    pair_store4(hi + n, lo + n, o);
  }
}

__global__ void sigmoid_rows_kernel(const float* __restrict__ x, int x_pitch, int64_t M, int C, float* __restrict__ out) {
  const int64_t total = M * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / C;
    const int c = (int)(i - r * C);
    out[i] = sigmoid_f(x[r * x_pitch + c]);
  }
}

static inline unsigned grid_1d(int64_t work, int threads) {
  const int64_t b = cdiv(work, threads);
  return (unsigned)(b < 1 ? 1 : (b > kNumSMs * 32 ? kNumSMs * 32 : b));
}

}  // namespace fb200
using namespace fb200;

extern "C" int fb200_layernorm_ex(const float* x, int x_pitch, const float* res, const int* gather_idx, int gather_k, const uint8_t* valid, int S, const float* fill,
                                  const float* gamma, const float* beta, float eps, int64_t M, int C, float* out_f32, void* out_pair, const float* pos,
                                  int64_t pos_rows, void* out_pair_pos, void* stream) {
  FB_CHECK_ARG(x && gamma && beta && M > 0 && C > 0 && C % 4 == 0 && C <= 1024 && x_pitch % 4 == 0 && x_pitch >= C, "layernorm_ex: bad arguments (C=%d pitch=%d)", C, x_pitch);
  FB_CHECK_ARG(out_f32 || out_pair || out_pair_pos, "layernorm_ex: no output");
  FB_CHECK_ARG(!gather_idx || (gather_k > 0 && S > 0), "layernorm_ex: gather needs gather_k and S");
  FB_CHECK_ARG(!valid || (S > 0 && fill), "layernorm_ex: valid mask needs S and fill");
  FB_CHECK_ARG(!out_pair_pos || (pos && pos_rows > 0), "layernorm_ex: out_pair_pos needs pos");
  LnExArgs a;
  a.x = x; a.x_pitch = x_pitch; a.res = res; a.gather = gather_idx; a.gK = gather_k; a.S = S > 0 ? S : 1; a.valid = valid; a.fill = fill;
  a.gamma = gamma; a.beta = beta; a.eps = eps; a.M = M; a.C = C; a.out_f32 = out_f32; a.out_pair = (__half*)out_pair; a.pos = pos;
  a.pos_rows = pos_rows > 0 ? pos_rows : 1; a.out_pair_pos = (__half*)out_pair_pos;
  const unsigned grid = (unsigned)cdiv(M, 8);
  cudaStream_t st = (cudaStream_t)stream;
  if (C <= 256) layernorm_ex_kernel<2><<<grid, 256, 0, st>>>(a);
  else layernorm_ex_kernel<8><<<grid, 256, 0, st>>>(a);
  FB_CHECK_LAUNCH("layernorm_ex");
  return FB200_OK;
}

extern "C" int fb200_split_pair_ex(const float* x, int64_t rows, int C, int x_pitch, int act, const float* pos, int64_t pos_rows, void* out_pair, void* out_pair_pos,
                                   void* stream) {
  FB_CHECK_ARG(x && rows > 0 && C % 4 == 0 && x_pitch % 4 == 0 && x_pitch >= C && (out_pair || out_pair_pos), "split_pair_ex: bad arguments");
  FB_CHECK_ARG(!out_pair_pos || (pos && pos_rows > 0), "split_pair_ex: out_pair_pos needs pos");
  split_pair_ex_kernel<<<grid_1d(rows * (C / 4), 256), 256, 0, (cudaStream_t)stream>>>(x, rows, C, x_pitch, act, pos, pos_rows > 0 ? pos_rows : 1, (__half*)out_pair,
                                                                                         (__half*)out_pair_pos);
  FB_CHECK_LAUNCH("split_pair_ex");
  return FB200_OK;
}

extern "C" int fb200_box_refine_qpos(const float* delta, const float* ref_in, float* ref_out, const float* w0, const float* b0, int N, void* qpos_pair, int64_t M,
                                     void* stream) {
  FB_CHECK_ARG(ref_in && M > 0 && (delta || qpos_pair), "box_refine_qpos: bad arguments");
  FB_CHECK_ARG(!delta || ref_out, "box_refine_qpos: delta needs ref_out");
  FB_CHECK_ARG(!qpos_pair || (w0 && b0 && N > 0 && N % 64 == 0 && N <= 2048), "box_refine_qpos: the query_pos layer needs w0 [N,4], b0 [N], N %% 64 == 0");
  const size_t smem = qpos_pair ? (size_t)5 * N * sizeof(float) : 0;
  box_refine_qpos_kernel<<<(unsigned)cdiv(M, 8), 128, smem, (cudaStream_t)stream>>>(delta, ref_in, ref_out, w0, b0, N, (__half*)qpos_pair, M);
  FB_CHECK_LAUNCH("box_refine_qpos");
  return FB200_OK;
}

extern "C" int fb200_sigmoid_rows(const float* x, int x_pitch, int64_t M, int C, float* out, void* stream) {
  FB_CHECK_ARG(x && out && M > 0 && C > 0 && x_pitch >= C, "sigmoid_rows: bad arguments");
  sigmoid_rows_kernel<<<grid_1d(M * C, 256), 256, 0, (cudaStream_t)stream>>>(x, x_pitch, M, C, out);
  FB_CHECK_LAUNCH("sigmoid_rows");
  return FB200_OK;
}

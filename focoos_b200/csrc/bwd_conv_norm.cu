// Backward / training-mode kernels of the convolutional part of the path (SURVEY §8 a21: what autograd runs for
// ConvNormLayer, BottleNeck, RepVggBlock, the pools and F.interpolate when the reference fine-tunes, trainer.py:757).
// fp32 throughout (the reference's CPU training path is fp32; its CUDA path is fp16 autocast with fp32 master weights).
//
//   conv weight gradient   dW[co,kh,kw,ci] = sum_p dY[p,co] * X[pix(p,kh,kw),ci]      (aten conv backward, weight)
//   conv data gradient     = forward conv of dY (zero-dilated for stride 2) with flipped/transposed weights - host side
//   BatchNorm2d, training  batch statistics (biased var for normalisation, unbiased for running_var), fused +residual, ReLU/SiLU
//   column sums            bias gradients, LayerNorm parameter gradients
//   pools / resize         adjoint of max_pool2d(3,2,1), AvgPool2d(2,2,ceil), F.interpolate(bilinear, align_corners=False)
//
// All reductions are two-phase with a fixed summation order (per-block partials, then one pass in double) => reproducible.
#include "common.cuh"

namespace fb200 {
namespace {

// ------------------------------------------------------------------------------------------------------------------
// conv weight gradient: C[M=Cout, N=Cin] per filter tap, K = output pixels; both operands are "K-outer" in NHWC, so
// 16-pixel x 64-channel tiles of dY and X load coalesced; 256 threads, 4x4 micro-tiles; split-K over gridDim.z.
constexpr int WG_TM = 64, WG_TN = 64, WG_TK = 16;

__global__ void __launch_bounds__(256) conv_wgrad_kernel(const float* __restrict__ x, int x_pitch, const float* __restrict__ dy, int dy_pitch, int B, int H,
                                                         int W, int Cin, int Ho, int Wo, int Cout, int KH, int KW, int stride, int pad, int64_t pix_per_split,
                                                         float* __restrict__ part) {
  __shared__ float sA[WG_TK][WG_TM + 4];  // dY tile  [k][co]
  __shared__ float sB[WG_TK][WG_TN + 4];  // X tile   [k][ci]
  const int tiles_n = (Cin + WG_TN - 1) / WG_TN;
  const int m0 = (blockIdx.x / tiles_n) * WG_TM, n0 = (blockIdx.x % tiles_n) * WG_TN;
  const int kh = blockIdx.y / KW, kw = blockIdx.y % KW;
  const int64_t P = (int64_t)B * Ho * Wo;
  const int64_t p_begin = (int64_t)blockIdx.z * pix_per_split, p_end = min(P, p_begin + pix_per_split);
  const int tid = threadIdx.x, tr = tid >> 4, tc = (tid & 15) * 4;  // loader: row tr (0..15), 4 channels at tc
  const int ty = tid >> 4, tx = tid & 15;                             // compute: rows ty*4.., cols tx*4..
  float acc[4][4] = {};
  for (int64_t p0 = p_begin; p0 < p_end; p0 += WG_TK) {
    const int64_t p = p0 + tr;
    float a[4] = {0.f, 0.f, 0.f, 0.f}, b[4] = {0.f, 0.f, 0.f, 0.f};
    if (p < p_end) {
      const int wo = p % Wo, ho = (p / Wo) % Ho, bi = p / ((int64_t)Wo * Ho);
      const float* dyp = dy + p * dy_pitch + m0 + tc;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (m0 + tc + j < Cout) a[j] = dyp[j];
      const int hi = ho * stride + kh - pad, wi = wo * stride + kw - pad;
      if (hi >= 0 && hi < H && wi >= 0 && wi < W) {
        const float* xp = x + (((int64_t)bi * H + hi) * W + wi) * x_pitch + n0 + tc;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (n0 + tc + j < Cin) b[j] = xp[j];
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) { sA[tr][tc + j] = a[j]; sB[tr][tc + j] = b[j]; }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < WG_TK; ++k) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { av[i] = sA[k][ty * 4 + i]; bv[i] = sB[k][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
  }
  float* out = part + (int64_t)blockIdx.z * Cout * KH * KW * Cin;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int co = m0 + ty * 4 + i;
    if (co >= Cout) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ci = n0 + tx * 4 + j;
      if (ci < Cin) out[(((int64_t)co * KH + kh) * KW + kw) * Cin + ci] = acc[i][j];
    }
  }
}

// Weight gradient of the stem conv (3x3, stride 2, pad 1, Cin <= 4, Cout = 32): 864 outputs reduced over B*Ho*Wo pixels.  The generic 64x64 tile would waste
// 31/32 of its FMAs on the 3-channel operand; here a block stages an 8 x 16 tile of dY and the (17 x 33) x Cin input halo in shared memory and thread
// (co = t % 32, g = t / 32) accumulates the (tap, ci) pairs j = g, g + 8, ... < 9*Cin for its output channel.  Per-block partials, fixed-order reduce.
constexpr int SW_TH = 8, SW_TW = 16;
__global__ void __launch_bounds__(256) conv_wgrad_stem_kernel(const float* __restrict__ x, int x_pitch, const float* __restrict__ dy, int dy_pitch, int B, int H, int W,
                                                              int Cin, int Ho, int Wo, int tiles_w, int tiles_h, float* __restrict__ part) {
  __shared__ float sdy[SW_TH * SW_TW][33];
  __shared__ float sx[(2 * SW_TH + 1) * (2 * SW_TW + 1) * 4];
  const int co = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int K = 9 * Cin;  // <= 36
  float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
  const int PW = 2 * SW_TW + 1, PH = 2 * SW_TH + 1;
  const int64_t ntiles = (int64_t)B * tiles_h * tiles_w;
  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int b = t / (tiles_h * tiles_w), rem = t % (tiles_h * tiles_w);
    const int ho0 = (rem / tiles_w) * SW_TH, wo0 = (rem % tiles_w) * SW_TW;
    __syncthreads();
    for (int i = threadIdx.x; i < SW_TH * SW_TW * 32; i += 256) {
      const int c = i & 31, p = i >> 5, ho = ho0 + p / SW_TW, wo = wo0 + p % SW_TW;
      sdy[p][c] = (ho < Ho && wo < Wo) ? dy[(((int64_t)b * Ho + ho) * Wo + wo) * dy_pitch + c] : 0.f;
    }
    for (int i = threadIdx.x; i < PH * PW * Cin; i += 256) {
      const int ci = i % Cin, pp = i / Cin, hi = 2 * ho0 - 1 + pp / PW, wi = 2 * wo0 - 1 + pp % PW;
      sx[pp * 4 + ci] = (hi >= 0 && hi < H && wi >= 0 && wi < W) ? x[(((int64_t)b * H + hi) * W + wi) * x_pitch + ci] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < 5; ++u) {
      const int j = g + 8 * u;
      if (j >= K) break;
      const int tap = j / Cin, ci = j - tap * Cin, kh = tap / 3, kw = tap - kh * 3;
      float a = 0.f;
      for (int py = 0; py < SW_TH; ++py)
#pragma unroll 8
        for (int px = 0; px < SW_TW; ++px) a = fmaf(sdy[py * SW_TW + px][co], sx[((2 * py + kh) * PW + 2 * px + kw) * 4 + ci], a);
      acc[u] += a;
    }
  }
  float* out = part + (int64_t)blockIdx.x * 32 * K;
#pragma unroll
  for (int u = 0; u < 5; ++u) {
    const int j = g + 8 * u;
    if (j < K) out[co * K + j] = acc[u];  // j = tap * Cin + ci: the [Cout][KH][KW][Cin] order
  }
}

__global__ void split_reduce_kernel(const float* __restrict__ part, int splits, int64_t n, float* __restrict__ out, int accumulate) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int k = 0; k < splits; ++k) s += (double)part[(int64_t)k * n + i];
  out[i] = accumulate ? out[i] + (float)s : (float)s;
}

// out[b,h,w,:] = (h,w both even and inside) ? dy[b,h/2,w/2,:] : 0     (zero-dilation for the stride-2 data gradient)
__global__ void dilate2_kernel(const float* __restrict__ dy, int B, int Ho, int Wo, int C, int Hd, int Wd, float* __restrict__ out) {
  const int cv = C / 4;
  const int64_t total = (int64_t)B * Hd * Wd * cv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (i % cv) * 4;
    const int64_t pix = i / cv;
    const int w = pix % Wd, h = (pix / Wd) % Hd, b = pix / ((int64_t)Wd * Hd);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!(h & 1) && !(w & 1) && (h >> 1) < Ho && (w >> 1) < Wo) v = *reinterpret_cast<const float4*>(dy + (((int64_t)b * Ho + (h >> 1)) * Wo + (w >> 1)) * C + c);
    *reinterpret_cast<float4*>(out + pix * C + c) = v;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// column reductions over [R, C] (row pitch).  MODE 0: sum x   1: sum (x-mean)^2   2: BN backward (sum g, sum g*xhat)
// partial[blockIdx.y][c] per row-slice; 32 channels x 8 row lanes per block.
constexpr int CR_ROWS = 2 * kNumSMs;  // row slices (two per SM)

__device__ __forceinline__ float act_grad(int act, float z, float y) {  // y = forward output where one exists, else pass z twice
  if (act == FB200_ACT_RELU) return y > 0.f ? 1.f : 0.f;
  if (act == FB200_ACT_SILU) { const float s = 1.f / (1.f + expf(-z)); return s * (1.f + z * (1.f - s)); }
  if (act == FB200_ACT_GELU) { return 0.5f * (1.f + erff(z * 0.70710678118654752f)) + z * 0.3989422804014327f * expf(-0.5f * z * z); }
  return 1.f;
}
__device__ __forceinline__ float act_fwd(int act, float z) {
  if (act == FB200_ACT_RELU) return fmaxf(z, 0.f);
  if (act == FB200_ACT_SILU) return z / (1.f + expf(-z));
  if (act == FB200_ACT_GELU) return 0.5f * z * (1.f + erff(z * 0.70710678118654752f));
  return z;
}

// MODE 3 (single-pass mean / variance): each thread sums (x - q) and (x - q)^2 about its OWN first row q, so the squares never cancel against a
// pivot far from the data; per thread that gives (n, mean, M2 = sum of squared deviations from the mean), which the block merges over its row
// lanes with Chan's pairwise update.  The part written is p0 = sum (x - x[0,c]) (the mean relative to the global pivot row) and p1 = M2 about
// the part's own mean; bn_stats_finalize_kernel adds the between-part term in double.  (One pivot for all rows, row 0, lost the variance to
// fp32 cancellation when row 0 lay far from the mean: ~1e-5 relative at 40 sigma.)
struct LaneRows {  // rows of the lane starting at row r0 < rstep (a grid-stride walk r0, r0 + rstep, ... < R): full or full + 1
  float full;
  int64_t rem;
  __device__ __forceinline__ LaneRows(int64_t R, int64_t rstep) : full((float)(R / rstep)), rem(R % rstep) {}
  __device__ __forceinline__ float operator()(int64_t r0) const { return full + (r0 < rem ? 1.f : 0.f); }
};
struct Moments {
  float n, mean, m2;  // rows, mean relative to the global pivot, sum of squared deviations from `mean`
  __device__ __forceinline__ void merge(float nb, float mb, float m2b) {
    if (nb == 0.f) return;
    const float nt = n + nb, d = mb - mean, w = nb * __frcp_rn(nt);
    mean += d * w;
    m2 += m2b + d * d * n * w;
    n = nt;
  }
};
__device__ __forceinline__ void lane_moments(float n, float q_rel, float s0, float s1, float& mean, float& m2) {  // (x - q) sums -> mean, M2
  const float m = n > 0.f ? s0 * __frcp_rn(n) : 0.f;
  mean = q_rel + m;
  m2 = fmaxf(s1 - s0 * m, 0.f);
}

template <int MODE>
__global__ void __launch_bounds__(256) col_partial_kernel(const float* __restrict__ x, int x_pitch, int64_t R, int C, const float* __restrict__ mean,
                                                          const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                                                          const float* __restrict__ dy, int dy_pitch, const float* __restrict__ y, int y_pitch, int act,
                                                          float* __restrict__ p0, float* __restrict__ p1) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int lane_r = threadIdx.x >> 5;  // 0..7
  const int64_t rstep = (int64_t)gridDim.y * 8;
  float s0 = 0.f, s1 = 0.f, q_rel = 0.f;
  if (c < C) {
    const float mu = (MODE >= 1) ? mean[c] : 0.f;
    const float rs = (MODE == 2) ? rstd[c] : 0.f;
    const float ga = (MODE == 2) ? gamma[c] : 0.f, be = (MODE == 2) ? beta[c] : 0.f;
    int64_t r = (int64_t)blockIdx.y * 8 + lane_r;
    const float pivot = (MODE == 3 && r < R) ? x[r * x_pitch + c] : 0.f;  // this thread's first row
    if (MODE == 3) q_rel = pivot - x[c];
    if (MODE == 2) {  // four independent rows per iteration: 8-12 loads in flight per thread instead of 2-3 (the kernel is latency-, not bandwidth-bound otherwise)
      for (; r + 3 * rstep < R; r += 4 * rstep) {
        float xv[4], gv[4], yv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          xv[u] = x[(r + u * rstep) * x_pitch + c];
          gv[u] = dy[(r + u * rstep) * dy_pitch + c];
          yv[u] = (act != FB200_ACT_NONE && y) ? y[(r + u * rstep) * y_pitch + c] : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const float xh = (xv[u] - mu) * rs;
          float g = gv[u];
          if (act != FB200_ACT_NONE) {
            const float z = xh * ga + be;
            g *= act_grad(act, z, y ? yv[u] : z);
          }
          s0 += g;
          s1 += g * xh;
        }
      }
    } else if (MODE == 3) {
      for (; r + 3 * rstep < R; r += 4 * rstep) {
        float xv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) xv[u] = x[(r + u * rstep) * x_pitch + c];
#pragma unroll
        for (int u = 0; u < 4; ++u) { const float d = xv[u] - pivot; s0 += d; s1 += d * d; }
      }
    }
    for (; r < R; r += rstep) {
      const float v = x[r * x_pitch + c];
      if (MODE == 0) s0 += v;
      else if (MODE == 1) { const float d = v - mu; s0 += d * d; }
      else if (MODE == 3) { const float d = v - pivot; s0 += d; s1 += d * d; }
      else {
        const float xh = (v - mu) * rs;
        float g = dy[r * dy_pitch + c];
        if (act != FB200_ACT_NONE) {
          const float z = xh * ga + be;
          g *= act_grad(act, z, y ? y[r * y_pitch + c] : z);
        }
        s0 += g;
        s1 += g * xh;
      }
    }
  }
  const LaneRows rows(R, rstep);
  if (MODE == 3) lane_moments(rows((int64_t)blockIdx.y * 8 + lane_r), q_rel, s0, s1, s0, s1);
  __shared__ float r0[8][33], r1[8][33];
  r0[lane_r][threadIdx.x & 31] = s0;
  r1[lane_r][threadIdx.x & 31] = s1;
  __syncthreads();
  if (lane_r == 0 && c < C) {
    float a = 0.f, b = 0.f;
    if (MODE == 3) {
      Moments m{0.f, 0.f, 0.f};
      for (int k = 0; k < 8; ++k) m.merge(rows((int64_t)blockIdx.y * 8 + k), r0[k][threadIdx.x], r1[k][threadIdx.x]);
      a = m.n * m.mean;
      b = m.m2;
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) { a += r0[k][threadIdx.x]; b += r1[k][threadIdx.x]; }
    }
    p0[(int64_t)blockIdx.y * C + c] = a;
    if (MODE >= 2) p1[(int64_t)blockIdx.y * C + c] = b;
  }
}

// float4 version of col_partial_kernel for MODE 0 / 2 / 3 (the passes that read whole activation tensors): a thread owns FOUR consecutive channels of a row, a block covers a
// chunk of CW = min(C, 128) channels x (1024 / CW) rows per step, four row steps unrolled -> 64 B (MODE 0 / 3) or 128-192 B (MODE 2) of loads in flight per thread.  The
// scalar kernel keeps 16 B per thread in flight and ran the BatchNorm statistics passes at about a third of the HBM bandwidth (trip r02-14: bn_train_fwd 9.5 ms,
// bn_train_bwd 15.4 ms per fine-tune step).  Requires C in {32, 64, 128} or C % 128 == 0, pitches % 4 == 0, 16-byte aligned bases (col_vec_ok).
template <int MODE>
__global__ void __launch_bounds__(256) col_partial4_kernel(const float* __restrict__ x, int x_pitch, int64_t R, int C, const float* __restrict__ mean,
                                                           const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                                                           const float* __restrict__ dy, int dy_pitch, const float* __restrict__ y, int y_pitch, int act,
                                                           float* __restrict__ p0, float* __restrict__ p1) {
  const int CW = C < 128 ? C : 128;           // channels of this block's chunk
  const int TPR = CW / 4;                     // threads per row (8, 16 or 32)
  const int RPB = 256 / TPR;                  // rows per block step
  const int tc = threadIdx.x % TPR, tr = threadIdx.x / TPR;
  const int c = blockIdx.x * CW + tc * 4;
  float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
  float mu[4] = {0.f, 0.f, 0.f, 0.f}, rs[4] = {0.f, 0.f, 0.f, 0.f}, ga[4] = {0.f, 0.f, 0.f, 0.f}, be[4] = {0.f, 0.f, 0.f, 0.f}, pv[4] = {0.f, 0.f, 0.f, 0.f};
  if (MODE == 2) { load4(mean + c, mu); load4(rstd + c, rs); load4(gamma + c, ga); load4(beta + c, be); }
  const bool has_y = (MODE == 2) && act != FB200_ACT_NONE && y != nullptr;
  const int64_t rstep = (int64_t)gridDim.y * RPB;
  int64_t r = (int64_t)blockIdx.y * RPB + tr;
  float q_rel[4] = {0.f, 0.f, 0.f, 0.f};
  if (MODE == 3) {  // pivot: this thread's first row (see col_partial_kernel)
    float p_row0[4];
    load4(x + c, p_row0);
    if (r < R) load4(x + r * x_pitch + c, pv);
#pragma unroll
    for (int j = 0; j < 4; ++j) q_rel[j] = pv[j] - p_row0[j];
  }
  auto accum = [&](const float (&xv)[4], const float (&gv)[4], const float (&yv)[4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (MODE == 0) s0[j] += xv[j];
      else if (MODE == 3) { const float d = xv[j] - pv[j]; s0[j] += d; s1[j] += d * d; }
      else {
        const float xh = (xv[j] - mu[j]) * rs[j];
        float g = gv[j];
        if (act != FB200_ACT_NONE) {
          const float z = xh * ga[j] + be[j];
          g *= act_grad(act, z, has_y ? yv[j] : z);
        }
        s0[j] += g;
        s1[j] += g * xh;
      }
    }
  };
  for (; r + 3 * rstep < R; r += 4 * rstep) {
    float xv[4][4], gv[4][4], yv[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      load4(x + (r + u * rstep) * x_pitch + c, xv[u]);
      if (MODE == 2) load4(dy + (r + u * rstep) * dy_pitch + c, gv[u]);
      if (MODE == 2 && has_y) load4(y + (r + u * rstep) * y_pitch + c, yv[u]);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) accum(xv[u], gv[u], yv[u]);
  }
  for (; r < R; r += rstep) {
    float xv[4], gv[4] = {0.f, 0.f, 0.f, 0.f}, yv[4] = {0.f, 0.f, 0.f, 0.f};
    load4(x + r * x_pitch + c, xv);
    if (MODE == 2) load4(dy + r * dy_pitch + c, gv);
    if (MODE == 2 && has_y) load4(y + r * y_pitch + c, yv);
    accum(xv, gv, yv);
  }
  const LaneRows rows(R, rstep);
  if (MODE == 3) {
    const float n = rows((int64_t)blockIdx.y * RPB + tr);
#pragma unroll
    for (int j = 0; j < 4; ++j) lane_moments(n, q_rel[j], s0[j], s1[j], s0[j], s1[j]);
  }
  __shared__ float red0[32][129], red1[32][129];   // [row lane][channel of the chunk]
#pragma unroll
  for (int j = 0; j < 4; ++j) { red0[tr][tc * 4 + j] = s0[j]; if (MODE >= 2) red1[tr][tc * 4 + j] = s1[j]; }
  __syncthreads();
  if ((int)threadIdx.x < CW) {
    float a = 0.f, b = 0.f;
    if (MODE == 3) {
      Moments m{0.f, 0.f, 0.f};
      for (int k = 0; k < RPB; ++k) m.merge(rows((int64_t)blockIdx.y * RPB + k), red0[k][threadIdx.x], red1[k][threadIdx.x]);
      a = m.n * m.mean;
      b = m.m2;
    } else {
      for (int k = 0; k < RPB; ++k) { a += red0[k][threadIdx.x]; if (MODE >= 2) b += red1[k][threadIdx.x]; }
    }
    const int co = blockIdx.x * CW + threadIdx.x;
    p0[(int64_t)blockIdx.y * C + co] = a;
    if (MODE >= 2) p1[(int64_t)blockIdx.y * C + co] = b;
  }
}

// FIN 0: out0 = sum                       (colsum)
// FIN 1: out0 = mean = sum / R            (BN pass 1)
// FIN 2: out0 = rstd from sum of squared deviations; running stats update (BN pass 2)
// FIN 3: out0 = dbeta = sum p0, out1 = dgamma = sum p1 (BN backward)
template <int FIN>
__global__ void col_finalize_kernel(const float* __restrict__ p0, const float* __restrict__ p1, int nparts, int C, double R, float eps, float momentum,
                                    const float* __restrict__ mean, float* __restrict__ run_mean, float* __restrict__ run_var, float* __restrict__ out0,
                                    float* __restrict__ out1, int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double a = 0.0, b = 0.0;
  for (int k = 0; k < nparts; ++k) {
    a += (double)p0[(int64_t)k * C + c];
    if (FIN >= 3) b += (double)p1[(int64_t)k * C + c];
  }
  if (FIN == 0) out0[c] = accumulate ? out0[c] + (float)a : (float)a;
  if (FIN == 1) out0[c] = (float)(a / R);
  if (FIN == 2) {
    const double var = a / R;
    out0[c] = (float)(1.0 / sqrt(var + (double)eps));
    if (run_mean) {
      run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * mean[c];
      run_var[c] = (1.f - momentum) * run_var[c] + momentum * (float)(R > 1.0 ? a / (R - 1.0) : var);
    }
  }
  if (FIN == 3) {
    out0[c] = accumulate ? out0[c] + (float)a : (float)a;
    out1[c] = accumulate ? out1[c] + (float)b : (float)b;
  }
}

__device__ __forceinline__ double warp_sum_f64(double v) {  // butterfly: the same fixed order on every lane
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// BN statistics from col_partial<3>'s parts: p0 = sum (x - pivot row), p1 = squared deviations about the part's own mean, in part k the rows whose
// (r mod nparts * rpb) lies in [k * rpb, (k + 1) * rpb).  Total squared deviations = sum p1_k + sum n_k (mean_k - mean)^2, the latter as
// sum p0_k^2 / n_k - (sum p0_k)^2 / R in double.  One warp per channel (lanes take every 32nd part, then a butterfly sum), so the walk over the
// parts is not one long chain of dependent loads.
// FIN 4: out0 = mean, out1 = rstd, running statistics updated (bn_train_fwd); `mean` carries the pivot row
// FIN 5: out0 = mean, out1 = BIASED variance: the raw local moments SyncBatchNorm exchanges (fb200_bn_stats)
template <int FIN>
__global__ void __launch_bounds__(256) bn_stats_finalize_kernel(const float* __restrict__ p0, const float* __restrict__ p1, int nparts, int rpb, int C, int64_t R,
                                                                float eps, float momentum, const float* __restrict__ pivot, float* __restrict__ run_mean,
                                                                float* __restrict__ run_var, float* __restrict__ out0, float* __restrict__ out1) {
  const int c = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (c >= C) return;
  // with rem = R mod (nparts * rpb), part k holds nfull rows, plus rpb for k < kpart and rem mod rpb for k == kpart
  const int64_t rstep = (int64_t)nparts * rpb, rem = R % rstep, nfull = (R / rstep) * rpb, npart = nfull + rem % rpb;
  const int kpart = (int)(rem / rpb);
  const double inv_more = 1.0 / (double)(nfull + rpb), inv_part = npart > 0 ? 1.0 / (double)npart : 0.0, inv_full = nfull > 0 ? 1.0 / (double)nfull : 0.0;
  double a = 0.0, b = 0.0, e = 0.0;
  for (int k = lane; k < nparts; k += 32) {
    const double p = (double)p0[(int64_t)k * C + c];
    a += p;
    b += (double)p1[(int64_t)k * C + c];
    e += p * p * (k < kpart ? inv_more : k == kpart ? inv_part : inv_full);
  }
  a = warp_sum_f64(a);
  b = warp_sum_f64(b);
  e = warp_sum_f64(e);
  if (lane != 0) return;
  const double Rd = (double)R, m1 = a / Rd;
  const double var = (b + fmax(e - a * m1, 0.0)) / Rd;
  const float mu = (float)((double)pivot[c] + m1);
  out0[c] = mu;
  if (FIN == 5) {
    out1[c] = (float)var;
    return;
  }
  out1[c] = (float)(1.0 / sqrt(var + (double)eps));
  if (run_mean) {
    run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * mu;
    run_var[c] = (1.f - momentum) * run_var[c] + momentum * (float)(R > 1 ? var * Rd / (Rd - 1.0) : var);
  }
}

// y = act((x - mean) * rstd * gamma + beta + res)
__global__ void bn_apply_kernel(const float* __restrict__ x, int x_pitch, const float* __restrict__ res, int res_pitch, int64_t R, int C,
                                const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                                int act, float* __restrict__ y, int y_pitch) {
  const int cv = C / 4;
  const int64_t total = R * cv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / cv;
    const int c = (i % cv) * 4;
    const float4 v = *reinterpret_cast<const float4*>(x + r * x_pitch + c);
    const float4 mu = *reinterpret_cast<const float4*>(mean + c), rs = *reinterpret_cast<const float4*>(rstd + c);
    const float4 ga = *reinterpret_cast<const float4*>(gamma + c), be = *reinterpret_cast<const float4*>(beta + c);
    float4 z = make_float4((v.x - mu.x) * rs.x * ga.x + be.x, (v.y - mu.y) * rs.y * ga.y + be.y, (v.z - mu.z) * rs.z * ga.z + be.z, (v.w - mu.w) * rs.w * ga.w + be.w);
    if (res) {
      const float4 q = *reinterpret_cast<const float4*>(res + r * res_pitch + c);
      z.x += q.x; z.y += q.y; z.z += q.z; z.w += q.w;
    }
    *reinterpret_cast<float4*>(y + r * y_pitch + c) = make_float4(act_fwd(act, z.x), act_fwd(act, z.y), act_fwd(act, z.z), act_fwd(act, z.w));
  }
}

// "column-fixed" variants of the two element-wise BatchNorm passes: the launch has a multiple of C/4 threads, so a thread keeps ONE group of four channels for its whole
// grid-stride walk over the rows - the per-channel parameters are loaded once, the loop has no 64-bit division (the generic kernels spend ~150 instructions per float4 on
// index arithmetic and parameter reloads and were instruction-bound at ~2.3 TB/s), and two rows are in flight per iteration.
__global__ void __launch_bounds__(256) bn_apply_cf_kernel(const float* __restrict__ x, int x_pitch, const float* __restrict__ res, int res_pitch, int64_t R, int C,
                                                          const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                                                          const float* __restrict__ beta, int act, float* __restrict__ y, int y_pitch) {
  const int cv = C / 4;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, T = (int64_t)gridDim.x * blockDim.x;
  const int c = (int)(tid % cv) * 4;
  const int64_t rstep = T / cv;
  float mu[4], rs[4], ga[4], b[4];
  load4(mean + c, mu); load4(rstd + c, rs); load4(gamma + c, ga); load4(beta + c, b);
  auto one = [&](int64_t r, const float (&v)[4], const float (&q)[4]) {
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float z = (v[j] - mu[j]) * rs[j] * ga[j] + b[j];   // the arithmetic (and rounding order) of bn_apply_kernel
      if (res) z += q[j];
      o[j] = act_fwd(act, z);
    }
    store4(y + r * y_pitch + c, o);
  };
  int64_t r = tid / cv;
  for (; r + rstep < R; r += 2 * rstep) {
    float v0[4], v1[4], q0[4] = {0.f, 0.f, 0.f, 0.f}, q1[4] = {0.f, 0.f, 0.f, 0.f};
    load4(x + r * x_pitch + c, v0);
    load4(x + (r + rstep) * x_pitch + c, v1);
    if (res) { load4(res + r * res_pitch + c, q0); load4(res + (r + rstep) * res_pitch + c, q1); }
    one(r, v0, q0);
    one(r + rstep, v1, q1);
  }
  if (r < R) {
    float v0[4], q0[4] = {0.f, 0.f, 0.f, 0.f};
    load4(x + r * x_pitch + c, v0);
    if (res) load4(res + r * res_pitch + c, q0);
    one(r, v0, q0);
  }
}

__global__ void __launch_bounds__(256) bn_bwd_apply_cf_kernel(const float* __restrict__ x, int x_pitch, const float* __restrict__ dy, int dy_pitch, const float* __restrict__ y,
                                                              int y_pitch, int64_t R, int C, const float* __restrict__ mean, const float* __restrict__ rstd,
                                                              const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ dgamma,
                                                              const float* __restrict__ dbeta, int act, float inv_R, float* __restrict__ dx, int dx_pitch,
                                                              float* __restrict__ dres, int dres_pitch) {
  const int cv = C / 4;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, T = (int64_t)gridDim.x * blockDim.x;
  const int c = (int)(tid % cv) * 4;
  const int64_t rstep = T / cv;
  float mu[4], rs[4], ga[4], be[4], dg[4], db[4];
  load4(mean + c, mu); load4(rstd + c, rs); load4(gamma + c, ga); load4(beta + c, be); load4(dgamma + c, dg); load4(dbeta + c, db);
  const bool has_y = act != FB200_ACT_NONE && y != nullptr;
  auto one = [&](int64_t r, const float (&xv)[4], const float (&gv)[4], const float (&yv)[4]) {
    float o[4], gr[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {   // the arithmetic of bn_bwd_apply4_kernel
      const float xh = (xv[j] - mu[j]) * rs[j];
      float g = gv[j];
      if (act != FB200_ACT_NONE) {
        const float z = xh * ga[j] + be[j];
        g *= act_grad(act, z, y ? yv[j] : z);
      }
      gr[j] = g;
      o[j] = ga[j] * rs[j] * (g - db[j] * inv_R - xh * dg[j] * inv_R);
    }
    store4(dx + r * dx_pitch + c, o);
    if (dres) store4(dres + r * dres_pitch + c, gr);
  };
  int64_t r = tid / cv;
  for (; r + rstep < R; r += 2 * rstep) {
    float x0[4], x1[4], g0[4], g1[4], y0[4] = {0.f, 0.f, 0.f, 0.f}, y1[4] = {0.f, 0.f, 0.f, 0.f};
    load4(x + r * x_pitch + c, x0);
    load4(x + (r + rstep) * x_pitch + c, x1);
    load4(dy + r * dy_pitch + c, g0);
    load4(dy + (r + rstep) * dy_pitch + c, g1);
    if (has_y) { load4(y + r * y_pitch + c, y0); load4(y + (r + rstep) * y_pitch + c, y1); }
    one(r, x0, g0, y0);
    one(r + rstep, x1, g1, y1);
  }
  if (r < R) {
    float x0[4], g0[4], y0[4] = {0.f, 0.f, 0.f, 0.f};
    load4(x + r * x_pitch + c, x0);
    load4(dy + r * dy_pitch + c, g0);
    if (has_y) load4(y + r * y_pitch + c, y0);
    one(r, x0, g0, y0);
  }
}

// float4 version of bn_bwd_apply_kernel (C % 4 == 0, 16-byte aligned rows): no per-element 64-bit division, per-channel parameters loaded as vectors
__global__ void bn_bwd_apply4_kernel(const float* __restrict__ x, int x_pitch, const float* __restrict__ dy, int dy_pitch, const float* __restrict__ y, int y_pitch,
                                     int64_t R, int C, const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, const float* __restrict__ dgamma, const float* __restrict__ dbeta, int act, float inv_R,
                                     float* __restrict__ dx, int dx_pitch, float* __restrict__ dres, int dres_pitch) {
  const int cv = C / 4;
  const int64_t total = R * cv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / cv;
    const int c = (int)(i - r * cv) * 4;
    const float4 xv = *reinterpret_cast<const float4*>(x + r * x_pitch + c), gv = *reinterpret_cast<const float4*>(dy + r * dy_pitch + c);
    float4 yv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (act != FB200_ACT_NONE && y) yv = *reinterpret_cast<const float4*>(y + r * y_pitch + c);
    const float4 mu = *reinterpret_cast<const float4*>(mean + c), rs = *reinterpret_cast<const float4*>(rstd + c);
    const float4 ga = *reinterpret_cast<const float4*>(gamma + c), be = *reinterpret_cast<const float4*>(beta + c);
    const float4 dg = *reinterpret_cast<const float4*>(dgamma + c), db = *reinterpret_cast<const float4*>(dbeta + c);
    const float xa[4] = {xv.x, xv.y, xv.z, xv.w}, ga4[4] = {gv.x, gv.y, gv.z, gv.w}, ya[4] = {yv.x, yv.y, yv.z, yv.w};
    const float m4[4] = {mu.x, mu.y, mu.z, mu.w}, r4[4] = {rs.x, rs.y, rs.z, rs.w}, g4[4] = {ga.x, ga.y, ga.z, ga.w}, b4[4] = {be.x, be.y, be.z, be.w};
    const float dg4[4] = {dg.x, dg.y, dg.z, dg.w}, db4[4] = {db.x, db.y, db.z, db.w};
    float o[4], gr[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float xh = (xa[j] - m4[j]) * r4[j];
      float g = ga4[j];
      if (act != FB200_ACT_NONE) {
        const float z = xh * g4[j] + b4[j];
        g *= act_grad(act, z, y ? ya[j] : z);
      }
      gr[j] = g;
      o[j] = g4[j] * r4[j] * (g - db4[j] * inv_R - xh * dg4[j] * inv_R);
    }
    *reinterpret_cast<float4*>(dx + r * dx_pitch + c) = make_float4(o[0], o[1], o[2], o[3]);
    if (dres) *reinterpret_cast<float4*>(dres + r * dres_pitch + c) = make_float4(gr[0], gr[1], gr[2], gr[3]);
  }
}

// dx = gamma * rstd * (g - dbeta/R - xhat * dgamma/R),  g = dy * act'(.);  dres = g
__global__ void bn_bwd_apply_kernel(const float* __restrict__ x, int x_pitch, const float* __restrict__ dy, int dy_pitch, const float* __restrict__ y, int y_pitch,
                                    int64_t R, int C, const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, const float* __restrict__ dgamma, const float* __restrict__ dbeta, int act, float inv_R,
                                    float* __restrict__ dx, int dx_pitch, float* __restrict__ dres, int dres_pitch) {
  const int64_t total = R * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / C;
    const int c = i % C;
    const float xh = (x[r * x_pitch + c] - mean[c]) * rstd[c];
    float g = dy[r * dy_pitch + c];
    if (act != FB200_ACT_NONE) {
      const float z = xh * gamma[c] + beta[c];
      g *= act_grad(act, z, y ? y[r * y_pitch + c] : z);
    }
    dx[r * dx_pitch + c] = gamma[c] * rstd[c] * (g - dbeta[c] * inv_R - xh * dgamma[c] * inv_R);
    if (dres) dres[r * dres_pitch + c] = g;
  }
}

// out = act(a + b) ; backward: da = db = dy * act'(a + b)
__global__ void add_act_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ dy, int act, int64_t n, float* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float z = a[i] + (b ? b[i] : 0.f);
    out[i] = dy ? dy[i] * act_grad(act, z, act_fwd(act, z)) : act_fwd(act, z);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// max_pool2d(3, 2, 1) backward: each input pixel collects from the <=4 windows that contain it where it is the FIRST maximum
// (row-major scan order, the tie rule of aten's max_pool2d_with_indices).
__global__ void maxpool_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, int B, int H, int W, int C, int Ho, int Wo, float* __restrict__ dx) {
  const int64_t total = (int64_t)B * H * W * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = i % C;
    const int64_t pix = i / C;
    const int w = pix % W, h = (pix / W) % H, b = pix / ((int64_t)W * H);
    const float* xb = x + (int64_t)b * H * W * C + c;
    float acc = 0.f;
    for (int ho = (h + 1 - 2 + 1) / 2; ho <= (h + 1) / 2 && ho < Ho; ++ho) {   // windows rows: 2*ho-1 <= h <= 2*ho+1
      if (ho < 0) continue;
      for (int wo = (w + 1 - 2 + 1) / 2; wo <= (w + 1) / 2 && wo < Wo; ++wo) {
        if (wo < 0) continue;
        float best = -INFINITY;
        int bh = -1, bw = -1;
        for (int dh = 0; dh < 3; ++dh) {
          const int hh = 2 * ho - 1 + dh;
          if (hh < 0 || hh >= H) continue;
          for (int dw = 0; dw < 3; ++dw) {
            const int ww = 2 * wo - 1 + dw;
            if (ww < 0 || ww >= W) continue;
            const float v = xb[((int64_t)hh * W + ww) * C];
            if (v > best || isnan(v)) { if (!(best != best)) { best = v; bh = hh; bw = ww; } }
          }
        }
        if (bh == h && bw == w) acc += dy[(((int64_t)b * Ho + ho) * Wo + wo) * C + c];
      }
    }
    dx[i] = acc;
  }
}

// four channels per thread (16-byte loads): same first-maximum rule per channel
__global__ void maxpool_bwd4_kernel(const float* __restrict__ x, const float* __restrict__ dy, int B, int H, int W, int C, int Ho, int Wo, float* __restrict__ dx) {
  const int cv = C / 4;
  const int64_t total = (int64_t)B * H * W * cv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) * 4;
    const int64_t pix = i / cv;
    const int w = pix % W, h = (pix / W) % H, b = pix / ((int64_t)W * H);
    const float* xb = x + (int64_t)b * H * W * C + c;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int ho = h / 2; ho <= (h + 1) / 2 && ho < Ho; ++ho) {
      for (int wo = w / 2; wo <= (w + 1) / 2 && wo < Wo; ++wo) {
        float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
        int bidx[4] = {-1, -1, -1, -1};
#pragma unroll
        for (int dh = 0; dh < 3; ++dh) {
          const int hh = 2 * ho - 1 + dh;
          if (hh < 0 || hh >= H) continue;
#pragma unroll
          for (int dw = 0; dw < 3; ++dw) {
            const int ww = 2 * wo - 1 + dw;
            if (ww < 0 || ww >= W) continue;
            const float4 v4 = *reinterpret_cast<const float4*>(xb + ((int64_t)hh * W + ww) * C);
            const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (v[j] > best[j]) { best[j] = v[j]; bidx[j] = hh * W + ww; }
          }
        }
        const float4 g4 = *reinterpret_cast<const float4*>(dy + (((int64_t)b * Ho + ho) * Wo + wo) * C + c);
        const float g[4] = {g4.x, g4.y, g4.z, g4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (bidx[j] == h * W + w) acc[j] += g[j];
      }
    }
    *reinterpret_cast<float4*>(dx + pix * C + c) = make_float4(acc[0], acc[1], acc[2], acc[3]);
  }
}

// AvgPool2d(2, 2, 0, ceil_mode=True) backward (divisor = number of in-bounds elements, as count_include_pad only affects padding)
__global__ void avgpool_bwd_kernel(const float* __restrict__ dy, int B, int H, int W, int C, int Ho, int Wo, float* __restrict__ dx) {
  const int64_t total = (int64_t)B * H * W * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = i % C;
    const int64_t pix = i / C;
    const int w = pix % W, h = (pix / W) % H, b = pix / ((int64_t)W * H);
    const int ho = h >> 1, wo = w >> 1;
    const int nh = min(2, H - 2 * ho), nw = min(2, W - 2 * wo);
    dx[i] = dy[(((int64_t)b * Ho + ho) * Wo + wo) * C + c] / (float)(nh * nw);
  }
}

// bilinear (align_corners=False) backward as a GATHER over the input grid: dx[h,w] = sum over output pixels whose 2x2 footprint
// touches (h,w) of weight * dy.  For every output row only two source rows have non-zero weight, so we invert the map by scanning the
// output rows/cols that can reference h / w (bounded by ceil(scale)+1 each side).
__global__ void resize_bwd_kernel(const float* __restrict__ dy, int dy_pitch, int B, int H, int W, int C, int Ho, int Wo, float* __restrict__ dx) {
  const float sh = (float)H / Ho, sw = (float)W / Wo;
  const int64_t total = (int64_t)B * H * W * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = i % C;
    const int64_t pix = i / C;
    const int w = pix % W, h = (pix / W) % H, b = pix / ((int64_t)W * H);
    // candidate output rows: source coordinate (ho+0.5)*sh-0.5 in (h-1, h+1) (plus clamping at the borders)
    int ho_lo = (int)floorf((h - 1 + 0.5f) / sh - 0.5f), ho_hi = (int)ceilf((h + 1 + 0.5f) / sh - 0.5f);
    int wo_lo = (int)floorf((w - 1 + 0.5f) / sw - 0.5f), wo_hi = (int)ceilf((w + 1 + 0.5f) / sw - 0.5f);
    if (h == 0) ho_lo = 0;
    if (w == 0) wo_lo = 0;
    if (h == H - 1) ho_hi = Ho - 1;
    if (w == W - 1) wo_hi = Wo - 1;
    ho_lo = max(ho_lo, 0); wo_lo = max(wo_lo, 0); ho_hi = min(ho_hi, Ho - 1); wo_hi = min(wo_hi, Wo - 1);
    float acc = 0.f;
    for (int ho = ho_lo; ho <= ho_hi; ++ho) {
      float fy = ((float)ho + 0.5f) * sh - 0.5f;
      fy = fy < 0.f ? 0.f : fy;
      const int y0 = min((int)fy, H - 1), y1 = min(y0 + 1, H - 1);
      const float ly = fy - (float)y0;
      const float wy = (y0 == h ? 1.f - ly : 0.f) + (y1 == h ? ly : 0.f);
      if (wy == 0.f) continue;
      for (int wo = wo_lo; wo <= wo_hi; ++wo) {
        float fx = ((float)wo + 0.5f) * sw - 0.5f;
        fx = fx < 0.f ? 0.f : fx;
        const int x0 = min((int)fx, W - 1), x1 = min(x0 + 1, W - 1);
        const float lx = fx - (float)x0;
        const float wx = (x0 == w ? 1.f - lx : 0.f) + (x1 == w ? lx : 0.f);
        if (wx != 0.f) acc += wy * wx * dy[(((int64_t)b * Ho + ho) * Wo + wo) * dy_pitch + c];
      }
    }
    dx[i] = acc;
  }
}

// LayerNorm backward over s = x (+ res): one warp per row (C <= 1024, C % 32 == 0), row statistics recomputed;
// dx = rstd * (g - mean(g) - xhat * mean(g * xhat)), g = dy * gamma.  Per-block partial sums of dy*xhat / dy for dgamma / dbeta.
constexpr int LN_MAXV = 32;
// MAXV = register slots per thread (C <= 32 * MAXV): the C = 256 LayerNorms of the decoder take the 8-slot instantiation (the 32-slot one keeps 128 array registers live)
template <int MAXV>
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ res, const float* __restrict__ gamma,
                                                            const float* __restrict__ dy, int64_t M, int C, float eps, float* __restrict__ dx,
                                                            float* __restrict__ pg, float* __restrict__ pb) {
  extern __shared__ float ln_sm[];  // [2][C] block accumulators
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nv = C / 32;
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) ln_sm[i] = 0.f;
  __syncthreads();
  float ag[MAXV], ab[MAXV];
#pragma unroll
  for (int k = 0; k < MAXV; ++k) { ag[k] = 0.f; ab[k] = 0.f; }
  for (int64_t row = (int64_t)blockIdx.x * 8 + wid; row < M; row += (int64_t)gridDim.x * 8) {
    float v[MAXV], g[MAXV];
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k)
      if (k < nv) {
        const int c = k * 32 + lane;
        v[k] = x[row * C + c] + (res ? res[row * C + c] : 0.f);
        sum += v[k];
      }
    const float mean = warp_sum(sum) / (float)C;
    float sq = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k)
      if (k < nv) { const float d = v[k] - mean; sq += d * d; }
    const float rstd = rsqrtf(warp_sum(sq) / (float)C + eps);
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k)
      if (k < nv) {
        const int c = k * 32 + lane;
        const float d = dy[row * C + c];
        v[k] = (v[k] - mean) * rstd;
        g[k] = d * gamma[c];
        sg += g[k];
        sgx += g[k] * v[k];
        ag[k] += d * v[k];
        ab[k] += d;
      }
    sg = warp_sum(sg) / (float)C;
    sgx = warp_sum(sgx) / (float)C;
#pragma unroll
    for (int k = 0; k < MAXV; ++k)
      if (k < nv) dx[row * C + k * 32 + lane] = rstd * (g[k] - sg - v[k] * sgx);
  }
  // deterministic in-block combine: warps add their accumulators one after the other
  for (int w = 0; w < 8; ++w) {
    if (wid == w) {
#pragma unroll
      for (int k = 0; k < MAXV; ++k)
        if (k < nv) { ln_sm[k * 32 + lane] += ag[k]; ln_sm[C + k * 32 + lane] += ab[k]; }
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < C; i += blockDim.x) { pg[(int64_t)blockIdx.x * C + i] = ln_sm[i]; pb[(int64_t)blockIdx.x * C + i] = ln_sm[C + i]; }
}

inline unsigned grid_for(int64_t n, int threads = 256) { return (unsigned)std::min<int64_t>(cdiv(n, threads), kNumSMs * 16); }

}  // namespace
}  // namespace fb200

using namespace fb200;

extern "C" int64_t fb200_conv_wgrad_workspace_bytes(int B, int Ho, int Wo, int Cin, int Cout, int KH, int KW) {
  const int64_t tiles = (int64_t)cdiv(Cout, WG_TM) * cdiv(Cin, WG_TN) * KH * KW;
  const int64_t P = (int64_t)B * Ho * Wo;
  int64_t splits = std::max<int64_t>(1, std::min<int64_t>(cdiv(kNumSMs * 4, tiles), cdiv(P, 512)));
  splits = std::max<int64_t>(splits, 2 * kNumSMs);  // the stem kernel writes one partial per block (<= 2 per SM)
  return splits * Cout * KH * KW * Cin * 4 + 16;
}

extern "C" int fb200_conv_wgrad(const float* x, int B, int H, int W, int Cin, int x_pitch, const float* dy, int Ho, int Wo, int Cout, int dy_pitch, int KH,
                                int KW, int stride, int pad, float* dw, int accumulate, void* workspace, void* stream) {
  FB_CHECK_ARG(x && dy && dw && workspace, "conv_wgrad: null pointer");
  FB_CHECK_ARG(B > 0 && Cin > 0 && Cout > 0 && KH > 0 && KW > 0 && stride >= 1, "conv_wgrad: bad sizes");
  FB_CHECK_ARG(Ho == (H + 2 * pad - KH) / stride + 1 && Wo == (W + 2 * pad - KW) / stride + 1, "conv_wgrad: output size does not match");
  if (KH == 3 && KW == 3 && stride == 2 && pad == 1 && Cin <= 4 && Cout == 32 && 2LL * kNumSMs * 32 * 9 * Cin * 4 + 16 <= fb200_conv_wgrad_workspace_bytes(B, Ho, Wo, Cin, Cout, KH, KW)) {
    const int tiles_w = (int)cdiv(Wo, SW_TW), tiles_h = (int)cdiv(Ho, SW_TH);
    const int nblk = (int)std::min<int64_t>(2 * kNumSMs, (int64_t)B * tiles_w * tiles_h);
    cudaStream_t st0 = (cudaStream_t)stream;
    conv_wgrad_stem_kernel<<<nblk, 256, 0, st0>>>(x, x_pitch, dy, dy_pitch, B, H, W, Cin, Ho, Wo, tiles_w, tiles_h, reinterpret_cast<float*>(workspace));
    FB_CHECK_LAUNCH("conv_wgrad(stem)");
    const int64_t n0 = (int64_t)Cout * 9 * Cin;
    split_reduce_kernel<<<(unsigned)cdiv(n0, 256), 256, 0, st0>>>(reinterpret_cast<float*>(workspace), nblk, n0, dw, accumulate);
    FB_CHECK_LAUNCH("conv_wgrad(stem reduce)");
    return FB200_OK;
  }
  const int64_t tiles = (int64_t)cdiv(Cout, WG_TM) * cdiv(Cin, WG_TN);
  const int64_t P = (int64_t)B * Ho * Wo;
  const int64_t splits = std::max<int64_t>(1, std::min<int64_t>(cdiv(kNumSMs * 4, tiles * KH * KW), cdiv(P, 512)));
  const int64_t per = cdiv(cdiv(P, splits), WG_TK) * WG_TK;
  float* part = reinterpret_cast<float*>(workspace);
  cudaStream_t st = (cudaStream_t)stream;
  conv_wgrad_kernel<<<dim3((unsigned)tiles, KH * KW, (unsigned)splits), 256, 0, st>>>(x, x_pitch, dy, dy_pitch, B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad, per, part);
  FB_CHECK_LAUNCH("conv_wgrad");
  const int64_t n = (int64_t)Cout * KH * KW * Cin;
  split_reduce_kernel<<<(unsigned)cdiv(n, 256), 256, 0, st>>>(part, (int)splits, n, dw, accumulate);
  FB_CHECK_LAUNCH("conv_wgrad(reduce)");
  return FB200_OK;
}

extern "C" int fb200_dilate2(const float* dy, int B, int Ho, int Wo, int C, int Hd, int Wd, float* out, void* stream) {
  FB_CHECK_ARG(dy && out && C % 4 == 0 && Hd >= 2 * Ho - 1 && Wd >= 2 * Wo - 1, "dilate2: bad arguments");
  dilate2_kernel<<<grid_for((int64_t)B * Hd * Wd * (C / 4)), 256, 0, (cudaStream_t)stream>>>(dy, B, Ho, Wo, C, Hd, Wd, out);
  FB_CHECK_LAUNCH("dilate2");
  return FB200_OK;
}

extern "C" int64_t fb200_col_workspace_bytes(int C) { return (int64_t)(2 * CR_ROWS + 2) * C * 4 + 16; }

static inline dim3 col_grid(int C, int64_t R) { return dim3((unsigned)cdiv(C, 32), (unsigned)std::min<int64_t>(CR_ROWS, cdiv(R, 8))); }

static inline bool col_vec_ok(int C, const void* x, int x_pitch, const void* dy, int dy_pitch, const void* y, int y_pitch) {
  if (!(C == 32 || C == 64 || C == 128 || (C > 128 && C % 128 == 0))) return false;
  if (x_pitch % 4 || (dy && dy_pitch % 4) || (y && y_pitch % 4)) return false;
  return ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
}
// grid of the column-fixed element-wise kernels: a multiple of C/4 threads (0 = use the generic kernel)
static inline unsigned cf_grid(int64_t R, int C) {
  const int cv = C / 4;
  if (C % 4 || cv <= 0) return 0;
  int64_t blocks = std::min<int64_t>(cdiv(R * cv, 256), kNumSMs * 16);
  if (cv <= 256) { if (256 % cv) return 0; }           // every block holds whole rows' worth of column groups
  else { if (cv % 256) return 0; const int64_t m = cv / 256; blocks = blocks / m * m; }
  return (unsigned)std::max<int64_t>(blocks, cv > 256 ? cv / 256 : 1);
}
static void bn_apply_launch(const float* x, int x_pitch, const float* res, int res_pitch, int64_t R, int C, const float* mean, const float* rstd, const float* gamma,
                            const float* beta, int act, float* y, int y_pitch, cudaStream_t st) {
  const unsigned g = cf_grid(R, C);
  const bool al = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(res) | reinterpret_cast<uintptr_t>(y)) & 15) == 0 && x_pitch % 4 == 0 && y_pitch % 4 == 0 &&
                  (!res || res_pitch % 4 == 0);
  if (g && al) bn_apply_cf_kernel<<<g, 256, 0, st>>>(x, x_pitch, res, res_pitch, R, C, mean, rstd, gamma, beta, act, y, y_pitch);
  else bn_apply_kernel<<<grid_for(R * (C / 4)), 256, 0, st>>>(x, x_pitch, res, res_pitch, R, C, mean, rstd, gamma, beta, act, y, y_pitch);
}

// one column pass (MODE 0 colsum / 2 BN backward sums / 3 moments) -> partials p0 / p1 [parts][C]; returns the number of parts (and in *rpb the rows
// each part takes per row step)
template <int MODE>
static int col_partial_launch(const float* x, int x_pitch, int64_t R, int C, const float* mean, const float* rstd, const float* gamma, const float* beta, const float* dy,
                              int dy_pitch, const float* y, int y_pitch, int act, float* p0, float* p1, cudaStream_t st, int* rpb = nullptr) {
  if (col_vec_ok(C, x, x_pitch, dy, dy_pitch, y, y_pitch)) {
    const int CW = C < 128 ? C : 128, RPB = 256 / (CW / 4);
    const dim3 g((unsigned)(C / CW), (unsigned)std::min<int64_t>(CR_ROWS, cdiv(R, (int64_t)RPB)));
    col_partial4_kernel<MODE><<<g, 256, 0, st>>>(x, x_pitch, R, C, mean, rstd, gamma, beta, dy, dy_pitch, y, y_pitch, act, p0, p1);
    if (rpb) *rpb = RPB;
    return (int)g.y;
  }
  const dim3 g = col_grid(C, R);
  col_partial_kernel<MODE><<<g, 256, 0, st>>>(x, x_pitch, R, C, mean, rstd, gamma, beta, dy, dy_pitch, y, y_pitch, act, p0, p1);
  if (rpb) *rpb = 8;
  return (int)g.y;
}

extern "C" int fb200_colsum(const float* x, int64_t R, int C, int pitch, float* out, int accumulate, void* workspace, void* stream) {
  FB_CHECK_ARG(x && out && workspace && R > 0 && C > 0, "colsum: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  float* p0 = reinterpret_cast<float*>(workspace);
  const int parts = col_partial_launch<0>(x, pitch, R, C, nullptr, nullptr, nullptr, nullptr, nullptr, 0, nullptr, 0, 0, p0, nullptr, st);
  FB_CHECK_LAUNCH("colsum");
  col_finalize_kernel<0><<<cdiv(C, 128), 128, 0, st>>>(p0, nullptr, parts, C, (double)R, 0.f, 0.f, nullptr, nullptr, nullptr, out, nullptr, accumulate);
  FB_CHECK_LAUNCH("colsum(finalize)");
  return FB200_OK;
}

extern "C" int fb200_bn_train_fwd(const float* x, int x_pitch, int64_t R, int C, const float* gamma, const float* beta, const float* res, int res_pitch, int act,
                                  float eps, float momentum, float* running_mean, float* running_var, float* save_mean, float* save_rstd, float* y, int y_pitch,
                                  void* workspace, void* stream) {
  FB_CHECK_ARG(x && gamma && beta && save_mean && save_rstd && y && workspace && R > 0 && C % 4 == 0, "bn_train_fwd: bad arguments");
  FB_CHECK_ARG(act == FB200_ACT_NONE || act == FB200_ACT_RELU || (act == FB200_ACT_SILU && !res), "bn_train_fwd: act must be none/relu (or silu without residual)");
  cudaStream_t st = (cudaStream_t)stream;
  float* p0 = reinterpret_cast<float*>(workspace);
  float* p1 = p0 + (int64_t)CR_ROWS * C;
  // ONE pass over x for both moments (per-part mean and squared deviations, combined in double); `x` itself serves as the pivot row for the finaliser
  int rpb = 0;
  const int parts = col_partial_launch<3>(x, x_pitch, R, C, nullptr, nullptr, nullptr, nullptr, nullptr, 0, nullptr, 0, 0, p0, p1, st, &rpb);
  bn_stats_finalize_kernel<4><<<cdiv(C, 8), 256, 0, st>>>(p0, p1, parts, rpb, C, R, eps, momentum, x, running_mean, running_var, save_mean, save_rstd);
  bn_apply_launch(x, x_pitch, res, res_pitch, R, C, save_mean, save_rstd, gamma, beta, act, y, y_pitch, st);
  FB_CHECK_LAUNCH("bn_train_fwd");
  return FB200_OK;
}

extern "C" int fb200_bn_train_bwd(const float* x, int x_pitch, const float* dy, int dy_pitch, const float* y, int y_pitch, int64_t R, int C, const float* gamma,
                                  const float* beta, const float* save_mean, const float* save_rstd, int act, float* dx, int dx_pitch, float* dres, int dres_pitch,
                                  float* dgamma, float* dbeta, int accumulate, void* workspace, void* stream) {
  FB_CHECK_ARG(x && dy && gamma && beta && save_mean && save_rstd && dx && dgamma && dbeta && workspace && R > 0, "bn_train_bwd: bad arguments");
  FB_CHECK_ARG(act == FB200_ACT_NONE || y || !dres, "bn_train_bwd: with a fused residual the activation gradient needs the forward output");
  cudaStream_t st = (cudaStream_t)stream;
  float* p0 = reinterpret_cast<float*>(workspace);
  float* p1 = p0 + (int64_t)CR_ROWS * C;
  float* f0 = p1 + (int64_t)CR_ROWS * C;  // this step's dbeta / dgamma: needed by dx before they may be accumulated into the caller's buffers
  float* f1 = f0 + C;
  const int parts = col_partial_launch<2>(x, x_pitch, R, C, save_mean, save_rstd, gamma, beta, dy, dy_pitch, y, y_pitch, act, p0, p1, st);
  col_finalize_kernel<3><<<cdiv(C, 128), 128, 0, st>>>(p0, p1, parts, C, (double)R, 0.f, 0.f, nullptr, nullptr, nullptr, f0, f1, 0);
  const bool v4 = C % 4 == 0 && x_pitch % 4 == 0 && dy_pitch % 4 == 0 && dx_pitch % 4 == 0 && (!y || y_pitch % 4 == 0) && (!dres || dres_pitch % 4 == 0) &&
                  ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx) | reinterpret_cast<uintptr_t>(y) |
                    reinterpret_cast<uintptr_t>(dres)) & 15) == 0;
  if (v4 && cf_grid(R, C))
    bn_bwd_apply_cf_kernel<<<cf_grid(R, C), 256, 0, st>>>(x, x_pitch, dy, dy_pitch, y, y_pitch, R, C, save_mean, save_rstd, gamma, beta, f1, f0, act, (float)(1.0 / (double)R),
                                                         dx, dx_pitch, dres, dres_pitch);
  else if (v4)
    bn_bwd_apply4_kernel<<<grid_for(R * (C / 4)), 256, 0, st>>>(x, x_pitch, dy, dy_pitch, y, y_pitch, R, C, save_mean, save_rstd, gamma, beta, f1, f0, act,
                                                               (float)(1.0 / (double)R), dx, dx_pitch, dres, dres_pitch);
  else
    bn_bwd_apply_kernel<<<grid_for(R * C), 256, 0, st>>>(x, x_pitch, dy, dy_pitch, y, y_pitch, R, C, save_mean, save_rstd, gamma, beta, f1, f0, act, (float)(1.0 / (double)R),
                                                         dx, dx_pitch, dres, dres_pitch);
  col_finalize_kernel<3><<<cdiv(C, 128), 128, 0, st>>>(f0, f1, 1, C, (double)R, 0.f, 0.f, nullptr, nullptr, nullptr, dbeta, dgamma, accumulate);
  FB_CHECK_LAUNCH("bn_train_bwd");
  return FB200_OK;
}

// ---- BatchNorm in phases (SyncBatchNorm across data-parallel ranks, FrozenBatchNorm2d): statistics | apply | backward sums | backward apply ----------
extern "C" int fb200_bn_stats(const float* x, int x_pitch, int64_t R, int C, float* mean, float* var_biased, void* workspace, void* stream) {
  FB_CHECK_ARG(x && mean && var_biased && workspace && R > 0 && C % 4 == 0, "bn_stats: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  float* p0 = reinterpret_cast<float*>(workspace);
  float* p1 = p0 + (int64_t)CR_ROWS * C;
  int rpb = 0;
  const int parts = col_partial_launch<3>(x, x_pitch, R, C, nullptr, nullptr, nullptr, nullptr, nullptr, 0, nullptr, 0, 0, p0, p1, st, &rpb);
  bn_stats_finalize_kernel<5><<<cdiv(C, 8), 256, 0, st>>>(p0, p1, parts, rpb, C, R, 0.f, 0.f, x, nullptr, nullptr, mean, var_biased);
  FB_CHECK_LAUNCH("bn_stats");
  return FB200_OK;
}

// SyncBatchNorm: combine the per-rank moments gathered by all_gather (row r = [mean_r (C) | biased var_r (C) | row count n_r]) into the global mean / rstd, update the
// running statistics (unbiased variance over the GLOBAL count, like aten's batch_norm_gather_stats_with_counts) and leave 1 / total on the device for the backward pass -
// one launch instead of a dozen small torch kernels and two host read-backs per layer
__global__ void bn_sync_combine_kernel(const float* __restrict__ allst, int world, int C, float eps, float momentum, float* __restrict__ run_mean,
                                       float* __restrict__ run_var, float* __restrict__ mean, float* __restrict__ rstd, float* __restrict__ inv_total) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int pitch = 2 * C + 1;
  double total = 0.0;
  for (int r = 0; r < world; ++r) total += (double)allst[(int64_t)r * pitch + 2 * C];
  if (c == 0) inv_total[0] = (float)(1.0 / total);
  if (c >= C) return;
  double m = 0.0;
  for (int r = 0; r < world; ++r) m += (double)allst[(int64_t)r * pitch + c] * (double)allst[(int64_t)r * pitch + 2 * C];
  m /= total;
  double v = 0.0;
  for (int r = 0; r < world; ++r) {
    const double d = (double)allst[(int64_t)r * pitch + c] - m;
    v += ((double)allst[(int64_t)r * pitch + C + c] + d * d) * (double)allst[(int64_t)r * pitch + 2 * C];
  }
  v /= total;
  mean[c] = (float)m;
  rstd[c] = (float)(1.0 / sqrt(v + (double)eps));
  if (run_mean) {
    run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * (float)m;
    run_var[c] = (1.f - momentum) * run_var[c] + momentum * (float)(total > 1.0 ? v * total / (total - 1.0) : v);
  }
}

extern "C" int fb200_bn_sync_combine(const float* all_stats, int world, int C, float eps, float momentum, float* running_mean, float* running_var, float* mean,
                                     float* rstd, float* inv_total, void* stream) {
  FB_CHECK_ARG(all_stats && mean && rstd && inv_total && world > 0 && C > 0, "bn_sync_combine: bad arguments");
  FB_CHECK_ARG((running_mean == nullptr) == (running_var == nullptr), "bn_sync_combine: running_mean and running_var go together");
  bn_sync_combine_kernel<<<cdiv(C, 128), 128, 0, (cudaStream_t)stream>>>(all_stats, world, C, eps, momentum, running_mean, running_var, mean, rstd, inv_total);
  FB_CHECK_LAUNCH("bn_sync_combine");
  return FB200_OK;
}

extern "C" int fb200_bn_apply(const float* x, int x_pitch, int64_t R, int C, const float* mean, const float* rstd, const float* gamma, const float* beta,
                              const float* res, int res_pitch, int act, float* y, int y_pitch, void* stream) {
  FB_CHECK_ARG(x && mean && rstd && gamma && beta && y && R > 0 && C % 4 == 0, "bn_apply: bad arguments");
  FB_CHECK_ARG(act == FB200_ACT_NONE || act == FB200_ACT_RELU || (act == FB200_ACT_SILU && !res), "bn_apply: act must be none/relu (or silu without residual)");
  bn_apply_launch(x, x_pitch, res, res_pitch, R, C, mean, rstd, gamma, beta, act, y, y_pitch, (cudaStream_t)stream);
  FB_CHECK_LAUNCH("bn_apply");
  return FB200_OK;
}

extern "C" int fb200_bn_bwd_reduce(const float* x, int x_pitch, const float* dy, int dy_pitch, const float* y, int y_pitch, int64_t R, int C, const float* gamma,
                                   const float* beta, const float* mean, const float* rstd, int act, float* sum_dy, float* sum_dy_xhat, void* workspace, void* stream) {
  FB_CHECK_ARG(x && dy && gamma && beta && mean && rstd && sum_dy && sum_dy_xhat && workspace && R > 0, "bn_bwd_reduce: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  float* p0 = reinterpret_cast<float*>(workspace);
  float* p1 = p0 + (int64_t)CR_ROWS * C;
  const int parts = col_partial_launch<2>(x, x_pitch, R, C, mean, rstd, gamma, beta, dy, dy_pitch, y, y_pitch, act, p0, p1, st);
  col_finalize_kernel<3><<<cdiv(C, 128), 128, 0, st>>>(p0, p1, parts, C, (double)R, 0.f, 0.f, nullptr, nullptr, nullptr, sum_dy, sum_dy_xhat, 0);
  FB_CHECK_LAUNCH("bn_bwd_reduce");
  return FB200_OK;
}

extern "C" int fb200_bn_bwd_apply(const float* x, int x_pitch, const float* dy, int dy_pitch, const float* y, int y_pitch, int64_t R, int C, const float* gamma,
                                  const float* beta, const float* mean, const float* rstd, const float* sum_dy, const float* sum_dy_xhat, float inv_count, int act,
                                  float* dx, int dx_pitch, float* dres, int dres_pitch, void* stream) {
  FB_CHECK_ARG(x && dy && gamma && beta && mean && rstd && sum_dy && sum_dy_xhat && dx && R > 0, "bn_bwd_apply: bad arguments");
  FB_CHECK_ARG(act == FB200_ACT_NONE || y || !dres, "bn_bwd_apply: with a fused residual the activation gradient needs the forward output");
  const bool v4 = C % 4 == 0 && x_pitch % 4 == 0 && dy_pitch % 4 == 0 && dx_pitch % 4 == 0 && (!y || y_pitch % 4 == 0) && (!dres || dres_pitch % 4 == 0) &&
                  ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx) | reinterpret_cast<uintptr_t>(y) |
                    reinterpret_cast<uintptr_t>(dres)) & 15) == 0;
  if (v4 && cf_grid(R, C))
    bn_bwd_apply_cf_kernel<<<cf_grid(R, C), 256, 0, (cudaStream_t)stream>>>(x, x_pitch, dy, dy_pitch, y, y_pitch, R, C, mean, rstd, gamma, beta, sum_dy_xhat, sum_dy, act,
                                                                           inv_count, dx, dx_pitch, dres, dres_pitch);
  else if (v4)
    bn_bwd_apply4_kernel<<<grid_for(R * (C / 4)), 256, 0, (cudaStream_t)stream>>>(x, x_pitch, dy, dy_pitch, y, y_pitch, R, C, mean, rstd, gamma, beta, sum_dy_xhat, sum_dy, act,
                                                                                  inv_count, dx, dx_pitch, dres, dres_pitch);
  else
    bn_bwd_apply_kernel<<<grid_for(R * C), 256, 0, (cudaStream_t)stream>>>(x, x_pitch, dy, dy_pitch, y, y_pitch, R, C, mean, rstd, gamma, beta, sum_dy_xhat, sum_dy, act, inv_count,
                                                                           dx, dx_pitch, dres, dres_pitch);
  FB_CHECK_LAUNCH("bn_bwd_apply");
  return FB200_OK;
}

extern "C" int fb200_add_act(const float* a, const float* b, const float* dy, int act, int64_t n, float* out, void* stream) {
  FB_CHECK_ARG(a && out && n > 0 && act >= 0 && act <= FB200_ACT_GELU, "add_act: bad arguments");
  add_act_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(a, b, dy, act, n, out);
  FB_CHECK_LAUNCH("add_act");
  return FB200_OK;
}

extern "C" int fb200_maxpool3x3s2_bwd(const float* x, const float* dy, int B, int H, int W, int C, float* dx, void* stream) {
  FB_CHECK_ARG(x && dy && dx, "maxpool3x3s2_bwd: null pointer");
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  if (C % 4 == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0)
    maxpool_bwd4_kernel<<<grid_for((int64_t)B * H * W * (C / 4)), 256, 0, (cudaStream_t)stream>>>(x, dy, B, H, W, C, Ho, Wo, dx);
  else
    maxpool_bwd_kernel<<<grid_for((int64_t)B * H * W * C), 256, 0, (cudaStream_t)stream>>>(x, dy, B, H, W, C, Ho, Wo, dx);
  FB_CHECK_LAUNCH("maxpool3x3s2_bwd");
  return FB200_OK;
}

extern "C" int fb200_avgpool2x2_ceil_bwd(const float* dy, int B, int H, int W, int C, float* dx, void* stream) {
  FB_CHECK_ARG(dy && dx, "avgpool2x2_ceil_bwd: null pointer");
  avgpool_bwd_kernel<<<grid_for((int64_t)B * H * W * C), 256, 0, (cudaStream_t)stream>>>(dy, B, H, W, C, (H + 1) / 2, (W + 1) / 2, dx);
  FB_CHECK_LAUNCH("avgpool2x2_ceil_bwd");
  return FB200_OK;
}

extern "C" int fb200_resize_bilinear_bwd(const float* dy, int dy_pitch, int B, int H, int W, int C, int Ho, int Wo, float* dx, void* stream) {
  FB_CHECK_ARG(dy && dx && H > 0 && W > 0 && Ho > 0 && Wo > 0, "resize_bilinear_bwd: bad arguments");
  resize_bwd_kernel<<<grid_for((int64_t)B * H * W * C), 256, 0, (cudaStream_t)stream>>>(dy, dy_pitch, B, H, W, C, Ho, Wo, dx);
  FB_CHECK_LAUNCH("resize_bilinear_bwd");
  return FB200_OK;
}

extern "C" int fb200_layernorm_bwd(const float* x, const float* res, const float* gamma, const float* dy, int64_t M, int C, float eps, float* dx, float* dgamma,
                                   float* dbeta, int accumulate, void* workspace, void* stream) {
  FB_CHECK_ARG(x && gamma && dy && dx && dgamma && dbeta && workspace && M > 0, "layernorm_bwd: bad arguments");
  FB_CHECK_ARG(C % 32 == 0 && C <= 32 * LN_MAXV, "layernorm_bwd: C must be a multiple of 32 and <= %d", 32 * LN_MAXV);
  cudaStream_t st = (cudaStream_t)stream;
  const int nblk = (int)std::min<int64_t>(CR_ROWS, cdiv(M, 8));
  float* pg = reinterpret_cast<float*>(workspace);
  float* pb = pg + (int64_t)CR_ROWS * C;
  if (C <= 256) layernorm_bwd_kernel<8><<<nblk, 256, 2 * C * sizeof(float), st>>>(x, res, gamma, dy, M, C, eps, dx, pg, pb);
  else layernorm_bwd_kernel<LN_MAXV><<<nblk, 256, 2 * C * sizeof(float), st>>>(x, res, gamma, dy, M, C, eps, dx, pg, pb);
  FB_CHECK_LAUNCH("layernorm_bwd");
  col_finalize_kernel<3><<<cdiv(C, 128), 128, 0, st>>>(pb, pg, nblk, C, 1.0, 0.f, 0.f, nullptr, nullptr, nullptr, dbeta, dgamma, accumulate);
  FB_CHECK_LAUNCH("layernorm_bwd(finalize)");
  return FB200_OK;
}

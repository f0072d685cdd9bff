// SIMT (CUDA-core, fp32 accumulate) convolution kernels:
//   * fb200_stem_conv3x3s2 — normalise + 3x3/s2 conv + BN + act straight from the NCHW fp32 image.
//   * conv_igemm_simt      — generic implicit-GEMM conv / linear with fused scale/bias/residual/act
//                            epilogue.  This is the fp32 parity path and the fall-back for shapes the
//                            tensor-core kernel (conv_tc.cu) does not take (Cin % 64 != 0, fp32 activations).
#include <stdarg.h>

#include "common.cuh"

namespace fb200 {

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// Tiled stem: a CTA computes a 16 x 16 tile of output pixels.  The 33 x 33 x 3 input patch is read ONCE (coalesced rows), normalised ONCE per input pixel and kept in
// shared memory as even / odd column planes (the stride-2 taps of 16 neighbouring threads then hit 16 consecutive floats: no bank conflicts); the 27 x 32 weights are
// read as float4 broadcasts.  Each input byte is loaded and normalised (with a division) once, not once for each of the up to nine taps that use it.
template <typename TOut, bool U8_NHWC, bool RELU>   // RELU: the activation is known to be ReLU (every model family's stem): no generic activation code in the kernel at all
__global__ void __launch_bounds__(256) stem_conv_tiled_kernel(const void* __restrict__ img_, int B, int H, int W, const float* __restrict__ w,
                                                              const float* __restrict__ scale, const float* __restrict__ bias, float m0, float m1, float m2,
                                                              float s0, float s1, float s2, int act, TOut* __restrict__ out, int tiles_w, int tiles_h) {
  constexpr int COUT = 32, T = 16, PR = 2 * T + 1, HC = T + 1;   // patch rows, columns per parity plane
  __shared__ __align__(16) float ws[27 * COUT];
  __shared__ float sc[COUT], bi[COUT];
  __shared__ float sin_[3][PR][2][HC + 1];
  const int tid = threadIdx.x;
  for (int i = tid; i < 27 * COUT; i += 256) { const int co = i % COUT, t = i / COUT; ws[i] = w[co * 27 + t]; }
  if (tid < COUT) { sc[tid] = scale ? scale[tid] : 1.f; bi[tid] = bias ? bias[tid] : 0.f; }
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  int t = blockIdx.x;
  const int tw = t % tiles_w; t /= tiles_w;
  const int th = t % tiles_h; const int b = t / tiles_h;
  const int ho0 = th * T, wo0 = tw * T;
  const int hi0 = 2 * ho0 - 1, wi0 = 2 * wo0 - 1;
  const float mean[3] = {m0, m1, m2}, stdv[3] = {s0, s1, s2};
  // the patch: all of a thread's (up to 13) loads are issued before the first one is consumed - as a rolled loop every iteration waited for its own global load
  // (13 dependent round trips per CTA in front of ~2 us of arithmetic)
  constexpr int NP = PR * PR * 3, NIT = (NP + 255) / 256;
  float raw[NIT];
  if (U8_NHWC) {
    // patch row r = 99 consecutive bytes (33 pixels x 3 channels) of image row hi0 + r: element i = r * 99 + j, walked incrementally (256 = 2 * 99 + 58) with 32-bit
    // offsets inside the image - the kernel is instruction-bound (ncu: 3340 instructions per warp for 864 FMAs, ALU pipe busier than the FMA pipe)
    constexpr int RB = PR * 3;
    const uint8_t* ub = reinterpret_cast<const uint8_t*>(img_) + (int64_t)b * H * W * 3;
    // (x - mean) / std takes only 3 x 256 values for uint8 input: one IEEE division per table entry (3 per thread) instead of one per patch element (13 per thread,
    // ~25 instructions each) - same arithmetic, same bits
    __shared__ float lut[3][256];
    lut[0][tid] = ((float)tid - m0) / s0; lut[1][tid] = ((float)tid - m1) / s1; lut[2][tid] = ((float)tid - m2) / s2;
    int r = tid / RB, j = tid - r * RB;
    int rr[NIT], jj[NIT];
#pragma unroll
    for (int u = 0; u < NIT; ++u) {  // consecutive threads -> consecutive bytes of a patch row
      rr[u] = r; jj[u] = j;
      const int c = j / 3;
      const int hi = hi0 + r, wi = wi0 + c;
      raw[u] = -1.f;  // marks "outside": the conv pads the NORMALISED image with zeros
      if (r < PR && hi >= 0 && hi < H && wi >= 0 && wi < W) raw[u] = (float)ub[(hi * W + wi0) * 3 + j];
      j += 256 - 2 * RB; r += 2;
      if (j >= RB) { j -= RB; r += 1; }
    }
    __syncthreads();  // the table
#pragma unroll
    for (int u = 0; u < NIT; ++u) {
      if (rr[u] < PR) {
        const int c = jj[u] / 3, ci = jj[u] - 3 * c;
        sin_[ci][rr[u]][c & 1][c >> 1] = raw[u] < 0.f ? 0.f : lut[ci][(int)raw[u]];
      }
    }
  } else {
    const float* ib = reinterpret_cast<const float*>(img_) + (int64_t)b * 3 * H * W;
    bool inb[NIT];
#pragma unroll
    for (int u = 0; u < NIT; ++u) {
      const int i = tid + u * 256;
      const int c = i % PR, r = (i / PR) % PR, ci = i / (PR * PR);
      const int hi = hi0 + r, wi = wi0 + c;
      inb[u] = i < NP && hi >= 0 && hi < H && wi >= 0 && wi < W;
      raw[u] = inb[u] ? ib[((int64_t)ci * H + hi) * W + wi] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < NIT; ++u) {
      const int i = tid + u * 256;
      if (i < NP) {
        const int c = i % PR, r = (i / PR) % PR, ci = i / (PR * PR);
        sin_[ci][r][c & 1][c >> 1] = inb[u] ? (raw[u] - mean[ci]) / stdv[ci] : 0.f;
      }
    }
  }
  __syncthreads();
  const int tx = tid & 15, ty = tid >> 4;
  float acc[COUT];
#pragma unroll
  for (int i = 0; i < COUT; ++i) acc[i] = 0.f;
#pragma unroll
  for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
#pragma unroll
      for (int ci = 0; ci < 3; ++ci) {
        const float v = sin_[ci][2 * ty + kh][kw & 1][tx + (kw >> 1)];
        const float4* wr = reinterpret_cast<const float4*>(&ws[((kh * 3 + kw) * 3 + ci) * COUT]);
#pragma unroll
        for (int q = 0; q < COUT / 4; ++q) {
          const float4 wv = wr[q];
          acc[q * 4 + 0] = fmaf(v, wv.x, acc[q * 4 + 0]); acc[q * 4 + 1] = fmaf(v, wv.y, acc[q * 4 + 1]);
          acc[q * 4 + 2] = fmaf(v, wv.z, acc[q * 4 + 2]); acc[q * 4 + 3] = fmaf(v, wv.w, acc[q * 4 + 3]);
        }
      }
    }
  }
  const int ho = ho0 + ty, wo = wo0 + tx;
  if (ho >= Ho || wo >= Wo) return;
  const int64_t pix = ((int64_t)b * Ho + ho) * Wo + wo;
  // folded BN + activation with the activation switch OUTSIDE the element loop (a per-element switch on the runtime `act` was a third of the kernel's instructions)
#pragma unroll
  for (int co = 0; co < COUT; ++co) acc[co] = acc[co] * sc[co] + bi[co];
  if constexpr (RELU) {
#pragma unroll
    for (int co = 0; co < COUT; ++co) acc[co] = fmaxf(acc[co], 0.f);
  } else if ((act & 15) != FB200_ACT_NONE) {
#pragma unroll
    for (int co = 0; co < COUT; ++co) acc[co] = apply_act(acc[co], act);
  }
  if (act & 256) {  // FB200_F16PAIR output: [hi(32) | lo(32)] fp16 per pixel, written as 16-byte vectors (8 halves): half the store instructions of 8-byte pieces
    __half* o = reinterpret_cast<__half*>(out) + pix * 2 * COUT;
#pragma unroll
    for (int co = 0; co < COUT; co += 8) {
      __half2 h2[4], l2[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float v0 = acc[co + 2 * j], v1 = acc[co + 2 * j + 1];
        const __half a0 = __float2half_rn(v0), a1 = __float2half_rn(v1);
        h2[j] = __halves2half2(a0, a1);
        l2[j] = __halves2half2(__float2half_rn(v0 - __half2float(a0)), __float2half_rn(v1 - __half2float(a1)));
      }
      *reinterpret_cast<uint4*>(o + co) = *reinterpret_cast<const uint4*>(h2);
      *reinterpret_cast<uint4*>(o + COUT + co) = *reinterpret_cast<const uint4*>(l2);
    }
    return;
  }
  TOut* o = out + pix * COUT;
#pragma unroll
  for (int co = 0; co < COUT; co += 4) {
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = acc[co + j];
    store4(o + co, v);
  }
}

// Two output pixels per thread (rows ty and ty + 8 of the 16 x 16 tile, 128 threads): every float4 weight broadcast feeds 8 FMAs instead of 4 and the per-thread
// preamble / epilogue instructions are shared by two pixels - the one-pixel kernel above is instruction-bound (2184 SASS instructions per pixel for 864 FMAs).
// uint8 NHWC input + ReLU only (the deployment path of all three model families); PAIR selects the [hi(32) | lo(32)] fp16 output.
template <typename TOut, bool PAIR>
__global__ void __launch_bounds__(128) stem_conv_tiled2_kernel(const uint8_t* __restrict__ img, int B, int H, int W, const float* __restrict__ w,
                                                               const float* __restrict__ scale, const float* __restrict__ bias, float m0, float m1, float m2, float s0,
                                                               float s1, float s2, TOut* __restrict__ out, int tiles_w, int tiles_h) {
  constexpr int COUT = 32, T = 16, PR = 2 * T + 1, HC = T + 1, NT = 128, RB = PR * 3;
  __shared__ __align__(16) float ws[27 * COUT];
  __shared__ float sc[COUT], bi[COUT];
  __shared__ float lut[3][256];
  __shared__ float sin_[3][PR][2][HC + 3];  // two patch rows = 80 floats = 16 banks apart: the two half-warps (rows ty, ty + 1) do not collide
  const int tid = threadIdx.x;
  for (int i = tid; i < 27 * COUT; i += NT) { const int co = i % COUT, t = i / COUT; ws[i] = w[co * 27 + t]; }
  if (tid < COUT) { sc[tid] = scale ? scale[tid] : 1.f; bi[tid] = bias ? bias[tid] : 0.f; }
#pragma unroll
  for (int v = tid; v < 256; v += NT) { lut[0][v] = ((float)v - m0) / s0; lut[1][v] = ((float)v - m1) / s1; lut[2][v] = ((float)v - m2) / s2; }
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  int t = blockIdx.x;
  const int tw = t % tiles_w; t /= tiles_w;
  const int th = t % tiles_h; const int b = t / tiles_h;
  const int ho0 = th * T, wo0 = tw * T;
  const int hi0 = 2 * ho0 - 1, wi0 = 2 * wo0 - 1;
  const uint8_t* ub = img + (int64_t)b * H * W * 3;
  __syncthreads();  // the table
  {  // patch: element i = r * 99 + j, two batches of 13 loads per thread, each batch issued before it is consumed (128 = 99 + 29)
    constexpr int NB = 13;
    int r = tid / RB, j = tid - r * RB;
#pragma unroll
    for (int batch = 0; batch < 2; ++batch) {
      float raw[NB];
      int rr[NB], jj[NB];
#pragma unroll
      for (int u = 0; u < NB; ++u) {
        rr[u] = r; jj[u] = j;
        const int c = j / 3, hi = hi0 + r, wi = wi0 + c;
        raw[u] = -1.f;
        if (r < PR && hi >= 0 && hi < H && wi >= 0 && wi < W) raw[u] = (float)ub[(hi * W + wi0) * 3 + j];
        j += NT - RB; r += 1;
        if (j >= RB) { j -= RB; r += 1; }
      }
#pragma unroll
      for (int u = 0; u < NB; ++u) {
        if (rr[u] < PR) {
          const int c = jj[u] / 3, ci = jj[u] - 3 * c;
          sin_[ci][rr[u]][c & 1][c >> 1] = raw[u] < 0.f ? 0.f : lut[ci][(int)raw[u]];
        }
      }
    }
  }
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  const int tx = lane & 15, ty = warp * 2 + (lane >> 4);   // rows ty and ty + 8
  float acc[2][COUT];
#pragma unroll
  for (int i = 0; i < COUT; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
#pragma unroll
  for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
#pragma unroll
      for (int ci = 0; ci < 3; ++ci) {
        const float v0 = sin_[ci][2 * ty + kh][kw & 1][tx + (kw >> 1)];
        const float v1 = sin_[ci][2 * (ty + 8) + kh][kw & 1][tx + (kw >> 1)];
        const float4* wr = reinterpret_cast<const float4*>(&ws[((kh * 3 + kw) * 3 + ci) * COUT]);
#pragma unroll
        for (int q = 0; q < COUT / 4; ++q) {
          const float4 wv = wr[q];
          acc[0][q * 4 + 0] = fmaf(v0, wv.x, acc[0][q * 4 + 0]); acc[0][q * 4 + 1] = fmaf(v0, wv.y, acc[0][q * 4 + 1]);
          acc[0][q * 4 + 2] = fmaf(v0, wv.z, acc[0][q * 4 + 2]); acc[0][q * 4 + 3] = fmaf(v0, wv.w, acc[0][q * 4 + 3]);
          acc[1][q * 4 + 0] = fmaf(v1, wv.x, acc[1][q * 4 + 0]); acc[1][q * 4 + 1] = fmaf(v1, wv.y, acc[1][q * 4 + 1]);
          acc[1][q * 4 + 2] = fmaf(v1, wv.z, acc[1][q * 4 + 2]); acc[1][q * 4 + 3] = fmaf(v1, wv.w, acc[1][q * 4 + 3]);
        }
      }
    }
  }
#pragma unroll
  for (int px = 0; px < 2; ++px) {
    const int ho = ho0 + ty + 8 * px, wo = wo0 + tx;
    if (ho >= Ho || wo >= Wo) continue;
    const int64_t pix = ((int64_t)b * Ho + ho) * Wo + wo;
#pragma unroll
    for (int co = 0; co < COUT; ++co) acc[px][co] = fmaxf(acc[px][co] * sc[co] + bi[co], 0.f);
    if constexpr (PAIR) {
      __half* o = reinterpret_cast<__half*>(out) + pix * 2 * COUT;
#pragma unroll
      for (int co = 0; co < COUT; co += 8) {
        __half2 h2[4], l2[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float v0 = acc[px][co + 2 * j], v1 = acc[px][co + 2 * j + 1];
          const __half a0 = __float2half_rn(v0), a1 = __float2half_rn(v1);
          h2[j] = __halves2half2(a0, a1);
          l2[j] = __halves2half2(__float2half_rn(v0 - __half2float(a0)), __float2half_rn(v1 - __half2float(a1)));
        }
        *reinterpret_cast<uint4*>(o + co) = *reinterpret_cast<const uint4*>(h2);
        *reinterpret_cast<uint4*>(o + COUT + co) = *reinterpret_cast<const uint4*>(l2);
      }
    } else {
      TOut* o = out + pix * COUT;
#pragma unroll
      for (int co = 0; co < COUT; co += 4) {
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = acc[px][co + j];
        store4(o + co, v);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// generic implicit GEMM.  M = B*Ho*Wo, N = Cout, K = KH*KW*Cin (k = (kh*KW+kw)*Cin + c).
// 64x64x16 tile, 256 threads, 4x4 micro-tile, register-prefetch double buffering.
// Requirements: Cin % 4 == 0, pitches % 4 == 0 (vector loads along the channel axis).
// ------------------------------------------------------------------------------------------------

constexpr int BM = 64, BN = 64, BK = 16, PADS = 4;

template <typename TIn, typename TOut>
__global__ void __launch_bounds__(256) conv_igemm_simt(const ConvParams p) {
  __shared__ __align__(16) float As[2][BK][BM + PADS];
  __shared__ __align__(16) float Bs[2][BK][BN + PADS];
  const TIn* __restrict__ x = reinterpret_cast<const TIn*>(p.x);
  const TIn* __restrict__ w = reinterpret_cast<const TIn*>(p.w);
  const int tid = threadIdx.x;
  const int64_t m0 = (int64_t)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  // loader mapping: row = tid/4 (0..63), kq = (tid%4)*4
  const int lrow = tid >> 2, lkq = (tid & 3) * 4;
  const int64_t am = m0 + lrow;
  const bool a_row_ok = am < p.M;
  int ab = 0, aho = 0, awo = 0;
  if (a_row_ok) {
    awo = am % p.Wo;
    aho = (am / p.Wo) % p.Ho;
    ab = am / ((int64_t)p.Wo * p.Ho);
  }
  const int bn = n0 + lrow;
  const bool b_row_ok = bn < p.Cout;
  const TIn* wrow = w + (int64_t)bn * p.K;

  float ra[4], rb[4];
  auto fetch = [&](int kt) {
    const int k = kt * BK + lkq;
#pragma unroll
    for (int j = 0; j < 4; ++j) { ra[j] = 0.f; rb[j] = 0.f; }
    if (k < p.K) {
      if (a_row_ok) {
        const int tap = k / p.Cin, c = k - tap * p.Cin;
        const int kh = tap / p.KW, kw = tap - kh * p.KW;
        const int hi = aho * p.stride - p.pad + kh, wi = awo * p.stride - p.pad + kw;
        if (hi >= 0 && hi < p.H && wi >= 0 && wi < p.W)
          load4(x + (((int64_t)ab * p.H + hi) * p.W + wi) * p.x_pitch + c, ra);
      }
      if (b_row_ok) load4(wrow + k, rb);
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      As[buf][lkq + j][lrow] = ra[j];
      Bs[buf][lkq + j][lrow] = rb[j];
    }
  };

  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int KT = (p.K + BK - 1) / BK;
  fetch(0);
  stash(0);
  __syncthreads();
  for (int kt = 0; kt < KT; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < KT) fetch(kt + 1);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kt + 1 < KT) stash(buf ^ 1);
    __syncthreads();
  }

  // epilogue
  const int n = n0 + tx * 4;
  if (n >= p.Cout) return;
  float sc[4], bi[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const bool ok = n + j < p.Cout;
    sc[j] = (p.scale && ok) ? p.scale[n + j] : 1.f;
    bi[j] = (p.bias && ok) ? p.bias[n + j] : 0.f;
  }
  TOut* out = reinterpret_cast<TOut*>(p.out);
  const TOut* res = reinterpret_cast<const TOut*>(p.res);
  const bool full = (n + 3 < p.Cout) && p.vec_ok;
  const bool post = (p.act & FB200_ACT_RESIDUAL_AFTER) != 0;
  const int64_t hw = (int64_t)p.Ho * p.Wo;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t m = m0 + ty * 4 + i;
    if (m >= p.M) continue;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = acc[i][j] * sc[j] + bi[j];
    const int64_t img = m / hw, o_off = img * p.out_bs + (m - img * hw) * p.out_pitch + n;
    if (full) {
      float r[4] = {0.f, 0.f, 0.f, 0.f};
      if (res) load4(res + m * p.res_pitch + n, r);
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = post ? apply_act(v[j], p.act) + r[j] : apply_act(v[j] + r[j], p.act);
      store4(out + o_off, v);
    } else {
      for (int j = 0; j < 4 && n + j < p.Cout; ++j) {
        const float r = res ? to_f(res[m * p.res_pitch + n + j]) : 0.f;
        out[o_off + j] = from_f<TOut>(post ? apply_act(v[j], p.act) + r : apply_act(v[j] + r, p.act));
      }
    }
  }
}

int conv2d_simt(const ConvParams& p, int x_dtype, int out_dtype, cudaStream_t st) {
  FB_CHECK_ARG(p.Cin % 4 == 0 && p.x_pitch % 4 == 0, "conv2d(simt): Cin (%d) and x_pitch (%d) must be multiples of 4", p.Cin, p.x_pitch);
  dim3 grid((unsigned)cdiv(p.M, BM), (unsigned)cdiv(p.Cout, BN));
  if (x_dtype == FB200_F32 && out_dtype == FB200_F32) conv_igemm_simt<float, float><<<grid, 256, 0, st>>>(p);
  else if (x_dtype == FB200_F16 && out_dtype == FB200_F16) conv_igemm_simt<__half, __half><<<grid, 256, 0, st>>>(p);
  else if (x_dtype == FB200_F16 && out_dtype == FB200_F32) conv_igemm_simt<__half, float><<<grid, 256, 0, st>>>(p);
  else if (x_dtype == FB200_F32 && out_dtype == FB200_F16) conv_igemm_simt<float, __half><<<grid, 256, 0, st>>>(p);
  else { set_error("conv2d: bad dtypes %d/%d", x_dtype, out_dtype); return FB200_ERR_INVALID; }
  FB_CHECK_LAUNCH("conv_igemm_simt");
  return FB200_OK;
}

int conv2d_tc(const ConvParams& p, cudaStream_t st);          // conv_tc.cu
bool conv2d_tc_supported(const ConvParams& p, int x_dtype, int out_dtype);

}  // namespace fb200

using namespace fb200;

extern "C" const char* fb200_last_error(void) { return fb200::g_err; }
extern "C" int fb200_version(void) { return 100; }

static int stem_launch(const void* img, bool u8, int B, int H, int W, const float* w, const float* scale, const float* bias, const float* mean3,
                       const float* std3, int act, void* out, int out_dtype, int Cout, void* stream) {
  FB_CHECK_ARG(img && w && out && mean3 && std3, "stem_conv: null pointer");
  FB_CHECK_ARG(Cout == 32, "stem_conv: only Cout=32 is instantiated (got %d)", Cout);
  FB_CHECK_ARG(B > 0 && H > 0 && W > 0, "stem_conv: bad shape");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  cudaStream_t st = (cudaStream_t)stream;
  const float* m = mean3; const float* s = std3;  // HOST pointers (3 floats each)
  const int tiles_w = (Wo + 15) / 16, tiles_h = (Ho + 15) / 16;
  const unsigned grid = (unsigned)((int64_t)B * tiles_w * tiles_h);
  // uint8 input with ReLU: two pixels per thread; everything else: one pixel per thread
#define STEM_LAUNCH(T, U8)                                                                                                                                              \
  do {                                                                                                                                                                  \
    if (U8 && (act & 15) == FB200_ACT_RELU) {                                                                                                                           \
      if (act & 256) stem_conv_tiled2_kernel<T, true><<<grid, 128, 0, st>>>((const uint8_t*)img, B, H, W, w, scale, bias, m[0], m[1], m[2], s[0], s[1], s[2], (T*)out, tiles_w, tiles_h);   \
      else stem_conv_tiled2_kernel<T, false><<<grid, 128, 0, st>>>((const uint8_t*)img, B, H, W, w, scale, bias, m[0], m[1], m[2], s[0], s[1], s[2], (T*)out, tiles_w, tiles_h);           \
    } else if ((act & 15) == FB200_ACT_RELU) stem_conv_tiled_kernel<T, U8, true><<<grid, 256, 0, st>>>(img, B, H, W, w, scale, bias, m[0], m[1], m[2], s[0], s[1], s[2], act, (T*)out, tiles_w, tiles_h);   \
    else stem_conv_tiled_kernel<T, U8, false><<<grid, 256, 0, st>>>(img, B, H, W, w, scale, bias, m[0], m[1], m[2], s[0], s[1], s[2], act, (T*)out, tiles_w, tiles_h);   \
  } while (0)
  if (out_dtype == FB200_F32) { if (u8) STEM_LAUNCH(float, true); else STEM_LAUNCH(float, false); }
  else if (out_dtype == FB200_F16) { if (u8) STEM_LAUNCH(__half, true); else STEM_LAUNCH(__half, false); }
  else if (out_dtype == FB200_F16PAIR) { act |= 256; if (u8) STEM_LAUNCH(__half, true); else STEM_LAUNCH(__half, false); }  // dense [hi(32) | lo(32)] pair per pixel
  else { set_error("stem_conv: bad dtype"); return FB200_ERR_INVALID; }
#undef STEM_LAUNCH
  FB_CHECK_LAUNCH("stem_conv_kernel");
  return FB200_OK;
}

extern "C" int fb200_stem_conv3x3s2(const float* img, int B, int H, int W, const float* w, const float* scale,
                                    const float* bias, const float* mean3, const float* std3, int act, void* out,
                                    int out_dtype, int Cout, void* stream) {
  return stem_launch(img, false, B, H, W, w, scale, bias, mean3, std3, act, out, out_dtype, Cout, stream);
}
extern "C" int fb200_stem_conv3x3s2_u8(const uint8_t* img_nhwc, int B, int H, int W, const float* w, const float* scale,
                                       const float* bias, const float* mean3, const float* std3, int act, void* out,
                                       int out_dtype, int Cout, void* stream) {
  return stem_launch(img_nhwc, true, B, H, W, w, scale, bias, mean3, std3, act, out, out_dtype, Cout, stream);
}

// The ConvParams of every conv entry point.  x_lo_off != 0: x is the hi plane of a pair with C logical channels and w the [W_hi | W_lo | W_hi] triple,
// so K runs over 3C per tap (the fp32-accurate split products); otherwise Cin = C.  out_batch_stride 0: dense images of Ho x Wo x out_pitch.
static int conv_params(ConvParams* q, const char* who, const void* x, int x_dtype, int B, int H, int W, int C, int x_pitch, int64_t x_lo_off, const void* w,
                       int64_t w_bs, int KH, int KW, int stride, int pad, const float* scale, const float* bias, const void* residual, int res_pitch,
                       int64_t res_lo_off, int act, void* out, int out_dtype, int out_pitch, int64_t out_lo_off, int64_t out_batch_stride, int Cout) {
  FB_CHECK_ARG(x && w && out, "%s: null pointer", who);
  FB_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && Cout > 0 && KH > 0 && KW > 0 && stride > 0 && pad >= 0, "%s: bad shape", who);
  ConvParams& p = *q;
  p.split3 = x_lo_off != 0;
  p.x = x; p.w = w; p.scale = scale; p.bias = bias; p.res = residual; p.out = out;
  p.B = B; p.H = H; p.W = W; p.Cin = p.split3 ? 3 * C : C; p.x_pitch = x_pitch; p.KH = KH; p.KW = KW; p.stride = stride; p.pad = pad;
  p.Ho = (H + 2 * pad - KH) / stride + 1; p.Wo = (W + 2 * pad - KW) / stride + 1;
  FB_CHECK_ARG(p.Ho > 0 && p.Wo > 0, "%s: empty output", who);
  p.Cout = Cout; p.res_pitch = res_pitch; p.out_pitch = out_pitch; p.act = act;
  p.M = (int64_t)B * p.Ho * p.Wo; p.K = KH * KW * p.Cin; p.x_dtype = x_dtype; p.out_dtype = out_dtype;
  p.out_bs = out_batch_stride > 0 ? out_batch_stride : (int64_t)p.Ho * p.Wo * out_pitch;
  p.vec_ok = (out_pitch % 4 == 0) && (!residual || res_pitch % 4 == 0) && (p.out_bs % 4 == 0);  // the SIMT epilogue's 16-byte stores
  p.w_bs = w_bs;
  FB_CHECK_ARG(w_bs == 0 || w_bs >= (int64_t)Cout * p.K, "%s: weight batch stride smaller than one weight set", who);
  FB_CHECK_ARG(w_bs == 0 || !residual, "%s: per-image weights take no residual", who);
  p.x_lo_off = x_lo_off; p.out_lo_off = out_lo_off; p.res_lo_off = res_lo_off;
  return FB200_OK;
}

extern "C" int fb200_conv2d(const void* x, int x_dtype, int B, int H, int W, int Cin, int x_pitch, const void* w, int64_t w_batch_stride, int KH,
                            int KW, int stride, int pad, const float* scale, const float* bias, const void* residual,
                            int res_pitch, int act, void* out, int out_dtype, int out_pitch, int64_t out_batch_stride, int Cout,
                            int algo, void* stream) {
  FB_CHECK_ARG(algo == FB200_ALGO_AUTO || algo == FB200_ALGO_SIMT || algo == FB200_ALGO_TCGEN05,
               "conv2d: unknown algo %d (split-precision products on [hi | lo] pairs are fb200_conv2d_pair)", algo);
  FB_CHECK_ARG(x_pitch >= Cin && out_pitch >= Cout, "conv2d: pitch smaller than channel count");
  ConvParams p;
  if (int rc = conv_params(&p, "conv2d", x, x_dtype, B, H, W, Cin, x_pitch, 0, w, w_batch_stride, KH, KW, stride, pad, scale, bias, residual, res_pitch, 0, act,
                           out, out_dtype, out_pitch, 0, out_batch_stride, Cout))
    return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const bool tc_ok = conv2d_tc_supported(p, x_dtype, out_dtype);
  if (algo == FB200_ALGO_TCGEN05 && !tc_ok) {
    set_error("conv2d: tensor-core path does not support this shape/dtype (Cin=%d Cout=%d k=%dx%d s=%d dtype=%d/%d)", Cin, Cout, KH, KW, stride, x_dtype, out_dtype);
    return FB200_ERR_UNSUPPORTED;
  }
  if ((algo == FB200_ALGO_AUTO && tc_ok) || algo == FB200_ALGO_TCGEN05) return conv2d_tc(p, st);
  if (w_batch_stride != 0) {  // CUDA-core path: one launch per image (the parity mode; the tensor-core path batches them)
    const size_t xe = x_dtype == FB200_F16 ? 2 : 4, oe = out_dtype == FB200_F16 ? 2 : 4;
    ConvParams q = p;
    q.B = 1; q.M = (int64_t)p.Ho * p.Wo; q.w_bs = 0;
    for (int b = 0; b < B; ++b) {
      q.x = static_cast<const char*>(x) + (size_t)b * H * W * x_pitch * xe;
      q.w = static_cast<const char*>(w) + (size_t)b * w_batch_stride * xe;
      q.out = static_cast<char*>(out) + (size_t)b * p.out_bs * oe;
      const int rc = conv2d_simt(q, x_dtype, out_dtype, st);
      if (rc) return rc;
    }
    return FB200_OK;
  }
  return conv2d_simt(p, x_dtype, out_dtype, st);
}

extern "C" int fb200_conv2d_pair(const void* x, int B, int H, int W, int C, int x_pitch, int64_t x_lo_off, const void* w3, int64_t w_batch_stride, int KH, int KW,
                                 int stride, int pad, const float* scale, const float* bias, const void* residual, int res_pitch, int64_t res_lo_off, int act,
                                 void* out, int out_dtype, int out_pitch, int64_t out_lo_off, int64_t out_batch_stride, int Cout, void* stream) {
  FB_CHECK_ARG(out_dtype == FB200_F32 || out_dtype == FB200_F16 || out_dtype == FB200_F16PAIR, "conv2d_pair: bad output dtype %d", out_dtype);
  FB_CHECK_ARG(x_lo_off >= C && x_pitch >= x_lo_off + C, "conv2d_pair: the lo plane must lie inside the pixel pitch, after the hi plane");
  ConvParams p;
  if (int rc = conv_params(&p, "conv2d_pair", x, FB200_F16, B, H, W, C, x_pitch, x_lo_off, w3, w_batch_stride, KH, KW, stride, pad, scale, bias, residual,
                           res_pitch, res_lo_off, act, out, out_dtype, out_pitch, out_lo_off, out_batch_stride, Cout))
    return rc;
  if (!conv2d_tc_supported(p, FB200_F16, out_dtype)) {
    set_error("conv2d_pair: tensor-core path does not support this shape / alignment / output (C=%d Cout=%d k=%dx%d s=%d out_dtype=%d); split-precision convs write fp32 or "
              "the fp16 pair", C, Cout, KH, KW, stride, out_dtype);
    return FB200_ERR_UNSUPPORTED;
  }
  return conv2d_tc(p, (cudaStream_t)stream);
}

// rowmax: a linear over M rows is the 1x1 conv of one [1, 1, M, K] image whose epilogue keeps only the row maxima; `out` is never written, the tensor
// map of the absent output only needs a valid aligned address.
static int linear_rowmax_launch(const char* who, const void* x, int64_t M, int K, int x_pitch, int64_t x_lo_off, const void* w, const float* bias, int Cout,
                                float* rowmax, void* stream) {
  FB_CHECK_ARG(x && w && rowmax && M > 0 && M <= 0x7fffffffLL && K > 0 && Cout > 0, "%s: bad arguments", who);
  ConvParams p;
  if (int rc = conv_params(&p, who, x, FB200_F16, 1, 1, (int)M, K, x_pitch, x_lo_off, w, 0, 1, 1, 1, 0, nullptr, bias, nullptr, 0, 0, FB200_ACT_NONE,
                           const_cast<void*>(x), FB200_F32, (Cout + 3) / 4 * 4, 0, 0, Cout))
    return rc;
  p.rowmax = rowmax;
  if (!conv2d_tc_supported(p, FB200_F16, FB200_F32)) {
    set_error("%s: shape not supported by the tensor-core path (K=%d must be a multiple of 32, fp16 operands, 16-byte aligned)", who, K);
    return FB200_ERR_UNSUPPORTED;
  }
  return conv2d_tc(p, (cudaStream_t)stream);
}

extern "C" int fb200_linear_rowmax(const void* x, int64_t M, int K, int x_pitch, const void* w, const float* bias, int Cout, float* rowmax, void* stream) {
  return linear_rowmax_launch("linear_rowmax", x, M, K, x_pitch, 0, w, bias, Cout, rowmax, stream);
}

extern "C" int fb200_linear_rowmax_pair(const void* x, int64_t M, int K, int x_pitch, int64_t x_lo_off, const void* w3, const float* bias, int Cout, float* rowmax, void* stream) {
  FB_CHECK_ARG(x_lo_off >= K && x_pitch >= x_lo_off + K && K % 64 == 0, "linear_rowmax_pair: K must be a multiple of 64 and the lo plane must lie inside the row pitch");
  return linear_rowmax_launch("linear_rowmax_pair", x, M, K, x_pitch, x_lo_off, w3, bias, Cout, rowmax, stream);
}

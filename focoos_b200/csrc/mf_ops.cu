// MaskFormer-family kernels (SURVEY §8 rows a14-a17): nearest-upsample+add, attention-mask construction, masked
// cross-attention (streaming over keys, online softmax), class softmax, fused sigmoid + bilinear mask upsampling to the
// reference's [B,Q,H,W] layout, and the post-processing reductions over that tensor.
#include <algorithm>

#include "common.cuh"

namespace fb200 {

static inline unsigned grid_cap(int64_t total, int threads) {
  int64_t g = cdiv(total, threads);
  const int64_t cap = (int64_t)kNumSMs * 32;
  return (unsigned)(g < cap ? (g > 0 ? g : 1) : cap);
}

// ---------------------------------------------------------------------------------------------------------------------
// out = cur + nearest_upsample(y)      (fai_mf/modelling.py:364; ATen nearest: src = min(floor(dst * in/out), in-1))
// ---------------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void upsample_nearest_add_kernel(const T* __restrict__ y, const T* __restrict__ cur, T* __restrict__ out, int B, int h, int w,
                                            int H, int W, int C, float sh, float sw) {
  const int cv = C / 4;
  const int64_t total = (int64_t)B * H * W * cv;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (i % cv) * 4;
    const int64_t pix = i / cv;
    const int X = pix % W, Y = (pix / W) % H, b = pix / ((int64_t)W * H);
    const int ys = min((int)floorf((float)Y * sh), h - 1), xs = min((int)floorf((float)X * sw), w - 1);
    float a[4], v[4];
    load4(cur + pix * C + c, a);
    load4(y + (((int64_t)b * h + ys) * w + xs) * C + c, v);
#pragma unroll
    for (int j = 0; j < 4; ++j) a[j] += v[j];
    store4(out + pix * C + c, a);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// mask[b,q,k] = (x[b,k,q] < 0) ; allowed[b,q] = #keys with x >= 0.   32x32 tiled transpose through shared memory.
// ---------------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) attn_mask_build_kernel(const T* __restrict__ x, int Lk, int Qp, int Q, uint8_t* __restrict__ mask,
                                                              int LkP, int* __restrict__ allowed) {
  __shared__ uint8_t tile[32][33];
  const int b = blockIdx.z, k0 = blockIdx.x * 32, q0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int r = ty; r < 32; r += 8) {
    const int k = k0 + r, q = q0 + tx;
    uint8_t m = 1;  // padding keys / queries: not allowed
    if (k < Lk && q < Q) m = to_f(x[((int64_t)b * Lk + k) * Qp + q]) < 0.f ? 1 : 0;
    tile[r][tx] = m;
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int q = q0 + r, k = k0 + tx;
    if (q >= Q) continue;
    const uint8_t m = tile[tx][r];
    if (k < LkP) mask[((int64_t)b * Q + q) * LkP + k] = m;
    const unsigned ok = __ballot_sync(0xffffffffu, (k < Lk) && !m);
    if (tx == 0 && ok) atomicAdd(&allowed[b * Q + q], __popc(ok));
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// masked attention, head_dim 32: one warp per query, 8 queries per CTA, keys streamed through smem in chunks of 128 with an
// online softmax.  mask[b,q,k] != 0 => key not allowed, unless allowed[b,q] == 0 (row fully masked -> attend everywhere,
// fai_mf/modelling.py:510-512).  mask == nullptr => plain attention.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int MA_CHUNK = 128, MA_QPB = 8;
template <typename T>
__global__ void __launch_bounds__(256) attention_masked_kernel(const T* __restrict__ q, int q_pitch, const T* __restrict__ k, int k_pitch,
                                                               const T* __restrict__ v, int v_pitch, const uint8_t* __restrict__ mask, int LkP,
                                                               const int* __restrict__ allowed, T* __restrict__ out, int out_pitch, int Lq,
                                                               int Lk, int heads, float scale) {
  __shared__ float Ks[MA_CHUNK][33];
  __shared__ float Vs[MA_CHUNK][32];
  __shared__ float Ps[MA_QPB][MA_CHUNK];
  __shared__ float Qs[MA_QPB][32];
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qi = blockIdx.y * MA_QPB + warp;
  const bool q_ok = qi < Lq;
  if (q_ok) Qs[warp][lane] = to_f(q[((int64_t)b * Lq + qi) * q_pitch + h * 32 + lane]) * scale;
  const bool use_mask = mask != nullptr && q_ok && allowed[b * Lq + qi] > 0;
  const uint8_t* mrow = mask ? mask + ((int64_t)b * Lq + (q_ok ? qi : 0)) * LkP : nullptr;
  float m_run = -INFINITY, l_run = 0.f, o = 0.f;
  for (int c0 = 0; c0 < Lk; c0 += MA_CHUNK) {
    __syncthreads();  // previous chunk fully consumed
    for (int i = threadIdx.x; i < MA_CHUNK * 8; i += 256) {
      const int r = i >> 3, c = (i & 7) * 4;
      float kv[4] = {0.f, 0.f, 0.f, 0.f}, vv[4] = {0.f, 0.f, 0.f, 0.f};
      if (c0 + r < Lk) {
        load4(k + ((int64_t)b * Lk + c0 + r) * k_pitch + h * 32 + c, kv);
        load4(v + ((int64_t)b * Lk + c0 + r) * v_pitch + h * 32 + c, vv);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) { Ks[r][c + j] = kv[j]; Vs[r][c + j] = vv[j]; }
    }
    __syncthreads();
    if (!q_ok) continue;
    float s[MA_CHUNK / 32];
    float cmax = -INFINITY;
#pragma unroll
    for (int t = 0; t < MA_CHUNK / 32; ++t) {
      const int j = t * 32 + lane, key = c0 + j;
      float acc = 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) acc = fmaf(Qs[warp][d], Ks[j][d], acc);
      const bool dead = key >= Lk || (use_mask && mrow[key] != 0);
      s[t] = dead ? -INFINITY : acc;
      cmax = fmaxf(cmax, s[t]);
    }
    cmax = warp_max(cmax);
    if (cmax == -INFINITY) continue;  // whole chunk masked for this query (warp-uniform)
    const float m_new = fmaxf(m_run, cmax);
    const float alpha = (m_run == -INFINITY) ? 0.f : expf(m_run - m_new);
    float psum = 0.f;
#pragma unroll
    for (int t = 0; t < MA_CHUNK / 32; ++t) {
      const float p = (s[t] == -INFINITY) ? 0.f : expf(s[t] - m_new);
      Ps[warp][t * 32 + lane] = p;
      psum += p;
    }
    psum = warp_sum(psum);
    __syncwarp();
    float acc = 0.f;
#pragma unroll 8
    for (int j = 0; j < MA_CHUNK; ++j) acc = fmaf(Ps[warp][j], Vs[j][lane], acc);
    o = o * alpha + acc;
    l_run = l_run * alpha + psum;
    m_run = m_new;
    __syncwarp();
  }
  if (q_ok) out[((int64_t)b * Lq + qi) * out_pitch + h * 32 + lane] = from_f<T>(o / l_run);
}

// fp32 / fp16 rows (k / v pitches multiples of 4); also the streaming fallback of fb200_attention (mask == nullptr) above the resident kernel's key count
int attention_masked_simt(const void* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, const uint8_t* mask, int LkP, const int* allowed, void* out,
                          int out_pitch, int dtype, int B, int Lq, int Lk, int heads, float scale, cudaStream_t st) {
  dim3 grid((unsigned)(B * heads), (unsigned)cdiv(Lq, MA_QPB));
  FB_DISPATCH_DTYPE(dtype, T, (attention_masked_kernel<T><<<grid, 256, 0, st>>>((const T*)q, q_pitch, (const T*)k, k_pitch, (const T*)v, v_pitch, mask, LkP, allowed, (T*)out, out_pitch, Lq, Lk, heads, scale)));
  FB_CHECK_LAUNCH("attention_masked");
  return FB200_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// out[r, 0..N-2] = softmax(x[r, 0..N-1])[..., :-1]     (one warp per row)
// ---------------------------------------------------------------------------------------------------------------------
__global__ void softmax_drop_last_kernel(const float* __restrict__ x, int64_t rows, int N, int pitch, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* xr = x + row * pitch;
  float m = -INFINITY;
  for (int j = lane; j < N; j += 32) m = fmaxf(m, xr[j]);
  m = warp_max(m);
  float s = 0.f;
  for (int j = lane; j < N; j += 32) s += expf(xr[j] - m);
  s = warp_sum(s);
  for (int j = lane; j < N - 1; j += 32) out[row * (N - 1) + j] = expf(xr[j] - m) / s;
}

// ---------------------------------------------------------------------------------------------------------------------
// probs[b,q,Y,X] = bilinear( sigmoid(x[b,:,:,q]) )  (align_corners=False).  One CTA per 16x64 output tile: the low-resolution
// patch it needs is loaded once for ALL queries (channel-contiguous, coalesced), passed through the sigmoid once per low-res
// element, kept in smem, and every query plane of the tile is then written with coalesced 256-byte rows.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int MU_TH = 16, MU_TW = 64;
// ARGMAX = true: the semantic post-process fused in (fai_mf/processor.py:208-220): instead of writing the [B,Q,H,W] probabilities (13.4 GB at
// 64 x 100 x 512 x 1024) and reading them back, each output pixel keeps argmax_q(score[b,q] * prob) -> uint8 label + per-(b,q) pixel counts.
// The probability is computed by the very same expression, so labels equal mask_argmax(mask_sigmoid_upsample(x)) bit for bit.
template <typename T, bool ARGMAX>
__global__ void __launch_bounds__(256) mask_sigmoid_upsample_kernel(const T* __restrict__ x, int h, int w, int Qp, int Q, float* __restrict__ out,
                                                                    int H, int W, float sh, float sw, int ph_max, int pw_max,
                                                                    const float* __restrict__ scores, uint8_t* __restrict__ labels, int* __restrict__ counts) {
  extern __shared__ float patch[];  // [ph][pw][Q] (+ ARGMAX: [Q] scores, [Q] int histogram behind the largest possible patch)
  float* s_sc = patch + (size_t)ph_max * pw_max * Q;
  int* s_hist = reinterpret_cast<int*>(s_sc + Q);
  if (ARGMAX)
    for (int i = threadIdx.x; i < Q; i += 256) { s_sc[i] = scores[blockIdx.z * Q + i]; s_hist[i] = 0; }
  const int b = blockIdx.z, oy0 = blockIdx.y * MU_TH, ox0 = blockIdx.x * MU_TW;
  const int oy1 = min(oy0 + MU_TH, H) - 1, ox1 = min(ox0 + MU_TW, W) - 1;
  const int ys0 = (int)fmaxf(((float)oy0 + 0.5f) * sh - 0.5f, 0.f), xs0 = (int)fmaxf(((float)ox0 + 0.5f) * sw - 0.5f, 0.f);
  const int ys1 = min((int)fmaxf(((float)oy1 + 0.5f) * sh - 0.5f, 0.f) + 1, h - 1), xs1 = min((int)fmaxf(((float)ox1 + 0.5f) * sw - 0.5f, 0.f) + 1, w - 1);
  const int ph = ys1 - ys0 + 1, pw = xs1 - xs0 + 1;  // <= ph_max, pw_max by construction
  for (int i = threadIdx.x; i < ph * pw * Q; i += 256) {
    const int qq = i % Q, pp = i / Q, px = pp % pw, py = pp / pw;
    const float v = to_f(x[(((int64_t)b * h + ys0 + py) * w + xs0 + px) * Qp + qq]);
    patch[i] = 1.f / (1.f + expf(-v));
  }
  __syncthreads();
  // 4 output pixels per thread: (row r0 + 4*i, column tx)
  const int tx = threadIdx.x & 63, r0 = threadIdx.x >> 6;
  int o00[4], o01[4], o10[4], o11[4];
  float wy[4], wx;
  const int X = ox0 + tx;
  const bool x_ok = X < W;
  {
    const float fx = fmaxf(((float)X + 0.5f) * sw - 0.5f, 0.f);
    const int x0 = min((int)fx, w - 1), x1 = min(x0 + 1, w - 1);
    wx = fx - (float)x0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int Y = oy0 + r0 + 4 * i;
      const float fy = fmaxf(((float)min(Y, H - 1) + 0.5f) * sh - 0.5f, 0.f);
      const int y0 = min((int)fy, h - 1), y1 = min(y0 + 1, h - 1);
      wy[i] = fy - (float)y0;
      o00[i] = ((y0 - ys0) * pw + (x0 - xs0)) * Q; o01[i] = ((y0 - ys0) * pw + (x1 - xs0)) * Q;
      o10[i] = ((y1 - ys0) * pw + (x0 - xs0)) * Q; o11[i] = ((y1 - ys0) * pw + (x1 - xs0)) * Q;
    }
  }
  if (!ARGMAX && !x_ok) return;
  float best[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
  int bi[4] = {0, 0, 0, 0};
  if (x_ok && ARGMAX && (Q & 3) == 0) {
    // four queries per shared-memory load (the patch is query-contiguous and every tap offset is a multiple of Q): the fused kernel is
    // bound by shared-memory bandwidth, not HBM
    for (int qq = 0; qq < Q; qq += 4) {
      const float4 sq = *reinterpret_cast<const float4*>(s_sc + qq);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int Y = oy0 + r0 + 4 * i;
        if (Y >= H) continue;
        const float4 v00 = *reinterpret_cast<const float4*>(patch + o00[i] + qq), v01 = *reinterpret_cast<const float4*>(patch + o01[i] + qq);
        const float4 v10 = *reinterpret_cast<const float4*>(patch + o10[i] + qq), v11 = *reinterpret_cast<const float4*>(patch + o11[i] + qq);
        const float lw1 = wx, lw0 = 1.f - wx, lh1 = wy[i], lh0 = 1.f - wy[i];
        const float p0 = lh0 * (lw0 * v00.x + lw1 * v01.x) + lh1 * (lw0 * v10.x + lw1 * v11.x);
        const float p1 = lh0 * (lw0 * v00.y + lw1 * v01.y) + lh1 * (lw0 * v10.y + lw1 * v11.y);
        const float p2 = lh0 * (lw0 * v00.z + lw1 * v01.z) + lh1 * (lw0 * v10.z + lw1 * v11.z);
        const float p3 = lh0 * (lw0 * v00.w + lw1 * v01.w) + lh1 * (lw0 * v10.w + lw1 * v11.w);
        float v = sq.x * p0; if (v > best[i]) { best[i] = v; bi[i] = qq; }
        v = sq.y * p1; if (v > best[i]) { best[i] = v; bi[i] = qq + 1; }
        v = sq.z * p2; if (v > best[i]) { best[i] = v; bi[i] = qq + 2; }
        v = sq.w * p3; if (v > best[i]) { best[i] = v; bi[i] = qq + 3; }
      }
    }
  } else if (x_ok) {
    for (int qq = 0; qq < Q; ++qq) {
      float* op = ARGMAX ? nullptr : out + (((int64_t)b * Q + qq) * H) * W;
      const float sq = ARGMAX ? s_sc[qq] : 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int Y = oy0 + r0 + 4 * i;
        if (Y >= H) continue;
        const float v00 = patch[o00[i] + qq], v01 = patch[o01[i] + qq], v10 = patch[o10[i] + qq], v11 = patch[o11[i] + qq];
        const float lw1 = wx, lw0 = 1.f - wx, lh1 = wy[i], lh0 = 1.f - wy[i];
        const float pr = lh0 * (lw0 * v00 + lw1 * v01) + lh1 * (lw0 * v10 + lw1 * v11);
        if (ARGMAX) {
          const float v = sq * pr;
          if (v > best[i]) { best[i] = v; bi[i] = qq; }
        } else {
          op[(int64_t)Y * W + X] = pr;
        }
      }
    }
  }
  if (ARGMAX) {
    if (x_ok) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int Y = oy0 + r0 + 4 * i;
        if (Y >= H) continue;
        labels[((int64_t)b * H + Y) * W + X] = (uint8_t)bi[i];
        atomicAdd(&s_hist[bi[i]], 1);
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < Q; i += 256)
      if (s_hist[i]) atomicAdd(&counts[b * Q + i], s_hist[i]);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Instance post-process fused into the upsampling (fai_mf/processor.py:222-257 on top of modelling.py:619,722-723): per (b,q) the number of pixels with
// prob >= thr and their probability mass, straight from the low-resolution logits - the [B,Q,H,W] tensor (4.1 GB at 16 x 100 x 800 x 800) is never written
// or re-read.  Same tiling and the same probability expression as mask_sigmoid_upsample_kernel; counts are exact, the mass is summed with float atomics
// (order not fixed: ~1e-7 relative).
template <typename T>
__global__ void __launch_bounds__(256) mask_upsample_stats_kernel(const T* __restrict__ x, int h, int w, int Qp, int Q, int H, int W, float sh, float sw, int ph_max,
                                                                  int pw_max, float thr, int* __restrict__ count, float* __restrict__ psum) {
  extern __shared__ float patch[];  // [ph][pw][Q], then [Q] float mass, [Q] int count
  float* s_sum = patch + (size_t)ph_max * pw_max * Q;
  int* s_cnt = reinterpret_cast<int*>(s_sum + Q);
  const int b = blockIdx.z, oy0 = blockIdx.y * MU_TH, ox0 = blockIdx.x * MU_TW;
  const int oy1 = min(oy0 + MU_TH, H) - 1, ox1 = min(ox0 + MU_TW, W) - 1;
  const int ys0 = (int)fmaxf(((float)oy0 + 0.5f) * sh - 0.5f, 0.f), xs0 = (int)fmaxf(((float)ox0 + 0.5f) * sw - 0.5f, 0.f);
  const int ys1 = min((int)fmaxf(((float)oy1 + 0.5f) * sh - 0.5f, 0.f) + 1, h - 1), xs1 = min((int)fmaxf(((float)ox1 + 0.5f) * sw - 0.5f, 0.f) + 1, w - 1);
  const int ph = ys1 - ys0 + 1, pw = xs1 - xs0 + 1;
  for (int i = threadIdx.x; i < Q; i += 256) { s_sum[i] = 0.f; s_cnt[i] = 0; }
  for (int i = threadIdx.x; i < ph * pw * Q; i += 256) {
    const int qq = i % Q, pp = i / Q, px = pp % pw, py = pp / pw;
    const float v = to_f(x[(((int64_t)b * h + ys0 + py) * w + xs0 + px) * Qp + qq]);
    patch[i] = 1.f / (1.f + expf(-v));
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  if ((Q & 3) == 0 && Q <= 128) {
    // thread = (query quad qg, pixel group pgp): four queries per 16-byte shared-memory load, counts / mass for its quad kept in registers over the
    // tile's pixels - no per-query warp reductions, 4x fewer shared-memory instructions than the pixel-per-thread mapping
    const int nq4 = Q >> 2, ngroups = 256 / nq4;
    const int qg = threadIdx.x % nq4, pgp = threadIdx.x / nq4;
    if (pgp < ngroups) {
      int c[4] = {0, 0, 0, 0};
      float m[4] = {0.f, 0.f, 0.f, 0.f};
      const int tw = min(MU_TW, W - ox0), th = min(MU_TH, H - oy0);
      for (int p = pgp; p < tw * th; p += ngroups) {
        const int py = p / tw, px = p - py * tw;
        const float fx = fmaxf(((float)(ox0 + px) + 0.5f) * sw - 0.5f, 0.f), fy = fmaxf(((float)(oy0 + py) + 0.5f) * sh - 0.5f, 0.f);
        const int x0 = min((int)fx, w - 1), x1 = min(x0 + 1, w - 1), y0 = min((int)fy, h - 1), y1 = min(y0 + 1, h - 1);
        const float lw1 = fx - (float)x0, lw0 = 1.f - lw1, lh1 = fy - (float)y0, lh0 = 1.f - lh1;
        const float4 v00 = *reinterpret_cast<const float4*>(patch + ((y0 - ys0) * pw + (x0 - xs0)) * Q + qg * 4);
        const float4 v01 = *reinterpret_cast<const float4*>(patch + ((y0 - ys0) * pw + (x1 - xs0)) * Q + qg * 4);
        const float4 v10 = *reinterpret_cast<const float4*>(patch + ((y1 - ys0) * pw + (x0 - xs0)) * Q + qg * 4);
        const float4 v11 = *reinterpret_cast<const float4*>(patch + ((y1 - ys0) * pw + (x1 - xs0)) * Q + qg * 4);
        const float pr[4] = {lh0 * (lw0 * v00.x + lw1 * v01.x) + lh1 * (lw0 * v10.x + lw1 * v11.x), lh0 * (lw0 * v00.y + lw1 * v01.y) + lh1 * (lw0 * v10.y + lw1 * v11.y),
                             lh0 * (lw0 * v00.z + lw1 * v01.z) + lh1 * (lw0 * v10.z + lw1 * v11.z), lh0 * (lw0 * v00.w + lw1 * v01.w) + lh1 * (lw0 * v10.w + lw1 * v11.w)};
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (pr[k] >= thr) { ++c[k]; m[k] += pr[k]; }
      }
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (c[k]) { atomicAdd(&s_cnt[qg * 4 + k], c[k]); atomicAdd(&s_sum[qg * 4 + k], m[k]); }
    }
  } else {
  const int tx = threadIdx.x & 63, r0 = threadIdx.x >> 6;
  int o00[4], o01[4], o10[4], o11[4];
  float wy[4], wx;
  bool ok[4];
  const int X = ox0 + tx;
  {
    const float fx = fmaxf(((float)min(X, W - 1) + 0.5f) * sw - 0.5f, 0.f);
    const int x0 = min((int)fx, w - 1), x1 = min(x0 + 1, w - 1);
    wx = fx - (float)x0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int Y = oy0 + r0 + 4 * i;
      ok[i] = X < W && Y < H;
      const float fy = fmaxf(((float)min(Y, H - 1) + 0.5f) * sh - 0.5f, 0.f);
      const int y0 = min((int)fy, h - 1), y1 = min(y0 + 1, h - 1);
      wy[i] = fy - (float)y0;
      o00[i] = ((y0 - ys0) * pw + (x0 - xs0)) * Q; o01[i] = ((y0 - ys0) * pw + (x1 - xs0)) * Q;
      o10[i] = ((y1 - ys0) * pw + (x0 - xs0)) * Q; o11[i] = ((y1 - ys0) * pw + (x1 - xs0)) * Q;
    }
  }
  for (int qq = 0; qq < Q; ++qq) {
    int c = 0;
    float m = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float v00 = patch[o00[i] + qq], v01 = patch[o01[i] + qq], v10 = patch[o10[i] + qq], v11 = patch[o11[i] + qq];
      const float lw1 = wx, lw0 = 1.f - wx, lh1 = wy[i], lh0 = 1.f - wy[i];
      const float pr = lh0 * (lw0 * v00 + lw1 * v01) + lh1 * (lw0 * v10 + lw1 * v11);
      if (ok[i] && pr >= thr) { ++c; m += pr; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { c += __shfl_xor_sync(0xffffffffu, c, o); m += __shfl_xor_sync(0xffffffffu, m, o); }
    if (lane == 0 && c) { atomicAdd(&s_cnt[qq], c); atomicAdd(&s_sum[qq], m); }
  }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < Q; i += 256)
    if (s_cnt[i]) { atomicAdd(&count[b * Q + i], s_cnt[i]); atomicAdd(&psum[b * Q + i], s_sum[i]); }
}

// out[i] = bilinear(sigmoid(x[b_i, :, :, q_i])) for the n kept (b,q) pairs only: [n,H,W] fp32, same expression as the full upsampling
template <typename T>
__global__ void __launch_bounds__(256) mask_upsample_select_kernel(const T* __restrict__ x, int h, int w, int Qp, const int* __restrict__ bq, float* __restrict__ out,
                                                                   int H, int W, float sh, float sw) {
  extern __shared__ float patch[];  // [ph][pw]
  const int i_ = blockIdx.z, b = bq[i_ * 2], q = bq[i_ * 2 + 1];
  const int oy0 = blockIdx.y * MU_TH, ox0 = blockIdx.x * MU_TW;
  const int oy1 = min(oy0 + MU_TH, H) - 1, ox1 = min(ox0 + MU_TW, W) - 1;
  const int ys0 = (int)fmaxf(((float)oy0 + 0.5f) * sh - 0.5f, 0.f), xs0 = (int)fmaxf(((float)ox0 + 0.5f) * sw - 0.5f, 0.f);
  const int ys1 = min((int)fmaxf(((float)oy1 + 0.5f) * sh - 0.5f, 0.f) + 1, h - 1), xs1 = min((int)fmaxf(((float)ox1 + 0.5f) * sw - 0.5f, 0.f) + 1, w - 1);
  const int ph = ys1 - ys0 + 1, pw = xs1 - xs0 + 1;
  for (int i = threadIdx.x; i < ph * pw; i += 256) {
    const int px = i % pw, py = i / pw;
    const float v = to_f(x[(((int64_t)b * h + ys0 + py) * w + xs0 + px) * Qp + q]);
    patch[i] = 1.f / (1.f + expf(-v));
  }
  __syncthreads();
  const int tx = threadIdx.x & 63, r0 = threadIdx.x >> 6;
  const int X = ox0 + tx;
  if (X >= W) return;
  const float fx = fmaxf(((float)X + 0.5f) * sw - 0.5f, 0.f);
  const int x0 = min((int)fx, w - 1), x1 = min(x0 + 1, w - 1);
  const float wx = fx - (float)x0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int Y = oy0 + r0 + 4 * i;
    if (Y >= H) continue;
    const float fy = fmaxf(((float)Y + 0.5f) * sh - 0.5f, 0.f);
    const int y0 = min((int)fy, h - 1), y1 = min(y0 + 1, h - 1);
    const float wyv = fy - (float)y0;
    const float v00 = patch[(y0 - ys0) * pw + (x0 - xs0)], v01 = patch[(y0 - ys0) * pw + (x1 - xs0)];
    const float v10 = patch[(y1 - ys0) * pw + (x0 - xs0)], v11 = patch[(y1 - ys0) * pw + (x1 - xs0)];
    const float lw1 = wx, lw0 = 1.f - wx, lh1 = wyv, lh0 = 1.f - wyv;
    out[((int64_t)i_ * H + Y) * W + X] = lh0 * (lw0 * v00 + lw1 * v01) + lh1 * (lw0 * v10 + lw1 * v11);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// per plane: count(p >= thr), sum(p * [p >= thr])
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) mask_stats_kernel(const float* __restrict__ masks, int64_t hw, float thr, int* __restrict__ count,
                                                         float* __restrict__ psum) {
  const float* p = masks + (int64_t)blockIdx.x * hw;
  int c = 0;
  float s = 0.f;
  const int64_t n4 = (hw & 3) ? 0 : hw / 4;  // planes are only 16-byte aligned when hw % 4 == 0; otherwise the scalar loop below covers everything
  for (int64_t i = threadIdx.x; i < n4; i += 256) {
    const float4 v = reinterpret_cast<const float4*>(p)[i];
    if (v.x >= thr) { ++c; s += v.x; }
    if (v.y >= thr) { ++c; s += v.y; }
    if (v.z >= thr) { ++c; s += v.z; }
    if (v.w >= thr) { ++c; s += v.w; }
  }
  for (int64_t i = n4 * 4 + threadIdx.x; i < hw; i += 256) {
    const float v = p[i];
    if (v >= thr) { ++c; s += v; }
  }
  __shared__ int sc[8];
  __shared__ float ss[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { c += __shfl_xor_sync(0xffffffffu, c, o); s += __shfl_xor_sync(0xffffffffu, s, o); }
  if ((threadIdx.x & 31) == 0) { sc[threadIdx.x >> 5] = c; ss[threadIdx.x >> 5] = s; }
  __syncthreads();
  if (threadIdx.x == 0) {
    int tc = 0; float ts = 0.f;
    for (int i = 0; i < 8; ++i) { tc += sc[i]; ts += ss[i]; }
    count[blockIdx.x] = tc;
    psum[blockIdx.x] = ts;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// kept (b,q): bin = (p >= thr) -> bilinear resize to (Ho,Wo) -> > 0 -> uint8 mask + xyxy bbox (masks_to_xyxy)
// ---------------------------------------------------------------------------------------------------------------------
__global__ void bbox_init_kernel(int* bbox, int n, int Wo, int Ho) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { bbox[i * 4 + 0] = Wo; bbox[i * 4 + 1] = Ho; bbox[i * 4 + 2] = -1; bbox[i * 4 + 3] = -1; }
}
__global__ void bbox_finish_kernel(int* bbox, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && bbox[i * 4 + 2] < 0) { bbox[i * 4 + 0] = 0; bbox[i * 4 + 1] = 0; bbox[i * 4 + 2] = 0; bbox[i * 4 + 3] = 0; }
}
__global__ void __launch_bounds__(256) mask_resize_bbox_kernel(const float* __restrict__ masks, int Q, int H, int W, const int* __restrict__ bq,
                                                               float thr, uint8_t* __restrict__ out, int Ho, int Wo, float sh, float sw,
                                                               int* __restrict__ bbox) {
  const int i = blockIdx.y;
  const float* p = masks + ((int64_t)bq[i * 2] * Q + bq[i * 2 + 1]) * H * W;
  int xmin = Wo, ymin = Ho, xmax = -1, ymax = -1;
  for (int64_t o = (int64_t)blockIdx.x * 256 + threadIdx.x; o < (int64_t)Ho * Wo; o += (int64_t)gridDim.x * 256) {
    const int X = o % Wo, Y = o / Wo;
    const float fy = fmaxf(((float)Y + 0.5f) * sh - 0.5f, 0.f), fx = fmaxf(((float)X + 0.5f) * sw - 0.5f, 0.f);
    const int y0 = min((int)fy, H - 1), x0 = min((int)fx, W - 1), y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
    const float ly = fy - (float)y0, lx = fx - (float)x0;
    const float b00 = p[(int64_t)y0 * W + x0] >= thr ? 1.f : 0.f, b01 = p[(int64_t)y0 * W + x1] >= thr ? 1.f : 0.f;
    const float b10 = p[(int64_t)y1 * W + x0] >= thr ? 1.f : 0.f, b11 = p[(int64_t)y1 * W + x1] >= thr ? 1.f : 0.f;
    const float r = (1.f - ly) * ((1.f - lx) * b00 + lx * b01) + ly * ((1.f - lx) * b10 + lx * b11);
    const bool on = r != 0.f;  // .bool() of the resized float mask
    out[(int64_t)i * Ho * Wo + o] = on ? 1 : 0;
    if (on) { xmin = min(xmin, X); xmax = max(xmax, X); ymin = min(ymin, Y); ymax = max(ymax, Y); }
  }
  if (xmax >= 0) {
    atomicMin(&bbox[i * 4 + 0], xmin); atomicMin(&bbox[i * 4 + 1], ymin);
    atomicMax(&bbox[i * 4 + 2], xmax); atomicMax(&bbox[i * 4 + 3], ymax);
  }
}

int attention_mma_stream(const __half* q, int q_pitch, const __half* k, int k_pitch, const __half* v, int v_pitch, const uint8_t* mask, int LkP,
                         const int* allowed, __half* out, int out_pitch, int B, int Lq, int Lk, int heads, float scale, cudaStream_t st);
}  // namespace fb200
using namespace fb200;

extern "C" int fb200_upsample_nearest_add(const void* y, const void* cur, void* out, int dtype, int B, int h, int w, int H, int W, int C, void* stream) {
  FB_CHECK_ARG(y && cur && out && C % 4 == 0 && h > 0 && w > 0 && H > 0 && W > 0, "upsample_nearest_add: bad arguments");
  const int64_t total = (int64_t)B * H * W * (C / 4);
  FB_DISPATCH_DTYPE(dtype, T, (upsample_nearest_add_kernel<T><<<grid_cap(total, 256), 256, 0, (cudaStream_t)stream>>>((const T*)y, (const T*)cur, (T*)out, B, h, w, H, W, C, (float)h / (float)H, (float)w / (float)W)));
  FB_CHECK_LAUNCH("upsample_nearest_add");
  return FB200_OK;
}

extern "C" int fb200_attn_mask_build(const void* x, int dtype, int B, int Lk, int Qp, int Q, uint8_t* mask, int LkP, int* allowed, void* stream) {
  FB_CHECK_ARG(x && mask && allowed && Q <= Qp && LkP >= Lk, "attn_mask_build: bad arguments");
  dim3 grid((unsigned)cdiv(LkP, 32), (unsigned)cdiv(Q, 32), (unsigned)B);
  FB_DISPATCH_DTYPE(dtype, T, (attn_mask_build_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>((const T*)x, Lk, Qp, Q, mask, LkP, allowed)));
  FB_CHECK_LAUNCH("attn_mask_build");
  return FB200_OK;
}

extern "C" int fb200_attention_masked(const void* q, int q_pitch, const void* k, int k_pitch, const void* v, int v_pitch, const uint8_t* mask, int LkP,
                                      const int* allowed, void* out, int out_pitch, int dtype, int B, int Lq, int Lk, int heads, int head_dim, float scale,
                                      void* stream) {
  FB_CHECK_ARG(q && k && v && out && head_dim == 32, "attention_masked: null pointer or head_dim != 32");
  FB_CHECK_ARG((mask == nullptr) == (allowed == nullptr), "attention_masked: mask and allowed go together");
  FB_CHECK_ARG(B > 0 && Lq > 0 && Lk > 0 && heads > 0, "attention_masked: B, Lq, Lk and heads must be positive (got %d, %d, %d, %d)", B, Lq, Lk, heads);
  FB_CHECK_ARG(k_pitch % 4 == 0 && v_pitch % 4 == 0, "attention_masked: k/v pitches must be multiples of 4");
  const int w = heads * 32;  // a pitch below the row width would make neighbouring rows overlap
  FB_CHECK_ARG(q_pitch >= w, "attention_masked: q_pitch (%d) < heads*32 (%d)", q_pitch, w);
  FB_CHECK_ARG(k_pitch >= w, "attention_masked: k_pitch (%d) < heads*32 (%d)", k_pitch, w);
  FB_CHECK_ARG(v_pitch >= w, "attention_masked: v_pitch (%d) < heads*32 (%d)", v_pitch, w);
  FB_CHECK_ARG(out_pitch >= w, "attention_masked: out_pitch (%d) < heads*32 (%d)", out_pitch, w);
  FB_CHECK_ARG(mask == nullptr || LkP >= Lk, "attention_masked: LkP (%d) < Lk (%d): every key needs a mask byte", LkP, Lk);
  if (dtype == FB200_F16 && q_pitch % 8 == 0 && k_pitch % 8 == 0 && v_pitch % 8 == 0 && out_pitch % 2 == 0 && (mask == nullptr || LkP % 4 == 0) &&
      (((uintptr_t)q | (uintptr_t)k | (uintptr_t)v) & 15) == 0 && ((uintptr_t)out & 3) == 0)  // tensor-core path (norm_attn.cu)
    return attention_mma_stream((const __half*)q, q_pitch, (const __half*)k, k_pitch, (const __half*)v, v_pitch, mask, LkP, allowed, (__half*)out, out_pitch,
                                B, Lq, Lk, heads, scale, (cudaStream_t)stream);
  return attention_masked_simt(q, q_pitch, k, k_pitch, v, v_pitch, mask, LkP, allowed, out, out_pitch, dtype, B, Lq, Lk, heads, scale, (cudaStream_t)stream);
}

extern "C" int fb200_softmax_drop_last(const float* x, int64_t rows, int N, int pitch, float* out, void* stream) {
  FB_CHECK_ARG(x && out && N >= 2 && pitch >= N, "softmax_drop_last: bad arguments");
  softmax_drop_last_kernel<<<(unsigned)cdiv(rows, 8), 256, 0, (cudaStream_t)stream>>>(x, rows, N, pitch, out);
  FB_CHECK_LAUNCH("softmax_drop_last");
  return FB200_OK;
}

static int mask_upsample_launch(const void* x, int dtype, int B, int h, int w, int Qp, int Q, float* out, int H, int W, const float* scores, uint8_t* labels,
                                int* counts, void* stream) {
  const bool argmax = labels != nullptr;
  const float sh = (float)h / (float)H, sw = (float)w / (float)W;
  const int ph = (int)(MU_TH * sh) + 3, pw = (int)(MU_TW * sw) + 3;
  const size_t smem = (size_t)ph * pw * Q * sizeof(float) + (argmax ? (size_t)Q * 8 : 0);
  FB_CHECK_ARG(smem <= 200 * 1024, "mask_sigmoid_upsample: low-resolution patch does not fit shared memory (%zu B)", smem);
  dim3 grid((unsigned)cdiv(W, MU_TW), (unsigned)cdiv(H, MU_TH), (unsigned)B);
  cudaStream_t st = (cudaStream_t)stream;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(mask_sigmoid_upsample_kernel<float, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(mask_sigmoid_upsample_kernel<__half, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(mask_sigmoid_upsample_kernel<float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(mask_sigmoid_upsample_kernel<__half, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    configured = true;
  }
  if (argmax) {
    cudaMemsetAsync(counts, 0, (size_t)B * Q * sizeof(int), st);
    FB_DISPATCH_DTYPE(dtype, T, (mask_sigmoid_upsample_kernel<T, true><<<grid, 256, smem, st>>>((const T*)x, h, w, Qp, Q, nullptr, H, W, sh, sw, ph, pw, scores, labels, counts)));
  } else {
    FB_DISPATCH_DTYPE(dtype, T, (mask_sigmoid_upsample_kernel<T, false><<<grid, 256, smem, st>>>((const T*)x, h, w, Qp, Q, out, H, W, sh, sw, ph, pw, nullptr, nullptr, nullptr)));
  }
  FB_CHECK_LAUNCH("mask_sigmoid_upsample");
  return FB200_OK;
}

extern "C" int fb200_mask_sigmoid_upsample(const void* x, int dtype, int B, int h, int w, int Qp, int Q, float* out, int H, int W, void* stream) {
  FB_CHECK_ARG(x && out && Q <= Qp && H >= h && W >= w, "mask_sigmoid_upsample: bad arguments (upsampling only)");
  return mask_upsample_launch(x, dtype, B, h, w, Qp, Q, out, H, W, nullptr, nullptr, nullptr, stream);
}

extern "C" int fb200_mask_sigmoid_upsample_argmax(const void* x, int dtype, int B, int h, int w, int Qp, int Q, const float* scores, int H, int W, uint8_t* labels,
                                                  int* counts, void* stream) {
  FB_CHECK_ARG(x && scores && labels && counts && Q <= Qp && Q <= 255 && H >= h && W >= w, "mask_sigmoid_upsample_argmax: bad arguments (upsampling only, Q <= 255)");
  return mask_upsample_launch(x, dtype, B, h, w, Qp, Q, nullptr, H, W, scores, labels, counts, stream);
}

extern "C" int fb200_mask_sigmoid_upsample_stats(const void* x, int dtype, int B, int h, int w, int Qp, int Q, int H, int W, float thr, int* count, float* psum,
                                                 void* stream) {
  FB_CHECK_ARG(x && count && psum && Q <= Qp && H >= h && W >= w, "mask_sigmoid_upsample_stats: bad arguments (upsampling only)");
  const float sh = (float)h / (float)H, sw = (float)w / (float)W;
  const int ph = (int)(MU_TH * sh) + 3, pw = (int)(MU_TW * sw) + 3;
  const size_t smem = (size_t)ph * pw * Q * sizeof(float) + (size_t)Q * 8;
  FB_CHECK_ARG(smem <= 200 * 1024, "mask_sigmoid_upsample_stats: low-resolution patch does not fit shared memory (%zu B)", smem);
  cudaStream_t st = (cudaStream_t)stream;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(mask_upsample_stats_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(mask_upsample_stats_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    configured = true;
  }
  cudaMemsetAsync(count, 0, (size_t)B * Q * sizeof(int), st);
  cudaMemsetAsync(psum, 0, (size_t)B * Q * sizeof(float), st);
  dim3 grid((unsigned)cdiv(W, MU_TW), (unsigned)cdiv(H, MU_TH), (unsigned)B);
  FB_DISPATCH_DTYPE(dtype, T, (mask_upsample_stats_kernel<T><<<grid, 256, smem, st>>>((const T*)x, h, w, Qp, Q, H, W, sh, sw, ph, pw, thr, count, psum)));
  FB_CHECK_LAUNCH("mask_sigmoid_upsample_stats");
  return FB200_OK;
}

extern "C" int fb200_mask_sigmoid_upsample_select(const void* x, int dtype, int h, int w, int Qp, const int* bq, int n, float* out, int H, int W, void* stream) {
  FB_CHECK_ARG(x && bq && out && n > 0 && H >= h && W >= w, "mask_sigmoid_upsample_select: bad arguments (upsampling only)");
  const float sh = (float)h / (float)H, sw = (float)w / (float)W;
  const int ph = (int)(MU_TH * sh) + 3, pw = (int)(MU_TW * sw) + 3;
  dim3 grid((unsigned)cdiv(W, MU_TW), (unsigned)cdiv(H, MU_TH), (unsigned)n);
  FB_DISPATCH_DTYPE(dtype, T, (mask_upsample_select_kernel<T><<<grid, 256, (size_t)ph * pw * sizeof(float), (cudaStream_t)stream>>>((const T*)x, h, w, Qp, bq, out, H, W, sh, sw)));
  FB_CHECK_LAUNCH("mask_sigmoid_upsample_select");
  return FB200_OK;
}

extern "C" int fb200_mask_stats(const float* masks, int64_t planes, int64_t hw, float thr, int* count, float* psum, void* stream) {
  FB_CHECK_ARG(masks && count && psum && planes > 0 && hw > 0, "mask_stats: bad arguments");
  mask_stats_kernel<<<(unsigned)planes, 256, 0, (cudaStream_t)stream>>>(masks, hw, thr, count, psum);
  FB_CHECK_LAUNCH("mask_stats");
  return FB200_OK;
}

extern "C" int fb200_mask_resize_bbox(const float* masks, int Q, int H, int W, const int* bq, int n, float thr, uint8_t* out, int Ho, int Wo, int* bbox,
                                      void* stream) {
  FB_CHECK_ARG(masks && bq && out && bbox && n > 0 && Ho > 0 && Wo > 0, "mask_resize_bbox: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  bbox_init_kernel<<<(unsigned)cdiv(n, 128), 128, 0, st>>>(bbox, n, Wo, Ho);
  dim3 grid((unsigned)std::min<int64_t>(cdiv((int64_t)Ho * Wo, 256), 64), (unsigned)n);
  mask_resize_bbox_kernel<<<grid, 256, 0, st>>>(masks, Q, H, W, bq, thr, out, Ho, Wo, (float)H / (float)Ho, (float)W / (float)Wo, bbox);
  bbox_finish_kernel<<<(unsigned)cdiv(n, 128), 128, 0, st>>>(bbox, n);
  FB_CHECK_LAUNCH("mask_resize_bbox");
  return FB200_OK;
}

// Backward of the two attention cores of the decoder/encoder (SURVEY §8 a21, what autograd runs for nn.MultiheadAttention and
// ms_deform_attn_core_pytorch when the reference fine-tunes): fp32, recomputation instead of stored probabilities.
//
//   attention_bwd   softmax(Q K^T s) V per (batch, head), L <= ~400 tokens, head_dim 32: Q,K,V,dO of one (b,h) resident in shared
//                   memory; phase 1 (thread per query) row log-sum-exp, D = rowsum(dO*O), dQ; phase 2 (thread per key) dK, dV.
//                   No atomics: every output element has exactly one writer, sums run in a fixed order.
//   msda_bwd        adjoint of msda_kernel (msda.cu): one warp per (batch, query, head), lane = channel; d(value) by 32-lane
//                   coalesced red.add (fp32 atomics: summation order not fixed), d(offsets) / d(attention logits) by warp reductions,
//                   softmax backward fused.  Reference points carry no gradient (detached at modelling.py:1018, :1228).
#include "common.cuh"

namespace fb200 {
namespace {

constexpr int HD = 32;
// HDP (template parameter of attention_bwd_kernel) = 36: row pitch a multiple of 4 floats so the inner loops read the (broadcast) rows as float4 - one shared-memory load per four FMAs
// (with the 33-float pitch every FMA needed its own LDS and the kernel ran at the shared-memory pipe's rate: 545 us per call)

// 33 = the conflict-free scalar pitch, kept for sequences whose four planes do not fit shared memory at 36 (the 400-token AIFI layer at 640x640)
template <bool VEC>
__device__ __forceinline__ float dot32(const float (&a)[HD], const float* __restrict__ row) {
  float s = 0.f;
  if constexpr (!VEC) {
#pragma unroll
    for (int d = 0; d < HD; ++d) s = fmaf(a[d], row[d], s);
    return s;
  }
#pragma unroll
  for (int d = 0; d < HD; d += 4) {
    const float4 r = *reinterpret_cast<const float4*>(row + d);
    s = fmaf(a[d], r.x, s); s = fmaf(a[d + 1], r.y, s); s = fmaf(a[d + 2], r.z, s); s = fmaf(a[d + 3], r.w, s);
  }
  return s;
}
template <bool VEC>
__device__ __forceinline__ void axpy32(float (&acc)[HD], float a, const float* __restrict__ row) {
  if constexpr (!VEC) {
#pragma unroll
    for (int d = 0; d < HD; ++d) acc[d] = fmaf(a, row[d], acc[d]);
    return;
  }
#pragma unroll
  for (int d = 0; d < HD; d += 4) {
    const float4 r = *reinterpret_cast<const float4*>(row + d);
    acc[d] = fmaf(a, r.x, acc[d]); acc[d + 1] = fmaf(a, r.y, acc[d + 1]); acc[d + 2] = fmaf(a, r.z, acc[d + 2]); acc[d + 3] = fmaf(a, r.w, acc[d + 3]);
  }
}

template <int HDP>
__global__ void __launch_bounds__(384) attention_bwd_kernel(const float* __restrict__ q, int q_pitch, const float* __restrict__ k, int k_pitch,
                                                            const float* __restrict__ v, int v_pitch, const float* __restrict__ o, int o_pitch,
                                                            const float* __restrict__ dout, int do_pitch, int Lq, int Lk, int heads, float scale,
                                                            float* __restrict__ dq, int dq_pitch, float* __restrict__ dk, int dk_pitch,
                                                            float* __restrict__ dv, int dv_pitch) {
  extern __shared__ float sm[];
  float* sQ = sm;                  // [Lq][33]
  float* sdO = sQ + Lq * HDP;      // [Lq][33]
  float* sK = sdO + Lq * HDP;      // [Lk][33]
  float* sV = sK + Lk * HDP;       // [Lk][33]
  float* sL = sV + Lk * HDP;       // [Lq] log-sum-exp of the scaled scores
  float* sD = sL + Lq;             // [Lq] rowsum(dO * O)
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int64_t qb = (int64_t)b * Lq, kb = (int64_t)b * Lk;
  for (int i = threadIdx.x; i < Lq * HD; i += blockDim.x) {
    const int r = i / HD, c = i % HD;
    sQ[r * HDP + c] = q[(qb + r) * q_pitch + h * HD + c];
    sdO[r * HDP + c] = dout[(qb + r) * do_pitch + h * HD + c];
  }
  for (int i = threadIdx.x; i < Lk * HD; i += blockDim.x) {
    const int r = i / HD, c = i % HD;
    sK[r * HDP + c] = k[(kb + r) * k_pitch + h * HD + c];
    sV[r * HDP + c] = v[(kb + r) * v_pitch + h * HD + c];
  }
  __syncthreads();
  // ---- phase 1: per query row
  for (int i = threadIdx.x; i < Lq; i += blockDim.x) {
    float qi[HD], gi[HD], acc[HD];
    float D = 0.f;
#pragma unroll
    for (int d = 0; d < HD; ++d) {
      qi[d] = sQ[i * HDP + d];
      gi[d] = sdO[i * HDP + d];
      D += gi[d] * o[(qb + i) * o_pitch + h * HD + d];
      acc[d] = 0.f;
    }
    float m = -INFINITY;
    for (int j = 0; j < Lk; ++j) m = fmaxf(m, dot32<HDP % 4 == 0>(qi, sK + j * HDP) * scale);
    float l = 0.f;
    for (int j = 0; j < Lk; ++j) l += expf(dot32<HDP % 4 == 0>(qi, sK + j * HDP) * scale - m);
    const float lse = m + logf(l);
    for (int j = 0; j < Lk; ++j) {
      const float s = dot32<HDP % 4 == 0>(qi, sK + j * HDP), dp = dot32<HDP % 4 == 0>(gi, sV + j * HDP);
      const float p = expf(s * scale - lse);
      const float ds = p * (dp - D) * scale;
      axpy32<HDP % 4 == 0>(acc, ds, sK + j * HDP);
    }
    sL[i] = lse;
    sD[i] = D;
#pragma unroll
    for (int d = 0; d < HD; ++d) dq[(qb + i) * dq_pitch + h * HD + d] = acc[d];
  }
  __syncthreads();
  // ---- phase 2: per key row
  for (int j = threadIdx.x; j < Lk; j += blockDim.x) {
    float kj[HD], vj[HD], ak[HD], av[HD];
#pragma unroll
    for (int d = 0; d < HD; ++d) { kj[d] = sK[j * HDP + d]; vj[d] = sV[j * HDP + d]; ak[d] = 0.f; av[d] = 0.f; }
    for (int i = 0; i < Lq; ++i) {
      const float s = dot32<HDP % 4 == 0>(kj, sQ + i * HDP), dp = dot32<HDP % 4 == 0>(vj, sdO + i * HDP);
      const float p = expf(s * scale - sL[i]);
      const float ds = p * (dp - sD[i]) * scale;
      axpy32<HDP % 4 == 0>(av, p, sdO + i * HDP);
      axpy32<HDP % 4 == 0>(ak, ds, sQ + i * HDP);
    }
#pragma unroll
    for (int d = 0; d < HD; ++d) { dk[(kb + j) * dk_pitch + h * HD + d] = ak[d]; dv[(kb + j) * dv_pitch + h * HD + d] = av[d]; }
  }
}

constexpr int MSDA_MAX_LEVELS = 4;
struct MsdaShapesB { int h[MSDA_MAX_LEVELS], w[MSDA_MAX_LEVELS], start[MSDA_MAX_LEVELS]; };

__global__ void __launch_bounds__(256) msda_bwd_kernel(const float* __restrict__ value, int v_pitch, const float* __restrict__ oa, int oa_pitch,
                                                       const float* __restrict__ ref, const float* __restrict__ dout, int do_pitch, MsdaShapesB sh, int L, int P,
                                                       int S, int Q, int heads, int64_t total, float* __restrict__ dvalue, int dv_pitch,
                                                       float* __restrict__ doa, int doa_pitch) {
  const int lane = threadIdx.x & 31;
  const int64_t wid = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= total) return;
  const int h = wid % heads;
  const int64_t bq = wid / heads;
  const int b = bq / Q;
  const int LP = L * P;
  const float* row = oa + bq * oa_pitch;
  float logit = -INFINITY;
  if (lane < LP) logit = row[heads * LP * 2 + h * LP + lane];
  const float mx = warp_max(logit);
  const float e = lane < LP ? expf(logit - mx) : 0.f;
  const float wgt = e / warp_sum(e);
  float ox = 0.f, oy = 0.f;
  if (lane < LP) { ox = row[(h * LP + lane) * 2 + 0]; oy = row[(h * LP + lane) * 2 + 1]; }
  const float4 r = *reinterpret_cast<const float4*>(ref + bq * 4);
  const float locx = r.x + ox / (float)P * r.z * 0.5f, locy = r.y + oy / (float)P * r.w * 0.5f;
  const float go = dout[bq * do_pitch + h * 32 + lane];
  const float* vb = value + (int64_t)b * S * v_pitch + h * 32 + lane;
  float* dvb = dvalue + (int64_t)b * S * dv_pitch + h * 32 + lane;
  float my_dw = 0.f, my_dx = 0.f, my_dy = 0.f;  // lane `pt` keeps the gradients of point pt
  for (int pt = 0; pt < LP; ++pt) {
    const int lvl = pt / P;
    const float lx = __shfl_sync(0xffffffffu, locx, pt), ly = __shfl_sync(0xffffffffu, locy, pt);
    const float aw = __shfl_sync(0xffffffffu, wgt, pt);
    const int H = sh.h[lvl], W = sh.w[lvl];
    const float gx = 2.f * lx - 1.f, gy = 2.f * ly - 1.f;
    const float ix = ((gx + 1.f) * (float)W - 1.f) * 0.5f, iy = ((gy + 1.f) * (float)H - 1.f) * 0.5f;
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
    const float tx = ix - fx, ty = iy - fy;
    const bool xin0 = x0 >= 0 && x0 < W, xin1 = x1 >= 0 && x1 < W, yin0 = y0 >= 0 && y0 < H, yin1 = y1 >= 0 && y1 < H;
    const int64_t base = (int64_t)sh.start[lvl];
    const int64_t o_nw = (base + (int64_t)y0 * W + x0), o_ne = (base + (int64_t)y0 * W + x1), o_sw = (base + (int64_t)y1 * W + x0), o_se = (base + (int64_t)y1 * W + x1);
    const float v_nw = (yin0 && xin0) ? vb[o_nw * v_pitch] : 0.f, v_ne = (yin0 && xin1) ? vb[o_ne * v_pitch] : 0.f;
    const float v_sw = (yin1 && xin0) ? vb[o_sw * v_pitch] : 0.f, v_se = (yin1 && xin1) ? vb[o_se * v_pitch] : 0.f;
    const float s = v_nw * (1.f - tx) * (1.f - ty) + v_ne * tx * (1.f - ty) + v_sw * (1.f - tx) * ty + v_se * tx * ty;
    const float gs = go * aw;  // d out / d s
    if (yin0 && xin0) atomicAdd(dvb + o_nw * dv_pitch, gs * (1.f - tx) * (1.f - ty));
    if (yin0 && xin1) atomicAdd(dvb + o_ne * dv_pitch, gs * tx * (1.f - ty));
    if (yin1 && xin0) atomicAdd(dvb + o_sw * dv_pitch, gs * (1.f - tx) * ty);
    if (yin1 && xin1) atomicAdd(dvb + o_se * dv_pitch, gs * tx * ty);
    const float dsdx = (v_ne - v_nw) * (1.f - ty) + (v_se - v_sw) * ty, dsdy = (v_sw - v_nw) * (1.f - tx) + (v_se - v_ne) * tx;
    const float dw = warp_sum(go * s);
    const float dix = warp_sum(gs * dsdx), diy = warp_sum(gs * dsdy);
    if (lane == pt) {
      my_dw = dw;
      my_dx = dix * (float)W * (r.z * 0.5f / (float)P);   // ix = lx*W - 0.5, lx = ref_x + ox/P * ref_w * 0.5
      my_dy = diy * (float)H * (r.w * 0.5f / (float)P);
    }
  }
  // softmax backward over the L*P logits of this head
  const float dot = warp_sum(lane < LP ? wgt * my_dw : 0.f);
  if (lane < LP) {
    float* drow = doa + bq * doa_pitch;
    drow[(h * LP + lane) * 2 + 0] = my_dx;
    drow[(h * LP + lane) * 2 + 1] = my_dy;
    drow[heads * LP * 2 + h * LP + lane] = wgt * (my_dw - dot);
  }
}

}  // namespace
}  // namespace fb200

using namespace fb200;

extern "C" int fb200_attention_bwd(const float* q, int q_pitch, const float* k, int k_pitch, const float* v, int v_pitch, const float* o, int o_pitch,
                                   const float* dout, int do_pitch, int B, int Lq, int Lk, int heads, int head_dim, float scale, float* dq, int dq_pitch,
                                   float* dk, int dk_pitch, float* dv, int dv_pitch, void* stream) {
  FB_CHECK_ARG(q && k && v && o && dout && dq && dk && dv, "attention_bwd: null pointer");
  FB_CHECK_ARG(head_dim == HD, "attention_bwd: head_dim must be 32");
  FB_CHECK_ARG(B > 0 && Lq > 0 && Lk > 0 && heads > 0, "attention_bwd: B, Lq, Lk and heads must be positive (got %d, %d, %d, %d)", B, Lq, Lk, heads);
  // a pitch below the row width would make neighbouring rows overlap (and the gradients of one row overwrite another's)
  const int w = heads * HD;
  FB_CHECK_ARG(q_pitch >= w, "attention_bwd: q_pitch (%d) < heads*32 (%d)", q_pitch, w);
  FB_CHECK_ARG(k_pitch >= w, "attention_bwd: k_pitch (%d) < heads*32 (%d)", k_pitch, w);
  FB_CHECK_ARG(v_pitch >= w, "attention_bwd: v_pitch (%d) < heads*32 (%d)", v_pitch, w);
  FB_CHECK_ARG(o_pitch >= w, "attention_bwd: o_pitch (%d) < heads*32 (%d)", o_pitch, w);
  FB_CHECK_ARG(do_pitch >= w, "attention_bwd: do_pitch (%d) < heads*32 (%d)", do_pitch, w);
  FB_CHECK_ARG(dq_pitch >= w, "attention_bwd: dq_pitch (%d) < heads*32 (%d)", dq_pitch, w);
  FB_CHECK_ARG(dk_pitch >= w, "attention_bwd: dk_pitch (%d) < heads*32 (%d)", dk_pitch, w);
  FB_CHECK_ARG(dv_pitch >= w, "attention_bwd: dv_pitch (%d) < heads*32 (%d)", dv_pitch, w);
  auto bytes = [&](int pitch) { return ((size_t)2 * Lq * pitch + (size_t)2 * Lk * pitch + 2 * Lq) * sizeof(float); };
  const bool vec = bytes(36) <= 227 * 1024;   // float4 rows when the four planes fit at the 36-float pitch, else the 33-float scalar layout
  const size_t smem = bytes(vec ? 36 : 33);
  FB_CHECK_ARG(smem <= 227 * 1024, "attention_bwd: Lq=%d Lk=%d exceed the shared-memory-resident design (Lq+Lk <= ~850)", Lq, Lk);
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(attention_bwd_kernel<36>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(attention_bwd_kernel<33>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    attr = true;
  }
  // one thread per query (phase 1) / key (phase 2): with 256 threads the 300 decoder queries took two rounds, the second with 44 active threads
  int threads = ((Lq > Lk ? Lq : Lk) + 31) / 32 * 32;
  threads = threads < 128 ? 128 : (threads > 384 ? 384 : threads);
  if (vec)
    attention_bwd_kernel<36><<<B * heads, threads, smem, (cudaStream_t)stream>>>(q, q_pitch, k, k_pitch, v, v_pitch, o, o_pitch, dout, do_pitch, Lq, Lk, heads, scale, dq,
                                                                                 dq_pitch, dk, dk_pitch, dv, dv_pitch);
  else
    attention_bwd_kernel<33><<<B * heads, threads, smem, (cudaStream_t)stream>>>(q, q_pitch, k, k_pitch, v, v_pitch, o, o_pitch, dout, do_pitch, Lq, Lk, heads, scale, dq,
                                                                                 dq_pitch, dk, dk_pitch, dv, dv_pitch);
  FB_CHECK_LAUNCH("attention_bwd");
  return FB200_OK;
}

extern "C" int fb200_msda_bwd(const float* value, int v_pitch, const float* oa, int oa_pitch, const float* ref, const float* dout, int do_pitch,
                              const int* shapes_host, int L, int P, int B, int S, int Q, int heads, float* dvalue, int dv_pitch, float* doa, int doa_pitch,
                              void* stream) {
  FB_CHECK_ARG(value && oa && ref && dout && shapes_host && dvalue && doa, "msda_bwd: null pointer");
  FB_CHECK_ARG(L >= 1 && L <= MSDA_MAX_LEVELS && L * P <= 32, "msda_bwd: levels*points must be <= 32 (L=%d P=%d)", L, P);
  MsdaShapesB sh;
  int start = 0;
  for (int l = 0; l < L; ++l) { sh.h[l] = shapes_host[2 * l]; sh.w[l] = shapes_host[2 * l + 1]; sh.start[l] = start; start += sh.h[l] * sh.w[l]; }
  FB_CHECK_ARG(start == S, "msda_bwd: sum of level sizes (%d) != S (%d)", start, S);
  // a pitch below the row width would make the warps of neighbouring rows read, and accumulate into, each other's elements
  const int oa_w = heads * L * P * 3, v_w = heads * 32;
  FB_CHECK_ARG(oa_pitch >= oa_w, "msda_bwd: oa_pitch (%d) < heads*L*P*3 (%d)", oa_pitch, oa_w);
  FB_CHECK_ARG(doa_pitch >= oa_w, "msda_bwd: doa_pitch (%d) < heads*L*P*3 (%d)", doa_pitch, oa_w);
  FB_CHECK_ARG(v_pitch >= v_w, "msda_bwd: v_pitch (%d) < heads*32 (%d)", v_pitch, v_w);
  FB_CHECK_ARG(dv_pitch >= v_w, "msda_bwd: dv_pitch (%d) < heads*32 (%d)", dv_pitch, v_w);
  FB_CHECK_ARG(do_pitch >= v_w, "msda_bwd: do_pitch (%d) < heads*32 (%d)", do_pitch, v_w);
  const int64_t total = (int64_t)B * Q * heads;
  msda_bwd_kernel<<<(unsigned)cdiv(total, 8), 256, 0, (cudaStream_t)stream>>>(value, v_pitch, oa, oa_pitch, ref, dout, do_pitch, sh, L, P, S, Q, heads, total, dvalue,
                                                                             dv_pitch, doa, doa_pitch);
  FB_CHECK_LAUNCH("msda_bwd");
  return FB200_OK;
}

// Multi-scale deformable attention core (RT-DETR decoder cross-attention), fully fused:
//   softmax over levels*points  +  sampling-location arithmetic  +  bilinear gather  +  weighted sum.
// One warp per (batch, query, head); lane = channel of the 32-wide head, so each bilinear tap is one
// coalesced 64/128-byte row segment of `value` (L2-resident: B*S*256 elements).  Gather/latency bound.
#include "common.cuh"

namespace fb200 {

constexpr int MSDA_MAX_LEVELS = 4;
struct MsdaShapes { int h[MSDA_MAX_LEVELS], w[MSDA_MAX_LEVELS], start[MSDA_MAX_LEVELS]; };

template <typename TV, typename TOA, typename TO>
__global__ void __launch_bounds__(256) msda_kernel(const TV* __restrict__ value, int v_pitch, const TOA* __restrict__ oa,
                                                   int oa_pitch, const float* __restrict__ ref, MsdaShapes sh, int L, int P,
                                                   int S, int Q, int heads, int64_t total, TO* __restrict__ out, int out_pitch) {
  const int lane = threadIdx.x & 31;
  const int64_t wid = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);  // (b*Q + q)*heads + h
  if (wid >= total) return;
  const int h = wid % heads;
  const int64_t bq = wid / heads;
  const int b = bq / Q;
  const int LP = L * P;
  const TOA* row = oa + bq * oa_pitch;
  // attention logits -> softmax (every lane holds logit of point `lane` if lane < LP)
  float logit = -INFINITY;
  if (lane < LP) logit = to_f(row[heads * LP * 2 + h * LP + lane]);
  const float mx = warp_max(logit);
  const float e = lane < LP ? expf(logit - mx) : 0.f;
  const float wgt = e / warp_sum(e);
  // sampling offsets for point `lane`
  float ox = 0.f, oy = 0.f;
  if (lane < LP) {
    ox = to_f(row[(h * LP + lane) * 2 + 0]);
    oy = to_f(row[(h * LP + lane) * 2 + 1]);
  }
  const float4 r = *reinterpret_cast<const float4*>(ref + bq * 4);
  // loc = ref_xy + off / P * ref_wh * 0.5   (modelling.py:871-874, same association order)
  const float locx = r.x + ox / (float)P * r.z * 0.5f;
  const float locy = r.y + oy / (float)P * r.w * 0.5f;
  const TV* vb = value + (int64_t)b * S * v_pitch + h * 32 + lane;
  float acc = 0.f;
#pragma unroll 4  // 16 independent gathers in flight per lane: the kernel is L2/HBM-latency bound
  for (int pt = 0; pt < LP; ++pt) {
    const int lvl = pt / P;
    const float lx = __shfl_sync(0xffffffffu, locx, pt), ly = __shfl_sync(0xffffffffu, locy, pt);
    const float aw = __shfl_sync(0xffffffffu, wgt, pt);
    const int H = sh.h[lvl], W = sh.w[lvl];
    // grid = 2*loc-1 ; grid_sample unnormalise (align_corners=False): ((g+1)*size-1)/2   (deformable.py:16,24-30)
    const float gx = 2.f * lx - 1.f, gy = 2.f * ly - 1.f;
    const float ix = ((gx + 1.f) * (float)W - 1.f) * 0.5f, iy = ((gy + 1.f) * (float)H - 1.f) * 0.5f;
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
    const float tx = ix - fx, ty = iy - fy;
    const float w_nw = (1.f - tx) * (1.f - ty), w_ne = tx * (1.f - ty), w_sw = (1.f - tx) * ty, w_se = tx * ty;
    const TV* vl = vb + (int64_t)sh.start[lvl] * v_pitch;
    float s = 0.f;
    const bool xin0 = x0 >= 0 && x0 < W, xin1 = x1 >= 0 && x1 < W, yin0 = y0 >= 0 && y0 < H, yin1 = y1 >= 0 && y1 < H;
    if (yin0 && xin0) s += to_f(vl[((int64_t)y0 * W + x0) * v_pitch]) * w_nw;
    if (yin0 && xin1) s += to_f(vl[((int64_t)y0 * W + x1) * v_pitch]) * w_ne;
    if (yin1 && xin0) s += to_f(vl[((int64_t)y1 * W + x0) * v_pitch]) * w_sw;
    if (yin1 && xin1) s += to_f(vl[((int64_t)y1 * W + x1) * v_pitch]) * w_se;
    acc = fmaf(s, aw, acc);
  }
  out[bq * out_pitch + h * 32 + lane] = from_f<TO>(acc);
}

// Vectorised variant (the one launched): a warp still owns one (batch, query, head), but the four bilinear corners of a sampling point are
// fetched by ONE load instruction - lane = (corner = lane >> 3, channel quad = lane & 7), each lane reads 4 consecutive channels (8 B fp16 /
// 16 B fp32) of its corner - so a warp issues L*P loads of 4 x 64/128 B instead of 4*L*P loads of 64/128 B, and every lane accumulates its own
// corner over all points (the sum over corners is linear: one cross-group reduction at the end).  Same arithmetic per tap as msda_kernel;
// the only difference is the order in which the 4*L*P products are added (per corner first, then across corners).
template <typename TV> struct Quad;
template <> struct Quad<float> { static __device__ __forceinline__ void load(const float* p, float (&v)[4]) { const float4 t = *reinterpret_cast<const float4*>(p); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; } };
template <> struct Quad<__half> {
  static __device__ __forceinline__ void load(const __half* p, float (&v)[4]) {
    const uint2 t = *reinterpret_cast<const uint2*>(p);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&t.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&t.y));
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
};

template <typename TV, typename TOA, typename TO>
__global__ void __launch_bounds__(256) msda_quad_kernel(const TV* __restrict__ value, int v_pitch, const TOA* __restrict__ oa, int oa_pitch,
                                                        const float* __restrict__ ref, MsdaShapes sh, int L, int P, int S, int Q, int heads, int64_t total,
                                                        TO* __restrict__ out, int out_pitch, int pair_lo_off = 0) {
  const int lane = threadIdx.x & 31;
  const int64_t wid = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= total) return;
  const int h = wid % heads;
  const int64_t bq = wid / heads;
  const int b = bq / Q;
  const int LP = L * P;
  const TOA* row = oa + bq * oa_pitch;
  float logit = -INFINITY;
  if (lane < LP) logit = to_f(row[heads * LP * 2 + h * LP + lane]);
  const float mx = warp_max(logit);
  const float e = lane < LP ? expf(logit - mx) : 0.f;
  const float wgt = e / warp_sum(e);
  float ox = 0.f, oy = 0.f;
  if (lane < LP) { ox = to_f(row[(h * LP + lane) * 2 + 0]); oy = to_f(row[(h * LP + lane) * 2 + 1]); }
  const float4 r = *reinterpret_cast<const float4*>(ref + bq * 4);
  const float locx = r.x + ox / (float)P * r.z * 0.5f, locy = r.y + oy / (float)P * r.w * 0.5f;
  const int corner = lane >> 3, cx = corner & 1, cy = corner >> 1;
  const TV* vb = value + (int64_t)b * S * v_pitch + h * 32 + (lane & 7) * 4;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
  for (int pt = 0; pt < LP; ++pt) {
    const int lvl = pt / P;
    const float lx = __shfl_sync(0xffffffffu, locx, pt), ly = __shfl_sync(0xffffffffu, locy, pt);
    const float aw = __shfl_sync(0xffffffffu, wgt, pt);
    const int H = sh.h[lvl], W = sh.w[lvl];
    const float gx = 2.f * lx - 1.f, gy = 2.f * ly - 1.f;
    const float ix = ((gx + 1.f) * (float)W - 1.f) * 0.5f, iy = ((gy + 1.f) * (float)H - 1.f) * 0.5f;
    const float fx = floorf(ix), fy = floorf(iy);
    const float tx = ix - fx, ty = iy - fy;
    const int x = (int)fx + cx, y = (int)fy + cy;
    const float wc = (cx ? tx : 1.f - tx) * (cy ? ty : 1.f - ty);   // w_nw, w_ne, w_sw, w_se of msda_kernel
    if (x >= 0 && x < W && y >= 0 && y < H) {
      float v[4];
      Quad<TV>::load(vb + ((int64_t)sh.start[lvl] + (int64_t)y * W + x) * v_pitch, v);
      const float k = wc * aw;
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = fmaf(v[j], k, acc[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], 8);
    acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], 16);
  }
  if (lane < 8) {
    TO* o = out + bq * out_pitch + h * 32 + lane * 4;
    float v[4] = {acc[0], acc[1], acc[2], acc[3]};
    if (pair_lo_off) {  // FB200_F16PAIR rows [hi | lo] (TO = __half): the operand format of the output_proj tensor-core linear
      float hi[4], lo[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) { hi[j] = __half2float(__float2half_rn(v[j])); lo[j] = v[j] - hi[j]; }
      store4(o, hi);
      store4(o + pair_lo_off, lo);
    } else {
      store4(o, v);
    }
  }
}

}  // namespace fb200
using namespace fb200;

extern "C" int fb200_msda(const void* value, int v_dtype, int v_pitch, const void* oa, int oa_dtype, int oa_pitch,
                          const float* ref, const int* shapes_host, int L, int P, int B, int S, int Q, int heads, void* out,
                          int out_dtype, int out_pitch, void* stream) {
  FB_CHECK_ARG(value && oa && ref && shapes_host && out, "msda: null pointer");
  FB_CHECK_ARG(L >= 1 && L <= MSDA_MAX_LEVELS && L * P <= 32, "msda: levels*points must be <= 32 (L=%d P=%d)", L, P);
  MsdaShapes sh;
  int start = 0;
  for (int l = 0; l < L; ++l) {
    sh.h[l] = shapes_host[2 * l];
    sh.w[l] = shapes_host[2 * l + 1];
    sh.start[l] = start;
    start += sh.h[l] * sh.w[l];
  }
  FB_CHECK_ARG(start == S, "msda: sum of level sizes (%d) != S (%d)", start, S);
  FB_CHECK_ARG(oa_pitch >= heads * L * P * 3, "msda: oa_pitch too small");
  const int64_t total = (int64_t)B * Q * heads;
  const unsigned grid = (unsigned)cdiv(total, 8);
  cudaStream_t st = (cudaStream_t)stream;
  // 4-channel vector loads need 8/16-byte aligned rows; other rows take the one-tap-per-load kernel
  const size_t velt = v_dtype == FB200_F16 ? 2 : 4, oelt = out_dtype == FB200_F32 ? 4 : 2;
  const bool quad = (v_pitch * velt) % (4 * velt) == 0 && (reinterpret_cast<uintptr_t>(value) % (4 * velt)) == 0 && (out_pitch * oelt) % (4 * oelt) == 0 &&
                    (reinterpret_cast<uintptr_t>(out) % (4 * oelt)) == 0;
#define MSDA_LAUNCH(TV, TOA, TO)                                                                                                                                   \
  do {                                                                                                                                                             \
    if (quad) msda_quad_kernel<TV, TOA, TO><<<grid, 256, 0, st>>>((const TV*)value, v_pitch, (const TOA*)oa, oa_pitch, ref, sh, L, P, S, Q, heads, total, (TO*)out, out_pitch); \
    else msda_kernel<TV, TOA, TO><<<grid, 256, 0, st>>>((const TV*)value, v_pitch, (const TOA*)oa, oa_pitch, ref, sh, L, P, S, Q, heads, total, (TO*)out, out_pitch);        \
  } while (0)
  if (v_dtype == FB200_F32 && oa_dtype == FB200_F32 && out_dtype == FB200_F16PAIR) {
    FB_CHECK_ARG(quad && out_pitch >= 2 * heads * 32, "msda: pair output needs 16-byte aligned rows of [hi(heads*32) | lo(heads*32)] halves");
    msda_quad_kernel<float, float, __half><<<grid, 256, 0, st>>>((const float*)value, v_pitch, (const float*)oa, oa_pitch, ref, sh, L, P, S, Q, heads, total, (__half*)out, out_pitch,
                                                                 heads * 32);
  } else if (v_dtype == FB200_F32 && oa_dtype == FB200_F32 && out_dtype == FB200_F32) MSDA_LAUNCH(float, float, float);
  else if (v_dtype == FB200_F16 && oa_dtype == FB200_F32 && out_dtype == FB200_F16) MSDA_LAUNCH(__half, float, __half);
  else if (v_dtype == FB200_F16 && oa_dtype == FB200_F16 && out_dtype == FB200_F16) MSDA_LAUNCH(__half, __half, __half);
  else { set_error("msda: unsupported dtype combination %d/%d/%d", v_dtype, oa_dtype, out_dtype); return FB200_ERR_UNSUPPORTED; }
#undef MSDA_LAUNCH
  FB_CHECK_LAUNCH("msda");
  return FB200_OK;
}

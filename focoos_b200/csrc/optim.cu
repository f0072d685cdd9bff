// Optimiser side of the fine-tune step (SURVEY §8 a21): what TrainerLoop.run_step does after backward
// (focoos/trainer/trainer.py:757-773) - GradScaler.unscale_ + inf check, clip_grad_norm_ (twice: trainer.py:793 and
// FullModelGradientClippingOptimizer.step, trainer/solver/build.py:29-37), AdamW.step with one hyper-parameter set per
// tensor (build.py:40-101), GradScaler.update - as three launches over ONE flat fp32 parameter / gradient / moment
// buffer: grad_stats (sum of squares + non-finite flag), optim_finalize (norm, clip coefficient, loss-scale update,
// bias corrections; one thread) and adamw_step (HBM-bound: reads g,p,m,v, writes p,m,v = 28 B/parameter).
// Nothing is read back by the host: the control block lives in device memory.
#include "common.cuh"

namespace fb200 {
namespace {

constexpr int STATS_BLOCKS = kNumSMs * 4;

__global__ void __launch_bounds__(256) grad_stats_kernel(const float* __restrict__ g, int64_t n, double* __restrict__ partial, int* __restrict__ flags) {
  const int tid = threadIdx.x;
  float acc = 0.f;
  int bad = 0;
  const int64_t n4 = n >> 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + tid; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    bad |= !(isfinite(v.x) && isfinite(v.y) && isfinite(v.z) && isfinite(v.w));
  }
  if (blockIdx.x == 0 && tid < (int)(n & 3)) {
    const float v = g[(n4 << 2) + tid];
    acc += v * v;
    bad |= !isfinite(v);
  }
  __shared__ double red[256];
  __shared__ int rbad[256];
  red[tid] = (double)acc;
  rbad[tid] = bad;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (tid < o) { red[tid] += red[tid + o]; rbad[tid] |= rbad[tid + o]; }
    __syncthreads();
  }
  if (tid == 0) { partial[blockIdx.x] = red[0]; flags[blockIdx.x] = rbad[0]; }
}

// ctrl words: see include/focoos_b200.h (FB200_CTRL_*)
__global__ void optim_finalize_kernel(const double* __restrict__ partial, const int* __restrict__ flags, int nblk, float* __restrict__ ctrl, float max_norm,
                                      int clip_passes, float inv_world, int use_scaler, float growth, float backoff, int growth_interval,
                                      float one_minus_beta1, float one_minus_beta2) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int* ictrl = reinterpret_cast<int*>(ctrl);
  double s = 0.0;
  int bad = 0;
  for (int i = 0; i < nblk; ++i) { s += partial[i]; bad |= flags[i]; }
  const float scale = use_scaler ? ctrl[0] : 1.f;
  const float pre = inv_world / scale;                    // gradients hold  scale * sum_over_ranks(grad)
  float norm = (float)sqrt(s) * pre;
  bad |= !isfinite(norm);
  float coef = 1.f;
  float nrm = norm;
  for (int k = 0; k < clip_passes && max_norm > 0.f; ++k) {   // clip_grad_norm_: coef = clamp(max_norm / (norm + 1e-6), max=1)
    const float c = fminf(max_norm / (nrm + 1e-6f), 1.f);
    coef *= c;
    nrm *= c;
  }
  ictrl[2] = bad;
  ctrl[3] = norm;
  ctrl[4] = pre * coef;
  ctrl[8] = coef;
  if (!bad) {
    const int step = ictrl[5] + 1;
    ictrl[5] = step;
    ctrl[6] = (float)(1.0 - pow(1.0 - (double)one_minus_beta1, (double)step));
    ctrl[7] = (float)sqrt(1.0 - pow(1.0 - (double)one_minus_beta2, (double)step));
  }
  if (use_scaler) {                                       // GradScaler.update (torch/amp/grad_scaler.py: _amp_update_scale_)
    if (bad) { ctrl[0] = scale * backoff; ictrl[1] = 0; }
    else {
      const int t = ictrl[1] + 1;
      if (t == growth_interval) { ctrl[0] = scale * growth; ictrl[1] = 0; }
      else ictrl[1] = t;
    }
  }
}

// torch.optim.AdamW (single-tensor path, torch/optim/adam.py): p *= 1 - lr*wd; m = lerp(m, g, 1-b1); v = b2*v + (1-b2)*g*g;
// p -= (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps).   One CTA per chunk; a chunk never straddles two tensors.
// omb1 / omb2 = 1 - beta as the caller formed it before rounding to fp32, as torch's scalars are (1 - fp32(0.999) is 1.3e-5 smaller than
// fp32(0.001)).
__global__ void __launch_bounds__(256) adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                                     const int64_t* __restrict__ chunk_start, const int* __restrict__ chunk_len, const int* __restrict__ chunk_seg,
                                                     const float* __restrict__ seg_lr, const float* __restrict__ seg_wd, const int* __restrict__ seg_active, float lr_factor,
                                                     float omb1, float beta2, float omb2, float eps, const float* __restrict__ ctrl) {
  if (reinterpret_cast<const int*>(ctrl)[2]) return;      // non-finite gradients: the step is skipped (GradScaler.step)
  const float gmul = ctrl[4], bc1 = ctrl[6], bc2s = ctrl[7];
  const int c = blockIdx.x;
  const int64_t s0 = chunk_start[c];
  const int len = chunk_len[c], seg = chunk_seg[c];
  if (seg_active && !seg_active[seg]) return;  // tensor received no gradient this step: torch.optim skips it entirely (p.grad is None), decay included
  const float lr = seg_lr[seg] * lr_factor, wd = seg_wd[seg];
  const float decay = 1.f - lr * wd, step_size = lr / bc1;
  float4* p4 = reinterpret_cast<float4*>(p + s0);
  float4* m4 = reinterpret_cast<float4*>(m + s0);
  float4* v4 = reinterpret_cast<float4*>(v + s0);
  const float4* g4 = reinterpret_cast<const float4*>(g + s0);
  auto upd = [&](float& pp, float gg, float& mm, float& vv) {
    gg *= gmul;
    pp *= decay;
    mm = mm + (gg - mm) * omb1;
    vv = vv * beta2 + omb2 * (gg * gg);
    pp -= step_size * (mm / (sqrtf(vv) / bc2s + eps));
  };
  for (int i = threadIdx.x; i < (len >> 2); i += blockDim.x) {
    float4 P = p4[i], M = m4[i], V = v4[i];
    const float4 G = g4[i];
    upd(P.x, G.x, M.x, V.x); upd(P.y, G.y, M.y, V.y); upd(P.z, G.z, M.z, V.z); upd(P.w, G.w, M.w, V.w);
    p4[i] = P; m4[i] = M; v4[i] = V;
  }
}

// Model EMA (focoos/trainer/solver/ema.py:112-140), one launch per step.  Blocks [0, arena_blocks) stride over the EMA arena, which has the
// layout of the flat parameter buffer: torch._foreach_mul_(ema, d) then torch._foreach_add_(ema, p, alpha=omd).  torch's foreach add is
// `a + alpha * b` in fp32 and nvcc contracts it into one FMA, so the update is fma(omd, p, fl(ema * d)) - two roundings, as on the device.
// Every further block owns one chunk of the table {src address, EMA address, length, kind}: the entries outside the flat buffer (frozen
// parameters, BatchNorm buffers).  Kind 1 is an int64 entry, updated as `ema.copy_(ema * decay + val * (1.0 - decay))` is: both products
// in fp32 (the int64 values converted to fp32), an fp32 sum, truncation back to int64.
__global__ void __launch_bounds__(256) ema_kernel(float* __restrict__ ema, const float* __restrict__ p, int64_t n4, int arena_blocks,
                                                  const int64_t* __restrict__ chunks, float d, float omd) {
  if ((int)blockIdx.x < arena_blocks) {
    float4* e4 = reinterpret_cast<float4*>(ema);
    const float4* p4 = reinterpret_cast<const float4*>(p);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)arena_blocks * blockDim.x) {
      float4 E = e4[i];
      const float4 P = p4[i];
      E.x = __fmaf_rn(omd, P.x, __fmul_rn(E.x, d));
      E.y = __fmaf_rn(omd, P.y, __fmul_rn(E.y, d));
      E.z = __fmaf_rn(omd, P.z, __fmul_rn(E.z, d));
      E.w = __fmaf_rn(omd, P.w, __fmul_rn(E.w, d));
      e4[i] = E;
    }
    return;
  }
  const int64_t* c = chunks + 4 * (int64_t)(blockIdx.x - arena_blocks);
  const int64_t len = c[2];
  if (c[3] == 1) {
    const long long* s = reinterpret_cast<const long long*>(c[0]);
    long long* e = reinterpret_cast<long long*>(c[1]);
    for (int64_t i = threadIdx.x; i < len; i += blockDim.x)
      e[i] = (long long)__fadd_rn(__fmul_rn(__ll2float_rn(e[i]), d), __fmul_rn(__ll2float_rn(s[i]), omd));
  } else {
    const float* s = reinterpret_cast<const float*>(c[0]);
    float* e = reinterpret_cast<float*>(c[1]);
    for (int64_t i = threadIdx.x; i < len; i += blockDim.x) e[i] = __fmaf_rn(omd, s[i], __fmul_rn(e[i], d));
  }
}

}  // namespace
}  // namespace fb200

using namespace fb200;

extern "C" int fb200_ema_update(float* ema, const float* params, int64_t n, const int64_t* chunks, int nchunks, float decay, float one_minus_decay,
                                void* stream) {
  FB_CHECK_ARG(n >= 0 && (n & 3) == 0 && nchunks >= 0 && (n > 0 || nchunks > 0) && (n == 0 || (ema && params)) && (nchunks == 0 || chunks),
               "ema_update: bad arguments");
  FB_CHECK_ARG(((reinterpret_cast<uintptr_t>(ema) | reinterpret_cast<uintptr_t>(params)) & 15) == 0, "ema_update: arena and parameters must be 16-byte aligned");
  const int64_t n4 = n >> 2;
  const int arena_blocks = (int)std::min<int64_t>((n4 + 255) / 256, (int64_t)kNumSMs * 8);
  ema_kernel<<<arena_blocks + nchunks, 256, 0, (cudaStream_t)stream>>>(ema, params, n4, arena_blocks, chunks, decay, one_minus_decay);
  FB_CHECK_LAUNCH("ema_update");
  return FB200_OK;
}

extern "C" int64_t fb200_optim_workspace_bytes(void) { return (int64_t)STATS_BLOCKS * (8 + 4) + 64; }

extern "C" int fb200_grad_stats(const float* grads, int64_t n, void* workspace, void* stream) {
  FB_CHECK_ARG(grads && workspace && n > 0, "grad_stats: bad arguments");
  FB_CHECK_ARG((reinterpret_cast<uintptr_t>(grads) & 15) == 0, "grad_stats: gradient buffer must be 16-byte aligned");
  double* partial = reinterpret_cast<double*>(workspace);
  int* flags = reinterpret_cast<int*>(partial + STATS_BLOCKS);
  grad_stats_kernel<<<STATS_BLOCKS, 256, 0, (cudaStream_t)stream>>>(grads, n, partial, flags);
  FB_CHECK_LAUNCH("grad_stats");
  return FB200_OK;
}

extern "C" int fb200_optim_finalize(const void* workspace, float* ctrl, float max_norm, int clip_passes, float inv_world, int use_scaler, float growth,
                                    float backoff, int growth_interval, float one_minus_beta1, float one_minus_beta2, void* stream) {
  FB_CHECK_ARG(workspace && ctrl && inv_world > 0.f && clip_passes >= 0, "optim_finalize: bad arguments");
  const double* partial = reinterpret_cast<const double*>(workspace);
  const int* flags = reinterpret_cast<const int*>(partial + STATS_BLOCKS);
  optim_finalize_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(partial, flags, STATS_BLOCKS, ctrl, max_norm, clip_passes, inv_world, use_scaler, growth, backoff,
                                                            growth_interval, one_minus_beta1, one_minus_beta2);
  FB_CHECK_LAUNCH("optim_finalize");
  return FB200_OK;
}

extern "C" int fb200_adamw_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const int64_t* chunk_start, const int* chunk_len,
                                const int* chunk_seg, int nchunks, const float* seg_lr, const float* seg_wd, const int* seg_active, float lr_factor,
                                float one_minus_beta1, float one_minus_beta2, float eps, const float* ctrl, void* stream) {
  FB_CHECK_ARG(params && grads && exp_avg && exp_avg_sq && chunk_start && chunk_len && chunk_seg && seg_lr && seg_wd && ctrl && nchunks > 0,
               "adamw_step: bad arguments");
  adamw_kernel<<<nchunks, 256, 0, (cudaStream_t)stream>>>(params, grads, exp_avg, exp_avg_sq, chunk_start, chunk_len, chunk_seg, seg_lr, seg_wd, seg_active, lr_factor,
                                                          one_minus_beta1, 1.f - one_minus_beta2, one_minus_beta2, eps, ctrl);
  FB_CHECK_LAUNCH("adamw_step");
  return FB200_OK;
}

// wgmma weight-gradient GEMM for sm_90a, fp32-accurate through split-precision fp16 products.
//
//   dW[co, kh, kw, ci] = sum over output pixels p of  dY[p, co] * X[pix(p, kh, kw), ci]          (stride-1 convs and linears)
//
// GEMM view per filter tap: D[M = Cout, N = Cin] = A^T B with the reduction over PIXELS.  In NHWC both operands are stored
// pixel-major with channels contiguous, i.e. they are "MN-major" for the tensor core: a TMA box of 64 pixels x 64 channels lands in
// shared memory as 8 swizzle atoms of (8 pixels x 128 B) - exactly the canonical SWIZZLE_128B MN-major layout
// ((8,8,n),(8,k)):((1,8,LBO),(64,SBO)) in elements (cute/arch/mma_sm90_desc.hpp), so no transpose is ever materialised:
//   SBO = 1024 B (next 8-pixel group), LBO = 8192 B (next 64-channel block = the next TMA box), wgmma with both operands
//   transposed (MN-major).  The X box is the dY box shifted by the tap offset; out-of-bounds rows/columns (conv zero padding, ragged
//   pixel tiles) are zero-filled by the TMA unit for BOTH operands, so ragged tiles contribute exact zeros.
// fp32 accuracy: operands are the [hi | lo] fp16 pairs of the fp32 tensors (fb200_split_f32_pair); each 64-pixel K chunk issues
//   dY_hi*X_hi + dY_hi*X_lo + dY_lo*X_hi  into one fp32 register accumulator per chunk, and the chunks are added in fp32 (round to nearest)
//   (error ~2^-21 relative, like the forward mode).
// Parallelism: work item = (128 x BLOCK_N weight tile, tap, pixel split); persistent CTAs, warp-specialised (one TMA producer thread,
//   two consumer warp-groups that each own 64 output channels of the tile), 3-stage smem ring;
//   split partials are reduced in a fixed order by wgrad_reduce_kernel (reproducible, no atomics).
#include <cuda.h>

#include <cstdlib>

#include "common.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace fb200 {
namespace wg {

constexpr int BLOCK_M = 128;   // Cout tile
constexpr int BLOCK_K = 64;    // pixels per chunk
constexpr int STAGES = 3;
constexpr int BOX_BYTES = BLOCK_K * 64 * 2;  // one TMA box: 64 pixels x 64 channels fp16 = 8 KiB

struct WParams {
  int Cout, Cin, KH, KW, pad, stride;
  int BW, BH, tiles_w, tiles_h, B;     // pixel tile rectangle (BW*BH == 64) and counts
  int m_tiles, n_tiles, taps, splits;  // work decomposition
  int pt_total, pt_per_split;          // pixel tiles
  int total_items;
  float* part;                         // [splits][Cout][KH*KW][Cin]
  int single;                          // 1: plain fp16 operands, ONE product per chunk (the reference's fp16-autocast numerics class); 0: [hi | lo] pairs, three products
};

// MN-major SWIZZLE_128B shared-memory matrix descriptor (sm_90 format): LBO = stride between 64-element MN blocks, SBO = stride between 8-row K groups
__device__ __forceinline__ uint64_t make_desc_mn(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)(BOX_BYTES >> 4) << 16;  // leading byte offset: next 64-channel block (next TMA box)
  d |= (uint64_t)(1024 >> 4) << 32;       // stride byte offset: next group of 8 pixels
  d |= (uint64_t)1 << 62;                 // SWIZZLE_128B
  return d;
}

template <int BLOCK_N> __host__ __device__ constexpr int a_boxes() { return 2 * (BLOCK_M / 64); }   // hi + lo, 64 channels per box
template <int BLOCK_N> __host__ __device__ constexpr int b_boxes() { return 2 * (BLOCK_N / 64); }
template <int BLOCK_N> __host__ __device__ constexpr int stage_bytes() { return (a_boxes<BLOCK_N>() + b_boxes<BLOCK_N>()) * BOX_BYTES; }
template <int BLOCK_N> constexpr int smem_bytes() { return STAGES * stage_bytes<BLOCK_N>() + 2 * STAGES * 8 + 1024; }

template <int BLOCK_N>
__global__ void __launch_bounds__(384, 1) wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmap_dy, const __grid_constant__ CUtensorMap tmap_x, const WParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int A_BOXES = a_boxes<BLOCK_N>(), B_BOXES = b_boxes<BLOCK_N>();
  constexpr int STAGE_BYTES = stage_bytes<BLOCK_N>();
  constexpr int A_HALF = (A_BOXES / 2) * BOX_BYTES, B_HALF = (B_BOXES / 2) * BOX_BYTES;  // bytes of the hi (or lo) part
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_dy) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_x) : "memory");
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }  // one arrival per consumer warp
    fence_barrier_init();
  }
  __syncthreads();
  const int tiles_per_img = p.tiles_w * p.tiles_h;

  // work item -> (split, tap, n tile, m tile); n fastest so CTAs running together share dY boxes in L2
  auto decode = [&](int item, int& mt, int& nt, int& tap, int& split) {
    nt = item % p.n_tiles; item /= p.n_tiles;
    mt = item % p.m_tiles; item /= p.m_tiles;
    tap = item % p.taps;
    split = item / p.taps;
  };

  if (warp < 4) {
    if (threadIdx.x != 0) return;  // ================================================================= TMA producer
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < p.total_items; item += gridDim.x) {
      int mt, nt, tap, split;
      decode(item, mt, nt, tap, split);
      const int m0 = mt * BLOCK_M, n0 = nt * BLOCK_N;
      const int kh = tap / p.KW, kw = tap - kh * p.KW;
      const int pt_begin = split * p.pt_per_split, pt_end = min(p.pt_total, pt_begin + p.pt_per_split);
      for (int pt = pt_begin; pt < pt_end; ++pt) {
        const int img = pt / tiles_per_img, rem = pt - img * tiles_per_img;
        const int h0 = (rem / p.tiles_w) * p.BH, w0 = (rem % p.tiles_w) * p.BW;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)(p.single ? STAGE_BYTES / 2 : STAGE_BYTES));
        uint8_t* sa = smem + stage * STAGE_BYTES;
        uint8_t* sb = sa + A_BOXES * BOX_BYTES;
        const int halves = p.single ? 1 : 2;
        for (int half = 0; half < halves; ++half) {  // 0 = hi, 1 = lo (channel offset C in the pair tensor)
#pragma unroll
          for (int j = 0; j < BLOCK_M / 64; ++j)
            tma_load_4d(&tmap_dy, &full_bar[stage], sa + half * A_HALF + j * BOX_BYTES, half * p.Cout + m0 + j * 64, w0, h0, img);
#pragma unroll
          for (int j = 0; j < BLOCK_N / 64; ++j)
            tma_load_4d(&tmap_x, &full_bar[stage], sb + half * B_HALF + j * BOX_BYTES, half * p.Cin + n0 + j * 64, w0 * p.stride + kw - p.pad,
                        h0 * p.stride + kh - p.pad, img);  // stride 2: the X map traverses every second pixel (TMA element strides)
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }
  // ===================================================================== consumers: warp-group g owns output channels m0 + 64g .. +63 (= dY box g)
  const int ct = threadIdx.x - 128;
  const int g = ct >> 7;
  const int row = g * 64 + ((ct & 127) >> 5) * 16 + (lane >> 2);  // accumulator rows row and row + 8
  const int cq = 2 * (lane & 3);
  // The wgmma accumulator does not round its additions to nearest: summed in it over a whole split (up to ~10^4 chunks for the stem's 1.6 M-pixel
  // weight gradients), products of one sign drift by many ulps.  So each 64-pixel chunk is summed in `acc` alone and added to `tot` with an fp32
  // (round-to-nearest) add; the drift stays that of one chunk's 4 (single) or 12 (split) products per element.
  float acc[BLOCK_N / 2], tot[BLOCK_N / 2];
  int stage = 0;
  uint32_t phase = 0;
  for (int item = blockIdx.x; item < p.total_items; item += gridDim.x) {
    int mt, nt, tap, split;
    decode(item, mt, nt, tap, split);
    const int pt_begin = split * p.pt_per_split, pt_end = min(p.pt_total, pt_begin + p.pt_per_split);
    for (int pt = pt_begin; pt < pt_end; ++pt) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + (uint32_t)(g * BOX_BYTES), sb = smem_u32(smem + stage * STAGE_BYTES) + A_BOXES * BOX_BYTES;
      const uint64_t a_hi = make_desc_mn(sa), a_lo = make_desc_mn(sa + A_HALF);
      const uint64_t b_hi = make_desc_mn(sb), b_lo = make_desc_mn(sb + B_HALF);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BLOCK_K / 16; ++k) {  // 16 pixels = two 8-pixel groups = 2048 B: +128 in 16-byte units
        const uint64_t adv = (uint64_t)(k * 128);
        Wgmma<BLOCK_N, 1>::mma(acc, a_hi + adv, b_hi + adv, k > 0 ? 1u : 0u);
        if (!p.single) {
          Wgmma<BLOCK_N, 1>::mma(acc, a_hi + adv, b_lo + adv, 1u);
          Wgmma<BLOCK_N, 1>::mma(acc, a_lo + adv, b_hi + adv, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();  // this chunk's products are done: its stage may be refilled (the producer keeps the next stages loaded meanwhile)
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) {
        asm volatile("" : "+f"(acc[i])::"memory");  // read acc only after the wait above (it carries no register dependence on the async products)
        tot[i] = pt > pt_begin ? tot[i] + acc[i] : acc[i];
      }
    }
    // registers -> split partial in global memory (Cin % 8 == 0: a column pair never straddles the end of a row)
    const int n0 = nt * BLOCK_N;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int co = mt * BLOCK_M + row + 8 * h;
      if (co >= p.Cout) continue;
      float* dst = p.part + (((int64_t)split * p.Cout + co) * p.taps + tap) * p.Cin + n0;
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int c = 8 * j + cq;
        if (n0 + c < p.Cin) *reinterpret_cast<float2*>(dst + c) = make_float2(tot[4 * j + 2 * h], tot[4 * j + 2 * h + 1]);
      }
    }
  }
}

__global__ void wgrad_reduce_kernel(const float* __restrict__ part, int splits, int64_t n, float* __restrict__ out, int accumulate) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int k = 0; k < splits; ++k) s += part[(int64_t)k * n + i];
  out[i] = accumulate ? out[i] + s : s;
}

// pair tensor [B,H,W,2C] fp16 -> 4-D map (channel, w, h, b) with a 64-channel x BW x BH box, SWIZZLE_128B, OOB = zero
static int encode_pair(CUtensorMap* m, const void* base, int C2, int W, int H, int B, int BW, int BH, const char* what, int stride = 1) {
  const uint64_t C = (uint64_t)C2;
  const uint64_t dims[4] = {C, (uint64_t)W, (uint64_t)H, (uint64_t)B}, str[4] = {1, C, C * W, C * W * H};
  // with a traversal stride s the box spans s*BW x s*BH input pixels and delivers ceil(s*BW / s) x ceil(s*BH / s) = BW x BH of them
  const uint32_t box[4] = {64, (uint32_t)(BW * stride), (uint32_t)(BH * stride), 1}, estr[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
  return encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, const_cast<void*>(base), dims, str, box, what, CU_TENSOR_MAP_SWIZZLE_128B, estr);
}

// pixel rectangle with EXACTLY 64 pixels (power-of-two width), maximising the covered fraction of the Ho x Wo map
static void choose_rect(int Ho, int Wo, int* BW, int* BH) {
  double best = -1.0;
  for (int bw = 1; bw <= 64; bw *= 2) {
    const int bh = 64 / bw;
    const double tiles = (double)((Wo + bw - 1) / bw) * (double)((Ho + bh - 1) / bh);
    const double eff = (double)Wo * Ho / (tiles * 64.0);
    if (eff > best + 1e-9 || (eff > best - 1e-9 && bw > *BW)) { best = eff; *BW = bw; *BH = bh; }
  }
}

struct Plan { int BW, BH, tiles_w, tiles_h, m_tiles, n_tiles, block_n, splits, pt_total, pt_per_split; };
static Plan make_plan(int B, int Ho, int Wo, int Cin, int Cout, int taps) {
  Plan pl;
  pl.BW = 1; pl.BH = 64;
  choose_rect(Ho, Wo, &pl.BW, &pl.BH);
  pl.tiles_w = (Wo + pl.BW - 1) / pl.BW; pl.tiles_h = (Ho + pl.BH - 1) / pl.BH;
  pl.pt_total = B * pl.tiles_w * pl.tiles_h;
  pl.block_n = Cin > 64 ? 128 : 64;
  pl.m_tiles = (Cout + BLOCK_M - 1) / BLOCK_M;
  pl.n_tiles = (Cin + pl.block_n - 1) / pl.block_n;
  const int64_t base = (int64_t)pl.m_tiles * pl.n_tiles * taps;
  int64_t splits = (2 * (int64_t)num_sms() + base - 1) / base;           // ~2 work items per SM
  const int64_t max_splits = pl.pt_total / 8 > 0 ? pl.pt_total / 8 : 1;   // at least 8 pixel tiles (512 pixels) per item
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  pl.pt_per_split = (int)((pl.pt_total + splits - 1) / splits);
  pl.splits = (pl.pt_total + pl.pt_per_split - 1) / pl.pt_per_split;
  return pl;
}

}  // namespace wg
}  // namespace fb200

using namespace fb200;

/* 1 if fb200_conv_wgrad_tc supports the shape (else the caller uses fb200_conv_wgrad) */
extern "C" int fb200_conv_wgrad_tc_supported(int B, int H, int W, int Cin, int Ho, int Wo, int Cout, int KH, int KW, int stride, int pad) {
  if ((stride != 1 && stride != 2) || KH != KW || (KH != 1 && KH != 3) || 2 * pad != KH - 1) return 0;
  if (Ho != (H + 2 * pad - KH) / stride + 1 || Wo != (W + 2 * pad - KW) / stride + 1) return 0;
  if (stride == 2 && KH != 3) return 0;
  if (Cin % 8 != 0 || Cout % 8 != 0) return 0;            // 16-byte global strides of the fp16 pair tensors
  if ((int64_t)B * Ho * Wo < 512) return 0;
  return 1;
}

extern "C" int64_t fb200_conv_wgrad_tc_workspace_bytes(int B, int Ho, int Wo, int Cin, int Cout, int KH, int KW) {
  const wg::Plan pl = wg::make_plan(B, Ho, Wo, Cin, Cout, KH * KW);
  return (int64_t)pl.splits * Cout * KH * KW * Cin * 4 + 16;
}

static int wgrad_tc_launch(const void* x_pair, int B, int H, int W, int Cin, const void* dy_pair, int Cout, int KH, int KW, int stride, int pad, float* dw,
                           int accumulate, void* workspace, void* stream, int single) {
  FB_CHECK_ARG(x_pair && dy_pair && dw && workspace, "conv_wgrad_tc: null pointer");
  const int Ho = (H + 2 * pad - KH) / stride + 1, Wo = (W + 2 * pad - KW) / stride + 1;
  FB_CHECK_ARG(fb200_conv_wgrad_tc_supported(B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad), "conv_wgrad_tc: unsupported shape (B=%d H=%d W=%d Cin=%d Cout=%d k=%d s=%d)", B, H, W,
               Cin, Cout, KH, stride);
  FB_CHECK_ARG(((reinterpret_cast<uintptr_t>(x_pair) | reinterpret_cast<uintptr_t>(dy_pair) | reinterpret_cast<uintptr_t>(workspace) | reinterpret_cast<uintptr_t>(dw)) & 15) == 0,
               "conv_wgrad_tc: pointers must be 16-byte aligned");
  using namespace wg;
  const int taps = KH * KW;
  const Plan pl = make_plan(B, Ho, Wo, Cin, Cout, taps);
  CUtensorMap tdy, tx;
  const int planes = single ? 1 : 2;  // channels per pixel of the operand tensors: C (plain fp16) or 2C ([hi | lo] pair)
  int rc = encode_pair(&tdy, dy_pair, planes * Cout, Wo, Ho, B, pl.BW, pl.BH, "wgrad_tc: dY");
  if (rc) return rc;
  rc = encode_pair(&tx, x_pair, planes * Cin, W, H, B, pl.BW, pl.BH, "wgrad_tc: X", stride);
  if (rc) return rc;
  WParams p;
  p.Cout = Cout; p.Cin = Cin; p.KH = KH; p.KW = KW; p.pad = pad; p.stride = stride;
  p.BW = pl.BW; p.BH = pl.BH; p.tiles_w = pl.tiles_w; p.tiles_h = pl.tiles_h; p.B = B;
  p.m_tiles = pl.m_tiles; p.n_tiles = pl.n_tiles; p.taps = taps; p.splits = pl.splits;
  p.pt_total = pl.pt_total; p.pt_per_split = pl.pt_per_split;
  const int64_t items = (int64_t)pl.m_tiles * pl.n_tiles * taps * pl.splits;
  FB_CHECK_ARG(items <= 0x7fffffffLL, "conv_wgrad_tc: too many work items");
  p.total_items = (int)items;
  p.part = reinterpret_cast<float*>(workspace);
  p.single = single;
  cudaStream_t st = (cudaStream_t)stream;
  rc = pl.block_n == 128 ? launch_persistent<wgrad_tc_kernel<128>, smem_bytes<128>()>("conv_wgrad_tc", items, 384, st, tdy, tx, p)
                         : launch_persistent<wgrad_tc_kernel<64>, smem_bytes<64>()>("conv_wgrad_tc", items, 384, st, tdy, tx, p);
  if (rc) return rc;
  const int64_t n = (int64_t)Cout * taps * Cin;
  wgrad_reduce_kernel<<<(unsigned)cdiv(n, 256), 256, 0, st>>>(p.part, pl.splits, n, dw, accumulate);
  FB_CHECK_LAUNCH("conv_wgrad_tc(reduce)");
  return FB200_OK;
}

/* x_pair [B,H,W,2*Cin] fp16, dy_pair [B,Ho,Wo,2*Cout] fp16 (both from fb200_split_f32_pair, dense) -> dw [Cout][KH][KW][Cin] fp32 */
extern "C" int fb200_conv_wgrad_tc(const void* x_pair, int B, int H, int W, int Cin, const void* dy_pair, int Cout, int KH, int KW, int stride, int pad, float* dw,
                                   int accumulate, void* workspace, void* stream) {
  return wgrad_tc_launch(x_pair, B, H, W, Cin, dy_pair, Cout, KH, KW, stride, pad, dw, accumulate, workspace, stream, 0);
}

/* the same GEMM on PLAIN fp16 operands (x [B,H,W,Cin], dy [B,Ho,Wo,Cout], dense), one tensor-core product, fp32 accumulation and output: the arithmetic of
   the reference's training under torch.autocast(fp16) (trainer/trainer.py:735), used by the "amp" training precision */
extern "C" int fb200_conv_wgrad_tc_f16(const void* x, int B, int H, int W, int Cin, const void* dy, int Cout, int KH, int KW, int stride, int pad, float* dw,
                                       int accumulate, void* workspace, void* stream) {
  return wgrad_tc_launch(x, B, H, W, Cin, dy, Cout, KH, KW, stride, pad, dw, accumulate, workspace, stream, 1);
}

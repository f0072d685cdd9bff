// wgmma implicit-GEMM convolution / linear for sm_90a  (fp16 operands, fp32 accumulate in registers).
//
//   D[m, n] = act( (sum_k A[m,k] * W[n,k]) * scale[n] + bias[n] + residual[m,n] )
//   m = output pixel (b, ho, wo), n = output channel, k = (kh, kw, c).
//
// Design: PERSISTENT, warp-specialised CTAs (grid = #SMs); each CTA walks 128 x BLOCK_N output tiles
// (N tiles fastest so CTAs that share an A tile run together and A comes from L2).
//   warp-group 0   TMA producer (one thread).  A is never materialised as im2col: an M-tile is a BW x BH rectangle of output
//                  pixels of one image, and the A block for filter tap (kh,kw), channel chunk c0 is the SAME rectangle of the
//                  NHWC input shifted by (kh-pad, kw-pad) — one 4-D tiled TMA load whose out-of-bounds rows/columns (the conv zero
//                  padding, and ragged tile edges) are zero-filled by the TMA unit.  Stride-2 convs on even maps use a 5-D view
//                  (c', w/2, h&1, h/2, b) of the same tensor so that every tap is again a dense box.  That view cannot describe an odd
//                  H or W, so 3x3 stride-2 convs on odd maps use the 4-D (c, w, h, b) view with traversal strides {1, 2, 2, 1}: tap
//                  (kh,kw) is the box at (2*w0 + kw - pad, 2*h0 + kh - pad) taking every other pixel, zero-filled against the true
//                  W x H, and it lands as the same dense smem tile.  1x1 convs and linears are the
//                  degenerate W = M, H = 1 case.  Smem tiles land in the canonical K-major SWIZZLE_128B (or _64B for 32-channel
//                  chunks) layout wgmma reads through its shared-memory descriptors.  After a tile's last k-block the producer loads
//                  the tile's residual (if any) into the next ring entries, so it is in flight while the consumers finish the previous tile.
//   warp-groups 1-2  consumers: group g owns tile rows 64g..64g+63.  Per k-block it issues BLOCK_K/16 x wgmma.m64nBLOCK_Nk16
//                  into its register accumulator and releases the ring stage once they have retired (wgmma.wait_group 1 in the next
//                  k-block).  In the fp32-accurate fused-split mode a step is three products; at BLOCK_N = 128 they take A from registers
//                  (A_hi and A_lo loaded by ldmatrix), one wgmma group per step.  The epilogue of its rows follows: folded-BN scale/bias, residual (before
//                  or after the activation), ReLU/SiLU/GELU -> fp16/fp32/pair -> swizzled smem staging (double buffered, shared by
//                  both groups) -> TMA store (clips ragged tiles / Cout tails).  The producer keeps filling the ring with the next
//                  tile's operands meanwhile.
//
// Algorithmic bytes: A (M x Cin, each input pixel counted once), W, D (+ residual) once each.
#include <cuda.h>

#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace fb200 {

namespace tc {

constexpr int BLOCK_M = 128;
constexpr int STAGING_BYTES = BLOCK_M * 128;  // one staging tile: 128 rows x 128 B
constexpr int NUM_THREADS = 384;              // producer warp-group + two consumer warp-groups
constexpr int CONSUMER_WARPS = 8;

// Output / residual stored as the fp16 [hi | lo] PAIR of the fp32 value (hi = fp16(v), lo = fp16(v - hi)): the operand format of the fp32-accurate convs,
// written straight from the epilogue so that no separate split pass runs between two convs.  sizeof == 4: a staging chunk is 32 columns like fp32, laid out as
// two dense [128 rows x 64 B] tiles (hi, then lo at +8 KiB), 64-byte swizzle, each stored / loaded with its own tensor map.
struct PairOut { __half hi, lo; };
template <typename T> struct is_pair { static constexpr bool value = false; };
template <> struct is_pair<PairOut> { static constexpr bool value = true; };

struct KParams {
  const float* scale; const float* bias; const void* res;
  int act, Cout;
  int KH, KW, pad, cchunks;        // cchunks = C / BLOCK_K, C = channels of the input (split-precision: of one of its [hi | lo] planes)
  int w_batched;                   // 1: weights differ per image (3-D weight map, third coordinate = image)
  int lo_off;                      // split-precision: channel offset of the A operand's lo half (C unless the input is a channel slice of a wider pair buffer)
  int w_seg;                       // split-precision: channels per weight segment ([W_hi | W_lo | W_hi] per tap)
  int BW, BH, tiles_w, tiles_h;    // output tile rectangle and tile counts per image
  int Ho, Wo;                      // output spatial size (validity of rows)
  int x_pitch;                     // stride-2 view only (c' = wp * pitch + c)
  int stride2;                     // 0: 4-D stride-1 view, 1: 5-D stride-2 view (even maps), 2: 4-D view with traversal stride 2 (odd maps)
  int num_k_blocks;
  int n_tiles, total_tiles;        // N tiles per M tile; total = m_tiles * n_tiles
  float* rowmax;                   // not null: row-max-only epilogue (query selection scores), nothing is stored
};

__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// K-major swizzled shared-memory matrix descriptor (sm_90 format: layout type at bits 62-63, 1 = SWIZZLE_128B, 2 = SWIZZLE_64B)
template <int BLOCK_K>
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);   // start address, 16-byte units
  d |= (uint64_t)1 << 16;                         // leading byte offset (unused for swizzled K-major) = 1
  d |= (uint64_t)((8 * BLOCK_K * 2) >> 4) << 32;  // stride byte offset: 8 rows x (BLOCK_K*2) B
  d |= (uint64_t)(BLOCK_K == 64 ? 1 : 2) << 62;
  return d;
}

template <bool GELU>
__device__ __forceinline__ float act1(float v, int act) {
  if constexpr (GELU) return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));  // exact-erf GELU (AIFI FFN only): its own instantiation
  switch (act & 15) {
    case FB200_ACT_RELU: return fmaxf(v, 0.f);
    case FB200_ACT_SILU: return __fdividef(v, 1.f + __expf(-v));
    default: return v;
  }
}

// max of floats through integer atomics (buffer initialised to -inf): non-negative values order like ints, negative ones like reversed uints
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
  if (v >= 0.f) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
  else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

// ---------------------------------------------------------------------------------------------- epilogue pieces of both kernels
// A consumer thread's place in the 128-row accumulator tile (fragment layout: wgmma.cuh)
struct AccThread {
  int ct;  // consumer thread 0..255; thread 0 issues the TMA stores
  int g;   // warp-group: tile rows 64g .. 64g + 63
  int r0;  // accumulator rows r0 and r0 + 8 of this thread
  int cq;  // first of the two adjacent accumulator columns
};
__device__ __forceinline__ AccThread acc_thread() {
  const int ct = threadIdx.x - 128, lane = threadIdx.x & 31;
  return {ct, ct >> 7, (ct >> 7) * 64 + ((ct & 127) >> 5) * 16 + (lane >> 2), 2 * (lane & 3)};
}

// Byte offset of (row, lc = column inside the chunk) in a swizzled staging tile - the layout a TMA store reads and a residual box lands in: the 16-byte piece
// index XOR the row phase.  A pair has two planes of 64-byte rows (64-byte swizzle), the same offset in each; fp16 and fp32 have 128-byte rows.
template <typename TOut>
__device__ __forceinline__ int staging_offset(int row, int lc) {
  if constexpr (is_pair<TOut>::value) return row * 64 + ((((lc >> 3) ^ ((row >> 1) & 3)) << 4) | ((lc & 7) * 2));
  else if constexpr (sizeof(TOut) == 2) return row * 128 + ((((lc >> 3) ^ (row & 7)) << 4) | ((lc & 7) * 2));
  else return row * 128 + ((((lc >> 2) ^ (row & 7)) << 4) | ((lc & 3) * 4));
}

// the adjacent columns (v0, v1) -> the staging tile at `off`; a pair is split again: hi = fp16(v), lo = fp16(v - hi) on the second plane
template <typename TOut>
__device__ __forceinline__ void staging_store(uint8_t* stg, int off, float v0, float v1) {
  if constexpr (is_pair<TOut>::value) {
    const __half2 hi = __floats2half2_rn(v0, v1);
    const float2 hf = __half22float2(hi);
    *reinterpret_cast<__half2*>(stg + off) = hi;
    *reinterpret_cast<__half2*>(stg + STAGING_BYTES / 2 + off) = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
  } else if constexpr (sizeof(TOut) == 2) {
    *reinterpret_cast<__half2*>(stg + off) = __floats2half2_rn(v0, v1);
  } else {
    *reinterpret_cast<float2*>(stg + off) = make_float2(v0, v1);
  }
}

// The consumers write a staging buffer between staging_open and staging_close.  open: thread 0 waits until the TMA store that last used the buffer
// (NSTG chunks ago) has finished READING it and runs `then` (what else it must start once the buffer is free), then the consumers meet.
template <int NSTG, typename F>
__device__ __forceinline__ void staging_open(int ct, F&& then) {
  if (ct == 0) {
    tma_store_wait_read<NSTG - 1>();
    then();
  }
  consumer_bar();
}
// close: every consumer's writes are made visible to the TMA unit, the consumers meet, and thread 0 stores the chunk at channel n of the tile at
// (w0, h0, img) - both planes of a pair - as one bulk group; the TMA unit clips ragged tiles, and Cout tails to whole 16-byte pieces (so
// conv2d_tc_supported takes only Cout that end on one)
template <typename TOut>
__device__ __forceinline__ void staging_close(int ct, const uint8_t* stg, const CUtensorMap* tmap_d, const CUtensorMap* tmap_d2, int n, int w0, int h0, int img) {
  fence_proxy_async();
  consumer_bar();
  if (ct == 0) {
    tma_store_4d(tmap_d, stg, n, w0, h0, img);
    if constexpr (is_pair<TOut>::value) tma_store_4d(tmap_d2, stg + STAGING_BYTES / 2, n, w0, h0, img);
    tma_store_commit();
  }
}

// FS ("fused split", fp32-accurate mode): one ring stage holds the hi AND lo halves of both operands of a channel chunk - A_hi, A_lo, B_hi, B_lo are loaded ONCE
// and feed the three products hi x W_hi, hi x W_lo, lo x W_hi
template <int BLOCK_K, bool FS> __host__ __device__ constexpr int a_stage_bytes() { return (FS ? 2 : 1) * BLOCK_M * BLOCK_K * 2; }
template <int BLOCK_N, int BLOCK_K, bool FS> __host__ __device__ constexpr int b_stage_bytes() { return (FS ? 2 : 1) * BLOCK_N * BLOCK_K * 2; }
template <int BLOCK_N, int STAGES, int BLOCK_K, int NSTG, bool FS> constexpr int smem_bytes() {
  return STAGES * (a_stage_bytes<BLOCK_K, FS>() + b_stage_bytes<BLOCK_N, BLOCK_K, FS>()) + NSTG * STAGING_BYTES + (2 * STAGES + 1) * 8 + 1024 /*align slack*/;
}

// The FS products of the N = 128 configurations take A from registers: each warp loads A_hi and A_lo of its 16 rows once per 16-channel step with ldmatrix
// and feeds both A_hi products from the same fragment, where descriptors would have the tensor pipe read A_hi from shared memory twice.
// Byte offset of the row this lane hands ldmatrix_x4 for the A fragment of rows row0 .. row0 + 15, channels 16k .. 16k + 15, inside an operand tile of
// BLOCK_K channels.  The ring's tiles have the staging tiles' swizzles (64 channels: 128-byte rows like fp16 staging; 32 channels: 64-byte rows like a pair
// plane), and every tile starts on a multiple of the swizzle's repeat.
template <int BLOCK_K>
__device__ __forceinline__ uint32_t a_frag_offset(int row0, int k, int lane) {
  typedef std::conditional_t<BLOCK_K == 64, __half, PairOut> Layout;
  return (uint32_t)staging_offset<Layout>(row0 + (lane & 15), 16 * k + 8 * (lane >> 4));
}

// One 16-channel FS step as one wgmma group: ldmatrix A_hi and A_lo at a_hi / a_lo into fr, then hi x W_hi, hi x W_lo, lo x W_hi.  Callers alternate two
// fragment buffers; the wait retires the previous step's group, so the other buffer may be reloaded while this step's products run.
template <int BLOCK_N>
__device__ __forceinline__ void fs_step(float (&acc)[BLOCK_N / 2], uint32_t (&fr)[2][4], uint32_t a_hi, uint32_t a_lo, uint64_t db_hi, uint64_t db_lo,
                                        uint32_t scale_d) {
  ldmatrix_x4(fr[0], a_hi);
  ldmatrix_x4(fr[1], a_lo);
  wgmma_fence();
  WgmmaRS<BLOCK_N>::mma(acc, fr[0], db_hi, scale_d);
  WgmmaRS<BLOCK_N>::mma(acc, fr[0], db_lo, 1u);
  WgmmaRS<BLOCK_N>::mma(acc, fr[1], db_hi, 1u);
  wgmma_commit();
  wgmma_wait<1>();
}

// ---------------------------------------------------------------------------------------------- kernel
template <int BLOCK_N, int STAGES, typename TOut, int BLOCK_K, int NSTG, bool GELU, bool FS>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const __grid_constant__ CUtensorMap tmap_d, const __grid_constant__ CUtensorMap tmap_r,
               const __grid_constant__ CUtensorMap tmap_d2, const __grid_constant__ CUtensorMap tmap_r2, const KParams p) {
  constexpr bool PAIR = is_pair<TOut>::value;  // tmap_d2 / tmap_r2: the lo planes of the output / residual (pair format only)
  static_assert(BLOCK_K == 32 || BLOCK_K == 64, "one swizzle row per channel chunk");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int A_STAGE_BYTES = a_stage_bytes<BLOCK_K, FS>();
  constexpr int B_STAGE_BYTES = b_stage_bytes<BLOCK_N, BLOCK_K, FS>();
  constexpr int A_HALF = BLOCK_M * BLOCK_K * 2;   // FS: bytes of one A half (hi or lo) inside a stage
  constexpr int B_HALF = BLOCK_N * BLOCK_K * 2;   // FS: bytes of one B half
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;
  uint8_t* staging = smem_b + STAGES * B_STAGE_BYTES;  // NSTG x 16 KiB
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + NSTG * STAGING_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* res_bar = empty_bar + STAGES;  // residual chunk landed in the staging buffer (configurations without ring slots only)

  // Residual tile: a 16 KiB box per staging chunk (CHUNK_COLS columns x 128 rows).  Where a ring stage has room for such boxes (A part first, then B part),
  // the producer loads the whole residual tile into the ring entries that follow the tile's last k-block, so it is in flight while the previous tile's
  // epilogue runs; the consumers release each entry after reading its last chunk.  The 32-channel non-split stages (8 KiB parts) have no room: there
  // one consumer thread loads each chunk into the staging buffer inside the epilogue.
  constexpr int CHUNK_COLS = 128 / (int)sizeof(TOut);  // output columns per 128-byte staging row
  constexpr int NCHUNKS = (BLOCK_N + CHUNK_COLS - 1) / CHUNK_COLS;
  constexpr int RES_SLOTS_A = A_STAGE_BYTES / STAGING_BYTES;
  constexpr int RES_SLOTS = RES_SLOTS_A + B_STAGE_BYTES / STAGING_BYTES;  // residual chunks per ring entry
  constexpr bool RES_RING = RES_SLOTS > 0;
  const bool res_ring = RES_RING && p.res != nullptr && p.rowmax == nullptr;
  auto res_slot = [&](int s, int slot) -> uint8_t* {
    return slot < RES_SLOTS_A ? smem_a + s * A_STAGE_BYTES + slot * STAGING_BYTES : smem_b + s * B_STAGE_BYTES + (slot - RES_SLOTS_A) * STAGING_BYTES;
  };
  // chunks of the N tile at n0 that hold output columns (the Cout tail of the last N tile has fewer)
  auto chunks_of = [&](int n0) { return min(NCHUNKS, (p.Cout - n0 + CHUNK_COLS - 1) / CHUNK_COLS); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_b) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_d) : "memory");
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], CONSUMER_WARPS); }
    if constexpr (!RES_RING) mbar_init(res_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  const int tiles_per_img = p.tiles_w * p.tiles_h;
  struct TileXY { int n0, img, h0, w0; };
  auto tile_of = [&](int t) {
    TileXY r;
    r.n0 = (t % p.n_tiles) * BLOCK_N;
    const int mt = t / p.n_tiles;
    r.img = mt / tiles_per_img;
    const int rem = mt - r.img * tiles_per_img;
    r.h0 = (rem / p.tiles_w) * p.BH;
    r.w0 = (rem % p.tiles_w) * p.BW;
    return r;
  };

  if (warp < 4) {
    // ===================================================================== TMA producer
    if (threadIdx.x != 0) return;
    const uint32_t a_bytes = (uint32_t)(p.BW * p.BH * BLOCK_K * 2);
    auto load_a = [&](uint64_t* bar, void* dst, int c, int kh, int kw, int h0, int w0, int img) {
      if (!p.stride2) {
        tma_load_4d(&tmap_a, bar, dst, c, w0 + kw - p.pad, h0 + kh - p.pad, img);
      } else if (p.stride2 == 2) {  // every other pixel of a 2BW x 2BH box from the tap's first input pixel
        tma_load_4d(&tmap_a, bar, dst, c, 2 * w0 + kw - p.pad, 2 * h0 + kh - p.pad, img);
      } else {
        // input h = 2*ho + kh - pad -> (h>>1, h&1).  3x3/pad 1: kh=0 -> (ho-1,1); 1 -> (ho,0); 2 -> (ho,1).  2x2/pad 0: kh -> (ho,kh)
        const int th = kh - p.pad, tw = kw - p.pad;  // arithmetic shift: -1 -> (-1, 1)
        tma_load_5d(&tmap_a, bar, dst, (tw & 1) * p.x_pitch + c, w0 + (tw >> 1), th & 1, h0 + (th >> 1), img);
      }
    };
    auto load_b = [&](uint64_t* bar, void* dst, int k, int n0, int img) {
      if (p.w_batched) tma_load_3d(&tmap_b, bar, dst, k, n0, img);  // per-image weights (the mask product of the MaskFormer-family heads)
      else tma_load_2d(&tmap_b, bar, dst, k, n0);
    };
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
      const TileXY tc = tile_of(t);
      // No L2 prefetch of the next tile's A: every CTA of the persistent grid would pull a whole tile ahead (256 KiB of A for a 512-channel pair input),
      // about as much again as the tiles in flight, into the 50 MB L2.  On H100 that made the HBM-bound 1x1 convs slower (1x1 512->128 @80^2: 0.27 ms without, 0.34 with).
      for (int kb = 0; kb < p.num_k_blocks; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        const int tap = kb / p.cchunks, cc = kb - tap * p.cchunks;
        const int kh = tap / p.KW, kw = tap - kh * p.KW;
        uint8_t* dst_a = smem_a + stage * A_STAGE_BYTES;
        uint8_t* dst_b = smem_b + stage * B_STAGE_BYTES;
        if constexpr (FS) {  // the stored input is [hi(C) | lo(C)]; k-block = (tap, channel chunk): A_hi, A_lo, W_hi, W_lo once each
          const int k_hi = tap * 3 * p.w_seg + cc * BLOCK_K, k_lo = k_hi + p.w_seg;  // weights packed [W_hi | W_lo | W_hi] per tap
          mbar_arrive_expect_tx(&full_bar[stage], 2u * a_bytes + (uint32_t)B_STAGE_BYTES);
          load_a(&full_bar[stage], dst_a, cc * BLOCK_K, kh, kw, tc.h0, tc.w0, tc.img);
          load_a(&full_bar[stage], dst_a + A_HALF, p.lo_off + cc * BLOCK_K, kh, kw, tc.h0, tc.w0, tc.img);
          load_b(&full_bar[stage], dst_b, k_hi, tc.n0, tc.img);
          load_b(&full_bar[stage], dst_b + B_HALF, k_lo, tc.n0, tc.img);
        } else {
          mbar_arrive_expect_tx(&full_bar[stage], a_bytes + (uint32_t)B_STAGE_BYTES);
          load_a(&full_bar[stage], dst_a, cc * BLOCK_K, kh, kw, tc.h0, tc.w0, tc.img);
          load_b(&full_bar[stage], dst_b, kb * BLOCK_K, tc.n0, tc.img);
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      if constexpr (RES_RING) if (res_ring) {  // the residual tile: RES_SLOTS chunk boxes per ring entry
        const int nch = chunks_of(tc.n0);
        for (int ch = 0; ch < nch; ++ch) {
          const int slot = ch % RES_SLOTS;
          if (slot == 0) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)(min(RES_SLOTS, nch - ch) * p.BW * p.BH * 128));
          }
          uint8_t* dst = res_slot(stage, slot);
          tma_load_4d(&tmap_r, &full_bar[stage], dst, tc.n0 + ch * CHUNK_COLS, tc.w0, tc.h0, tc.img);
          if constexpr (PAIR) tma_load_4d(&tmap_r2, &full_bar[stage], dst + STAGING_BYTES / 2, tc.n0 + ch * CHUNK_COLS, tc.w0, tc.h0, tc.img);
          if (slot == RES_SLOTS - 1 || ch == nch - 1) {
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ===================================================================== consumers: wgmma main loop + epilogue
  const AccThread th = acc_thread();
  constexpr int NACC = BLOCK_N / 2;
  const bool post = (p.act & FB200_ACT_RESIDUAL_AFTER) != 0;
  const bool has_res = p.res != nullptr;
  float acc[NACC];
  // The fused-split products take A from registers at N = 128 only.  At N = 64 a step's products are too short for it: the register form gained nothing on
  // those convs (-1% to +4% in five sessions, H100 80GB HBM3, 700 W), and it slowed the small-channel kernel's N = 32 / 64 products.
  constexpr bool RS = FS && BLOCK_N == 128;
  uint32_t frag[2][2][4];  // RS: two buffers of this warp's (A_hi, A_lo) fragments
  int stage = 0;
  uint32_t phase = 0, res_phase = 0, chunk_ctr = 0;
  for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
    const TileXY tc = tile_of(t);
    int prev = -1;
    for (int kb = 0; kb < p.num_k_blocks; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem_a + stage * A_STAGE_BYTES) + (uint32_t)(th.g * 64 * BLOCK_K * 2);
      const uint32_t sb = smem_u32(smem_b + stage * B_STAGE_BYTES);
      const uint64_t db = make_smem_desc<BLOCK_K>(sb);
      if constexpr (RS) {  // hi x W_hi, hi x W_lo, lo x W_hi into the same fp32 accumulator, one group per step
        const uint64_t db_lo = make_smem_desc<BLOCK_K>(sb + B_HALF);
        const int row0 = ((th.ct & 127) >> 5) * 16;
#pragma unroll
        for (int k = 0; k < BLOCK_K / 16; ++k) {  // an even number of steps: step 0 of the next k-block takes buffer 0 again
          const uint32_t ao = a_frag_offset<BLOCK_K>(row0, k, lane);
          fs_step<BLOCK_N>(acc, frag[k & 1], sa + ao, sa + A_HALF + ao, db + (uint64_t)(k * 2), db_lo + (uint64_t)(k * 2), (kb > 0 || k > 0) ? 1u : 0u);
          // at k = 0 the previous k-block's last group has retired: its stage may be refilled
          if (k == 0 && prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        }
      } else {
        const uint64_t da = make_smem_desc<BLOCK_K>(sa);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / 16; ++k) {
          // advance 16 halves = 32 B inside the swizzle row: +2 in 16-byte units
          const uint64_t ko = (uint64_t)(k * 2);
          Wgmma<BLOCK_N, 0>::mma(acc, da + ko, db + ko, (kb > 0 || k > 0) ? 1u : 0u);
          if constexpr (FS) {  // hi x W_lo, lo x W_hi into the same fp32 accumulator
            const uint64_t da_lo = make_smem_desc<BLOCK_K>(sa + A_HALF), db_lo = make_smem_desc<BLOCK_K>(sb + B_HALF);
            Wgmma<BLOCK_N, 0>::mma(acc, da + ko, db_lo + ko, 1u);
            Wgmma<BLOCK_N, 0>::mma(acc, da_lo + ko, db + ko, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's products are done: its stage may be refilled
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);

    auto scale_of = [&](int n) { return (p.scale && n < p.Cout) ? __ldg(p.scale + n) : 1.f; };
    auto bias_of = [&](int n) { return (p.bias && n < p.Cout) ? __ldg(p.bias + n) : 0.f; };
    auto row_valid = [&](int row, int64_t& pix) {
      const int bh = row / p.BW, bw = row - bh * p.BW;
      const int ho = tc.h0 + bh, wo = tc.w0 + bw;
      pix = ((int64_t)tc.img * p.Ho + ho) * p.Wo + wo;
      return row < p.BW * p.BH && ho < p.Ho && wo < p.Wo;
    };
    if (p.rowmax) {  // row-max-only epilogue: enc_outputs_class.max(-1) without materialising the [B*S, num_classes] logits
      float m[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int n = tc.n0 + 8 * j + th.cq + e;
          if (n < p.Cout) {
            const float s = scale_of(n), b = bias_of(n);
            m[0] = fmaxf(m[0], fmaf(acc[4 * j + e], s, b));
            m[1] = fmaxf(m[1], fmaf(acc[4 * j + 2 + e], s, b));
          }
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 1));
        m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 2));
        int64_t pix;
        if ((lane & 3) == 0 && row_valid(th.r0 + 8 * h, pix)) atomic_max_float(p.rowmax + pix, m[h]);
      }
      continue;
    }
    const int nch = chunks_of(tc.n0);
#pragma unroll
    for (int ch = 0; ch < NCHUNKS; ++ch) {
      const int c0 = ch * CHUNK_COLS;
      if (ch >= nch) break;  // uniform across the consumers
      uint8_t* stg = staging + (chunk_ctr % NSTG) * STAGING_BYTES;
      const uint8_t* res = stg;  // residual chunk, same swizzled layout as the staging tile
      staging_open<NSTG>(th.ct, [&] {
        if constexpr (!RES_RING) if (has_res) {  // the [BW x BH x CHUNK_COLS] residual box lands in the staging buffer; each thread adds and overwrites its own elements
          mbar_arrive_expect_tx(res_bar, (uint32_t)(p.BW * p.BH * 128));
          tma_load_4d(&tmap_r, res_bar, stg, tc.n0 + c0, tc.w0, tc.h0, tc.img);
          if constexpr (PAIR) tma_load_4d(&tmap_r2, res_bar, stg + STAGING_BYTES / 2, tc.n0 + c0, tc.w0, tc.h0, tc.img);
        }
      });
      if constexpr (RES_RING) {
        if (res_ring) {
          if (ch % RES_SLOTS == 0) mbar_wait(&full_bar[stage], phase);
          res = res_slot(stage, ch % RES_SLOTS);
        }
      } else if (has_res) {
        mbar_wait(res_bar, res_phase);
        res_phase ^= 1;
      }
#pragma unroll
      for (int jj = 0; jj < CHUNK_COLS / 8; ++jj) {
        const int j = c0 / 8 + jj;
        if (j >= BLOCK_N / 8) break;
        const int lc = 8 * jj + th.cq;  // column inside the chunk
        const int n = tc.n0 + c0 + lc;
        const float s0 = scale_of(n), s1 = scale_of(n + 1), b0 = bias_of(n), b1 = bias_of(n + 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = th.r0 + 8 * h;
          float v0 = fmaf(acc[4 * j + 2 * h], s0, b0), v1 = fmaf(acc[4 * j + 2 * h + 1], s1, b1);
          const int off = staging_offset<TOut>(row, lc);
          auto add_residual = [&]() {
            if (!has_res) return;
            if constexpr (PAIR) {
              const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(res + off));
              const float2 fl = __half22float2(*reinterpret_cast<const __half2*>(res + STAGING_BYTES / 2 + off));
              v0 += fh.x + fl.x;
              v1 += fh.y + fl.y;
            } else if constexpr (sizeof(TOut) == 2) {
              const float2 f = __half22float2(*reinterpret_cast<const __half2*>(res + off));
              v0 += f.x;
              v1 += f.y;
            } else {
              const float2 f = *reinterpret_cast<const float2*>(res + off);
              v0 += f.x;
              v1 += f.y;
            }
          };
          if (!post) add_residual();
          v0 = act1<GELU>(v0, p.act);
          v1 = act1<GELU>(v1, p.act);
          if (post) add_residual();
          staging_store<TOut>(stg, off, v0, v1);
        }
      }
      if constexpr (RES_RING) {
        if (res_ring && (ch % RES_SLOTS == RES_SLOTS - 1 || ch == nch - 1)) {  // last chunk of this ring entry read by the whole warp: release it
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
      staging_close<TOut>(th.ct, stg, &tmap_d, &tmap_d2, tc.n0 + c0, tc.w0, tc.h0, tc.img);
      ++chunk_ctr;
    }
  }
  if (th.ct == 0) tma_store_wait_all();
}

// ---------------------------------------------------------------------------------------------- small-channel 3x3 fused-split kernel
// 3x3 / stride 1 / pad 1 fp32-accurate convs with 32 input channels and 32 or 64 output channels (the ResNet-vd stem's conv1_2 and conv1_3).  The
// general kernel streams A_hi, A_lo, W_hi, W_lo through its ring once per filter tap.  Here BLOCK_N = Cout and the whole [W_hi | W_lo] (9 taps x 2 x
// Cout x 64 B: 36 or 72 KiB) is loaded into shared memory once, at kernel start, and an output tile takes ONE ring entry: three kw-shifted boxes of
// SC_BW x (SC_BH + 2) input pixels per plane.  Tap (kh, kw) is box kw from pixel row kh * SC_BW on, a 128-row operand whose start is a multiple of the
// 512-byte repeat of the 64-byte swizzle, so the usual descriptors address it.  That is 3 x 160 instead of 9 x 128 A rows per tile and no weights in the
// stream.  Products run in the general kernel's order (tap, 16-channel step, then hi x W_hi, hi x W_lo, lo x W_hi) with N = Cout, so the outputs are the
// same bits.  Same warp roles and epilogue (folded BN, activation, fp32 or pair output through TMA stores) without residual or row-max.
// A stays in shared memory, as in the general kernel's N = 64 configurations: the register form (with two or four fragment buffers) made conv1_2 and
// conv1_3 4-11% slower (H100 80GB HBM3, 700 W).
constexpr int SC_BW = 16, SC_BH = 8;                 // output tile: 16 x 8 pixels = BLOCK_M rows
constexpr int SC_BOX_ROWS = SC_BW * (SC_BH + 2);     // one kw-shifted input box
constexpr int SC_BOX_BYTES = SC_BOX_ROWS * 64;       // 32 channels of fp16: 64-byte rows, 64-byte swizzle
constexpr int SC_STAGE_BYTES = 2 * 3 * SC_BOX_BYTES;  // hi and lo planes x three kw shifts: 60 KiB
constexpr int SC_STAGES = 2;
template <int BLOCK_N> __host__ __device__ constexpr int sc_w_bytes() { return 9 * 2 * BLOCK_N * 64; }
template <int BLOCK_N> constexpr int sc_smem_bytes() {
  return sc_w_bytes<BLOCK_N>() + SC_STAGES * SC_STAGE_BYTES + 2 * STAGING_BYTES + (2 * SC_STAGES + 1) * 8 + 1024 /*align slack*/;
}

template <int BLOCK_N, typename TOut>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_tc_smallc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                      const __grid_constant__ CUtensorMap tmap_d, const __grid_constant__ CUtensorMap tmap_d2, const KParams p) {
  constexpr int W_BYTES = sc_w_bytes<BLOCK_N>();
  constexpr int W_TAP = 2 * BLOCK_N * 64;  // [W_hi | W_lo] of one tap
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_w = smem;
  uint8_t* smem_a = smem_w + W_BYTES;
  uint8_t* staging = smem_a + SC_STAGES * SC_STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + 2 * STAGING_BYTES);
  uint64_t* empty_bar = full_bar + SC_STAGES;
  uint64_t* w_bar = empty_bar + SC_STAGES;
  constexpr int CHUNK_COLS = 32;  // pair and fp32 staging rows alike
  constexpr int NCHUNKS = BLOCK_N / CHUNK_COLS;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_d) : "memory");
    for (int i = 0; i < SC_STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], CONSUMER_WARPS); }
    mbar_init(w_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  const int tiles_per_img = p.tiles_w * p.tiles_h;
  struct TileXY { int img, h0, w0; };
  auto tile_of = [&](int t) {  // BLOCK_N = Cout: one N tile
    TileXY r;
    r.img = t / tiles_per_img;
    const int rem = t - r.img * tiles_per_img;
    r.h0 = (rem / p.tiles_w) * SC_BH;
    r.w0 = (rem % p.tiles_w) * SC_BW;
    return r;
  };

  if (warp < 4) {
    // ===================================================================== TMA producer
    if (threadIdx.x != 0) return;
    mbar_arrive_expect_tx(w_bar, (uint32_t)W_BYTES);
    for (int tap = 0; tap < 9; ++tap) {  // weights packed [W_hi | W_lo | W_hi] per tap
      tma_load_2d(&tmap_b, w_bar, smem_w + tap * W_TAP, tap * 3 * p.w_seg, 0);
      tma_load_2d(&tmap_b, w_bar, smem_w + tap * W_TAP + W_TAP / 2, tap * 3 * p.w_seg + p.w_seg, 0);
    }
    int stage = 0;
    uint32_t phase = 0;
    for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
      const TileXY tc = tile_of(t);
      mbar_wait(&empty_bar[stage], phase ^ 1);
      mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)SC_STAGE_BYTES);
      uint8_t* dst = smem_a + stage * SC_STAGE_BYTES;
      for (int kw = 0; kw < 3; ++kw) {  // box kw: input pixels (h0 - 1 .. h0 + SC_BH, w0 + kw - 1 ..); the TMA unit zero-fills the padding
        tma_load_4d(&tmap_a, &full_bar[stage], dst + kw * SC_BOX_BYTES, 0, tc.w0 + kw - 1, tc.h0 - 1, tc.img);
        tma_load_4d(&tmap_a, &full_bar[stage], dst + (3 + kw) * SC_BOX_BYTES, p.lo_off, tc.w0 + kw - 1, tc.h0 - 1, tc.img);
      }
      if (++stage == SC_STAGES) { stage = 0; phase ^= 1; }
    }
    return;
  }

  // ===================================================================== consumers: wgmma over the nine taps of one patch + epilogue
  const AccThread th = acc_thread();
  float acc[BLOCK_N / 2];
  float sc[BLOCK_N / 4], bi[BLOCK_N / 4];  // folded BN of this thread's columns, the same for every tile
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int n = 8 * j + th.cq + e;
      sc[2 * j + e] = p.scale ? __ldg(p.scale + n) : 1.f;
      bi[2 * j + e] = p.bias ? __ldg(p.bias + n) : 0.f;
    }
  mbar_wait(w_bar, 0);
  const uint32_t sw = smem_u32(smem_w);
  int stage = 0;
  uint32_t phase = 0, chunk_ctr = 0;
  for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
    const TileXY tc = tile_of(t);
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sa = smem_u32(smem_a + stage * SC_STAGE_BYTES) + (uint32_t)(th.g * 64 * 64);
    wgmma_fence();
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int kh = tap / 3, kw = tap - 3 * (tap / 3);
      const uint32_t a_tap = sa + (uint32_t)(kw * SC_BOX_BYTES + kh * SC_BW * 64);
      const uint64_t da = make_smem_desc<32>(a_tap), da_lo = make_smem_desc<32>(a_tap + 3 * SC_BOX_BYTES);
      const uint64_t db = make_smem_desc<32>(sw + tap * W_TAP), db_lo = make_smem_desc<32>(sw + tap * W_TAP + W_TAP / 2);
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const uint64_t ko = (uint64_t)(k * 2);
        Wgmma<BLOCK_N, 0>::mma(acc, da + ko, db + ko, (tap > 0 || k > 0) ? 1u : 0u);
        Wgmma<BLOCK_N, 0>::mma(acc, da + ko, db_lo + ko, 1u);
        Wgmma<BLOCK_N, 0>::mma(acc, da_lo + ko, db + ko, 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);  // the producer refills this entry with a later tile's patch while the epilogue runs
    if (++stage == SC_STAGES) { stage = 0; phase ^= 1; }

#pragma unroll
    for (int ch = 0; ch < NCHUNKS; ++ch) {
      uint8_t* stg = staging + (chunk_ctr & 1) * STAGING_BYTES;
      staging_open<2>(th.ct, [] {});
#pragma unroll
      for (int jj = 0; jj < CHUNK_COLS / 8; ++jj) {
        const int j = ch * (CHUNK_COLS / 8) + jj;
        const int lc = 8 * jj + th.cq;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = th.r0 + 8 * h;
          const float v0 = act1<false>(fmaf(acc[4 * j + 2 * h], sc[2 * j], bi[2 * j]), p.act);
          const float v1 = act1<false>(fmaf(acc[4 * j + 2 * h + 1], sc[2 * j + 1], bi[2 * j + 1]), p.act);
          staging_store<TOut>(stg, staging_offset<TOut>(row, lc), v0, v1);
        }
      }
      staging_close<TOut>(th.ct, stg, &tmap_d, &tmap_d2, ch * CHUNK_COLS, tc.w0, tc.h0, tc.img);
      ++chunk_ctr;
    }
  }
  if (th.ct == 0) tma_store_wait_all();
}

// ---------------------------------------------------------------------------------------------- host
// best output rectangle (BW x BH <= 128 pixels) for an Ho x Wo map
static void choose_tile(int Ho, int Wo, int* BW, int* BH) {
  double best = -1.0;
  for (int bw = 1; bw <= (Wo < 128 ? Wo : 128); ++bw) {
    int bh = 128 / bw;
    if (bh > Ho) bh = Ho;
    if (bh < 1) continue;
    const double tiles = (double)((Wo + bw - 1) / bw) * (double)((Ho + bh - 1) / bh);
    const double eff = (double)Wo * Ho / (tiles * 128.0);
    if (eff > best + 1e-9 || (eff > best - 1e-9 && bw > *BW)) { best = eff; *BW = bw; *BH = bh; }
  }
}

// Tensor maps of the output (d; d2 = the lo plane of a pair) and of the residual (r, r2), which has the output's format and geometry with its own pointer /
// pitch.  One box is a staging chunk of a BW x BH tile: 128-byte rows of fp16 / fp32, or per plane of a pair 32 channels with 64-byte swizzle (hi at `out`,
// lo `out_lo_off` elements further).  Maps the kernel does not read (no residual, no pair) are copies of d.
struct OutMaps { CUtensorMap d, d2, r, r2; };
static int encode_out_maps(OutMaps* m, const ConvParams& p, int Wo, int Ho, int B, int BW, int BH, uint64_t batch_stride) {
  const bool pair = p.out_dtype == FB200_F16PAIR, f32 = p.out_dtype == FB200_F32;
  const CUtensorMapDataType dt = f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  const int elt = f32 ? 4 : 2;
  const CUtensorMapSwizzle swz = pair ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
  const uint64_t OP = (uint64_t)p.out_pitch, RP = (uint64_t)p.res_pitch;
  const uint64_t dims[4] = {(uint64_t)p.Cout, (uint64_t)Wo, (uint64_t)Ho, (uint64_t)B};
  const uint64_t str[4] = {1, OP, OP * Wo, batch_stride}, rstr[4] = {1, RP, RP * Wo, RP * Wo * Ho};
  const uint32_t box[4] = {(uint32_t)(pair || f32 ? 32 : 64), (uint32_t)BW, (uint32_t)BH, 1};
  int rc = encode(&m->d, dt, elt, 4, p.out, dims, str, box, pair ? "conv_tc: D(hi)" : "conv_tc: D", swz);
  if (rc) return rc;
  m->d2 = m->d;
  if (pair) rc = encode(&m->d2, dt, elt, 4, static_cast<__half*>(p.out) + p.out_lo_off, dims, str, box, "conv_tc: D(lo)", swz);
  if (rc) return rc;
  m->r = m->d; m->r2 = m->d2;
  if (!p.res) return FB200_OK;
  rc = encode(&m->r, dt, elt, 4, const_cast<void*>(p.res), dims, rstr, box, pair ? "conv_tc: R(hi)" : "conv_tc: R", swz);
  if (rc || !pair) return rc;
  return encode(&m->r2, dt, elt, 4, const_cast<__half*>(static_cast<const __half*>(p.res)) + p.res_lo_off, dims, rstr, box, "conv_tc: R(lo)", swz);
}

// fused-split 3x3 / stride 1 / pad 1, Cin = 32, Cout = 32 or 64, no residual, fp32 or pair output
static bool smallc_fits(const ConvParams& p) {
  return p.split3 && p.Cin == 3 * 32 && (p.Cout == 32 || p.Cout == 64) && p.KH == 3 && p.KW == 3 && p.stride == 1 && p.pad == 1 &&
         !p.res && !p.rowmax && p.w_bs == 0 && (p.out_dtype == FB200_F32 || p.out_dtype == FB200_F16PAIR);
}

static int conv2d_tc_smallc(const ConvParams& p, cudaStream_t st) {
  KParams kp{};
  kp.scale = p.scale; kp.bias = p.bias; kp.act = p.act; kp.Cout = p.Cout;
  kp.lo_off = (int)p.x_lo_off;
  kp.w_seg = 32;
  kp.tiles_w = (p.Wo + SC_BW - 1) / SC_BW; kp.tiles_h = (p.Ho + SC_BH - 1) / SC_BH; kp.Ho = p.Ho; kp.Wo = p.Wo;
  const int64_t total = (int64_t)p.B * kp.tiles_w * kp.tiles_h;
  if (total > 0x7fffffffLL) { set_error("conv_tc: too many tiles (%lld)", (long long)total); return FB200_ERR_UNSUPPORTED; }
  kp.total_tiles = (int)total;
  CUtensorMap ta, tb;
  OutMaps om;
  const uint64_t P = (uint64_t)p.x_pitch;
  {
    const uint64_t dims[4] = {(uint64_t)kp.lo_off + 32, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.B};
    const uint64_t str[4] = {1, P, P * p.W, P * p.W * p.H};
    const uint32_t box[4] = {32, SC_BW, SC_BH + 2, 1};
    int rc = encode(&ta, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, const_cast<void*>(p.x), dims, str, box, "conv_tc: A(patch)", CU_TENSOR_MAP_SWIZZLE_64B);
    if (rc) return rc;
  }
  {
    const uint64_t dims[2] = {(uint64_t)p.K, (uint64_t)p.Cout};
    const uint64_t str[2] = {1, (uint64_t)p.K};
    const uint32_t box[2] = {32, (uint32_t)p.Cout};
    int rc = encode(&tb, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 2, const_cast<void*>(p.w), dims, str, box, "conv_tc: W", CU_TENSOR_MAP_SWIZZLE_64B);
    if (rc) return rc;
  }
  if (int rc = encode_out_maps(&om, p, p.Wo, p.Ho, p.B, SC_BW, SC_BH, (uint64_t)p.out_bs)) return rc;
  auto run = [&](auto blockn_tag, auto out_tag) -> int {
    constexpr int BN_ = decltype(blockn_tag)::value;
    return launch_persistent<conv_tc_smallc_kernel<BN_, decltype(out_tag)>, sc_smem_bytes<BN_>()>("conv_tc_smallc_kernel", kp.total_tiles, NUM_THREADS, st, ta, tb,
                                                                                                 om.d, om.d2, kp);
  };
  typedef std::integral_constant<int, 32> N32;
  typedef std::integral_constant<int, 64> N64;
  const bool outp = p.out_dtype == FB200_F16PAIR;
  if (p.Cout == 32) return outp ? run(N32{}, PairOut{}) : run(N32{}, float{});
  return outp ? run(N64{}, PairOut{}) : run(N64{}, float{});
}

}  // namespace tc

bool conv2d_tc_supported(const ConvParams& p, int x_dtype, int out_dtype) {
  if (x_dtype != FB200_F16) return false;
  if (out_dtype != FB200_F16 && out_dtype != FB200_F32 && out_dtype != FB200_F16PAIR) return false;
  if (p.split3 && out_dtype == FB200_F16) return false;  // split-precision convs write fp32 or the pair
  const int Clog = p.split3 ? p.Cin / 3 : p.Cin;  // channels of one K segment
  if (out_dtype == FB200_F16PAIR) {  // pair output: fused-split layers, planes 16-byte aligned
    if (!p.split3 || p.rowmax || p.w_bs != 0 || p.Cout % 8 != 0) return false;
    if ((p.out_lo_off * 2) % 16 != 0 || (p.out_pitch * 2) % 16 != 0 || (p.out_bs * 2) % 16 != 0) return false;
    if (p.res && ((p.res_lo_off * 2) % 16 != 0 || (p.res_pitch * 2) % 16 != 0 || p.Cout % 32 != 0)) return false;
  }
  if (p.split3 && (p.x_lo_off * 2) % 16 != 0) return false;
  if (Clog % 32 != 0 || p.x_pitch % 8 != 0) return false;
  if (p.split3 && p.Cin % 3 != 0) return false;
  if ((reinterpret_cast<uintptr_t>(p.x) | reinterpret_cast<uintptr_t>(p.w) | reinterpret_cast<uintptr_t>(p.out)) & 15) return false;
  const int oelt = out_dtype == FB200_F32 ? 4 : 2;   // element size of one stored plane
  if ((p.out_pitch * oelt) % 16 != 0) return false;
  // a TMA store clips the channel dimension only to whole 16-byte pieces: with a Cout tail inside one (365 fp32, 100 fp16 channels) it would also write
  // the columns up to the next 16-byte boundary, past the output view into the rest of the pitch.  The row-max epilogue stores nothing.
  if (!p.rowmax && (p.Cout * oelt) % 16 != 0) return false;
  if (p.res && ((p.res_pitch * oelt) % 16 != 0 || (reinterpret_cast<uintptr_t>(p.res) & 15))) return false;
  if (p.res && out_dtype != FB200_F16PAIR && p.Cout % (128 / oelt) != 0) return false;  // residual is consumed in whole 128-byte row chunks
  if (p.KH != p.KW) return false;
  if (p.w_bs != 0 && (p.w_bs * 2) % 16 != 0) return false;
  if ((p.act & 15) == FB200_ACT_GELU && (out_dtype != FB200_F16 || Clog % 64 != 0)) return false;
  if ((p.act & 15) == FB200_ACT_SIGMOID) return false;  // gates are [B, C] vectors: SIMT path
  if ((p.out_bs * oelt) % 16 != 0) return false;
  if (p.stride == 1) return (2 * p.pad == p.KH - 1) || (p.KH == 1 && p.pad == 0);
  if (p.stride == 2) {
    if (p.KH == 3 && p.pad == 1) return true;  // even maps: the 5-D parity view; odd H or W: the strided 4-D view (one box <= 256 per dimension: 2 * BW, 2 * BH)
    return p.KH == 2 && p.pad == 0 && p.H % 2 == 0 && p.W % 2 == 0;
  }
  return false;
}

int conv2d_tc(const ConvParams& p, cudaStream_t st) {
  using namespace tc;
  if (smallc_fits(p)) return conv2d_tc_smallc(p, st);  // fp32-accurate 3x3 with 32 input channels: resident weights, one input patch per tile
  KParams kp;
  kp.scale = p.scale; kp.bias = p.bias; kp.res = p.res; kp.act = p.act; kp.Cout = p.Cout;
  kp.KH = p.KH; kp.KW = p.KW; kp.pad = p.pad;
  const int Clog = p.split3 ? p.Cin / 3 : p.Cin;
  const int BK = (Clog % 64 == 0) ? 64 : 32;
  kp.lo_off = p.split3 ? (int)p.x_lo_off : Clog;
  kp.w_seg = Clog;
  const CUtensorMapSwizzle swz = BK == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  kp.cchunks = Clog / BK; kp.x_pitch = p.x_pitch;  // split-precision: a k-block is (tap, channel chunk) with the hi / lo halves of both operands together
  kp.stride2 = (p.stride != 2) ? 0 : (p.H % 2 == 0 && p.W % 2 == 0) ? 1 : 2;
  kp.num_k_blocks = p.KH * p.KW * kp.cchunks;
  // geometry: 1x1 stride-1 convs and linears flatten to W = M, H = 1, B = 1
  int B = p.B, H = p.H, W = p.W, Ho = p.Ho, Wo = p.Wo;
  const bool flat = (p.KH == 1 && p.stride == 1 && p.out_bs == (int64_t)p.Ho * p.Wo * p.out_pitch) && p.w_bs == 0;
  kp.w_batched = p.w_bs != 0 ? 1 : 0;
  kp.rowmax = p.rowmax;
  if (flat) {
    if (p.M > 0x7fffffffLL) { set_error("conv_tc: M too large"); return FB200_ERR_UNSUPPORTED; }
    W = Wo = (int)p.M; H = Ho = 1; B = 1;
  }
  int BW = 1, BH = 1;
  choose_tile(Ho, Wo, &BW, &BH);
  kp.BW = BW; kp.BH = BH; kp.tiles_w = (Wo + BW - 1) / BW; kp.tiles_h = (Ho + BH - 1) / BH; kp.Ho = Ho; kp.Wo = Wo;
  const int64_t m_tiles = (int64_t)B * kp.tiles_w * kp.tiles_h;

  CUtensorMap ta, tb;
  OutMaps om;
  int rc;
  const uint64_t P = (uint64_t)p.x_pitch;
  if (!kp.stride2) {
    const uint64_t dims[4] = {(uint64_t)(p.split3 ? kp.lo_off + Clog : p.Cin), (uint64_t)W, (uint64_t)H, (uint64_t)B};
    const uint64_t str[4] = {1, P, P * W, P * W * H};
    const uint32_t box[4] = {(uint32_t)BK, (uint32_t)BW, (uint32_t)BH, 1};
    rc = encode(&ta, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, const_cast<void*>(p.x), dims, str, box, "conv_tc: A", swz);
  } else if (kp.stride2 == 2) {
    // odd H or W: the true (c, w, h, b) geometry, every other pixel of a 2BW x 2BH box.  The last tile's box runs one row / column past the
    // map, which the TMA unit zero-fills like the conv padding.  choose_tile keeps BW, BH <= 128, so the box stays within 256.
    const uint64_t dims[4] = {(uint64_t)(p.split3 ? kp.lo_off + Clog : p.Cin), (uint64_t)W, (uint64_t)H, (uint64_t)B};
    const uint64_t str[4] = {1, P, P * W, P * W * H};
    const uint32_t box[4] = {(uint32_t)BK, 2 * (uint32_t)BW, 2 * (uint32_t)BH, 1};
    const uint32_t estr[4] = {1, 2, 2, 1};
    rc = encode(&ta, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 4, const_cast<void*>(p.x), dims, str, box, "conv_tc: A(s2 odd)", swz, estr);
  } else {
    const uint64_t dims[5] = {2 * P, (uint64_t)W / 2, 2, (uint64_t)H / 2, (uint64_t)B};
    const uint64_t str[5] = {1, 2 * P, P * W, 2 * P * W, P * W * H};
    const uint32_t box[5] = {(uint32_t)BK, (uint32_t)BW, 1, (uint32_t)BH, 1};
    rc = encode(&ta, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, 5, const_cast<void*>(p.x), dims, str, box, "conv_tc: A(s2)", swz);
  }
  if (rc) return rc;
  rc = encode_out_maps(&om, p, Wo, Ho, B, BW, BH, flat ? (uint64_t)p.out_pitch * Wo * Ho : (uint64_t)p.out_bs);
  if (rc) return rc;

  auto run = [&](auto blockn_tag, auto stages_tag, auto bk_tag, auto gelu_tag, auto fs_tag) -> int {
    constexpr bool FS_ = decltype(fs_tag)::value;
    constexpr int BN_ = decltype(blockn_tag)::value;
    constexpr int ST_ = decltype(stages_tag)::value;
    constexpr int BK_ = decltype(bk_tag)::value;
    constexpr int NS_ = 2;  // double-buffered output staging
    {
      const uint64_t dims[3] = {(uint64_t)p.K, (uint64_t)p.Cout, (uint64_t)p.B};
      const uint64_t str[3] = {1, (uint64_t)p.K, (uint64_t)p.w_bs};
      const uint32_t box[3] = {(uint32_t)BK_, (uint32_t)BN_, 1};
      int r2 = encode(&tb, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, p.w_bs ? 3 : 2, const_cast<void*>(p.w), dims, str, box, "conv_tc: W", swz);
      if (r2) return r2;
    }
    kp.n_tiles = (p.Cout + BN_ - 1) / BN_;
    const int64_t total = m_tiles * kp.n_tiles;
    if (total > 0x7fffffffLL) { set_error("conv_tc: too many tiles (%lld)", (long long)total); return FB200_ERR_UNSUPPORTED; }
    kp.total_tiles = (int)total;
    auto launch = [&](auto out_tag) -> int {
      return launch_persistent<conv_tc_kernel<BN_, ST_, decltype(out_tag), BK_, NS_, decltype(gelu_tag)::value, FS_>, smem_bytes<BN_, ST_, BK_, NS_, FS_>()>(
          "conv_tc_kernel", kp.total_tiles, NUM_THREADS, st, ta, tb, om.d, om.r, om.d2, om.r2, kp);
    };
    const bool outp = p.out_dtype == FB200_F16PAIR;
    if constexpr (decltype(gelu_tag)::value) return launch(__half{});
    else if constexpr (FS_) return outp ? launch(PairOut{}) : launch(float{});  // fp32 or pair output (checked by the caller)
    else {
      if (outp) { set_error("conv_tc: pair output is only produced by the fused-split configurations"); return FB200_ERR_UNSUPPORTED; }
      return p.out_dtype == FB200_F16 ? launch(__half{}) : launch(float{});
    }
  };
  using std::integral_constant;
  typedef std::false_type NF;  // fp16 operands, one product
  typedef std::true_type FS;   // split-precision operands, fused split
  typedef integral_constant<int, 64> K64;
  typedef integral_constant<int, 32> K32;
  typedef integral_constant<int, 128> N128;
  typedef integral_constant<int, 64> N64;
  typedef integral_constant<int, 4> S4;
  typedef integral_constant<int, 3> S3;
  if ((p.act & 15) == FB200_ACT_GELU)  // exact-erf GELU: dedicated instantiation (fp16 out, Cin % 64 == 0; checked in conv2d_tc_supported)
    return run(N128{}, S4{}, K64{}, std::true_type{}, NF{});
  if (p.split3) {  // fp32-accurate mode: fused split (one TMA pass over A_hi, A_lo, W_hi, W_lo per chunk feeds the three products)
    if (BK == 64) {
      if (p.Cout > 64) return run(N128{}, S3{}, K64{}, std::false_type{}, FS{});   // 3 x 64 + 32 KiB
      return run(N64{}, S4{}, K64{}, std::false_type{}, FS{});                     // 4 x 48 + 32 KiB
    }
    if (p.Cout > 64) return run(N128{}, S4{}, K32{}, std::false_type{}, FS{});     // 4 x 32 + 32 KiB
    return run(N64{}, S4{}, K32{}, std::false_type{}, FS{});                       // 4 x 24 + 32 KiB
  }
  if (BK == 32) {  // stem convs (Cin = 32)
    if (p.Cout > 64) return run(N128{}, S4{}, K32{}, std::false_type{}, NF{});
    return run(N64{}, S4{}, K32{}, std::false_type{}, NF{});
  }
  if (p.Cout > 64) return run(N128{}, S4{}, K64{}, std::false_type{}, NF{});       // 4 x 32 + 32 KiB
  return run(N64{}, S4{}, K64{}, std::false_type{}, NF{});                         // 4 x 24 + 32 KiB
}

}  // namespace fb200

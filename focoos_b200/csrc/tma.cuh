// The sm_90a asynchronous-copy pipeline, written once for the kernels that stream operands through shared memory (conv_tc.cu, wgrad_tc.cu):
// mbarriers, TMA tensor loads / stores, and on the host the tensor-map encoder and the launch of a persistent kernel.
#pragma once
#include <cuda.h>
#include <stdint.h>

#include "common.cuh"

namespace fb200 {

// ---------------------------------------------------------------------------------------------- PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  uint32_t spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) break;
    if (++spins > (1u << 26)) __trap();  // a descriptor / phase bug must not hang the GPU
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------- host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// Tiled tensor map of rank `rank` (dimension 0 contiguous; strides in elements of `elt` bytes), out-of-bounds elements read as zero.  `what` names the
// caller and the operand in error messages ("conv_tc: A").
inline int encode(CUtensorMap* m, CUtensorMapDataType dt, int elt, int rank, void* base, const uint64_t* dims, const uint64_t* strides_elts,
                  const uint32_t* box, const char* what, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B,
                  const uint32_t* elem_strides = nullptr) {
  // elem_strides (null = all 1): traversal stride per dimension; a load then takes ceil(box[i] / elem_strides[i]) elements along dimension i
  EncodeTiledFn fn = get_encode();
  if (!fn) { set_error("%s: cuTensorMapEncodeTiled unavailable", what); return FB200_ERR_CUDA; }
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bdim[i] = box[i]; estr[i] = elem_strides ? elem_strides[i] : 1; }
  for (int i = 1; i < rank; ++i) gstr[i - 1] = strides_elts[i] * (uint64_t)elt;  // bytes; dim0 stride is implicit
  CUresult r = fn(m, dt, (cuuint32_t)rank, base, gdim, gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("%s: cuTensorMapEncodeTiled failed with %d (rank %d dims %llu,%llu,%llu,%llu box %u,%u,%u,%u)", what, (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)(rank > 2 ? dims[2] : 0),
              (unsigned long long)(rank > 3 ? dims[3] : 0), box[0], box[1], rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
    return FB200_ERR_CUDA;
  }
  return FB200_OK;
}

inline int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// Launches the persistent kernel KERN on min(items, #SMs) CTAs of `threads` threads with SMEM bytes of dynamic shared memory, which the kernel is
// allowed once, on its first launch.  `name` is the kernel's name in error messages.
template <auto KERN, int SMEM, typename... Args>
int launch_persistent(const char* name, int64_t items, int threads, cudaStream_t st, const Args&... args) {
  static_assert(SMEM <= 227 * 1024, "shared memory budget exceeded");
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(KERN, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    if (e != cudaSuccess) { set_error("%s: cudaFuncSetAttribute(%d B) failed: %s", name, SMEM, cudaGetErrorString(e)); return FB200_ERR_CUDA; }
    configured = true;
  }
  const int64_t cap = num_sms();
  const unsigned grid = (unsigned)(items < cap ? items : cap);
  KERN<<<grid, threads, SMEM, st>>>(args...);
  FB_CHECK_LAUNCH(name);
  return FB200_OK;
}

}  // namespace fb200

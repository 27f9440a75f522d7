// PTX wrappers shared by the TMA / mbarrier pipelines (agg_tma.cu, agg_nchw_tma.cu, gn72.cu, tc_gemm.cu, tc_wgrad.cu), sm_90a,
// and the host-side tensor-map encoder of those that use tensor maps.
// Every wait is a BOUNDED try_wait spin that __trap()s: a broken pipeline aborts the launch instead of hanging the GPU.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>

namespace cotb200 {

// ---------------------------------------------------------------- host: tensor maps
template <typename T> CUtensorMapDataType tma_dtype();
template <> inline CUtensorMapDataType tma_dtype<float>() { return CU_TENSOR_MAP_DATA_TYPE_FLOAT32; }
template <> inline CUtensorMapDataType tma_dtype<__nv_bfloat16>() { return CU_TENSOR_MAP_DATA_TYPE_BFLOAT16; }
template <> inline CUtensorMapDataType tma_dtype<__half>() { return CU_TENSOR_MAP_DATA_TYPE_FLOAT16; }

// cuTensorMapEncodeTiled with what every map of the library shares: unit element strides, no interleave, 128-byte L2
// promotion, zero fill out of bounds.  dims[rank] (dims[0] innermost, unit stride), strides[rank - 1] in BYTES of dims[1..],
// box[rank].  The driver entry point is looked up through the runtime (the library links no libcuda) once per process;
// CUDA_ERROR_NOT_FOUND when the driver does not have it.
inline CUresult tma_encode(CUtensorMap* m, CUtensorMapDataType dtype, int rank, const void* base, const cuuint64_t* dims,
                           const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle swizzle) {
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static const EncodeFn enc = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    const bool ok = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
                    q == cudaDriverEntryPointSuccess;
    return ok ? (EncodeFn)p : nullptr;
  }();
  if (!enc) return CUDA_ERROR_NOT_FOUND;
  if (rank < 1 || rank > 5) return CUDA_ERROR_INVALID_VALUE;
  const cuuint32_t es[5] = {1, 1, 1, 1, 1};
  return enc(m, dtype, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
             CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

// ---------------------------------------------------------------- device: mbarriers and bulk copies

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  for (int spin = 0; !done; ++spin) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (!done && spin > (1 << 22)) __trap();   // never hang the GPU: a broken pipeline aborts the launch
  }
}

// tiled tensor loads: global (tensor map, coordinates) -> shared, completion on an mbarrier (complete_tx::bytes)
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3,
                                            int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// 1-D bulk copies (no tensor map): contiguous bytes, 16-byte aligned addresses and sizes
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_store_and_wait(void* dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// generic-proxy writes to shared memory -> visible to the async proxy (bulk / TMA stores reading that memory)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

}  // namespace cotb200

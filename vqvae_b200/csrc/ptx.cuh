// ptx.cuh -- thin inline-PTX wrappers for the Hopper (sm_90a) async machinery: mbarrier and TMA
// (cp.async.bulk[.tensor]).  The warpgroup MMA wrappers are in wgmma.cuh.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Wait for the phase with the given parity.  try_wait carries a suspend-time hint: the hardware parks the thread until
// the phase completes (or the hint expires) instead of returning early and being re-polled.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "LAB_WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
        "@p bra LAB_DONE_%=;\n\t"
        "bra LAB_WAIT_%=;\n\t"
        "LAB_DONE_%=:\n\t"
        "}" ::"r"(bar), "r"(parity), "r"(0x989680u) : "memory");
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap *m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tiled load: coordinate c0 is the innermost (contiguous) dimension.
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *m, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::
            "r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap *m, uint32_t bar, int c0, int c1,
                                            int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::
            "r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
// 1-D bulk copy global -> shared (size multiple of 16, both 16-byte aligned).
__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
                     "r"(dst), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar) : "memory");
}

__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

}  // namespace ptx

// ---------------------------------------------------------------- host: tensor maps
// cuTensorMapEncodeTiled is fetched through the runtime (cudaGetDriverEntryPoint) so
// the library does not link libcuda and still loads on a machine without a driver.
int vqb_encode_tmap_2d(CUtensorMap *map, CUtensorMapDataType dtype, const void *base, uint64_t inner,
                       uint64_t outer, uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer,
                       CUtensorMapSwizzle swizzle);
int vqb_encode_tmap_4d(CUtensorMap *map, CUtensorMapDataType dtype, const void *base, const uint64_t dims[4],
                       const uint64_t strides_bytes[3], const uint32_t box[4], const uint32_t elem_strides[4],
                       CUtensorMapSwizzle swizzle);
int vqb_encode_tmap_nd(CUtensorMap *map, CUtensorMapDataType dtype, const void *base, int rank,
                       const unsigned long long *dims, const unsigned long long *strides_bytes, const uint32_t *box,
                       CUtensorMapSwizzle swizzle);

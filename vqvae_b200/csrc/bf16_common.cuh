// bf16_common.cuh -- helpers shared by the sources that write bf16 (wgconv.cu, conv_edge.cu, vq_exact.cu).
#pragma once
#include <cuda_bf16.h>


namespace {

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t *>(&h);
}


}  // namespace

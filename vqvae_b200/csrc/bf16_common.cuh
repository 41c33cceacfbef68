// bf16_common.cuh -- helpers shared by the bf16 pipeline's sources (hconv.cu, conv_edge.cu).
#pragma once
#include <cuda_bf16.h>


namespace {

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t *>(&h);
}


}  // namespace

// internal weight-packing kind (next to enum vqb_conv_kind): the 1x1 conv of a residual layer, Cmid <= 64 input
// channels zero-padded to one 64-channel K chunk
#define VQB_RES_W2_KIND 6

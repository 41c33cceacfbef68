// common.cuh -- shared declarations of the sm_90a VQ-VAE kernels (internal).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/vqvae_b200.h"

#define VQB_MAX_TAPS 16

// The environment knobs for experiments (VQB_PDL, VQB_MEMCPY_RUNTIME) are read only by a library built with
// -DVQB_DIAG=1 (VQB_DIAG=1 python -m vqvae_b200.build).  The release library never reads the environment:
// vqb_getenv() is a constant nullptr there.
#ifndef VQB_DIAG
#define VQB_DIAG 0
#endif
#include <stdlib.h>
static inline const char *vqb_getenv(const char *name) { return VQB_DIAG ? getenv(name) : nullptr; }

// A conv layer on an H x W input: its output size and its sub-pixel phases.  A conv or a stride-1 transposed conv
// is one phase; a stride-s transposed conv is s*s phases (decoder.py:31-35).  No pointers: the fp32 and the bf16
// entry points share it.
struct ConvGeom {
    int kh, kw, stride, pad, transposed;
    int OH, OW;
    int nph;
};

// One sub-pixel phase of a layer as a gather-form convolution
//   out[n, gy*out_step+out_py, gx*out_step+out_px, co] =
//       act( bias[co] + skip + sum_{t<ntaps, ci} in[n, gy*in_step+dy[t], gx*in_step+dx[t], ci]
//                                                * w[tap_w[t]][co][ci] )
// which covers nn.Conv2d (in_step = stride, out_step = 1, dy = r - pad), stride-1
// nn.ConvTranspose2d (dy = pad - r) and one sub-pixel phase of a stride-s
// nn.ConvTranspose2d (in_step = 1, out_step = s, taps of matching parity).
struct ConvPhase {
    int OHg, OWg;                 // output grid of this phase
    int in_step, out_step, out_py, out_px;
    int ntaps;
    int tap_w[VQB_MAX_TAPS], tap_dy[VQB_MAX_TAPS], tap_dx[VQB_MAX_TAPS];
};

// element strides (batch, row, column, channel) of a (B, C, H, W) activation stored in `layout` (VQB_NCHW or VQB_NHWC)
static inline void layout_strides(int layout, int C, int H, int W, long long &sn, long long &sh, long long &sw,
                                  long long &sc) {
    if (layout == VQB_NCHW) {
        sn = (long long)C * H * W; sc = (long long)H * W; sh = W; sw = 1;
    } else {
        sn = (long long)H * W * C; sh = (long long)W * C; sw = C; sc = 1;
    }
}

ConvGeom conv_geom(int kh, int kw, int stride, int pad, int transposed, int H, int W);
// phase i < g.nph of g; false when its output grid is empty
bool conv_phase(const ConvGeom &g, int i, ConvPhase &ph);

// One launch of a CUDA-core conv kernel: one phase of a layer on fp32 tensors.
struct ConvLaunch : ConvPhase {
    const float *in, *w, *bias, *skip;         // w: the K-major rows [kh*kw][Cout][Cin] of vqb_pack_conv_weight_f32
    float *out;
    int B, Cin, H, W, Cout;
    long long in_sn, in_sh, in_sw, in_sc;      // element strides of `in`
    long long out_sn, out_sh, out_sw, out_sc;  // element strides of `out` (and `skip`)
    int relu;
};

int launch_conv_ffma(const ConvLaunch &p, cudaStream_t s);
int launch_conv_small_cout(const ConvLaunch &p, cudaStream_t s);

// vqb_pack_conv_weight_f32 writes the K-major rows [kh*kw][Cout][Cin] from element 0; the [9][16][Cin] pixel-shuffle
// form of a k4 s2 transposed conv to Cout <= 4 channels starts here, in floats.
static inline size_t conv_pack_shuffle_offset(int Cout, int Cin, int kh, int kw) { return (size_t)kh * kw * Cout * Cin; }

// The weight vqb_pack_conv_weight_bf16 writes: K-major bf16 rows [kh*kw][Cout][Cin_pad] (zero padded from Cin), or
// for shuffle != 0 the [9][16][Cin] form of the k4 s2 output layer.
int launch_pack_weight_bf16(const float *w, void *out, int Cout, int Cin, int Cin_pad, int kh, int kw, int transposed,
                            int shuffle, cudaStream_t s);

// process-wide count of kernels launched through the C ABI (vqb_launch_count)
extern unsigned long long g_vqb_launches;
#define VQB_COUNT_LAUNCH(n) (g_vqb_launches += (n))

// Programmatic dependent launch: the next kernel of the layer chain may start its prologue (barrier init,
// tensor-map prefetch) while this one drains; it blocks in pdl_wait() until the previous
// grid has completed and its writes are visible.  VQB_PDL=0 in the environment disables the attribute.
int vqb_pdl_enabled();
#ifdef __CUDACC__
#include <utility>
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
template <typename... KArgs, typename... Args>
static inline cudaError_t vqb_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                                     Args &&...args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = vqb_pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
#endif

static inline int vqb_cuda_status(cudaError_t e) { return e == cudaSuccess ? 0 : (int)e; }

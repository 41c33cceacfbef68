// conv_edge.cu -- the two HBM-bound end layers of the hot path (sm_90a, CUDA cores).
//
//   conv_in_k4s2:   encoder.py:29-31  Conv2d(3 -> 64, k4 s2 p1) + ReLU, reads the NCHW module
//                   input, writes NHWC (fp32, or bf16 for the bf16 pipeline).  K_red = 48: far too thin for a
//                   tensor-core tile (SURVEY 7.3.4); arithmetic intensity ~20 F/B.
//   convt_out_k4s2: decoder.py:34-35  ConvTranspose2d(64 -> 3, k4 s2 p1), reads NHWC, writes
//                   the NCHW module output.  One thread owns one INPUT pixel and produces its
//                   2x2 output block for every output channel from the 3x3 input
//                   neighbourhood (the four sub-pixel phases share the loads).
// Both keep the (tiny) weight tensor in shared memory, read activations through L1 and
// write fully coalesced rows.  fp32 FFMA arithmetic in every precision mode.
#include "common.cuh"
#include "bf16_common.cuh"

namespace {

// ------------------------------------------------------------------ Conv2d(Cin<=4 -> Cout), k4 s2 p1
// thread = (output pixel, group of 32 output channels); warp = 32 consecutive pixels of one
// channel group, so weight reads are warp-wide broadcasts.
template <int CIN, bool OUT_BF16>
__global__ void __launch_bounds__(256, 2)
conv_in_k4s2_kernel(const float *__restrict__ x, const float *__restrict__ wp, const float *__restrict__ bias,
                    void *__restrict__ y, int B, int H, int W, int Cout, int relu) {
    extern __shared__ __align__(16) float wsm[];          // [16*CIN][Cout], from the K-major packing [16][Cout][CIN]
    // a warp copies the K-major rows of 32 output channels of one tap: 32 * CIN contiguous floats
    for (int g = threadIdx.x >> 5; g < 16 * (Cout / 32); g += blockDim.x >> 5) {
        const int tap = g % 16, co = (g / 16) * 32 + (threadIdx.x & 31);
#pragma unroll
        for (int ci = 0; ci < CIN; ++ci) wsm[(tap * CIN + ci) * Cout + co] = __ldg(wp + (tap * Cout + co) * CIN + ci);
    }
    __syncthreads();
    const int OH = H / 2, OW = W / 2;                      // (H + 2 - 4)/2 + 1
    const int groups = Cout / 32;
    const long long npix = (long long)B * OH * OW;
    const long long gwarp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const long long pix = (gwarp / groups) * 32 + lane;
    const int cg = (int)(gwarp % groups);
    if (pix >= npix) return;
    const int ox = (int)(pix % OW);
    const long long t = pix / OW;
    const int oy = (int)(t % OH);
    const int n = (int)(t / OH);

    float acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = bias ? __ldg(bias + cg * 32 + j) : 0.f;
    // one kernel row per iteration: 4*CIN inputs in registers, body small enough for the I-cache
#pragma unroll 1
    for (int r = 0; r < 4; ++r) {
        const int iy = 2 * oy - 1 + r;
        float in[4 * CIN];
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            const int ix = 2 * ox - 1 + s;
            const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
#pragma unroll
            for (int c = 0; c < CIN; ++c)
                in[s * CIN + c] = ok ? __ldg(x + (((long long)n * CIN + c) * H + iy) * W + ix) : 0.f;
        }
#pragma unroll
        for (int k = 0; k < 4 * CIN; ++k) {
            const float4 *w4 = reinterpret_cast<const float4 *>(wsm + (size_t)(r * 4 * CIN + k) * Cout + cg * 32);
            const float a = in[k];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float4 w = w4[j];
                acc[4 * j + 0] = fmaf(a, w.x, acc[4 * j + 0]); acc[4 * j + 1] = fmaf(a, w.y, acc[4 * j + 1]);
                acc[4 * j + 2] = fmaf(a, w.z, acc[4 * j + 2]); acc[4 * j + 3] = fmaf(a, w.w, acc[4 * j + 3]);
            }
        }
    }
    if (relu) {
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[j] = fmaxf(acc[j], 0.f);
    }
    if constexpr (OUT_BF16) {
        uint4 *dst = reinterpret_cast<uint4 *>(reinterpret_cast<__nv_bfloat16 *>(y) + pix * Cout + cg * 32);
#pragma unroll
        for (int j = 0; j < 4; ++j)
            dst[j] = make_uint4(pack_bf16(acc[8 * j], acc[8 * j + 1]), pack_bf16(acc[8 * j + 2], acc[8 * j + 3]),
                                pack_bf16(acc[8 * j + 4], acc[8 * j + 5]), pack_bf16(acc[8 * j + 6], acc[8 * j + 7]));
    } else {
        float4 *dst = reinterpret_cast<float4 *>(reinterpret_cast<float *>(y) + pix * Cout + cg * 32);
#pragma unroll
        for (int j = 0; j < 8; ++j) dst[j] = make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]);
    }
}

// ------------------------------------------------------------------ ConvTranspose2d(Cin -> Cout<=4), k4 s2 p1
// out[2j+py][2i+px] = sum over the two kernel rows/cols of matching parity:
//   py = 0: (kh=1, dy=0), (kh=3, dy=-1)      py = 1: (kh=0, dy=+1), (kh=2, dy=0)     (same in x)
// A group of L = Cin/4 lanes owns one input pixel: lane c reads channels 4c..4c+3 of the nine
// neighbours (one fully coalesced Cin*4-byte row per neighbour and group), accumulates its
// share of the 2x2xCOUT output block, and the group reduces with shuffles.  Persistent CTAs:
// the 16*COUT*Cin weights are staged in shared memory once per CTA.
template <int COUT>
__global__ void __launch_bounds__(256, 2)
convt_out_k4s2_kernel(const float *__restrict__ x, const float *__restrict__ wk, const float *__restrict__ bias,
                      float *__restrict__ y, int B, int H, int W, int Cin, int relu) {
    extern __shared__ __align__(16) float wsm[];          // [16 taps][COUT][Cin] = the K-major packing
    for (int i = threadIdx.x; i < 16 * COUT * Cin / 4; i += blockDim.x)
        reinterpret_cast<float4 *>(wsm)[i] = __ldg(reinterpret_cast<const float4 *>(wk) + i);
    __syncthreads();
    const int L = Cin / 4;                                 // lanes per pixel (power of two <= 32)
    const int per_warp = 32 / L;
    const int lane = threadIdx.x & 31;
    const int c4 = (lane % L) * 4, sub = lane / L;
    const long long npix = (long long)B * H * W;
    const long long warps_total = (long long)gridDim.x * (blockDim.x >> 5);
    const long long gwarp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int OH = 2 * H, OW = 2 * W;
    for (long long base = gwarp * per_warp; base < npix; base += warps_total * per_warp) {
        const long long pix = base + sub;
        const bool live = pix < npix;
        const long long pp = live ? pix : npix - 1;
        const int i0 = (int)(pp % W);
        const long long t = pp / W;
        const int j0 = (int)(t % H);
        const int n = (int)(t / H);
        float acc[2][2][COUT];
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
                for (int c = 0; c < COUT; ++c) acc[a][b][c] = 0.f;
        float4 xin[3][3];
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                const int iy = j0 + dy, ix = i0 + dx;
                xin[dy + 1][dx + 1] = (iy >= 0 && iy < H && ix >= 0 && ix < W)
                    ? __ldg(reinterpret_cast<const float4 *>(x + (((long long)n * H + iy) * W + ix) * Cin + c4))
                    : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
        for (int py = 0; py < 2; ++py)
#pragma unroll
            for (int px = 0; px < 2; ++px)
#pragma unroll
                for (int a = 0; a < 2; ++a)
#pragma unroll
                    for (int b = 0; b < 2; ++b) {
                        const int kh = (py == 0) ? (a == 0 ? 1 : 3) : (a == 0 ? 0 : 2);
                        const int dy = (py == 0) ? (a == 0 ? 0 : -1) : (a == 0 ? 1 : 0);
                        const int kw = (px == 0) ? (b == 0 ? 1 : 3) : (b == 0 ? 0 : 2);
                        const int dx = (px == 0) ? (b == 0 ? 0 : -1) : (b == 0 ? 1 : 0);
                        const float4 xv = xin[dy + 1][dx + 1];
#pragma unroll
                        for (int c = 0; c < COUT; ++c) {
                            const float4 w = *reinterpret_cast<const float4 *>(
                                wsm + ((size_t)(kh * 4 + kw) * COUT + c) * Cin + c4);
                            acc[py][px][c] = fmaf(xv.x, w.x, acc[py][px][c]);
                            acc[py][px][c] = fmaf(xv.y, w.y, acc[py][px][c]);
                            acc[py][px][c] = fmaf(xv.z, w.z, acc[py][px][c]);
                            acc[py][px][c] = fmaf(xv.w, w.w, acc[py][px][c]);
                        }
                    }
        // reduce over the L lanes of the pixel (butterfly: every lane ends with the total)
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
                for (int c = 0; c < COUT; ++c) {
                    float v = acc[a][b][c];
                    for (int off = L >> 1; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
                    acc[a][b][c] = v;
                }
        if (live && (lane % L) == 0) {
#pragma unroll
            for (int c = 0; c < COUT; ++c) {
                const float bv = bias ? __ldg(bias + c) : 0.f;
#pragma unroll
                for (int py = 0; py < 2; ++py) {
                    float2 o = make_float2(acc[py][0][c] + bv, acc[py][1][c] + bv);
                    if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
                    *reinterpret_cast<float2 *>(y + (((long long)n * COUT + c) * OH + 2 * j0 + py) * OW + 2 * i0) = o;
                }
            }
        }
    }
}

}  // namespace

// Conv2d(Cin in {1..4} -> Cout % 32 == 0), k4 s2 p1, NCHW in, NHWC out (fp32, or bf16 when out_bf16).
// wp = vqb_pack_conv_weight_f32.
int launch_conv_in_k4s2(const float *x, const float *wp, const float *bias, void *y, int out_bf16, int B, int Cin, int H,
                        int W, int Cout, int relu, cudaStream_t s) {
    if (Cin != 3 || Cout % 32 != 0 || H % 2 || W % 2) return VQB_ERR_UNSUPPORTED;
    const size_t smem = (size_t)16 * Cin * Cout * sizeof(float);
    if (smem > 48 * 1024) return VQB_ERR_UNSUPPORTED;
    const long long npix = (long long)B * (H / 2) * (W / 2);
    const long long warps = (npix + 31) / 32 * (Cout / 32);
    const long long blocks = (warps + 7) / 8;
    if (blocks > 0x7fffffffLL) return VQB_ERR_UNSUPPORTED;
    if (out_bf16)
        conv_in_k4s2_kernel<3, true><<<(unsigned)blocks, 256, smem, s>>>(x, wp, bias, y, B, H, W, Cout, relu);
    else
        conv_in_k4s2_kernel<3, false><<<(unsigned)blocks, 256, smem, s>>>(x, wp, bias, y, B, H, W, Cout, relu);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

// ConvTranspose2d(Cin % 4 == 0 -> Cout == 3), k4 s2 p1, NHWC in, NCHW out.  wp = vqb_pack_conv_weight_f32.
int launch_convt_out_k4s2(const float *x, const float *wp, const float *bias, float *y, int B, int Cin, int H, int W,
                          int Cout, int relu, cudaStream_t s) {
    const int L = Cin / 4;
    if (Cout != 3 || Cin % 4 != 0 || L < 1 || L > 32 || (L & (L - 1)) != 0) return VQB_ERR_UNSUPPORTED;
    const size_t smem = (size_t)16 * Cout * Cin * sizeof(float);
    if (smem > 48 * 1024) return VQB_ERR_UNSUPPORTED;
    const long long npix = (long long)B * H * W;
    const long long warps = (npix + (32 / L) - 1) / (32 / L);
    long long blocks = (warps + 7) / 8;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (blocks > (long long)sms * 2) blocks = (long long)sms * 2;       // persistent: weights staged once per CTA
    if (blocks < 1) blocks = 1;
    convt_out_k4s2_kernel<3><<<(unsigned)blocks, 256, smem, s>>>(x, wp, bias, y, B, H, W, Cin, relu);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

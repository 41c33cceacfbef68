// vq_backward.cu -- backward of VectorQuantizer.forward (quantizer.py:63-67) for training-mode callers (main.py:74-79).
//
// Forward (reference):  loss = mean((sg[z_q] - z)^2) + beta * mean((z_q - sg[z])^2),   z_q_out = z + sg[z_q - z]
// with z_q = E[idx] and sg = stop-gradient.  Hence, for upstream gradients g_loss (scalar) and g_zq (N, D):
//     dz[i]  = g_zq[i] + g_loss * 2 / (N D) * (z[i] - E[idx[i]])                      (straight-through + first loss term)
//     dE[k]  = g_loss * 2 beta / (N D) * sum_{i : idx[i] = k} (E[k] - z[i])           (second loss term: scatter-add by index)
// The argmin, the one-hot and the perplexity carry no gradient.  One thread per float4 of a row; the codebook gradient is
// accumulated with red.global.add.f32 (order-dependent in the last bits, like torch's own embedding backward).
#include "common.cuh"

namespace {

__global__ void vq_backward_kernel(const float *__restrict__ g_zq, const float *__restrict__ g_loss, const float *__restrict__ z,
                                   const float *__restrict__ E, const long long *__restrict__ idx, long long N, int K, int D,
                                   float beta, float *__restrict__ dz, float *__restrict__ dE) {
    const int d4 = D / 4;
    const long long total = N * d4;
    const float gl = g_loss ? __ldg(g_loss) : 0.f;
    const float c1 = gl * 2.0f / ((float)N * (float)D), c2 = c1 * beta;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / d4;
        const int c = (int)(i - row * d4);
        long long k = idx[row];
        k = k < 0 ? 0 : (k >= K ? K - 1 : k);
        const float4 zv = __ldg(reinterpret_cast<const float4 *>(z) + i);
        const float4 ev = __ldg(reinterpret_cast<const float4 *>(E + (size_t)k * D) + c);
        float4 g = g_zq ? __ldg(reinterpret_cast<const float4 *>(g_zq) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 df = make_float4(zv.x - ev.x, zv.y - ev.y, zv.z - ev.z, zv.w - ev.w);
        g.x = fmaf(c1, df.x, g.x); g.y = fmaf(c1, df.y, g.y); g.z = fmaf(c1, df.z, g.z); g.w = fmaf(c1, df.w, g.w);
        reinterpret_cast<float4 *>(dz)[i] = g;
        float *de = dE + (size_t)k * D + 4 * c;
        atomicAdd(de + 0, -c2 * df.x); atomicAdd(de + 1, -c2 * df.y); atomicAdd(de + 2, -c2 * df.z); atomicAdd(de + 3, -c2 * df.w);
    }
}

}  // namespace

extern "C" int vqb_vq_backward_f32(const float *g_zq, const float *g_loss, const float *z, const float *codebook,
                                   const int64_t *idx, int64_t N, int K, int D, float beta, float *dz, float *dE, void *stream) {
    if (!z || !codebook || !idx || !dz || !dE) return VQB_ERR_BAD_ARG;
    if (N <= 0 || K <= 0 || D <= 0) return VQB_ERR_BAD_ARG;
    if (D % 4 != 0) return VQB_ERR_UNSUPPORTED;
    const uintptr_t al = reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(codebook) | reinterpret_cast<uintptr_t>(dz) |
                         reinterpret_cast<uintptr_t>(dE) | reinterpret_cast<uintptr_t>(g_zq);
    if (al & 15) return VQB_ERR_ALIGNMENT;
    cudaStream_t s = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(dE, 0, sizeof(float) * (size_t)K * D, s);
    if (e != cudaSuccess) return (int)e;
    const long long total = N * (D / 4);
    long long blocks = (total + 255) / 256;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (blocks > (long long)sms * 16) blocks = (long long)sms * 16;
    vq_backward_kernel<<<(unsigned)blocks, 256, 0, s>>>(g_zq, g_loss, z, codebook, reinterpret_cast<const long long *>(idx), N, K, D, beta,
                                                        dz, dE);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

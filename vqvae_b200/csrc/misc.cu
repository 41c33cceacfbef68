// misc.cu -- small bandwidth kernels around the hot path (sm_90a).
#include <cuda_bf16.h>

#include "common.cuh"
#include "pack.cuh"

namespace {

// the K-major packing of pack_kmajor_at.  T = float or __nv_bfloat16 (rounded to nearest even).
template <typename T>
__global__ void pack_weight_kernel(const float *__restrict__ w, T *__restrict__ out, int Cout, int Cin, int Cin_pad,
                                   int kh, int kw, int transposed) {
    const long long total = (long long)Cout * Cin_pad * kh * kw;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x)
        out[i] = T(pack_kmajor_at(w, i, Cout, Cin, Cin_pad, kh, kw, transposed));
}

// the [9][16][Cin] pixel-shuffle packing of pack_shuffle_at
template <typename T>
__global__ void pack_convt_shuffle_kernel(const float *__restrict__ w, T *__restrict__ out, int Cout, int Cin) {
    const int total = 9 * 16 * Cin;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x)
        out[i] = T(pack_shuffle_at(w, i, Cout, Cin));
}

// tiled transpose of the innermost two logical axes: in[b][R][Ccols] -> out[b][Ccols][R]
__global__ void transpose_kernel(const float *__restrict__ in, float *__restrict__ out, int R, int Cc) {
    __shared__ float tile[32][33];
    const long long b = blockIdx.z;
    const float *src = in + b * (long long)R * Cc;
    float *dst = out + b * (long long)R * Cc;
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int j = threadIdx.y; j < 32; j += 8) {
        const int r = r0 + j, c = c0 + threadIdx.x;
        if (r < R && c < Cc) tile[j][threadIdx.x] = src[(long long)r * Cc + c];
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += 8) {
        const int c = c0 + j, r = r0 + threadIdx.x;
        if (r < R && c < Cc) dst[(long long)c * R + r] = tile[threadIdx.x][j];
    }
}

// quantizer.py:63-64 and :70-71 in fp32, like the reference's scalar ops.  COMMIT_ONLY (the EMA codebook): the loss is
// the commitment term beta * mse alone.
template <bool COMMIT_ONLY>
__global__ void vq_finish_kernel(const double *__restrict__ sse, const int *__restrict__ hist, long long N,
                                 int K, int D, float beta, float *__restrict__ loss, float *__restrict__ perp) {
    __shared__ float sh[256];
    float ent = 0.f;
    for (int k = threadIdx.x; k < K; k += 256) {
        const float p = __fdiv_rn((float)hist[k], (float)N);
        ent += p * logf(p + 1e-10f);
    }
    sh[threadIdx.x] = ent;
    __syncthreads();
    for (int off = 128; off >= 1; off >>= 1) {
        if (threadIdx.x < off) sh[threadIdx.x] += sh[threadIdx.x + off];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float mse = (float)(*sse / ((double)N * (double)D));
        *loss = COMMIT_ONLY ? __fmul_rn(beta, mse) : __fadd_rn(mse, __fmul_rn(beta, mse));
        *perp = expf(-sh[0]);
    }
}

__global__ void onehot_kernel(const long long *__restrict__ idx, long long N, int K, float *__restrict__ out) {
    // one CTA per row group; every element written exactly once (zeros + the one)
    const long long total4 = N * (long long)(K / 4);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total4;
         i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / (K / 4);
        const int c = (int)(i % (K / 4)) * 4;
        const int k = (int)idx[row];
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k == c) v.x = 1.f; else if (k == c + 1) v.y = 1.f;
        else if (k == c + 2) v.z = 1.f; else if (k == c + 3) v.w = 1.f;
        *reinterpret_cast<float4 *>(out + row * K + c) = v;
    }
}

__global__ void onehot_scalar_kernel(const long long *__restrict__ idx, long long N, int K,
                                     float *__restrict__ out) {
    const long long total = N * (long long)K;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / K;
        out[i] = ((long long)(i % K) == idx[row]) ? 1.f : 0.f;
    }
}

__global__ void gather_rows_kernel(const long long *__restrict__ idx, const float *__restrict__ E, long long N,
                                   int K, int D, float *__restrict__ rows) {
    const long long total = N * (long long)D;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / D;
        const int d = (int)(i % D);
        long long k = idx[row];
        k = k < 0 ? 0 : (k >= K ? K - 1 : k);
        rows[i] = __ldg(E + k * D + d);
    }
}

__global__ void relu_kernel(float *__restrict__ x, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x)
        x[i] = fmaxf(x[i], 0.f);
}

// out = y > 0 ? g : 0 (out may be g): the gradient through a ReLU whose output y was kept
__global__ void relu_backward_kernel(const float *g, const float *__restrict__ y, float *out, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x)
        out[i] = __ldg(y + i) > 0.f ? g[i] : 0.f;
}

unsigned grid_for(long long total, int block) {
    long long g = (total + block - 1) / block;
    if (g > 148LL * 32) g = 148LL * 32;
    if (g < 1) g = 1;
    return (unsigned)g;
}

}  // namespace

extern "C" int vqb_pack_conv_weight_f32(const float *w, float *packed, int Cout, int Cin, int kh, int kw,
                                        int transposed, void *stream) {
    if (!w || !packed || Cout <= 0 || Cin <= 0 || kh <= 0 || kw <= 0) return VQB_ERR_BAD_ARG;
    pack_weight_kernel<float><<<grid_for((long long)Cout * Cin * kh * kw, 256), 256, 0, (cudaStream_t)stream>>>(
        w, packed, Cout, Cin, Cin, kh, kw, transposed);
    if (transposed && kh == 4 && kw == 4 && Cout <= 4) {
        pack_convt_shuffle_kernel<float><<<grid_for(9 * 16 * Cin, 256), 256, 0, (cudaStream_t)stream>>>(
            w, packed + conv_pack_shuffle_offset(Cout, Cin, kh, kw), Cout, Cin);
        VQB_COUNT_LAUNCH(1);
    }
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

int launch_pack_weight_bf16(const float *w, void *out, int Cout, int Cin, int Cin_pad, int kh, int kw, int transposed,
                            int shuffle, cudaStream_t s) {
    __nv_bfloat16 *o = reinterpret_cast<__nv_bfloat16 *>(out);
    if (shuffle)
        pack_convt_shuffle_kernel<<<grid_for(9 * 16 * Cin, 256), 256, 0, s>>>(w, o, Cout, Cin);
    else
        pack_weight_kernel<<<grid_for((long long)Cout * Cin_pad * kh * kw, 256), 256, 0, s>>>(w, o, Cout, Cin, Cin_pad,
                                                                                            kh, kw, transposed);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

static int transpose_launch(const float *in, float *out, int Bt, int R, int Cc, cudaStream_t s) {
    if (Bt > 65535) return VQB_ERR_UNSUPPORTED;
    dim3 grid((Cc + 31) / 32, (R + 31) / 32, Bt), block(32, 8);
    if (grid.y > 65535) return VQB_ERR_UNSUPPORTED;
    transpose_kernel<<<grid, block, 0, s>>>(in, out, R, Cc);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" int vqb_nchw_to_nhwc_f32(const float *in, float *out, int B, int C, int H, int W, void *stream) {
    if (!in || !out || B <= 0 || C <= 0 || H <= 0 || W <= 0) return VQB_ERR_BAD_ARG;
    return transpose_launch(in, out, B, C, H * W, (cudaStream_t)stream);  // [C][HW] -> [HW][C]
}

extern "C" int vqb_nhwc_to_nchw_f32(const float *in, float *out, int B, int C, int H, int W, void *stream) {
    if (!in || !out || B <= 0 || C <= 0 || H <= 0 || W <= 0) return VQB_ERR_BAD_ARG;
    return transpose_launch(in, out, B, H * W, C, (cudaStream_t)stream);  // [HW][C] -> [C][HW]
}

extern "C" int vqb_vq_finish_f32(const double *sse, const int32_t *hist, int64_t N, int K, int D, float beta,
                                 float *loss, float *perplexity, void *stream) {
    if (!sse || !hist || !loss || !perplexity || N <= 0 || K <= 0 || D <= 0) return VQB_ERR_BAD_ARG;
    vq_finish_kernel<false><<<1, 256, 0, (cudaStream_t)stream>>>(sse, hist, N, K, D, beta, loss, perplexity);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" int vqb_vq_finish_ema_f32(const double *sse, const int32_t *hist, int64_t N, int K, int D, float beta,
                                     float *loss, float *perplexity, void *stream) {
    if (!sse || !hist || !loss || !perplexity || N <= 0 || K <= 0 || D <= 0) return VQB_ERR_BAD_ARG;
    vq_finish_kernel<true><<<1, 256, 0, (cudaStream_t)stream>>>(sse, hist, N, K, D, beta, loss, perplexity);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" int vqb_onehot_f32(const int64_t *idx, int64_t N, int K, float *onehot, void *stream) {
    if (!idx || !onehot || N <= 0 || K <= 0) return VQB_ERR_BAD_ARG;
    const long long *ip = reinterpret_cast<const long long *>(idx);
    if (K % 4 == 0 && (reinterpret_cast<uintptr_t>(onehot) & 15) == 0)
        onehot_kernel<<<grid_for(N * (long long)(K / 4), 256), 256, 0, (cudaStream_t)stream>>>(ip, N, K, onehot);
    else
        onehot_scalar_kernel<<<grid_for(N * (long long)K, 256), 256, 0, (cudaStream_t)stream>>>(ip, N, K, onehot);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" int vqb_gather_rows_f32(const int64_t *idx, const float *codebook, int64_t N, int K, int D,
                                   float *rows, void *stream) {
    if (!idx || !codebook || !rows || N <= 0 || K <= 0 || D <= 0) return VQB_ERR_BAD_ARG;
    gather_rows_kernel<<<grid_for(N * (long long)D, 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const long long *>(idx), codebook, N, K, D, rows);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" int vqb_relu_f32(float *x, int64_t n, void *stream) {
    if (!x || n < 0) return VQB_ERR_BAD_ARG;
    if (n == 0) return 0;
    relu_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(x, n);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" int vqb_relu_backward_f32(const float *g, const float *y, float *out, int64_t n, void *stream) {
    if (!g || !y || !out || n < 0) return VQB_ERR_BAD_ARG;
    if (n == 0) return 0;
    relu_backward_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(g, y, out, n);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

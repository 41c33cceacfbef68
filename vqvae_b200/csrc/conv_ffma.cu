// conv_ffma.cu -- fp32 (FFMA, CUDA-core) gather-form convolution for sm_90a.
//
// This is the VQB_FP32 arithmetic of vqb_conv2d_f32: every product and every
// accumulation is fp32, like the reference's CPU path (oneDNN), so it is the path
// the parity tests hold to the tightest tolerance, the fallback for shapes the
// wgmma implicit-GEMM kernels do not cover, and their on-GPU cross-check.
// Replaces nn.Conv2d / nn.ConvTranspose2d call sites: encoder.py:29-36,
// residual.py:20-24, vqvae.py:16-17, decoder.py:28-35.
//
// Implicit GEMM:  C[m][co] = sum_k A[m][k] * Wp[k][co],  m = (n, gy, gx) output
// pixel, k = (tap, ci).  A is gathered on the fly (never materialised); Wp[k][co] is
// read from the K-major packed weight [tap][co][ci] and stored transposed into shared
// memory.  Tile BM x BN x 16, 256 threads, TM x TN registers per thread,
// global->register prefetch of the next k-tile overlapped with the FFMAs.
#include "common.cuh"

namespace {

constexpr int BK = 16;
constexpr int NT = 256;

template <int BM, int BN, int TM, int TN, bool VEC_A>
__global__ void __launch_bounds__(NT) conv_ffma_kernel(const ConvLaunch p) {
    static_assert((BM / TM) * (BN / TN) == NT, "thread tiling");
    constexpr int APAD = 4, BPAD = 4;
    __shared__ __align__(16) float As[2][BK][BM + APAD];
    __shared__ __align__(16) float Bs[2][BK][BN + BPAD];
    __shared__ long long row_in[BM];   // n * in_sn
    __shared__ long long row_out[BM];  // full output offset (without co)
    __shared__ int row_iy[BM], row_ix[BM];

    const int tid = threadIdx.x;
    const long long M = (long long)p.B * p.OHg * p.OWg;
    const long long m0 = (long long)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    const int Ktot = p.ntaps * p.Cin;

    for (int r = tid; r < BM; r += NT) {
        long long m = m0 + r;
        if (m < M) {
            int gx = (int)(m % p.OWg);
            long long t = m / p.OWg;
            int gy = (int)(t % p.OHg);
            int n = (int)(t / p.OHg);
            row_in[r] = (long long)n * p.in_sn;
            row_iy[r] = gy * p.in_step;
            row_ix[r] = gx * p.in_step;
            row_out[r] = (long long)n * p.out_sn + (long long)(gy * p.out_step + p.out_py) * p.out_sh +
                         (long long)(gx * p.out_step + p.out_px) * p.out_sw;
        } else {
            row_in[r] = 0;
            row_iy[r] = -(1 << 28);   // forces the bounds check to fail
            row_ix[r] = -(1 << 28);
            row_out[r] = -1;
        }
    }
    __syncthreads();

    // ---- global -> register staging of one k-tile --------------------------------
    constexpr int A_PER_THREAD = BM * BK / NT;          // scalars
    constexpr int A_VEC_PER_THREAD = BM * BK / 4 / NT;  // float4s
    constexpr int B_VEC_PER_THREAD = (BK * BN / 4 + NT - 1) / NT;
    float a_reg[A_PER_THREAD];
    float4 b_reg[B_VEC_PER_THREAD];   // Bs[k][c..c+3], k = f % BK, c = (f / BK) * 4

    auto load_tile = [&](int k0) {
        if (VEC_A) {
            // NHWC input, Cin % 4 == 0: a float4 never straddles a tap.
#pragma unroll
            for (int i = 0; i < A_VEC_PER_THREAD; ++i) {
                int f = tid + i * NT;
                int row = f / (BK / 4);
                int k = (f % (BK / 4)) * 4;
                int gk = k0 + k;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (gk < Ktot) {
                    int t = gk / p.Cin, ci = gk - t * p.Cin;
                    int iy = row_iy[row] + p.tap_dy[t], ix = row_ix[row] + p.tap_dx[t];
                    if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W)
                        v = __ldg(reinterpret_cast<const float4 *>(
                            p.in + row_in[row] + (long long)iy * p.in_sh + (long long)ix * p.in_sw + ci));
                }
                a_reg[i * 4 + 0] = v.x; a_reg[i * 4 + 1] = v.y;
                a_reg[i * 4 + 2] = v.z; a_reg[i * 4 + 3] = v.w;
            }
        } else {
            // generic strides (NCHW input or odd Cin): lanes run along m so that an
            // NCHW row of pixels is read contiguously.
#pragma unroll
            for (int i = 0; i < A_PER_THREAD; ++i) {
                int e = tid + i * NT;
                int row = e % BM, k = e / BM;
                int gk = k0 + k;
                float v = 0.f;
                if (gk < Ktot) {
                    int t = gk / p.Cin, ci = gk - t * p.Cin;
                    int iy = row_iy[row] + p.tap_dy[t], ix = row_ix[row] + p.tap_dx[t];
                    if (iy >= 0 && iy < p.H && ix >= 0 && ix < p.W)
                        v = __ldg(p.in + row_in[row] + (long long)iy * p.in_sh + (long long)ix * p.in_sw +
                                  (long long)ci * p.in_sc);
                }
                a_reg[i] = v;
            }
        }
#pragma unroll
        for (int i = 0; i < B_VEC_PER_THREAD; ++i) {
            int f = tid + i * NT;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            const int gk = k0 + f % BK, co = n0 + (f / BK) * 4;
            if (f < BK * BN / 4 && gk < Ktot) {
                // B[k = t*Cin + ci][co] is w[tap_w[t]][co][ci]: lanes run along ci, so a warp reads 64 contiguous
                // bytes of each of its weight rows
                const int t = gk / p.Cin, ci = gk - t * p.Cin;
                const float *wr = p.w + ((long long)p.tap_w[t] * p.Cout + co) * p.Cin + ci;
                if (co + 0 < p.Cout) v.x = __ldg(wr);
                if (co + 1 < p.Cout) v.y = __ldg(wr + p.Cin);
                if (co + 2 < p.Cout) v.z = __ldg(wr + 2 * p.Cin);
                if (co + 3 < p.Cout) v.w = __ldg(wr + 3 * p.Cin);
            }
            b_reg[i] = v;
        }
    };
    auto store_tile = [&](int buf) {
        if (VEC_A) {
#pragma unroll
            for (int i = 0; i < A_VEC_PER_THREAD; ++i) {
                int f = tid + i * NT;
                int row = f / (BK / 4), k = (f % (BK / 4)) * 4;
#pragma unroll
                for (int j = 0; j < 4; ++j) As[buf][k + j][row] = a_reg[i * 4 + j];
            }
        } else {
#pragma unroll
            for (int i = 0; i < A_PER_THREAD; ++i) {
                int e = tid + i * NT;
                As[buf][e / BM][e % BM] = a_reg[i];
            }
        }
#pragma unroll
        for (int i = 0; i < B_VEC_PER_THREAD; ++i) {
            int f = tid + i * NT;
            // (row pitch BN + BPAD = 4 mod 32 floats: the eight float4s of a quarter warp, k = 0..7 or 8..15, hit
            // distinct banks)
            if (f < BK * BN / 4) *reinterpret_cast<float4 *>(&Bs[buf][f % BK][(f / BK) * 4]) = b_reg[i];
        }
    };

    const int ty = tid / (BN / TN), tx = tid % (BN / TN);
    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    const int nk = (Ktot + BK - 1) / BK;
    load_tile(0);
    store_tile(0);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nk) load_tile((kt + 1) * BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[TM], b[TN];
#pragma unroll
            for (int i = 0; i < TM; i += 4) {
                float4 v = *reinterpret_cast<const float4 *>(&As[buf][k][ty * TM + i]);
                a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
            }
#pragma unroll
            for (int j = 0; j < TN; j += 4) {
                float4 v = *reinterpret_cast<const float4 *>(&Bs[buf][k][tx * TN + j]);
                b[j] = v.x; b[j + 1] = v.y; b[j + 2] = v.z; b[j + 3] = v.w;
            }
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (kt + 1 < nk) store_tile(buf ^ 1);
        __syncthreads();
    }

    // ---- epilogue: bias, skip, ReLU, store ---------------------------------------
    const bool vec_out = (p.out_sc == 1) && (p.Cout % 4 == 0);
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int r = ty * TM + i;
        const long long ob = row_out[r];
        if (ob < 0) continue;
#pragma unroll
        for (int j = 0; j < TN; j += 4) {
            const int co = n0 + tx * TN + j;
            float v[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                float x = acc[i][j + q];
                if (co + q < p.Cout) {
                    if (p.bias) x += __ldg(p.bias + co + q);
                    if (p.skip) x += __ldg(p.skip + ob + (long long)(co + q) * p.out_sc);
                    if (p.relu) x = fmaxf(x, 0.f);
                }
                v[q] = x;
            }
            if (vec_out && co + 3 < p.Cout) {
                *reinterpret_cast<float4 *>(p.out + ob + co) = make_float4(v[0], v[1], v[2], v[3]);
            } else {
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (co + q < p.Cout) p.out[ob + (long long)(co + q) * p.out_sc] = v[q];
            }
        }
    }
}

// ---- Cout <= 4 (decoder.py:34-35, ConvT 64->3): HBM-bound, one thread per pixel ----
// The packed weights of the launch's taps live in shared memory; each thread reads
// its NHWC input rows as float4 and keeps <= 4 accumulators.  The NCHW store of the
// module boundary is coalesced because consecutive threads own consecutive gx.
__global__ void __launch_bounds__(256) conv_small_cout_kernel(const ConvLaunch p) {
    extern __shared__ float wsm[];  // [ntaps][Cin][4]
    const int Cin = p.Cin;
    // each tap's K-major rows, read along ci, padded with zero rows to 4 output channels
    for (int i = threadIdx.x; i < p.ntaps * 4 * Cin; i += blockDim.x) {
        const int ci = i % Cin, row = i / Cin, co = row & 3, t = row >> 2;
        wsm[(t * Cin + ci) * 4 + co] = co < p.Cout ? __ldg(p.w + ((long long)p.tap_w[t] * p.Cout + co) * Cin + ci) : 0.f;
    }
    __syncthreads();
    const long long M = (long long)p.B * p.OHg * p.OWg;
    const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    const int gx = (int)(m % p.OWg);
    const long long tt = m / p.OWg;
    const int gy = (int)(tt % p.OHg);
    const int n = (int)(tt / p.OHg);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const bool vec = (p.in_sc == 1) && (Cin % 4 == 0);
    for (int t = 0; t < p.ntaps; ++t) {
        const int iy = gy * p.in_step + p.tap_dy[t], ix = gx * p.in_step + p.tap_dx[t];
        if (iy < 0 || iy >= p.H || ix < 0 || ix >= p.W) continue;
        const float *src = p.in + (long long)n * p.in_sn + (long long)iy * p.in_sh + (long long)ix * p.in_sw;
        const float4 *w4 = reinterpret_cast<const float4 *>(wsm + (size_t)t * Cin * 4);
        if (vec) {
            for (int ci = 0; ci < Cin; ci += 4) {
                const float4 x = __ldg(reinterpret_cast<const float4 *>(src + ci));
                const float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float4 w = w4[ci + q];
                    acc[0] = fmaf(xs[q], w.x, acc[0]); acc[1] = fmaf(xs[q], w.y, acc[1]);
                    acc[2] = fmaf(xs[q], w.z, acc[2]); acc[3] = fmaf(xs[q], w.w, acc[3]);
                }
            }
        } else {
            for (int ci = 0; ci < Cin; ++ci) {
                const float x = __ldg(src + (long long)ci * p.in_sc);
                const float4 w = w4[ci];
                acc[0] = fmaf(x, w.x, acc[0]); acc[1] = fmaf(x, w.y, acc[1]);
                acc[2] = fmaf(x, w.z, acc[2]); acc[3] = fmaf(x, w.w, acc[3]);
            }
        }
    }
    const long long ob = (long long)n * p.out_sn + (long long)(gy * p.out_step + p.out_py) * p.out_sh +
                         (long long)(gx * p.out_step + p.out_px) * p.out_sw;
    for (int co = 0; co < p.Cout; ++co) {
        float v = acc[co];
        if (p.bias) v += __ldg(p.bias + co);
        if (p.skip) v += __ldg(p.skip + ob + (long long)co * p.out_sc);
        if (p.relu) v = fmaxf(v, 0.f);
        p.out[ob + (long long)co * p.out_sc] = v;
    }
}

}  // namespace

int launch_conv_ffma(const ConvLaunch &p, cudaStream_t s) {
    const long long M = (long long)p.B * p.OHg * p.OWg;
    if (M <= 0) return 0;
    const bool vec_a = (p.in_sc == 1) && (p.Cin % 4 == 0) &&
                       (p.in_sn % 4 == 0) && (p.in_sh % 4 == 0) && (p.in_sw % 4 == 0);
    if (p.Cout > 32) {
        dim3 grid((unsigned)((M + 127) / 128), (unsigned)((p.Cout + 63) / 64));
        if (vec_a) conv_ffma_kernel<128, 64, 8, 4, true><<<grid, NT, 0, s>>>(p);
        else conv_ffma_kernel<128, 64, 8, 4, false><<<grid, NT, 0, s>>>(p);
    } else {
        dim3 grid((unsigned)((M + 127) / 128), (unsigned)((p.Cout + 31) / 32));
        if (vec_a) conv_ffma_kernel<128, 32, 4, 4, true><<<grid, NT, 0, s>>>(p);
        else conv_ffma_kernel<128, 32, 4, 4, false><<<grid, NT, 0, s>>>(p);
    }
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

int launch_conv_small_cout(const ConvLaunch &p, cudaStream_t s) {
    const long long M = (long long)p.B * p.OHg * p.OWg;
    if (M <= 0) return 0;
    const size_t smem = (size_t)p.ntaps * p.Cin * 4 * sizeof(float);
    if (smem > 48 * 1024) return VQB_ERR_UNSUPPORTED;
    conv_small_cout_kernel<<<(unsigned)((M + 255) / 256), 256, smem, s>>>(p);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

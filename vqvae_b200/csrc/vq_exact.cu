// vq_exact.cu -- fused VectorQuantizer.forward in canonical fp32 arithmetic (sm_90a).
//
// Replaces quantizer.py:45-71 (distance matrix, argmin, one-hot, one-hot @ codebook,
// loss numerator, straight-through, code histogram) with ONE persistent kernel that
// never materialises the (N,K) distance / one-hot matrices:
//   * a CTA owns 64 latent rows at a time and streams the codebook through shared
//     memory in 64-code chunks (so K*D of any size works);
//   * each thread owns a 4x4 (row, code) block and runs the dot products as
//     sequential fmaf chains over d = 0..D-1 -- exactly the canonical order of
//     oracle/csrc/oracle.c, which matched the reference bit for bit on every golden
//     case -- then d = fl(fl(A+B) - fl(2*M)) with non-contracted intrinsics;
//   * (min, idx) is kept per thread (ascending k => first minimum wins, NaN wins like
//     torch.argmin), merged across the 16 threads of a row with shuffles;
//   * the same launch gathers e_idx, writes z_q = z + (e - z), accumulates the SSE and a
//     shared-memory code histogram that is flushed once per CTA.
// The bf16 pipeline takes z_q as bf16 rows from the same launch (zq_bf16).  vq_tc_kernel (below) gives the same
// outputs with the distance GEMM on tensor cores.
#include <math.h>

#include "common.cuh"
#include "bf16_common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace {

constexpr int VR = 64;    // rows per tile
constexpr int VC = 64;    // codes per chunk
constexpr int VNT = 256;  // threads
constexpr int VPAD = 4;

__device__ __forceinline__ bool vq_better(float dn, int kn, float db, int kb) {
    // torch.argmin order (quantizer.py:54): NaN is the minimum; ties -> lowest index.
    const bool nn = dn != dn, nb = db != db;
    if (nn || nb) return nn && (!nb || kn < kb);
    return dn < db || (dn == db && kn < kb);
}

__global__ void code_norms_kernel(const float *__restrict__ E, int K, int D, float *__restrict__ bn) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= K) return;
    const float *e = E + (size_t)k * D;
    float s = 0.f;
    for (int d = 0; d < D; ++d) s = __fadd_rn(s, __fmul_rn(e[d], e[d]));  // quantizer.py:50
    bn[k] = s;
}

__global__ void __launch_bounds__(VNT)
vq_exact_kernel(const float *__restrict__ z, const float *__restrict__ E, const float *__restrict__ bn,
                long long N, int K, int D, long long *__restrict__ idx, void *__restrict__ zq, int zq_bf16,
                double *__restrict__ partials, int *__restrict__ hist, int use_smem_hist) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *zs = reinterpret_cast<float *>(smem_raw);          // [D][VR+VPAD]
    float *es = zs + (size_t)D * (VR + VPAD);                 // [D][VC+VPAD]
    float *an = es + (size_t)D * (VC + VPAD);                 // [VR]
    float *bs = an + VR;                                      // [VC]
    int *best_k = reinterpret_cast<int *>(bs + VC);           // [VR]
    int *shist = best_k + VR;                                 // [K] when use_smem_hist
    __shared__ double red[VNT / 32];

    const int tid = threadIdx.x;
    const int ty = tid >> 4, tx = tid & 15;
    const long long ntiles = (N + VR - 1) / VR;
    double my_sse = 0.0;
    if (use_smem_hist)
        for (int k = tid; k < K; k += VNT) shist[k] = 0;

    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long r0 = tile * VR;
        __syncthreads();
        // z tile -> smem, transposed to [d][row]; rows past N read as zero
        for (int e4 = tid; e4 < VR * (D / 4); e4 += VNT) {
            const int row = e4 / (D / 4), d = (e4 % (D / 4)) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r0 + row < N) v = __ldg(reinterpret_cast<const float4 *>(z + (size_t)(r0 + row) * D + d));
            zs[(size_t)(d + 0) * (VR + VPAD) + row] = v.x;
            zs[(size_t)(d + 1) * (VR + VPAD) + row] = v.y;
            zs[(size_t)(d + 2) * (VR + VPAD) + row] = v.z;
            zs[(size_t)(d + 3) * (VR + VPAD) + row] = v.w;
        }
        __syncthreads();
        if (tid < VR) {  // A_i = sum_d fl(z^2), left to right (quantizer.py:49)
            float s = 0.f;
            for (int d = 0; d < D; ++d) {
                const float v = zs[(size_t)d * (VR + VPAD) + tid];
                s = __fadd_rn(s, __fmul_rn(v, v));
            }
            an[tid] = s;
        }
        float bd[4];
        int bk[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { bd[i] = 0.f; bk[i] = -1; }

        for (int c0 = 0; c0 < K; c0 += VC) {
            __syncthreads();
            for (int e4 = tid; e4 < VC * (D / 4); e4 += VNT) {
                const int c = e4 / (D / 4), d = (e4 % (D / 4)) * 4;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (c0 + c < K) v = __ldg(reinterpret_cast<const float4 *>(E + (size_t)(c0 + c) * D + d));
                es[(size_t)(d + 0) * (VC + VPAD) + c] = v.x;
                es[(size_t)(d + 1) * (VC + VPAD) + c] = v.y;
                es[(size_t)(d + 2) * (VC + VPAD) + c] = v.z;
                es[(size_t)(d + 3) * (VC + VPAD) + c] = v.w;
            }
            if (tid < VC) bs[tid] = (c0 + tid < K) ? __ldg(bn + c0 + tid) : 0.f;
            __syncthreads();
            float acc[4][4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 4
            for (int d = 0; d < D; ++d) {
                const float4 a = *reinterpret_cast<const float4 *>(zs + (size_t)d * (VR + VPAD) + ty * 4);
                const float4 b = *reinterpret_cast<const float4 *>(es + (size_t)d * (VC + VPAD) + tx * 4);
                const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = __fmaf_rn(av[i], bv[j], acc[i][j]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float A = an[ty * 4 + i];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int k = c0 + tx * 4 + j;
                    if (k < K) {
                        // d = fl(fl(A + B) - fl(2*M))   quantizer.py:49-51
                        const float dist = __fsub_rn(__fadd_rn(A, bs[tx * 4 + j]), __fmul_rn(2.0f, acc[i][j]));
                        if (bk[i] < 0 || vq_better(dist, k, bd[i], bk[i])) { bd[i] = dist; bk[i] = k; }
                    }
                }
            }
        }
        // merge the 16 threads (tx) that share a row: lanes differ in the low 4 bits
#pragma unroll
        for (int i = 0; i < 4; ++i) {
#pragma unroll
            for (int off = 8; off >= 1; off >>= 1) {
                const float od = __shfl_xor_sync(0xffffffffu, bd[i], off);
                const int ok = __shfl_xor_sync(0xffffffffu, bk[i], off);
                if (ok >= 0 && (bk[i] < 0 || vq_better(od, ok, bd[i], bk[i]))) { bd[i] = od; bk[i] = ok; }
            }
            if (tx == 0) best_k[ty * 4 + i] = bk[i];
        }
        __syncthreads();
        // gather + straight-through + SSE + histogram; 16 threads per row, float4 each
        for (int rr = 0; rr < VR; rr += VNT / 16) {
            const int row = rr + (tid >> 4);
            const long long grow = r0 + row;
            if (grow < N) {
                const int k = best_k[row];
                const float *zr = z + (size_t)grow * D;
                const float *er = E + (size_t)k * D;
                for (int d = tx * 4; d < D; d += 64) {
                    const float4 zv = __ldg(reinterpret_cast<const float4 *>(zr + d));
                    const float4 ev = __ldg(reinterpret_cast<const float4 *>(er + d));
                    float4 df, q;
                    df.x = __fsub_rn(ev.x, zv.x); df.y = __fsub_rn(ev.y, zv.y);
                    df.z = __fsub_rn(ev.z, zv.z); df.w = __fsub_rn(ev.w, zv.w);
                    q.x = __fadd_rn(zv.x, df.x); q.y = __fadd_rn(zv.y, df.y);   // quantizer.py:67
                    q.z = __fadd_rn(zv.z, df.z); q.w = __fadd_rn(zv.w, df.w);
                    if (zq_bf16)            // bf16 pipeline: z_q rows feed the decoder's bf16 conv
                        *reinterpret_cast<uint2 *>(reinterpret_cast<__nv_bfloat16 *>(zq) + (size_t)grow * D + d) =
                            make_uint2(pack_bf16(q.x, q.y), pack_bf16(q.z, q.w));
                    else
                        *reinterpret_cast<float4 *>(reinterpret_cast<float *>(zq) + (size_t)grow * D + d) = q;
                    my_sse += (double)df.x * df.x + (double)df.y * df.y + (double)df.z * df.z + (double)df.w * df.w;
                }
                if (tx == 0) {
                    idx[grow] = k;
                    if (use_smem_hist) atomicAdd(&shist[k], 1);
                    else atomicAdd(&hist[k], 1);
                }
            }
        }
    }
    // CTA reduction of the SSE partial (fixed order => deterministic)
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) my_sse += __shfl_xor_sync(0xffffffffu, my_sse, off);
    if ((tid & 31) == 0) red[tid >> 5] = my_sse;
    __syncthreads();
    if (tid == 0) {
        double s = 0.0;
        for (int w = 0; w < VNT / 32; ++w) s += red[w];
        partials[blockIdx.x] = s;
    }
    if (use_smem_hist)
        for (int k = tid; k < K; k += VNT) {
            const int c = shist[k];
            if (c) atomicAdd(&hist[k], c);
        }
}

__global__ void sum_partials_kernel(const double *__restrict__ partials, int n, double *__restrict__ out) {
    __shared__ double sh[256];
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) s += partials[i];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int off = 128; off >= 1; off >>= 1) {
        if (threadIdx.x < off) sh[threadIdx.x] += sh[threadIdx.x + off];
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = sh[0];
}

}  // namespace

// workspace: [K floats code norms | pad to 256 B | VQ_MAX_CTAS doubles]
constexpr int VQ_MAX_CTAS = 2048;

size_t vq_exact_workspace_bytes(int K) {
    return (((size_t)K * sizeof(float) + 255) / 256) * 256 + (size_t)VQ_MAX_CTAS * sizeof(double);
}

int launch_vq_exact(const float *z, const float *E, long long N, int K, int D, long long *idx, void *zq, int zq_bf16,
                    double *sse, int *hist, void *ws, cudaStream_t s) {
    float *bn = reinterpret_cast<float *>(ws);
    double *partials = reinterpret_cast<double *>(reinterpret_cast<unsigned char *>(ws) +
                                                  (((size_t)K * sizeof(float) + 255) / 256) * 256);
    cudaError_t e = cudaMemsetAsync(hist, 0, sizeof(int) * (size_t)K, s);
    if (e != cudaSuccess) return (int)e;
    code_norms_kernel<<<(K + 127) / 128, 128, 0, s>>>(E, K, D, bn);
    const size_t base = ((size_t)D * (VR + VPAD) + (size_t)D * (VC + VPAD) + VR + VC) * sizeof(float) +
                        VR * sizeof(int);
    const int use_smem_hist = (base + (size_t)K * sizeof(int) <= 200 * 1024) ? 1 : 0;
    const size_t smem = base + (use_smem_hist ? (size_t)K * sizeof(int) : 0);
    constexpr size_t kMaxDyn = 227 * 1024 - 1024;   // 227 KB per CTA minus static smem
    if (smem > kMaxDyn) return VQB_ERR_UNSUPPORTED;
    static bool attr_set = false;
    if (!attr_set) {
        e = cudaFuncSetAttribute(vq_exact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxDyn);
        if (e != cudaSuccess) return (int)e;
        attr_set = true;
    }
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int per_sm = (int)((227 * 1024) / (smem + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 4) per_sm = 4;
    const long long ntiles = (N + VR - 1) / VR;
    long long grid = (long long)sms * per_sm;
    if (grid > ntiles) grid = ntiles;
    if (grid > VQ_MAX_CTAS) grid = VQ_MAX_CTAS;
    if (grid < 1) grid = 1;
    vq_exact_kernel<<<(unsigned)grid, VNT, smem, s>>>(z, E, bn, N, K, D, idx, zq, zq_bf16, partials, hist, use_smem_hist);
    sum_partials_kernel<<<1, 256, 0, s>>>(partials, (int)grid, sse);
    VQB_COUNT_LAUNCH(3);
    return vqb_cuda_status(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ tensor-core VQ (D = 64)
// The same outputs as vq_exact_kernel, bit for bit, with the (N x K) distance work on Hopper tensor cores:
//   1. per 128-row tile (z rows in shared memory, 128-byte swizzle) the codebook streams through in chunks of 128 codes;
//      two warpgroups run wgmma m64n128k8 tf32 for the approximate scores s = ||e||^2 - 2 z.e, keep the running row
//      minimum and
//   2. collect every code whose score lies within the TF32 error bound of the minimum so far
//      (bound: 2^-6 ||z|| max||e|| + 2^-15 (||z||^2 + max||e||^2 + 2 ||z|| max||e||), far above the
//      2 * 2^-10 sum|z||e| of TF32 operand rounding plus the fp32 rounding of the canonical distance);
//   3. one thread per row re-scores its candidates in the canonical fp32 order of vq_exact_kernel and keeps the winner
//      with the same tie / NaN rule.  A row whose list overflows, or whose scores or norms are not finite, is re-scored
//      over all K codes: the result never depends on the approximation.
namespace {

constexpr int TC_ROWS = 128, TC_CODES = 128, TC_THREADS = 256, TC_CAP = 32;
constexpr int TC_TILE = 128 * 128;                            // one [128][128 B] operand chunk

__device__ __forceinline__ void tc_stage_rows(uint32_t base, const float *src, long long row0, long long nrows, int tid) {
    // rows of 64 fp32 -> two 128-byte-swizzled K chunks; rows past nrows are zero
    for (int e = tid; e < 128 * 16; e += TC_THREADS) {
        const int r = e >> 4, q = e & 15, chunk = q >> 3, j = q & 7;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row0 + r < nrows) v = __ldg(reinterpret_cast<const float4 *>(src + (size_t)(row0 + r) * 64) + q);
        const uint32_t addr = base + (uint32_t)(chunk * TC_TILE + r * 128 + ((j ^ (r & 7)) << 4));
        asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
    }
}

__global__ void __launch_bounds__(TC_THREADS, 1)
vq_tc_kernel(const float *__restrict__ z, const float *__restrict__ E, const float *__restrict__ bn, long long N, int K,
             int nchunks, long long *__restrict__ idx, void *__restrict__ zq, int zq_bf16, double *__restrict__ partials,
             int *__restrict__ hist, float *__restrict__ dbg, int dbg_cols) {
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    const uint32_t sbase = (raw + 1023u) & ~1023u;
    unsigned char *sm = smem_raw + (sbase - raw);
    const uint32_t zt = sbase, et = sbase + 2 * TC_TILE;
    float *bnc = reinterpret_cast<float *>(sm + 4 * TC_TILE);              // [TC_CODES]
    float *thr = bnc + TC_CODES;                                           // [TC_ROWS] running row minimum
    float *arow = thr + TC_ROWS;                                           // [TC_ROWS] canonical ||z||^2
    int *cnt = reinterpret_cast<int *>(arow + TC_ROWS);                    // [TC_ROWS] candidates (> TC_CAP: full scan)
    int *cand = cnt + TC_ROWS;                                             // [TC_ROWS][TC_CAP] candidate codes
    float *cands = reinterpret_cast<float *>(cand + TC_ROWS * TC_CAP);     // [TC_ROWS][TC_CAP] their approximate scores
    float *mg = cands + TC_ROWS * TC_CAP;                                  // [TC_ROWS] selection margin
    __shared__ float bmax_s;
    __shared__ double red[TC_THREADS / 32];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = warp >> 2, wl = warp & 3, cq = 2 * (lane & 3);
    if (tid == 0) bmax_s = 0.f;
    __syncthreads();
    {
        float m = 0.f;
        for (int k = tid; k < K; k += TC_THREADS) m = fmaxf(m, __ldg(bn + k));      // NaN norms: rows re-scored fully below
        for (int o = 16; o >= 1; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) atomicMax(reinterpret_cast<int *>(&bmax_s), __float_as_int(m));      // m >= 0: int order = float order
    }
    double my_sse = 0.0;
    const long long ntiles = (N + TC_ROWS - 1) / TC_ROWS;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long r0 = tile * TC_ROWS;
        __syncthreads();
        tc_stage_rows(zt, z, r0, N, tid);
        if (tid < TC_ROWS) {
            float s = 0.f;                                                  // quantizer.py:49, canonical order
            if (r0 + tid < N) {
                const float *zr = z + (size_t)(r0 + tid) * 64;
                for (int d = 0; d < 64; ++d) { const float v = __ldg(zr + d); s = __fadd_rn(s, __fmul_rn(v, v)); }
            }
            arow[tid] = s;
            thr[tid] = INFINITY;
            cnt[tid] = 0;
        }
        __syncthreads();
        if (tid < TC_ROWS) {           // the row's selection margin (see the header); not finite -> full re-scoring
            const float A = arow[tid], zn = sqrtf(A), en = sqrtf(bmax_s);
            const float mgv = 0.015625f * zn * en + 3.0517578125e-5f * (A + bmax_s + 2.f * zn * en);
            mg[tid] = mgv;
            if (!isfinite(mgv)) cnt[tid] = TC_CAP + 1;
        }
        // one sweep over the codebook: running row minimum of the approximate scores, and every code within the margin
        // of the minimum so far (codes that fall outside the final bound are dropped before re-scoring)
        const int np = dbg ? dbg_cols / TC_CODES : nchunks;
        for (int c = 0; c < np; ++c) {
            const int k0 = c * TC_CODES;
            __syncthreads();
            tc_stage_rows(et, E, k0, K, tid);
            if (tid < TC_CODES) bnc[tid] = k0 + tid < K ? __ldg(bn + k0 + tid) : INFINITY;
            ptx::fence_proxy_async();
            __syncthreads();
            float acc[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = 0.f;
            wg::fence();
#pragma unroll
            for (int ch = 0; ch < 2; ++ch)
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)
                    wg::mma<false, 128>(acc, wg::desc_sw128(zt + (uint32_t)(ch * TC_TILE + wgi * 64 * 128 + 32 * kk)),
                                        wg::desc_sw128(et + (uint32_t)(ch * TC_TILE + 32 * kk)), 1u);
            wg::commit();
            wg::wait<0>();
            wg::fence_regs<128>(acc);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = wgi * 64 + wl * 16 + (lane >> 2) + 8 * h;
                const bool live = r0 + row < N;
                float mn = INFINITY;
                bool bad = false;
#pragma unroll
                for (int j = 0; j < 16; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = 8 * j + cq + e;
                        const float sc = __fsub_rn(bnc[col], 2.f * acc[4 * j + 2 * h + e]);
                        acc[4 * j + 2 * h + e] = sc;
                        if (dbg && live) dbg[(size_t)(r0 + row) * dbg_cols + k0 + col] = sc;
                        if (k0 + col < K) { bad |= !(sc == sc); mn = fminf(mn, sc); }
                    }
                mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, 1));
                mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, 2));
                const float rm = fminf(thr[row], mn);
                const float t = rm + mg[row];
                if (live) {
#pragma unroll
                    for (int j = 0; j < 16; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = 8 * j + cq + e;
                            const float sc = acc[4 * j + 2 * h + e];
                            if (k0 + col < K && sc <= t) {
                                const int pos = atomicAdd(&cnt[row], 1);
                                if (pos < TC_CAP) { cand[row * TC_CAP + pos] = k0 + col; cands[row * TC_CAP + pos] = sc; }
                            }
                        }
                }
                __syncwarp();
                if ((lane & 3) == 0) thr[row] = rm;          // the row's four lanes read thr[row] above
                if (bad) cnt[row] = TC_CAP + 1;
            }
        }
        __syncthreads();
        // canonical re-scoring of the candidates within the final bound (all K codes when the list overflowed or a score /
        // norm was not finite)
        if (tid < TC_ROWS && r0 + tid < N) {
            const long long grow = r0 + tid;
            const float *zr = z + (size_t)grow * 64;
            const float A = arow[tid], t = thr[tid] + mg[tid];
            const int nc = cnt[tid];
            const bool full_scan = nc > TC_CAP || nc == 0;
            const int n_try = full_scan ? K : nc;
            float zv[64];
#pragma unroll
            for (int d = 0; d < 64; d += 4) {
                const float4 v = __ldg(reinterpret_cast<const float4 *>(zr + d));
                zv[d] = v.x; zv[d + 1] = v.y; zv[d + 2] = v.z; zv[d + 3] = v.w;
            }
            float bd = 0.f;
            int bk = -1;
            for (int i = 0; i < n_try; ++i) {
                if (!full_scan && cands[tid * TC_CAP + i] > t) continue;      // outside the final bound: cannot win
                const int k = full_scan ? i : cand[tid * TC_CAP + i];
                const float4 *er4 = reinterpret_cast<const float4 *>(E + (size_t)k * 64);
                float m = 0.f;
#pragma unroll
                for (int d = 0; d < 64; d += 4) {
                    const float4 ev = __ldg(er4 + d / 4);
                    m = __fmaf_rn(zv[d], ev.x, m); m = __fmaf_rn(zv[d + 1], ev.y, m);
                    m = __fmaf_rn(zv[d + 2], ev.z, m); m = __fmaf_rn(zv[d + 3], ev.w, m);
                }
                const float dist = __fsub_rn(__fadd_rn(A, __ldg(bn + k)), __fmul_rn(2.0f, m));   // quantizer.py:49-51
                if (bk < 0 || vq_better(dist, k, bd, bk)) { bd = dist; bk = k; }
            }
            const float *er = E + (size_t)bk * 64;
            for (int d = 0; d < 64; d += 4) {
                const float4 zv = __ldg(reinterpret_cast<const float4 *>(zr + d));
                const float4 ev = __ldg(reinterpret_cast<const float4 *>(er + d));
                float4 df, q;
                df.x = __fsub_rn(ev.x, zv.x); df.y = __fsub_rn(ev.y, zv.y);
                df.z = __fsub_rn(ev.z, zv.z); df.w = __fsub_rn(ev.w, zv.w);
                q.x = __fadd_rn(zv.x, df.x); q.y = __fadd_rn(zv.y, df.y);           // quantizer.py:67
                q.z = __fadd_rn(zv.z, df.z); q.w = __fadd_rn(zv.w, df.w);
                if (zq_bf16)
                    *reinterpret_cast<uint2 *>(reinterpret_cast<__nv_bfloat16 *>(zq) + (size_t)grow * 64 + d) =
                        make_uint2(pack_bf16(q.x, q.y), pack_bf16(q.z, q.w));
                else
                    *reinterpret_cast<float4 *>(reinterpret_cast<float *>(zq) + (size_t)grow * 64 + d) = q;
                my_sse += (double)df.x * df.x + (double)df.y * df.y + (double)df.z * df.z + (double)df.w * df.w;
            }
            idx[grow] = bk;
            atomicAdd(&hist[bk], 1);
        }
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) my_sse += __shfl_xor_sync(0xffffffffu, my_sse, off);
    if (lane == 0) red[warp] = my_sse;
    __syncthreads();
    if (tid == 0) {
        double s = 0.0;
        for (int w = 0; w < TC_THREADS / 32; ++w) s += red[w];
        partials[blockIdx.x] = s;
    }
}

}  // namespace

bool vq_tc_supported(long long N, int K, int D) { return D == 64 && N >= 1 && K >= 1 && K <= (1 << 20); }

// dbg != null: also writes the approximate scores as (N, ceil(K / 256) * 256) floats (padding codes score +inf)
int launch_vq_tc(const float *z, const float *E, long long N, int K, int D, long long *idx, void *zq, int zq_bf16, double *sse,
                 int *hist, void *ws, float *dbg, cudaStream_t s) {
    if (!vq_tc_supported(N, K, D)) return VQB_ERR_UNSUPPORTED;
    float *bn = reinterpret_cast<float *>(ws);
    double *partials = reinterpret_cast<double *>(reinterpret_cast<unsigned char *>(ws) +
                                                  (((size_t)K * sizeof(float) + 255) / 256) * 256);
    cudaError_t e = cudaMemsetAsync(hist, 0, sizeof(int) * (size_t)K, s);
    if (e != cudaSuccess) return (int)e;
    code_norms_kernel<<<(K + 127) / 128, 128, 0, s>>>(E, K, D, bn);
    const int smem = 4 * TC_TILE + (TC_CODES + 3 * TC_ROWS) * 4 + TC_ROWS * (1 + 2 * TC_CAP) * 4 + 1024;
    static bool attr_set = false;
    if (!attr_set) {
        e = cudaFuncSetAttribute(vq_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return (int)e;
        attr_set = true;
    }
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long ntiles = (N + TC_ROWS - 1) / TC_ROWS;
    long long grid = (long long)sms * 2;
    if (grid > ntiles) grid = ntiles;
    if (grid > VQ_MAX_CTAS) grid = VQ_MAX_CTAS;
    const int nchunks = (K + TC_CODES - 1) / TC_CODES;
    const int dbg_cols = (K + 255) / 256 * 256;
    vq_tc_kernel<<<(unsigned)grid, TC_THREADS, smem, s>>>(z, E, bn, N, K, nchunks, idx, zq, zq_bf16, partials, hist, dbg, dbg_cols);
    sum_partials_kernel<<<1, 256, 0, s>>>(partials, (int)grid, sse);
    VQB_COUNT_LAUNCH(3);
    return vqb_cuda_status(cudaGetLastError());
}

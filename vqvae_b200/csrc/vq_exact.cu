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

// workspace: [Kpad floats code norms (+inf past K) | VQ_MAX_CTAS doubles SSE partials | Kpad / 128 floats per-block
// maxima of the code norms | one counter of finished CTAs], Kpad = K rounded up to 256
constexpr int VQ_MAX_CTAS = 2048;

struct VqWorkspace {
    float *bn;
    double *partials;
    float *bmax_part;
    unsigned *done;
};

static size_t vq_kpad(int K) { return ((size_t)K + 255) / 256 * 256; }

static VqWorkspace vq_workspace(void *ws, int K) {
    unsigned char *p = reinterpret_cast<unsigned char *>(ws);
    const size_t kpad = vq_kpad(K);
    VqWorkspace w;
    w.bn = reinterpret_cast<float *>(p);
    w.partials = reinterpret_cast<double *>(p + kpad * sizeof(float));
    w.bmax_part = reinterpret_cast<float *>(w.partials + VQ_MAX_CTAS);
    w.done = reinterpret_cast<unsigned *>(w.bmax_part + kpad / 128);
    return w;
}

size_t vq_exact_workspace_bytes(int K) {
    const size_t kpad = vq_kpad(K);
    return kpad * sizeof(float) + (size_t)VQ_MAX_CTAS * sizeof(double) + kpad / 128 * sizeof(float) + 16;
}

constexpr size_t VQ_EXACT_MAX_DYN = 227 * 1024 - 1024;   // 227 KB per CTA minus static smem

// dynamic shared memory of vq_exact_kernel: its tiles, plus the code histogram when that fits
static size_t vq_exact_smem(int K, int D, int &use_smem_hist) {
    const size_t base = ((size_t)D * (VR + VPAD) + (size_t)D * (VC + VPAD) + VR + VC) * sizeof(float) +
                        VR * sizeof(int);
    use_smem_hist = (base + (size_t)K * sizeof(int) <= 200 * 1024) ? 1 : 0;
    return base + (use_smem_hist ? (size_t)K * sizeof(int) : 0);
}

bool vq_exact_supported(int K, int D) {
    int use_smem_hist;
    return vq_exact_smem(K, D, use_smem_hist) <= VQ_EXACT_MAX_DYN;
}

int launch_vq_exact(const float *z, const float *E, long long N, int K, int D, long long *idx, void *zq, int zq_bf16,
                    double *sse, int *hist, void *ws, cudaStream_t s) {
    const VqWorkspace w = vq_workspace(ws, K);
    float *bn = w.bn;
    double *partials = w.partials;
    cudaError_t e = cudaMemsetAsync(hist, 0, sizeof(int) * (size_t)K, s);
    if (e != cudaSuccess) return (int)e;
    code_norms_kernel<<<(K + 127) / 128, 128, 0, s>>>(E, K, D, bn);
    int use_smem_hist;
    const size_t smem = vq_exact_smem(K, D, use_smem_hist);
    if (smem > VQ_EXACT_MAX_DYN) return VQB_ERR_UNSUPPORTED;
    static bool attr_set = false;
    if (!attr_set) {
        e = cudaFuncSetAttribute(vq_exact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)VQ_EXACT_MAX_DYN);
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
//   1. per 128-row tile (z rows in shared memory, 128-byte swizzle) the codebook passes in chunks of 128 codes; two
//      warpgroups run wgmma m64n128k8 tf32 for the approximate scores s = ||e||^2 - 2 z.e, keep the running row
//      minimum and
//   2. collect every code whose score lies within the TF32 error bound of the minimum so far
//      (bound: 2^-6 ||z|| max||e|| + 2^-15 (||z||^2 + max||e||^2 + 2 ||z|| max||e||), far above the
//      2 * 2^-10 sum|z||e| of TF32 operand rounding plus the fp32 rounding of the canonical distance);
//   3. two threads per row re-score its candidates in the canonical fp32 order of vq_exact_kernel and keep the winner
//      with the same tie / NaN rule (a total order on (dist, k), so the split does not change the result).  A row whose
//      list overflows, or whose scores or norms are not finite, is re-scored over all K codes: the result never depends
//      on the approximation.
//
// Structure: one persistent CTA per SM, warp-specialised.  A producer warp loads z tiles (double-buffered, so the next
// tile arrives during this one's re-scoring) and codebook chunks with their code norms by TMA into an mbarrier ring.
// When the whole codebook fits in the ring (K <= 512 with the K-bin shared histogram beside it) it is loaded once per
// CTA and stays; otherwise it streams through the ring continuously across tiles.  The two consumer warpgroups own 64
// rows each and synchronise only through the ring and their own named barriers, so one warpgroup's epilogue runs while
// the other's wgmma are in flight.  The norms of the codes (canonical order) and their maximum are computed once per
// call by vq_prep_kernel; the row norms, the re-scoring and z_q all read z from the staged tile.  The SSE partials of
// the CTAs are summed in CTA order by the last CTA to finish, so a call is two launches (prep, main) and gives a
// bitwise-reproducible `sse`.
namespace {

constexpr int TC_ROWS = 128, TC_CODES = 128, TC_CAP = 24, TC_MAX_STAGES = 8;
constexpr int TC_CONSUMERS = 256, TC_THREADS = TC_CONSUMERS + 32;   // two consumer warpgroups + the producer warp
constexpr int TC_TILE = 128 * 128;                  // [128 rows][128 B]: 32 fp32 of K, 128-byte swizzle
constexpr int TC_CHUNK = 2 * TC_TILE;               // a z tile or a codebook chunk: 128 rows x 64 fp32
constexpr int TC_STAGE = TC_CHUNK + TC_CODES * 4;   // a chunk and its code norms
constexpr int TC_HIST_SMEM = 1024;                  // histogram in shared memory up to this K
constexpr int TC_BAR_ALL = 3;                       // named barrier of both consumer warpgroups (1, 2: one each)

struct TcArgs {
    const float *E, *bn, *bmax_part;
    long long N;
    int K, nch, stages, resident, nbpart, use_smem_hist, zq_bf16, dbg_cols;
    long long *idx;
    void *zq;
    double *partials, *sse;
    unsigned *done;
    int *hist;
    float *dbg;
};

// fp32 4q .. 4q+3 of row r of a [128][64] fp32 tile staged as two 128-byte-swizzled halves
__device__ __forceinline__ float4 ld_tile4(const unsigned char *tile, int r, int q) {
    return *reinterpret_cast<const float4 *>(tile + (q >> 3) * TC_TILE + r * 128 + (((q & 7) ^ (r & 7)) << 4));
}

// Code norms in the canonical order (quantizer.py:50; the arithmetic of code_norms_kernel), +inf for the padding codes
// up to the grid's end, the per-block maxima over the real codes (NaN norms drop out: those rows are re-scored fully),
// the zeroed histogram and the zeroed finished-CTA counter of vq_tc_kernel.
__global__ void __launch_bounds__(128)
vq_prep_kernel(const float *__restrict__ E, int K, float *__restrict__ bn, float *__restrict__ bmax_part,
               int *__restrict__ hist, unsigned *__restrict__ done) {
    __shared__ float wmax[4];
    pdl_wait();                        // hist may still be read by the stream's earlier work
    const int k = blockIdx.x * 128 + threadIdx.x;
    float s = INFINITY, m = 0.f;
    if (k < K) {
        const float4 *e4 = reinterpret_cast<const float4 *>(E + (size_t)k * 64);
        float4 v[16];
#pragma unroll
        for (int q = 0; q < 16; ++q) v[q] = __ldg(e4 + q);
        s = 0.f;
#pragma unroll
        for (int q = 0; q < 16; ++q) {
            s = __fadd_rn(s, __fmul_rn(v[q].x, v[q].x)); s = __fadd_rn(s, __fmul_rn(v[q].y, v[q].y));
            s = __fadd_rn(s, __fmul_rn(v[q].z, v[q].z)); s = __fadd_rn(s, __fmul_rn(v[q].w, v[q].w));
        }
        m = fmaxf(m, s);
        hist[k] = 0;
    }
    bn[k] = s;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) bmax_part[blockIdx.x] = fmaxf(fmaxf(wmax[0], wmax[1]), fmaxf(wmax[2], wmax[3]));
    if (k == 0) *done = 0u;
}

// DBG: also dump the approximate scores (vqb_debug_vq_scores_f32); a separate instantiation keeps the dump's address
// arithmetic out of the release kernel's registers.
template <bool DBG>
__global__ void __launch_bounds__(TC_THREADS, 1)
vq_tc_kernel(const __grid_constant__ CUtensorMap tma_z, const __grid_constant__ CUtensorMap tma_e,
             const __grid_constant__ TcArgs p) {
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    const uint32_t sbase = (raw + 1023u) & ~1023u;
    unsigned char *sm = smem_raw + (sbase - raw);
    const int S = p.stages;
    // [z tile][z tile][S codebook chunks][S x 128 code norms][K histogram bins when use_smem_hist]
    const uint32_t ring = sbase + 2 * TC_CHUNK;
    const unsigned char *rings = sm + 2 * TC_CHUNK;
    float *bnr = reinterpret_cast<float *>(sm + (size_t)(2 + S) * TC_CHUNK);
    int *shist = reinterpret_cast<int *>(bnr + S * TC_CODES);
    __shared__ __align__(8) uint64_t bars[2 * TC_MAX_STAGES + 4];
    __shared__ float thr[TC_ROWS], arow[TC_ROWS], mg[TC_ROWS];     // running row minimum, canonical ||z||^2, margin
    __shared__ int cnt[TC_ROWS], best_k[TC_ROWS];                    // candidates (> TC_CAP: full scan), winner
    __shared__ int cand[TC_ROWS * TC_CAP];                           // candidate codes
    __shared__ float cands[TC_ROWS * TC_CAP];                        // their approximate scores
    __shared__ float bmax_s;
    __shared__ double red[TC_CONSUMERS / 32];
    auto full = [&](int s) { return ptx::smem_u32(&bars[s]); };                     // chunk landed (TMA bytes)
    auto empty = [&](int s) { return ptx::smem_u32(&bars[TC_MAX_STAGES + s]); };    // 8 consumer warps done with it
    auto zfull = [&](int b) { return ptx::smem_u32(&bars[2 * TC_MAX_STAGES + b]); };
    auto zempty = [&](int b) { return ptx::smem_u32(&bars[2 * TC_MAX_STAGES + 2 + b]); };   // both warpgroups done

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const long long ntiles = (p.N + TC_ROWS - 1) / TC_ROWS;
    if (tid == 0) {
        for (int s = 0; s < S; ++s) { ptx::mbar_init(full(s), 1); ptx::mbar_init(empty(s), TC_CONSUMERS / 32); }
        for (int b = 0; b < 2; ++b) { ptx::mbar_init(zfull(b), 1); ptx::mbar_init(zempty(b), 2); }
        ptx::fence_mbar_init();
        bmax_s = 0.f;
    }
    if (tid == TC_CONSUMERS) { ptx::prefetch_tmap(&tma_z); ptx::prefetch_tmap(&tma_e); }
    if (p.use_smem_hist)
        for (int k = tid; k < p.K; k += TC_THREADS) shist[k] = 0;
    __syncthreads();
    // z, the code norms, and every output: a previous call's consumers (a graph replay's decoder) may still read z_q
    pdl_wait();

    if (warp == TC_CONSUMERS / 32) {   // ------------------------------------------------ producer
        if (lane == 0) {
            int rs = 0;                // ring slot and the number of times the ring has wrapped, continued across tiles
            uint32_t wraps = 0;
            int it = 0;
            for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
                const int b = it & 1;
                const int row0 = (int)(tile * TC_ROWS);
                if (it >= 2) ptx::mbar_wait(zempty(b), (uint32_t)(((it >> 1) - 1) & 1));
                ptx::mbar_expect_tx(zfull(b), (uint32_t)TC_CHUNK);
                ptx::tma_load_2d(sbase + (uint32_t)(b * TC_CHUNK), &tma_z, zfull(b), 0, row0);
                ptx::tma_load_2d(sbase + (uint32_t)(b * TC_CHUNK + TC_TILE), &tma_z, zfull(b), 32, row0);
                if (p.resident && it > 0) continue;          // the whole codebook stays in the ring
                for (int c = 0; c < p.nch; ++c) {
                    const int s = rs;
                    if (wraps > 0) ptx::mbar_wait(empty(s), (wraps - 1) & 1);
                    if (++rs == S) { rs = 0; ++wraps; }
                    ptx::mbar_expect_tx(full(s), (uint32_t)TC_STAGE);
                    const uint32_t dst = ring + (uint32_t)(s * TC_CHUNK);
                    ptx::tma_load_2d(dst, &tma_e, full(s), 0, c * TC_CODES);
                    ptx::tma_load_2d(dst + TC_TILE, &tma_e, full(s), 32, c * TC_CODES);
                    ptx::bulk_load_1d(ptx::smem_u32(bnr + s * TC_CODES), p.bn + (size_t)c * TC_CODES, TC_CODES * 4, full(s));
                }
            }
        }
        __syncwarp();
        return;
    }

    // ------------------------------------------------------------------------------------ consumers
    const int wgi = warp >> 2, wl = warp & 3, wt = tid & 127, cq = 2 * (lane & 3);
    const uint32_t wg_bar = 1u + (uint32_t)wgi;
    {
        float m = 0.f;
        for (int i = tid; i < p.nbpart; i += TC_CONSUMERS) m = fmaxf(m, __ldg(p.bmax_part + i));
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) atomicMax(reinterpret_cast<int *>(&bmax_s), __float_as_int(m));      // m >= 0: int order = float order
        ptx::named_bar_sync(TC_BAR_ALL, TC_CONSUMERS);
    }
    const float bmax = bmax_s;
    // E row k, fp32 4q .. 4q+3: from the resident ring, or from L2
    auto ld_code4 = [&](int k, int q) -> float4 {
        if (p.resident) return ld_tile4(rings + (size_t)(k >> 7) * TC_CHUNK, k & 127, q);
        return __ldg(reinterpret_cast<const float4 *>(p.E + (size_t)k * 64) + q);
    };

    double my_sse = 0.0;
    int rs = 0;                        // ring slot and its fill parity, as the producer steps them
    uint32_t rpar = 0;
    int it = 0;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
        const long long r0 = tile * TC_ROWS;
        const int b = it & 1;
        const uint32_t zt = sbase + (uint32_t)(b * TC_CHUNK);
        const unsigned char *zs = sm + b * TC_CHUNK;
        ptx::mbar_wait(zfull(b), (uint32_t)((it >> 1) & 1));
        if (wt < 64) {                 // A_i (quantizer.py:49, canonical order) and the selection margin (see the header)
            const int row = wgi * 64 + wt;
            float s = 0.f;             // rows past N were zero-filled by the TMA: never written out
#pragma unroll
            for (int q = 0; q < 16; ++q) {
                const float4 v = ld_tile4(zs, row, q);
                s = __fadd_rn(s, __fmul_rn(v.x, v.x)); s = __fadd_rn(s, __fmul_rn(v.y, v.y));
                s = __fadd_rn(s, __fmul_rn(v.z, v.z)); s = __fadd_rn(s, __fmul_rn(v.w, v.w));
            }
            const float zn = sqrtf(s), en = sqrtf(bmax);
            const float mgv = 0.015625f * zn * en + 3.0517578125e-5f * (s + bmax + 2.f * zn * en);
            arow[row] = s;
            thr[row] = INFINITY;
            mg[row] = mgv;
            cnt[row] = isfinite(mgv) ? 0 : TC_CAP + 1;     // not finite -> full re-scoring
        }
        ptx::named_bar_sync(wg_bar, 128);
        // one sweep over the codebook: running row minimum of the approximate scores, and every code within the margin
        // of the minimum so far (codes that fall outside the final bound are dropped before re-scoring)
        for (int c = 0; c < p.nch; ++c) {
            const int k0 = c * TC_CODES;
            int s;
            uint32_t par;
            if (p.resident) { s = c; par = 0u; }
            else {
                s = rs; par = rpar;
                if (++rs == S) { rs = 0; rpar ^= 1u; }
            }
            ptx::mbar_wait(full(s), par);
            const uint32_t et = ring + (uint32_t)(s * TC_CHUNK);
            const float *bnc = bnr + s * TC_CODES;
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
                const bool live = r0 + row < p.N;
                float mn = INFINITY;
                bool bad = false;
#pragma unroll
                for (int j = 0; j < 16; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int col = 8 * j + cq + e;
                        const float sc = __fsub_rn(bnc[col], 2.f * acc[4 * j + 2 * h + e]);
                        acc[4 * j + 2 * h + e] = sc;
                        if (DBG && live) p.dbg[(size_t)(r0 + row) * p.dbg_cols + k0 + col] = sc;
                        if (k0 + col < p.K) { bad |= !(sc == sc); mn = fminf(mn, sc); }
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
                            if (k0 + col < p.K && sc <= t) {
                                const int pos = atomicAdd(&cnt[row], 1);
                                if (pos < TC_CAP) { cand[row * TC_CAP + pos] = k0 + col; cands[row * TC_CAP + pos] = sc; }
                            }
                        }
                }
                __syncwarp();
                if ((lane & 3) == 0) thr[row] = rm;          // the row's four lanes read thr[row] above
                if (bad) cnt[row] = TC_CAP + 1;
            }
            __syncwarp();                                    // the warp's reads of the chunk and its norms are done
            if (!p.resident && lane == 0) ptx::mbar_arrive(empty(s));
        }
        ptx::named_bar_sync(wg_bar, 128);
        // canonical re-scoring of the candidates within the final bound (all K codes when the list overflowed or a score /
        // norm was not finite): two threads per row, two independent dot-product chains per thread
        {
            const int row = wgi * 64 + (wt >> 1), half = wt & 1;
            const long long grow = r0 + row;
            float bd = 0.f;
            int bk = -1;
            if (grow < p.N) {
                const float A = arow[row], t = thr[row] + mg[row];
                const int nc = cnt[row];
                const bool full_scan = nc > TC_CAP || nc == 0;
                const int n_try = full_scan ? p.K : nc;
                auto pick = [&](int i) -> int {          // -1: outside the final bound, cannot win
                    if (full_scan) return i;
                    return cands[row * TC_CAP + i] > t ? -1 : cand[row * TC_CAP + i];
                };
                for (int i = half; i < n_try; i += 4) {
                    int ka = pick(i), kb = i + 2 < n_try ? pick(i + 2) : -1;
                    if (ka < 0) { ka = kb; kb = -1; }
                    if (ka < 0) continue;
                    const int kb2 = kb >= 0 ? kb : ka;
                    float ma = 0.f, mb = 0.f;
#pragma unroll
                    for (int q = 0; q < 16; ++q) {
                        const float4 zv = ld_tile4(zs, row, q), ea = ld_code4(ka, q), eb = ld_code4(kb2, q);
                        ma = __fmaf_rn(zv.x, ea.x, ma); mb = __fmaf_rn(zv.x, eb.x, mb);
                        ma = __fmaf_rn(zv.y, ea.y, ma); mb = __fmaf_rn(zv.y, eb.y, mb);
                        ma = __fmaf_rn(zv.z, ea.z, ma); mb = __fmaf_rn(zv.z, eb.z, mb);
                        ma = __fmaf_rn(zv.w, ea.w, ma); mb = __fmaf_rn(zv.w, eb.w, mb);
                    }
                    const float da = __fsub_rn(__fadd_rn(A, __ldg(p.bn + ka)), __fmul_rn(2.0f, ma));   // quantizer.py:49-51
                    if (bk < 0 || vq_better(da, ka, bd, bk)) { bd = da; bk = ka; }
                    if (kb >= 0) {
                        const float db = __fsub_rn(__fadd_rn(A, __ldg(p.bn + kb)), __fmul_rn(2.0f, mb));
                        if (vq_better(db, kb, bd, bk)) { bd = db; bk = kb; }
                    }
                }
            }
            const float od = __shfl_xor_sync(0xffffffffu, bd, 1);
            const int ok = __shfl_xor_sync(0xffffffffu, bk, 1);
            if (ok >= 0 && (bk < 0 || vq_better(od, ok, bd, bk))) { bd = od; bk = ok; }
            if (half == 0 && grow < p.N) best_k[row] = bk;
        }
        ptx::named_bar_sync(wg_bar, 128);
        // gather + straight-through + SSE + histogram from the staged tile: 16 threads per row, coalesced row stores
        {
            const int q = wt & 15;
#pragma unroll 2
            for (int pass = 0; pass < 8; ++pass) {
                const int row = wgi * 64 + pass * 8 + (wt >> 4);
                const long long grow = r0 + row;
                if (grow >= p.N) continue;
                const int k = best_k[row];
                const float4 zv = ld_tile4(zs, row, q);
                const float4 ev = ld_code4(k, q);
                float4 df, o;
                df.x = __fsub_rn(ev.x, zv.x); df.y = __fsub_rn(ev.y, zv.y);
                df.z = __fsub_rn(ev.z, zv.z); df.w = __fsub_rn(ev.w, zv.w);
                o.x = __fadd_rn(zv.x, df.x); o.y = __fadd_rn(zv.y, df.y);           // quantizer.py:67
                o.z = __fadd_rn(zv.z, df.z); o.w = __fadd_rn(zv.w, df.w);
                if (p.zq_bf16)
                    *reinterpret_cast<uint2 *>(reinterpret_cast<__nv_bfloat16 *>(p.zq) + (size_t)grow * 64 + 4 * q) =
                        make_uint2(pack_bf16(o.x, o.y), pack_bf16(o.z, o.w));
                else
                    *reinterpret_cast<float4 *>(reinterpret_cast<float *>(p.zq) + (size_t)grow * 64 + 4 * q) = o;
                my_sse += (double)df.x * df.x + (double)df.y * df.y + (double)df.z * df.z + (double)df.w * df.w;
                if (q == 0) {
                    p.idx[grow] = k;
                    if (p.use_smem_hist) atomicAdd(&shist[k], 1);
                    else atomicAdd(&p.hist[k], 1);
                }
            }
        }
        ptx::named_bar_sync(wg_bar, 128);            // the warpgroup is done with the z tile and the row state
        if (wt == 0) ptx::mbar_arrive(zempty(b));
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) my_sse += __shfl_xor_sync(0xffffffffu, my_sse, off);
    if (lane == 0) red[warp] = my_sse;
    ptx::named_bar_sync(TC_BAR_ALL, TC_CONSUMERS);
    if (p.use_smem_hist)
        for (int k = tid; k < p.K; k += TC_CONSUMERS) {
            const int c = shist[k];
            if (c) atomicAdd(&p.hist[k], c);
        }
    if (tid == 0) {
        double s = 0.0;
        for (int w = 0; w < TC_CONSUMERS / 32; ++w) s += red[w];
        p.partials[blockIdx.x] = s;
        __threadfence();
        if (atomicAdd(p.done, 1u) == gridDim.x - 1) {      // the last CTA: sum the partials in CTA order
            __threadfence();
            double tot = 0.0;
            for (unsigned i = 0; i < gridDim.x; ++i) tot += __ldcg(p.partials + i);
            *p.sse = tot;
        }
    }
}

}  // namespace

bool vq_tc_supported(long long N, int K, int D) {
    return D == 64 && N >= 1 && N <= 0x7fffffffLL - TC_ROWS && K >= 1 && K <= (1 << 20);
}

// dbg != null: also writes the approximate scores as (N, ceil(K / 256) * 256) floats (padding codes score +inf)
int launch_vq_tc(const float *z, const float *E, long long N, int K, int D, long long *idx, void *zq, int zq_bf16, double *sse,
                 int *hist, void *ws, float *dbg, cudaStream_t s) {
    if (!vq_tc_supported(N, K, D)) return VQB_ERR_UNSUPPORTED;
    const VqWorkspace w = vq_workspace(ws, K);
    const int kpad = (int)vq_kpad(K);
    CUtensorMap tz, te;
    int rc = vqb_encode_tmap_2d(&tz, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, z, 64, (uint64_t)N, 256, 32, TC_ROWS,
                                CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    rc = vqb_encode_tmap_2d(&te, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, E, 64, (uint64_t)K, 256, 32, TC_CODES,
                            CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    auto *kernel = dbg ? vq_tc_kernel<true> : vq_tc_kernel<false>;
    static int max_dyn[2] = {-1, -1};
    int &md = max_dyn[dbg ? 1 : 0];
    if (md < 0) {
        cudaFuncAttributes fa;
        cudaError_t e = cudaFuncGetAttributes(&fa, kernel);
        if (e != cudaSuccess) return (int)e;
        const int m = 227 * 1024 - (int)fa.sharedSizeBytes;
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, m);
        if (e != cudaSuccess) return (int)e;
        md = m;
    }
    TcArgs a = {};
    a.E = E; a.bn = w.bn; a.bmax_part = w.bmax_part; a.N = N; a.K = K;
    a.nch = dbg ? kpad / TC_CODES : (K + TC_CODES - 1) / TC_CODES;
    a.nbpart = kpad / 128;
    a.use_smem_hist = K <= TC_HIST_SMEM;
    a.zq_bf16 = zq_bf16; a.dbg_cols = kpad;
    a.idx = idx; a.zq = zq; a.partials = w.partials; a.sse = sse; a.done = w.done; a.hist = hist; a.dbg = dbg;
    const int fixed = 1024 + 2 * TC_CHUNK + (a.use_smem_hist ? K * 4 : 0);
    int stages = (md - fixed) / TC_STAGE;
    if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
    if (stages > a.nch) stages = a.nch;
    if (stages < 1) return VQB_ERR_UNSUPPORTED;
    a.stages = stages;
    a.resident = a.nch <= stages;
    const size_t smem = (size_t)fixed + (size_t)stages * TC_STAGE;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long ntiles = (N + TC_ROWS - 1) / TC_ROWS;
    long long grid = sms;
    if (grid > ntiles) grid = ntiles;
    if (grid > VQ_MAX_CTAS) grid = VQ_MAX_CTAS;
    cudaError_t e = vqb_launch(vq_prep_kernel, dim3((unsigned)(kpad / 128)), dim3(128), 0, s, E, K, w.bn, w.bmax_part, hist,
                               w.done);
    if (e != cudaSuccess) return (int)e;
    e = vqb_launch(kernel, dim3((unsigned)grid), dim3(TC_THREADS), smem, s, tz, te, a);
    VQB_COUNT_LAUNCH(2);
    return vqb_cuda_status(e);
}

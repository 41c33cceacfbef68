// ffma_gemm.cuh -- the fp32 CUDA-core GEMM of both backwards (internal; shared by prior_gemm.cu and conv_wgrad.cu),
// the deterministic split of a weight gradient's reduction over positions, and the reduction of its chunk partials
// into the parameter's layout.
//
// gemm_kernel computes out(m, n) = sum over k of A(m, k) * B(k, n), one chunk of k per blockIdx.z.  It reads its
// operands through small accessor structs and writes through an epilogue.  Per CTA: a 64 x 64 tile, 16 k per step
// staged in shared memory, 4 x 4 outputs per thread, each one fmaf chain in ascending k.
// A weight gradient is an (M x cols) product reduced over positions.  The positions are cut into `splits` chunks of
// `chunk` positions (a function of the shapes only); one CTA sums one chunk into partials [splits][M][cols], and
// `wgrad_reduce_kernel` adds the chunks in chunk order.  No float atomics: the result is bitwise reproducible.
#pragma once
#include <type_traits>

#include "common.cuh"

namespace {

constexpr int BM = 64, BN = 64, BK = 16, GT = 256;       // CTA tile, k-step, threads (16 x 16, 4 x 4 outputs each)

constexpr long long WGRAD_CHUNK = 2048;          // at most this many positions per partial

struct WgradSplit {                              // `splits` chunks of `chunk` positions
    int splits, chunk;
};

inline int wgrad_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// about two CTAs per SM over the (bm x bn) tiles of an (M x N) gradient, chunks of at most WGRAD_CHUNK positions
// rounded to the k-step bk
inline WgradSplit wgrad_split(int M, int N, long long K, int bm, int bn, int bk) {
    const long long tiles = (long long)wgrad_cdiv(M, bm) * wgrad_cdiv(N, bn);
    long long s = wgrad_cdiv(2 * 132, tiles);
    s = s > wgrad_cdiv(K, WGRAD_CHUNK) ? s : wgrad_cdiv(K, WGRAD_CHUNK);
    s = s < wgrad_cdiv(K, bk) ? s : wgrad_cdiv(K, bk);
    const int chunk = wgrad_cdiv(wgrad_cdiv(K, s), bk) * bk;
    return {wgrad_cdiv(K, chunk), chunk};
}

// Job: partials [splits][M][cols] with cols = taps*Cin (+1 for the bias); column tap*Cin + ci -> w[m][ci][tap]
// (the (M, Cin, kh, kw) layout with tap = r*kw + s), the ones column -> bias[m].
struct RJob {
    const float *part;
    float *w, *bias;
    int M, Cin, taps, cols, splits;
};
constexpr int MAX_JOBS = 5;
struct RJobs {
    RJob j[MAX_JOBS];
};

__global__ void wgrad_reduce_kernel(RJobs jobs) {
    const RJob J = jobs.j[blockIdx.y];
    const long long total = (long long)J.M * J.cols, stride = total;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        float v = 0.f;
        for (int z = 0; z < J.splits; ++z) v += J.part[z * stride + i];
        const int m = (int)(i / J.cols), j = (int)(i % J.cols);
        if (j >= J.taps * J.Cin) {
            J.bias[m] = v;
        } else {
            const int tap = j / J.Cin, ci = j % J.Cin;
            J.w[((long long)m * J.Cin + ci) * J.taps + tap] = v;
        }
    }
}

// one launch reducing the first n jobs; `most` = the largest M * cols among them
inline void wgrad_reduce(cudaStream_t st, const RJobs &jobs, int n, long long most) {
    constexpr int threads = 256;
    const int blocks = wgrad_cdiv(most, threads) < 1024 ? wgrad_cdiv(most, threads) : 1024;
    wgrad_reduce_kernel<<<dim3(blocks, n), threads, 0, st>>>(jobs);
}

// ---- operand accessors: (i, j) -> float; j_fast: consecutive j are consecutive addresses -------------------------
// An accessor may also hand the kernel four consecutive rows (A operand) or columns (B operand) at once: it has a
// `vec` member, set when those four are contiguous and 16-byte aligned, and four(i, j), which returns (i..i+3, j) of
// an A operand or (i, j..j+3) of a B operand.  The kernel calls four() only when `vec` is set, for groups starting
// inside the tile's bounds.
template <class L, class = void>
constexpr bool has_vec = false;
template <class L>
constexpr bool has_vec<L, std::void_t<decltype(L::vec)>> = true;

struct Mat {                      // p[i][j], row length ld
    const float *p;
    int ld;
    static constexpr bool j_fast = true;
    __device__ __forceinline__ float operator()(int i, int j) const { return __ldg(p + (long long)i * ld + j); }
    // tc_gemm.cuh: 32 consecutive j of row i; a 32-wide k-step stays in a row when ld % 32 == 0
    __device__ __forceinline__ const float *seg(int i, long long j0) const { return p + (long long)i * ld + j0; }
    bool seg_ok() const { return ld % 32 == 0 && ((uintptr_t)p & 15) == 0; }
};

struct MatT {                     // p[j][i]
    const float *p;
    int ld;
    static constexpr bool j_fast = false;
    __device__ __forceinline__ float operator()(int i, int j) const { return __ldg(p + (long long)j * ld + i); }
};

template <class L>
struct WithOnes : L {             // column `cols` of ones after the columns of L: the bias gradient's column
    int cols;
    __device__ __forceinline__ float operator()(long long k, int n) const { return n < cols ? L::operator()(k, n) : 1.f; }
    // a group reaching the ones column goes element by element (the columns after it are never stored)
    __device__ __forceinline__ float4 four(long long k, int n) const {
        if (n + 3 < cols) return L::four(k, n);
        return make_float4((*this)(k, n), (*this)(k, n + 1), (*this)(k, n + 2), (*this)(k, n + 3));
    }
};

// ---- epilogue: (m, n, value) --------------------------------------------------------------------------------------
struct Partial {                  // wgrad: chunk z's partial of element (m, n) of an (M x cols) gradient
    float *part;
    long long M, cols;
    __device__ __forceinline__ void operator()(int m, int n, float v) const {
        part[(long long)blockIdx.z * M * cols + (long long)m * cols + n] = v;
    }
};

// ---- the GEMM: out(m, n) = sum over k in [z*chunk, min(K, (z+1)*chunk)) of A(m, k) * B(k, n), k ascending ----------
static_assert(BM == BN, "stage() fills both operands' tiles");

// Stage one k-step of operand l into S[kk][rr]: row (A) or column (B) r0 + rr < R at k = k0 + kk, kk < kn; 0 elsewhere.
template <bool IsB, class L>
__device__ __forceinline__ void stage(const L &l, float (&S)[BK][BM + 4], int r0, int R, long long k0, int kn) {
    const int tid = threadIdx.x;
    if constexpr (has_vec<L>) {
        if (l.vec) {                                   // one group of four per thread
            const int kk = tid / 16, rr = tid % 16 * 4, r = r0 + rr;
            const long long k = k0 + kk;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r < R && kk < kn) {
                if constexpr (IsB) v = l.four(k, r);
                else v = l.four(r, k);
            }
            *reinterpret_cast<float4 *>(&S[kk][rr]) = v;
            return;
        }
    }
    const bool r_fast = IsB ? l.j_fast : !l.j_fast;   // consecutive threads: consecutive addresses
#pragma unroll
    for (int q = 0; q < BM * BK / GT; ++q) {
        const int e = tid + q * GT;
        const int rr = r_fast ? e % BM : e / BK, kk = r_fast ? e / BM : e % BK, r = r0 + rr;
        const long long k = k0 + kk;
        float v = 0.f;
        if (r < R && kk < kn) {
            if constexpr (IsB) v = l(k, r);
            else v = l(r, k);
        }
        S[kk][rr] = v;
    }
}

template <class LA, class LB, class EP>
__global__ void __launch_bounds__(GT) gemm_kernel(LA a, LB b, EP ep, int M, int N, long long K, int chunk) {
    __shared__ __align__(16) float As[BK][BM + 4];
    __shared__ __align__(16) float Bs[BK][BN + 4];
    const int tid = threadIdx.x, tm = tid / 16, tn = tid % 16;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const long long k_begin = (long long)blockIdx.z * chunk;
    const int kc = (int)min((long long)chunk, K - k_begin);     // this chunk's k, counted in 32 bits
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int kd = 0; kd < kc; kd += BK) {
        stage<false>(a, As, m0, M, k_begin + kd, min(BK, kc - kd));
        stage<true>(b, Bs, n0, N, k_begin + kd, min(BK, kc - kd));
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            const float4 av = *reinterpret_cast<const float4 *>(&As[kk][tm * 4]);
            const float4 bv = *reinterpret_cast<const float4 *>(&Bs[kk][tn * 4]);
            const float ar[4] = {av.x, av.y, av.z, av.w}, br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int m = m0 + tm * 4 + i, n = n0 + tn * 4 + j;
            if (m < M && n < N) ep(m, n, acc[i][j]);
        }
}

// one launch: the (M x N) product over K, chunk z of sp on blockIdx.z
template <class LA, class LB, class EP>
void gemm(cudaStream_t st, LA a, LB b, EP ep, int M, int N, long long K, WgradSplit sp) {
    const dim3 grid(wgrad_cdiv(M, BM), wgrad_cdiv(N, BN), sp.splits);
    gemm_kernel<LA, LB, EP><<<grid, GT, 0, st>>>(a, b, ep, M, N, K, sp.chunk);
}

}  // namespace

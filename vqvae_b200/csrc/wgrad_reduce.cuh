// wgrad_reduce.cuh -- the deterministic split of a weight gradient's reduction over positions, and the reduction of
// its chunk partials into the parameter's layout (internal; shared by prior_bwd.cu and conv_wgrad.cu).
//
// A weight gradient is an (M x cols) product reduced over positions.  The positions are cut into `splits` chunks of
// `chunk` positions (a function of the shapes only); one CTA sums one chunk into partials [splits][M][cols], and
// `wgrad_reduce_kernel` adds the chunks in chunk order.  No float atomics: the result is bitwise reproducible.
#pragma once
#include "common.cuh"

namespace {

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

}  // namespace

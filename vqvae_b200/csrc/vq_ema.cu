// vq_ema.cu -- exponential-moving-average codebook update of a VectorQuantizer (van den Oord et al. 2017, app. A.1),
// with per-code row sums in a fixed order, the backward / loss finisher of the EMA model (commitment term only), and
// the dead-code restarts that may follow an update (see "dead-code restarts" below).
//
// One update, from the rows z (N, D) the VQ kernel quantized, their codes idx (clamped to [0, K-1]) and its hist:
//   N_k <- g N_k + (1-g) hist_k,   m_k <- g m_k + (1-g) s_k,   n = sum_k N_k,
//   e_k <- m_k / ((N_k + eps) / (n + K eps) * n)
// s_k = sum of the rows of code k in this order: the rows of k by ascending row index, cut into consecutive segments
// of EMA_SEG rows; each segment is one fp32 add chain, and the segment partials are added in segment order.  The bits
// depend on (z, idx) only.
//
// Five launches, no atomics on floats, no host synchronisation:
//   1 ema_count    one warp per chunk of rows: the chunk's count of every code -> cnt[(code, chunk)]; also
//                  N_k' into the workspace and the scan's tile flags zeroed
//   2 ema_scan     exclusive scan of cnt in (code, chunk) order (single pass, decoupled look-back) -> base
//   3 ema_scatter  one warp per chunk: each row id to base[(code, chunk)] + its rank among the chunk's rows of that
//                  code -- a stable counting sort of the row ids by code
//   4 ema_partial  one lane group (D/4 lanes, float4 loads) per segment: its fp32 add chain -> one partial
//   5 ema_finish   every CTA sums n = sum N_k' in the same fixed order; then per code: s_k, N, m and e
// A segment's partial lives in slot floor(cb_k / S) + k + j (cb_k = first sorted position of code k, j = segment
// number): strictly increasing in (k, j), so slots are unique and fewer than N / S + K + 1.
#include "common.cuh"

namespace {

constexpr int EMA_SEG = 256;          // rows per segment of s_k (part of the summation order: never change silently)
constexpr int EMA_KTILE = 4096;       // codes a chunk warp keeps in shared memory per pass
constexpr int EMA_SCAN_THREADS = 256, EMA_SCAN_ITEMS = 8, EMA_SCAN_TILE = EMA_SCAN_THREADS * EMA_SCAN_ITEMS;
constexpr int EMA_THREADS = 128;      // ema_partial / ema_finish
constexpr long long EMA_MATRIX_CAP = 1LL << 21;   // (code, chunk) counts kept at most (unless K alone is larger)

constexpr unsigned long long FLAG_AGG = 1ULL << 62, FLAG_PREFIX = 2ULL << 62, VALUE_MASK = (1ULL << 62) - 1;

struct EmaPlan {
    long long nchunks, rows_per_chunk, M, ntiles, nslots;
    size_t off_cnt, off_base, off_status, off_rows, off_part, off_nnew, total;
};

inline size_t align16(size_t x) { return (x + 15) & ~size_t(15); }

EmaPlan ema_plan(long long N, int K, int D) {
    EmaPlan p{};
    long long nch = (N + 255) / 256;                                  // at least 256 rows per chunk
    const long long cap = EMA_MATRIX_CAP / K > 1 ? EMA_MATRIX_CAP / K : 1;
    if (nch > cap) nch = cap;
    long long r = (N + nch - 1) / nch;
    r = (r + 31) / 32 * 32;
    p.rows_per_chunk = r;
    p.nchunks = (N + r - 1) / r;
    p.M = (long long)K * p.nchunks;
    p.ntiles = (p.M + 1 + EMA_SCAN_TILE - 1) / EMA_SCAN_TILE;
    p.nslots = N / EMA_SEG + K + 1;
    size_t o = 0;
    p.off_cnt = o;    o = align16(o + sizeof(unsigned) * (size_t)p.M);
    p.off_base = o;   o = align16(o + sizeof(long long) * (size_t)(p.M + 1));
    p.off_status = o; o = align16(o + sizeof(unsigned long long) * (size_t)(p.ntiles + 1));   // + the tile counter
    p.off_rows = o;   o = align16(o + sizeof(long long) * (size_t)N);
    p.off_part = o;   o = align16(o + sizeof(float) * (size_t)p.nslots * D);
    p.off_nnew = o;   o = align16(o + sizeof(float) * (size_t)K);
    p.total = o;
    return p;
}

__device__ __forceinline__ int clamp_code(long long k, int K) { return k < 0 ? 0 : (k >= K ? K - 1 : (int)k); }

__global__ void __launch_bounds__(32) ema_count(const long long *__restrict__ idx, const int *__restrict__ hist,
                                                const float *__restrict__ cluster_size, long long N, int K,
                                                long long rows_per_chunk, long long nchunks, float decay,
                                                unsigned *__restrict__ cnt, float *__restrict__ nnew,
                                                unsigned long long *__restrict__ status, long long ntiles) {
    __shared__ unsigned sc[EMA_KTILE];
    const int lane = threadIdx.x;
    const long long c = blockIdx.x;
    // side jobs, grid-stride: N_k' for the finisher's n, and the scan's tile flags (+ its tile counter) zeroed
    const float omg = 1.0f - decay;
    for (long long k = c * 32 + lane; k < K; k += (long long)gridDim.x * 32)
        nnew[k] = __fadd_rn(__fmul_rn(decay, cluster_size[k]), __fmul_rn(omg, (float)hist[k]));
    for (long long t = c * 32 + lane; t <= ntiles; t += (long long)gridDim.x * 32) status[t] = 0ULL;
    const long long r0 = c * rows_per_chunk;
    const long long r1 = r0 + rows_per_chunk < N ? r0 + rows_per_chunk : N;
    for (int kt = 0; kt < K; kt += EMA_KTILE) {
        const int kn = K - kt < EMA_KTILE ? K - kt : EMA_KTILE;
        for (int k = lane; k < kn; k += 32) sc[k] = 0u;
        __syncwarp();
        for (long long r = r0 + lane; r - lane < r1; r += 32) {
            const int k = r < r1 ? clamp_code(__ldg(idx + r), K) - kt : -1;
            const bool in = r < r1 && k >= 0 && k < kn;
            const unsigned peers = __match_any_sync(0xffffffffu, in ? k : -1);
            if (in && lane == __ffs(peers) - 1) sc[k] += __popc(peers);
            __syncwarp();
        }
        for (int k = lane; k < kn; k += 32) cnt[(long long)(kt + k) * nchunks + c] = sc[k];
        __syncwarp();
    }
}

// base[i] = sum_{j < i} cnt[j] for i in [0, M]; tiles taken in launch order from a counter so that every tile a CTA
// waits for has started.
__global__ void __launch_bounds__(EMA_SCAN_THREADS) ema_scan(const unsigned *__restrict__ cnt, long long M,
                                                             long long *__restrict__ base,
                                                             unsigned long long *status, long long ntiles) {
    __shared__ long long s_warp[EMA_SCAN_THREADS / 32];
    __shared__ long long s_prefix;
    __shared__ unsigned long long s_tile;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t == 0) s_tile = atomicAdd(status + ntiles, 1ULL);
    __syncthreads();
    const long long tile = (long long)s_tile;
    const long long i0 = tile * EMA_SCAN_TILE + (long long)t * EMA_SCAN_ITEMS;
    unsigned v[EMA_SCAN_ITEMS];
    long long sum = 0;
#pragma unroll
    for (int i = 0; i < EMA_SCAN_ITEMS; ++i) {
        v[i] = i0 + i < M ? cnt[i0 + i] : 0u;
        sum += v[i];
    }
    long long incl = sum;                          // inclusive scan of the thread sums: warp, then block
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    long long wpre = 0, agg = 0;
    for (int w = 0; w < EMA_SCAN_THREADS / 32; ++w) {
        if (w < warp) wpre += s_warp[w];
        agg += s_warp[w];
    }
    if (t == 0) {
        long long prefix = 0;
        if (tile == 0) {
            atomicExch(status + tile, FLAG_PREFIX | (unsigned long long)agg);
        } else {
            atomicExch(status + tile, FLAG_AGG | (unsigned long long)agg);
            for (long long j = tile - 1; j >= 0; --j) {
                unsigned long long s;
                do { s = atomicAdd(status + j, 0ULL); } while ((s >> 62) == 0);
                prefix += (long long)(s & VALUE_MASK);
                if ((s >> 62) == 2) break;
            }
            atomicExch(status + tile, FLAG_PREFIX | (unsigned long long)(prefix + agg));
        }
        s_prefix = prefix;
    }
    __syncthreads();
    long long run = s_prefix + wpre + incl - sum;
#pragma unroll
    for (int i = 0; i < EMA_SCAN_ITEMS; ++i) {
        if (i0 + i <= M) base[i0 + i] = run;
        run += v[i];
    }
}

__global__ void __launch_bounds__(32) ema_scatter(const long long *__restrict__ idx, long long N, int K,
                                                  long long rows_per_chunk, long long nchunks,
                                                  const long long *__restrict__ base, long long *__restrict__ rows) {
    __shared__ long long sp[EMA_KTILE];
    const int lane = threadIdx.x;
    const long long c = blockIdx.x;
    const unsigned lt = (1u << lane) - 1u;
    const long long r0 = c * rows_per_chunk;
    const long long r1 = r0 + rows_per_chunk < N ? r0 + rows_per_chunk : N;
    for (int kt = 0; kt < K; kt += EMA_KTILE) {
        const int kn = K - kt < EMA_KTILE ? K - kt : EMA_KTILE;
        for (int k = lane; k < kn; k += 32) sp[k] = base[(long long)(kt + k) * nchunks + c];
        __syncwarp();
        for (long long r = r0 + lane; r - lane < r1; r += 32) {
            const int k = r < r1 ? clamp_code(__ldg(idx + r), K) - kt : -1;
            const bool in = r < r1 && k >= 0 && k < kn;
            const unsigned peers = __match_any_sync(0xffffffffu, in ? k : -1);
            if (in) rows[sp[k] + __popc(peers & lt)] = r;
            __syncwarp();
            if (in && lane == __ffs(peers) - 1) sp[k] += __popc(peers);
            __syncwarp();
        }
    }
}

// first sorted position of code k and its row count
__device__ __forceinline__ void code_span(const long long *base, long long nchunks, int k, long long &cb, long long &n) {
    cb = base[(long long)k * nchunks];
    n = base[(long long)(k + 1) * nchunks] - cb;
}

__device__ __forceinline__ long long seg_slot(long long cb, int k) { return cb / EMA_SEG + k; }

__device__ __forceinline__ float4 add4(float4 a, float4 b) {
    return make_float4(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z), __fadd_rn(a.w, b.w));
}

// lanes per code / segment: D/4 float4 columns, at most one CTA's worth (wider rows loop over their columns)
__host__ __device__ __forceinline__ int group_lanes(int D) { return D / 4 < EMA_THREADS ? D / 4 : EMA_THREADS; }

__global__ void __launch_bounds__(EMA_THREADS) ema_partial(const float *__restrict__ z, int K, int D, long long nchunks,
                                                           const long long *__restrict__ base,
                                                           const long long *__restrict__ rows, long long nslots,
                                                           float *__restrict__ part) {
    const int L = group_lanes(D), G = EMA_THREADS / L, d4 = D / 4;
    const int g = threadIdx.x / L, lane = threadIdx.x - g * L;
    const long long s = (long long)blockIdx.x * G + g;
    if (g >= G || s >= nslots) return;
    int lo = 0, hi = K - 1;                     // the last code whose first slot is <= s
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (seg_slot(base[(long long)mid * nchunks], mid) <= s) lo = mid; else hi = mid - 1;
    }
    long long cb, n;
    code_span(base, nchunks, lo, cb, n);
    const long long j = s - seg_slot(cb, lo);
    if (j * EMA_SEG >= n) return;               // a slot no segment uses
    const long long start = cb + j * EMA_SEG;
    const int len = n - j * EMA_SEG < EMA_SEG ? (int)(n - j * EMA_SEG) : EMA_SEG;
    const float4 *z4 = reinterpret_cast<const float4 *>(z);
    for (int c = lane; c < d4; c += L) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
        for (int r = 0; r < len; ++r) acc = add4(acc, __ldg(z4 + rows[start + r] * d4 + c));
        reinterpret_cast<float4 *>(part)[s * d4 + c] = acc;
    }
}

__global__ void __launch_bounds__(EMA_THREADS) ema_finish(int K, int D, long long nchunks,
                                                          const long long *__restrict__ base,
                                                          const float *__restrict__ part,
                                                          const float *__restrict__ nnew, float decay, float eps,
                                                          float *__restrict__ cluster_size,
                                                          float *__restrict__ embed_sum, float *__restrict__ codebook) {
    __shared__ float sh[EMA_THREADS];
    // n = sum_k N_k': per thread in k order, then a fixed tree -- the same order in every CTA
    float acc = 0.f;
    for (int k = threadIdx.x; k < K; k += EMA_THREADS) acc = __fadd_rn(acc, nnew[k]);
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int o = EMA_THREADS / 2; o >= 1; o >>= 1) {
        if (threadIdx.x < o) sh[threadIdx.x] = __fadd_rn(sh[threadIdx.x], sh[threadIdx.x + o]);
        __syncthreads();
    }
    const float n = sh[0];
    const float denom = __fadd_rn(n, __fmul_rn((float)K, eps));
    const float omg = 1.0f - decay;
    const int L = group_lanes(D), G = EMA_THREADS / L, d4 = D / 4;
    const int g = threadIdx.x / L, lane = threadIdx.x - g * L;
    if (g >= G) return;
    for (int k = blockIdx.x * G + g; k < K; k += gridDim.x * G) {
        const float Nk = nnew[k];
        const float Nt = __fmul_rn(__fdiv_rn(__fadd_rn(Nk, eps), denom), n);
        long long cb, cnt;
        code_span(base, nchunks, k, cb, cnt);
        const long long s0 = seg_slot(cb, k), nseg = (cnt + EMA_SEG - 1) / EMA_SEG;
        for (int c = lane; c < d4; c += L) {
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 8
            for (long long j = 0; j < nseg; ++j) s = add4(s, reinterpret_cast<const float4 *>(part)[(s0 + j) * d4 + c]);
            float4 *m4 = reinterpret_cast<float4 *>(embed_sum) + (long long)k * d4 + c;
            float4 m = *m4;
            m.x = __fadd_rn(__fmul_rn(decay, m.x), __fmul_rn(omg, s.x));
            m.y = __fadd_rn(__fmul_rn(decay, m.y), __fmul_rn(omg, s.y));
            m.z = __fadd_rn(__fmul_rn(decay, m.z), __fmul_rn(omg, s.z));
            m.w = __fadd_rn(__fmul_rn(decay, m.w), __fmul_rn(omg, s.w));
            *m4 = m;
            reinterpret_cast<float4 *>(codebook)[(long long)k * d4 + c] =
                make_float4(__fdiv_rn(m.x, Nt), __fdiv_rn(m.y, Nt), __fdiv_rn(m.z, Nt), __fdiv_rn(m.w, Nt));
        }
        if (lane == 0) cluster_size[k] = Nk;
    }
}

// dz = g_zq + g_loss * 2 beta / (N D) * (z - zq): the commitment term's gradient, from the forward's own z_q rows
__global__ void vq_commit_backward_kernel(const float *__restrict__ g_zq, const float *__restrict__ g_loss,
                                          const float *__restrict__ z, const float *__restrict__ zq, long long total4,
                                          long long N, int D, float beta, float *__restrict__ dz) {
    const float gl = g_loss ? __ldg(g_loss) : 0.f;
    const float c = gl * 2.0f / ((float)N * (float)D) * beta;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
        const float4 zv = __ldg(reinterpret_cast<const float4 *>(z) + i);
        const float4 qv = __ldg(reinterpret_cast<const float4 *>(zq) + i);
        float4 g = g_zq ? __ldg(reinterpret_cast<const float4 *>(g_zq) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        g.x = fmaf(c, zv.x - qv.x, g.x); g.y = fmaf(c, zv.y - qv.y, g.y);
        g.z = fmaf(c, zv.z - qv.z, g.z); g.w = fmaf(c, zv.w - qv.w, g.w);
        reinterpret_cast<float4 *>(dz)[i] = g;
    }
}

int sm_count() {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms;
}

// ---- dead-code restarts (vqb_vq_ema_restart_f32), run after an update --------------------------------------------
// From the rows z (N, D) the update consumed, uniforms u (N) in [0, 1) and a threshold t:
//   dead codes k_0 < k_1 < ... < k_{M-1}: N_k < t (strict, so a NaN N_k is not dead)
//   rows r_0, r_1, ...: the rows ordered by (u_i, i) ascending -- uniform sampling without replacement
//   for j < R = min(M, N):  e_{k_j} <- z_{r_j},  m_{k_j} <- fl(t z_{r_j}),  N_{k_j} <- t;   *n_restarted = R
// Row i's key is (bits of u_i) << 32 | i.  For u >= 0 the bit order is the value order, and the row index makes every
// key unique, so the R rows are the R smallest keys and their order is the keys' order.
//
// Twelve launches, no host synchronisation, no float atomics; every kernel after the first returns at once when R = 0:
//   1      rs_compact  one CTA: the dead flags in code order -> dead list, M, *n_restarted; counts zeroed
//   2..9   rs_digits   pass p: counts of digit p (8 bits, from the top) over the keys whose digits 0..p-1 are those of
//                      T, the R-th smallest key (every CTA derives them from passes 0..p-1); integer atomics only
//   10     rs_collect  the R keys <= T into a list (integer atomics pick the slots: the set is fixed, not the order)
//   11     rs_rank     each listed key's rank j among the R: the count of listed keys below it, one CTA per (256 keys,
//                      chunk of RS_RANK_CHUNK keys), the chunk counts added with integer atomics -- a sort, R^2 compares
//                      spread over the GPU
//   12     rs_assign   one thread per (listed key, float4 column): the copies into e, m and N of code k_j
constexpr int RS_MAX_K = 8192;                       // one CTA compacts the flags (8 per thread); R^2 rank compares
constexpr long long RS_MAX_N = 0xFFFFFFFFLL;         // the row index fills the key's low 32 bits; counts fit unsigned
constexpr int RS_THREADS = 256, RS_PASSES = 8, RS_COMPACT_THREADS = 1024, RS_RANK_CHUNK = 1024;

struct RestartPlan {
    size_t off_meta, off_dead, off_digits, off_keys, off_rank, total;
};

RestartPlan restart_plan(int K) {
    RestartPlan p{};
    size_t o = 0;
    p.off_meta = o;   o = align16(o + 2 * sizeof(int));                                  // M, the collect counter
    p.off_dead = o;   o = align16(o + sizeof(int) * (size_t)K);
    p.off_digits = o; o = align16(o + sizeof(unsigned) * RS_PASSES * 256);
    p.off_keys = o;   o = align16(o + sizeof(unsigned long long) * (size_t)K);
    p.off_rank = o;   o = align16(o + sizeof(int) * (size_t)K);
    p.total = o;
    return p;
}

__device__ __forceinline__ unsigned long long rs_key(const float *u, long long i) {
    return ((unsigned long long)__float_as_uint(__ldg(u + i)) << 32) | (unsigned long long)i;
}

__device__ __forceinline__ long long rs_count(const int *meta, long long N) {
    return (long long)meta[0] < N ? (long long)meta[0] : N;
}

// The digits 0..npass-1 of T, the R-th smallest key, from the counts of those passes (every thread of the CTA calls
// it; blockDim.x == 256, one digit per thread).  After all eight passes this is T itself.
__device__ unsigned long long rs_prefix(const unsigned *digits, int npass, long long R) {
    __shared__ unsigned long long s_prefix;
    __shared__ long long s_rank;
    __shared__ unsigned s_warp[RS_THREADS / 32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t == 0) { s_prefix = 0ULL; s_rank = R; }
    __syncthreads();
    for (int q = 0; q < npass; ++q) {
        const long long rank = s_rank;              // 1-based rank of T among the keys matching the digits so far
        const unsigned c = digits[q * 256 + t];
        unsigned incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        for (int w = 0; w < warp; ++w) incl += s_warp[w];
        const long long before = (long long)incl - c;
        if (before < rank && rank <= (long long)incl) {    // exactly one digit holds the rank
            s_prefix |= (unsigned long long)t << (56 - 8 * q);
            s_rank = rank - before;
        }
        __syncthreads();
    }
    return s_prefix;
}

__global__ void __launch_bounds__(RS_COMPACT_THREADS) rs_compact(const float *__restrict__ cluster_size, int K,
                                                                 long long N, float thr, int *__restrict__ meta,
                                                                 int *__restrict__ dead, unsigned *__restrict__ digits,
                                                                 int *__restrict__ rank, int *__restrict__ n_restarted) {
    __shared__ int s_warp[RS_COMPACT_THREADS / 32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    for (int i = t; i < RS_PASSES * 256; i += RS_COMPACT_THREADS) digits[i] = 0u;
    for (int i = t; i < K; i += RS_COMPACT_THREADS) rank[i] = 0;
    if (t == 0) meta[1] = 0;
    const int per = (K + RS_COMPACT_THREADS - 1) / RS_COMPACT_THREADS;    // <= 8 codes per thread, in code order
    const int k0 = t * per;
    unsigned flags = 0u;
    for (int q = 0; q < per; ++q)
        if (k0 + q < K && cluster_size[k0 + q] < thr) flags |= 1u << q;
    const int cnt = __popc(flags);
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int pos = incl - cnt, M = 0;
    for (int w = 0; w < RS_COMPACT_THREADS / 32; ++w) {
        if (w < warp) pos += s_warp[w];
        M += s_warp[w];
    }
    for (int q = 0; q < per; ++q)
        if (flags >> q & 1u) dead[pos++] = k0 + q;
    if (t == 0) {
        meta[0] = M;
        n_restarted[0] = (int)((long long)M < N ? (long long)M : N);
    }
}

__global__ void __launch_bounds__(RS_THREADS) rs_digits(const float *__restrict__ u, long long N,
                                                        const int *__restrict__ meta, unsigned *digits, int pass) {
    __shared__ unsigned h[256];
    const long long R = rs_count(meta, N);
    if (R == 0) return;
    const unsigned long long prefix = rs_prefix(digits, pass, R);
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    h[t] = 0u;
    __syncthreads();
    const int shift = 56 - 8 * pass;
    const unsigned long long high = pass == 0 ? 0ULL : ~0ULL << (shift + 8);
    for (long long i0 = (long long)blockIdx.x * RS_THREADS + warp * 32; i0 < N; i0 += (long long)gridDim.x * RS_THREADS) {
        const long long i = i0 + lane;
        int d = -1;
        if (i < N) {
            const unsigned long long key = rs_key(u, i);
            if ((key & high) == prefix) d = (int)(key >> shift) & 255;
        }
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        if (d >= 0 && lane == __ffs(peers) - 1) atomicAdd(h + d, (unsigned)__popc(peers));
    }
    __syncthreads();
    if (h[t]) atomicAdd(digits + pass * 256 + t, h[t]);
}

__global__ void __launch_bounds__(RS_THREADS) rs_collect(const float *__restrict__ u, long long N, int *meta,
                                                         const unsigned *__restrict__ digits,
                                                         unsigned long long *__restrict__ keys) {
    const long long R = rs_count(meta, N);
    if (R == 0) return;
    const unsigned long long T = rs_prefix(digits, RS_PASSES, R);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned *counter = reinterpret_cast<unsigned *>(meta + 1);
    for (long long i0 = (long long)blockIdx.x * RS_THREADS + warp * 32; i0 < N; i0 += (long long)gridDim.x * RS_THREADS) {
        const long long i = i0 + lane;
        const unsigned long long key = i < N ? rs_key(u, i) : ~0ULL;
        const bool take = i < N && key <= T;
        const unsigned b = __ballot_sync(0xffffffffu, take);
        unsigned slot = 0u;
        if (lane == 0 && b) slot = atomicAdd(counter, (unsigned)__popc(b));
        slot = __shfl_sync(0xffffffffu, slot, 0);
        if (take) keys[slot + __popc(b & ((1u << lane) - 1u))] = key;
    }
}

// rank[q] += the number of listed keys in chunk blockIdx.y below key q (keys are unique: the ranks are 0..R-1)
__global__ void __launch_bounds__(RS_THREADS) rs_rank(const int *__restrict__ meta, long long N,
                                                      const unsigned long long *__restrict__ keys, int *rank) {
    __shared__ unsigned long long s_key[RS_RANK_CHUNK];
    const long long R = rs_count(meta, N);
    const long long c0 = (long long)blockIdx.y * RS_RANK_CHUNK, q0 = (long long)blockIdx.x * RS_THREADS;
    if (c0 >= R || q0 >= R) return;
    const int cn = R - c0 < RS_RANK_CHUNK ? (int)(R - c0) : RS_RANK_CHUNK;
    for (int i = threadIdx.x; i < cn; i += RS_THREADS) s_key[i] = keys[c0 + i];
    __syncthreads();
    const long long q = q0 + threadIdx.x;
    if (q >= R) return;
    const unsigned long long key = keys[q];
    int below = 0;
#pragma unroll 8
    for (int i = 0; i < cn; ++i) below += s_key[i] < key;
    if (below) atomicAdd(rank + q, below);
}

__global__ void __launch_bounds__(RS_THREADS) rs_assign(const float *__restrict__ z, long long N, int D, float thr,
                                                        const int *__restrict__ meta, const int *__restrict__ dead,
                                                        const unsigned long long *__restrict__ keys,
                                                        const int *__restrict__ rank, float *__restrict__ cluster_size,
                                                        float *__restrict__ embed_sum, float *__restrict__ codebook) {
    const long long R = rs_count(meta, N);
    if (R == 0) return;
    const int d4 = D / 4;
    const float4 *z4 = reinterpret_cast<const float4 *>(z);
    for (long long g = (long long)blockIdx.x * RS_THREADS + threadIdx.x; g < R * d4; g += (long long)gridDim.x * RS_THREADS) {
        const long long q = g / d4;
        const int c = (int)(g - q * d4);
        const long long k = dead[rank[q]];
        const long long r = (long long)(keys[q] & 0xFFFFFFFFULL);
        const float4 v = __ldg(z4 + r * d4 + c);
        reinterpret_cast<float4 *>(codebook)[k * d4 + c] = v;
        reinterpret_cast<float4 *>(embed_sum)[k * d4 + c] =
            make_float4(__fmul_rn(thr, v.x), __fmul_rn(thr, v.y), __fmul_rn(thr, v.z), __fmul_rn(thr, v.w));
        if (c == 0) cluster_size[k] = thr;
    }
}

}  // namespace

extern "C" size_t vqb_vq_ema_workspace_bytes(int64_t N, int K, int D) {
    if (N <= 0 || K <= 0 || D <= 0 || D % 4 != 0) return 0;
    return ema_plan(N, K, D).total;
}

extern "C" int vqb_vq_ema_update_f32(const float *z, const int64_t *idx, const int32_t *hist, int64_t N, int K, int D,
                                     float decay, float eps, float *cluster_size, float *embed_sum, float *codebook,
                                     void *workspace, size_t workspace_bytes, void *stream) {
    if (!z || !idx || !hist || !cluster_size || !embed_sum || !codebook || !workspace) return VQB_ERR_BAD_ARG;
    if (N <= 0 || K <= 0 || D <= 0) return VQB_ERR_BAD_ARG;
    if (!(decay >= 0.f && decay < 1.f) || !(eps > 0.f && eps <= 3.4e38f)) return VQB_ERR_BAD_ARG;
    if (D % 4 != 0) return VQB_ERR_UNSUPPORTED;
    const EmaPlan p = ema_plan(N, K, D);
    if (workspace_bytes < p.total) return VQB_ERR_WORKSPACE;
    const uintptr_t al = reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(embed_sum) |
                         reinterpret_cast<uintptr_t>(codebook) | reinterpret_cast<uintptr_t>(workspace);
    if (al & 15) return VQB_ERR_ALIGNMENT;
    char *ws = static_cast<char *>(workspace);
    unsigned *cnt = reinterpret_cast<unsigned *>(ws + p.off_cnt);
    long long *base = reinterpret_cast<long long *>(ws + p.off_base);
    unsigned long long *status = reinterpret_cast<unsigned long long *>(ws + p.off_status);
    long long *rows = reinterpret_cast<long long *>(ws + p.off_rows);
    float *part = reinterpret_cast<float *>(ws + p.off_part);
    float *nnew = reinterpret_cast<float *>(ws + p.off_nnew);
    const long long *ip = reinterpret_cast<const long long *>(idx);
    cudaStream_t s = (cudaStream_t)stream;
    const int G = EMA_THREADS / group_lanes(D);
    long long fin = ((long long)K + G - 1) / G;
    if (fin > 2LL * sm_count()) fin = 2LL * sm_count();
    ema_count<<<(unsigned)p.nchunks, 32, 0, s>>>(ip, hist, cluster_size, N, K, p.rows_per_chunk, p.nchunks, decay, cnt,
                                                 nnew, status, p.ntiles);
    ema_scan<<<(unsigned)p.ntiles, EMA_SCAN_THREADS, 0, s>>>(cnt, p.M, base, status, p.ntiles);
    ema_scatter<<<(unsigned)p.nchunks, 32, 0, s>>>(ip, N, K, p.rows_per_chunk, p.nchunks, base, rows);
    ema_partial<<<(unsigned)((p.nslots + G - 1) / G), EMA_THREADS, 0, s>>>(z, K, D, p.nchunks, base, rows, p.nslots, part);
    ema_finish<<<(unsigned)fin, EMA_THREADS, 0, s>>>(K, D, p.nchunks, base, part, nnew, decay, eps, cluster_size,
                                                     embed_sum, codebook);
    VQB_COUNT_LAUNCH(5);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" size_t vqb_vq_ema_restart_workspace_bytes(int64_t N, int K) {
    if (N <= 0 || K <= 0 || K > RS_MAX_K || N > RS_MAX_N) return 0;
    return restart_plan(K).total;
}

extern "C" int vqb_vq_ema_restart_f32(const float *z, const float *u, int64_t N, int K, int D, float threshold,
                                      float *cluster_size, float *embed_sum, float *codebook, int32_t *n_restarted,
                                      void *workspace, size_t workspace_bytes, void *stream) {
    if (!z || !u || !cluster_size || !embed_sum || !codebook || !n_restarted || !workspace) return VQB_ERR_BAD_ARG;
    if (N <= 0 || K <= 0 || D <= 0) return VQB_ERR_BAD_ARG;
    if (!(threshold > 0.f && threshold <= 3.4028235e38f)) return VQB_ERR_BAD_ARG;
    if (D % 4 != 0 || K > RS_MAX_K || N > RS_MAX_N) return VQB_ERR_UNSUPPORTED;
    const RestartPlan p = restart_plan(K);
    if (workspace_bytes < p.total) return VQB_ERR_WORKSPACE;
    const uintptr_t al = reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(embed_sum) |
                         reinterpret_cast<uintptr_t>(codebook) | reinterpret_cast<uintptr_t>(workspace);
    if (al & 15) return VQB_ERR_ALIGNMENT;
    const long long rmax = (long long)K < N ? (long long)K : N;
    char *ws = static_cast<char *>(workspace);
    int *meta = reinterpret_cast<int *>(ws + p.off_meta);
    int *dead = reinterpret_cast<int *>(ws + p.off_dead);
    unsigned *digits = reinterpret_cast<unsigned *>(ws + p.off_digits);
    unsigned long long *keys = reinterpret_cast<unsigned long long *>(ws + p.off_keys);
    int *rank = reinterpret_cast<int *>(ws + p.off_rank);
    cudaStream_t s = (cudaStream_t)stream;
    const int sms = sm_count();
    long long scan = (N + RS_THREADS - 1) / RS_THREADS;
    if (scan > 4LL * sms) scan = 4LL * sms;
    long long asg = (rmax * (D / 4) + RS_THREADS - 1) / RS_THREADS;
    if (asg > 4LL * sms) asg = 4LL * sms;
    rs_compact<<<1, RS_COMPACT_THREADS, 0, s>>>(cluster_size, K, N, threshold, meta, dead, digits, rank,
                                                 n_restarted);
    for (int pass = 0; pass < RS_PASSES; ++pass)
        rs_digits<<<(unsigned)scan, RS_THREADS, 0, s>>>(u, N, meta, digits, pass);
    rs_collect<<<(unsigned)scan, RS_THREADS, 0, s>>>(u, N, meta, digits, keys);
    const dim3 rank_grid((unsigned)((rmax + RS_THREADS - 1) / RS_THREADS),
                         (unsigned)((rmax + RS_RANK_CHUNK - 1) / RS_RANK_CHUNK));
    rs_rank<<<rank_grid, RS_THREADS, 0, s>>>(meta, N, keys, rank);
    rs_assign<<<(unsigned)asg, RS_THREADS, 0, s>>>(z, N, D, threshold, meta, dead, keys, rank, cluster_size,
                                                   embed_sum, codebook);
    VQB_COUNT_LAUNCH(4 + RS_PASSES);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" int vqb_vq_commit_backward_f32(const float *g_zq, const float *g_loss, const float *z, const float *zq,
                                          int64_t N, int D, float beta, float *dz, void *stream) {
    if (!z || !zq || !dz) return VQB_ERR_BAD_ARG;
    if (N <= 0 || D <= 0) return VQB_ERR_BAD_ARG;
    if (D % 4 != 0) return VQB_ERR_UNSUPPORTED;
    const uintptr_t al = reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(zq) |
                         reinterpret_cast<uintptr_t>(dz) | reinterpret_cast<uintptr_t>(g_zq);
    if (al & 15) return VQB_ERR_ALIGNMENT;
    const long long total4 = N * (D / 4);
    long long blocks = (total4 + 255) / 256;
    if (blocks > 16LL * sm_count()) blocks = 16LL * sm_count();
    vq_commit_backward_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(g_zq, g_loss, z, zq, total4, N, D, beta,
                                                                                   dz);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

// wgconv.cu -- implicit-GEMM convolution on Hopper tensor cores (wgmma, sm_90a): the tensor-core conv of the TF32
// mode (fp32 NHWC activations read as TF32) and of the bf16 pipeline (bf16 NHWC activations).
//
// GEMM view (one CTA = one 128-pixel output tile = BN images x BH rows x BW cols, all N columns):
//   D[128 px][N] = sum over k-steps i of A_i[128 px][128 B of channels] * B_i[N][128 B]^T
//   * A_i is ONE 4-D TMA box {128 B of channels, BW, BH, BN} of the NHWC input shifted by the step's tap
//     (dy, dx): it lands as 128 rows of 128 bytes in the 128-byte-swizzled K-major layout wgmma reads;
//     out-of-image pixels are zero-filled by TMA (= the zero padding), stride-2 convolutions use the tensor
//     map's element strides.  No im2col matrix exists.
//   * B_i is a 2-D TMA box of N K-major weight rows.
//   * warp 0 = TMA producer over an mbarrier ring of up to 8 stages; warpgroups 1 and 2 = consumers, each owns
//     64 pixel rows of the tile: 4 wgmma per stage (m64nNk8 tf32 / m64nNk16 bf16) into N/2 fp32 registers per
//     thread, then the epilogue straight from the registers: + bias, + skip, ReLU, fp32 or bf16 stores.
//   * the sub-pixel phases of a stride-2 transposed conv run in one launch (blockIdx.y = phase).
//   * N2 > 0 (residual layer of the bf16 pipeline): the first GEMM's result is ReLU'd, rounded to bf16 and written
//     to shared memory as the A operand of a second GEMM against an N2 x 64 weight tile loaded once, so
//     out = act(skip + W2 . relu(W1 (*) r)) and the intermediate never leaves the SM.
//   * TAIL (TF32, N = 64, the decoder's k4 s2 transposed conv on whole-image tiles): the CTA runs all four phases
//     itself, keeps h = relu(convT + b) of its images in shared memory and chains the output layer on it (below).
// The TF32 residual stack on whole-image tiles has its own kernel, res_scatter_kernel, which can also run the k3 conv
// before the stack and the 1x1 conv after it in the same launch (the latent block of the inference forward).
// The decoder's output layer (k4 s2 transposed conv to <= 4 channels) has its own persistent kernel at the end of this
// file, convt_scatter_kernel: one GEMM per tile over the input pixels and their halo, read once per channel chunk.
#include "ptx.cuh"
#include "bf16_common.cuh"
#include "wgconv.h"
#include "wgmma.cuh"

namespace {

constexpr int WG_THREADS = 384;
constexpr int WG_MAX_STAGES = 8;
constexpr int A_BYTES = 128 * 128;             // 128 pixels x 128 bytes

struct WgParams {
    const float *bias;
    const void *skip;
    void *out;
    int B, ncols, mid_cols;
    int BW, BH, BN, tiles_x, tiles_y;
    int in_step, out_step, stages;
    int relu, out_bf16;
    int OHg[4], OWg[4], out_py[4], out_px[4], nsteps[4];
    long long out_sn, out_sh, out_sw, out_sc;
    int4 steps[4][WG_MAX_STEPS];              // x = c0, y = dx, z = dy, w = w_row
    // TAIL: the output layer (w_shuffle rows as convt_scatter_kernel reads them, bias may be null) -> x_hat NCHW fp32;
    // `out` is h (NHWC) or null
    const void *tail_w;
    const float *tail_bias;
    float *tail_out;
    int tail_cout, tail_relu;
};

// The output layer's weight in scatter form (see convt_scatter_kernel): 64 GEMM columns (phase, neighbour (ky, kx),
// co), gathered once per CTA.
constexpr int SC_N = 64;                   // GEMM columns: 4 phases x 4 neighbours (ky, kx) x 4 channels
constexpr int SC_BBYTES = SC_N * 128;      // one 128-byte channel chunk of the gathered weight

// Gather the output layer's 64 live weight rows from w_shuffle ([9 taps (dy, dx)][16][Cin], row (py * 2 + px) * Cout
// + co of tap (dy + 1) * 3 + dx + 1) into nc chunks [64][128 B] at wres, by 256 threads (t = 0..255): row r = phase *
// 16 + k * 4 + co in the 128-byte swizzle wgmma reads (16-byte piece j of row r at j ^ (r & 7)), channels co >= Cout
// zero.  Ends with the proxy fence; the caller's barrier makes the rows complete.
template <bool BF16>
__device__ __forceinline__ void gather_shuffle_weight(uint32_t wres, const void *w, int Cin, int Cout, int nc, int t) {
    const size_t row_bytes = (size_t)Cin * (BF16 ? 2 : 4);
    for (int i = t; i < nc * SC_N * 8; i += 256) {
        const int j = i & 7, r = (i >> 3) % SC_N, c = i / (8 * SC_N);
        const int ph = r >> 4, k = (r >> 2) & 3, co = r & 3;
        const int tap = ((k >> 1) + (ph >> 1)) * 3 + (k & 1) + (ph & 1);
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (co < Cout)
            v = __ldg(reinterpret_cast<const uint4 *>(reinterpret_cast<const unsigned char *>(w) +
                      (size_t)(tap * 16 + ph * Cout + co) * row_bytes + c * 128 + j * 16));
        const uint32_t dst = wres + (uint32_t)(c * SC_BBYTES + r * 128 + ((j ^ (r & 7)) << 4));
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
    }
    ptx::fence_proxy_async();                      // generic-proxy writes -> visible to wgmma
}

// Epilogue of one accumulator fragment (wgmma D layout, see wgmma.cuh) for the pixel rows of this thread.
template <int N>
__device__ __forceinline__ void store_tile(const WgParams &p, const float *acc, int ph, int wgi, int gx0, int gy0, int n0,
                                           const void *skip, int relu) {
    const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = wgi * 64 + warp * 16 + (lane >> 2) + 8 * h;
        const int bw = row % p.BW, bh = (row / p.BW) % p.BH, bn = row / (p.BW * p.BH);
        const int gx = gx0 + bw, gy = gy0 + bh, n = n0 + bn;
        if (gx >= p.OWg[ph] || gy >= p.OHg[ph] || n >= p.B) continue;
        const long long ob = (long long)n * p.out_sn + (long long)(gy * p.out_step + p.out_py[ph]) * p.out_sh +
                             (long long)(gx * p.out_step + p.out_px[ph]) * p.out_sw;
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
            const int c = 8 * j + cq;
            if (c >= p.ncols) continue;                 // ncols is even: a pair is wholly in or out
            float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            if (p.bias) { v0 += __ldg(p.bias + c); v1 += __ldg(p.bias + c + 1); }
            if (p.out_bf16) {
                if (skip) {
                    const __nv_bfloat162 sk = *reinterpret_cast<const __nv_bfloat162 *>(
                        reinterpret_cast<const __nv_bfloat16 *>(skip) + ob + c);
                    v0 += __bfloat162float(sk.x); v1 += __bfloat162float(sk.y);
                }
                if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                *reinterpret_cast<uint32_t *>(reinterpret_cast<__nv_bfloat16 *>(p.out) + ob + c) = pack_bf16(v0, v1);
            } else {
                if (skip) {
                    const float2 sk = *reinterpret_cast<const float2 *>(reinterpret_cast<const float *>(skip) + ob + c);
                    v0 += sk.x; v1 += sk.y;
                }
                if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                *reinterpret_cast<float2 *>(reinterpret_cast<float *>(p.out) + ob + c) = make_float2(v0, v1);
            }
        }
    }
}

// chunks of the chained second GEMM's K (the first GEMM's N columns): one 64-channel bf16 chunk, or 32-channel fp32 ones
template <bool BF16, int N>
__host__ __device__ constexpr int chain_chunks() { return BF16 ? 1 : (N >= 32 ? N / 32 : 1); }

// TAIL: h of the tile's images stays in shared memory as the A operand of the output layer's GEMM.  Each of the 4 phases
// runs the k-steps of the per-phase launch (the same table, ring and chain), then its epilogue (+ bias, ReLU, in
// store_tile's order) writes the values to h (and to `out` when given).  h: KC2 = 2 chunks [4 x 128 rows][128 B] of 32
// channels, 128-byte swizzle, rows in tile raster order (image, 2 BH, 2 BW), so every 64-row block is 1024-byte aligned
// and warpgroup wgi's phase rows all land in h rows 256 wgi .. + 255.  Then, per 64-row block, the output layer's
//   Y[q][phase, k, co] = h[q] . w_out[tap of (phase, k)][phase, co]      (m64n64, chunk outer, from zero)
// as in convt_scatter_kernel, and Y overwrites the block's h rows in place (the block's GEMM has read them): columns
// 0..31 in the chunk 0 row, 32..63 in the chunk 1 row, word w of the 32 at (w + 2 q) mod 32 against bank conflicts.
// Finally x_hat(2 gy + py, 2 gx + px, co) = sum over k in raster (ky, kx) order of Y[(gy + ky + py - 1, gx + kx + px
// - 1)][phase, k, co] (+0 for a neighbour outside the image, the term of convt_scatter_kernel's zero-filled halo row),
// + bias, optional ReLU.  So h and x_hat are bitwise the two separate launches'.
// Shared memory (1024-byte aligned): ring S x (A box + 64 weight rows) | h 128 KB | gathered output weight 16 KB | bars.
constexpr int TAIL_PHASE_ROWS = 4 * 128;   // h rows per tile: 4 phases x 128 pixels

template <bool BF16, int N, int N2, bool TAIL = false>
__global__ void __launch_bounds__(WG_THREADS, 1)
wgconv_kernel(const __grid_constant__ CUtensorMap tma_in, const __grid_constant__ CUtensorMap tma_w,
              const __grid_constant__ CUtensorMap tma_w2, const __grid_constant__ WgParams p) {
    static_assert(!TAIL || (!BF16 && N == SC_N && N2 == 0), "TAIL: TF32, 64 channels of h, no second GEMM");
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    const uint32_t sbase = (raw + 1023u) & ~1023u;
    constexpr int STAGE = A_BYTES + N * 128;
    constexpr int KC2 = chain_chunks<BF16, N>();
    constexpr int HCHUNK = TAIL_PHASE_ROWS * 128;      // TAIL: one 32-channel chunk of h
    const int S = p.stages;
    // N2 > 0: KC2 intermediate tiles [128 px][128 B], then the KC2 W2 tiles [N2][128 B]
    // TAIL: KC2 chunks of h, then the KC2 chunks of the gathered output weight [64][128 B]
    const uint32_t mid = sbase + (uint32_t)(S * STAGE);
    const uint32_t w2s = mid + (uint32_t)(KC2 * (TAIL ? HCHUNK : A_BYTES));
    const uint32_t bars = mid + (N2 > 0 ? (uint32_t)(KC2 * (A_BYTES + N2 * 128))
                                 : TAIL ? (uint32_t)(KC2 * (HCHUNK + SC_BBYTES)) : 0u);
    auto full = [&](int s) { return bars + 8u * s; };
    auto empty = [&](int s) { return bars + 8u * (WG_MAX_STAGES + s); };
    const uint32_t w2bar = bars + 8u * (2 * WG_MAX_STAGES);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ph0 = TAIL ? 0 : blockIdx.y, nph = TAIL ? 4 : 1;      // the phases this CTA runs
    int tile = blockIdx.x;
    const int tx = tile % p.tiles_x; tile /= p.tiles_x;
    const int ty = tile % p.tiles_y; tile /= p.tiles_y;
    const int gx0 = tx * p.BW, gy0 = ty * p.BH, n0 = tile * p.BN;

    if (tid == 0) {
        for (int s = 0; s < S; ++s) { ptx::mbar_init(full(s), 1); ptx::mbar_init(empty(s), 2); }
        ptx::mbar_init(w2bar, 1);
        ptx::fence_mbar_init();
    }
    if (tid == 32) {
        ptx::prefetch_tmap(&tma_in);
        ptx::prefetch_tmap(&tma_w);
        if (N2 > 0) ptx::prefetch_tmap(&tma_w2);
    }
    __syncthreads();
    pdl_launch_dependents();           // the next layer may start its prologue

    if (warp == 0) {
        if constexpr (N2 > 0) {        // weights do not depend on the previous layer
            if (lane == 0) {
                constexpr int ck = BF16 ? 64 : 32;
                ptx::mbar_expect_tx(w2bar, (uint32_t)(KC2 * N2 * 128));
                for (int c = 0; c < KC2; ++c) ptx::tma_load_2d(w2s + (uint32_t)(c * N2 * 128), &tma_w2, w2bar, c * ck, 0);
            }
        }
        pdl_wait();                    // ... the activations do
        if (lane == 0) {
            int g = 0;                 // ring slot counter over the CTA's phases
            for (int ph = ph0; ph < ph0 + nph; ++ph)
                for (int i = 0; i < p.nsteps[ph]; ++i, ++g) {
                    const int s = g % S;
                    if (g >= S) ptx::mbar_wait(empty(s), (uint32_t)((g / S - 1) & 1));
                    const int4 st = p.steps[ph][i];
                    const uint32_t dst = sbase + (uint32_t)(s * STAGE);
                    ptx::mbar_expect_tx(full(s), (uint32_t)STAGE);
                    ptx::tma_load_4d(dst, &tma_in, full(s), st.x, gx0 * p.in_step + st.y, gy0 * p.in_step + st.z, n0);
                    ptx::tma_load_2d(dst + A_BYTES, &tma_w, full(s), st.x, st.w);
                }
        }
        return;
    }
    if (warp < 4) return;

    // TAIL: the output weight does not depend on the previous layer
    if constexpr (TAIL) gather_shuffle_weight<false>(w2s, p.tail_w, N, p.tail_cout, KC2, tid - 128);
    pdl_wait();                        // skip / out may belong to the previous layer
    const int wgi = (warp >> 2) - 1;   // pixel rows 64 * wgi .. + 63 of the tile
    float acc[N / 2];
    int g = 0;
    for (int ph = ph0; ph < ph0 + nph; ++ph) {
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
        for (int i = 0; i < p.nsteps[ph]; ++i, ++g) {
            const int s = g % S;
            ptx::mbar_wait(full(s), (uint32_t)((g / S) & 1));
            const uint32_t a = sbase + (uint32_t)(s * STAGE) + (uint32_t)(wgi * 64 * 128), b = sbase + (uint32_t)(s * STAGE) + A_BYTES;
            wg::fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) wg::mma<BF16, N>(acc, wg::desc_sw128(a + 32u * kk), wg::desc_sw128(b + 32u * kk), 1u);
            wg::commit();
            wg::wait<0>();
            wg::fence_regs<N>(acc);
            if ((warp & 3) == 0 && lane == 0) ptx::mbar_arrive(empty(s));
        }
        if constexpr (TAIL) {
            // + bias, ReLU (store_tile's order) -> h in shared memory, and to `out` when given
            const int wl = warp & 3, cq = 2 * (lane & 3);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = wgi * 64 + wl * 16 + (lane >> 2) + 8 * h;
                const int bw = row % p.BW, bh = (row / p.BW) % p.BH, bn = row / (p.BW * p.BH);
                const int hr = (bn * 2 * p.BH + 2 * bh + p.out_py[ph]) * 2 * p.BW + 2 * bw + p.out_px[ph];
                const bool live = gx0 + bw < p.OWg[ph] && gy0 + bh < p.OHg[ph] && n0 + bn < p.B;
                float *o = reinterpret_cast<float *>(p.out) + (long long)(n0 + bn) * p.out_sn +
                           (long long)((gy0 + bh) * p.out_step + p.out_py[ph]) * p.out_sh +
                           (long long)((gx0 + bw) * p.out_step + p.out_px[ph]) * p.out_sw;
#pragma unroll
                for (int j = 0; j < N / 8; ++j) {
                    const int c = 8 * j + cq;
                    float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                    if (p.bias) { v0 += __ldg(p.bias + c); v1 += __ldg(p.bias + c + 1); }
                    if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                    const uint32_t addr = mid + (uint32_t)((c >> 5) * HCHUNK + hr * 128 + ((((c & 31) >> 2) ^ (hr & 7)) << 4) + (c & 3) * 4);
                    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v0), "f"(v1) : "memory");
                    if (p.out && live) *reinterpret_cast<float2 *>(o + c) = make_float2(v0, v1);
                }
            }
        }
    }

    if constexpr (TAIL) {
        ptx::fence_proxy_async();                        // h (generic-proxy writes) -> visible to wgmma
        ptx::named_bar_sync(1, 256);                     // h and the gathered output weight are complete
        const int wl = warp & 3, cq = 2 * (lane & 3);
        for (int blk = 4 * wgi; blk < 4 * wgi + 4; ++blk) {
            float y[SC_N / 2];
#pragma unroll
            for (int i = 0; i < SC_N / 2; ++i) y[i] = 0.f;
            wg::fence();
#pragma unroll
            for (int c = 0; c < KC2; ++c) {
                const uint32_t a = mid + (uint32_t)(c * HCHUNK + blk * 64 * 128), b = w2s + (uint32_t)(c * SC_BBYTES);
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) wg::mma<false, SC_N>(y, wg::desc_sw128(a + 32u * kk), wg::desc_sw128(b + 32u * kk), 1u);
            }
            wg::commit();
            wg::wait<0>();
            wg::fence_regs<SC_N>(y);
            ptx::named_bar_sync(2 + wgi, 128);           // the whole warpgroup's GEMM has read the block's h rows
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int q = blk * 64 + wl * 16 + (lane >> 2) + 8 * h;
#pragma unroll
                for (int j = 0; j < SC_N / 8; ++j) {
                    const int c = 8 * j + cq;
                    const uint32_t addr = mid + (uint32_t)((c >> 5) * HCHUNK + q * 128 + (((c & 31) + 2 * q) & 31) * 4);
                    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(y[4 * j + 2 * h]), "f"(y[4 * j + 2 * h + 1]) : "memory");
                }
            }
        }
        ptx::named_bar_sync(1, 256);                     // Y of the whole tile is staged
        // one output pixel per thread and step, (image, co, oy, ox) with ox fastest: coalesced NCHW rows
        const int H = p.OHg[0], W = p.OWg[0];            // the latent: every phase of the k4 s2 p1 layer is H x W
        const int lw = __ffs(4 * p.BW) - 1, lh = __ffs(4 * p.BH) - 1, Cout = p.tail_cout;
        const float *const ys = reinterpret_cast<const float *>(smem_raw + (mid - raw));
        auto yat = [&](int q, int col) {                 // Y[q][col]
            return ys[(col >> 5) * (HCHUNK / 4) + q * 32 + (((col & 31) + 2 * q) & 31)];
        };
        const int total = (p.BN * Cout) << (lw + lh);
        for (int e = tid - 128; e < total; e += 256) {
            const int ox = e & (4 * p.BW - 1), oy = (e >> lw) & (4 * p.BH - 1), co = (e >> (lw + lh)) % Cout;
            const int bn = (e >> (lw + lh)) / Cout;
            if (ox >= 4 * W || oy >= 4 * H || n0 + bn >= p.B) continue;
            const int gy = oy >> 1, py = oy & 1, gx = ox >> 1, px = ox & 1;
            const int base = bn * 4 * p.BH * p.BW, col = (py * 2 + px) * 16 + co;
            float t[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int hy = gy + (k >> 1) + py - 1, hx = gx + (k & 1) + px - 1;
                t[k] = hy >= 0 && hy < 2 * H && hx >= 0 && hx < 2 * W ? yat(base + hy * 2 * p.BW + hx, col + 4 * k) : 0.f;
            }
            float v = t[0];
            v += t[1];
            v += t[2];
            v += t[3];
            v += p.tail_bias ? __ldg(p.tail_bias + co) : 0.f;
            if (p.tail_relu) v = fmaxf(v, 0.f);
            p.tail_out[(long long)(n0 + bn) * Cout * 16 * H * W + (long long)co * 16 * H * W + oy * 4 * W + ox] = v;
        }
    } else if constexpr (N2 == 0) {
        store_tile<N>(p, acc, ph0, wgi, gx0, gy0, n0, p.skip, p.relu);
    } else {
        // relu(first GEMM) -> rows of 128 bytes (64 bf16 / 32 fp32 channels per chunk), 128-byte swizzle: 16-byte
        // piece j of row r sits at j ^ (r & 7)
        const int wl = warp & 3, cq = 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = wgi * 64 + wl * 16 + (lane >> 2) + 8 * h;
            const uint32_t rb = mid + (uint32_t)(row * 128);
            if constexpr (BF16) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = 8 * j + cq;
                    float v0 = 0.f, v1 = 0.f;
                    if (j < N / 8 && c < p.mid_cols) { v0 = fmaxf(acc[4 * j + 2 * h], 0.f); v1 = fmaxf(acc[4 * j + 2 * h + 1], 0.f); }
                    const uint32_t addr = rb + (uint32_t)(((j ^ (row & 7)) << 4) + cq * 2);
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(pack_bf16(v0, v1)) : "memory");
                }
            } else {
#pragma unroll
                for (int j = 0; j < N / 8; ++j) {
                    const int c = 8 * j + cq, piece = (c & 31) >> 2;
                    const float v0 = fmaxf(acc[4 * j + 2 * h], 0.f), v1 = fmaxf(acc[4 * j + 2 * h + 1], 0.f);
                    const uint32_t addr = rb + (uint32_t)((c >> 5) * A_BYTES) + (uint32_t)(((piece ^ (row & 7)) << 4) + (c & 3) * 4);
                    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v0), "f"(v1) : "memory");
                }
            }
        }
        ptx::fence_proxy_async();                        // generic-proxy writes -> visible to wgmma
        ptx::named_bar_sync(1 + wgi, 128);               // this warpgroup's 64 rows are complete
        ptx::mbar_wait(w2bar, 0);
        float acc2[N2 > 0 ? N2 / 2 : 1];
#pragma unroll
        for (int i = 0; i < N2 / 2; ++i) acc2[i] = 0.f;
        wg::fence();
#pragma unroll
        for (int c = 0; c < KC2; ++c) {
            const uint32_t a = mid + (uint32_t)(c * A_BYTES + wgi * 64 * 128), b = w2s + (uint32_t)(c * N2 * 128);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                wg::mma<BF16, N2>(acc2, wg::desc_sw128(a + 32u * kk), wg::desc_sw128(b + 32u * kk), 1u);
        }
        wg::commit();
        wg::wait<0>();
        wg::fence_regs<N2>(acc2);
        store_tile<N2>(p, acc2, ph0, wgi, gx0, gy0, n0, p.skip, p.relu);
    }
}

int pow2_ceil(int x) {
    int p = 1;
    while (p < x) p <<= 1;
    return p;
}

typedef void (*wg_fn)(CUtensorMap, CUtensorMap, CUtensorMap, WgParams);

template <bool BF16, int N2>
wg_fn pick_n(int N) {
    switch (N) {
        case 16: return wgconv_kernel<BF16, 16, N2>;
        case 32: return wgconv_kernel<BF16, 32, N2>;
        case 64: return wgconv_kernel<BF16, 64, N2>;
        case 128: return wgconv_kernel<BF16, 128, N2>;
        case 256: return N2 == 0 ? wgconv_kernel<BF16, 256, 0> : nullptr;
        default: return nullptr;
    }
}

wg_fn pick(int bf16, int N, int N2) {
    if (!bf16) {
        switch (N2) {
            case 0: return pick_n<false, 0>(N);
            case 64: return (N == 32 || N == 64) ? pick_n<false, 64>(N) : nullptr;
            case 128: return (N == 32 || N == 64) ? pick_n<false, 128>(N) : nullptr;
            default: return nullptr;
        }
    }
    switch (N2) {
        case 0: return pick_n<true, 0>(N);
        case 64: return N <= 64 ? pick_n<true, 64>(N) : nullptr;
        case 128: return N <= 64 ? pick_n<true, 128>(N) : nullptr;
        default: return nullptr;
    }
}

}  // namespace

int wg_gemm_cols(int ncols) {
    for (int n : {16, 32, 64, 128, 256})
        if (ncols <= n) return n;
    return 0;
}

int launch_wgconv(const WgLaunch &L, cudaStream_t s) {
    if (L.nph < 1 || L.nph > 4 || wg_gemm_cols(L.N) != L.N || L.ncols > L.N) return VQB_ERR_UNSUPPORTED;
    const bool tail = L.tail_out != nullptr;
    if (tail && (L.bf16 || L.N != SC_N || L.ncols != SC_N || L.N2 != 0 || L.nph != 4 || L.out_step != 2 ||
                 L.tail_cout < 1 || L.tail_cout > 4))
        return VQB_ERR_UNSUPPORTED;
    const wg_fn fn = tail ? wgconv_kernel<false, SC_N, 0, true> : pick(L.bf16, L.N, L.N2);
    if (!fn) return VQB_ERR_UNSUPPORTED;
    const int esz = L.bf16 ? 2 : 4, ck = 128 / esz;       // elements per 128-byte K chunk
    if (L.Cin % ck != 0 || L.w_inner % ck != 0) return VQB_ERR_UNSUPPORTED;
    if (L.out_sc != 1) return VQB_ERR_UNSUPPORTED;
    WgParams q;
    memset(&q, 0, sizeof(q));
    q.bias = L.bias; q.skip = L.skip; q.out = L.out;
    q.B = L.B; q.ncols = L.ncols; q.mid_cols = L.ncols;
    q.in_step = L.in_step; q.out_step = L.out_step;
    q.relu = L.relu; q.out_bf16 = L.out_bf16;
    q.out_sn = L.out_sn; q.out_sh = L.out_sh; q.out_sw = L.out_sw; q.out_sc = L.out_sc;
    q.tail_w = L.tail_w; q.tail_bias = L.tail_bias; q.tail_out = L.tail_out; q.tail_cout = L.tail_cout;
    q.tail_relu = L.tail_relu;
    int maxw = 0, maxh = 0, maxk = 1;
    for (int i = 0; i < L.nph; ++i) {
        if (L.nsteps[i] > WG_MAX_STEPS) return VQB_ERR_UNSUPPORTED;
        q.OHg[i] = L.OHg[i]; q.OWg[i] = L.OWg[i]; q.out_py[i] = L.out_py[i]; q.out_px[i] = L.out_px[i];
        q.nsteps[i] = L.nsteps[i];
        for (int t = 0; t < L.nsteps[i]; ++t) {
            const WgStep &st = L.steps[i][t];
            q.steps[i][t] = make_int4(st.c0, st.dx, st.dy, st.w_row);
        }
        if (L.OWg[i] > maxw) maxw = L.OWg[i];
        if (L.OHg[i] > maxh) maxh = L.OHg[i];
        if (L.nsteps[i] > maxk) maxk = L.nsteps[i];
    }
    if (maxw <= 0 || maxh <= 0) return 0;
    q.BW = pow2_ceil(maxw) < 16 ? pow2_ceil(maxw) : 16;
    q.BH = pow2_ceil(maxh) < 128 / q.BW ? pow2_ceil(maxh) : 128 / q.BW;
    q.BN = 128 / (q.BW * q.BH);
    q.tiles_x = (maxw + q.BW - 1) / q.BW;
    q.tiles_y = (maxh + q.BH - 1) / q.BH;
    const long long tiles_n = (L.B + q.BN - 1) / q.BN;
    if (tail) {      // whole images per tile, and every phase over the same H x W grid
        if (q.tiles_x != 1 || q.tiles_y != 1) return VQB_ERR_UNSUPPORTED;
        for (int i = 0; i < 4; ++i)
            if (L.OHg[i] != maxh || L.OWg[i] != maxw) return VQB_ERR_UNSUPPORTED;
    }

    const CUtensorMapDataType dt = L.bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    CUtensorMap tin, tw, tw2;
    const uint64_t dims[4] = {(uint64_t)L.Cin, (uint64_t)L.W, (uint64_t)L.H, (uint64_t)L.B};
    const uint64_t strides[3] = {(uint64_t)L.Cin * esz, (uint64_t)L.W * L.Cin * esz, (uint64_t)L.H * L.W * L.Cin * esz};
    const uint32_t box[4] = {(uint32_t)ck, (uint32_t)(q.BW * L.in_step), (uint32_t)(q.BH * L.in_step), (uint32_t)q.BN};
    const uint32_t es[4] = {1u, (uint32_t)L.in_step, (uint32_t)L.in_step, 1u};
    int rc = vqb_encode_tmap_4d(&tin, dt, L.in, dims, strides, box, es, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    rc = vqb_encode_tmap_2d(&tw, dt, L.w, (uint64_t)L.w_inner, (uint64_t)L.w_rows, (uint64_t)L.w_inner * esz, (uint32_t)ck,
                            (uint32_t)L.N, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    tw2 = tw;
    int kc2 = 0;
    if (L.N2 > 0) {
        if (L.ncols > 64 || L.w2_inner % ck != 0) return VQB_ERR_UNSUPPORTED;
        if (!L.bf16 && L.ncols != L.N) return VQB_ERR_UNSUPPORTED;          // fp32 intermediate: whole 32-channel chunks
        kc2 = L.bf16 ? 1 : L.N / 32;
        q.mid_cols = L.ncols; q.ncols = L.N2;
        rc = vqb_encode_tmap_2d(&tw2, dt, L.w2, (uint64_t)L.w2_inner, (uint64_t)L.w2_rows, (uint64_t)L.w2_inner * esz, (uint32_t)ck,
                                (uint32_t)L.N2, CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    const long long grid = (long long)q.tiles_x * q.tiles_y * tiles_n;
    if (grid <= 0 || grid > 0x7fffffffLL) return VQB_ERR_UNSUPPORTED;
    const int stage = A_BYTES + L.N * 128;
    const int fixed = (tail ? (SC_N / 32) * (TAIL_PHASE_ROWS * 128 + SC_BBYTES) : kc2 * (A_BYTES + L.N2 * 128)) +
                      8 * (2 * WG_MAX_STAGES + 1) + 1024;
    auto ring = [&](int budget) {
        const int st = (budget - fixed) / stage;
        return st > WG_MAX_STAGES ? WG_MAX_STAGES : st > maxk ? maxk : st;
    };
    int stages = ring(220 * 1024);
    if (stages < 1) return VQB_ERR_UNSUPPORTED;
    static bool attr_set[64] = {false};      // per instantiation (slot below): every ring size fits in 220 KB
    const int slot = tail ? 24 : (L.bf16 ? 32 : 0) + (L.N2 == 128 ? 16 : L.N2 == 64 ? 8 : 0) + (L.N == 16 ? 0 : L.N == 32 ? 1 : L.N == 64 ? 2 : L.N == 128 ? 3 : 4);
    if (!attr_set[slot]) {
        cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
        if (e != cudaSuccess) return (int)e;
        attr_set[slot] = true;
    }
    // More CTAs than SMs: a CTA spends its prologue, ring fill and epilogue with the tensor cores idle, and one per SM
    // leaves them so.  Size the ring for two CTAs per SM (228 KB of shared memory, 1 KB of it reserved per CTA) when
    // that keeps at least 3 stages and the registers allow it, so each CTA's k-steps cover the other's idle phases.
    // The k-step order, and so every result bit, does not depend on the ring size.
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int shared = ring(113 * 1024);
    if (!tail && grid * L.nph > sms && shared >= (maxk < 3 ? maxk : 3) && shared < stages) {
        int per_sm = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, WG_THREADS, (size_t)(shared * stage + fixed)) ==
                cudaSuccess && per_sm >= 2)
            stages = shared;
    }
    q.stages = stages;
    const int smem = stages * stage + fixed;
    if (cudaError_t le = vqb_launch(fn, dim3((unsigned)grid, tail ? 1u : (unsigned)L.nph), dim3(WG_THREADS), (size_t)smem, s,
                                    tin, tw, tw2, q))
        return (int)le;
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ layer launchers
// The k-steps of one phase: each tap of the phase x each 128-byte channel chunk (32 fp32 / 64 bf16 channels), tap t
// reading the N weight rows from tap_w[t] * rows_per_tap.  Every k-step adds into the fp32 accumulators, so the
// order fixes the result bits: tap outer / chunk inner, or chunk outer / tap inner (chunk_outer).
static bool set_phase(WgLaunch &L, int i, const ConvPhase &ph, int rows_per_tap, bool chunk_outer) {
    const int ck = L.bf16 ? 64 : 32, nc = L.Cin / ck;
    if (ph.ntaps * nc > WG_MAX_STEPS) return false;
    L.in_step = ph.in_step; L.out_step = ph.out_step;
    L.OHg[i] = ph.OHg; L.OWg[i] = ph.OWg; L.out_py[i] = ph.out_py; L.out_px[i] = ph.out_px;
    int n = 0;
    for (int a = 0; a < (chunk_outer ? nc : ph.ntaps); ++a)
        for (int b = 0; b < (chunk_outer ? ph.ntaps : nc); ++b) {
            const int t = chunk_outer ? b : a, c0 = (chunk_outer ? a : b) * ck;
            L.steps[i][n++] = WgStep{c0, ph.tap_dx[t], ph.tap_dy[t], ph.tap_w[t] * rows_per_tap};
        }
    L.nsteps[i] = n;
    return true;
}

// the 3x3 neighbourhood of an output pixel of a stride-1 layer: taps t = r * 3 + s, dy = r - 1, dx = s - 1
static ConvPhase taps3x3(int H, int W) {
    ConvPhase ph;
    conv_phase(conv_geom(3, 3, 1, 1, 0, H, W), 0, ph);
    return ph;
}

bool conv_tc_supported(const ConvLaunch &p) {
    const bool in_nhwc = p.in_sc == 1 && p.in_sw == p.Cin;
    const bool out_nhwc = p.out_sc == 1 && p.out_sw == p.Cout;
    return in_nhwc && out_nhwc && p.Cin % 32 == 0 && p.Cout % 16 == 0 && p.Cout >= 16 && p.Cout <= 256 &&
           (reinterpret_cast<uintptr_t>(p.in) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.out) & 15) == 0 &&
           (p.skip == nullptr || (reinterpret_cast<uintptr_t>(p.skip) & 15) == 0);
}

int launch_conv_tc(WgLaunch &L, const ConvPhase *ph, int nph, int total_taps, bool chunk_outer, cudaStream_t s) {
    if (nph < 1 || nph > 4) return VQB_ERR_UNSUPPORTED;
    L.w_rows = (long long)total_taps * L.ncols; L.w_inner = L.Cin;
    L.N = wg_gemm_cols(L.ncols);
    L.nph = nph;
    for (int i = 0; i < nph; ++i)
        if (!set_phase(L, i, ph[i], L.ncols, chunk_outer)) return VQB_ERR_UNSUPPORTED;
    return launch_wgconv(L, s);
}

// ------------------------------------------------------------------------------------------------ residual layer
// residual.py:18-29 on NHWC activations: the 3x3 GEMM (C -> Cmid), ReLU, the 1x1 GEMM (Cmid -> C) on the intermediate
// held in shared memory (fp32, or rounded to bf16), + r, ReLU.  Two kernels:
//   * res_scatter_kernel (TF32, Cmid = 32, a 128-pixel tile holds whole images): the 3x3 conv in scatter form, and
//     every application of a ResidualStack in the same launch.  Per CTA the tile r_i is loaded once, one unshifted
//     TMA box per 32-channel chunk, and stays in shared memory as the A operand.  Per kernel row dy (3 passes):
//         Y[p][dx, co] = r_i[p] . w1[tap (dy, dx)][co]                       (m64n96, N = 3 taps x 32 channels)
//     staged in shared memory; each consumer thread owns 16 (pixel, co) outputs of the intermediate and adds the
//     neighbours' terms, m[q][co] = sum over t = 0..8 in raster order of Y[q + (dy, dx)][dx, co], dropping the
//     neighbours outside the image (the zero padding).  Then relu(m) -> the 1x1 GEMM, + r_i (from the resident
//     tile), ReLU.  Between applications the result overwrites the resident tile in place (pixels outside the image
//     or past the batch as zero: the next application's padding); only the last application stores to `out`.
//     Two optional phases make it the whole latent block of a VQVAE inference forward (vqb_latent_block_tf32):
//       - head: r_0 = relu(conv(x) + b) of the k3 s1 conv (or stride-1 transposed conv) that feeds the stack, C
//         output channels, computed into the resident tile instead of loaded: wgconv_kernel's k-steps for that
//         layer from the same builder (set_phase: tap outer, chunk inner; shifted 4-D boxes of x, zero filled;
//         the same weight rows), accumulated from zero, then + bias and ReLU as store_tile does them.  So r_0 is
//         bitwise the separate conv launch's output, and so is everything after it.
//       - tail: z_e = r_n . Wpq^T + b (a 1x1 conv to TAIL_N channels, the k1 launch's 4 wgmma per 32-channel chunk
//         in one chain from zero, then the bias), stored as fp32 NHWC rows instead of r_n.
//   * otherwise wgconv_kernel with N2 = C: per tile the 3x3 GEMM's k-steps (the two separate conv launches' order
//     and operands in TF32), ReLU, the chained 1x1 GEMM.  One application per launch.
// Which kernel runs depends only on (bf16, C, Cmid, H, W), so a stack and its layers one by one compute the same bits.
constexpr int RS_MID = 32;                 // Cmid
constexpr int RS_N = 3 * RS_MID;           // GEMM columns per pass: one kernel row's 3 taps x Cmid
constexpr int RS_WBYTES = RS_N * 128;      // one pass's weight rows, one 128-byte channel chunk
constexpr int RS_YS = RS_N + 8;            // staged floats per pixel: + 8 against bank conflicts of the fragment stores
constexpr int RS_MAX_STAGES = 4;           // of the w1 ring, and of the head's ring
constexpr int TAIL_N = 64;                 // output channels of the tail (the VQ's embedding dim)

struct RsParams {
    float *out;                            // r_n, or z_e rows with a tail
    const float *head_bias, *tail_bias;
    int B, H, W, BW, BH, BN, napps, relu, stages;
    int head_steps, head_stages, tail;     // head_steps = 0: r_0 is loaded from tma_in
    int4 head[WG_MAX_STEPS];               // the head's k-steps: x = c0, y = dx, z = dy, w = w_row
};

// Shared memory (1024-byte aligned, C = 128 / 64):
//   act   NC chunks [128 px][128 B]                the resident tile r_i, the A operand          64 / 32 KB
//   ring  S stages of one pass's w1 rows [96][128 B]                                           48 KB
//   mid   relu(m) [128 px][128 B]                                                               16 KB
//   Y     [128 px][RS_YS] floats                                                                52 KB
//   w2s   w2 [C][128 B]                                                                         16 / 8 KB
//   bars  full[4], empty[4], hfull[4], hempty[4], abar, w2bar, tbar
// The head runs before any of ring .. w2s is used: its ring of head_stages x (A box [128 px][128 B] + C weight rows
// [C][128 B]) starts at `ring` and may reach the end of w2s, so the stack's w1 and w2 loads wait until every head stage
// is consumed.  The tail's weight [NC][TAIL_N][128 B] goes into the w1 ring once its last stage is consumed.
template <int C>
__global__ void __launch_bounds__(WG_THREADS, 1)
res_scatter_kernel(const __grid_constant__ CUtensorMap tma_in, const __grid_constant__ CUtensorMap tma_w1,
                   const __grid_constant__ CUtensorMap tma_w2, const __grid_constant__ CUtensorMap tma_hw,
                   const __grid_constant__ CUtensorMap tma_tw, const __grid_constant__ RsParams p) {
    constexpr int NC = C / 32;
    constexpr int HSTAGE = A_BYTES + C * 128;
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    const uint32_t act = (raw + 1023u) & ~1023u;
    const uint32_t ring = act + (uint32_t)(NC * A_BYTES);
    const uint32_t mid = ring + (uint32_t)(p.stages * RS_WBYTES);
    const uint32_t ysm = mid + (uint32_t)A_BYTES;
    const uint32_t w2s = ysm + (uint32_t)(128 * RS_YS * 4);
    const uint32_t bars = w2s + (uint32_t)(C * 128);
    float *const Y = reinterpret_cast<float *>(smem_raw + (ysm - raw));
    auto full = [&](int s) { return bars + 8u * s; };
    auto empty = [&](int s) { return bars + 8u * (RS_MAX_STAGES + s); };
    auto hfull = [&](int s) { return bars + 8u * (2 * RS_MAX_STAGES + s); };
    auto hempty = [&](int s) { return bars + 8u * (3 * RS_MAX_STAGES + s); };
    const uint32_t abar = bars + 8u * (4 * RS_MAX_STAGES), w2bar = abar + 8u, tbar = abar + 16u;
    const int S = p.stages, HS = p.head_stages, nh = p.head_steps;
    const int total = p.napps * 3 * NC;        // ring slots: application, pass (kernel row), chunk, innermost last
    const int n0 = blockIdx.x * p.BN;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int s = 0; s < S; ++s) { ptx::mbar_init(full(s), 1); ptx::mbar_init(empty(s), 2); }
        for (int s = 0; s < HS; ++s) { ptx::mbar_init(hfull(s), 1); ptx::mbar_init(hempty(s), 2); }
        ptx::mbar_init(abar, 1);
        ptx::mbar_init(w2bar, 1);
        ptx::mbar_init(tbar, 1);
        ptx::fence_mbar_init();
    }
    if (tid == 32) {
        ptx::prefetch_tmap(&tma_in);
        ptx::prefetch_tmap(&tma_w1);
        ptx::prefetch_tmap(&tma_w2);
        if (nh) ptx::prefetch_tmap(&tma_hw);
        if (p.tail) ptx::prefetch_tmap(&tma_tw);
    }
    __syncthreads();
    pdl_launch_dependents();

    if (warp == 0) {
        auto load_w1 = [&](int g) {
            const int s = g % S;
            ptx::mbar_expect_tx(full(s), (uint32_t)RS_WBYTES);
            ptx::tma_load_2d(ring + (uint32_t)(s * RS_WBYTES), &tma_w1, full(s), (g % NC) * 32, ((g / NC) % 3) * RS_N);
        };
        auto load_weights = [&] {
            ptx::mbar_expect_tx(w2bar, (uint32_t)(C * 128));
            ptx::tma_load_2d(w2s, &tma_w2, w2bar, 0, 0);
            for (int g = 0; g < S; ++g) load_w1(g);
        };
        if (lane == 0 && !nh) load_weights();      // weights do not depend on the previous layer
        pdl_wait();                                // ... the activations do
        if (lane == 0) {
            if (nh) {
                for (int i = 0; i < nh; ++i) {
                    const int s = i % HS;
                    if (i >= HS) ptx::mbar_wait(hempty(s), (uint32_t)((i / HS - 1) & 1));
                    const int4 st = p.head[i];
                    const uint32_t dst = ring + (uint32_t)(s * HSTAGE);
                    ptx::mbar_expect_tx(hfull(s), (uint32_t)HSTAGE);
                    ptx::tma_load_4d(dst, &tma_in, hfull(s), st.x, st.y, st.z, n0);
                    ptx::tma_load_2d(dst + A_BYTES, &tma_hw, hfull(s), st.x, st.w);
                }
                // the head's ring lies over the stack's weights: wait until its last stages are consumed
                for (int i = nh > HS ? nh - HS : 0; i < nh; ++i) ptx::mbar_wait(hempty(i % HS), (uint32_t)((i / HS) & 1));
                load_weights();
            } else {
                ptx::mbar_expect_tx(abar, (uint32_t)(NC * A_BYTES));
                for (int c = 0; c < NC; ++c) ptx::tma_load_4d(act + (uint32_t)(c * A_BYTES), &tma_in, abar, c * 32, 0, 0, n0);
            }
            for (int g = S; g < total; ++g) {
                ptx::mbar_wait(empty(g % S), (uint32_t)((g / S - 1) & 1));
                load_w1(g);
            }
            if (p.tail) {              // into the w1 ring once its last stages are consumed
                for (int g = total - S; g < total; ++g) ptx::mbar_wait(empty(g % S), (uint32_t)((g / S) & 1));
                ptx::mbar_expect_tx(tbar, (uint32_t)(NC * TAIL_N * 128));
                for (int c = 0; c < NC; ++c) ptx::tma_load_2d(ring + (uint32_t)(c * TAIL_N * 128), &tma_tw, tbar, c * 32, 0);
            }
        }
        return;
    }
    if (warp < 4) return;

    pdl_wait();                        // `out` may still be read by the previous layer
    const int wgi = (warp >> 2) - 1, wl = warp & 3, cw = warp - 4, cq = 2 * (lane & 3);
    const int lbw = __ffs(p.BW) - 1, lbh = __ffs(p.BH) - 1;
    // address in the resident tile of channels (c, c + 1) of tile row `row` (128-byte swizzle: piece j of row r at
    // j ^ (r & 7))
    auto act_addr = [&](int row, int c) {
        return act + (uint32_t)((c >> 5) * A_BYTES + row * 128 + ((((c & 31) >> 2) ^ (row & 7)) << 4) + (c & 3) * 4);
    };
    auto live_row = [&](int row) {
        const int bw = row & (p.BW - 1), bh = (row >> lbw) & (p.BH - 1), bn = row >> (lbw + lbh);
        return bw < p.W && bh < p.H && n0 + bn < p.B;
    };
    if (nh) {
        float acc[C / 2];
#pragma unroll
        for (int i = 0; i < C / 2; ++i) acc[i] = 0.f;
        for (int i = 0; i < nh; ++i) {
            const int s = i % HS;
            ptx::mbar_wait(hfull(s), (uint32_t)((i / HS) & 1));
            const uint32_t a = ring + (uint32_t)(s * HSTAGE + wgi * 64 * 128), b = ring + (uint32_t)(s * HSTAGE + A_BYTES);
            wg::fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) wg::mma<false, C>(acc, wg::desc_sw128(a + 32u * kk), wg::desc_sw128(b + 32u * kk), 1u);
            wg::commit();
            wg::wait<0>();
            wg::fence_regs<C>(acc);
            if (wl == 0 && lane == 0) ptx::mbar_arrive(hempty(s));
        }
        // relu(acc + bias) -> the resident tile as r_0, padding pixels as zero
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = wgi * 64 + wl * 16 + (lane >> 2) + 8 * h;
            const bool live = live_row(row);
#pragma unroll
            for (int j = 0; j < C / 8; ++j) {
                const int c = 8 * j + cq;
                float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                if (p.head_bias) { v0 += __ldg(p.head_bias + c); v1 += __ldg(p.head_bias + c + 1); }
                v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f);
                if (!live) { v0 = 0.f; v1 = 0.f; }
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(act_addr(row, c)), "f"(v0), "f"(v1) : "memory");
            }
        }
        ptx::fence_proxy_async();                    // r_0 -> the first application's wgmma
        ptx::named_bar_sync(2 + wgi, 128);
    } else {
        ptx::mbar_wait(abar, 0);
    }
    int g = 0;
    for (int app = 0; app < p.napps; ++app) {
        const bool last = app + 1 == p.napps;
        float m[16];                   // intermediate channel `lane` of pixels 16 cw .. + 15, taps added in raster order
#pragma unroll
        for (int i = 0; i < 16; ++i) m[i] = 0.f;
#pragma unroll 1
        for (int r = 0; r < 3; ++r) {
            float acc[RS_N / 2];       // the first k-step overwrites (scale-d 0): no register writes between the wgmma
            for (int c = 0; c < NC; ++c, ++g) {
                const int s = g % S;
                ptx::mbar_wait(full(s), (uint32_t)((g / S) & 1));
                const uint32_t a = act + (uint32_t)(c * A_BYTES + wgi * 64 * 128), b = ring + (uint32_t)(s * RS_WBYTES);
                wg::fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk) wg::mma<false, RS_N>(acc, wg::desc_sw128(a + 32u * kk), wg::desc_sw128(b + 32u * kk), (c | kk) != 0);
                wg::commit();
                wg::wait<0>();
                wg::fence_regs<RS_N>(acc);
                if (wl == 0 && lane == 0) ptx::mbar_arrive(empty(s));
            }
            ptx::named_bar_sync(1, 256);             // every thread has added the previous pass's terms
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float *yr = Y + (wgi * 64 + wl * 16 + (lane >> 2) + 8 * h) * RS_YS + cq;
#pragma unroll
                for (int j = 0; j < RS_N / 8; ++j)
                    *reinterpret_cast<float2 *>(yr + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
            ptx::named_bar_sync(1, 256);             // Y of all 128 pixels is staged
            const int dy = r - 1;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                // neighbours by (bn, bh, bw), never by flat row: no wrap into the next row or image.  A dropped term
                // adds +0, which leaves m bitwise as it was (m starts at +0 and so is never -0).
                const int q = cw * 16 + i, bw = q & (p.BW - 1), bh = (q >> lbw) & (p.BH - 1);
                const bool row_in = bh + dy >= 0 && bh + dy < p.H;
                const float *yq = Y + (row_in ? q + dy * p.BW : q) * RS_YS + lane;
                const float t0 = row_in && bw > 0 ? yq[-RS_YS] : 0.f;
                const float t1 = row_in ? yq[RS_MID] : 0.f;
                const float t2 = row_in && bw + 1 < p.W ? yq[RS_YS + 2 * RS_MID] : 0.f;
                m[i] += t0;
                m[i] += t1;
                m[i] += t2;
            }
        }
        // relu(m) -> this warp's 16 rows of the mid tile (fp32, 128-byte swizzle: piece j of row r at j ^ (r & 7))
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int row = cw * 16 + i;
            const uint32_t addr = mid + (uint32_t)(row * 128 + (((lane >> 2) ^ (row & 7)) << 4) + (lane & 3) * 4);
            asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(fmaxf(m[i], 0.f)) : "memory");
        }
        ptx::fence_proxy_async();                    // generic-proxy writes -> visible to wgmma
        ptx::named_bar_sync(2 + wgi, 128);           // this warpgroup's 64 rows are complete
        if (app == 0) ptx::mbar_wait(w2bar, 0);
        float acc2[C / 2];
        wg::fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
            wg::mma<false, C>(acc2, wg::desc_sw128(mid + (uint32_t)(wgi * 64 * 128) + 32u * kk), wg::desc_sw128(w2s + 32u * kk), kk != 0);
        wg::commit();
        wg::wait<0>();
        wg::fence_regs<C>(acc2);
        // + r_i from the resident tile, ReLU, back into the resident tile as r_{i+1} (pixels outside the image or past
        // the batch as zero: the next application's padding).  A warpgroup's GEMMs read only its own 64 rows of the
        // tile, and each element is read and written by one thread.
        const int relu = last ? p.relu : 1;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = wgi * 64 + wl * 16 + (lane >> 2) + 8 * h;
            const bool live = live_row(row);
#pragma unroll
            for (int j = 0; j < C / 8; ++j) {
                const int c = 8 * j + cq;
                const uint32_t addr = act_addr(row, c);
                float s0, s1;
                asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(s0), "=f"(s1) : "r"(addr) : "memory");
                float v0 = acc2[4 * j + 2 * h] + s0, v1 = acc2[4 * j + 2 * h + 1] + s1;
                if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                if (!live) { v0 = 0.f; v1 = 0.f; }
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v0), "f"(v1) : "memory");
            }
        }
        if (!last || p.tail) {
            ptx::fence_proxy_async();                // r_{i+1} -> the next application's (or the tail's) wgmma
            ptx::named_bar_sync(2 + wgi, 128);
        }
    }
    if (p.tail) {
        // z_e = r_n . Wpq^T + b for this warpgroup's 64 rows -> fp32 NHWC rows
        ptx::mbar_wait(tbar, 0);
        float acc3[TAIL_N / 2];
#pragma unroll
        for (int i = 0; i < TAIL_N / 2; ++i) acc3[i] = 0.f;
        wg::fence();
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            const uint32_t a = act + (uint32_t)(c * A_BYTES + wgi * 64 * 128), b = ring + (uint32_t)(c * TAIL_N * 128);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) wg::mma<false, TAIL_N>(acc3, wg::desc_sw128(a + 32u * kk), wg::desc_sw128(b + 32u * kk), 1u);
        }
        wg::commit();
        wg::wait<0>();
        wg::fence_regs<TAIL_N>(acc3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = wgi * 64 + wl * 16 + (lane >> 2) + 8 * h;
            const int bw = row & (p.BW - 1), bh = (row >> lbw) & (p.BH - 1), bn = row >> (lbw + lbh);
            if (bw >= p.W || bh >= p.H || n0 + bn >= p.B) continue;
            float *o = p.out + (((long long)(n0 + bn) * p.H + bh) * p.W + bw) * TAIL_N;
#pragma unroll
            for (int j = 0; j < TAIL_N / 8; ++j) {
                const int c = 8 * j + cq;
                float v0 = acc3[4 * j + 2 * h], v1 = acc3[4 * j + 2 * h + 1];
                if (p.tail_bias) { v0 += __ldg(p.tail_bias + c); v1 += __ldg(p.tail_bias + c + 1); }
                *reinterpret_cast<float2 *>(o + c) = make_float2(v0, v1);
            }
        }
        return;
    }
    // the last application's 16 rows of this warp (written by its own lanes) -> `out`, 16 bytes per lane
    __syncwarp();
    for (int e = lane; e < 16 * (C / 4); e += 32) {
        const int row = wgi * 64 + wl * 16 + e / (C / 4), c = (e % (C / 4)) * 4;
        const int bw = row & (p.BW - 1), bh = (row >> lbw) & (p.BH - 1), bn = row >> (lbw + lbh);
        if (bw >= p.W || bh >= p.H || n0 + bn >= p.B) continue;
        float4 v;
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(act_addr(row, c)) : "memory");
        *reinterpret_cast<float4 *>(p.out + (((long long)(n0 + bn) * p.H + bh) * p.W + bw) * C + c) = v;
    }
}

bool res_scatter_supported(int C, int Cmid, int H, int W) {
    return (C == 64 || C == 128) && Cmid == RS_MID && H >= 1 && W >= 1 && W <= 16 && pow2_ceil(W) * pow2_ceil(H) <= 128;
}

// The conv that feeds the stack (x: NHWC fp32 (B, H, W, Cin); w: its vqb_pack_conv_weight_f32 rows [9][C][Cin]) and
// the 1x1 conv after it (w: [TAIL_N][C]); null members: no such phase.
struct RsHead { const void *x, *w; const float *bias; int Cin, transposed; };
struct RsTail { const void *w; const float *bias; };

// r, out: NHWC fp32 (B, H, W, C) (out: (B, H, W, TAIL_N) with a tail); w1: [9][32][C]; w2: [C][32].  With a head, r is
// not read.
static int launch_res_scatter(const RsHead &head, const RsTail &tail, const void *r, const void *w1, const void *w2,
                              void *out, int B, int H, int W, int C, int relu_out, int napps, cudaStream_t s) {
    RsParams q;
    memset(&q, 0, sizeof(q));
    q.out = static_cast<float *>(out);
    q.head_bias = head.bias; q.tail_bias = tail.bias; q.tail = tail.w != nullptr;
    q.B = B; q.H = H; q.W = W; q.napps = napps; q.relu = relu_out;
    q.BW = pow2_ceil(W); q.BH = pow2_ceil(H); q.BN = 128 / (q.BW * q.BH);      // the tile launch_wgconv would pick
    const int total = napps * 3 * (C / 32);
    q.stages = total < RS_MAX_STAGES ? total : RS_MAX_STAGES;
    const long long grid = ((long long)B + q.BN - 1) / q.BN;
    if (grid > 0x7fffffffLL) return VQB_ERR_UNSUPPORTED;
    const int region = q.stages * RS_WBYTES + A_BYTES + 128 * RS_YS * 4 + C * 128;     // ring .. the end of w2s
    if (q.tail && (C / 32) * TAIL_N * 128 > q.stages * RS_WBYTES) return VQB_ERR_UNSUPPORTED;

    const CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    CUtensorMap tin, tw1, tw2, thw, ttw;
    const int Cin = head.x ? head.Cin : C;
    const uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    const uint64_t strides[3] = {(uint64_t)Cin * 4, (uint64_t)W * Cin * 4, (uint64_t)H * W * Cin * 4};
    const uint32_t box[4] = {32u, (uint32_t)q.BW, (uint32_t)q.BH, (uint32_t)q.BN};
    const uint32_t es[4] = {1u, 1u, 1u, 1u};
    int rc = vqb_encode_tmap_4d(&tin, dt, head.x ? head.x : r, dims, strides, box, es, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    rc = vqb_encode_tmap_2d(&tw1, dt, w1, (uint64_t)C, 9ull * RS_MID, (uint64_t)C * 4, 32u, (uint32_t)RS_N,
                            CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    rc = vqb_encode_tmap_2d(&tw2, dt, w2, (uint64_t)RS_MID, (uint64_t)C, (uint64_t)RS_MID * 4, 32u, (uint32_t)C,
                            CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    thw = ttw = tw1;
    if (head.x) {
        // the k-steps of the separate launch of this conv (vqb_conv2d_f32 -> launch_conv_tc): the same builder
        WgLaunch L;
        L.bf16 = 0; L.Cin = Cin;
        ConvPhase ph;
        conv_phase(conv_geom(3, 3, 1, 1, head.transposed, H, W), 0, ph);
        if (!set_phase(L, 0, ph, C, false)) return VQB_ERR_UNSUPPORTED;
        q.head_steps = L.nsteps[0];
        for (int i = 0; i < q.head_steps; ++i) {
            const WgStep &st = L.steps[0][i];
            q.head[i] = make_int4(st.c0, st.dx, st.dy, st.w_row);
        }
        const int hstage = A_BYTES + C * 128;
        q.head_stages = region / hstage < RS_MAX_STAGES ? region / hstage : RS_MAX_STAGES;
        if (q.head_stages > q.head_steps) q.head_stages = q.head_steps;
        rc = vqb_encode_tmap_2d(&thw, dt, head.w, (uint64_t)Cin, 9ull * C, (uint64_t)Cin * 4, 32u, (uint32_t)C,
                                CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    if (q.tail) {
        rc = vqb_encode_tmap_2d(&ttw, dt, tail.w, (uint64_t)C, (uint64_t)TAIL_N, (uint64_t)C * 4, 32u, (uint32_t)TAIL_N,
                                CU_TENSOR_MAP_SWIZZLE_128B);
        if (rc) return rc;
    }
    const int smem = 1024 + (C / 32) * A_BYTES + region + 8 * (4 * RS_MAX_STAGES + 3);
    auto kernel = C == 128 ? res_scatter_kernel<128> : res_scatter_kernel<64>;
    static bool attr_set[2] = {false, false};
    if (!attr_set[C == 128]) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
        if (e != cudaSuccess) return (int)e;
        attr_set[C == 128] = true;
    }
    if (cudaError_t le = vqb_launch(kernel, dim3((unsigned)grid), dim3(WG_THREADS), (size_t)smem, s, tin, tw1, tw2, thw,
                                    ttw, q))
        return (int)le;
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

bool latent_block_supported(int Cin, int C, int Cmid, int H, int W, int tail_cout) {
    return res_scatter_supported(C, Cmid, H, W) && Cin % 32 == 0 && 9 * (Cin / 32) <= WG_MAX_STEPS &&
           (tail_cout == 0 || tail_cout == TAIL_N);
}

int launch_latent_block(const void *x, const void *head_w, const float *head_bias, int Cin, int transposed,
                        const void *w1, const void *w2, int napps, const void *tail_w, const float *tail_bias,
                        int tail_cout, void *out, int B, int H, int W, int C, int Cmid, cudaStream_t s) {
    if (!latent_block_supported(Cin, C, Cmid, H, W, tail_cout) || (tail_w != nullptr) != (tail_cout != 0) || napps < 1 ||
        x == out)
        return VQB_ERR_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) return VQB_ERR_UNSUPPORTED;
    return launch_res_scatter(RsHead{x, head_w, head_bias, Cin, transposed}, RsTail{tail_w, tail_bias}, nullptr, w1, w2,
                              out, B, H, W, C, 1, napps, s);
}

bool res_wg_supported(int bf16, int C, int Cmid) {
    return (C == 64 || C == 128) && (bf16 ? Cmid % 16 == 0 && Cmid >= 16 && Cmid <= 64 : Cmid == 32 || Cmid == 64);
}

// w1: [9][Cmid][C]; w2: [C][Cmid] (TF32) or [C][64] (bf16, Cmid zero padded to one chunk).  napps > 1 (a ResidualStack
// of one shared layer) runs on res_scatter_kernel only and answers VQB_ERR_UNSUPPORTED elsewhere.
int launch_res_wg(int bf16, const void *r, const void *w1, const void *w2, void *out, int B, int H, int W, int C, int Cmid,
                  int relu_out, int napps, cudaStream_t s) {
    if (!res_wg_supported(bf16, C, Cmid) || r == out || napps < 1) return VQB_ERR_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(r) | reinterpret_cast<uintptr_t>(out)) & 15) return VQB_ERR_UNSUPPORTED;
    if (!bf16 && res_scatter_supported(C, Cmid, H, W))
        return launch_res_scatter(RsHead{}, RsTail{}, r, w1, w2, out, B, H, W, C, relu_out, napps, s);
    if (napps > 1) return VQB_ERR_UNSUPPORTED;
    WgLaunch L;
    L.bf16 = bf16;
    L.in = r; L.B = B; L.Cin = C; L.H = H; L.W = W;
    L.w = w1; L.w_rows = 9LL * Cmid; L.w_inner = C;
    L.N = wg_gemm_cols(Cmid); L.ncols = Cmid;
    L.w2 = w2; L.w2_rows = C; L.w2_inner = bf16 ? 64 : Cmid; L.N2 = C;
    L.skip = r; L.out = out; L.out_bf16 = bf16; L.relu = relu_out;
    L.out_sn = (long long)H * W * C; L.out_sh = (long long)W * C; L.out_sw = C; L.out_sc = 1;
    set_phase(L, 0, taps3x3(H, W), Cmid, bf16);
    return launch_wgconv(L, s);
}

// ------------------------------------------------------------------------------------------------ output layer
// decoder.py:34-35, ConvTranspose2d(Cin -> Cout <= 4, k4 s2 p1), NHWC in, NCHW fp32 out, in scatter form.  Output
// pixel (2 gy + py, 2 gx + px) takes input pixel (gy + dy, gx + dx) through kernel tap (py - 2 dy + 1, px - 2 dx + 1):
// for each phase (py, px) the 2 x 2 neighbours dy = ky + py - 1, dx = kx + px - 1 (ky, kx in {0, 1}).  So every input
// pixel p of a tile and its one-pixel halo is multiplied once by the 64 weight rows (phase, (ky, kx), co):
//   Y[p][phase, k, co] = in[p] . w[tap of (phase, k)][phase, co]          (one m64n64 GEMM per warpgroup and chunk)
// and the epilogue gathers
//   out(2 gy + py, 2 gx + px, co) = act(Y[(gy + dy, gx + dx)][phase, k, co] summed over k = 0..3 in raster (dy, dx)
//                                       order, + bias[co])
// through shared memory.  The A operand is one 4-D TMA box {128 B of channels, TW + 2, TH + 2, 1} per chunk: the
// tile's (TW + 2) x (TH + 2) halo pixels as plain rows (at most 128; TMA zero fills outside the image, which is the
// padding).  Persistent CTAs: each gathers the 64 rows it needs from w_shuffle into shared memory once (in the 128-byte
// swizzle wgmma reads, channels co >= Cout zero), then warp 8 streams the A boxes of the CTA's tiles through a ring
// while warpgroups 0 and 1 run the GEMM and the epilogue.
// w_shuffle: [9 taps (dy, dx)][16][Cin] (the region of vqb_pack_conv_weight_f32 at conv_pack_shuffle_offset, or
// vqb_pack_conv_weight_bf16); row (py * 2 + px) * Cout + co of tap (dy + 1) * 3 + dx + 1.
constexpr int SC_ROW = 66;                 // staged floats per halo pixel: the 64 columns + 2 against bank conflicts
constexpr int SC_STAGE_BYTES = 128 * SC_ROW * 4;
constexpr int SC_MAX_STAGES = 4;
constexpr int SC_THREADS = 288;            // warpgroups 0 and 1 (weight gather, GEMM, epilogue), warp 8 (TMA producer)

struct ScParams {
    const void *w;
    const float *bias;
    float *out;
    int B, H, W, Cin, Cout, nc, ck, TW, TH, tiles_x, tiles_y, ntiles, stages, relu;
    long long out_sn, out_sc, out_sh;
};

template <bool BF16>
__global__ void __launch_bounds__(SC_THREADS, 2)
convt_scatter_kernel(const __grid_constant__ CUtensorMap tma_in, const __grid_constant__ ScParams p) {
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    const uint32_t wres = (raw + 1023u) & ~1023u;                        // nc gathered weight chunks [64][128 B]
    const uint32_t ring = wres + (uint32_t)(p.nc * SC_BBYTES);           // stages of one A box [128 px][128 B]
    const uint32_t bars = ring + (uint32_t)(p.stages * A_BYTES);
    float *const st = reinterpret_cast<float *>(smem_raw + (bars + 128u - raw));     // [128 px][SC_ROW]
    auto full = [&](int s) { return bars + 8u * s; };
    auto empty = [&](int s) { return bars + 8u * (SC_MAX_STAGES + s); };
    const int S = p.stages, HW2 = p.TW + 2;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int s = 0; s < S; ++s) { ptx::mbar_init(full(s), 1); ptx::mbar_init(empty(s), 2); }
        ptx::fence_mbar_init();
    }
    if (tid == 256) ptx::prefetch_tmap(&tma_in);
    __syncthreads();
    pdl_launch_dependents();

    if (warp == 8) {
        pdl_wait();                   // the activations come from the previous layer
        if (lane == 0) {
            const uint32_t abytes = (uint32_t)(HW2 * (p.TH + 2) * 128);
            int g = 0;
            for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
                const int tx = tile % p.tiles_x, ty = (tile / p.tiles_x) % p.tiles_y, n = tile / (p.tiles_x * p.tiles_y);
                for (int c = 0; c < p.nc; ++c, ++g) {
                    const int s = g % S;
                    if (g >= S) ptx::mbar_wait(empty(s), (uint32_t)((g / S - 1) & 1));
                    ptx::mbar_expect_tx(full(s), abytes);
                    ptx::tma_load_4d(ring + (uint32_t)(s * A_BYTES), &tma_in, full(s), c * p.ck, tx * p.TW - 1, ty * p.TH - 1, n);
                }
            }
        }
        return;
    }

    // gather the weight (it does not depend on the previous layer)
    gather_shuffle_weight<BF16>(wres, p.w, p.Cin, p.Cout, p.nc, tid);
    float bias[4];
#pragma unroll
    for (int co = 0; co < 4; ++co) bias[co] = p.bias && co < p.Cout ? __ldg(p.bias + co) : 0.f;
    pdl_wait();                       // `out` may still be read by the previous layer's consumers of it
    const int wgi = warp >> 2, wl = warp & 3, cq = 2 * (lane & 3);
    int g = 0;
    for (int tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
        const int tx = tile % p.tiles_x, ty = (tile / p.tiles_x) % p.tiles_y, n = tile / (p.tiles_x * p.tiles_y);
        float acc[SC_N / 2];
#pragma unroll
        for (int i = 0; i < SC_N / 2; ++i) acc[i] = 0.f;
        // first tile: the gathered weight is complete; later tiles: the previous epilogue has read the staging rows
        ptx::named_bar_sync(1, 256);
        for (int c = 0; c < p.nc; ++c, ++g) {
            const int s = g % S;
            ptx::mbar_wait(full(s), (uint32_t)((g / S) & 1));
            const uint32_t a = ring + (uint32_t)(s * A_BYTES + wgi * 64 * 128), b = wres + (uint32_t)(c * SC_BBYTES);
            wg::fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) wg::mma<BF16, SC_N>(acc, wg::desc_sw128(a + 32u * kk), wg::desc_sw128(b + 32u * kk), 1u);
            wg::commit();
            wg::wait<0>();
            wg::fence_regs<SC_N>(acc);
            if (wl == 0 && lane == 0) ptx::mbar_arrive(empty(s));
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float *sr = st + (wgi * 64 + wl * 16 + (lane >> 2) + 8 * h) * SC_ROW + cq;
#pragma unroll
            for (int j = 0; j < SC_N / 8; ++j)
                *reinterpret_cast<float2 *>(sr + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
        ptx::named_bar_sync(1, 256);
        // lane = output column ox = 2 bx + px of the tile, warps over the output rows (co, by, py)
        const int gx0 = tx * p.TW, gy0 = ty * p.TH, bx = lane >> 1, px = lane & 1;
        float *out = p.out + (long long)n * p.out_sn + 2 * gx0 + lane;
        const bool live = lane < 2 * p.TW && gx0 + bx < p.W;
#pragma unroll
        for (int co = 0; co < 4; ++co) {
            if (co >= p.Cout || !live) break;
            for (int r = warp; r < 2 * p.TH; r += 8) {
                const int by = r >> 1, py = r & 1;
                if (gy0 + by >= p.H) break;
                // neighbour k = (ky, kx) of phase (py, px): halo row by + ky + py, halo column bx + kx + px
                const float *s0 = st + ((by + py) * HW2 + bx + px) * SC_ROW + (py * 2 + px) * 16 + co;
                float v = s0[0];
                v += s0[SC_ROW + 4];
                v += s0[HW2 * SC_ROW + 8];
                v += s0[(HW2 + 1) * SC_ROW + 12];
                v += bias[co];
                if (p.relu) v = fmaxf(v, 0.f);
                out[(long long)co * p.out_sc + (long long)(2 * (gy0 + by) + py) * p.out_sh] = v;
            }
        }
    }
}

bool convt_shuffle_supported(int Cin, int Cout) { return Cout >= 1 && Cout <= 4 && Cin % 32 == 0 && Cin <= 256; }

int launch_convt_shuffle_wg(int bf16, const void *in, const void *w_shuffle, const float *bias, float *out, int B, int Cin,
                            int H, int W, int Cout, int relu, cudaStream_t s) {
    if (!convt_shuffle_supported(Cin, Cout)) return VQB_ERR_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(w_shuffle)) & 15) return VQB_ERR_UNSUPPORTED;
    const int esz = bf16 ? 2 : 4, ck = 128 / esz;
    if (Cin % ck != 0) return VQB_ERR_UNSUPPORTED;
    ScParams q;
    memset(&q, 0, sizeof(q));
    q.w = w_shuffle; q.bias = bias; q.out = out; q.relu = relu;
    q.B = B; q.H = H; q.W = W; q.Cin = Cin; q.Cout = Cout; q.nc = Cin / ck; q.ck = ck;
    // tiles of at most 16 columns whose halo (TW + 2) x (TH + 2) fits 128 rows, split evenly over the image
    q.tiles_x = (W + 15) / 16;
    q.TW = (W + q.tiles_x - 1) / q.tiles_x;
    const int th_max = 128 / (q.TW + 2) - 2;
    q.tiles_y = (H + th_max - 1) / th_max;
    q.TH = (H + q.tiles_y - 1) / q.tiles_y;
    const long long ntiles = (long long)q.tiles_x * q.tiles_y * B;
    if (ntiles <= 0 || ntiles > 0x7fffffffLL) return VQB_ERR_UNSUPPORTED;
    q.ntiles = (int)ntiles;
    q.out_sn = 4LL * Cout * H * W; q.out_sc = 4LL * H * W; q.out_sh = 2LL * W;

    CUtensorMap tin;
    const uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    const uint64_t strides[3] = {(uint64_t)Cin * esz, (uint64_t)W * Cin * esz, (uint64_t)H * W * Cin * esz};
    const uint32_t box[4] = {(uint32_t)ck, (uint32_t)(q.TW + 2), (uint32_t)(q.TH + 2), 1u};
    const uint32_t es[4] = {1u, 1u, 1u, 1u};
    const int rc = vqb_encode_tmap_4d(&tin, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, in,
                                      dims, strides, box, es, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;

    // the gathered weight, the ring, the barriers and the staging rows: two CTAs per SM (113 KB each) when that keeps
    // 2 stages, so one CTA's epilogue overlaps the other's GEMM; else one CTA with up to 4 stages
    auto smem_for = [&](int stages) { return 1024 + q.nc * SC_BBYTES + stages * A_BYTES + 128 + SC_STAGE_BYTES; };
    auto kernel = bf16 ? convt_scatter_kernel<true> : convt_scatter_kernel<false>;
    static bool attr_set[2] = {false, false};
    if (!attr_set[bf16 ? 1 : 0]) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
        if (e != cudaSuccess) return (int)e;
        attr_set[bf16 ? 1 : 0] = true;
    }
    int dev = 0, sms = 132, per_sm = 1, occ = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int stages = SC_MAX_STAGES;
    while (stages > 2 && smem_for(stages) > 113 * 1024) --stages;
    if (smem_for(stages) <= 113 * 1024 && ntiles > sms &&
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, SC_THREADS, (size_t)smem_for(stages)) == cudaSuccess &&
        occ >= 2) {
        per_sm = 2;
    } else {
        stages = SC_MAX_STAGES;
        while (stages > 1 && smem_for(stages) > 220 * 1024) --stages;
    }
    q.stages = stages;
    const long long grid = ntiles < (long long)per_sm * sms ? ntiles : (long long)per_sm * sms;
    if (cudaError_t le = vqb_launch(kernel, dim3((unsigned)grid), dim3(SC_THREADS), (size_t)smem_for(stages), s, tin, q))
        return (int)le;
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------ decoder tail
// decoder.py:32-35 from d_out: the k4 s2 transposed conv Cin -> 64 with ReLU and the output layer 64 -> Cout <= 4 as one
// wgconv_kernel launch in TAIL mode (see above the kernel), one CTA per whole-image tile.
bool decoder_tail_supported(int Cin, int H, int W, int C, int Cout) {
    return C == SC_N && Cout >= 1 && Cout <= 4 && Cin % 32 == 0 && Cin >= 32 && Cin <= 256 && H >= 1 && W >= 1 &&
           W <= 16 && pow2_ceil(W) * pow2_ceil(H) <= 128;
}

int launch_decoder_tail(const void *d_out, const void *convt_w, const float *convt_bias, const void *out_w,
                        const float *out_bias, void *h_out, float *x_hat, int B, int Cin, int H, int W, int C, int Cout,
                        int relu_out, cudaStream_t s) {
    if (!decoder_tail_supported(Cin, H, W, C, Cout) || d_out == h_out || d_out == x_hat) return VQB_ERR_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(d_out) | reinterpret_cast<uintptr_t>(h_out) | reinterpret_cast<uintptr_t>(x_hat) |
         reinterpret_cast<uintptr_t>(convt_w) | reinterpret_cast<uintptr_t>(out_w)) & 15)
        return VQB_ERR_UNSUPPORTED;
    // the separate launch of the transposed conv (vqb_conv2d_f32 -> launch_conv_tc): the same phases and k-steps
    const ConvGeom g = conv_geom(4, 4, 2, 1, 1, H, W);
    ConvPhase phases[4];
    for (int i = 0; i < 4; ++i)
        if (!conv_phase(g, i, phases[i])) return VQB_ERR_UNSUPPORTED;
    WgLaunch L;
    L.in = d_out; L.B = B; L.Cin = Cin; L.H = H; L.W = W;
    L.w = convt_w; L.ncols = C;
    L.bias = convt_bias; L.out = h_out; L.relu = 1;
    layout_strides(VQB_NHWC, C, g.OH, g.OW, L.out_sn, L.out_sh, L.out_sw, L.out_sc);
    L.tail_w = static_cast<const float *>(out_w) + conv_pack_shuffle_offset(Cout, C, 4, 4);
    L.tail_bias = out_bias; L.tail_out = x_hat; L.tail_cout = Cout; L.tail_relu = relu_out;
    return launch_conv_tc(L, phases, 4, 16, false, s);
}

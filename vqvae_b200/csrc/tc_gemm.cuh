// tc_gemm.cuh -- the TF32 tensor-core GEMM (wgmma, sm_90a) behind the FFMA GEMM's interface (ffma_gemm.cuh): the same
// operand accessors, epilogues and WgradSplit chunking, so a product written for `gemm` runs on tensor cores by
// calling `tc_gemm` instead.  Internal; used by the prior's TF32 forward and backward (prior_gemm.cu).
//
// tc_gemm_kernel computes out(m, n) = sum over k in chunk z of A(m, k) * B(k, n).  Per CTA: a 128-row tile, two
// warpgroups of m64nBNk8 (BN = 64 or 128, chosen per call from N), k-steps of 32 floats.  Both operands are staged
// K-major into 128-byte swizzled shared-memory rows, A as [m][k] and B as [n][k], through registers: each thread loads
// the next k-step while the tensor cores run the current one, then writes it to the other of two stages.  That k-loop
// is `tc_tile`, which prior_gemm.cu's log_prob head (`tc_lse_kernel`) also runs, tile after tile, with the staging
// modes `tc_modes` and the tile width `tc_bn` choose here: its products are bitwise this kernel's.
//
// Staging.  An operand accessor may offer 32 consecutive k of one row as a pointer (A: `seg(i, k0)`, contiguous along
// j; B: `segT(k0, j)`, contiguous along i), or nullptr for a row of zeros (a tap outside the grid).  When the product's
// k-steps never cross such a row (K and the chunk multiples of 32, and the accessor's `seg_ok()`), the tile is loaded
// with one 16-byte load and one position decode per four values, eight threads per 128-byte row.  Otherwise each value
// goes through the accessor's operator(), with consecutive threads on whichever index is contiguous in memory, and
// is transposed on its way into shared memory.
//
// Rounding.  Every staged value is rounded to TF32 with cvt.rna (round to nearest, ties away from zero: the low 13
// mantissa bits become zero) before it is stored, so the tensor cores see exact TF32 operands and the rounding does
// not depend on how the hardware treats the low bits of an fp32 input.  Products of two TF32 values are exact in fp32;
// the accumulation is the hardware's fp32 accumulation in a fixed order, so results are bitwise reproducible.
// `tf32_round` in tests/prior_tf32_port.py restates this rounding.
#pragma once
#include <type_traits>

#include "ffma_gemm.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace {

constexpr int TC_BM = 128, TC_BK = 32, TC_T = 256;     // CTA rows, k-step, threads (two warpgroups)

template <int BN>
struct TcTile {
    static constexpr int A_BYTES = TC_BM * 128, B_BYTES = BN * 128, STAGE = A_BYTES + B_BYTES;
    static constexpr int SMEM = 2 * STAGE + 1024;      // two stages, plus slack to align the base to 1024 bytes
};

template <class L, class = void>
constexpr bool has_seg = false;
template <class L>
constexpr bool has_seg<L, std::void_t<decltype(&L::seg)>> = true;
template <class L, class = void>
constexpr bool has_segT = false;
template <class L>
constexpr bool has_segT<L, std::void_t<decltype(&L::segT)>> = true;

__device__ __forceinline__ float tf32_rna(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

// byte offset of element kk of row r: 16-byte piece kk/4 of the 128-byte row sits at (kk/4) ^ (r % 8)
__device__ __forceinline__ uint32_t swz(int r, int kk) {
    return (uint32_t)(r * 128 + ((((kk >> 2) ^ r) & 7) << 4) + (kk & 3) * 4);
}

// How an operand is staged: value by value through operator(), or 16 bytes at a time from a pointer that the accessor
// gives for 32 consecutive k of one row (A: seg(i, k0); B: segT(k0, j)), or (B only) for consecutive columns n of one
// k (seg(k, n)), four of which go to four rows of the K-major tile.
enum StageMode { BY_VALUE = 0, ALONG_K = 1, ALONG_N = 2 };

// One operand's share of a k-step: ROWS rows (A: m, B: n) of TC_BK k each, staged in two halves (`part`) so that
// only half of a thread's values are live in registers between the global loads and the shared-memory stores.
// Row r0 + rr < R at k = k0 + kk, kk < kn; 0 elsewhere.
template <bool IsB, int ROWS, class L>
struct Stager {
    static constexpr int NV = ROWS * TC_BK / TC_T / 2;             // values per thread and part
    static constexpr bool r_fast = IsB ? L::j_fast : !L::j_fast;   // consecutive threads: consecutive addresses
    float v[NV];

    __device__ __forceinline__ void load(const L &l, int mode, int part, int r0, int R, long long k0, int kn) {
        const int tid = threadIdx.x;
        if constexpr (IsB ? has_segT<L> : has_seg<L>) {
            if (mode == ALONG_K) {                      // whole rows of 32 k: kn == TC_BK
#pragma unroll
                for (int q = 0; q < NV / 4; ++q) {
                    const int u = tid + (part * NV / 4 + q) * TC_T, rr = u >> 3, kq = u & 7, r = r0 + rr;
                    const float *p = nullptr;
                    if (r < R) {
                        if constexpr (IsB) p = l.segT(k0, r);
                        else p = l.seg(r, k0);
                    }
                    float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (p) f = __ldg(reinterpret_cast<const float4 *>(p) + kq);
                    v[4 * q] = f.x; v[4 * q + 1] = f.y; v[4 * q + 2] = f.z; v[4 * q + 3] = f.w;
                }
                return;
            }
        }
        if constexpr (IsB && has_seg<L>) {
            if (mode == ALONG_N) {                      // four columns per load; R % 4 == 0
#pragma unroll
                for (int q = 0; q < NV / 4; ++q) {
                    const int u = tid + (part * NV / 4 + q) * TC_T, rq = u % (ROWS / 4), kk = u / (ROWS / 4);
                    const int r = r0 + 4 * rq;
                    float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
                    const float *p = r < R && kk < kn ? l.seg(k0 + kk, r) : nullptr;
                    if (p) f = __ldg(reinterpret_cast<const float4 *>(p));
                    v[4 * q] = f.x; v[4 * q + 1] = f.y; v[4 * q + 2] = f.z; v[4 * q + 3] = f.w;
                }
                return;
            }
        }
#pragma unroll
        for (int q = 0; q < NV; ++q) {
            const int e = tid + (part * NV + q) * TC_T;
            const int rr = r_fast ? e % ROWS : e / TC_BK, kk = r_fast ? e / ROWS : e % TC_BK, r = r0 + rr;
            float x = 0.f;
            if (r < R && kk < kn) {
                if constexpr (IsB) x = l(k0 + kk, r);
                else x = l(r, k0 + kk);
            }
            v[q] = x;
        }
    }

    __device__ __forceinline__ void store(uint32_t base, int mode, int part) const {
        const int tid = threadIdx.x;
        if (mode == ALONG_K) {
#pragma unroll
            for (int q = 0; q < NV / 4; ++q) {
                const int u = tid + (part * NV / 4 + q) * TC_T, rr = u >> 3, kq = u & 7;
                const uint32_t addr = base + (uint32_t)(rr * 128 + ((kq ^ (rr & 7)) << 4));
                asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(tf32_rna(v[4 * q])),
                             "f"(tf32_rna(v[4 * q + 1])), "f"(tf32_rna(v[4 * q + 2])), "f"(tf32_rna(v[4 * q + 3]))
                             : "memory");
            }
            return;
        }
        if (mode == ALONG_N) {
#pragma unroll
            for (int q = 0; q < NV / 4; ++q) {
                const int u = tid + (part * NV / 4 + q) * TC_T, rq = u % (ROWS / 4), kk = u / (ROWS / 4);
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    asm volatile("st.shared.f32 [%0], %1;" ::"r"(base + swz(4 * rq + i, kk)), "f"(tf32_rna(v[4 * q + i]))
                                 : "memory");
            }
            return;
        }
#pragma unroll
        for (int q = 0; q < NV; ++q) {
            const int e = tid + (part * NV + q) * TC_T;
            const int rr = r_fast ? e % ROWS : e / TC_BK, kk = r_fast ? e / ROWS : e % TC_BK;
            asm volatile("st.shared.f32 [%0], %1;" ::"r"(base + swz(rr, kk)), "f"(tf32_rna(v[q])) : "memory");
        }
    }
};

// The (128 x BN) tile at rows m0, columns n0 of the product over k in [k_begin, k_begin + kc), into acc in wgmma's
// accumulator layout (wgmma.cuh), staged through the two stages at `base` (TcTile<BN>).  Every thread of the CTA
// calls it.  On return no wgmma of this thread is in flight, but the other warpgroup may still read the stage of the
// last k-step: a caller that runs the loop again first waits for the whole CTA.
template <int BN, class LA, class LB>
__device__ __forceinline__ void tc_tile(float (&acc)[BN / 2], const LA &a, const LB &b, uint32_t base, int m0, int M,
                                        int n0, int N, long long k_begin, int kc, int a_mode, int b_mode) {
    using T = TcTile<BN>;
    const int wgi = threadIdx.x >> 7;
    const int steps = (kc + TC_BK - 1) / TC_BK;
    Stager<false, TC_BM, LA> sa;
    Stager<true, BN, LB> sb;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    // k-step s of both operands into stage s % 2
    auto stage = [&](int s) {
        const long long k0 = k_begin + (long long)s * TC_BK;
        const int kn = min(TC_BK, kc - s * TC_BK);
        const uint32_t at = base + (uint32_t)((s & 1) * T::STAGE);
#pragma unroll
        for (int part = 0; part < 2; ++part) {
            sa.load(a, a_mode, part, m0, M, k0, kn);
            sa.store(at, a_mode, part);
        }
#pragma unroll
        for (int part = 0; part < 2; ++part) {
            sb.load(b, b_mode, part, n0, N, k0, kn);
            sb.store(at + T::A_BYTES, b_mode, part);
        }
    };
    if (steps > 0) stage(0);
    for (int s = 0; s < steps; ++s) {
        // stage s % 2 is written (by every thread) and stage (s + 1) % 2 is no longer read (both warpgroups waited)
        const uint32_t cur = base + (uint32_t)((s & 1) * T::STAGE);
        ptx::fence_proxy_async();                       // generic-proxy stores -> visible to wgmma
        __syncthreads();
        wg::fence();
        const uint32_t da = cur + (uint32_t)(wgi * 64 * 128), db = cur + T::A_BYTES;
#pragma unroll
        for (int kk = 0; kk < TC_BK / 8; ++kk)
            wg::mma<false, BN>(acc, wg::desc_sw128(da + 32u * kk), wg::desc_sw128(db + 32u * kk), 1u);
        wg::commit();
        if (s + 1 < steps) stage(s + 1);                 // overlaps the tensor cores' work on step s
        wg::wait<0>();
        wg::fence_regs<BN>(acc);
    }
}

template <int BN, class LA, class LB, class EP>
__global__ void __launch_bounds__(TC_T) tc_gemm_kernel(LA a, LB b, EP ep, int M, int N, long long K, int chunk,
                                                       int a_mode, int b_mode) {
    extern __shared__ unsigned char tc_smem[];
    const uint32_t base = (ptx::smem_u32(tc_smem) + 1023u) & ~1023u;
    const int tid = threadIdx.x, wgi = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const int m0 = blockIdx.x * TC_BM, n0 = blockIdx.y * BN;
    const long long k_begin = (long long)blockIdx.z * chunk;
    const int kc = (int)min((long long)chunk, K - k_begin);     // this chunk's k, counted in 32 bits
    float acc[BN / 2];
    tc_tile<BN>(acc, a, b, base, m0, M, n0, N, k_begin, kc, a_mode, b_mode);
    // wgmma's accumulator layout (wgmma.cuh): row 16*warp + lane/4 (+8), columns 8j + 2*(lane%4) + {0,1}
    const int row = m0 + wgi * 64 + warp * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int m = row + 8 * h, n = n0 + 8 * j + 2 * (lane & 3) + e;
                if (m < M && n < N) ep(m, n, acc[4 * j + 2 * h + e]);
            }
}

template <int BN, class LA, class LB, class EP>
void tc_launch(cudaStream_t st, const LA &a, const LB &b, const EP &ep, int M, int N, long long K, WgradSplit sp,
               int a_mode, int b_mode) {
    static bool attr_set = false;                       // if this fails, so does the launch, and the caller reports it
    if (!attr_set)
        attr_set = cudaFuncSetAttribute(tc_gemm_kernel<BN, LA, LB, EP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        TcTile<BN>::SMEM) == cudaSuccess;
    const dim3 grid(wgrad_cdiv(M, TC_BM), wgrad_cdiv(N, BN), sp.splits);
    tc_gemm_kernel<BN, LA, LB, EP><<<grid, TC_T, TcTile<BN>::SMEM, st>>>(a, b, ep, M, N, K, sp.chunk, a_mode, b_mode);
}

// How tc_tile stages each operand of a product over K in chunks of sp.chunk
template <class LA, class LB>
void tc_modes(const LA &a, const LB &b, int N, long long K, WgradSplit sp, int &a_mode, int &b_mode) {
    const bool whole = K % TC_BK == 0 && sp.chunk % TC_BK == 0;     // no k-step leaves a row of 32
    a_mode = b_mode = BY_VALUE;
    if constexpr (has_seg<LA>)
        if (whole && a.seg_ok()) a_mode = ALONG_K;
    if constexpr (has_segT<LB>)
        if (whole && b.seg_ok()) b_mode = ALONG_K;
    // (never a WithOnes operand: its N = cols + 1 is odd, as cols is a multiple of 32)
    if constexpr (has_seg<LB>)
        if (N % 4 == 0 && b.seg_ok()) b_mode = ALONG_N;
}

// the tile width of a product with N columns
inline int tc_bn(int N) { return N <= 64 ? 64 : 128; }

// one launch: the (M x N) product over K, chunk z of sp on blockIdx.z (as `gemm`)
template <class LA, class LB, class EP>
void tc_gemm(cudaStream_t st, LA a, LB b, EP ep, int M, int N, long long K, WgradSplit sp) {
    int a_mode, b_mode;
    tc_modes(a, b, N, K, sp, a_mode, b_mode);
    if (tc_bn(N) == 64) tc_launch<64>(st, a, b, ep, M, N, K, sp, a_mode, b_mode);
    else tc_launch<128>(st, a, b, ep, M, N, K, sp, a_mode, b_mode);
}

}  // namespace

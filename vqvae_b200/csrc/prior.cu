// prior.cu -- the Gated PixelCNN prior (pixelcnn/models.py of the reference), fp32 on CUDA cores (sm_90a).
//
// Activations are NHWC rows.  A buffer holds `ring` rows of a (B, ring, W, C) grid and row r lives in slot r % ring:
// ring = H is a whole grid (the teacher-forced forward, and completion's vertical outputs), ring = 1 or gen_ring(H)
// the rows the incremental sampler keeps.  Every output element is one fmaf chain over its inputs in a fixed order
// (taps, then input channels), started from 0, then the bias: the value of an element does not depend on which
// positions share a block or on how many do.  The forward's kernels and the sampler's position step call the same device functions below, so the
// sampler's logits are bitwise the forward's logits on the grid it produced.
#include <cfloat>
#include <type_traits>

#include "pack.cuh"
#include "prior.cuh"

namespace {

// one block's positions: image, row, column and clamped label of each of its P slots (b < 0: slot unused).  Q: output
// channels per thread of the 2*dim-wide products, so the block holds dim <= Q*NT/2 channels; Q = 2 is dim <= MAXC.
template <int P, int Q = 2>
struct Smem {
    static constexpr int CAP = Q * NT / 2;
    float x[CAP * P];             // [ci][p]: one tap of the input, or the gated activations
    float pre[(Q * NT > HID ? Q * NT : HID) * P];  // [c][p]: pre-activations (2*dim) or the head's hidden layer (512)
    int b[P], r[P], c[P], lab[P];
};

// The block's Smem: static shared memory for the dim <= MAXC kernels, dynamic (above 48 KB, opted in by `wide_attr`)
// for the wide ones
template <int P, int Q>
__device__ __forceinline__ Smem<P, Q> &block_smem() {
    if constexpr (Q == 2) {
        __shared__ __align__(16) Smem<P, Q> s;
        return s;
    } else {
        extern __shared__ __align__(16) unsigned char wide_smem[];
        return *reinterpret_cast<Smem<P, Q> *>(wide_smem);
    }
}

template <int P>
__device__ __forceinline__ void load_vec(float (&v)[P], const float *s) {
    if constexpr (P % 4 == 0) {
#pragma unroll
        for (int q = 0; q < P / 4; ++q) {
            const float4 t = reinterpret_cast<const float4 *>(s)[q];
            v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
        }
    } else {
#pragma unroll
        for (int p = 0; p < P; ++p) v[p] = s[p];
    }
}

// acc[q][p] = fmaf-chain over k < n of x[k][p] * Wt[k][c0 + tid + q*NT]   (Wt: [n][Cout], output channel fastest)
template <int P, int Q>
__device__ __forceinline__ void mac(float (&acc)[Q][P], const float *xs, const float *__restrict__ Wt, int n,
                                    int Cout, int c0) {
    const int tid = threadIdx.x;
    for (int k = 0; k < n; ++k) {
        float v[P];
        load_vec<P>(v, xs + k * P);
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            const int c = c0 + tid + q * NT;
            if (c < Cout) {
                const float w = __ldg(Wt + (long long)k * Cout + c);
#pragma unroll
                for (int p = 0; p < P; ++p) acc[q][p] = fmaf(v[p], w, acc[q][p]);
            }
        }
    }
}

// x[ci][p] = in at (b, r + dy, c + dx) of slot p, 0 outside the grid or for an unused slot
template <int P, int Q>
__device__ __forceinline__ void load_tap(Smem<P, Q> &s, const Act &in, int dy, int dx, int H, int W) {
    const int C = in.C;
    for (int i = threadIdx.x; i < P * C; i += NT) {
        const int p = i / C, ci = i % C;
        const int rr = s.r[p] + dy, cc = s.c[p] + dx;
        float v = 0.f;
        if (s.b[p] >= 0 && rr >= 0 && rr < H && cc >= 0 && cc < W) v = in.at(s.b[p], rr, cc, W)[ci];
        s.x[ci * P + p] = v;
    }
}

// kept taps of a masked conv: vert_stack (kernel//2+1, kernel) and horiz_stack (1, kernel//2+1); mask A drops the
// last row / column (models.py:61-63).  Tap (t_r, t_c) reads offset (t_r - kernel//2, t_c - kernel//2).
__device__ __forceinline__ int vert_rows(const vqb_prior_layer_weights &w) { return w.kernel / 2 + 1 - (w.mask_a ? 1 : 0); }
__device__ __forceinline__ int horiz_cols(const vqb_prior_layer_weights &w) { return w.kernel / 2 + 1 - (w.mask_a ? 1 : 0); }

// Vertical stack of one layer at the P positions of the block (models.py:69-72, :77):
//   h_vert = vert_stack(x_v) ; out_v = gate(h_vert + emb[label]) ; vh = vert_to_horiz(h_vert) + emb[label]
// keep.p != nullptr (the training forward) also stores h_vert there for the backward.  vh.p == nullptr skips vh
// (completion's prefix rows, whose horizontal stacks never run).
template <int P, int Q>
__device__ void vert_positions(Smem<P, Q> &s, const vqb_prior_layer_weights &w, const Act &in, const Act &out_v,
                               const Act &vh, int H, int W, const Act &keep) {
    const int C = in.C, C2 = 2 * C, tid = threadIdx.x;
    float acc[Q][P];
#pragma unroll
    for (int q = 0; q < Q; ++q)
#pragma unroll
        for (int p = 0; p < P; ++p) acc[q][p] = 0.f;
    const int rows = vert_rows(w), k = w.kernel, half = k / 2;
    for (int tr = 0; tr < rows; ++tr)
        for (int tc = 0; tc < k; ++tc) {
            __syncthreads();
            load_tap(s, in, tr - half, tc - half, H, W);
            __syncthreads();
            mac<P, Q>(acc, s.x, w.vert_w + (long long)(tr * k + tc) * C * C2, C, C2, 0);
        }
#pragma unroll
    for (int q = 0; q < Q; ++q) {
        const int c = tid + q * NT;
        if (c < C2)
#pragma unroll
            for (int p = 0; p < P; ++p) {
                s.pre[c * P + p] = acc[q][p] + __ldg(w.vert_b + c);
                if (keep.p && s.b[p] >= 0) keep.at(s.b[p], s.r[p], s.c[p], W)[c] = s.pre[c * P + p];
            }
    }
    __syncthreads();
    for (int i = tid; i < P * C; i += NT) {
        const int p = i / C, c = i % C;
        if (s.b[p] < 0) continue;
        const float *e = w.class_emb + (long long)s.lab[p] * C2;
        out_v.at(s.b[p], s.r[p], s.c[p], W)[c] = gate(s.pre[c * P + p] + __ldg(e + c), s.pre[(c + C) * P + p] + __ldg(e + c + C));
    }
    if (!vh.p) return;
#pragma unroll
    for (int q = 0; q < Q; ++q)
#pragma unroll
        for (int p = 0; p < P; ++p) acc[q][p] = 0.f;
    mac<P, Q>(acc, s.pre, w.v2h_w, C2, C2, 0);
#pragma unroll
    for (int q = 0; q < Q; ++q) {
        const int c = tid + q * NT;
        if (c >= C2) continue;
#pragma unroll
        for (int p = 0; p < P; ++p)
            if (s.b[p] >= 0)
                vh.at(s.b[p], s.r[p], s.c[p], W)[c] =
                    (acc[q][p] + __ldg(w.v2h_b + c)) + __ldg(w.class_emb + (long long)s.lab[p] * C2 + c);
    }
}

// Horizontal stack of one layer at the P positions of the block (models.py:74-83):
//   out = gate(horiz_stack(x_h) + vh) ; out_h = horiz_resid(out) [+ x_h]
// The forward's per-layer kernel and the sampler's position step both run this.  keep.p != nullptr (the training
// forward) also stores the gate's pre-activation there.
template <int P, int Q>
__device__ void horiz_positions(Smem<P, Q> &s, const vqb_prior_layer_weights &w, const Act &in, const Act &vh,
                                const Act &out_h, int H, int W, const Act &keep) {
    const int C = in.C, C2 = 2 * C, tid = threadIdx.x;
    float acc[Q][P];
#pragma unroll
    for (int q = 0; q < Q; ++q)
#pragma unroll
        for (int p = 0; p < P; ++p) acc[q][p] = 0.f;
    const int cols = horiz_cols(w), half = w.kernel / 2;
    for (int tc = 0; tc < cols; ++tc) {
        __syncthreads();
        load_tap(s, in, 0, tc - half, H, W);
        __syncthreads();
        mac<P, Q>(acc, s.x, w.horiz_w + (long long)tc * C * C2, C, C2, 0);
    }
#pragma unroll
    for (int q = 0; q < Q; ++q) {
        const int c = tid + q * NT;
        if (c >= C2) continue;
#pragma unroll
        for (int p = 0; p < P; ++p) {
            s.pre[c * P + p] = s.b[p] >= 0 ? (acc[q][p] + __ldg(w.horiz_b + c)) + vh.at(s.b[p], s.r[p], s.c[p], W)[c] : 0.f;
            if (keep.p && s.b[p] >= 0) keep.at(s.b[p], s.r[p], s.c[p], W)[c] = s.pre[c * P + p];
        }
    }
    __syncthreads();
    for (int i = tid; i < P * C; i += NT) {
        const int p = i % P, c = i / P;
        s.x[c * P + p] = gate(s.pre[c * P + p], s.pre[(c + C) * P + p]);
    }
    __syncthreads();
    constexpr int R = (Q + 1) / 2;                  // output channels per thread of the dim-wide product
    float r[R][P];
#pragma unroll
    for (int q = 0; q < R; ++q)
#pragma unroll
        for (int p = 0; p < P; ++p) r[q][p] = 0.f;
    mac<P, R>(r, s.x, w.resid_w, C, C, 0);
#pragma unroll
    for (int q = 0; q < R; ++q) {
        const int c = tid + q * NT;
        if (c >= C) continue;
#pragma unroll
        for (int p = 0; p < P; ++p) {
            if (s.b[p] < 0) continue;
            float v = r[q][p] + __ldg(w.resid_b + c);
            if (w.residual) v = v + in.at(s.b[p], s.r[p], s.c[p], W)[c];
            out_h.at(s.b[p], s.r[p], s.c[p], W)[c] = v;
        }
    }
}

// Where head_positions sends logit k of slot p: sink(p, k, value), each (p, k) once, by thread k % NT, in increasing
// k per thread.  ToHbm stores it at out[p] + k * kstride (the forward's and the sampler's logits); Lse reduces it.
template <int P>
struct ToHbm {
    float *const *out;
    long long kstride;
    __device__ __forceinline__ void operator()(int p, int k, float v) const { out[p][k * kstride] = v; }
};

// The cross-entropy options' sum of w_k * l_k per slot over the logits this thread sees, in fp64 (nothing without)
template <int P, bool OPT>
struct WlSum {
    __device__ __forceinline__ void add(int, int, float) {}
};
template <int P>
struct WlSum<P, true> {
    double wl[P];
    CeOpt o;
    __device__ __forceinline__ void add(int p, int k, float v) { wl[p] += (double)v * o.wt(k); }
};

// A running log-sum-exp per slot over the logits this thread sees, and the logit of the slot's target code (the
// thread that sees it stores it in t[p], shared memory); OPT: also WlSum's sum
template <int P, bool OPT = false>
struct Lse : WlSum<P, OPT> {
    float m[P], s[P];
    int tgt[P];
    float *t;
    __device__ __forceinline__ void operator()(int p, int k, float v) {
        if (v > m[p]) {
            s[p] = s[p] * expf(m[p] - v) + 1.f;
            m[p] = v;
        } else {
            s[p] += expf(v - m[p]);
        }
        if (k == tgt[p]) t[p] = v;
        this->add(p, k, v);
    }
};

// lse_head_kernel's per-warp sums of w_k * l_k (OPT only)
template <int P>
__device__ __forceinline__ double (&wl_warps())[NT / 32][P] {
    __shared__ double w[NT / 32][P];
    return w;
}

// (m, s) <- the log-sum-exp pair of the union of (m, s) and (m2, s2); an empty pair (-INFINITY, 0) changes nothing
__device__ __forceinline__ void lse_merge(float &m, float &s, float m2, float s2) {
    const float M = fmaxf(m, m2);
    if (M == -INFINITY) return;
    s = s * expf(m - M) + s2 * expf(m2 - M);
    m = M;
}

// output_conv (models.py:107-111): logits = W2 . relu(W1 . x_h + b1) + b2 at the P positions of the block, each
// handed to `sink`.  keep.p != nullptr (the training forward) also stores the hidden layer there.
template <int P, int Q, class Sink>
__device__ void head_positions(Smem<P, Q> &s, const Net &n, const Act &in, Sink &sink, int H, int W, const Act &keep) {
    const int C = n.C, tid = threadIdx.x;
    __syncthreads();
    load_tap(s, in, 0, 0, H, W);
    __syncthreads();
    for (int c0 = 0; c0 < HID; c0 += NT) {
        float acc[1][P];
#pragma unroll
        for (int p = 0; p < P; ++p) acc[0][p] = 0.f;
        mac<P, 1>(acc, s.x, n.w1, C, HID, c0);
#pragma unroll
        for (int p = 0; p < P; ++p) {
            s.pre[(c0 + tid) * P + p] = fmaxf(acc[0][p] + __ldg(n.b1 + c0 + tid), 0.f);
            if (keep.p && s.b[p] >= 0) keep.at(s.b[p], s.r[p], s.c[p], W)[c0 + tid] = s.pre[(c0 + tid) * P + p];
        }
    }
    __syncthreads();
    for (int c0 = 0; c0 < n.K; c0 += NT) {
        float acc[1][P];
#pragma unroll
        for (int p = 0; p < P; ++p) acc[0][p] = 0.f;
        mac<P, 1>(acc, s.pre, n.w2, HID, n.K, c0);
        const int k = c0 + tid;
        if (k < n.K)
#pragma unroll
            for (int p = 0; p < P; ++p)
                if (s.b[p] >= 0) sink(p, k, acc[0][p] + __ldg(n.b2 + k));
    }
}

// Slots of a block over the positions [row0, row0 + nrows) x [col0, col0 + ncols) of all B images, position-major in
// (b, row, col).
template <int P, int Q>
__device__ void set_slots(Smem<P, Q> &s, int B, int row0, int nrows, int col0, int ncols, const long long *labels,
                          int NC) {
    if (threadIdx.x < P) {
        const int p = threadIdx.x;
        const long long g = (long long)blockIdx.x * P + p;
        const long long per = (long long)nrows * ncols;
        if (g < B * per) {
            s.b[p] = (int)(g / per);
            s.r[p] = row0 + (int)((g % per) / ncols);
            s.c[p] = col0 + (int)(g % ncols);
            s.lab[p] = clampi(labels[s.b[p]], NC);
        } else {
            s.b[p] = -1; s.r[p] = 0; s.c[p] = 0; s.lab[p] = 0;
        }
    }
    __syncthreads();
}

template <int P, int Q = 2>
__global__ void __launch_bounds__(NT) vert_kernel(vqb_prior_layer_weights w, Act in, Act out_v, Act vh,
                                                  const long long *labels, int NC, int B, int H, int W, int row0,
                                                  int nrows, Act keep) {
    Smem<P, Q> &s = block_smem<P, Q>();
    set_slots(s, B, row0, nrows, 0, W, labels, NC);
    vert_positions(s, w, in, out_v, vh, H, W, keep);
}

// over rows [row0, row0 + nrows) x columns [col0, col0 + ncols)
template <int P, int Q = 2>
__global__ void __launch_bounds__(NT) horiz_kernel(vqb_prior_layer_weights w, Act in, Act vh, Act out_h,
                                                   const long long *labels, int NC, int B, int H, int W, int row0,
                                                   int nrows, int col0, int ncols, Act keep) {
    Smem<P, Q> &s = block_smem<P, Q>();
    set_slots(s, B, row0, nrows, col0, ncols, labels, NC);
    horiz_positions(s, w, in, vh, out_h, H, W, keep);
}

// logits NCHW (B, K, H, W)
template <int P, int Q = 2>
__global__ void __launch_bounds__(NT) head_kernel(Net n, Act in, const long long *labels, int B, int H, int W,
                                                  float *logits, Act keep) {
    Smem<P, Q> &s = block_smem<P, Q>();
    __shared__ float *out[P];
    set_slots(s, B, 0, H, 0, W, labels, n.NC);
    if (threadIdx.x < P) {
        const int p = threadIdx.x;
        out[p] = s.b[p] >= 0 ? logits + (long long)s.b[p] * n.K * H * W + (long long)s.r[p] * W + s.c[p] : nullptr;
    }
    ToHbm<P> sink{out, (long long)H * W};
    head_positions(s, n, in, sink, H, W, keep);
}

// head_kernel's logits reduced on chip: each position's one partial (M, S, l_t) (prior.cuh) over all K codes, its
// target the clamped code codes[b, i, j].  A block owns all K logits of its P positions: each thread keeps a running
// log-sum-exp per slot over its codes k = tid (mod NT), then the warps' pairs are merged by xor butterflies and the
// eight warps' in warp order.
// keep.p != nullptr (the cross-entropy's training forward) also stores the hidden layer there, as head_kernel does.
// OPT (the cross-entropy's options): also each position's sum of w_k * l_k (o's weights) in fp64 into wl[g], merged
// over the lanes and the warps in the order of (M, S).
template <int P, int Q = 2, bool OPT = false>
__global__ void __launch_bounds__(NT) lse_head_kernel(Net n, Act in, const long long *labels, const long long *codes,
                                                      int B, int H, int W, float *part, Act keep, CeOpt o = {},
                                                      double *wl = nullptr) {
    Smem<P, Q> &s = block_smem<P, Q>();
    __shared__ float t[P], wm[NT / 32][P], wsum[NT / 32][P];
    set_slots(s, B, 0, H, 0, W, labels, n.NC);
    Lse<P, OPT> sink;
#pragma unroll
    for (int p = 0; p < P; ++p) {
        sink.m[p] = -INFINITY;
        sink.s[p] = 0.f;
        sink.tgt[p] = s.b[p] >= 0 ? clampi(codes[((long long)s.b[p] * H + s.r[p]) * W + s.c[p]], n.K) : -1;
        if constexpr (OPT) sink.wl[p] = 0.0;
    }
    if constexpr (OPT) sink.o = o;
    sink.t = t;
    head_positions(s, n, in, sink, H, W, keep);
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
#pragma unroll
    for (int p = 0; p < P; ++p) {
        float m = sink.m[p], sm = sink.s[p];
        for (int o = 16; o; o >>= 1) {
            const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, sm, o);
            lse_merge(m, sm, m2, s2);
        }
        if (lane == 0) {
            wm[warp][p] = m;
            wsum[warp][p] = sm;
        }
        if constexpr (OPT) {
            double a = sink.wl[p];
            for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
            if (lane == 0) wl_warps<P>()[warp][p] = a;
        }
    }
    __syncthreads();
    if (threadIdx.x < P) {
        const int p = threadIdx.x;
        if (s.b[p] < 0) return;
        float m = wm[0][p], sm = wsum[0][p];
        for (int w = 1; w < NT / 32; ++w) lse_merge(m, sm, wm[w][p], wsum[w][p]);
        const long long g = ((long long)s.b[p] * H + s.r[p]) * W + s.c[p];
        float *q = part + g * 3;
        q[0] = m;
        q[1] = sm;
        q[2] = t[p];
        if constexpr (OPT) {
            double a = wl_warps<P>()[0][p];
            for (int w = 1; w < NT / 32; ++w) a += wl_warps<P>()[w][p];
            wl[g] = a;
        }
    }
}

// The draw's knobs (vqb_prior_sampling, checked by the entry point) and its extra outputs.  Samp{} is generate's draw
// from the plain softmax.
struct Samp {
    float T = 1.f;                // temperature
    int top_k = 0;                // 0 or >= K: no top-k truncation
    float top_p = 1.f;            // >= 1: no nucleus truncation
    float *scratch = nullptr;     // the kept-set search's keys and probabilities: search_floats(1, K) per image
    float *log_prob = nullptr;    // (B) sum of log p_model(code) over the sampled steps, or nullptr
    float *log_c = nullptr;       // (B) the compensation of log_prob's Kahan sum
};

// floats of the draw's scratch for B images: per image, per lane of the draw's warp, ceil(K/32) keys and as many
// probabilities, interleaved by lane so that each warp access is one contiguous 128-byte line; then B floats of
// log_prob's compensation
long long search_floats(long long B, long long K) { return B * 64 * ((K + 31) / 32) + B; }

// order-preserving map from fp32 to uint32: a < b  <=>  fkey(a) < fkey(b) (-0 below +0)
__device__ __forceinline__ unsigned fkey(float z) {
    const unsigned v = __float_as_uint(z);
    return (v & 0x80000000u) ? ~v : (v | 0x80000000u);
}

// z = l / T in fp32, saturated to the finite range so that max(z) - z stays defined for tiny T; l itself at T = 1
__device__ __forceinline__ float tempered(float l, float T) {
    return T == 1.f ? l : fminf(fmaxf(l / T, -FLT_MAX), FLT_MAX);
}

// Warp sums (xor butterfly: every lane ends with the same value, since each pairwise fp32 add is commutative)
__device__ __forceinline__ float warp_sum(float v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// One sampling step at (i, j) for P images: every layer's horizontal stack, the head, the softmax and the inverse-CDF
// draw.  The code goes to codes[b, i, j] and its embedding to x0[b, i, j], which later steps and row passes read.
// `first`: the first sampled step of the call, which writes log_prob instead of adding to it.
// RAGGED: image b keeps its raster positions p < g_b = clamp_given(ragged[b], H*W) as given (`first` is not read).
// In a row it has given whole the step does nothing for it; at a given position of its first free row it runs only
// the horizontal stacks, which the row's later steps read; from p = g_b on it is the step above, first at p = g_b.
template <int P, int Q = 2, bool RAGGED = false>
__global__ void __launch_bounds__(NT) step_kernel(Net n, Act x0, Act xrow0, Act vh0, long long vh_stride,
                                                  long long x_stride, const long long *labels, const float *u, int B,
                                                  int H, int W, int i, int j, float *logits, long long logit_img,
                                                  long long *codes, Samp sp, bool first, const long long *ragged) {
    Smem<P, Q> &s = block_smem<P, Q>();
    __shared__ float *out[P];
    const long long HW = (long long)H * W, at = (long long)i * W + j;
    if (threadIdx.x < P) {
        const int p = threadIdx.x, b = blockIdx.x * P + p;
        s.b[p] = b < B ? b : -1;
        if constexpr (RAGGED)
            if (b < B && (long long)(i + 1) * W <= clamp_given(ragged[b], HW)) s.b[p] = -1;
        s.r[p] = i; s.c[p] = j;
        s.lab[p] = b < B ? clampi(labels[b], n.NC) : 0;
        out[p] = b < B ? logits + (long long)b * logit_img : nullptr;
    }
    __syncthreads();
    if constexpr (RAGGED) {
        bool live = false;
#pragma unroll
        for (int p = 0; p < P; ++p) live |= s.b[p] >= 0;
        if (!live) return;
    }
    for (int l = 0; l < n.L; ++l) {
        const Act in = l == 0 ? x0 : Act{xrow0.p + (l - 1) * x_stride, 1, n.C};
        const Act vh{vh0.p + l * vh_stride, 1, 2 * n.C};
        const Act o{xrow0.p + l * x_stride, 1, n.C};
        horiz_positions(s, n.layer[l], in, vh, o, H, W, Act{});
        __syncthreads();
    }
    if constexpr (RAGGED) {         // given positions: no head, no draw
        if (threadIdx.x < P && s.b[threadIdx.x] >= 0 && at < clamp_given(ragged[s.b[threadIdx.x]], HW))
            s.b[threadIdx.x] = -1;
        __syncthreads();
        bool live = false;
#pragma unroll
        for (int p = 0; p < P; ++p) live |= s.b[p] >= 0;
        if (!live) return;
    }
    ToHbm<P> sink{out, 1};
    head_positions(s, n, Act{xrow0.p + (n.L - 1) * x_stride, 1, n.C}, sink, H, W, Act{});
    __syncthreads();
    // softmax + inverse CDF, one warp per image: lane L owns logits [L*cs, L*cs + cs).  z = l / T; the kept set is
    // S = {k : fkey(z_k) >= t} (t = 0: every code); the CDF is the fp32 running sum of q_k = expf(z_k - max) / sum_S
    // over k in S, over the lanes' chunk sums scanned in lane order and then within the chunk.  With the default knobs
    // this is the plain softmax's arithmetic, bit for bit.
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int K = n.K;
    const bool by_k = sp.top_k > 0 && sp.top_k < K, by_p = sp.top_p < 1.f;
    for (int p = warp; p < P; p += NT / 32) {
        if (s.b[p] < 0) continue;
        const int b = s.b[p];
        const float *lg = out[p];
        const int cs = (K + 31) / 32, k0 = min(K, lane * cs), k1 = min(K, k0 + cs);
        float m = -INFINITY;
        for (int k = k0; k < k1; ++k) m = fmaxf(m, tempered(lg[k], sp.T));
        m = warp_max(m);
        float sum = 0.f;
        for (int k = k0; k < k1; ++k) sum += expf(tempered(lg[k], sp.T) - m);
        sum = warp_sum(sum);
        unsigned t = 0;
        float sum_s = sum;
        if (by_k || by_p) {
            // t = max(t_k, t_p), each the largest threshold whose kept set still has top_k codes / top_p of the
            // tempered softmax's mass, found bit by bit from the MSB: 32 sweeps over the cached keys and probabilities
            unsigned *key = reinterpret_cast<unsigned *>(sp.scratch + (long long)b * 64 * cs) + lane;
            float *prob = sp.scratch + (long long)b * 64 * cs + 32 * cs + lane;
            for (int k = k0; k < k1; ++k) {
                const float z = tempered(lg[k], sp.T);
                key[(k - k0) * 32] = fkey(z);
                prob[(k - k0) * 32] = expf(z - m) / sum;
            }
            unsigned t_k = 0, t_p = 0;
            for (int bit = 31; bit >= 0; --bit) {
                const unsigned ck = t_k | 1u << bit, cp = t_p | 1u << bit;
                int cnt = 0;
                float mass = 0.f;
                for (int q = 0; q < k1 - k0; ++q) {
                    const unsigned kq = key[q * 32];
                    if (by_k) cnt += kq >= ck;
                    if (by_p && kq >= cp) mass += prob[q * 32];
                }
                for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
                mass = warp_sum(mass);
                if (by_k && cnt >= sp.top_k) t_k = ck;
                if (by_p && mass >= sp.top_p) t_p = cp;
            }
            t = max(t_k, t_p);
            sum_s = 0.f;
            for (int k = k0; k < k1; ++k) {
                const float z = tempered(lg[k], sp.T);
                if (fkey(z) >= t) sum_s += expf(z - m);
            }
            sum_s = warp_sum(sum_s);
        }
        float part = 0.f;
        int last = -1;
        for (int k = k0; k < k1; ++k) {
            const float z = tempered(lg[k], sp.T);
            if (fkey(z) < t) continue;
            const float pk = expf(z - m) / sum_s;
            part += pk;
            if (pk > 0.f) last = k;
        }
        float incl = part;
        for (int o = 1; o < 32; o <<= 1) {
            const float t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        float cdf = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) cdf = 0.f;
        const float uu = u[((long long)b * H + i) * W + j];
        int hit = -1;
        for (int k = k0; k < k1; ++k) {
            const float z = tempered(lg[k], sp.T);
            if (fkey(z) < t) continue;
            cdf += expf(z - m) / sum_s;
            if (uu < cdf) { hit = k; break; }
        }
        const unsigned found = __ballot_sync(0xffffffffu, hit >= 0);
        int code;
        if (found) {
            code = __shfl_sync(0xffffffffu, hit, __ffs(found) - 1);
        } else {                    // u above the rounded total: the last kept code with non-zero probability
            for (int o = 16; o; o >>= 1) last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
            code = last < 0 ? K - 1 : last;
        }
        if (lane == 0) codes[((long long)b * H + i) * W + j] = code;
        if (sp.log_prob) {          // log p_model(code): the raw logits' softmax, the draw's max and sum when T = 1
            float ml = m, suml = sum;
            if (sp.T != 1.f) {
                ml = -INFINITY;
                for (int k = k0; k < k1; ++k) ml = fmaxf(ml, lg[k]);
                ml = warp_max(ml);
                suml = 0.f;
                for (int k = k0; k < k1; ++k) suml += expf(lg[k] - ml);
                suml = warp_sum(suml);
            }
            if (lane == 0) {        // compensated fp32 sum in raster order: 4096 near-equal terms stay accurate
                const float lp = (lg[code] - ml) - logf(suml);
                if constexpr (RAGGED) first = at == clamp_given(ragged[b], HW);
                if (first) {
                    sp.log_prob[b] = lp;
                    sp.log_c[b] = 0.f;
                } else {
                    const float acc = sp.log_prob[b], y = lp - sp.log_c[b], t = acc + y;
                    sp.log_c[b] = (t - acc) - y;
                    sp.log_prob[b] = t;
                }
            }
        }
        float *x = x0.at(b, i, j, W);
        for (int c = lane; c < n.C; c += 32) x[c] = __ldg(n.emb + (long long)code * n.C + c);
    }
}

// Completion's given prefix: codes[b, p] = given[b, p] as given and x0[b, p] = E[clamp(given[b, p])] (embed_kernel's
// clamp) for the raster positions p < n of every image; positions >= n are not read.  zero: nullptr, or the (B)
// log_prob of a call that samples nothing (n = HW), set to 0 here since no step writes it.
__global__ void given_kernel(const long long *__restrict__ given, const float *__restrict__ E, int B, long long HW,
                             long long n, int K, int C, float *__restrict__ x0, long long *__restrict__ codes,
                             float *__restrict__ zero) {
    const long long total = (long long)B * n * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long q = i / C, pos = q / n * HW + q % n;
        const int c = (int)(i % C);
        const long long code = given[pos];
        x0[pos * C + c] = __ldg(E + (long long)clampi(code, K) * C + c);
        if (c == 0) codes[pos] = code;
    }
    if (zero)
        for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (long long)gridDim.x * blockDim.x)
            zero[b] = 0.f;
}

// given_kernel with image b's own bound g_b = clamp_given(n_given[b], HW), over every position of the grid; zero:
// nullptr, or the (B) log_prob, set to 0 for the images with nothing to sample (g_b = HW).
__global__ void given_ragged_kernel(const long long *__restrict__ given, const long long *__restrict__ n_given,
                                    const float *__restrict__ E, int B, long long HW, int K, int C,
                                    float *__restrict__ x0, long long *__restrict__ codes, float *__restrict__ zero) {
    const long long total = (long long)B * HW * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long pos = i / C;
        if (pos % HW >= clamp_given(n_given[pos / HW], HW)) continue;
        const int c = (int)(i % C);
        const long long code = given[pos];
        x0[pos * C + c] = __ldg(E + (long long)clampi(code, K) * C + c);
        if (c == 0) codes[pos] = code;
    }
    if (zero)
        for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (long long)gridDim.x * blockDim.x)
            if (clamp_given(n_given[b], HW) == HW) zero[b] = 0.f;
}

// the kept-tap packing of pack_prior_at
__global__ void pack_kernel(const float *__restrict__ w, float *__restrict__ out, int Cout, int Cin, int kh, int kw,
                            int rows, int cols) {
    const long long total = (long long)rows * cols * Cin * Cout;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
        out[i] = pack_prior_at(w, i, Cout, Cin, kh, kw, cols);
}

__global__ void gate_kernel(const float *__restrict__ x, float *__restrict__ out, long long outer, int C,
                            long long inner) {
    const long long total = outer * C * inner;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long o = i / ((long long)C * inner), rest = i % ((long long)C * inner);
        const float *src = x + o * 2 * C * inner + rest;
        out[i] = gate(src[0], src[(long long)C * inner]);
    }
}

// Rows of each layer's vertical output the sampler keeps: a layer l >= 1 with kernel k reads rows i - k/2 .. i of
// layer l - 1's at row i.  The workspace does not see the kernels, so it holds the most any kernel reads; generate
// uses the rows its own net reads (2 for the reference's 3x3 layers).
int gen_ring(int H, int reach = VQB_PRIOR_MAX_KERNEL / 2 + 1) { return H < reach ? H : reach; }

// workspace regions, in floats
struct Ws {
    long long fwd_v, fwd_vh, fwd_x;               // forward: x0 | v[2] | vh | x[2]  (whole grids)
    long long gen_x0, gen_vh, gen_x, gen_lg, gen_v;  // sampler: x0 | vh[L] (1 row) | x[L] (1 row) | logits | v[L] (gen_ring)
    long long fwd_total, gen_total;
    long long comp_total;                         // completion: the sampler's regions with v[L] whole grids (ring = H)
};

Ws ws_layout(long long B, long long H, long long W, long long C, long long L, long long K) {
    Ws w;
    const long long grid = B * H * W * C;
    w.fwd_v = grid;
    w.fwd_vh = 3 * grid;
    w.fwd_x = 5 * grid;
    w.fwd_total = 7 * grid;
    w.gen_x0 = 0;
    w.gen_vh = grid;
    w.gen_x = w.gen_vh + L * B * W * 2 * C;
    w.gen_lg = w.gen_x + L * B * W * C;
    w.gen_v = w.gen_lg + B * K;                   // last: generate uses the first L * B * ring * W * C floats
    w.gen_total = w.gen_v + L * B * gen_ring((int)H) * W * C;
    w.comp_total = w.gen_v + L * grid;
    return w;
}

constexpr int PF = 8;             // positions per block of the whole-grid kernels and the row pass
constexpr int PS = 4;             // images per block of the sampling step
constexpr int PF_WIDE = 8;        // the same for dim > MAXC (DESIGN §8.4)
constexpr int PS_WIDE = 4;

unsigned blocks(long long positions, int P) { return (unsigned)((positions + P - 1) / P); }

// Output channels per thread of the 2*dim-wide products: 2 up to dim = MAXC (the original instantiations), else
// ceil(2*dim / NT), 3 .. 8
int q_of(int C) { return 2 * C <= 2 * NT ? 2 : (2 * C + NT - 1) / NT; }

// f(std::integral_constant<int, q_of(C)>{}): the per-position kernels' instantiation for dim C
template <int Q = 2, class F>
void by_q(int C, F &&f) {
    if constexpr (Q < 2 * MAXC_WIDE / NT) {
        if (q_of(C) != Q) return by_q<Q + 1>(C, f);
    }
    f(std::integral_constant<int, Q>{});
}

template <int Q> constexpr int pf() { return Q == 2 ? PF : PF_WIDE; }
template <int Q> constexpr int ps() { return Q == 2 ? PS : PS_WIDE; }

// Dynamic shared memory of kernel Kern, an instantiation on Smem<P, Q>: none for Q = 2; else sizeof(Smem<P, Q>),
// opted in once (above 48 KB, at most 227 KB per block).  If the opt-in fails, so does the launch, and the caller
// reports it.
template <auto Kern, int P, int Q>
size_t smem_of() {
    if constexpr (Q == 2) {
        return 0;
    } else {
        constexpr size_t bytes = sizeof(Smem<P, Q>);
        static_assert(bytes + 1024 <= 227 * 1024, "Smem<P, Q> exceeds the H100's shared memory per block");
        static bool attr_set = false;
        if (!attr_set)
            attr_set = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) == cudaSuccess;
        return bytes;
    }
}

// The per-position kernels' launches at dim = in.C's instantiation (vert_kernel's and horiz_kernel's over rows
// [row0, row0 + nrows) x columns [col0, col0 + ncols) of B images; the heads over every position)
void launch_vert(cudaStream_t s, const vqb_prior_layer_weights &w, const Act &in, const Act &out_v, const Act &vh,
                 const long long *lab, int NC, int B, int H, int W, int row0, int nrows, const Act &keep) {
    by_q(in.C, [&](auto q) {
        constexpr int Q = decltype(q)::value, P = pf<Q>();
        vert_kernel<P, Q><<<blocks((long long)B * nrows * W, P), NT, smem_of<vert_kernel<P, Q>, P, Q>(), s>>>(
            w, in, out_v, vh, lab, NC, B, H, W, row0, nrows, keep);
    });
}

void launch_horiz(cudaStream_t s, const vqb_prior_layer_weights &w, const Act &in, const Act &vh, const Act &out_h,
                  const long long *lab, int NC, int B, int H, int W, int row0, int nrows, int col0, int ncols,
                  const Act &keep) {
    by_q(in.C, [&](auto q) {
        constexpr int Q = decltype(q)::value, P = pf<Q>();
        horiz_kernel<P, Q><<<blocks((long long)B * nrows * ncols, P), NT, smem_of<horiz_kernel<P, Q>, P, Q>(), s>>>(
            w, in, vh, out_h, lab, NC, B, H, W, row0, nrows, col0, ncols, keep);
    });
}

void launch_head(cudaStream_t s, const Net &n, const Act &in, const long long *lab, int B, int H, int W, float *logits,
                 const Act &keep) {
    by_q(n.C, [&](auto q) {
        constexpr int Q = decltype(q)::value, P = pf<Q>();
        head_kernel<P, Q><<<blocks((long long)B * H * W, P), NT, smem_of<head_kernel<P, Q>, P, Q>(), s>>>(
            n, in, lab, B, H, W, logits, keep);
    });
}

template <bool OPT = false>
void launch_lse_head(cudaStream_t s, const Net &n, const Act &in, const long long *lab, const long long *codes, int B,
                     int H, int W, float *part, const Act &keep, const CeOpt &o = {}, double *wl = nullptr) {
    by_q(n.C, [&](auto q) {
        constexpr int Q = decltype(q)::value, P = pf<Q>();
        lse_head_kernel<P, Q, OPT><<<blocks((long long)B * H * W, P), NT,
                                     smem_of<lse_head_kernel<P, Q, OPT>, P, Q>(), s>>>(n, in, lab, codes, B, H, W, part,
                                                                                       keep, o, wl);
    });
}

// The sampler of generate and complete, from raster position n_given = i0*W + j0 on (generate: n_given = 0).  The
// positions before it are final and their embeddings are in x0.  When i0 > 0, every layer's vertical output is first
// computed for rows [0, i0) in one launch per layer, into whole-grid rings (ring = H: the completion workspace) that
// the later row passes read; those rows' vh and horizontal stacks have no reader and are not computed.  Then rows
// i0 .. H-1 as generate runs them: per row one vertical pass per layer, then one step per position.  In row i0 with
// j0 > 0, one horizontal launch per layer over columns [0, j0) first fills the one-row x[l] that the step at (i0, j0)
// reads.  Every value is the fmaf chain generate computes at that position, so the logits are bitwise generate's.
// Launches: L*[i0 > 0] + L*(H - i0) + L*[j0 > 0] + (H*W - n_given).  sp: the draw's knobs, the same for every step.
// ragged (with n_given = 0): the (B) per-image prefix lengths on the device, which the steps read (step_kernel's
// RAGGED instantiation); the schedule is generate's, H*(L + W) launches whatever their values.
void sample_from(const Net &n, const long long *lab, const float *u, int B, int H, int W, long long n_given,
                 const Samp &sp, long long *codes, float *step_logits, float *ws, cudaStream_t s,
                 const long long *ragged = nullptr) {
    const Ws wl = ws_layout(B, H, W, n.C, n.L, n.K);
    const int i0 = (int)(n_given / W), j0 = (int)(n_given % W);
    int reach = 1;
    for (int l = 1; l < n.L; ++l) reach = max(reach, n.layer[l].kernel / 2 + 1);
    const int ring = i0 > 0 ? H : gen_ring(H, reach);
    const long long v_stride = (long long)B * ring * W * n.C, vh_stride = (long long)B * W * 2 * n.C,
                    x_stride = (long long)B * W * n.C;
    const Act x0{ws + wl.gen_x0, H, n.C};
    const auto v = [&](int l) { return Act{ws + wl.gen_v + l * v_stride, ring, n.C}; };
    const auto vh = [&](int l) { return Act{ws + wl.gen_vh + l * vh_stride, 1, 2 * n.C}; };
    const auto x = [&](int l) { return Act{ws + wl.gen_x + l * x_stride, 1, n.C}; };
    unsigned long long launches = 0;
    if (i0 > 0) {
        for (int l = 0; l < n.L; ++l)
            launch_vert(s, n.layer[l], l == 0 ? x0 : v(l - 1), v(l), Act{}, lab, n.NC, B, H, W, 0, i0, Act{});
        launches += n.L;
    }
    for (int i = i0; i < H; ++i) {
        // row pass: every layer's vertical stack at row i (codes of rows < i are final)
        for (int l = 0; l < n.L; ++l)
            launch_vert(s, n.layer[l], l == 0 ? x0 : v(l - 1), v(l), vh(l), lab, n.NC, B, H, W, i, 1, Act{});
        launches += n.L;
        const int jstart = i == i0 ? j0 : 0;
        if (jstart > 0) {
            for (int l = 0; l < n.L; ++l)
                launch_horiz(s, n.layer[l], l == 0 ? x0 : x(l - 1), vh(l), x(l), lab, n.NC, B, H, W, i, 1, 0, jstart,
                             Act{});
            launches += n.L;
        }
        for (int j = jstart; j < W; ++j) {
            float *lg = step_logits ? step_logits + ((long long)i * W + j) * n.K : ws + wl.gen_lg;
            const long long img = step_logits ? (long long)H * W * n.K : n.K;
            const bool first = (long long)i * W + j == n_given;
            by_q(n.C, [&](auto q) {
                constexpr int Q = decltype(q)::value, P = ps<Q>();
                if (ragged)
                    step_kernel<P, Q, true><<<blocks(B, P), NT, smem_of<step_kernel<P, Q, true>, P, Q>(), s>>>(
                        n, x0, x(0), vh(0), vh_stride, x_stride, lab, u, B, H, W, i, j, lg, img, codes, sp, false,
                        ragged);
                else
                    step_kernel<P, Q><<<blocks(B, P), NT, smem_of<step_kernel<P, Q>, P, Q>(), s>>>(
                        n, x0, x(0), vh(0), vh_stride, x_stride, lab, u, B, H, W, i, j, lg, img, codes, sp, first,
                        nullptr);
            });
        }
        launches += W - jstart;
    }
    VQB_COUNT_LAUNCH(launches);
}

// generate's, complete's and sample's body after their argument checks: the given prefix (n_given > 0), then the
// sampler from n_given on.
void sample_call(const Net &n, const int64_t *labels, const float *u, const int64_t *given, long long n_given, int B,
                 int H, int W, const Samp &sp, int64_t *codes, float *step_logits, void *workspace, cudaStream_t s) {
    const long long HW = (long long)H * W;
    float *ws = static_cast<float *>(workspace);
    long long *out = reinterpret_cast<long long *>(codes);
    if (n_given > 0) {
        given_kernel<<<grid_for((long long)B * n_given * n.C), NT, 0, s>>>(
            reinterpret_cast<const long long *>(given), n.emb, B, HW, n_given, n.K, n.C,
            ws + ws_layout(B, H, W, n.C, n.L, n.K).gen_x0, out, n_given == HW ? sp.log_prob : nullptr);
        VQB_COUNT_LAUNCH(1);
    }
    if (n_given < HW)
        sample_from(n, reinterpret_cast<const long long *>(labels), u, B, H, W, n_given, sp, out, step_logits, ws, s);
}

// The ragged sampler's body after its argument checks: every image's given prefix in one launch, then generate's
// schedule with each step deciding per image.  1 + H*(L + W) launches.
void sample_ragged_call(const Net &n, const int64_t *labels, const float *u, const int64_t *given,
                        const int64_t *n_given, int B, int H, int W, const Samp &sp, int64_t *codes,
                        float *step_logits, void *workspace, cudaStream_t s) {
    const long long HW = (long long)H * W;
    float *ws = static_cast<float *>(workspace);
    long long *out = reinterpret_cast<long long *>(codes);
    const long long *ng = reinterpret_cast<const long long *>(n_given);
    given_ragged_kernel<<<grid_for((long long)B * HW * n.C), NT, 0, s>>>(
        reinterpret_cast<const long long *>(given), ng, n.emb, B, HW, n.K, n.C,
        ws + ws_layout(B, H, W, n.C, n.L, n.K).gen_x0, out, sp.log_prob);
    VQB_COUNT_LAUNCH(1);
    sample_from(n, reinterpret_cast<const long long *>(labels), u, B, H, W, 0, sp, out, step_logits, ws, s, ng);
}

// The draw's knobs of a sampling entry point (NULL: the defaults) into sp; false for a knob outside its range
bool knobs_from(const vqb_prior_sampling *sampling, int K, Samp &sp) {
    if (sampling) {
        sp.T = sampling->temperature;
        sp.top_k = sampling->top_k;
        sp.top_p = sampling->top_p;
    }
    return sp.T > 0.f && sp.T <= FLT_MAX && sp.top_k >= 0 && sp.top_k <= K && sp.top_p > 0.f && sp.top_p <= 1.f;
}

// Floats of the sampler's regions from raster position n_given: a prefix shorter than a row keeps generate's rings,
// a longer one every layer's vertical output as a whole grid.  The kept-set search's scratch follows them.
long long ring_floats(const Ws &w, long long W, long long n_given) { return n_given < W ? w.gen_total : w.comp_total; }

// bytes a sampler call from n_given needs: generate's workspace at least, so one buffer also serves the forward
size_t sampler_bytes(int B, int H, int W, int dim, int n_layers, int K, long long n_given, bool search) {
    const size_t base = vqb_prior_workspace_bytes(B, H, W, dim, n_layers, K);
    const long long f = ring_floats(ws_layout(B, H, W, dim, n_layers, K), W, n_given) + (search ? search_floats(B, K) : 0);
    return (size_t)f * sizeof(float) > base ? (size_t)f * sizeof(float) : base;
}

}  // namespace

extern "C" int vqb_prior_pack_f32(const float *w, float *packed, int Cout, int Cin, int kh, int kw, int rows, int cols,
                                  void *stream) {
    if (!w || !packed || Cout <= 0 || Cin <= 0 || kh <= 0 || kw <= 0 || rows < 0 || cols < 0 || rows > kh || cols > kw)
        return VQB_ERR_BAD_ARG;
    const long long total = (long long)rows * cols * Cin * Cout;
    if (total == 0) return 0;
    pack_kernel<<<grid_for(total), NT, 0, (cudaStream_t)stream>>>(w, packed, Cout, Cin, kh, kw, rows, cols);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" size_t vqb_prior_workspace_bytes(int B, int H, int W, int dim, int n_layers, int K) {
    if (B <= 0 || H <= 0 || W <= 0 || dim <= 0 || n_layers <= 0 || K <= 0) return 0;
    const Ws w = ws_layout(B, H, W, dim, n_layers, K);
    return (size_t)(w.fwd_total > w.gen_total ? w.fwd_total : w.gen_total) * sizeof(float);
}

extern "C" int vqb_prior_gate_f32(const float *x, float *out, int64_t outer, int C, int64_t inner, void *stream) {
    if (!x || !out || outer <= 0 || C <= 0 || inner <= 0) return VQB_ERR_BAD_ARG;
    gate_kernel<<<grid_for(outer * C * inner), NT, 0, (cudaStream_t)stream>>>(x, out, outer, C, inner);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" int vqb_prior_layer_f32(const vqb_prior_layer_weights *layer, const float *x_v, const float *x_h,
                                   const int64_t *labels, int B, int H, int W, int dim, int n_classes, float *out_v,
                                   float *out_h, float *vh, void *stream) {
    if (!layer || !x_v || !x_h || !labels || !out_v || !out_h || !vh || B <= 0 || H <= 0 || W <= 0 || dim <= 0 ||
        n_classes <= 0 || !layer_ok(*layer))
        return VQB_ERR_BAD_ARG;
    if (!dim_ok(dim)) return VQB_ERR_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    const long long *lab = reinterpret_cast<const long long *>(labels);
    Act in_v{const_cast<float *>(x_v), H, dim}, in_h{const_cast<float *>(x_h), H, dim};
    Act ov{out_v, H, dim}, oh{out_h, H, dim}, vha{vh, H, 2 * dim};
    launch_vert(s, *layer, in_v, ov, vha, lab, n_classes, B, H, W, 0, H, Act{});
    launch_horiz(s, *layer, in_h, vha, oh, lab, n_classes, B, H, W, 0, H, 0, W, Act{});
    VQB_COUNT_LAUNCH(2);
    return vqb_cuda_status(cudaGetLastError());
}

namespace {

// The teacher-forced forward up to the head, in the workspace's ping-pong grids: the embedding, then per layer the
// vertical and the horizontal stack over every position.  Returns x_h of the last layer.  1 + 2*L launches.
Act forward_layers(const Net &n, const long long *codes, const long long *lab, int B, int H, int W, float *ws,
                   cudaStream_t s) {
    const Ws wl = ws_layout(B, H, W, n.C, n.L, n.K);
    const long long npos = (long long)B * H * W, grid = npos * n.C;
    Act x0{ws, H, n.C}, vh{ws + wl.fwd_vh, H, 2 * n.C};
    Act v[2] = {{ws + wl.fwd_v, H, n.C}, {ws + wl.fwd_v + grid, H, n.C}};
    Act x[2] = {{ws + wl.fwd_x, H, n.C}, {ws + wl.fwd_x + grid, H, n.C}};
    embed_kernel<<<grid_for(grid), NT, 0, s>>>(codes, n.emb, npos, n.K, n.C, x0.p);
    for (int l = 0; l < n.L; ++l) {
        const Act vin = l == 0 ? x0 : v[(l - 1) & 1], xin = l == 0 ? x0 : x[(l - 1) & 1];
        launch_vert(s, n.layer[l], vin, v[l & 1], vh, lab, n.NC, B, H, W, 0, H, Act{});
        launch_horiz(s, n.layer[l], xin, vh, x[l & 1], lab, n.NC, B, H, W, 0, H, 0, W, Act{});
    }
    VQB_COUNT_LAUNCH(1 + 2 * n.L);
    return x[(n.L - 1) & 1];
}

// The training forward's walk up to the head: the same kernels as forward_layers, every activation into the Saved
// layout at sp (the three stores the backward needs switched on).  Returns x_h of the last layer.  1 + 2*L launches.
Act train_layers(const Net &n, const long long *codes, const long long *lab, int B, int H, int W, float *sp,
                 cudaStream_t s) {
    const long long npos = (long long)B * H * W;
    const Saved sv{npos, n.C, n.L};
    const Act vh{sp + sv.vh(), H, 2 * n.C};
    embed_kernel<<<grid_for(npos * n.C), NT, 0, s>>>(codes, n.emb, npos, n.K, n.C, sp + sv.xv(0));
    for (int l = 0; l < n.L; ++l) {
        launch_vert(s, n.layer[l], Act{sp + sv.xv(l), H, n.C}, Act{sp + sv.xv(l + 1), H, n.C}, vh, lab, n.NC, B, H,
                    W, 0, H, Act{sp + sv.hv(l), H, 2 * n.C});
        launch_horiz(s, n.layer[l], Act{sp + sv.xh(l), H, n.C}, vh, Act{sp + sv.xh(l + 1), H, n.C}, lab, n.NC, B, H,
                     W, 0, H, 0, W, Act{sp + sv.ph(l), H, 2 * n.C});
    }
    VQB_COUNT_LAUNCH(1 + 2 * n.L);
    return Act{sp + sv.xh(n.L), H, n.C};
}

}  // namespace

extern "C" int vqb_prior_forward_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B,
                                     int H, int W, float *logits, void *workspace, size_t workspace_bytes,
                                     void *stream) {
    Net n;
    const int st = net_from(net, n);
    if (st) return st;
    if (!codes || !labels || !logits || !workspace || B <= 0 || H <= 0 || W <= 0) return VQB_ERR_BAD_ARG;
    if (workspace_bytes < vqb_prior_workspace_bytes(B, H, W, n.C, n.L, n.K)) return VQB_ERR_WORKSPACE;
    cudaStream_t s = (cudaStream_t)stream;
    const long long *lab = reinterpret_cast<const long long *>(labels);
    const Act xL = forward_layers(n, reinterpret_cast<const long long *>(codes), lab, B, H, W,
                                  static_cast<float *>(workspace), s);
    launch_head(s, n, xL, lab, B, H, W, logits, Act{});
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" size_t vqb_prior_log_prob_workspace_bytes(int B, int H, int W, int dim, int n_layers, int K) {
    const size_t base = vqb_prior_workspace_bytes(B, H, W, dim, n_layers, K);
    if (!base) return 0;
    return base + (size_t)B * H * W * 3 * sizeof(float);
}

namespace {

// log_prob's launches after the checks: the forward's layer walk, then lse_head_kernel in place of head_kernel (the
// same logits, reduced on chip: one partial per position, after the forward's workspace) and the finish, which reads
// n_given or, with ragged != nullptr, image b's own ragged[b].  3 + 2*n_layers launches.
void log_prob_f32(const Net &n, const int64_t *codes, const int64_t *labels, int64_t n_given, const int64_t *ragged,
                  int B, int H, int W, float *log_prob, float *pos_log_prob, void *workspace, cudaStream_t s) {
    const long long *lab = reinterpret_cast<const long long *>(labels), *cd = reinterpret_cast<const long long *>(codes);
    float *ws = static_cast<float *>(workspace);
    float *part = ws + vqb_prior_workspace_bytes(B, H, W, n.C, n.L, n.K) / sizeof(float);
    const Act xL = forward_layers(n, cd, lab, B, H, W, ws, s);
    launch_lse_head(s, n, xL, lab, cd, B, H, W, part, Act{});
    if (ragged)
        log_prob_finish_kernel<true><<<B, NT, 0, s>>>(part, 1, (long long)H * W, 0, log_prob, pos_log_prob,
                                                      reinterpret_cast<const long long *>(ragged));
    else
        log_prob_finish_kernel<<<B, NT, 0, s>>>(part, 1, (long long)H * W, n_given, log_prob, pos_log_prob);
    VQB_COUNT_LAUNCH(2);
}

}  // namespace

extern "C" int vqb_prior_log_prob_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels,
                                      int64_t n_given, int B, int H, int W, float *log_prob, float *pos_log_prob,
                                      void *workspace, size_t workspace_bytes, void *stream) {
    Net n;
    const int st = log_prob_args(net, n, codes, labels, n_given, B, H, W, log_prob, pos_log_prob, workspace);
    if (st) return st;
    if (workspace_bytes < vqb_prior_log_prob_workspace_bytes(B, H, W, n.C, n.L, n.K)) return VQB_ERR_WORKSPACE;
    log_prob_f32(n, codes, labels, n_given, nullptr, B, H, W, log_prob, pos_log_prob, workspace, (cudaStream_t)stream);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" int vqb_prior_log_prob_ragged_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels,
                                             const int64_t *n_given, int B, int H, int W, float *log_prob,
                                             void *workspace, size_t workspace_bytes, void *stream) {
    Net n;
    const int st = log_prob_ragged_args(net, n, codes, labels, n_given, B, H, W, log_prob, workspace);
    if (st) return st;
    if (workspace_bytes < vqb_prior_log_prob_workspace_bytes(B, H, W, n.C, n.L, n.K)) return VQB_ERR_WORKSPACE;
    log_prob_f32(n, codes, labels, 0, n_given, B, H, W, log_prob, nullptr, workspace, (cudaStream_t)stream);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" int vqb_prior_generate_f32(const vqb_prior_net *net, const int64_t *labels, const float *u, int B, int H,
                                      int W, int64_t *codes, float *step_logits, void *workspace,
                                      size_t workspace_bytes, void *stream) {
    Net n;
    const int st = net_from(net, n);
    if (st) return st;
    if (!labels || !u || !codes || !workspace || B <= 0 || H <= 0 || W <= 0) return VQB_ERR_BAD_ARG;
    if (workspace_bytes < vqb_prior_workspace_bytes(B, H, W, n.C, n.L, n.K)) return VQB_ERR_WORKSPACE;
    // Layer 0 must read only codes before (i, j): mask B reads row i and column j, a residual adds x_h at (i, j).
    if (!n.layer[0].mask_a || n.layer[0].residual) return VQB_ERR_UNSUPPORTED;
    sample_call(n, labels, u, nullptr, 0, B, H, W, Samp{}, codes, step_logits, workspace, (cudaStream_t)stream);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" size_t vqb_prior_complete_workspace_bytes(int B, int H, int W, int dim, int n_layers, int K) {
    const size_t base = vqb_prior_workspace_bytes(B, H, W, dim, n_layers, K);
    if (!base) return 0;
    const size_t comp = (size_t)ws_layout(B, H, W, dim, n_layers, K).comp_total * sizeof(float);
    return comp > base ? comp : base;
}

extern "C" int vqb_prior_complete_f32(const vqb_prior_net *net, const int64_t *labels, const float *u,
                                      const int64_t *given, int64_t n_given, int B, int H, int W, int64_t *codes,
                                      float *step_logits, void *workspace, size_t workspace_bytes, void *stream) {
    Net n;
    const int st = net_from(net, n);
    if (st) return st;
    if (!labels || !u || !given || !codes || !workspace || B <= 0 || H <= 0 || W <= 0) return VQB_ERR_BAD_ARG;
    const long long HW = (long long)H * W;
    if (n_given < 0 || n_given > HW) return VQB_ERR_BAD_ARG;
    if (workspace_bytes < sampler_bytes(B, H, W, n.C, n.L, n.K, n_given, false)) return VQB_ERR_WORKSPACE;
    if (!n.layer[0].mask_a || n.layer[0].residual) return VQB_ERR_UNSUPPORTED;
    sample_call(n, labels, u, given, n_given, B, H, W, Samp{}, codes, step_logits, workspace, (cudaStream_t)stream);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" size_t vqb_prior_sample_workspace_bytes(int B, int H, int W, int dim, int n_layers, int K,
                                                   int64_t n_given) {
    if (!vqb_prior_workspace_bytes(B, H, W, dim, n_layers, K) || n_given < 0 || n_given > (long long)H * W) return 0;
    return sampler_bytes(B, H, W, dim, n_layers, K, n_given, true);
}

extern "C" int vqb_prior_sample_f32(const vqb_prior_net *net, const int64_t *labels, const float *u,
                                    const int64_t *given, int64_t n_given, int B, int H, int W,
                                    const vqb_prior_sampling *sampling, int64_t *codes, float *log_prob,
                                    float *step_logits, void *workspace, size_t workspace_bytes, void *stream) {
    Net n;
    const int st = net_from(net, n);
    if (st) return st;
    if (!labels || !u || !codes || !workspace || B <= 0 || H <= 0 || W <= 0) return VQB_ERR_BAD_ARG;
    if (n_given < 0 || n_given > (long long)H * W || (n_given > 0 && !given)) return VQB_ERR_BAD_ARG;
    Samp sp;
    if (!knobs_from(sampling, n.K, sp)) return VQB_ERR_BAD_ARG;
    if (workspace_bytes < vqb_prior_sample_workspace_bytes(B, H, W, n.C, n.L, n.K, n_given)) return VQB_ERR_WORKSPACE;
    if (!n.layer[0].mask_a || n.layer[0].residual) return VQB_ERR_UNSUPPORTED;
    sp.scratch = static_cast<float *>(workspace) + ring_floats(ws_layout(B, H, W, n.C, n.L, n.K), W, n_given);
    sp.log_prob = log_prob;
    sp.log_c = sp.scratch + search_floats(B, n.K) - B;
    sample_call(n, labels, u, given, n_given, B, H, W, sp, codes, step_logits, workspace, (cudaStream_t)stream);
    return vqb_cuda_status(cudaGetLastError());
}

// vqb_prior_sample_f32's checks with a device n_given; generate's rings and the search's scratch after them
extern "C" int vqb_prior_sample_ragged_f32(const vqb_prior_net *net, const int64_t *labels, const float *u,
                                           const int64_t *given, const int64_t *n_given, int B, int H, int W,
                                           const vqb_prior_sampling *sampling, int64_t *codes, float *log_prob,
                                           float *step_logits, void *workspace, size_t workspace_bytes,
                                           void *stream) {
    Net n;
    const int st = net_from(net, n);
    if (st) return st;
    if (!labels || !u || !given || !n_given || !codes || !workspace || B <= 0 || H <= 0 || W <= 0)
        return VQB_ERR_BAD_ARG;
    Samp sp;
    if (!knobs_from(sampling, n.K, sp)) return VQB_ERR_BAD_ARG;
    if (workspace_bytes < vqb_prior_sample_workspace_bytes(B, H, W, n.C, n.L, n.K, 0)) return VQB_ERR_WORKSPACE;
    if (!n.layer[0].mask_a || n.layer[0].residual) return VQB_ERR_UNSUPPORTED;
    sp.scratch = static_cast<float *>(workspace) + ring_floats(ws_layout(B, H, W, n.C, n.L, n.K), W, 0);
    sp.log_prob = log_prob;
    sp.log_c = sp.scratch + search_floats(B, n.K) - B;
    sample_ragged_call(n, labels, u, given, n_given, B, H, W, sp, codes, step_logits, workspace, (cudaStream_t)stream);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" size_t vqb_prior_train_saved_bytes(int B, int H, int W, int dim, int n_layers) {
    if (B <= 0 || H <= 0 || W <= 0 || dim <= 0 || n_layers <= 0) return 0;
    return (size_t)Saved{(long long)B * H * W, dim, n_layers}.total() * sizeof(float);
}

// The teacher-forced forward's kernels, writing every activation into `saved` (prior.cuh: Saved) instead of the
// ping-pong workspace, plus the three stores the backward needs: the same arithmetic, so bitwise the same logits.
extern "C" int vqb_prior_forward_train_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels,
                                           int B, int H, int W, float *logits, void *saved, size_t saved_bytes,
                                           void *stream) {
    Net n;
    const int st = net_from(net, n);
    if (st) return st;
    if (!codes || !labels || !logits || !saved || B <= 0 || H <= 0 || W <= 0) return VQB_ERR_BAD_ARG;
    if (saved_bytes < vqb_prior_train_saved_bytes(B, H, W, n.C, n.L)) return VQB_ERR_WORKSPACE;
    cudaStream_t s = (cudaStream_t)stream;
    const long long *lab = reinterpret_cast<const long long *>(labels);
    const long long npos = (long long)B * H * W;
    const Saved sv{npos, n.C, n.L};
    float *sp = static_cast<float *>(saved);
    train_layers(n, reinterpret_cast<const long long *>(codes), lab, B, H, W, sp, s);
    launch_head(s, n, Act{sp + sv.xh(n.L), H, n.C}, lab, B, H, W, logits, Act{sp + sv.hid(), H, HID});
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" size_t vqb_prior_ce_saved_bytes(int B, int H, int W, int dim, int n_layers) {
    return vqb_prior_ce_saved_bytes_ex(B, H, W, dim, n_layers, nullptr);
}

extern "C" size_t vqb_prior_ce_saved_bytes_ex(int B, int H, int W, int dim, int n_layers,
                                              const vqb_prior_ce_options *options) {
    if (B <= 0 || H <= 0 || W <= 0 || dim <= 0 || n_layers <= 0) return 0;
    return (size_t)ce_saved_floats(Saved{(long long)B * H * W, dim, n_layers}, options != nullptr) * sizeof(float);
}

extern "C" size_t vqb_prior_ce_workspace_bytes(int B, int H, int W, int dim, int n_layers, int K, int train) {
    const size_t base = vqb_prior_log_prob_workspace_bytes(B, H, W, dim, n_layers, K);
    if (!base) return 0;
    const size_t npos = (size_t)B * H * W;
    return (train ? 3 * npos * sizeof(float) : base) + npos * sizeof(float);
}

extern "C" size_t vqb_prior_ce_workspace_bytes_ex(int B, int H, int W, int dim, int n_layers, int K, int train,
                                                  const vqb_prior_ce_options *options) {
    const size_t base = vqb_prior_ce_workspace_bytes(B, H, W, dim, n_layers, K, train);
    return base && options ? ce_opt_ws_bytes(base, (long long)B * H * W, 1) : base;
}

namespace {

// log_prob's launches with the finish of the cross-entropy; with `saved`, train_layers in place of forward_layers and
// the hidden layer kept, so that `saved` is bitwise vqb_prior_forward_train_f32's.  Workspace: the forward's (saved
// NULL), then one partial per position, then the per-position losses of MEAN and SUM; with options, then
// ce_opt_ws_bytes's regions.
int ce_forward_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H, int W,
                   int reduction, const vqb_prior_ce_options *opt, float *loss, void *saved, size_t saved_bytes,
                   void *workspace, size_t workspace_bytes, void *stream) {
    Net n;
    int st = ce_args(net, n, codes, labels, B, H, W, reduction, loss, workspace);
    if (st) return st;
    CeOpt o{};
    if (opt && (st = ce_opt_args(opt, o))) return st;
    if (saved && saved_bytes < vqb_prior_ce_saved_bytes_ex(B, H, W, n.C, n.L, opt)) return VQB_ERR_WORKSPACE;
    if (workspace_bytes < vqb_prior_ce_workspace_bytes_ex(B, H, W, n.C, n.L, n.K, saved != nullptr, opt))
        return VQB_ERR_WORKSPACE;
    cudaStream_t s = (cudaStream_t)stream;
    const long long *lab = reinterpret_cast<const long long *>(labels), *cd = reinterpret_cast<const long long *>(codes);
    const long long npos = (long long)B * H * W;
    const Saved sv{npos, n.C, n.L};
    float *ws = static_cast<float *>(workspace), *sp = static_cast<float *>(saved);
    float *part = ws + (saved ? 0 : vqb_prior_workspace_bytes(B, H, W, n.C, n.L, n.K) / sizeof(float));
    Act xL, keep{};
    if (saved) {
        xL = train_layers(n, cd, lab, B, H, W, sp, s);
        keep = Act{sp + sv.hid(), H, HID};
    } else {
        xL = forward_layers(n, cd, lab, B, H, W, ws, s);
    }
    float *lse = saved ? sp + sv.total() : nullptr;
    if (opt) {
        double *wl = ce_opt_wl(workspace, vqb_prior_ce_workspace_bytes(B, H, W, n.C, n.L, n.K, saved != nullptr), npos);
        launch_lse_head<true>(s, n, xL, lab, cd, B, H, W, part, keep, o, wl);
        VQB_COUNT_LAUNCH(1 + ce_finish<true>(s, part, 1, npos, reduction, loss, lse, part + 3 * npos,
                                             CeX{o, cd, wl, nullptr, saved ? sp + ce_saved_floats(sv) : nullptr, n.K}));
    } else {
        launch_lse_head(s, n, xL, lab, cd, B, H, W, part, keep);
        VQB_COUNT_LAUNCH(1 + ce_finish(s, part, 1, npos, reduction, loss, lse, part + 3 * npos));
    }
    return vqb_cuda_status(cudaGetLastError());
}

}  // namespace

extern "C" int vqb_prior_ce_forward_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B,
                                        int H, int W, int reduction, float *loss, void *saved, size_t saved_bytes,
                                        void *workspace, size_t workspace_bytes, void *stream) {
    return ce_forward_f32(net, codes, labels, B, H, W, reduction, nullptr, loss, saved, saved_bytes, workspace,
                          workspace_bytes, stream);
}

extern "C" int vqb_prior_ce_forward_ex_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B,
                                           int H, int W, int reduction, const vqb_prior_ce_options *options,
                                           float *loss, void *saved, size_t saved_bytes, void *workspace,
                                           size_t workspace_bytes, void *stream) {
    return ce_forward_f32(net, codes, labels, B, H, W, reduction, options, loss, saved, saved_bytes, workspace,
                          workspace_bytes, stream);
}

extern "C" size_t vqb_prior_layer_train_saved_bytes(int B, int H, int W, int dim) {
    if (B <= 0 || H <= 0 || W <= 0 || dim <= 0) return 0;
    return (size_t)LayerSaved{(long long)B * H * W, dim}.total() * sizeof(float);
}

// vqb_prior_layer_f32's two launches with the vertical and horizontal stores of the net's training forward switched
// on: the same arithmetic, so bitwise the same outputs.
extern "C" int vqb_prior_layer_forward_train_f32(const vqb_prior_layer_weights *layer, const float *x_v,
                                                 const float *x_h, const int64_t *labels, int B, int H, int W, int dim,
                                                 int n_classes, float *out_v, float *out_h, float *vh, void *saved,
                                                 size_t saved_bytes, void *stream) {
    if (!layer || !x_v || !x_h || !labels || !out_v || !out_h || !vh || !saved || B <= 0 || H <= 0 || W <= 0 || dim <= 0 ||
        n_classes <= 0 || !layer_ok(*layer))
        return VQB_ERR_BAD_ARG;
    if (!dim_ok(dim)) return VQB_ERR_UNSUPPORTED;
    if (saved_bytes < vqb_prior_layer_train_saved_bytes(B, H, W, dim)) return VQB_ERR_WORKSPACE;
    cudaStream_t s = (cudaStream_t)stream;
    const long long *lab = reinterpret_cast<const long long *>(labels);
    const LayerSaved sv{(long long)B * H * W, dim};
    float *sp = static_cast<float *>(saved);
    Act in_v{const_cast<float *>(x_v), H, dim}, in_h{const_cast<float *>(x_h), H, dim};
    Act ov{out_v, H, dim}, oh{out_h, H, dim}, vha{vh, H, 2 * dim};
    launch_vert(s, *layer, in_v, ov, vha, lab, n_classes, B, H, W, 0, H, Act{sp + sv.hv(), H, 2 * dim});
    launch_horiz(s, *layer, in_h, vha, oh, lab, n_classes, B, H, W, 0, H, 0, W, Act{sp + sv.ph(), H, 2 * dim});
    VQB_COUNT_LAUNCH(2);
    return vqb_cuda_status(cudaGetLastError());
}

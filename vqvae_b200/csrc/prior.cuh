// prior.cuh -- what the Gated PixelCNN's per-position kernels (prior.cu) and its matrix products (prior_gemm.cu) share:
// shape limits, the NHWC activation view, the host-side weight table and its argument checks, and the gate.
#pragma once
#include "common.cuh"

namespace {

constexpr int NT = 256;           // threads of every prior kernel
constexpr int MAXC = 256;         // dim <= 256: the per-position kernels' original instantiations (prior.cu)
constexpr int MAXC_WIDE = 1024;   // dim <= 1024, dim % 32 == 0: every dim the prior accepts
constexpr int HID = 512;          // output_conv.0: dim -> 512 (models.py:109)
constexpr int MAXK = 8192;

struct Act {                      // one NHWC activation buffer, C channels, `ring` rows of W positions per image
    float *p;
    int ring, C;
    __device__ __forceinline__ float *at(int b, int r, int c, int W) const {
        return p + (((long long)b * ring + r % ring) * W + c) * C;
    }
};

struct Net {
    vqb_prior_layer_weights layer[VQB_PRIOR_MAX_LAYERS];
    const float *emb, *w1, *b1, *w2, *b2;
    int L, C, K, NC;
};

__device__ __forceinline__ float gate(float a, float g) {      // GatedActivation: tanh(x) * sigmoid(y)
    return tanhf(a) * (1.f / (1.f + expf(-g)));
}

__device__ __forceinline__ int clampi(long long v, int n) { return v < 0 ? 0 : (v >= n ? n - 1 : (int)v); }

// A per-image prefix length (the ragged entry points' n_given[b]) clamped to [0, HW], as codes and labels are clamped
__device__ __forceinline__ long long clamp_given(long long v, long long HW) { return v < 0 ? 0 : (v > HW ? HW : v); }

inline unsigned grid_for(long long total) {
    long long g = (total + NT - 1) / NT;
    return (unsigned)(g > 148LL * 32 ? 148LL * 32 : (g < 1 ? 1 : g));
}

// embedding (models.py:122): x0[n] = E[clamp(codes[n])]
__global__ void embed_kernel(const long long *__restrict__ codes, const float *__restrict__ E, long long N, int K,
                             int C, float *__restrict__ x0) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < N * C; i += (long long)gridDim.x * blockDim.x)
        x0[i] = __ldg(E + (long long)clampi(codes[i / C], K) * C + i % C);
}

inline bool layer_ok(const vqb_prior_layer_weights &w) {
    return w.vert_w && w.vert_b && w.v2h_w && w.v2h_b && w.horiz_w && w.horiz_b && w.resid_w && w.resid_b &&
           w.class_emb && w.kernel >= 1 && w.kernel <= VQB_PRIOR_MAX_KERNEL && (w.kernel & 1);
}

inline bool dim_ok(int C) { return C % 32 == 0 && C <= MAXC_WIDE; }

inline int net_from(const vqb_prior_net *net, Net &n) {
    if (!net || !net->layers || !net->embedding || !net->out1_w || !net->out1_b || !net->out2_w || !net->out2_b)
        return VQB_ERR_BAD_ARG;
    if (net->n_layers <= 0 || net->dim <= 0 || net->input_dim <= 0 || net->n_classes <= 0) return VQB_ERR_BAD_ARG;
    if (net->n_layers > VQB_PRIOR_MAX_LAYERS || !dim_ok(net->dim) || net->input_dim > MAXK) return VQB_ERR_UNSUPPORTED;
    for (int l = 0; l < net->n_layers; ++l) {
        if (!layer_ok(net->layers[l])) return VQB_ERR_BAD_ARG;
        n.layer[l] = net->layers[l];
    }
    n.emb = net->embedding; n.w1 = net->out1_w; n.b1 = net->out1_b; n.w2 = net->out2_w; n.b2 = net->out2_b;
    n.L = net->n_layers; n.C = net->dim; n.K = net->input_dim; n.NC = net->n_classes;
    return 0;
}

// ---- log_prob (vqb_prior_log_prob_*): what both precisions' heads hand to one finish launch ----------------------
// The head of either precision reduces each position's logits, N range by N range, to one partial (M, S, l_t):
// M the range's largest logit, S the sum of expf(l - M) over the range, l_t the logit of the position's clamped code
// (-INFINITY when the code lies outside the range).  Partials of position g (g = (b*H + i)*W + j) are
// part[(g*splits + z)*3 + {0, 1, 2}] for ranges z = 0 .. splits-1.

// lp = (l_t - M) - logf(S) with M = max_z M_z, S = sum over z in order of S_z * expf(M_z - M), l_t = max_z l_t_z.
// lse: nullptr, or where (M, logf(S)) go (the cross-entropy's backward reads softmax_k = expf((l_k - M) - logf(S)))
__device__ __forceinline__ float lp_of(const float *q, int splits, float *lse = nullptr) {
    float M = -INFINITY, lt = -INFINITY;
    for (int z = 0; z < splits; ++z) {
        M = fmaxf(M, q[3 * z]);
        lt = fmaxf(lt, q[3 * z + 2]);
    }
    float S = 0.f;
    for (int z = 0; z < splits; ++z) S += q[3 * z + 1] * expf(q[3 * z] - M);
    const float ls = logf(S);
    if (lse) {
        lse[0] = M;
        lse[1] = ls;
    }
    return (lt - M) - ls;
}

// One block per image: every position's lp into pos (if non-null), and into log_prob[b] (if non-null) the
// compensated fp32 sum of lp over the raster positions p >= n_given, in raster order, with the sampler's Kahan step
// (prior.cu: step_kernel), so 4096 near-equal terms stay accurate and the result does not depend on the launch.
// RAGGED: image b's own n_given is clamp_given(ragged[b], HW) (the scalar n_given is not read).
template <bool RAGGED = false>
__global__ void __launch_bounds__(NT) log_prob_finish_kernel(const float *__restrict__ part, int splits, long long HW,
                                                              long long n_given, float *__restrict__ log_prob,
                                                              float *__restrict__ pos,
                                                              const long long *__restrict__ ragged = nullptr) {
    __shared__ float lp[NT];
    const int b = blockIdx.x, tid = threadIdx.x;
    if constexpr (RAGGED) n_given = clamp_given(ragged[b], HW);
    float acc = 0.f, comp = 0.f;
    for (long long p0 = 0; p0 < HW; p0 += NT) {
        const long long p = p0 + tid;
        if (p < HW) {
            const float v = lp_of(part + ((long long)b * HW + p) * splits * 3, splits);
            lp[tid] = v;
            if (pos) pos[(long long)b * HW + p] = v;
        }
        __syncthreads();
        if (tid == 0 && log_prob) {
            const int n = (int)(HW - p0 < NT ? HW - p0 : NT);
            for (int q = 0; q < n; ++q) {
                if (p0 + q < n_given) continue;
                const float y = lp[q] - comp, t = acc + y;
                comp = (t - acc) - y;
                acc = t;
            }
        }
        __syncthreads();
    }
    if (tid == 0 && log_prob) log_prob[b] = acc;
}

// The C entry points' checks shared by both precisions, in their order; fills n.
inline int log_prob_args(const vqb_prior_net *net, Net &n, const int64_t *codes, const int64_t *labels,
                         int64_t n_given, int B, int H, int W, const float *log_prob, const float *pos,
                         const void *workspace) {
    const int st = net_from(net, n);
    if (st) return st;
    if (!codes || !labels || !workspace || (!log_prob && !pos) || B <= 0 || H <= 0 || W <= 0) return VQB_ERR_BAD_ARG;
    if (n_given < 0 || n_given > (long long)H * W) return VQB_ERR_BAD_ARG;
    return 0;
}

// The ragged entry points' checks (vqb_prior_log_prob_ragged_*): log_prob_args with log_prob required, then n_given
inline int log_prob_ragged_args(const vqb_prior_net *net, Net &n, const int64_t *codes, const int64_t *labels,
                                const int64_t *n_given, int B, int H, int W, const float *log_prob,
                                const void *workspace) {
    const int st = log_prob_args(net, n, codes, labels, 0, B, H, W, log_prob, nullptr, workspace);
    if (st) return st;
    return n_given ? 0 : VQB_ERR_BAD_ARG;
}

// ---- the cross-entropy (vqb_prior_ce_*): log_prob's head partials, then the loss ----------------------------------
// The options of the _ex entry points (vqb_prior_ce_options, checked by ce_opt_args).  A position is ignored iff its
// raw code equals `ignore` (has_ignore); its target is the clamped code y, its weight w_y (1 without a weight vector).
struct CeOpt {
    const float *w;               // K weights, or nullptr: all ones
    long long ignore;
    int has_ignore;
    float eps;                    // label smoothing
    __device__ __forceinline__ float wt(int k) const { return w ? __ldg(w + k) : 1.f; }
    __device__ __forceinline__ bool ignored(long long code) const { return has_ignore && code == ignore; }
};

// What the options' finish reads and writes besides the no-options finish's arguments
struct CeX {
    CeOpt o;
    const long long *codes;
    const double *wl;             // the heads' sum of w_k * l_k per partial (splits per position, in range order)
    float *wy;                    // MEAN: each position's w_y, 0 if ignored (the divisor's terms); else nullptr
    float *tail;                  // the saved options tail (ce_saved_floats): tail[0] = W, tail[1] = MEAN's 1 / divisor
    int K;
};

// Every position g's loss -lp (lp_of: bitwise -log_prob's term) into loss[g], and (M, logf(S)) into lse[2g], lse[2g+1]
// (lse == nullptr: not kept).  OPT: loss_p = (1 - eps) * w_y * (-lp) + (eps / K) * (W * lse - sum_k w_k l_k), 0 if
// ignored; W = sum_k w_k in fp64 (thread t adds k = t, t + NT, ... in turn, then a pairwise tree), in every block.  The
// smoothing term is fp64: W*logf(S) + (W*M - sum_k w_k l_k), so a common offset of the logits cancels exactly.
template <bool OPT = false>
__global__ void __launch_bounds__(NT) ce_finish_kernel(const float *__restrict__ part, int splits, long long npos,
                                                       float *__restrict__ loss, float *__restrict__ lse, CeX x = {}) {
    if constexpr (!OPT) {
        for (long long g = (long long)blockIdx.x * NT + threadIdx.x; g < npos; g += (long long)gridDim.x * NT)
            loss[g] = -lp_of(part + g * splits * 3, splits, lse ? lse + 2 * g : nullptr);
    } else {
        __shared__ double red[NT];
        double a = 0.0;
        for (int k = threadIdx.x; k < x.K; k += NT) a += x.o.wt(k);
        red[threadIdx.x] = a;
        __syncthreads();
        for (int h = NT / 2; h > 0; h >>= 1) {
            if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
            __syncthreads();
        }
        const double Wt = red[0];
        if (x.tail && blockIdx.x == 0 && threadIdx.x == 0) x.tail[0] = (float)Wt;
        for (long long g = (long long)blockIdx.x * NT + threadIdx.x; g < npos; g += (long long)gridDim.x * NT) {
            float ml[2];
            const float lp = lp_of(part + g * splits * 3, splits, ml);
            if (lse) {
                lse[2 * g] = ml[0];
                lse[2 * g + 1] = ml[1];
            }
            const long long c = x.codes[g];
            const bool ign = x.o.ignored(c);
            const float wy = ign ? 0.f : x.o.wt(clampi(c, x.K));
            float v = ign ? 0.f : (1.f - x.o.eps) * wy * -lp;
            if (x.o.eps != 0.f && !ign) {
                double wl = 0.0;
                for (int z = 0; z < splits; ++z) wl += x.wl[g * splits + z];
                v = (float)((double)v + (double)x.o.eps / x.K * (Wt * ml[1] + (Wt * ml[0] - wl)));
            }
            loss[g] = v;
            if (x.wy) x.wy[g] = wy;
        }
    }
}

// One block: *out = (sum of loss[0 .. npos)) / div, rounded to fp32 once.  The sum is fp64 in a fixed order: thread t
// adds positions t, t + CE_RT, t + 2*CE_RT, ... in turn, then the threads' sums meet in a pairwise tree.
// OPT with wy (MEAN): the divisor is the sum of wy in the same order (NaN if it is 0, as torch), and
// scale (if non-null) receives (float)(1.0 / divisor), the backward's factor.
constexpr int CE_RT = 1024;
template <bool OPT = false>
__global__ void __launch_bounds__(CE_RT) ce_total_kernel(const float *__restrict__ loss, long long npos, double div,
                                                         float *__restrict__ out, const float *__restrict__ wy = nullptr,
                                                         float *__restrict__ scale = nullptr) {
    __shared__ double s[OPT ? 2 : 1][CE_RT];
    const bool den = OPT && wy;
    double a = 0.0, d = 0.0;
    for (long long g = threadIdx.x; g < npos; g += CE_RT) {
        a += loss[g];
        if (den) d += wy[g];
    }
    s[0][threadIdx.x] = a;
    if constexpr (OPT) s[1][threadIdx.x] = d;
    __syncthreads();
    for (int h = CE_RT / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) {
            s[0][threadIdx.x] += s[0][threadIdx.x + h];
            if constexpr (OPT) s[1][threadIdx.x] += s[1][threadIdx.x + h];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        if (den) {
            const double q = s[OPT ? 1 : 0][0];
            *out = q == 0.0 ? NAN : (float)(s[0][0] / q);
            if (scale) *scale = (float)(1.0 / q);
        } else {
            *out = (float)(s[0][0] / div);
        }
    }
}

// The finish of both precisions' forwards: reduction "none" writes the per-position loss to out, "mean" and "sum" to
// `scratch` and then the scalar to out.  OPT: x's codes, options, wl and tail filled in; MEAN's w_y go to
// scratch + npos.  1 or 2 launches, returned.
template <bool OPT = false>
inline int ce_finish(cudaStream_t st, const float *part, int splits, long long npos, int reduction, float *out,
                     float *lse, float *scratch, CeX x = {}) {
    float *loss = reduction == VQB_PRIOR_CE_NONE ? out : scratch;
    if (OPT && reduction == VQB_PRIOR_CE_MEAN) x.wy = scratch + npos;
    ce_finish_kernel<OPT><<<grid_for(npos), NT, 0, st>>>(part, splits, npos, loss, lse, x);
    if (reduction == VQB_PRIOR_CE_NONE) return 1;
    ce_total_kernel<OPT><<<1, CE_RT, 0, st>>>(loss, npos, reduction == VQB_PRIOR_CE_MEAN ? (double)npos : 1.0, out,
                                              x.wy, x.tail ? x.tail + 1 : nullptr);
    return 2;
}

// The options' checks (after ce_args): has_ignore 0 or 1, label_smoothing in [0, 1] (NaN rejected); fills o
inline int ce_opt_args(const vqb_prior_ce_options *opt, CeOpt &o) {
    if (opt->has_ignore != 0 && opt->has_ignore != 1) return VQB_ERR_BAD_ARG;
    if (!(opt->label_smoothing >= 0.f && opt->label_smoothing <= 1.f)) return VQB_ERR_BAD_ARG;
    o = CeOpt{opt->weight, (long long)opt->ignore_index, opt->has_ignore, opt->label_smoothing};
    return 0;
}

// The options path's extra workspace after the no-options bytes `base` of npos positions and `splits` head ranges:
// MEAN's w_y (4*npos bytes, right after the per-position losses), then, 8-byte aligned, the heads' sums of w_k l_k
inline size_t ce_opt_ws_bytes(size_t base, long long npos, int splits) {
    return ((base + 4 * (size_t)npos + 7) & ~(size_t)7) + 8 * (size_t)npos * splits;
}
inline double *ce_opt_wl(void *ws, size_t base, long long npos) {
    return reinterpret_cast<double *>(static_cast<char *>(ws) + ((base + 4 * (size_t)npos + 7) & ~(size_t)7));
}

// The cross-entropy entry points' checks shared by both precisions and directions, in their order; fills n.
inline int ce_args(const vqb_prior_net *net, Net &n, const int64_t *codes, const int64_t *labels, int B, int H, int W,
                   int reduction, const float *loss, const void *workspace) {
    const int st = net_from(net, n);
    if (st) return st;
    if (!codes || !labels || !loss || !workspace || B <= 0 || H <= 0 || W <= 0) return VQB_ERR_BAD_ARG;
    if (reduction != VQB_PRIOR_CE_NONE && reduction != VQB_PRIOR_CE_MEAN && reduction != VQB_PRIOR_CE_SUM)
        return VQB_ERR_BAD_ARG;
    return 0;
}

// Activations the training forward keeps for the backward, in floats; N = B*H*W positions, all NHWC grids:
//   xv[l], l = 0..L   input of layer l's vertical stack (xv[0] the embedding, also x_h of layer 0); xv[L] unused
//   xh[l], l = 1..L   input of layer l's horizontal stack (xh[L] the head's input)
//   hv[l]  (2C)       vertical stack output h_vert, bias included, class embedding not
//   ph[l]  (2C)       horizontal gate pre-activation: horiz_stack(x_h) + bias + vert_to_horiz(h_vert) + bias + class
//   vh     (2C)       scratch between the vertical and the horizontal launch of a layer
//   hid    (512)      the head's hidden layer after the ReLU
struct Saved {
    long long N, C, L;
    long long xv(int l) const { return (long long)l * N * C; }
    long long xh(int l) const { return l == 0 ? 0 : (L + l) * N * C; }
    long long hv(int l) const { return (2 * L + 1) * N * C + 2LL * l * N * C; }
    long long ph(int l) const { return (4 * L + 1) * N * C + 2LL * l * N * C; }
    long long vh() const { return (6 * L + 1) * N * C; }
    long long hid() const { return (6 * L + 3) * N * C; }
    long long total() const { return hid() + N * HID; }
};

// The cross-entropy forward's `saved`: Saved, then each position's (M, logf(S)) at total() (ce_finish_kernel's lse);
// with options, then two floats: W = sum_k w_k and MEAN's 1 / sum of w_y (CeX::tail)
inline long long ce_saved_floats(const Saved &sv, bool opt = false) { return sv.total() + 2 * sv.N + (opt ? 2 : 0); }

// What one layer's training forward (vqb_prior_layer_forward_train_f32) keeps, in floats, NHWC (2C) grids: hv and
// ph as in Saved.
struct LayerSaved {
    long long N, C;
    long long hv() const { return 0; }
    long long ph() const { return 2 * N * C; }
    long long total() const { return 4 * N * C; }
};

}  // namespace

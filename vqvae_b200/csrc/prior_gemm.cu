// prior_gemm.cu -- the Gated PixelCNN prior (GatedPixelCNN.forward, pixelcnn/models.py:121-130) as matrix products
// (sm_90a): the backward in both precisions and the TF32 teacher-forced forward.
//
// Every gradient is a matrix product, run by the FFMA GEMM the conv weight gradients also use (ffma_gemm.cuh:
// `gemm_kernel`).  This file gives it the prior's operands as accessor structs: the activations the training forward
// saved (prior.cuh: Saved), NHWC grids read at a tap's shifted position (im2col on the fly), the forward's packed
// weights, a one-hot of codes or labels; and the epilogues that apply the gates' and the ReLU's derivatives.
//   dgrad: rows = positions, columns = input channels, reduction = kept taps x output channels
//   wgrad: rows = output channels, columns = taps x input channels (+ a column of ones: the bias), reduction =
//          positions, split into fixed chunks; the chunk partials are summed in chunk order by
//          `wgrad_reduce_kernel`, which also writes each gradient in its parameter's layout.
// Every output element is one fmaf chain in a fixed order and no float atomics are used, so the gradients are bitwise
// reproducible.  Weight gradients cover all kh*kw taps, mask A's included (the reference convolves with the full,
// zeroed weight, so autograd gives those taps a gradient); dgrad reads the taps the forward kept.
//
// The TF32 mode (vqb_prior_*_tf32) runs the same products on the wgmma GEMM of tc_gemm.cuh, which takes the same
// accessors and epilogues: the backward is this file's backward with `tc_gemm` in place of `gemm` (the one-hot sums of
// the class and code embeddings stay on the FFMA GEMM), and the forward is written below as four products per layer
// and two for the head, with the same Saved layout as the fp32 training forward.  log_prob in TF32 runs that forward
// up to the head's hidden layer and reduces the logits on chip (`tc_lse_kernel`).  The fp32 forward stays on prior.cu's
// per-position kernels: on the FFMA GEMM it is faster on large grids but slower on the reference's 8x8 default
// (DESIGN §8.1).
#include "prior.cuh"
#include "ffma_gemm.cuh"
#include "tc_gemm.cuh"

namespace {

struct Grid {                     // position n of a (B, H, W) grid
    int H, W;
    __device__ __forceinline__ void split(int n, int &b, int &r, int &c) const {
        b = n / (H * W);
        const int rem = n - b * H * W;
        r = rem / W;
        c = rem - r * W;
    }
};

// ---- the prior's operand accessors (ffma_gemm.cuh: Mat, MatT, WithOnes) -----------------------------------------
struct Nchw {                     // d_logits (B, K, H, W) as a (positions x K) matrix
    const float *p;
    int K, HW;
    static constexpr bool j_fast = false;
    __device__ __forceinline__ float operator()(int n, int k) const {
        const int b = n / HW;
        return __ldg(p + ((long long)b * K + k) * HW + (n - b * HW));
    }
};

struct NchwT {                    // the same as a (K x positions) matrix
    Nchw a;
    static constexpr bool j_fast = true;
    __device__ __forceinline__ float operator()(int k, int n) const { return a(n, k); }
};

// NHWC grid g (C channels) as (positions x taps*C): column j = tap*C + c reads channel c at row r + sgn*(tr - hr),
// column c + sgn*(tc - hc) of tap (tr, tc) = (tap / cols, tap % cols); 0 outside the grid.  sgn = +1 is the forward
// conv's im2col (wgrad), sgn = -1 the transposed conv (dgrad).
struct Tap {
    const float *g;
    int C, cols, hr, hc, sgn;
    Grid grid;
    static constexpr bool j_fast = true;
    __device__ __forceinline__ float operator()(int n, int j) const {
        const int tap = j / C, c = j - tap * C, tr = tap / cols, tc = tap - tr * cols;
        int b, r, col;
        grid.split(n, b, r, col);
        const int rr = r + sgn * (tr - hr), cc = col + sgn * (tc - hc);
        if (rr < 0 || rr >= grid.H || cc < 0 || cc >= grid.W) return 0.f;
        return __ldg(g + (((long long)b * grid.H + rr) * grid.W + cc) * C + c);
    }
    // tc_gemm.cuh: columns j0 .. j0 + 31 at position n, one position decode (nullptr: the tap is outside the grid).
    // C % 32 == 0 keeps a 32-wide k-step inside one tap.
    __device__ __forceinline__ const float *seg(int n, long long j0) const {
        const int j = (int)j0, tap = j / C, c = j - tap * C, tr = tap / cols, tc = tap - tr * cols;
        int b, r, col;
        grid.split(n, b, r, col);
        const int rr = r + sgn * (tr - hr), cc = col + sgn * (tc - hc);
        if (rr < 0 || rr >= grid.H || cc < 0 || cc >= grid.W) return nullptr;
        return g + (((long long)b * grid.H + rr) * grid.W + cc) * C + c;
    }
    bool seg_ok() const { return C % 32 == 0 && ((uintptr_t)g & 15) == 0; }
};

struct Gated {                    // gate(pre) of a saved (positions x 2C) pre-activation: the gated layer's output
    const float *pre;
    int C;
    static constexpr bool j_fast = true;
    __device__ __forceinline__ float operator()(int n, int c) const {
        const float *q = pre + (long long)n * 2 * C;
        return gate(__ldg(q + c), __ldg(q + c + C));
    }
};

// a forward packing [tap][ci][co] (vqb_prior_pack_f32) as the dgrad operand (tap*Cout + co) x ci
struct WPacked {
    const float *p;
    int Cin, Cout;
    static constexpr bool j_fast = false;
    __device__ __forceinline__ float operator()(int k, int ci) const {
        const int tap = k / Cout, co = k - tap * Cout;
        return __ldg(p + ((long long)tap * Cin + ci) * Cout + co);
    }
    // tc_gemm.cuh: rows k0 .. k0 + 31 of column ci, contiguous when Cout % 32 == 0
    __device__ __forceinline__ const float *segT(long long k0, int ci) const {
        const int k = (int)k0, tap = k / Cout, co = k - tap * Cout;
        return p + ((long long)tap * Cin + ci) * Cout + co;
    }
    bool seg_ok() const { return Cout % 32 == 0 && ((uintptr_t)p & 15) == 0; }
};

struct OneHot {                   // (m, n) -> 1 if the clamped index of position n is m: idx[n / per]
    const long long *idx;
    int per, count;
    static constexpr bool j_fast = true;
    __device__ __forceinline__ float operator()(int m, int n) const { return clampi(idx[n / per], count) == m ? 1.f : 0.f; }
};

// ---- epilogues: (m, n, value) -----------------------------------------------------------------------------------
struct Store {                    // out[m][n] = v (+ add[m][n])
    float *out;
    const float *add;
    int ld;
    __device__ __forceinline__ void operator()(int m, int n, float v) const {
        const long long i = (long long)m * ld + n;
        out[i] = add ? v + add[i] : v;
    }
};

struct ReluBack {                 // d_hidden = relu'(hidden) * v
    float *out;
    const float *hid;
    __device__ __forceinline__ void operator()(int m, int n, float v) const {
        const long long i = (long long)m * HID + n;
        out[i] = __ldg(hid + i) > 0.f ? v : 0.f;
    }
};

// d(tanh(a) * sigmoid(g)) by a and by g, times d
__device__ __forceinline__ void gate_back(float a, float g, float d, float &da, float &dg) {
    const float t = tanhf(a), s = 1.f / (1.f + expf(-g));
    da = d * (1.f - t * t) * s;
    dg = d * t * s * (1.f - s);
}

struct GateBack {                 // v = d out[m][c] of the horizontal gate -> d pre_h[m][c], d pre_h[m][c + C]
    float *dpre;
    const float *pre;
    int C;
    __device__ __forceinline__ void operator()(int m, int c, float v) const {
        const long long i = (long long)m * 2 * C + c;
        float da, dg;
        gate_back(__ldg(pre + i), __ldg(pre + i + C), v, da, dg);
        dpre[i] = da;
        dpre[i + C] = dg;
    }
};

// v = (W_v2h^T d pre_h)[m][c]: d h_vert = v + d pre_v, with d pre_v = gate'(h_vert + class) * d x_v of the next layer
// (gv == nullptr: the last layer, whose vertical output nothing reads).  Also writes cls = d pre_v + d pre_h, the
// per-position gradient of the class embedding, which enters both gates.
struct VertBack {
    float *dhv, *cls;
    const float *hv, *gv, *dph, *emb;
    const long long *labels;
    int C, HW, NC;
    __device__ __forceinline__ void operator()(int m, int c, float v) const {
        const long long i = (long long)m * 2 * C + c;
        float dpv = 0.f;
        if (gv) {
            const int c0 = c < C ? c : c - C;
            const float *e = emb + (long long)clampi(labels[m / HW], NC) * 2 * C;
            const long long i0 = (long long)m * 2 * C + c0;
            float da, dg;
            gate_back(__ldg(hv + i0) + __ldg(e + c0), __ldg(hv + i0 + C) + __ldg(e + c0 + C),
                      __ldg(gv + (long long)m * C + c0), da, dg);
            dpv = c < C ? da : dg;
        }
        dhv[i] = v + dpv;
        cls[i] = dpv + __ldg(dph + i);
    }
};

// Partial, added to what the earlier chunks of positions left there (first: the first chunk, which stores)
struct PartialAdd {
    float *part;
    long long M, cols;
    bool first;
    __device__ __forceinline__ void operator()(int m, int n, float v) const {
        float &o = part[(long long)blockIdx.z * M * cols + (long long)m * cols + n];
        o = first ? v : o + v;
    }
};

// What the options' CeGrad reads besides the no-options one's: the options, and the saved tail (W, MEAN's factor)
template <bool OPT>
struct CeGradX {};
template <>
struct CeGradX<true> {
    CeOpt o;
    const float *tail;
    bool mean;
};

// The cross-entropy's d_logits of row m of a chunk of positions starting at c0, from logit n without its bias:
// l = v + bias (bitwise the forward's logit), d = g * (expf((l - M) - logS) - [n = c]), into out[m][n] (ld K).
// g = d_loss[p * gstride] * scale; (M, logS) from lse[2p] (ce_finish_kernel); c the clamped code of position p.
// OPT: d = g * (q * c_p - (1 - e) * w_c * [n = c] - (e / K) * w_n), c_p = (1 - e) * w_c + (e / K) * W, evaluated as
// g * (a * (q - [n = c]) + b * (W * q - w_n)), a = (1 - e) * w_c, b = e / K, so that it is exactly 0 where the
// gradient is (K = 1) and unit weights, nothing ignored and e = 0 give the same bits; g = 0 at an ignored position,
// and MEAN's scale is tail[1].
template <bool OPT = false>
struct CeGrad : CeGradX<OPT> {
    float *out;
    const float *bias, *lse, *d_loss;
    const long long *codes;
    float scale;
    int K, gstride;
    long long c0;
    __device__ __forceinline__ void operator()(int m, int n, float v) const {
        const long long p = c0 + m;
        const float l = v + __ldg(bias + n);
        const float q = expf((l - __ldg(lse + 2 * p)) - __ldg(lse + 2 * p + 1));
        if constexpr (!OPT) {
            const float g = __ldg(d_loss + p * gstride) * scale;
            out[(long long)m * K + n] = g * (n == clampi(codes[p], K) ? q - 1.f : q);
        } else {
            const CeOpt &o = this->o;
            const long long c = codes[p];
            const int y = clampi(c, K);
            const float g = o.ignored(c) ? 0.f : __ldg(d_loss + p * gstride) * (this->mean ? __ldg(this->tail + 1) : scale);
            const float a = (1.f - o.eps) * o.wt(y), b = o.eps / K;
            out[(long long)m * K + n] = g * (a * (n == y ? q - 1.f : q) + b * (__ldg(this->tail) * q - o.wt(n)));
        }
    }
};

// ---- epilogues of the TF32 forward ------------------------------------------------------------------------------
struct BiasStore {                // out[m][n] = v + bias[n] (+ add[m][n])
    float *out;
    const float *bias, *add;
    int ld;
    __device__ __forceinline__ void operator()(int m, int n, float v) const {
        const long long i = (long long)m * ld + n;
        const float r = v + __ldg(bias + n);
        out[i] = add ? r + __ldg(add + i) : r;
    }
};

// v = (W_v2h h_vert)[m][n]: vh = v + bias + class (2C wide); for n < C also out_v = gate(h_vert + class)
struct VertOut {
    float *vh, *out_v;
    const float *hv, *bias, *emb;
    const long long *labels;
    int C, HW, NC;
    __device__ __forceinline__ void operator()(int m, int n, float v) const {
        const float *e = emb + (long long)clampi(labels[m / HW], NC) * 2 * C;
        vh[(long long)m * 2 * C + n] = (v + __ldg(bias + n)) + __ldg(e + n);
        if (n < C) {
            const float *h = hv + (long long)m * 2 * C;
            out_v[(long long)m * C + n] = gate(__ldg(h + n) + __ldg(e + n), __ldg(h + n + C) + __ldg(e + n + C));
        }
    }
};

struct ReluBias {                 // the head's hidden layer: out[m][n] = relu(v + bias[n])
    float *out;
    const float *bias;
    __device__ __forceinline__ void operator()(int m, int n, float v) const {
        out[(long long)m * HID + n] = fmaxf(v + __ldg(bias + n), 0.f);
    }
};

struct Logits {                   // logit n of position m into NCHW (B, K, H, W)
    float *out;
    const float *bias;
    int K, HW;
    __device__ __forceinline__ void operator()(int m, int n, float v) const {
        const int b = m / HW;
        out[((long long)b * K + n) * HW + (m - b * HW)] = v + __ldg(bias + n);
    }
};

// ---- host side ---------------------------------------------------------------------------------------------------
struct Ffma {                     // the arithmetic of a product: fp32 FFMA (ffma_gemm.cuh) or TF32 wgmma (tc_gemm.cuh)
    template <class LA, class LB, class EP>
    static void run(cudaStream_t st, LA a, LB b, EP ep, int M, int N, long long K, WgradSplit sp) {
        gemm(st, a, b, ep, M, N, K, sp);
    }
};

struct Tf32 {
    template <class LA, class LB, class EP>
    static void run(cudaStream_t st, LA a, LB b, EP ep, int M, int N, long long K, WgradSplit sp) {
        tc_gemm(st, a, b, ep, M, N, K, sp);
    }
};

// one product over all of K in one chunk (positions x channels): dgrad and the TF32 forward
template <class G, class LA, class LB, class EP>
void product(cudaStream_t st, LA a, LB b, EP ep, int M, int N, int K) {
    G::run(st, a, b, ep, M, N, K, WgradSplit{1, K});
}

// The split of a reduction over npos positions whose partials must not grow with npos: about two CTAs per SM over
// the gradient's tiles, never more chunks than that
WgradSplit bounded_split(int M, int N, long long npos) {
    const long long tiles = (long long)wgrad_cdiv(M, BM) * wgrad_cdiv(N, BN);
    long long s = wgrad_cdiv(2 * 132, tiles);
    s = s < wgrad_cdiv(npos, BK) ? s : wgrad_cdiv(npos, BK);
    const int chunk = wgrad_cdiv(wgrad_cdiv(npos, s), BK) * BK;
    return {wgrad_cdiv(npos, chunk), chunk};
}

// A wgrad job in the partial region: M x cols partials of a reduction over `npos` positions, at `off` floats.
struct WJob {
    int M, Cin, taps;
    bool bias;
    WgradSplit sp;
    long long off;
    int cols() const { return Cin * taps + (bias ? 1 : 0); }
    long long floats() const { return (long long)sp.splits * M * cols(); }
};

// The wgrad jobs of one phase, laid out one after the other.
struct Phase {
    WJob job[MAX_JOBS];
    int n = 0;
    long long floats = 0;
    WJob &add(int M, int Cin, int taps, bool bias, long long npos, bool bounded = false) {
        WJob &j = job[n++];
        j.M = M; j.Cin = Cin; j.taps = taps; j.bias = bias;
        j.sp = bounded ? bounded_split(M, j.cols(), npos) : wgrad_split(M, j.cols(), npos, BM, BN, BK);
        j.off = floats;
        floats += j.floats();
        return j;
    }
};

int vrows(const vqb_prior_layer_weights &w) { return w.kernel / 2 + 1; }     // vert_stack (k/2 + 1, k)
int hcols(const vqb_prior_layer_weights &w) { return w.kernel / 2 + 1; }     // horiz_stack (1, k/2 + 1)

// Positions per chunk of the cross-entropy's head backward (the d_logits buffer holds CE_CHUNK x K floats)
constexpr long long CE_CHUNK = 4096;
long long ce_rows(long long npos) { return npos < CE_CHUNK ? npos : CE_CHUNK; }

// The split of the cross-entropy's output_conv.2 gradient within one chunk of positions; its partials are added
// chunk after chunk (PartialAdd), so they do not grow with the positions either
WgradSplit ce_w2_split(const Net &n, long long npos) { return wgrad_split(n.K, HID + 1, ce_rows(npos), BM, BN, BK); }

// the wgrad jobs of the head (dW2, dW1; the cross-entropy's dW1 only), of layer l (resid, horiz, v2h, class, vert)
// and of the embedding (the cross-entropy's on bounded_split)
Phase head_phase(const Net &n, long long npos, bool ce = false) {
    Phase p;
    if (!ce) p.add(n.K, HID, 1, true, npos);
    p.add(HID, n.C, 1, true, npos);
    return p;
}

Phase layer_phase(const vqb_prior_layer_weights &w, int C, int NC, long long npos) {
    Phase p;
    p.add(C, C, 1, true, npos);
    p.add(2 * C, C, hcols(w), true, npos);
    p.add(2 * C, 2 * C, 1, true, npos);
    p.add(NC, 2 * C, 1, false, npos);
    p.add(2 * C, C, vrows(w) * w.kernel, true, npos);
    return p;
}

Phase emb_phase(const Net &n, long long npos, bool ce = false) {
    Phase p;
    p.add(n.K, n.C, 1, false, npos, ce);
    return p;
}

// workspace regions, in floats: d x_h (2 grids), d x_v (2 grids), the head's d_hidden or a layer's d pre_h, d h_vert
// and class gradient (union), then the wgrad partials of the largest phase; the cross-entropy's (ce) then adds one
// chunk of d_logits (dl, ce_rows x K) and the output_conv.2 partials (acc)
struct Bws {
    long long gh, gv, work, part, dl, acc, total;
};

Bws bws_layout(const Net &n, long long npos, bool ce = false) {
    Bws w;
    const long long grid = npos * n.C;
    w.gh = 0;
    w.gv = 2 * grid;
    w.work = 4 * grid;
    const long long head = npos * HID, layer = 6 * grid;
    w.part = w.work + (head > layer ? head : layer);
    long long part = head_phase(n, npos, ce).floats;
    const long long e = emb_phase(n, npos, ce).floats;
    part = part > e ? part : e;
    for (int l = 0; l < n.L; ++l) {
        const long long f = layer_phase(n.layer[l], n.C, n.NC, npos).floats;
        part = part > f ? part : f;
    }
    w.dl = w.part + part;
    w.acc = w.dl + (ce ? ce_rows(npos) * n.K : 0);
    w.total = w.acc + (ce ? (long long)ce_w2_split(n, npos).splits * n.K * (HID + 1) : 0);
    return w;
}

void reduce(cudaStream_t st, const Phase &p, float *part, float *const (&w)[MAX_JOBS], float *const (&b)[MAX_JOBS]) {
    RJobs jobs;
    long long most = 0;
    for (int i = 0; i < p.n; ++i) {
        const WJob &j = p.job[i];
        jobs.j[i] = RJob{part + j.off, w[i], b[i], j.M, j.Cin, j.taps, j.cols(), j.sp.splits};
        most = most > (long long)j.M * j.cols() ? most : (long long)j.M * j.cols();
    }
    wgrad_reduce(st, jobs, p.n, most);
}

// One layer's backward: 10 launches.  xv, xh: the layer's inputs; hv, ph: h_vert and the horizontal gate's
// pre-activation its training forward kept; ghi = d out_h, gvi = d out_v (nullptr: zero, as for the net's last
// layer) -> gho = d x_h, gvo = d x_v (+ fold, the net's layer 0: x_v and x_h are both the embedding) and the nine
// weight gradients of q.  work: 6 grids of scratch; part: the wgrad partials of layer_phase.
template <class G>
void layer_backward(cudaStream_t st, const vqb_prior_layer_weights &w, const vqb_prior_layer_grads &q, int C, int NC,
                    const long long *lab, Grid g, int npos, const float *xv, const float *xh, const float *hv,
                    const float *ph, const float *ghi, const float *gvi, float *gho, float *gvo, const float *fold,
                    float *work, float *part) {
    const int C2 = 2 * C, half = w.kernel / 2, vr = vrows(w) - (w.mask_a ? 1 : 0), hc = hcols(w) - (w.mask_a ? 1 : 0);
    const long long grid = (long long)npos * C;
    float *dph = work, *dhv = dph + 2 * grid, *cls = dhv + 2 * grid;
    const Phase p = layer_phase(w, C, NC, npos);
    // out_h = horiz_resid(gate(pre_h)) [+ x_h]: d pre_h, then d x_h = [d out_h +] horiz_stack^T * d pre_h
    product<G>(st, Mat{ghi, C}, WPacked{w.resid_w, C, C}, GateBack{dph, ph, C}, npos, C, C);
    G::run(st, MatT{ghi, C}, WithOnes<Gated>{Gated{ph, C}, C}, Partial{part + p.job[0].off, C, C + 1}, C, C + 1,
           npos, p.job[0].sp);
    product<G>(st, Tap{dph, C2, hc, 0, half, -1, g}, WPacked{w.horiz_w, C, C2},
               Store{gho, w.residual ? ghi : nullptr, C}, npos, C, hc * C2);
    G::run(st, MatT{dph, C2}, WithOnes<Tap>{Tap{xh, C, hcols(w), 0, half, 1, g}, hcols(w) * C},
           Partial{part + p.job[1].off, C2, p.job[1].cols()}, C2, p.job[1].cols(), npos, p.job[1].sp);
    G::run(st, MatT{dph, C2}, WithOnes<Mat>{Mat{hv, C2}, C2}, Partial{part + p.job[2].off, C2, C2 + 1}, C2, C2 + 1,
           npos, p.job[2].sp);
    // d h_vert = W_v2h^T d pre_h + gate'(h_vert + class) * d out_v; class gradient; d x_v = vert_stack^T * d h_vert
    product<G>(st, Mat{dph, C2}, WPacked{w.v2h_w, C2, C2},
               VertBack{dhv, cls, hv, gvi, dph, w.class_emb, lab, C, g.H * g.W, NC}, npos, C2, C2);
    gemm(st, OneHot{lab, g.H * g.W, NC}, Mat{cls, C2}, Partial{part + p.job[3].off, NC, C2}, NC, C2, npos,
         p.job[3].sp);
    G::run(st, MatT{dhv, C2}, WithOnes<Tap>{Tap{xv, C, w.kernel, half, half, 1, g}, vrows(w) * w.kernel * C},
           Partial{part + p.job[4].off, C2, p.job[4].cols()}, C2, p.job[4].cols(), npos, p.job[4].sp);
    product<G>(st, Tap{dhv, C2, w.kernel, half, half, -1, g}, WPacked{w.vert_w, C, C2}, Store{gvo, fold, C}, npos,
               C, vr * w.kernel * C2);
    reduce(st, p, part, {q.resid_w, q.horiz_w, q.v2h_w, q.class_emb, q.vert_w},
           {q.resid_b, q.horiz_b, q.v2h_b, nullptr, q.vert_b});
}

// GatedActivation's backward: d x (outer, 2C, inner) from x and d out (outer, C, inner); one thread per output element
__global__ void gate_backward_kernel(const float *__restrict__ x, const float *__restrict__ d_out,
                                     float *__restrict__ d_x, long long outer, int C, long long inner) {
    const long long total = outer * C * inner;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long o = i / ((long long)C * inner), rest = i % ((long long)C * inner);
        const long long a = o * 2 * C * inner + rest, b = a + (long long)C * inner;
        float da, dg;
        gate_back(__ldg(x + a), __ldg(x + b), __ldg(d_out + i), da, dg);
        d_x[a] = da;
        d_x[b] = dg;
    }
}

bool layer_grads_ok(const vqb_prior_layer_grads &q) {
    return q.vert_w && q.vert_b && q.v2h_w && q.v2h_b && q.horiz_w && q.horiz_b && q.resid_w && q.resid_b && q.class_emb;
}

bool grads_ok(const vqb_prior_grads *g, int L) {
    if (!g || !g->layers || g->n_layers != L || !g->embedding || !g->out1_w || !g->out1_b || !g->out2_w || !g->out2_b)
        return false;
    for (int l = 0; l < L; ++l)
        if (!layer_grads_ok(g->layers[l])) return false;
    return true;
}

// ---- the TF32 forward --------------------------------------------------------------------------------------------
// Workspace of the inference call (vqb_prior_forward_tf32), in floats, with Saved's accessors: x_v and x_h ping-pong
// between two grids each (layer 0 reads the embedding in grid 0 for both), one h_vert, pre_h and vh (2C), the hidden
// layer (512).
struct TcWs {
    long long N, C;
    long long xv(int l) const { return l == 0 ? 0 : (1 + ((l - 1) & 1)) * N * C; }
    long long xh(int l) const { return l == 0 ? 0 : (3 + ((l - 1) & 1)) * N * C; }
    long long hv(int) const { return 5 * N * C; }
    long long ph(int) const { return 7 * N * C; }
    long long vh() const { return 9 * N * C; }
    long long hid() const { return 11 * N * C; }
    long long total() const { return hid() + N * HID; }
};

// GatedPixelCNN.forward in TF32, every activation at lay's offsets from sp: the embedding gather, per layer
//   h_vert = vert_stack * x_v + b                      (kept taps)
//   vh = v2h(h_vert) + b + class, out_v = gate(h_vert + class)
//   pre_h = horiz_stack * x_h + b + vh                 (kept taps)
//   out_h = horiz_resid(gate(pre_h)) + b [+ x_h]       (the gate computed as the operand is staged)
// and the head's hidden layer hid = relu(W1 x_h + b1), left at lay.hid().  2 + 4*n_layers launches.
template <class Lay>
void forward_hid_tf32(cudaStream_t st, const Net &n, const long long *codes, const long long *lab, int B, int H, int W,
                      float *sp, const Lay &lay) {
    const int npos = B * H * W, C = n.C, C2 = 2 * C;
    const Grid g{H, W};
    embed_kernel<<<grid_for((long long)npos * C), NT, 0, st>>>(codes, n.emb, npos, n.K, C, sp + lay.xv(0));
    float *vh = sp + lay.vh();
    for (int l = 0; l < n.L; ++l) {
        const vqb_prior_layer_weights &w = n.layer[l];
        const int half = w.kernel / 2, vr = vrows(w) - (w.mask_a ? 1 : 0), hc = hcols(w) - (w.mask_a ? 1 : 0);
        const float *xv = sp + lay.xv(l), *xh = sp + lay.xh(l);
        float *hv = sp + lay.hv(l), *ph = sp + lay.ph(l);
        product<Tf32>(st, Tap{xv, C, w.kernel, half, half, 1, g}, Mat{w.vert_w, C2},
                      BiasStore{hv, w.vert_b, nullptr, C2}, npos, C2, vr * w.kernel * C);
        product<Tf32>(st, Mat{hv, C2}, Mat{w.v2h_w, C2},
                      VertOut{vh, sp + lay.xv(l + 1), hv, w.v2h_b, w.class_emb, lab, C, H * W, n.NC}, npos, C2, C2);
        product<Tf32>(st, Tap{xh, C, hcols(w), 0, half, 1, g}, Mat{w.horiz_w, C2}, BiasStore{ph, w.horiz_b, vh, C2},
                      npos, C2, hc * C);
        product<Tf32>(st, Gated{ph, C}, Mat{w.resid_w, C},
                      BiasStore{sp + lay.xh(l + 1), w.resid_b, w.residual ? xh : nullptr, C}, npos, C, C);
    }
    product<Tf32>(st, Mat{sp + lay.xh(n.L), C}, Mat{n.w1, HID}, ReluBias{sp + lay.hid(), n.b1}, npos, HID, C);
}

// GatedPixelCNN.forward in TF32: forward_hid_tf32, then logits = W2 hid + b2 (NCHW).  3 + 4*n_layers launches.
template <class Lay>
void forward_tf32(cudaStream_t st, const Net &n, const long long *codes, const long long *lab, int B, int H, int W,
                  float *logits, float *sp, const Lay &lay) {
    forward_hid_tf32(st, n, codes, lab, B, H, W, sp, lay);
    product<Tf32>(st, Mat{sp + lay.hid(), HID}, Mat{n.w2, n.K}, Logits{logits, n.b2, n.K, H * W}, B * H * W, n.K, HID);
}

// ---- log_prob in TF32 ----------------------------------------------------------------------------------------------
// The logits product of forward_tf32 with its epilogue replaced by a running log-sum-exp: CTA (x, y) takes the
// 128-position tile x and the N tiles [y*per, min((y+1)*per, tiles)) of the K codes, in order.  Each N tile is
// tc_tile's product (the forward's staging, k order and BN), plus the bias: bitwise the forward's logits.  A row's
// BN logits sit on the four lanes of a quad (wgmma's accumulator layout), so each row's tile max and sum of exp are
// quad shuffles; the running (m, s) of a row is rescaled to the new max tile by tile, and the logit at the row's
// clamped code is kept.  One partial (prior.cuh) per position and CTA column y; no logit goes to memory.
// OPT (the cross-entropy's options): also each row's sum of w_n * l_n (o's weights) in fp64, each lane's codes in
// order, then over the quad, into wl[row * splits + y].
template <int BN, class LA, class LB, bool OPT = false>
__global__ void __launch_bounds__(TC_T) tc_lse_kernel(LA a, LB b, const float *__restrict__ bias,
                                                      const long long *__restrict__ codes, int M, int N, int K,
                                                      int per, int a_mode, int b_mode, float *__restrict__ part,
                                                      CeOpt o = {}, double *__restrict__ wl = nullptr) {
    extern __shared__ unsigned char tc_smem[];
    const uint32_t base = (ptx::smem_u32(tc_smem) + 1023u) & ~1023u;
    const int tid = threadIdx.x, wgi = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const int m0 = blockIdx.x * TC_BM, splits = gridDim.y;
    const int t0 = blockIdx.y * per, t1 = min((N + BN - 1) / BN, t0 + per);
    const int row = m0 + wgi * 64 + warp * 16 + (lane >> 2);
    float m[2] = {-INFINITY, -INFINITY}, s[2] = {0.f, 0.f}, lt[2] = {-INFINITY, -INFINITY};
    double swl[2] = {0.0, 0.0};
    int tgt[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) tgt[h] = row + 8 * h < M ? clampi(codes[row + 8 * h], N) : -1;
    float acc[BN / 2];
    for (int t = t0; t < t1; ++t) {
        const int n0 = t * BN;
        __syncthreads();                                // the previous tile's last stage is read by both warpgroups
        tc_tile<BN>(acc, a, b, base, m0, M, n0, N, 0, K, a_mode, b_mode);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float mt = -INFINITY;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int n = n0 + 8 * j + 2 * (lane & 3) + e;
                    float &v = acc[4 * j + 2 * h + e];
                    if (n < N) {
                        v = v + __ldg(bias + n);
                        mt = fmaxf(mt, v);
                        if (n == tgt[h]) lt[h] = v;
                        if constexpr (OPT) swl[h] += (double)v * o.wt(n);
                    }
                }
            mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 1));
            mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 2));
            const float Mn = fmaxf(m[h], mt);
            float st = 0.f;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    if (n0 + 8 * j + 2 * (lane & 3) + e < N) st += expf(acc[4 * j + 2 * h + e] - Mn);
            st += __shfl_xor_sync(0xffffffffu, st, 1);
            st += __shfl_xor_sync(0xffffffffu, st, 2);
            s[h] = s[h] * expf(m[h] - Mn) + st;
            m[h] = Mn;
        }
    }
    // the target logit sits on one lane of the quad (or none, outside this CTA's N tiles)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        lt[h] = fmaxf(lt[h], __shfl_xor_sync(0xffffffffu, lt[h], 1));
        lt[h] = fmaxf(lt[h], __shfl_xor_sync(0xffffffffu, lt[h], 2));
        if constexpr (OPT) {
            swl[h] += __shfl_xor_sync(0xffffffffu, swl[h], 1);
            swl[h] += __shfl_xor_sync(0xffffffffu, swl[h], 2);
        }
        const int r = row + 8 * h;
        if ((lane & 3) == 0 && r < M) {
            float *q = part + ((long long)r * splits + blockIdx.y) * 3;
            q[0] = m[h];
            q[1] = s[h];
            q[2] = lt[h];
            if constexpr (OPT) wl[(long long)r * splits + blockIdx.y] = swl[h];
        }
    }
}

// N ranges of tc_lse_kernel over npos positions and K codes: enough CTAs for about two per SM of an H100 (132 SMs,
// a constant: the split, and with it the result's bits, depends on the shape only), at most one N tile per range.
// per: N tiles per range.
int lse_splits(long long npos, int K, int *per = nullptr) {
    const int tiles = wgrad_cdiv(K, tc_bn(K)), ptiles = wgrad_cdiv(npos, TC_BM);
    int splits = wgrad_cdiv(2 * 132, ptiles);
    splits = splits < 1 ? 1 : (splits > tiles ? tiles : splits);
    const int p = wgrad_cdiv(tiles, splits);
    if (per) *per = p;
    return wgrad_cdiv(tiles, p);                    // no empty range
}

template <int BN, bool OPT = false, class LA, class LB>
void tc_lse_launch(cudaStream_t st, const LA &a, const LB &b, const float *bias, const long long *codes, int M, int N,
                   int K, float *part, const CeOpt &o = {}, double *wl = nullptr) {
    static bool attr_set = false;                   // if this fails, so does the launch, and the caller reports it
    if (!attr_set)
        attr_set = cudaFuncSetAttribute(tc_lse_kernel<BN, LA, LB, OPT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        TcTile<BN>::SMEM) == cudaSuccess;
    int per;
    const int splits = lse_splits(M, N, &per);
    int a_mode, b_mode;
    tc_modes(a, b, N, K, WgradSplit{1, K}, a_mode, b_mode);
    tc_lse_kernel<BN, LA, LB, OPT><<<dim3(wgrad_cdiv(M, TC_BM), splits), TC_T, TcTile<BN>::SMEM, st>>>(
        a, b, bias, codes, M, N, K, per, a_mode, b_mode, part, o, wl);
}

}  // namespace

extern "C" size_t vqb_prior_workspace_bytes_tf32(int B, int H, int W, int dim, int n_layers, int K) {
    if (B <= 0 || H <= 0 || W <= 0 || dim <= 0 || n_layers <= 0 || K <= 0) return 0;
    return (size_t)TcWs{(long long)B * H * W, dim}.total() * sizeof(float);
}

extern "C" int vqb_prior_forward_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B,
                                      int H, int W, float *logits, void *workspace, size_t workspace_bytes,
                                      void *stream) {
    Net n;
    const int st = net_from(net, n);
    if (st) return st;
    if (!codes || !labels || !logits || !workspace || B <= 0 || H <= 0 || W <= 0) return VQB_ERR_BAD_ARG;
    if (workspace_bytes < vqb_prior_workspace_bytes_tf32(B, H, W, n.C, n.L, n.K)) return VQB_ERR_WORKSPACE;
    forward_tf32((cudaStream_t)stream, n, reinterpret_cast<const long long *>(codes),
                 reinterpret_cast<const long long *>(labels), B, H, W, logits, static_cast<float *>(workspace),
                 TcWs{(long long)B * H * W, n.C});
    VQB_COUNT_LAUNCH(3 + 4 * n.L);
    return vqb_cuda_status(cudaGetLastError());
}

// vqb_prior_forward_tf32's launches with every activation in the Saved layout of the fp32 training forward: the same
// products on the same values, so bitwise the same logits.
extern "C" int vqb_prior_forward_train_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels,
                                            int B, int H, int W, float *logits, void *saved, size_t saved_bytes,
                                            void *stream) {
    Net n;
    const int st = net_from(net, n);
    if (st) return st;
    if (!codes || !labels || !logits || !saved || B <= 0 || H <= 0 || W <= 0) return VQB_ERR_BAD_ARG;
    if (saved_bytes < vqb_prior_train_saved_bytes(B, H, W, n.C, n.L)) return VQB_ERR_WORKSPACE;
    forward_tf32((cudaStream_t)stream, n, reinterpret_cast<const long long *>(codes),
                 reinterpret_cast<const long long *>(labels), B, H, W, logits, static_cast<float *>(saved),
                 Saved{(long long)B * H * W, n.C, n.L});
    VQB_COUNT_LAUNCH(3 + 4 * n.L);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" size_t vqb_prior_log_prob_workspace_bytes_tf32(int B, int H, int W, int dim, int n_layers, int K) {
    const size_t base = vqb_prior_workspace_bytes_tf32(B, H, W, dim, n_layers, K);
    if (!base) return 0;
    const long long npos = (long long)B * H * W;
    return base + (size_t)npos * lse_splits(npos, K) * 3 * sizeof(float);
}

namespace {

// log_prob's launches after the checks: forward_tf32 up to hid (the same launches and values), then tc_lse_kernel in
// place of the logits product, and the finish, which reads n_given or, with ragged != nullptr, image b's own
// ragged[b].  4 + 4*n_layers launches.
void log_prob_tf32(const Net &n, const int64_t *codes, const int64_t *labels, int64_t n_given, const int64_t *ragged,
                   int B, int H, int W, float *log_prob, float *pos_log_prob, void *workspace, cudaStream_t s) {
    const long long *cd = reinterpret_cast<const long long *>(codes);
    const int npos = B * H * W;
    const TcWs lay{npos, n.C};
    float *sp = static_cast<float *>(workspace), *part = sp + lay.total();
    forward_hid_tf32(s, n, cd, reinterpret_cast<const long long *>(labels), B, H, W, sp, lay);
    const Mat a{sp + lay.hid(), HID}, b{n.w2, n.K};
    if (tc_bn(n.K) == 64) tc_lse_launch<64>(s, a, b, n.b2, cd, npos, n.K, HID, part);
    else tc_lse_launch<128>(s, a, b, n.b2, cd, npos, n.K, HID, part);
    if (ragged)
        log_prob_finish_kernel<true><<<B, NT, 0, s>>>(part, lse_splits(npos, n.K), (long long)H * W, 0, log_prob,
                                                      pos_log_prob, reinterpret_cast<const long long *>(ragged));
    else
        log_prob_finish_kernel<<<B, NT, 0, s>>>(part, lse_splits(npos, n.K), (long long)H * W, n_given, log_prob,
                                                pos_log_prob);
    VQB_COUNT_LAUNCH(4 + 4 * n.L);
}

}  // namespace

extern "C" int vqb_prior_log_prob_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels,
                                       int64_t n_given, int B, int H, int W, float *log_prob, float *pos_log_prob,
                                       void *workspace, size_t workspace_bytes, void *stream) {
    Net n;
    const int st = log_prob_args(net, n, codes, labels, n_given, B, H, W, log_prob, pos_log_prob, workspace);
    if (st) return st;
    if (workspace_bytes < vqb_prior_log_prob_workspace_bytes_tf32(B, H, W, n.C, n.L, n.K)) return VQB_ERR_WORKSPACE;
    log_prob_tf32(n, codes, labels, n_given, nullptr, B, H, W, log_prob, pos_log_prob, workspace, (cudaStream_t)stream);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" int vqb_prior_log_prob_ragged_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels,
                                              const int64_t *n_given, int B, int H, int W, float *log_prob,
                                              void *workspace, size_t workspace_bytes, void *stream) {
    Net n;
    const int st = log_prob_ragged_args(net, n, codes, labels, n_given, B, H, W, log_prob, workspace);
    if (st) return st;
    if (workspace_bytes < vqb_prior_log_prob_workspace_bytes_tf32(B, H, W, n.C, n.L, n.K)) return VQB_ERR_WORKSPACE;
    log_prob_tf32(n, codes, labels, 0, n_given, B, H, W, log_prob, nullptr, workspace, (cudaStream_t)stream);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" size_t vqb_prior_ce_workspace_bytes_tf32(int B, int H, int W, int dim, int n_layers, int K, int train) {
    const size_t base = vqb_prior_log_prob_workspace_bytes_tf32(B, H, W, dim, n_layers, K);
    if (!base) return 0;
    const long long npos = (long long)B * H * W;
    return (train ? (size_t)npos * lse_splits(npos, K) * 3 * sizeof(float) : base) + (size_t)npos * sizeof(float);
}

extern "C" size_t vqb_prior_ce_workspace_bytes_ex_tf32(int B, int H, int W, int dim, int n_layers, int K, int train,
                                                       const vqb_prior_ce_options *options) {
    const size_t base = vqb_prior_ce_workspace_bytes_tf32(B, H, W, dim, n_layers, K, train);
    const long long npos = (long long)B * H * W;
    return base && options ? ce_opt_ws_bytes(base, npos, lse_splits(npos, K)) : base;
}

namespace {

// vqb_prior_log_prob_tf32's launches with the finish of the cross-entropy; with `saved`, every activation in the Saved
// layout (forward_train_tf32's walk up to the hidden layer, so `saved` is bitwise its).  Workspace: the inference
// forward's (saved NULL), then the head's partials, then the per-position losses of MEAN and SUM; with options, then
// ce_opt_ws_bytes's regions.
int ce_forward_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H, int W,
                    int reduction, const vqb_prior_ce_options *opt, float *loss, void *saved, size_t saved_bytes,
                    void *workspace, size_t workspace_bytes, void *stream) {
    Net n;
    int st = ce_args(net, n, codes, labels, B, H, W, reduction, loss, workspace);
    if (st) return st;
    CeOpt o{};
    if (opt && (st = ce_opt_args(opt, o))) return st;
    if (saved && saved_bytes < vqb_prior_ce_saved_bytes_ex(B, H, W, n.C, n.L, opt)) return VQB_ERR_WORKSPACE;
    if (workspace_bytes < vqb_prior_ce_workspace_bytes_ex_tf32(B, H, W, n.C, n.L, n.K, saved != nullptr, opt))
        return VQB_ERR_WORKSPACE;
    cudaStream_t s = (cudaStream_t)stream;
    const long long *cd = reinterpret_cast<const long long *>(codes), *lab = reinterpret_cast<const long long *>(labels);
    const int npos = B * H * W;
    float *ws = static_cast<float *>(workspace), *sp = static_cast<float *>(saved), *part, *hid;
    if (saved) {
        const Saved lay{npos, n.C, n.L};
        forward_hid_tf32(s, n, cd, lab, B, H, W, sp, lay);
        hid = sp + lay.hid();
        part = ws;
    } else {
        const TcWs lay{npos, n.C};
        forward_hid_tf32(s, n, cd, lab, B, H, W, ws, lay);
        hid = ws + lay.hid();
        part = ws + lay.total();
    }
    const Mat a{hid, HID}, b{n.w2, n.K};
    const int splits = lse_splits(npos, n.K);
    const Saved sv{npos, n.C, n.L};
    float *lse = saved ? sp + sv.total() : nullptr, *scratch = part + (long long)npos * splits * 3;
    if (opt) {
        double *wl = ce_opt_wl(workspace, vqb_prior_ce_workspace_bytes_tf32(B, H, W, n.C, n.L, n.K, saved != nullptr),
                               npos);
        if (tc_bn(n.K) == 64) tc_lse_launch<64, true>(s, a, b, n.b2, cd, npos, n.K, HID, part, o, wl);
        else tc_lse_launch<128, true>(s, a, b, n.b2, cd, npos, n.K, HID, part, o, wl);
        VQB_COUNT_LAUNCH(3 + 4 * n.L + ce_finish<true>(s, part, splits, npos, reduction, loss, lse, scratch,
                                                       CeX{o, cd, wl, nullptr, saved ? sp + ce_saved_floats(sv) : nullptr,
                                                           n.K}));
    } else {
        if (tc_bn(n.K) == 64) tc_lse_launch<64>(s, a, b, n.b2, cd, npos, n.K, HID, part);
        else tc_lse_launch<128>(s, a, b, n.b2, cd, npos, n.K, HID, part);
        VQB_COUNT_LAUNCH(3 + 4 * n.L + ce_finish(s, part, splits, npos, reduction, loss, lse, scratch));
    }
    return vqb_cuda_status(cudaGetLastError());
}

}  // namespace

extern "C" int vqb_prior_ce_forward_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B,
                                         int H, int W, int reduction, float *loss, void *saved, size_t saved_bytes,
                                         void *workspace, size_t workspace_bytes, void *stream) {
    return ce_forward_tf32(net, codes, labels, B, H, W, reduction, nullptr, loss, saved, saved_bytes, workspace,
                           workspace_bytes, stream);
}

extern "C" int vqb_prior_ce_forward_ex_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels,
                                            int B, int H, int W, int reduction, const vqb_prior_ce_options *options,
                                            float *loss, void *saved, size_t saved_bytes, void *workspace,
                                            size_t workspace_bytes, void *stream) {
    return ce_forward_tf32(net, codes, labels, B, H, W, reduction, options, loss, saved, saved_bytes, workspace,
                           workspace_bytes, stream);
}

extern "C" size_t vqb_prior_backward_workspace_bytes(const vqb_prior_net *net, int B, int H, int W) {
    Net n;
    if (net_from(net, n) || B <= 0 || H <= 0 || W <= 0) return 0;
    return (size_t)bws_layout(n, (long long)B * H * W).total * sizeof(float);
}

namespace {

// The layers, last to first, from d x_h of the last layer in gh[0] (wl's regions), then the embedding (ce: on the
// cross-entropy's bounded split).  Returns the launches: 10*L + 2.
template <class G>
unsigned long long body_backward(cudaStream_t st, const Net &n, const long long *codes, const long long *lab, Grid g,
                                 int npos, const float *sp, const vqb_prior_grads *grads, float *ws, const Bws &wl,
                                 bool ce) {
    const int C = n.C;
    const long long grid = (long long)npos * C;
    const Saved sv{npos, C, n.L};
    float *gh[2] = {ws + wl.gh, ws + wl.gh + grid}, *gv[2] = {ws + wl.gv, ws + wl.gv + grid};
    float *part = ws + wl.part;
    // gh[cur] = d x_h^{l+1}, gv[cur] = d x_v^{l+1} (none for the last layer)
    int cur = 0;
    for (int l = n.L - 1; l >= 0; --l) {
        float *gho = gh[cur ^ 1];
        // layer 0: x_v and x_h are both the embedding, so d x_v^0 + d x_h^0 is its gradient per position
        layer_backward<G>(st, n.layer[l], grads->layers[l], C, n.NC, lab, g, npos, sp + sv.xv(l), sp + sv.xh(l),
                          sp + sv.hv(l), sp + sv.ph(l), gh[cur], l == n.L - 1 ? nullptr : gv[cur], gho, gv[cur ^ 1],
                          l == 0 ? gho : nullptr, ws + wl.work, part);
        cur ^= 1;
    }
    // embedding: the per-position gradient summed by (clamped) code
    const Phase p = emb_phase(n, npos, ce);
    gemm(st, OneHot{codes, 1, n.K}, Mat{gv[cur], C}, Partial{part + p.job[0].off, n.K, C}, n.K, C, npos, p.job[0].sp);
    reduce(st, p, part, {grads->embedding}, {nullptr});
    return 10ULL * n.L + 2;
}

// vqb_prior_backward_f32 (G = Ffma) and vqb_prior_backward_tf32 (G = Tf32): the same products, launches and workspace
template <class G>
int net_backward(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H, int W,
                 const float *d_logits, const void *saved, const vqb_prior_grads *grads, void *workspace,
                 size_t workspace_bytes, void *stream) {
    Net n;
    const int st_ = net_from(net, n);
    if (st_) return st_;
    if (!codes || !labels || !d_logits || !saved || !workspace || B <= 0 || H <= 0 || W <= 0 || !grads_ok(grads, n.L))
        return VQB_ERR_BAD_ARG;
    if (workspace_bytes < vqb_prior_backward_workspace_bytes(net, B, H, W)) return VQB_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    const int npos = B * H * W, C = n.C, K = n.K;
    const long long *lab = reinterpret_cast<const long long *>(labels);
    const Saved sv{npos, C, n.L};
    const float *sp = static_cast<const float *>(saved);
    float *ws = static_cast<float *>(workspace);
    const Bws wl = bws_layout(n, npos);
    float *part = ws + wl.part;
    unsigned long long launches = 0;

    // head: d_hidden = relu' * (W2^T d_logits); dW2, db2; dW1, db1; d x_h^L = W1^T d_hidden
    {
        float *dhid = ws + wl.work;
        const float *hid = sp + sv.hid(), *xL = sp + sv.xh(n.L);
        const Nchw dl{d_logits, K, H * W};
        product<G>(st, dl, WPacked{n.w2, HID, K}, ReluBack{dhid, hid}, npos, HID, K);
        const Phase p = head_phase(n, npos);
        G::run(st, NchwT{dl}, WithOnes<Mat>{Mat{hid, HID}, HID}, Partial{part + p.job[0].off, K, HID + 1}, K,
               HID + 1, npos, p.job[0].sp);
        G::run(st, MatT{dhid, HID}, WithOnes<Mat>{Mat{xL, C}, C}, Partial{part + p.job[1].off, HID, C + 1}, HID,
               C + 1, npos, p.job[1].sp);
        product<G>(st, Mat{dhid, HID}, WPacked{n.w1, C, HID}, Store{ws + wl.gh, nullptr, C}, npos, C, HID);
        reduce(st, p, part, {grads->out2_w, grads->out1_w}, {grads->out2_b, grads->out1_b});
        launches += 5;
    }
    launches += body_backward<G>(st, n, reinterpret_cast<const long long *>(codes), lab, Grid{H, W}, npos, sp, grads,
                                 ws, wl, false);
    VQB_COUNT_LAUNCH(launches);
    return vqb_cuda_status(cudaGetLastError());
}

// vqb_prior_ce_backward_f32 (G = Ffma) and _tf32 (G = Tf32): net_backward with the head's d_logits made per chunk of
// ce_rows positions.  Per chunk: the logits product of the forward (Mat hid x Mat W2, one k chunk: bitwise the
// forward's logits) with the CeGrad epilogue into dl; d_hidden = relu' * (dl W2^T); dW2, db2 partials added to acc.
// Then dW1, db1 and d x_h^L over all positions, one reduce for both head gradients, and body_backward.
// opt (the _ex entry points): the CeGrad<true> epilogue, with W and MEAN's factor from the saved tail.
template <class G>
int ce_backward(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H, int W,
                int reduction, const vqb_prior_ce_options *opt, const float *d_loss, const void *saved,
                const vqb_prior_grads *grads, void *workspace, size_t workspace_bytes, void *stream) {
    Net n;
    int st_ = ce_args(net, n, codes, labels, B, H, W, reduction, d_loss, workspace);
    if (st_) return st_;
    CeOpt o{};
    if (opt && (st_ = ce_opt_args(opt, o))) return st_;
    if (!saved || !grads_ok(grads, n.L)) return VQB_ERR_BAD_ARG;
    if (workspace_bytes < vqb_prior_ce_backward_workspace_bytes(net, B, H, W)) return VQB_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    const int npos = B * H * W, C = n.C, K = n.K;
    const long long *cd = reinterpret_cast<const long long *>(codes);
    const Saved sv{npos, C, n.L};
    const float *sp = static_cast<const float *>(saved);
    float *ws = static_cast<float *>(workspace);
    const Bws wl = bws_layout(n, npos, true);
    float *part = ws + wl.part, *dl = ws + wl.dl, *acc = ws + wl.acc, *dhid = ws + wl.work;
    const float *hid = sp + sv.hid(), *xL = sp + sv.xh(n.L), *lse = sp + sv.total();
    const int rows = (int)ce_rows(npos);
    const WgradSplit s2 = ce_w2_split(n, npos);
    const float scale = reduction == VQB_PRIOR_CE_MEAN ? (float)(1.0 / npos) : 1.f;
    const int gstride = reduction == VQB_PRIOR_CE_NONE ? 1 : 0;
    unsigned long long launches = 0;
    for (int c0 = 0; c0 < npos; c0 += rows) {
        const int P = npos - c0 < rows ? npos - c0 : rows;
        const float *hc = hid + (long long)c0 * HID;
        if (opt)
            product<G>(st, Mat{hc, HID}, Mat{n.w2, K},
                       CeGrad<true>{{o, lse + 2LL * npos, reduction == VQB_PRIOR_CE_MEAN}, dl, n.b2, lse, d_loss, cd,
                                    1.f, K, gstride, c0},
                       P, K, HID);
        else
            product<G>(st, Mat{hc, HID}, Mat{n.w2, K}, CeGrad<>{{}, dl, n.b2, lse, d_loss, cd, scale, K, gstride, c0},
                       P, K, HID);
        product<G>(st, Mat{dl, K}, WPacked{n.w2, HID, K}, ReluBack{dhid + (long long)c0 * HID, hc}, P, HID, K);
        G::run(st, MatT{dl, K}, WithOnes<Mat>{Mat{hc, HID}, HID}, PartialAdd{acc, K, HID + 1, c0 == 0}, K, HID + 1, P,
               s2);
        launches += 3;
    }
    const Phase p = head_phase(n, npos, true);
    G::run(st, MatT{dhid, HID}, WithOnes<Mat>{Mat{xL, C}, C}, Partial{part + p.job[0].off, HID, C + 1}, HID, C + 1,
           npos, p.job[0].sp);
    product<G>(st, Mat{dhid, HID}, WPacked{n.w1, C, HID}, Store{ws + wl.gh, nullptr, C}, npos, C, HID);
    RJobs jobs;
    jobs.j[0] = RJob{acc, grads->out2_w, grads->out2_b, K, HID, 1, HID + 1, s2.splits};
    jobs.j[1] = RJob{part + p.job[0].off, grads->out1_w, grads->out1_b, HID, C, 1, C + 1, p.job[0].sp.splits};
    const long long w2 = (long long)K * (HID + 1), w1 = (long long)HID * (C + 1);
    wgrad_reduce(st, jobs, 2, w2 > w1 ? w2 : w1);
    launches += 3 + body_backward<G>(st, n, cd, reinterpret_cast<const long long *>(labels), Grid{H, W}, npos, sp,
                                     grads, ws, wl, true);
    VQB_COUNT_LAUNCH(launches);
    return vqb_cuda_status(cudaGetLastError());
}

}  // namespace

extern "C" int vqb_prior_backward_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B,
                                      int H, int W, const float *d_logits, const void *saved,
                                      const vqb_prior_grads *grads, void *workspace, size_t workspace_bytes,
                                      void *stream) {
    return net_backward<Ffma>(net, codes, labels, B, H, W, d_logits, saved, grads, workspace, workspace_bytes, stream);
}

extern "C" int vqb_prior_backward_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B,
                                       int H, int W, const float *d_logits, const void *saved,
                                       const vqb_prior_grads *grads, void *workspace, size_t workspace_bytes,
                                       void *stream) {
    return net_backward<Tf32>(net, codes, labels, B, H, W, d_logits, saved, grads, workspace, workspace_bytes, stream);
}

extern "C" size_t vqb_prior_ce_backward_workspace_bytes(const vqb_prior_net *net, int B, int H, int W) {
    Net n;
    if (net_from(net, n) || B <= 0 || H <= 0 || W <= 0) return 0;
    return (size_t)bws_layout(n, (long long)B * H * W, true).total * sizeof(float);
}

extern "C" int vqb_prior_ce_backward_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B,
                                         int H, int W, int reduction, const float *d_loss, const void *saved,
                                         const vqb_prior_grads *grads, void *workspace, size_t workspace_bytes,
                                         void *stream) {
    return ce_backward<Ffma>(net, codes, labels, B, H, W, reduction, nullptr, d_loss, saved, grads, workspace,
                             workspace_bytes, stream);
}

extern "C" int vqb_prior_ce_backward_ex_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels,
                                            int B, int H, int W, int reduction, const vqb_prior_ce_options *options,
                                            const float *d_loss, const void *saved, const vqb_prior_grads *grads,
                                            void *workspace, size_t workspace_bytes, void *stream) {
    return ce_backward<Ffma>(net, codes, labels, B, H, W, reduction, options, d_loss, saved, grads, workspace,
                             workspace_bytes, stream);
}

extern "C" int vqb_prior_ce_backward_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B,
                                          int H, int W, int reduction, const float *d_loss, const void *saved,
                                          const vqb_prior_grads *grads, void *workspace, size_t workspace_bytes,
                                          void *stream) {
    return ce_backward<Tf32>(net, codes, labels, B, H, W, reduction, nullptr, d_loss, saved, grads, workspace,
                             workspace_bytes, stream);
}

extern "C" int vqb_prior_ce_backward_ex_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels,
                                            int B, int H, int W, int reduction, const vqb_prior_ce_options *options,
                                            const float *d_loss, const void *saved, const vqb_prior_grads *grads,
                                            void *workspace, size_t workspace_bytes, void *stream) {
    return ce_backward<Tf32>(net, codes, labels, B, H, W, reduction, options, d_loss, saved, grads, workspace,
                             workspace_bytes, stream);
}

extern "C" int vqb_prior_gate_backward_f32(const float *x, const float *d_out, float *d_x, int64_t outer, int C,
                                          int64_t inner, void *stream) {
    if (!x || !d_out || !d_x || outer <= 0 || C <= 0 || inner <= 0) return VQB_ERR_BAD_ARG;
    gate_backward_kernel<<<grid_for(outer * C * inner), NT, 0, (cudaStream_t)stream>>>(x, d_out, d_x, outer, C, inner);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

namespace {

// One layer's backward for dims up to maxc (MAXC: the ABI-3 pair vqb_prior_layer_backward_*, which has always
// refused dim > 256; MAXC_WIDE: vqb_prior_layer_backward_wide_*).  Workspace: the 6 grids of layer_backward's
// scratch, then its wgrad partials (0 = bad arguments).
size_t layer_backward_ws(int maxc, const vqb_prior_layer_weights *layer, int B, int H, int W, int dim, int n_classes) {
    if (!layer || !layer_ok(*layer) || B <= 0 || H <= 0 || W <= 0 || n_classes <= 0 || !dim_ok(dim) || dim > maxc)
        return 0;
    const long long npos = (long long)B * H * W;
    return (size_t)(6 * npos * dim + layer_phase(*layer, dim, n_classes, npos).floats) * sizeof(float);
}

int layer_backward_call(int maxc, const vqb_prior_layer_weights *layer, const float *x_v, const float *x_h,
                        const int64_t *labels, int B, int H, int W, int dim, int n_classes, const float *d_out_v,
                        const float *d_out_h, const void *saved, const vqb_prior_layer_grads *grads, float *d_x_v,
                        float *d_x_h, void *workspace, size_t workspace_bytes, void *stream) {
    if (!layer || !x_v || !x_h || !labels || !d_out_h || !saved || !grads || !d_x_v || !d_x_h || !workspace ||
        B <= 0 || H <= 0 || W <= 0 || dim <= 0 || n_classes <= 0 || !layer_ok(*layer) || !layer_grads_ok(*grads))
        return VQB_ERR_BAD_ARG;
    if (!dim_ok(dim) || dim > maxc) return VQB_ERR_UNSUPPORTED;
    if (workspace_bytes < layer_backward_ws(maxc, layer, B, H, W, dim, n_classes)) return VQB_ERR_WORKSPACE;
    const int npos = B * H * W;
    const LayerSaved sv{npos, dim};
    const float *sp = static_cast<const float *>(saved);
    float *ws = static_cast<float *>(workspace);
    layer_backward<Ffma>((cudaStream_t)stream, *layer, *grads, dim, n_classes, reinterpret_cast<const long long *>(labels),
                   Grid{H, W}, npos, x_v, x_h, sp + sv.hv(), sp + sv.ph(), d_out_h, d_out_v, d_x_h, d_x_v, nullptr, ws,
                   ws + 6LL * npos * dim);
    VQB_COUNT_LAUNCH(10);
    return vqb_cuda_status(cudaGetLastError());
}

}  // namespace

extern "C" size_t vqb_prior_layer_backward_workspace_bytes(const vqb_prior_layer_weights *layer, int B, int H, int W,
                                                           int dim, int n_classes) {
    return layer_backward_ws(MAXC, layer, B, H, W, dim, n_classes);
}

extern "C" int vqb_prior_layer_backward_f32(const vqb_prior_layer_weights *layer, const float *x_v, const float *x_h,
                                           const int64_t *labels, int B, int H, int W, int dim, int n_classes,
                                           const float *d_out_v, const float *d_out_h, const void *saved,
                                           const vqb_prior_layer_grads *grads, float *d_x_v, float *d_x_h,
                                           void *workspace, size_t workspace_bytes, void *stream) {
    return layer_backward_call(MAXC, layer, x_v, x_h, labels, B, H, W, dim, n_classes, d_out_v, d_out_h, saved, grads,
                               d_x_v, d_x_h, workspace, workspace_bytes, stream);
}

extern "C" size_t vqb_prior_layer_backward_wide_workspace_bytes(const vqb_prior_layer_weights *layer, int B, int H,
                                                                int W, int dim, int n_classes) {
    return layer_backward_ws(MAXC_WIDE, layer, B, H, W, dim, n_classes);
}

extern "C" int vqb_prior_layer_backward_wide_f32(const vqb_prior_layer_weights *layer, const float *x_v,
                                                const float *x_h, const int64_t *labels, int B, int H, int W, int dim,
                                                int n_classes, const float *d_out_v, const float *d_out_h,
                                                const void *saved, const vqb_prior_layer_grads *grads, float *d_x_v,
                                                float *d_x_h, void *workspace, size_t workspace_bytes, void *stream) {
    return layer_backward_call(MAXC_WIDE, layer, x_v, x_h, labels, B, H, W, dim, n_classes, d_out_v, d_out_h, saved,
                               grads, d_x_v, d_x_h, workspace, workspace_bytes, stream);
}

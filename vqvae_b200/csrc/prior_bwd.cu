// prior_bwd.cu -- backward of the Gated PixelCNN prior (GatedPixelCNN.forward, pixelcnn/models.py:121-130), fp32 on
// CUDA cores (sm_90a).
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
#include "prior.cuh"
#include "ffma_gemm.cuh"

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

// ---- host side ---------------------------------------------------------------------------------------------------
template <class LA, class LB, class EP>
void dgrad(cudaStream_t st, LA a, LB b, EP ep, int M, int N, int K) { gemm(st, a, b, ep, M, N, K, WgradSplit{1, K}); }

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
    WJob &add(int M, int Cin, int taps, bool bias, long long npos) {
        WJob &j = job[n++];
        j.M = M; j.Cin = Cin; j.taps = taps; j.bias = bias;
        j.sp = wgrad_split(M, j.cols(), npos, BM, BN, BK);
        j.off = floats;
        floats += j.floats();
        return j;
    }
};

int vrows(const vqb_prior_layer_weights &w) { return w.kernel / 2 + 1; }     // vert_stack (k/2 + 1, k)
int hcols(const vqb_prior_layer_weights &w) { return w.kernel / 2 + 1; }     // horiz_stack (1, k/2 + 1)

// the wgrad jobs of the head (dW2, dW1), of layer l (resid, horiz, v2h, class, vert) and of the embedding
Phase head_phase(const Net &n, long long npos) {
    Phase p;
    p.add(n.K, HID, 1, true, npos);
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

Phase emb_phase(const Net &n, long long npos) {
    Phase p;
    p.add(n.K, n.C, 1, false, npos);
    return p;
}

// workspace regions, in floats: d x_h (2 grids), d x_v (2 grids), the head's d_hidden or a layer's d pre_h, d h_vert
// and class gradient (union), then the wgrad partials of the largest phase
struct Bws {
    long long gh, gv, work, part, total;
};

Bws bws_layout(const Net &n, long long npos) {
    Bws w;
    const long long grid = npos * n.C;
    w.gh = 0;
    w.gv = 2 * grid;
    w.work = 4 * grid;
    const long long head = npos * HID, layer = 6 * grid;
    w.part = w.work + (head > layer ? head : layer);
    long long part = head_phase(n, npos).floats;
    const long long e = emb_phase(n, npos).floats;
    part = part > e ? part : e;
    for (int l = 0; l < n.L; ++l) {
        const long long f = layer_phase(n.layer[l], n.C, n.NC, npos).floats;
        part = part > f ? part : f;
    }
    w.total = w.part + part;
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
void layer_backward(cudaStream_t st, const vqb_prior_layer_weights &w, const vqb_prior_layer_grads &q, int C, int NC,
                    const long long *lab, Grid g, int npos, const float *xv, const float *xh, const float *hv,
                    const float *ph, const float *ghi, const float *gvi, float *gho, float *gvo, const float *fold,
                    float *work, float *part) {
    const int C2 = 2 * C, half = w.kernel / 2, vr = vrows(w) - (w.mask_a ? 1 : 0), hc = hcols(w) - (w.mask_a ? 1 : 0);
    const long long grid = (long long)npos * C;
    float *dph = work, *dhv = dph + 2 * grid, *cls = dhv + 2 * grid;
    const Phase p = layer_phase(w, C, NC, npos);
    // out_h = horiz_resid(gate(pre_h)) [+ x_h]: d pre_h, then d x_h = [d out_h +] horiz_stack^T * d pre_h
    dgrad(st, Mat{ghi, C}, WPacked{w.resid_w, C, C}, GateBack{dph, ph, C}, npos, C, C);
    gemm(st, MatT{ghi, C}, WithOnes<Gated>{Gated{ph, C}, C}, Partial{part + p.job[0].off, C, C + 1}, C, C + 1,
         npos, p.job[0].sp);
    dgrad(st, Tap{dph, C2, hc, 0, half, -1, g}, WPacked{w.horiz_w, C, C2}, Store{gho, w.residual ? ghi : nullptr, C},
          npos, C, hc * C2);
    gemm(st, MatT{dph, C2}, WithOnes<Tap>{Tap{xh, C, hcols(w), 0, half, 1, g}, hcols(w) * C},
         Partial{part + p.job[1].off, C2, p.job[1].cols()}, C2, p.job[1].cols(), npos, p.job[1].sp);
    gemm(st, MatT{dph, C2}, WithOnes<Mat>{Mat{hv, C2}, C2}, Partial{part + p.job[2].off, C2, C2 + 1}, C2, C2 + 1,
         npos, p.job[2].sp);
    // d h_vert = W_v2h^T d pre_h + gate'(h_vert + class) * d out_v; class gradient; d x_v = vert_stack^T * d h_vert
    dgrad(st, Mat{dph, C2}, WPacked{w.v2h_w, C2, C2},
          VertBack{dhv, cls, hv, gvi, dph, w.class_emb, lab, C, g.H * g.W, NC}, npos, C2, C2);
    gemm(st, OneHot{lab, g.H * g.W, NC}, Mat{cls, C2}, Partial{part + p.job[3].off, NC, C2}, NC, C2, npos,
         p.job[3].sp);
    gemm(st, MatT{dhv, C2}, WithOnes<Tap>{Tap{xv, C, w.kernel, half, half, 1, g}, vrows(w) * w.kernel * C},
         Partial{part + p.job[4].off, C2, p.job[4].cols()}, C2, p.job[4].cols(), npos, p.job[4].sp);
    dgrad(st, Tap{dhv, C2, w.kernel, half, half, -1, g}, WPacked{w.vert_w, C, C2}, Store{gvo, fold, C}, npos, C,
          vr * w.kernel * C2);
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

}  // namespace

extern "C" size_t vqb_prior_backward_workspace_bytes(const vqb_prior_net *net, int B, int H, int W) {
    Net n;
    if (net_from(net, n) || B <= 0 || H <= 0 || W <= 0) return 0;
    return (size_t)bws_layout(n, (long long)B * H * W).total * sizeof(float);
}

extern "C" int vqb_prior_backward_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B,
                                      int H, int W, const float *d_logits, const void *saved,
                                      const vqb_prior_grads *grads, void *workspace, size_t workspace_bytes,
                                      void *stream) {
    Net n;
    const int st_ = net_from(net, n);
    if (st_) return st_;
    if (!codes || !labels || !d_logits || !saved || !workspace || B <= 0 || H <= 0 || W <= 0 || !grads_ok(grads, n.L))
        return VQB_ERR_BAD_ARG;
    if (workspace_bytes < vqb_prior_backward_workspace_bytes(net, B, H, W)) return VQB_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    const int npos = B * H * W, C = n.C, K = n.K;
    const long long grid = (long long)npos * C;
    const long long *lab = reinterpret_cast<const long long *>(labels);
    const Saved sv{npos, C, n.L};
    const float *sp = static_cast<const float *>(saved);
    float *ws = static_cast<float *>(workspace);
    const Bws wl = bws_layout(n, npos);
    float *gh[2] = {ws + wl.gh, ws + wl.gh + grid}, *gv[2] = {ws + wl.gv, ws + wl.gv + grid};
    float *part = ws + wl.part;
    const Grid g{H, W};
    unsigned long long launches = 0;

    // head: d_hidden = relu' * (W2^T d_logits); dW2, db2; dW1, db1; d x_h^L = W1^T d_hidden
    {
        float *dhid = ws + wl.work;
        const float *hid = sp + sv.hid(), *xL = sp + sv.xh(n.L);
        const Nchw dl{d_logits, K, H * W};
        dgrad(st, dl, WPacked{n.w2, HID, K}, ReluBack{dhid, hid}, npos, HID, K);
        const Phase p = head_phase(n, npos);
        gemm(st, NchwT{dl}, WithOnes<Mat>{Mat{hid, HID}, HID}, Partial{part + p.job[0].off, K, HID + 1}, K, HID + 1,
             npos, p.job[0].sp);
        gemm(st, MatT{dhid, HID}, WithOnes<Mat>{Mat{xL, C}, C}, Partial{part + p.job[1].off, HID, C + 1}, HID, C + 1,
             npos, p.job[1].sp);
        dgrad(st, Mat{dhid, HID}, WPacked{n.w1, C, HID}, Store{gh[0], nullptr, C}, npos, C, HID);
        reduce(st, p, part, {grads->out2_w, grads->out1_w}, {grads->out2_b, grads->out1_b});
        launches += 5;
    }
    // layers, last to first.  gh[cur] = d x_h^{l+1}, gv[cur] = d x_v^{l+1} (none for the last layer)
    int cur = 0;
    for (int l = n.L - 1; l >= 0; --l) {
        float *gho = gh[cur ^ 1];
        // layer 0: x_v and x_h are both the embedding, so d x_v^0 + d x_h^0 is its gradient per position
        layer_backward(st, n.layer[l], grads->layers[l], C, n.NC, lab, g, npos, sp + sv.xv(l), sp + sv.xh(l),
                       sp + sv.hv(l), sp + sv.ph(l), gh[cur], l == n.L - 1 ? nullptr : gv[cur], gho, gv[cur ^ 1],
                       l == 0 ? gho : nullptr, ws + wl.work, part);
        launches += 10;
        cur ^= 1;
    }
    // embedding: the per-position gradient summed by (clamped) code
    {
        const Phase p = emb_phase(n, npos);
        gemm(st, OneHot{reinterpret_cast<const long long *>(codes), 1, K}, Mat{gv[cur], C},
             Partial{part + p.job[0].off, K, C}, K, C, npos, p.job[0].sp);
        reduce(st, p, part, {grads->embedding}, {nullptr});
        launches += 2;
    }
    VQB_COUNT_LAUNCH(launches);
    return vqb_cuda_status(cudaGetLastError());
}

extern "C" int vqb_prior_gate_backward_f32(const float *x, const float *d_out, float *d_x, int64_t outer, int C,
                                          int64_t inner, void *stream) {
    if (!x || !d_out || !d_x || outer <= 0 || C <= 0 || inner <= 0) return VQB_ERR_BAD_ARG;
    gate_backward_kernel<<<grid_for(outer * C * inner), NT, 0, (cudaStream_t)stream>>>(x, d_out, d_x, outer, C, inner);
    VQB_COUNT_LAUNCH(1);
    return vqb_cuda_status(cudaGetLastError());
}

// workspace of one layer's backward: the 6 grids of layer_backward's scratch, then its wgrad partials
extern "C" size_t vqb_prior_layer_backward_workspace_bytes(const vqb_prior_layer_weights *layer, int B, int H, int W,
                                                           int dim, int n_classes) {
    if (!layer || !layer_ok(*layer) || B <= 0 || H <= 0 || W <= 0 || n_classes <= 0 || !dim_ok(dim)) return 0;
    const long long npos = (long long)B * H * W;
    return (size_t)(6 * npos * dim + layer_phase(*layer, dim, n_classes, npos).floats) * sizeof(float);
}

extern "C" int vqb_prior_layer_backward_f32(const vqb_prior_layer_weights *layer, const float *x_v, const float *x_h,
                                           const int64_t *labels, int B, int H, int W, int dim, int n_classes,
                                           const float *d_out_v, const float *d_out_h, const void *saved,
                                           const vqb_prior_layer_grads *grads, float *d_x_v, float *d_x_h,
                                           void *workspace, size_t workspace_bytes, void *stream) {
    if (!layer || !x_v || !x_h || !labels || !d_out_h || !saved || !grads || !d_x_v || !d_x_h || !workspace ||
        B <= 0 || H <= 0 || W <= 0 || dim <= 0 || n_classes <= 0 || !layer_ok(*layer) || !layer_grads_ok(*grads))
        return VQB_ERR_BAD_ARG;
    if (!dim_ok(dim)) return VQB_ERR_UNSUPPORTED;
    if (workspace_bytes < vqb_prior_layer_backward_workspace_bytes(layer, B, H, W, dim, n_classes))
        return VQB_ERR_WORKSPACE;
    const int npos = B * H * W;
    const LayerSaved sv{npos, dim};
    const float *sp = static_cast<const float *>(saved);
    float *ws = static_cast<float *>(workspace);
    layer_backward((cudaStream_t)stream, *layer, *grads, dim, n_classes, reinterpret_cast<const long long *>(labels),
                   Grid{H, W}, npos, x_v, x_h, sp + sv.hv(), sp + sv.ph(), d_out_h, d_out_v, d_x_h, d_x_v, nullptr, ws,
                   ws + 6LL * npos * dim);
    VQB_COUNT_LAUNCH(10);
    return vqb_cuda_status(cudaGetLastError());
}

// api.cu -- the extern "C" boundary declared in include/vqvae_b200.h.
#include <cstdlib>

#include "common.cuh"

size_t vq_exact_workspace_bytes(int K);
int launch_vq_exact(const float *z, const float *E, long long N, int K, int D, long long *idx, void *zq, int zq_bf16,
                    double *sse, int *hist, void *ws, cudaStream_t s);
int launch_conv_in_k4s2(const float *x, const float *wp, const float *bias, void *y, int out_bf16, int B, int Cin, int H,
                        int W, int Cout, int relu, cudaStream_t s);
int launch_convt_out_k4s2(const float *x, const float *wp, const float *bias, float *y, int B, int Cin, int H, int W,
                          int Cout, int relu, cudaStream_t s);
#include "wgconv.h"
bool vq_tc_supported(long long N, int K, int D);
bool vq_exact_supported(int K, int D);
int launch_vq_tc(const float *z, const float *E, long long N, int K, int D, long long *idx, void *zq, int zq_bf16, double *sse,
                 int *hist, void *ws, float *dbg, cudaStream_t s);

int vqb_pdl_enabled() {
    static int on = -1;
    if (on < 0) {
        const char *e = vqb_getenv("VQB_PDL");
        on = e ? (atoi(e) != 0) : 1;
    }
    return on;
}

unsigned long long g_vqb_launches = 0;
static int g_vq_kernel = 0;   // 0 auto (tensor-core kernel when D == 64), 1 exact FFMA kernel, 2 tensor-core kernel
extern "C" int vqb_set_vq_kernel(int which) {
    if (which < 0 || which > 2) return VQB_ERR_BAD_ARG;
    g_vq_kernel = which;
    return 0;
}
extern "C" unsigned long long vqb_launch_count(void) { return g_vqb_launches; }

extern "C" int vqb_abi_version(void) { return VQB_ABI_VERSION; }

// 0 = release library (never reads the environment, no work-skipping paths compiled in); 1 = diagnostic build
extern "C" int vqb_diag_build(void) { return VQB_DIAG; }

extern "C" const char *vqb_error_string(int code) {
    switch (code) {
        case VQB_OK: return "success";
        case VQB_ERR_BAD_ARG: return "bad argument (null pointer, non-positive size or bad enum)";
        case VQB_ERR_UNSUPPORTED: return "shape not supported by the sm_90a kernels";
        case VQB_ERR_WORKSPACE: return "workspace too small";
        case VQB_ERR_NO_DEVICE: return "no CUDA device";
        case VQB_ERR_ALIGNMENT: return "pointer not 16-byte aligned";
        default: return code > 0 ? cudaGetErrorString((cudaError_t)code) : "unknown vqb error";
    }
}

extern "C" int vqb_device_info(int *sm_count, int *cc_major, int *cc_minor) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return VQB_ERR_NO_DEVICE;
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, dev);
    if (e != cudaSuccess) return VQB_ERR_NO_DEVICE;
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    return 0;
}

extern "C" int vqb_conv2d_f32(const float *in, const float *w_packed, const float *bias, const float *skip,
                              float *out, int B, int Cin, int H, int W, int Cout, int kh, int kw, int stride,
                              int pad, int transposed, int in_layout, int out_layout, int relu, int precision,
                              void *stream) {
    if (!in || !w_packed || !out) return VQB_ERR_BAD_ARG;
    if (B <= 0 || Cin <= 0 || H <= 0 || W <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || stride <= 0 || pad < 0)
        return VQB_ERR_BAD_ARG;
    if ((in_layout != VQB_NCHW && in_layout != VQB_NHWC) || (out_layout != VQB_NCHW && out_layout != VQB_NHWC))
        return VQB_ERR_BAD_ARG;
    if (precision < VQB_FP32 || precision > VQB_BF16) return VQB_ERR_BAD_ARG;
    if (precision == VQB_BF16) return VQB_ERR_UNSUPPORTED;      // bf16 operands need bf16 activations: vqb_conv2d_bf16
    if (skip && out_layout != VQB_NHWC) return VQB_ERR_BAD_ARG;
    if (kh * kw > VQB_MAX_TAPS) return VQB_ERR_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;

    const ConvGeom g = conv_geom(kh, kw, stride, pad, transposed, H, W);
    if (g.OH <= 0 || g.OW <= 0) return VQB_ERR_BAD_ARG;

    // the two end layers: the output ConvTranspose2d (Cout <= 4) as one wgmma GEMM per tile over its input pixels and
    // their halo, summed into the pixel-shuffled output (wgconv.cu, scatter form); the input conv (Cin = 3: K = 48
    // fp32 values per pixel straight from the NCHW image, HBM bound) and the fp32 mode on dedicated CUDA-core kernels
    // (conv_edge.cu)
    if (kh == 4 && kw == 4 && stride == 2 && pad == 1 && !skip) {
        if (transposed && precision != VQB_FP32 && in_layout == VQB_NHWC && out_layout == VQB_NCHW &&
            convt_shuffle_supported(Cin, Cout)) {
            const int rc = launch_convt_shuffle_wg(0, in, w_packed + conv_pack_shuffle_offset(Cout, Cin, kh, kw), bias, out,
                                                   B, Cin, H, W, Cout, relu, s);
            if (rc != VQB_ERR_UNSUPPORTED) return rc;
        }
        if (!transposed && Cin == 3 && Cout % 32 == 0 && in_layout == VQB_NCHW && out_layout == VQB_NHWC &&
            H % 2 == 0 && W % 2 == 0 && (size_t)16 * Cin * Cout * 4 <= 48 * 1024)
            return launch_conv_in_k4s2(in, w_packed, bias, out, 0, B, Cin, H, W, Cout, relu, s);
        if (transposed && Cout == 3 && Cin % 4 == 0 && Cin <= 128 && ((Cin / 4) & (Cin / 4 - 1)) == 0 &&
            in_layout == VQB_NHWC && out_layout == VQB_NCHW)
            return launch_convt_out_k4s2(in, w_packed, bias, out, B, Cin, H, W, Cout, relu, s);
    }

    ConvLaunch p = {};
    p.in = in; p.w = w_packed; p.bias = bias; p.skip = skip; p.out = out;
    p.B = B; p.Cin = Cin; p.H = H; p.W = W; p.Cout = Cout; p.relu = relu;
    layout_strides(in_layout, Cin, H, W, p.in_sn, p.in_sh, p.in_sw, p.in_sc);
    layout_strides(out_layout, Cout, g.OH, g.OW, p.out_sn, p.out_sh, p.out_sw, p.out_sc);
    auto run_ffma = [&](const ConvPhase &ph) {
        static_cast<ConvPhase &>(p) = ph;
        return Cout <= 4 ? launch_conv_small_cout(p, s) : launch_conv_ffma(p, s);
    };
    // the wgmma path takes every phase of the layer in one launch (blockIdx.y = phase); a phase no tap reaches still
    // gets bias/skip/activation
    const bool tc = precision != VQB_FP32 && stride <= 2 && conv_tc_supported(p);
    ConvPhase phases[4];
    int nph = 0;
    for (int i = 0; i < g.nph; ++i) {
        ConvPhase ph;
        if (!conv_phase(g, i, ph)) continue;
        if (tc) { phases[nph++] = ph; continue; }
        const int rc = run_ffma(ph);
        if (rc != 0) return rc;
    }
    if (tc && nph > 0) {
        WgLaunch L;
        L.in = in; L.B = B; L.Cin = Cin; L.H = H; L.W = W;
        L.w = w_packed; L.ncols = Cout;
        L.bias = bias; L.skip = skip; L.out = out; L.relu = relu;
        L.out_sn = p.out_sn; L.out_sh = p.out_sh; L.out_sw = p.out_sw; L.out_sc = p.out_sc;
        // the launcher answers VQB_ERR_UNSUPPORTED before launching anything when it cannot take the shape (step
        // table, shared memory): the FFMA kernels run it then
        const int rc = launch_conv_tc(L, phases, nph, kh * kw, false, s);
        if (rc != VQB_ERR_UNSUPPORTED) return rc;
        for (int i = 0; i < nph; ++i) {
            const int rc2 = run_ffma(phases[i]);
            if (rc2 != 0) return rc2;
        }
    }
    return 0;
}

ConvGeom conv_geom(int kh, int kw, int stride, int pad, int transposed, int H, int W) {
    ConvGeom g = {kh, kw, stride, pad, transposed};
    g.OH = transposed ? (H - 1) * stride - 2 * pad + kh : (H + 2 * pad - kh) / stride + 1;
    g.OW = transposed ? (W - 1) * stride - 2 * pad + kw : (W + 2 * pad - kw) / stride + 1;
    g.nph = transposed ? stride * stride : 1;
    return g;
}

// Phase i = py * s + px.  A conv reads in(gy * stride + r - pad) through kernel row r; output row y = s gy + py of a
// stride-s transposed conv takes input row gy + dy through kernel row r = py + pad - s dy, so phase (py, px) is a
// stride-1 gather conv over the taps whose (py + pad - r, px + pad - c) are multiples of s.
bool conv_phase(const ConvGeom &g, int i, ConvPhase &ph) {
    const int up = g.transposed ? g.stride : 1;
    ph.in_step = g.transposed ? 1 : g.stride;
    ph.out_step = up;
    ph.out_py = i / up; ph.out_px = i % up;
    ph.OHg = (g.OH - ph.out_py + up - 1) / up;
    ph.OWg = (g.OW - ph.out_px + up - 1) / up;
    ph.ntaps = 0;
    for (int r = 0; r < g.kh; ++r)
        for (int c = 0; c < g.kw; ++c) {
            const int ny = g.transposed ? ph.out_py + g.pad - r : r - g.pad;
            const int nx = g.transposed ? ph.out_px + g.pad - c : c - g.pad;
            if (ny % up != 0 || nx % up != 0) continue;
            ph.tap_w[ph.ntaps] = r * g.kw + c;
            ph.tap_dy[ph.ntaps] = ny / up;
            ph.tap_dx[ph.ntaps] = nx / up;
            ++ph.ntaps;
        }
    return ph.OHg > 0 && ph.OWg > 0;
}

extern "C" size_t vqb_vq_workspace_bytes(int64_t N, int K, int D) {
    (void)N; (void)D;
    if (K <= 0) return 0;
    return vq_exact_workspace_bytes(K);
}

// The shape checks of vqb_vq_forward_f32's dispatch under the current vqb_set_vq_kernel choice, answered before it
// launches anything (vq_ema.cu's k-means asks them before its first launch).
int vq_forward_check(long long N, int K, int D) {
    if (N <= 0 || K <= 0 || D <= 0) return VQB_ERR_BAD_ARG;
    if (D % 4 != 0) return VQB_ERR_UNSUPPORTED;
    const bool tc = vq_tc_supported(N, K, D);
    if (g_vq_kernel == 2 && !tc) return VQB_ERR_UNSUPPORTED;
    if ((!tc || g_vq_kernel == 1) && !vq_exact_supported(K, D)) return VQB_ERR_UNSUPPORTED;
    return 0;
}

static int vq_forward_impl(const float *z, const float *codebook, int64_t N, int K, int D, int64_t *idx, void *zq,
                           int zq_bf16, double *sse, int32_t *hist, void *workspace, size_t workspace_bytes, void *stream) {
    if (!z || !codebook || !idx || !zq || !sse || !hist || !workspace) return VQB_ERR_BAD_ARG;
    const int rc = vq_forward_check(N, K, D);
    if (rc != 0) return rc;
    const bool tc_ok = vq_tc_supported(N, K, D);
    if (workspace_bytes < vqb_vq_workspace_bytes(N, K, D)) return VQB_ERR_WORKSPACE;
    const uintptr_t al = reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(codebook) |
                         reinterpret_cast<uintptr_t>(zq) | reinterpret_cast<uintptr_t>(workspace);
    if (al & 15) return VQB_ERR_ALIGNMENT;
    if (tc_ok && g_vq_kernel != 1)
        return launch_vq_tc(z, codebook, N, K, D, reinterpret_cast<long long *>(idx), zq, zq_bf16, sse, hist, workspace,
                            nullptr, (cudaStream_t)stream);
    return launch_vq_exact(z, codebook, N, K, D, reinterpret_cast<long long *>(idx), zq, zq_bf16, sse, hist, workspace,
                           (cudaStream_t)stream);
}

extern "C" int vqb_vq_forward_f32(const float *z, const float *codebook, int64_t N, int K, int D, int64_t *idx,
                                  float *zq, double *sse, int32_t *hist, void *workspace,
                                  size_t workspace_bytes, void *stream) {
    return vq_forward_impl(z, codebook, N, K, D, idx, zq, 0, sse, hist, workspace, workspace_bytes, stream);
}

// VQB_BF16 pipeline: same contract as vqb_vq_forward_f32 (fp32 z in, bit-exact idx) but z_q leaves as bf16
// rows for the decoder's first conv.
extern "C" int vqb_vq_forward_bf16zq_f32(const float *z, const float *codebook, int64_t N, int K, int D, int64_t *idx,
                                         void *zq_bf16, double *sse, int32_t *hist, void *workspace,
                                         size_t workspace_bytes, void *stream) {
    return vq_forward_impl(z, codebook, N, K, D, idx, zq_bf16, 1, sse, hist, workspace, workspace_bytes, stream);
}

// encoder.py:29-31 in the VQB_BF16 pipeline: fp32 NCHW image in, bf16 NHWC activation out (Cout == 64), fp32 FFMA
// arithmetic (conv_edge.cu).  w_packed: vqb_pack_conv_weight_f32 of the layer (K-major rows, the same as the fp32 mode).
extern "C" int vqb_conv_in_bf16(const float *x, const float *w_packed, const float *bias, void *out, int B, int H, int W,
                                int Cout, int relu, void *stream) {
    if (!x || !w_packed || !out) return VQB_ERR_BAD_ARG;
    if (B <= 0 || H <= 0 || W <= 0 || Cout <= 0) return VQB_ERR_BAD_ARG;
    if (Cout != 64) return VQB_ERR_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(out) & 15)) return VQB_ERR_ALIGNMENT;
    return launch_conv_in_k4s2(x, w_packed, bias, out, 1, B, 3, H, W, Cout, relu, (cudaStream_t)stream);
}

extern "C" int vqb_debug_vq_scores_f32(const float *z, const float *codebook, int64_t N, int K, int D, int64_t *idx,
                                       float *zq, double *sse, int32_t *hist, void *workspace,
                                       size_t workspace_bytes, float *scores, void *stream) {
    if (!z || !codebook || !idx || !zq || !sse || !hist || !workspace || !scores) return VQB_ERR_BAD_ARG;
    if (!vq_tc_supported(N, K, D)) return VQB_ERR_UNSUPPORTED;
    if (workspace_bytes < vqb_vq_workspace_bytes(N, K, D)) return VQB_ERR_WORKSPACE;
    return launch_vq_tc(z, codebook, N, K, D, reinterpret_cast<long long *>(idx), zq, 0, sse, hist, workspace, scores,
                        (cudaStream_t)stream);
}

extern "C" int vqb_residual_layer_f32(const float *r, const float *w1_packed, const float *w2_packed, float *out,
                                      float *tmp, int B, int H, int W, int C, int Cmid, int relu_out, int precision,
                                      void *stream) {
    if (!r || !w1_packed || !w2_packed || !out || !tmp) return VQB_ERR_BAD_ARG;
    if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || Cmid <= 0) return VQB_ERR_BAD_ARG;
    if (precision < VQB_FP32 || precision > VQB_BF16) return VQB_ERR_BAD_ARG;
    if (precision == VQB_BF16) return VQB_ERR_UNSUPPORTED;      // see vqb_residual_layer_bf16
    if (precision == VQB_TF32 && res_wg_supported(0, C, Cmid)) {      // one wgmma launch, the intermediate stays on chip
        const int rc = launch_res_wg(0, r, w1_packed, w2_packed, out, B, H, W, C, Cmid, relu_out, 1, (cudaStream_t)stream);
        if (rc != VQB_ERR_UNSUPPORTED) return rc;
    }
    // two launches (residual.py:20-24 then :23-24,:28)

    int rc = vqb_conv2d_f32(r, w1_packed, nullptr, nullptr, tmp, B, C, H, W, Cmid, 3, 3, 1, 1, 0, VQB_NHWC, VQB_NHWC, 1,
                            precision, stream);
    if (rc) return rc;
    return vqb_conv2d_f32(tmp, w2_packed, nullptr, r, out, B, Cmid, H, W, C, 1, 1, 1, 0, 0, VQB_NHWC, VQB_NHWC,
                          relu_out, precision, stream);
}

extern "C" int vqb_residual_stack_f32(const float *r, const float *w1_packed, const float *w2_packed, float *out,
                                      float *scratch, float *tmp, int B, int H, int W, int C, int Cmid, int n_layers,
                                      int precision, void *stream) {
    if (!r || !w1_packed || !w2_packed || !out || !tmp) return VQB_ERR_BAD_ARG;
    if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || Cmid <= 0 || n_layers < 1) return VQB_ERR_BAD_ARG;
    if (n_layers > 1 && !scratch) return VQB_ERR_BAD_ARG;
    if (precision < VQB_FP32 || precision > VQB_BF16) return VQB_ERR_BAD_ARG;
    if (precision == VQB_BF16) return VQB_ERR_UNSUPPORTED;
    if (n_layers > 1 && precision == VQB_TF32 && res_wg_supported(0, C, Cmid)) {
        // all applications in ONE launch when a tile holds whole images and Cmid = 32 (res_scatter_kernel; answers
        // VQB_ERR_UNSUPPORTED otherwise)
        const int rc = launch_res_wg(0, r, w1_packed, w2_packed, out, B, H, W, C, Cmid, 1, n_layers, (cudaStream_t)stream);
        if (rc != VQB_ERR_UNSUPPORTED) return rc;
    }
    // one launch per application, ping-ponging so that the last one lands in `out`
    const float *src = r;
    for (int i = 0; i < n_layers; ++i) {
        float *dst = ((n_layers - 1 - i) % 2 == 0) ? out : scratch;
        const int rc = vqb_residual_layer_f32(src, w1_packed, w2_packed, dst, tmp, B, H, W, C, Cmid, 1, precision, stream);
        if (rc) return rc;
        src = dst;
    }
    return 0;
}

extern "C" int vqb_latent_block_tf32(const float *x, const float *head_w_packed, const float *head_bias,
                                     int head_transposed, const float *w1_packed, const float *w2_packed, int n_layers,
                                     const float *tail_w_packed, const float *tail_bias, int tail_cout, float *out,
                                     int B, int Cin, int H, int W, int C, int Cmid, void *stream) {
    if (!x || !head_w_packed || !w1_packed || !w2_packed || !out) return VQB_ERR_BAD_ARG;
    if (B <= 0 || Cin <= 0 || H <= 0 || W <= 0 || C <= 0 || Cmid <= 0 || n_layers < 1 || tail_cout < 0)
        return VQB_ERR_BAD_ARG;
    if (head_transposed != 0 && head_transposed != 1) return VQB_ERR_BAD_ARG;
    if ((tail_w_packed != nullptr) != (tail_cout != 0)) return VQB_ERR_BAD_ARG;
    return launch_latent_block(x, head_w_packed, head_bias, Cin, head_transposed, w1_packed, w2_packed, n_layers,
                               tail_w_packed, tail_bias, tail_cout, out, B, H, W, C, Cmid, (cudaStream_t)stream);
}

extern "C" int vqb_latent_block_supported(int Cin, int H, int W, int C, int Cmid, int tail_cout) {
    return Cin > 0 && H > 0 && W > 0 && tail_cout >= 0 && latent_block_supported(Cin, C, Cmid, H, W, tail_cout) ? 1 : 0;
}

extern "C" int vqb_decoder_tail_tf32(const float *d_out, const float *convt_w_packed, const float *convt_bias,
                                     const float *out_w_packed, const float *out_bias, float *h_out, float *x_hat, int B,
                                     int Cin, int H, int W, int C, int Cout, int relu_out, void *stream) {
    if (!d_out || !convt_w_packed || !out_w_packed || !x_hat) return VQB_ERR_BAD_ARG;
    if (B <= 0 || Cin <= 0 || H <= 0 || W <= 0 || C <= 0 || Cout <= 0) return VQB_ERR_BAD_ARG;
    if (relu_out != 0 && relu_out != 1) return VQB_ERR_BAD_ARG;
    return launch_decoder_tail(d_out, convt_w_packed, convt_bias, out_w_packed, out_bias, h_out, x_hat, B, Cin, H, W, C,
                               Cout, relu_out, (cudaStream_t)stream);
}

extern "C" int vqb_decoder_tail_supported(int Cin, int H, int W, int C, int Cout) {
    return decoder_tail_supported(Cin, H, W, C, Cout) ? 1 : 0;
}

// Thin stream-ordered copy for the host-buffer front end (vqvae_b200/pipeline.py): one ctypes call instead of
// a torch stream context + Tensor.copy_ per transfer (the Python overhead per step was larger than the kernels).
extern "C" int vqb_memcpy_async(void *dst, const void *src, size_t bytes, int kind, void *stream) {
    if (!dst || !src) return VQB_ERR_BAD_ARG;
    if (bytes == 0) return 0;
    if (kind < 1 || kind > 3) return VQB_ERR_BAD_ARG;
    // Driver entry point (unified addressing: the driver knows which side is pinned host memory).  The copy must
    // not go through THIS library's statically linked runtime: host buffers pinned by another runtime instance
    // (torch's) were copied at pageable speed, synchronously, through cudaMemcpyAsync (measured: 8 GB/s).
    typedef int (*PFN_cuMemcpyAsync)(unsigned long long, unsigned long long, size_t, void *);
    static PFN_cuMemcpyAsync fn = [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuMemcpyAsync", &p, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            p = nullptr;
        return reinterpret_cast<PFN_cuMemcpyAsync>(p);
    }();
    static const bool use_rt = [] { const char *e = vqb_getenv("VQB_MEMCPY_RUNTIME"); return e && e[0] == '1'; }();
    if (fn && !use_rt) {
        const int rc = fn((unsigned long long)(uintptr_t)dst, (unsigned long long)(uintptr_t)src, bytes, stream);
        return rc == 0 ? 0 : VQB_ERR_BAD_ARG;
    }
    const cudaMemcpyKind k = kind == 1 ? cudaMemcpyHostToDevice : kind == 2 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    return vqb_cuda_status(cudaMemcpyAsync(dst, src, bytes, k, (cudaStream_t)stream));
}

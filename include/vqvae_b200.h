/*
 * vqvae_b200.h -- C ABI of the H100 (sm_90a) VQ-VAE inference hot path.
 *
 * The reference (MishaLaskin/vqvae) is pure Python on top of PyTorch and exposes no
 * FFI of its own (SURVEY.md 8b); its "plugin API" for this path is the nn.Module
 * tree models.{vqvae,quantizer,encoder,decoder,residual}.  This header is the
 * boundary UNDER those modules: each entry point replaces one PyTorch operator call
 * site of the reference (file:line cited per function, paths under the reference
 * root).  models/*.py in this repo binds them with ctypes; INTEGRATION.md shows the
 * stub a maintainer of the reference would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (PyTorch in practice)
 *     unless stated otherwise;
 *     the library never allocates, frees or retains device memory;
 *   - `stream` is a cudaStream_t passed as void*; all calls are asynchronous, make no
 *     host synchronisation and are CUDA-graph capturable;
 *   - one CUDA device per process (the deployment model is one process per GPU,
 *     SURVEY.md 8e): the opt-in shared-memory size of each kernel is configured once
 *     per process, on the device that is current at its first launch; calls may come
 *     from any host thread but are not re-entrant on the same workspace;
 *   - host pointers appear only in vqb_memcpy_async and the weight tables of the
 *     vqb_prior_* entry points;
 *   - return value: 0 = success, >0 = cudaError_t, <0 = vqb_status below; no C++
 *     exception crosses the boundary;
 *   - activations between layers are NHWC ("pixel rows": (B*H*W, C) row-major); the
 *     module boundary of the reference is NCHW, so every conv entry point takes an
 *     explicit layout for its input and output.
 */
#ifndef VQVAE_B200_H
#define VQVAE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VQB_ABI_VERSION 3

enum vqb_status {
    VQB_OK = 0,
    VQB_ERR_BAD_ARG = -1,       /* NULL pointer, non-positive size, bad enum          */
    VQB_ERR_UNSUPPORTED = -2,   /* shape outside what the kernels implement          */
    VQB_ERR_WORKSPACE = -3,     /* workspace too small (see *_workspace_bytes)       */
    VQB_ERR_NO_DEVICE = -4,     /* no sm_90 device / driver                          */
    VQB_ERR_ALIGNMENT = -5      /* pointer not aligned as documented                 */
};

enum vqb_layout { VQB_NCHW = 0, VQB_NHWC = 1 };

/* arithmetic of a convolution entry point that takes fp32 activations (vqb_conv2d_f32,
 * vqb_residual_*_f32).  VQB_BF16 names the bf16-operand pipeline, whose activations are bf16:
 * the *_f32 entry points answer VQB_ERR_UNSUPPORTED to it -- use vqb_conv2d_bf16 & co.   */
enum vqb_precision {
    VQB_FP32 = 0,  /* fp32 FFMA accumulate (CUDA cores): the reference's CPU numerics   */
    VQB_TF32 = 1,  /* wgmma tf32, fp32 accumulate (cuDNN's default)                    */
    VQB_BF16 = 2   /* wgmma on bf16 operands and activations (bf16 entry points only) */
};

int vqb_abi_version(void);
/* 0: release library -- never reads the environment, no diagnostic / work-skipping code paths
 * compiled in.  1: built with -DVQB_DIAG=1 (environment knobs for experiments).         */
int vqb_diag_build(void);
const char *vqb_error_string(int code);
/* SM count and compute capability of the current device. */
int vqb_device_info(int *sm_count, int *cc_major, int *cc_minor);

/* Number of kernels this process has launched through the library so far (bench.py
 * reports it as gpu_launches).                                                     */
unsigned long long vqb_launch_count(void);

/* ---- weight packing (once per load_state_dict) --------------------------------
 * nn.Conv2d weight (Cout,Cin,kh,kw)          encoder.py:29-36, residual.py:20-24,
 *                                            vqvae.py:16-17
 * nn.ConvTranspose2d weight (Cin,Cout,kh,kw) decoder.py:28-35   (transposed = 1)
 * -> `packed` holds Cout*Cin*kh*kw + 144*Cin floats (a larger buffer also does): the
 *    tap-major K-major rows [(r*kw+s)][co][ci] that every conv kernel reads; for a k4 s2
 *    transposed conv with Cout <= 4 the [9][16][Cin] form follows them: per input
 *    neighbour (dy, dx), the rows (sub-pixel phase, channel) of decoder.py:34-35.   */
int vqb_pack_conv_weight_f32(const float *w, float *packed, int Cout, int Cin, int kh,
                             int kw, int transposed, void *stream);

/* ---- convolution layers ---------------------------------------------------------
 * One call = one nn.Conv2d (transposed=0) or nn.ConvTranspose2d (transposed=1)
 * forward, optionally fused with what follows it in the reference:
 *   out = act( conv(in) + bias [+ skip] ),  act = ReLU if relu else identity
 * `skip` (NHWC, shape of out, may be NULL) implements `x + res_block(x)` of
 * residual.py:27-29; out_layout must be NHWC when skip is given.
 * w_packed comes from vqb_pack_conv_weight_f32.  Stride-2 transposed convs are run
 * as 4 sub-pixel phase launches.  Replaces: encoder.py:29-36 (stride 2/2/1, pad 1),
 * residual.py:20-24, vqvae.py:16-17 (1x1), decoder.py:28-35.                      */
int vqb_conv2d_f32(const float *in, const float *w_packed, const float *bias,
                   const float *skip, float *out, int B, int Cin, int H, int W, int Cout,
                   int kh, int kw, int stride, int pad, int transposed, int in_layout,
                   int out_layout, int relu, int precision, void *stream);

/* ---- bf16 activation path (VQB_BF16): wgmma kernels on bf16 operands ----------------------
 * Between layers the activations are bf16 NHWC; weights are packed to bf16 once per
 * load_state_dict; accumulation is fp32 in registers.  This is the arithmetic the reference
 * reaches through torch.autocast(dtype=torch.bfloat16) around vqvae.py:29-44 (SURVEY Q6).
 * The layer shapes are named, not parameterised:                                         */
enum vqb_conv_kind {
    VQB_CONV_K1 = 0,        /* nn.Conv2d k1 s1 p0           vqvae.py:16-17                 */
    VQB_CONV_K3 = 1,        /* nn.Conv2d k3 s1 p1           encoder.py:35-36               */
    VQB_CONVT_K3 = 2,       /* nn.ConvTranspose2d k3 s1 p1  decoder.py:28-29               */
    VQB_CONV_K4S2 = 3,      /* nn.Conv2d k4 s2 p1           encoder.py:32-33 (H, W even)   */
    VQB_CONVT_K4S2 = 4,     /* nn.ConvTranspose2d k4 s2 p1  decoder.py:31-32 (Cout % 32 == 0, Cout <= 128) */
    VQB_CONVT_K4S2_OUT = 5  /* same to Cout <= 4 channels, fp32 NCHW output: decoder.py:34-35 */
};
/* Bytes of the packed bf16 weight of one layer (0 = shape not covered: Cin % 64 != 0, ...). */
size_t vqb_conv_bf16_packed_bytes(int kind, int Cout, int Cin);
/* w: the layer's fp32 weight as PyTorch stores it ((Cout,Cin,kh,kw), or (Cin,Cout,kh,kw) for
 * the transposed kinds) -> `packed` (128-byte aligned): K-major bf16 rows, tap-major,
 * [kh*kw][Cout][Cin] (VQB_RES_W2: Cin zero padded to 64), or [9][16][Cin] for
 * VQB_CONVT_K4S2_OUT -- the layouts vqb_pack_conv_weight_f32 writes, in bf16.              */
int vqb_pack_conv_weight_bf16(const float *w, void *packed, int kind, int Cout, int Cin,
                              void *stream);
/* One layer forward on bf16 NHWC input (B,H,W,Cin):  out = act(conv(in) + bias).
 * out: bf16 NHWC, or fp32 NHWC when out_f32 != 0 (z_e for the bit-exact VQ), or fp32 NCHW
 * (B,Cout,2H,2W) for VQB_CONVT_K4S2_OUT.  All pointers 16-byte aligned.                   */
int vqb_conv2d_bf16(const void *in, const void *packed, const float *bias, void *out, int B,
                    int Cin, int H, int W, int Cout, int kind, int relu, int out_f32,
                    void *stream);

/* encoder.py:29-31 for the bf16 pipeline: fp32 NCHW image (B,3,H,W) -> bf16 NHWC (B,H/2,W/2,Cout),
 * Cout == 64; w_packed from vqb_pack_conv_weight_f32 (its fp32 K-major rows, as in the fp32
 * and tf32 modes).                                                                          */
int vqb_conv_in_bf16(const float *x, const float *w_packed, const float *bias, void *out, int B,
                     int H, int W, int Cout, int relu, void *stream);
/* VectorQuantizer core for the bf16 pipeline: as vqb_vq_forward_f32 (fp32 z, bit-exact idx,
 * final sse) but zq is written as bf16 rows (N, D); D == 64 only.                            */
int vqb_vq_forward_bf16zq_f32(const float *z, const float *codebook, int64_t N, int K, int D,
                              int64_t *idx, void *zq_bf16, double *sse, int32_t *hist,
                              void *workspace, size_t workspace_bytes, void *stream);

/* One ResidualLayer application on bf16 NHWC activations (residual.py:18-29 as evaluated,
 * SURVEY Q2):  out = act( r + W2 . relu( W1 (*) r ) ),  act = ReLU iff relu_out.
 * w1_packed: vqb_pack_conv_weight_bf16(kind VQB_CONV_K3, Cout = Cmid, Cin = C) of res_block.1.weight;
 * w2_packed: vqb_pack_conv_weight_bf16(kind VQB_RES_W2 = 6, Cout = C, Cin = Cmid) of res_block.3.weight.
 * One wgmma launch: per 128-pixel tile both GEMMs chained, the bf16 intermediate and W2 in shared memory.
 * C in {64, 128}, Cmid % 16 == 0, Cmid <= 64; other shapes return VQB_ERR_UNSUPPORTED.      */
#define VQB_RES_W2 6
int vqb_residual_layer_bf16(const void *r, const void *w1_packed, const void *w2_packed, void *out,
                            int B, int H, int W, int C, int Cmid, int relu_out, void *stream);

/* ---- one ResidualLayer application, residual.py:18-29 -----------------------------
 * As the reference evaluates it (the in-place ReLU of :19 has already replaced x by
 * r = relu(x), SURVEY Q2):   out = act( r + W2 . relu( W1 (*) r ) )
 * r, out NHWC (B,H,W,C); W1 = res_block.1.weight (Cmid,C,3,3), W2 = res_block.3.weight
 * (C,Cmid,1,1), both packed by vqb_pack_conv_weight_f32; act = ReLU iff relu_out (inside
 * a ResidualStack the next consumer always applies ReLU first, residual.py:19,50).
 * tmp: B*H*W*Cmid floats of scratch (used only by the two-launch paths).
 * With precision VQB_TF32, C in {64, 128} and Cmid in {32, 64} this is ONE wgmma launch
 * (two chained GEMMs, the Cmid-channel intermediate never leaves the SM).            */
int vqb_residual_layer_f32(const float *r, const float *w1_packed, const float *w2_packed,
                           float *out, float *tmp, int B, int H, int W, int C, int Cmid,
                           int relu_out, int precision, void *stream);

/* ---- a whole ResidualStack, residual.py:45-51 --------------------------------------
 * n_layers applications of ONE shared-weight layer (residual.py:43 builds the list as
 * [layer] * n), each followed by the ReLU its consumer applies (the next layer's in-place
 * ReLU, or the stack's F.relu at :50):  r_{i+1} = relu( r_i + W2 . relu( W1 (*) r_i ) ),
 * r_0 = r = relu(stack input), out = r_{n_layers}.   r, out NHWC (B,H,W,C).
 * scratch: B*H*W*C floats (needed when n_layers > 1; used when the applications run as
 * separate launches), tmp: B*H*W*Cmid floats (two-launch paths only).
 * With precision VQB_TF32, the layer shapes the one-launch vqb_residual_layer_f32 takes and
 * whole images per 128-pixel tile (pow2(W) <= 16 and pow2(W) * pow2(H) <= 128), ALL
 * applications run inside ONE wgmma launch: each tile's output goes to `out` and is read
 * back by the next application (no other CTA touches those images).                   */
int vqb_residual_stack_f32(const float *r, const float *w1_packed, const float *w2_packed,
                           float *out, float *scratch, float *tmp, int B, int H, int W, int C,
                           int Cmid, int n_layers, int precision, void *stream);

/* ---- the latent block of a VQVAE forward in one launch, TF32 only -------------------
 * head: out0 = relu( conv(x) + head_bias ), the k3 s1 p1 layer that feeds the stack:
 *   nn.Conv2d(Cin, C) (head_transposed = 0, encoder.py:35) or nn.ConvTranspose2d(Cin, C)
 *   (head_transposed = 1, decoder.py:28); x NHWC (B,H,W,Cin), head_w_packed from
 *   vqb_pack_conv_weight_f32; head_bias may be NULL.
 * then the ResidualStack of vqb_residual_stack_f32 on out0 (n_layers >= 1, w1/w2 as there),
 * then, when tail_cout > 0, the 1x1 conv C -> tail_cout of vqvae.py:16-17 (tail_w_packed
 * from vqb_pack_conv_weight_f32, + tail_bias, may be NULL), whose output replaces the stack's.
 * tail_w_packed must be NULL exactly when tail_cout == 0 (VQB_ERR_BAD_ARG otherwise).
 * out: NHWC (B,H,W,C), or the (B*H*W, tail_cout) rows of z_e with the tail.
 * Bitwise the separate calls (vqb_conv2d_f32 with VQB_TF32, vqb_residual_stack_f32 [,
 * vqb_conv2d_f32 1x1]).  Shapes: those vqb_residual_stack_f32 runs in one launch (C in {64,
 * 128}, Cmid = 32, whole images per 128-pixel tile), Cin % 32 == 0, Cin <= 256, tail_cout 0
 * or 64; anything else, x == out or a pointer not 16-byte aligned returns VQB_ERR_UNSUPPORTED
 * and launches nothing: run the separate calls then.
 * vqb_latent_block_supported answers 1 for the shapes vqb_latent_block_tf32 takes, else 0
 * (no CUDA call: callers ask before allocating the output).                               */
int vqb_latent_block_tf32(const float *x, const float *head_w_packed, const float *head_bias,
                          int head_transposed, const float *w1_packed, const float *w2_packed,
                          int n_layers, const float *tail_w_packed, const float *tail_bias,
                          int tail_cout, float *out, int B, int Cin, int H, int W, int C, int Cmid,
                          void *stream);
int vqb_latent_block_supported(int Cin, int H, int W, int C, int Cmid, int tail_cout);

/* ---- the decoder's last two layers in one launch, TF32 only -------------------------
 * h = relu( convT(d_out) + convt_bias ), the k4 s2 p1 nn.ConvTranspose2d(Cin, C) of
 *   decoder.py:31-33 on d_out NHWC (B,H,W,Cin),
 * x_hat = act( convT(h) + out_bias ), the k4 s2 p1 nn.ConvTranspose2d(C, Cout) of
 *   decoder.py:34-35, act = ReLU iff relu_out; x_hat fp32 NCHW (B,Cout,4H,4W).
 * Both weights packed by vqb_pack_conv_weight_f32; the biases may be NULL.  h_out: NULL, or
 * NHWC (B,2H,2W,C), which then receives h.  Bitwise the separate calls (vqb_conv2d_f32 with
 * VQB_TF32, NHWC out with ReLU, then NHWC in, NCHW out).  Shapes: C == 64, 1 <= Cout <= 4,
 * Cin % 32 == 0, Cin <= 256, whole latent images per 128-pixel tile (pow2(W) <= 16 and
 * pow2(W) * pow2(H) <= 128); anything else, d_out aliasing an output or a pointer not
 * 16-byte aligned returns VQB_ERR_UNSUPPORTED and launches nothing: run the separate calls
 * then.  vqb_decoder_tail_supported answers 1 for the shapes vqb_decoder_tail_tf32 takes,
 * else 0 (no CUDA call).                                                                  */
int vqb_decoder_tail_tf32(const float *d_out, const float *convt_w_packed, const float *convt_bias,
                          const float *out_w_packed, const float *out_bias, float *h_out,
                          float *x_hat, int B, int Cin, int H, int W, int C, int Cout,
                          int relu_out, void *stream);
int vqb_decoder_tail_supported(int Cin, int H, int W, int C, int Cout);

/* ---- VectorQuantizer.forward, quantizer.py:45-76 --------------------------------
 * z        (N, D) fp32 pixel rows (= z.permute(0,2,3,1).view(-1, e_dim), :45-46)
 * codebook (K, D) fp32 embedding.weight (:26)
 * idx      (N)    int64 min_encoding_indices, first minimum wins, NaN wins (:54)
 * zq       (N, D) fp32 straight-through value fl(z + fl(e_idx - z)) (:60,:67)
 * hist     (K)    int32 code counts, ZEROED by the call (column sums of the one-hot
 *                 of :55-57; feeds the perplexity of :70-71)
 * sse      (1)    double, sum of fl(e_idx - z)^2, OVERWRITTEN by the call (numerator
 *                 of the two mean() terms of :63-64)
 * workspace       vqb_vq_workspace_bytes(N,K,D) bytes, 16-byte aligned
 * Distances follow the canonical fp32 order documented in DESIGN.md / oracle.c, so
 * idx and zq are bit-exact against the oracle.                                    */
size_t vqb_vq_workspace_bytes(int64_t N, int K, int D);
int vqb_vq_forward_f32(const float *z, const float *codebook, int64_t N, int K, int D,
                       int64_t *idx, float *zq, double *sse, int32_t *hist,
                       void *workspace, size_t workspace_bytes, void *stream);

/* Kernel choice of vqb_vq_forward_f32: 0 = auto (see vqb_vq_forward_f32's dispatch),
 * 1 = always the exact FFMA kernel, 2 = require the wgmma kernel (TF32 candidate
 * selection + canonical fp32 re-scoring; D == 64, 1 <= K <= 2^20); anything else is
 * VQB_ERR_BAD_ARG.  All produce bit-identical idx / zq; the switch exists for tests
 * and benchmarks.                                                                     */
int vqb_set_vq_kernel(int which);

/* Diagnostic twin of vqb_vq_forward_f32 (wgmma kernel, D == 64): additionally dumps the
 * approximate TF32 scores s = ||e||^2 - 2 z.e as (N, ceil(K/256)*256) floats.        */
int vqb_debug_vq_scores_f32(const float *z, const float *codebook, int64_t N, int K, int D,
                            int64_t *idx, float *zq, double *sse, int32_t *hist,
                            void *workspace, size_t workspace_bytes, float *scores,
                            void *stream);

/* ---- backward of VectorQuantizer.forward, quantizer.py:63-67 (training-mode callers, main.py:74-79) ----
 * g_zq (N,D) = gradient arriving at the returned z_q (straight-through: passes to z unchanged), g_loss = device
 * scalar gradient of the returned loss (either may be NULL = zero).  Writes
 *   dz (N,D) = g_zq + g_loss * 2/(N D) * (z - E[idx])
 *   dE (K,D) = g_loss * 2 beta/(N D) * sum_{i: idx[i]=k} (E[k] - z[i])      (zeroed, then scatter-added by index)
 * argmin / one-hot / perplexity carry no gradient.  D % 4 == 0, 16-byte aligned pointers.                */
int vqb_vq_backward_f32(const float *g_zq, const float *g_loss, const float *z, const float *codebook,
                        const int64_t *idx, int64_t N, int K, int D, float beta, float *dz, float *dE,
                        void *stream);

/* loss = (1+beta)*sse/(N*D) and perplexity = exp(-sum p log(p+1e-10)), p = hist/N,
 * written as two fp32 device scalars (quantizer.py:63-64, :70-71).  Separate from
 * the VQ kernel so a batch-sharded caller can all-reduce (hist, sse) in between.  */
int vqb_vq_finish_f32(const double *sse, const int32_t *hist, int64_t N, int K, int D,
                      float beta, float *loss, float *perplexity, void *stream);

/* ---- exponential-moving-average codebook (VectorQuantizer(decay=...), van den Oord et al. 2017, A.1) ----
 * One update from the rows z (N,D) fp32 that vqb_vq_forward_f32 quantized, their codes idx (N) int64 (clamped to
 * [0, K-1]) and its hist (K) int32 (n_k):
 *   cluster_size N_k <- decay N_k + (1-decay) n_k        embed_sum m_k <- decay m_k + (1-decay) s_k
 *   n = sum_k N_k,   codebook e_k <- m_k / ((N_k + eps) / (n + K eps) * n)          (all three in place, fp32)
 * s_k = sum of the rows of code k in a fixed order: by ascending row index, in consecutive segments of 256 rows, each
 * one fp32 add chain, the segment partials added in segment order; the result bits depend on (z, idx) only.  Five
 * launches, no float atomics, no host synchronisation.  decay in [0, 1), eps finite and > 0 and NULL pointers:
 * VQB_ERR_BAD_ARG; D % 4 != 0: VQB_ERR_UNSUPPORTED; both before any launch.  z, embed_sum, codebook and the
 * workspace (vqb_vq_ema_workspace_bytes(N,K,D) bytes, 0 for a shape it refuses) 16-byte aligned.              */
size_t vqb_vq_ema_workspace_bytes(int64_t N, int K, int D);
int vqb_vq_ema_update_f32(const float *z, const int64_t *idx, const int32_t *hist, int64_t N, int K,
                          int D, float decay, float eps, float *cluster_size, float *embed_sum,
                          float *codebook, void *workspace, size_t workspace_bytes, void *stream);

/* Dead-code restart, run after vqb_vq_ema_update_f32 on the same rows z (N,D) fp32 and state, with uniforms u (N)
 * fp32 in [0, 1) and a threshold t:
 *   dead codes k_0 < k_1 < ... < k_{M-1}: cluster_size N_k < t (strict; a NaN N_k is not dead)
 *   rows r_0, r_1, ...: the rows ordered by (u_i, i) ascending (uniform sampling without replacement)
 *   for j < R = min(M, N):  codebook e_{k_j} <- z_{r_j},  embed_sum m_{k_j} <- fl(t z_{r_j}),  N_{k_j} <- t
 *   *n_restarted (int32, device) <- R;  every other element keeps its bits.
 * Twelve launches, no float atomics, no host synchronisation; with no dead code every kernel after the first returns
 * at once.  NULL pointers, N, K or D <= 0, t not finite or <= 0: VQB_ERR_BAD_ARG; D % 4 != 0, K > 8192 or
 * N > 2^32 - 1: VQB_ERR_UNSUPPORTED; a workspace shorter than vqb_vq_ema_restart_workspace_bytes(N,K) (0 for a shape
 * it refuses): VQB_ERR_WORKSPACE; all before any launch.  z, embed_sum, codebook and the workspace 16-byte aligned. */
size_t vqb_vq_ema_restart_workspace_bytes(int64_t N, int K);
int vqb_vq_ema_restart_f32(const float *z, const float *u, int64_t N, int K, int D, float threshold,
                           float *cluster_size, float *embed_sum, float *codebook, int32_t *n_restarted,
                           void *workspace, size_t workspace_bytes, void *stream);

/* k-means initialisation of a codebook (K, D) fp32 from rows z (N, D) fp32, N >= K, with uniforms u (N) fp32 in [0, 1):
 *   seed: code j <- the row of rank j when the rows are ordered by (u_i, i) ascending (vqb_vq_ema_restart_f32's
 *         sampling without replacement, with every code dead), copied exactly
 *   then iters Lloyd steps, t = 0 .. iters-1:  idx and sse[t] from vqb_vq_forward_f32 on the current codebook (the
 *         canonical fp32 distances; sse[t] is the inertia before step t); n_k and s_k as vqb_vq_ema_update_f32 forms
 *         them; e_k <- fl(s_k / (float)n_k) where n_k > 0 (a code no row picks keeps its bits)
 * sse: iters doubles, may be NULL iff iters == 0.  Non-finite rows are used as they are: a row holding a NaN takes
 * code 0 (NaN wins the argmin), whose centroid then turns NaN and takes every row -- the call cannot check for one
 * without a host synchronisation.  12 + iters * (v + 5) launches, v = vqb_vq_forward_f32's launches for the shape (2 on
 * the tensor-core kernel, 3 on the exact kernel); no float atomics, no host synchronisation, CUDA-graph capturable.
 * NULL pointers, N, K or D <= 0, N < K, iters < 0: VQB_ERR_BAD_ARG; D % 4 != 0, K > 8192, N > 2^32 - 1, or a shape the
 * VQ dispatch refuses when iters > 0: VQB_ERR_UNSUPPORTED; a workspace shorter than
 * vqb_vq_kmeans_workspace_bytes(N,K,D) (0 for a shape it refuses): VQB_ERR_WORKSPACE; all before any launch.
 * z, codebook and the workspace 16-byte aligned.                                                                  */
size_t vqb_vq_kmeans_workspace_bytes(int64_t N, int K, int D);
int vqb_vq_kmeans_f32(const float *z, const float *u, int64_t N, int K, int D, int iters, float *codebook,
                      double *sse, void *workspace, size_t workspace_bytes, void *stream);

/* Backward of the EMA quantizer, whose loss is the commitment term alone (the codebook gets no gradient):
 *   dz (N,D) = g_zq + g_loss * 2 beta/(N D) * (z - zq)
 * zq = the forward's fp32 z_q rows (not the codebook, which the update has overwritten).  g_zq / g_loss may be
 * NULL (= zero).  One launch, no atomics.  D % 4 == 0, 16-byte aligned pointers.                              */
int vqb_vq_commit_backward_f32(const float *g_zq, const float *g_loss, const float *z, const float *zq,
                               int64_t N, int D, float beta, float *dz, void *stream);

/* vqb_vq_finish_f32 for the EMA quantizer: loss = beta * sse/(N*D) (fp32), the same perplexity.             */
int vqb_vq_finish_ema_f32(const double *sse, const int32_t *hist, int64_t N, int K, int D,
                          float beta, float *loss, float *perplexity, void *stream);

/* Dense one-hot min_encodings (N,K) fp32 for direct VectorQuantizer.forward callers
 * (quantizer.py:55-57,76); VQVAE.forward discards it (vqvae.py:34) so it is never
 * built on that path.                                                             */
int vqb_onehot_f32(const int64_t *idx, int64_t N, int K, float *onehot, void *stream);

/* z_q rows from indices: matmul(one_hot, embedding.weight) of quantizer.py:60 and of
 * the notebook's generate_samples (visualization.ipynb cell 13) as a row gather.
 * Indices outside [0, K) are clamped to the nearest valid row.                    */
int vqb_gather_rows_f32(const int64_t *idx, const float *codebook, int64_t N, int K, int D,
                        float *rows, void *stream);

/* In-place ReLU over n floats: the nn.ReLU(True) of residual.py:19, which mutates
 * the caller's tensor when a ResidualLayer is called directly (SURVEY Q2).         */
int vqb_relu_f32(float *x, int64_t n, void *stream);

/* Gradient through a ReLU from its kept output y: out = y > 0 ? g : 0 over n floats (out may be g).
 * The backward of VQVAE.forward's ReLUs (residual.py:19,21,50, encoder.py:30,33, decoder.py:33). */
int vqb_relu_backward_f32(const float *g, const float *y, float *out, int64_t n, void *stream);

/* ---- layout changes at the module boundary (quantizer.py:45, :74) ---------------- */
int vqb_nchw_to_nhwc_f32(const float *in, float *out, int B, int C, int H, int W, void *stream);
int vqb_nhwc_to_nchw_f32(const float *in, float *out, int B, int C, int H, int W, void *stream);
/* The same changes between C real channels and Cp >= C stored ones (a standalone GatedMaskedConv2d at a dim the prior
 * kernels run padded, VQB_PACK_PRIOR_PAD_F32): NCHW (B,C,H,W) -> NHWC (B,H,W,Cp) with channels C..Cp-1 zero, and
 * NHWC (B,H,W,Cp) -> NCHW (B,C,H,W) reading channels 0..C-1 only.  One launch each.                              */
int vqb_nchw_to_nhwc_pad_f32(const float *in, float *out, int B, int C, int Cp, int H, int W, void *stream);
int vqb_nhwc_to_nchw_unpad_f32(const float *in, float *out, int B, int C, int Cp, int H, int W, void *stream);

/* Stream-ordered copy used by the host-buffer streaming front end (vqvae_b200.HostPipeline):
 * kind 1 = host -> device, 2 = device -> host, 3 = device -> device.  Host buffers should be
 * pinned (the copy is only asynchronous then).                                          */
int vqb_memcpy_async(void *dst, const void *src, size_t bytes, int kind, void *stream);

/* ---- weight gradient of one convolution layer (training VQVAE.forward, main.py:74-79) ------------------
 * dW (and dbias unless NULL) of the layer vqb_conv2d_f32 runs with the same geometry: `in` is the layer's
 * input (B,Cin,H,W) in in_layout, g_out the gradient of its output (B,Cout,OH,OW) in gout_layout.  dW is
 * written in the parameter's own layout, (Cout,Cin,kh,kw) or, transposed, (Cin,Cout,kh,kw); dbias (Cout).
 * Both are OVERWRITTEN.  Any kernel size, stride, padding and channel counts.  fp32 on CUDA cores; the
 * reduction over images and pixels runs in fixed chunks summed in a fixed order, with no atomics: two calls
 * give bitwise-equal results.  A weight applied several times (a shared ResidualLayer) gets one reduction
 * over all its applications when their inputs and output gradients are passed as one batch of n*B images.
 * 2 launches, 3 for a transposed conv with a bias.  workspace: vqb_conv_wgrad_workspace_bytes bytes,
 * enough with or without dbias (0 = bad geometry).                                                       */
size_t vqb_conv_wgrad_workspace_bytes(int B, int Cin, int H, int W, int Cout, int kh, int kw, int stride,
                                      int pad, int transposed);
int vqb_conv_wgrad_f32(const float *in, const float *g_out, float *dW, float *dbias, int B, int Cin, int H,
                       int W, int Cout, int kh, int kw, int stride, int pad, int transposed, int in_layout,
                       int gout_layout, void *workspace, size_t workspace_bytes, void *stream);

/* ---- Gated PixelCNN prior, pixelcnn/models.py (inference, fp32 on CUDA cores) ----------------------------
 * The prior over VQ code grids: teacher-forced logits (GatedPixelCNN.forward, models.py:121-130) and the whole
 * sampling loop (GatedPixelCNN.generate, :132-143) in one call.  Activations are NHWC rows.  Shapes: dim % 32 == 0
 * and dim <= 1024 (the reference script's dim = img_dim**2 up to 32x32 latents), 1 <= input_dim (K) <= 8192, 1 <= n_layers <= VQB_PRIOR_MAX_LAYERS, odd kernel <= 15, any
 * n_classes; other dims return VQB_ERR_UNSUPPORTED.  Out-of-range codes and labels are clamped to the nearest
 * valid row in the kernels (as vqb_gather_rows_f32 does): a host-side range check would need a device sync.
 * The weight tables below are HOST structs holding device pointers; they are read during the call only.     */
#define VQB_PRIOR_MAX_LAYERS 32
#define VQB_PRIOR_MAX_KERNEL 15

/* One GatedMaskedConv2d (models.py:29-86).  *_w from vqb_prior_pack_f32, *_b the conv biases, class_emb the
 * class_cond_embedding weight (n_classes, 2*dim).  vert_w keeps rows [0, kernel/2 + 1 - mask_a) of vert_stack's
 * (2dim, dim, kernel/2+1, kernel) weight, horiz_w columns [0, kernel/2 + 1 - mask_a) of horiz_stack's
 * (2dim, dim, 1, kernel/2+1) weight: mask A's zeroed taps (models.py:61-63) are not stored.                   */
typedef struct vqb_prior_layer_weights {
    const float *vert_w, *vert_b, *v2h_w, *v2h_b, *horiz_w, *horiz_b, *resid_w, *resid_b, *class_emb;
    int kernel, mask_a, residual;
} vqb_prior_layer_weights;

/* The whole GatedPixelCNN: `layers` is a host array of n_layers entries; embedding (input_dim, dim);
 * output_conv.0 (dim -> 512) and output_conv.2 (512 -> input_dim) packed by vqb_prior_pack_f32 (1x1).        */
typedef struct vqb_prior_net {
    const vqb_prior_layer_weights *layers;
    int n_layers;
    const float *embedding, *out1_w, *out1_b, *out2_w, *out2_b;
    int input_dim, dim, n_classes;
} vqb_prior_net;

/* Conv weight (Cout, Cin, kh, kw) -> [(r*cols + s)*Cin + ci][co] for the taps r < rows, s < cols.            */
int vqb_prior_pack_f32(const float *w, float *packed, int Cout, int Cin, int kh, int kw, int rows, int cols,
                       void *stream);
/* Workspace of vqb_prior_forward_f32 and vqb_prior_generate_f32 on a (B, H, W) grid (0 = bad sizes).        */
size_t vqb_prior_workspace_bytes(int B, int H, int W, int dim, int n_layers, int K);
/* GatedActivation (models.py:20-26): x (outer, 2C, inner) -> out (outer, C, inner) = tanh(x_a) * sigmoid(x_b). */
int vqb_prior_gate_f32(const float *x, float *out, int64_t outer, int C, int64_t inner, void *stream);
/* GatedMaskedConv2d.forward (models.py:65-86) on NHWC x_v, x_h (B,H,W,dim), labels (B) int64 ->
 * out_v, out_h NHWC (B,H,W,dim); vh: B*H*W*2*dim floats of scratch.  Two launches.                        */
int vqb_prior_layer_f32(const vqb_prior_layer_weights *layer, const float *x_v, const float *x_h,
                        const int64_t *labels, int B, int H, int W, int dim, int n_classes, float *out_v,
                        float *out_h, float *vh, void *stream);
/* GatedPixelCNN.forward: codes (B,H,W) int64, labels (B) int64 -> logits (B, input_dim, H, W) fp32 NCHW.
 * 2 + 2*n_layers launches.                                                                               */
int vqb_prior_forward_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H,
                          int W, float *logits, void *workspace, size_t workspace_bytes, void *stream);
/* GatedPixelCNN.generate: samples codes (B,H,W) int64 in raster order.  Code (b,i,j) is the smallest k with
 * u[b,i,j] < CDF_k, CDF the fp32 running sum of the softmax of the logits at (i,j) (DESIGN.md gives the order).
 * u: (B,H,W) uniforms in [0,1).  H*(n_layers + W) launches: per row one vertical-stack pass per layer, then one
 * launch per position running every layer's horizontal stack, the head and the draw.  No host synchronisation.
 * The workspace keeps min(H, VQB_PRIOR_MAX_KERNEL/2 + 1) rows of each layer's vertical output, the most a later
 * layer reads (a layer with kernel k reads k/2 + 1 rows of the previous one's).  Layer 0 must be mask A without residual (anything else reads the code being drawn, so the logits are not
 * causal in raster order): VQB_ERR_UNSUPPORTED before any launch otherwise.
 * step_logits: NULL, or (B,H,W,input_dim) fp32 receiving the logits each step sampled from -- bitwise equal to
 * vqb_prior_forward_f32's logits on the returned codes.                                                    */
int vqb_prior_generate_f32(const vqb_prior_net *net, const int64_t *labels, const float *u, int B, int H, int W,
                           int64_t *codes, float *step_logits, void *workspace, size_t workspace_bytes,
                           void *stream);
/* Workspace of vqb_prior_complete_f32 for any n_given: at least vqb_prior_workspace_bytes, plus every layer's
 * vertical output as a whole grid, 4*n_layers*B*H*W*dim bytes (0 = bad sizes).                               */
size_t vqb_prior_complete_workspace_bytes(int B, int H, int W, int dim, int n_layers, int K);
/* GatedPixelCNN completion: the raster positions p = i*W + j < n_given of every image are given, the rest are
 * sampled as vqb_prior_generate_f32 samples them.  given (B,H,W) int64: codes[b,p] = given[b,p] for p < n_given,
 * as given (out-of-range values included; the kernels clamp them where they embed them); given[b,p] for
 * p >= n_given is never read.  Code (b,p) for p >= n_given is the smallest k with u[b,p] < CDF_k of that step's
 * logits, which are bitwise vqb_prior_forward_f32's logits at p on the returned codes (clamped); so with the same
 * u, completing a prefix of vqb_prior_generate_f32's output returns that output bitwise.  u at p < n_given is
 * not read; step_logits (NULL or (B,H,W,input_dim)) is written only at p >= n_given.
 * With i0 = n_given / W and j0 = n_given % W: one launch copies the given codes and embeds them; if i0 > 0, one
 * launch per layer computes its vertical output on rows [0, i0); rows i0 .. H-1 then run as in generate, with, in
 * row i0 when j0 > 0, one launch per layer of horizontal stacks over columns [0, j0) before the steps from j0.
 * 0 < n_given < H*W: 1 + n_layers*[i0 > 0] + n_layers*(H - i0) + n_layers*[j0 > 0] + (H*W - n_given) launches;
 * n_given = 0 is vqb_prior_generate_f32 (its launches and codes); n_given = H*W is the copy alone.
 * workspace: n_given < W needs vqb_prior_workspace_bytes (generate's rings), n_given >= W
 * vqb_prior_complete_workspace_bytes (whole-grid vertical outputs).  VQB_ERR_BAD_ARG for n_given outside
 * [0, H*W]; VQB_ERR_UNSUPPORTED, before any launch, for a layer 0 generate refuses.  No host synchronisation.  */
int vqb_prior_complete_f32(const vqb_prior_net *net, const int64_t *labels, const float *u, const int64_t *given,
                           int64_t n_given, int B, int H, int W, int64_t *codes, float *step_logits,
                           void *workspace, size_t workspace_bytes, void *stream);
/* The draw's knobs, one set for the whole batch.  With z = l / T in fp32 (saturated to +-FLT_MAX) and fkey the
 * order-preserving map from fp32 to uint32, the kept set is S = {k : fkey(z_k) >= t}, t = max(t_k, t_p):
 *   t_k  the largest t with at least top_k codes kept (ties at the threshold are kept);
 *   t_p  the largest t whose kept codes hold at least top_p of the tempered softmax expf(z - max) / sum.
 * top_k = 0 (or K) and top_p = 1 turn their truncation off; temperature 1, top_k 0, top_p 1 is generate's draw.   */
typedef struct vqb_prior_sampling {
    float temperature;                        /* finite, > 0 */
    int top_k;                                /* 0 (off) .. input_dim */
    float top_p;                              /* (0, 1]; 1 is off */
} vqb_prior_sampling;
/* Workspace of vqb_prior_sample_f32 from raster position n_given: at least what vqb_prior_complete_f32 needs there,
 * plus 256*ceil(input_dim/32) + 4 bytes per image for the kept-set search and log_prob (0 = bad sizes or n_given outside [0, H*W]). */
size_t vqb_prior_sample_workspace_bytes(int B, int H, int W, int dim, int n_layers, int K, int64_t n_given);
/* vqb_prior_complete_f32 (n_given = 0: vqb_prior_generate_f32) drawing each code from the softmax of that step's
 * tempered logits truncated to S: the smallest k in S with u < CDF_k, CDF the fp32 running sum over S of
 * q_k = expf(z_k - max) / sum over S, in generate's order (the last k in S with q_k > 0 if rounding leaves u above
 * the total).  sampling NULL, or knobs off, is complete's draw: the same codes and step logits, bit for bit.
 * log_prob: NULL, or (B) fp32 receiving, per image, the compensated (Kahan) fp32 sum in raster order over the
 * sampled positions of l_code - max(l) - logf(sum expf(l - max(l))), the model's untempered, untruncated
 * log-probability (0 when n_given = H*W).  step_logits stay the raw logits.  given may be NULL when n_given = 0.  The same launches as
 * vqb_prior_complete_f32 for this n_given, no host synchronisation, the knobs passed as kernel arguments.
 * VQB_ERR_BAD_ARG for a knob outside its range, VQB_ERR_UNSUPPORTED for a layer 0 generate refuses, both before
 * any launch.                                                                                                    */
int vqb_prior_sample_f32(const vqb_prior_net *net, const int64_t *labels, const float *u, const int64_t *given,
                         int64_t n_given, int B, int H, int W, const vqb_prior_sampling *sampling, int64_t *codes,
                         float *log_prob, float *step_logits, void *workspace, size_t workspace_bytes, void *stream);
/* vqb_prior_sample_f32 with one prefix length per image: n_given (B) int64 on the device, never read on the host, so
 * a captured graph follows new values written there.  Each value is clamped to [0, H*W], as codes and labels are.
 * Image b's codes, log_prob[b] and step logits are bitwise those of vqb_prior_sample_f32 on image b alone with
 * n_given = clamp(n_given[b]) and the same u and knobs (log_prob[b] = 0 when that is H*W); step_logits are written
 * at image b's positions >= n_given[b] only.  sampling NULL is complete's draw (the ragged complete), log_prob may
 * be NULL, given may not.  Schedule: one launch copies and embeds every image's given prefix, then generate's
 * row passes and steps, each step skipping the images that have that position given: 1 + H*(n_layers + W) launches
 * whatever the values.  workspace: vqb_prior_sample_workspace_bytes(..., n_given = 0) (generate's rings and the
 * draw's scratch).  VQB_ERR_BAD_ARG for a NULL given or n_given and for vqb_prior_sample_f32's other bad
 * arguments; VQB_ERR_UNSUPPORTED for a layer 0 generate refuses; both before any launch.                        */
int vqb_prior_sample_ragged_f32(const vqb_prior_net *net, const int64_t *labels, const float *u,
                                const int64_t *given, const int64_t *n_given, int B, int H, int W,
                                const vqb_prior_sampling *sampling, int64_t *codes, float *log_prob,
                                float *step_logits, void *workspace, size_t workspace_bytes, void *stream);

/* ---- Gated PixelCNN prior, training (fp32 on CUDA cores) ------------------------------------------------------
 * The forward keeps its activations in `saved`; the backward turns d_logits into the gradient of every parameter.
 * Shape limits and argument checks are those of vqb_prior_forward_f32.                                          */
/* Bytes of `saved` on a (B, H, W) grid: 4*B*H*W*(dim*(6*n_layers + 3) + 512) (0 = bad sizes).                   */
size_t vqb_prior_train_saved_bytes(int B, int H, int W, int dim, int n_layers);
/* vqb_prior_forward_f32 that also stores, per layer, x_v, x_h, h_vert (bias included, class embedding not) and the
 * horizontal gate's pre-activation, and the head's 512-wide hidden layer.  The same kernels and arithmetic: the
 * logits are bitwise those of vqb_prior_forward_f32.  2 + 2*n_layers launches.                                   */
int vqb_prior_forward_train_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H,
                                int W, float *logits, void *saved, size_t saved_bytes, void *stream);

/* Device output pointers of every gradient, shaped like vqb_prior_layer_weights / vqb_prior_net, each in its
 * parameter's own layout: (Cout, Cin, kh, kw) for the convs, (rows, cols) for the embeddings.  The conv gradients
 * cover all kh*kw taps, mask A's included.                                                                        */
typedef struct vqb_prior_layer_grads {
    float *vert_w, *vert_b, *v2h_w, *v2h_b, *horiz_w, *horiz_b, *resid_w, *resid_b, *class_emb;
} vqb_prior_layer_grads;

typedef struct vqb_prior_grads {
    const vqb_prior_layer_grads *layers;      /* host array of n_layers entries */
    int n_layers;
    float *embedding, *out1_w, *out1_b, *out2_w, *out2_b;
} vqb_prior_grads;

/* Workspace of vqb_prior_backward_f32 for this net on a (B, H, W) grid (0 = bad arguments).                     */
size_t vqb_prior_backward_workspace_bytes(const vqb_prior_net *net, int B, int H, int W);
/* Gradients of every parameter from d_logits (B, input_dim, H, W) fp32 NCHW, codes, labels and the `saved` of a
 * vqb_prior_forward_train_f32 call with the same net and inputs.  Overwrites every gradient (no accumulation).
 * Deterministic: fixed-order sums, no atomics; two calls give bitwise-equal gradients.  No host synchronisation.
 * 7 + 10*n_layers launches.                                                                                      */
int vqb_prior_backward_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H, int W,
                           const float *d_logits, const void *saved, const vqb_prior_grads *grads, void *workspace,
                           size_t workspace_bytes, void *stream);

/* One layer and the gate on their own (GatedMaskedConv2d / GatedActivation called as modules).  The same rules as the
 * net: fp32, no float atomics (two calls give bitwise-equal results), no host synchronisation, argument checks
 * before any launch, and vqb_prior_layer_f32's shape limits.                                                    */
/* GatedActivation's backward: x (outer, 2C, inner) and d_out (outer, C, inner) -> d_x (outer, 2C, inner).  One
 * launch.                                                                                                        */
int vqb_prior_gate_backward_f32(const float *x, const float *d_out, float *d_x, int64_t outer, int C, int64_t inner,
                                void *stream);
/* Bytes of a layer's `saved` on a (B, H, W) grid: 16*B*H*W*dim (0 = bad sizes).                                  */
size_t vqb_prior_layer_train_saved_bytes(int B, int H, int W, int dim);
/* vqb_prior_layer_f32 that also stores h_vert (bias included, class embedding not) and the horizontal gate's
 * pre-activation in `saved`; vh is the same B*H*W*2*dim floats of scratch, free after the call.  out_v and out_h
 * are bitwise vqb_prior_layer_f32's.  Two launches.                                                              */
int vqb_prior_layer_forward_train_f32(const vqb_prior_layer_weights *layer, const float *x_v, const float *x_h,
                                      const int64_t *labels, int B, int H, int W, int dim, int n_classes,
                                      float *out_v, float *out_h, float *vh, void *saved, size_t saved_bytes,
                                      void *stream);
/* Workspace of vqb_prior_layer_backward_f32 (0 = bad arguments).  This pair keeps the dim <= 256 limit it was
 * published with (VQB_ERR_UNSUPPORTED / 0 above it); vqb_prior_layer_backward_wide_* below take every dim the net
 * takes.                                                                                                        */
size_t vqb_prior_layer_backward_workspace_bytes(const vqb_prior_layer_weights *layer, int B, int H, int W, int dim,
                                                int n_classes);
/* Gradients of one layer from d_out_v, d_out_h (B,H,W,dim) NHWC, the layer's inputs x_v, x_h and the `saved` of a
 * vqb_prior_layer_forward_train_f32 call with the same layer and inputs: overwrites the nine gradients of `grads`
 * (each in its parameter's layout, mask A's taps included) and d_x_v, d_x_h (B,H,W,dim) NHWC.  d_out_v == NULL is a
 * zero gradient.  The body of one layer of vqb_prior_backward_f32, without layer 0's d_x_v + d_x_h fold (that is the
 * net's embedding gradient): 10 launches.                                                                        */
int vqb_prior_layer_backward_f32(const vqb_prior_layer_weights *layer, const float *x_v, const float *x_h,
                                 const int64_t *labels, int B, int H, int W, int dim, int n_classes,
                                 const float *d_out_v, const float *d_out_h, const void *saved,
                                 const vqb_prior_layer_grads *grads, float *d_x_v, float *d_x_h, void *workspace,
                                 size_t workspace_bytes, void *stream);
/* vqb_prior_layer_backward_workspace_bytes / vqb_prior_layer_backward_f32 for dim % 32 == 0 up to 1024: the same
 * arguments, checks, launches and bits.                                                                         */
size_t vqb_prior_layer_backward_wide_workspace_bytes(const vqb_prior_layer_weights *layer, int B, int H, int W,
                                                     int dim, int n_classes);
int vqb_prior_layer_backward_wide_f32(const vqb_prior_layer_weights *layer, const float *x_v, const float *x_h,
                                      const int64_t *labels, int B, int H, int W, int dim, int n_classes,
                                      const float *d_out_v, const float *d_out_h, const void *saved,
                                      const vqb_prior_layer_grads *grads, float *d_x_v, float *d_x_h, void *workspace,
                                      size_t workspace_bytes, void *stream);

/* ---- Gated PixelCNN prior in TF32 (wgmma tensor cores) ---------------------------------------------------------
 * The teacher-forced forward and the backward with every matrix product on a TF32 wgmma GEMM: each operand is
 * rounded to TF32 (round to nearest, ties away from zero) as it is staged, products accumulate in fp32.  The one-hot
 * sums of the class and code embedding gradients stay fp32.  Same arguments, shape limits and error codes as the fp32
 * entry points (never an fp32 fall-back); `saved` has the same layout and size (vqb_prior_train_saved_bytes), and the
 * backward the same workspace (vqb_prior_backward_workspace_bytes) and properties: every gradient overwritten in its
 * parameter's layout, mask A's taps included; no float atomics (bitwise reproducible); no host synchronisation.
 * generate stays fp32 (vqb_prior_generate_f32).                                                                    */
/* Workspace of vqb_prior_forward_tf32: 4*B*H*W*(11*dim + 512) bytes (0 = bad sizes).                               */
size_t vqb_prior_workspace_bytes_tf32(int B, int H, int W, int dim, int n_layers, int K);
/* GatedPixelCNN.forward in TF32: 3 + 4*n_layers launches (embedding; per layer the vertical stack, vert_to_horiz with
 * the vertical gate, the horizontal stack, the gate with horiz_resid; the head's two 1x1 convs).                   */
int vqb_prior_forward_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H, int W,
                           float *logits, void *workspace, size_t workspace_bytes, void *stream);
/* vqb_prior_forward_tf32 keeping its activations in `saved`: the same launches, bitwise the same logits.           */
int vqb_prior_forward_train_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H,
                                 int W, float *logits, void *saved, size_t saved_bytes, void *stream);
/* Gradients from a vqb_prior_forward_train_tf32 call's `saved`: 7 + 10*n_layers launches.                          */
int vqb_prior_backward_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H, int W,
                            const float *d_logits, const void *saved, const vqb_prior_grads *grads, void *workspace,
                            size_t workspace_bytes, void *stream);

/* ---- Gated PixelCNN prior: log-likelihood of given code grids (fp32 and TF32) -----------------------------------
 * With l = the logits vqb_prior_forward_f32 (or _tf32) computes on codes and labels, and c = codes clamped to
 * [0, input_dim - 1], the term of position p = i*W + j of image b is
 *   lp[b, p] = (l_c - M) - logf(S),  M = max_k l_k,  S = sum_k expf(l_k - M)      (l at b, p; a fixed-order sum)
 * The logits are never written to memory: the layers are the forward's launches (bitwise the same activations), the
 * head's logits, bitwise the forward's, are reduced on chip to a running (M, S, l_c) per position, and one finish
 * launch combines them.  pos_log_prob: NULL or (B, H, W) fp32 receiving every lp; log_prob: NULL or (B) fp32
 * receiving, per image, the compensated (Kahan) fp32 sum of lp over p >= n_given in raster order (0 when
 * n_given = H*W), vqb_prior_sample_f32's sum.  At least one of them non-NULL, n_given in [0, H*W]: VQB_ERR_BAD_ARG
 * otherwise.  Shape limits and the other checks are vqb_prior_forward_*'s; any layer 0 is taken (with a layer 0 that
 * reads the code it scores, the sum is the reference's cross-entropy, not a likelihood).  Deterministic (no float
 * atomics; two calls are bitwise equal), no host synchronisation.
 * Launches: fp32 3 + 2*n_layers (embedding, two per layer, head, finish); TF32 4 + 4*n_layers (embedding, four per
 * layer, the hidden layer, head, finish).                                                                         */
/* vqb_prior_workspace_bytes + 12*B*H*W bytes (0 = bad sizes).                                                      */
size_t vqb_prior_log_prob_workspace_bytes(int B, int H, int W, int dim, int n_layers, int K);
/* vqb_prior_workspace_bytes_tf32 + 12*B*H*W*splits bytes (0 = bad sizes): the TF32 head splits the K codes over
 * `splits` CTAs per 128 positions, from the shape only.  With T = ceil(K / BN) tiles of BN = (K <= 64 ? 64 : 128)
 * codes and s = min(T, max(1, ceil(264 / ceil(B*H*W / 128)))): splits = ceil(T / ceil(T / s)).                   */
size_t vqb_prior_log_prob_workspace_bytes_tf32(int B, int H, int W, int dim, int n_layers, int K);
int vqb_prior_log_prob_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int64_t n_given,
                           int B, int H, int W, float *log_prob, float *pos_log_prob, void *workspace,
                           size_t workspace_bytes, void *stream);
int vqb_prior_log_prob_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int64_t n_given,
                            int B, int H, int W, float *log_prob, float *pos_log_prob, void *workspace,
                            size_t workspace_bytes, void *stream);
/* log_prob with one prefix length per image: n_given (B) int64 on the device (never read on the host, each value
 * clamped to [0, H*W]); log_prob[b] is bitwise entry b of vqb_prior_log_prob_* on the same inputs with the scalar
 * n_given = clamp(n_given[b]).
 * No per-position output.  The same launches and workspace as vqb_prior_log_prob_* in the same precision;
 * VQB_ERR_BAD_ARG for a NULL log_prob or n_given and for their other bad arguments.                              */
int vqb_prior_log_prob_ragged_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels,
                                  const int64_t *n_given, int B, int H, int W, float *log_prob, void *workspace,
                                  size_t workspace_bytes, void *stream);
int vqb_prior_log_prob_ragged_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels,
                                   const int64_t *n_given, int B, int H, int W, float *log_prob, void *workspace,
                                   size_t workspace_bytes, void *stream);

/* ---- Gated PixelCNN prior: the training cross-entropy without the logits (fp32 and TF32) -------------------------
 * The reference's loss, nn.CrossEntropyLoss(reduction)(logits.permute(0, 2, 3, 1).reshape(-1, K), codes.reshape(-1)),
 * with the logits of vqb_prior_forward_f32 (or _tf32) and codes clamped to [0, input_dim - 1], and its gradient with
 * respect to every parameter, without storing the B*K*H*W logits or their gradient.
 * Forward: vqb_prior_log_prob_*'s layer walk and head, then the finish.  The per-position loss is -lp[b, p] of
 * vqb_prior_log_prob_* bitwise; VQB_PRIOR_CE_SUM is their sum in fp64 (thread t of one 1024-thread block adds
 * positions t, t + 1024, ... in order, then a pairwise tree over the threads), rounded to fp32 once, and
 * VQB_PRIOR_CE_MEAN that fp64 sum over B*H*W, rounded once.  With `saved` non-NULL the walk is the training forward's
 * (vqb_prior_forward_train_*): `saved` receives bitwise that call's activations, then each position's (M, logf(S)).
 * Backward: the head's products per chunk of P = min(4096, B*H*W) positions in raster order: the chunk's logits are
 * recomputed (bitwise the forward's) and turned into d_l[n, k] = g_n * (expf((l_k - M) - logf(S)) - [k = c_n]) in a
 * P x K buffer (g_n = d_loss[n] for VQB_PRIOR_CE_NONE, d_loss[0] / (B*H*W) for MEAN, d_loss[0] for SUM), which feed
 * d_hidden and the output_conv.2 gradient; the chunks' output_conv.2 partials are added in chunk order.  The rest is
 * vqb_prior_backward_*'s, with the embedding gradient's position chunks bounded in number.  No buffer grows with
 * B*H*W*K.  Checks and limits are vqb_prior_forward_*'s, plus the reduction (VQB_ERR_BAD_ARG); any layer 0 is taken.
 * Deterministic (no float atomics; two calls are bitwise equal), no host synchronisation.
 * Launches, forward: fp32 3 + 2*n_layers, TF32 4 + 4*n_layers, one more for MEAN and SUM; backward, both
 * precisions: 5 + 10*n_layers + 3*ceil(B*H*W / 4096).                                                            */
#define VQB_PRIOR_CE_NONE 0     /* loss (B, H, W) */
#define VQB_PRIOR_CE_MEAN 1     /* loss (1): the mean over B*H*W positions */
#define VQB_PRIOR_CE_SUM 2      /* loss (1): the sum */
/* Bytes of the forward's `saved`: vqb_prior_train_saved_bytes + 8*B*H*W (0 = bad sizes).                           */
size_t vqb_prior_ce_saved_bytes(int B, int H, int W, int dim, int n_layers);
/* Forward workspace (0 = bad sizes).  train = 0 (saved NULL): vqb_prior_log_prob_workspace_bytes(_tf32) + 4*B*H*W;
 * train = 1: 4*B*H*W*(3*splits + 1), splits 1 in fp32 and vqb_prior_log_prob_workspace_bytes_tf32's in TF32.     */
size_t vqb_prior_ce_workspace_bytes(int B, int H, int W, int dim, int n_layers, int K, int train);
size_t vqb_prior_ce_workspace_bytes_tf32(int B, int H, int W, int dim, int n_layers, int K, int train);
/* loss: (B, H, W) fp32 for VQB_PRIOR_CE_NONE, one fp32 otherwise.  saved: NULL (inference), or
 * vqb_prior_ce_saved_bytes for the backward.                                                                      */
int vqb_prior_ce_forward_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H,
                             int W, int reduction, float *loss, void *saved, size_t saved_bytes, void *workspace,
                             size_t workspace_bytes, void *stream);
int vqb_prior_ce_forward_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H,
                              int W, int reduction, float *loss, void *saved, size_t saved_bytes, void *workspace,
                              size_t workspace_bytes, void *stream);
/* Backward workspace, both precisions (0 = bad arguments): vqb_prior_backward_workspace_bytes's regions without the
 * output_conv.2 partials and with at most ceil(264 / tiles) embedding-gradient chunks, plus 4*P*K bytes for d_l and
 * 4*s*K*513 for the output_conv.2 partials, s the chunks of a 513-column gradient over P positions (ffma_gemm.cuh). */
size_t vqb_prior_ce_backward_workspace_bytes(const vqb_prior_net *net, int B, int H, int W);
/* Every parameter gradient (overwritten, as vqb_prior_backward_*) from d_loss, the upstream gradient in device memory
 * ((B, H, W) fp32 for VQB_PRIOR_CE_NONE, one fp32 otherwise), and the `saved` of a vqb_prior_ce_forward_* call with
 * the same net, inputs, reduction and precision.                                                                  */
int vqb_prior_ce_backward_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H,
                              int W, int reduction, const float *d_loss, const void *saved,
                              const vqb_prior_grads *grads, void *workspace, size_t workspace_bytes, void *stream);
int vqb_prior_ce_backward_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H,
                               int W, int reduction, const float *d_loss, const void *saved,
                               const vqb_prior_grads *grads, void *workspace, size_t workspace_bytes, void *stream);

/* ---- the cross-entropy's options: class weights, an ignored code and label smoothing (fp32 and TF32) --------------
 * nn.CrossEntropyLoss(weight, ignore_index, label_smoothing, reduction) of the same logits, with codes clamped as above.
 * With w the weights (all ones when weight is NULL), e = label_smoothing, y the clamped code of a position, lse its
 * log-sum-exp, l its logits and W = sum_k w_k (fp64, on the device in a fixed order):
 *   loss_p = (1 - e) * w_y * (-lp) + (e / K) * (W * lse - sum_k w_k * l_k)   (lp as vqb_prior_log_prob_*'s term)
 * and loss_p = 0 at an ignored position: one whose raw code (before clamping) equals ignore_index, when has_ignore.
 * sum_k w_k * l_k is an fp64 sum in the head (each thread's codes in order, then the lanes' and warps' in a fixed
 * order, as (M, S)), and the smoothing term is W * logf(S) + (W * M - sum_k w_k l_k) in fp64.  SUM adds loss_p as
 * VQB_PRIOR_CE_SUM does; MEAN divides that sum by the sum of w_y over the positions not ignored (fp64, the same
 * order), NaN when it is 0.  The backward's d_l[n, k] = g_n * (q_k * c_n - (1 - e) * w_y * [k = y] - (e / K) * w_k),
 * q_k = expf((l_k - M) - logf(S)), c_n = (1 - e) * w_y + (e / K) * W, is evaluated in fp32 as
 * g_n * ((1 - e) * w_y * (q_k - [k = y]) + (e / K) * (W * q_k - w_k)); g_n = 0 at an ignored position, and MEAN's
 * factor (float)(1.0 / divisor) is read from `saved` on the device.  The weights are read on the device only.
 * With unit weights, no position ignored and e = 0 every value is bitwise the call without options.
 * The _ex entry points take a NULL options pointer as the call without options (the same launches and sizes), and
 * return VQB_ERR_BAD_ARG for has_ignore not 0 or 1 or label_smoothing outside [0, 1] (NaN included), after the
 * checks above.  The same launch counts as without options.                                                       */
typedef struct {
    const float *weight;        /* input_dim fp32 weights on the device, or NULL: all ones */
    int64_t ignore_index;       /* read when has_ignore = 1 */
    int has_ignore;
    float label_smoothing;      /* in [0, 1] */
} vqb_prior_ce_options;
/* vqb_prior_ce_saved_bytes, plus 8 bytes (W and MEAN's factor) with options.                                      */
size_t vqb_prior_ce_saved_bytes_ex(int B, int H, int W, int dim, int n_layers, const vqb_prior_ce_options *options);
/* vqb_prior_ce_workspace_bytes(_tf32) = b, and with options: round_up(b + 4*B*H*W, 8) + 8*B*H*W*splits, splits 1 in
 * fp32 and vqb_prior_log_prob_workspace_bytes_tf32's in TF32 (0 = bad sizes).                                     */
size_t vqb_prior_ce_workspace_bytes_ex(int B, int H, int W, int dim, int n_layers, int K, int train,
                                       const vqb_prior_ce_options *options);
size_t vqb_prior_ce_workspace_bytes_ex_tf32(int B, int H, int W, int dim, int n_layers, int K, int train,
                                            const vqb_prior_ce_options *options);
int vqb_prior_ce_forward_ex_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H,
                                int W, int reduction, const vqb_prior_ce_options *options, float *loss, void *saved,
                                size_t saved_bytes, void *workspace, size_t workspace_bytes, void *stream);
int vqb_prior_ce_forward_ex_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H,
                                 int W, int reduction, const vqb_prior_ce_options *options, float *loss, void *saved,
                                 size_t saved_bytes, void *workspace, size_t workspace_bytes, void *stream);
/* The backward workspace is vqb_prior_ce_backward_workspace_bytes's; `saved` from the _ex forward with the same
 * options.                                                                                                          */
int vqb_prior_ce_backward_ex_f32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H,
                                 int W, int reduction, const vqb_prior_ce_options *options, const float *d_loss,
                                 const void *saved, const vqb_prior_grads *grads, void *workspace,
                                 size_t workspace_bytes, void *stream);
int vqb_prior_ce_backward_ex_tf32(const vqb_prior_net *net, const int64_t *codes, const int64_t *labels, int B, int H,
                                  int W, int reduction, const vqb_prior_ce_options *options, const float *d_loss,
                                  const void *saved, const vqb_prior_grads *grads, void *workspace,
                                  size_t workspace_bytes, void *stream);

/* ---- optimizer step on device: Adam over many tensors, then every weight packing refreshed --------------------
 * One training step's update of a parameter group is two calls, each normally ONE launch: vqb_adam_multi_f32 updates
 * every parameter and its moments, then vqb_repack_multi rebuilds every packing read from those parameters and
 * advances their step counters.  The descriptor arrays are HOST arrays, read during the call only; each launch carries
 * its whole table as one by-value kernel parameter (needs a driver of the CUDA 12.1 line or newer), so both calls
 * capture into a CUDA graph with no host-to-device copy, and a replay runs with the hyper-parameters and pointers of
 * the capture.  A list longer than the per-launch capacity is split into several launches, in order.              */

/* One parameter of vqb_adam_multi_f32: numel fp32 elements each of param, grad, exp_avg, exp_avg_sq and, with amsgrad,
 * max_exp_avg_sq (NULL otherwise).  step: the device fp32 count of steps this parameter has taken (torch's
 * state["step"]), read, not written: vqb_repack_multi advances it.                                                   */
typedef struct vqb_adam_tensor {
    float *param;
    const float *grad;
    float *exp_avg, *exp_avg_sq, *max_exp_avg_sq;
    const float *step;
    int64_t numel;
} vqb_adam_tensor;

/* Tensors per launch of vqb_adam_multi_f32 (480).                                                                     */
int vqb_adam_capacity(void);
/* torch.optim.Adam's update (weight decay as an L2 term on the grad, not decoupled), per element in fp32 in the order
 * of torch's single-tensor Adam: g += wd*p; exp_avg lerps towards g by 1 - beta1; exp_avg_sq = exp_avg_sq*beta2 +
 * (1 - beta2)*g*g; amsgrad max; denom = sqrt(v)/sqrt(bc2) + eps; p -= (lr/bc1)*exp_avg/denom, with bc_i = 1 - beta_i^t
 * for t = step + 1 formed in double and rounded to fp32 once.  float4 accesses where a tensor's five pointers are
 * 16-byte aligned.  No atomics: bitwise reproducible.  Hyper-parameters outside torch's ranges (lr, eps, weight_decay
 * < 0, betas outside [0, 1)) are VQB_ERR_BAD_ARG.  ceil(n / vqb_adam_capacity()) launches (none for empty tensors). */
int vqb_adam_multi_f32(const vqb_adam_tensor *tensors, int n, double lr, double beta1, double beta2, double eps,
                       double weight_decay, int amsgrad, void *stream);

/* The layouts of vqb_repack_multi: each writes one packing of the fp32 parameter `src` (as PyTorch stores it) into
 * `dst`, as the single-packing entry point named writes it.                                                        */
enum vqb_pack_layout {
    VQB_PACK_F32 = 0,           /* K-major fp32 [kh*kw][Cout][Cin_pad] of a conv (transposed = 0) or transposed conv
                                   (1), zero padded from Cin: vqb_pack_conv_weight_f32 (Cin_pad = Cin)              */
    VQB_PACK_SHUFFLE_F32 = 1,   /* the [9][16][Cin] pixel-shuffle region of a k4 s2 transposed conv to Cout <= 4
                                   channels (vqb_pack_conv_weight_f32 writes it after the K-major rows)             */
    VQB_PACK_BF16 = 2,          /* VQB_PACK_F32 in bf16: vqb_pack_conv_weight_bf16                                 */
    VQB_PACK_SHUFFLE_BF16 = 3,  /* VQB_PACK_SHUFFLE_F32 in bf16: vqb_pack_conv_weight_bf16, VQB_CONVT_K4S2_OUT     */
    VQB_PACK_PRIOR_F32 = 4,     /* [(r*cols + s)*Cin + ci][co] over the kept taps r < rows, s < cols: vqb_prior_pack_f32 */
    VQB_PACK_MASK_ZERO = 5,     /* no packing: zeroes the taps r >= rows or s >= cols of the (Cout,Cin,kh,kw)
                                   parameter `dst` itself (a mask-A layer's); `src` unused.  Those taps are read by
                                   no packing of the same call                                                      */
    /* The prior at a dim the kernels do not take (dim % 32 != 0): GatedPixelCNN runs them at Cp = roundup(dim, 32)
     * channels on zero-padded copies of its parameters.  These three layouts take the padded channel count Cp in
     * Cin_pad and say which axes pad in `transposed` = kout + 4*kin, one kind per axis (Cout, Cin):
     *   0  the axis is not padded (output_conv's 512 and K axes, an embedding's rows);
     *   1  a dim-wide axis: n = dim real channels, then Cp - dim zeros (width Cp);
     *   2  a gate axis of n = 2*dim channels, padded per half: [dim real, Cp - dim zeros | dim real, Cp - dim zeros]
     *      (width 2*Cp), because the kernels pair channel c with channel c + Cp.
     * A padded width below the real one, a kind outside 0..2, an odd gate axis or no padded axis: VQB_ERR_BAD_ARG.
     * A bias is Cout = its length, Cin = 1; an embedding (rows, cols) is Cout = rows, Cin = cols; both kh = kw = 1. */
    VQB_PACK_PRIOR_PAD_F32,     /* (6) VQB_PACK_PRIOR_F32 at the padded widths: [(r*cols + s)*Cin' + ci'][co'], zero
                                   at every padding channel; what vqb_prior_pack_f32 makes of the padded weight     */
    VQB_PACK_PAD_F32,           /* (7) the parameter in its own layout (Cout, Cin, kh, kw) at the padded widths
                                   (Cout', Cin', kh, kw), zero at every padding channel                             */
    VQB_PACK_UNPAD_F32          /* (8) the inverse of VQB_PACK_PAD_F32, for gradients: `dst` (Cout, Cin, kh, kw)
                                   receives the real entries of the padded `src` (Cout', Cin', kh, kw)              */
};

typedef struct vqb_pack_desc {
    void *dst;
    const float *src;
    int layout, Cout, Cin, Cin_pad, kh, kw, transposed, rows, cols;
} vqb_pack_desc;

/* Descriptors plus step counters per launch of vqb_repack_multi (480).                                              */
int vqb_repack_capacity(void);
/* Every packing of `descs`, then steps[i] += 1 for each of the n_steps device fp32 counters (issue it after the
 * vqb_adam_multi_f32 calls that read them).  A single packing is one descriptor and no counters; so is a gradient's
 * VQB_PACK_UNPAD_F32 copy.  The descriptors must not write what another one reads.  Unknown layouts,
 * NULL pointers, non-positive sizes, Cin_pad < Cin, rows / cols outside the kernel: VQB_ERR_BAD_ARG.
 * ceil((n + n_steps) / vqb_repack_capacity()) launches.                                                             */
int vqb_repack_multi(const vqb_pack_desc *descs, int n, float *const *steps, int n_steps, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* VQVAE_B200_H */

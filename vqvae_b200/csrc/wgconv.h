// wgconv.h -- host description of one launch of the wgmma implicit-GEMM convolution (wgconv.cu).
#pragma once
#include "common.cuh"

#define WG_MAX_STEPS 72        // k-steps per phase: taps x 128-byte channel chunks (e.g. 9 taps x 8 chunks)

// One k-step over channels [c0, c0 + chunk): the A box is those channels of the input pixel shifted by (dy, dx); the
// B box is the same channels of the N weight rows starting at w_row.
struct WgStep { int c0, dx, dy, w_row; };

struct WgLaunch {
    int bf16 = 0;                         // operands: 0 = fp32 activations read as TF32, 1 = bf16
    const void *in = nullptr;             // NHWC (B, H, W, Cin)
    int B = 0, Cin = 0, H = 0, W = 0, in_step = 1;
    const void *w = nullptr;              // weight rows, w_inner elements each (K-major)
    long long w_rows = 0;
    int w_inner = 0;
    int N = 0;                            // GEMM columns per tile: 16, 32, 64, 128 or 256
    int ncols = 0;                        // columns that carry output (<= N)
    // chained second GEMM (residual layer): N2 output columns from N2 rows of w2_inner channels; 0 = none
    const void *w2 = nullptr;
    long long w2_rows = 0;
    int w2_inner = 64;
    int N2 = 0;
    const float *bias = nullptr;          // per output channel, may be null
    const void *skip = nullptr;           // same layout and type as out, may be null
    void *out = nullptr;
    int out_bf16 = 0, relu = 0;
    int out_step = 1;
    long long out_sn = 0, out_sh = 0, out_sw = 0, out_sc = 1;    // element strides of out (and skip)
    int nph = 1;
    int OHg[4] = {0, 0, 0, 0}, OWg[4] = {0, 0, 0, 0}, out_py[4] = {0, 0, 0, 0}, out_px[4] = {0, 0, 0, 0};
    int nsteps[4] = {0, 0, 0, 0};
    WgStep steps[4][WG_MAX_STEPS];
    // the decoder's output layer chained on whole-image tiles of this k4 s2 transposed conv (N = 64, TF32, 4 phases):
    // x_hat NCHW (B, tail_cout, 2 OH, 2 OW) from w_shuffle rows (vqb_pack_conv_weight_f32's shuffle region); out
    // (h) may then be null.  tail_out = null: no tail.
    const void *tail_w = nullptr;
    const float *tail_bias = nullptr;
    float *tail_out = nullptr;
    int tail_cout = 0, tail_relu = 0;
};

int launch_wgconv(const WgLaunch &L, cudaStream_t s);
int wg_gemm_cols(int ncols);           // smallest supported N >= ncols, 0 if none

// The layer launchers take the operand type (bf16 = 0: fp32 activations read as TF32, 1: bf16) and a weight of
// K-major rows per tap, [tap][rows][Cin], as vqb_pack_conv_weight_f32 and vqb_pack_conv_weight_bf16 write them.
bool conv_tc_supported(const ConvLaunch &p);
// L: the tensors, ncols = Cout, output strides and epilogue of one layer; ph[0..nph): its phases, one launch
// (blockIdx.y = phase) over the weight [total_taps][Cout][Cin]
int launch_conv_tc(WgLaunch &L, const ConvPhase *ph, int nph, int total_taps, bool chunk_outer, cudaStream_t s);
bool res_wg_supported(int bf16, int C, int Cmid);
int launch_res_wg(int bf16, const void *r, const void *w1, const void *w2, void *out, int B, int H, int W, int C, int Cmid,
                  int relu_out, int napps, cudaStream_t s);
// A stride-1 k3 conv (or transposed conv) Cin -> C with bias and ReLU, a ResidualStack of napps applications and, when
// tail_cout > 0, the 1x1 conv tail_w (C -> tail_cout) with bias, in one launch (res_scatter_kernel): the separate
// launches' bits.  out: (B, H, W, C) NHWC, or (B, H, W, tail_cout) with the tail.  Answers VQB_ERR_UNSUPPORTED,
// launching nothing, when latent_block_supported fails (tail_cout = 0: no tail), tail_w is given without tail_cout or
// the other way round, x == out, or a pointer is not 16-byte aligned.
bool latent_block_supported(int Cin, int C, int Cmid, int H, int W, int tail_cout);
int launch_latent_block(const void *x, const void *head_w, const float *head_bias, int Cin, int transposed,
                        const void *w1, const void *w2, int napps, const void *tail_w, const float *tail_bias,
                        int tail_cout, void *out, int B, int H, int W, int C, int Cmid, cudaStream_t s);
// The decoder's k4 s2 transposed conv Cin -> C (bias, ReLU) and the output layer C -> Cout (k4 s2 transposed, + bias,
// optional ReLU) in one launch (wgconv_kernel in TAIL mode): x_hat NCHW (B, Cout, 4H, 4W) and, when h_out is not
// null, h NHWC (B, 2H, 2W, C), bitwise the two separate launches.  w: vqb_pack_conv_weight_f32 packings of both
// layers.  Answers VQB_ERR_UNSUPPORTED, launching nothing, when decoder_tail_supported fails, d_out aliases an
// output or a pointer is not 16-byte aligned.
bool decoder_tail_supported(int Cin, int H, int W, int C, int Cout);
int launch_decoder_tail(const void *d_out, const void *convt_w, const float *convt_bias, const void *out_w,
                        const float *out_bias, void *h_out, float *x_hat, int B, int Cin, int H, int W, int C, int Cout,
                        int relu_out, cudaStream_t s);
bool convt_shuffle_supported(int Cin, int Cout);
int launch_convt_shuffle_wg(int bf16, const void *in, const void *w_shuffle, const float *bias, float *out, int B, int Cin,
                            int H, int W, int Cout, int relu, cudaStream_t s);

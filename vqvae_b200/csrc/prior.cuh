// prior.cuh -- what the Gated PixelCNN's per-position kernels (prior.cu) and its matrix products (prior_gemm.cu) share:
// shape limits, the NHWC activation view, the host-side weight table and its argument checks, and the gate.
#pragma once
#include "common.cuh"

namespace {

constexpr int NT = 256;           // threads of every prior kernel
constexpr int MAXC = 256;         // dim <= 256, dim % 32 == 0
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

inline bool dim_ok(int C) { return C % 32 == 0 && C <= MAXC; }

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

// What one layer's training forward (vqb_prior_layer_forward_train_f32) keeps, in floats, NHWC (2C) grids: hv and
// ph as in Saved.
struct LayerSaved {
    long long N, C;
    long long hv() const { return 0; }
    long long ph() const { return 2 * N * C; }
    long long total() const { return 4 * N * C; }
};

}  // namespace

// hconv.cu -- the bf16 pipeline's convolution layers (VQB_BF16 mode): the shapes each layer kind takes, the weight
// packing and the entry points vqb_conv2d_bf16 / vqb_residual_layer_bf16, all computed by the wgmma implicit-GEMM
// kernel of wgconv.cu on bf16 NHWC activations with fp32 accumulation:
//   encoder.py:32-34  Conv2d k4 s2 p1          (taps read through stride-2 element strides of the input tensor map)
//   encoder.py:35-36  Conv2d k3 s1 p1
//   vqvae.py:16-17    Conv2d k1                 (fp32 output: z_e feeds the bit-exact VQ)
//   decoder.py:28-29  ConvTranspose2d k3 s1 p1
//   decoder.py:31-33  ConvTranspose2d k4 s2 p1  (four sub-pixel phases of 4 taps in one launch)
//   decoder.py:34-35  ConvTranspose2d k4 s2 p1 to <= 4 channels (scatter form: one GEMM over each tile's input pixels
//                                                and halo, N = 64, neighbour sums writing the NCHW fp32 module output)
//   residual.py:18-29 one ResidualLayer: 3x3 conv, ReLU and 1x1 conv chained inside one CTA per tile
// A packed weight is the K-major layout the TF32 mode reads, in bf16: [kh*kw taps][Cout][Cin] (VQB_RES_W2: Cin zero
// padded to 64), or [9 neighbour taps][16][Cin] for VQB_CONVT_K4S2_OUT.  The kernel reads the N rows of one k-step
// as one TMA box.
#include "common.cuh"
#include "wgconv.h"

namespace {

// enum vqb_conv_kind -> the layer, and the shapes it takes: Cin % cin_step == 0 and cin_step <= Cin <= cin_max, the
// same for Cout.  chunk_outer: k-step order 64-channel chunk outer, tap inner (else tap outer, chunk inner).
struct Kind { int k, stride, pad, transposed, chunk_outer, cin_step, cin_max, cout_step, cout_max; };
constexpr Kind KINDS[] = {
    {1, 1, 0, 0, 1, 64, 512, 16, 256},     // VQB_CONV_K1
    {3, 1, 1, 0, 1, 64, 256, 16, 256},     // VQB_CONV_K3
    {3, 1, 1, 1, 1, 64, 256, 16, 256},     // VQB_CONVT_K3
    {4, 2, 1, 0, 0, 64, 128, 16, 256},     // VQB_CONV_K4S2
    {4, 2, 1, 1, 0, 64, 384, 32, 128},     // VQB_CONVT_K4S2
    {4, 2, 1, 1, 1, 64, 256, 1, 4},        // VQB_CONVT_K4S2_OUT
    {1, 1, 0, 0, 0, 16, 64, 16, 256},      // VQB_RES_W2 (Cin = Cmid)
};

const Kind *kind_of(int kind, int Cout, int Cin) {
    if (kind < 0 || kind > VQB_RES_W2) return nullptr;
    const Kind &k = KINDS[kind];
    const bool ok = Cin % k.cin_step == 0 && Cin >= k.cin_step && Cin <= k.cin_max &&
                    Cout % k.cout_step == 0 && Cout >= k.cout_step && Cout <= k.cout_max;
    return ok ? &k : nullptr;
}

int cin_pad(int Cin) { return (Cin + 63) / 64 * 64; }

}  // namespace

extern "C" size_t vqb_conv_bf16_packed_bytes(int kind, int Cout, int Cin) {
    const Kind *k = kind_of(kind, Cout, Cin);
    if (!k) return 0;
    const size_t elems = kind == VQB_CONVT_K4S2_OUT ? (size_t)9 * 16 * Cin : (size_t)k->k * k->k * Cout * cin_pad(Cin);
    return elems * 2;
}

extern "C" int vqb_pack_conv_weight_bf16(const float *w, void *packed, int kind, int Cout, int Cin, void *stream) {
    if (!w || !packed) return VQB_ERR_BAD_ARG;
    const Kind *k = kind_of(kind, Cout, Cin);
    if (!k) return VQB_ERR_UNSUPPORTED;
    if (reinterpret_cast<uintptr_t>(packed) & 127) return VQB_ERR_ALIGNMENT;
    return launch_pack_weight_bf16(w, packed, Cout, Cin, cin_pad(Cin), k->k, k->k, k->transposed,
                                   kind == VQB_CONVT_K4S2_OUT, (cudaStream_t)stream);
}

// in: bf16 NHWC (B, H, W, Cin).  out: bf16 NHWC (out_f32 = 0) / fp32 NHWC (out_f32 = 1) / fp32 NCHW (VQB_CONVT_K4S2_OUT).
extern "C" int vqb_conv2d_bf16(const void *in, const void *packed, const float *bias, void *out, int B, int Cin, int H, int W,
                               int Cout, int kind, int relu, int out_f32, void *stream) {
    if (!in || !packed || !out) return VQB_ERR_BAD_ARG;
    if (B <= 0 || Cin <= 0 || H <= 0 || W <= 0 || Cout <= 0) return VQB_ERR_BAD_ARG;
    const Kind *k = kind_of(kind, Cout, Cin);
    if (!k) return VQB_ERR_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(packed)) & 15) return VQB_ERR_ALIGNMENT;
    cudaStream_t s = (cudaStream_t)stream;
    if (kind == VQB_CONVT_K4S2_OUT)
        return launch_convt_shuffle_wg(1, in, packed, bias, reinterpret_cast<float *>(out), B, Cin, H, W, Cout, relu, s);
    if (kind == VQB_CONV_K4S2 && ((H | W) & 1)) return VQB_ERR_UNSUPPORTED;

    const ConvGeom g = conv_geom(k->k, k->k, k->stride, k->pad, k->transposed, H, W);
    ConvPhase ph[4];
    int nph = 0;
    for (int i = 0; i < g.nph; ++i)
        if (conv_phase(g, i, ph[nph])) ++nph;
    WgLaunch L;
    L.bf16 = 1;
    L.in = in; L.B = B; L.Cin = Cin; L.H = H; L.W = W;
    L.w = packed; L.ncols = Cout;
    L.bias = bias; L.out = out; L.out_bf16 = !out_f32; L.relu = relu;
    L.out_sn = (long long)g.OH * g.OW * Cout; L.out_sh = (long long)g.OW * Cout; L.out_sw = Cout; L.out_sc = 1;
    return launch_conv_tc(L, ph, nph, k->k * k->k, k->chunk_outer, s);
}

// r, out: bf16 NHWC (B,H,W,C).  w1: packing of kind VQB_CONV_K3 with (Cout = Cmid, Cin = C); w2: VQB_RES_W2 with
// (Cout = C, Cin = Cmid) -- both made by vqb_pack_conv_weight_bf16.  One launch: per 128-pixel tile the 3x3 GEMM, ReLU,
// and the 1x1 GEMM on the bf16 intermediate held in shared memory, + r, optional ReLU.
extern "C" int vqb_residual_layer_bf16(const void *r, const void *w1_packed, const void *w2_packed, void *out, int B, int H,
                                       int W, int C, int Cmid, int relu_out, void *stream) {
    if (!r || !w1_packed || !w2_packed || !out) return VQB_ERR_BAD_ARG;
    if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || Cmid <= 0) return VQB_ERR_BAD_ARG;
    if (!res_wg_supported(1, C, Cmid)) return VQB_ERR_UNSUPPORTED;
    if (r == out) return VQB_ERR_BAD_ARG;                       // neighbouring tiles read each other's halo: not in place
    if ((reinterpret_cast<uintptr_t>(r) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(w1_packed) |
         reinterpret_cast<uintptr_t>(w2_packed)) & 15) return VQB_ERR_ALIGNMENT;
    return launch_res_wg(1, r, w1_packed, w2_packed, out, B, H, W, C, Cmid, relu_out, 1, (cudaStream_t)stream);
}

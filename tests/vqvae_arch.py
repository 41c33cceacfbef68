"""VQ-VAE architectures that main.py's flags build, and the kernel every layer must run at each of them.

ARCHS is shared by tests/test_vqvae_arch_cpu.py, tests/test_gpu_vqvae_arch.py and oracle/make_arch_golden.py.  The
second half restates the dispatch rules of include/vqvae_b200.h and the launchers (vqb_conv2d_f32, the residual
entry points, the latent block, the decoder tail, the VQ and the bf16 pipeline) as plain Python, from the documented
shape limits.  It never asks the library which shapes it takes: the CPU test checks the restatement against the
library's own queries, and the GPU test checks it against the kernel names the profiler records.
"""
from collections import Counter

import numpy as np

from oracle.weights import make_state_dict

# name -> (h_dim, res_h_dim, n_res_layers, K, embedding_dim, batch, (H, W), codebook scale, seed)
ARCHS = {
    # 128-channel input conv, N = 256 GEMMs with 8 chunks, a stack outside res_wg, both fusions declined
    "h256": (256, 64, 2, 512, 64, 3, (32, 32), 0.05, 31),
    # N = 16 (W1), W2 with Cin 16 on FFMA, exact VQ at D = 32, output layer Cin 32
    "h64": (64, 16, 1, 256, 32, 5, (32, 32), 0.07, 32),
    # 48-channel layers on FFMA, N = 128 with 96 live, D = 40, K = 1000, ragged 12 x 20 latents
    "h96": (96, 48, 3, 1000, 40, 2, (48, 80), 0.06, 33),
    # N = 256 with 160 live, 80-channel layers on FFMA, N = 128 with 80 live
    "h160": (160, 32, 2, 512, 64, 3, (32, 32), 0.05, 34),
    # conv_in_k4s2 at its 48 KB limit, Cout 512 on FFMA, shuffle output layer at Cin 256, exact VQ at D = 256
    "h512": (512, 128, 1, 512, 256, 2, (32, 32), 0.03, 35),
    # TF32 res_wg per application; bf16 Cmid 64
    "r64": (128, 64, 2, 512, 64, 4, (32, 32), 0.05, 36),
    # 16 x 16 latents, two-launch stack with W2 on FFMA; bf16 Cmid 16
    "r16": (128, 16, 3, 512, 64, 2, (64, 64), 0.05, 37),
    # W1 at N = 64 with 48 live; bf16 Cmid 48
    "r48": (128, 48, 4, 512, 64, 3, (32, 32), 0.05, 38),
    # empty stacks
    "n0": (128, 32, 0, 512, 64, 3, (32, 32), 0.05, 39),
    # latent blocks with 6 chained applications
    "n6": (128, 32, 6, 512, 64, 3, (32, 32), 0.05, 40),
}
GOLDEN_ARCHS = ("h96", "h160", "h512", "r16")
HP_KEYS = ("h_dim", "res_h_dim", "n_res_layers", "n_embeddings", "embedding_dim")


def arch_inputs(name):
    """(hyper-parameters, numpy state dict, fp32 images (B, 3, H, W) in [-1, 1)) of a row, from its seed."""
    h, r, n, K, D, B, (H, W), scale, seed = ARCHS[name]
    hp = dict(zip(HP_KEYS, (h, r, n, K, D)))
    sd = make_state_dict(seed=seed, codebook="normal", codebook_scale=scale, **hp)
    x = np.random.RandomState(100 + seed).uniform(-1, 1, (B, 3, H, W)).astype(np.float32)
    return hp, sd, x


# ---------------------------------------------------------------------------------------------- dispatch rules
# The kernels restated here; every other kernel (weight packing, layout changes, ReLU, the VQ's helper launches, the
# weight gradients and the VQ backward) is left out of the comparison.
KERNELS = ("wgconv_kernel", "res_scatter_kernel", "convt_scatter_kernel", "conv_ffma_kernel", "conv_small_cout_kernel",
           "conv_in_k4s2_kernel", "convt_out_k4s2_kernel", "vq_tc_kernel", "vq_exact_kernel")
BF16 = "<bf16>"                 # suffix of the bf16 instantiations of convt_scatter_kernel and conv_in_k4s2_kernel
WG_MAX_STEPS = 72               # k-steps per phase of the wgmma conv: taps x 32-channel chunks (wgconv.h)


def _pow2(v):
    p = 1
    while p < v:
        p *= 2
    return p


def gemm_cols(ncols):
    """N of the wgmma GEMM that computes ncols output columns: the next of 16, 32, 64, 128, 256."""
    return next(n for n in (16, 32, 64, 128, 256) if ncols <= n)


def wg(N, N2=0, bf16=False, tail=False):
    """The wgconv_kernel instantiation <BF16, N, N2, TAIL>, named as the profiler demangles it: N2 > 0 is the residual
    layer's second GEMM chained in the same CTA, TAIL the decoder tail's output layer."""
    return f"wgconv_kernel<{str(bf16).lower()}, {N}, {N2}, {str(tail).lower()}>"


def whole_images(H, W):
    """A 128-pixel tile holds whole H x W images: pow2(W) <= 16 and pow2(W) * pow2(H) <= 128."""
    return W <= 16 and _pow2(W) * _pow2(H) <= 128


def conv_kernels(prec, Cin, Cout, k, s, transposed, H, W, in_nchw=False, out_nchw=False, skip=False):
    """The kernels of one vqb_conv2d_f32 call ("fp32" or "tf32") on an (H, W) input, in launch order:
    - k4 s2 p1 without skip: the transposed conv to 1..4 channels, NHWC in, NCHW out, Cin % 32 == 0, Cin <= 256 in
      TF32: convt_scatter_kernel; the conv from 3 channels, NCHW in, NHWC out, Cout % 32 == 0, H and W even and its
      16 * 3 * Cout fp32 weights within 48 KB: conv_in_k4s2_kernel; the transposed conv to 3 channels, NHWC in, NCHW
      out, Cin % 4 == 0, Cin <= 128, Cin / 4 a power of two: convt_out_k4s2_kernel;
    - TF32, NHWC on both sides, Cin % 32 == 0, Cout % 16 == 0, 16 <= Cout <= 256 and at most WG_MAX_STEPS k-steps per
      phase: one wgconv_kernel for every phase, N = gemm_cols(Cout);
    - else one FFMA launch per phase (a stride-s transposed conv has s * s): conv_small_cout_kernel to <= 4 channels,
      conv_ffma_kernel otherwise."""
    assert prec in ("fp32", "tf32")
    tf32 = prec == "tf32"
    if k == 4 and s == 2 and not skip:
        if transposed and tf32 and not in_nchw and out_nchw and 1 <= Cout <= 4 and Cin % 32 == 0 and Cin <= 256:
            return ["convt_scatter_kernel"]
        if not transposed and Cin == 3 and Cout % 32 == 0 and in_nchw and not out_nchw and H % 2 == 0 and \
                W % 2 == 0 and 16 * Cin * Cout * 4 <= 48 * 1024:
            return ["conv_in_k4s2_kernel"]
        L = Cin // 4
        if transposed and Cout == 3 and Cin % 4 == 0 and Cin <= 128 and L & (L - 1) == 0 and not in_nchw and out_nchw:
            return ["convt_out_k4s2_kernel"]
    taps = (k // s) ** 2 if transposed else k * k               # taps per phase
    if tf32 and not in_nchw and not out_nchw and Cin % 32 == 0 and Cout % 16 == 0 and 16 <= Cout <= 256 and \
            taps * (Cin // 32) <= WG_MAX_STEPS:
        return [wg(gemm_cols(Cout))]
    nph = s * s if transposed else 1
    return ["conv_small_cout_kernel" if Cout <= 4 else "conv_ffma_kernel"] * nph


def res_wg(C, Cmid):
    """The TF32 residual layer runs as one launch: C in {64, 128}, Cmid in {32, 64}."""
    return C in (64, 128) and Cmid in (32, 64)


def res_scatter(C, Cmid, H, W):
    """... on res_scatter_kernel: additionally Cmid = 32 and whole images per tile."""
    return res_wg(C, Cmid) and Cmid == 32 and whole_images(H, W)


def res_layer_kernels(prec, C, Cmid, H, W):
    """One vqb_residual_layer_f32 call: one launch where res_wg takes it, else the 3x3 conv and the 1x1 conv + skip."""
    if prec == "tf32" and res_wg(C, Cmid):
        return ["res_scatter_kernel" if res_scatter(C, Cmid, H, W) else wg(gemm_cols(Cmid), C)]
    return conv_kernels(prec, C, Cmid, 3, 1, False, H, W) + conv_kernels(prec, Cmid, C, 1, 1, False, H, W, skip=True)


def stack_kernels(prec, C, Cmid, n, H, W):
    """vqb_residual_stack_f32: every application in one res_scatter_kernel launch when it takes the layer, else one
    vqb_residual_layer_f32 per application; nothing for an empty stack."""
    if n == 0:
        return []
    if prec == "tf32" and n > 1 and res_scatter(C, Cmid, H, W):
        return ["res_scatter_kernel"]
    return res_layer_kernels(prec, C, Cmid, H, W) * n


def latent_block_shape(Cin, C, Cmid, H, W, tail_cout):
    """vqb_latent_block_supported: a res_scatter stack, Cin % 32 == 0 with 9 * Cin / 32 k-steps at most, a tail of 0 or
    64 channels."""
    return res_scatter(C, Cmid, H, W) and Cin % 32 == 0 and 9 * (Cin // 32) <= WG_MAX_STEPS and tail_cout in (0, 64)


def decoder_tail_shape(Cin, H, W, C, Cout):
    """vqb_decoder_tail_supported: C = 64, 1 <= Cout <= 4, Cin % 32 == 0, 32 <= Cin <= 256, whole latent images."""
    return C == 64 and 1 <= Cout <= 4 and Cin % 32 == 0 and 32 <= Cin <= 256 and whole_images(H, W)


def vq_kernels(D):
    """vqb_vq_forward_f32: the tensor-core kernel at D = 64, the exact FFMA kernel otherwise."""
    return ["vq_tc_kernel" if D == 64 else "vq_exact_kernel"]


# bf16 layer kinds (include/vqvae_b200.h, hconv.cu): (cin_step, cin_max, cout_step, cout_max)
BF16_KINDS = {"K1": (64, 512, 16, 256), "K3": (64, 256, 16, 256), "CONVT_K3": (64, 256, 16, 256),
              "K4S2": (64, 128, 16, 256), "CONVT_K4S2": (64, 384, 32, 128), "CONVT_K4S2_OUT": (64, 256, 1, 4),
              "RES_W2": (16, 64, 16, 256)}


def bf16_kind_ok(kind, Cout, Cin):
    """vqb_conv_bf16_packed_bytes != 0: Cin and Cout multiples of their steps, within [step, max]."""
    cs, cm, os_, om = BF16_KINDS[kind]
    return Cin % cs == 0 and cs <= Cin <= cm and Cout % os_ == 0 and os_ <= Cout <= om


def bf16_layers(h, r, n, D):
    """(kind, Cout, Cin) of every conv that takes a bf16 packing."""
    out = [("K4S2", h, h // 2), ("K3", h, h), ("K1", D, h), ("CONVT_K3", h, D), ("CONVT_K4S2", h // 2, h),
           ("CONVT_K4S2_OUT", 3, h // 2)]
    if n:
        out += [("K3", r, h), ("RES_W2", h, r)]
    return out


def bf16_covered(name):
    """The bf16 pipeline runs the row: a 64-channel input conv (vqb_conv_in_bf16), residual layers with C in {64, 128}
    and Cmid % 16 == 0, 16 <= Cmid <= 64 (vqb_residual_layer_bf16), D = 64 (vqb_vq_forward_bf16zq_f32) and a bf16
    packing for every other conv."""
    h, r, n, K, D = ARCHS[name][:5]
    if h // 2 != 64 or D != 64:
        return False
    if n and not (h in (64, 128) and r % 16 == 0 and 16 <= r <= 64):
        return False
    return all(bf16_kind_ok(*layer) for layer in bf16_layers(h, r, n, D))


def _geometry(name):
    h, r, n, K, D, B, (H, W) = ARCHS[name][:7]
    return h, r, n, D, H, W, H // 2, W // 2, H // 4, W // 4


def fused_blocks(name):
    """(encoder latent block, decoder latent block, decoder tail): which one-launch fusions the TF32 walks take.  The
    latent blocks need the reference's [layer] * n stack with n >= 1 and run in the eval walk only; the tail runs in
    both."""
    h, r, n, D, H, W, H1, W1, H2, W2 = _geometry(name)
    return (n >= 1 and latent_block_shape(h, h, r, H2, W2, D), n >= 1 and latent_block_shape(D, h, r, H2, W2, 0),
            decoder_tail_shape(h, H2, W2, h // 2, 3))


def forward_kernels(name, prec, walk):
    """The restated kernels of one VQVAE forward in `prec` ("fp32", "tf32", "bf16"); walk "eval" (model.eval(), the
    inference walk) or "train" (the training walk that keeps the activations the backward reads)."""
    h, r, n, D, H, W, H1, W1, H2, W2 = _geometry(name)
    if prec == "bf16" and walk == "eval" and bf16_covered(name):
        conv, res = (lambda cout: wg(gemm_cols(cout), bf16=True)), [wg(gemm_cols(r), h, bf16=True)] * n
        return ["conv_in_k4s2_kernel" + BF16, conv(h), conv(h)] + res + [conv(D)] + vq_kernels(D) + [conv(h)] + res + \
            [conv(h // 2), "convt_scatter_kernel" + BF16]
    p = "fp32" if prec == "fp32" else "tf32"         # bf16 outside the pipeline runs the TF32 kernels
    enc_block, dec_block, tail = fused_blocks(name) if p == "tf32" else (False, False, False)
    ks = conv_kernels(p, 3, h // 2, 4, 2, False, H, W, in_nchw=True)
    ks += conv_kernels(p, h // 2, h, 4, 2, False, H1, W1)
    if enc_block and walk == "eval":
        ks += ["res_scatter_kernel"]
    else:
        ks += conv_kernels(p, h, h, 3, 1, False, H2, W2) + stack_kernels(p, h, r, n, H2, W2)
        ks += conv_kernels(p, h, D, 1, 1, False, H2, W2)
    ks += vq_kernels(D)
    if dec_block and walk == "eval":
        ks += ["res_scatter_kernel"]
    else:
        ks += conv_kernels(p, D, h, 3, 1, True, H2, W2) + stack_kernels(p, h, r, n, H2, W2)
    if tail:
        ks += [wg(64, tail=True)]
    else:
        ks += conv_kernels(p, h, h // 2, 4, 2, True, H2, W2)
        ks += conv_kernels(p, h // 2, 3, 4, 2, True, H1, W1, out_nchw=True)
    return ks


def stack_backward_kernels(p, C, Cmid, n, H, W):
    """_stack_backward: the n - 1 recomputed applications, every application's 3x3 conv in one call, then per
    application the adjoints of the 1x1 conv (a k1 transposed conv) and of the 3x3 conv (+ skip)."""
    if n == 0:
        return []
    ks = res_layer_kernels(p, C, Cmid, H, W) * (n - 1) + conv_kernels(p, C, Cmid, 3, 1, False, H, W)
    return ks + (conv_kernels(p, C, Cmid, 1, 1, True, H, W) + conv_kernels(p, Cmid, C, 3, 1, True, H, W, skip=True)) * n


def train_step_kernels(name, prec):
    """The restated kernels of one training step (the training walk, then _VQVAEFunction.backward with the image
    gradient): every input gradient is the adjoint conv (Conv2d <-> ConvTranspose2d) on vqb_conv2d_f32.  bf16 mode
    trains on the TF32 kernels."""
    h, r, n, D, H, W, H1, W1, H2, W2 = _geometry(name)
    p = "fp32" if prec == "fp32" else "tf32"
    ks = forward_kernels(name, p, "train")
    ks += conv_kernels(p, 3, h // 2, 4, 2, False, H, W, in_nchw=True)           # output layer
    ks += conv_kernels(p, h // 2, h, 4, 2, False, H1, W1)                       # decoder k4 s2
    ks += stack_backward_kernels(p, h, r, n, H2, W2)
    ks += conv_kernels(p, h, D, 3, 1, False, H2, W2)                            # decoder k3
    ks += conv_kernels(p, D, h, 1, 1, True, H2, W2)                             # pre-quantization conv
    ks += stack_backward_kernels(p, h, r, n, H2, W2)
    ks += conv_kernels(p, h, h, 3, 1, True, H2, W2)                             # encoder k3
    ks += conv_kernels(p, h, h // 2, 4, 2, True, H2, W2)                        # encoder k4 s2
    ks += conv_kernels(p, h // 2, 3, 4, 2, True, H1, W1, out_nchw=True)         # input conv (image gradient)
    return ks


def expected_kernels(name, prec, walk):
    """Multiset of restated kernel names: walk "eval" (one inference forward) or "train" (one training step)."""
    return Counter(forward_kernels(name, prec, "eval") if walk == "eval" else train_step_kernels(name, prec))

"""The VQ-VAE forward restated with every ReLU given, for fp64 checks of the GPU's gradients at the GPU's own ReLU masks.

An fp64 forward flips some ReLU masks against a TF32 (or fp32) forward, and a flipped mask moves a gradient by far more
than the backward's own rounding.  Restated with ``relu = masked_relu(masks)``, each ReLU multiplies by the next mask
of a list built from the activations the GPU's training walk kept, in the order the restatement applies its ReLUs
(``model_masks``), so fp64 autograd of the restatement differentiates the same piecewise-linear function the GPU's
backward does.  With ``relu = torch.relu`` the functions are the plain forward of oracle/torch_port.py.
tests/test_vqvae_masked_cpu.py pins the mask order without a GPU.
"""
import torch.nn.functional as F

from oracle.vqvae_train_port import vector_quantizer


def res64(x, w1, w2, n, relu, final):
    """residual.py with every ReLU given: n applications of one layer, then the stack's ReLU if `final` (an empty stack,
    n = 0, has no weights: w1 and w2 None)."""
    for _ in range(n):
        r = relu(x)
        x = r + F.conv2d(relu(F.conv2d(r, w1, None, 1, 1)), w2)
    return relu(x) if final else x


def enc64(x, p, n, relu, e="encoder.conv_stack."):
    h = relu(F.conv2d(x, p[e + "0.weight"], p[e + "0.bias"], 2, 1))
    h = relu(F.conv2d(h, p[e + "2.weight"], p[e + "2.bias"], 2, 1))
    h = F.conv2d(h, p[e + "4.weight"], p[e + "4.bias"], 1, 1)
    return res64(h, p.get(e + "5.stack.0.res_block.1.weight"), p.get(e + "5.stack.0.res_block.3.weight"), n, relu, True)


def dec64(z, p, n, relu, d="decoder.inverse_conv_stack."):
    h = F.conv_transpose2d(z, p[d + "0.weight"], p[d + "0.bias"], 1, 1)
    h = res64(h, p.get(d + "1.stack.0.res_block.1.weight"), p.get(d + "1.stack.0.res_block.3.weight"), n, relu, True)
    h = relu(F.conv_transpose2d(h, p[d + "2.weight"], p[d + "2.bias"], 2, 1))
    return F.conv_transpose2d(h, p[d + "4.weight"], p[d + "4.bias"], 2, 1)


def vqvae64(x, p, n, relu, idx, beta=0.25):
    """VQVAE.forward (oracle/vqvae_train_port.py) with every ReLU given, at the codes idx -> (embedding_loss, x_hat)."""
    z_e = F.conv2d(enc64(x, p, n, relu), p["pre_quantization_conv.weight"], p["pre_quantization_conv.bias"])
    loss, z_q, _, _ = vector_quantizer(z_e, p["vector_quantization.embedding.weight"], beta, idx)
    return loss, dec64(z_q, p, n, relu)


def stack_mask_list(r0, out, n, mid, step, relu_out=True):
    """The masks of res64 over a stack of n applications of one layer, from its input r0 = relu(x) and its output:
    each application's input r_i > 0 and m_i = mid(r_i) > 0, with r_{i+1} = step(r_i), then out > 0 if `relu_out`."""
    masks, r = [], r0
    for i in range(n):
        masks += [r > 0, mid(r) > 0]
        if i < n - 1:
            r = step(r)
    if relu_out:
        masks.append(out > 0)
    return masks


def model_masks(enc, dec, stack):
    """The masks of vqvae64, in order, from the encoder's kept activations (a1, a2, a3, e_out), the decoder's
    (d1, d_out, d2) and stack(side, r0, out), the masks of the residual stack of side "enc" or "dec"."""
    a1, a2, a3, e_out = enc
    d1, d_out, d2 = dec
    return [a1 > 0, a2 > 0] + stack("enc", a3, e_out) + stack("dec", d1, d_out) + [d2 > 0]


def masked_relu(masks):
    """(relu, done): relu(t) = t * the next of `masks` (NCHW, t's dtype and device); done() is True once every mask
    has been used exactly once."""
    it = iter(masks)

    def relu(t):
        m = next(it)
        assert m.shape == t.shape, (tuple(m.shape), tuple(t.shape))
        return t * m.to(t.dtype)

    return relu, lambda: next(it, None) is None


def nchw64(masks):
    """NHWC CUDA masks -> NCHW fp64 CPU tensors."""
    return [t.permute(0, 3, 1, 2).double().cpu() for t in masks]


def stack_masks(layer, r0, out, n, relu_out=True, precision=None):
    """The ReLU masks a stack backward in `precision` (default TF32) reads, in the order res64 applies its ReLUs: each
    application's input r_i > 0 and m_i = relu(W1 (*) r_i) > 0, recomputed from r0 (NHWC) as _stack_backward does,
    then out > 0."""
    from vqvae_b200 import ops
    from vqvae_b200._lib import TF32
    from vqvae_b200.modules import _packed
    precision = TF32 if precision is None else precision
    c1, c2 = layer.res_block[1], layer.res_block[3]
    w1, w2 = _packed(c1.weight, ("f32", False)), _packed(c2.weight, ("f32", False))
    B, H, W, C = r0.shape
    geo = dict(B=B, H=H, W=W)
    mid = lambda r: ops.conv2d(r, w1, None, Cin=C, Cout=c1.out_channels, kh=3, kw=3, stride=1, pad=1,  # noqa: E731
                               relu=True, precision=precision, **geo)
    step = lambda r: ops.residual_layer(r, w1, w2, C=C, Cmid=c1.out_channels, relu_out=True,  # noqa: E731
                                        precision=precision, **geo)
    return stack_mask_list(r0, out, n, mid, step, relu_out)

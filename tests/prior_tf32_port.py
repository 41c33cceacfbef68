"""The emulated-TF32 restatement of the Gated PixelCNN prior (GatedPixelCNN.precision = "tf32") -- TEST INFRASTRUCTURE
ONLY.

``prior_logits_tf32`` is ``oracle.prior_train_port.prior_logits`` (the reference's GatedPixelCNN.forward on a dict of
leaf tensors, mask A zeroing its layer's weights in place) with every convolution replaced by ``_Tf32Conv``, which
rounds its operands with ``tf32_round`` as the kernels' TF32 GEMM (vqvae_b200/csrc/tc_gemm.cuh) does, in the forward and
in both products of its backward.  Everything else is exact in the tensors' dtype (fp64 in the tests), so the
restatement differs from the kernels only by their fp32 accumulation.  The product never imports this module.
"""
import torch
import torch.nn.functional as F

from oracle.prior_port import _stack


def tf32_round(t):
    """t rounded to TF32 as the kernels' `cvt.rna.tf32.f32` does: to nearest on the 10 kept mantissa bits, ties away
    from zero (the low 13 bits of the fp32 value become zero).  fp32 first, so an fp64 tensor is rounded from the fp32
    value a kernel would hold; returned in t's dtype."""
    u = t.detach().float().contiguous().view(torch.int32)
    u = ((u & 0x7FFFFFFF) + 0x1000) & 0x7FFFE000 | (u & -0x80000000)
    return u.view(torch.float32).to(t.dtype)


class _Tf32Conv(torch.autograd.Function):
    """F.conv2d (stride 1) whose forward and both backward products take TF32-rounded operands: the forward
    rnd(x) * rnd(w); d x from rnd(d y) and rnd(w); d w from rnd(x) and rnd(d y); d bias the sum of rnd(d y) (the
    kernels' bias column of ones)."""

    @staticmethod
    def forward(ctx, x, w, b, padding):
        ctx.save_for_backward(x, w)
        ctx.padding = padding
        return F.conv2d(tf32_round(x), tf32_round(w), b, 1, padding)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        r = tf32_round(dy)
        dx = torch.nn.grad.conv2d_input(x.shape, tf32_round(w), r, 1, ctx.padding)
        dw = torch.nn.grad.conv2d_weight(tf32_round(x), w.shape, r, 1, ctx.padding)
        return dx, dw, r.sum((0, 2, 3)), None


def _conv(x, w, b, padding=0):
    return _Tf32Conv.apply(x, w, b, padding)


def _gate(t):
    a, b = t.chunk(2, dim=1)
    return torch.tanh(a) * torch.sigmoid(b)


def prior_logits_tf32(g, x, label, n_layers, layers=None):
    """Logits (B, K, H, W) of codes x (B,H,W) int64 and labels (B,) int64 in the TF32 mode's arithmetic; g maps keys to
    (leaf) tensors; layers: (mask_type, kernel, residual) per layer, default the reference's stack."""
    h = F.embedding(x, g["embedding.weight"]).permute(0, 3, 1, 2)
    x_v = x_h = h
    for i, (mask, k, residual) in enumerate(_stack(n_layers, layers)):
        p = f"layers.{i}."
        wv, wh = g[p + "vert_stack.weight"], g[p + "horiz_stack.weight"]
        if mask == "A":                                   # mask A (models.py:61-63): in place, on the parameter
            wv.data[:, :, -1].zero_()
            wh.data[:, :, :, -1].zero_()
        c = F.embedding(label, g[p + "class_cond_embedding.weight"])[:, :, None, None]
        hv = _conv(x_v, wv, g[p + "vert_stack.bias"], (k // 2, k // 2))[:, :, :x_v.size(-1), :]
        out_v = _gate(hv + c)
        hh = _conv(x_h, wh, g[p + "horiz_stack.bias"], (0, k // 2))[:, :, :, :x_h.size(-2)]
        v2h = _conv(hv, g[p + "vert_to_horiz.weight"], g[p + "vert_to_horiz.bias"])
        out = _gate(v2h + hh + c)
        r = _conv(out, g[p + "horiz_resid.weight"], g[p + "horiz_resid.bias"])
        x_h = r + x_h if residual else r
        x_v = out_v
    y = F.relu(_conv(x_h, g["output_conv.0.weight"], g["output_conv.0.bias"]))
    return _conv(y, g["output_conv.2.weight"], g["output_conv.2.bias"])

"""The emulated-TF32 restatement of the Gated PixelCNN prior (GatedPixelCNN.precision = "tf32") -- TEST INFRASTRUCTURE
ONLY.

``prior_logits_tf32`` is ``oracle.prior_train_port.prior_logits`` (the reference's GatedPixelCNN.forward on a dict of
leaf tensors, mask A zeroing its layer's weights in place) with every convolution replaced by ``_Tf32Conv``, which
rounds its operands with ``tf32_round`` as the kernels' TF32 GEMM (vqvae_b200/csrc/tc_gemm.cuh) does, in the forward and
in both products of its backward.  Everything else is exact in the tensors' dtype (fp64 in the tests), so the
restatement differs from the kernels only by their fp32 accumulation.  The product never imports this module.

Evaluated on its own, the restatement drifts from the GPU with depth: the GPU's fp32 activations and the fp64 ones
round to different TF32 neighbours, and a gate or ReLU pre-activation near zero can then take the other branch.  With
``at`` (the activations the GPU's training forward kept, ``decode_saved``) every product is evaluated at the GPU's own
operands instead, one product deep, and every gate and ReLU derivative of the backward at the GPU's values.

``decode_saved`` reads the buffer of ``vqb_prior_forward_train_f32`` / ``_tf32``: the layout ``Saved`` of
vqvae_b200/csrc/prior.cuh, restated here once.
"""
import torch
import torch.nn.functional as F

from oracle.prior_port import HIDDEN, _stack


def tf32_round(t):
    """t rounded to TF32 as the kernels' `cvt.rna.tf32.f32` does: to nearest on the 10 kept mantissa bits, ties away
    from zero (the low 13 bits of the fp32 value become zero).  fp32 first, so an fp64 tensor is rounded from the fp32
    value a kernel would hold; returned in t's dtype."""
    u = t.detach().float().contiguous().view(torch.int32)
    u = ((u & 0x7FFFFFFF) + 0x1000) & 0x7FFFE000 | (u & -0x80000000)
    return u.view(torch.float32).to(t.dtype)


def tf32_truncate(t):
    """t with the low 13 bits of its fp32 value cleared (rounded toward zero to TF32): the rounding the kernels do not
    use, for showing that they round to nearest."""
    u = t.detach().float().contiguous().view(torch.int32) & -0x2000
    return u.view(torch.float32).to(t.dtype)


def no_rounding(t):
    """The identity: the restatement of the fp32 mode's products."""
    return t.detach()


class _Tf32Conv(torch.autograd.Function):
    """F.conv2d (stride 1) whose forward and both backward products take rounded operands (`rnd`, tf32_round for the
    kernels' TF32 GEMM): the forward rnd(x) * rnd(w); d x from rnd(d y) and rnd(w); d w from rnd(x) and rnd(d y);
    d bias the sum of rnd(d y) (the kernels' bias column of ones)."""

    @staticmethod
    def forward(ctx, x, w, b, padding, rnd):
        ctx.save_for_backward(x, w)
        ctx.padding, ctx.rnd = padding, rnd
        return F.conv2d(rnd(x), rnd(w), b, 1, padding)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        rnd = ctx.rnd
        r = rnd(dy)
        dx = torch.nn.grad.conv2d_input(x.shape, rnd(w), r, 1, ctx.padding)
        dw = torch.nn.grad.conv2d_weight(rnd(x), w.shape, r, 1, ctx.padding)
        return dx, dw, r.sum((0, 2, 3)), None, None


def _gate(t):
    a, b = t.chunk(2, dim=1)
    return torch.tanh(a) * torch.sigmoid(b)


def saved_points(n_layers):
    """Names of the activations the training forward keeps and ``at`` / ``record`` take, in forward order: per layer
    l, hv{l} (h_vert, bias included, class embedding not) and ph{l} (the horizontal gate's pre-activation), then
    xh{l+1} (the next layer's horizontal input; xh{L} is the head's) and xv{l+1} (the next layer's vertical input, for
    l + 1 < L: nothing reads the last layer's); last hid (the head's hidden layer after the ReLU)."""
    out = []
    for l in range(n_layers):
        out += [f"hv{l}", f"ph{l}", f"xh{l + 1}"] + ([f"xv{l + 1}"] if l + 1 < n_layers else [])
    return out + ["hid"]


def prior_logits_tf32(g, x, label, n_layers, layers=None, at=None, record=None, rounding=tf32_round, terms=None):
    """Logits (B, K, H, W) of codes x (B,H,W) int64 and labels (B,) int64 in the TF32 mode's arithmetic; g maps keys to
    (leaf) tensors; layers: (mask_type, kernel, residual) per layer, default the reference's stack.

    at: None, or {name: NCHW tensor} for every name of ``saved_points``.  Each such activation then takes the given
    value in straight-through form, t + (at[name] - t).detach(): the products after it read the given value, the
    gates' derivatives are taken at it, and autograd still runs the restatement's backward through t.  The head's
    ReLU passes the gradient where at["hid"] > 0, as the kernels' backward reads it from the saved hidden layer.
    record: None, or a dict that receives each point's recomputed value (detached, before the replacement).
    rounding: the operand rounding of every product, tf32_round (the TF32 mode) or no_rounding (fp32).
    terms: None, or a dict that receives, for every point computed by products (all but xv) and for "logits", the sum
    over each element's terms of their magnitudes (|rounded operands| in every product, |bias|, |class|, |skip|): the
    scale of that element's fp32 accumulation error."""
    def point(name, t, keep=None):
        if record is not None:
            record[name] = (t if keep is None else keep).detach()
        return t if at is None else t + (at[name].to(t) - t).detach()

    def conv(x, w, b, padding=0):
        return _Tf32Conv.apply(x, w, b, padding, rounding)

    def mag(x, w, b, padding=0):
        return F.conv2d(rounding(x).abs(), rounding(w).abs(), b.detach().abs(), 1, padding)

    def term(name, t):
        if terms is not None:
            with torch.no_grad():
                terms[name] = t()

    h = F.embedding(x, g["embedding.weight"]).permute(0, 3, 1, 2)
    x_v = x_h = h
    stack = _stack(n_layers, layers)
    for i, (mask, k, residual) in enumerate(stack):
        p = f"layers.{i}."
        wv, wh = g[p + "vert_stack.weight"], g[p + "horiz_stack.weight"]
        if mask == "A":                                   # mask A (models.py:61-63): in place, on the parameter
            wv.data[:, :, -1].zero_()
            wh.data[:, :, :, -1].zero_()
        c = F.embedding(label, g[p + "class_cond_embedding.weight"])[:, :, None, None]
        bv, bh = g[p + "vert_stack.bias"], g[p + "horiz_stack.bias"]
        wvh, bvh = g[p + "vert_to_horiz.weight"], g[p + "vert_to_horiz.bias"]
        wr, br = g[p + "horiz_resid.weight"], g[p + "horiz_resid.bias"]
        term(f"hv{i}", lambda: mag(x_v, wv, bv, (k // 2, k // 2))[:, :, :x_v.size(-1), :])
        hv = point(f"hv{i}", conv(x_v, wv, bv, (k // 2, k // 2))[:, :, :x_v.size(-1), :])
        out_v = _gate(hv + c)
        term(f"ph{i}", lambda: mag(x_h, wh, bh, (0, k // 2))[:, :, :, :x_h.size(-2)] + mag(hv, wvh, bvh) + c.abs())
        hh = conv(x_h, wh, bh, (0, k // 2))[:, :, :, :x_h.size(-2)]
        v2h = conv(hv, wvh, bvh)
        out = _gate(point(f"ph{i}", v2h + hh + c))
        term(f"xh{i + 1}", lambda: mag(out, wr, br) + (x_h.abs() if residual else 0))
        r = conv(out, wr, br)
        x_h = point(f"xh{i + 1}", r + x_h if residual else r)
        x_v = point(f"xv{i + 1}", out_v) if i + 1 < len(stack) else out_v
    w1, b1, w2, b2 = (g["output_conv." + k] for k in ("0.weight", "0.bias", "2.weight", "2.bias"))
    term("hid", lambda: mag(x_h, w1, b1))
    z = conv(x_h, w1, b1)
    y = F.relu(z)
    if at is not None:
        y = z * (at["hid"] > 0)
    y = point("hid", y, F.relu(z))
    term("logits", lambda: mag(y, w2, b2))
    return conv(y, w2, b2)


def saved_offsets(B, H, W, dim, n_layers):
    """{name: (offset, channels)} of the training forward's `saved` buffer, in floats, and its total length: the layout
    ``Saved`` of vqvae_b200/csrc/prior.cuh with N = B*H*W positions, every grid NHWC.  xv{0} (the embedding, also
    layer 0's x_h) and xv{L} (a grid nothing reads) are included; the scratch between a layer's launches is not."""
    N, C, L = B * H * W, dim, n_layers
    off = {f"xv{l}": (l * N * C, C) for l in range(L + 1)}
    off.update({f"xh{l}": ((L + l) * N * C, C) for l in range(1, L + 1)})
    off.update({f"hv{l}": ((2 * L + 1) * N * C + 2 * l * N * C, 2 * C) for l in range(L)})
    off.update({f"ph{l}": ((4 * L + 1) * N * C + 2 * l * N * C, 2 * C) for l in range(L)})
    off["hid"] = ((6 * L + 3) * N * C, HIDDEN)
    return off, (6 * L + 3) * N * C + HIDDEN * N


def decode_saved(saved, B, H, W, dim, n_layers):
    """{name: NCHW fp64 tensor} of a `saved` buffer (a uint8 or fp32 tensor, on any device), for every name of
    ``saved_offsets``."""
    f = saved.view(torch.float32) if saved.dtype == torch.uint8 else saved
    off, total = saved_offsets(B, H, W, dim, n_layers)
    assert f.numel() >= total, (f.numel(), total)
    N = B * H * W
    return {k: f[o:o + N * c].view(B, H, W, c).permute(0, 3, 1, 2).double() for k, (o, c) in off.items()}


def encode_saved(grids, B, H, W, dim, n_layers):
    """The inverse of decode_saved: an fp32 buffer of the full length holding each NCHW grid of `grids` at its offset,
    NaN everywhere else."""
    off, total = saved_offsets(B, H, W, dim, n_layers)
    f = torch.full((total,), float("nan"), dtype=torch.float32)
    N = B * H * W
    for k, t in grids.items():
        o, c = off[k]
        f[o:o + N * c] = t.permute(0, 2, 3, 1).reshape(-1).float()
    return f

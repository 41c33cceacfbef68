"""Host-side mirror of the reference's Gated PixelCNN prior (``pixelcnn/models.py``), trainable.

Same class names, constructor signatures, attribute names and state-dict keys as the reference, so a state dict saved
by its ``gated_pixelcnn.py`` loads unchanged and ``from pixelcnn.models import GatedPixelCNN`` (the top-level
``pixelcnn`` package re-exports these classes) drops in.  As in ``modules.py`` the nn.Conv2d / nn.Embedding children
are parameter containers only: every forward runs the sm_90a kernels of ``csrc/prior.cu`` / ``csrc/prior_gemm.cu``
through the C ABI, in the model's ``precision`` (fp32 by default) whatever ``set_precision`` says.

``GatedPixelCNN.forward`` is differentiable with respect to every parameter when grad is enabled and a parameter
requires grad (``_PriorFunction``: the training forward keeps its activations, and the backward of
``csrc/prior_gemm.cu`` writes one gradient per parameter), so the reference's training loop runs unchanged.  Under
``torch.no_grad()`` it is the inference forward.  ``GatedPixelCNN.precision`` (a plain attribute, not in the state
dict) selects the arithmetic of ``forward`` (inference and training alike) and of ``log_prob``: "fp32" (the default, CUDA cores) or
"tf32" (every matrix product on the wgmma TF32 GEMM, operands rounded to TF32, fp32 accumulation; the one-hot
embedding-gradient sums stay fp32).  ``generate``, ``complete``, ``sample``, ``sample_completion``,
``GatedMaskedConv2d`` and ``GatedActivation`` stay fp32 in both modes, and ``set_precision`` does not affect the
prior.  ``GatedMaskedConv2d`` and ``GatedActivation`` called on their own are differentiable too, under the same rule
(grad enabled and an input or a parameter requiring grad):
``_GatedLayerFunction`` runs the layer's training forward and single-layer backward (vqb_prior_layer_*_f32),
``_GateFunction`` the gate and its backward.  Their outputs are bitwise the inference call's.

Reference behaviour kept on purpose:
  P2  ``self.apply(weights_init)``: Xavier-uniform conv weights, zero biases, and one "Skipping initialization of"
      line per GatedMaskedConv2d (it matches 'Conv' by name but has no weight of its own)
  P3  mask A zeroes the last row of ``vert_stack.weight`` and the last column of ``horiz_stack.weight`` in the
      caller's parameters.  Here that happens when a mask-A layer's weights are (re)packed, i.e. once per change of
      the parameter, so the packing cache and CUDA graphs around a forward stay valid
  P4  square grids only: the reference crops the vertical stack with the width and the horizontal one with the
      height, which fails for H != W; here that is a RuntimeError before any launch
  P5  ``layers`` may be replaced by any GatedMaskedConv2d stack (odd kernels up to 15, either mask, with or without
      residual), as the reference's forward walks whatever ``self.layers`` holds.  Every layer must have the model's
      ``dim`` and layer 0's class count (the reference fails on such a model too, with a shape or index error); a
      RuntimeError before any launch otherwise.  ``generate`` and ``complete`` also need layer 0 to be mask A without
      residual: anything else reads the code being drawn, so the reference's one-forward-per-position loop is not
      causal in raster order there, and the sampler refuses it (C ABI: VQB_ERR_UNSUPPORTED)

Limits: any dim from 1 to 1024, so gated_pixelcnn.py's GatedPixelCNN(K, img_dim**2, n_layers) runs for every latent
grid up to 32x32.  The library's kernels take dim % 32 == 0 only; at any other dim the module runs them at
Cp = roundup(dim, 32) channels on zero-padded packings of its parameters, each gate axis padded per half, and copies
the real entries of the Cp-shaped gradients back (DESIGN §8.5).  Results are bitwise those of GatedPixelCNN(K, Cp) with
the zero-padded weights; state dicts stay the reference's at dim.  A dim above 1024 raises a RuntimeError before any
launch (at a multiple of 32, the library's VQB_ERR_UNSUPPORTED).
"""
import math
import numbers
import operator

import torch
import torch.nn as nn

from . import ops
from ._lib import (PACK_UNPAD_F32, PRIOR_MAX_KERNEL, C, PackDesc, PriorGrads, PriorLayerGrads, PriorLayerWeights,
                   PriorNet, PriorSampling)
from .modules import _packed, _packed_current, pad_geometry

HIDDEN = 512          # output_conv's hidden width


def weights_init(m):
    """Xavier-uniform weight and zero bias for every module whose class name contains 'Conv'."""
    name = type(m).__name__
    if "Conv" not in name:
        return
    try:
        nn.init.xavier_uniform_(m.weight.data)
        m.bias.data.fill_(0)
    except AttributeError:
        print("Skipping initialization of ", name)


def _f32(t):
    t = t.detach()
    t = t if t.dtype == torch.float32 else t.float()
    return t if t.is_contiguous() else t.contiguous()


def _square(H, W, what):
    if H != W:
        raise RuntimeError(f"{what}: the Gated PixelCNN takes square code grids only, got {H}x{W} (the reference "
                           "crops its vertical stack by the width and its horizontal stack by the height)")


def _labels(label, B, dev, what):
    if not torch.is_tensor(label):
        label = torch.as_tensor(label, device=dev)
    ops._require_cuda(label, what + " label")
    label = label.reshape(-1)
    if label.numel() != B:
        raise RuntimeError(f"{what}: expected {B} labels, got {label.numel()}")
    return label.to(torch.int64).contiguous()


def _per_image(n_given):
    """Whether n_given gives one prefix length per image (a 1-D tensor, a list or a tuple) rather than one for the
    batch (an int or a 0-d tensor)."""
    return isinstance(n_given, (list, tuple)) or (torch.is_tensor(n_given) and n_given.dim() != 0)


def _ragged(n_given, x, what):
    """A per-image n_given for the codes x (B,H,W) -> int64 (B,) on x's device.  A tensor must be 1-D with B entries of
    an integer dtype, on x's device; its values are never read on the host (the kernels clamp them to [0, H*W]), and an
    int64 contiguous one is used in place.  A list or tuple must hold B ints in [0, H*W], checked here.  ValueError
    for the shape, dtype, length or a value; RuntimeError for the device."""
    B, H, W = x.shape
    if torch.is_tensor(n_given):
        if n_given.dim() != 1 or n_given.numel() != B:
            raise ValueError(f"{what}: a per-image n_given must be a 1-D tensor of {B} entries, got shape "
                             f"{tuple(n_given.shape)}")
        if n_given.dtype == torch.bool or n_given.is_floating_point() or n_given.is_complex():
            raise ValueError(f"{what}: a per-image n_given must have an integer dtype, got {n_given.dtype}")
        if n_given.device != x.device:
            raise RuntimeError(f"{what}: n_given is on {n_given.device}, the codes on {x.device}")
        return n_given.to(torch.int64).contiguous()
    if len(n_given) != B:
        raise ValueError(f"{what}: a per-image n_given must have {B} entries, got {len(n_given)}")
    for v in n_given:
        if isinstance(v, bool) or not isinstance(v, numbers.Integral) or not 0 <= v <= H * W:
            raise ValueError(f"{what}: every n_given must be an int in [0, H*W] = [0, {H * W}], got {v!r}")
    return torch.tensor([int(v) for v in n_given], dtype=torch.int64, device=x.device)


def _grad_call(inputs, module=None):
    """Whether a prior module's call is differentiable (GatedPixelCNN's rule): grad enabled and an input, or a
    parameter of `module`, requiring grad."""
    return torch.is_grad_enabled() and (any(x.requires_grad for x in inputs) or
                                        (module is not None and any(p.requires_grad for p in module.parameters())))


MAX_DIM = 1024        # the widest prior the kernels run (dim % 32 == 0 up to it; any other dim padded up to it)

# The kinds of a prior parameter's first two axes at a padded dim (vqb_pack_layout): 1 a dim-wide axis, padded at its
# end, 2 a gate axis of 2*dim channels, padded per half (the kernels pair channel c with c + Cp), 0 not padded.  Every
# parameter not listed (output_conv.0.bias, output_conv.2) is the same at every Cp.
_PAD_KINDS = {"vert_stack.weight": (2, 1), "vert_stack.bias": (2, 0), "vert_to_horiz.weight": (2, 2),
              "vert_to_horiz.bias": (2, 0), "horiz_stack.weight": (2, 1), "horiz_stack.bias": (2, 0),
              "horiz_resid.weight": (1, 1), "horiz_resid.bias": (1, 0), "class_cond_embedding.weight": (0, 2),
              "embedding.weight": (0, 1), "output_conv.0.weight": (0, 1)}


def _kinds(name):
    """_PAD_KINDS of a parameter named as in GatedPixelCNN or GatedMaskedConv2d.named_parameters()."""
    if name.startswith("layers."):
        name = name.split(".", 2)[2]
    return _PAD_KINDS.get(name, (0, 0))


def _padded_dim(dim):
    """The channel count the kernels run a dim-wide prior at: dim when they take it (dim % 32 == 0), else
    roundup(dim, 32), on zero-padded packings of the parameters (DESIGN §8.5).  RuntimeError, before any packing or
    launch, for a dim above MAX_DIM that would need padding."""
    cp = -(-dim // 32) * 32
    if cp != dim and dim > MAX_DIM:
        raise RuntimeError(f"GatedPixelCNN: dim {dim} is above the {MAX_DIM} channels the prior kernels run")
    return cp


def _conv_key(cp, dim, name, rows=1, cols=1):
    """Packing-cache key of the prior conv weight `name` (a _PAD_KINDS entry) keeping taps rows x cols, at Cp."""
    return ("prior", rows, cols) if cp == dim else ("prior_pad", rows, cols, cp) + _PAD_KINDS[name]


def _vector(p, cp, dim, name):
    """A bias or embedding as the kernels read it: the parameter itself (fp32, contiguous), or at a padded dim its
    zero-padded copy, cached and refreshed like a weight packing."""
    return _f32(p) if cp == dim else _packed(p, ("pad", cp) + _PAD_KINDS[name])


class _Grads:
    """One fp32 gradient per parameter of `module` (a GatedPixelCNN or a GatedMaskedConv2d of channel count `dim`) and
    the tensors the backward kernels write them into.  At a padded dim those are Cp-shaped buffers for the padded
    parameters, and finish() copies their real entries into the gradients in one vqb_repack_multi launch
    (VQB_PACK_UNPAD_F32), with no host synchronisation; otherwise the gradients themselves."""

    def __init__(self, module, dev, dim):
        cp = _padded_dim(dim)
        self.params = dict(module.named_parameters())
        self.grads = {k: torch.empty(p.shape, dtype=torch.float32, device=dev) for k, p in self.params.items()}
        self.out = dict(self.grads)
        descs = []
        for k, p in self.params.items():
            kout, kin = _kinds(k)
            if cp == dim or not (kout or kin):
                continue
            g = pad_geometry(p.shape, cp, kout, kin)
            shape = list(p.shape)
            shape[0] = ops.pad_width(shape[0], kout, cp)
            if len(shape) > 1:
                shape[1] = ops.pad_width(shape[1], kin, cp)
            self.out[k] = torch.empty(shape, dtype=torch.float32, device=dev)
            descs.append(PackDesc(dst=self.grads[k].data_ptr(), src=self.out[k].data_ptr(), layout=PACK_UNPAD_F32,
                                  rows=0, cols=0, **g))
        self.descs = (PackDesc * len(descs))(*descs) if descs else None

    def ptr(self, name):
        return self.out[name].data_ptr()

    def finish(self):
        """The gradients in parameters() order, each in its parameter's dtype."""
        if self.descs is not None:
            ops.repack_multi(self.descs, len(self.descs), None, 0)
        self.out = None
        return tuple(self.grads[k].to(p.dtype) for k, p in self.params.items())


class _GateFunction(torch.autograd.Function):
    """GatedActivation with a gradient: vqb_prior_gate_f32 forward, vqb_prior_gate_backward_f32 backward."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return ops.prior_gate(x)

    @staticmethod
    def backward(ctx, d_out):
        x, = ctx.saved_tensors
        return ops.prior_gate_backward(x, d_out)


class GatedActivation(nn.Module):
    """tanh(first half of the channels) * sigmoid(second half) (models.py:20-26).  Differentiable when grad is enabled
    and x requires grad (_GateFunction), else the inference call.  Always fp32."""

    def forward(self, x):
        if _grad_call([x]):
            return _GateFunction.apply(x)
        return ops.prior_gate(x)


class GatedMaskedConv2d(nn.Module):
    """One gated layer with a vertical and a horizontal stack (models.py:29-86).  Differentiable with respect to x_v,
    x_h and its nine parameters when grad is enabled and one of them requires grad (_GatedLayerFunction), else the
    inference call.  Always fp32 on its own (a model's ``precision`` applies to ``GatedPixelCNN.forward``)."""

    def __init__(self, mask_type, dim, kernel, residual=True, n_classes=10):
        super().__init__()
        if kernel % 2 != 1:
            raise AssertionError("Kernel size must be odd")
        self.mask_type = mask_type
        self.residual = residual
        half = kernel // 2
        self.class_cond_embedding = nn.Embedding(n_classes, 2 * dim)
        self.vert_stack = nn.Conv2d(dim, dim * 2, (half + 1, kernel), 1, (half, half))
        self.vert_to_horiz = nn.Conv2d(2 * dim, 2 * dim, 1)
        self.horiz_stack = nn.Conv2d(dim, dim * 2, (1, half + 1), 1, (0, half))
        self.horiz_resid = nn.Conv2d(dim, dim, 1)
        self.gate = GatedActivation()
        self._mark_mask_a()

    def _mark_mask_a(self):
        """A mask-A layer marks its two stacks' weights with the taps make_causal keeps, (rows, cols), so that
        vqvae_b200.optim.Adam zeroes the others after each update.  Done when the layer is built, and again before each
        packing (a parameter replaced or deep-copied since has lost the mark)."""
        if self.mask_type == "A":
            vs, hs = self.vert_stack, self.horiz_stack
            vs.weight._vqb_mask_a = (vs.kernel_size[0] - 1, vs.kernel_size[1])
            hs.weight._vqb_mask_a = (1, hs.kernel_size[1] - 1)

    def make_causal(self):
        """Zero the taps mask A excludes: the vertical stack's last row, the horizontal stack's last column."""
        self.vert_stack.weight.data[:, :, -1].zero_()
        self.horiz_stack.weight.data[:, :, :, -1].zero_()

    def _weights(self, keep):
        """struct vqb_prior_layer_weights of this layer; tensors it points into are appended to `keep`.  At a dim the
        kernels do not take, the packings of the zero-padded layer at _padded_dim(dim) channels (DESIGN §8.5)."""
        dim = self.horiz_resid.in_channels
        cp = _padded_dim(dim)
        mask_a = self.mask_type == "A"
        vs, hs = self.vert_stack, self.horiz_stack
        vkey = _conv_key(cp, dim, "vert_stack.weight", vs.kernel_size[0] - mask_a, vs.kernel_size[1])
        hkey = _conv_key(cp, dim, "horiz_stack.weight", 1, hs.kernel_size[1] - mask_a)
        self._mark_mask_a()
        if mask_a and not (_packed_current(vs.weight, vkey) and _packed_current(hs.weight, hkey)):
            self.make_causal()          # P3: once per change of the parameters, right before they are packed
        v2h, res, emb = self.vert_to_horiz, self.horiz_resid, self.class_cond_embedding
        t = dict(vert_w=_packed(vs.weight, vkey), vert_b=_vector(vs.bias, cp, dim, "vert_stack.bias"),
                 v2h_w=_packed(v2h.weight, _conv_key(cp, dim, "vert_to_horiz.weight")),
                 v2h_b=_vector(v2h.bias, cp, dim, "vert_to_horiz.bias"),
                 horiz_w=_packed(hs.weight, hkey), horiz_b=_vector(hs.bias, cp, dim, "horiz_stack.bias"),
                 resid_w=_packed(res.weight, _conv_key(cp, dim, "horiz_resid.weight")),
                 resid_b=_vector(res.bias, cp, dim, "horiz_resid.bias"),
                 class_emb=_vector(emb.weight, cp, dim, "class_cond_embedding.weight"))
        keep.extend(t.values())
        return PriorLayerWeights(**{k: v.data_ptr() for k, v in t.items()}, kernel=vs.kernel_size[1],
                                 mask_a=int(mask_a), residual=int(bool(self.residual)))

    def forward(self, x_v, x_h, h):
        dim = self.horiz_resid.in_channels
        for x, what in ((x_v, "x_v"), (x_h, "x_h")):
            if x.dim() != 4 or x.shape[1] != dim:
                raise RuntimeError(f"GatedMaskedConv2d: expected {what} of shape (B,{dim},H,W), got {tuple(x.shape)}")
            ops._require_cuda(x, "GatedMaskedConv2d " + what)
        if x_v.shape != x_h.shape:
            raise RuntimeError(f"GatedMaskedConv2d: x_v {tuple(x_v.shape)} and x_h {tuple(x_h.shape)} differ")
        B, _, H, W = x_v.shape
        _square(H, W, "GatedMaskedConv2d")
        label = _labels(h, B, x_v.device, "GatedMaskedConv2d")
        if _grad_call([x_v, x_h], self):
            return _GatedLayerFunction.apply(self, x_v, x_h, label, *self.parameters())
        keep = []
        w = self._weights(keep)
        cp = _padded_dim(dim)
        out_v, out_h = ops.prior_layer(w, ops.nchw_to_nhwc_pad(x_v.detach(), cp), ops.nchw_to_nhwc_pad(x_h.detach(), cp),
                                       label, B=B, H=H, W=W, dim=cp,
                                       n_classes=self.class_cond_embedding.num_embeddings)
        return ops.nhwc_to_nchw_unpad(out_v, dim), ops.nhwc_to_nchw_unpad(out_h, dim)


# PriorLayerGrads / PriorGrads field -> parameter name (within a layer / the model)
_LAYER_GRADS = dict(vert_w="vert_stack.weight", vert_b="vert_stack.bias", v2h_w="vert_to_horiz.weight",
                    v2h_b="vert_to_horiz.bias", horiz_w="horiz_stack.weight", horiz_b="horiz_stack.bias",
                    resid_w="horiz_resid.weight", resid_b="horiz_resid.bias", class_emb="class_cond_embedding.weight")
_NET_GRADS = dict(embedding="embedding.weight", out1_w="output_conv.0.weight", out1_b="output_conv.0.bias",
                  out2_w="output_conv.2.weight", out2_b="output_conv.2.bias")


class _GatedLayerFunction(torch.autograd.Function):
    """GatedMaskedConv2d.forward with gradients: inputs are the layer, x_v, x_h (NCHW), the labels and the layer's
    parameters in ``parameters()`` order.  NCHW <-> NHWC at the boundary (at a padded dim, NCHW with dim channels <->
    NHWC with Cp, zero-filled); the forward keeps x_v, x_h (NHWC) and vqb_prior_layer_forward_train_f32's `saved`; the
    backward (vqb_prior_layer_backward_wide_f32) returns the gradients of x_v, x_h and every parameter, mask A's taps
    included.  The labels get none."""

    @staticmethod
    def forward(ctx, layer, x_v, x_h, label, *params):
        B, dim, H, W = x_v.shape
        cp = _padded_dim(dim)
        keep = []
        w = layer._weights(keep)
        xv, xh = ops.nchw_to_nhwc_pad(x_v.detach(), cp), ops.nchw_to_nhwc_pad(x_h.detach(), cp)
        nc = layer.class_cond_embedding.num_embeddings
        out_v, out_h, saved = ops.prior_layer_forward_train(w, xv, xh, label, B=B, H=H, W=W, dim=cp, n_classes=nc)
        ctx.layer, ctx.w, ctx.keep, ctx.saved = layer, w, keep, (xv, xh, label, saved)
        ctx.shape = (B, H, W, dim, cp, nc)
        ctx.save_for_backward(x_v, x_h, *params)
        ctx.set_materialize_grads(False)
        return ops.nhwc_to_nchw_unpad(out_v, dim), ops.nhwc_to_nchw_unpad(out_h, dim)

    @staticmethod
    def backward(ctx, g_v, g_h):
        if ctx.saved is None:
            raise RuntimeError("GatedMaskedConv2d: backward through the same forward twice is not supported "
                               "(its saved activations are freed by the first backward)")
        ctx.saved_tensors                 # autograd's check that nothing saved was modified in place
        xv, xh, label, saved = ctx.saved
        B, H, W, dim, cp, nc = ctx.shape
        if g_h is None:
            g_h = torch.zeros((B, dim, H, W), dtype=torch.float32, device=xv.device)
        dv = ops.nchw_to_nhwc_pad(g_v, cp) if g_v is not None else None
        grads = _Grads(ctx.layer, xv.device, dim)
        table = PriorLayerGrads(**{f: grads.ptr(k) for f, k in _LAYER_GRADS.items()})
        d_x_v, d_x_h = ops.prior_layer_backward(ctx.w, xv, xh, label, dv, ops.nchw_to_nhwc_pad(g_h, cp), saved, table,
                                                B=B, H=H, W=W, dim=cp, n_classes=nc)
        ctx.saved = ctx.keep = None
        need = ctx.needs_input_grad
        return (None, ops.nhwc_to_nchw_unpad(d_x_v, dim) if need[1] else None,
                ops.nhwc_to_nchw_unpad(d_x_h, dim) if need[2] else None, None) + grads.finish()


class _PriorFunction(torch.autograd.Function):
    """GatedPixelCNN.forward with gradients: inputs are the model, the precision, codes, labels and every parameter in
    ``parameters()`` order.  The forward keeps the activations vqb_prior_backward_f32 (or _tf32) reads; the backward
    runs in the precision the forward ran in and returns one gradient per parameter in its shape and dtype, mask A's
    taps included (the reference's autograd gives them one)."""

    @staticmethod
    def forward(ctx, model, precision, codes, labels, *params):
        keep = []
        net = model._net(keep)
        logits, saved = ops.prior_forward_train(net, codes, labels, precision)
        ctx.model, ctx.net, ctx.keep, ctx.saved, ctx.precision = model, net, keep, saved, precision
        ctx.save_for_backward(codes, labels)
        return logits

    @staticmethod
    def backward(ctx, d_logits):
        if ctx.saved is None:           # the first backward freed the saved activations
            raise RuntimeError("GatedPixelCNN: backward through the same forward twice is not supported "
                               "(its saved activations are freed by the first backward)")
        codes, labels = ctx.saved_tensors
        grads, table, _layers = _grad_table(ctx.model, codes.device)
        ops.prior_backward(ctx.net, codes, labels, _f32(d_logits), ctx.saved, table, ctx.precision)
        ctx.saved = ctx.keep = None
        return (None, None, None, None) + grads.finish()


def _grad_table(model, dev):
    """(the model's _Grads, the PriorGrads struct pointing at the tensors the backward writes, its layer array, which
    must outlive the backward call)."""
    grads = _Grads(model, dev, model.dim)
    n_layers = len(model.layers)
    layers = (PriorLayerGrads * n_layers)(*[
        PriorLayerGrads(**{f: grads.ptr(f"layers.{i}.{k}") for f, k in _LAYER_GRADS.items()})
        for i in range(n_layers)])
    table = PriorGrads(layers=C.cast(layers, C.POINTER(PriorLayerGrads)), n_layers=n_layers,
                       **{f: grads.ptr(k) for f, k in _NET_GRADS.items()})
    return grads, table, layers


class _PriorCEFunction(torch.autograd.Function):
    """GatedPixelCNN.cross_entropy and cross_entropy_ex with gradients: inputs are the model, the precision, the reduction, the options
    (None, or (fp32 weight or None, ignore_index, label_smoothing)), codes, labels and every parameter in
    ``parameters()`` order.  The forward keeps the training activations and each position's log-sum-exp
    (vqb_prior_ce_forward_*), not the logits; the backward (vqb_prior_ce_backward_*, in the forward's precision)
    recomputes the logits chunk by chunk and returns one gradient per parameter, as _PriorFunction does.  The weight
    takes no gradient."""

    @staticmethod
    def forward(ctx, model, precision, reduction, options, codes, labels, *params):
        keep = []
        net = model._net(keep)
        if options is None:
            opt = None
            loss, saved = ops.prior_ce_forward(net, codes, labels, reduction, precision, train=True)
        else:
            opt = ops.prior_ce_options(*options)
            loss, saved = ops.prior_ce_forward(net, codes, labels, reduction, precision, train=True, options=opt)
        ctx.model, ctx.net, ctx.keep, ctx.saved = model, net, keep, saved
        # options keeps alive the fp32 weight the struct points at, for the backward
        ctx.precision, ctx.reduction, ctx.options = precision, reduction, (options, opt)
        ctx.save_for_backward(codes, labels)
        return loss

    @staticmethod
    def backward(ctx, d_loss):
        if ctx.saved is None:           # the first backward freed the saved activations
            raise RuntimeError("GatedPixelCNN.cross_entropy: backward through the same call twice is not supported "
                               "(its saved activations are freed by the first backward)")
        codes, labels = ctx.saved_tensors
        grads, table, _layers = _grad_table(ctx.model, codes.device)
        if ctx.options[1] is None:
            ops.prior_ce_backward(ctx.net, codes, labels, ctx.reduction, _f32(d_loss), ctx.saved, table, ctx.precision)
        else:
            ops.prior_ce_backward(ctx.net, codes, labels, ctx.reduction, _f32(d_loss), ctx.saved, table, ctx.precision,
                                  ctx.options[1])
        ctx.saved = ctx.keep = ctx.options = None
        return (None,) * 6 + grads.finish()


class GatedPixelCNN(nn.Module):
    """Prior over code grids (models.py:89-143): layer 0 is a mask-A 7x7 layer without residual, the others mask-B
    3x3 layers with residual, then a 1x1 -> ReLU -> 1x1 head to input_dim logits.

    ``precision``: "fp32" (default) or "tf32", the arithmetic of ``forward`` (see the module docstring).  A plain
    attribute, so state dicts are the reference's; any other value raises ValueError from ``forward``.  ``generate``
    and ``complete`` are fp32 either way."""

    def __init__(self, input_dim=256, dim=64, n_layers=15, n_classes=10):
        super().__init__()
        self.precision = "fp32"
        self.dim = dim
        self.embedding = nn.Embedding(input_dim, dim)
        self.layers = nn.ModuleList()
        for i in range(n_layers):
            first = i == 0
            self.layers.append(GatedMaskedConv2d("A" if first else "B", dim, 7 if first else 3, not first, n_classes))
        self.output_conv = nn.Sequential(
            nn.Conv2d(dim, HIDDEN, 1),
            nn.ReLU(True),
            nn.Conv2d(HIDDEN, input_dim, 1),
        )
        self.apply(weights_init)

    def _check_layers(self):
        """P5: the kernels take one channel count and one class count for the whole net."""
        n_classes = self.layers[0].class_cond_embedding.num_embeddings if len(self.layers) else 1
        for i, l in enumerate(self.layers):
            dim, nc = l.horiz_resid.in_channels, l.class_cond_embedding.num_embeddings
            kernel = l.vert_stack.kernel_size[1]
            if dim != self.dim:
                raise RuntimeError(f"GatedPixelCNN: layer {i} has {dim} channels, the model has dim={self.dim}")
            if nc != n_classes:
                raise RuntimeError(f"GatedPixelCNN: layer {i} has {nc} classes, layer 0 has {n_classes}")
            if kernel > PRIOR_MAX_KERNEL:
                raise RuntimeError(f"GatedPixelCNN: layer {i} has kernel {kernel}; the kernels take odd kernels up to "
                                   f"{PRIOR_MAX_KERNEL}")

    def _net(self, keep):
        """(struct vqb_prior_net, its layer array); every tensor it points into is appended to `keep`.  At a dim the
        kernels do not take, the net at _padded_dim(dim) channels on zero-padded packings (DESIGN §8.5)."""
        self._check_layers()
        cp = _padded_dim(self.dim)
        layers = (PriorLayerWeights * len(self.layers))(*[l._weights(keep) for l in self.layers])
        o1, o2 = self.output_conv[0], self.output_conv[2]
        t = dict(embedding=_vector(self.embedding.weight, cp, self.dim, "embedding.weight"),
                 out1_w=_packed(o1.weight, _conv_key(cp, self.dim, "output_conv.0.weight")), out1_b=_f32(o1.bias),
                 out2_w=_packed(o2.weight, ("prior", 1, 1)), out2_b=_f32(o2.bias))
        keep.extend(t.values())
        keep.append(layers)
        return PriorNet(layers=layers, n_layers=len(self.layers), input_dim=self.embedding.num_embeddings, dim=cp,
                        n_classes=self.layers[0].class_cond_embedding.num_embeddings if len(self.layers) else 1,
                        **{k: v.data_ptr() for k, v in t.items()})

    def forward(self, x, label):
        """int64 codes (B,H,W) and labels (B,) -> fp32 logits (B, input_dim, H, W), in ``self.precision``.
        Differentiable with respect to the parameters when grad is enabled and any parameter requires grad."""
        precision = self.precision
        if precision not in ops.PRIOR_PRECISIONS:
            raise ValueError(f"GatedPixelCNN.precision must be one of {ops.PRIOR_PRECISIONS}, got {precision!r}")
        if x.dim() != 3:
            raise RuntimeError(f"GatedPixelCNN: expected codes of shape (B,H,W), got {tuple(x.shape)}")
        B, H, W = x.shape
        _square(H, W, "GatedPixelCNN")
        ops._require_cuda(x, "GatedPixelCNN codes")
        label = _labels(label, B, x.device, "GatedPixelCNN")
        x = x.detach().to(torch.int64).contiguous()
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            return _PriorFunction.apply(self, precision, x, label, *self.parameters())
        keep = []
        return ops.prior_forward(self._net(keep), x, label, precision)

    def _log_prob_args(self, x, label, n_given, per_position):
        """log_prob()'s host-side checks, in order, before any CUDA check or launch: the precision, n_given (an int),
        the codes' rank, n_given in [0, H*W], per_position only with n_given = 0, a square grid, the layers (P5),
        the label count (ValueError for the arguments, RuntimeError for the shapes, as forward and complete).  A
        per-image n_given is checked by _ragged and returned as an int64 device tensor."""
        what = "GatedPixelCNN.log_prob"
        if self.precision not in ops.PRIOR_PRECISIONS:
            raise ValueError(f"GatedPixelCNN.precision must be one of {ops.PRIOR_PRECISIONS}, got {self.precision!r}")
        ragged = _per_image(n_given)
        if not ragged and (isinstance(n_given, bool) or not isinstance(n_given, numbers.Integral)):
            raise ValueError(f"{what}: n_given must be an int, got {n_given!r}")
        if ragged and per_position:
            raise ValueError(f"{what}: per_position=True scores every position; n_given must be 0, got a per-image "
                             "n_given")
        if x.dim() != 3:
            raise RuntimeError(f"{what}: expected codes of shape (B,H,W), got {tuple(x.shape)}")
        B, H, W = x.shape
        if ragged:
            n_given = _ragged(n_given, x, what)
        else:
            if not 0 <= n_given <= H * W:
                raise ValueError(f"{what}: n_given must be in [0, H*W] = [0, {H * W}], got {n_given}")
            if per_position and n_given != 0:
                raise ValueError(f"{what}: per_position=True scores every position; n_given must be 0, got {n_given}")
        _square(H, W, what)
        self._check_layers()
        n = (label if torch.is_tensor(label) else torch.as_tensor(label)).numel()
        if n != B:
            raise RuntimeError(f"{what}: expected {B} labels, got {n}")
        return n_given if ragged else int(n_given)

    def _log_prob(self, x, label, n_given=0, per_position=False):
        """log_prob() as a graph-capturable call: the same checks and result, and for int64 contiguous codes and
        labels on the device no copy of either, so a CUDA graph captured around it reads x and label in place."""
        n_given = self._log_prob_args(x, label, n_given, per_position)
        B, H, W = x.shape
        ops._require_cuda(x, "GatedPixelCNN.log_prob codes")
        label = _labels(label, B, x.device, "GatedPixelCNN.log_prob")
        x = x.detach().to(torch.int64).contiguous()
        keep = []
        if torch.is_tensor(n_given):
            return ops.prior_log_prob_ragged(self._net(keep), x, label, n_given, self.precision)
        if n_given == H * W:                # nothing to score: no packing, no launch
            return torch.zeros((B,), dtype=torch.float32, device=x.device)
        return ops.prior_log_prob(self._net(keep), x, label, n_given, self.precision, per_position)

    def log_prob(self, x, label, *, n_given=0, per_position=False):
        """Log-likelihood of given code grids: int64 codes x (B,H,W) and labels (B,) (as forward takes them) ->
        fp32 (B,), entry b the sum over raster positions p = i*W + j >= n_given of
        log_softmax(forward(x, label)[b, :, i, j])[x[b, i, j]], in the model's ``precision``.  per_position=True
        returns the (B,H,W) fp32 map of every position's term instead (n_given must then be 0).  The first n_given
        positions are context, not scored, as in sample_completion; n_given = H*W gives zeros without a launch.

        n_given may also be per image: a 1-D integer tensor of B entries on x's device, or a list or tuple of B ints
        in [0, H*W].  Entry b is then the sum over image b's positions >= n_given[b], bitwise entry b of the scalar
        call on the same batch with n_given = n_given[b], in either precision (in fp32 also the call on image b
        alone), in one call with the scalar call's launches.  A
        tensor is never read on the host (no synchronisation: a captured graph follows new values written into it),
        and its values are clamped to [0, H*W] as codes are clamped; a list's values are checked (ValueError).
        per_position=True takes no per-image n_given (ValueError).  A 0-d tensor is not an int here (ValueError).

        -log_prob(x, label).sum() / x.numel() is the reference's validation loss (nn.CrossEntropyLoss on forward's
        logits), without writing the B*K*H*W logits: each position's logits are reduced on chip and the per-image
        sums are compensated fp32 sums in raster order, deterministic.  Codes outside [0, K-1] are clamped, as the
        embedding clamps them, and scored as the clamped code (torch's cross-entropy would raise).  Any layer stack
        forward takes is taken; with a layer 0 that reads the code it scores (not mask A without residual, P5) the
        result is the reference loop's cross-entropy, not a likelihood.

        Never differentiable: it runs the inference kernels even with grad enabled and parameters requiring grad,
        keeps no training activations, and returns a tensor without grad.  Train with forward plus the
        cross-entropy.  cross_entropy() is that training loss without the logits, and differentiable.  ValueError for a bad precision, n_given or per_position with n_given != 0; RuntimeError for
        forward's shape, layer (P5), label and device checks; every host-side check runs before any CUDA check."""
        return self._log_prob(x, label, n_given, per_position)

    def cross_entropy(self, x, label, *, reduction="mean"):
        """The reference's training loss without the B*K*H*W logits: int64 codes x (B,H,W) and labels (B,) (as forward
        takes them) -> the value of nn.CrossEntropyLoss(reduction=reduction)(forward(x, label).permute(0, 2, 3, 1)
        .reshape(-1, K), x.reshape(-1)), in the model's ``precision``: a 0-d fp32 tensor for reduction "mean" (over
        B*H*W) or "sum", the (B,H,W) fp32 map for "none".  The "none" values are bitwise -log_prob(x, label,
        per_position=True) in the same precision; "sum" and "mean" add them in fp64 in a fixed order (DESIGN §8.3).

        Differentiable with respect to every parameter under forward's rule (grad enabled and a parameter requiring
        grad): the call keeps the training activations and each position's log-sum-exp, and the backward recomputes
        the logits a chunk of positions at a time, so neither the logits nor their gradient is ever stored whole.
        Otherwise it runs the inference kernels and returns the same bits without a graph.  The upstream gradient is
        read on the device (no host synchronisation), so the loss, its backward and vqvae_b200.optim.Adam.step()
        capture into one CUDA graph; a second backward through the same call raises.

        Codes outside [0, K-1] are clamped, as the embedding clamps them, and scored and differentiated as the clamped
        code (torch's cross-entropy would raise).  For nn.CrossEntropyLoss's weight, ignore_index and label_smoothing
        use cross_entropy_ex, the same loss on the same kernels with those options.  Any layer stack forward takes is
        taken.  ValueError for a bad precision or reduction; RuntimeError for forward's shape, layer (P5), label and
        device checks; every host-side check runs before any CUDA check."""
        return self._cross_entropy("GatedPixelCNN.cross_entropy", x, label, reduction, None, None, 0.0)

    def cross_entropy_ex(self, x, label, *, reduction="mean", weight=None, ignore_index=None, label_smoothing=0.0):
        """cross_entropy with nn.CrossEntropyLoss's options: the value of nn.CrossEntropyLoss(weight=weight,
        ignore_index=ignore_index, label_smoothing=label_smoothing, reduction=reduction)(forward(x, label)
        .permute(0, 2, 3, 1).reshape(-1, K), x.reshape(-1)), in the model's ``precision``, without the B*K*H*W logits,
        differentiable and graph-capturable as cross_entropy is.  With every option at its default it is
        cross_entropy: the same calls and bits.

        Codes are clamped as in cross_entropy.  The options follow torch, with y the clamped code of a position, lse
        its log-sum-exp, l its logits, w the weights (all ones for None), W = sum_k w_k and e = label_smoothing:
        loss_p = (1 - e) * w_y * (lse - l_y) + (e / K) * (W * lse - sum_k w_k * l_k).
          weight: None, or a 1-D floating tensor of K class weights on the codes' device, used as contiguous fp32.
            It takes no gradient, and its values are only read on the device, so a captured graph uses the values
            it holds at each replay.
          ignore_index: None (the default: nothing is ignored; torch's default is -100, which here is a code that is
            clamped and scored like any other), or an int: a position is ignored iff its raw code, before clamping,
            equals it.  ignore_index=-100 gives torch's behaviour.  An ignored position scores 0 and takes no
            gradient, but is still embedded (clamped) as the model's input, since x is both input and target.
          label_smoothing: a float in [0, 1].
        "sum" adds loss_p; "mean" divides that sum by the sum of w_y over the positions not ignored, as torch does: a
        NaN loss when that is 0 (every position ignored gives zero gradients; scored targets of weight 0 give NaN
        gradients).  Both sums are fp64 in a fixed order, rounded once.  Options at their neutral values (unit
        weights, an ignore_index that occurs nowhere, 0 smoothing) give the same bits as cross_entropy.

        ValueError for a bad precision, reduction, label_smoothing (not a finite float in [0, 1]), ignore_index (not
        None or an int; bools rejected) or weight (rank, length, dtype); RuntimeError for a weight on another device
        than x, then cross_entropy's shape, layer (P5), label and device checks; every host-side check runs before any
        CUDA check."""
        return self._cross_entropy("GatedPixelCNN.cross_entropy_ex", x, label, reduction, weight, ignore_index,
                                   label_smoothing)

    def _cross_entropy(self, what, x, label, reduction, weight, ignore_index, label_smoothing):
        """cross_entropy and cross_entropy_ex: the checks in their order, then the call (without options when every
        option is at its default)."""
        precision = self.precision
        if precision not in ops.PRIOR_PRECISIONS:
            raise ValueError(f"GatedPixelCNN.precision must be one of {ops.PRIOR_PRECISIONS}, got {precision!r}")
        if not isinstance(reduction, str) or reduction not in ops.PRIOR_CE_REDUCTIONS:
            raise ValueError(f"{what}: reduction must be one of {ops.PRIOR_CE_REDUCTIONS}, got {reduction!r}")
        if (isinstance(label_smoothing, bool) or not isinstance(label_smoothing, numbers.Real)
                or not math.isfinite(label_smoothing) or not 0.0 <= label_smoothing <= 1.0):
            raise ValueError(f"{what}: label_smoothing must be a finite float in [0, 1], got {label_smoothing!r}")
        if ignore_index is not None and (isinstance(ignore_index, bool) or not isinstance(ignore_index, numbers.Integral)):
            raise ValueError(f"{what}: ignore_index must be None or an int, got {ignore_index!r}")
        if weight is not None:
            K = self.embedding.num_embeddings
            if not torch.is_tensor(weight) or weight.dim() != 1 or weight.numel() != K:
                shape = tuple(weight.shape) if torch.is_tensor(weight) else type(weight).__name__
                raise ValueError(f"{what}: weight must be a 1-D tensor of {K} entries, got {shape}")
            if not weight.is_floating_point():
                raise ValueError(f"{what}: weight must be a floating tensor, got {weight.dtype}")
            if weight.device != x.device:
                raise RuntimeError(f"{what}: weight is on {weight.device}, the codes on {x.device}")
        if x.dim() != 3:
            raise RuntimeError(f"{what}: expected codes of shape (B,H,W), got {tuple(x.shape)}")
        B, H, W = x.shape
        _square(H, W, what)
        self._check_layers()
        n = (label if torch.is_tensor(label) else torch.as_tensor(label)).numel()
        if n != B:
            raise RuntimeError(f"{what}: expected {B} labels, got {n}")
        ops._require_cuda(x, what + " codes")
        label = _labels(label, B, x.device, what)
        x = x.detach().to(torch.int64).contiguous()
        options = None
        if weight is not None or ignore_index is not None or label_smoothing != 0.0:
            w = weight.detach().to(torch.float32).contiguous() if weight is not None else None
            options = (w, None if ignore_index is None else int(ignore_index), float(label_smoothing))
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            return _PriorCEFunction.apply(self, precision, reduction, options, x, label, *self.parameters())
        keep = []
        if options is None:
            return ops.prior_ce_forward(self._net(keep), x, label, reduction, precision)[0]
        return ops.prior_ce_forward(self._net(keep), x, label, reduction, precision,
                                    options=ops.prior_ce_options(*options))[0]

    def _check_causal(self, what):
        """P5: the sampler needs a layer 0 that reads only the codes before the one being drawn."""
        first = self.layers[0] if len(self.layers) else None
        if first is not None and (first.mask_type != "A" or first.residual):
            raise RuntimeError(f"{what}: layer 0 must be mask A without residual (P5): this one reads "
                               "the code being drawn, so the logits are not causal in raster order")

    def _sample(self, label, u, step_logits=None):
        """generate() with given uniforms u (B,H,W) fp32: the code at (b,i,j) is the smallest k with u < CDF_k.
        fp32 whatever ``precision`` says."""
        B, H, W = u.shape
        _square(H, W, "GatedPixelCNN.generate")
        self._check_causal("GatedPixelCNN.generate")
        ops._require_cuda(u, "GatedPixelCNN.generate uniforms")
        label = _labels(label, B, u.device, "GatedPixelCNN.generate")
        keep = []
        return ops.prior_generate(self._net(keep), label, _f32(u), step_logits)

    def generate(self, label, shape=(8, 8), batch_size=64):
        """Sample (batch_size, *shape) int64 codes in raster order on the model's device.  Draws exactly one
        torch.rand((batch_size, H, W)) from the current CUDA generator, so torch.manual_seed makes it reproducible.
        fp32 whatever ``precision`` says: the per-position step kernels are bound by latency, not by FLOPs."""
        H, W = shape
        _square(H, W, "GatedPixelCNN.generate")
        dev = next(self.parameters()).device
        ops._require_cuda(torch.empty(0, device=dev), "GatedPixelCNN parameters")
        u = torch.rand((batch_size, H, W), device=dev)
        return self._sample(label, u)

    def _given(self, x, label, n_given):
        """complete()'s host-side checks, in order, before any CUDA check or launch: the codes' rank, n_given (an
        int, ValueError outside [0, H*W]), a square grid, layer 0 (P5), the label count.  Returns n_given: an int, or
        a per-image n_given as an int64 device tensor (_ragged's checks)."""
        ragged = _per_image(n_given)
        if not ragged:
            n_given = operator.index(n_given)
        if x.dim() != 3:
            raise RuntimeError(f"GatedPixelCNN.complete: expected codes of shape (B,H,W), got {tuple(x.shape)}")
        B, H, W = x.shape
        if ragged:
            n_given = _ragged(n_given, x, "GatedPixelCNN.complete")
        elif not 0 <= n_given <= H * W:
            raise ValueError(f"GatedPixelCNN.complete: n_given must be in [0, H*W] = [0, {H * W}], got {n_given}")
        _square(H, W, "GatedPixelCNN.complete")
        self._check_causal("GatedPixelCNN.complete")
        n = (label if torch.is_tensor(label) else torch.as_tensor(label)).numel()
        if n != B:
            raise RuntimeError(f"GatedPixelCNN.complete: expected {B} labels, got {n}")
        return n_given

    def _complete(self, label, u, x, n_given, step_logits=None):
        """complete() with given uniforms u (B,H,W) fp32: positions p = i*W + j < n_given are x's codes as given,
        the code at each later (b,i,j) is the smallest k with u < CDF_k of that step's logits.  step_logits: None or
        (B,H,W,K) fp32, written at the positions >= n_given only.  fp32 whatever ``precision`` says."""
        n_given = self._given(x, label, n_given)
        B, H, W = x.shape
        if tuple(u.shape) != (B, H, W):
            raise RuntimeError(f"GatedPixelCNN.complete: uniforms of shape {tuple(u.shape)} for codes {(B, H, W)}")
        ops._require_cuda(x, "GatedPixelCNN.complete codes")
        ops._require_cuda(u, "GatedPixelCNN.complete uniforms")
        label = _labels(label, B, x.device, "GatedPixelCNN.complete")
        x = x.detach().to(torch.int64).contiguous()
        keep = []
        if torch.is_tensor(n_given):
            return ops.prior_sample_ragged(self._net(keep), label, _f32(u), x, n_given, None, step_logits,
                                           log_prob=False)[0]
        if n_given == H * W:                # nothing to sample: no packing, no launch
            return x.clone()
        return ops.prior_complete(self._net(keep), label, _f32(u), x, n_given, step_logits)

    def complete(self, x, label, n_given):
        """Complete the code grids x (B,H,W) from their first n_given positions in raster order (p = i*W + j):
        positions < n_given are returned as x holds them, the rest are sampled as generate() samples them, each
        conditioned on everything before it; x's values there are never read.  A new int64 (B,H,W) tensor; x is not
        modified.  Draws exactly one torch.rand((B, H, W)) from the current CUDA generator whatever n_given is, so
        after the same torch.manual_seed, completing any prefix of generate()'s output returns that output.
        n_given = 0 is generate(); the restrictions are generate()'s (square grids, P5, fp32).

        n_given may also be per image: a 1-D integer tensor of B entries on x's device, or a list or tuple of B ints
        in [0, H*W].  Image b then keeps its positions < n_given[b] and is bitwise what complete() returns for image b
        alone with n_given = n_given[b] and the same uniforms.  One call runs generate()'s schedule, 1 + H*(L + W)
        launches for L layers whatever the values, each step skipping the images that have that position given.  A
        tensor is never read on the host (no synchronisation: a graph captured around _complete follows new values
        written into it), and its values are clamped to [0, H*W] as codes are clamped; a list's values are checked
        (ValueError).  An int or a 0-d integer tensor is one n_given for the batch, as before; a 1-D tensor of one
        entry takes the per-image path, with the same bits and its own launch count."""
        n_given = self._given(x, label, n_given)
        ops._require_cuda(x, "GatedPixelCNN.complete codes")
        u = torch.rand(tuple(x.shape), device=x.device)
        return self._complete(label, u, x, n_given)

    def _knobs(self, temperature, top_k, top_p, what):
        """The sampling knobs' checks (ValueError), as the C ABI sees them (fp32 temperature and top_p) ->
        PriorSampling; top_k None is 0 and top_p None is 1 (off)."""
        K = self.embedding.num_embeddings
        if isinstance(temperature, bool) or not isinstance(temperature, numbers.Real):
            raise ValueError(f"{what}: temperature must be a real number, got {temperature!r}")
        t32 = C.c_float(temperature).value
        if not (math.isfinite(t32) and t32 > 0):
            raise ValueError(f"{what}: temperature must be finite and > 0 in fp32, got {temperature!r}")
        if top_k is not None and (isinstance(top_k, bool) or not isinstance(top_k, numbers.Integral)
                                  or not 1 <= top_k <= K):
            raise ValueError(f"{what}: top_k must be None or an int in [1, {K}], got {top_k!r}")
        if top_p is not None:
            if isinstance(top_p, bool) or not isinstance(top_p, numbers.Real):
                raise ValueError(f"{what}: top_p must be None or a float in (0, 1], got {top_p!r}")
            p32 = C.c_float(top_p).value
            if not (0 < p32 <= 1 and 0 < top_p <= 1):
                raise ValueError(f"{what}: top_p must be None or a float in (0, 1] (fp32), got {top_p!r}")
        return PriorSampling(temperature=t32, top_k=0 if top_k is None else int(top_k),
                             top_p=1.0 if top_p is None else C.c_float(top_p).value)

    def _sample_with(self, label, u, x, n_given, temperature, top_k, top_p, step_logits=None):
        """sample() / sample_completion() with given uniforms u (B,H,W) fp32 -> (codes, log_prob).  x: the codes
        whose first n_given raster positions are kept (None with n_given = 0).  step_logits: None or (B,H,W,K) fp32,
        the raw logits of every sampled step.  fp32 whatever ``precision`` says."""
        what = "GatedPixelCNN.sample" if x is None else "GatedPixelCNN.sample_completion"
        if x is None:
            if u.dim() != 3:
                raise RuntimeError(f"{what}: expected uniforms of shape (B,H,W), got {tuple(u.shape)}")
            if _per_image(n_given) or n_given != 0:
                raise ValueError(f"{what}: n_given must be 0 without codes, got {n_given!r}")
            B, H, W = u.shape
            _square(H, W, what)
            self._check_causal(what)
        else:
            n_given = self._given(x, label, n_given)
            B, H, W = x.shape
            if tuple(u.shape) != (B, H, W):
                raise RuntimeError(f"{what}: uniforms of shape {tuple(u.shape)} for codes {(B, H, W)}")
        sampling = self._knobs(temperature, top_k, top_p, what)
        if x is not None:
            ops._require_cuda(x, what + " codes")
        ops._require_cuda(u, what + " uniforms")
        label = _labels(label, B, u.device, what)
        keep = []
        if x is not None:
            x = x.detach().to(torch.int64).contiguous()
            if torch.is_tensor(n_given):
                return ops.prior_sample_ragged(self._net(keep), label, _f32(u), x, n_given, sampling, step_logits)
            if n_given == H * W:            # nothing to sample: no packing, no launch
                return x.clone(), torch.zeros((B,), dtype=torch.float32, device=x.device)
        return ops.prior_sample(self._net(keep), label, _f32(u), x, n_given, sampling, step_logits)

    def sample(self, label, shape=(8, 8), batch_size=64, *, temperature=1.0, top_k=None, top_p=None):
        """generate() with control over the draw -> (codes (batch_size, H, W) int64, log_prob (batch_size,) fp32).
        Each code is drawn from the softmax of that step's logits divided by `temperature`, restricted to the top_k
        codes (ties at the threshold kept) and to the smallest top set holding top_p of the tempered probability
        (nucleus sampling), then renormalized; None turns a truncation off.  log_prob is the sum over the grid of the
        model's own log-probability of each sampled code (untempered, untruncated softmax), for ranking samples.
        Draws exactly one torch.rand((batch_size, H, W)), so with the default knobs and the same seed the codes are
        generate()'s.  ValueError for a knob out of range; the other restrictions are generate()'s (square grids,
        P5, fp32, one set of knobs for the batch)."""
        H, W = shape
        what = "GatedPixelCNN.sample"
        _square(H, W, what)
        self._check_causal(what)
        self._knobs(temperature, top_k, top_p, what)
        dev = next(self.parameters()).device
        ops._require_cuda(torch.empty(0, device=dev), "GatedPixelCNN parameters")
        u = torch.rand((batch_size, H, W), device=dev)
        return self._sample_with(label, u, None, 0, temperature, top_k, top_p)

    def sample_completion(self, x, label, n_given, *, temperature=1.0, top_k=None, top_p=None):
        """complete() with sample()'s knobs -> (codes (B,H,W) int64, log_prob (B,) fp32).  log_prob sums the
        model's log-probability over the sampled positions only (0 when n_given = H*W).  Draws exactly one
        torch.rand((B, H, W)), so with the default knobs and the same seed the codes are complete()'s.  n_given may be
        per image, as complete() takes it: log_prob[b] then sums over image b's sampled positions only (0 when
        n_given[b] = H*W), and codes, log_prob and step logits are bitwise the scalar call's on image b alone."""
        what = "GatedPixelCNN.sample_completion"
        n_given = self._given(x, label, n_given)
        self._knobs(temperature, top_k, top_p, what)
        ops._require_cuda(x, what + " codes")
        u = torch.rand(tuple(x.shape), device=x.device)
        return self._sample_with(label, u, x, n_given, temperature, top_k, top_p)

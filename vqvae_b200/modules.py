"""Host-side mirror of the reference's nn.Module API for the VQVAE.forward hot path.

Same class names, constructor signatures, attribute names and state-dict keys as
MishaLaskin/vqvae ``models/{vqvae,quantizer,encoder,decoder,residual}.py`` (SURVEY 8b),
so ``from models.vqvae import VQVAE`` keeps working (the top-level ``models`` package
re-exports these classes).  The nn.Conv2d / nn.ConvTranspose2d / nn.Embedding children
are kept ONLY as parameter containers (identical init order => identical weights under
the same torch seed, identical ``state_dict()``); their own ``forward`` is never used.
Every ``forward`` here launches the hand-written sm_90a kernels through the C ABI
(``include/vqvae_b200.h``).  ``VQVAE.forward`` is differentiable in training mode (``_VQVAEFunction``: model.train(),
grad enabled, a parameter or the image requiring grad), so the reference's ``main.py`` loop runs unchanged.  The
sub-modules (Encoder, Decoder, ResidualStack, ResidualLayer, the pre-quantization conv) follow the same rule when
called on their own, each through its own autograd Function whose backward is its slice of _VQVAEFunction.backward,
so notebook-style piecewise walks train too.  In eval mode and under no_grad the outputs carry no autograd graph
(unlike the reference, whose eval-mode outputs do).

Reference semantics reproduced on purpose (SURVEY 3.3):
  Q1  ResidualStack applies ONE shared ResidualLayer n times (residual.py:44-45)
  Q2  the in-place ReLU makes a layer relu(x) + f(relu(x)) and mutates the caller's x
  Q3  final F.relu after the stack; no activation after encoder conv 4 / decoder convT 0
  Q4  z_q is bitwise z + (e - z)
  Q7  the dense one-hot is built only for direct VectorQuantizer.forward callers
  Q8  verbose=True prints three shapes and then ``assert False``
"""
import contextlib
import math
import numbers

import torch
import torch.nn as nn

from . import _lib, ops
from .dist import reduce_vq_stats
from ._lib import NCHW, NHWC, PRECISIONS, RES_W2

# Default = what the reference itself computes on a GPU: fp32 tensors, convolutions on tensor cores in TF32 with fp32
# accumulation (PyTorch's torch.backends.cudnn.allow_tf32 default, SURVEY 2.2), bit-exact fp32 VQ.
DEFAULT_PRECISION = "tf32"
_PRECISION = {"value": DEFAULT_PRECISION}


def set_precision(name: str):
    """Arithmetic of the convolution layers:
    "tf32" (default) wgmma tf32 on fp32 activations, fp32 accumulation -- the reference's GPU arithmetic;
    "fp32"  FFMA on CUDA cores -- the reference's CPU numerics (end-to-end indices equal the CPU reference);
    "bf16"  bf16 activations and operands between layers (wgmma bf16), fp32 accumulation -- the arithmetic the
            reference reaches through torch.autocast(dtype=torch.bfloat16); fastest.
    The VQ distances / argmin are bit-exact fp32 in every mode."""
    if name not in PRECISIONS:
        raise ValueError(f"precision must be one of {sorted(PRECISIONS)}")
    _PRECISION["value"] = name


def get_precision() -> str:
    return _PRECISION["value"]


@contextlib.contextmanager
def precision(name: str):
    old = get_precision()
    set_precision(name)
    try:
        yield
    finally:
        set_precision(old)


def _param_tag(param):
    """Identity of a parameter's current value as far as torch tracks it.  ``.data`` edits (``w.data.mul_()``) do
    not bump ``_version`` and inference-mode tensors have no version counter at all: call
    ``vqvae_b200.invalidate_packed(model)`` after such edits (documented in INTEGRATION.md)."""
    try:
        ver = param._version
    except RuntimeError:            # "Inference tensors do not track version counter"
        ver = None
    return (ver, param.data_ptr(), str(param.device))


def _pack_key(conv, bf16):
    """The packing of a conv container's weight that the forward reads in a mode: ("f32", transposed), the K-major
    fp32 layout of vqb_pack_conv_weight_f32, or in the bf16 pipeline ("bf16", kind), the same K-major layout in bf16
    from vqb_pack_conv_weight_bf16, for the kind the layer's geometry names.  A container that the bf16 pipeline
    reads differently carries its key as ``_bf16_key``, set by the module that builds it."""
    transposed = isinstance(conv, nn.ConvTranspose2d)
    if not bf16:
        return ("f32", transposed)
    return getattr(conv, "_bf16_key", None) or \
        ("bf16", ops.conv_kind(conv.kernel_size[0], conv.stride[0], transposed, conv.out_channels))


def _packed_current(param, key):
    """Whether _packed(param, key) would return its cached packing without packing again."""
    tag = _param_tag(param)
    hit = getattr(param, "_vqb_packed", {}).get(key)
    return hit is not None and hit[0] == tag and tag[0] is not None


def pad_geometry(shape, cp, kout, kin):
    """The PackDesc geometry of a prior parameter of `shape` at Cp channels (the padded layouts of vqb_pack_layout):
    Cp in Cin_pad and the axis kinds in `transposed` = kout + 4*kin.  A 1-D parameter is (Cout, 1), a 2-D one
    (Cout, Cin), a conv weight (Cout, Cin, kh, kw)."""
    shape = tuple(shape)
    kh, kw = shape[2:4] if len(shape) == 4 else (1, 1)
    return dict(Cout=shape[0], Cin=shape[1] if len(shape) > 1 else 1, Cin_pad=cp, kh=kh, kw=kw,
                transposed=kout + 4 * kin)


def pack_spec(param, key):
    """The one place a packing-cache key becomes a layout and its geometry, for the conv weight `param`:
    ("f32", transposed), ("bf16", kind) (the residual 1x1's RES_W2 kind pads Cin to the kernels' 64) or
    ("prior", rows, cols), the kept taps of a prior conv (vqvae_b200/prior.py).  Returns (pack, layouts):
    pack(param, out) runs the key's single-packing entry point (refilling `out` when it has the right size) and returns
    the buffer, or None for a bf16 shape the kernels do not cover; layouts is the same packing as vqb_repack_multi
    descriptors, a list of (byte offset into that buffer, PackDesc fields), empty when there is no packing.

    A prior at a dim the kernels do not take runs them at Cp channels on zero-padded copies (DESIGN §8.5), under two
    more keys: ("prior_pad", rows, cols, Cp, kout, kin), the ("prior", rows, cols) packing of the padded conv weight,
    and ("pad", Cp, kout, kin), any prior parameter (bias, embedding, conv weight) in its own layout at the padded
    widths; kout and kin are the kinds of its first two axes (vqb_pack_layout: 0 kept, 1 dim-wide, 2 a gate axis
    padded per half).  Both are filled by one vqb_repack_multi descriptor, padding included."""
    kind = key[0]
    if kind in ("prior_pad", "pad"):
        cp, kout, kin = key[-3:]
        g = pad_geometry(param.shape, cp, kout, kin)
        coutp, cinp = ops.pad_width(g["Cout"], kout, cp), ops.pad_width(g["Cin"], kin, cp)
        if kind == "prior_pad":
            f = dict(g, layout=_lib.PACK_PRIOR_PAD_F32, rows=key[1], cols=key[2])
            n = key[1] * key[2] * cinp * coutp
        else:
            f = dict(g, layout=_lib.PACK_PAD_F32, rows=0, cols=0)
            n = coutp * cinp * g["kh"] * g["kw"]
        return (lambda p, out: ops.pack_one(p, f, n, out=out)), [(0, f)]
    if kind == "prior":
        cout, cin, kh, kw = param.shape
        f = dict(layout=_lib.PACK_PRIOR_F32, Cout=cout, Cin=cin, Cin_pad=cin, kh=kh, kw=kw, transposed=0,
                 rows=key[1], cols=key[2])
        return (lambda p, out: ops.prior_pack_weight(p, key[1], key[2], out=out)), [(0, f)]
    transposed = bool(key[1]) if kind == "f32" else ops.KIND_GEOMETRY[key[1]][2]
    cin, cout, kh, kw = param.shape if transposed else (param.shape[1], param.shape[0]) + tuple(param.shape[2:])
    geo = dict(Cout=cout, Cin=cin, kh=kh, kw=kw, transposed=int(transposed), rows=0, cols=0)
    if kind == "f32":
        layouts = [(0, dict(geo, layout=_lib.PACK_F32, Cin_pad=cin))]
        if transposed and kh == 4 and kw == 4 and cout <= 4:         # vqb_pack_conv_weight_f32 adds the shuffle form
            layouts.append((4 * kh * kw * cout * cin, dict(geo, layout=_lib.PACK_SHUFFLE_F32, Cin_pad=cin)))
        return (lambda p, out: ops.pack_conv_weight(p, key[1], out=out)), layouts
    nbytes = ops.lib().vqb_conv_bf16_packed_bytes(key[1], cout, cin)
    if nbytes == 0:
        layouts = []
    elif key[1] == _lib.CONVT_K4S2_OUT:
        layouts = [(0, dict(geo, layout=_lib.PACK_SHUFFLE_BF16, Cin_pad=cin))]
    else:                                                               # the padded channel count, from the byte size
        layouts = [(0, dict(geo, layout=_lib.PACK_BF16, Cin_pad=nbytes // (2 * kh * kw * cout)))]
    return (lambda p, out: ops.pack_conv_weight_bf16(p, key[1], out=out)), layouts


def _packed(param, key):
    """The packing `key` (see _pack_key, pack_spec) of a conv weight, cached ON the parameter object (so the cache
    dies with it).  When the parameter changes (load_state_dict, optimizer step, .to()) the SAME device buffer is
    repacked in place whenever its size still fits, so CUDA graphs captured around a forward keep reading current
    weights after ``repack`` (HostPipeline checks the tags before every replay).  vqvae_b200.optim.Adam refreshes
    every cached packing of the parameters it updates in the same buffers, and their tags with them."""
    cache = getattr(param, "_vqb_packed", None)
    if cache is None:
        cache = {}
        param._vqb_packed = cache
    hit = cache.get(key)
    if _packed_current(param, key):
        return hit[1]
    tag = _param_tag(param)
    old = hit[1] if hit is not None and hit[1] is not None and hit[1].device == param.device else None
    pack, _ = pack_spec(param, key)
    buf = pack(param, old)
    cache[key] = (tag, buf)
    return buf


def _convs(module):
    """Every conv container under `module`, each once (a shared ResidualLayer included once)."""
    return [m for m in module.modules() if isinstance(m, (nn.Conv2d, nn.ConvTranspose2d))]


_INVALIDATIONS = {"n": 0}


def invalidate_packed(model):
    """Drop every cached weight packing of ``model`` (after ``param.data`` edits, which torch does not version).
    Buffers are kept and refilled in place at the next forward / ``HostPipeline.push``."""
    _INVALIDATIONS["n"] += 1
    for p in model.parameters():
        cache = getattr(p, "_vqb_packed", None)
        if cache:
            for k, (tag, buf) in list(cache.items()):
                cache[k] = ((None, None, None), buf)


def packed_state(model):
    """Tuple of the parameters' tags: changes whenever a weight packing may be stale."""
    return tuple(_param_tag(p) for p in model.parameters())


def _conv_precision():
    """Arithmetic of the fp32-activation entry points (vqb_conv2d_f32 & co): "bf16" has no meaning for them -- bf16
    operands exist only inside the fused VQVAE.forward / encode / decode pipeline -- so piecewise sub-module calls
    run the TF32 kernels in that mode (more accurate than asked, never less)."""
    name = get_precision()
    return PRECISIONS["tf32" if name == "bf16" else name]


def _bias(conv):
    if conv.bias is None:
        return None
    b = conv.bias.detach()
    return b if b.dtype == torch.float32 else b.float()


def _run_conv(conv, x, B, H, W, bf16=False, *, in_layout=NHWC, out_layout=NHWC, relu=False, out_f32=False):
    """Forward of one nn.Conv2d / nn.ConvTranspose2d container -> (output, OH, OW): vqb_conv2d_f32 on fp32
    activations in `in_layout` / `out_layout`, or (bf16) vqb_conv2d_bf16 on bf16 NHWC activations, fp32 out if
    `out_f32` (the output layer's kind always writes the fp32 NCHW module output)."""
    kh, kw = conv.kernel_size
    stride, pad = conv.stride[0], conv.padding[0]
    key = _pack_key(conv, bf16)
    w = _packed(conv.weight, key)
    if bf16:
        y = ops.conv2d_bf16(x, w, _bias(conv), B=B, Cin=conv.in_channels, H=H, W=W, Cout=conv.out_channels,
                            kind=key[1], relu=relu, out_f32=out_f32)
    else:
        y = ops.conv2d(x, w, _bias(conv), B=B, Cin=conv.in_channels, H=H, W=W, Cout=conv.out_channels,
                       kh=kh, kw=kw, stride=stride, pad=pad, transposed=key[1], in_layout=in_layout,
                       out_layout=out_layout, relu=relu, precision=_conv_precision())
    return (y,) + ops.conv_out_hw(H, W, kh, kw, stride, pad, isinstance(conv, nn.ConvTranspose2d))


def _trains(module, *inputs):
    """Whether a call of `module` on `inputs` takes the differentiable path: training mode, grad enabled, and an input
    or one of the module's parameters requiring grad (VQVAE.forward's rule, for every module of the family)."""
    return module.training and torch.is_grad_enabled() and \
        (any(x.requires_grad for x in inputs) or any(p.requires_grad for p in module.parameters()))


def _check_input(x, channels, what):
    if x.dim() != 4:
        raise RuntimeError(f"{what}: expected a 4-D (B,C,H,W) tensor, got {tuple(x.shape)}")
    if x.shape[1] != channels:
        raise RuntimeError(f"{what}: expected {channels} input channels, got {x.shape[1]}")
    ops._require_cuda(x, what + " input")


def _prep_input(x, channels, what):
    _check_input(x, channels, what)
    x = x.detach()
    if x.dtype != torch.float32:
        x = x.float()
    return x if x.is_contiguous() else x.contiguous()


def _prep_relu_input(x, channels, what, in_place=True):
    """(relu(x) NHWC, B, H, W) for a residual module's forward.  Q2: nn.ReLU(True) rewrites the caller's tensor before
    the sum is formed, so with `in_place` a contiguous fp32 `x` is ReLU'd where it lies."""
    xp = _prep_input(x, channels, what)
    B, _, H, W = xp.shape
    if in_place and x.is_contiguous() and x.dtype == torch.float32 and not x.requires_grad:
        xp = ops.relu_(x)
    else:
        xp = ops.relu_(xp.clone())
    return ops.nchw_to_nhwc(xp), B, H, W


class ResidualLayer(nn.Module):
    """One residual layer (reference models/residual.py:8-29)."""

    def __init__(self, in_dim, h_dim, res_h_dim):
        super().__init__()
        self.res_block = nn.Sequential(
            nn.ReLU(True),
            nn.Conv2d(in_dim, res_h_dim, kernel_size=3, stride=1, padding=1, bias=False),
            nn.ReLU(True),
            nn.Conv2d(res_h_dim, h_dim, kernel_size=1, stride=1, bias=False),
        )
        self.res_block[3]._bf16_key = ("bf16", RES_W2)      # bf16: the fused layer's second GEMM, Cmid padded to 64

    def _apply_nhwc(self, r, B, H, W, relu_out, bf16=False):
        """r = relu(x) in NHWC (bf16 in the bf16 pipeline).  Returns r + W2.relu(W1 (*) r), optionally ReLU'd
        (the next consumer always applies ReLU first, residual.py:19,50).  One fused launch in either mode."""
        c1, c2 = self.res_block[1], self.res_block[3]
        w1, w2 = _packed(c1.weight, _pack_key(c1, bf16)), _packed(c2.weight, _pack_key(c2, bf16))
        if bf16:
            return ops.residual_layer_bf16(r, w1, w2, B=B, H=H, W=W, C=c1.in_channels, Cmid=c1.out_channels,
                                           relu_out=relu_out)
        return ops.residual_layer(r, w1, w2, B=B, H=H, W=W, C=c1.in_channels, Cmid=c1.out_channels, relu_out=relu_out,
                                  precision=_conv_precision())

    def forward(self, x):
        if _trains(self, x):
            return _residual_train(self, [self], x, self.res_block[1].in_channels, "ResidualLayer")
        r, B, H, W = _prep_relu_input(x, self.res_block[1].in_channels, "ResidualLayer")
        return ops.nhwc_to_nchw(self._apply_nhwc(r, B, H, W, relu_out=False))


class ResidualStack(nn.Module):
    """n applications of ONE shared ResidualLayer, then ReLU (models/residual.py:32-51)."""

    def __init__(self, in_dim, h_dim, res_h_dim, n_res_layers):
        super().__init__()
        self.n_res_layers = n_res_layers
        self.stack = nn.ModuleList([ResidualLayer(in_dim, h_dim, res_h_dim)] * n_res_layers)

    def _apply_nhwc(self, r, B, H, W, bf16=False):
        """r = relu(stack input), NHWC (bf16 in the bf16 pipeline).  Output = the stack's result (post F.relu)."""
        if len(self.stack) == 0:
            return r
        layer = self.stack[0]
        # bf16: one launch per application.  fp32 / tf32: one per layer when the layers are not the reference's
        # [layer] * n construction, else the whole stack in one call.
        if bf16 or any(l is not layer for l in self.stack):
            for l in self.stack:
                r = l._apply_nhwc(r, B, H, W, relu_out=True, bf16=bf16)
            return r
        c1, c2 = layer.res_block[1], layer.res_block[3]
        return ops.residual_stack(r, _packed(c1.weight, _pack_key(c1, False)), _packed(c2.weight, _pack_key(c2, False)),
                                  B=B, H=H, W=W, C=c1.in_channels, Cmid=c1.out_channels, n_layers=len(self.stack),
                                  precision=_conv_precision())

    def forward(self, x):
        ch = self.stack[0].res_block[1].in_channels if len(self.stack) else x.shape[1]
        if _trains(self, x):
            return _residual_train(self, list(self.stack), x, ch, "ResidualStack")
        # an empty stack has no in-place ReLU: only its final F.relu, on a copy
        r, B, H, W = _prep_relu_input(x, ch, "ResidualStack", in_place=len(self.stack) > 0)
        return ops.nhwc_to_nchw(self._apply_nhwc(r, B, H, W))


def _latent_block(head, stack, h, B, H, W, tail=None):
    """VQVAE._walk's TF32 inference path: the k3 s1 conv `head` (its ReLU folded in), the ResidualStack `stack` and, given,
    the 1x1 conv `tail` on NHWC h as one launch (ops.latent_block) -> the output of the last of them, bitwise the
    separate launches.  None (nothing allocated or launched) when the stack is not the reference's [layer] * n
    construction with n >= 1 or the library does not take the shapes (the tail's Cout included): the caller runs the
    separate launches then."""
    if len(stack.stack) == 0 or any(l is not stack.stack[0] for l in stack.stack):
        return None
    c1, c2 = stack.stack[0].res_block[1], stack.stack[0].res_block[3]
    transposed = isinstance(head, nn.ConvTranspose2d)
    return ops.latent_block(h, _packed(head.weight, _pack_key(head, False)), _bias(head),
                            _packed(c1.weight, _pack_key(c1, False)), _packed(c2.weight, _pack_key(c2, False)),
                            None if tail is None else _packed(tail.weight, _pack_key(tail, False)),
                            None if tail is None else _bias(tail),
                            B=B, Cin=head.in_channels, H=H, W=W, C=head.out_channels, Cmid=c1.out_channels,
                            n_layers=len(stack.stack), transposed=transposed,
                            tail_cout=0 if tail is None else tail.out_channels)


def _decoder_tail(convt, out, d_out, B, H, W, keep_h):
    """VQVAE._walk's TF32 path: the k4 s2 transposed conv `convt` (its ReLU folded in) and the output layer `out` on
    NHWC d_out as one launch (ops.decoder_tail) -> (x_hat NCHW, h NHWC if keep_h else None), bitwise the separate
    launches.  None (nothing allocated or launched) when the library does not take the shapes: the caller runs the
    separate launches then."""
    return ops.decoder_tail(d_out, _packed(convt.weight, _pack_key(convt, False)), _bias(convt),
                            _packed(out.weight, _pack_key(out, False)), _bias(out), B=B, Cin=convt.in_channels, H=H,
                            W=W, C=convt.out_channels, Cout=out.out_channels, keep_h=keep_h)


class Encoder(nn.Module):
    """q_theta(z|x): models/encoder.py:9-43."""

    def __init__(self, in_dim, h_dim, n_res_layers, res_h_dim):
        super().__init__()
        kernel, stride = 4, 2
        self.conv_stack = nn.Sequential(
            nn.Conv2d(in_dim, h_dim // 2, kernel_size=kernel, stride=stride, padding=1),
            nn.ReLU(),
            nn.Conv2d(h_dim // 2, h_dim, kernel_size=kernel, stride=stride, padding=1),
            nn.ReLU(),
            nn.Conv2d(h_dim, h_dim, kernel_size=kernel - 1, stride=stride - 1, padding=1),
            ResidualStack(h_dim, h_dim, res_h_dim, n_res_layers),
        )
        self.conv_stack[0]._bf16_key = ("f32", False)      # bf16: vqb_conv_in_bf16 reads the fp32 packing

    def _forward_nhwc(self, x, bf16=False, acts=None, tail=None, fuse=False):
        """x: prepared NCHW fp32 CUDA tensor -> (NHWC activation, bf16 in the bf16 pipeline, B, H, W).  `acts` (a
        dict, training walk) receives the post-ReLU outputs of the three convs and the stack's output as "enc".
        `tail` (VQVAE's pre-quantization conv): applied to the stack's output, which makes the result z_e (fp32 in
        every mode).  `fuse` (VQVAE._walk's TF32 inference path): conv 4, the stack and `tail` in one launch when
        _latent_block takes them."""
        B, _, H, W = x.shape
        cs = self.conv_stack
        if bf16:      # the 3-channel image has its own entry point: fp32 NCHW in, bf16 NHWC out
            h = ops.conv_in_bf16(x, _packed(cs[0].weight, _pack_key(cs[0], True)), _bias(cs[0]), B=B, H=H, W=W,
                                 Cout=cs[0].out_channels, relu=True)
            H, W = H // 2, W // 2
        else:
            h, H, W = _run_conv(cs[0], x, B, H, W, in_layout=NCHW, relu=True)
        a1 = h
        h, H, W = _run_conv(cs[2], h, B, H, W, bf16, relu=True)
        a2 = h
        z = _latent_block(cs[4], cs[5], h, B, H, W, tail) if fuse else None      # k3 s1 p1: H, W unchanged
        if z is not None:
            return z, B, H, W
        # the only consumer of conv 4 is the stack, whose first op is ReLU (or, with an
        # empty stack, its final F.relu): fold that ReLU into this epilogue (Q2/Q3).
        h, H, W = _run_conv(cs[4], h, B, H, W, bf16, relu=True)
        a3 = h
        h = cs[5]._apply_nhwc(h, B, H, W, bf16)
        if acts is not None:
            acts["enc"] = (a1, a2, a3, h)
        if tail is not None:
            h = _run_conv(tail, h, B, H, W, bf16, out_f32=True)[0]
        return h, B, H, W

    def forward(self, x):
        if _trains(self, x):
            if x.dim() == 4 and (x.shape[2] % 4 or x.shape[3] % 4):
                # the input gradients run the adjoint convs, which map the 2x-strided grids back onto exactly twice
                # their size: an image side that is not a multiple of 4 has rows no adjoint reaches (Q11)
                raise RuntimeError("Encoder: training needs an image height and width divisible by 4 (Q11); the "
                                   "inference call (model.eval() or torch.no_grad()) takes any size")
            return _EncoderFunction.apply(self, x, *self.parameters())
        x = _prep_input(x, self.conv_stack[0].in_channels, "Encoder")
        h, _, _, _ = self._forward_nhwc(x)
        return ops.nhwc_to_nchw(h)


class Decoder(nn.Module):
    """p_phi(x|z): models/decoder.py:9-39."""

    def __init__(self, in_dim, h_dim, n_res_layers, res_h_dim):
        super().__init__()
        kernel, stride = 4, 2
        self.inverse_conv_stack = nn.Sequential(
            nn.ConvTranspose2d(in_dim, h_dim, kernel_size=kernel - 1, stride=stride - 1, padding=1),
            ResidualStack(h_dim, h_dim, res_h_dim, n_res_layers),
            nn.ConvTranspose2d(h_dim, h_dim // 2, kernel_size=kernel, stride=stride, padding=1),
            nn.ReLU(),
            nn.ConvTranspose2d(h_dim // 2, 3, kernel_size=kernel, stride=stride, padding=1),
        )

    def _forward_from_nhwc(self, z, B, H, W, bf16=False, acts=None, fuse=False, fuse_tail=False):
        """z: NHWC (B,H,W,in_dim), bf16 in the bf16 pipeline -> x_hat fp32 NCHW.  `acts` (a dict, training walk)
        receives the stack's input and output and the last hidden activation as "dec".  `fuse` (VQVAE._walk's TF32
        inference path): the first conv and the stack in one launch when _latent_block takes them.  `fuse_tail`
        (VQVAE._walk in TF32, both walks): the last two layers in one launch when _decoder_tail takes them."""
        ics = self.inverse_conv_stack
        h = _latent_block(ics[0], ics[1], z, B, H, W) if fuse else None      # k3 s1 p1: H, W unchanged
        if h is None:
            h, H, W = _run_conv(ics[0], z, B, H, W, bf16, relu=True)     # ReLU of the stack folded in (Q2/Q3)
            d1 = h
            h = ics[1]._apply_nhwc(h, B, H, W, bf16)
        d_out = h
        tail = _decoder_tail(ics[2], ics[4], d_out, B, H, W, acts is not None) if fuse_tail else None
        if tail is not None:
            x_hat, h = tail
        else:
            h, H, W = _run_conv(ics[2], h, B, H, W, bf16, relu=True)
            x_hat = _run_conv(ics[4], h, B, H, W, bf16, out_layout=NCHW)[0]
        if acts is not None:
            acts["dec"] = (d1, d_out, h)
        return x_hat

    def forward(self, x):
        if _trains(self, x):
            return _DecoderFunction.apply(self, x, *self.parameters())
        x = _prep_input(x, self.inverse_conv_stack[0].in_channels, "Decoder")
        B, _, H, W = x.shape
        return self._forward_from_nhwc(ops.nchw_to_nhwc(x), B, H, W)


class _VQFunction(torch.autograd.Function):
    """Training-mode VectorQuantizer core (SURVEY 8f rank 3): the fused forward kernel plus vqb_vq_backward_f32 --
    straight-through gradient to z, commitment / codebook gradients scatter-added by index (quantizer.py:63-67).
    With an EMA codebook (`vq.decay` set) the loss is the commitment term alone, `update` runs the EMA update right
    after the VQ kernel, and the backward is vqb_vq_commit_backward_f32 on the forward's own z_q rows: the codebook is
    neither saved (the update rewrites it in place) nor given a gradient."""

    @staticmethod
    def forward(ctx, z_rows, codebook, beta, vq, update):
        z_rows, codebook = z_rows.detach().contiguous(), codebook.detach().contiguous()
        idx, zq, sse, hist = ops.vq_forward(z_rows, codebook)
        N, D = z_rows.shape
        ctx.beta, ctx.ema = beta, vq.decay is not None
        if ctx.ema:
            loss, perp = ops.vq_finish_ema(sse, hist, N, codebook.shape[0], D, beta)
            if update:
                vq._ema_update(z_rows, idx, hist)
            ctx.save_for_backward(z_rows, zq)
        else:
            loss, perp = ops.vq_finish(sse, hist, N, codebook.shape[0], D, beta)
            ctx.save_for_backward(z_rows, codebook, idx)
        ctx.mark_non_differentiable(perp, idx)
        return loss, zq, perp, idx

    @staticmethod
    def backward(ctx, g_loss, g_zq, _g_perp, _g_idx):
        if ctx.ema:
            z_rows, zq = ctx.saved_tensors
            return ops.vq_commit_backward(g_zq, g_loss, z_rows, zq, ctx.beta), None, None, None, None
        z_rows, codebook, idx = ctx.saved_tensors
        dz, dE = ops.vq_backward(g_zq, g_loss, z_rows, codebook, idx, ctx.beta)
        return dz, dE, None, None, None


def _check_ema(decay, eps):
    """ValueError unless decay is None or in [0, 1) and eps is finite and > 0."""
    if decay is not None:
        try:
            d = float(decay)
        except (TypeError, ValueError):
            raise ValueError(f"decay must be None or a number in [0, 1), got {decay!r}") from None
        if not 0.0 <= d < 1.0:
            raise ValueError(f"decay must be None or a number in [0, 1), got {decay!r}")
    try:
        e = float(eps)
    except (TypeError, ValueError):
        raise ValueError(f"eps must be a finite number > 0, got {eps!r}") from None
    if not (math.isfinite(e) and e > 0.0):
        raise ValueError(f"eps must be a finite number > 0, got {eps!r}")


class VectorQuantizer(nn.Module):
    """Discretisation bottleneck: models/quantizer.py:10-76.

    ``decay`` (keyword only, default None = the reference's module): learn the codebook by exponential moving averages
    (van den Oord et al. 2017, appendix A.1) instead of by gradient.  ``embedding.weight`` then takes no gradient, two
    fp32 buffers hold the averages -- ``ema_cluster_size`` N (K,) and ``ema_embed_sum`` m (K, D), initialised as if
    each code had been assigned one vector equal to itself (N = 1, m = e) -- and every differentiable call in training
    mode (grad enabled, z requiring grad) updates N, m and the codebook in place (vqb_vq_ema_update_f32):
    N <- decay N + (1-decay) n_k,  m <- decay m + (1-decay) s_k,  e = m / ((N + eps) / (n + K eps) * n).  The loss is
    the commitment term beta * mse((sg[z_q], z)) on every path.

    ``dead_code_threshold`` (attribute, default None = off; EMA codebooks of at most 8192 codes): after each update,
    every code whose N fell below it moves onto a row of the batch just quantized, drawn uniformly without replacement
    from one ``torch.rand`` per update (vqb_vq_ema_restart_f32): e <- z_row, m <- t z_row, N <- t.  ``last_restarts``,
    a device int32 (1,) tensor written in place, holds how many codes the last update restarted."""

    _MAX_RESTART_CODES = 8192

    def __init__(self, n_e, e_dim, beta, *, decay=None, eps=1e-5):
        _check_ema(decay, eps)
        super().__init__()
        self.n_e = n_e
        self.e_dim = e_dim
        self.beta = beta
        self.decay = None if decay is None else float(decay)
        self.eps = float(eps)
        self._dead_code_threshold = None
        self.embedding = nn.Embedding(self.n_e, self.e_dim)
        self.embedding.weight.data.uniform_(-1.0 / self.n_e, 1.0 / self.n_e)
        if self.decay is not None:
            self.embedding.weight.requires_grad_(False)
            self.register_buffer("ema_cluster_size", torch.ones(self.n_e))
            self.register_buffer("ema_embed_sum", self.embedding.weight.detach().clone())
            self.register_buffer("last_restarts", torch.zeros(1, dtype=torch.int32), persistent=False)
        else:
            self.last_restarts = None

    _EMA_KEYS = ("ema_cluster_size", "ema_embed_sum")

    @property
    def dead_code_threshold(self):
        """None (no restarts) or the cluster size t below which an EMA code is restarted after each update."""
        return self._dead_code_threshold

    @dead_code_threshold.setter
    def dead_code_threshold(self, value):
        if value is None:
            self._dead_code_threshold = None
            return
        if isinstance(value, bool) or not isinstance(value, numbers.Real) or not math.isfinite(value) or value <= 0:
            raise ValueError(f"dead_code_threshold must be None or a finite number > 0, got {value!r}")
        if self.decay is None:
            raise ValueError("dead_code_threshold needs an EMA codebook (decay=...): the gradient-trained codebook "
                             "has no cluster sizes")
        if self.n_e > self._MAX_RESTART_CODES:
            raise ValueError(f"dead_code_threshold supports at most {self._MAX_RESTART_CODES} codes, not {self.n_e}")
        self._dead_code_threshold = float(value)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        """A state dict without the EMA buffers (a reference checkpoint, a decay=None model) loads into an EMA model:
        the buffers restart from the loaded codebook (N = 1, m = e)."""
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                                      error_msgs)
        w = state_dict.get(prefix + "embedding.weight")
        keys = [prefix + k for k in self._EMA_KEYS]
        if self.decay is None or w is None or not all(k in missing_keys for k in keys):
            return
        with torch.no_grad():
            self.ema_cluster_size.fill_(1.0)
            self.ema_embed_sum.copy_(w)
        for k in keys:
            missing_keys.remove(k)

    def _ema_update(self, rows, idx, hist):
        """One EMA update of N, m and the codebook from the rows the VQ kernel just quantized; bumps their version
        counters as an optimizer step does.  With a dead_code_threshold, the restart follows on the same stream, its
        uniforms drawn whether or not any code is dead, so the RNG stream does not depend on the data."""
        w = self.embedding.weight
        ops.vq_ema_update(rows, idx, hist, self.decay, self.eps, self.ema_cluster_size, self.ema_embed_sum, w.detach())
        if self._dead_code_threshold is not None:
            u = torch.rand((rows.shape[0],), device=rows.device)
            ops.vq_ema_restart(rows, u, self._dead_code_threshold, self.ema_cluster_size, self.ema_embed_sum,
                               w.detach(), self.last_restarts)
        torch.autograd.graph.increment_version([w, self.ema_cluster_size, self.ema_embed_sum])

    def init_codebook_kmeans(self, z, iters=10):
        """Fit the codebook to one batch by k-means, in place (vqb_vq_kmeans_f32).  z is (B, e_dim, H, W) fp32 CUDA, what
        forward takes; its rows, in forward's order, are the data.  The K codes start on K distinct rows drawn uniformly
        without replacement (one ``torch.rand((B*H*W,))`` from the current generator); each of the `iters` Lloyd steps
        then assigns every row to its nearest code by forward's fp32 distances and moves every code that took a row to
        their mean (a code that took none stays).  iters=0 only seeds.  Returns the sum of squared distances before each
        step, a float64 (iters,) device tensor that the library never reads back.

        Records no autograd graph and leaves ``training`` as it is; the codebook's version counter moves, as after an
        optimizer step.  An EMA codebook's averages restart from the new codebook (N = 1, m = e).  A row holding a NaN
        takes over the codebook: finding one would need a host synchronisation, so the call does not look."""
        self._check_kmeans(iters)
        _check_input(z, self.e_dim, "VectorQuantizer")
        self._check_kmeans_rows(z.shape[0] * z.shape[2] * z.shape[3])
        with torch.no_grad():
            z = _prep_input(z, self.e_dim, "VectorQuantizer")
            return self._kmeans_rows(ops.nchw_to_nhwc(z).view(-1, self.e_dim), iters)

    def _check_kmeans(self, iters):
        """init_codebook_kmeans's checks of its arguments, then (_check_kmeans_rows) of the batch, made before anything
        is allocated or launched."""
        if isinstance(iters, bool) or not isinstance(iters, numbers.Integral) or iters < 0:
            raise ValueError(f"iters must be an int >= 0, got {iters!r}")
        if self.n_e > self._MAX_RESTART_CODES:
            raise ValueError(f"init_codebook_kmeans supports at most {self._MAX_RESTART_CODES} codes, not {self.n_e}")
        if self.e_dim % 4:
            raise ValueError(f"init_codebook_kmeans needs e_dim % 4 == 0, not {self.e_dim}")

    def _check_kmeans_rows(self, n_rows):
        if n_rows < self.n_e:
            raise ValueError(f"init_codebook_kmeans needs at least one row per code: {n_rows} rows, {self.n_e} codes")
        ops._require_cuda(self.embedding.weight, "VectorQuantizer codebook")

    def _kmeans_rows(self, rows, iters):
        """init_codebook_kmeans on checked (N, e_dim) fp32 rows, under no_grad."""
        w = self.embedding.weight
        cb = self._codebook()
        sse = ops.vq_kmeans(rows, torch.rand((rows.shape[0],), device=rows.device), int(iters), cb)
        if cb.data_ptr() == w.data_ptr():
            torch.autograd.graph.increment_version([w])          # the kernels wrote it in place
        else:
            w.copy_(cb)
        if self.decay is not None:                               # as _load_from_state_dict restarts them
            self.ema_cluster_size.fill_(1.0)
            self.ema_embed_sum.copy_(w)
        return sse

    def _codebook(self):
        w = self.embedding.weight.detach()
        if w.dtype != torch.float32:
            w = w.float()
        return w if w.is_contiguous() else w.contiguous()

    def _scalars(self, sse, hist, n_local, group=None):
        """(loss, perplexity) from the VQ kernel's sufficient statistics (quantizer.py:63-64, :70-71)."""
        n_total = n_local
        if group is not None and torch.distributed.get_world_size(group) > 1:
            # batch-sharded forward (SURVEY 8e): loss and perplexity are the only
            # cross-sample quantities; reduce their sufficient statistics.
            # one tiny all-reduce of [hist (K) | sse]; shards are equal-sized (contiguous batch
            # split), so the global row count is n_local * world_size: no host sync needed
            hist, sse = reduce_vq_stats(hist, sse, group)
            n_total = n_total * torch.distributed.get_world_size(group)
        finish = ops.vq_finish if self.decay is None else ops.vq_finish_ema
        return finish(sse, hist, n_total, self.n_e, self.e_dim, self.beta)

    def _quantize_rows(self, rows, group=None):
        """rows (N, e_dim) fp32 CUDA -> (loss, zq_rows, perplexity, idx (N,))."""
        idx, zq, sse, hist = ops.vq_forward(rows, self._codebook())
        loss, perp = self._scalars(sse, hist, rows.shape[0], group)
        return loss, zq, perp, idx

    def _forward_train(self, z):
        """Differentiable path (z or the codebook requires grad): same kernels, gradients through _VQFunction; the
        NCHW <-> row layout changes are plain torch views/copies so autograd carries them."""
        if z.dim() != 4 or z.shape[1] != self.e_dim:
            raise RuntimeError(f"VectorQuantizer: expected (B,{self.e_dim},H,W), got {tuple(z.shape)}")
        ops._require_cuda(z, "VectorQuantizer input")
        B, D, H, W = z.shape
        rows = z.float().permute(0, 2, 3, 1).contiguous().view(-1, D)                   # quantizer.py:45-46
        update = self.training and self.decay is not None and z.requires_grad
        loss, zq, perp, idx = _VQFunction.apply(rows, self.embedding.weight.float(), float(self.beta), self, update)
        z_q = zq.view(B, H, W, D).permute(0, 3, 1, 2).contiguous()                      # :74
        return loss, z_q, perp, ops.onehot(idx, self.n_e), idx.view(-1, 1)

    def forward(self, z):
        if torch.is_grad_enabled() and (z.requires_grad or self.embedding.weight.requires_grad) and z.is_cuda:
            return self._forward_train(z)
        z = _prep_input(z, self.e_dim, "VectorQuantizer")   # Q11: channels must equal e_dim
        B, D, H, W = z.shape
        rows = ops.nchw_to_nhwc(z).view(-1, D)                              # quantizer.py:45-46
        loss, zq, perp, idx = self._quantize_rows(rows)
        z_q = ops.nhwc_to_nchw(zq.view(B, H, W, D))                         # :74
        min_encoding_indices = idx.view(-1, 1)                              # :54
        min_encodings = ops.onehot(idx, self.n_e)                           # :55-57 (Q7)
        return loss, z_q, perp, min_encodings, min_encoding_indices


class _PointwiseConv2d(nn.Conv2d):
    """nn.Conv2d container whose forward runs vqb_conv2d_f32 (vqvae.py:16-17,33)."""

    def forward(self, x):
        if _trains(self, x):
            return _PointwiseFunction.apply(self, x, *self.parameters())
        x = _prep_input(x, self.in_channels, "pre_quantization_conv")
        B, _, H, W = x.shape
        return _run_conv(self, x, B, H, W, in_layout=NCHW, out_layout=NCHW)[0]


def _conv_dgrad(conv, g, B, H, W, prec, *, in_layout=NHWC, out_layout=NHWC, skip=None, out=None):
    """Gradient of a conv container's input from `g`, the gradient of its (B, ., H, W) output: the adjoint conv
    (Conv2d <-> ConvTranspose2d, same weight, stride and padding) on vqb_conv2d_f32, from the ("f32", not transposed)
    packing, which is built the first time a backward needs it and refreshed by _packed like the forward's."""
    transposed = isinstance(conv, nn.ConvTranspose2d)
    kh, kw = conv.kernel_size
    w = _packed(conv.weight, ("f32", not transposed))
    return ops.conv2d(g, w, None, B=B, Cin=conv.out_channels, H=H, W=W, Cout=conv.in_channels, kh=kh, kw=kw,
                      stride=conv.stride[0], pad=conv.padding[0], transposed=not transposed, in_layout=in_layout,
                      out_layout=out_layout, skip=skip, precision=prec, out=out)


def _conv_wgrad(conv, x, g, B, H, W, grads, *, in_layout=NHWC, gout_layout=NHWC):
    """grads[id(param)] = the weight (and bias) gradient of a conv container from its (B, ., H, W) input `x` and
    its output gradient `g` (vqb_conv_wgrad_f32)."""
    kh, kw = conv.kernel_size
    dW = torch.empty(conv.weight.shape, dtype=torch.float32, device=g.device)
    db = torch.empty(conv.bias.shape, dtype=torch.float32, device=g.device) if conv.bias is not None else None
    ops.conv_wgrad(x, g, dW, db, B=B, Cin=conv.in_channels, H=H, W=W, Cout=conv.out_channels, kh=kh, kw=kw,
                   stride=conv.stride[0], pad=conv.padding[0], transposed=isinstance(conv, nn.ConvTranspose2d),
                   in_layout=in_layout, gout_layout=gout_layout)
    grads[id(conv.weight)] = dW
    if db is not None:
        grads[id(conv.bias)] = db


def _stack_backward(layers, g, r0, out, B, H, W, prec, grads, relu_out=True):
    """Gradient of a ResidualStack's input r0 = relu(x) (NHWC) from g, the gradient of its output `out`; the weight
    gradients of its `layers` (the stack's list, or [layer] for a lone ResidualLayer, whose output has no final ReLU:
    `relu_out` False) go to `grads`.  Per application r' = relu(r + W2.m), m = relu(W1 (*) r), with t = g' [r' > 0]
    and g_m = (W2^T t) [m > 0]:  dW2 += t (x) m,  dW1 += g_m (x) r,  g_r = t + W1^T (*) g_m  (Q2: every mask is taken
    from a kept post-ReLU activation).  The one-launch forward keeps r_1 .. r_{n-1} and every m on chip: they are
    recomputed here by the per-application entry points.  The applications of one layer (Q1: all of them in the
    reference's stack) take consecutive slots of the n-image-batch buffers, so each of its weights gets ONE wgrad
    call, a single fixed-order reduction over all its applications."""
    n = len(layers)
    if n == 0:
        return g
    first = {}
    for i, l in enumerate(layers):
        first.setdefault(id(l), i)
    order = sorted(range(n), key=lambda i: (first[id(layers[i])], i))
    slot = {i: s for s, i in enumerate(order)}
    groups = []                                     # (layer, first slot, end slot)
    for s, i in enumerate(order):
        if groups and groups[-1][0] is layers[i]:
            groups[-1][2] = s + 1
        else:
            groups.append([layers[i], s, s + 1])
    c1 = layers[0].res_block[1]
    C, Cmid = c1.in_channels, c1.out_channels
    f32 = dict(dtype=torch.float32, device=g.device)
    R = torch.empty((n, B, H, W, C), **f32)         # application inputs r_0 .. r_{n-1}
    M = torch.empty((n, B, H, W, Cmid), **f32)      # m_i
    T = torch.empty((n, B, H, W, C), **f32)         # t_i
    GM = torch.empty((n, B, H, W, Cmid), **f32)     # g_m of each application
    R[slot[0]].copy_(r0)
    for i in range(n - 1):
        w1, w2 = (_packed(layers[i].res_block[k].weight, ("f32", False)) for k in (1, 3))
        ops.residual_layer(R[slot[i]], w1, w2, B=B, H=H, W=W, C=C, Cmid=Cmid, relu_out=True, precision=prec,
                           out=R[slot[i + 1]])
    for l, s0, s1 in groups:
        ops.conv2d(R[s0:s1], _packed(l.res_block[1].weight, ("f32", False)), None, B=(s1 - s0) * B, Cin=C, H=H, W=W,
                   Cout=Cmid, kh=3, kw=3, stride=1, pad=1, relu=True, precision=prec, out=M[s0:s1])
    for i in reversed(range(n)):
        s, l = slot[i], layers[i]
        if i == n - 1 and not relu_out:
            T[s].copy_(g)
        else:
            ops.relu_backward(g, out if i == n - 1 else R[slot[i + 1]], out=T[s])
        ops.relu_backward(_conv_dgrad(l.res_block[3], T[s], B, H, W, prec), M[s], out=GM[s])
        g = _conv_dgrad(l.res_block[1], GM[s], B, H, W, prec, skip=T[s])
    for l, s0, s1 in groups:
        _conv_wgrad(l.res_block[3], M[s0:s1], T[s0:s1], (s1 - s0) * B, H, W, grads)
        _conv_wgrad(l.res_block[1], R[s0:s1], GM[s0:s1], (s1 - s0) * B, H, W, grads)
    return g


def _decoder_backward(dec, gx, z, acts, B, H, W, prec, grads, out_layout=NHWC, need_dz=True):
    """Gradient of a Decoder's (B, H, W) latent input z (NHWC) from gx, the fp32 NCHW gradient of its output, with the
    activations `acts` ("dec") its training walk kept; weight gradients go to `grads`.  The input gradient is
    returned in `out_layout` (None unless `need_dz`)."""
    ics = dec.inverse_conv_stack
    d1, d_out, d2 = acts
    H1, W1 = 2 * H, 2 * W
    # last layer first: convT 4 (NCHW out), ReLU, convT 2, the stack, convT 0 (its ReLU folded in)
    _conv_wgrad(ics[4], d2, gx, B, H1, W1, grads, gout_layout=NCHW)
    g = ops.relu_backward(_conv_dgrad(ics[4], gx, B, 2 * H1, 2 * W1, prec, in_layout=NCHW), d2)
    _conv_wgrad(ics[2], d_out, g, B, H, W, grads)
    g = _conv_dgrad(ics[2], g, B, H1, W1, prec)
    g = _stack_backward(list(ics[1].stack), g, d1, d_out, B, H, W, prec, grads)
    g = ops.relu_backward(g, d1, out=g)
    _conv_wgrad(ics[0], z, g, B, H, W, grads)
    return _conv_dgrad(ics[0], g, B, H, W, prec, out_layout=out_layout) if need_dz else None


def _encoder_backward(enc, g, x, acts, prec, grads, need_dx):
    """Gradient of an Encoder's image x (fp32 NCHW; None unless `need_dx`) from g, the NHWC gradient of its output,
    with the activations `acts` ("enc") its training walk kept; weight gradients go to `grads`."""
    cs = enc.conv_stack
    a1, a2, a3, e_out = acts
    B, _, H0, W0 = x.shape
    if H0 % 4 or W0 % 4:                # the adjoints of the two strided convs map back onto exactly 2x their grids
        raise RuntimeError("Encoder: the backward needs an image height and width divisible by 4 (Q11)")
    H1, W1, H2, W2 = H0 // 2, W0 // 2, H0 // 4, W0 // 4
    # the stack, then convs 4, 2, 0, each followed by a ReLU
    g = _stack_backward(list(cs[5].stack), g, a3, e_out, B, H2, W2, prec, grads)
    g = ops.relu_backward(g, a3, out=g)
    _conv_wgrad(cs[4], a2, g, B, H2, W2, grads)
    g = _conv_dgrad(cs[4], g, B, H2, W2, prec)
    g = ops.relu_backward(g, a2, out=g)
    _conv_wgrad(cs[2], a1, g, B, H1, W1, grads)
    g = _conv_dgrad(cs[2], g, B, H2, W2, prec)
    g = ops.relu_backward(g, a1, out=g)
    _conv_wgrad(cs[0], x, g, B, H0, W0, grads, in_layout=NCHW)
    return _conv_dgrad(cs[0], g, B, H1, W1, prec, out_layout=NCHW) if need_dx else None


def _param_grads(module, grads):
    """One gradient per parameter of `module`, in ``parameters()`` order and each parameter's dtype."""
    return tuple(grads[id(p)].to(p.dtype) for p in module.parameters())


class _ModuleFunction(torch.autograd.Function):
    """What the sub-module Functions share: inputs are the module, its input and its parameters; the forward keeps its
    saved activations on ctx (``ctx.acts``) and saves the input and parameters so that autograd raises, as for the
    reference, when one is modified in place before the backward; a second backward raises."""

    @staticmethod
    def _open(ctx, what):
        if ctx.acts is None:
            raise RuntimeError(f"{what}: backward through the same forward twice is not supported "
                               "(its saved activations are freed by the first backward)")
        ctx.saved_tensors                 # autograd's check that nothing saved was modified in place
        acts, ctx.acts = ctx.acts, None
        return acts


class _EncoderFunction(_ModuleFunction):
    """Encoder.forward in training mode: the inference walk keeping a1, a2, a3 and the stack output."""

    @staticmethod
    def forward(ctx, enc, x, *params):
        xp = _prep_input(x, enc.conv_stack[0].in_channels, "Encoder")
        acts = {}
        h, _, _, _ = enc._forward_nhwc(xp, False, acts)
        ctx.module, ctx.acts, ctx.prec = enc, (xp, acts["enc"]), _conv_precision()
        ctx.save_for_backward(x, *params)
        return ops.nhwc_to_nchw(h)

    @staticmethod
    def backward(ctx, g):
        xp, acts = _ModuleFunction._open(ctx, "Encoder")
        grads = {}
        dx = _encoder_backward(ctx.module, ops.nchw_to_nhwc(g), xp, acts, ctx.prec, grads, ctx.needs_input_grad[1])
        return (None, dx) + _param_grads(ctx.module, grads)


class _DecoderFunction(_ModuleFunction):
    """Decoder.forward in training mode: the inference walk keeping its NHWC input, d1, d_out and d2."""

    @staticmethod
    def forward(ctx, dec, x, *params):
        xp = _prep_input(x, dec.inverse_conv_stack[0].in_channels, "Decoder")
        B, _, H, W = xp.shape
        z = ops.nchw_to_nhwc(xp)
        acts = {}
        y = dec._forward_from_nhwc(z, B, H, W, acts=acts)
        ctx.module, ctx.acts, ctx.prec = dec, (z, acts["dec"]), _conv_precision()
        ctx.save_for_backward(x, *params)
        return y

    @staticmethod
    def backward(ctx, g):
        z, acts = _ModuleFunction._open(ctx, "Decoder")
        B, H, W, _ = z.shape
        grads = {}
        dz = _decoder_backward(ctx.module, ops._f32c(g), z, acts, B, H, W, ctx.prec, grads, out_layout=NCHW,
                               need_dz=ctx.needs_input_grad[1])
        return (None, dz) + _param_grads(ctx.module, grads)


class _PointwiseFunction(_ModuleFunction):
    """The pre-quantization conv in training mode: one dgrad and one wgrad, NCHW on both sides."""

    @staticmethod
    def forward(ctx, conv, x, *params):
        xp = _prep_input(x, conv.in_channels, "pre_quantization_conv")
        B, _, H, W = xp.shape
        ctx.module, ctx.acts, ctx.prec = conv, xp, _conv_precision()
        ctx.save_for_backward(x, *params)
        return _run_conv(conv, xp, B, H, W, in_layout=NCHW, out_layout=NCHW)[0]

    @staticmethod
    def backward(ctx, g):
        xp = _ModuleFunction._open(ctx, "pre_quantization_conv")
        B, _, H, W = xp.shape
        g = ops._f32c(g)
        grads = {}
        _conv_wgrad(ctx.module, xp, g, B, H, W, grads, in_layout=NCHW, gout_layout=NCHW)
        dx = _conv_dgrad(ctx.module, g, B, H, W, ctx.prec, in_layout=NCHW, out_layout=NCHW) \
            if ctx.needs_input_grad[1] else None
        return (None, dx) + _param_grads(ctx.module, grads)


class _ReluInPlace(torch.autograd.Function):
    """Q2 under autograd: nn.ReLU(True) rewrites the caller's tensor and is recorded on it (mark_dirty bumps its
    version and routes its gradient through the mask, as torch's relu_ does)."""

    @staticmethod
    def forward(ctx, x):
        if x.is_contiguous() and x.dtype == torch.float32:
            ops.relu_(x)
        else:
            x.copy_(ops.relu_(ops._f32c(x.detach()).clone()))
        ctx.mark_dirty(x)
        ctx.save_for_backward(x)
        return x

    @staticmethod
    def backward(ctx, g):
        y, = ctx.saved_tensors
        return ops.relu_backward(ops._f32c(g), ops._f32c(y))


class _ReluFunction(torch.autograd.Function):
    """An empty ResidualStack in training mode: its final F.relu, on a copy (vqb_relu_f32 / vqb_relu_backward_f32)."""

    @staticmethod
    def forward(ctx, x):
        y = ops.relu_(ops._f32c(x.detach()).clone())
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, g):
        y, = ctx.saved_tensors
        return ops.relu_backward(ops._f32c(g), y)


class _StackFunction(_ModuleFunction):
    """A ResidualStack (or a lone ResidualLayer) in training mode on r = relu(x), already taken in place: the inference
    launches keeping r (NHWC) and the output; the backward is _stack_backward."""

    @staticmethod
    def forward(ctx, module, layers, relu_out, r, *params):
        B, _, H, W = r.shape
        rn = ops.nchw_to_nhwc(r)
        out = module._apply_nhwc(rn, B, H, W) if relu_out else module._apply_nhwc(rn, B, H, W, relu_out=False)
        ctx.module, ctx.layers, ctx.relu_out, ctx.acts, ctx.prec = module, layers, relu_out, (rn, out), _conv_precision()
        ctx.save_for_backward(r, *params)
        return ops.nhwc_to_nchw(out)

    @staticmethod
    def backward(ctx, g):
        rn, out = _ModuleFunction._open(ctx, type(ctx.module).__name__)
        B, H, W, _ = rn.shape
        grads = {}
        dr = _stack_backward(ctx.layers, ops.nchw_to_nhwc(g), rn, out, B, H, W, ctx.prec, grads, ctx.relu_out)
        return (None, None, None, ops.nhwc_to_nchw(dr) if ctx.needs_input_grad[3] else None) + \
            _param_grads(ctx.module, grads)


def _residual_train(module, layers, x, channels, what):
    """The differentiable call of a ResidualStack (layers = its list) or a ResidualLayer (layers = [itself]): the
    in-place ReLU on the caller's x (Q2), then _StackFunction; an empty stack is its final ReLU only."""
    _check_input(x, channels, what)
    if not layers:
        return _ReluFunction.apply(x)
    if x.is_leaf and x.requires_grad:       # torch's own check, before the caller's tensor is touched
        raise RuntimeError("a leaf Variable that requires grad is being used in an in-place operation.")
    r = _ReluInPlace.apply(x)
    return _StackFunction.apply(module, layers, isinstance(module, ResidualStack), r, *module.parameters())


class _VQVAEFunction(torch.autograd.Function):
    """VQVAE.forward in training mode: inputs are the model, the image and every parameter in ``parameters()`` order
    (a shared ResidualLayer once).  The forward is the inference walk (fp32 activations; the bf16 mode runs the TF32
    kernels) keeping the activations it already produces; the backward runs every input gradient on the forward conv
    kernels (vqb_conv2d_f32 with the transposed flag flipped), every conv weight gradient on vqb_conv_wgrad_f32 and
    the VQ step on vqb_vq_backward_f32, and returns one gradient per parameter."""

    @staticmethod
    def forward(ctx, model, x, *params):
        acts = {}
        embedding_loss, x_hat, perplexity = model._walk(x, False, acts)
        ctx.model, ctx.acts, ctx.prec = model, acts, _conv_precision()
        # saved so that autograd raises, as it does for the reference, when the image or a parameter is modified in
        # place between this forward and its backward (the backward reads the weights as they are then).  An EMA
        # codebook is not: the forward's own update rewrites it, and the backward does not read it.
        vq = model.vector_quantization
        if vq.decay is not None:
            params = [p for p in params if p is not vq.embedding.weight]
        ctx.save_for_backward(x, *params)
        ctx.mark_non_differentiable(perplexity)
        return embedding_loss, x_hat, perplexity

    @staticmethod
    def backward(ctx, g_loss, g_xhat, _g_perp):
        if ctx.acts is None:            # the first backward freed the saved activations
            raise RuntimeError("VQVAE: backward through the same forward twice is not supported "
                               "(its saved activations are freed by the first backward)")
        ctx.saved_tensors                 # autograd's check that nothing saved was modified in place
        model, a, prec = ctx.model, ctx.acts, ctx.prec
        ctx.acts = None
        vq = model.vector_quantization
        x = a["x"]
        B, _, H0, W0 = x.shape
        H2, W2 = H0 // 4, W0 // 4
        grads = {}
        g = _decoder_backward(model.decoder, ops._f32c(g_xhat), a["zq"], a["dec"], B, H2, W2, prec, grads)
        if vq.decay is None:
            # the VQ step: straight-through to z_e plus the loss terms; the codebook gradient (float atomics)
            dz, dE = ops.vq_backward(g.view(-1, vq.e_dim), g_loss, a["z_e"], a["codebook"], a["idx"], float(vq.beta))
        else:
            # EMA codebook: the commitment term only, from the forward's z_q rows; no codebook gradient
            dz, dE = ops.vq_commit_backward(g.view(-1, vq.e_dim), g_loss, a["z_e"], a["zq"], float(vq.beta)), None
        grads[id(vq.embedding.weight)] = dE
        pq = model.pre_quantization_conv
        _conv_wgrad(pq, a["enc"][3], dz, B, H2, W2, grads)
        g = _conv_dgrad(pq, dz, B, H2, W2, prec)
        dx = _encoder_backward(model.encoder, g, x, a["enc"], prec, grads, ctx.needs_input_grad[1])
        params = list(model.parameters())
        return (None, dx) + tuple(None if grads[id(p)] is None else grads[id(p)].to(p.dtype) for p in params)


class VQVAE(nn.Module):
    """models/vqvae.py:10-44."""

    def __init__(self, h_dim, res_h_dim, n_res_layers, n_embeddings, embedding_dim, beta,
                 save_img_embedding_map=False, *, ema_decay=None, ema_eps=1e-5):
        """``ema_decay`` / ``ema_eps``: the quantizer's ``decay`` / ``eps`` (VectorQuantizer): None keeps the reference's
        gradient-trained codebook."""
        _check_ema(ema_decay, ema_eps)
        super().__init__()
        self.encoder = Encoder(3, h_dim, n_res_layers, res_h_dim)
        self.pre_quantization_conv = _PointwiseConv2d(h_dim, embedding_dim, kernel_size=1, stride=1)
        self.vector_quantization = VectorQuantizer(n_embeddings, embedding_dim, beta, decay=ema_decay, eps=ema_eps)
        self.decoder = Decoder(embedding_dim, h_dim, n_res_layers, res_h_dim)
        if save_img_embedding_map:
            self.img_to_embedding_map = {i: [] for i in range(n_embeddings)}
        else:
            self.img_to_embedding_map = None
        # batch-sharded inference: set to a torch.distributed process group so that
        # embedding_loss / perplexity equal the single-process values (SURVEY 8e)
        self.process_group = None
        # True: every sharded forward all-reduces the VQ statistics (one 4 KB collective per step: every step is a
        # rank rendezvous).  False: forward returns THIS SHARD's loss / perplexity and keeps the statistics;
        # reduce_scalars() all-reduces them on demand (e.g. every M steps, or when a caller reads the scalars).
        self.sync_scalars = True
        self.last_vq_stats = None            # (hist int32 (K,), sse f64 (1,), rows of this shard) of the last forward
        self._side_stream = None
        self.last_min_encoding_indices = None
        self._bf16_covered = None            # _bf16_pipeline's answer for this architecture, once asked

    def _bf16_pipeline(self):
        """True when set_precision("bf16") is active AND every layer of this model has a bf16 kernel
        (h_dim = 128 family: 64-channel first layer, channel counts in multiples of 64, embedding_dim = 64).
        Other shapes run the TF32 kernels on fp32 activations, with a one-time warning.  The constructor fixes the
        architecture, so the answer is worked out on first use and kept."""
        if get_precision() != "bf16":
            return False
        if self._bf16_covered is None:
            self._bf16_covered = self._bf16_coverage()
            if not self._bf16_covered:
                import warnings
                warnings.warn("vqvae_b200: this model shape has no bf16 kernels; precision 'bf16' runs the TF32 kernels")
        return self._bf16_covered

    def _bf16_coverage(self):
        """Whether the library has a bf16 kernel for every layer.  vqb_conv_bf16_packed_bytes answers for each conv that
        takes a bf16 packing; the entry points with no such query take the shapes include/vqvae_b200.h documents."""
        conv_in = self.encoder.conv_stack[0]
        if (conv_in.in_channels, conv_in.out_channels) != (3, 64):                      # vqb_conv_in_bf16
            return False
        for st in (m for m in self.modules() if isinstance(m, ResidualStack) and len(m.stack)):
            layer = st.stack[0]                                                         # vqb_residual_layer_bf16
            if any(l is not layer for l in st.stack) or layer.res_block[1].in_channels not in (64, 128):
                return False
        if self.vector_quantization.e_dim != 64:                                        # vqb_vq_forward_bf16zq_f32
            return False
        keys = [(c, _pack_key(c, True)) for c in _convs(self)]
        return all(ops.lib().vqb_conv_bf16_packed_bytes(key[1], c.out_channels, c.in_channels) != 0
                   for c, key in keys if key[0] == "bf16")

    def _encode_rows(self, x, bf16=False, acts=None, fuse=False):
        x = _prep_input(x, 3, "VQVAE")
        if x.shape[2] % 4 or x.shape[3] % 4:
            raise RuntimeError("VQVAE: image height and width must be divisible by 4 (Q11)")
        if acts is not None:
            acts["x"] = x
        # NHWC (B,H,W,D) rows, fp32 in every mode: they feed the exact VQ
        return self.encoder._forward_nhwc(x, bf16, acts, self.pre_quantization_conv, fuse)

    def _trains(self, x):
        """Whether forward(x) takes the differentiable path (see forward)."""
        return _trains(self, x)

    def forward(self, x, verbose=False):
        """vqvae.py:29-44 -> (embedding_loss, x_hat, perplexity).  In training mode with grad enabled and a parameter
        (or x) requiring grad, the outputs are differentiable (_VQVAEFunction): the same launches, so the same values,
        as the eval-mode forward, which records no autograd graph."""
        if self._trains(x):
            if self.process_group is not None:
                raise RuntimeError("VQVAE: training with process_group set is not supported (the loss gradient of a "
                                   "batch-sharded forward would need an all-reduce)")
            embedding_loss, x_hat, perplexity = _VQVAEFunction.apply(self, x, *self.parameters())
        else:
            embedding_loss, x_hat, perplexity = self._walk(x, self._bf16_pipeline())
        if verbose:                                                          # :38-42 (Q8)
            B, _, H, W = x.shape
            print('original data shape:', x.shape)
            print('encoded data shape:', torch.Size((B, self.vector_quantization.e_dim, H // 4, W // 4)))
            print('recon data shape:', x_hat.shape)
            assert False
        return embedding_loss, x_hat, perplexity

    def _walk(self, x, bf16, acts=None):
        """The forward's launches -> (embedding_loss, x_hat, perplexity).  `acts` (a dict) receives the tensors the
        training backward reads."""
        # Inference in TF32: each side's k3 conv, its ResidualStack and (encoder) the pre-quantization conv run as one
        # launch where _latent_block takes the shape, bitwise the separate launches.  The training walk keeps those,
        # since its backward reads the activations between them.  The decoder's last two layers run as one launch in
        # both walks: it can also store the hidden activation the backward reads.
        tf32 = not bf16 and _conv_precision() == PRECISIONS["tf32"]
        fuse = acts is None and tf32
        z_e, B, H, W = self._encode_rows(x, bf16, acts, fuse)                # vqvae.py:31-33
        vq = self.vector_quantization
        D = vq.e_dim
        group = self.process_group
        # The decoder does not depend on the loss / perplexity scalars (vqvae.py:36 vs quantizer.py:63-71), so
        # the batch-sharded all-reduce of (sse, hist) (SURVEY 8e) and the scalar finisher run on a side stream
        # and overlap the decoder; fork/join with events, so the whole forward stays capturable in one CUDA graph.
        n_rows = z_e.shape[0] * H * W
        codebook = vq._codebook()
        idx, zq, sse, hist = ops.vq_forward(z_e.view(-1, D), codebook,
                                            zq_dtype=torch.bfloat16 if bf16 else torch.float32)
        main = torch.cuda.current_stream()
        if self._side_stream is None or self._side_stream.device != z_e.device:
            self._side_stream = torch.cuda.Stream(device=z_e.device)
        side = self._side_stream
        side.wait_stream(main)
        # A training call of an EMA model updates the codebook there too: the decoder reads z_q, not the codebook.
        ema = acts is not None and vq.decay is not None
        with torch.cuda.stream(side):
            embedding_loss, perplexity = vq._scalars(sse, hist, n_rows, group if self.sync_scalars else None)
            self.last_vq_stats = (hist, sse, n_rows)
            if ema:
                vq._ema_update(z_e.view(-1, D), idx, hist)
            if not torch.cuda.is_current_stream_capturing():
                for t in (sse, hist, embedding_loss, perplexity) + ((z_e, idx) if ema else ()):
                    t.record_stream(side)
        x_hat = self.decoder._forward_from_nhwc(zq.view(B, H, W, D), B, H, W, bf16, acts, fuse, tf32)  # :36
        main.wait_stream(side)
        if not torch.cuda.is_current_stream_capturing():
            # the two scalars were allocated in the side stream's pool and are consumed on the caller's stream: without this
            # their block could be handed out again on the side stream while the caller still reads them (ADVICE r1)
            embedding_loss.record_stream(main)
            perplexity.record_stream(main)
        self.last_min_encoding_indices = idx.view(-1, 1)
        if acts is not None:
            acts.update(z_e=z_e.view(-1, D), codebook=codebook, idx=idx, zq=zq)
        return embedding_loss, x_hat, perplexity

    def init_codebook_kmeans(self, x, iters=10):
        """VectorQuantizer.init_codebook_kmeans on the z_e rows of the images x, from the encoder walk that forward
        quantizes (in the active precision, the bf16 pipeline included).  Call it on the first batch before training;
        an optimizer built earlier keeps its moments of the codebook.  Returns the (iters,) float64 device SSE."""
        vq = self.vector_quantization
        vq._check_kmeans(iters)
        _check_input(x, 3, "VQVAE")
        vq._check_kmeans_rows(x.shape[0] * (x.shape[2] // 4) * (x.shape[3] // 4))
        with torch.no_grad():
            z_e, _, _, _ = self._encode_rows(x, self._bf16_pipeline())
            return vq._kmeans_rows(z_e.view(-1, vq.e_dim), iters)

    def reduce_scalars(self):
        """(embedding_loss, perplexity) over the WHOLE sharded batch from the statistics of the last forward: the one
        collective of the path (SURVEY 8e), issued on demand when ``sync_scalars`` is False.  Equals the
        single-process values on the concatenated batch (tests/test_dist_cpu.py, tests/test_gpu_dist.py)."""
        if self.last_vq_stats is None:
            raise RuntimeError("reduce_scalars: no forward has run yet")
        hist, sse, n_rows = self.last_vq_stats
        return self.vector_quantization._scalars(sse, hist, n_rows, self.process_group)

    def repack(self):
        """Refresh every cached weight packing whose parameter changed (load_state_dict, optimizer step), IN PLACE
        in the buffers earlier forwards -- and CUDA graphs captured around them -- already read: the forward's, and
        the input-gradient packing of a training backward once one exists.  A plain forward (backward) does this by
        itself; HostPipeline calls it before replaying a captured graph."""
        bf16 = self._bf16_pipeline()
        for conv in _convs(self):
            fwd = _pack_key(conv, bf16)
            _packed(conv.weight, fwd)
            for key in [k for k in getattr(conv.weight, "_vqb_packed", {}) if k[0] == "f32" and k != fwd]:
                _packed(conv.weight, key)           # a training backward's input-gradient packing, once it exists

    # ---- SURVEY 8(f) rank 1: the two halves callers use around the path ----------
    def encode(self, x):
        """images -> min_encoding_indices (N,1) int64 (README step 2 / notebook cell 1)."""
        z_e, B, H, W = self._encode_rows(x, self._bf16_pipeline())
        _, _, _, idx = self.vector_quantization._quantize_rows(z_e.view(-1, self.vector_quantization.e_dim))
        return idx.view(-1, 1)

    def decode(self, indices, latent_hw):
        """min_encoding_indices -> images (notebook cell 13 ``generate_samples``): the
        one-hot matmul replaced by a codebook row gather."""
        H, W = latent_hw
        vq = self.vector_quantization
        rows = ops.gather_rows(indices, vq._codebook())
        B = rows.shape[0] // (H * W)
        bf16 = self._bf16_pipeline()
        if bf16:
            rows = rows.to(torch.bfloat16)
        return self.decoder._forward_from_nhwc(rows.view(B, H, W, vq.e_dim), B, H, W, bf16)

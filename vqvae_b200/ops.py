"""Torch-tensor front end of the C ABI: allocation and stream plumbing only.

PyTorch owns every buffer and the current stream; all arithmetic happens inside
libvqvae_b200.so.  There is NO CPU path: a non-CUDA tensor raises.
"""
import torch

from . import _lib
from ._lib import BF16, FP32, NCHW, NHWC, TF32, check, lib  # noqa: F401


def _require_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError(
            f"vqvae_b200: {what} must be a CUDA tensor -- this implementation is sm_90a (H100) only "
            "and has no CPU fallback")
    if t.device.index != torch.cuda.current_device():
        # the C ABI launches on the CURRENT device's stream (header: "the caller selects the device"); a tensor that lives
        # elsewhere would be read through a peer mapping at best and fault at worst (ADVICE r1)
        raise RuntimeError(
            f"vqvae_b200: {what} is on {t.device} but the current CUDA device is cuda:{torch.cuda.current_device()}; "
            "wrap the call in `with torch.cuda.device(tensor.device):`")


def _stream():
    return torch.cuda.current_stream().cuda_stream


# Optional per-call CUDA-event timing (bench.py's kernel breakdown): when PROFILE is a
# list, every C-ABI compute call appends (label, start_event, end_event).
PROFILE = None


class _Span:
    __slots__ = ("label", "start", "end")

    def __init__(self, label):
        self.label = label
        self.start = self.end = None
        if PROFILE is not None:
            self.start = torch.cuda.Event(enable_timing=True)
            self.end = torch.cuda.Event(enable_timing=True)
            self.start.record()

    def done(self):
        if self.start is not None:
            self.end.record()
            PROFILE.append((self.label, self.start, self.end))


def launch_count() -> int:
    """Kernels launched so far through the C ABI by this process."""
    return int(lib().vqb_launch_count())


def _f32c(t):
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


def pack_conv_weight(w, transposed, out=None):
    """(Cout,Cin,kh,kw) conv / (Cin,Cout,kh,kw) conv-transpose weight -> the fp32 packing of
    vqb_pack_conv_weight_f32: K-major rows [(r*kw+s)][co][ci], which every conv kernel reads, then
    room for the [9][16][Cin] pixel-shuffle form that a k4 s2 transposed conv to <= 4 channels adds."""
    _require_cuda(w, "weight")
    w = _f32c(w.detach())
    if transposed:
        cin, cout, kh, kw = w.shape
    else:
        cout, cin, kh, kw = w.shape
    n = kh * kw * cin * cout + 9 * 16 * cin
    if out is None or out.numel() != n or out.dtype != torch.float32 or out.device != w.device:
        out = torch.empty((n,), dtype=torch.float32, device=w.device)      # else: repacked in place
    check(lib().vqb_pack_conv_weight_f32(w.data_ptr(), out.data_ptr(), cout, cin, kh, kw,
                                         int(bool(transposed)), _stream()), "pack_conv_weight")
    return out


def conv_out_hw(h, w, kh, kw, stride, pad, transposed):
    if transposed:
        return (h - 1) * stride - 2 * pad + kh, (w - 1) * stride - 2 * pad + kw
    return (h + 2 * pad - kh) // stride + 1, (w + 2 * pad - kw) // stride + 1


def conv2d(x, w_packed, bias, *, B, Cin, H, W, Cout, kh, kw, stride, pad, transposed=False,
           in_layout=NHWC, out_layout=NHWC, relu=False, skip=None, precision=FP32, out=None):
    """One nn.Conv2d / nn.ConvTranspose2d forward (+bias, +skip, +ReLU) on raw buffers.
    `x` is any contiguous CUDA fp32 tensor holding the (B,Cin,H,W) activation in
    `in_layout`; returns a new tensor in `out_layout` ((B,Cout,OH,OW) or (B,OH,OW,Cout)), or writes `out`
    (a contiguous fp32 tensor of that many elements) when given."""
    _require_cuda(x, "input")
    oh, ow = conv_out_hw(H, W, kh, kw, stride, pad, transposed)
    if oh <= 0 or ow <= 0:
        raise RuntimeError(f"conv output size is non-positive ({oh}x{ow})")
    shape = (B, Cout, oh, ow) if out_layout == NCHW else (B, oh, ow, Cout)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=x.device)
    span = _Span(f"conv{'T' if transposed else ''} {Cin}->{Cout} k{kh}s{stride} {H}x{W}"
                 f"{' +skip' if skip is not None else ''}")
    check(lib().vqb_conv2d_f32(
        x.data_ptr(), w_packed.data_ptr(), bias.data_ptr() if bias is not None else None,
        skip.data_ptr() if skip is not None else None, out.data_ptr(),
        B, Cin, H, W, Cout, kh, kw, stride, pad, int(bool(transposed)), in_layout, out_layout,
        int(bool(relu)), precision, _stream()), "conv2d")
    span.done()
    return out


# enum vqb_conv_kind -> (kernel size, stride, transposed) of the layer it names
KIND_GEOMETRY = {_lib.CONV_K1: (1, 1, False), _lib.CONV_K3: (3, 1, False), _lib.CONVT_K3: (3, 1, True),
                 _lib.CONV_K4S2: (4, 2, False), _lib.CONVT_K4S2: (4, 2, True), _lib.CONVT_K4S2_OUT: (4, 2, True),
                 _lib.RES_W2: (1, 1, False)}


def conv_kind(kh, stride, transposed, cout):
    """enum vqb_conv_kind of a layer of the hot path, or None when the bf16 kernels do not cover it.  (RES_W2, the
    residual layer's 1x1 weight, is never a layer of its own.)"""
    if cout <= 4 and KIND_GEOMETRY[_lib.CONVT_K4S2_OUT] == (kh, stride, bool(transposed)):
        return _lib.CONVT_K4S2_OUT
    for kind in (_lib.CONV_K1, _lib.CONV_K3, _lib.CONVT_K3, _lib.CONV_K4S2, _lib.CONVT_K4S2):
        if KIND_GEOMETRY[kind] == (kh, stride, bool(transposed)):
            return kind
    return None


def pack_conv_weight_bf16(w, kind, out=None):
    """fp32 conv / conv-transpose weight -> the bf16 K-major tap-major packing of vqb_pack_conv_weight_bf16
    (None when the shape is not covered).  `out`: repack into an existing buffer (same shape) in place."""
    _require_cuda(w, "weight")
    w = _f32c(w.detach())
    transposed = KIND_GEOMETRY[kind][2]
    cin, cout = (w.shape[0], w.shape[1]) if transposed else (w.shape[1], w.shape[0])
    nbytes = lib().vqb_conv_bf16_packed_bytes(kind, cout, cin)
    if nbytes == 0:
        return None
    if out is None or out.numel() != nbytes or out.dtype != torch.uint8 or out.device != w.device:
        # (torch's caching allocator hands out 512-byte aligned blocks: the 128-byte alignment the TMA maps need)
        out = torch.empty((nbytes,), dtype=torch.uint8, device=w.device)
    check(lib().vqb_pack_conv_weight_bf16(w.data_ptr(), out.data_ptr(), kind, cout, cin, _stream()), "pack_conv_weight_bf16")
    return out


def conv2d_bf16(x, packed, bias, *, B, Cin, H, W, Cout, kind, relu=False, out_f32=False):
    """One layer on bf16 NHWC input through vqb_conv2d_bf16; returns bf16 NHWC, fp32 NHWC (out_f32) or, for
    CONVT_K4S2_OUT, the fp32 NCHW module output."""
    _require_cuda(x, "input")
    if x.dtype != torch.bfloat16 or not x.is_contiguous():
        raise RuntimeError("conv2d_bf16: input must be a contiguous bf16 NHWC tensor")
    k, stride, transposed = KIND_GEOMETRY[kind]
    oh, ow = (H * stride, W * stride) if transposed else (H // stride, W // stride)
    if kind == _lib.CONVT_K4S2_OUT:
        shape, dt = (B, Cout, oh, ow), torch.float32
    else:
        shape, dt = (B, oh, ow, Cout), (torch.float32 if out_f32 else torch.bfloat16)
    out = torch.empty(shape, dtype=dt, device=x.device)
    span = _Span(f"bf16 conv{'T' if transposed else ''} {Cin}->{Cout} k{k}s{stride} {H}x{W}")
    check(lib().vqb_conv2d_bf16(x.data_ptr(), packed.data_ptr(), bias.data_ptr() if bias is not None else None,
                                out.data_ptr(), B, Cin, H, W, Cout, kind, int(bool(relu)), int(bool(out_f32)),
                                _stream()), "conv2d_bf16")
    span.done()
    return out


def conv_in_bf16(x, w_packed_f32, bias, *, B, H, W, Cout, relu=True):
    """encoder.py:29-31 for the bf16 pipeline: fp32 NCHW image -> bf16 NHWC (B, H/2, W/2, Cout) (vqb_conv_in_bf16)."""
    _require_cuda(x, "input")
    out = torch.empty((B, H // 2, W // 2, Cout), dtype=torch.bfloat16, device=x.device)
    span = _Span(f"bf16 conv 3->{Cout} k4s2 {H}x{W}")
    check(lib().vqb_conv_in_bf16(x.data_ptr(), w_packed_f32.data_ptr(), bias.data_ptr() if bias is not None else None,
                                 out.data_ptr(), B, H, W, Cout, int(bool(relu)), _stream()), "conv_in_bf16")
    span.done()
    return out


def residual_layer_bf16(r, w1_packed, w2_packed, *, B, H, W, C, Cmid, relu_out):
    """out = act(r + W2.relu(W1 (*) r)) on bf16 NHWC buffers, one wgmma launch (vqb_residual_layer_bf16)."""
    _require_cuda(r, "input")
    if r.dtype != torch.bfloat16 or not r.is_contiguous():
        raise RuntimeError("residual_layer_bf16: input must be a contiguous bf16 NHWC tensor")
    out = torch.empty((B, H, W, C), dtype=torch.bfloat16, device=r.device)
    span = _Span(f"bf16 res {C}->{Cmid}->{C} {H}x{W}")
    check(lib().vqb_residual_layer_bf16(r.data_ptr(), w1_packed.data_ptr(), w2_packed.data_ptr(), out.data_ptr(),
                                        B, H, W, C, Cmid, int(bool(relu_out)), _stream()), "residual_layer_bf16")
    span.done()
    return out


def residual_layer(r, w1_packed, w2_packed, *, B, H, W, C, Cmid, relu_out, precision=FP32, out=None):
    """out = act(r + W2.relu(W1 (*) r)) on NHWC buffers (vqb_residual_layer_f32), into `out` when given."""
    _require_cuda(r, "input")
    if out is None:
        out = torch.empty((B, H, W, C), dtype=torch.float32, device=r.device)
    tmp = torch.empty((B, H, W, Cmid), dtype=torch.float32, device=r.device)
    span = _Span(f"res {C}->{Cmid}->{C} {H}x{W}")
    check(lib().vqb_residual_layer_f32(r.data_ptr(), w1_packed.data_ptr(), w2_packed.data_ptr(), out.data_ptr(),
                                       tmp.data_ptr(), B, H, W, C, Cmid, int(bool(relu_out)), precision,
                                       _stream()), "residual_layer")
    span.done()
    return out


def residual_stack(r, w1_packed, w2_packed, *, B, H, W, C, Cmid, n_layers, precision=FP32):
    """n_layers applications of one shared-weight layer, each followed by ReLU, on NHWC buffers
    (vqb_residual_stack_f32; one kernel in tensor-core mode when a tile holds whole images)."""
    _require_cuda(r, "input")
    if n_layers < 1:
        return r
    out = torch.empty((B, H, W, C), dtype=torch.float32, device=r.device)
    scratch = torch.empty((B, H, W, C), dtype=torch.float32, device=r.device) if n_layers > 1 else out
    tmp = torch.empty((B, H, W, Cmid), dtype=torch.float32, device=r.device)
    span = _Span(f"res x{n_layers} {C}->{Cmid}->{C} {H}x{W}")
    check(lib().vqb_residual_stack_f32(r.data_ptr(), w1_packed.data_ptr(), w2_packed.data_ptr(), out.data_ptr(),
                                       scratch.data_ptr(), tmp.data_ptr(), B, H, W, C, Cmid, n_layers, precision,
                                       _stream()), "residual_stack")
    span.done()
    return out


def latent_block(x, head_w, head_bias, w1_packed, w2_packed, tail_w=None, tail_bias=None, *, B, Cin, H, W, C, Cmid,
                 n_layers, transposed, tail_cout=0):
    """relu(k3 s1 conv or transposed conv of NHWC x + head_bias), the ResidualStack of residual_stack and, given
    tail_w, the 1x1 conv to tail_cout channels + tail_bias, as ONE TF32 launch (vqb_latent_block_tf32), bitwise the
    separate calls.  Returns the NHWC stack output, or the tail's (B, H, W, tail_cout) rows; None (nothing allocated or
    launched) for a shape the launch does not take."""
    _require_cuda(x, "input")
    if (tail_w is None) != (tail_cout == 0):
        raise ValueError("latent_block: tail_w and tail_cout > 0 go together")
    if not lib().vqb_latent_block_supported(Cin, H, W, C, Cmid, tail_cout):
        return None
    out = torch.empty((B, H, W, tail_cout or C), dtype=torch.float32, device=x.device)
    conv = f"+conv{'T' if transposed else ''} {Cin}->{C} k3s1"
    tail = "" if tail_w is None else f" +conv {C}->{tail_cout} k1s1"
    span = _Span(f"res x{n_layers} {C}->{Cmid}->{C} {H}x{W} {conv}{tail}")
    rc = lib().vqb_latent_block_tf32(x.data_ptr(), head_w.data_ptr(), head_bias.data_ptr() if head_bias is not None else None,
                                     int(bool(transposed)), w1_packed.data_ptr(), w2_packed.data_ptr(), n_layers,
                                     tail_w.data_ptr() if tail_w is not None else None,
                                     tail_bias.data_ptr() if tail_bias is not None else None, tail_cout, out.data_ptr(),
                                     B, Cin, H, W, C, Cmid, _stream())
    if rc == _lib.ERR_UNSUPPORTED:      # a supported shape declined only for aliasing or alignment
        return None
    check(rc, "latent_block")
    span.done()
    return out


def decoder_tail(d_out, convt_w, convt_bias, out_w, out_bias, *, B, Cin, H, W, C, Cout, relu_out=False, keep_h=False):
    """relu(k4 s2 transposed conv of NHWC d_out + convt_bias) -> h, then the k4 s2 transposed conv of h to Cout channels +
    out_bias (ReLU'd if relu_out), as ONE TF32 launch (vqb_decoder_tail_tf32), bitwise the separate calls.  Returns
    (x_hat NCHW (B, Cout, 4H, 4W), h NHWC (B, 2H, 2W, C) if keep_h else None); None (nothing allocated or launched) for a
    shape the launch does not take."""
    _require_cuda(d_out, "input")
    if not lib().vqb_decoder_tail_supported(Cin, H, W, C, Cout):
        return None
    x_hat = torch.empty((B, Cout, 4 * H, 4 * W), dtype=torch.float32, device=d_out.device)
    h = torch.empty((B, 2 * H, 2 * W, C), dtype=torch.float32, device=d_out.device) if keep_h else None
    span = _Span(f"convT {Cin}->{C} k4s2 {H}x{W} +convT {C}->{Cout} k4s2")
    rc = lib().vqb_decoder_tail_tf32(d_out.data_ptr(), convt_w.data_ptr(),
                                     convt_bias.data_ptr() if convt_bias is not None else None, out_w.data_ptr(),
                                     out_bias.data_ptr() if out_bias is not None else None,
                                     h.data_ptr() if h is not None else None, x_hat.data_ptr(), B, Cin, H, W, C, Cout,
                                     int(bool(relu_out)), _stream())
    if rc == _lib.ERR_UNSUPPORTED:      # a supported shape declined only for aliasing or alignment
        return None
    check(rc, "decoder_tail")
    span.done()
    return x_hat, h


def vq_forward(z_rows, codebook, zq_dtype=torch.float32):
    """Fused VectorQuantizer core on (N,D) fp32 rows -> (idx int64 (N,), zq (N,D), sse f64 (1,),
    hist int32 (K,)); `sse` is final when the call returns.  zq_dtype=torch.bfloat16
    (vqb_vq_forward_bf16zq_f32, D == 64) writes z_q as bf16 rows for the bf16 pipeline."""
    _require_cuda(z_rows, "z")
    bf16zq = zq_dtype == torch.bfloat16
    if zq_dtype not in (torch.float32, torch.bfloat16):
        raise ValueError("vq_forward: z_q is fp32 or bf16 rows")
    N, D = z_rows.shape
    K = codebook.shape[0]
    dev = z_rows.device
    idx = torch.empty((N,), dtype=torch.int64, device=dev)
    zq = torch.empty((N, D), dtype=zq_dtype, device=dev)
    sse = torch.empty((1,), dtype=torch.float64, device=dev)
    hist = torch.empty((K,), dtype=torch.int32, device=dev)
    ws_bytes = lib().vqb_vq_workspace_bytes(N, K, D)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    span = _Span(f"vq N={N} K={K} D={D}{' (bf16 zq)' if bf16zq else ''}")
    fn = lib().vqb_vq_forward_bf16zq_f32 if bf16zq else lib().vqb_vq_forward_f32
    check(fn(z_rows.data_ptr(), codebook.data_ptr(), N, K, D, idx.data_ptr(), zq.data_ptr(), sse.data_ptr(),
             hist.data_ptr(), ws.data_ptr(), ws_bytes, _stream()), "vq_forward")
    span.done()
    return idx, zq, sse, hist


def vq_finish(sse, hist, N, K, D, beta):
    """(loss, perplexity) fp32 0-dim CUDA tensors from the (all-reduced) sse / hist."""
    out = torch.empty((2,), dtype=torch.float32, device=hist.device)
    check(lib().vqb_vq_finish_f32(sse.data_ptr(), hist.data_ptr(), N, K, D, float(beta),
                                  out.data_ptr(), out.data_ptr() + 4, _stream()), "vq_finish")
    return out[0], out[1]


def vq_backward(g_zq, g_loss, z_rows, codebook, idx, beta):
    """(dz (N,D), dE (K,D)) of the VectorQuantizer forward (vqb_vq_backward_f32); g_zq / g_loss may be None."""
    _require_cuda(z_rows, "z")
    N, D = z_rows.shape
    K = codebook.shape[0]
    dz = torch.empty_like(z_rows)
    dE = torch.empty((K, D), dtype=torch.float32, device=z_rows.device)
    gz = _f32c(g_zq) if g_zq is not None else None
    gl = _f32c(g_loss).reshape(1) if g_loss is not None else None
    check(lib().vqb_vq_backward_f32(gz.data_ptr() if gz is not None else None, gl.data_ptr() if gl is not None else None,
                                    z_rows.data_ptr(), codebook.data_ptr(), idx.data_ptr(), N, K, D, float(beta),
                                    dz.data_ptr(), dE.data_ptr(), _stream()), "vq_backward")
    return dz, dE


def vq_finish_ema(sse, hist, N, K, D, beta):
    """(loss, perplexity) of the EMA quantizer: loss = beta * mse, the commitment term alone (vqb_vq_finish_ema_f32)."""
    out = torch.empty((2,), dtype=torch.float32, device=hist.device)
    check(lib().vqb_vq_finish_ema_f32(sse.data_ptr(), hist.data_ptr(), N, K, D, float(beta),
                                      out.data_ptr(), out.data_ptr() + 4, _stream()), "vq_finish_ema")
    return out[0], out[1]


def vq_commit_backward(g_zq, g_loss, z_rows, zq_rows, beta):
    """dz (N,D) of the EMA quantizer from the forward's fp32 z_q rows (vqb_vq_commit_backward_f32); g_zq / g_loss may
    be None."""
    _require_cuda(z_rows, "z")
    N, D = z_rows.shape
    dz = torch.empty_like(z_rows)
    gz = _f32c(g_zq) if g_zq is not None else None
    gl = _f32c(g_loss).reshape(1) if g_loss is not None else None
    check(lib().vqb_vq_commit_backward_f32(gz.data_ptr() if gz is not None else None,
                                           gl.data_ptr() if gl is not None else None, z_rows.data_ptr(),
                                           zq_rows.data_ptr(), N, D, float(beta), dz.data_ptr(), _stream()),
          "vq_commit_backward")
    return dz


def vq_ema_update(z_rows, idx, hist, decay, eps, cluster_size, embed_sum, codebook):
    """One EMA codebook update in place (vqb_vq_ema_update_f32): cluster_size (K,), embed_sum (K,D) and codebook
    (K,D), fp32 contiguous CUDA tensors, from the rows z_rows (N,D) the VQ kernel quantized, their codes idx (N,) and
    its hist (K,).  Version counters are the caller's to bump."""
    _require_cuda(z_rows, "z")
    N, D = z_rows.shape
    K = codebook.shape[0]
    for t in (cluster_size, embed_sum, codebook):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.device != z_rows.device:
            raise RuntimeError("vq_ema_update: the EMA state and the codebook must be contiguous fp32 on z's device")
    ws_bytes = lib().vqb_vq_ema_workspace_bytes(N, K, D)
    ws = torch.empty((max(ws_bytes, 16),), dtype=torch.uint8, device=z_rows.device)
    span = _Span(f"vq_ema N={N} K={K} D={D}")
    check(lib().vqb_vq_ema_update_f32(z_rows.data_ptr(), idx.data_ptr(), hist.data_ptr(), N, K, D, float(decay),
                                      float(eps), cluster_size.data_ptr(), embed_sum.data_ptr(), codebook.data_ptr(),
                                      ws.data_ptr(), ws_bytes, _stream()), "vq_ema_update")
    span.done()


def vq_ema_restart(z_rows, u, threshold, cluster_size, embed_sum, codebook, n_restarted):
    """Dead-code restart in place after an EMA update (vqb_vq_ema_restart_f32): every code with cluster_size < threshold
    moves onto a row of z_rows (N,D), the rows taken by ascending (u, row index) from the uniforms u (N,) fp32;
    n_restarted (1,) int32 receives the count.  Same tensor requirements as vq_ema_update."""
    _require_cuda(z_rows, "z")
    N, D = z_rows.shape
    K = codebook.shape[0]
    for t in (cluster_size, embed_sum, codebook, u):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.device != z_rows.device:
            raise RuntimeError("vq_ema_restart: the EMA state, the codebook and u must be contiguous fp32 on z's device")
    if u.numel() != N or n_restarted.dtype != torch.int32 or n_restarted.numel() != 1 or \
            n_restarted.device != z_rows.device:
        raise RuntimeError("vq_ema_restart: u must hold N values and n_restarted be one int32 on z's device")
    ws_bytes = lib().vqb_vq_ema_restart_workspace_bytes(N, K)
    ws = torch.empty((max(ws_bytes, 16),), dtype=torch.uint8, device=z_rows.device)
    span = _Span(f"vq_ema_restart N={N} K={K} D={D}")
    check(lib().vqb_vq_ema_restart_f32(z_rows.data_ptr(), u.data_ptr(), N, K, D, float(threshold),
                                       cluster_size.data_ptr(), embed_sum.data_ptr(), codebook.data_ptr(),
                                       n_restarted.data_ptr(), ws.data_ptr(), ws_bytes, _stream()), "vq_ema_restart")
    span.done()


def vq_kmeans(z_rows, u, iters, codebook):
    """k-means fit of codebook (K,D), a contiguous fp32 CUDA tensor, in place (vqb_vq_kmeans_f32): seeded with the rows
    of z_rows (N,D) ranked 0..K-1 by ascending (u, row index) from the uniforms u (N,) fp32, then `iters` Lloyd steps.
    Returns sse, a float64 (iters,) device tensor: the inertia before each step.  Version counters are the caller's to
    bump."""
    _require_cuda(z_rows, "z")
    N, D = z_rows.shape
    K = codebook.shape[0]
    for t in (codebook, u):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.device != z_rows.device:
            raise RuntimeError("vq_kmeans: the codebook and u must be contiguous fp32 on z's device")
    if u.numel() != N:
        raise RuntimeError("vq_kmeans: u must hold N values")
    sse = torch.empty((iters,), dtype=torch.float64, device=z_rows.device)
    ws_bytes = lib().vqb_vq_kmeans_workspace_bytes(N, K, D)
    ws = torch.empty((max(ws_bytes, 16),), dtype=torch.uint8, device=z_rows.device)
    span = _Span(f"vq_kmeans N={N} K={K} D={D} iters={iters}")
    check(lib().vqb_vq_kmeans_f32(z_rows.data_ptr(), u.data_ptr(), N, K, D, iters, codebook.data_ptr(),
                                  sse.data_ptr() if iters else None, ws.data_ptr(), ws_bytes, _stream()), "vq_kmeans")
    span.done()
    return sse


def onehot(idx, K):
    N = idx.numel()
    out = torch.empty((N, K), dtype=torch.float32, device=idx.device)
    check(lib().vqb_onehot_f32(idx.data_ptr(), N, K, out.data_ptr(), _stream()), "onehot")
    return out


def gather_rows(idx, codebook):
    _require_cuda(idx, "indices")
    idx = idx.reshape(-1).to(torch.int64).contiguous()
    K, D = codebook.shape
    out = torch.empty((idx.numel(), D), dtype=torch.float32, device=idx.device)
    check(lib().vqb_gather_rows_f32(idx.data_ptr(), codebook.data_ptr(), idx.numel(), K, D,
                                    out.data_ptr(), _stream()), "gather_rows")
    return out


def nchw_to_nhwc(x):
    _require_cuda(x, "input")
    x = _f32c(x)
    B, C, H, W = x.shape
    out = torch.empty((B, H, W, C), dtype=torch.float32, device=x.device)
    check(lib().vqb_nchw_to_nhwc_f32(x.data_ptr(), out.data_ptr(), B, C, H, W, _stream()), "nchw_to_nhwc")
    return out


def nhwc_to_nchw(x):
    B, H, W, C = x.shape
    out = torch.empty((B, C, H, W), dtype=torch.float32, device=x.device)
    check(lib().vqb_nhwc_to_nchw_f32(x.data_ptr(), out.data_ptr(), B, C, H, W, _stream()), "nhwc_to_nchw")
    return out


def nchw_to_nhwc_pad(x, cp):
    """nchw_to_nhwc with the channels zero-padded to cp (vqb_nchw_to_nhwc_pad_f32); nchw_to_nhwc itself at cp = C."""
    _require_cuda(x, "input")
    x = _f32c(x)
    B, C, H, W = x.shape
    if cp == C:
        return nchw_to_nhwc(x)
    out = torch.empty((B, H, W, cp), dtype=torch.float32, device=x.device)
    check(lib().vqb_nchw_to_nhwc_pad_f32(x.data_ptr(), out.data_ptr(), B, C, cp, H, W, _stream()), "nchw_to_nhwc_pad")
    return out


def nhwc_to_nchw_unpad(x, c):
    """nhwc_to_nchw of the first c channels of x (B,H,W,Cp) (vqb_nhwc_to_nchw_unpad_f32); nhwc_to_nchw at c = Cp."""
    B, H, W, cp = x.shape
    if cp == c:
        return nhwc_to_nchw(x)
    out = torch.empty((B, c, H, W), dtype=torch.float32, device=x.device)
    check(lib().vqb_nhwc_to_nchw_unpad_f32(x.data_ptr(), out.data_ptr(), B, c, cp, H, W, _stream()),
          "nhwc_to_nchw_unpad")
    return out


def relu_(x):
    """In-place ReLU on a contiguous fp32 CUDA tensor (residual.py:19 side effect)."""
    check(lib().vqb_relu_f32(x.data_ptr(), x.numel(), _stream()), "relu_")
    return x


def relu_backward(g, y, out=None):
    """out = y > 0 ? g : 0 elementwise (vqb_relu_backward_f32); g, y contiguous fp32 of one size, `out` may be g."""
    if g.numel() != y.numel() or (out is not None and out.numel() != y.numel()):
        raise RuntimeError(f"relu_backward: gradient {tuple(g.shape)} and activation {tuple(y.shape)} differ in size")
    if out is None:
        out = torch.empty_like(y)
    check(lib().vqb_relu_backward_f32(g.data_ptr(), y.data_ptr(), out.data_ptr(), y.numel(), _stream()), "relu_backward")
    return out


def conv_wgrad(x, g_out, dW, dbias, *, B, Cin, H, W, Cout, kh, kw, stride, pad, transposed=False, in_layout=NHWC,
               gout_layout=NHWC):
    """Overwrite dW (the parameter's layout) and dbias (None: not computed) with the weight and bias gradient of one
    conv layer from its input `x` and output gradient `g_out` (vqb_conv_wgrad_f32)."""
    _require_cuda(x, "input")
    n = lib().vqb_conv_wgrad_workspace_bytes(B, Cin, H, W, Cout, kh, kw, stride, pad, int(bool(transposed)))
    if n == 0:
        raise RuntimeError("conv_wgrad: bad geometry")
    ws = torch.empty((n,), dtype=torch.uint8, device=x.device)
    span = _Span(f"wgrad{'T' if transposed else ''} {Cin}->{Cout} k{kh}s{stride} {H}x{W} B={B}")
    check(lib().vqb_conv_wgrad_f32(x.data_ptr(), g_out.data_ptr(), dW.data_ptr(),
                                   dbias.data_ptr() if dbias is not None else None, B, Cin, H, W, Cout, kh, kw, stride,
                                   pad, int(bool(transposed)), in_layout, gout_layout, ws.data_ptr(), n, _stream()),
          "conv_wgrad")
    span.done()


VQ_KERNELS = {"auto": 0, "exact": 1, "tc": 2}


def set_vq_kernel(name: str):
    """Kernel used by vq_forward: "auto" (see vqb_vq_forward_f32), "exact" (FFMA) or "tc"."""
    check(lib().vqb_set_vq_kernel(VQ_KERNELS[name]), "set_vq_kernel")


def vq_debug_scores(z_rows, codebook):
    """Diagnostic: wgmma VQ kernel + dump of its approximate TF32 scores (N, Kpad)."""
    N, D = z_rows.shape
    K = codebook.shape[0]
    dev = z_rows.device
    kpad = (K + 255) // 256 * 256
    idx = torch.empty((N,), dtype=torch.int64, device=dev)
    zq = torch.empty((N, D), dtype=torch.float32, device=dev)
    sse = torch.empty((1,), dtype=torch.float64, device=dev)
    hist = torch.empty((K,), dtype=torch.int32, device=dev)
    scores = torch.full((N, kpad), float("nan"), dtype=torch.float32, device=dev)
    ws_bytes = lib().vqb_vq_workspace_bytes(N, K, D)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    check(lib().vqb_debug_vq_scores_f32(z_rows.data_ptr(), codebook.data_ptr(), N, K, D, idx.data_ptr(),
                                        zq.data_ptr(), sse.data_ptr(), hist.data_ptr(), ws.data_ptr(),
                                        ws_bytes, scores.data_ptr(), _stream()), "vq_debug_scores")
    return idx, zq, sse, hist, scores


# ---- Gated PixelCNN prior (vqb_prior_*) ------------------------------------------------------------------------
def prior_pack_weight(w, rows, cols, out=None):
    """(Cout,Cin,kh,kw) conv weight -> [(r*cols+s)*Cin+ci][co] for the taps r < rows, s < cols (vqb_prior_pack_f32)."""
    _require_cuda(w, "weight")
    w = _f32c(w.detach())
    cout, cin, kh, kw = w.shape
    n = max(rows * cols * cin * cout, 1)
    if out is None or out.numel() != n or out.dtype != torch.float32 or out.device != w.device:
        out = torch.empty((n,), dtype=torch.float32, device=w.device)
    check(lib().vqb_prior_pack_f32(w.data_ptr(), out.data_ptr(), cout, cin, kh, kw, rows, cols, _stream()),
          "prior_pack_weight")
    return out


def prior_gate(x):
    """GatedActivation on (B, 2C, ...) fp32 CUDA -> (B, C, ...) (vqb_prior_gate_f32)."""
    _require_cuda(x, "input")
    x = _f32c(x.detach())
    if x.dim() < 2 or x.shape[1] % 2:
        raise RuntimeError(f"GatedActivation: expected (B, 2C, ...) with an even channel count, got {tuple(x.shape)}")
    c = x.shape[1] // 2
    inner = x[0, 0].numel()
    out = torch.empty((x.shape[0], c) + tuple(x.shape[2:]), dtype=torch.float32, device=x.device)
    if out.numel():
        check(lib().vqb_prior_gate_f32(x.data_ptr(), out.data_ptr(), x.shape[0], c, inner, _stream()), "prior_gate")
    return out


def prior_gate_backward(x, d_out):
    """d x of GatedActivation from its (B, 2C, ...) input and the (B, C, ...) gradient of its output
    (vqb_prior_gate_backward_f32)."""
    x, d_out = _f32c(x.detach()), _f32c(d_out)
    c = x.shape[1] // 2
    d_x = torch.empty_like(x)
    if d_x.numel():
        check(lib().vqb_prior_gate_backward_f32(x.data_ptr(), d_out.data_ptr(), d_x.data_ptr(), x.shape[0], c,
                                                x[0, 0].numel(), _stream()), "prior_gate_backward")
    return d_x


def prior_layer(layer_w, x_v, x_h, labels, *, B, H, W, dim, n_classes):
    """One GatedMaskedConv2d on NHWC (B,H,W,dim) fp32 buffers -> (out_v, out_h) NHWC (vqb_prior_layer_f32)."""
    out_v = torch.empty((B, H, W, dim), dtype=torch.float32, device=x_v.device)
    out_h = torch.empty_like(out_v)
    vh = torch.empty((B, H, W, 2 * dim), dtype=torch.float32, device=x_v.device)
    span = _Span(f"prior layer dim={dim} {H}x{W}")
    check(lib().vqb_prior_layer_f32(_lib.C.byref(layer_w), x_v.data_ptr(), x_h.data_ptr(), labels.data_ptr(), B, H, W,
                                    dim, n_classes, out_v.data_ptr(), out_h.data_ptr(), vh.data_ptr(), _stream()),
          "prior_layer")
    span.done()
    return out_v, out_h


def prior_layer_forward_train(layer_w, x_v, x_h, labels, *, B, H, W, dim, n_classes):
    """prior_layer that also keeps what its backward reads -> (out_v, out_h, saved), saved a uint8 buffer of
    vqb_prior_layer_train_saved_bytes (vqb_prior_layer_forward_train_f32; the outputs are bitwise prior_layer's)."""
    n = lib().vqb_prior_layer_train_saved_bytes(B, H, W, dim)
    if n == 0:
        raise RuntimeError("prior layer: bad sizes")
    saved = torch.empty((n,), dtype=torch.uint8, device=x_v.device)
    out_v = torch.empty((B, H, W, dim), dtype=torch.float32, device=x_v.device)
    out_h = torch.empty_like(out_v)
    vh = torch.empty((B, H, W, 2 * dim), dtype=torch.float32, device=x_v.device)
    span = _Span(f"prior layer (train) dim={dim} {H}x{W}")
    check(lib().vqb_prior_layer_forward_train_f32(_lib.C.byref(layer_w), x_v.data_ptr(), x_h.data_ptr(),
                                                  labels.data_ptr(), B, H, W, dim, n_classes, out_v.data_ptr(),
                                                  out_h.data_ptr(), vh.data_ptr(), saved.data_ptr(), saved.numel(),
                                                  _stream()),
          "prior_layer_forward_train")
    span.done()
    return out_v, out_h, saved


def prior_layer_backward(layer_w, x_v, x_h, labels, d_out_v, d_out_h, saved, grads, *, B, H, W, dim, n_classes):
    """One layer's gradients (vqb_prior_layer_backward_wide_f32, any dim the prior takes): the nine weight gradients into the tensors `grads` (a
    PriorLayerGrads struct) points at -> (d_x_v, d_x_h) NHWC.  d_out_v None: a zero gradient."""
    n = lib().vqb_prior_layer_backward_wide_workspace_bytes(_lib.C.byref(layer_w), B, H, W, dim, n_classes)
    if n == 0:
        raise RuntimeError("prior layer backward: bad sizes")
    ws = torch.empty((n,), dtype=torch.uint8, device=x_v.device)
    d_x_v = torch.empty((B, H, W, dim), dtype=torch.float32, device=x_v.device)
    d_x_h = torch.empty_like(d_x_v)
    span = _Span(f"prior layer backward dim={dim} {H}x{W}")
    check(lib().vqb_prior_layer_backward_wide_f32(_lib.C.byref(layer_w), x_v.data_ptr(), x_h.data_ptr(),
                                                  labels.data_ptr(), B, H, W, dim, n_classes,
                                                  d_out_v.data_ptr() if d_out_v is not None else None,
                                                  d_out_h.data_ptr(), saved.data_ptr(), _lib.C.byref(grads),
                                                  d_x_v.data_ptr(), d_x_h.data_ptr(), ws.data_ptr(), n, _stream()),
          "prior_layer_backward")
    span.done()
    return d_x_v, d_x_h


def _prior_workspace(net, B, H, W, dev, size=None, *extra):
    n = (size or lib().vqb_prior_workspace_bytes)(B, H, W, net.dim, net.n_layers, net.input_dim, *extra)
    if n == 0:
        raise RuntimeError("prior: bad sizes")
    return torch.empty((n,), dtype=torch.uint8, device=dev)


PRIOR_PRECISIONS = ("fp32", "tf32")


def _prior_precision(precision):
    """The C-ABI suffix of a prior precision: "fp32" -> "f32" (CUDA cores), "tf32" -> "tf32" (wgmma tensor cores)."""
    if precision not in PRIOR_PRECISIONS:
        raise ValueError(f"prior precision must be one of {PRIOR_PRECISIONS}, got {precision!r}")
    return "f32" if precision == "fp32" else "tf32"


def prior_forward(net, codes, labels, precision="fp32"):
    """Teacher-forced logits (B, K, H, W) of int64 codes (B,H,W) and labels (B,) (vqb_prior_forward_f32, or
    vqb_prior_forward_tf32 for precision="tf32")."""
    sfx = _prior_precision(precision)
    B, H, W = codes.shape
    dev = codes.device
    logits = torch.empty((B, net.input_dim, H, W), dtype=torch.float32, device=dev)
    ws = _prior_workspace(net, B, H, W, dev, lib().vqb_prior_workspace_bytes_tf32 if sfx == "tf32" else None)
    span = _Span(f"prior forward ({precision}) K={net.input_dim} dim={net.dim} L={net.n_layers} {H}x{W}")
    check(getattr(lib(), "vqb_prior_forward_" + sfx)(_lib.C.byref(net), codes.data_ptr(), labels.data_ptr(), B, H, W,
                                                      logits.data_ptr(), ws.data_ptr(), ws.numel(), _stream()),
          "prior_forward")
    span.done()
    return logits


def prior_log_prob(net, codes, labels, n_given, precision="fp32", per_position=False):
    """log softmax of the teacher-forced logits at each int64 code of codes (B,H,W) (clamped to [0, K-1]), without
    writing the logits (vqb_prior_log_prob_f32, or _tf32 for precision="tf32") -> per_position=False: (B,) fp32, the
    compensated sum over the raster positions >= n_given; per_position=True: the (B,H,W) fp32 map of every term."""
    sfx = _prior_precision(precision)
    B, H, W = codes.shape
    dev = codes.device
    ws = _prior_workspace(net, B, H, W, dev, getattr(lib(), "vqb_prior_log_prob_workspace_bytes" +
                                                     ("_tf32" if sfx == "tf32" else "")))
    out = torch.empty((B, H, W) if per_position else (B,), dtype=torch.float32, device=dev)
    span = _Span(f"prior log_prob ({precision}) K={net.input_dim} dim={net.dim} L={net.n_layers} {H}x{W} "
                 f"n_given={n_given}")
    check(getattr(lib(), "vqb_prior_log_prob_" + sfx)(_lib.C.byref(net), codes.data_ptr(), labels.data_ptr(), n_given,
                                                       B, H, W, None if per_position else out.data_ptr(),
                                                       out.data_ptr() if per_position else None, ws.data_ptr(),
                                                       ws.numel(), _stream()),
          "prior_log_prob")
    span.done()
    return out


def prior_log_prob_ragged(net, codes, labels, n_given, precision="fp32"):
    """prior_log_prob with one prefix length per image, n_given int64 (B,) on the device (vqb_prior_log_prob_ragged_f32
    / _tf32) -> (B,) fp32, entry b the compensated sum over the raster positions >= n_given[b] (clamped to [0, H*W])."""
    sfx = _prior_precision(precision)
    B, H, W = codes.shape
    dev = codes.device
    ws = _prior_workspace(net, B, H, W, dev, getattr(lib(), "vqb_prior_log_prob_workspace_bytes" +
                                                     ("_tf32" if sfx == "tf32" else "")))
    out = torch.empty((B,), dtype=torch.float32, device=dev)
    span = _Span(f"prior log_prob ragged ({precision}) K={net.input_dim} dim={net.dim} L={net.n_layers} {H}x{W}")
    check(getattr(lib(), "vqb_prior_log_prob_ragged_" + sfx)(_lib.C.byref(net), codes.data_ptr(), labels.data_ptr(),
                                                              n_given.data_ptr(), B, H, W, out.data_ptr(),
                                                              ws.data_ptr(), ws.numel(), _stream()),
          "prior_log_prob_ragged")
    span.done()
    return out


PRIOR_CE_REDUCTIONS = ("none", "mean", "sum")      # VQB_PRIOR_CE_NONE, _MEAN, _SUM


def _prior_ce_reduction(reduction):
    if reduction not in PRIOR_CE_REDUCTIONS:
        raise ValueError(f"reduction must be one of {PRIOR_CE_REDUCTIONS}, got {reduction!r}")
    return PRIOR_CE_REDUCTIONS.index(reduction)


_INT64 = (-2 ** 63, 2 ** 63 - 1)


def prior_ce_options(weight=None, ignore_index=None, label_smoothing=0.0):
    """The vqb_prior_ce_options struct of cross_entropy's options, or None when they are all neutral by default
    (weight None, ignore_index None, label_smoothing 0): the call without options.  weight: None or a contiguous fp32
    tensor of K entries on the device, which the struct points at (the caller keeps it alive for the call, or for the
    graph).  An ignore_index outside int64 matches no code."""
    if weight is None and ignore_index is None and label_smoothing == 0.0:
        return None
    has_ignore = ignore_index is not None and _INT64[0] <= ignore_index <= _INT64[1]
    return _lib.PriorCeOptions(weight=weight.data_ptr() if weight is not None else None,
                               ignore_index=int(ignore_index) if has_ignore else 0, has_ignore=int(has_ignore),
                               label_smoothing=float(label_smoothing))


def prior_ce_forward(net, codes, labels, reduction, precision="fp32", train=False, options=None):
    """The cross-entropy of the teacher-forced logits at int64 codes (B,H,W) (clamped to [0, K-1]) without writing the
    logits (vqb_prior_ce_forward_f32, or _tf32 for precision="tf32") -> (loss, saved): loss (B,H,W) fp32 for
    reduction="none", a 0-d fp32 tensor otherwise; saved None, or with train=True the uint8 buffer of
    vqb_prior_ce_saved_bytes that prior_ce_backward reads.  options: None, or a prior_ce_options struct (the _ex
    entry points, vqb_prior_ce_saved_bytes_ex and vqb_prior_ce_workspace_bytes_ex)."""
    sfx = _prior_precision(precision)
    r = _prior_ce_reduction(reduction)
    B, H, W = codes.shape
    dev = codes.device
    saved = None
    opt = _lib.C.byref(options) if options is not None else None
    if train:
        n = (lib().vqb_prior_ce_saved_bytes(B, H, W, net.dim, net.n_layers) if options is None else
             lib().vqb_prior_ce_saved_bytes_ex(B, H, W, net.dim, net.n_layers, opt))
        if n == 0:
            raise RuntimeError("prior: bad sizes")
        saved = torch.empty((n,), dtype=torch.uint8, device=dev)
    tf = "_tf32" if sfx == "tf32" else ""
    if options is None:
        ws = _prior_workspace(net, B, H, W, dev, getattr(lib(), "vqb_prior_ce_workspace_bytes" + tf), int(train))
    else:
        ws = _prior_workspace(net, B, H, W, dev, getattr(lib(), "vqb_prior_ce_workspace_bytes_ex" + tf), int(train),
                              opt)
    loss = torch.empty((B, H, W) if r == 0 else (), dtype=torch.float32, device=dev)
    span = _Span(f"prior cross_entropy ({precision}, {reduction}) K={net.input_dim} dim={net.dim} L={net.n_layers} "
                 f"{H}x{W}")
    args = (_lib.C.byref(net), codes.data_ptr(), labels.data_ptr(), B, H, W, r)
    rest = (loss.data_ptr(), saved.data_ptr() if saved is not None else None, saved.numel() if saved is not None else 0,
            ws.data_ptr(), ws.numel(), _stream())
    if options is None:
        check(getattr(lib(), "vqb_prior_ce_forward_" + sfx)(*args, *rest), "prior_ce_forward")
    else:
        check(getattr(lib(), "vqb_prior_ce_forward_ex_" + sfx)(*args, opt, *rest), "prior_ce_forward")
    span.done()
    return loss, saved


def prior_ce_backward(net, codes, labels, reduction, d_loss, saved, grads, precision="fp32", options=None):
    """Every parameter gradient of the prior's cross-entropy (vqb_prior_ce_backward_f32 / _tf32) into the tensors
    `grads` (a PriorGrads struct) points at; d_loss fp32 contiguous on the device, (B,H,W) for reduction="none" and
    one element otherwise, saved from prior_ce_forward(train=True) on the same net, inputs, reduction and options."""
    sfx = _prior_precision(precision)
    r = _prior_ce_reduction(reduction)
    B, H, W = codes.shape
    n = lib().vqb_prior_ce_backward_workspace_bytes(_lib.C.byref(net), B, H, W)
    if n == 0:
        raise RuntimeError("prior backward: bad sizes")
    ws = torch.empty((n,), dtype=torch.uint8, device=codes.device)
    span = _Span(f"prior cross_entropy backward ({precision}, {reduction}) K={net.input_dim} dim={net.dim} "
                 f"L={net.n_layers} {H}x{W}")
    args = (_lib.C.byref(net), codes.data_ptr(), labels.data_ptr(), B, H, W, r)
    rest = (d_loss.data_ptr(), saved.data_ptr(), _lib.C.byref(grads), ws.data_ptr(), ws.numel(), _stream())
    if options is None:
        check(getattr(lib(), "vqb_prior_ce_backward_" + sfx)(*args, *rest), "prior_ce_backward")
    else:
        check(getattr(lib(), "vqb_prior_ce_backward_ex_" + sfx)(*args, _lib.C.byref(options), *rest),
              "prior_ce_backward")
    span.done()


def prior_generate(net, labels, u, step_logits=None):
    """The whole sampling loop (vqb_prior_generate_f32): int64 codes (B,H,W) drawn with the uniforms u (B,H,W).
    step_logits: None, or a (B,H,W,K) fp32 tensor receiving the logits of every step."""
    B, H, W = u.shape
    dev = u.device
    codes = torch.empty((B, H, W), dtype=torch.int64, device=dev)
    ws = _prior_workspace(net, B, H, W, dev)
    span = _Span(f"prior generate K={net.input_dim} dim={net.dim} L={net.n_layers} {H}x{W}")
    check(lib().vqb_prior_generate_f32(_lib.C.byref(net), labels.data_ptr(), u.data_ptr(), B, H, W, codes.data_ptr(),
                                       step_logits.data_ptr() if step_logits is not None else None, ws.data_ptr(),
                                       ws.numel(), _stream()), "prior_generate")
    span.done()
    return codes


def prior_complete(net, labels, u, given, n_given, step_logits=None):
    """The sampling loop from raster position n_given on (vqb_prior_complete_f32): int64 codes (B,H,W) whose positions
    < n_given are the int64 `given` (B,H,W) and the rest are drawn with the uniforms u (B,H,W).  step_logits: None,
    or a (B,H,W,K) fp32 tensor receiving the logits of every step (positions >= n_given)."""
    B, H, W = u.shape
    dev = u.device
    codes = torch.empty((B, H, W), dtype=torch.int64, device=dev)
    ws = _prior_workspace(net, B, H, W, dev, lib().vqb_prior_sample_workspace_bytes, n_given)
    span = _Span(f"prior complete K={net.input_dim} dim={net.dim} L={net.n_layers} {H}x{W} n_given={n_given}")
    check(lib().vqb_prior_complete_f32(_lib.C.byref(net), labels.data_ptr(), u.data_ptr(), given.data_ptr(), n_given,
                                       B, H, W, codes.data_ptr(),
                                       step_logits.data_ptr() if step_logits is not None else None, ws.data_ptr(),
                                       ws.numel(), _stream()), "prior_complete")
    span.done()
    return codes


def prior_sample(net, labels, u, given, n_given, sampling, step_logits=None):
    """prior_complete drawing from the tempered, truncated softmax that `sampling` (a PriorSampling struct) sets
    (vqb_prior_sample_f32) -> (codes (B,H,W) int64, log_prob (B,) fp32: the model's log-probability of the sampled
    positions).  given: None when n_given = 0."""
    B, H, W = u.shape
    dev = u.device
    codes = torch.empty((B, H, W), dtype=torch.int64, device=dev)
    log_prob = torch.empty((B,), dtype=torch.float32, device=dev)
    ws = _prior_workspace(net, B, H, W, dev, lib().vqb_prior_sample_workspace_bytes, n_given)
    span = _Span(f"prior sample K={net.input_dim} dim={net.dim} L={net.n_layers} {H}x{W} n_given={n_given} "
                 f"T={sampling.temperature:g} top_k={sampling.top_k} top_p={sampling.top_p:g}")
    check(lib().vqb_prior_sample_f32(_lib.C.byref(net), labels.data_ptr(), u.data_ptr(),
                                     given.data_ptr() if given is not None else None, n_given, B, H, W,
                                     _lib.C.byref(sampling), codes.data_ptr(), log_prob.data_ptr(),
                                     step_logits.data_ptr() if step_logits is not None else None, ws.data_ptr(),
                                     ws.numel(), _stream()), "prior_sample")
    span.done()
    return codes, log_prob


def prior_sample_ragged(net, labels, u, given, n_given, sampling=None, step_logits=None, log_prob=True):
    """prior_sample with one prefix length per image (vqb_prior_sample_ragged_f32): n_given int64 (B,) on the device,
    never read here; given the int64 codes (B,H,W) whose positions < n_given[b] image b keeps.  sampling None is
    complete's draw.  -> (codes (B,H,W) int64, log_prob (B,) fp32, or None with log_prob=False)."""
    B, H, W = u.shape
    dev = u.device
    codes = torch.empty((B, H, W), dtype=torch.int64, device=dev)
    lp = torch.empty((B,), dtype=torch.float32, device=dev) if log_prob else None
    ws = _prior_workspace(net, B, H, W, dev, lib().vqb_prior_sample_workspace_bytes, 0)
    knobs = "" if sampling is None else \
        f" T={sampling.temperature:g} top_k={sampling.top_k} top_p={sampling.top_p:g}"
    span = _Span(f"prior sample ragged K={net.input_dim} dim={net.dim} L={net.n_layers} {H}x{W}{knobs}")
    check(lib().vqb_prior_sample_ragged_f32(_lib.C.byref(net), labels.data_ptr(), u.data_ptr(), given.data_ptr(),
                                            n_given.data_ptr(), B, H, W,
                                            _lib.C.byref(sampling) if sampling is not None else None,
                                            codes.data_ptr(), lp.data_ptr() if lp is not None else None,
                                            step_logits.data_ptr() if step_logits is not None else None,
                                            ws.data_ptr(), ws.numel(), _stream()), "prior_sample_ragged")
    span.done()
    return codes, lp


def prior_forward_train(net, codes, labels, precision="fp32"):
    """prior_forward that also keeps the activations the backward needs: (logits, saved) with saved a uint8 buffer
    of vqb_prior_train_saved_bytes (vqb_prior_forward_train_f32 / _tf32; the logits are bitwise prior_forward's in the
    same precision)."""
    sfx = _prior_precision(precision)
    B, H, W = codes.shape
    dev = codes.device
    n = lib().vqb_prior_train_saved_bytes(B, H, W, net.dim, net.n_layers)
    if n == 0:
        raise RuntimeError("prior: bad sizes")
    saved = torch.empty((n,), dtype=torch.uint8, device=dev)
    logits = torch.empty((B, net.input_dim, H, W), dtype=torch.float32, device=dev)
    span = _Span(f"prior forward (train, {precision}) K={net.input_dim} dim={net.dim} L={net.n_layers} {H}x{W}")
    check(getattr(lib(), "vqb_prior_forward_train_" + sfx)(_lib.C.byref(net), codes.data_ptr(), labels.data_ptr(), B,
                                                            H, W, logits.data_ptr(), saved.data_ptr(), saved.numel(),
                                                            _stream()),
          "prior_forward_train")
    span.done()
    return logits, saved


def prior_backward(net, codes, labels, d_logits, saved, grads, precision="fp32"):
    """Every parameter gradient of the prior (vqb_prior_backward_f32 / _tf32) into the tensors `grads` (a PriorGrads
    struct) points at; d_logits (B, K, H, W) fp32 contiguous, saved from prior_forward_train on the same net and
    inputs, in the same precision."""
    sfx = _prior_precision(precision)
    B, H, W = codes.shape
    n = lib().vqb_prior_backward_workspace_bytes(_lib.C.byref(net), B, H, W)
    if n == 0:
        raise RuntimeError("prior backward: bad sizes")
    ws = torch.empty((n,), dtype=torch.uint8, device=codes.device)
    span = _Span(f"prior backward ({precision}) K={net.input_dim} dim={net.dim} L={net.n_layers} {H}x{W}")
    check(getattr(lib(), "vqb_prior_backward_" + sfx)(_lib.C.byref(net), codes.data_ptr(), labels.data_ptr(), B, H,
                                                       W, d_logits.data_ptr(), saved.data_ptr(), _lib.C.byref(grads),
                                                       ws.data_ptr(), ws.numel(), _stream()), "prior_backward")
    span.done()


# ---- optimizer step (vqb_adam_multi_f32 / vqb_repack_multi) -------------------------------------------------------
def adam_multi(tensors, n, lr, beta1, beta2, eps, weight_decay, amsgrad):
    """Adam over a ctypes array of n AdamTensor descriptors (device pointers; read during the call only)."""
    span = _Span(f"adam x{n}")
    check(lib().vqb_adam_multi_f32(tensors, n, float(lr), float(beta1), float(beta2), float(eps), float(weight_decay),
                                   int(bool(amsgrad)), _stream()), "adam_multi")
    span.done()


def repack_multi(descs, n, steps, n_steps):
    """Every packing of a ctypes array of n PackDesc descriptors, then +1 on each of the n_steps device fp32 step
    counters of the ctypes pointer array `steps`."""
    span = _Span(f"repack x{n}")
    check(lib().vqb_repack_multi(descs, n, steps, n_steps, _stream()), "repack_multi")
    span.done()


def pad_width(n, kind, cp):
    """Width at Cp channels of an axis of n real channels and kind 0 (kept), 1 (dim-wide) or 2 (a gate axis, padded
    per half): vqb_pack_layout's padded layouts."""
    return kind * cp if kind else n


def pack_one(w, fields, n, out=None):
    """One packing of the fp32 CUDA parameter w into n fp32 elements, described by the PackDesc fields `fields`
    (layout and geometry), through vqb_repack_multi with one descriptor; `out` is refilled when it has that size."""
    _require_cuda(w, "weight")
    w = _f32c(w.detach())
    n = max(n, 1)
    if out is None or out.numel() != n or out.dtype != torch.float32 or out.device != w.device:
        out = torch.empty((n,), dtype=torch.float32, device=w.device)
    desc = (_lib.PackDesc * 1)(_lib.PackDesc(dst=out.data_ptr(), src=w.data_ptr(), **fields))
    repack_multi(desc, 1, None, 0)
    return out

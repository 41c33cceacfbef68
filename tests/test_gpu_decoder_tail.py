"""The decoder's output layer (decoder.py:34-35, ConvTranspose2d k4 s2 p1 to <= 4 channels) in scatter form
(wgconv.cu, convt_scatter_kernel): each tile's input pixels and their one-pixel halo are multiplied once by the 64 weight
rows (phase, neighbour, channel) gathered from the [9][16][Cin] packing, and the epilogue sums the four neighbour terms
of every output pixel.

Held to the C oracle at the layer tolerances of the existing tests (TF32: 4e-3 abs + 2e-3 rel; bf16 operands, fp32
output: the oracle on the same bf16-rounded operands, 2e-4 abs + 1e-4 rel) on shapes the model does not reach: odd and
non-power-of-two images, tiles split over the width, more tiles than the persistent grid holds (CTAs looping around
the ring, at two CTAs per SM and at one with 8 chunks), every channel count from 1 to 4, 32 to 256 input channels, ReLU
on and off.  Which kernel ran is read from the profiler, so a fall-back to the CUDA-core kernel fails the test.  Also:
a CUDA-graph replay and a second call are bitwise equal to the first eager call.  Needs an H100 (``-m gpu``).
"""
import numpy as np
import pytest
import torch

from oracle import cref

pytestmark = pytest.mark.gpu


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bf(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.bfloat16).float().numpy()


def _kernels(call):
    """(result of call(), names of the CUDA kernels it launched)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        y = call()
        torch.cuda.synchronize()
    return y, [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def _inputs(seed, B, Cin, H, W, Cout, bf16):
    rng = np.random.RandomState(seed)
    x = rng.standard_normal((B, Cin, H, W)).astype(np.float32)
    w = (rng.standard_normal((Cin, Cout, 4, 4)) / np.sqrt(Cin * 16)).astype(np.float32)
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    if bf16:
        x = _bf(x)
    return x, w, b


def _run(x, w, b, relu, bf16):
    """The output layer through the C ABI: fp32 NHWC (TF32 mode) or bf16 NHWC input, fp32 NCHW output."""
    from vqvae_b200 import _lib, ops
    B, Cin, H, W = x.shape
    Cout = w.shape[1]
    if bf16:
        kind = _lib.CONVT_K4S2_OUT
        xin = torch.from_numpy(np.ascontiguousarray(x.transpose(0, 2, 3, 1))).to(torch.bfloat16).cuda()
        wp, bd = ops.pack_conv_weight_bf16(_cuda(w), kind), _cuda(b)
        return lambda: ops.conv2d_bf16(xin, wp, bd, B=B, Cin=Cin, H=H, W=W, Cout=Cout, kind=kind, relu=relu,
                                       out_f32=True)
    wp = ops.pack_conv_weight(_cuda(w), True)
    xin, bd = _cuda(x.transpose(0, 2, 3, 1)), _cuda(b)
    return lambda: ops.conv2d(xin, wp, bd, B=B, Cin=Cin, H=H, W=W, Cout=Cout, kh=4, kw=4, stride=2, pad=1,
                              transposed=True, in_layout=_lib.NHWC, out_layout=_lib.NCHW,
                              relu=relu, precision=_lib.TF32)


def _check(case, bf16, kernel):
    B, Cin, H, W, Cout, relu = case
    x, w, b = _inputs(sum(case) + (3 if bf16 else 0), B, Cin, H, W, Cout, bf16)
    ref = cref.conv_transpose2d(x, _bf(w) if bf16 else w, b, 2, 1)
    if relu:
        ref = np.maximum(ref, 0)
    y, names = _kernels(_run(x, w, b, relu, bf16))
    convs = [n for n in names if "conv" in n]
    assert len(convs) == 1 and kernel in convs[0], names       # one conv launch, of the expected kernel
    y = y.float().cpu().numpy()
    assert y.shape == ref.shape == (B, Cout, 2 * H, 2 * W)
    if bf16:
        np.testing.assert_allclose(y, ref, atol=2e-4, rtol=1e-4)
    else:
        np.testing.assert_allclose(y, ref, atol=4e-3, rtol=2e-3)


OUT_CASES = [
    # B, Cin, H, W, Cout, relu
    (3, 64, 5, 6, 3, False),        # one small tile per image
    (2, 32, 3, 17, 4, True),        # width split into two tiles of 9 and 8 columns
    (1, 64, 33, 20, 3, False),      # 33 rows: ragged last tile row, two column tiles
    (5, 128, 7, 9, 2, True),        # 5 images, 4 chunks (TF32)
    (2, 256, 8, 8, 1, False),       # 256 input channels, one output channel
    (3, 32, 16, 16, 4, True),       # cfg2 tile shape, 4 output channels
    (45, 64, 16, 16, 3, False),     # 180 tiles: more CTAs than SMs, one tile each
    (70, 64, 16, 16, 3, False),     # 280 tiles, more than two CTAs per SM: CTAs loop over tiles around the ring
    (40, 256, 16, 16, 3, True),     # 160 tiles at 8 chunks: one CTA per SM with the 4-stage ring, looping
    (7, 64, 1, 1, 3, True),         # one input pixel per image: everything else is padding
]


@pytest.mark.parametrize("case", OUT_CASES)
def test_tf32_output_layer_vs_oracle(case):
    _check(case, False, "convt_scatter_kernel")


BF16_OUT_CASES = [
    (3, 64, 5, 6, 3, False),
    (2, 64, 3, 17, 1, True),
    (1, 128, 33, 20, 2, False),
    (5, 256, 7, 9, 4, True),
    (45, 64, 16, 16, 3, False),     # 180 tiles: more CTAs than SMs, one tile each
    (70, 64, 16, 16, 3, False),     # 280 tiles: CTAs loop over tiles
]


@pytest.mark.parametrize("case", BF16_OUT_CASES)
def test_bf16_output_layer_vs_oracle(case):
    _check(case, True, "convt_scatter_kernel")


@pytest.mark.parametrize("bf16", [False, True])
def test_output_layer_is_deterministic_and_graph_capturable(bf16):
    """Two eager calls and a CUDA-graph replay of the same call give bitwise-equal outputs."""
    _deterministic_and_graph_capturable(bf16, 3)


def _deterministic_and_graph_capturable(bf16, Cout):
    x, w, b = _inputs(17, 9, 64, 13, 19, Cout, bf16)
    call = _run(x, w, b, False, bf16)
    y0 = call().clone()
    y1 = call().clone()
    assert torch.equal(y0, y1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()                                         # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        yg = call()
    yg.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, y0)

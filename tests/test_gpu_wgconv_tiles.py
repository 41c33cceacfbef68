"""Tile edges of the wgmma convolution (wgconv.cu), where each k-step's A box is the tile's input shifted by a tap and
zero filled outside the image: taps that reach into neighbouring tiles on all four sides, ragged right / bottom tiles
with stride-2 taps, several small images per tile (zero padding between images and past the batch), chained residual
applications that read the previous application's output back, the widest shapes the launcher takes (8 chunks,
N = 256), and the training backward's adjoint convs over interior tiles.  The model's forward layers reach none of
these.  Held to the C oracle at the TF32 / bf16 tolerances of the existing layer tests; every TF32 case is checked by
kernel name, through the profiler, to run on the wgmma kernel.  Needs an H100 (``-m gpu``).
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


def _layer(rng, B, Cin, H, W, Cout, k, stride, transposed, bf16):
    x = rng.standard_normal((B, Cin, H, W)).astype(np.float32)
    w = (rng.standard_normal((Cin, Cout, k, k) if transposed else (Cout, Cin, k, k)) / np.sqrt(Cin * k * k)).astype(np.float32)
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    if bf16:
        x = _bf(x)
    wq = _bf(w) if bf16 else w
    pad = 0 if k == 1 else 1
    ref = cref.conv_transpose2d(x, wq, b, stride, pad) if transposed else cref.conv2d(x, wq, b, stride, pad)
    return x, w, b, np.maximum(ref, 0)


TF32_CASES = [
    # B, Cin, H, W, Cout, k, stride, transposed
    (1, 64, 24, 40, 64, 3, 1, False),     # 3 x 3 tiles of 16 x 8: taps cross every tile side
    (1, 64, 20, 20, 64, 4, 2, True),      # four sub-pixel phases over 2 x 3 tiles
    (2, 32, 34, 46, 32, 4, 2, False),     # stride 2, 17 x 23 outputs: ragged right and bottom tiles
    (6, 64, 4, 4, 64, 3, 1, False),       # 8 images per tile, 6 in the batch
    (5, 32, 6, 6, 32, 4, 2, False),       # stride 2, 3 x 3 outputs, 8 images per tile
    (1, 256, 16, 16, 256, 3, 1, False),   # 8 chunks x 9 taps, N = 256
    # adjoint convs of the training backward (modules._conv_dgrad) with an interior tile: 3 x 3 tiles of 16 x 8
    (2, 32, 24, 40, 128, 3, 1, True),     # residual W1's adjoint: transposed k3, 1 chunk, N = 128
    (2, 128, 24, 40, 128, 3, 1, True),    # encoder conv 4's adjoint: transposed k3, 4 chunks
    (2, 128, 20, 36, 32, 1, 1, True),     # residual W2's adjoint: transposed 1x1 over 3 x 3 tiles, ragged on both axes
]


def _pad(k):
    return 0 if k == 1 else 1


@pytest.fixture(scope="module")
def tf32_kernels():
    """case -> the CUDA kernels one call of each TF32_CASES case ran, from torch.profiler."""
    from tests.helpers import tf32_conv_kernels
    from vqvae_b200._lib import NHWC
    calls = [(B, Cin, H, W, Cout, k, s, _pad(k), t, NHWC, NHWC, True, False) for B, Cin, H, W, Cout, k, s, t in TF32_CASES]
    return dict(zip(TF32_CASES, tf32_conv_kernels(calls)))


@pytest.mark.parametrize("case", TF32_CASES)
def test_tf32_tile_edge_layers_vs_oracle(case, tf32_kernels):
    from vqvae_b200 import ops
    from vqvae_b200._lib import NHWC, TF32
    B, Cin, H, W, Cout, k, stride, transposed = case
    x, w, b, ref = _layer(np.random.RandomState(sum(case) + 7), *case, bf16=False)
    wp = ops.pack_conv_weight(_cuda(w), transposed)
    l0 = ops.launch_count()
    y = ops.conv2d(_cuda(x.transpose(0, 2, 3, 1)), wp, _cuda(b), B=B, Cin=Cin,
                   H=H, W=W, Cout=Cout, kh=k, kw=k, stride=stride, pad=_pad(k), transposed=transposed, in_layout=NHWC,
                   out_layout=NHWC, relu=True, precision=TF32)
    assert ops.launch_count() - l0 == 1
    np.testing.assert_allclose(y.cpu().numpy().transpose(0, 3, 1, 2), ref, atol=4e-3, rtol=2e-3)
    names = tf32_kernels[case]                    # the wgmma kernel, not the CUDA-core fallback
    assert len(names) == 1 and "wgconv_kernel" in names[0], names


BF16_CASES = [
    # B, Cin, H, W, Cout, k, stride, transposed
    (1, 192, 24, 40, 64, 3, 1, False),    # chunk outer over 3 chunks, 3 x 3 tiles
    (1, 128, 20, 20, 64, 4, 2, True),     # four sub-pixel phases over 2 x 3 tiles
    (2, 64, 34, 46, 64, 4, 2, False),     # stride 2, ragged right and bottom tiles
    (6, 128, 4, 4, 64, 3, 1, False),      # 8 images per tile, 6 in the batch
    (5, 64, 6, 6, 64, 4, 2, False),       # stride 2, 8 images per tile
]


@pytest.mark.parametrize("case", BF16_CASES)
def test_bf16_tile_edge_layers_vs_oracle(case):
    from vqvae_b200 import ops
    B, Cin, H, W, Cout, k, stride, transposed = case
    x, w, b, ref = _layer(np.random.RandomState(sum(case) + 11), *case, bf16=True)
    kind = ops.conv_kind(k, stride, transposed, Cout)
    xin = torch.from_numpy(np.ascontiguousarray(x.transpose(0, 2, 3, 1))).to(torch.bfloat16).cuda()
    y = ops.conv2d_bf16(xin, ops.pack_conv_weight_bf16(_cuda(w), kind), _cuda(b), B=B, Cin=Cin, H=H, W=W, Cout=Cout,
                        kind=kind, relu=True, out_f32=False)
    np.testing.assert_allclose(y.float().cpu().numpy().transpose(0, 3, 1, 2), ref, atol=2e-3, rtol=2.0 ** -8)


def test_tf32_residual_stack_three_applications_ragged_images():
    """Three chained applications in one launch on 5 x 6 images, two per tile: each application reads back what the
    previous one stored, with the padding around and between the images zero."""
    from vqvae_b200 import ops
    from vqvae_b200._lib import TF32
    B, H, W, C, Cmid, n = 3, 5, 6, 64, 32, 3
    rng = np.random.RandomState(5)
    r = np.maximum(rng.standard_normal((B, C, H, W)).astype(np.float32), 0)
    w1 = (rng.standard_normal((Cmid, C, 3, 3)) / np.sqrt(C * 9)).astype(np.float32)
    w2 = (rng.standard_normal((C, Cmid, 1, 1)) / np.sqrt(Cmid)).astype(np.float32)
    ref = r
    for _ in range(n):
        ref = np.maximum(ref + cref.conv2d(np.maximum(cref.conv2d(ref, w1, None, 1, 1), 0), w2, None, 1, 0), 0)
    p1, p2 = ops.pack_conv_weight(_cuda(w1), False), ops.pack_conv_weight(_cuda(w2), False)
    l0 = ops.launch_count()
    y = ops.residual_stack(_cuda(r.transpose(0, 2, 3, 1)), p1, p2, B=B, H=H, W=W, C=C, Cmid=Cmid, n_layers=n,
                           precision=TF32)
    assert ops.launch_count() - l0 == 1
    np.testing.assert_allclose(y.cpu().numpy().transpose(0, 3, 1, 2), ref, atol=6e-3 * n, rtol=2e-3 * n)


def test_bf16_residual_layer_small_images():
    """The bf16 residual layer (chunk outer over two chunks) with 8 images of 4 x 4 per tile and 7 in the batch."""
    from vqvae_b200 import ops, _lib
    B, H, W, C, Cmid = 7, 4, 4, 128, 32
    rng = np.random.RandomState(9)
    r = _bf(np.maximum(rng.standard_normal((B, C, H, W)).astype(np.float32), 0))
    w1 = (rng.standard_normal((Cmid, C, 3, 3)) / np.sqrt(C * 9)).astype(np.float32)
    w2 = (rng.standard_normal((C, Cmid, 1, 1)) / np.sqrt(Cmid)).astype(np.float32)
    mid = _bf(np.maximum(cref.conv2d(r, _bf(w1), None, 1, 1), 0))
    ref = np.maximum(r + cref.conv2d(mid, _bf(w2), None, 1, 0), 0)
    p1 = ops.pack_conv_weight_bf16(_cuda(w1), _lib.CONV_K3)
    p2 = ops.pack_conv_weight_bf16(_cuda(w2), _lib.RES_W2)
    rin = torch.from_numpy(np.ascontiguousarray(r.transpose(0, 2, 3, 1))).to(torch.bfloat16).cuda()
    y = ops.residual_layer_bf16(rin, p1, p2, B=B, H=H, W=W, C=C, Cmid=Cmid, relu_out=True)
    np.testing.assert_allclose(y.float().cpu().numpy().transpose(0, 3, 1, 2), ref, atol=6e-3, rtol=2.0 ** -7)

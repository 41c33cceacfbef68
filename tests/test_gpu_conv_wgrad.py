"""The conv weight and bias gradient (vqb_conv_wgrad_f32) called directly, against fp64 autograd on the CPU.  The cases
reach each way the GEMM stages its operands: four channels per float4 load (channels contiguous, C % 4 == 0, 16-byte
aligned) or element by element, the group of four that runs from the last tap column into the bias's column of ones,
and a transposed conv's bias as a second product over an NCHW output gradient."""
import pytest
import torch
import torch.nn.functional as F

from vqvae_b200._lib import NCHW, NHWC

pytestmark = pytest.mark.gpu

# name -> (transposed, B, Cin, H, W, Cout, k, stride, pad, in_layout, gout_layout, bias, input offset in floats)
CASES = {
    "nhwc_vec_bias": (0, 4, 16, 9, 9, 32, 3, 1, 1, NHWC, NHWC, True, 0),
    "enc_input_k4s2_nchw": (0, 3, 3, 16, 16, 32, 4, 2, 1, NCHW, NHWC, True, 0),
    "nhwc_scalar_3_to_6": (0, 4, 3, 9, 9, 6, 3, 1, 1, NHWC, NHWC, True, 0),
    "nhwc_unaligned_input": (0, 4, 16, 9, 9, 32, 3, 1, 1, NHWC, NHWC, True, 1),
    "convt_k4s2_nchw_gout_bias": (1, 3, 32, 8, 8, 3, 4, 2, 1, NHWC, NCHW, True, 0),
    "ones_column_in_last_group": (0, 4, 3, 9, 9, 8, 3, 1, 1, NHWC, NHWC, True, 0),
    "conv1x1_no_bias": (0, 2, 16, 5, 5, 8, 1, 1, 0, NHWC, NHWC, False, 0),
    # the position split under test: cfg3's input conv on 256 x 256 NCHW images, 32 768 positions staged element by
    # element over hundreds of chunks; 3 * 7 * 9 = 189 positions, not a multiple of the 16-position k-step, so the
    # last chunk is short; the output layer's bias as a second product over a 128 x 128 NCHW output gradient; the
    # residual W1 at 64 x 64 latents over n * B = 4 images
    "cfg3_input_k4s2_256": (0, 2, 3, 256, 256, 64, 4, 2, 1, NCHW, NHWC, True, 0),
    "short_last_chunk_3x7x9": (0, 3, 16, 7, 9, 32, 3, 1, 1, NHWC, NHWC, True, 0),
    "convt_k4s2_out_128_nchw_gout_bias": (1, 2, 64, 64, 64, 3, 4, 2, 1, NHWC, NCHW, True, 0),
    "residual_w1_64x64_4_images": (0, 4, 128, 64, 64, 32, 3, 1, 1, NHWC, NHWC, False, 0),
}


def out_size(case):
    transposed, _, _, H, W, _, k, s, p = case[:9]
    if transposed:
        return (H - 1) * s - 2 * p + k, (W - 1) * s - 2 * p + k
    return (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1


def inputs(case, seed=0):
    """The layer's input and output gradient, (B, C, H, W) float32 on the CPU."""
    _, B, Cin, H, W, Cout = case[:6]
    OH, OW = out_size(case)
    gen = torch.Generator().manual_seed(seed)
    return torch.randn((B, Cin, H, W), generator=gen), torch.randn((B, Cout, OH, OW), generator=gen)


def _device(t, layout, offset=0):
    """t on the GPU in `layout`, starting `offset` floats into a larger buffer."""
    t = t.permute(0, 2, 3, 1) if layout == NHWC else t
    buf = torch.zeros(t.numel() + offset, device="cuda")
    buf[offset:] = t.contiguous().reshape(-1).cuda()
    return buf[offset:]


def wgrad(case, x, g):
    """vqb_conv_wgrad_f32 on the case's layouts -> (dW, dbias or None) on the CPU."""
    from vqvae_b200 import ops
    from vqvae_b200._lib import check
    lib = ops.lib()
    transposed, B, Cin, H, W, Cout, k, s, p, in_layout, gout_layout, bias, offset = case
    geom = (B, Cin, H, W, Cout, k, k, s, p, transposed)
    n = lib.vqb_conv_wgrad_workspace_bytes(*geom)
    assert n > 0
    ws = torch.empty((n,), dtype=torch.uint8, device="cuda")
    dW = torch.full((Cin, Cout, k, k) if transposed else (Cout, Cin, k, k), float("nan"), device="cuda")
    db = torch.full((Cout,), float("nan"), device="cuda") if bias else None
    xc, gc = _device(x, in_layout, offset), _device(g, gout_layout)
    check(lib.vqb_conv_wgrad_f32(xc.data_ptr(), gc.data_ptr(), dW.data_ptr(), db.data_ptr() if bias else None, *geom,
                                 in_layout, gout_layout, ws.data_ptr(), n, torch.cuda.current_stream().cuda_stream),
          "conv_wgrad")
    torch.cuda.synchronize()
    return dW.cpu(), db.cpu() if bias else None


def _fp64(case, x, g):
    transposed, _, Cin, _, _, Cout, k, s, p = case[:9]
    w = torch.zeros((Cin, Cout, k, k) if transposed else (Cout, Cin, k, k), dtype=torch.float64, requires_grad=True)
    b = torch.zeros((Cout,), dtype=torch.float64, requires_grad=True)
    with torch.enable_grad():
        conv = F.conv_transpose2d if transposed else F.conv2d
        conv(x.double(), w, b, stride=s, padding=p).backward(g.double())
    return w.grad, b.grad


@pytest.mark.parametrize("name", list(CASES))
def test_conv_wgrad_matches_fp64(name):
    case = CASES[name]
    x, g = inputs(case)
    dW, db = wgrad(case, x, g)
    want_w, want_b = _fp64(case, x, g)
    assert float((dW.double() - want_w).abs().max() / want_w.abs().max()) <= 1e-5
    if case[11]:
        assert float((db.double() - want_b).abs().max() / want_b.abs().max()) <= 1e-5

"""CPU-only checks of vqb_decoder_tail_tf32's argument handling and of vqb_decoder_tail_supported: every answer here is
given before any CUDA call, so it runs without a GPU."""
import ctypes

import pytest

from vqvae_b200 import _lib


@pytest.mark.parametrize("Cin,H,W,C,Cout,ok", [
    (128, 8, 8, 64, 3, True),        # the decoder at cfg2
    (64, 8, 8, 64, 3, True),
    (32, 4, 4, 64, 1, True),
    (256, 8, 16, 64, 4, True),       # one image per 128-pixel tile
    (128, 16, 8, 64, 2, True),
    (128, 1, 1, 64, 3, True),
    (128, 8, 8, 64, 5, False),       # the output layer's scatter form takes at most 4 channels
    (128, 8, 8, 64, 0, False),
    (128, 8, 8, 128, 3, False),      # h of 128 channels does not fit in shared memory
    (128, 8, 8, 32, 3, False),
    (16, 8, 8, 64, 3, False),        # Cin % 32 != 0
    (288, 8, 8, 64, 3, False),       # more k-steps than the step table holds
    (128, 16, 16, 64, 3, False),     # two tiles per image
    (128, 8, 32, 64, 3, False),
])
def test_supported_shapes(Cin, H, W, C, Cout, ok):
    assert _lib.lib().vqb_decoder_tail_supported(Cin, H, W, C, Cout) == int(ok)


def test_arguments_are_checked_without_a_gpu():
    lib = _lib.lib()
    bufs = [(ctypes.c_float * 4)() for _ in range(2)]
    p, q = (ctypes.cast(b, ctypes.c_void_p) for b in bufs)

    def call(d=p, cw=p, ow=p, x_hat=q, B=4, Cin=128, H=8, W=8, C=64, Cout=3, relu=0, h_out=None):
        return lib.vqb_decoder_tail_tf32(d, cw, None, ow, None, h_out, x_hat, B, Cin, H, W, C, Cout, relu, None)

    assert call(d=None) == -1
    assert call(cw=None) == -1
    assert call(ow=None) == -1
    assert call(x_hat=None) == -1
    assert call(B=0) == -1
    assert call(Cout=-1) == -1
    assert call(relu=2) == -1
    assert call(Cout=5) == -2                      # unsupported: the caller runs the separate calls
    assert call(C=128) == -2
    assert call(H=16, W=16) == -2
    assert call(x_hat=p) == -2                     # d_out aliases x_hat: nothing is launched
    assert call(h_out=p) == -2                     # ... or h

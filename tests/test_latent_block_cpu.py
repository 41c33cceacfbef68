"""CPU-only checks of vqb_latent_block_tf32's argument handling and of vqb_latent_block_supported: every answer here is
given before any CUDA call, so it runs without a GPU."""
import ctypes

import pytest

from vqvae_b200 import _lib


@pytest.mark.parametrize("Cin,H,W,C,Cmid,tail_cout,ok", [
    (128, 8, 8, 128, 32, 64, True),      # the encoder's block at cfg2
    (64, 8, 8, 128, 32, 0, True),        # the decoder's
    (32, 8, 8, 128, 32, 0, True),
    (128, 8, 16, 128, 32, 64, True),     # one image per 128-pixel tile
    (128, 8, 8, 128, 32, 32, False),     # a tail of any other width
    (128, 8, 8, 128, 32, 128, False),
    (16, 8, 8, 128, 32, 0, False),       # Cin % 32 != 0
    (288, 8, 8, 128, 32, 0, False),      # more k-steps than the step table holds
    (128, 16, 16, 128, 32, 64, False),   # two tiles per image
    (128, 8, 8, 128, 64, 64, False),     # Cmid = 64 has no scatter form
    (128, 8, 8, 96, 32, 64, False),
])
def test_supported_shapes(Cin, H, W, C, Cmid, tail_cout, ok):
    assert _lib.lib().vqb_latent_block_supported(Cin, H, W, C, Cmid, tail_cout) == int(ok)


def test_arguments_are_checked_without_a_gpu():
    lib = _lib.lib()
    buf = (ctypes.c_float * 4)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    call = lambda tw, tcout, n=2, B=4, Cin=128: lib.vqb_latent_block_tf32(  # noqa: E731
        p, p, None, 0, p, p, n, tw, None, tcout, p, B, Cin, 8, 8, 128, 32, None)
    assert call(p, 0) == -1                        # a tail weight without its width
    assert call(None, 64) == -1                    # a width without the weight
    assert call(p, -64) == -1
    assert call(None, 0, n=0) == -1
    assert call(None, 0, B=0) == -1
    assert call(p, 32) == -2                       # a tail not 64 wide: unsupported, the caller runs the separate calls
    assert call(None, 0, Cin=16) == -2

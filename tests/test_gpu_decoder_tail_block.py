"""The decoder's last two layers in one launch (vqb_decoder_tail_tf32: wgconv_kernel in TAIL mode): the k4 s2 transposed
conv to 64 channels with its ReLU, and the output layer on the hidden activation kept in shared memory.  It must be
bitwise the separate launches, because the eval forward and the training walk both take it and the walk's outputs are
held equal to the layer-by-layer calls.  Needs an H100 (``-m gpu``).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHAPES = [
    # B, H, W (the latent): B odd or 1, so the last tile is partly past the batch
    (5, 8, 8),       # two images per tile, the model's shape
    (257, 8, 8),
    (3, 4, 4),       # eight images per tile
    (1, 5, 6),       # ragged images in 8 x 8 tile slots: padding rows and columns inside the tile
    (3, 6, 7),
    (5, 1, 1),       # 128 one-pixel images per tile
    (3, 8, 16),      # one image per tile, spanning both consumer warpgroups
    (1, 16, 8),
]


def _weights(seed, Cin, Cout, C=64):
    from vqvae_b200 import ops
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s, scale: (torch.randn(s, generator=g) * scale).cuda()  # noqa: E731
    return dict(cw=ops.pack_conv_weight(rnd(Cin, C, 4, 4, scale=1 / np.sqrt(4 * Cin)), True), cb=rnd(C, scale=0.1),
                ow=ops.pack_conv_weight(rnd(C, Cout, 4, 4, scale=1 / np.sqrt(4 * C)), True), ob=rnd(Cout, scale=0.1))


def _separate(d, cw, cb, ow, ob, B, Cin, H, W, Cout, relu_out, C=64):
    from vqvae_b200 import ops
    from vqvae_b200._lib import NCHW, TF32
    h = ops.conv2d(d, cw, cb, B=B, Cin=Cin, H=H, W=W, Cout=C, kh=4, kw=4, stride=2, pad=1, transposed=True, relu=True,
                   precision=TF32)
    x_hat = ops.conv2d(h, ow, ob, B=B, Cin=C, H=2 * H, W=2 * W, Cout=Cout, kh=4, kw=4, stride=2, pad=1, transposed=True,
                       out_layout=NCHW, relu=relu_out, precision=TF32)
    return x_hat, h


@pytest.mark.parametrize("keep_h", [False, True])
@pytest.mark.parametrize("relu_out", [False, True])
@pytest.mark.parametrize("Cout", [1, 2, 3, 4])
@pytest.mark.parametrize("Cin", [64, 128])
@pytest.mark.parametrize("B,H,W", SHAPES)
def test_decoder_tail_is_bitwise_the_separate_launches(B, H, W, Cin, Cout, relu_out, keep_h):
    from vqvae_b200 import ops
    w = _weights(B * 100 + H * 10 + W + Cin + Cout, Cin, Cout)
    d = torch.relu(torch.randn((B, H, W, Cin), generator=torch.Generator().manual_seed(Cout))).cuda()
    l0 = ops.launch_count()
    got = ops.decoder_tail(d, w["cw"], w["cb"], w["ow"], w["ob"], B=B, Cin=Cin, H=H, W=W, C=64, Cout=Cout,
                           relu_out=relu_out, keep_h=keep_h)
    assert got is not None and ops.launch_count() - l0 == 1
    x_hat, h = got
    ref_x_hat, ref_h = _separate(d, w["cw"], w["cb"], w["ow"], w["ob"], B, Cin, H, W, Cout, relu_out)
    assert x_hat.shape == ref_x_hat.shape and torch.equal(x_hat, ref_x_hat)
    if keep_h:
        assert torch.equal(h, ref_h)
    else:
        assert h is None


def test_decoder_tail_without_biases():
    from vqvae_b200 import ops
    w = _weights(3, 128, 3)
    d = torch.relu(torch.randn((5, 8, 8, 128), generator=torch.Generator().manual_seed(4))).cuda()
    x_hat, h = ops.decoder_tail(d, w["cw"], None, w["ow"], None, B=5, Cin=128, H=8, W=8, C=64, Cout=3, keep_h=True)
    ref_x_hat, ref_h = _separate(d, w["cw"], None, w["ow"], None, 5, 128, 8, 8, 3, False)
    assert torch.equal(x_hat, ref_x_hat) and torch.equal(h, ref_h)


def test_decoder_tail_declines_shapes_without_whole_image_tiles():
    from vqvae_b200 import ops
    w = _weights(1, 128, 3)
    d = torch.rand((2, 16, 16, 128), device="cuda")
    l0 = ops.launch_count()
    assert ops.decoder_tail(d, w["cw"], w["cb"], w["ow"], w["ob"], B=2, Cin=128, H=16, W=16, C=64, Cout=3) is None
    assert ops.launch_count() == l0


def test_decoder_tail_repeats_and_replays_bitwise():
    from vqvae_b200 import ops
    w = _weights(2, 128, 3)
    d = torch.relu(torch.randn((256, 8, 8, 128), generator=torch.Generator().manual_seed(5))).cuda()
    run = lambda: ops.decoder_tail(d, w["cw"], w["cb"], w["ow"], w["ob"], B=256, Cin=128, H=8, W=8, C=64,  # noqa: E731
                                   Cout=3, keep_h=True)
    a, b = run(), run()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c = run()
    g.replay()
    torch.cuda.synchronize()
    for u, v, t in zip(a, b, c):
        assert torch.equal(u, v) and torch.equal(u, t)


def _model(seed=0):
    from models.vqvae import VQVAE
    torch.manual_seed(seed)
    return VQVAE(128, 32, 2, 512, 64, 0.25).cuda().eval()


def _layer_by_layer(model, d_out, B, H, W):
    from vqvae_b200.modules import _bias, _pack_key, _packed
    ics = model.decoder.inverse_conv_stack
    c, o = ics[2], ics[4]
    return _separate(d_out, _packed(c.weight, _pack_key(c, False)), _bias(c), _packed(o.weight, _pack_key(o, False)),
                     _bias(o), B, c.in_channels, H, W, o.out_channels, False)


@pytest.mark.parametrize("B", [5, 256])
def test_vqvae_forwards_are_bitwise_the_layer_by_layer_tail(B, monkeypatch):
    """The eval forward and the training walk take the fused tail: their x_hat, and the walk's saved h, are the
    layer-by-layer calls' on the walk's own d_out.  The eval forward launches one kernel fewer than with the separate
    launches (7 on the main stream at cfg2 instead of 8)."""
    import vqvae_b200
    from vqvae_b200 import modules, ops
    model = _model()
    x = torch.rand((B, 3, 32, 32), generator=torch.Generator().manual_seed(B)).cuda()
    with vqvae_b200.precision("tf32"), torch.no_grad():
        model(x)                                     # packs the weights
        l0 = ops.launch_count()
        loss, x_hat, perp = model(x)
        l1 = ops.launch_count()
        acts = {}
        w_loss, w_x_hat, w_perp = model._walk(x, False, acts=acts)
        d1, d_out, h = acts["dec"]
        ref_x_hat, ref_h = _layer_by_layer(model, d_out, B, 8, 8)
        monkeypatch.setattr(modules, "_decoder_tail", lambda *a, **k: None)
        l2 = ops.launch_count()
        s_loss, s_x_hat, s_perp = model(x)
        l3 = ops.launch_count()
    torch.cuda.synchronize()
    assert (l3 - l2) - (l1 - l0) == 1
    assert torch.equal(w_x_hat, ref_x_hat) and torch.equal(h, ref_h)
    assert torch.equal(x_hat, w_x_hat) and torch.equal(x_hat, s_x_hat)
    assert torch.equal(loss, w_loss) and torch.equal(perp, w_perp) and torch.equal(loss, s_loss)


_PROFILE_SCRIPT = """
import json
import torch
from torch.profiler import ProfilerActivity, profile
import vqvae_b200
from models.vqvae import VQVAE
torch.manual_seed(0)
model = VQVAE(128, 32, 2, 512, 64, 0.25).cuda().eval()
x = torch.rand((4, 3, 32, 32), device="cuda")
with vqvae_b200.precision("tf32"), torch.no_grad():
    model(x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model(x)
        torch.cuda.synchronize()
print(json.dumps([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]))
"""


def test_profiler_shows_no_separate_output_layer_at_cfg2_shapes():
    """32 x 32 images: the output layer runs inside the decoder's wgconv_kernel launch, so no convt_scatter_kernel."""
    run = subprocess.run([sys.executable, "-c", _PROFILE_SCRIPT], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-3000:]
    names = json.loads(run.stdout.strip().splitlines()[-1])
    assert sum("convt_scatter_kernel" in n for n in names) == 0, names
    assert sum("wgconv_kernel" in n for n in names) == 2, names

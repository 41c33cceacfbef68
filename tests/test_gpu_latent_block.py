"""The latent block in one launch (vqb_latent_block_tf32: res_scatter_kernel with its head conv and 1x1 tail): the k3
conv that feeds a ResidualStack, the stack and the pre-quantization conv, computed per whole-image tile without leaving
shared memory between them.  It must be bitwise the separate launches, because the training walk keeps those and its
outputs are held equal to the eval forward's.  Which kernels a whole forward runs is read from the profiler in a fresh
interpreter.  Needs an H100 (``-m gpu``).
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
    # B, H, W, C: B odd, so the last tile is partly past the batch
    (5, 8, 8, 128),      # two images per tile, the model's shape
    (9, 4, 4, 64),       # eight images per tile
    (3, 5, 6, 64),       # ragged images in 8 x 8 tile slots: padding rows and columns inside the tile
    (3, 6, 7, 128),
    (131, 1, 1, 128),    # 128 one-pixel images per tile: every neighbour is padding
    (3, 8, 16, 128),     # one image per tile, spanning both consumer warpgroups
    (3, 16, 8, 64),
]


def _weights(seed, Cin, C, transposed, Cmid=32, D=64):
    from vqvae_b200 import ops
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s, scale: (torch.randn(s, generator=g) * scale).cuda()  # noqa: E731
    hw = rnd(*((Cin, C, 3, 3) if transposed else (C, Cin, 3, 3)), scale=1 / np.sqrt(9 * Cin))
    return dict(hw=ops.pack_conv_weight(hw, transposed), hb=rnd(C, scale=0.1),
                w1=ops.pack_conv_weight(rnd(Cmid, C, 3, 3, scale=1 / np.sqrt(9 * C)), False),
                w2=ops.pack_conv_weight(rnd(C, Cmid, 1, 1, scale=1 / np.sqrt(Cmid)), False),
                tw=ops.pack_conv_weight(rnd(D, C, 1, 1, scale=1 / np.sqrt(C)), False), tb=rnd(D, scale=0.1))


def _separate(x, w, B, Cin, H, W, C, n, transposed, tail):
    from vqvae_b200 import ops
    from vqvae_b200._lib import TF32
    h = ops.conv2d(x, w["hw"], w["hb"], B=B, Cin=Cin, H=H, W=W, Cout=C, kh=3, kw=3, stride=1, pad=1,
                   transposed=transposed, relu=True, precision=TF32)
    h = ops.residual_stack(h, w["w1"], w["w2"], B=B, H=H, W=W, C=C, Cmid=32, n_layers=n, precision=TF32)
    if tail:
        h = ops.conv2d(h, w["tw"], w["tb"], B=B, Cin=C, H=H, W=W, Cout=64, kh=1, kw=1, stride=1, pad=0, precision=TF32)
    return h


@pytest.mark.parametrize("tail", [False, True])
@pytest.mark.parametrize("n", [1, 2, 3, 4])
@pytest.mark.parametrize("Cin,transposed", [(128, False), (64, True), (64, False), (128, True)])
@pytest.mark.parametrize("B,H,W,C", SHAPES)
def test_latent_block_is_bitwise_the_separate_launches(B, H, W, C, Cin, transposed, n, tail):
    from vqvae_b200 import ops
    w = _weights(B * 100 + H * 10 + W + C + Cin + 7 * n, Cin, C, transposed)
    x = torch.relu(torch.randn((B, H, W, Cin), generator=torch.Generator().manual_seed(n))).cuda()
    l0 = ops.launch_count()
    y = ops.latent_block(x, w["hw"], w["hb"], w["w1"], w["w2"], w["tw"] if tail else None, w["tb"] if tail else None,
                         B=B, Cin=Cin, H=H, W=W, C=C, Cmid=32, n_layers=n, transposed=transposed,
                         tail_cout=64 if tail else 0)
    assert y is not None and ops.launch_count() - l0 == 1
    ref = _separate(x, w, B, Cin, H, W, C, n, transposed, tail)
    assert y.shape == ref.shape
    assert torch.equal(y, ref)


def test_latent_block_declines_shapes_without_whole_image_tiles():
    """16 x 16 latents need two tiles per image: nothing is launched and the caller runs the separate launches."""
    from vqvae_b200 import ops
    w = _weights(1, 128, 128, False)
    x = torch.rand((2, 16, 16, 128), device="cuda")
    l0 = ops.launch_count()
    assert ops.latent_block(x, w["hw"], w["hb"], w["w1"], w["w2"], w["tw"], w["tb"], B=2, Cin=128, H=16, W=16, C=128,
                            Cmid=32, n_layers=2, transposed=False, tail_cout=64) is None
    assert ops.launch_count() == l0


def _model(seed=0, D=64):
    from models.vqvae import VQVAE
    torch.manual_seed(seed)
    return VQVAE(128, 32, 2, 512, D, 0.25).cuda().eval()


@pytest.mark.parametrize("B,size,D,fewer", [
    (5, 32, 64, 3),
    (256, 32, 64, 3),
    (2, 64, 64, 0),      # 16 x 16 latents: no whole-image tiles
    (5, 32, 32, 1),      # a 1x1 conv to 32 channels is no tail: only the decoder's block (Cin = 32) is one launch
    (5, 32, 16, 0),      # and a decoder head with Cin = 16 is not a shape the gather launch takes on tensor cores
])
def test_vqvae_eval_forward_is_bitwise_the_separate_launches(B, size, D, fewer):
    """The eval forward against the walk that keeps every layer's launch (the one training uses): same loss, x_hat,
    perplexity and indices, with `fewer` launches fewer."""
    import vqvae_b200
    from vqvae_b200 import ops
    model = _model(D=D)
    x = torch.rand((B, 3, size, size), generator=torch.Generator().manual_seed(B)).cuda()
    with vqvae_b200.precision("tf32"), torch.no_grad():
        model(x)                                     # packs the weights
        l0 = ops.launch_count()
        loss, x_hat, perp = model(x)
        l1 = ops.launch_count()
        idx = model.last_min_encoding_indices.clone()
        ref_loss, ref_x_hat, ref_perp = model._walk(x, False, acts={})
        l2 = ops.launch_count()
        ref_idx = model.last_min_encoding_indices.clone()
    torch.cuda.synchronize()
    assert (l2 - l1) - (l1 - l0) == fewer
    assert torch.equal(loss, ref_loss) and torch.equal(perp, ref_perp)
    assert torch.equal(x_hat, ref_x_hat) and torch.equal(idx, ref_idx)


def test_vqvae_eval_forward_repeats_and_replays_bitwise():
    import vqvae_b200
    model = _model(1)
    x = torch.rand((256, 3, 32, 32), generator=torch.Generator().manual_seed(3)).cuda()
    with vqvae_b200.precision("tf32"), torch.no_grad():
        a, b = model(x), model(x)
        for u, v in zip(a, b):
            assert torch.equal(u, v)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            model(x)
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            c = model(x)
        g.replay()
        torch.cuda.synchronize()
    for u, v in zip(a, c):
        assert torch.equal(u, v)


_PROFILE_SCRIPT = """
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
import vqvae_b200
from models.vqvae import VQVAE
torch.manual_seed(0)
model = VQVAE(128, 32, 2, 512, 64, 0.25).cuda().eval()
out = []
for size in json.loads(sys.argv[1]):
    x = torch.rand((4, 3, size, size), device="cuda")
    with vqvae_b200.precision("tf32"), torch.no_grad():
        model(x)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            model(x)
            torch.cuda.synchronize()
    out.append([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA])
print(json.dumps(out))
"""


def test_profiler_shows_the_fused_launches_only_for_whole_image_latents():
    """32 x 32 images (8 x 8 latents): the two latent blocks are res_scatter_kernel launches and only the two k4 s2
    layers run wgconv_kernel.  64 x 64 images (16 x 16 latents): no res_scatter_kernel; the k3 convs, each stack
    application and the 1x1 conv run wgconv_kernel."""
    run = subprocess.run([sys.executable, "-c", _PROFILE_SCRIPT, json.dumps([32, 64])], cwd=ROOT, capture_output=True,
                         text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-3000:]
    small, big = json.loads(run.stdout.strip().splitlines()[-1])
    count = lambda names, k: sum(k in n for n in names)  # noqa: E731
    assert count(small, "res_scatter_kernel") == 2 and count(small, "wgconv_kernel") == 2, small
    assert count(big, "res_scatter_kernel") == 0 and count(big, "wgconv_kernel") == 2 + 3 + 2 * 2, big

"""The TF32 residual layer and stack in scatter form (res_scatter_kernel in wgconv.cu): whole-image tiles of 1 to 128
images, the tile loaded once and kept in shared memory across the applications of a stack, neighbour terms summed by
(image, row, column) with the out-of-image ones dropped.  Held to the C oracle at the TF32 bars of the existing
residual tests.  Which kernel every case ran is read from the profiler in a fresh interpreter, so the check does not
depend on what earlier tests did to the process's profiling state.  Needs an H100 (``-m gpu``).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import cref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _case(seed, B, H, W, C, Cmid=32):
    rng = np.random.RandomState(seed)
    r = np.maximum(rng.standard_normal((B, C, H, W)).astype(np.float32), 0)
    w1 = (rng.standard_normal((Cmid, C, 3, 3)) / np.sqrt(C * 9)).astype(np.float32)
    w2 = (rng.standard_normal((C, Cmid, 1, 1)) / np.sqrt(Cmid)).astype(np.float32)
    return r, w1, w2


def _ref(r, w1, w2, n, relu_out):
    """residual.py: n applications of one layer, every one but the last always ReLU'd."""
    y = r
    for i in range(n):
        y = y + cref.conv2d(np.maximum(cref.conv2d(y, w1, None, 1, 1), 0), w2, None, 1, 0)
        if relu_out or i + 1 < n:
            y = np.maximum(y, 0)
    return y


def _ops(r, w1, w2):
    from vqvae_b200 import ops
    return _cuda(r.transpose(0, 2, 3, 1)), ops.pack_conv_weight(_cuda(w1), False), ops.pack_conv_weight(_cuda(w2), False)


def _nchw(y):
    return y.cpu().numpy().transpose(0, 3, 1, 2)


SHAPES = [
    # B, H, W, C: B odd, so the last tile is partly past the batch
    (5, 8, 8, 128),      # two images per tile, the model's shape
    (9, 4, 4, 64),       # eight images per tile
    (3, 5, 6, 64),       # ragged images in 8 x 8 tile slots: padding rows and columns inside the tile
    (3, 6, 7, 128),
    (131, 1, 1, 128),    # 128 one-pixel images per tile: every neighbour is padding
]


@pytest.mark.parametrize("relu_out", [True, False])
@pytest.mark.parametrize("B,H,W,C", SHAPES)
def test_tf32_residual_layer_scatter_vs_oracle(B, H, W, C, relu_out):
    from vqvae_b200 import ops
    from vqvae_b200._lib import TF32
    r, w1, w2 = _case(B * 100 + H * 10 + W + C, B, H, W, C)
    rn, p1, p2 = _ops(r, w1, w2)
    l0 = ops.launch_count()
    y = ops.residual_layer(rn, p1, p2, B=B, H=H, W=W, C=C, Cmid=32, relu_out=relu_out, precision=TF32)
    assert ops.launch_count() - l0 == 1
    np.testing.assert_allclose(_nchw(y), _ref(r, w1, w2, 1, relu_out), atol=6e-3, rtol=2e-3)


@pytest.mark.parametrize("n", [1, 2, 3, 4])
@pytest.mark.parametrize("B,H,W,C", SHAPES)
def test_tf32_residual_stack_scatter_vs_oracle_and_layers(B, H, W, C, n):
    """One launch for the whole stack (bitwise the layers one by one), within n times the layer bar of the oracle."""
    from vqvae_b200 import ops
    from vqvae_b200._lib import TF32
    r, w1, w2 = _case(B * 100 + H * 10 + W + C + 7 * n, B, H, W, C)
    rn, p1, p2 = _ops(r, w1, w2)
    l0 = ops.launch_count()
    y = ops.residual_stack(rn, p1, p2, B=B, H=H, W=W, C=C, Cmid=32, n_layers=n, precision=TF32)
    assert ops.launch_count() - l0 == 1
    np.testing.assert_allclose(_nchw(y), _ref(r, w1, w2, n, True), atol=6e-3 * n, rtol=2e-3 * n)
    seq = rn
    for _ in range(n):
        seq = ops.residual_layer(seq, p1, p2, B=B, H=H, W=W, C=C, Cmid=32, relu_out=True, precision=TF32)
    assert torch.equal(y, seq)
    assert torch.equal(rn.cpu(), torch.from_numpy(np.ascontiguousarray(r.transpose(0, 2, 3, 1))))   # input untouched


def test_tf32_residual_stack_scatter_repeats_and_replays_bitwise():
    """Two calls, and a CUDA-graph replay, give the same bits: fixed tap order, no atomics."""
    from vqvae_b200 import ops
    from vqvae_b200._lib import TF32
    B, H, W, C, n = 256, 8, 8, 128, 2
    r, w1, w2 = _case(11, B, H, W, C)
    rn, p1, p2 = _ops(r, w1, w2)
    call = lambda: ops.residual_stack(rn, p1, p2, B=B, H=H, W=W, C=C, Cmid=32, n_layers=n, precision=TF32)  # noqa: E731
    y0, y1 = call(), call()
    assert torch.equal(y0, y1)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        yg = call()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(yg, y0)


def test_residual_layer_without_whole_image_tiles_vs_oracle():
    """16 x 16 images need two tiles per image: a stack runs one launch per application."""
    from vqvae_b200 import ops
    from vqvae_b200._lib import TF32
    B, H, W, C, n = 2, 16, 16, 128, 2
    r, w1, w2 = _case(3, B, H, W, C)
    rn, p1, p2 = _ops(r, w1, w2)
    y = ops.residual_layer(rn, p1, p2, B=B, H=H, W=W, C=C, Cmid=32, relu_out=True, precision=TF32)
    np.testing.assert_allclose(_nchw(y), _ref(r, w1, w2, 1, True), atol=6e-3, rtol=2e-3)
    l0 = ops.launch_count()
    y = ops.residual_stack(rn, p1, p2, B=B, H=H, W=W, C=C, Cmid=32, n_layers=n, precision=TF32)
    assert ops.launch_count() - l0 == n
    np.testing.assert_allclose(_nchw(y), _ref(r, w1, w2, n, True), atol=6e-3 * n, rtol=2e-3 * n)


_PROFILE_SCRIPT = """
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
from vqvae_b200 import ops
from vqvae_b200._lib import TF32
out = []
for B, H, W, C, n in json.loads(sys.argv[1]):
    r = torch.rand((B, H, W, C), device="cuda")
    p1 = ops.pack_conv_weight(torch.randn((32, C, 3, 3), device="cuda") * 0.05, False)
    p2 = ops.pack_conv_weight(torch.randn((C, 32, 1, 1), device="cuda") * 0.1, False)
    for layer in (True, False):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            if layer:
                ops.residual_layer(r, p1, p2, B=B, H=H, W=W, C=C, Cmid=32, relu_out=True, precision=TF32)
            else:
                ops.residual_stack(r, p1, p2, B=B, H=H, W=W, C=C, Cmid=32, n_layers=n, precision=TF32)
            torch.cuda.synchronize()
        out.append([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA])
print(json.dumps(out))
"""


def test_profiler_shows_which_kernel_each_shape_runs():
    """From torch.profiler: every whole-image shape above runs res_scatter_kernel, once per layer and once per stack;
    16 x 16 images run wgconv_kernel, once per application."""
    cases = [[B, H, W, C, 3] for B, H, W, C in SHAPES] + [[2, 16, 16, 128, 2]]
    run = subprocess.run([sys.executable, "-c", _PROFILE_SCRIPT, json.dumps(cases)], cwd=ROOT, capture_output=True,
                         text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-3000:]
    names = json.loads(run.stdout.strip().splitlines()[-1])
    for i, case in enumerate(cases):
        for k, what in enumerate(("layer", "stack")):
            got = names[2 * i + k]
            scatter = [x for x in got if "res_scatter_kernel" in x]
            gather = [x for x in got if "wgconv_kernel" in x]
            if case[1] == 16:
                assert not scatter and len(gather) == (1 if what == "layer" else case[4]), (case, what, got)
            else:
                assert len(scatter) == 1 and not gather, (case, what, got)

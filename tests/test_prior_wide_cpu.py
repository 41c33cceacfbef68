"""The Gated PixelCNN prior at dims above 256 (up to 1024, the reference script's dim = img_dim**2 for 24x24 and 32x32
latents), without a GPU: the C ABI takes every dim % 32 == 0 up to 1024 and refuses the rest before any launch; the
workspace and saved-activation queries are their documented formulas at those dims, in 64-bit arithmetic; the module
built as the reference script builds it has the reference's state-dict keys and shapes; and the wide goldens come
from the reference with the seeded weights."""
import contextlib
import ctypes
import io
import json
import os

import numpy as np
import pytest
import torch

from oracle.make_prior_wide_golden import PRIOR_WIDE_CASES
from oracle.prior_port import make_prior_inputs, make_prior_state_dict, prior_forward, prior_shapes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAD, UNSUP, WS = -1, -2, -3


def _lib():
    from vqvae_b200 import _lib
    return _lib, _lib.lib()


def _net(_lib, p, dim, L=2, K=16):
    lw = _lib.PriorLayerWeights(*([p.value] * 9), 3, 0, 1)
    layers = (_lib.PriorLayerWeights * L)(*([lw] * L))
    net = _lib.PriorNet(layers=layers, n_layers=L, embedding=p.value, out1_w=p.value, out1_b=p.value, out2_w=p.value,
                        out2_b=p.value, input_dim=K, dim=dim, n_classes=2)
    return net, layers


@pytest.mark.parametrize("dim", [288, 576, 1024, 40, 48, 1056])
def test_c_abi_takes_wide_dims_and_refuses_the_rest(dim):
    """An accepted dim gets past every shape check to the next argument check (a short workspace: -3, or a missing
    pointer: -1); a refused one returns VQB_ERR_UNSUPPORTED, so nothing is launched."""
    _l, lib = _lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    ok = dim % 32 == 0 and dim <= 1024
    net, _keep = _net(_l, p, dim)
    n = ctypes.byref(net)
    want = WS if ok else UNSUP
    assert lib.vqb_prior_forward_f32(n, p, p, 1, 4, 4, p, p, 4, None) == want
    assert lib.vqb_prior_forward_tf32(n, p, p, 1, 4, 4, p, p, 4, None) == want
    assert lib.vqb_prior_forward_train_f32(n, p, p, 1, 4, 4, p, p, 4, None) == want
    assert lib.vqb_prior_generate_f32(n, p, p, 1, 4, 4, p, None, p, 4, None) == want
    assert lib.vqb_prior_log_prob_f32(n, p, p, 0, 1, 4, 4, p, None, p, 4, None) == want
    assert lib.vqb_prior_ce_forward_f32(n, p, p, 1, 4, 4, 1, p, None, 0, p, 4, None) == want
    assert lib.vqb_prior_ce_forward_tf32(n, p, p, 1, 4, 4, 1, p, None, 0, p, 4, None) == want
    assert (lib.vqb_prior_backward_workspace_bytes(n, 1, 4, 4) > 0) == ok
    assert (lib.vqb_prior_ce_backward_workspace_bytes(n, 1, 4, 4) > 0) == ok
    lw = _l.PriorLayerWeights(*([p.value] * 9), 3, 0, 1)
    assert lib.vqb_prior_layer_f32(ctypes.byref(lw), p, p, None, 1, 4, 4, dim, 2, p, p, p, None) == BAD
    if not ok:                                      # an accepted dim would launch: not called with fake pointers
        assert lib.vqb_prior_layer_f32(ctypes.byref(lw), p, p, p, 1, 4, 4, dim, 2, p, p, p, None) == UNSUP
    assert (lib.vqb_prior_layer_backward_wide_workspace_bytes(ctypes.byref(lw), 1, 4, 4, dim, 2) > 0) == ok
    # the ABI-3 single-layer backward pair keeps the dim <= 256 it was published with
    assert lib.vqb_prior_layer_backward_workspace_bytes(ctypes.byref(lw), 1, 4, 4, dim, 2) == 0


def _gen_floats(B, H, W, C, L, K):
    ring = min(H, 15 // 2 + 1)
    return B * H * W * C + L * B * W * 2 * C + L * B * W * C + B * K + L * B * ring * W * C


@pytest.mark.parametrize("shape", [(2, 6, 6, 576, 3, 512), (3, 4, 4, 1024, 2, 512), (32, 32, 32, 1024, 15, 512),
                                   (16, 24, 24, 576, 15, 512), (1, 1, 1, 288, 1, 1)])
def test_workspace_and_saved_bytes_are_their_formulas_at_wide_dims(shape):
    """In Python integers, so a 32-bit product anywhere in the library shows as a mismatch.  At B=32 on 32x32 with
    15 layers and dim = 1024, the saved activations are (6L + 3)*N*dim + 512*N floats, about 12.5 GB."""
    _l, lib = _lib()
    B, H, W, C, L, K = shape
    N = B * H * W
    fwd = max(7 * N * C, _gen_floats(B, H, W, C, L, K))
    assert lib.vqb_prior_workspace_bytes(*shape) == 4 * fwd
    comp = _gen_floats(B, H, W, C, L, K) - L * B * min(H, 8) * W * C + L * N * C
    assert lib.vqb_prior_complete_workspace_bytes(*shape) == 4 * max(fwd, comp)
    assert lib.vqb_prior_log_prob_workspace_bytes(*shape) == 4 * fwd + 12 * N
    saved = (6 * L + 3) * N * C + 512 * N
    assert lib.vqb_prior_train_saved_bytes(B, H, W, C, L) == 4 * saved
    assert lib.vqb_prior_ce_saved_bytes(B, H, W, C, L) == 4 * saved + 8 * N
    assert lib.vqb_prior_workspace_bytes_tf32(*shape) == 4 * (11 * N * C + 512 * N)
    assert lib.vqb_prior_layer_train_saved_bytes(B, H, W, C) == 16 * N * C
    search = B * 64 * ((K + 31) // 32) + B
    assert lib.vqb_prior_sample_workspace_bytes(*shape, 0) == max(4 * fwd, 4 * (_gen_floats(B, H, W, C, L, K) + search))
    if shape[:5] == (32, 32, 32, 1024, 15):
        assert 12.4e9 < lib.vqb_prior_train_saved_bytes(B, H, W, C, L) < 12.6e9


def test_backward_workspace_grows_linearly_in_positions_at_dim_1024():
    """The backward's workspace at dim = 1024 is activation grids plus weight-gradient partials whose chunk count
    grows with the positions; doubling B at least doubles the grids and never wraps."""
    _l, lib = _lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    net, _keep = _net(_l, p, 1024, L=15, K=512)
    n = ctypes.byref(net)
    for q in (lib.vqb_prior_backward_workspace_bytes, lib.vqb_prior_ce_backward_workspace_bytes):
        a, b, c = q(n, 16, 32, 32), q(n, 32, 32, 32), q(n, 64, 32, 32)
        assert 0 < a < b < c and b - a >= 6 * 16 * 1024 * 1024 * 4 and c - b >= 2 * (b - a) - 4
        assert c > 2 ** 32                          # more than a 32-bit size can hold


def test_module_matches_the_reference_state_dict_at_dim_1024():
    """GatedPixelCNN(512, 32**2, 2), as gated_pixelcnn.py builds it for --img_dim 32."""
    from pixelcnn.models import GatedPixelCNN
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(512, 1024, 2)
    got = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    assert got == [(k, tuple(s)) for k, s in prior_shapes(512, 1024, 2, 10)]
    assert m.layers[0].vert_stack.weight.shape == (2048, 1024, 4, 7)
    assert (m.layers[0].mask_type, m.layers[0].residual, m.layers[1].mask_type) == ("A", False, "B")


@pytest.mark.parametrize("name", list(PRIOR_WIDE_CASES))
def test_port_reproduces_the_wide_goldens(name):
    """The fp64 restatement at the goldens' seeded weights and inputs matches the reference's logits, and the
    fixture records the case it was made from."""
    c = PRIOR_WIDE_CASES[name]
    with np.load(os.path.join(ROOT, "tests", "golden", name + ".npz")) as d:
        assert json.loads(str(d["case"])) == c
        gold = torch.from_numpy(d["logits"])
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"])
    codes, labels, _ = make_prior_inputs(c)
    want = prior_forward(sd, codes, labels, c["n_layers"], torch.float64)
    assert gold.shape == (c["batch"], c["K"], c["size"], c["size"])
    err = float((gold.double() - want).abs().max() / want.abs().max())
    assert err <= 2e-5, err


def test_wide_single_layer_backward_validates_arguments_without_a_gpu():
    """vqb_prior_layer_backward_wide_*: the ABI-3 single-layer backward's argument checks in the same order and the
    same workspace, with dims up to 1024 accepted (288 here, which the ABI-3 pair refuses) and 1056 refused."""
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p).value
    lw = _lib.PriorLayerWeights(*([p] * 9), 3, 0, 1)
    ok = ctypes.byref(lw)
    wsb, old_wsb = lib.vqb_prior_layer_backward_wide_workspace_bytes, lib.vqb_prior_layer_backward_workspace_bytes
    assert wsb(None, 1, 4, 4, 32, 2) == 0
    assert wsb(ok, 1, 0, 4, 32, 2) == 0
    assert wsb(ok, 1, 4, 4, 1056, 2) == 0 and wsb(ok, 1, 4, 4, 40, 2) == 0
    for dim in (32, 160, 256):
        assert wsb(ok, 2, 5, 5, dim, 3) == old_wsb(ok, 2, 5, 5, dim, 3) > 0
    assert old_wsb(ok, 1, 4, 4, 288, 2) == 0
    ws = wsb(ok, 1, 4, 4, 288, 2)
    assert ws > 4 * 6 * 16 * 288
    lg = _lib.PriorLayerGrads(*([p] * 9))
    g = ctypes.byref(lg)
    bwd, old = lib.vqb_prior_layer_backward_wide_f32, lib.vqb_prior_layer_backward_f32
    assert bwd(ok, p, p, p, 1, 4, 4, 288, 2, p, None, p, g, p, p, p, ws, None) == -1          # d_out_h
    assert bwd(ok, p, p, p, 1, 4, 4, 288, 2, p, p, None, g, p, p, p, ws, None) == -1          # saved
    assert bwd(ok, p, p, p, 1, 4, 4, 288, 2, p, p, p, None, p, p, p, ws, None) == -1          # grads
    assert bwd(ok, p, p, p, 1, 4, 4, 288, 2, p, p, p, ctypes.byref(_lib.PriorLayerGrads(*([p] * 8), None)), p, p, p,
               ws, None) == -1
    assert bwd(ok, p, p, p, 1, 4, 4, 288, 2, p, p, p, g, None, p, p, ws, None) == -1          # d_x_v
    assert bwd(ok, p, p, p, 1, 4, 4, 288, 2, p, p, p, g, p, p, None, ws, None) == -1          # workspace
    assert bwd(ok, p, p, p, 1, 4, 4, 288, 0, p, p, p, g, p, p, p, ws, None) == -1
    assert bwd(ok, p, p, p, 1, 4, 4, 1056, 2, p, p, p, g, p, p, p, ws, None) == -2
    assert bwd(ok, p, p, p, 1, 4, 4, 288, 2, p, p, p, g, p, p, p, ws - 4, None) == -3
    assert old(ok, p, p, p, 1, 4, 4, 288, 2, p, p, p, g, p, p, p, ws, None) == -2

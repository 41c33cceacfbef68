"""GatedPixelCNN.complete without a GPU: its signature, the checks that run before any CUDA call, and the C ABI's
argument checks for vqb_prior_complete_f32 and its workspace query."""
import contextlib
import ctypes
import inspect
import io

import pytest
import torch


def _model(first="A"):
    from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(37, 32, 2, 3)
    if first != "A":
        m.layers[0] = GatedMaskedConv2d("B", 32, 7, False, 3)
    return m


def test_complete_signature():
    from pixelcnn.models import GatedPixelCNN
    assert list(inspect.signature(GatedPixelCNN.complete).parameters) == ["self", "x", "label", "n_given"]
    assert list(inspect.signature(GatedPixelCNN._complete).parameters) == \
        ["self", "label", "u", "x", "n_given", "step_logits"]


@pytest.mark.parametrize("n_given", [-1, 26, 2**40])
def test_out_of_range_n_given_raises_value_error_before_the_cuda_check(n_given):
    m = _model()
    x, lab = torch.zeros((2, 5, 5), dtype=torch.int64), torch.zeros(2, dtype=torch.int64)
    with pytest.raises(ValueError, match="n_given"):
        m.complete(x, lab, n_given)
    with pytest.raises(ValueError, match="n_given"):
        m._complete(lab, torch.zeros((2, 5, 5)), x, n_given)


@pytest.mark.parametrize("n_given", [2.0, 3.5, "3", None])
def test_non_integer_n_given_is_refused(n_given):
    m = _model()
    with pytest.raises((TypeError, ValueError)):
        m.complete(torch.zeros((2, 5, 5), dtype=torch.int64), torch.zeros(2, dtype=torch.int64), n_given)


@pytest.mark.parametrize("n_given", [0, 1, 12, 25])
def test_valid_n_given_on_cpu_tensors_raises_the_cuda_error(n_given):
    m = _model()
    x, lab = torch.zeros((2, 5, 5), dtype=torch.int64), torch.zeros(2, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.complete(x, lab, n_given)
    with pytest.raises(RuntimeError, match="CUDA"):
        m._complete(lab, torch.zeros((2, 5, 5)), x, n_given)


def test_complete_refuses_what_generate_refuses():
    m = _model()
    lab = torch.zeros(2, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="square"):
        m.complete(torch.zeros((2, 6, 8), dtype=torch.int64), lab, 3)
    with pytest.raises(RuntimeError, match="square"):
        m.generate(lab, shape=(6, 8), batch_size=2)
    with pytest.raises(RuntimeError, match="shape"):
        m.complete(torch.zeros((5, 5), dtype=torch.int64), lab, 3)
    with pytest.raises(RuntimeError, match="shape"):
        m.complete(torch.zeros((1, 2, 5, 5), dtype=torch.int64), lab, 3)
    with pytest.raises(RuntimeError, match="expected 2 labels, got 3"):
        m.complete(torch.zeros((2, 5, 5), dtype=torch.int64), torch.zeros(3, dtype=torch.int64), 3)
    with pytest.raises(RuntimeError, match="expected 2 labels, got 1"):
        m.complete(torch.zeros((2, 5, 5), dtype=torch.int64), [0], 3)
    b = _model("B")
    with pytest.raises(RuntimeError, match="mask A without residual"):
        b.complete(torch.zeros((2, 5, 5), dtype=torch.int64), lab, 3)
    with pytest.raises(RuntimeError, match="mask A without residual"):
        b._sample(lab, torch.zeros((2, 5, 5)))


def test_complete_entry_points_validate_arguments_without_a_gpu():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    q = lib.vqb_prior_complete_workspace_bytes
    for bad in ((0, 4, 4, 32, 2, 16), (1, 0, 4, 32, 2, 16), (1, 4, -1, 32, 2, 16), (1, 4, 4, 0, 2, 16),
                (1, 4, 4, 32, 0, 16), (1, 4, 4, 32, 2, 0)):
        assert q(*bad) == 0
    for shape in ((1, 4, 4, 32, 2, 16), (100, 8, 8, 64, 15, 512), (16, 64, 64, 64, 15, 1024), (3, 1, 1, 32, 1, 8192),
                  (2, 48, 48, 32, 2, 512)):
        B, H, W, dim, L, K = shape
        assert q(*shape) >= lib.vqb_prior_workspace_bytes(*shape)
        assert q(*shape) >= 4 * L * B * H * W * dim                 # every layer's vertical output, whole grids
    lw = _lib.PriorLayerWeights(*([p.value] * 9), 7, 1, 0)
    layers = (_lib.PriorLayerWeights * 2)(lw, lw)
    net = _lib.PriorNet(layers=layers, n_layers=2, embedding=p.value, out1_w=p.value, out1_b=p.value, out2_w=p.value,
                        out2_b=p.value, input_dim=16, dim=32, n_classes=2)
    ws, ws_gen = q(1, 4, 4, 32, 2, 16), lib.vqb_prior_workspace_bytes(1, 4, 4, 32, 2, 16)
    comp = lib.vqb_prior_complete_f32
    n = ctypes.byref(net)
    assert comp(n, p, p, None, 5, 1, 4, 4, p, None, p, ws, None) == -1              # null given
    assert comp(n, None, p, p, 5, 1, 4, 4, p, None, p, ws, None) == -1
    assert comp(n, p, p, p, 5, 1, 4, 4, None, None, p, ws, None) == -1
    assert comp(n, p, p, p, 5, 1, 4, 4, p, None, None, ws, None) == -1
    assert comp(None, p, p, p, 5, 1, 4, 4, p, None, p, ws, None) == -1
    assert comp(n, p, p, p, 5, 0, 4, 4, p, None, p, ws, None) == -1
    assert comp(n, p, p, p, -1, 1, 4, 4, p, None, p, ws, None) == -1
    assert comp(n, p, p, p, 17, 1, 4, 4, p, None, p, ws, None) == -1
    assert comp(n, p, p, p, 2**40, 1, 4, 4, p, None, p, ws, None) == -1
    assert comp(n, p, p, p, 5, 1, 4, 4, p, None, p, ws - 4, None) == -3            # short workspace
    assert comp(n, p, p, p, 16, 1, 4, 4, p, None, p, ws - 4, None) == -3
    assert comp(n, p, p, p, 3, 1, 4, 4, p, None, p, ws_gen - 4, None) == -3        # shorter than a row: generate's
    assert comp(ctypes.byref(_lib.PriorNet(layers=layers, n_layers=2, embedding=p.value, out1_w=p.value,
                                           out1_b=p.value, out2_w=p.value, out2_b=p.value, input_dim=16, dim=40,
                                           n_classes=2)), p, p, p, 5, 1, 4, 4, p, None, p, ws, None) == -2
    mask_b = _lib.PriorLayerWeights(*([p.value] * 9), 7, 0, 0)
    resid = _lib.PriorLayerWeights(*([p.value] * 9), 7, 1, 1)
    for first in (mask_b, resid):                                                   # refused before any launch
        ls = (_lib.PriorLayerWeights * 2)(first, lw)
        bad = _lib.PriorNet(layers=ls, n_layers=2, embedding=p.value, out1_w=p.value, out1_b=p.value, out2_w=p.value,
                            out2_b=p.value, input_dim=16, dim=32, n_classes=2)
        assert comp(ctypes.byref(bad), p, p, p, 5, 1, 4, 4, p, None, p, ws, None) == -2

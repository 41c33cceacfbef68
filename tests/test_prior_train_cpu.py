"""CPU checks of the trainable Gated PixelCNN prior: the differentiable restatement against the reference's gradient
goldens (mask A's taps included), argument checks of the training entry points, and the CUDA-only rule in grad mode."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle.prior_port import PRIOR_CASES, make_prior_inputs, make_prior_state_dict
from oracle.prior_train_port import fingerprint, leaf_params, prior_logits, prior_loss

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden(name):
    with np.load(os.path.join(ROOT, "tests", "golden", name + ".npz")) as d:
        return {k: d[k] for k in d.files}


def _grads(name):
    c = PRIOR_CASES[name]
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"])
    codes, labels, _ = make_prior_inputs(c)
    threads = torch.get_num_threads()
    torch.set_num_threads(1)            # the goldens were made single-threaded
    try:
        with torch.enable_grad():
            g = leaf_params(sd)
            x = torch.from_numpy(codes)
            loss = prior_loss(prior_logits(g, x, torch.from_numpy(labels), c["n_layers"]), x)
            loss.backward()
    finally:
        torch.set_num_threads(threads)
    return c, list(sd), loss.item(), {k: v.grad.numpy() for k, v in g.items()}


def test_restatement_reproduces_the_reference_gradients_in_full():
    c, keys, loss, grads = _grads("prior_ragged")
    want = _golden("prior_grad_ragged")
    assert json.loads(str(want["case"])) == c
    assert abs(loss - float(want["loss"])) <= 1e-6 * abs(float(want["loss"]))
    assert sorted(k[5:] for k in want if k.startswith("grad/")) == sorted(keys)
    for k in keys:
        w = want["grad/" + k]
        assert grads[k].shape == w.shape, k
        np.testing.assert_allclose(grads[k], w, atol=1e-5 * np.abs(w).max(), rtol=0, err_msg=k)


def test_restatement_reproduces_the_reference_gradient_fingerprints():
    c, keys, loss, grads = _grads("prior_default")
    want = _golden("prior_grad_default")
    assert json.loads(str(want["case"])) == c
    assert abs(loss - float(want["loss"])) <= 1e-6 * abs(float(want["loss"]))
    for i, k in enumerate(keys):
        w = want["grad/" + k]
        got = fingerprint(grads[k], i)
        # each value is a sum over the tensor; 1e-5 of its max |g| per element, scaled by the L2 norm of the probe
        tol = 1e-5 * np.abs(grads[k]).max() * np.sqrt(grads[k].size)
        np.testing.assert_allclose(got, w, atol=tol, rtol=0, err_msg=k)


def test_reference_gives_mask_a_taps_a_gradient():
    want = _golden("prior_grad_ragged")
    assert np.abs(want["grad/layers.0.vert_stack.weight"][:, :, -1]).max() > 1e-4
    assert np.abs(want["grad/layers.0.horiz_stack.weight"][:, :, :, -1]).max() > 1e-4


def test_training_entry_points_validate_arguments_without_a_gpu():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.vqb_prior_train_saved_bytes(0, 8, 8, 64, 15) == 0
    assert lib.vqb_prior_train_saved_bytes(4, 8, 8, 64, 0) == 0
    assert lib.vqb_prior_train_saved_bytes(4, 8, 8, 64, 15) == 4 * 4 * 8 * 8 * (64 * (6 * 15 + 3) + 512)
    lw = _lib.PriorLayerWeights(*([p.value] * 9), 3, 0, 1)
    layers = (_lib.PriorLayerWeights * 2)(lw, lw)

    def net(**kw):
        a = dict(layers=layers, n_layers=2, embedding=p.value, out1_w=p.value, out1_b=p.value, out2_w=p.value,
                 out2_b=p.value, input_dim=16, dim=32, n_classes=2)
        a.update(kw)
        return _lib.PriorNet(**a)

    sv = lib.vqb_prior_train_saved_bytes(1, 4, 4, 32, 2)
    fwd = lib.vqb_prior_forward_train_f32
    assert fwd(None, p, p, 1, 4, 4, p, p, sv, None) == -1
    assert fwd(ctypes.byref(net()), None, p, 1, 4, 4, p, p, sv, None) == -1
    assert fwd(ctypes.byref(net()), p, p, 1, 4, 4, p, None, sv, None) == -1
    assert fwd(ctypes.byref(net()), p, p, 0, 4, 4, p, p, sv, None) == -1
    assert fwd(ctypes.byref(net()), p, p, 1, 4, 4, p, p, sv - 4, None) == -3
    assert fwd(ctypes.byref(net(dim=40)), p, p, 1, 4, 4, p, p, sv, None) == -2
    assert fwd(ctypes.byref(net(input_dim=8193)), p, p, 1, 4, 4, p, p, sv, None) == -2

    wsb = lib.vqb_prior_backward_workspace_bytes
    assert wsb(None, 1, 4, 4) == 0
    assert wsb(ctypes.byref(net()), 0, 4, 4) == 0
    assert wsb(ctypes.byref(net(dim=40)), 1, 4, 4) == 0
    ws = wsb(ctypes.byref(net()), 1, 4, 4)
    assert ws > 0
    lg = _lib.PriorLayerGrads(*([p.value] * 9))
    glayers = (_lib.PriorLayerGrads * 2)(lg, lg)

    def grads(**kw):
        a = dict(layers=glayers, n_layers=2, embedding=p.value, out1_w=p.value, out1_b=p.value, out2_w=p.value,
                 out2_b=p.value)
        a.update(kw)
        return _lib.PriorGrads(**a)

    bwd = lib.vqb_prior_backward_f32
    ok = ctypes.byref(grads())
    assert bwd(None, p, p, 1, 4, 4, p, p, ok, p, ws, None) == -1
    assert bwd(ctypes.byref(net()), p, p, 1, 4, 4, None, p, ok, p, ws, None) == -1          # d_logits
    assert bwd(ctypes.byref(net()), p, p, 1, 4, 4, p, None, ok, p, ws, None) == -1          # saved
    assert bwd(ctypes.byref(net()), p, p, 1, 4, 0, p, p, ok, p, ws, None) == -1
    assert bwd(ctypes.byref(net()), p, p, 1, 4, 4, p, p, None, p, ws, None) == -1
    assert bwd(ctypes.byref(net()), p, p, 1, 4, 4, p, p, ctypes.byref(grads(n_layers=1)), p, ws, None) == -1
    assert bwd(ctypes.byref(net()), p, p, 1, 4, 4, p, p, ctypes.byref(grads(out2_b=None)), p, ws, None) == -1
    bad = (_lib.PriorLayerGrads * 2)(lg, _lib.PriorLayerGrads(*([p.value] * 8), None))
    assert bwd(ctypes.byref(net()), p, p, 1, 4, 4, p, p, ctypes.byref(grads(layers=bad)), p, ws, None) == -1
    assert bwd(ctypes.byref(net()), p, p, 1, 4, 4, p, p, ok, p, ws - 4, None) == -3
    assert bwd(ctypes.byref(net(dim=300)), p, p, 1, 4, 4, p, p, ok, p, ws, None) == -2
    assert bwd(ctypes.byref(net(n_layers=33)), p, p, 1, 4, 4, p, p, ok, p, ws, None) == -2


def test_grad_mode_still_rejects_cpu_tensors():
    from pixelcnn.models import GatedPixelCNN
    m = GatedPixelCNN(37, 32, 2, 3)
    with torch.enable_grad():
        assert torch.is_grad_enabled() and all(p.requires_grad for p in m.parameters())
        with pytest.raises(RuntimeError, match="CUDA"):
            m(torch.zeros((2, 5, 5), dtype=torch.int64), torch.zeros(2, dtype=torch.int64))

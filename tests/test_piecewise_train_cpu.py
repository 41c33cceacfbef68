"""CPU checks of training through the sub-modules: the torch restatements the GPU tests use against the reference's
piecewise gradients (tests/golden/piecewise_grad.npz), the differentiability rule of every module, CPU tensors refused
before any launch, and the argument checks of the single-layer prior entry points."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle.piecewise_port import (GATE, GATED, PRIOR_LAYER_KEYS, RES, gate, gate_inputs, gated_inputs, gated_layer,
                                   res_inputs, residual_layer, residual_stack)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden():
    with np.load(os.path.join(ROOT, "tests", "golden", "piecewise_grad.npz")) as d:
        return {k: d[k] for k in d.files}


def _close(got, want, what):
    np.testing.assert_allclose(got, want, atol=1e-5 * max(np.abs(want).max(), 1e-30), rtol=0, err_msg=what)


def test_restatements_reproduce_the_reference_piecewise_gradients():
    want = _golden()
    assert json.loads(str(want["case"])) == dict(res=RES, gated=GATED, gate=GATE)
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        with torch.enable_grad():
            r = {k: torch.from_numpy(v) for k, v in res_inputs().items()}
            for n in [None] + RES["stacks"]:
                name = "layer" if n is None else f"stack{n}"
                w1, w2 = r["w1"].clone().requires_grad_(), r["w2"].clone().requires_grad_()
                x0 = r["x"].clone().requires_grad_()
                y = residual_layer(x0, w1, w2) if n is None else residual_stack(x0, [(w1, w2)] * n)
                (y * r["g/" + name]).sum().backward()
                _close(x0.grad.numpy(), want[f"res/{name}/dx"], name)
                after = torch.relu(r["x"]) if n != 0 else r["x"]        # Q2: the caller's tensor is ReLU'd in place
                assert np.array_equal(after.numpy(), want[f"res/{name}/x_after"]), name
                if n != 0:
                    _close(w1.grad.numpy(), want[f"res/{name}/dw1"], name + " w1")
                    _close(w2.grad.numpy(), want[f"res/{name}/dw2"], name + " w2")
            for name, mask, k, residual in GATED["layers"]:
                d = gated_inputs(name)
                p = {key: torch.from_numpy(d[key]).requires_grad_() for key in PRIOR_LAYER_KEYS}
                xv, xh = (torch.from_numpy(d[key]).requires_grad_() for key in ("x_v", "x_h"))
                ov, oh = gated_layer(p, xv, xh, torch.from_numpy(d["label"]), mask, k, residual)
                ((ov * torch.from_numpy(d["g_v"])).sum() + (oh * torch.from_numpy(d["g_h"])).sum()).backward()
                _close(xv.grad.numpy(), want[f"gated/{name}/dx_v"], name + " x_v")
                _close(xh.grad.numpy(), want[f"gated/{name}/dx_h"], name + " x_h")
                for key in PRIOR_LAYER_KEYS:
                    _close(p[key].grad.numpy(), want[f"gated/{name}/d/{key}"], f"{name} {key}")
                if mask == "A":
                    assert np.abs(want[f"gated/{name}/d/vert_stack.weight"][:, :, -1]).max() > 1e-4
            gi = gate_inputs()
            x = torch.from_numpy(gi["x"]).requires_grad_()
            (gate(x) * torch.from_numpy(gi["g"])).sum().backward()
            _close(x.grad.numpy(), want["gate/dx"], "gate")
    finally:
        torch.set_num_threads(threads)


def _vqvae_modules():
    from models.vqvae import VQVAE
    m = VQVAE(32, 8, 2, 16, 8, 0.25)
    return [m.encoder, m.decoder, m.encoder.conv_stack[5], m.encoder.conv_stack[5].stack[0], m.pre_quantization_conv]


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("grad", [True, False])
@pytest.mark.parametrize("what", ["nothing", "input", "params", "both"])
def test_vqvae_family_rule(training, grad, what):
    from vqvae_b200.modules import _trains
    for mod in _vqvae_modules():
        mod.train(training)
        for p in mod.parameters():
            p.requires_grad_(what in ("params", "both"))
        x = torch.zeros(1, requires_grad=what in ("input", "both"))
        with torch.set_grad_enabled(grad):
            assert _trains(mod, x) == (training and grad and what != "nothing"), type(mod).__name__


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("grad", [True, False])
@pytest.mark.parametrize("what", ["nothing", "x_v", "x_h", "params"])
def test_prior_family_rule(training, grad, what):
    from pixelcnn.models import GatedMaskedConv2d
    from vqvae_b200.prior import _grad_call
    layer = GatedMaskedConv2d("B", 32, 3).train(training)
    for p in layer.parameters():
        p.requires_grad_(what == "params")
    x_v, x_h = torch.zeros(1, requires_grad=what == "x_v"), torch.zeros(1, requires_grad=what == "x_h")
    with torch.set_grad_enabled(grad):
        assert _grad_call([x_v, x_h], layer) == (grad and what != "nothing")      # the mode plays no part
        assert _grad_call([x_v]) == (grad and what == "x_v")                      # GatedActivation: x only


def test_cpu_tensors_raise_before_any_launch():
    from pixelcnn.models import GatedActivation, GatedMaskedConv2d
    from vqvae_b200 import ops
    enc, dec, stack, layer, pq = _vqvae_modules()
    n0 = ops.launch_count()
    with torch.enable_grad():
        for mod, ch in ((enc, 3), (dec, 8), (stack, 32), (layer, 32), (pq, 32)):
            mod.train()
            x = torch.randn((1, ch, 8, 8)) * 1
            before = x.clone()
            with pytest.raises(RuntimeError, match="CUDA"):
                mod(x)
            assert torch.equal(x, before), type(mod).__name__      # the in-place ReLU did not run either
        x = torch.randn((1, 64, 4, 4), requires_grad=True)
        with pytest.raises(RuntimeError, match="CUDA"):
            GatedMaskedConv2d("A", 64, 7)(x, x, torch.zeros(1, dtype=torch.int64))
        with pytest.raises(RuntimeError, match="CUDA"):
            GatedActivation()(x)
    assert ops.launch_count() == n0


def test_training_an_encoder_needs_sides_divisible_by_4():
    """Q11 for the differentiable Encoder call: refused before any launch (and before the CUDA check), where the
    inference call takes any size; relu_backward refuses operands of different sizes."""
    from vqvae_b200 import ops
    enc = _vqvae_modules()[0].train()
    n0 = ops.launch_count()
    with torch.enable_grad():
        for hw in ((30, 32), (32, 30), (18, 18)):
            with pytest.raises(RuntimeError, match="divisible by 4"):
                enc(torch.zeros((1, 3) + hw))
    assert ops.launch_count() == n0
    with pytest.raises(RuntimeError, match="differ in size"):
        ops.relu_backward(torch.zeros(4), torch.zeros(5))


def test_single_layer_prior_entry_points_validate_arguments_without_a_gpu():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p).value
    assert lib.vqb_prior_gate_backward_f32(None, p, p, 1, 4, 4, None) == -1
    assert lib.vqb_prior_gate_backward_f32(p, p, None, 1, 4, 4, None) == -1
    assert lib.vqb_prior_gate_backward_f32(p, p, p, 1, 0, 4, None) == -1

    assert lib.vqb_prior_layer_train_saved_bytes(2, 5, 5, 32) == 4 * 4 * 2 * 5 * 5 * 32
    assert lib.vqb_prior_layer_train_saved_bytes(0, 5, 5, 32) == 0
    lw = _lib.PriorLayerWeights(*([p] * 9), 3, 0, 1)
    bad_k = _lib.PriorLayerWeights(*([p] * 9), 4, 0, 1)
    sv = lib.vqb_prior_layer_train_saved_bytes(1, 4, 4, 32)
    fwd = lib.vqb_prior_layer_forward_train_f32
    ok = ctypes.byref(lw)
    assert fwd(None, p, p, p, 1, 4, 4, 32, 2, p, p, p, p, sv, None) == -1
    assert fwd(ok, p, p, None, 1, 4, 4, 32, 2, p, p, p, p, sv, None) == -1                    # labels
    assert fwd(ok, p, p, p, 1, 4, 4, 32, 2, p, p, None, p, sv, None) == -1                 # vh scratch
    assert fwd(ok, p, p, p, 1, 4, 4, 32, 2, p, p, p, None, sv, None) == -1                 # saved
    assert fwd(ctypes.byref(bad_k), p, p, p, 1, 4, 4, 32, 2, p, p, p, p, sv, None) == -1      # even kernel
    assert fwd(ok, p, p, p, 1, 4, 4, 32, 0, p, p, p, p, sv, None) == -1
    assert fwd(ok, p, p, p, 1, 4, 4, 40, 2, p, p, p, p, sv, None) == -2                       # dim % 32
    assert fwd(ok, p, p, p, 1, 4, 4, 32, 2, p, p, p, p, sv - 4, None) == -3

    wsb = lib.vqb_prior_layer_backward_workspace_bytes
    assert wsb(None, 1, 4, 4, 32, 2) == 0
    assert wsb(ok, 1, 4, 4, 288, 2) == 0
    assert wsb(ok, 1, 0, 4, 32, 2) == 0
    ws = wsb(ok, 1, 4, 4, 32, 2)
    assert ws > 4 * 6 * 16 * 32
    lg = _lib.PriorLayerGrads(*([p] * 9))
    g = ctypes.byref(lg)
    bwd = lib.vqb_prior_layer_backward_f32
    assert bwd(ok, p, p, p, 1, 4, 4, 32, 2, p, None, p, g, p, p, p, ws, None) == -1           # d_out_h
    assert bwd(ok, p, p, p, 1, 4, 4, 32, 2, p, p, None, g, p, p, p, ws, None) == -1           # saved
    assert bwd(ok, p, p, p, 1, 4, 4, 32, 2, p, p, p, None, p, p, p, ws, None) == -1           # grads
    assert bwd(ok, p, p, p, 1, 4, 4, 32, 2, p, p, p, ctypes.byref(_lib.PriorLayerGrads(*([p] * 8), None)), p, p, p,
               ws, None) == -1
    assert bwd(ok, p, p, p, 1, 4, 4, 32, 2, p, p, p, g, None, p, p, ws, None) == -1           # d_x_v
    assert bwd(ok, p, p, p, 1, 4, 4, 32, 2, p, p, p, g, p, p, None, ws, None) == -1           # workspace
    assert bwd(ok, p, p, p, 1, 4, 4, 32, 0, p, p, p, g, p, p, p, ws, None) == -1
    assert bwd(ok, p, p, p, 1, 4, 4, 288, 2, p, p, p, g, p, p, p, ws, None) == -2
    assert bwd(ok, p, p, p, 1, 4, 4, 32, 2, p, p, p, g, p, p, p, ws - 4, None) == -3


def test_signature_table_has_the_single_layer_entry_points():
    from vqvae_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vqvae_b200.h")).read()
    for name in ("vqb_prior_gate_backward_f32", "vqb_prior_layer_train_saved_bytes", "vqb_prior_layer_forward_train_f32",
                 "vqb_prior_layer_backward_workspace_bytes", "vqb_prior_layer_backward_f32"):
        assert name in _lib.SIGNATURES and name + "(" in src

"""CPU checks of the Gated PixelCNN prior over its documented shape range: the per-layer restatement against the
reference's goldens for a stack of every kernel path, causality of such stacks, and the rules that keep a model the
kernels cannot run from reaching them (layers that do not match the model, a layer 0 the sampler cannot run)."""
import contextlib
import ctypes
import io
import json
import os

import numpy as np
import pytest
import torch

from oracle.prior_port import (PRIOR_SHAPE_CASES, make_prior_inputs, make_prior_state_dict, prior_forward,
                               prior_shapes, reference_layers)
from oracle.prior_train_port import fingerprint, leaf_params, prior_logits, prior_loss

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden(name):
    with np.load(os.path.join(ROOT, "tests", "golden", name + ".npz")) as d:
        return {k: d[k] for k in d.files}


def _case(name):
    c = PRIOR_SHAPE_CASES[name]
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], c["layers"])
    codes, labels, _ = make_prior_inputs(c)
    return c, sd, codes, labels


@contextlib.contextmanager
def _one_thread():                      # the goldens were made single-threaded: the same oneDNN blocking
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        yield
    finally:
        torch.set_num_threads(threads)


def _model(c):
    """GatedPixelCNN of a case with layers[i] replaced by GatedMaskedConv2d(mask, dim, kernel, residual, n_classes)."""
    from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
    for i, (mask, k, residual) in enumerate(c["layers"]):
        m.layers[i] = GatedMaskedConv2d(mask, c["dim"], k, residual, c["n_classes"])
    return m


def test_layer_stack_restatement_reproduces_reference_logits():
    c, sd, codes, labels = _case("kernels")
    g = _golden("prior_layers")
    assert json.loads(str(g["case"])) == c
    with _one_thread():
        got = prior_forward(sd, codes, labels, c["n_layers"], layers=c["layers"]).numpy()
    assert got.shape == g["logits"].shape
    np.testing.assert_allclose(got, g["logits"], atol=1e-6, rtol=0)


def test_layer_stack_restatement_reproduces_reference_gradients():
    """Every mask-A layer's taps get a gradient in the reference (it masks in place, then convolves the full weight)."""
    c, sd, codes, labels = _case("kernels")
    want = _golden("prior_grad_layers")
    assert json.loads(str(want["case"])) == c
    with _one_thread(), torch.enable_grad():
        g = leaf_params(sd)
        x = torch.from_numpy(codes)
        loss = prior_loss(prior_logits(g, x, torch.from_numpy(labels), c["n_layers"], c["layers"]), x)
        loss.backward()
    assert abs(loss.item() - float(want["loss"])) <= 1e-6 * abs(float(want["loss"]))
    keys = list(sd)
    full = {k[5:] for k in want if k.startswith("grad/")}
    printed = {k[12:] for k in want if k.startswith("fingerprint/")}
    assert full | printed == set(keys) and not full & printed and len(printed) == 2
    for i, k in enumerate(keys):
        got = g[k].grad.numpy()
        if k in full:
            w = want["grad/" + k]
            assert got.shape == w.shape, k
            np.testing.assert_allclose(got, w, atol=1e-5 * np.abs(w).max(), rtol=0, err_msg=k)
        else:
            # each value is a sum over the tensor: 1e-5 of its max |g| per element, scaled by the probe's L2 norm
            tol = 1e-5 * np.abs(got).max() * np.sqrt(got.size)
            np.testing.assert_allclose(fingerprint(got, i), want["fingerprint/" + k], atol=tol, rtol=0, err_msg=k)
    for i, (mask, k, _) in enumerate(c["layers"]):
        if mask == "A":
            assert np.abs(g[f"layers.{i}.vert_stack.weight"].grad.numpy()[:, :, -1]).max() > 0, i


def test_default_stack_is_the_reference_stack():
    for n in (1, 2, 15):
        assert prior_shapes(37, 32, n, 3) == prior_shapes(37, 32, n, 3, reference_layers(n))
    sd = make_prior_state_dict(37, 32, 4, 3, 32)
    codes = np.random.RandomState(0).randint(0, 37, size=(2, 5, 5))
    labels = np.array([0, 2])
    want = prior_forward(sd, codes, labels, 4, layers=reference_layers(4))
    assert torch.equal(prior_forward(sd, codes, labels, 4), want)


@pytest.mark.parametrize("name", list(PRIOR_SHAPE_CASES))
def test_shape_case_state_dicts_fit_the_module(name):
    c = PRIOR_SHAPE_CASES[name]
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], c["layers"])
    m = _model(c)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [(k, v.shape) for k, v in sd.items()]
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    m._check_layers()


def _causal(c, sd, codes, labels):
    """True when the logits at every (i, j) are unchanged by redrawing every code at or after (i, j)."""
    S = c["size"]
    base = prior_forward(sd, codes, labels, c["n_layers"], layers=c["layers"])
    rng = np.random.RandomState(7)
    for i in range(S):
        for j in range(S):
            x = codes.copy().reshape(c["batch"], -1)
            x[:, i * S + j:] = rng.randint(0, c["K"], size=x[:, i * S + j:].shape)
            got = prior_forward(sd, x.reshape(codes.shape), labels, c["n_layers"], layers=c["layers"])
            if not torch.equal(got[:, :, i, j], base[:, :, i, j]):
                return False
    return True


def test_layer_stacks_are_causal_only_with_a_plain_mask_a_first_layer():
    """The sampler's premise holds for any stack whose layer 0 is mask A without residual, whatever comes after; a
    mask-B or residual layer 0 reads the code at (i, j) itself, so generate refuses those."""
    c, sd, codes, labels = _case("kernels")
    assert _causal(c, sd, codes, labels)
    for first in (["B", 3, False], ["A", 3, True]):
        c2 = dict(c, layers=[first] + c["layers"][1:])
        sd2 = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], c2["layers"])
        assert not _causal(c2, sd2, codes, labels), first


def test_generate_refuses_a_layer_0_that_reads_the_code_being_drawn():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    ws = lib.vqb_prior_workspace_bytes(1, 4, 4, 32, 2, 16)
    for mask_a, residual in ((0, 0), (0, 1), (1, 1)):
        first = _lib.PriorLayerWeights(*([p.value] * 9), 3, mask_a, residual)
        rest = _lib.PriorLayerWeights(*([p.value] * 9), 3, 0, 1)
        layers = (_lib.PriorLayerWeights * 2)(first, rest)
        net = _lib.PriorNet(layers=layers, n_layers=2, embedding=p.value, out1_w=p.value, out1_b=p.value,
                            out2_w=p.value, out2_b=p.value, input_dim=16, dim=32, n_classes=2)
        n0 = lib.vqb_launch_count()
        assert lib.vqb_prior_generate_f32(ctypes.byref(net), p, p, 1, 4, 4, p, None, p, ws, None) == -2
        assert lib.vqb_launch_count() == n0
    from pixelcnn.models import GatedMaskedConv2d
    c = PRIOR_SHAPE_CASES["narrow"]
    for first in (["B", 3, True], ["A", 7, True]):
        m = _model(dict(c, layers=[first] + c["layers"][1:]))
        with pytest.raises(RuntimeError, match="layer 0 must be mask A without residual"):
            m._sample(torch.zeros(2, dtype=torch.int64), torch.rand((2, 4, 4)))
    m.layers[0] = GatedMaskedConv2d("A", c["dim"], 3, False, c["n_classes"])
    with pytest.raises(RuntimeError, match="CUDA"):
        m._sample(torch.zeros(2, dtype=torch.int64), torch.rand((2, 4, 4)))


def test_sampler_workspace_keeps_eight_vertical_rows_per_layer():
    """Sampler region: x0 grid + L layers x min(H, 8) rows of dim + L rows of 2*dim + L rows of dim + B*K logits."""
    from vqvae_b200 import _lib
    lib = _lib.lib()
    for B, H, C, L, K in ((100, 8, 64, 15, 512), (3, 5, 32, 7, 37), (2, 64, 32, 32, 8192)):
        gen = B * H * H * C + L * B * min(H, 8) * H * C + L * B * H * 2 * C + L * B * H * C + B * K
        assert lib.vqb_prior_workspace_bytes(B, H, H, C, L, K) == 4 * max(7 * B * H * H * C, gen), (B, H)


def test_net_rejects_layers_that_do_not_match_the_model():
    from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(37, 32, 3, 3)
    keep = []
    for bad, what in ((GatedMaskedConv2d("B", 64, 3, True, 3), "64 channels"),
                      (GatedMaskedConv2d("B", 32, 3, True, 4), "4 classes"),
                      (GatedMaskedConv2d("B", 32, 3, True, 2), "2 classes"),
                      (GatedMaskedConv2d("B", 32, 17, True, 3), "kernel 17")):
        m.layers[1] = bad
        with pytest.raises(RuntimeError, match=what):
            m._net(keep)
        assert keep == []               # refused before anything was packed
    m.layers[1] = GatedMaskedConv2d("A", 32, 15, False, 3)
    m._check_layers()

"""CPU checks of the Gated PixelCNN prior: the torch restatement against the reference's goldens, the causality the
incremental sampler relies on, the drop-in module tree and init, and argument checks of the C ABI."""
import contextlib
import ctypes
import inspect
import io
import json
import os

import numpy as np
import pytest
import torch

from oracle.prior_port import PRIOR_CASES, make_prior_inputs, make_prior_state_dict, prior_forward

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(name):
    c = PRIOR_CASES[name]
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"])
    codes, labels, pos = make_prior_inputs(c)
    return c, sd, codes, labels, pos


def _golden(name):
    with np.load(os.path.join(ROOT, "tests", "golden", name + ".npz")) as d:
        return {k: d[k] for k in d.files}


@pytest.mark.parametrize("name", list(PRIOR_CASES))
def test_port_reproduces_reference_logits(name):
    c, sd, codes, labels, pos = _case(name)
    g = _golden(name)
    assert json.loads(str(g["case"])) == c
    threads = torch.get_num_threads()
    torch.set_num_threads(1)            # the goldens were made single-threaded: the same oneDNN blocking
    try:
        got = prior_forward(sd, codes, labels, c["n_layers"]).numpy()
    finally:
        torch.set_num_threads(threads)
    if pos is not None:
        got, want = got[:, :, pos[:, 0], pos[:, 1]], g["logits_at"]
    else:
        want = g["logits"]
    assert got.shape == want.shape
    np.testing.assert_allclose(got, want, atol=1e-6, rtol=0)


@pytest.mark.parametrize("name", ["prior_default", "prior_ragged"])
def test_logits_are_causal_in_raster_order(name):
    """The premise of the incremental sampler: logits at (i, j) do not depend on codes at or after (i, j)."""
    c, sd, codes, labels, _ = _case(name)
    S = c["size"]
    base = prior_forward(sd, codes, labels, c["n_layers"])
    rng = np.random.RandomState(7)
    for i in range(S):
        for j in range(S):
            x = codes.copy().reshape(c["batch"], -1)
            x[:, i * S + j:] = rng.randint(0, c["K"], size=x[:, i * S + j:].shape)
            got = prior_forward(sd, x.reshape(codes.shape), labels, c["n_layers"])
            assert torch.equal(got[:, :, i, j], base[:, :, i, j]), (i, j)


def test_module_tree_signatures_and_init_match_the_reference():
    from pixelcnn.models import GatedActivation, GatedMaskedConv2d, GatedPixelCNN  # noqa: F401
    import vqvae_b200
    assert vqvae_b200.GatedPixelCNN is GatedPixelCNN
    assert str(inspect.signature(GatedPixelCNN.__init__)) == "(self, input_dim=256, dim=64, n_layers=15, n_classes=10)"
    assert str(inspect.signature(GatedMaskedConv2d.__init__)) == "(self, mask_type, dim, kernel, residual=True, n_classes=10)"
    assert list(inspect.signature(GatedPixelCNN.generate).parameters) == ["self", "label", "shape", "batch_size"]
    assert list(inspect.signature(GatedMaskedConv2d.forward).parameters) == ["self", "x_v", "x_h", "h"]
    with open(os.path.join(ROOT, "tests", "golden", "prior_init_fingerprint.json")) as f:
        fp = json.load(f)
    for name, want in fp.items():
        c = PRIOR_CASES[name]
        torch.manual_seed(0)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
        assert buf.getvalue() == "Skipping initialization of  GatedMaskedConv2d\n" * c["n_layers"]
        sd = m.state_dict()
        assert [k for k, *_ in want] == list(sd.keys())
        import hashlib
        for k, shape, total, digest in want:
            assert list(sd[k].shape) == shape, k
            assert hashlib.sha256(sd[k].contiguous().numpy().tobytes()).hexdigest() == digest, k
        m1 = m.layers[1]
        assert (m.layers[0].mask_type, m.layers[0].residual, m1.mask_type, m1.residual) == ("A", False, "B", True)
        assert m.layers[0].vert_stack.kernel_size == (4, 7) and m1.horiz_stack.kernel_size == (1, 2)


def test_prior_port_state_dict_layout_matches_the_module():
    from pixelcnn.models import GatedPixelCNN
    c = PRIOR_CASES["prior_ragged"]
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"])
    m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [(k, v.shape) for k, v in sd.items()]
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})


def test_prior_entry_points_validate_arguments_without_a_gpu():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.vqb_prior_pack_f32(None, p, 4, 4, 1, 1, 1, 1, None) == -1
    assert lib.vqb_prior_pack_f32(p, p, 4, 4, 2, 3, 3, 3, None) == -1                 # more rows kept than exist
    assert lib.vqb_prior_workspace_bytes(0, 8, 8, 64, 15, 512) == 0
    assert lib.vqb_prior_workspace_bytes(4, 8, 8, 64, 15, 512) > 0
    assert lib.vqb_prior_gate_f32(None, p, 1, 4, 1, None) == -1
    assert lib.vqb_prior_gate_f32(p, p, 1, 0, 1, None) == -1
    lw = _lib.PriorLayerWeights(*([p.value] * 9), 3, 0, 1)
    assert lib.vqb_prior_layer_f32(ctypes.byref(lw), p, p, None, 1, 4, 4, 32, 2, p, p, p, None) == -1
    assert lib.vqb_prior_layer_f32(ctypes.byref(lw), p, p, p, 1, 4, 4, 48, 2, p, p, p, None) == -2   # dim % 32
    bad = _lib.PriorLayerWeights(*([p.value] * 9), 4, 0, 1)                                         # even kernel
    assert lib.vqb_prior_layer_f32(ctypes.byref(bad), p, p, p, 1, 4, 4, 32, 2, p, p, p, None) == -1
    layers = (_lib.PriorLayerWeights * 2)(lw, lw)

    def net(**kw):
        a = dict(layers=layers, n_layers=2, embedding=p.value, out1_w=p.value, out1_b=p.value, out2_w=p.value,
                 out2_b=p.value, input_dim=16, dim=32, n_classes=2)
        a.update(kw)
        return _lib.PriorNet(**a)

    ws = lib.vqb_prior_workspace_bytes(1, 4, 4, 32, 2, 16)
    fwd, gen = lib.vqb_prior_forward_f32, lib.vqb_prior_generate_f32
    assert fwd(None, p, p, 1, 4, 4, p, p, ws, None) == -1
    assert fwd(ctypes.byref(net()), None, p, 1, 4, 4, p, p, ws, None) == -1
    assert fwd(ctypes.byref(net()), p, p, 0, 4, 4, p, p, ws, None) == -1
    assert fwd(ctypes.byref(net()), p, p, 1, 4, 4, p, p, ws - 4, None) == -3
    assert fwd(ctypes.byref(net(dim=300)), p, p, 1, 4, 4, p, p, ws, None) == -2
    assert fwd(ctypes.byref(net(dim=40)), p, p, 1, 4, 4, p, p, ws, None) == -2
    assert fwd(ctypes.byref(net(input_dim=8193)), p, p, 1, 4, 4, p, p, ws, None) == -2
    assert fwd(ctypes.byref(net(n_layers=33)), p, p, 1, 4, 4, p, p, ws, None) == -2
    assert fwd(ctypes.byref(net(embedding=None)), p, p, 1, 4, 4, p, p, ws, None) == -1
    assert gen(ctypes.byref(net()), p, None, 1, 4, 4, p, None, p, ws, None) == -1
    assert gen(ctypes.byref(net()), p, p, 1, 4, 4, p, None, p, ws - 4, None) == -3
    assert gen(ctypes.byref(net(n_classes=0)), p, p, 1, 4, 4, p, None, p, ws, None) == -1


def test_prior_modules_reject_cpu_tensors_and_non_square_grids():
    from pixelcnn.models import GatedActivation, GatedMaskedConv2d, GatedPixelCNN
    m = GatedPixelCNN(37, 32, 2, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros((2, 5, 5), dtype=torch.int64), torch.zeros(2, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="square"):
        m(torch.zeros((2, 6, 8), dtype=torch.int64), torch.zeros(2, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="square"):
        m.generate(torch.zeros(2, dtype=torch.int64), shape=(8, 6), batch_size=2)
    with pytest.raises(RuntimeError, match="CUDA"):
        GatedActivation()(torch.zeros((1, 4, 2, 2)))
    layer = GatedMaskedConv2d("B", 32, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        layer(torch.zeros((1, 32, 4, 4)), torch.zeros((1, 32, 4, 4)), torch.zeros(1, dtype=torch.int64))
    with pytest.raises(AssertionError):
        GatedMaskedConv2d("B", 32, 4)


def test_prior_product_never_imports_the_oracle_or_the_tests():
    import re
    paths = [os.path.join(ROOT, "vqvae_b200", "prior.py")]
    for root, _, files in os.walk(os.path.join(ROOT, "pixelcnn")):
        paths += [os.path.join(root, f) for f in files if f.endswith(".py")]
    assert len(paths) >= 3
    for path in paths:
        src = open(path).read()
        assert not re.search(r"^\s*(from|import)\s+(oracle|tests)\b", src, flags=re.M), path

"""GatedPixelCNN.cross_entropy without a GPU: signature and docstring, the checks that run before any CUDA call and
their order, the C ABI's argument checks for vqb_prior_ce_*, the header against the _lib prototypes, the workspace
arithmetic (no term grows with B*H*W*K), and an fp64 restatement of the head's d_logits on hand-made logits."""
import contextlib
import ctypes
import inspect
import io
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
X, LAB = torch.zeros((2, 5, 5), dtype=torch.int64), torch.zeros(2, dtype=torch.int64)


def _model(precision="fp32"):
    from pixelcnn.models import GatedPixelCNN
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(37, 32, 2, 3)
    m.precision = precision
    return m


def test_signature_and_docstring():
    from pixelcnn.models import GatedPixelCNN
    s = inspect.signature(GatedPixelCNN.cross_entropy)
    assert list(s.parameters) == ["self", "x", "label", "reduction"]
    assert s.parameters["reduction"].kind is inspect.Parameter.KEYWORD_ONLY
    assert s.parameters["reduction"].default == "mean"
    doc = " ".join(GatedPixelCNN.cross_entropy.__doc__.split())
    for phrase in ("nn.CrossEntropyLoss(reduction=reduction)", "bitwise -log_prob(x, label, per_position=True)",
                   "clamped", "Differentiable", "CUDA graph", "second backward"):
        assert phrase in doc, phrase
    assert "cross_entropy() is that training loss" in " ".join(GatedPixelCNN.log_prob.__doc__.split())


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("reduction", ["none", "mean", "sum"])
def test_valid_arguments_on_cpu_tensors_raise_the_cuda_error(precision, reduction):
    for grad in (False, True):
        with torch.set_grad_enabled(grad), pytest.raises(RuntimeError, match="CUDA"):
            _model(precision).cross_entropy(X, LAB, reduction=reduction)


def test_errors_and_their_order():
    from pixelcnn.models import GatedMaskedConv2d
    m = _model()
    m.precision = "bf16"                                        # the precision first
    with pytest.raises(ValueError, match="precision"):
        m.cross_entropy(torch.zeros((5, 5), dtype=torch.int64), LAB, reduction="batchmean")
    m.precision = "fp32"
    for bad in ("batchmean", "Mean", None, 1, ("mean",)):      # then the reduction, before the rank
        with pytest.raises(ValueError, match="reduction"):
            m.cross_entropy(torch.zeros((5, 5), dtype=torch.int64), LAB, reduction=bad)
    with pytest.raises(RuntimeError, match="shape"):           # the rank, before the square check
        m.cross_entropy(torch.zeros((5, 5), dtype=torch.int64), LAB)
    with pytest.raises(RuntimeError, match="square"):          # square, before the layers and the label count
        m.cross_entropy(torch.zeros((2, 6, 8), dtype=torch.int64), torch.zeros(3, dtype=torch.int64))
    m.layers[1] = GatedMaskedConv2d("B", 64, 3, True, 3)       # P5, before the label count
    with pytest.raises(RuntimeError, match="layer 1 has 64 channels"):
        m.cross_entropy(X, torch.zeros(3, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="expected 2 labels, got 3"):
        _model().cross_entropy(X, torch.zeros(3, dtype=torch.int64))
    m = _model()
    m.layers[0] = GatedMaskedConv2d("B", 32, 7, True, 3)       # any layer 0 is taken: the CUDA check is reached
    with pytest.raises(RuntimeError, match="CUDA"):
        m.cross_entropy(X, LAB)


def _header_text():
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "vqvae_b200.h")).read(), flags=re.S)


_CTYPES = {"int": "_i", "int64_t": "_i64", "size_t": "_sz"}


def test_header_declarations_match_the_lib_prototypes():
    from vqvae_b200 import _lib
    src = " ".join(_header_text().split())
    names = ["vqb_prior_ce_saved_bytes", "vqb_prior_ce_workspace_bytes", "vqb_prior_ce_workspace_bytes_tf32",
             "vqb_prior_ce_forward_f32", "vqb_prior_ce_forward_tf32", "vqb_prior_ce_backward_workspace_bytes",
             "vqb_prior_ce_backward_f32", "vqb_prior_ce_backward_tf32"]
    lib = _lib.lib()
    for name in names:
        m = re.search(r"(\w+) " + name + r"\(([^)]*)\);", src)
        assert m, name
        ret, args = m.group(1), [a.strip() for a in m.group(2).split(",")]
        restype, argtypes = _lib.SIGNATURES[name]
        assert restype is getattr(_lib, _CTYPES[ret]), name
        want = [getattr(_lib, "_vp") if "*" in a else getattr(_lib, _CTYPES[a.rsplit(" ", 1)[0]]) for a in args]
        assert argtypes == want, name
        assert hasattr(lib, name)
    for v, k in ((0, "NONE"), (1, "MEAN"), (2, "SUM")):
        assert f"#define VQB_PRIOR_CE_{k} {v}" in src
    assert lib.vqb_abi_version() == 3
    doc = " ".join(open(os.path.join(ROOT, "include", "vqvae_b200.h")).read().split())
    assert "fp32 3 + 2*n_layers, TF32 4 + 4*n_layers, one more for MEAN and SUM" in doc
    assert "5 + 10*n_layers + 3*ceil(B*H*W / 4096)" in doc


def _net(p, dim=32, K=16, L=2):
    from vqvae_b200 import _lib
    lw = _lib.PriorLayerWeights(*([p.value] * 9), 7, 1, 0)
    layers = (_lib.PriorLayerWeights * L)(*([lw] + [_lib.PriorLayerWeights(*([p.value] * 9), 3, 0, 1)] * (L - 1)))
    net = _lib.PriorNet(layers=layers, n_layers=L, embedding=p.value, out1_w=p.value, out1_b=p.value,
                        out2_w=p.value, out2_b=p.value, input_dim=K, dim=dim, n_classes=2)
    return net, layers


def _grads(p, L=2):
    from vqvae_b200 import _lib
    lg = (_lib.PriorLayerGrads * L)(*([_lib.PriorLayerGrads(*([p.value] * 9))] * L))
    return _lib.PriorGrads(layers=ctypes.cast(lg, ctypes.POINTER(_lib.PriorLayerGrads)), n_layers=L,
                           embedding=p.value, out1_w=p.value, out1_b=p.value, out2_w=p.value, out2_b=p.value), lg


BAD, UNSUP, WS = -1, -2, -3


@pytest.mark.parametrize("sfx", ["f32", "tf32"])
def test_forward_entry_points_validate_arguments_without_a_gpu(sfx):
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    f = getattr(lib, "vqb_prior_ce_forward_" + sfx)
    q = getattr(lib, "vqb_prior_ce_workspace_bytes" + ("_tf32" if sfx == "tf32" else ""))
    net, _l = _net(p)
    n = ctypes.byref(net)
    sv, ws, ws_inf = lib.vqb_prior_ce_saved_bytes(1, 4, 4, 32, 2), q(1, 4, 4, 32, 2, 16, 1), q(1, 4, 4, 32, 2, 16, 0)
    assert f(None, p, p, 1, 4, 4, 1, p, p, sv, p, ws, None) == BAD
    assert f(n, None, p, 1, 4, 4, 1, p, p, sv, p, ws, None) == BAD
    assert f(n, p, None, 1, 4, 4, 1, p, p, sv, p, ws, None) == BAD
    assert f(n, p, p, 1, 4, 4, 1, None, p, sv, p, ws, None) == BAD        # no loss
    assert f(n, p, p, 1, 4, 4, 1, p, p, sv, None, ws, None) == BAD        # no workspace
    for shape in ((0, 4, 4), (1, 0, 4), (1, 4, 0), (-2, 4, 4)):
        assert f(n, p, p, *shape, 1, p, p, sv, p, ws, None) == BAD, shape
    for r in (-1, 3, 100):
        assert f(n, p, p, 1, 4, 4, r, p, p, sv, p, ws, None) == BAD, r
    assert f(n, p, p, 1, 4, 4, 1, p, p, sv - 4, p, ws, None) == WS
    assert f(n, p, p, 1, 4, 4, 1, p, p, sv, p, ws - 4, None) == WS
    assert f(n, p, p, 1, 4, 4, 0, p, None, 0, p, ws_inf - 4, None) == WS
    wide, _w = _net(p, dim=40)
    assert f(ctypes.byref(wide), p, p, 1, 4, 4, 1, p, p, sv, p, ws, None) == UNSUP
    big, _b = _net(p, K=8193)
    assert f(ctypes.byref(big), None, p, 1, 4, 4, 7, p, p, sv, p, ws, None) == UNSUP   # the net is checked first


@pytest.mark.parametrize("sfx", ["f32", "tf32"])
def test_backward_entry_points_validate_arguments_without_a_gpu(sfx):
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    f = getattr(lib, "vqb_prior_ce_backward_" + sfx)
    net, _l = _net(p)
    n = ctypes.byref(net)
    g, _g = _grads(p)
    gr = ctypes.byref(g)
    ws = lib.vqb_prior_ce_backward_workspace_bytes(n, 1, 4, 4)
    assert ws > 0
    assert f(None, p, p, 1, 4, 4, 1, p, p, gr, p, ws, None) == BAD
    assert f(n, None, p, 1, 4, 4, 1, p, p, gr, p, ws, None) == BAD
    assert f(n, p, None, 1, 4, 4, 1, p, p, gr, p, ws, None) == BAD
    assert f(n, p, p, 1, 4, 4, 1, None, p, gr, p, ws, None) == BAD        # no d_loss
    assert f(n, p, p, 1, 4, 4, 1, p, None, gr, p, ws, None) == BAD        # no saved
    assert f(n, p, p, 1, 4, 4, 1, p, p, None, p, ws, None) == BAD         # no gradients
    assert f(n, p, p, 1, 4, 4, 1, p, p, gr, None, ws, None) == BAD
    g1, _g1 = _grads(p, L=1)
    assert f(n, p, p, 1, 4, 4, 1, p, p, ctypes.byref(g1), p, ws, None) == BAD   # a table for another depth
    for r in (-1, 3):
        assert f(n, p, p, 1, 4, 4, r, p, p, gr, p, ws, None) == BAD
    assert f(n, p, p, 0, 4, 4, 1, p, p, gr, p, ws, None) == BAD
    assert f(n, p, p, 1, 4, 4, 1, p, p, gr, p, ws - 4, None) == WS
    big, _b = _net(p, K=8193)
    assert f(ctypes.byref(big), p, p, 1, 4, 4, 1, p, p, gr, p, ws, None) == UNSUP
    assert lib.vqb_prior_ce_backward_workspace_bytes(None, 1, 4, 4) == 0
    assert lib.vqb_prior_ce_backward_workspace_bytes(n, 0, 4, 4) == 0


def test_saved_and_forward_workspace_sizes():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    for shape in ((1, 4, 4, 32, 2, 16), (32, 8, 8, 64, 15, 512), (16, 64, 64, 64, 2, 8192), (3, 1, 1, 32, 1, 8192)):
        B, H, W, dim, L, K = shape
        npos = B * H * W
        assert lib.vqb_prior_ce_saved_bytes(B, H, W, dim, L) == lib.vqb_prior_train_saved_bytes(B, H, W, dim, L) + \
            8 * npos
        assert lib.vqb_prior_ce_workspace_bytes(*shape, 0) == lib.vqb_prior_log_prob_workspace_bytes(*shape) + 4 * npos
        assert lib.vqb_prior_ce_workspace_bytes(*shape, 1) == 16 * npos
        lp = lib.vqb_prior_log_prob_workspace_bytes_tf32(*shape)
        splits = (lp - lib.vqb_prior_workspace_bytes_tf32(*shape)) // (12 * npos)
        assert lib.vqb_prior_ce_workspace_bytes_tf32(*shape, 0) == lp + 4 * npos
        assert lib.vqb_prior_ce_workspace_bytes_tf32(*shape, 1) == 4 * npos * (3 * splits + 1)
    for q in (lib.vqb_prior_ce_workspace_bytes, lib.vqb_prior_ce_workspace_bytes_tf32):
        assert q(0, 4, 4, 32, 2, 16, 1) == 0 and q(1, 4, 4, 32, 2, 0, 0) == 0
    assert lib.vqb_prior_ce_saved_bytes(1, 4, 4, 0, 2) == 0


def test_backward_workspace_has_no_term_in_positions_times_codes():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)

    def ws(B, K, dim=64, L=2, H=64):
        net, _l = _net(p, dim=dim, K=K, L=L)
        return lib.vqb_prior_ce_backward_workspace_bytes(ctypes.byref(net), B, H, H)
    for K1, K2 in ((512, 8192), (1024, 4096), (37, 300)):
        for B in (16, 64):
            assert ws(2 * B, K2) - ws(2 * B, K1) == ws(B, K2) - ws(B, K1), (K1, K2, B)
    # the forward + CE backward's workspace at B=16, 64x64, K=8192 keeps about 0.5 GiB of output_conv.2 partials
    net, _l = _net(p, dim=64, K=8192, L=2)
    old = lib.vqb_prior_backward_workspace_bytes(ctypes.byref(net), 16, 64, 64)
    assert ws(16, 8192) < old - 2 ** 28
    assert ws(16, 8192) < 2 ** 29


# ---- the fp64 restatement of the head's d_logits ------------------------------------------------------------------
def d_logits(l, codes, g):
    """g_n * (softmax(l_n) - onehot(clamp(c_n))) for logits l (N, K), codes (N,) and g scalar or (N,)"""
    l = np.asarray(l, dtype=np.float64)
    K = l.shape[1]
    M = l.max(1, keepdims=True)
    p = np.exp(l - M)
    p /= p.sum(1, keepdims=True)
    p[np.arange(l.shape[0]), np.clip(codes, 0, K - 1)] -= 1
    return p * np.broadcast_to(np.asarray(g, dtype=np.float64), (l.shape[0],))[:, None]


def test_d_logits_restatement_on_hand_made_logits():
    l = np.array([[0.0, 0.0, 0.0, 0.0], [np.log(0.5), np.log(0.25), np.log(0.125), np.log(0.125)],
                  [10.0, 0.0, 0.0, -1000.0]])
    d = d_logits(l, np.array([2, 1, 0]), 1.0)
    np.testing.assert_allclose(d[0], [0.25, 0.25, -0.75, 0.25], rtol=1e-15)
    np.testing.assert_allclose(d[1], [0.5, -0.75, 0.125, 0.125], rtol=1e-15)
    assert d[2, 3] == 0.0 and abs(d[2].sum()) < 1e-15
    # rows sum to zero, per-position g scales rows, scalar g scales all
    g = np.array([2.0, -1.0, 0.5])
    np.testing.assert_allclose(d_logits(l, np.array([2, 1, 0]), g), d * g[:, None], rtol=1e-15)
    np.testing.assert_allclose(d_logits(l, np.array([2, 1, 0]), 1 / 3), d / 3, rtol=1e-15)
    # clamped codes are differentiated as the clamped code
    np.testing.assert_array_equal(d_logits(l, np.array([-5, 9, 100]), 1.0), d_logits(l, np.array([0, 3, 3]), 1.0))
    # against torch's autograd of the cross-entropy in fp64, every reduction
    rng = np.random.default_rng(0)
    lt = rng.standard_normal((12, 7))
    c = rng.integers(0, 7, 12)
    for red, gt in (("mean", 1 / 12), ("sum", 1.0), ("none", rng.standard_normal(12))):
        t = torch.tensor(lt, requires_grad=True)
        with torch.enable_grad():
            loss = torch.nn.functional.cross_entropy(t, torch.from_numpy(c), reduction=red)
            loss.backward(torch.from_numpy(gt) if red == "none" else None)
        np.testing.assert_allclose(t.grad.numpy(), d_logits(lt, c, gt), rtol=1e-12, atol=1e-15)

"""GatedPixelCNN.log_prob without a GPU: signature and docstring, the checks that run before any CUDA call and their
order, the C ABI's argument checks for vqb_prior_log_prob_* and the workspace queries' arithmetic, the header, and the
fp64 restatement of the contract (tests/prior_log_prob_ref.py) on hand-made logits."""
import contextlib
import ctypes
import inspect
import io
import os
import re

import numpy as np
import pytest
import torch

from tests import prior_log_prob_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model(first="A", precision="fp32"):
    from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(37, 32, 2, 3)
    if first != "A":
        m.layers[0] = GatedMaskedConv2d("B", 32, 7, True, 3)
    m.precision = precision
    return m


def test_signature_and_docstring():
    from pixelcnn.models import GatedPixelCNN
    s = inspect.signature(GatedPixelCNN.log_prob)
    assert list(s.parameters) == ["self", "x", "label", "n_given", "per_position"]
    for name, default in (("n_given", 0), ("per_position", False)):
        assert s.parameters[name].kind is inspect.Parameter.KEYWORD_ONLY and s.parameters[name].default == default
    assert list(inspect.signature(GatedPixelCNN._log_prob).parameters) == \
        ["self", "x", "label", "n_given", "per_position"]
    doc = " ".join(GatedPixelCNN.log_prob.__doc__.split())
    for phrase in ("Never differentiable", "forward plus the cross-entropy", "clamped", "not a likelihood",
                   "n_given = H*W gives zeros", "-log_prob(x, label).sum() / x.numel()"):
        assert phrase in doc, phrase


X, LAB = torch.zeros((2, 5, 5), dtype=torch.int64), torch.zeros(2, dtype=torch.int64)


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("n_given", [-1, 26, 2**40, 2.0, 3.5, "3", None, True])
def test_bad_n_given_raises_value_error_before_the_cuda_check(precision, n_given):
    m = _model(precision=precision)
    with pytest.raises(ValueError, match="n_given"):
        m.log_prob(X, LAB, n_given=n_given)
    with pytest.raises(ValueError, match="n_given"):
        m._log_prob(X, LAB, n_given, False)


@pytest.mark.parametrize("n_given", [1, 12, 25])
def test_per_position_with_n_given_is_a_value_error(n_given):
    with pytest.raises(ValueError, match="per_position"):
        _model().log_prob(X, LAB, n_given=n_given, per_position=True)


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("n_given,per_position", [(0, False), (1, False), (25, False), (0, True)])
def test_valid_arguments_on_cpu_tensors_raise_the_cuda_error(precision, n_given, per_position):
    m = _model(precision=precision)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.log_prob(X, LAB, n_given=n_given, per_position=per_position)
    with pytest.raises(RuntimeError, match="CUDA"):
        m._log_prob(X, LAB, n_given, per_position)


def test_errors_and_their_order():
    from pixelcnn.models import GatedMaskedConv2d
    m = _model()
    m.precision = "bf16"                                    # the precision first
    with pytest.raises(ValueError, match="precision"):
        m.log_prob(torch.zeros((5, 5), dtype=torch.int64), LAB, n_given=-1)
    m.precision = "fp32"
    with pytest.raises(ValueError, match="n_given"):       # then n_given's type, before the rank
        m.log_prob(torch.zeros((5, 5), dtype=torch.int64), LAB, n_given=1.0)
    with pytest.raises(RuntimeError, match="shape"):       # the rank, before n_given's range
        m.log_prob(torch.zeros((5, 5), dtype=torch.int64), LAB, n_given=-1)
    with pytest.raises(ValueError, match="n_given"):       # the range, before the square check
        m.log_prob(torch.zeros((2, 6, 8), dtype=torch.int64), LAB, n_given=49)
    with pytest.raises(ValueError, match="per_position"):  # per_position, before the square check
        m.log_prob(torch.zeros((2, 6, 8), dtype=torch.int64), LAB, n_given=3, per_position=True)
    with pytest.raises(RuntimeError, match="square"):
        m.log_prob(torch.zeros((2, 6, 8), dtype=torch.int64), torch.zeros(3, dtype=torch.int64))
    m.layers[1] = GatedMaskedConv2d("B", 64, 3, True, 3)   # P5, before the label count
    with pytest.raises(RuntimeError, match="layer 1 has 64 channels"):
        m.log_prob(X, torch.zeros(3, dtype=torch.int64))
    m = _model()
    m.layers[1] = GatedMaskedConv2d("B", 32, 3, True, 4)
    with pytest.raises(RuntimeError, match="classes"):
        m.log_prob(X, LAB)
    m.layers[1] = GatedMaskedConv2d("B", 32, 17, True, 3)
    with pytest.raises(RuntimeError, match="kernel 17"):
        m.log_prob(X, LAB)
    with pytest.raises(RuntimeError, match="expected 2 labels, got 3"):
        _model().log_prob(X, torch.zeros(3, dtype=torch.int64))


def test_any_layer_zero_is_taken():
    """No causality check: a mask-B, residual layer 0 reaches the CUDA check (forward takes it too)."""
    for precision in ("fp32", "tf32"):
        with pytest.raises(RuntimeError, match="CUDA"):
            _model("B", precision).log_prob(X, LAB, n_given=3)


def _header_text():
    src = open(os.path.join(ROOT, "include", "vqvae_b200.h")).read()
    return re.sub(r"/\*.*?\*/", "", src, flags=re.S)


def test_header_declares_and_the_library_exports_the_log_prob_abi():
    from vqvae_b200 import _lib
    src = " ".join(_header_text().split())
    for sfx in ("", "_tf32"):
        assert f"size_t vqb_prior_log_prob_workspace_bytes{sfx}(int B, int H, int W, int dim, int n_layers, int K);" \
            in src
    for sfx in ("f32", "tf32"):
        assert re.search(rf"int vqb_prior_log_prob_{sfx}\(const vqb_prior_net \*net, const int64_t \*codes, const "
                         r"int64_t \*labels, int64_t n_given, int B, int H, int W, float \*log_prob, float "
                         r"\*pos_log_prob, void \*workspace, size_t workspace_bytes, void \*stream\);", src), sfx
    lib = _lib.lib()
    for name in ("vqb_prior_log_prob_workspace_bytes", "vqb_prior_log_prob_workspace_bytes_tf32",
                 "vqb_prior_log_prob_f32", "vqb_prior_log_prob_tf32"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES
    assert lib.vqb_abi_version() == 3
    doc = " ".join(open(os.path.join(ROOT, "include", "vqvae_b200.h")).read().split())
    assert "fp32 3 + 2*n_layers" in doc and "TF32 4 + 4*n_layers" in doc


def _splits(npos, K):
    bn = 64 if K <= 64 else 128
    tiles = -(-K // bn)
    s = min(tiles, max(1, -(-264 // -(-npos // 128))))
    return -(-tiles // -(-tiles // s))


def test_workspace_queries():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    q32, qtf = lib.vqb_prior_log_prob_workspace_bytes, lib.vqb_prior_log_prob_workspace_bytes_tf32
    for bad in ((0, 4, 4, 32, 2, 16), (1, 0, 4, 32, 2, 16), (1, 4, 0, 32, 2, 16), (1, 4, 4, 0, 2, 16),
                (1, 4, 4, 32, 0, 16), (1, 4, 4, 32, 2, 0), (-1, 4, 4, 32, 2, 16)):
        assert q32(*bad) == 0 and qtf(*bad) == 0, bad
    for shape in ((1, 4, 4, 32, 2, 16), (32, 8, 8, 64, 15, 512), (16, 64, 64, 64, 15, 1024),
                  (16, 64, 64, 64, 2, 8192), (3, 1, 1, 32, 1, 8192), (2, 48, 48, 32, 2, 512), (3, 6, 6, 256, 2, 8192)):
        B, H, W, dim, L, K = shape
        npos = B * H * W
        assert q32(*shape) == lib.vqb_prior_workspace_bytes(*shape) + 12 * npos, shape
        assert qtf(*shape) == lib.vqb_prior_workspace_bytes_tf32(*shape) + 12 * npos * _splits(npos, K), shape
    assert _splits(32 * 64, 512) == 4                  # the reference's default: 16 position tiles, K over 4 CTAs
    assert _splits(16 * 64 * 64, 1024) == 1            # 64x64: no split
    assert _splits(16 * 64 * 64, 8192) == 1
    assert _splits(3 * 36, 8192) == 64
    # K-independent beyond the splits: 64x64 at K = 8192 needs no more than at K = 1024
    assert qtf(16, 64, 64, 64, 2, 8192) == qtf(16, 64, 64, 64, 2, 1024)


def _net(p, dim=32, K=16):
    from vqvae_b200 import _lib
    lw = _lib.PriorLayerWeights(*([p.value] * 9), 7, 1, 0)
    layers = (_lib.PriorLayerWeights * 2)(lw, _lib.PriorLayerWeights(*([p.value] * 9), 3, 0, 1))
    net = _lib.PriorNet(layers=layers, n_layers=2, embedding=p.value, out1_w=p.value, out1_b=p.value, out2_w=p.value,
                        out2_b=p.value, input_dim=K, dim=dim, n_classes=2)
    return net, layers


@pytest.mark.parametrize("sfx", ["f32", "tf32"])
def test_entry_points_validate_arguments_without_a_gpu(sfx):
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    f = getattr(lib, "vqb_prior_log_prob_" + sfx)
    q = lib.vqb_prior_log_prob_workspace_bytes_tf32 if sfx == "tf32" else lib.vqb_prior_log_prob_workspace_bytes
    net, layers = _net(p)
    n = ctypes.byref(net)
    ws = q(1, 4, 4, 32, 2, 16)
    BAD, WS, UNSUP = -1, -3, -2
    assert f(None, p, p, 0, 1, 4, 4, p, p, p, ws, None) == BAD
    assert f(n, None, p, 0, 1, 4, 4, p, p, p, ws, None) == BAD
    assert f(n, p, None, 0, 1, 4, 4, p, p, p, ws, None) == BAD
    assert f(n, p, p, 0, 1, 4, 4, None, None, p, ws, None) == BAD          # no output
    assert f(n, p, p, 0, 1, 4, 4, p, p, None, ws, None) == BAD
    for shape in ((0, 4, 4), (1, 0, 4), (1, 4, 0), (-2, 4, 4)):
        assert f(n, p, p, 0, *shape, p, p, p, ws, None) == BAD, shape
    for n_given in (-1, 17, 2**40, -2**40):
        assert f(n, p, p, n_given, 1, 4, 4, p, None, p, ws, None) == BAD, n_given
        assert f(n, p, p, n_given, 1, 4, 4, None, p, p, ws, None) == BAD, n_given
    assert f(n, p, p, 0, 1, 4, 4, p, p, p, ws - 4, None) == WS
    assert f(n, p, p, 16, 1, 4, 4, None, p, p, ws - 4, None) == WS
    wide, _l = _net(p, dim=40)
    assert f(ctypes.byref(wide), p, p, 0, 1, 4, 4, p, p, p, ws, None) == UNSUP
    big, _l = _net(p, K=8193)
    assert f(ctypes.byref(big), p, p, 0, 1, 4, 4, p, p, p, ws, None) == UNSUP
    assert f(ctypes.byref(big), None, p, 0, 1, 4, 4, p, p, p, ws, None) == UNSUP  # the net is checked first


# ---- the fp64 restatement on hand-made logits --------------------------------------------------------------------

def test_position_terms_and_clamping():
    l = np.zeros((1, 4, 1, 3))
    l[0, :, 0, 0] = [0.0, 0.0, 0.0, 0.0]
    l[0, :, 0, 1] = [np.log(0.5), np.log(0.25), np.log(0.125), np.log(0.125)]
    l[0, :, 0, 2] = [10.0, 0.0, 0.0, -1000.0]
    lp = ref.position_terms(l, np.array([[[2, 1, 0]]]))
    np.testing.assert_allclose(lp[0, 0], [np.log(0.25), np.log(0.25), -np.log1p(2 * np.exp(-10.0))], rtol=1e-12)
    # out-of-range codes are scored as the clamped code
    np.testing.assert_array_equal(ref.position_terms(l, np.array([[[-5, 9, 100]]])),
                                  ref.position_terms(l, np.array([[[0, 3, 3]]])))
    np.testing.assert_allclose(ref.position_terms(l, np.array([[[0, 4, 3]]]))[0, 0, 1], np.log(0.125), rtol=1e-12)


def test_n_given_restricts_the_sum_in_raster_order():
    rng = np.random.default_rng(0)
    l = rng.standard_normal((3, 7, 4, 4))
    c = rng.integers(0, 7, (3, 4, 4))
    lp = ref.position_terms(l, c)
    flat = lp.reshape(3, -1)
    for n in (0, 1, 3, 4, 8, 15, 16):
        np.testing.assert_allclose(ref.log_prob(l, c, n), flat[:, n:].sum(-1), rtol=1e-12)
    assert (ref.log_prob(l, c, 16) == 0).all()
    # raster order: p = i*W + j, so n_given = W leaves out exactly row 0
    np.testing.assert_allclose(ref.log_prob(l, c, 4), lp[:, 1:].reshape(3, -1).sum(-1), rtol=1e-12)
    assert ref.scored(3, 4, 4, 5)[0].tolist()[1] == [False, True, True, True]


def test_compensated_raster_sum():
    rng = np.random.default_rng(1)
    t = (-6.9 + 1e-3 * rng.standard_normal((2, 4096))).astype(np.float32)
    exact = t.astype(np.float64).sum(-1)
    naive = np.zeros(2, dtype=np.float32)
    for v in t.T:
        naive = (naive + v).astype(np.float32)
    k = ref.kahan32(t)
    assert (np.abs(k - exact) <= 1e-6 * np.abs(exact)).all()
    assert np.abs(k - exact).max() < np.abs(naive - exact).max()
    np.testing.assert_array_equal(ref.kahan32(t, 4096), np.zeros(2, dtype=np.float32))
    np.testing.assert_allclose(ref.kahan32(t, 100), t[:, 100:].astype(np.float64).sum(-1), rtol=1e-6)

"""GatedPixelCNN.sample / sample_completion without a GPU: signatures, the knob checks that run before any CUDA call,
the C ABI's argument checks for vqb_prior_sample_f32 and its workspace query, the header, and the fp64 restatement
of the draw's contract (tests/prior_sample_ref.py) on hand-made logits."""
import contextlib
import ctypes
import inspect
import io
import math
import os
import re

import numpy as np
import pytest
import torch

from tests import prior_sample_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model(first="A"):
    from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(37, 32, 2, 3)
    if first != "A":
        m.layers[0] = GatedMaskedConv2d("B", 32, 7, False, 3)
    return m


def _knobs(knobs):
    return {**dict(temperature=1.0, top_k=None, top_p=None), **knobs}


def test_signatures():
    from pixelcnn.models import GatedPixelCNN
    s = inspect.signature(GatedPixelCNN.sample)
    assert list(s.parameters) == ["self", "label", "shape", "batch_size", "temperature", "top_k", "top_p"]
    assert s.parameters["shape"].default == (8, 8) and s.parameters["batch_size"].default == 64
    for f in (GatedPixelCNN.sample, GatedPixelCNN.sample_completion):
        ps = inspect.signature(f).parameters
        for name, default in (("temperature", 1.0), ("top_k", None), ("top_p", None)):
            assert ps[name].kind is inspect.Parameter.KEYWORD_ONLY and ps[name].default == default
    assert list(inspect.signature(GatedPixelCNN.sample_completion).parameters) == \
        ["self", "x", "label", "n_given", "temperature", "top_k", "top_p"]
    assert list(inspect.signature(GatedPixelCNN._sample_with).parameters) == \
        ["self", "label", "u", "x", "n_given", "temperature", "top_k", "top_p", "step_logits"]


BAD_KNOBS = [dict(temperature=0.0), dict(temperature=-1.0), dict(temperature=math.inf), dict(temperature=math.nan),
             dict(temperature=1e-50), dict(temperature=1e39), dict(temperature="1"), dict(temperature=True),
             dict(top_k=0), dict(top_k=-1), dict(top_k=38), dict(top_k=2.0), dict(top_k=True),
             dict(top_p=0.0), dict(top_p=-0.5), dict(top_p=1.5), dict(top_p=math.nan), dict(top_p=1e-50),
             dict(top_p="0.5")]


@pytest.mark.parametrize("knobs", BAD_KNOBS, ids=lambda k: f"{next(iter(k))}={next(iter(k.values()))!r}")
def test_bad_knobs_raise_value_error_before_the_cuda_check(knobs):
    m = _model()
    x, lab = torch.zeros((2, 5, 5), dtype=torch.int64), torch.zeros(2, dtype=torch.int64)
    full = _knobs(knobs)
    with pytest.raises(ValueError):
        m.sample(lab, shape=(5, 5), batch_size=2, **knobs)
    with pytest.raises(ValueError):
        m.sample_completion(x, lab, 3, **knobs)
    with pytest.raises(ValueError):
        m._sample_with(lab, torch.zeros((2, 5, 5)), None, 0, full["temperature"], full["top_k"], full["top_p"])
    with pytest.raises(ValueError):
        m._sample_with(lab, torch.zeros((2, 5, 5)), x, 3, full["temperature"], full["top_k"], full["top_p"])


@pytest.mark.parametrize("knobs", [{}, dict(temperature=0.5), dict(top_k=1), dict(top_k=37), dict(top_p=1.0),
                                   dict(top_p=1e-3), dict(temperature=3, top_k=5, top_p=0.9)])
def test_valid_knobs_on_cpu_tensors_raise_the_cuda_error(knobs):
    m = _model()
    x, lab = torch.zeros((2, 5, 5), dtype=torch.int64), torch.zeros(2, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.sample(lab, shape=(5, 5), batch_size=2, **knobs)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.sample_completion(x, lab, 3, **knobs)
    k = _knobs(knobs)
    with pytest.raises(RuntimeError, match="CUDA"):
        m._sample_with(lab, torch.zeros((2, 5, 5)), x, 3, k["temperature"], k["top_k"], k["top_p"])


def test_sample_refuses_what_complete_refuses():
    m = _model()
    lab = torch.zeros(2, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="square"):
        m.sample(lab, shape=(6, 8), batch_size=2)
    with pytest.raises(ValueError, match="n_given"):
        m.sample_completion(torch.zeros((2, 5, 5), dtype=torch.int64), lab, 26)
    with pytest.raises(RuntimeError, match="shape"):
        m.sample_completion(torch.zeros((5, 5), dtype=torch.int64), lab, 3)
    with pytest.raises(RuntimeError, match="expected 2 labels, got 3"):
        m.sample_completion(torch.zeros((2, 5, 5), dtype=torch.int64), torch.zeros(3, dtype=torch.int64), 3)
    with pytest.raises(RuntimeError, match="mask A without residual"):
        _model("B").sample(lab, shape=(5, 5), batch_size=2)
    with pytest.raises(RuntimeError, match="mask A without residual"):
        _model("B").sample_completion(torch.zeros((2, 5, 5), dtype=torch.int64), lab, 3)


def _header_text():
    src = open(os.path.join(ROOT, "include", "vqvae_b200.h")).read()
    return re.sub(r"/\*.*?\*/", "", src, flags=re.S)


def test_header_declares_and_the_library_exports_the_sampling_abi():
    from vqvae_b200 import _lib
    src = _header_text()
    assert re.search(r"typedef struct vqb_prior_sampling \{\s*float temperature;\s*int top_k;\s*float top_p;\s*\}"
                     r" vqb_prior_sampling;", src)
    assert re.search(r"size_t vqb_prior_sample_workspace_bytes\(int B, int H, int W, int dim, int n_layers, int K,"
                     r"\s*int64_t n_given\);", src)
    assert "int vqb_prior_sample_f32(" in src
    lib = _lib.lib()
    for name in ("vqb_prior_sample_workspace_bytes", "vqb_prior_sample_f32"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES
    assert lib.vqb_abi_version() == 3
    assert ctypes.sizeof(_lib.PriorSampling) == 12


def _net(p, first=(7, 1, 0), dim=32, K=16):
    from vqvae_b200 import _lib
    lw = _lib.PriorLayerWeights(*([p.value] * 9), 7, 1, 0)
    layers = (_lib.PriorLayerWeights * 2)(_lib.PriorLayerWeights(*([p.value] * 9), *first), lw)
    net = _lib.PriorNet(layers=layers, n_layers=2, embedding=p.value, out1_w=p.value, out1_b=p.value, out2_w=p.value,
                        out2_b=p.value, input_dim=K, dim=dim, n_classes=2)
    return net, layers


def test_sample_entry_points_validate_arguments_without_a_gpu():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    q = lib.vqb_prior_sample_workspace_bytes
    for bad in ((0, 4, 4, 32, 2, 16, 0), (1, 0, 4, 32, 2, 16, 0), (1, 4, 4, 0, 2, 16, 0), (1, 4, 4, 32, 2, 0, 0),
                (1, 4, 4, 32, 2, 16, -1), (1, 4, 4, 32, 2, 16, 17)):
        assert q(*bad) == 0
    for shape in ((1, 4, 4, 32, 2, 16), (100, 8, 8, 64, 15, 512), (16, 64, 64, 64, 15, 1024), (3, 1, 1, 32, 1, 8192),
                  (2, 48, 48, 32, 2, 512)):
        B, H, W, dim, L, K = shape
        for n in (0, W - 1, W, H * W):
            got = q(*shape, n)
            assert got >= lib.vqb_prior_workspace_bytes(*shape)
            if n >= W:
                assert got >= lib.vqb_prior_complete_workspace_bytes(*shape)
            assert got >= (256 * ((K + 31) // 32) + 4) * B                  # the draw's scratch
    net, layers = _net(p)
    n = ctypes.byref(net)
    ws = q(1, 4, 4, 32, 2, 16, 5)
    f = lib.vqb_prior_sample_f32
    S = _lib.PriorSampling
    ok = ctypes.byref(S(1.0, 0, 1.0))
    BAD, WS, UNSUP = -1, -3, -2
    assert f(n, p, p, None, 5, 1, 4, 4, ok, p, p, None, p, ws, None) == BAD        # null given with n_given > 0
    assert f(n, None, p, p, 5, 1, 4, 4, ok, p, p, None, p, ws, None) == BAD
    assert f(n, p, None, p, 5, 1, 4, 4, ok, p, p, None, p, ws, None) == BAD
    assert f(n, p, p, p, 5, 1, 4, 4, ok, None, p, None, p, ws, None) == BAD
    assert f(n, p, p, p, 5, 1, 4, 4, ok, p, p, None, None, ws, None) == BAD
    assert f(None, p, p, p, 5, 1, 4, 4, ok, p, p, None, p, ws, None) == BAD
    assert f(n, p, p, p, 5, 0, 4, 4, ok, p, p, None, p, ws, None) == BAD
    for n_given in (-1, 17, 2**40):
        assert f(n, p, p, p, n_given, 1, 4, 4, ok, p, p, None, p, ws, None) == BAD
    for knobs in ((0.0, 0, 1.0), (-1.0, 0, 1.0), (math.inf, 0, 1.0), (math.nan, 0, 1.0), (1.0, -1, 1.0),
                  (1.0, 17, 1.0), (1.0, 0, 0.0), (1.0, 0, -0.1), (1.0, 0, 1.5), (1.0, 0, math.nan)):
        assert f(n, p, p, p, 5, 1, 4, 4, ctypes.byref(S(*knobs)), p, p, None, p, ws, None) == BAD, knobs
    assert f(n, p, p, p, 5, 1, 4, 4, ok, p, p, None, p, ws - 4, None) == WS
    assert f(n, p, p, p, 5, 1, 4, 4, None, p, None, None, p, ws - 4, None) == WS    # NULL sampling, NULL log_prob
    assert f(n, p, p, None, 0, 1, 4, 4, None, p, None, None, p, q(1, 4, 4, 32, 2, 16, 0) - 4, None) == WS
    wide, _l = _net(p, dim=40)
    assert f(ctypes.byref(wide), p, p, p, 5, 1, 4, 4, ok, p, p, None, p, ws, None) == UNSUP
    for first in ((7, 0, 0), (7, 1, 1)):                                           # mask-B or residual layer 0
        bad, _l = _net(p, first=first)
        assert f(ctypes.byref(bad), p, p, p, 5, 1, 4, 4, ok, p, p, None, p, ws, None) == UNSUP
        assert f(ctypes.byref(bad), p, p, None, 0, 1, 4, 4, None, p, None, None, p, ws, None) == UNSUP
        assert f(ctypes.byref(bad), p, p, p, 5, 1, 4, 4, ctypes.byref(S(0.0, 0, 1.0)), p, p, None, p, ws,
                 None) == BAD                                                       # knobs are checked first


# ---- the fp64 restatement on hand-made logits --------------------------------------------------------------------

def test_ties_at_the_top_k_threshold_are_kept():
    l = np.array([[1.0, 3.0, 2.0, 2.0, 0.5, 2.0]])
    assert ref.kept(l, top_k=2).tolist() == [[False, True, True, True, False, True]]
    assert ref.kept(l, top_k=1).tolist() == [[False, True, False, False, False, False]]
    assert ref.kept(l, top_k=5).tolist() == [[True, True, True, True, False, True]]
    q = ref.probs(l, top_k=2)[0]
    np.testing.assert_allclose(q[[2, 3, 5]], q[2])
    np.testing.assert_allclose(q.sum(), 1.0)
    assert ref.kept(np.array([[0.0, -0.0, 1.0]]), top_k=2).tolist() == [[True, False, True]]   # -0 < +0


def test_top_k_one_is_the_argmax_and_top_k_k_keeps_everything():
    rng = np.random.default_rng(0)
    l = rng.standard_normal((50, 37)).astype(np.float32)
    S = ref.kept(l, top_k=1)
    assert (S.sum(-1) == 1).all() and (S.argmax(-1) == l.argmax(-1)).all()
    assert ref.kept(l, top_k=37).all()
    assert (ref.draw(l, rng.random(50), top_k=1) == l.argmax(-1)).all()
    np.testing.assert_array_equal(ref.probs(l, top_k=37), ref.probs(l))


def test_top_p_just_above_and_below_a_cumulative_mass():
    l = np.log(np.array([[0.5, 0.3, 0.15, 0.05]], dtype=np.float64)).astype(np.float32)
    p = ref.softmax64(ref.tempered(l, 1.0))[0]
    c1, c2 = p[0], p[0] + p[1]
    assert ref.kept(l, top_p=float(c1) * (1 - 1e-4)).tolist() == [[True, False, False, False]]
    assert ref.kept(l, top_p=float(c1) * (1 + 1e-4)).tolist() == [[True, True, False, False]]
    assert ref.kept(l, top_p=float(c2) * (1 - 1e-4)).tolist() == [[True, True, False, False]]
    assert ref.kept(l, top_p=float(c2) * (1 + 1e-4)).tolist() == [[True, True, True, False]]
    assert ref.kept(l, top_p=1e-6).tolist() == [[True, False, False, False]]
    assert ref.kept(l, top_p=1.0).all()
    np.testing.assert_allclose(ref.probs(l, top_p=0.7)[0], [0.5 / 0.8, 0.3 / 0.8, 0, 0], rtol=1e-6)
    # both knobs: the smaller kept set wins
    assert ref.kept(l, top_k=3, top_p=0.6).tolist() == [[True, True, False, False]]
    assert ref.kept(l, top_k=1, top_p=0.9).tolist() == [[True, False, False, False]]


def test_temperature():
    l = np.array([[0.0, 1.0, 2.0]], dtype=np.float32)
    np.testing.assert_allclose(ref.probs(l, T=2.0)[0], ref.softmax64(np.array([[0.0, 0.5, 1.0]]))[0])
    assert (ref.tempered(l, 1.0) == l).all()
    q = ref.probs(l, T=1e-3)[0]                         # T -> 0: the argmax
    assert q[2] == 1.0 and q[0] == 0.0 and q[1] == 0.0
    assert (ref.draw(np.repeat(l, 5, 0), np.array([0.0, 0.3, 0.5, 0.9, 0.999999]), T=1e-3) == 2).all()
    z = ref.tempered(np.array([[3.0, -3.0, 1e-40]], dtype=np.float32), 1e-40)   # saturates, no inf
    assert np.isfinite(z).all() and z[0, 0] == ref.FLT_MAX and z[0, 1] == -ref.FLT_MAX
    # temperature reorders nothing: the kept set of top_k is the same at any T
    rng = np.random.default_rng(1)
    l = rng.standard_normal((20, 33)).astype(np.float32)
    for T in (0.25, 0.5, 2.0, 7.0):
        np.testing.assert_array_equal(ref.kept(l, T, top_k=5), ref.kept(l, 1.0, top_k=5))
    # a lower temperature keeps fewer codes for the same top_p
    assert (ref.kept(l, 0.5, top_p=0.9).sum(-1) <= ref.kept(l, 2.0, top_p=0.9).sum(-1)).all()


def test_draw_and_log_softmax():
    l = np.array([[0.0, 0.0, 0.0, 0.0]], dtype=np.float32)
    u = np.array([0.1, 0.3, 0.6, 0.9])
    assert ref.draw(np.repeat(l, 4, 0), u).tolist() == [0, 1, 2, 3]
    assert ref.draw(np.repeat(l, 4, 0), u, top_k=2).tolist() == [0, 1, 2, 3]  # all tied: all kept
    l2 = np.array([[0.0, 1.0, 1.0, 0.0]], dtype=np.float32)
    assert ref.draw(np.repeat(l2, 4, 0), u, top_k=1).tolist() == [1, 1, 2, 2]
    np.testing.assert_allclose(ref.log_softmax64(l), np.log(0.25))

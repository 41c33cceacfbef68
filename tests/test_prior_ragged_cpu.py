"""Per-image prefix lengths for GatedPixelCNN.complete / sample_completion / log_prob without a GPU: the argument
refusals that run before any CUDA check, the CUDA error for valid arguments on CPU tensors, the header and SIGNATURES
for the ragged entry points, and their C argument checks."""
import contextlib
import ctypes
import io
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, S = 3, 5


def _model(first="A"):
    from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(37, 32, 2, 3)
    if first != "A":
        m.layers[0] = GatedMaskedConv2d("B", 32, 7, False, 3)
    return m


def _calls(m, x, lab, n, **kw):
    """Every public and graph-capturable form that takes n_given, as thunks."""
    u = torch.zeros(tuple(x.shape)) if x.dim() == 3 else torch.zeros((B, S, S))
    return {
        "complete": lambda: m.complete(x, lab, n),
        "_complete": lambda: m._complete(lab, u, x, n),
        "sample_completion": lambda: m.sample_completion(x, lab, n),
        "_sample_with": lambda: m._sample_with(lab, u, x, n, 1.0, None, None),
        "log_prob": lambda: m.log_prob(x, lab, n_given=n, **kw),
        "_log_prob": lambda: m._log_prob(x, lab, n, **kw),
    }


BAD = {
    "2-D": torch.zeros((B, 1), dtype=torch.int64),
    "too short": torch.zeros((B - 1,), dtype=torch.int64),
    "too long": torch.zeros((B + 1,), dtype=torch.int64),
    "float": torch.zeros((B,), dtype=torch.float32),
    "double": torch.zeros((B,), dtype=torch.float64),
    "bool": torch.zeros((B,), dtype=torch.bool),
    "list short": [0] * (B - 1),
    "list negative": [0, -1, 3],
    "list above H*W": [0, S * S + 1, 3],
    "list float": [0, 1.0, 3],
    "list bool": [0, True, 3],
    "tuple above H*W": (S * S, S * S, S * S + 7),
}


@pytest.mark.parametrize("bad", list(BAD), ids=list(BAD))
def test_bad_per_image_n_given_raises_value_error_before_the_cuda_check(bad):
    m = _model()
    x, lab = torch.zeros((B, S, S), dtype=torch.int64), torch.zeros(B, dtype=torch.int64)
    for name, call in _calls(m, x, lab, BAD[bad]).items():
        with pytest.raises(ValueError, match="n_given"):
            call()
        m.precision = "tf32"
        if name.endswith("log_prob"):
            with pytest.raises(ValueError, match="n_given"):
                call()
        m.precision = "fp32"


def test_a_tensor_on_another_device_is_refused_before_the_cuda_check():
    m = _model()
    x, lab = torch.zeros((B, S, S), dtype=torch.int64), torch.zeros(B, dtype=torch.int64)
    n = torch.zeros((B,), dtype=torch.int64, device="meta")
    for call in _calls(m, x, lab, n).values():
        with pytest.raises(RuntimeError, match="n_given is on meta"):
            call()


def test_per_position_takes_no_per_image_n_given():
    m = _model()
    x, lab = torch.zeros((B, S, S), dtype=torch.int64), torch.zeros(B, dtype=torch.int64)
    for n in (torch.zeros((B,), dtype=torch.int64), [0] * B, torch.zeros((1,), dtype=torch.int64)):
        for precision in ("fp32", "tf32"):
            m.precision = precision
            with pytest.raises(ValueError, match="per_position"):
                m.log_prob(x, lab, n_given=n, per_position=True)
            with pytest.raises(ValueError, match="per_position"):
                m._log_prob(x, lab, n, per_position=True)


def test_sample_without_codes_takes_no_per_image_n_given():
    m = _model()
    lab = torch.zeros(B, dtype=torch.int64)
    for n in (torch.zeros((B,), dtype=torch.int64), [0] * B):
        with pytest.raises(ValueError, match="n_given must be 0 without codes"):
            m._sample_with(lab, torch.zeros((B, S, S)), None, n, 1.0, None, None)


GOOD = {
    "int64": torch.tensor([0, 7, S * S], dtype=torch.int64),
    "int32": torch.tensor([1, 2, 3], dtype=torch.int32),
    "uint8": torch.tensor([1, 2, 3], dtype=torch.uint8),
    "out of range values": torch.tensor([-5, 3, S * S + 7], dtype=torch.int64),   # clamped on the device
    "non-contiguous": torch.tensor([[0, 9], [4, 9], [25, 9]], dtype=torch.int64)[:, 0],
    "list": [0, 12, S * S],
    "tuple": (S * S, 0, 1),
}


@pytest.mark.parametrize("good", list(GOOD), ids=list(GOOD))
def test_valid_per_image_n_given_on_cpu_tensors_raises_the_cuda_error(good):
    m = _model()
    x, lab = torch.zeros((B, S, S), dtype=torch.int64), torch.zeros(B, dtype=torch.int64)
    for precision in ("fp32", "tf32"):
        m.precision = precision
        for call in _calls(m, x, lab, GOOD[good]).values():
            with pytest.raises(RuntimeError, match="CUDA"):
                call()


def test_per_image_n_given_keeps_the_scalar_paths_other_refusals():
    m = _model()
    n = torch.zeros((B,), dtype=torch.int64)
    lab = torch.zeros(B, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="square"):
        m.complete(torch.zeros((B, 5, 6), dtype=torch.int64), lab, n)
    with pytest.raises(RuntimeError, match="square"):
        m.log_prob(torch.zeros((B, 5, 6), dtype=torch.int64), lab, n_given=n)
    with pytest.raises(RuntimeError, match="shape"):
        m.complete(torch.zeros((5, 5), dtype=torch.int64), lab, n)
    with pytest.raises(RuntimeError, match=f"expected {B} labels, got 2"):
        m.sample_completion(torch.zeros((B, S, S), dtype=torch.int64), torch.zeros(2, dtype=torch.int64), n)
    with pytest.raises(RuntimeError, match=f"expected {B} labels, got 2"):
        m.log_prob(torch.zeros((B, S, S), dtype=torch.int64), torch.zeros(2, dtype=torch.int64), n_given=n)
    with pytest.raises(RuntimeError, match="mask A without residual"):
        _model("B").complete(torch.zeros((B, S, S), dtype=torch.int64), lab, n)
    with pytest.raises(RuntimeError, match="mask A without residual"):
        _model("B").sample_completion(torch.zeros((B, S, S), dtype=torch.int64), lab, [1, 2, 3])
    with pytest.raises(ValueError, match="temperature"):
        m.sample_completion(torch.zeros((B, S, S), dtype=torch.int64), lab, n, temperature=0.0)


def _header_text():
    src = open(os.path.join(ROOT, "include", "vqvae_b200.h")).read()
    return re.sub(r"/\*.*?\*/", "", src, flags=re.S)


def _params(src, name):
    m = re.search(r"\b(int|size_t) " + name + r"\((.*?)\);", src, flags=re.S)
    assert m, name
    return [" ".join(p.split()) for p in m.group(2).split(",")]


def test_header_and_signatures_agree_on_the_ragged_entry_points():
    from vqvae_b200 import _lib
    src = _header_text()
    assert _params(src, "vqb_prior_sample_ragged_f32") == [
        "const vqb_prior_net *net", "const int64_t *labels", "const float *u", "const int64_t *given",
        "const int64_t *n_given", "int B", "int H", "int W", "const vqb_prior_sampling *sampling", "int64_t *codes",
        "float *log_prob", "float *step_logits", "void *workspace", "size_t workspace_bytes", "void *stream"]
    for sfx in ("f32", "tf32"):
        assert _params(src, "vqb_prior_log_prob_ragged_" + sfx) == [
            "const vqb_prior_net *net", "const int64_t *codes", "const int64_t *labels", "const int64_t *n_given",
            "int B", "int H", "int W", "float *log_prob", "void *workspace", "size_t workspace_bytes",
            "void *stream"]
    ctype = {"int": ctypes.c_int, "size_t": ctypes.c_size_t}
    for name in ("vqb_prior_sample_ragged_f32", "vqb_prior_log_prob_ragged_f32", "vqb_prior_log_prob_ragged_tf32"):
        res, args = _lib.SIGNATURES[name]
        assert res is ctype["int"]
        want = [ctypes.c_void_p if "*" in p else ctype.get(p.split()[0], None) for p in _params(src, name)]
        assert args == want, name
    lib = _lib.lib()
    for name in ("vqb_prior_sample_ragged_f32", "vqb_prior_log_prob_ragged_f32", "vqb_prior_log_prob_ragged_tf32"):
        assert hasattr(lib, name)
    assert lib.vqb_abi_version() == 3


def _net(p, first=(7, 1, 0), dim=32, K=16):
    from vqvae_b200 import _lib
    lw = _lib.PriorLayerWeights(*([p.value] * 9), 7, 1, 0)
    layers = (_lib.PriorLayerWeights * 2)(_lib.PriorLayerWeights(*([p.value] * 9), *first), lw)
    net = _lib.PriorNet(layers=layers, n_layers=2, embedding=p.value, out1_w=p.value, out1_b=p.value, out2_w=p.value,
                        out2_b=p.value, input_dim=K, dim=dim, n_classes=2)
    return net, layers


BAD_ARG, UNSUP, WS = -1, -2, -3


def test_ragged_sample_entry_point_validates_arguments_without_a_gpu():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    net, _layers = _net(p)
    n = ctypes.byref(net)
    ws = lib.vqb_prior_sample_workspace_bytes(2, 4, 4, 32, 2, 16, 0)
    assert ws > 0
    f = lib.vqb_prior_sample_ragged_f32
    S_ = _lib.PriorSampling
    ok = ctypes.byref(S_(1.0, 0, 1.0))
    # (net, labels, u, given, n_given, B, H, W, sampling, codes, log_prob, step_logits, workspace, bytes, stream)
    assert f(None, p, p, p, p, 2, 4, 4, ok, p, p, None, p, ws, None) == BAD_ARG
    assert f(n, None, p, p, p, 2, 4, 4, ok, p, p, None, p, ws, None) == BAD_ARG
    assert f(n, p, None, p, p, 2, 4, 4, ok, p, p, None, p, ws, None) == BAD_ARG
    assert f(n, p, p, None, p, 2, 4, 4, ok, p, p, None, p, ws, None) == BAD_ARG          # NULL given
    assert f(n, p, p, p, None, 2, 4, 4, ok, p, p, None, p, ws, None) == BAD_ARG          # NULL n_given
    assert f(n, p, p, p, p, 2, 4, 4, ok, None, p, None, p, ws, None) == BAD_ARG
    assert f(n, p, p, p, p, 2, 4, 4, ok, p, p, None, None, ws, None) == BAD_ARG
    for shape in ((0, 4, 4), (-1, 4, 4), (2, 0, 4), (2, 4, -3)):
        assert f(n, p, p, p, p, *shape, ok, p, p, None, p, ws, None) == BAD_ARG, shape
    for knobs in ((0.0, 0, 1.0), (-1.0, 0, 1.0), (float("nan"), 0, 1.0), (1.0, -1, 1.0), (1.0, 17, 1.0),
                  (1.0, 0, 0.0), (1.0, 0, 1.5)):
        assert f(n, p, p, p, p, 2, 4, 4, ctypes.byref(S_(*knobs)), p, p, None, p, ws, None) == BAD_ARG, knobs
    assert f(n, p, p, p, p, 2, 4, 4, ok, p, p, None, p, ws - 4, None) == WS
    assert f(n, p, p, p, p, 2, 4, 4, None, p, None, None, p, ws - 4, None) == WS          # the ragged complete
    wide, _l = _net(p, dim=40)
    assert f(ctypes.byref(wide), p, p, p, p, 2, 4, 4, ok, p, p, None, p, ws, None) == UNSUP
    for first in ((7, 0, 0), (7, 1, 1)):                                                   # mask-B or residual layer 0
        bad, _l = _net(p, first=first)
        assert f(ctypes.byref(bad), p, p, p, p, 2, 4, 4, ok, p, p, None, p, ws, None) == UNSUP
        assert f(ctypes.byref(bad), p, p, p, p, 2, 4, 4, ctypes.byref(S_(0.0, 0, 1.0)), p, p, None, p, ws,
                 None) == BAD_ARG                                                          # knobs are checked first


@pytest.mark.parametrize("sfx", ["f32", "tf32"])
def test_ragged_log_prob_entry_points_validate_arguments_without_a_gpu(sfx):
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    net, _layers = _net(p)
    n = ctypes.byref(net)
    q = getattr(lib, "vqb_prior_log_prob_workspace_bytes" + ("_tf32" if sfx == "tf32" else ""))
    ws = q(2, 4, 4, 32, 2, 16)
    assert ws > 0
    f = getattr(lib, "vqb_prior_log_prob_ragged_" + sfx)
    # (net, codes, labels, n_given, B, H, W, log_prob, workspace, bytes, stream)
    assert f(None, p, p, p, 2, 4, 4, p, p, ws, None) == BAD_ARG
    assert f(n, None, p, p, 2, 4, 4, p, p, ws, None) == BAD_ARG
    assert f(n, p, None, p, 2, 4, 4, p, p, ws, None) == BAD_ARG
    assert f(n, p, p, None, 2, 4, 4, p, p, ws, None) == BAD_ARG                          # NULL n_given
    assert f(n, p, p, p, 2, 4, 4, None, p, ws, None) == BAD_ARG                          # NULL log_prob
    assert f(n, p, p, p, 2, 4, 4, p, None, ws, None) == BAD_ARG
    for shape in ((0, 4, 4), (-2, 4, 4), (2, 0, 4), (2, 4, -1)):
        assert f(n, p, p, p, *shape, p, p, ws, None) == BAD_ARG, shape
    assert f(n, p, p, p, 2, 4, 4, p, p, ws - 4, None) == WS
    wide, _l = _net(p, dim=40)
    assert f(ctypes.byref(wide), p, p, p, 2, 4, 4, p, p, ws, None) == UNSUP

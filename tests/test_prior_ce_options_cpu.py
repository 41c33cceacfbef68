"""GatedPixelCNN.cross_entropy_ex (cross_entropy with weight, ignore_index and label_smoothing) without a GPU: the signature and docstring,
the host checks and their order (all before any CUDA call), the C ABI's checks and size queries for the _ex entry
points, and the fp64 restatement (tests/prior_ce_options_ref.py) against torch's F.cross_entropy, edge cases
included."""
import ctypes
import inspect
import itertools
import math

import pytest
import torch

from tests.prior_ce_options_ref import ce_options, torch_ce
from tests.test_prior_ce_cpu import BAD, UNSUP, WS, X, LAB, _grads, _header_text, _model, _net

K = 37                                  # tests.test_prior_ce_cpu._model's input_dim


def test_signature_and_docstring():
    from pixelcnn.models import GatedPixelCNN
    s = inspect.signature(GatedPixelCNN.cross_entropy_ex)
    assert list(s.parameters) == ["self", "x", "label", "reduction", "weight", "ignore_index", "label_smoothing"]
    for name, default in (("reduction", "mean"), ("weight", None), ("ignore_index", None), ("label_smoothing", 0.0)):
        assert s.parameters[name].kind is inspect.Parameter.KEYWORD_ONLY
        assert s.parameters[name].default == default
    doc = " ".join(GatedPixelCNN.cross_entropy_ex.__doc__.split())
    for phrase in ("nn.CrossEntropyLoss(weight=weight, ignore_index=ignore_index, label_smoothing=label_smoothing, "
                   "reduction=reduction)", "clamped", "differentiable and graph-capturable", "takes no gradient",
                   "torch's default is -100", "ignore_index=-100 gives torch's behaviour", "raw code", "NaN",
                   "same bits as cross_entropy"):
        assert phrase in doc, phrase
    doc = " ".join(GatedPixelCNN.cross_entropy.__doc__.split())
    assert "No weight, ignore_index or label_smoothing" not in doc and "use cross_entropy_ex" in doc


def test_option_errors_and_their_order():
    m = _model()
    bad_x = torch.zeros((5, 5), dtype=torch.int64)               # a rank error that comes after the options
    for bad in (-0.1, 1.5, float("nan"), float("inf"), "0.1", None, True, torch.tensor(0.1)):
        with pytest.raises(ValueError, match="label_smoothing"):
            m.cross_entropy_ex(bad_x, LAB, reduction="mean", label_smoothing=bad, ignore_index=1.5)
    with pytest.raises(ValueError, match="reduction"):          # the reduction comes first
        m.cross_entropy_ex(bad_x, LAB, reduction="batchmean", label_smoothing=2.0)
    for bad in (1.5, True, False, "3", torch.tensor(3)):        # ignore_index after label_smoothing
        with pytest.raises(ValueError, match="ignore_index"):
            m.cross_entropy_ex(bad_x, LAB, ignore_index=bad, weight=torch.ones(3))
    for bad in (torch.ones(K, 1), torch.ones(K + 1), torch.ones(()), [1.0] * K):   # weight's rank and length
        with pytest.raises(ValueError, match="weight"):
            m.cross_entropy_ex(bad_x, LAB, ignore_index=3, weight=bad)
    for dt in (torch.int64, torch.int32, torch.bool):
        with pytest.raises(ValueError, match="floating"):
            m.cross_entropy_ex(bad_x, LAB, weight=torch.ones(K, dtype=dt))
    meta = torch.ones(K, device="meta")
    with pytest.raises(RuntimeError, match="weight is on meta"):  # the device, before the rank of x
        m.cross_entropy_ex(bad_x, LAB, weight=meta)
    with pytest.raises(RuntimeError, match="shape"):
        m.cross_entropy_ex(bad_x, LAB, weight=torch.ones(K, dtype=torch.float64), ignore_index=-100, label_smoothing=1)


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_valid_options_on_cpu_tensors_raise_the_cuda_error(precision):
    opts = [dict(weight=torch.rand(K)), dict(ignore_index=-100), dict(label_smoothing=0.1),
            dict(weight=torch.ones(K, dtype=torch.float16), ignore_index=2 ** 70, label_smoothing=1)]
    for o, grad, r in itertools.product(opts, (False, True), ("none", "mean", "sum")):
        with torch.set_grad_enabled(grad), pytest.raises(RuntimeError, match="CUDA"):
            _model(precision).cross_entropy_ex(X, LAB, reduction=r, **o)


def test_header_declarations_and_struct_match_the_lib():
    import re
    from vqvae_b200 import _lib
    from tests.test_prior_ce_cpu import _CTYPES
    src = " ".join(_header_text().split())
    lib = _lib.lib()
    names = ["vqb_prior_ce_saved_bytes_ex", "vqb_prior_ce_workspace_bytes_ex", "vqb_prior_ce_workspace_bytes_ex_tf32",
             "vqb_prior_ce_forward_ex_f32", "vqb_prior_ce_forward_ex_tf32", "vqb_prior_ce_backward_ex_f32",
             "vqb_prior_ce_backward_ex_tf32"]
    for name in names:
        m = re.search(r"(\w+) " + name + r"\(([^)]*)\);", src)
        assert m, name
        ret, args = m.group(1), [a.strip() for a in m.group(2).split(",")]
        restype, argtypes = _lib.SIGNATURES[name]
        assert restype is getattr(_lib, _CTYPES[ret]), name
        assert argtypes == [_lib._vp if "*" in a else getattr(_lib, _CTYPES[a.rsplit(" ", 1)[0]]) for a in args], name
        assert hasattr(lib, name)
    assert ("typedef struct { const float *weight; int64_t ignore_index; int has_ignore; float label_smoothing; } "
            "vqb_prior_ce_options;") in src
    assert [f[0] for f in _lib.PriorCeOptions._fields_] == ["weight", "ignore_index", "has_ignore", "label_smoothing"]
    assert ctypes.sizeof(_lib.PriorCeOptions) == 24
    assert lib.vqb_abi_version() == 3


def _opts(weight=None, ignore=0, has_ignore=0, eps=0.0):
    from vqvae_b200 import _lib
    return _lib.PriorCeOptions(weight=weight, ignore_index=ignore, has_ignore=has_ignore, label_smoothing=eps)


@pytest.mark.parametrize("sfx", ["f32", "tf32"])
def test_ex_entry_points_validate_arguments_without_a_gpu(sfx):
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    fwd, bwd = getattr(lib, "vqb_prior_ce_forward_ex_" + sfx), getattr(lib, "vqb_prior_ce_backward_ex_" + sfx)
    q = getattr(lib, "vqb_prior_ce_workspace_bytes_ex" + ("_tf32" if sfx == "tf32" else ""))
    net, _l = _net(p)
    n = ctypes.byref(net)
    g, _g = _grads(p)
    gr = ctypes.byref(g)
    good = _opts(p.value, -100, 1, 0.1)
    o = ctypes.byref(good)
    sv, ws = lib.vqb_prior_ce_saved_bytes_ex(1, 4, 4, 32, 2, o), q(1, 4, 4, 32, 2, 16, 1, o)
    bws = lib.vqb_prior_ce_backward_workspace_bytes(n, 1, 4, 4)

    def f(*a):
        return fwd(*a[:7], o, *a[7:])
    # the no-options checks, in their order, with options
    assert f(None, p, p, 1, 4, 4, 1, p, p, sv, p, ws, None) == BAD
    assert f(n, None, p, 1, 4, 4, 1, p, p, sv, p, ws, None) == BAD
    assert f(n, p, None, 1, 4, 4, 1, p, p, sv, p, ws, None) == BAD
    assert f(n, p, p, 1, 4, 4, 1, None, p, sv, p, ws, None) == BAD
    assert f(n, p, p, 1, 4, 4, 1, p, p, sv, None, ws, None) == BAD
    for r in (-1, 3):
        assert f(n, p, p, 1, 4, 4, r, p, p, sv, p, ws, None) == BAD
        assert bwd(n, p, p, 1, 4, 4, r, o, p, p, gr, p, bws, None) == BAD
    assert bwd(n, p, p, 1, 4, 4, 1, o, None, p, gr, p, bws, None) == BAD
    assert bwd(n, p, p, 1, 4, 4, 1, o, p, None, gr, p, bws, None) == BAD
    assert bwd(n, p, p, 1, 4, 4, 1, o, p, p, None, p, bws, None) == BAD
    # the options: smoothing outside [0, 1] or NaN, has_ignore not 0/1; before the sizes
    for bad in (_opts(eps=-1e-7), _opts(eps=1.0000001), _opts(eps=float("nan")), _opts(eps=float("inf")),
                _opts(has_ignore=2), _opts(has_ignore=-1)):
        assert fwd(n, p, p, 1, 4, 4, 1, ctypes.byref(bad), p, p, 0, p, 0, None) == BAD
        assert bwd(n, p, p, 1, 4, 4, 1, ctypes.byref(bad), p, p, gr, p, 0, None) == BAD
    for edge in (_opts(eps=0.0), _opts(eps=1.0, has_ignore=1)):             # valid: the size checks are reached
        assert fwd(n, p, p, 1, 4, 4, 1, ctypes.byref(edge), p, p, 0, p, ws, None) == WS
    # the sizes with options
    assert f(n, p, p, 1, 4, 4, 1, p, p, sv - 4, p, ws, None) == WS
    assert f(n, p, p, 1, 4, 4, 1, p, p, sv, p, ws - 4, None) == WS
    assert f(n, p, p, 1, 4, 4, 1, p, p, lib.vqb_prior_ce_saved_bytes(1, 4, 4, 32, 2), p, ws, None) == WS
    assert bwd(n, p, p, 1, 4, 4, 1, o, p, p, gr, p, bws - 4, None) == WS
    # K = 8193 is unsupported, the net checked first, as without options
    big, _b = _net(p, K=8193)
    assert fwd(ctypes.byref(big), None, p, 1, 4, 4, 7, ctypes.byref(_opts(has_ignore=5)), p, p, sv, p, ws, None) == UNSUP
    assert bwd(ctypes.byref(big), p, p, 1, 4, 4, 1, o, p, p, gr, p, bws, None) == UNSUP
    # a NULL options pointer is the call without options: its checks and sizes
    sv0 = lib.vqb_prior_ce_saved_bytes(1, 4, 4, 32, 2)
    ws0 = getattr(lib, "vqb_prior_ce_workspace_bytes" + ("_tf32" if sfx == "tf32" else ""))(1, 4, 4, 32, 2, 16, 1)
    assert fwd(n, p, p, 1, 4, 4, 1, None, p, p, sv0 - 4, p, ws0, None) == WS
    assert fwd(n, p, p, 1, 4, 4, 1, None, p, p, sv0, p, ws0 - 4, None) == WS
    assert bwd(n, p, p, 1, 4, 4, 3, None, p, p, gr, p, bws, None) == BAD


def test_ex_size_queries():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    good = _opts(None, 0, 0, 0.5)
    o = ctypes.byref(good)
    for shape in ((1, 4, 4, 32, 2, 16), (32, 8, 8, 64, 15, 512), (16, 64, 64, 64, 2, 8192), (3, 1, 1, 32, 1, 8192),
                  (1, 3, 3, 32, 1, 37)):
        B, H, W, dim, L, Kq = shape
        npos = B * H * W
        base = lib.vqb_prior_ce_saved_bytes(B, H, W, dim, L)
        assert lib.vqb_prior_ce_saved_bytes_ex(B, H, W, dim, L, None) == base
        assert lib.vqb_prior_ce_saved_bytes_ex(B, H, W, dim, L, o) == base + 8
        lp = lib.vqb_prior_log_prob_workspace_bytes_tf32(*shape)
        splits = (lp - lib.vqb_prior_workspace_bytes_tf32(*shape)) // (12 * npos)
        for train in (0, 1):
            for ex, plain, s in ((lib.vqb_prior_ce_workspace_bytes_ex, lib.vqb_prior_ce_workspace_bytes, 1),
                                 (lib.vqb_prior_ce_workspace_bytes_ex_tf32, lib.vqb_prior_ce_workspace_bytes_tf32,
                                  splits)):
                b = plain(*shape, train)
                assert ex(*shape, train, None) == b
                assert ex(*shape, train, o) == -(-(b + 4 * npos) // 8) * 8 + 8 * npos * s
    for q in (lib.vqb_prior_ce_workspace_bytes_ex, lib.vqb_prior_ce_workspace_bytes_ex_tf32):
        assert q(0, 4, 4, 32, 2, 16, 1, o) == 0 and q(1, 4, 4, 32, 2, 0, 0, o) == 0
    assert lib.vqb_prior_ce_saved_bytes_ex(1, 4, 4, 0, 2, o) == 0


# ---- the fp64 restatement against torch ---------------------------------------------------------------------------
def _close(a, b, rel=1e-12):
    a, b = a.double(), b.double()
    if a.dim() == 0 and math.isnan(float(b)):
        return math.isnan(float(a))
    return bool(((a - b).abs() <= rel * b.abs().clamp_min(1.0)).all())


def _inputs(seed=0, N=60, Kq=9):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn((N, Kq), generator=g, dtype=torch.float64) * 3 + 40.0     # a large common offset
    codes = torch.randint(-3, Kq + 3, (N,), generator=g)
    codes[::7] = -100
    return logits, codes, g


def test_restatement_equals_torch_for_every_combination():
    logits, codes, g = _inputs()
    Kq = logits.shape[1]
    weights = [None, torch.rand(Kq, generator=g, dtype=torch.float64) + 0.1,
               torch.where(torch.rand(Kq, generator=g) < 0.4, 0.0, 1.0).double() * 2.5]
    for w, ig, e, r in itertools.product(weights, (None, -100, 4, Kq + 1), (0.0, 0.1, 1.0), ("none", "sum", "mean")):
        want = torch_ce(logits, codes, w, ig, e, r)
        got = ce_options(logits, codes, w, ig, e, r)
        assert _close(got, want), (w is None, ig, e, r)


def test_restatement_edge_cases_and_gradients_match_torch():
    logits, codes, g = _inputs(1, N=24, Kq=6)
    Kq = logits.shape[1]
    # every position ignored: "mean" is NaN with zero gradients, "sum" and "none" are 0
    allig = torch.full_like(codes, 5)
    for e in (0.0, 0.3):
        assert math.isnan(float(ce_options(logits, allig, None, 5, e, "mean")))
        t = logits.clone().requires_grad_()
        with torch.enable_grad():
            loss = torch_ce(t, allig, None, 5, e, "mean")
            loss.backward()
        assert math.isnan(float(loss)) and torch.equal(t.grad, torch.zeros_like(t.grad))
        assert float(ce_options(logits, allig, None, 5, e, "sum")) == 0.0 == float(torch_ce(logits, allig, None, 5,
                                                                                             e, "sum"))
    # scored targets whose weights sum to 0: a NaN loss and NaN in the logits' gradient
    w = torch.ones(Kq, dtype=torch.float64)
    w[codes.clamp(0, Kq - 1)] = 0.0
    for e in (0.0, 0.2):
        assert math.isnan(float(ce_options(logits, codes, w, None, e, "mean")))
        t = logits.clone().requires_grad_()
        with torch.enable_grad():
            loss = torch_ce(t, codes, w, None, e, "mean")
            loss.backward()
        assert math.isnan(float(loss)) and torch.isnan(t.grad).any()
    # the backward formula of DESIGN §8.3 against torch's autograd, per reduction
    w = torch.rand(Kq, generator=g, dtype=torch.float64) + 0.2
    for ig, e, r in itertools.product((None, -100), (0.0, 0.25, 1.0), ("none", "sum", "mean")):
        up = torch.randn(codes.shape, generator=g, dtype=torch.float64)
        t = logits.clone().requires_grad_()
        with torch.enable_grad():
            loss = torch_ce(t, codes, w, ig, e, r)
            loss.backward(up if r == "none" else None)
        assert torch.allclose(t.grad, d_logits(logits, codes, w, ig, e, r, up), rtol=1e-12, atol=1e-15), (ig, e, r)


def d_logits(l, codes, w, ig, e, reduction, up):
    """g_p * (q * c_p - (1 - e) * w_y * onehot(y) - (e / K) * w), c_p = (1 - e) * w_y + (e / K) * W (DESIGN §8.3)"""
    N, Kq = l.shape
    y = codes.clamp(0, Kq - 1)
    ign = codes == ig if ig is not None else torch.zeros(N, dtype=torch.bool)
    q = torch.softmax(l, 1)
    wy = w[y]
    g = up if reduction == "none" else torch.ones(N, dtype=torch.float64)
    if reduction == "mean":
        g = g / torch.where(ign, 0.0, wy).sum()
    g = torch.where(ign, 0.0, g)
    c = (1 - e) * wy + e / Kq * w.sum()
    d = q * c[:, None] - e / Kq * w[None, :]
    d[torch.arange(N), y] -= (1 - e) * wy
    return d * g[:, None]

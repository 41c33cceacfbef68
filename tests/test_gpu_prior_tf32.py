"""The Gated PixelCNN prior in TF32 (GatedPixelCNN.precision = "tf32") on the H100: logits and every gradient against
the emulated-TF32 restatement (tests/prior_tf32_port.py: prior_logits_tf32, fp64 accumulation), against plain
fp64 and the reference's gradient golden at loose bars, across PRIOR_SHAPE_CASES; bitwise grad-mode
logits, the documented launch counts, determinism, CUDA-graph capture, the reference's Adam loop, fp32 results
untouched by a round trip through "tf32", and generate unaffected by the mode."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle.prior_port import PRIOR_CASES, PRIOR_SHAPE_CASES, make_prior_inputs, make_prior_state_dict
from oracle.prior_train_port import leaf_params, prior_logits, prior_loss
from tests.prior_tf32_port import prior_logits_tf32

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# Bars, relative to the tensor's max |.|.  The logits follow the emulated restatement to within a few TF32 roundings
# (measured <= 8.6e-4 on an H100).  The gradients do so on shallow nets (<= 6.4e-4 on prior_ragged, <= 6e-6 on the
# one-layer cases), but once the GPU's fp32 activations and the fp64 restatement's round a value to different TF32
# neighbours, a ReLU or gate pre-activation near zero can take the other branch, and the head's weight gradients (sums
# over positions that largely cancel) move by up to 7.4e-2 of their max (DESIGN.md section 8.2).  A layout or indexing
# error moves a gradient by O(1).
LOGITS, GRADS = 2e-3, 1e-1              # against the emulated restatement
LOGITS_FP64, GRADS_FP64 = 5e-3, 2.5e-1  # against plain fp64 and the reference's golden


def _model(c, layers=None):
    import contextlib
    import io
    from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], layers)
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
        for i, (mask, k, residual) in enumerate(layers or []):
            m.layers[i] = GatedMaskedConv2d(mask, c["dim"], k, residual, c["n_classes"])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    m.precision = "tf32"
    codes, labels, _ = make_prior_inputs(c)
    return sd, m.cuda(), torch.from_numpy(codes), torch.from_numpy(labels)


def _upstream(c, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((c["batch"], c["K"], c["size"], c["size"]), generator=g, dtype=torch.float64)


def _rel(got, want):
    return float((got.double().cpu() - want).abs().max() / want.abs().max().clamp_min(1e-30))


def _reference(c, sd, x, lab, kind, tf32, layers=None):
    """fp64 logits and gradients of the restatement, emulated TF32 or plain."""
    with torch.enable_grad():
        g = leaf_params(sd, torch.float64)
        lg = (prior_logits_tf32 if tf32 else prior_logits)(g, x, lab, c["n_layers"], layers)
        (prior_loss(lg, x) if kind == "ce" else (lg * _upstream(c, 9)).sum()).backward()
    return lg.detach(), {k: v.grad for k, v in g.items()}


def _ours(c, m, x, lab, kind):
    xc, lc = x.cuda(), lab.cuda()
    m.zero_grad(set_to_none=True)
    with torch.enable_grad():
        out = m(xc, lc)
        if kind == "ce":
            prior_loss(out, xc).backward()
        else:
            out.backward(_upstream(c, 9).float().cuda())
    return out.detach(), {k: p.grad for k, p in m.named_parameters()}


@pytest.mark.parametrize("kind", ["ce", "random"])
@pytest.mark.parametrize("name", ["prior_ragged", "prior_default", "prior_cfg3"])
def test_logits_and_gradients_match_the_emulated_restatement(name, kind):
    c = PRIOR_CASES[name]
    sd, m, x, lab = _model(c)
    out, got = _ours(c, m, x, lab, kind)
    lg, want = _reference(c, sd, x, lab, kind, True)
    assert all(got[k].shape == want[k].shape and got[k].dtype == torch.float32 for k in want)
    errs = {k: _rel(got[k], want[k]) for k in want}
    worst = max(errs, key=errs.get)
    err_l = _rel(out, lg)
    print(f"{name} {kind}: logits {err_l:.2e}, worst gradient {errs[worst]:.2e} ({worst}) against emulated TF32")
    assert err_l <= LOGITS
    assert errs[worst] <= GRADS


@pytest.mark.parametrize("kind", ["ce", "random"])
@pytest.mark.parametrize("name", ["prior_ragged", "prior_default", "prior_cfg3"])
def test_logits_and_gradients_are_near_plain_fp64(name, kind):
    c = PRIOR_CASES[name]
    sd, m, x, lab = _model(c)
    out, got = _ours(c, m, x, lab, kind)
    lg, want = _reference(c, sd, x, lab, kind, False)
    errs = {k: _rel(got[k], want[k]) for k in want}
    worst = max(errs, key=errs.get)
    err_l = _rel(out, lg)
    print(f"{name} {kind}: logits {err_l:.2e}, worst gradient {errs[worst]:.2e} ({worst}) against plain fp64")
    assert err_l <= LOGITS_FP64
    assert errs[worst] <= GRADS_FP64


def test_gradients_are_near_the_reference_golden():
    c = PRIOR_CASES["prior_ragged"]
    sd, m, x, lab = _model(c)
    _, got = _ours(c, m, x, lab, "ce")
    with np.load(os.path.join(ROOT, "tests", "golden", "prior_grad_ragged.npz")) as d:
        want = {k[5:]: torch.from_numpy(d[k]).double() for k in d.files if k.startswith("grad/")}
    errs = {k: _rel(got[k], want[k]) for k in want}
    worst = max(errs, key=errs.get)
    print(f"prior_ragged: worst gradient {errs[worst]:.2e} ({worst}) against the reference's golden")
    assert errs[worst] <= GRADS_FP64


@pytest.mark.parametrize("name", [n for n, c in PRIOR_SHAPE_CASES.items() if "backward" in c.get("parts", ["backward"])])
def test_shape_range_matches_the_emulated_restatement(name):
    c = PRIOR_SHAPE_CASES[name]
    sd, m, x, lab = _model(c, c["layers"])
    out, got = _ours(c, m, x, lab, "random")
    lg, want = _reference(c, sd, x, lab, "random", True, c["layers"])
    errs = {k: _rel(got[k], want[k]) for k in want}
    worst = max(errs, key=errs.get)
    err_l = _rel(out, lg)
    print(f"{name}: logits {err_l:.2e}, worst gradient {errs[worst]:.2e} ({worst}) against emulated TF32")
    assert err_l <= LOGITS
    assert errs[worst] <= GRADS


def test_grad_mode_logits_are_the_inference_logits_and_launch_counts_are_documented():
    from vqvae_b200 import ops
    c = PRIOR_CASES["prior_default"]
    _, m, x, lab = _model(c)
    xc, lc = x.cuda(), lab.cuda()
    L = c["n_layers"]
    with torch.no_grad():
        ref = m(xc, lc)                             # packs the weights
        n0 = ops.launch_count()
        assert torch.equal(m(xc, lc), ref)
        assert ops.launch_count() - n0 == 3 + 4 * L
    with torch.enable_grad():
        n0 = ops.launch_count()
        out = m(xc, lc)
        assert ops.launch_count() - n0 == 3 + 4 * L
        n0 = ops.launch_count()
        out.backward(_upstream(c, 3).float().cuda())
        assert ops.launch_count() - n0 == 7 + 10 * L
    assert out.requires_grad and torch.equal(out.detach(), ref)


def test_backward_is_deterministic_and_captures_in_a_cuda_graph():
    c = PRIOR_CASES["prior_ragged"]
    _, m, x, lab = _model(c)
    xc, lc = x.cuda(), lab.cuda()
    G = _upstream(c, 5).float().cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    runs = []
    with torch.cuda.stream(s), torch.enable_grad():
        for _ in range(2):
            m.zero_grad(set_to_none=True)
            m(xc, lc).backward(G)
            runs.append({k: p.grad.clone() for k, p in m.named_parameters()})
    torch.cuda.current_stream().wait_stream(s)
    assert all(torch.equal(runs[0][k], runs[1][k]) for k in runs[0])
    m.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph), torch.enable_grad():
        m(xc, lc).backward(G)
    for p in m.parameters():
        p.grad.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(p.grad, runs[0][k]) for k, p in m.named_parameters())


def test_reference_adam_loop_tracks_fp64():
    c = PRIOR_CASES["prior_ragged"]
    sd, m, x, lab = _model(c)
    g = leaf_params(sd, torch.float64)
    opt64 = torch.optim.Adam(list(g.values()), lr=3e-4)
    opt = torch.optim.Adam(m.parameters(), lr=3e-4)
    xc, lc = x.cuda(), lab.cuda()
    got, want = [], []
    with torch.enable_grad():
        for _ in range(100):
            loss = prior_loss(prior_logits(g, x, lab, c["n_layers"]), x)
            opt64.zero_grad()
            loss.backward()
            opt64.step()
            want.append(loss.item())
            loss = prior_loss(m(xc, lc), xc)
            opt.zero_grad()
            loss.backward()
            opt.step()
            got.append(loss.item())
    rel = max(abs(a - b) / abs(b) for a, b in zip(got, want))
    print(f"adam tf32: loss {got[0]:.5f} -> {got[99]:.5f} @99 (fp64 {want[99]:.5f}); worst relative to fp64 {rel:.2e}")
    assert rel <= 5e-3


def test_a_round_trip_through_tf32_leaves_fp32_results_unchanged():
    c = PRIOR_CASES["prior_default"]
    _, m, x, lab = _model(c)
    m.precision = "fp32"
    twin = copy.deepcopy(m)
    m.precision = "tf32"
    _ours(c, m, x, lab, "random")
    with torch.no_grad():
        m(x.cuda(), lab.cuda())
    m.precision = "fp32"
    out, got = _ours(c, m, x, lab, "random")
    out2, want = _ours(c, twin, x, lab, "random")
    assert torch.equal(out, out2)
    assert all(torch.equal(got[k], want[k]) for k in want)


def test_precision_is_fixed_per_forward():
    """A backward runs in the precision its forward ran in, whatever the attribute says by then."""
    c = PRIOR_CASES["prior_ragged"]
    _, m, x, lab = _model(c)
    G = _upstream(c, 7).float().cuda()
    xc, lc = x.cuda(), lab.cuda()
    _ours(c, m, x, lab, "random")                  # packs
    want = []
    for mode in ("tf32", "fp32"):
        m.precision = mode
        m.zero_grad(set_to_none=True)
        with torch.enable_grad():
            m(xc, lc).backward(G)
        want.append({k: p.grad.clone() for k, p in m.named_parameters()})
    for first, other in (("tf32", "fp32"), ("fp32", "tf32")):
        m.precision = first
        m.zero_grad(set_to_none=True)
        with torch.enable_grad():
            out = m(xc, lc)
            m.precision = other
            out.backward(G)
        ref = want[0] if first == "tf32" else want[1]
        assert all(torch.equal(p.grad, ref[k]) for k, p in m.named_parameters())


def test_generate_is_the_same_under_either_precision_and_mask_a_is_rezeroed():
    c = PRIOR_CASES["prior_default"]
    _, m, x, lab = _model(c)
    l0 = m.layers[0]
    draws = []
    for mode in ("fp32", "tf32"):
        m.precision = mode
        torch.manual_seed(3)
        draws.append(m.generate(torch.arange(4, device="cuda") % c["n_classes"], shape=(8, 8), batch_size=4))
    assert torch.equal(draws[0], draws[1])
    opt = torch.optim.SGD(m.parameters(), lr=0.05)
    with torch.enable_grad():
        loss = prior_loss(m(x.cuda(), lab.cuda()), x.cuda())
        opt.zero_grad()
        loss.backward()
        opt.step()
    assert float(l0.vert_stack.weight[:, :, -1].abs().max()) > 0       # the step moved mask A's taps
    with torch.no_grad():
        m(x.cuda(), lab.cuda())
    assert float(l0.vert_stack.weight[:, :, -1].abs().max()) == 0
    assert float(l0.horiz_stack.weight[:, :, :, -1].abs().max()) == 0

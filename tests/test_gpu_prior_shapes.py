"""The Gated PixelCNN prior on the H100 across its documented shape range (oracle.prior_port.PRIOR_SHAPE_CASES):
dim up to 256, K from 1 to 8192, 1 to 32 layers, odd kernels up to 15 with either mask anywhere in the stack, up to 65
classes, grids from 1x1 to 64x64.  Per case: teacher-forced logits against the fp64 restatement, the sampler's step
logits against the forward and its draws against the fp64 CDF of those logits, and every gradient against fp64
autograd.  Plus a standalone GatedMaskedConv2d sweep, and the models the kernels refuse."""
import contextlib
import io
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.prior_port import PRIOR_SHAPE_CASES, make_prior_inputs, make_prior_state_dict, prior_forward
from oracle.prior_train_port import leaf_params, prior_logits, prior_loss

pytestmark = pytest.mark.gpu

ALL_PARTS = ("forward", "sampler", "backward")


def _cases(part):
    return [n for n, c in PRIOR_SHAPE_CASES.items() if part in c.get("parts", ALL_PARTS)]


def _bar(name):
    """The training bars of test_gpu_prior_train.py: 2e-5 of max |ref|, 1e-4 where the chains are long (2*dim = 512
    and a 512 -> 8192 head; 32 layers; cfg3's 15 layers at 64x64)."""
    return 1e-4 if name in ("wide", "deep", "cfg3_sampler") else 2e-5


def _model(c):
    """GatedPixelCNN of a case with layers[i] replaced by GatedMaskedConv2d(mask, dim, kernel, residual, n_classes),
    holding the case's seeded weights (mask A's taps non-zero until the first forward zeroes them)."""
    from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], c["layers"])
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
    for i, (mask, k, residual) in enumerate(c["layers"]):
        m.layers[i] = GatedMaskedConv2d(mask, c["dim"], k, residual, c["n_classes"])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    codes, labels, _ = make_prior_inputs(c)
    return sd, m.cuda(), torch.from_numpy(codes), torch.from_numpy(labels)


def _rel(got, want):
    """max |got - want| / max |want|"""
    return float((got.double().cpu() - want).abs().max() / want.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("name", _cases("forward"))
def test_forward_matches_fp64(name):
    from vqvae_b200 import ops
    c = PRIOR_SHAPE_CASES[name]
    sd, m, x, lab = _model(c)
    xc, lc = x.cuda(), lab.cuda()
    L = c["n_layers"]
    with torch.no_grad():
        out = m(xc, lc)                             # packs the weights (and zeroes mask A's taps)
        n0 = ops.launch_count()
        assert torch.equal(m(xc, lc), out)
        assert ops.launch_count() - n0 == 2 + 2 * L
    assert out.shape == (c["batch"], c["K"], c["size"], c["size"])
    want = prior_forward(sd, x, lab, L, torch.float64, c["layers"])
    err = _rel(out, want)
    cpu = _rel(prior_forward(sd, x, lab, L, torch.float32, c["layers"]), want)
    print(f"{name} forward: |l - l64| / max|l64| = {err:.2e} (fp32 CPU torch {cpu:.2e})")
    with torch.enable_grad():
        n0 = ops.launch_count()
        g = m(xc, lc)
        assert ops.launch_count() - n0 == 2 + 2 * L
    assert g.requires_grad and torch.equal(g.detach(), out)
    assert err <= _bar(name)


@pytest.mark.parametrize("name", _cases("sampler"))
def test_sampler_steps_are_the_forward_and_invert_the_fp64_cdf(name):
    from vqvae_b200 import ops
    c = PRIOR_SHAPE_CASES[name]
    _, m, _, _ = _model(c)
    B, S, K, L = c["batch"], c["size"], c["K"], c["n_layers"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    torch.manual_seed(c["xseed"])
    u = torch.rand((B, S, S), device="cuda")
    step = torch.full((B, S, S, K), float("nan"), device="cuda")
    with torch.no_grad():
        codes = m._sample(labels, u, step)
        n0 = ops.launch_count()
        assert torch.equal(m._sample(labels, u), codes)          # step_logits changes nothing
        assert ops.launch_count() - n0 == S * (L + S)
        fwd = m(codes, labels).permute(0, 2, 3, 1)
    assert codes.dtype == torch.int64 and codes.shape == (B, S, S)
    assert int(codes.min()) >= 0 and int(codes.max()) < K
    bad = (step != fwd).any(-1)
    if bool(bad.any()):
        rows = sorted(set(torch.nonzero(bad)[:, 1].tolist()))
        pytest.fail(f"{name}: step_logits differ from forward(codes) at {int(bad.sum())} of {B * S * S} positions, "
                    f"in rows {rows[0]}..{rows[-1]}")
    # each draw against the fp64 softmax of its own logits: CDF_{k-1} <= u < CDF_k, up to a bound on the fp32
    # running sum of ceil(K/32) terms per lane after a 32-lane scan
    cdf = torch.cumsum(torch.softmax(step.double().cpu(), -1), -1)
    k = codes.cpu()[..., None]
    hi = cdf.gather(-1, k)[..., 0]
    lo = torch.where(k[..., 0] > 0, cdf.gather(-1, (k - 1).clamp(min=0))[..., 0], torch.zeros_like(hi))
    uu = u.double().cpu()
    allow = max(1e-5, (math.ceil(K / 32) + 32) * 2.0 ** -23)
    ok = (lo <= uu) & (uu < hi)
    near = (lo - allow <= uu) & (uu < hi + allow)
    print(f"{name} sampler: {int((~ok).sum())} of {ok.numel()} draws needed the allowance {allow:.1e}")
    assert bool(near.all())


def _upstream(c, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((c["batch"], c["K"], c["size"], c["size"]), generator=g, dtype=torch.float64)


def _reference_grads(c, sd, x, lab, kind, dtype):
    with torch.enable_grad():
        g = leaf_params(sd, dtype)
        lg = prior_logits(g, x, lab, c["n_layers"], c["layers"])
        (prior_loss(lg, x) if kind == "ce" else (lg * _upstream(c, 9).to(dtype)).sum()).backward()
    return {k: v.grad for k, v in g.items()}


def _worst(got, want):
    return max(_rel(got[k], want[k]) for k in want)


@pytest.mark.parametrize("kind", ["ce", "random"])
@pytest.mark.parametrize("name", _cases("backward"))
def test_gradients_match_fp64_autograd(name, kind):
    from vqvae_b200 import ops
    c = PRIOR_SHAPE_CASES[name]
    sd, m, x, lab = _model(c)
    want = _reference_grads(c, sd, x, lab, kind, torch.float64)
    cpu = _worst(_reference_grads(c, sd, x, lab, kind, torch.float32), want)
    xc, lc = x.cuda(), lab.cuda()
    with torch.enable_grad():
        out = m(xc, lc)
        n0 = ops.launch_count()
        if kind == "ce":
            prior_loss(out, xc).backward()
        else:
            out.backward(_upstream(c, 9).float().cuda())
        assert ops.launch_count() - n0 == 7 + 10 * c["n_layers"]
    got = {k: p.grad for k, p in m.named_parameters()}
    assert all(got[k].shape == want[k].shape and got[k].dtype == torch.float32 for k in want)
    if c["K"] == 1 and kind == "ce":                # log_softmax of one logit is 0: no gradient anywhere
        assert all(float(want[k].abs().max()) == 0 and float(got[k].abs().max()) == 0 for k in want)
        return
    worst = _worst(got, want)
    masked = 0.0
    for i, (mask, _, _) in enumerate(c["layers"]):
        if mask != "A":
            continue
        for key, sl in ((f"layers.{i}.vert_stack.weight", np.s_[:, :, -1]),
                        (f"layers.{i}.horiz_stack.weight", np.s_[:, :, :, -1])):
            assert float(want[key][sl].abs().max()) > 0, key
            masked = max(masked, float((got[key].double().cpu() - want[key])[sl].abs().max() / want[key].abs().max()))
    print(f"{name} {kind}: worst |g - g64| / max|g64| = {worst:.2e} (mask A taps {masked:.2e}; "
          f"fp32 CPU torch {cpu:.2e})")
    assert worst <= _bar(name)


def test_backward_is_bitwise_reproducible_over_many_weight_gradient_chunks():
    c = PRIOR_SHAPE_CASES["long"]
    _, m, x, lab = _model(c)
    xc, lc = x.cuda(), lab.cuda()
    G = _upstream(c, 3).float().cuda()
    runs = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        with torch.enable_grad():
            m(xc, lc).backward(G)
        runs.append({k: p.grad.clone() for k, p in m.named_parameters()})
    assert all(torch.equal(runs[0][k], runs[1][k]) for k in runs[0])


@pytest.mark.parametrize("first", [["B", 3, True], ["B", 7, False], ["A", 7, True]])
def test_generate_refuses_a_layer_0_that_reads_the_code_being_drawn(first):
    """The teacher-forced forward runs such a stack as the reference does; the sampler cannot, and raises before
    launching anything."""
    from vqvae_b200 import ops
    c = dict(PRIOR_SHAPE_CASES["narrow"])
    c["layers"] = [first] + c["layers"][1:]
    sd, m, x, lab = _model(c)
    with torch.no_grad():
        out = m(x.cuda(), lab.cuda())
        assert _rel(out, prior_forward(sd, x, lab, c["n_layers"], torch.float64, c["layers"])) <= 2e-5
        u = torch.rand((2, c["size"], c["size"]), device="cuda")
        n0 = ops.launch_count()
        with pytest.raises(RuntimeError, match="layer 0"):
            m._sample(torch.zeros(2, dtype=torch.int64, device="cuda"), u)
        assert ops.launch_count() == n0


def test_layers_with_another_class_count_are_refused():
    """One class count for the whole net: a layer with more classes than layer 0 would see its labels clamped to
    layer 0's count, where the reference indexes its own table."""
    from pixelcnn.models import GatedMaskedConv2d
    from vqvae_b200 import ops
    c = PRIOR_SHAPE_CASES["kernels"]
    _, m, x, lab = _model(c)
    m.layers[1] = GatedMaskedConv2d("B", c["dim"], 5, True, c["n_classes"] + 7).cuda()
    n0 = ops.launch_count()
    with torch.no_grad(), pytest.raises(RuntimeError, match="classes"):
        m(x.cuda(), lab.cuda())
    assert ops.launch_count() == n0


@pytest.mark.parametrize("size", [1, 7])
@pytest.mark.parametrize("dim", [32, 160, 256])
@pytest.mark.parametrize("residual", [True, False])
@pytest.mark.parametrize("kernel", [1, 3, 5, 15])
@pytest.mark.parametrize("mask", ["A", "B"])
def test_standalone_layer_matches_fp64(mask, kernel, residual, dim, size):
    from pixelcnn.models import GatedMaskedConv2d
    torch.manual_seed(1000 * kernel + dim + size + (mask == "A") + 2 * residual)
    layer = GatedMaskedConv2d(mask, dim, kernel, residual, n_classes=5).cuda()
    x_v = torch.randn((2, dim, size, size), device="cuda")
    x_h = torch.randn((2, dim, size, size), device="cuda")
    h = torch.tensor([4, 1], device="cuda")
    out_v, out_h = layer(x_v, x_h, h)
    p = {n: t.detach().cpu().double() for n, t in layer.state_dict().items()}     # mask A: zeroed by the call
    if mask == "A":
        assert p["vert_stack.weight"][:, :, -1].abs().max() == 0
        assert p["horiz_stack.weight"][:, :, :, -1].abs().max() == 0
    xv, xh, S, k = x_v.cpu().double(), x_h.cpu().double(), size, kernel
    e = p["class_cond_embedding.weight"][h.cpu()][:, :, None, None]
    g = lambda t: torch.tanh(t[:, :dim]) * torch.sigmoid(t[:, dim:])       # noqa: E731
    hv = F.conv2d(xv, p["vert_stack.weight"], p["vert_stack.bias"], 1, k // 2)[:, :, :S]
    hh = F.conv2d(xh, p["horiz_stack.weight"], p["horiz_stack.bias"], 1, (0, k // 2))[:, :, :, :S]
    o = g(F.conv2d(hv, p["vert_to_horiz.weight"], p["vert_to_horiz.bias"]) + hh + e)
    oh = F.conv2d(o, p["horiz_resid.weight"], p["horiz_resid.bias"]) + (xh if residual else 0)
    ev, eh = _rel(out_v, g(hv + e)), _rel(out_h, oh)
    assert ev <= 2e-5 and eh <= 2e-5, (ev, eh)

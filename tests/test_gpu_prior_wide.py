"""The Gated PixelCNN prior at dims above 256 on the H100: dim = 288, 576 (24**2) and 1024 (32**2), the reference
script's ``GatedPixelCNN(K, img_dim**2, n_layers)`` for 24x24 and 32x32 latents, on small grids.  Per dim: fp32
logits against the reference's goldens and the fp64 restatement; every gradient of forward and of cross_entropy
against fp64 autograd; bitwise-reproducible backwards; TF32 against the emulated restatement; the sampler's step
logits against the forward and its draws against the fp64 CDF, with and without knobs, and completion of generate's
prefix; log_prob and cross_entropy against fp64; a standalone GatedMaskedConv2d at dim = 1024; a captured training
step; and the script's own loop body on its own 24x24 and 32x32 grids."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.make_prior_wide_golden import PRIOR_WIDE_CASES
from oracle.prior_port import make_prior_inputs, make_prior_state_dict, prior_forward
from oracle.prior_train_port import leaf_params, prior_logits, prior_loss
from tests.prior_tf32_port import prior_logits_tf32
from tests.test_gpu_prior_sample import _check_contract, _check_log_prob

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = dict(PRIOR_WIDE_CASES)
# 2*dim = 576: three output channels per thread, the narrowest wide instantiation; K = 64
CASES["prior_wide_288"] = dict(K=64, dim=288, n_layers=2, n_classes=10, size=5, batch=3, wseed=74, xseed=75)
NAMES = ["prior_wide_288", "prior_wide_576", "prior_wide_1024"]
BAR = 1e-4                  # the shape tests' long-chain bar: 2*dim >= 576 deep products into a 512 -> K head
# test_gpu_prior_tf32.py's bars against the emulated restatement.  The head's output_conv.0 gradient is a sum over
# positions of relu'(hidden) * d_hidden * x_h: where the GPU's fp32 hidden value and the restatement's fp64 one round
# to different TF32 neighbours near zero, the ReLU takes the other branch, and over a 1024-deep input that moved it by
# up to 1.31e-1 of its max at dim = 1024 (DESIGN §8.4); it is held to that file's plain-fp64 bar instead.
LOGITS_TF32, GRADS_TF32, HEAD0_TF32 = 2e-3, 1e-1, 2.5e-1


def _model(name, precision="fp32"):
    from pixelcnn.models import GatedPixelCNN
    c = CASES[name]
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"])
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    m.precision = precision
    codes, labels, _ = make_prior_inputs(c)
    return c, sd, m.cuda(), torch.from_numpy(codes), torch.from_numpy(labels)


def _rel(got, want):
    return float((got.double().cpu() - want).abs().max() / want.abs().max().clamp_min(1e-30))


def _upstream(c, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((c["batch"], c["K"], c["size"], c["size"]), generator=g, dtype=torch.float64)


@pytest.mark.parametrize("name", NAMES)
def test_forward_matches_golden_and_fp64(name):
    from vqvae_b200 import ops
    c, sd, m, x, lab = _model(name)
    xc, lc = x.cuda(), lab.cuda()
    with torch.no_grad():
        out = m(xc, lc)
        n0 = ops.launch_count()
        assert torch.equal(m(xc, lc), out)
        assert ops.launch_count() - n0 == 2 + 2 * c["n_layers"]
    want = prior_forward(sd, x, lab, c["n_layers"], torch.float64)
    err = _rel(out, want)
    gold = os.path.join(ROOT, "tests", "golden", name + ".npz")
    errg = _rel(out, torch.from_numpy(np.load(gold)["logits"]).double()) if os.path.exists(gold) else float("nan")
    print(f"{name} forward: {err:.2e} of fp64, {errg:.2e} of the reference's golden")
    assert err <= BAR
    assert not errg > BAR


def _reference_grads(c, sd, x, lab, kind):
    with torch.enable_grad():
        g = leaf_params(sd, torch.float64)
        lg = prior_logits(g, x, lab, c["n_layers"])
        (prior_loss(lg, x) if kind == "ce" else (lg * _upstream(c, 9)).sum()).backward()
    return {k: v.grad for k, v in g.items()}


def _grads(m):
    return {k: p.grad.detach().clone() for k, p in m.named_parameters()}


@pytest.mark.parametrize("kind", ["forward_ce", "forward_random", "cross_entropy"])
@pytest.mark.parametrize("name", NAMES)
def test_gradients_match_fp64_autograd(name, kind):
    c, sd, m, x, lab = _model(name)
    want = _reference_grads(c, sd, x, lab, "random" if kind == "forward_random" else "ce")
    xc, lc = x.cuda(), lab.cuda()
    runs = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        with torch.enable_grad():
            if kind == "cross_entropy":
                m.cross_entropy(xc, lc).backward()
            elif kind == "forward_ce":
                prior_loss(m(xc, lc), xc).backward()
            else:
                m(xc, lc).backward(_upstream(c, 9).float().cuda())
        runs.append(_grads(m))
    assert all(torch.equal(runs[0][k], runs[1][k]) for k in want), "two backward passes differ"
    errs = {k: _rel(runs[0][k], want[k]) for k in want}
    worst = max(errs, key=errs.get)
    print(f"{name} {kind}: worst |g - g64| / max|g64| = {errs[worst]:.2e} ({worst})")
    assert errs[worst] <= BAR


@pytest.mark.parametrize("kind", ["ce", "random"])
@pytest.mark.parametrize("name", NAMES)
def test_tf32_matches_the_emulated_restatement(name, kind):
    c, sd, m, x, lab = _model(name, "tf32")
    xc, lc = x.cuda(), lab.cuda()
    with torch.enable_grad():
        g = leaf_params(sd, torch.float64)
        lg = prior_logits_tf32(g, x, lab, c["n_layers"])
        (prior_loss(lg, x) if kind == "ce" else (lg * _upstream(c, 9)).sum()).backward()
        out = m(xc, lc)
        prior_loss(out, xc).backward() if kind == "ce" else out.backward(_upstream(c, 9).float().cuda())
    errs = {k: _rel(p.grad, g[k].grad) for k, p in m.named_parameters()}
    worst = max(errs, key=errs.get)
    err_l = _rel(out.detach(), lg.detach())
    print(f"{name} tf32 {kind}: logits {err_l:.2e}, worst gradient {errs[worst]:.2e} ({worst})")
    assert err_l <= LOGITS_TF32
    assert max(e for k, e in errs.items() if not k.startswith("output_conv.0.")) <= GRADS_TF32
    assert errs[worst] <= HEAD0_TF32


@pytest.mark.parametrize("name", NAMES)
def test_log_prob_and_cross_entropy(name):
    for precision in ("fp32", "tf32"):
        c, sd, m, x, lab = _model(name, precision)
        xc, lc = x.cuda(), lab.cuda()
        with torch.no_grad():
            pos = m.log_prob(xc, lc, per_position=True)
            total = m.log_prob(xc, lc)
            none = m.cross_entropy(xc, lc, reduction="none")
            logits = m(xc, lc)
        assert torch.equal(none, -pos)
        lg = (prior_logits_tf32 if precision == "tf32" else prior_logits)(leaf_params(sd, torch.float64), x, lab,
                                                                           c["n_layers"]).detach()
        want = F.log_softmax(lg, 1).gather(1, x[:, None])[:, 0]
        own = F.log_softmax(logits.double().cpu(), 1).gather(1, x[:, None])[:, 0]
        err, err_own = float((pos.double().cpu() - want).abs().max()), float((pos.double().cpu() - own).abs().max())
        print(f"{name} {precision} log_prob: {err:.2e} from the fp64 restatement, {err_own:.2e} from its own logits")
        assert err_own <= 1e-5
        assert err <= (1e-4 if precision == "fp32" else 5e-2)
        np.testing.assert_allclose(total.double().cpu().numpy(), pos.double().sum((1, 2)).cpu().numpy(), rtol=1e-5,
                                   atol=1e-4)


SETTINGS = [(1.0, None, None), (0.7, None, None), (1.0, 5, None), (1.0, None, 0.8), (1.5, 10, 0.9)]


@pytest.mark.parametrize("name", NAMES)
def test_sampler_steps_are_the_forward_and_invert_the_fp64_cdf(name):
    c, _, m, _, _ = _model(name)
    m.eval()
    B, S, K = c["batch"], c["size"], c["K"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    torch.manual_seed(c["xseed"])
    u = torch.rand((B, S, S), device="cuda")
    everywhere = torch.ones((B, S, S), dtype=torch.bool)
    with torch.no_grad():
        step = torch.full((B, S, S, K), float("nan"), device="cuda")
        gen = m._sample(labels, u, step)
        assert torch.equal(m(gen, labels).permute(0, 2, 3, 1), step), "generate's step logits are not the forward's"
        _check_contract(step, gen, u, everywhere, 1.0, None, None, f"{name} generate")
        for n_given in (S + 2, S * S - 1):
            done = m._complete(labels, u, gen, n_given)
            assert torch.equal(done, gen), f"completing {n_given} given positions of generate's output"
        for T, top_k, top_p in SETTINGS:
            step = torch.full((B, S, S, K), float("nan"), device="cuda")
            codes, lp = m._sample_with(labels, u, None, 0, T, top_k, top_p, step)
            if (T, top_k, top_p) == (1.0, None, None):
                assert torch.equal(codes, gen)
            assert torch.equal(m(codes, labels).permute(0, 2, 3, 1), step), (T, top_k, top_p)
            _check_contract(step, codes, u, everywhere, T, top_k, top_p, f"{name} sample {(T, top_k, top_p)}")
            _check_log_prob(step, codes, everywhere, lp, f"{name} sample {(T, top_k, top_p)}")
        T, top_k, top_p = SETTINGS[-1]
        given = S + 1
        step = torch.full((B, S, S, K), float("nan"), device="cuda")
        codes, lp = m._sample_with(labels, u, gen, given, T, top_k, top_p, step)
        assert torch.equal(codes.reshape(B, -1)[:, :given], gen.reshape(B, -1)[:, :given])
        sampled = torch.arange(S * S) >= given
        fwd = m(codes, labels).permute(0, 2, 3, 1)
        assert torch.equal(fwd.reshape(B, -1, K)[:, sampled], step.reshape(B, -1, K)[:, sampled])
        mask = sampled.reshape(1, S, S).expand(B, S, S)
        _check_contract(step, codes, u, mask, T, top_k, top_p, f"{name} sample_completion")
        _check_log_prob(step, codes, mask, lp, f"{name} sample_completion")


@pytest.mark.parametrize("kernel", [3, 7])
@pytest.mark.parametrize("mask", ["A", "B"])
def test_standalone_layer_at_dim_1024_matches_fp64(mask, kernel):
    from pixelcnn.models import GatedMaskedConv2d
    dim, S = 1024, 4
    torch.manual_seed(7 * kernel + (mask == "A"))
    layer = GatedMaskedConv2d(mask, dim, kernel, True, n_classes=5).cuda()
    x_v = torch.randn((2, dim, S, S), device="cuda", requires_grad=True)
    x_h = torch.randn((2, dim, S, S), device="cuda", requires_grad=True)
    h = torch.tensor([4, 1], device="cuda")
    gv, gh = torch.randn((2, dim, S, S), device="cuda"), torch.randn((2, dim, S, S), device="cuda")
    with torch.enable_grad():
        out_v, out_h = layer(x_v, x_h, h)
        (out_v * gv).sum().add((out_h * gh).sum()).backward()
    p = {n: t.detach().cpu().double().requires_grad_() for n, t in layer.state_dict().items()}
    xv = x_v.detach().cpu().double().requires_grad_()
    xh = x_h.detach().cpu().double().requires_grad_()
    g = lambda t: torch.tanh(t[:, :dim]) * torch.sigmoid(t[:, dim:])       # noqa: E731
    k = kernel
    with torch.enable_grad():
        e = p["class_cond_embedding.weight"][h.cpu()][:, :, None, None]
        hv = F.conv2d(xv, p["vert_stack.weight"], p["vert_stack.bias"], 1, k // 2)[:, :, :S]
        hh = F.conv2d(xh, p["horiz_stack.weight"], p["horiz_stack.bias"], 1, (0, k // 2))[:, :, :, :S]
        o = g(F.conv2d(hv, p["vert_to_horiz.weight"], p["vert_to_horiz.bias"]) + hh + e)
        ov, oh = g(hv + e), F.conv2d(o, p["horiz_resid.weight"], p["horiz_resid.bias"]) + xh
        (ov * gv.cpu().double()).sum().add((oh * gh.cpu().double()).sum()).backward()
    errs = {"out_v": _rel(out_v.detach(), ov.detach()), "out_h": _rel(out_h.detach(), oh.detach()),
            "x_v": _rel(x_v.grad, xv.grad), "x_h": _rel(x_h.grad, xh.grad)}
    errs.update({n: _rel(t.grad, p[n].grad) for n, t in layer.named_parameters()})
    worst = max(errs, key=errs.get)
    print(f"layer {mask}{kernel} dim 1024: worst {errs[worst]:.2e} ({worst})")
    assert errs["out_v"] <= 2e-5 and errs["out_h"] <= 2e-5, errs
    assert errs[worst] <= BAR, errs


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_captured_training_step_replays_the_eager_step(precision):
    from vqvae_b200.optim import Adam

    def steps(graph):
        _, _, m, x, lab = _model("prior_wide_1024", precision)
        xc, lc = x.cuda(), lab.cuda()
        opt = Adam(m.parameters(), lr=3e-4)

        def step():
            opt.zero_grad(set_to_none=True)
            with torch.enable_grad():
                m.cross_entropy(xc, lc).backward()
            opt.step()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            step()
            if graph:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    step()
        torch.cuda.current_stream().wait_stream(s)
        for _ in range(2):
            g.replay() if graph else step()
        torch.cuda.synchronize()
        return {k: p.detach().clone() for k, p in m.named_parameters()}
    eager, replayed = steps(False), steps(True)
    assert all(torch.equal(eager[k], replayed[k]) for k in eager)


@pytest.mark.parametrize("img_dim", [24, 32])
def test_the_reference_scripts_model_on_its_own_grid(img_dim):
    """gated_pixelcnn.py's model and loop body: GatedPixelCNN(512, img_dim**2, n_layers), forward, permute,
    nn.CrossEntropyLoss, backward, torch.optim.Adam; then generate on the same grid, decoded by a VQ-VAE."""
    from pixelcnn.models import GatedPixelCNN
    from models.vqvae import VQVAE
    torch.manual_seed(img_dim)
    with contextlib.redirect_stdout(io.StringIO()):
        model = GatedPixelCNN(512, img_dim ** 2, 2).cuda()
    sd = {k: v.detach().cpu().numpy().copy() for k, v in model.state_dict().items()}
    criterion = torch.nn.CrossEntropyLoss().cuda()
    opt = torch.optim.Adam(model.parameters(), lr=3e-4)
    x = torch.randint(0, 512, (2, img_dim, img_dim), device="cuda")
    label = torch.tensor([3, 7], device="cuda")
    with torch.enable_grad():
        logits = model(x, label)
        logits = logits.permute(0, 2, 3, 1).contiguous()
        loss = criterion(logits.view(-1, 512), x.view(-1))
        opt.zero_grad()
        loss.backward()
        opt.step()
    want = prior_loss(prior_logits(leaf_params(sd, torch.float64), x.cpu(), label.cpu(), 2), x.cpu()).detach()
    print(f"img_dim {img_dim}: loss {loss.item():.6f}, fp64 {float(want):.6f}")
    assert abs(loss.item() - float(want)) <= 1e-5 * abs(float(want))
    assert all(torch.isfinite(p).all() for p in model.parameters())
    with torch.no_grad():
        codes = model.generate(label, shape=(img_dim, img_dim), batch_size=2)
    assert codes.shape == (2, img_dim, img_dim) and 0 <= int(codes.min()) and int(codes.max()) < 512
    vq = VQVAE(128, 32, 2, 512, 64, 0.25).cuda().eval()
    with torch.no_grad():
        img = vq.decode(codes.reshape(-1, 1), (img_dim, img_dim))
    assert img.shape == (2, 3, 4 * img_dim, 4 * img_dim) and bool(torch.isfinite(img).all())

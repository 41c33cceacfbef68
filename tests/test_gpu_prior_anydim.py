"""The Gated PixelCNN prior at dims that are not a multiple of 32, on the H100.  Such a prior runs the kernels at
Cp = roundup(dim, 32) channels on zero-padded packings of its parameters (DESIGN §8.5), so every result must be bitwise
that of GatedPixelCNN(K, Cp) loaded with the zero-padded weights: logits in fp32 and TF32, log_prob, cross_entropy and
every gradient, the sampler's codes, log-probs and step logits, and Adam steps, eager and replayed from a CUDA graph.
Then, against fp64 and the reference: logits at the reference script's own dim = img_dim**2 against the goldens,
gradients against fp64 autograd, a standalone GatedMaskedConv2d, and the script's own loop body on its own grid.
Multiples of 32 keep their packings and launches."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.make_prior_anydim_golden import PRIOR_ANYDIM_CASES
from oracle.prior_port import make_prior_inputs, make_prior_state_dict, prior_forward
from oracle.prior_train_port import leaf_params, prior_logits, prior_loss
from tests.prior_anydim_port import pad_prior_state_dict, padded_dim, real_entries
from tests.prior_tf32_port import prior_logits_tf32

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAR = 1e-4                                      # test_gpu_prior_wide.py's bars
LOGITS_TF32, GRADS_TF32, HEAD0_TF32 = 2e-3, 1e-1, 2.5e-1

# dim -> (K, n_layers, grid, batch): small cases for the bitwise and gradient checks
SMALL = {16: (37, 3, 5, 3), 49: (64, 3, 7, 2), 100: (512, 2, 5, 2), 196: (64, 2, 5, 2), 784: (64, 2, 4, 2)}


def _build(K, dim, L, nc=10):
    from pixelcnn.models import GatedPixelCNN
    with contextlib.redirect_stdout(io.StringIO()):
        return GatedPixelCNN(K, dim, L, nc)


def _pair(dim, seed=0):
    """(case, state dict, the dim model, GatedPixelCNN(K, Cp) with the padded weights, codes, labels), on the GPU."""
    K, L, S, B = SMALL[dim]
    sd = make_prior_state_dict(K, dim, L, 10, 100 + dim + seed)
    m = _build(K, dim, L)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    mp = _build(K, padded_dim(dim), L)
    mp.load_state_dict({k: v.float() for k, v in pad_prior_state_dict(sd, dim).items()})
    rng = np.random.RandomState(dim)
    x = torch.from_numpy(rng.randint(0, K, size=(B, S, S))).cuda()
    lab = torch.from_numpy(rng.randint(0, 10, size=(B,))).cuda()
    return dict(K=K, L=L, S=S, B=B, dim=dim), sd, m.cuda(), mp.cuda(), x, lab


def _same_grads(m, mp, dim, what):
    gp = dict(mp.named_parameters())
    for k, p in m.named_parameters():
        full = gp[k].grad
        real = real_entries(full, k, dim)
        assert torch.equal(p.grad, real), f"{what}: {k}"
        assert int(torch.count_nonzero(full)) == int(torch.count_nonzero(real)), f"{what}: {k}'s padding gradient"


@pytest.mark.parametrize("dim", list(SMALL))
def test_bitwise_the_padded_native_model(dim):
    c, _, m, mp, x, lab = _pair(dim)
    B, S, K = c["B"], c["S"], c["K"]
    for precision in ("fp32", "tf32"):
        m.precision = mp.precision = precision
        with torch.no_grad():
            assert torch.equal(m(x, lab), mp(x, lab)), precision
            assert torch.equal(m.log_prob(x, lab), mp.log_prob(x, lab)), precision
            assert torch.equal(m.log_prob(x, lab, per_position=True), mp.log_prob(x, lab, per_position=True))
            ng = torch.tensor([0, S * S // 2, S + 1][:B], device="cuda")
            assert torch.equal(m.log_prob(x, lab, n_given=ng), mp.log_prob(x, lab, n_given=ng)), precision
            assert torch.equal(m.cross_entropy(x, lab, reduction="none"), mp.cross_entropy(x, lab, reduction="none"))
        for kind in ("cross_entropy", "forward"):
            up = torch.randn((B, K, S, S), generator=torch.Generator().manual_seed(3)).cuda()
            for model in (m, mp):
                model.zero_grad(set_to_none=True)
                with torch.enable_grad():
                    if kind == "cross_entropy":
                        loss = model.cross_entropy(x, lab)
                        loss.backward()
                    else:
                        model(x, lab).backward(up)
            _same_grads(m, mp, dim, f"dim {dim} {precision} {kind}")
    m.eval()
    mp.eval()
    m.precision = mp.precision = "fp32"         # the sampler is fp32: its step logits are the fp32 forward's
    torch.manual_seed(dim)
    u = torch.rand((B, S, S), device="cuda")
    with torch.no_grad():
        steps = [torch.full((B, S, S, K), float("nan"), device="cuda") for _ in range(2)]
        gen, genp = m._sample(lab, u, steps[0]), mp._sample(lab, u, steps[1])
        assert torch.equal(gen, genp) and torch.equal(steps[0], steps[1]), "generate"
        assert torch.equal(m(gen, lab).permute(0, 2, 3, 1), steps[0]), "generate's step logits are not the forward's"
        for n_given in (S + 1, torch.tensor([0, S * S - 2, 3][:B], device="cuda")):
            assert torch.equal(m._complete(lab, u, gen, n_given), mp._complete(lab, u, gen, n_given))
            assert torch.equal(m._complete(lab, u, gen, n_given), gen), "completion of generate's output"
        for knobs in ((1.0, None, None), (1.5, 10, 0.9)):
            steps = [torch.full((B, S, S, K), float("nan"), device="cuda") for _ in range(2)]
            a = m._sample_with(lab, u, None, 0, *knobs, steps[0])
            b = mp._sample_with(lab, u, None, 0, *knobs, steps[1])
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(steps[0], steps[1]), knobs
            ng = torch.tensor([1, S * S, S][:B], device="cuda")
            a = m._sample_with(lab, u, gen, ng, *knobs)
            b = mp._sample_with(lab, u, gen, ng, *knobs)
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), knobs


@pytest.mark.parametrize("dim", [49, 100])
def test_adam_steps_eager_and_replayed_are_the_padded_native_models(dim):
    from vqvae_b200.optim import Adam

    def run(model, graph, precision="fp32"):
        model.precision = precision
        opt = Adam(model.parameters(), lr=3e-3)
        x, lab = xs

        def step():
            opt.zero_grad(set_to_none=True)
            with torch.enable_grad():
                model.cross_entropy(x, lab).backward()
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
        return {k: p.detach().clone() for k, p in model.named_parameters()}

    for precision in ("fp32", "tf32"):
        _, _, m, mp, x, lab = _pair(dim)
        xs = (x, lab)
        native = run(mp, False, precision)
        eager = run(m, False, precision)
        _, _, m2, _, _, _ = _pair(dim)
        replayed = run(m2, True, precision)
        for k in eager:
            assert torch.equal(eager[k], replayed[k]), (precision, k)
            assert torch.equal(eager[k], real_entries(native[k], k, dim)), (precision, k)
            assert int(torch.count_nonzero(native[k])) == int(torch.count_nonzero(real_entries(native[k], k, dim))), k
        # the packings the steps refreshed are what the next forward reads
        with torch.no_grad():
            assert torch.equal(m(x, lab), mp(x, lab)), precision


def _rel(got, want):
    return float((got.double().cpu() - want).abs().max() / want.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("name", list(PRIOR_ANYDIM_CASES))
def test_script_dims_match_the_goldens_and_fp64(name):
    c = PRIOR_ANYDIM_CASES[name]
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"])
    m = _build(c["K"], c["dim"], c["n_layers"], c["n_classes"])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    m.cuda()
    codes, labels, pos = make_prior_inputs(c)
    x, lab = torch.from_numpy(codes), torch.from_numpy(labels)
    with torch.no_grad():
        out = m(x.cuda(), lab.cuda()).cpu()
    gold = torch.from_numpy(np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))["logits_at"]).double()
    want = prior_forward(sd, x, lab, c["n_layers"], torch.float64)
    err, errg = _rel(out, want), _rel(out[:, :, pos[:, 0], pos[:, 1]], gold)
    print(f"{name}: {err:.2e} of fp64, {errg:.2e} of the reference's golden")
    assert err <= BAR and errg <= BAR


@pytest.mark.parametrize("kind", ["forward", "cross_entropy"])
@pytest.mark.parametrize("dim", list(SMALL))
def test_gradients_match_fp64(dim, kind):
    c, sd, m, _, x, lab = _pair(dim, seed=1)
    xc, lc = x.cpu(), lab.cpu()
    up = torch.randn((c["B"], c["K"], c["S"], c["S"]), generator=torch.Generator().manual_seed(9), dtype=torch.float64)
    for precision in ("fp32", "tf32"):
        g = leaf_params(sd, torch.float64)
        with torch.enable_grad():
            lg = (prior_logits_tf32 if precision == "tf32" else prior_logits)(g, xc, lc, c["L"])
            (prior_loss(lg, xc) if kind == "cross_entropy" else (lg * up).sum()).backward()
        m.precision = precision
        m.zero_grad(set_to_none=True)
        with torch.enable_grad():
            if kind == "cross_entropy":
                m.cross_entropy(x, lab).backward()
            else:
                out = m(x, lab)
                out.backward(up.float().cuda())
        errs = {k: _rel(p.grad, g[k].grad) for k, p in m.named_parameters()}
        worst = max(errs, key=errs.get)
        print(f"dim {dim} {precision} {kind}: worst gradient {errs[worst]:.2e} ({worst})")
        if precision == "fp32":
            assert errs[worst] <= BAR
        else:
            assert max(e for k, e in errs.items() if not k.startswith("output_conv.0.")) <= GRADS_TF32
            assert errs[worst] <= HEAD0_TF32
            if kind == "forward":
                assert _rel(out.detach(), lg.detach()) <= LOGITS_TF32


@pytest.mark.parametrize("residual", [True, False])
@pytest.mark.parametrize("mask", ["A", "B"])
@pytest.mark.parametrize("dim", [40, 49])
def test_standalone_layer_matches_fp64(dim, mask, residual):
    from pixelcnn.models import GatedMaskedConv2d
    S, kernel = 5, 3 if mask == "B" else 5
    torch.manual_seed(dim + 7 * (mask == "A") + residual)
    layer = GatedMaskedConv2d(mask, dim, kernel, residual, n_classes=5).cuda()
    x_v = torch.randn((2, dim, S, S), device="cuda", requires_grad=True)
    x_h = torch.randn((2, dim, S, S), device="cuda", requires_grad=True)
    h = torch.tensor([4, 1], device="cuda")
    gv, gh = torch.randn((2, dim, S, S), device="cuda"), torch.randn((2, dim, S, S), device="cuda")
    with torch.no_grad():
        inf_v, inf_h = layer(x_v, x_h, h)
    with torch.enable_grad():
        out_v, out_h = layer(x_v, x_h, h)
        (out_v * gv).sum().add((out_h * gh).sum()).backward()
    assert torch.equal(inf_v, out_v.detach()) and torch.equal(inf_h, out_h.detach())
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
        r = F.conv2d(o, p["horiz_resid.weight"], p["horiz_resid.bias"])
        ov, oh = g(hv + e), (r + xh if residual else r)
        (ov * gv.cpu().double()).sum().add((oh * gh.cpu().double()).sum()).backward()
    errs = {"out_v": _rel(out_v.detach(), ov.detach()), "out_h": _rel(out_h.detach(), oh.detach()),
            "x_v": _rel(x_v.grad, xv.grad), "x_h": _rel(x_h.grad, xh.grad)}
    errs.update({n: _rel(t.grad, p[n].grad) for n, t in layer.named_parameters()})
    worst = max(errs, key=errs.get)
    print(f"layer {mask}{kernel} residual={residual} dim {dim}: worst {errs[worst]:.2e} ({worst})")
    assert errs["out_v"] <= 2e-5 and errs["out_h"] <= 2e-5, errs
    assert errs[worst] <= BAR, errs


@pytest.mark.parametrize("img_dim", [4, 7, 12, 14, 20, 28])
def test_the_reference_scripts_model_on_its_own_grid(img_dim):
    """gated_pixelcnn.py's model and loop body: GatedPixelCNN(512, img_dim**2, n_layers), forward, permute,
    nn.CrossEntropyLoss, backward, torch.optim.Adam; then generate on the same grid, decoded by a VQ-VAE."""
    from models.vqvae import VQVAE
    torch.manual_seed(img_dim)
    model = _build(512, img_dim ** 2, 2).cuda()
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
    with torch.no_grad():
        want = prior_loss(prior_logits(leaf_params(sd, torch.float64), x.cpu(), label.cpu(), 2), x.cpu())
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


def test_multiples_of_32_keep_their_packings_and_launches():
    """At dim 64 no padded packing is ever made and a training step's launches are the parent's; at dim 49 the only
    extra launch of a warm step is the gradients' unpadding, one per backward."""
    from vqvae_b200 import ops
    from vqvae_b200.optim import Adam
    counts = {}
    for dim in (64, 49):
        L, S = 3, 6
        m = _build(64, dim, L).cuda()
        x = torch.randint(0, 64, (2, S, S), device="cuda")
        lab = torch.tensor([1, 2], device="cuda")
        opt = Adam(m.parameters(), lr=1e-3)
        for _ in range(2):                          # the second step is warm: every packing exists
            n0 = ops.launch_count()
            with torch.no_grad():
                m(x, lab)
            n1 = ops.launch_count()
            opt.zero_grad(set_to_none=True)
            with torch.enable_grad():
                m.cross_entropy(x, lab).backward()
            n2 = ops.launch_count()
            opt.step()
            n3 = ops.launch_count()
        counts[dim] = (n1 - n0, n2 - n1, n3 - n2)
        keys = {k[0] for p in m.parameters() for k in getattr(p, "_vqb_packed", {})}
        assert keys == ({"prior"} if dim == 64 else {"prior_pad", "pad", "prior"}), (dim, keys)
    assert counts[64][0] == 2 + 2 * L and counts[64][2] == 2, counts
    assert counts[49] == (counts[64][0], counts[64][1] + 1, 2), counts

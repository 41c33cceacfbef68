"""GatedPixelCNN.complete on the H100: completing a prefix of the sampler's own output reproduces it bitwise (codes
and step logits) across the documented shape range, foreign prefixes are kept and conditioned on, the draws follow the
fp64 softmax, the launch count follows the schedule, seeds line up with generate, graph capture, and an
encode -> complete -> decode pipeline."""
import contextlib
import io

import numpy as np
import pytest
import torch

from oracle.prior_port import PRIOR_CASES, PRIOR_SHAPE_CASES, make_prior_state_dict, prior_forward

pytestmark = pytest.mark.gpu

SAMPLER_CASES = ["prior_default", "prior_ragged"] + \
    [n for n, c in PRIOR_SHAPE_CASES.items() if "sampler" in c.get("parts", ("sampler",))]


def _model(name):
    """(case, numpy state dict, layer list or None, GatedPixelCNN on cuda in eval mode)."""
    from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
    c = PRIOR_CASES.get(name) or PRIOR_SHAPE_CASES[name]
    layers = c.get("layers")
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], layers)
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
    for i, (mask, k, residual) in enumerate(layers or []):
        m.layers[i] = GatedMaskedConv2d(mask, c["dim"], k, residual, c["n_classes"])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return c, sd, layers, m.cuda().eval()


def _prefixes(H, W):
    return sorted({n for n in (1, W - 1, W, W + 1, H * W // 2, H * W - 1) if 0 <= n <= H * W})


def _launches(H, W, L, n):
    """The completion schedule's launch count for 0 < n < H*W."""
    i0, j0 = divmod(n, W)
    return 1 + L * (i0 > 0) + L * (H - i0) + L * (j0 > 0) + (H * W - n)


def _junk(x, n, K, seed):
    """x with every raster position >= n replaced by random codes, out-of-range ones included."""
    B, H, W = x.shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    junk = torch.randint(-3, K + 5, (B, H, W), device="cuda", generator=g)
    keep = (torch.arange(H * W, device="cuda") < n).view(1, H, W)
    return torch.where(keep, x, junk)


def _inverts_fp64_cdf(sd, layers, L, codes, labels, u, mask, what):
    """Every code at a True position of `mask` is the inverse fp64 CDF of the fp64 forward's logits on `codes`, within
    test_generate_inverts_the_fp64_cdf's 1e-5 of a boundary."""
    lg = prior_forward(sd, codes.cpu(), labels.cpu(), L, torch.float64, layers)
    cdf = torch.cumsum(torch.softmax(lg, 1), 1)                       # (B, K, H, W)
    k = codes.cpu()[:, None]
    hi = cdf.gather(1, k)[:, 0]
    lo = torch.where(k[:, 0] > 0, cdf.gather(1, (k - 1).clamp(min=0))[:, 0], torch.zeros_like(hi))
    uu = u.double().cpu()
    ok = (lo <= uu) & (uu < hi)
    near = torch.minimum((uu - lo).abs(), (uu - hi).abs()) < 1e-5
    m = mask.cpu()
    print(f"{what}: {int((~ok & m).sum())} of {int(m.sum())} draws within 1e-5 of a CDF boundary")
    assert bool((ok | near | ~m).all())


@pytest.mark.parametrize("name", SAMPLER_CASES)
def test_completing_a_prefix_of_the_samplers_output_reproduces_it(name):
    from vqvae_b200 import ops
    c, _, _, m = _model(name)
    B, S, K, L = c["batch"], c["size"], c["K"], c["n_layers"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    torch.manual_seed(c["xseed"] + 1000)
    u = torch.rand((B, S, S), device="cuda")
    with torch.no_grad():
        step_g = torch.full((B, S, S, K), float("nan"), device="cuda")
        g = m._sample(labels, u, step_g)
        pos = torch.arange(S * S, device="cuda").view(1, S, S, 1)
        for n in _prefixes(S, S):
            x = _junk(g, n, K, seed=n)
            x_before = x.clone()
            step_c = torch.full((B, S, S, K), float("nan"), device="cuda")
            n0 = ops.launch_count()
            out = m._complete(labels, u, x, n, step_c)
            launches = ops.launch_count() - n0
            assert torch.equal(x, x_before)                              # x is not modified
            assert out.dtype == torch.int64 and out.shape == (B, S, S)
            if not torch.equal(out, g):
                bad = torch.nonzero((out != g).view(B, -1))[:, 1]
                pytest.fail(f"{name} n_given={n}: {int(bad.numel())} codes differ, first at raster position "
                            f"{int(bad.min())}")
            after = (pos >= n).expand_as(step_c)
            diff = (step_c != step_g) & after
            assert not bool(diff.any()), f"{name} n_given={n}: step logits differ at {int(diff.any(-1).sum())} positions"
            assert bool(torch.isnan(step_c[~after]).all())               # given positions untouched
            want = S * (L + S) if n == 0 else (0 if n == S * S else _launches(S, S, L, n))
            assert launches == want, (n, launches, want)


@pytest.mark.parametrize("name", ["prior_default", "prior_ragged"])
def test_foreign_prefixes_are_kept_and_conditioned_on(name):
    c, sd, _, m = _model(name)
    B, S, K, L = 6, c["size"], c["K"], c["n_layers"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    pos = torch.arange(S * S, device="cuda").view(1, S, S)
    for n in _prefixes(S, S):
        if n == S * S:
            continue
        gen = torch.Generator(device="cuda").manual_seed(200 + n)
        x = torch.randint(-4, K + 4, (B, S, S), device="cuda", generator=gen)    # out-of-range given codes too
        u = torch.rand((B, S, S), device="cuda", generator=gen)
        step = torch.full((B, S, S, K), float("nan"), device="cuda")
        with torch.no_grad():
            out = m._complete(labels, u, x, n, step)
            fwd = m(out.clamp(0, K - 1), labels).permute(0, 2, 3, 1)
        given = pos < n
        assert torch.equal(out[given.expand_as(out)], x[given.expand_as(x)])
        drawn = ~given.expand_as(out)
        assert int(out[drawn].min()) >= 0 and int(out[drawn].max()) < K
        after = drawn[..., None].expand_as(step)
        assert torch.equal(step[after], fwd[after])
        assert bool(torch.isnan(step[~after]).all())
        _inverts_fp64_cdf(sd, None, L, out.clamp(0, K - 1), labels, u, drawn, f"{name} n_given={n}")


def test_completion_distribution_chi_square():
    from scipy import stats
    c, sd, _, m = _model("prior_ragged")
    N, K, lab = 65536, c["K"], 1
    labels = torch.full((N,), lab, dtype=torch.int64, device="cuda")
    for first in (0, 5, K - 1):
        x = torch.zeros((N, 2, 2), dtype=torch.int64, device="cuda")
        x[:, 0, 0] = first
        torch.manual_seed(300 + first)
        with torch.no_grad():
            out = m.complete(x, labels, 1)
        assert bool((out[:, 0, 0] == first).all())
        counts = np.bincount(out[:, 0, 1].cpu().numpy(), minlength=K).astype(np.float64)
        grid = np.zeros((1, 2, 2), np.int64)
        grid[0, 0, 0] = first
        lg = prior_forward(sd, grid, np.array([lab]), c["n_layers"], dtype=torch.float64)
        p = torch.softmax(lg[0, :, 0, 1], 0).numpy()
        exp = p * N
        big = exp >= 5
        f_obs = np.append(counts[big], counts[~big].sum())
        f_exp = np.append(exp[big], exp[~big].sum())
        if f_exp[-1] == 0:
            f_obs, f_exp = f_obs[:-1], f_exp[:-1]
        assert counts[~big].sum() <= max(50.0, 10 * exp[~big].sum())
        pval = stats.chisquare(f_obs, f_exp * f_obs.sum() / f_exp.sum()).pvalue
        print(f"given first code {first}: chi-square p = {pval:.4f}")
        assert pval > 1e-3


def test_edges_and_launch_counts():
    from vqvae_b200 import ops
    c, _, _, m = _model("prior_default")
    B, S, K, L = 16, c["size"], c["K"], c["n_layers"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    u = torch.rand((B, S, S), device="cuda")
    x = torch.randint(0, K, (B, S, S), device="cuda")
    with torch.no_grad():
        want = m._sample(labels, u)                                       # packs the weights
        n0 = ops.launch_count()
        got = m._complete(labels, u, x, 0)
        assert ops.launch_count() - n0 == S * (L + S)
        assert torch.equal(got, want)
        x32 = torch.randint(-5, K + 5, (B, S, S), device="cuda", dtype=torch.int32)
        n0 = ops.launch_count()
        got = m._complete(labels, u, x32, S * S)
        assert ops.launch_count() - n0 == 0
        assert got.dtype == torch.int64 and torch.equal(got, x32.long())
        got = m._complete(labels, u, x, S * S)
        assert torch.equal(got, x) and got.data_ptr() != x.data_ptr()
        assert _launches(8, 8, 15, 32) == 108 and _launches(64, 64, 15, 2048) == 2544
        for n in (1, 7, 8, 9, 31, 32, 33, 40, 63):
            n0 = ops.launch_count()
            m._complete(labels, u, x, n)
            assert ops.launch_count() - n0 == _launches(S, S, L, n), n


def test_seeds_line_up_with_generate():
    c, _, _, m = _model("prior_ragged")
    B, S = 4, c["size"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    with torch.no_grad():
        torch.manual_seed(7)
        g = m.generate(labels, shape=(S, S), batch_size=B)
        before = g.clone()
        for n in range(S * S + 1):
            torch.manual_seed(7)
            out = m.complete(g, labels, n)
            assert torch.equal(out, g), n
            r = torch.rand(1, device="cuda")
            torch.manual_seed(7)
            torch.rand((B, S, S), device="cuda")
            assert torch.equal(r, torch.rand(1, device="cuda")), n      # exactly one draw of (B, H, W)
        assert torch.equal(g, before)
        torch.manual_seed(7)
        assert torch.equal(m.complete(g, labels.tolist(), 3), g)          # labels as generate takes them


def test_graph_capture():
    c, _, _, m = _model("prior_default")
    B, S, K = 8, c["size"], c["K"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    for n in (5, 32):
        u = torch.rand((B, S, S), device="cuda")
        x = torch.randint(0, K, (B, S, S), device="cuda")
        with torch.no_grad():
            first = m._complete(labels, u, x, n)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = m._complete(labels, u, x, n)
            u.copy_(torch.rand_like(u))
            x.view(B, -1)[:, :n].copy_(torch.randint(0, K, (B, n), device="cuda"))
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, m._complete(labels, u, x, n))
            assert not torch.equal(out, first)


def test_encode_complete_decode_pipeline():
    """VQVAE.encode -> (B, 8, 8) codes -> complete the bottom half with the prior -> VQVAE.decode (fp32 mode), against
    the C oracle's decoder on the codebook rows of the completed codes."""
    from models.vqvae import VQVAE
    from oracle import cref
    from vqvae_b200.synth import make_images, make_state_dict
    c, _, _, m = _model("prior_default")
    hp = dict(h_dim=128, res_h_dim=32, n_res_layers=2, n_embeddings=512, embedding_dim=64)
    sd = make_state_dict(seed=0, codebook="normal", codebook_scale=0.05, **hp)
    vq = VQVAE(128, 32, 2, 512, 64, 0.25)
    vq.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    vq = vq.cuda().eval()
    B = 4
    images = torch.from_numpy(make_images(B, 32, seed=3)).cuda()
    with torch.no_grad():
        codes = vq.encode(images).view(B, 8, 8)
        torch.manual_seed(0)
        done = m.complete(codes, torch.arange(B, device="cuda"), 32)
        x = vq.decode(done.view(-1, 1), (8, 8))
    assert torch.equal(done[:, :4], codes[:, :4])
    assert int(done.min()) >= 0 and int(done.max()) < 512
    assert x.shape == (B, 3, 32, 32)
    E = np.asarray(sd["vector_quantization.embedding.weight"])
    zq = np.ascontiguousarray(E[done.cpu().numpy()].transpose(0, 3, 1, 2))
    np.testing.assert_allclose(x.cpu().numpy(), cref.decoder(zq, sd, 2), atol=2e-6, rtol=0)

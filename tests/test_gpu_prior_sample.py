"""GatedPixelCNN.sample / sample_completion on the H100: with default knobs they are generate / complete bit for bit;
with temperature, top-k and top-p every draw follows the fp64 restatement of the contract (tests/prior_sample_ref.py)
on its own step logits; a chi-square test of the truncated distribution; log_prob against fp64 and against the
teacher-forced cross-entropy; determinism, graph capture, launch counts, and completion of a sample's prefix."""
import contextlib
import io
import math

import numpy as np
import pytest
import torch

from oracle.prior_port import PRIOR_CASES, PRIOR_SHAPE_CASES, make_prior_state_dict
from tests import prior_sample_ref as ref

pytestmark = pytest.mark.gpu

# the sampler's shape cases: K from 1 to 8192 (wide: 8192, long and prior_default: 512, single: 1)
CASES = ["prior_default"] + [n for n, c in PRIOR_SHAPE_CASES.items() if "sampler" in c.get("parts", ("sampler",))]

# (temperature, top_k, top_p); top_k "K" is the case's K
SETTINGS = [(0.5, None, None), (2.0, None, None), (1.0, 1, None), (1.0, 5, None), (1.0, "K", None),
            (1.0, None, 0.1), (1.0, None, 0.9), (0.5, 5, 0.9), (2.0, "K", 0.1)]


def _model(name):
    from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
    c = PRIOR_CASES.get(name) or PRIOR_SHAPE_CASES[name]
    layers = c.get("layers")
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], layers)
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
    for i, (mask, k, residual) in enumerate(layers or []):
        m.layers[i] = GatedMaskedConv2d(mask, c["dim"], k, residual, c["n_classes"])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return c, m.cuda().eval()


def _setting(s, K):
    T, k, p = s
    return T, (K if k == "K" else None if k is None else min(k, K)), p


def _allowance(K):
    return max(1e-5, (math.ceil(K / 32) + 32) * 2.0 ** -23)


def _check_contract(step, codes, u, mask, T, top_k, top_p, what):
    """Every code at a True position of `mask` lies in the fp64 kept set S of its step logits and satisfies the
    renormalized CDF bracket, except draws within the allowance of a CDF boundary and, for the bracket, positions
    whose S changes when the top_p mass moves by the allowance (the code must then lie in the larger set)."""
    K = step.shape[-1]
    tol = _allowance(K)
    m = mask.reshape(-1).cpu().numpy()
    lg = step.reshape(-1, K).cpu().numpy()[m]
    c = codes.reshape(-1).cpu().numpy()[m]
    uu = u.reshape(-1).double().cpu().numpy()[m]
    rows = np.arange(len(c))
    S = ref.kept(lg, T, top_k, top_p)
    if top_p is not None and top_p < 1:
        lo, hi = ref.kept(lg, T, top_k, max(top_p - tol, 1e-9)), ref.kept(lg, T, top_k, min(top_p + tol, 1.0))
    else:
        lo = hi = S
    assert hi[rows, c].all(), f"{what}: {int((~hi[rows, c]).sum())} codes outside the kept set"
    stable = (lo == hi).all(-1)
    q = ref.probs(lg, T, top_k, top_p)
    cdf = np.cumsum(q, -1)
    up = cdf[rows, c]
    low = up - q[rows, c]
    ok = (low <= uu) & (uu < up)
    near = np.minimum(np.abs(uu - low), np.abs(uu - up)) < tol
    bad = ~(ok | near) & stable
    print(f"{what}: {int((~ok & stable).sum())} of {len(c)} draws near a CDF boundary, {int((~stable).sum())} "
          f"positions with a top_p flip")
    assert not bad.any(), f"{what}: {int(bad.sum())} draws outside their CDF bracket"


def _check_log_prob(step, codes, mask, log_prob, what):
    """log_prob = fp64 sum over the True positions of log_softmax(step logits)[code], within 1e-5 relative plus
    1e-6 per position."""
    B, K = step.shape[0], step.shape[-1]
    ls = ref.log_softmax64(step.reshape(B, -1, K).cpu().numpy())
    lp = np.take_along_axis(ls, codes.reshape(B, -1, 1).cpu().numpy(), -1)[..., 0]
    m = mask.reshape(1, -1).expand(B, -1).cpu().numpy() if mask.dim() == 1 else mask.reshape(B, -1).cpu().numpy()
    want = np.where(m, lp, 0.0).sum(-1)                    # given positions' step logits are NaN
    n = m.sum(-1)
    got = log_prob.double().cpu().numpy()
    assert (np.abs(got - want) <= 1e-5 * np.abs(want) + 1e-6 * n).all(), (what, got, want)
    return want


@pytest.mark.parametrize("name", CASES)
def test_default_knobs_are_generate_and_complete_bitwise(name):
    c, m = _model(name)
    B, S, K = c["batch"], c["size"], c["K"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    torch.manual_seed(c["xseed"] + 2000)
    u = torch.rand((B, S, S), device="cuda")
    with torch.no_grad():
        step_g = torch.full((B, S, S, K), float("nan"), device="cuda")
        g = m._sample(labels, u, step_g)
        step_s = torch.full_like(step_g, float("nan"))
        codes, lp = m._sample_with(labels, u, None, 0, 1.0, None, None, step_s)
        assert codes.dtype == torch.int64 and lp.dtype == torch.float32 and lp.shape == (B,)
        assert torch.equal(codes, g) and torch.equal(step_s, step_g)
        pos = torch.arange(S * S, device="cuda")
        _check_log_prob(step_g, g, pos >= 0, lp, name)
        for n in sorted({0, min(S - 1, 1), S - 1, min(2 * S + 1, S * S - 1), S * S}):
            x = torch.randint(0, K, (B, S, S), device="cuda")
            x.view(B, -1)[:, :n] = g.view(B, -1)[:, :n]
            step_c = torch.full_like(step_g, float("nan"))
            want = m._complete(labels, u, x, n, step_c)
            step_w = torch.full_like(step_g, float("nan"))
            got, lpc = m._sample_with(labels, u, x, n, 1.0, None, None, step_w)
            assert torch.equal(got, want) and torch.equal(got, g), (name, n)
            assert torch.equal(step_w.nan_to_num(7.0), step_c.nan_to_num(7.0)), (name, n)
            _check_log_prob(step_g, g, pos >= n, lpc, f"{name} n_given={n}")


@pytest.mark.parametrize("name", CASES)
def test_every_draw_follows_the_contract_on_its_step_logits(name):
    c, m = _model(name)
    B, S, K = c["batch"], c["size"], c["K"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    pos = torch.arange(S * S, device="cuda").view(1, S, S)
    with torch.no_grad():
        for i, s in enumerate(SETTINGS):
            T, top_k, top_p = _setting(s, K)
            gen = torch.Generator(device="cuda").manual_seed(c["xseed"] + 100 * i)
            u = torch.rand((B, S, S), device="cuda", generator=gen)
            n = (S * S) // 2 if i % 2 else 0
            x = torch.randint(0, K, (B, S, S), device="cuda", generator=gen) if n else None
            step = torch.full((B, S, S, K), float("nan"), device="cuda")
            codes, lp = m._sample_with(labels, u, x, n, T, top_k, top_p, step)
            drawn = (pos >= n).expand(B, S, S)
            assert int(codes[drawn].min()) >= 0 and int(codes[drawn].max()) < K
            what = f"{name} T={T} top_k={top_k} top_p={top_p} n_given={n}"
            _check_contract(step, codes, u, drawn, T, top_k, top_p, what)
            _check_log_prob(step, codes, pos.view(-1) >= n, lp, what)
            if top_k == 1:                                  # the argmax of each step's logits
                best = step.max(-1).values
                assert torch.equal(step.gather(-1, codes[..., None])[..., 0][drawn], best[drawn])
            if n:
                assert torch.equal(codes[~drawn], x[~drawn])
            fwd = m(codes, labels).permute(0, 2, 3, 1)     # step logits stay the raw logits, bitwise
            assert torch.equal(step[drawn], fwd[drawn])


@pytest.mark.parametrize("knobs", [dict(temperature=0.5), dict(top_k=5), dict(top_p=0.8)],
                         ids=lambda k: f"{next(iter(k))}={next(iter(k.values()))}")
def test_distribution_chi_square(knobs):
    from scipy import stats
    c, m = _model("prior_ragged")
    N, K, lab = 65536, c["K"], 2
    labels = torch.full((N,), lab, dtype=torch.int64, device="cuda")
    torch.manual_seed(400)
    with torch.no_grad():
        codes, lp = m.sample(labels, shape=(1, 1), batch_size=N, **knobs)
        step = torch.empty((1, 1, 1, K), device="cuda")
        m._sample_with(labels[:1], torch.zeros((1, 1, 1), device="cuda"), None, 0, 1.0, None, None, step)
    k = {**dict(temperature=1.0, top_k=None, top_p=None), **knobs}
    p = ref.probs(step.reshape(1, K).cpu().numpy(), k["temperature"], k["top_k"], k["top_p"])[0]
    counts = np.bincount(codes.view(-1).cpu().numpy(), minlength=K).astype(np.float64)
    assert counts[p == 0].sum() == 0, "codes drawn outside the kept set"
    exp = p * N
    big = exp >= 5
    f_obs = np.append(counts[big], counts[~big & (p > 0)].sum())
    f_exp = np.append(exp[big], exp[~big & (p > 0)].sum())
    if f_exp[-1] == 0:
        f_obs, f_exp = f_obs[:-1], f_exp[:-1]
    pval = stats.chisquare(f_obs, f_exp * f_obs.sum() / f_exp.sum()).pvalue
    print(f"{knobs}: {int((p > 0).sum())} codes kept, chi-square p = {pval:.4f}")
    assert pval > 1e-3
    ls = ref.log_softmax64(step.reshape(1, K).cpu().numpy())[0]
    np.testing.assert_allclose(lp.double().cpu().numpy(), ls[codes.view(-1).cpu().numpy()], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("name", ["prior_default", "prior_ragged"])
def test_log_prob_is_the_teacher_forced_cross_entropy(name):
    c, m = _model(name)
    B, S, K = 6, c["size"], c["K"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    torch.manual_seed(11)
    with torch.no_grad():
        for knobs, n in ((dict(), 0), (dict(temperature=0.7, top_k=10, top_p=0.95), 0), (dict(top_p=0.5), S + 2)):
            if n:
                x = torch.randint(0, K, (B, S, S), device="cuda")
                codes, lp = m.sample_completion(x, labels, n, **knobs)
            else:
                codes, lp = m.sample(labels, shape=(S, S), batch_size=B, **knobs)
            ce = torch.nn.functional.cross_entropy(m(codes, labels).double(), codes, reduction="none")
            sampled = (torch.arange(S * S, device="cuda") >= n).view(1, S, S)
            want = -(ce * sampled).sum((1, 2))
            got = lp.double()
            assert bool(((got - want).abs() <= 1e-5 * want.abs() + 1e-6 * (S * S - n)).all()), (knobs, got, want)


def test_determinism_capture_launches_and_prefix_completion():
    from vqvae_b200 import ops
    c, m = _model("prior_default")
    B, S, K, L = 8, c["size"], c["K"], c["n_layers"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    knobs = (0.8, 50, 0.9)
    with torch.no_grad():
        u = torch.rand((B, S, S), device="cuda")
        m._sample(labels, u)                                           # packs the weights
        a = m._sample_with(labels, u, None, 0, *knobs)
        b = m._sample_with(labels, u, None, 0, *knobs)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        x = torch.randint(0, K, (B, S, S), device="cuda")
        for n in (0, 5, 32, S * S - 1):
            n0 = ops.launch_count()
            m._complete(labels, u, x, n)
            want = ops.launch_count() - n0
            n0 = ops.launch_count()
            m._sample_with(labels, u, x, n, *knobs)
            assert ops.launch_count() - n0 == want, n
        n0 = ops.launch_count()
        m._sample_with(labels, u, None, 0, *knobs)
        assert ops.launch_count() - n0 == S * (L + S) == 184
        # completing a prefix of sample()'s output with the same u and knobs returns that output
        for n in (1, S - 1, S, 33, S * S):
            got, lp = m._sample_with(labels, u, a[0], n, *knobs)
            assert torch.equal(got, a[0]), n
            if n == S * S:
                assert torch.equal(lp, torch.zeros_like(lp))
        # graph capture: the knobs are kernel arguments, nothing synchronises
        for n in (0, 5, 32):
            first = m._sample_with(labels, u, x, n, *knobs)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                out = m._sample_with(labels, u, x, n, *knobs)
            u.copy_(torch.rand_like(u))
            g.replay()
            torch.cuda.synchronize()
            eager = m._sample_with(labels, u, x, n, *knobs)
            assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1]), n
            assert not torch.equal(out[0], first[0])


def test_seeds_line_up_with_generate_and_complete():
    c, m = _model("prior_ragged")
    B, S = 4, c["size"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    with torch.no_grad():
        torch.manual_seed(9)
        g = m.generate(labels, shape=(S, S), batch_size=B)
        torch.manual_seed(9)
        codes, _ = m.sample(labels, shape=(S, S), batch_size=B)
        assert torch.equal(codes, g)
        for n in (0, 3, S * S):
            torch.manual_seed(10)
            want = m.complete(g, labels, n)
            torch.manual_seed(10)
            got, lp = m.sample_completion(g, labels, n)
            assert torch.equal(got, want), n
            r = torch.rand(1, device="cuda")
            torch.manual_seed(10)
            torch.rand((B, S, S), device="cuda")
            assert torch.equal(r, torch.rand(1, device="cuda")), n         # exactly one draw of (B, H, W)

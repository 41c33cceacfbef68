"""Per-image prefix lengths on the H100: one ragged call is, image by image, bitwise the scalar call with that image's
own n_given (codes, log_prob and step logits; log_prob scoring in fp32 and TF32), across the sampler's shape cases,
with generate's launch schedule whatever the values, clamping, fp64 draws, determinism, graph replay with new values
in the same tensor, and the workspace bound."""
import pytest
import torch

from tests.test_gpu_prior_complete import SAMPLER_CASES, _inverts_fp64_cdf, _junk, _model

pytestmark = pytest.mark.gpu


def _cycle(H, W):
    """The prefix lengths the per-image tests cycle through over the batch."""
    HW = H * W
    return [min(max(v, 0), HW) for v in (0, 1, W - 1, W, W + 1, HW // 2, HW - 1, HW)]


def _setup(name, B=None, seed=0):
    c, sd, layers, m = _model(name)
    B = B or max(c["batch"], 8)
    S, K = c["size"], c["K"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    cyc = _cycle(S, S)
    n = torch.tensor([cyc[b % len(cyc)] for b in range(B)], dtype=torch.int64, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(c["xseed"] + seed)
    u = torch.rand((B, S, S), device="cuda", generator=g)
    return c, sd, layers, m, B, S, K, labels, n, u


def _before(n, B, S):
    """(B, S, S) True at each image's given positions p < n[b]."""
    return torch.arange(S * S, device="cuda").view(1, S, S) < n.view(B, 1, 1)


def _junk_after(x, n, K, seed):
    """x with image b's positions >= n[b] replaced by junk codes, out-of-range ones included."""
    B, S, _ = x.shape
    return torch.where(_before(n, B, S), x, _junk(x, 0, K, seed))


def _knob_sets(K):
    return [(1.0, None, None), (0.7, min(5, K), 0.9)]


@pytest.mark.parametrize("name", SAMPLER_CASES)
def test_ragged_complete_reproduces_generate_and_launches_generates_schedule(name):
    from vqvae_b200 import ops
    c, _, _, m, B, S, K, labels, n, u = _setup(name)
    L = c["n_layers"]
    with torch.no_grad():
        step_g = torch.full((B, S, S, K), float("nan"), device="cuda")
        g = m._sample(labels, u, step_g)
        x = _junk_after(g, n, K, seed=1)
        x_before, n_before = x.clone(), n.clone()
        step_c = torch.full((B, S, S, K), float("nan"), device="cuda")
        n0 = ops.launch_count()
        out = m._complete(labels, u, x, n, step_c)
        assert ops.launch_count() - n0 == 1 + S * (L + S)
    assert torch.equal(x, x_before) and torch.equal(n, n_before)
    assert out.dtype == torch.int64 and out.shape == (B, S, S)
    if not torch.equal(out, g):
        bad = torch.nonzero(out != g)
        pytest.fail(f"{name}: {bad.shape[0]} codes differ, first at {bad[0].tolist()} (n = {n.tolist()})")
    after = (~_before(n, B, S))[..., None].expand_as(step_c)
    assert torch.equal(step_c[after], step_g[after])
    assert bool(torch.isnan(step_c[~after]).all())                   # given positions untouched


@pytest.mark.parametrize("name", SAMPLER_CASES)
def test_ragged_sample_is_the_per_image_scalar_calls(name):
    c, _, _, m, B, S, K, labels, n, u = _setup(name, seed=2)
    gen = torch.Generator(device="cuda").manual_seed(c["xseed"] + 3)
    x = torch.randint(-3, K + 3, (B, S, S), device="cuda", generator=gen)
    given = _before(n, B, S)
    for T, k, p in _knob_sets(K):
        with torch.no_grad():
            step = torch.full((B, S, S, K), float("nan"), device="cuda")
            codes, lp = m._sample_with(labels, u, x, n, T, k, p, step)
            for b in range(B):
                nb = int(n[b])
                step_b = torch.full((1, S, S, K), float("nan"), device="cuda")
                codes_b, lp_b = m._sample_with(labels[b:b + 1], u[b:b + 1], x[b:b + 1], nb, T, k, p, step_b)
                what = f"{name} T={T} top_k={k} top_p={p} image {b} n_given={nb}"
                assert torch.equal(codes[b:b + 1], codes_b), what
                assert torch.equal(lp[b:b + 1], lp_b), (what, float(lp[b]), float(lp_b[0]))
                assert torch.equal(step[b:b + 1].nan_to_num(7.0), step_b.nan_to_num(7.0)), what
        assert torch.equal(codes[given], x[given])
        assert bool(torch.isnan(step[given]).all())
        assert bool((lp[n == S * S] == 0).all())


@pytest.mark.parametrize("name", ["prior_default", "prior_ragged"])
def test_ragged_draws_invert_the_fp64_cdf(name):
    c, sd, layers, m, B, S, K, labels, n, u = _setup(name, seed=4)
    gen = torch.Generator(device="cuda").manual_seed(c["xseed"] + 5)
    x = torch.randint(-4, K + 4, (B, S, S), device="cuda", generator=gen)
    with torch.no_grad():
        out = m._complete(labels, u, x, n)
    _inverts_fp64_cdf(sd, layers, c["n_layers"], out.clamp(0, K - 1), labels, u, ~_before(n, B, S), name)


@pytest.mark.parametrize("name", ["prior_default", "prior_ragged", "kernels"])
def test_a_uniform_tensor_is_the_scalar_call(name):
    from vqvae_b200 import ops
    c, _, _, m, B, S, K, labels, _, u = _setup(name, seed=6)
    gen = torch.Generator(device="cuda").manual_seed(c["xseed"] + 7)
    x = torch.randint(0, K, (B, S, S), device="cuda", generator=gen)
    T, k, p = _knob_sets(K)[1]
    with torch.no_grad():
        for v in sorted({0, 1, S, S + 1, S * S // 2, S * S - 1, S * S}):
            t = torch.full((B,), v, dtype=torch.int64, device="cuda")
            sr = torch.full((B, S, S, K), float("nan"), device="cuda")
            ss = torch.full((B, S, S, K), float("nan"), device="cuda")
            cr, lr = m._sample_with(labels, u, x, t, T, k, p, sr)
            cs, ls = m._sample_with(labels, u, x, v, T, k, p, ss)
            assert torch.equal(cr, cs) and torch.equal(lr, ls), v
            assert torch.equal(sr.nan_to_num(7.0), ss.nan_to_num(7.0)), v
            assert torch.equal(m._complete(labels, u, x, t), m._complete(labels, u, x, v)), v
            for precision in ("fp32", "tf32"):
                m.precision = precision
                n0 = ops.launch_count()
                got = m.log_prob(x, labels, n_given=t)
                launches = ops.launch_count() - n0
                assert torch.equal(got, m.log_prob(x, labels, n_given=v)), (v, precision)
                assert launches == (3 + 2 * c["n_layers"] if precision == "fp32" else 4 + 4 * c["n_layers"])
            m.precision = "fp32"
        # a 1-D tensor of one entry is the per-image path, with the scalar call's bits
        one = torch.tensor([S + 1], device="cuda")
        assert torch.equal(m._complete(labels[:1], u[:1], x[:1], one), m._complete(labels[:1], u[:1], x[:1], S + 1))


def test_launches_do_not_depend_on_the_values():
    from vqvae_b200 import ops
    c, _, _, m, B, S, K, labels, n, u = _setup("prior_default")
    x = torch.randint(0, K, (B, S, S), device="cuda")
    L = c["n_layers"]
    assert 1 + S * (L + S) == 185
    with torch.no_grad():
        m._sample(labels, u)                                            # packs the weights
        for vals in ([0] * B, [S * S] * B, [S * S - 1] * B, n.tolist(), list(range(B))):
            t = torch.tensor(vals, device="cuda")
            for call in (lambda: m._complete(labels, u, x, t), lambda: m.sample_completion(x, labels, t, top_k=7)):
                n0 = ops.launch_count()
                call()
                assert ops.launch_count() - n0 == 1 + S * (L + S), vals


def test_values_are_clamped_to_the_grid():
    c, _, _, m, B, S, K, labels, _, u = _setup("prior_ragged", seed=8)
    x = torch.randint(0, K, (B, S, S), device="cuda")
    wild = torch.tensor([-5, S * S + 7, -1, 2**40, 3, -(2**40), S * S, 0][:B], device="cuda")
    tame = wild.clamp(0, S * S)
    with torch.no_grad():
        for T, k, p in _knob_sets(K):
            sw = torch.full((B, S, S, K), float("nan"), device="cuda")
            st = torch.full((B, S, S, K), float("nan"), device="cuda")
            cw, lw = m._sample_with(labels, u, x, wild, T, k, p, sw)
            ct, lt = m._sample_with(labels, u, x, tame, T, k, p, st)
            assert torch.equal(cw, ct) and torch.equal(lw, lt)
            assert torch.equal(sw.nan_to_num(7.0), st.nan_to_num(7.0))
        for precision in ("fp32", "tf32"):
            m.precision = precision
            assert torch.equal(m.log_prob(x, labels, n_given=wild), m.log_prob(x, labels, n_given=tame))
        m.precision = "fp32"


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("name", SAMPLER_CASES)
def test_ragged_log_prob_is_the_scalar_calls(name, precision):
    c, _, _, m, B, S, K, labels, n, _ = _setup(name, seed=9)
    m.precision = precision
    gen = torch.Generator(device="cuda").manual_seed(c["xseed"] + 10)
    x = torch.randint(-3, K + 3, (B, S, S), device="cuda", generator=gen)
    with torch.no_grad():
        got = m.log_prob(x, labels, n_given=n)
        assert torch.equal(got, m._log_prob(x, labels, n.tolist()))    # a list is the same call
        for v in sorted(set(n.tolist())):
            want = m.log_prob(x, labels, n_given=v)                      # the scalar call on the same batch
            sel = n == v
            assert torch.equal(got[sel], want[sel]), (name, precision, v)
        if precision == "fp32":                                          # and on each image alone
            for b in range(B):
                alone = m.log_prob(x[b:b + 1], labels[b:b + 1], n_given=int(n[b]))
                assert torch.equal(got[b:b + 1], alone), (name, b)
    assert bool((got[n == S * S] == 0).all())


@pytest.mark.parametrize("name", ["prior_default", "prior_ragged", "cfg3_sampler"])
def test_scoring_a_ragged_completion_reproduces_its_log_prob(name):
    c, _, _, m, B, S, K, labels, n, _ = _setup(name, seed=11)
    gen = torch.Generator(device="cuda").manual_seed(c["xseed"] + 12)
    x = torch.randint(0, K, (B, S, S), device="cuda", generator=gen)
    torch.manual_seed(c["xseed"] + 13)
    with torch.no_grad():
        codes, lp = m.sample_completion(x, labels, n)
        scored = m.log_prob(codes, labels, n_given=n)
    rel = ((scored.double() - lp.double()).abs() / lp.double().abs().clamp(min=1e-30))[n < S * S]
    print(f"{name}: worst relative difference {float(rel.max()) if rel.numel() else 0.0:.3g}")
    assert bool((rel <= 1e-5).all())
    assert bool((lp[n == S * S] == 0).all()) and bool((scored[n == S * S] == 0).all())


def test_determinism_and_graph_replay_with_new_values():
    c, _, _, m, B, S, K, labels, n, u = _setup("prior_default", seed=14)
    x = torch.randint(0, K, (B, S, S), device="cuda")
    T, k, p = _knob_sets(K)[1]
    with torch.no_grad():
        a = m._sample_with(labels, u, x, n, T, k, p)
        b = m._sample_with(labels, u, x, n, T, k, p)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        assert torch.equal(m._log_prob(x, labels, n), m._log_prob(x, labels, n))
        static = n.clone()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            codes, lp = m._sample_with(labels, u, x, static, T, k, p)
            score = m._log_prob(x, labels, static)
        for seed in range(3):
            g = torch.Generator(device="cuda").manual_seed(100 + seed)
            static.copy_(torch.randint(-2, S * S + 3, (B,), device="cuda", generator=g))
            graph.replay()
            torch.cuda.synchronize()
            want_codes, want_lp = m._sample_with(labels, u, x, static.clone(), T, k, p)
            assert torch.equal(codes, want_codes) and torch.equal(lp, want_lp), seed
            assert torch.equal(score, m._log_prob(x, labels, static.clone())), seed


def test_peak_memory_is_the_generate_workspace_and_the_search_scratch():
    from vqvae_b200 import _lib
    c, _, _, m, B, S, K, labels, _, u = _setup("cfg3_sampler", B=16, seed=15)
    x = torch.randint(0, K, (B, S, S), device="cuda")
    n = torch.randint(0, S * S + 1, (B,), device="cuda")
    with torch.no_grad():
        m.sample_completion(x[:1], labels[:1], n[:1])                  # packs the weights
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        m._sample_with(labels, u, x, n, 1.0, 9, 0.95)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
    lib = _lib.lib()
    ws = lib.vqb_prior_sample_workspace_bytes(B, S, S, c["dim"], c["n_layers"], K, 0)
    outputs = B * S * S * 8 + B * 4
    print(f"peak {peak / 2**20:.1f} MiB, workspace {ws / 2**20:.1f} MiB, completion's "
          f"{lib.vqb_prior_sample_workspace_bytes(B, S, S, c['dim'], c['n_layers'], K, S * S // 2) / 2**20:.1f} MiB")
    assert peak <= ws + outputs + 2 * 512

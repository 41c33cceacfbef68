"""The codebook's k-means initialisation on the H100: vqb_vq_kmeans_f32 bit for bit against tests/vq_kmeans_ref.py on
both VQ kernels, the seed against the restart's selection, determinism (two calls, a CUDA graph, the workspace bound,
the launches and random draws), the Lloyd property, the modules' behaviour, and what the initialisation is for: a
codebook that starts on the data."""
import ctypes

import numpy as np
import pytest
import torch

from oracle.weights import make_images
from tests.test_gpu_vq_ema import VAR
from tests.vq_kmeans_ref import kmeans
from tests.vq_restart_ref import row_order

pytestmark = pytest.mark.gpu

SEED_LAUNCHES, STEP_LAUNCHES = 12, 5        # + the VQ call's own: 2 on the tensor-core kernel, 3 on the exact one


def _rows(N, D, case, rng):
    if case == "distinct":
        return rng.standard_normal((N, D), dtype=np.float32)
    if case == "dup":                                      # few distinct rows: the seed repeats rows, codes go empty
        pool = rng.standard_normal((max(N // 8, 1), D), dtype=np.float32)
        return pool[rng.integers(0, pool.shape[0], N)]
    if case == "equal":
        return np.repeat(rng.standard_normal((1, D), dtype=np.float32), N, axis=0)
    assert case == "nan", case
    z = rng.standard_normal((N, D), dtype=np.float32)
    z[N // 2, D - 1] = np.nan
    return z


def _same(got, want):
    """Bit for bit, except that any NaN equals any NaN (the GPU's NaN is the canonical one, numpy's keeps a payload)."""
    g, w = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    nan = np.isnan(g)
    return np.array_equal(nan, np.isnan(w)) and np.array_equal(g[~nan].view(np.uint32), w[~nan].view(np.uint32))


def _kmeans_gpu(z, u, K, iters):
    from vqvae_b200 import ops
    cb = torch.full((K, z.shape[1]), float("nan"), device="cuda")      # the seed overwrites every code
    sse = ops.vq_kmeans(torch.from_numpy(z).cuda(), torch.from_numpy(u).cuda(), iters, cb)
    return cb.cpu().numpy(), sse.cpu().numpy()


# N in {K, 1000, 65536, 2^20}; N*K*D*max(iters, 1) <= ~2^34 keeps the C oracle's VQ affordable
GRID = [(1, 1, 4, 10, "distinct", "auto"), (7, 7, 64, 10, "distinct", "auto"), (1000, 1, 4, 10, "distinct", "auto"),
        (1000, 7, 4, 10, "dup", "auto"), (1000, 7, 256, 1, "nan", "auto"), (1000, 7, 64, 10, "nan", "exact"),
        (1000, 512, 64, 10, "distinct", "auto"), (1000, 512, 64, 10, "dup", "exact"),
        (1024, 1024, 64, 1, "equal", "auto"), (1024, 1024, 64, 10, "distinct", "exact"),
        (8192, 8192, 4, 1, "distinct", "auto"), (8192, 8192, 64, 1, "dup", "auto"),
        (65536, 7, 256, 10, "distinct", "auto"), (65536, 512, 4, 10, "dup", "auto"),
        (65536, 512, 64, 1, "distinct", "auto"), (65536, 512, 64, 1, "distinct", "exact"),
        (65536, 1024, 64, 1, "nan", "auto"), (65536, 1024, 256, 0, "distinct", "auto"),
        (65536, 8192, 4, 1, "equal", "auto"), (65536, 8192, 4, 0, "dup", "auto"),
        (1 << 20, 1, 256, 10, "equal", "auto"), (1 << 20, 7, 64, 10, "distinct", "auto"),
        (1 << 20, 512, 4, 1, "dup", "auto"), (1 << 20, 1024, 4, 1, "distinct", "auto"),
        (1 << 20, 1024, 4, 0, "distinct", "auto")]
LARGEST = max(GRID, key=lambda c: c[0] * c[1] * c[2] * max(c[3], 1))


@pytest.fixture
def vq_kernel():
    from vqvae_b200 import ops
    yield ops.set_vq_kernel
    ops.set_vq_kernel("auto")


@pytest.mark.parametrize("N, K, D, iters, case, kernel", GRID)
def test_kmeans_is_the_reference_bit_for_bit(N, K, D, iters, case, kernel, vq_kernel):
    rng = np.random.default_rng(N * 31 + K * 7 + D + iters)
    z = _rows(N, D, case, rng)
    u = rng.random(N, dtype=np.float32)
    vq_kernel("tc" if kernel == "auto" and D == 64 else kernel)
    e, sse = _kmeans_gpu(z, u, K, iters)
    want_e, want_sse = kmeans(z, u, K, iters)
    assert _same(e, want_e), f"{int((e.view(np.uint32) != want_e.view(np.uint32)).any(axis=1).sum())} codes differ"
    if case == "nan" and iters > 0:
        assert np.isnan(sse).all() and np.isnan(want_sse).all()
    else:
        np.testing.assert_allclose(sse, want_sse, rtol=2e-6, atol=0)
    if case == "equal" and iters > 0:
        assert want_sse[0] == 0.0
    if (N, K, D, iters, case, kernel) == LARGEST:
        print(f"largest case run: N={N} K={K} D={D} iters={iters}, N*K*D*max(iters, 1) = "
              f"2^{np.log2(N * K * D * max(iters, 1)):.2f}")


def test_zero_iterations_are_the_restart_with_every_code_dead():
    from vqvae_b200 import ops
    N, K, D = 65536, 8192, 64
    rng = np.random.default_rng(5)
    z = torch.from_numpy(rng.standard_normal((N, D), dtype=np.float32)).cuda()
    u = torch.from_numpy(rng.random(N, dtype=np.float32)).cuda()
    cb = torch.zeros((K, D), device="cuda")
    ops.vq_kmeans(z, u, 0, cb)
    state = [torch.zeros(K, device="cuda"), torch.zeros((K, D), device="cuda"), torch.zeros((K, D), device="cuda")]
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.vq_ema_restart(z, u, 1.0, *state, cnt)
    assert int(cnt) == K and torch.equal(cb, state[2])
    assert torch.equal(cb.cpu(), z.cpu()[torch.from_numpy(row_order(u.cpu().numpy())[:K])])


def test_two_calls_a_graph_replay_and_the_workspace_bound():
    from vqvae_b200 import _lib, ops
    N, K, D, iters = 1 << 18, 1024, 64, 4
    rng = np.random.default_rng(9)
    z = torch.from_numpy(rng.standard_normal((N, D), dtype=np.float32)).cuda()
    u = torch.from_numpy(rng.random(N, dtype=np.float32)).cuda()
    a, b = torch.zeros((K, D), device="cuda"), torch.ones((K, D), device="cuda")
    sa, sb = ops.vq_kmeans(z, u, iters, a), ops.vq_kmeans(z, u, iters, b)
    assert torch.equal(a, b) and torch.equal(sa, sb)
    # the workspace: guard bytes on both sides stay as they were
    L = ops.lib()
    ws_bytes = L.vqb_vq_kmeans_workspace_bytes(N, K, D)
    guard = 1 << 16
    buf = torch.full((guard + ws_bytes + guard,), 0xA5, dtype=torch.uint8, device="cuda")
    c = torch.zeros((K, D), device="cuda")
    sc = torch.empty(iters, dtype=torch.float64, device="cuda")
    n0 = ops.launch_count()
    _lib.check(L.vqb_vq_kmeans_f32(z.data_ptr(), u.data_ptr(), N, K, D, iters, c.data_ptr(), sc.data_ptr(),
                                   buf.data_ptr() + guard, ws_bytes,
                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "kmeans")
    assert ops.launch_count() - n0 == SEED_LAUNCHES + iters * (2 + STEP_LAUNCHES)
    torch.cuda.synchronize()
    assert bool((buf[:guard] == 0xA5).all()) and bool((buf[guard + ws_bytes:] == 0xA5).all())
    assert torch.equal(a, c) and torch.equal(sa, sc)
    ops.set_vq_kernel("exact")
    try:
        n0 = ops.launch_count()
        d = torch.zeros((K, D), device="cuda")
        sd = ops.vq_kmeans(z, u, iters, d)
        assert ops.launch_count() - n0 == SEED_LAUNCHES + iters * (3 + STEP_LAUNCHES)
    finally:
        ops.set_vq_kernel("auto")
    # both VQ kernels: the same assignments, so the same codebook bits; each sums its SSE in its own order
    assert torch.equal(a, d)
    torch.testing.assert_close(sd, sa, rtol=2e-6, atol=0)


def test_a_captured_call_replays_as_an_eager_call_and_draws_one_uniform_per_row():
    import vqvae_b200
    from vqvae_b200 import ops
    B, D, H, W, K, iters = 16, 64, 16, 16, 512, 3
    N = B * H * W
    z = torch.randn(B, D, H, W, device="cuda")
    va, vb = vqvae_b200.VectorQuantizer(K, D, 0.25).cuda(), vqvae_b200.VectorQuantizer(K, D, 0.25).cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        vb.init_codebook_kmeans(z, iters)                      # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        sse_b = vb.init_codebook_kmeans(z, iters)
    for seed in (2, 3):
        torch.cuda.manual_seed(seed)
        sse_a = va.init_codebook_kmeans(z, iters)
        after = torch.cuda.get_rng_state()
        torch.cuda.manual_seed(seed)
        n0 = ops.launch_count()
        g.replay()
        assert ops.launch_count() == n0
        torch.cuda.synchronize()
        assert torch.equal(va.embedding.weight, vb.embedding.weight) and torch.equal(sse_a, sse_b)
        torch.cuda.manual_seed(seed)
        torch.rand((N,), device="cuda")                         # exactly one draw of one uniform per row
        assert torch.equal(after, torch.cuda.get_rng_state())


def test_lloyd_steps_never_raise_the_inertia():
    from vqvae_b200 import ops
    rng = np.random.default_rng(4)
    K, D, N = 256, 64, 1 << 17
    centres = 4.0 * rng.standard_normal((K, D))
    z = (centres[rng.integers(0, K, N)] + 0.1 * rng.standard_normal((N, D))).astype(np.float32)
    cb = torch.empty((K, D), device="cuda")
    torch.manual_seed(0)
    sse = ops.vq_kmeans(torch.from_numpy(z).cuda(), torch.rand(N, device="cuda"), 10, cb).cpu().numpy()
    assert np.all(sse[1:] <= sse[:-1] * (1 + 1e-6)), sse
    assert sse[-1] < sse[0]


# ---- the modules ---------------------------------------------------------------------------------------------------
def test_module_state_after_the_call():
    import vqvae_b200
    from vqvae_b200 import ops
    from vqvae_b200.optim import Adam
    x = torch.from_numpy(make_images(8, 32, seed=3)).cuda()
    # EMA: the averages restart from the new codebook, bumped like a state-dict load
    torch.manual_seed(0)
    m = vqvae_b200.VQVAE(128, 32, 2, 64, 64, 0.25, ema_decay=0.99).cuda().eval()
    vq = m.vector_quantization
    vq.ema_cluster_size.fill_(7.0)
    vers = [t._version for t in (vq.embedding.weight, vq.ema_cluster_size, vq.ema_embed_sum)]
    m.init_codebook_kmeans(x, iters=2)
    assert not m.training
    assert torch.equal(vq.ema_cluster_size, torch.ones_like(vq.ema_cluster_size))
    assert torch.equal(vq.ema_embed_sum, vq.embedding.weight)
    assert all(t._version > v for t, v in zip((vq.embedding.weight, vq.ema_cluster_size, vq.ema_embed_sum), vers))
    # gradient codebook: no autograd graph, the version moves, and an on-device Adam step runs after it
    torch.manual_seed(0)
    m = vqvae_b200.VQVAE(128, 32, 2, 64, 64, 0.25).cuda().train()
    opt = Adam(m.parameters(), lr=3e-4)
    w = m.vector_quantization.embedding.weight
    v0 = w._version
    with torch.enable_grad():
        sse = m.init_codebook_kmeans(x.clone().requires_grad_(True), iters=2)
        zs = torch.randn(4, 64, 4, 4, device="cuda", requires_grad=True)
        sse2 = m.vector_quantization.init_codebook_kmeans(zs, iters=1)
    assert m.training and w._version > v0 and w.is_leaf and w.grad is None
    for t in (sse, sse2):
        assert t.dtype == torch.float64 and not t.requires_grad and t.grad_fn is None
    assert sse.shape == (2,) and sse2.shape == (1,) and zs.grad is None
    before = w.detach().clone()
    opt.zero_grad(set_to_none=True)
    with torch.enable_grad():
        embedding_loss, x_hat, _ = m(x)
        (torch.mean((x_hat - x) ** 2) / VAR + embedding_loss).backward()
    opt.step()
    torch.cuda.synchronize()
    assert torch.isfinite(w).all() and not torch.equal(w.detach(), before)
    # fewer rows than codes: ValueError before anything is drawn or launched
    few = torch.randn(1, 64, 4, 4, device="cuda")
    rng, n0 = torch.cuda.get_rng_state(), ops.launch_count()
    with pytest.raises(ValueError, match="row"):
        m.vector_quantization.init_codebook_kmeans(few)
    with pytest.raises(ValueError, match="row"):
        vqvae_b200.VQVAE(32, 8, 1, 512, 8, 0.25).cuda().init_codebook_kmeans(x[:1])
    assert ops.launch_count() == n0 and torch.equal(torch.cuda.get_rng_state(), rng)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_vqvae_fits_the_rows_forward_quantizes(precision):
    import vqvae_b200
    torch.manual_seed(0)
    m = vqvae_b200.VQVAE(128, 32, 2, 512, 64, 0.25).cuda().train()
    x = torch.from_numpy(make_images(16, 32, seed=4)).cuda()
    with vqvae_b200.precision(precision), torch.no_grad():
        z_e, _, _, _ = m._encode_rows(x, m._bf16_pipeline())
        rows = z_e.view(-1, 64).float().cpu().numpy()
        torch.cuda.manual_seed(7)
        u = torch.rand(rows.shape[0], device="cuda").cpu().numpy()
        torch.cuda.manual_seed(7)
        sse = m.init_codebook_kmeans(x, iters=3)
    e, want_sse = kmeans(rows, u, 512, 3)
    assert _same(m.vector_quantization.embedding.weight.detach().cpu().numpy(), e)
    np.testing.assert_allclose(sse.cpu().numpy(), want_sse, rtol=2e-6, atol=0)


# ---- what it is for ------------------------------------------------------------------------------------------------
def _clusters(K=32, D=8, per=64, sigma=0.05, radius=1.0):
    """The restart test's data: K tight clusters on a sphere around a far centre, as (rows (B, D, 8, 8), centres)."""
    rng = np.random.default_rng(11)
    c = np.zeros(D)
    c[0] = 5.0
    dirs = rng.standard_normal((K, D))
    centres = c + radius * dirs / np.linalg.norm(dirs, axis=1, keepdims=True)
    rows = (np.repeat(centres, per, axis=0) + sigma * rng.standard_normal((K * per, D))).astype(np.float32)
    rows = rows[rng.permutation(K * per)]
    return torch.from_numpy(rows).view(K * per // 64, 8, 8, D).permute(0, 3, 1, 2).contiguous().cuda(), centres


def test_a_lone_quantizer_starts_on_the_clusters():
    import vqvae_b200
    sigma = 0.05
    z, centres = _clusters(sigma=sigma)
    torch.manual_seed(0)
    vq = vqvae_b200.VectorQuantizer(32, 8, 0.25).cuda().eval()

    def covered_and_perplexity():
        with torch.no_grad():
            perp = float(vq(z)[2])
        e = vq.embedding.weight.detach().double().cpu().numpy()
        dist = np.linalg.norm(centres[:, None, :] - e[None, :, :], axis=2)
        return int((dist.min(axis=1) < 3 * sigma).sum()), perp
    covered0, perp0 = covered_and_perplexity()
    vq.init_codebook_kmeans(z, iters=10)
    covered, perp = covered_and_perplexity()
    print(f"reference init: {covered0} clusters covered, perplexity {perp0:.2f}; "
          f"after k-means: {covered} covered, perplexity {perp:.2f}")
    assert covered0 == 0 and perp0 < 4.0
    assert covered >= 12 and perp > 20.0


def test_main_py_model_first_forward_uses_more_codes():
    import vqvae_b200
    x = torch.from_numpy(make_images(32, 32, seed=1)).cuda()
    torch.manual_seed(0)
    m = vqvae_b200.VQVAE(128, 32, 2, 512, 64, 0.25).cuda().train()
    with torch.enable_grad():
        perp0 = float(m(x)[2])
    m.init_codebook_kmeans(x)
    with torch.enable_grad():
        perp = float(m(x)[2])
    print(f"main.py's model, B = 32: perplexity {perp0:.2f} at the reference init, {perp:.2f} after k-means")
    assert perp >= 4 * perp0, (perp0, perp)

"""The EMA codebook on the H100: vqb_vq_ema_update_f32's per-code sums bit for bit against the fp32 emulation of their
documented order, the update against fp64, determinism (eager and in a CUDA graph), one VQ-VAE training step against
fp64 autograd with the restated EMA and loss, the paths that must not update, main.py's loop reproducible bit for bit,
VectorQuantizer on its own, checkpoints and the workspace bound."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle.make_golden import MODEL_CASES
from oracle.prior_train_port import leaf_params
from oracle.vqvae_train_port import train_loss, vqvae_train_forward
from oracle.weights import make_images, make_state_dict
from tests.vq_ema_ref import commit_dz_fp64, commit_loss_fp64, counts, ema_update_fp64, segment_sums

pytestmark = pytest.mark.gpu

HP = ("h_dim", "res_h_dim", "n_res_layers", "n_embeddings", "embedding_dim")
VAR = 0.0625


def _codes(kind, N, K, rng):
    if kind == "uniform":
        return rng.integers(0, K, N)
    if kind == "one":                                  # the collapsed codebook: every row on one code
        return np.full(N, K // 2, dtype=np.int64)
    if kind == "half":                                 # half the codes unused
        return rng.integers(0, max(K // 2, 1), N) * 2 % K
    if kind == "oob":                                  # out-of-range codes, clamped
        return rng.integers(-3, K + 3, N)
    raise ValueError(kind)


def _state(K, D, rng, init=None):
    if init is None:
        N0 = torch.ones(K)
        m0 = torch.from_numpy(rng.standard_normal((K, D)).astype(np.float32) * 0.1)
    else:
        N0, m0 = init
    return [t.clone().cuda().contiguous() for t in (N0, m0, m0)]


def _update(z, idx, K, decay, eps, state):
    from vqvae_b200 import ops
    hist = torch.from_numpy(counts(idx.cpu().numpy(), K).astype(np.int32)).cuda()
    ops.vq_ema_update(z, idx, hist, decay, eps, *state)
    return hist


CASES = [(1, 1, 4, "uniform"), (1, 7, 64, "oob"), (1000, 7, 4, "uniform"), (1000, 7, 256, "one"),
         (1000, 512, 64, "half"), (16384, 1, 64, "uniform"), (16384, 512, 64, "uniform"), (16384, 512, 64, "one"),
         (16384, 1024, 256, "half"), (16384, 8192, 64, "oob"), (16384, 8192, 4, "one"),
         (524288, 1024, 64, "uniform"), (524288, 1024, 64, "one"), (524288, 8192, 64, "half"),
         (524288, 7, 256, "oob"), (524288, 512, 4, "uniform")]


@pytest.mark.parametrize("N, K, D, kind", CASES)
def test_row_sums_are_the_fp32_emulation_bit_for_bit_and_counts_exact(N, K, D, kind):
    rng = np.random.default_rng(N * 31 + K * 7 + D)
    zn = rng.standard_normal((N, D)).astype(np.float32)
    idx_np = _codes(kind, N, K, rng)
    z, idx = torch.from_numpy(zn).cuda(), torch.from_numpy(idx_np).cuda()
    state = _state(K, D, rng)
    hist = _update(z, idx, K, 0.0, 1e-5, state)             # decay 0: embed_sum = s_k, cluster_size = n_k, exactly
    torch.cuda.synchronize()
    want = segment_sums(zn, idx_np, K)
    got = state[1].cpu().numpy()
    bad = np.nonzero(~np.all(got.view(np.uint32) == want.view(np.uint32), axis=1))[0]
    assert bad.size == 0, f"{bad.size} codes differ, first {bad[:5]}"
    assert np.array_equal(state[0].cpu().numpy(), hist.cpu().numpy().astype(np.float32))


@pytest.mark.parametrize("N, K, D, kind", [(16384, 512, 64, "uniform"), (16384, 512, 64, "one"),
                                           (524288, 1024, 64, "half"), (1000, 7, 256, "oob")])
def test_update_matches_fp64_on_the_kernels_own_sums(N, K, D, kind):
    rng = np.random.default_rng(5)
    zn = rng.standard_normal((N, D)).astype(np.float32)
    idx_np = _codes(kind, N, K, rng)
    z, idx = torch.from_numpy(zn).cuda(), torch.from_numpy(idx_np).cuda()
    N0 = torch.from_numpy(rng.uniform(0.5, 50.0, K).astype(np.float32))
    m0 = torch.from_numpy(rng.standard_normal((K, D)).astype(np.float32))
    probe = _state(K, D, rng, (N0, m0))
    _update(z, idx, K, 0.0, 1e-5, probe)                    # the kernel's own s_k and n_k
    s, n = probe[1].cpu().numpy(), probe[0].cpu().numpy()
    state = _state(K, D, rng, (N0, m0))
    _update(z, idx, K, 0.9, 1e-5, state)
    N1, m1, e1 = ema_update_fp64(N0.numpy(), m0.numpy(), n, s, float(np.float32(0.9)), float(np.float32(1e-5)))
    for got, want in zip(state, (N1, m1, e1)):
        g = got.cpu().numpy().astype(np.float64)
        assert float(np.max(np.abs(g - want))) <= 1e-6 * float(np.abs(want).max())


def test_decay_zero_is_the_k_means_step_and_unused_codes_stay_put():
    rng = np.random.default_rng(1)
    N, K, D = 16384, 512, 64
    zn = rng.standard_normal((N, D)).astype(np.float32)
    idx_np = _codes("half", N, K, rng)
    z, idx = torch.from_numpy(zn).cuda(), torch.from_numpy(idx_np).cuda()
    state = _state(K, D, rng)
    _update(z, idx, K, 0.0, 1e-12, state)
    e = state[2].cpu().numpy().astype(np.float64)
    n = counts(idx_np, K)
    for k in np.nonzero(n)[0][:64]:
        mean = zn[idx_np == k].astype(np.float64).mean(0)
        assert np.max(np.abs(e[k] - mean)) <= 1e-6 * max(1.0, np.abs(mean).max()), k
    # decay 0.99 from N = 1, m = e: the codes no row picked keep their value up to the smoothing's rescale
    e0 = torch.from_numpy(rng.standard_normal((K, D)).astype(np.float32) * 0.01)
    state = _state(K, D, rng, (torch.ones(K), e0))
    _update(z, idx, K, 0.99, 1e-5, state)
    e1 = state[2].cpu().numpy()
    unused = n == 0
    assert unused.sum() > 0 and np.isfinite(e1).all()
    np.testing.assert_allclose(e1[unused], e0.numpy()[unused], rtol=1e-3, atol=1e-7)


@pytest.mark.parametrize("kind", ["uniform", "one"])
def test_two_calls_and_a_graph_replay_are_bitwise_equal(kind):
    from vqvae_b200 import ops
    rng = np.random.default_rng(2)
    N, K, D = 1 << 18, 1024, 64
    z = torch.from_numpy(rng.standard_normal((N, D)).astype(np.float32)).cuda()
    idx = torch.from_numpy(_codes(kind, N, K, rng)).cuda()
    init = (torch.rand(K) + 0.5, torch.randn(K, D))
    a, b, c = (_state(K, D, rng, init) for _ in range(3))
    hist = _update(z, idx, K, 0.95, 1e-5, a)
    _update(z, idx, K, 0.95, 1e-5, b)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.vq_ema_update(z, idx, hist, 0.95, 1e-5, *[t.clone() for t in c])      # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.vq_ema_update(z, idx, hist, 0.95, 1e-5, *c)
    n0 = ops.launch_count()
    g.replay()
    assert ops.launch_count() == n0
    torch.cuda.synchronize()
    for x, y, w in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, w)


def test_update_stays_inside_its_workspace():
    from vqvae_b200 import _lib, ops
    L = ops.lib()
    rng = np.random.default_rng(3)
    for N, K, D, kind in ((16384, 8192, 64, "one"), (1000, 7, 4, "oob"), (65536, 512, 256, "uniform")):
        z = torch.from_numpy(rng.standard_normal((N, D)).astype(np.float32)).cuda()
        idx_np = _codes(kind, N, K, rng)
        idx = torch.from_numpy(idx_np).cuda()
        hist = torch.from_numpy(counts(idx_np, K).astype(np.int32)).cuda()
        Nk, m, e = _state(K, D, rng)
        ws_bytes = L.vqb_vq_ema_workspace_bytes(N, K, D)
        guard = 1 << 16
        buf = torch.full((guard + ws_bytes + guard,), 0xA5, dtype=torch.uint8, device="cuda")
        _lib.check(L.vqb_vq_ema_update_f32(z.data_ptr(), idx.data_ptr(), hist.data_ptr(), N, K, D, 0.9, 1e-5,
                                           Nk.data_ptr(), m.data_ptr(), e.data_ptr(), buf.data_ptr() + guard,
                                           ws_bytes, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
                   "ema")
        torch.cuda.synchronize()
        assert bool((buf[:guard] == 0xA5).all()) and bool((buf[guard + ws_bytes:] == 0xA5).all()), (N, K, D)


# ---- the VQ-VAE ---------------------------------------------------------------------------------------------------
def _setup(name="small_odd", decay=0.9, eps=1e-5):
    from vqvae_b200 import VQVAE
    c = MODEL_CASES[name]
    sd = make_state_dict(seed=c["wseed"], codebook=c["codebook"], codebook_scale=c["codebook_scale"],
                         **{k: c[k] for k in HP})
    m = VQVAE(*(c[k] for k in HP), 0.25, ema_decay=decay, ema_eps=eps)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    return c, sd, m.cuda().train(), torch.from_numpy(make_images(c["batch"], c["size"], c["xseed"]))


def _step(m, xc):
    m.zero_grad(set_to_none=True)
    with torch.enable_grad():
        embedding_loss, x_hat, perplexity = m(xc)
        loss = torch.mean((x_hat - xc) ** 2) / VAR + embedding_loss
        loss.backward()
    return loss, embedding_loss


def _fp64_ema_step(c, sd, x, idx, beta=0.25):
    """fp64 autograd of the restatement with the EMA quantizer's loss (commitment term only) at the codes idx, and the
    restated EMA update from the fp64 z_e -> ({param: grad}, z_e rows fp64)."""
    with torch.enable_grad():
        g = leaf_params({k: sd[k] for k in sd if ".stack." not in k or ".stack.0." in k}, torch.float64)
        E = g["vector_quantization.embedding.weight"]
        captured = {}

        def vq(z, E_, beta_, idx=None):
            zr = z.permute(0, 2, 3, 1).contiguous()
            zf = zr.view(-1, E_.shape[1])
            captured["z"] = zf.detach().clone()
            z_q = E_.detach()[idx].view(zr.shape)
            loss = beta_ * torch.mean((z_q - zf.view(zr.shape)) ** 2)
            z_q = zr + (z_q - zr).detach()
            return loss, z_q.permute(0, 3, 1, 2).contiguous(), None, idx
        import oracle.vqvae_train_port as port
        orig = port.vector_quantizer
        port.vector_quantizer = vq
        try:
            emb, x_hat, _, _ = vqvae_train_forward(x.double(), g, c["n_res_layers"], beta, idx=idx.cpu().reshape(-1))
        finally:
            port.vector_quantizer = orig
        train_loss(x.double(), x_hat, emb, VAR)[0].backward()
    del E
    return {k: v.grad for k, v in g.items()}, captured["z"].numpy(), float(emb)


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_one_training_step_matches_fp64_with_the_restated_ema(precision):
    import vqvae_b200
    c, sd, m, x = _setup("small_odd", decay=0.9)
    vq = m.vector_quantization
    E0 = vq.embedding.weight.detach().cpu().numpy().astype(np.float64)
    with vqvae_b200.precision(precision):
        _, embedding_loss = _step(m, x.cuda())
    torch.cuda.synchronize()
    idx = m.last_min_encoding_indices.reshape(-1)
    want, z64, emb64 = _fp64_ema_step(c, sd, x, idx)
    assert vq.embedding.weight.grad is None
    K = vq.n_e
    np.testing.assert_allclose(emb64, commit_loss_fp64(z64, E0[idx.cpu().numpy()], 0.25), rtol=1e-12)
    np.testing.assert_allclose(float(embedding_loss), emb64, rtol=1e-2 if precision == "tf32" else 1e-4)
    for k, p in m.named_parameters():
        if k == "vector_quantization.embedding.weight":
            continue
        worst = float((p.grad.double().cpu() - want[k]).abs().max() / want[k].abs().max().clamp_min(1e-30))
        bar = 1e-4 if precision == "fp32" else (1e-3 if k.startswith("decoder.inverse_conv_stack.4") else 0.15)
        assert worst <= bar, (k, worst)
    # codebook and buffers: the restated update on the fp64 z_e rows (test_fp32_step_codebook_matches_fp64_on_the_
    # models_own_rows holds the 1e-6 bar on the rows the kernel read)
    n = counts(idx.cpu().numpy(), K)
    s = np.zeros_like(E0)
    np.add.at(s, idx.cpu().numpy(), z64)
    N1, m1, e1 = ema_update_fp64(np.ones(K), E0, n, s, 0.9, 1e-5)
    tol = 1e-5 if precision == "fp32" else 1e-2
    for got, want_t in ((vq.ema_cluster_size, N1), (vq.ema_embed_sum, m1), (vq.embedding.weight, e1)):
        g = got.detach().double().cpu().numpy()
        assert np.abs(g - want_t).max() <= tol * np.abs(want_t).max() + 1e-7, (np.abs(g - want_t).max())


def test_fp32_step_codebook_matches_fp64_on_the_models_own_rows():
    """fp32: the updated codebook and buffers within 1e-6 of fp64 applied to the exact z_e rows the kernel read."""
    import vqvae_b200
    c, sd, m, x = _setup("small_odd", decay=0.9)
    vq = m.vector_quantization
    K = vq.n_e
    E0 = vq.embedding.weight.detach().cpu().numpy().astype(np.float64)
    with vqvae_b200.precision("fp32"), torch.no_grad():
        z_e, _, _, _ = m._encode_rows(x.cuda(), False)
    zr = z_e.reshape(-1, vq.e_dim).cpu().numpy().astype(np.float64)
    with vqvae_b200.precision("fp32"):
        _step(m, x.cuda())
    torch.cuda.synchronize()
    idx = m.last_min_encoding_indices.reshape(-1).cpu().numpy()
    s = np.zeros_like(E0)
    np.add.at(s, idx, zr)
    N1, m1, e1 = ema_update_fp64(np.ones(K), E0, counts(idx, K), s, float(np.float32(0.9)), float(np.float32(1e-5)))
    for got, want in ((vq.ema_cluster_size, N1), (vq.ema_embed_sum, m1), (vq.embedding.weight, e1)):
        g = got.detach().double().cpu().numpy()
        assert np.abs(g - want).max() <= 1e-6 * np.abs(want).max(), np.abs(g - want).max() / np.abs(want).max()


def test_nothing_else_moves_and_launch_counts():
    import vqvae_b200
    from vqvae_b200 import ops
    c, sd, m, x = _setup("cifar_default", decay=0.99)
    _, _, m0, _ = _setup("cifar_default", decay=None)
    xc = x.cuda()
    vq = m.vector_quantization

    def snap():
        return [t.detach().clone() for t in (vq.ema_cluster_size, vq.ema_embed_sum, vq.embedding.weight)]

    def launches(model, fn):
        torch.cuda.synchronize()
        n0 = ops.launch_count()
        fn(model)
        torch.cuda.synchronize()
        return ops.launch_count() - n0
    before = snap()
    for mode in ("fp32", "tf32", "bf16"):
        with vqvae_b200.precision(mode):
            m.eval(), m0.eval()
            with torch.enable_grad():
                assert launches(m, lambda mm: mm(xc)) == launches(m0, lambda mm: mm(xc))   # eval, grad enabled
            m.train(), m0.train()
            with torch.no_grad():
                assert launches(m, lambda mm: mm(xc)) == launches(m0, lambda mm: mm(xc))   # no_grad
                assert launches(m, lambda mm: mm.encode(xc)) == launches(m0, lambda mm: mm.encode(xc))
                codes = m.encode(xc)
                hw = (xc.shape[2] // 4, xc.shape[3] // 4)
                assert launches(m, lambda mm: mm.decode(codes, hw)) == launches(m0, lambda mm: mm.decode(codes, hw))
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(before, snap()))
    # a training step: the gradient codebook's launches, minus its backward, plus the commit backward and the update
    with vqvae_b200.precision("fp32"):
        _step(m, xc), _step(m0, xc)                 # first steps build the backward packings
        ema, ref = launches(m, lambda mm: _step(mm, xc)), launches(m0, lambda mm: _step(mm, xc))
    assert ema == ref + 5, (ema, ref)
    assert not all(torch.equal(a, b) for a, b in zip(before, snap()))


def _snapshot(m, opt):
    out = {}
    for k, p in m.named_parameters():
        out[k] = p.detach().clone()
        for s in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq", "step"):
            if p in opt.state and s in opt.state[p]:
                out[k + "/" + s] = opt.state[p][s].clone()
    for k, b in m.named_buffers():
        out[k] = b.clone()
    return out


def _main_loop_model(decay=0.99):
    from vqvae_b200 import VQVAE
    hp = dict(h_dim=128, res_h_dim=32, n_res_layers=2, n_embeddings=512, embedding_dim=64)
    m = VQVAE(*hp.values(), 0.25, ema_decay=decay)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in make_state_dict(seed=0, **hp).items()})
    return m.cuda().train()


def _opt_step(m, x, opt):
    opt.zero_grad(set_to_none=True)
    with torch.enable_grad():
        embedding_loss, x_hat, _ = m(x)
        loss = torch.mean((x_hat - x) ** 2) / VAR + embedding_loss
        loss.backward()
    opt.step()
    return loss


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_main_py_loop_is_bitwise_reproducible_eager_and_replayed(precision):
    import vqvae_b200
    from vqvae_b200 import ops
    from vqvae_b200.optim import Adam
    x = torch.from_numpy(make_images(32, 32, seed=7)).cuda()
    with vqvae_b200.precision(precision):
        runs = []
        for _ in range(2):
            m = _main_loop_model()
            opt = Adam(m.parameters(), lr=3e-4, amsgrad=True)
            losses = [_opt_step(m, x, opt).item() for _ in range(10)]
            runs.append((losses, _snapshot(m, opt)))
        assert runs[0][0] == runs[1][0]
        a, b = runs[0][1], runs[1][1]
        assert all(torch.equal(a[k], b[k]) for k in a), [k for k in a if not torch.equal(a[k], b[k])][:5]
        # a captured step replayed 10 times after one eager warm-up step = 11 eager steps
        ma, mb = _main_loop_model(), _main_loop_model()
        oa, ob = Adam(ma.parameters(), lr=3e-4, amsgrad=True), Adam(mb.parameters(), lr=3e-4, amsgrad=True)
        eager = [_opt_step(ma, x, oa).item() for _ in range(11)]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            _opt_step(mb, x, ob)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            loss = _opt_step(mb, x, ob)
        got = []
        for _ in range(10):
            n0 = ops.launch_count()
            graph.replay()
            assert ops.launch_count() == n0
            got.append(loss.item())
        torch.cuda.synchronize()
    assert got == eager[1:]
    a, b = _snapshot(ma, oa), _snapshot(mb, ob)
    assert all(torch.equal(a[k], b[k]) for k in a), [k for k in a if not torch.equal(a[k], b[k])][:5]
    assert a["vector_quantization.ema_cluster_size"].sum().item() > 0


def test_vector_quantizer_alone_updates_in_training_only_and_its_dz_matches_fp64():
    import vqvae_b200
    rng = np.random.default_rng(4)
    K, D = 64, 16
    vq = vqvae_b200.VectorQuantizer(K, D, 0.25, decay=0.8).cuda()
    with torch.no_grad():
        vq.embedding.weight.copy_(torch.randn(K, D) * 0.5)
        vq.ema_embed_sum.copy_(vq.embedding.weight)
    z = torch.from_numpy(rng.standard_normal((2, D, 8, 8)).astype(np.float32)).cuda()
    E0 = vq.embedding.weight.detach().clone()
    vq.eval()
    zz = z.clone().requires_grad_(True)
    with torch.enable_grad():
        loss, z_q, _, _, idx = vq(zz)
    assert torch.equal(vq.embedding.weight, E0) and torch.equal(vq.ema_cluster_size, torch.ones(K, device="cuda"))
    vq.train()
    zz = z.clone().requires_grad_(True)
    g_zq = torch.from_numpy(rng.standard_normal(z.shape).astype(np.float32)).cuda()
    with torch.enable_grad():
        loss, z_q, _, _, idx = vq(zz)
        (loss * 3.0 + (z_q * g_zq).sum()).backward()
    torch.cuda.synchronize()
    assert vq.embedding.weight.grad is None
    rows = z.permute(0, 2, 3, 1).reshape(-1, D).cpu().numpy()
    ids = idx.reshape(-1).cpu().numpy()
    zq_rows = E0.cpu().numpy()[ids]
    np.testing.assert_allclose(float(loss), commit_loss_fp64(rows, zq_rows, 0.25), rtol=1e-5)
    g_rows = g_zq.permute(0, 2, 3, 1).reshape(-1, D).cpu().numpy()
    want = commit_dz_fp64(rows, zq_rows, g_rows, 3.0, 0.25)
    got = zz.grad.permute(0, 2, 3, 1).reshape(-1, D).cpu().numpy()
    np.testing.assert_allclose(got, want, atol=1e-6 * np.abs(want).max(), rtol=0)
    s = segment_sums(rows, ids, K)
    N1, m1, e1 = ema_update_fp64(np.ones(K), E0.cpu().numpy(), counts(ids, K), s, float(np.float32(0.8)),
                                 float(np.float32(1e-5)))
    np.testing.assert_allclose(vq.embedding.weight.detach().cpu().numpy(), e1, rtol=1e-5, atol=1e-6)
    assert not torch.equal(vq.embedding.weight, E0)


def test_checkpoint_round_trip_restores_the_buffers_and_a_reference_file_restarts_them(tmp_path):
    import vqvae_b200
    c, sd, m, x = _setup("small_odd", decay=0.9)
    with vqvae_b200.precision("fp32"):
        _step(m, x.cuda())
    hp = dict(n_hiddens=c["h_dim"], n_residual_hiddens=c["res_h_dim"], n_residual_layers=c["n_res_layers"],
              n_embeddings=c["n_embeddings"], embedding_dim=c["embedding_dim"], beta=0.25)
    path = str(tmp_path / "ema.pth")
    vqvae_b200.save_checkpoint(m, {}, hp, path)
    m2, _ = vqvae_b200.load_checkpoint(path)
    a, b = m.vector_quantization, m2.vector_quantization
    assert b.decay == 0.9
    for t in ("ema_cluster_size", "ema_embed_sum"):
        assert torch.equal(getattr(a, t), getattr(b, t))
    assert torch.equal(a.embedding.weight, b.embedding.weight)
    # the reference's own file (no vq_ema) into an EMA model: the buffers restart from its codebook
    m3 = _setup("small_odd", decay=0.9)[2]
    ref = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ckpt_small_odd.pth"),
                     map_location="cpu", weights_only=False)
    m3.load_state_dict(ref["model"])
    v3 = m3.vector_quantization
    assert torch.equal(v3.ema_cluster_size, torch.ones_like(v3.ema_cluster_size))
    assert torch.equal(v3.ema_embed_sum, v3.embedding.weight.detach())

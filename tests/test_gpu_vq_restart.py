"""Dead-code restarts of the EMA codebook on the H100: vqb_vq_ema_restart_f32 bit for bit against tests/vq_restart_ref.py
after a real update, determinism (eager and in a CUDA graph) and the workspace bound, main.py's loop with restarts on
reproducible eagerly and under replay, the launches and random draws each setting adds, and a collapsed codebook
brought back by restarts."""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_gpu_vq_ema import _main_loop_model, _opt_step, _setup, _snapshot, _step
from tests.vq_ema_ref import counts
from tests.vq_restart_ref import restart

pytestmark = pytest.mark.gpu

RESTART_LAUNCHES = 12


def _problem(N, K, D, case, seed):
    """(z, codes, N0, decay, t, u) for one case; the update runs from N0 with m = e = a random codebook."""
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((N, D), dtype=np.float32)
    codes = rng.integers(0, K, N)
    u = rng.random(N, dtype=np.float32)
    N0 = np.ones(K, np.float32)
    decay, t = 0.9, 1e30                                    # every code dead unless the case says otherwise
    if case == "none":
        N0 = rng.uniform(0.5, 2.0, K).astype(np.float32)
        t = 0.25
    elif case == "half":                                    # the odd codes take no row and start at 0
        codes = rng.integers(0, (K + 1) // 2, N) * 2
        N0 = np.where(np.arange(K) % 2 == 0, 5.0, 0.0).astype(np.float32)
        t = 0.5
    elif case == "equal":                                   # decay 0: N_k = n_k exactly; n_k == 1 is not dead
        decay, t = 0.0, 1.0
    elif case == "ties":
        u = (rng.integers(0, 8, N) / 8).astype(np.float32)
    elif case == "nan":
        N0[::3] = np.nan
    else:
        assert case == "all", case
    return z, codes, N0, decay, t, u


def _updated_state(z, codes, N0, decay, K, D, seed):
    from vqvae_b200 import ops
    rng = np.random.default_rng(seed + 1)
    e0 = torch.from_numpy(rng.standard_normal((K, D), dtype=np.float32) * 0.1)
    state = [torch.from_numpy(N0).cuda(), e0.cuda(), e0.clone().cuda()]
    zc, idx = torch.from_numpy(z).cuda(), torch.from_numpy(codes).cuda()
    hist = torch.from_numpy(counts(codes, K).astype(np.int32)).cuda()
    ops.vq_ema_update(zc, idx, hist, decay, 1e-5, *state)
    return zc, state


def _bits(t):
    return np.ascontiguousarray(t.detach().cpu().numpy()).view(np.uint32)


GRID = [(1, 1, 4, "all"), (1, 7, 64, "all"), (1, 7, 4, "none"), (1000, 7, 4, "half"), (1000, 7, 256, "nan"),
        (1000, 512, 64, "all"), (100, 1024, 64, "all"), (5000, 8192, 4, "all"), (2000, 1024, 64, "equal"),
        (16384, 512, 64, "none"), (16384, 512, 64, "half"), (16384, 8192, 64, "ties"), (16384, 8192, 64, "all"),
        (16384, 8192, 256, "equal"), (65536, 8192, 256, "half"), (65536, 1024, 256, "nan"),
        (262144, 7, 256, "all"), (524288, 1024, 64, "ties"), (1 << 20, 8192, 64, "all"), (1 << 20, 8192, 64, "none"),
        (1 << 20, 512, 4, "half"), (1 << 20, 1024, 64, "nan"), (1 << 20, 1, 64, "ties"), (1 << 20, 8192, 4, "ties")]


@pytest.mark.parametrize("N, K, D, case", GRID)
def test_restart_is_the_reference_bit_for_bit(N, K, D, case):
    from vqvae_b200 import ops
    seed = N * 31 + K * 7 + D
    z, codes, N0, decay, t, u = _problem(N, K, D, case, seed)
    zc, state = _updated_state(z, codes, N0, decay, K, D, seed)
    before = [s.clone() for s in state]
    cnt = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    ops.vq_ema_restart(zc, torch.from_numpy(u).cuda(), t, *state, cnt)
    torch.cuda.synchronize()
    want = restart(z, u, t, *(s.cpu().numpy() for s in before))
    for name, got, w in zip(("cluster_size", "embed_sum", "codebook"), state, want[:3]):
        bad = np.nonzero(_bits(got).reshape(got.shape[0], -1) != w.view(np.uint32).reshape(got.shape[0], -1))[0]
        assert bad.size == 0, f"{name}: {np.unique(bad).size} codes differ, first {np.unique(bad)[:5]}"
    assert int(cnt.item()) == want[3]
    if case == "none":                              # nothing dead: every bit is the update's
        assert want[3] == 0 and all(torch.equal(a, b) for a, b in zip(state, before))
    if case == "equal":
        n = counts(codes, K)
        assert (n == 1).any() and want[3] == min(int((n == 0).sum()), N)
    if case in ("all", "ties") or (case == "nan" and K > 1):
        assert want[3] > 0


@pytest.mark.parametrize("case", ["all", "none"])
def test_two_calls_and_a_graph_replay_are_bitwise_equal(case):
    from vqvae_b200 import ops
    N, K, D = 1 << 18, 8192, 64
    z, codes, N0, decay, t, u = _problem(N, K, D, case, 9)
    uc = torch.from_numpy(u).cuda()
    zc, s0 = _updated_state(z, codes, N0, decay, K, D, 9)
    a, b, c = ([x.clone() for x in s0] for _ in range(3))
    ca, cb, cc = (torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(3))
    ops.vq_ema_restart(zc, uc, t, *a, ca)
    ops.vq_ema_restart(zc, uc, t, *b, cb)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.vq_ema_restart(zc, uc, t, *[x.clone() for x in c], cc.clone())      # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.vq_ema_restart(zc, uc, t, *c, cc)
    n0 = ops.launch_count()
    g.replay()
    assert ops.launch_count() == n0
    torch.cuda.synchronize()
    for x, y, w in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, w)
    assert int(ca) == int(cb) == int(cc) == (K if case == "all" else 0)


def test_restart_stays_inside_its_workspace():
    from vqvae_b200 import _lib, ops
    L = ops.lib()
    for N, K, D, case in ((16384, 8192, 64, "all"), (1000, 7, 4, "half"), (3, 8192, 4, "ties"),
                          (65536, 512, 256, "none")):
        z, codes, N0, decay, t, u = _problem(N, K, D, case, 3)
        zc, (Nk, m, e) = _updated_state(z, codes, N0, decay, K, D, 3)
        uc = torch.from_numpy(u).cuda()
        cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
        ws_bytes = L.vqb_vq_ema_restart_workspace_bytes(N, K)
        guard = 1 << 16
        buf = torch.full((guard + ws_bytes + guard,), 0xA5, dtype=torch.uint8, device="cuda")
        _lib.check(L.vqb_vq_ema_restart_f32(zc.data_ptr(), uc.data_ptr(), N, K, D, t, Nk.data_ptr(), m.data_ptr(),
                                            e.data_ptr(), cnt.data_ptr(), buf.data_ptr() + guard, ws_bytes,
                                            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "restart")
        torch.cuda.synchronize()
        assert bool((buf[:guard] == 0xA5).all()) and bool((buf[guard + ws_bytes:] == 0xA5).all()), (N, K, D)


# ---- training ----------------------------------------------------------------------------------------------------
THRESHOLD = 0.95        # main.py's model: an unused code's N = 0.99^s falls below it after 6 updates


def _restart_model():
    m = _main_loop_model()
    m.vector_quantization.dead_code_threshold = THRESHOLD
    return m


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_main_py_loop_with_restarts_is_bitwise_reproducible_eager_and_replayed(precision):
    import vqvae_b200
    from oracle.weights import make_images
    from vqvae_b200 import ops
    from vqvae_b200.optim import Adam
    x = torch.from_numpy(make_images(32, 32, seed=7)).cuda()
    with vqvae_b200.precision(precision):
        runs = []
        for _ in range(2):
            torch.manual_seed(0)
            m = _restart_model()
            opt = Adam(m.parameters(), lr=3e-4, amsgrad=True)
            losses, restarts = [], []
            for _ in range(10):
                losses.append(_opt_step(m, x, opt).item())
                restarts.append(int(m.vector_quantization.last_restarts))
            runs.append((losses, restarts, _snapshot(m, opt)))
        assert runs[0][:2] == runs[1][:2]
        assert max(runs[0][1]) > 0, runs[0][1]                     # the loop does restart codes
        a, b = runs[0][2], runs[1][2]
        assert all(torch.equal(a[k], b[k]) for k in a), [k for k in a if not torch.equal(a[k], b[k])][:5]
        # a captured step replayed 10 times = 10 eager steps from the same generator state
        ma, mb = _restart_model(), _restart_model()
        oa, ob = Adam(ma.parameters(), lr=3e-4, amsgrad=True), Adam(mb.parameters(), lr=3e-4, amsgrad=True)
        torch.manual_seed(1)
        _opt_step(ma, x, oa)
        torch.manual_seed(1)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            _opt_step(mb, x, ob)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            loss = _opt_step(mb, x, ob)
        torch.cuda.manual_seed(2)
        eager = []
        for _ in range(10):
            eager.append((_opt_step(ma, x, oa).item(), int(ma.vector_quantization.last_restarts)))
        torch.cuda.manual_seed(2)
        got = []
        for _ in range(10):
            n0 = ops.launch_count()
            graph.replay()
            assert ops.launch_count() == n0
            got.append((loss.item(), int(mb.vector_quantization.last_restarts)))
        torch.cuda.synchronize()
    assert got == eager
    assert max(r for _, r in eager) > 0
    a, b = _snapshot(ma, oa), _snapshot(mb, ob)
    assert all(torch.equal(a[k], b[k]) for k in a), [k for k in a if not torch.equal(a[k], b[k])][:5]


def test_launches_and_random_draws_per_setting():
    import vqvae_b200
    from vqvae_b200 import ops
    _, _, m, x = _setup("cifar_default", decay=0.99)
    _, _, m0, _ = _setup("cifar_default", decay=None)
    xc = x.cuda()
    vq = m.vector_quantization
    n_rows = xc.shape[0] * (xc.shape[2] // 4) * (xc.shape[3] // 4)

    def launches(model):
        torch.cuda.synchronize()
        n0 = ops.launch_count()
        _step(model, xc)
        torch.cuda.synchronize()
        return ops.launch_count() - n0

    with vqvae_b200.precision("fp32"):
        _step(m, xc), _step(m0, xc)                 # first steps build the backward packings
        ref = launches(m0)
        rng = torch.cuda.get_rng_state()
        assert launches(m) == ref + 5               # threshold None: the EMA path's launches, no random numbers
        assert torch.equal(torch.cuda.get_rng_state(), rng)
        vq.dead_code_threshold = 0.5
        torch.cuda.manual_seed(3)
        assert launches(m) == ref + 5 + RESTART_LAUNCHES
        after_step = torch.cuda.get_rng_state()
        torch.cuda.manual_seed(3)
        torch.rand((n_rows,), device="cuda")        # exactly one draw of one uniform per row
        assert torch.equal(after_step, torch.cuda.get_rng_state())
        # eval, no_grad, encode and decode never restart
        vq.dead_code_threshold = 1e30
        snap = [t.clone() for t in (vq.ema_cluster_size, vq.ema_embed_sum, vq.embedding.weight, vq.last_restarts)]
        rng = torch.cuda.get_rng_state()
        m.eval()
        with torch.enable_grad():
            m(xc)
        m.train()
        with torch.no_grad():
            m(xc)
            codes = m.encode(xc)
            m.decode(codes, (xc.shape[2] // 4, xc.shape[3] // 4))
        torch.cuda.synchronize()
        assert torch.equal(torch.cuda.get_rng_state(), rng)
        assert all(torch.equal(a, b) for a, b in
                   zip(snap, (vq.ema_cluster_size, vq.ema_embed_sum, vq.embedding.weight, vq.last_restarts)))
        _step(m, xc)                                # a training step with every code dead restarts min(K, N)
        torch.cuda.synchronize()
        assert int(vq.last_restarts) == min(vq.n_e, n_rows)


def _collapse_run(threshold, calls=100):
    """A lone EMA quantizer, every code at the origin, on 32 tight clusters: (clusters holding a code within 3 sigma of
    their centre, the last call's perplexity)."""
    import vqvae_b200
    K, D, per, sigma, radius = 32, 8, 64, 0.05, 1.0
    rng = np.random.default_rng(11)
    c = np.zeros(D)
    c[0] = 5.0                                              # |c| > 2R + 3 sigma
    dirs = rng.standard_normal((K, D))
    centres = c + radius * dirs / np.linalg.norm(dirs, axis=1, keepdims=True)
    rows = (np.repeat(centres, per, axis=0) + sigma * rng.standard_normal((K * per, D))).astype(np.float32)
    rows = rows[rng.permutation(K * per)]
    z = torch.from_numpy(rows).view(32, 8, 8, D).permute(0, 3, 1, 2).contiguous().cuda()
    vq = vqvae_b200.VectorQuantizer(K, D, 0.25, decay=0.9).cuda().train()
    with torch.no_grad():
        vq.embedding.weight.zero_()
        vq.ema_embed_sum.zero_()
    vq.dead_code_threshold = threshold
    torch.manual_seed(0)
    for _ in range(calls):
        with torch.enable_grad():
            _, _, perp, _, _ = vq(z.clone().requires_grad_(True))
    torch.cuda.synchronize()
    e = vq.embedding.weight.detach().double().cpu().numpy()
    dist = np.linalg.norm(centres[:, None, :] - e[None, :, :], axis=2)
    return int((dist.min(axis=1) < 3 * sigma).sum()), float(perp)


def test_restarts_bring_back_a_collapsed_codebook():
    covered, perp = _collapse_run(None)
    assert perp < 1.5, perp
    covered, perp = _collapse_run(0.5)
    assert covered >= 14 and perp > 10, (covered, perp)

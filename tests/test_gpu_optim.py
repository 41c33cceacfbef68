"""vqvae_b200.optim.Adam on the H100: one step against torch.optim.Adam(foreach=False) within 2 ulp, every cached
packing refreshed bitwise as the single-packing entry points make it, mask A's taps zeroed, two launches per group, the
reference's training loops against fp64 and the reference, state-dict round trips with torch's Adam, a whole training
step as one CUDA graph, and a HostPipeline built before the steps."""
import contextlib
import copy
import io
import os

import numpy as np
import pytest
import torch

from oracle.prior_port import PRIOR_CASES, make_prior_inputs, make_prior_state_dict
from oracle.prior_train_port import leaf_params, prior_logits, prior_loss

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HP = dict(h_dim=128, res_h_dim=32, n_res_layers=2, n_embeddings=512, embedding_dim=64)   # main.py's model
VAR = 0.0625


def _vqvae(seed=0):
    from models.vqvae import VQVAE
    from oracle.weights import make_state_dict
    m = VQVAE(*HP.values(), 0.25)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in make_state_dict(seed=seed, **HP).items()})
    return m.cuda().train()


def _images(B, seed=7):
    from oracle.weights import make_images
    return torch.from_numpy(make_images(B, 32, seed=seed)).cuda()


def _prior(name="prior_ragged", precision="fp32"):
    from pixelcnn.models import GatedPixelCNN
    c = PRIOR_CASES[name]
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"])
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    m.precision = precision
    codes, labels, _ = make_prior_inputs(c)
    return c, sd, m.cuda(), torch.from_numpy(codes), torch.from_numpy(labels)


def _vq_loss(m, x):
    embedding_loss, x_hat, _ = m(x)
    return torch.mean((x_hat - x) ** 2) / VAR + embedding_loss


def _vq_step(m, x, opt):
    opt.zero_grad(set_to_none=True)
    with torch.enable_grad():
        loss = _vq_loss(m, x)
        loss.backward()
    opt.step()
    return loss


def _prior_step(m, x, lab, opt):
    opt.zero_grad(set_to_none=True)
    with torch.enable_grad():
        loss = prior_loss(m(x, lab), x)
        loss.backward()
    opt.step()
    return loss


def _ulps(a, b):
    """max distance in units in the last place between two fp32 tensors (0 = bitwise)."""
    def ordered(t):
        i = t.detach().contiguous().view(torch.int32).long()
        return torch.where(i < 0, -(i & 0x7FFFFFFF), i)
    return int((ordered(a) - ordered(b)).abs().max()) if a.numel() else 0


def _random_grads(params, gen, scale=1e-2):
    for p in params:
        p.grad = torch.randn(p.shape, generator=gen, device="cuda") * scale


# ---- one step against torch -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("wd", [0.0, 1e-2])
@pytest.mark.parametrize("amsgrad", [False, True])
@pytest.mark.parametrize("model", ["vqvae", "prior"])
def test_one_step_matches_torch_adam_within_2_ulp(model, amsgrad, wd):
    from vqvae_b200.optim import Adam
    base = list(_vqvae().parameters()) if model == "vqvae" else list(_prior("prior_default")[2].parameters())
    gen = torch.Generator(device="cuda").manual_seed(0)
    ref = [torch.nn.Parameter(p.detach().clone()) for p in base]
    ropt = torch.optim.Adam(ref, lr=1e-3, weight_decay=wd, amsgrad=amsgrad, foreach=False)
    for _ in range(3):                  # moments and step counts that are not the initial ones
        _random_grads(ref, gen)
        ropt.step()
    ours = [torch.nn.Parameter(p.detach().clone()) for p in ref]
    opt = Adam(ours, lr=1e-3, weight_decay=wd, amsgrad=amsgrad)
    opt.load_state_dict(copy.deepcopy(ropt.state_dict()))     # (state_dict() holds torch's own moment tensors)
    _random_grads(ref, gen)
    for p, q in zip(ours, ref):
        p.grad = q.grad.clone()
    ropt.step()
    opt.step()
    worst, n_equal, n = 0, 0, 0
    for p, q in zip(ours, ref):
        pairs = [(p, q)] + [(opt.state[p][k], ropt.state[q][k]) for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")
                            if k in ropt.state[q]]
        for a, b in pairs:
            u = _ulps(a, b)
            worst = max(worst, u)
            n_equal += int(torch.equal(a, b))
            n += 1
        assert float(opt.state[p]["step"]) == float(ropt.state[q]["step"]) == 4.0
    print(f"{model} amsgrad={amsgrad} wd={wd}: worst {worst} ulp over {n} tensors"
          + (" (bitwise)" if n_equal == n else f" ({n_equal} bitwise)"))
    assert worst <= 2


# ---- packings -------------------------------------------------------------------------------------------------------
def _check_packings(m):
    """Every cached packing of `m` is current and bitwise what its single-packing entry point makes now."""
    from vqvae_b200.modules import _packed_current, pack_spec
    from vqvae_b200.optim import _layout_bytes
    keys = set()
    for name, p in m.named_parameters():
        for key, (_, buf) in getattr(p, "_vqb_packed", {}).items():
            if buf is None:
                continue
            assert _packed_current(p, key), (name, key)
            pack, layouts = pack_spec(p, key)
            fresh = pack(p, None)
            for off, f in layouts:
                end = _layout_bytes(off, f)
                assert torch.equal(buf.view(torch.uint8)[off:end], fresh.view(torch.uint8)[off:end]), (name, key)
            keys.add(key[:1] + ((key[1],) if key[0] != "prior" else ()))
    return keys


def _mask_a_zero(m):
    l0 = m.layers[0]
    return bool((l0.vert_stack.weight[:, :, -1] == 0).all()) and bool((l0.horiz_stack.weight[:, :, :, -1] == 0).all())


def test_vqvae_packings_are_refreshed_bitwise_and_the_next_forward_packs_nothing():
    import vqvae_b200
    from vqvae_b200 import ops
    from vqvae_b200._lib import CONVT_K4S2_OUT, RES_W2
    from vqvae_b200.optim import Adam
    m, x = _vqvae(), _images(8)
    with torch.no_grad():
        m.eval()
        with vqvae_b200.precision("bf16"):
            m(x)                            # bf16 packings
        with vqvae_b200.precision("fp32"):
            m(x)                            # fp32 forward packings
        m.train()
    opt = Adam(m.parameters(), lr=1e-3)
    _random_grads(m.parameters(), torch.Generator(device="cuda").manual_seed(1))
    opt.step()
    keys = _check_packings(m)
    assert {("bf16", CONVT_K4S2_OUT), ("bf16", RES_W2), ("f32", False), ("f32", True)} <= keys
    dec_out = m.decoder.inverse_conv_stack[4].weight
    assert ("f32", False) not in dec_out._vqb_packed           # no input-gradient packing before the first backward
    with vqvae_b200.precision("fp32"):
        _vq_step(m, x, opt)                 # the backward creates the input-gradient packings: refreshed by this step
        assert ("f32", False) in dec_out._vqb_packed
        _check_packings(m)
        _vq_step(m, x, opt)
        _check_packings(m)
        counts = []
        with torch.no_grad():
            for _ in range(2):
                n0 = ops.launch_count()
                m(x)
                counts.append(ops.launch_count() - n0)
    assert counts[0] == counts[1]           # the forward right after the step packs nothing


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_prior_packings_are_refreshed_bitwise_and_mask_a_taps_are_zero(precision):
    from vqvae_b200 import ops
    from vqvae_b200.optim import Adam
    c, _, m, x, lab = _prior("prior_ragged", precision)
    xc, lc = x.cuda(), lab.cuda()
    opt = Adam(m.parameters(), lr=1e-2)
    for _ in range(3):
        _prior_step(m, xc, lc, opt)
        assert ("prior",) in _check_packings(m)
        assert _mask_a_zero(m)
        counts = []
        with torch.no_grad():
            for _ in range(2):
                n0 = ops.launch_count()
                m(xc, lc)
                counts.append(ops.launch_count() - n0)
        assert counts[0] == counts[1] == (2 + 2 * c["n_layers"] if precision == "fp32" else 3 + 4 * c["n_layers"])


def test_two_launches_per_group_whatever_the_model_size():
    from vqvae_b200 import ops
    from vqvae_b200.optim import Adam
    gen = torch.Generator(device="cuda").manual_seed(2)
    for name in ("prior_ragged", "prior_default"):
        c, _, m, x, lab = _prior(name)
        with torch.no_grad():
            m(x.cuda(), lab.cuda())
        for groups, want in (([{"params": m.parameters()}], 2),
                             ([{"params": m.layers.parameters()}, {"params": m.output_conv.parameters(), "lr": 1e-4},
                               {"params": m.embedding.parameters()}], 6)):
            opt = Adam(groups, amsgrad=True)
            _random_grads(m.parameters(), gen)
            n0 = ops.launch_count()
            opt.step()
            assert ops.launch_count() - n0 == want, (name, want)
    m = _vqvae()
    opt = Adam(m.parameters())
    _random_grads(m.parameters(), gen)
    m.encoder.conv_stack[0].weight.grad = None         # skipped: its step does not advance
    n0 = ops.launch_count()
    opt.step()
    assert ops.launch_count() - n0 == 2
    assert m.encoder.conv_stack[0].weight not in opt.state
    assert all(float(opt.state[p]["step"]) == 1.0 for p in m.parameters() if p.grad is not None)


# ---- trajectories -------------------------------------------------------------------------------------------------
def _prior_fp64_losses(c, sd, x, lab, steps):
    g = leaf_params(sd, torch.float64)
    opt = torch.optim.Adam(list(g.values()), lr=3e-4)
    losses = []
    with torch.enable_grad():
        for _ in range(steps):
            loss = prior_loss(prior_logits(g, x, lab, c["n_layers"]), x)
            opt.zero_grad()
            loss.backward()
            opt.step()
            losses.append(loss.item())
    return losses


def _prior_run(m, xc, lc, schedule):
    """Losses of the reference's Adam loop (lr 3e-4), switching optimizer at each (n_steps, make_opt) of `schedule`
    and carrying the state over by state_dict."""
    got, opt = [], None
    for n, make in schedule:
        new = make(m.parameters(), lr=3e-4)
        if opt is not None:
            new.load_state_dict(opt.state_dict())
        opt = new
        for _ in range(n):
            got.append(_prior_step(m, xc, lc, opt).item())
    return got


def test_prior_adam_loop_tracks_fp64_and_round_trips_through_torch_adam():
    from vqvae_b200.optim import Adam
    c, sd, m, x, lab = _prior("prior_ragged")
    want = _prior_fp64_losses(c, sd, x, lab, 100)
    xc, lc = x.cuda(), lab.cuda()
    got = _prior_run(m, xc, lc, [(100, Adam)])
    rel = max(abs(a - b) / abs(b) for a, b in zip(got, want))
    _, _, m2, _, _ = _prior("prior_ragged")
    mixed = _prior_run(m2, xc, lc, [(33, torch.optim.Adam), (33, Adam), (34, torch.optim.Adam)])
    rel_mixed = max(abs(a - b) / abs(b) for a, b in zip(mixed, want))
    print(f"prior adam: loss {got[0]:.5f} -> {got[99]:.5f}; worst relative to fp64 {rel:.2e} fused, "
          f"{rel_mixed:.2e} torch -> fused -> torch")
    assert rel <= 2e-6 and rel_mixed <= 2e-6


def _vq_run(m, x, schedule):
    """Losses of main.py's loop (Adam amsgrad, lr 3e-4), switching optimizer at each (n_steps, make_opt) of `schedule`
    and carrying the state over by state_dict."""
    got, opt = [], None
    for n, make in schedule:
        new = make(m.parameters(), lr=3e-4, amsgrad=True)
        if opt is not None:
            new.load_state_dict(opt.state_dict())
        opt = new
        for _ in range(n):
            got.append(_vq_step(m, x, opt).item())
    return np.array(got)


def _vq_run_shadowed(m, x, steps):
    """main.py's loop with the fused Adam, every step also applied by torch.optim.Adam(foreach=False) to a copy of the
    parameters from the same gradients: parameters and moments must stay bitwise equal.  -> losses"""
    from vqvae_b200.optim import Adam
    params = list(m.parameters())
    twin = [torch.nn.Parameter(p.detach().clone()) for p in params]
    opt = Adam(params, lr=3e-4, amsgrad=True)
    topt = torch.optim.Adam(twin, lr=3e-4, amsgrad=True, foreach=False)
    got = []
    for _ in range(steps):
        opt.zero_grad(set_to_none=True)
        with torch.enable_grad():
            loss = _vq_loss(m, x)
            loss.backward()
        for t, p in zip(twin, params):
            t.grad = p.grad.clone()
        opt.step()
        topt.step()
        for t, p in zip(twin, params):
            assert torch.equal(t, p)
            for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
                assert torch.equal(topt.state[t][k], opt.state[p][k]), k
        got.append(loss.item())
    return np.array(got)


def test_main_py_adam_loop_tracks_the_reference_and_round_trips_through_torch_adam():
    """main.py's loop on cifar_spread.  The VQ-VAE's codebook gradient is summed with float atomics, and at step 14 of
    this case an argmin flips with the last bits of that sum: the loop follows one of two trajectories, which are the
    reference's own two runs (4 threads and 1 thread, 1.5e-4 apart at the end).  torch's Adam on this model takes
    either, as does the fused one.  So each run must follow one of the reference's runs within 1e-4 at every step,
    and the fused step must be bitwise torch's Adam applied to the same gradients, step by step."""
    import vqvae_b200
    from oracle.make_golden import MODEL_CASES
    from oracle.weights import make_images, make_state_dict
    from models.vqvae import VQVAE
    from vqvae_b200.optim import Adam
    c = MODEL_CASES["cifar_spread"]
    keys = ("h_dim", "res_h_dim", "n_res_layers", "n_embeddings", "embedding_dim")
    sd = make_state_dict(seed=c["wseed"], codebook=c["codebook"], codebook_scale=c["codebook_scale"],
                         **{k: c[k] for k in keys})
    with np.load(os.path.join(ROOT, "tests", "golden", "vqvae_train_cifar_spread.npz")) as d:
        gold = {k: d[k] for k in d.files}
    steps = len(gold["trajectory"])
    x = torch.from_numpy(make_images(c["batch"], c["size"], c["xseed"])).cuda()

    def model():
        m = VQVAE(*(c[k] for k in keys), 0.25)
        m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
        return m.cuda().train()
    with vqvae_b200.precision("fp32"):
        torch_run = _vq_run(model(), x, [(steps, torch.optim.Adam)])
        fused = _vq_run_shadowed(model(), x, steps)
        third = steps // 3
        mixed = _vq_run(model(), x, [(third, torch.optim.Adam), (third, Adam), (steps - 2 * third, torch.optim.Adam)])
    refs = {"4 threads": gold["trajectory_threads4"][:, 0], "1 thread": gold["trajectory"][:, 0]}
    for name, got in (("torch", torch_run), ("fused", fused), ("torch -> fused -> torch", mixed)):
        rel = {k: float(np.max(np.abs(got - r) / np.abs(r))) for k, r in refs.items()}
        follows = min(rel, key=rel.get)
        print(f"main.py adam amsgrad, {name}: {got[0]:.5f} -> {got[-1]:.5f}; worst relative to the reference's run "
              + ", ".join(f"with {k} {v:.2e}" for k, v in rel.items()) + f": follows the run with {follows}")
        assert rel[follows] <= 1e-4


# ---- a whole training step as one CUDA graph ----------------------------------------------------------------------
def _capture(step_fn):
    """One eager warm-up step on a side stream, then the step captured as one graph -> (graph, its static loss)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step_fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = step_fn()
    return graph, loss


def _snapshot(m, opt):
    out = {}
    for k, p in m.named_parameters():
        out[k] = p.detach().clone()
        for s in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq", "step"):
            if s in opt.state[p]:
                out[k + "/" + s] = opt.state[p][s].clone()
    return out


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_prior_whole_step_graph_is_bitwise_the_eager_steps(precision):
    from vqvae_b200 import ops
    from vqvae_b200.optim import Adam
    _, _, ma, x, lab = _prior("prior_ragged", precision)
    _, _, mb, _, _ = _prior("prior_ragged", precision)
    xc, lc = x.cuda(), lab.cuda()
    oa, ob = Adam(ma.parameters(), lr=1e-3), Adam(mb.parameters(), lr=1e-3)
    eager = [_prior_step(ma, xc, lc, oa).item() for _ in range(11)]
    graph, loss = _capture(lambda: _prior_step(mb, xc, lc, ob))
    got = []
    for _ in range(10):
        n0 = ops.launch_count()
        graph.replay()
        assert ops.launch_count() == n0
        got.append(loss.item())
    torch.cuda.synchronize()
    a, b = _snapshot(ma, oa), _snapshot(mb, ob)
    assert all(torch.equal(a[k], b[k]) for k in a), [k for k in a if not torch.equal(a[k], b[k])][:5]
    assert got == eager[1:]
    assert float(ob.state[next(mb.parameters())]["step"]) == 11.0
    assert _mask_a_zero(mb)
    _check_packings(mb)                     # the tags of the capture match the replayed buffers


def test_vqvae_whole_step_graph_tracks_the_eager_steps():
    import vqvae_b200
    from vqvae_b200.optim import Adam
    ma, mb, x = _vqvae(), _vqvae(), _images(32)
    with vqvae_b200.precision("fp32"):
        oa, ob = Adam(ma.parameters(), lr=3e-4, amsgrad=True), Adam(mb.parameters(), lr=3e-4, amsgrad=True)
        eager = np.array([_vq_step(ma, x, oa).item() for _ in range(11)])
        graph, loss = _capture(lambda: _vq_step(mb, x, ob))
        got = []
        for _ in range(10):
            graph.replay()
            got.append(loss.item())
        got = np.array(got)
    rel = np.abs(got - eager[1:]) / np.abs(eager[1:])
    a, b = _snapshot(ma, oa), _snapshot(mb, ob)
    worst = max(float((a[k] - b[k]).abs().max() / a[k].abs().max().clamp_min(1e-30)) for k in a)
    print(f"vqvae graph: loss {got[0]:.5f} -> {got[-1]:.5f}; worst relative to eager {rel.max():.2e}; "
          f"worst state |graph - eager| / max|eager| {worst:.2e}")
    assert rel.max() <= 1e-4
    assert float(ob.state[next(mb.parameters())]["step"]) == 11.0


def test_host_pipeline_built_before_the_steps_matches_an_eager_forward_after_them():
    import vqvae_b200
    from vqvae_b200.optim import Adam
    m, x = _vqvae(), _images(16)
    rng = np.random.default_rng(3)
    batches = [torch.from_numpy(rng.standard_normal((16, 3, 32, 32)).astype(np.float32)).pin_memory()
               for _ in range(4)]
    with vqvae_b200.precision("fp32"):
        m.eval()
        pipe = vqvae_b200.HostPipeline(m, (16, 3, 32, 32), depth=2)
        m.train()
        opt = Adam(m.parameters(), lr=1e-3, amsgrad=True)
        for _ in range(3):
            _vq_step(m, x, opt)
        m.eval()
        with torch.no_grad():
            want = [(float(l), xh.cpu().clone(), float(p)) for l, xh, p in (m(b.cuda()) for b in batches)]
        got = []
        pipe.run(batches, lambda r: got.append((float(r.loss), r.x_hat.clone(), float(r.perplexity))))
    assert len(got) == len(want)
    for (l0, xh0, p0), (l1, xh1, p1) in zip(want, got):
        assert l0 == l1 and p0 == p1 and torch.equal(xh0, xh1)

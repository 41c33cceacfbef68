"""GatedPixelCNN.cross_entropy_ex: cross_entropy with weight, ignore_index and label_smoothing, on the H100, in fp32
and TF32.

Per case (PRIOR_CASES, the backward entries of PRIOR_SHAPE_CASES, a three-chunk case and a K=8192 head), precision,
option set and reduction:
  values     against tests/prior_ce_options_ref.torch_ce (F.cross_entropy) in fp64 on forward's logits of the same
             precision: "mean" and "sum" within 1e-6 relative, "none" within 1e-5 * max(1, |loss_p|); grad mode and
             no-grad mode give the same bits
  gradients  against forward + F.cross_entropy(options) + backward on the GPU in the same precision (SAME), and for
             PRIOR_CASES with all three options against fp64 autograd of oracle/prior_train_port.py (_fp64_bar)
Then: neutral options give the bits of cross_entropy, the _ex entry points with a NULL options pointer give
the bits of today's entry points, the "mean" edge cases, determinism, a CUDA graph of cross_entropy + backward + Adam
whose replays read new weight values, launch counts, and the peak memory at B=16, 64x64, K=8192."""
import contextlib
import ctypes
import functools
import io
import math

import pytest
import torch

from oracle.prior_port import PRIOR_CASES, PRIOR_SHAPE_CASES, make_prior_inputs, make_prior_state_dict
from oracle.prior_train_port import leaf_params, prior_logits
from tests.prior_ce_options_ref import torch_ce
from tests.test_gpu_prior_ce import CE_CASES, CHUNK, SAME, _fp64_bar, _grads, _rel, _upstream

pytestmark = pytest.mark.gpu

A7, B3 = ["A", 7, False], ["B", 3, True]
OPT_CASES = dict(CE_CASES, ce_k8192=dict(K=8192, dim=32, n_layers=2, n_classes=3, size=8, batch=4, wseed=80, xseed=81,
                                         layers=[A7, B3]))
CASES = (list(PRIOR_CASES) + [n for n, c in PRIOR_SHAPE_CASES.items() if "backward" in c.get("parts", ["backward"])]
         + list(OPT_CASES))
REDUCTIONS = ("mean", "sum", "none")
OPTION_SETS = ("weight", "weight_zeros", "ignore", "ignore_out_of_range", "smooth_0.1", "smooth_1", "all")


def _case(name):
    return PRIOR_CASES.get(name) or PRIOR_SHAPE_CASES.get(name) or OPT_CASES[name]


def _model(name, precision):
    from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
    c = _case(name)
    layers = c.get("layers")
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], layers)
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
        for i, (mask, k, residual) in enumerate(layers or []):
            m.layers[i] = GatedMaskedConv2d(mask, c["dim"], k, residual, c["n_classes"])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    m.precision = precision
    codes, labels, _ = make_prior_inputs(c)
    return c, sd, m.cuda(), torch.from_numpy(codes), torch.from_numpy(labels)


def _options(kind, c, x, seed=5):
    """(codes, options) of an option set: the codes change only where positions are to be ignored"""
    K = c["K"]
    g = torch.Generator().manual_seed(seed)
    x = x.clone()
    opts = {}
    if kind in ("weight", "all"):
        opts["weight"] = torch.rand(K, generator=g) + 0.1
    if kind == "weight_zeros":
        w = torch.rand(K, generator=g) + 0.1
        w[torch.rand(K, generator=g) < 0.3] = 0.0
        w[x.reshape(-1)[0].clamp(0, K - 1)] = 1.0                   # some target keeps a positive weight
        opts["weight"] = w
    if kind in ("ignore", "ignore_out_of_range", "all"):
        # an in-range code that occurs (or, with one position or one code, -7), or one the model clamps
        v = -7 if kind == "ignore_out_of_range" or K == 1 or x.numel() < 2 else int(x.reshape(-1)[1])
        x[torch.rand(x.shape, generator=g) < 0.2] = v
        if x.shape[0] > 1:
            x[-1] = v                                                # one image ignored whole
        x.reshape(-1)[0] = 0 if v != 0 else min(1, K - 1)            # and one position scored
        opts["ignore_index"] = v
    if kind.startswith("smooth") or kind == "all":
        opts["label_smoothing"] = 1.0 if kind == "smooth_1" else 0.1
    return x, opts


def _ref_loss(logits, x, opts, reduction, dtype):
    K = logits.shape[1]
    w = opts.get("weight")
    loss = torch_ce(logits.permute(0, 2, 3, 1).reshape(-1, K).to(dtype), x.reshape(-1).to(logits.device),
                    None if w is None else w.to(dtype).to(logits.device), opts.get("ignore_index"),
                    opts.get("label_smoothing", 0.0), reduction)
    return loss.reshape(x.shape) if reduction == "none" else loss


def _backward(loss, c, reduction):
    if reduction == "none":
        loss.backward(_upstream(c).to(loss.dtype).to(loss.device))
    else:
        loss.backward()


def _gpu_opts(opts):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in opts.items()}


@functools.lru_cache(maxsize=None)
def _fp64(name, kind, reduction):
    c = _case(name)
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], c.get("layers"))
    codes, labels, _ = make_prior_inputs(c)
    x, opts = _options(kind, c, torch.from_numpy(codes))
    lab = torch.from_numpy(labels)
    with torch.enable_grad():
        g = leaf_params(sd, torch.float64)
        lg = prior_logits(g, x.clamp(0, c["K"] - 1), lab, c["n_layers"], c.get("layers"))   # the embedding clamps
        _backward(_ref_loss(lg, x, opts, reduction, torch.float64), c, reduction)
    return {k: v.grad for k, v in g.items()}


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("name", CASES)
def test_values_and_gradients(name, precision):
    c, _, m, x0, lab = _model(name, precision)
    lc = lab.cuda()
    report = []
    for kind in OPTION_SETS:
        x, opts = _options(kind, c, x0)
        xc, go = x.cuda(), _gpu_opts(_options(kind, c, x0)[1])
        with torch.no_grad():
            logits = m(xc, lc)
            inf = {r: m.cross_entropy_ex(xc, lc, reduction=r, **go) for r in REDUCTIONS}
        for r in REDUCTIONS:
            want = _ref_loss(logits, x, opts, r, torch.float64)
            got = inf[r].double()
            if r == "none":
                err = float(((got - want).abs() / want.abs().clamp_min(1.0)).max())
                assert err <= 1e-5, (kind, r, err)
            else:
                err = abs(float(got - want)) / max(abs(float(want)), 1e-30)
                assert err <= 1e-6, (kind, r, err)
            with torch.enable_grad():
                loss = m.cross_entropy_ex(xc, lc, reduction=r, **go)
                assert loss.requires_grad and torch.equal(loss.detach(), inf[r])
                _backward(loss, c, r)
                got_g = _grads(m)
                _backward(_ref_loss(m(xc, lc), x, go, r, torch.float32), c, r)
                ref_g = _grads(m)
            same = max(_rel(got_g[k], ref_g[k]) for k in ref_g)
            assert same <= SAME[precision], (kind, r, same)
            line = f"{kind} {r}: value {err:.1e}, vs forward+CE {same:.1e}"
            if name in PRIOR_CASES and kind == "all":
                want_g = _fp64(name, kind, r)
                w64 = max(_rel(got_g[k], want_g[k]) for k in want_g)
                assert w64 <= _fp64_bar(name, precision), (kind, r, w64)
                line += f", vs fp64 {w64:.1e}"
            report.append(line)
    print(f"{name} {precision}:\n  " + "\n  ".join(report))


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_neutral_options_and_null_options_pointer_are_the_call_without_options(precision):
    from vqvae_b200 import _lib, ops
    from vqvae_b200.prior import _grad_table
    for name in ("prior_default", "ce_chunks"):
        c, _, m, x, lab = _model(name, precision)
        xc, lc = x.cuda(), lab.cuda()
        neutral = dict(weight=torch.ones(c["K"], device="cuda"), ignore_index=-12345, label_smoothing=0.0)
        for r in REDUCTIONS:
            with torch.enable_grad():
                a = m.cross_entropy(xc, lc, reduction=r)
                _backward(a, c, r)
                ga = _grads(m)
                b = m.cross_entropy_ex(xc, lc, reduction=r, **neutral)
                _backward(b, c, r)
                gb = _grads(m)
            assert torch.equal(a, b) and all(torch.equal(ga[k], gb[k]) for k in ga), (name, r)
            with torch.no_grad():
                assert torch.equal(m.cross_entropy_ex(xc, lc, reduction=r, **neutral), a.detach())
            # every option at its default: cross_entropy itself, the same launches and bits
            with torch.enable_grad():
                n0 = ops.launch_count()
                d = m.cross_entropy_ex(xc, lc, reduction=r)
                assert ops.launch_count() - n0 == (3 + 2 * c["n_layers"] if precision == "fp32" else
                                                   4 + 4 * c["n_layers"]) + (r != "none")
                _backward(d, c, r)
                gd = _grads(m)
            assert torch.equal(a, d) and all(torch.equal(ga[k], gd[k]) for k in ga), (name, r)

        # the _ex entry points with NULL options against today's, through ctypes
        keep = []
        net = m._net(keep)
        sfx = "tf32" if precision == "tf32" else "f32"
        lib = _lib.lib()
        B, H, W = x.shape
        for r in REDUCTIONS:
            loss, saved = ops.prior_ce_forward(net, xc, lc, r, precision, train=True)
            ri = ops.PRIOR_CE_REDUCTIONS.index(r)
            loss2, saved2 = torch.empty_like(loss), torch.empty_like(saved)
            ws = torch.empty(getattr(lib, "vqb_prior_ce_workspace_bytes" + ("_tf32" if sfx == "tf32" else ""))(
                B, H, W, net.dim, net.n_layers, net.input_dim, 1), dtype=torch.uint8, device="cuda")
            _lib.check(getattr(lib, "vqb_prior_ce_forward_ex_" + sfx)(
                ctypes.byref(net), xc.data_ptr(), lc.data_ptr(), B, H, W, ri, None, loss2.data_ptr(),
                saved2.data_ptr(), saved2.numel(), ws.data_ptr(), ws.numel(), ops._stream()), "forward_ex")
            assert torch.equal(loss, loss2) and torch.equal(saved, saved2)
            d = (_upstream(c).float() if r == "none" else torch.ones(())).cuda()
            out = []
            for ex in (False, True):
                grads, table, _layers = _grad_table(m, xc.device)
                if ex:
                    bws = torch.empty(lib.vqb_prior_ce_backward_workspace_bytes(ctypes.byref(net), B, H, W),
                                      dtype=torch.uint8, device="cuda")
                    _lib.check(getattr(lib, "vqb_prior_ce_backward_ex_" + sfx)(
                        ctypes.byref(net), xc.data_ptr(), lc.data_ptr(), B, H, W, ri, None, d.data_ptr(),
                        saved.data_ptr(), ctypes.byref(table), bws.data_ptr(), bws.numel(), ops._stream()),
                        "backward_ex")
                else:
                    ops.prior_ce_backward(net, xc, lc, r, d, saved, table, precision)
                out.append([t.clone() for t in grads.finish()])
            assert all(torch.equal(u, v) for u, v in zip(*out)), (name, r)


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_mean_edge_cases(precision):
    c, _, m, x, lab = _model("prior_ragged", precision)
    lc = lab.cuda()
    K = c["K"]
    # every position ignored: NaN, zero gradients ("sum": 0)
    v = int(x.reshape(-1)[0])
    xa = torch.full_like(x, v).cuda()
    for e in (0.0, 0.2):
        with torch.enable_grad():
            loss = m.cross_entropy_ex(xa, lc, ignore_index=v, label_smoothing=e)
            loss.backward()
        g = _grads(m)
        assert math.isnan(float(loss)) and all(torch.equal(t, torch.zeros_like(t)) for t in g.values())
        assert float(m.cross_entropy_ex(xa, lc, reduction="sum", ignore_index=v, label_smoothing=e)) == 0.0
    # scored targets of weight 0: NaN, non-finite gradients
    w = torch.ones(K)
    w[x.reshape(-1).clamp(0, K - 1)] = 0.0
    for e in (0.0, 0.2):
        with torch.enable_grad():
            loss = m.cross_entropy_ex(x.cuda(), lc, weight=w.cuda(), label_smoothing=e)
            loss.backward()
        g = _grads(m)
        assert math.isnan(float(loss)) and not all(bool(torch.isfinite(t).all()) for t in g.values())


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_deterministic_launch_counts_and_graph_replay_with_new_weights(precision):
    from vqvae_b200 import ops
    from vqvae_b200.optim import Adam
    for name in ("prior_default", "ce_chunks"):
        c, _, m, x0, lab = _model(name, precision)
        x, opts = _options("all", c, x0)
        xc, lc, go = x.cuda(), lab.cuda(), _gpu_opts(opts)
        L, npos = c["n_layers"], c["batch"] * c["size"] ** 2
        fwd = (3 + 2 * L) if precision == "fp32" else (4 + 4 * L)
        with torch.no_grad():
            m.cross_entropy_ex(xc, lc, **go)
        runs = []
        for r in ("mean", "none"):
            with torch.no_grad():
                n0 = ops.launch_count()
                m.cross_entropy_ex(xc, lc, reduction=r, **go)
                assert ops.launch_count() - n0 == fwd + (r != "none")
            for _ in range(2):
                with torch.enable_grad():
                    n0 = ops.launch_count()
                    loss = m.cross_entropy_ex(xc, lc, reduction=r, **go)
                    assert ops.launch_count() - n0 == fwd + (r != "none")
                    n0 = ops.launch_count()
                    _backward(loss, c, r)
                    assert ops.launch_count() - n0 == 5 + 10 * L + 3 * -(-npos // CHUNK)
                runs.append((loss.detach().clone(), _grads(m)))
        for a, b in ((runs[0], runs[1]), (runs[2], runs[3])):
            assert torch.equal(a[0], b[0]) and all(torch.equal(a[1][k], b[1][k]) for k in a[1])

    # cross_entropy_ex + backward + Adam.step() in one CUDA graph; new weight values before the second replay
    def steps(graph):
        c, _, m, x0, lab = _model("prior_ragged", precision)
        x, opts = _options("all", c, x0)
        xc, lc, go = x.cuda(), lab.cuda(), _gpu_opts(opts)
        w_new = (torch.rand(c["K"], generator=torch.Generator().manual_seed(3)) + 0.5).cuda()
        opt = Adam(m.parameters(), lr=3e-4)

        def step():
            opt.zero_grad(set_to_none=True)
            with torch.enable_grad():
                m.cross_entropy_ex(xc, lc, **go).backward()
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
        for i in range(3):
            if i == 1:
                go["weight"].copy_(w_new)
            g.replay() if graph else step()
        torch.cuda.synchronize()
        return {k: p.detach().clone() for k, p in m.named_parameters()}
    eager, replayed = steps(False), steps(True)
    assert all(torch.equal(eager[k], replayed[k]) for k in eager)


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_memory_at_b16_64x64_k8192(precision):
    from pixelcnn.models import GatedPixelCNN
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(8192, 64, 2, 10).cuda()
    m.precision = precision
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randint(0, 8192, (16, 64, 64), device="cuda", generator=gen)
    lab = torch.randint(0, 10, (16,), device="cuda", generator=gen)
    w = torch.rand(8192, device="cuda", generator=gen) + 0.1
    peaks = {}
    for arm in ("plain", "options"):
        for p in m.parameters():
            p.grad = torch.zeros_like(p)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        with torch.enable_grad():
            kw = dict(weight=w, ignore_index=int(x[0, 0, 0]), label_smoothing=0.1)
            loss = m.cross_entropy_ex(x, lab, **kw) if arm == "options" else m.cross_entropy(x, lab)
            loss.backward()
        del loss
        torch.cuda.synchronize()
        peaks[arm] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    print(f"{precision}: peak above the call, cross_entropy + backward {peaks['plain']:.4f} GiB, with options "
          f"{peaks['options']:.4f} GiB")
    assert peaks["options"] <= 1.02 * peaks["plain"]

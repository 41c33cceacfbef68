"""GatedPixelCNN.cross_entropy on the H100, in fp32 and TF32: the loss without the B*K*H*W logits, and its gradients.

Per case of PRIOR_CASES, of PRIOR_SHAPE_CASES with a backward part and of CE_CASES below, in both precisions:
  values     reduction="none" is bitwise -log_prob(per_position=True); "mean" is within 1e-6 relative of torch's
             F.cross_entropy on forward's logits; grad mode and no-grad mode give the same bits
  saved      the buffer the training call keeps starts with bitwise what vqb_prior_forward_train_* keeps
  gradients  for "mean", "sum" and "none" (a seeded random upstream map), against forward + F.cross_entropy on the
             GPU in the same precision, and against fp64 autograd of oracle/prior_train_port.py at the bars the
             existing tests apply to forward + cross-entropy
  head       output_conv.2's gradients against an fp64 product of forward's own logits and the saved hidden layer
Then determinism, launch counts, CUDA-graph replay of cross_entropy + backward + Adam.step(), the errors, the
reference's Adam loop against fp64, and the memory the call saves at B=16, 64x64, K=8192."""
import contextlib
import functools
import io

import pytest
import torch
import torch.nn.functional as F

from oracle.prior_port import PRIOR_CASES, PRIOR_SHAPE_CASES, make_prior_inputs, make_prior_state_dict
from oracle.prior_train_port import leaf_params, prior_logits
from tests.prior_tf32_port import saved_offsets, tf32_round

pytestmark = pytest.mark.gpu

A7, B3 = ["A", 7, False], ["B", 3, True]
# 9600 positions: three chunks of the head's backward (4096 positions each), the last one ragged (1408)
CE_CASES = {
    "ce_chunks": dict(K=37, dim=32, n_layers=3, n_classes=3, size=40, batch=6, wseed=70, xseed=71,
                      layers=[A7, B3, B3]),
}
CASES = (list(PRIOR_CASES) + [n for n, c in PRIOR_SHAPE_CASES.items() if "backward" in c.get("parts", ["backward"])]
         + list(CE_CASES))
REDUCTIONS = ("mean", "sum", "none")
CHUNK = 4096

# Against forward + F.cross_entropy on the GPU, relative to each tensor's max |g|
SAME = {"fp32": 1e-5, "tf32": 5e-3}
# fp32 ulps between the GPU's d_logits (expf, logf in fp32) and the fp64 softmax the head check restates
DL_ULPS = 8


def _fp64_bar(name, precision):
    """The bars of tests/test_gpu_prior_train.py and test_gpu_prior_shapes.py (fp32), test_gpu_prior_tf32.py (TF32)"""
    if precision == "tf32":
        return 2.5e-1
    return 1e-4 if name in ("prior_cfg3", "wide", "deep") else 2e-5


def _case(name):
    return PRIOR_CASES.get(name) or PRIOR_SHAPE_CASES.get(name) or CE_CASES[name]


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


def _upstream(c, seed=9):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((c["batch"], c["size"], c["size"]), generator=g, dtype=torch.float64)


def _loss_of_logits(lg, x, reduction):
    K = lg.shape[1]
    loss = F.cross_entropy(lg.permute(0, 2, 3, 1).reshape(-1, K), x.reshape(-1), reduction=reduction)
    return loss.reshape(x.shape) if reduction == "none" else loss


def _backward(loss, c, reduction):
    if reduction == "none":
        loss.backward(_upstream(c).to(loss.dtype).to(loss.device))
    else:
        loss.backward()


def _grads(m):
    out = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    return out


def _rel(got, want):
    return float((got.double().cpu() - want.double().cpu()).abs().max() / want.double().abs().max().clamp_min(1e-30))


@functools.lru_cache(maxsize=None)
def _fp64(name, reduction):
    c = _case(name)
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], c.get("layers"))
    codes, labels, _ = make_prior_inputs(c)
    x, lab = torch.from_numpy(codes), torch.from_numpy(labels)
    with torch.enable_grad():
        g = leaf_params(sd, torch.float64)
        _backward(_loss_of_logits(prior_logits(g, x, lab, c["n_layers"], c.get("layers")), x, reduction), c,
                  reduction)
    return {k: v.grad for k, v in g.items()}


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("name", CASES)
def test_values_saved_and_gradients(name, precision, monkeypatch):
    from vqvae_b200 import ops
    c, sd, m, x, lab = _model(name, precision)
    xc, lc = x.cuda(), lab.cuda()
    B, S, K = c["batch"], c["size"], c["K"]

    # values: bitwise -log_prob per position; grad and no-grad modes agree bitwise
    with torch.no_grad():
        pos = m.log_prob(xc, lc, per_position=True)
        inf = {r: m.cross_entropy(xc, lc, reduction=r) for r in REDUCTIONS}
        logits = m(xc, lc)
    assert inf["none"].shape == (B, S, S) and inf["mean"].shape == () and not inf["mean"].requires_grad
    assert torch.equal(inf["none"], -pos)
    want_mean = F.cross_entropy(logits.permute(0, 2, 3, 1).reshape(-1, K), xc.reshape(-1)).double()
    err_mean = abs(float(inf["mean"].double() - want_mean)) / max(abs(float(want_mean)), 1e-30)   # K = 1: 0
    assert err_mean <= 1e-6, err_mean
    want_sum = F.cross_entropy(logits.permute(0, 2, 3, 1).reshape(-1, K).double(), xc.reshape(-1), reduction="sum")
    assert abs(float(inf["sum"].double() - want_sum)) <= 1e-6 * abs(float(want_sum))

    kept = {}
    forward_train, ce_forward = ops.prior_forward_train, ops.prior_ce_forward

    def keep_train(net, codes, labels, precision="fp32"):
        out, saved = forward_train(net, codes, labels, precision)
        kept["train"] = saved
        return out, saved

    def keep_ce(net, codes, labels, reduction, precision="fp32", train=False):
        out, saved = ce_forward(net, codes, labels, reduction, precision, train)
        kept["ce"] = saved
        return out, saved

    monkeypatch.setattr(ops, "prior_forward_train", keep_train)
    monkeypatch.setattr(ops, "prior_ce_forward", keep_ce)
    worst_same, worst64 = {}, {}
    for r in REDUCTIONS:
        with torch.enable_grad():
            loss = m.cross_entropy(xc, lc, reduction=r)
            assert loss.requires_grad and torch.equal(loss.detach(), inf[r])
            _backward(loss, c, r)
            got = _grads(m)
            out = m(xc, lc)
            assert torch.equal(out.detach(), logits)
            _backward(_loss_of_logits(out, xc, r), c, r)
            ref = _grads(m)
        worst_same[r] = max(_rel(got[k], ref[k]) for k in ref)
        if precision == "fp32" or name in PRIOR_CASES:
            want = _fp64(name, r)
            worst64[r] = max(_rel(got[k], want[k]) for k in want)
        if r == "none":
            head = got
    print(f"{name} {precision}: mean {err_mean:.2e}; vs forward+CE {worst_same}; vs fp64 {worst64}")
    assert max(worst_same.values()) <= SAME[precision]
    assert all(v <= _fp64_bar(name, precision) for v in worst64.values())

    # the saved activations: bitwise the training forward's, then (M, logf(S)) per position
    n = kept["train"].numel()
    assert kept["ce"].numel() == n + 8 * B * S * S
    assert torch.equal(kept["ce"][:n], kept["train"])

    # output_conv.2's gradient at forward's own logits and the saved hidden layer (reduction "none")
    off, _ = saved_offsets(B, S, S, c["dim"], c["n_layers"])
    o, ch = off["hid"]
    hid = kept["train"].view(torch.float32)[o:o + B * S * S * ch].reshape(-1, ch).double().cpu()
    l64 = logits.permute(0, 2, 3, 1).reshape(-1, K).double().cpu()
    p = torch.softmax(l64, dim=1)
    p[torch.arange(p.shape[0]), x.reshape(-1)] -= 1
    dl = p * _upstream(c).reshape(-1, 1)
    ones = torch.ones((hid.shape[0], 1), dtype=torch.float64)
    slack = 0
    if precision == "tf32":
        # Both operands are staged as TF32 (tc_gemm.cuh).  hid is the GPU's own; d_logits is the GPU's fp32
        # arithmetic, a few ulps from this fp64 value, so where it lies within DL_ULPS of a TF32 rounding midpoint
        # either neighbour is right, and that term may move by the rounding step (as _gate_slack in
        # tests/test_gpu_prior_tf32_saved.py).
        d = dl.abs() * DL_ULPS * 2.0 ** -23
        step = (tf32_round(dl + d) - tf32_round(dl - d)).abs()
        dl, hid = tf32_round(dl), tf32_round(hid)
        slack = step.t() @ torch.cat([hid, ones], 1).abs()
    hid1 = torch.cat([hid, ones], 1)
    want = dl.t() @ hid1
    terms = dl.abs().t() @ hid1.abs()
    got = torch.cat([head["output_conv.2.weight"].reshape(K, -1), head["output_conv.2.bias"].reshape(K, 1)], 1)
    bar = terms.max().clamp_min(1e-30)
    err = float(((got.double().cpu() - want).abs() - slack).max() / bar)
    raw = float((got.double().cpu() - want).abs().max() / bar)
    print(f"{name} {precision}: output_conv.2 at the GPU's logits {err:.2e} of the largest sum of |terms| "
          f"({raw:.2e} without the rounding slack)")
    assert err <= 1e-5


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_deterministic_launch_counts_and_graph_replay_with_adam(precision):
    from vqvae_b200 import ops
    from vqvae_b200.optim import Adam
    for name in ("prior_default", "ce_chunks"):
        c, _, m, x, lab = _model(name, precision)
        xc, lc = x.cuda(), lab.cuda()
        L, npos = c["n_layers"], c["batch"] * c["size"] ** 2
        fwd = (3 + 2 * L) if precision == "fp32" else (4 + 4 * L)
        with torch.no_grad():
            m.cross_entropy(xc, lc)                     # packs the weights once (P3): not part of the counts
        runs = []
        for r in ("mean", "none"):
            with torch.no_grad():
                n0 = ops.launch_count()
                m.cross_entropy(xc, lc, reduction=r)
                assert ops.launch_count() - n0 == fwd + (r != "none")
            for _ in range(2):
                with torch.enable_grad():
                    n0 = ops.launch_count()
                    loss = m.cross_entropy(xc, lc, reduction=r)
                    assert ops.launch_count() - n0 == fwd + (r != "none")
                    n0 = ops.launch_count()
                    _backward(loss, c, r)
                    assert ops.launch_count() - n0 == 5 + 10 * L + 3 * -(-npos // CHUNK)
                    with pytest.raises(RuntimeError, match="twice"):
                        _backward(loss, c, r)
                runs.append(_grads(m))
        assert all(torch.equal(runs[0][k], runs[1][k]) and torch.equal(runs[2][k], runs[3][k]) for k in runs[0])

    # cross_entropy + backward + Adam.step() in one CUDA graph: three replays are three eager steps, bitwise
    def steps(graph):
        c, _, m, x, lab = _model("prior_ragged", precision)
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
            step()                                      # warm-up: Adam's state and the gradients exist
            if graph:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    step()
        torch.cuda.current_stream().wait_stream(s)
        for _ in range(3):
            g.replay() if graph else step()
        torch.cuda.synchronize()
        return {k: p.detach().clone() for k, p in m.named_parameters()}
    eager, replayed = steps(False), steps(True)
    assert all(torch.equal(eager[k], replayed[k]) for k in eager)


def test_errors():
    c, _, m, x, lab = _model("prior_ragged", "fp32")
    with pytest.raises(RuntimeError, match="CUDA"):
        m.cross_entropy(x, lab)
    with pytest.raises(ValueError, match="reduction"):
        m.cross_entropy(x.cuda(), lab.cuda(), reduction="batchmean")


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_reference_adam_loop_tracks_fp64(precision):
    c, sd, m, x, lab = _model("prior_ragged", precision)
    g = leaf_params(sd, torch.float64)
    opt64 = torch.optim.Adam(list(g.values()), lr=3e-4)
    opt = torch.optim.Adam(m.parameters(), lr=3e-4)
    xc, lc = x.cuda(), lab.cuda()
    got, want = [], []
    with torch.enable_grad():
        for _ in range(100):
            loss = _loss_of_logits(prior_logits(g, x, lab, c["n_layers"]), x, "mean")
            opt64.zero_grad()
            loss.backward()
            opt64.step()
            want.append(loss.item())
            loss = m.cross_entropy(xc, lc)
            opt.zero_grad()
            loss.backward()
            opt.step()
            got.append(loss.item())
    rel = max(abs(a - b) / abs(b) for a, b in zip(got, want))
    print(f"adam {precision}: loss {got[0]:.5f} -> {got[99]:.5f} @99 (fp64 {want[99]:.5f}); worst relative {rel:.2e}")
    assert rel <= (1e-3 if precision == "fp32" else 5e-3)


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_memory_at_b16_64x64_k8192(precision):
    from pixelcnn.models import GatedPixelCNN
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(8192, 64, 2, 10).cuda()
    m.precision = precision
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randint(0, 8192, (16, 64, 64), device="cuda", generator=gen)
    lab = torch.randint(0, 10, (16,), device="cuda", generator=gen)
    peaks = {}
    for arm in ("cross_entropy", "forward"):
        for p in m.parameters():
            p.grad = torch.zeros_like(p)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        with torch.enable_grad():
            loss = m.cross_entropy(x, lab) if arm == "cross_entropy" else _loss_of_logits(m(x, lab), x, "mean")
            loss.backward()
        del loss
        torch.cuda.synchronize()
        peaks[arm] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    print(f"{precision}: peak above the call, cross_entropy + backward {peaks['cross_entropy']:.3f} GiB, "
          f"forward + CE + backward {peaks['forward']:.3f} GiB")
    assert peaks["cross_entropy"] < 1.0

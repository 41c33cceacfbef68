"""GatedPixelCNN.log_prob on the H100, in fp32 and TF32: every position's term against fp64 log_softmax of that
precision's own forward logits (which only holds if the kernel reduces exactly those logits), TF32 against the
emulated restatement, the compensated sums over n_given, the reference's validation loss, the sampler's log_prob,
clamping, determinism and CUDA-graph replay, the documented launch counts, no autograd, and peak memory against the
B*K*H*W logits it does not write."""
import contextlib
import io

import numpy as np
import pytest
import torch

from oracle.prior_port import PRIOR_CASES, PRIOR_SHAPE_CASES, make_prior_inputs, make_prior_state_dict
from oracle.prior_train_port import leaf_params
from tests import prior_log_prob_ref as ref
from tests.prior_tf32_port import prior_logits_tf32

pytestmark = pytest.mark.gpu

CASES = ["prior_ragged", "prior_default", "prior_cfg3"] + list(PRIOR_SHAPE_CASES)
PRECISIONS = ["fp32", "tf32"]
TERM, SUM = 1e-5, 1e-5          # per position: relative to max(1, |lp|); sums: relative
EMULATED = 4e-3                 # TF32 terms against the emulated logits, relative to their max |l|


def _case(name):
    return PRIOR_CASES.get(name) or PRIOR_SHAPE_CASES[name]


def _model(name, precision="fp32"):
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
    return c, sd, m.cuda().eval(), torch.from_numpy(codes).cuda(), torch.from_numpy(labels).cuda()


def _n_givens(S):
    HW = S * S
    return sorted({0, min(1, HW), S - 1, S, HW // 2, HW - 1, HW})


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", CASES)
def test_terms_sums_and_the_reference_loss(name, precision):
    c, sd, m, x, lab = _model(name, precision)
    B, S, K = c["batch"], c["size"], c["K"]
    with torch.no_grad():
        logits = m(x, lab)
        pos = m.log_prob(x, lab, per_position=True)
        total = m.log_prob(x, lab)
    assert pos.shape == (B, S, S) and pos.dtype == torch.float32 and total.shape == (B,)
    want = ref.position_terms(logits.cpu().numpy(), x.cpu().numpy())
    got = pos.double().cpu().numpy()
    err = np.abs(got - want) / np.maximum(1.0, np.abs(want))
    print(f"{name} {precision}: per-position max error {err.max():.2e} (relative to max(1, |lp|))")
    assert err.max() <= TERM
    # sums over p >= n_given against the fp64 sum of the kernel's own terms
    flat = got.reshape(B, -1)
    for n in _n_givens(S):
        with torch.no_grad():
            lp = m.log_prob(x, lab, n_given=n).double().cpu().numpy()
        exact = flat[:, n:].sum(-1)
        assert (np.abs(lp - exact) <= SUM * np.abs(exact)).all(), (n, lp, exact)
    np.testing.assert_allclose(total.double().cpu().numpy(), flat.sum(-1), rtol=SUM, atol=0)
    # the reference's test() loop: CrossEntropyLoss on forward's logits, permuted and made contiguous
    with torch.no_grad():
        lg = logits.permute(0, 2, 3, 1).contiguous()
        ce = torch.nn.CrossEntropyLoss()(lg.view(-1, K), x.view(-1)).item()
    ours = -total.double().sum().item() / (B * S * S)
    print(f"{name} {precision}: loss {ours:.7f}, reference loop {ce:.7f}")
    assert abs(ours - ce) <= SUM * abs(ce) + 1e-7


@pytest.mark.parametrize("name", CASES)
def test_tf32_terms_follow_the_emulated_logits(name):
    c, sd, m, x, lab = _model(name, "tf32")
    with torch.no_grad():
        pos = m.log_prob(x, lab, per_position=True)
    lg = prior_logits_tf32(leaf_params(sd, torch.float64), x.cpu(), lab.cpu(), c["n_layers"], c.get("layers"))
    lg = lg.detach().numpy()
    want = ref.position_terms(lg, x.cpu().numpy())
    err = np.abs(pos.double().cpu().numpy() - want).max() / max(np.abs(lg).max(), 1e-30)
    print(f"{name}: TF32 terms against the emulated logits {err:.2e} of max |l|")
    assert err <= EMULATED


@pytest.mark.parametrize("name", ["prior_ragged", "prior_default", "long", "wide"])
def test_the_samplers_log_prob(name):
    c, _, m, _, _ = _model(name)
    B, S, K = c["batch"], c["size"], c["K"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    torch.manual_seed(c["xseed"] + 77)
    with torch.no_grad():
        codes, lp = m.sample(labels, shape=(S, S), batch_size=B)
        got = m.log_prob(codes, labels)
        assert torch.allclose(got.double(), lp.double(), rtol=SUM, atol=0), (got, lp)
        x = torch.randint(0, K, (B, S, S), device="cuda")
        for n in sorted({1, S, S * S // 2 + 1}):
            codes, lp = m.sample_completion(x, labels, n, temperature=0.8, top_k=min(K, 20))
            got = m.log_prob(codes, labels, n_given=n)
            assert torch.allclose(got.double(), lp.double(), rtol=SUM, atol=0), (n, got, lp)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_out_of_range_codes_are_scored_as_the_clamped_code(precision):
    c, _, m, x, lab = _model("prior_ragged", precision)
    K = c["K"]
    bad = x.clone()
    bad[0, 0, 0], bad[0, 1, 2], bad[1, 3, 3], bad[2, 4, 4] = -1, K, -(2 ** 40), 2 ** 50
    with torch.no_grad():
        a = m.log_prob(bad, lab, per_position=True)
        b = m.log_prob(bad.clamp(0, K - 1), lab, per_position=True)
        assert torch.equal(a, b)
        assert torch.equal(m.log_prob(bad, lab, n_given=3), m.log_prob(bad.clamp(0, K - 1), lab, n_given=3))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_determinism_graph_replay_and_launch_counts(precision):
    from vqvae_b200 import ops
    for name in ("prior_default", "kernels"):
        c, _, m, x, lab = _model(name, precision)
        L, S = c["n_layers"], c["size"]
        with torch.no_grad():
            a = m._log_prob(x, lab, 5, False)
            b = m._log_prob(x, lab, 5, False)
            assert torch.equal(a, b)
            for n, per in ((0, False), (5, False), (0, True)):
                n0 = ops.launch_count()
                m._log_prob(x, lab, n, per)
                assert ops.launch_count() - n0 == (3 + 2 * L if precision == "fp32" else 4 + 4 * L), (name, n)
            n0 = ops.launch_count()
            z = m.log_prob(x, lab, n_given=S * S)
            assert ops.launch_count() == n0 and torch.equal(z, torch.zeros_like(z))
            for per in (False, True):
                first = m._log_prob(x, lab, 0 if per else 5, per)
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    out = m._log_prob(x, lab, 0 if per else 5, per)
                x.copy_(torch.randint_like(x, 0, c["K"]))
                g.replay()
                torch.cuda.synchronize()
                eager = m._log_prob(x, lab, 0 if per else 5, per)
                assert torch.equal(out, eager), (name, per)
                assert not torch.equal(out, first)


def _ws(m, B, S, precision):
    from vqvae_b200 import ops
    q = ops.lib().vqb_prior_log_prob_workspace_bytes_tf32 if precision == "tf32" else \
        ops.lib().vqb_prior_log_prob_workspace_bytes
    return q(B, S, S, m.dim, len(m.layers), m.embedding.num_embeddings)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_no_autograd_and_the_inference_workspace_only(precision):
    from vqvae_b200 import ops
    c, _, m, x, lab = _model("prior_default", precision)
    B, S = c["batch"], c["size"]
    assert all(p.requires_grad for p in m.parameters())
    with torch.enable_grad():
        with torch.no_grad():
            m.log_prob(x, lab)                                  # packs the weights
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = m.log_prob(x, lab)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - before
    assert out.grad_fn is None and not out.requires_grad
    saved = ops.lib().vqb_prior_train_saved_bytes(B, S, S, m.dim, len(m.layers))
    ws = _ws(m, B, S, precision)
    print(f"{precision}: peak {peak} B, workspace {ws} B, training activations {saved} B")
    assert peak <= ws + 4 * B + (1 << 20)
    assert peak < saved // 2


@pytest.mark.parametrize("precision", PRECISIONS)
def test_memory_at_k8192_on_64x64(precision):
    from pixelcnn.models import GatedPixelCNN
    B, S, K = 16, 64, 8192
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(K, 64, 2, 10).cuda().eval()
    m.precision = precision
    x = torch.randint(0, K, (B, S, S), device="cuda")
    lab = torch.arange(B, device="cuda") % 10
    logits_bytes = B * K * S * S * 4
    with torch.no_grad():
        m.log_prob(x, lab)
        torch.cuda.synchronize()
        for per in (False, True):
            before = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            out = m.log_prob(x, lab, per_position=per)
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - before
            ws = _ws(m, B, S, precision)
            print(f"{precision} per_position={per}: peak {peak / 2**20:.1f} MiB, workspace {ws / 2**20:.1f} MiB, "
                  f"logits {logits_bytes / 2**20:.1f} MiB")
            assert peak <= ws + out.numel() * 4 + (1 << 20)
            assert peak < logits_bytes // 4
            assert bool(torch.isfinite(out).all()) and bool((out <= 0).all())

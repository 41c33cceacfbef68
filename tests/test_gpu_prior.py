"""The Gated PixelCNN prior on the H100: teacher-forced logits against the reference's goldens, the sampler's exactness
against the forward and against the fp64 restatement, its distribution, clamping, launch count and graph capture."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.prior_port import PRIOR_CASES, make_prior_inputs, make_prior_state_dict, prior_forward

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model(name):
    from pixelcnn.models import GatedPixelCNN
    c = PRIOR_CASES[name]
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"])
    m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    return c, sd, m.cuda().eval()


def _golden(name):
    with np.load(os.path.join(ROOT, "tests", "golden", name + ".npz")) as d:
        return {k: d[k] for k in d.files}


@pytest.mark.parametrize("name", list(PRIOR_CASES))
def test_forward_matches_reference_and_zeroes_mask_a(name):
    c, sd, m = _model(name)
    l0 = m.layers[0]
    assert l0.vert_stack.weight[:, :, -1].abs().sum() > 0 and l0.horiz_stack.weight[:, :, :, -1].abs().sum() > 0
    codes, labels, pos = make_prior_inputs(c)
    logits = m(torch.from_numpy(codes).cuda(), torch.from_numpy(labels).cuda())
    torch.cuda.synchronize()
    assert logits.shape == (c["batch"], c["K"], c["size"], c["size"]) and logits.dtype == torch.float32
    assert not logits.requires_grad
    g = _golden(name)
    got = logits.cpu().numpy()
    if pos is not None:
        got, want = got[:, :, pos[:, 0], pos[:, 1]], g["logits_at"]
    else:
        want = g["logits"]
    np.testing.assert_allclose(got, want, atol=1e-4, rtol=0)
    # P3: the masked taps of layer 0 are zero in the caller's parameters, and stay so without further repacks
    assert l0.vert_stack.weight[:, :, -1].abs().sum() == 0 and l0.horiz_stack.weight[:, :, :, -1].abs().sum() == 0
    v = l0.vert_stack.weight._version
    m(torch.from_numpy(codes).cuda(), torch.from_numpy(labels).cuda())
    assert l0.vert_stack.weight._version == v


@pytest.mark.parametrize("name", ["prior_default", "prior_ragged"])
def test_generate_step_logits_equal_forward_bitwise(name):
    c, _, m = _model(name)
    B, S, K = c["batch"], c["size"], c["K"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    torch.manual_seed(5)
    u = torch.rand((B, S, S), device="cuda")
    step = torch.full((B, S, S, K), float("nan"), device="cuda")
    codes = m._sample(labels, u, step)
    assert codes.dtype == torch.int64 and codes.shape == (B, S, S)
    assert int(codes.min()) >= 0 and int(codes.max()) < K
    fwd = m(codes, labels).permute(0, 2, 3, 1)
    assert torch.equal(step, fwd)
    assert torch.equal(m._sample(labels, u), codes)                   # step_logits changes nothing


@pytest.mark.parametrize("name", ["prior_default", "prior_ragged"])
def test_generate_inverts_the_fp64_cdf(name):
    c, sd, m = _model(name)
    B, S = 8, c["size"]
    labels = torch.arange(B, device="cuda") % c["n_classes"]
    torch.manual_seed(11)
    codes = m.generate(labels, shape=(S, S), batch_size=B)
    torch.manual_seed(11)
    u = torch.rand((B, S, S), device="cuda").double().cpu()
    assert codes.device.type == "cuda"
    lg = prior_forward(sd, codes.cpu(), labels.cpu(), c["n_layers"], dtype=torch.float64)
    cdf = torch.cumsum(torch.softmax(lg, 1), 1)                       # (B, K, S, S)
    k = codes.cpu()[:, None]
    hi = cdf.gather(1, k)[:, 0]
    lo = torch.where(k[:, 0] > 0, cdf.gather(1, (k - 1).clamp(min=0))[:, 0], torch.zeros_like(hi))
    ok = (lo <= u) & (u < hi)
    near = torch.minimum((u - lo).abs(), (u - hi).abs()) < 1e-5
    assert bool((ok | near).all())
    print(f"{name}: {int((~ok).sum())} of {ok.numel()} draws within 1e-5 of a CDF boundary")


def test_generate_distribution_chi_square():
    from scipy import stats
    c, sd, m = _model("prior_ragged")
    N = 65536
    for lab in range(c["n_classes"]):
        labels = torch.full((N,), lab, dtype=torch.int64, device="cuda")
        torch.manual_seed(100 + lab)
        codes = m.generate(labels, shape=(1, 1), batch_size=N)
        counts = np.bincount(codes.cpu().numpy().ravel(), minlength=c["K"]).astype(np.float64)
        lg = prior_forward(sd, np.zeros((1, 1, 1), np.int64), np.array([lab]), c["n_layers"], dtype=torch.float64)
        p = torch.softmax(lg[0, :, 0, 0], 0).numpy()
        exp = p * N
        big = exp >= 5
        f_obs = np.append(counts[big], counts[~big].sum())
        f_exp = np.append(exp[big], exp[~big].sum())
        if f_exp[-1] == 0:
            f_obs, f_exp = f_obs[:-1], f_exp[:-1]
        assert counts[~big].sum() <= max(50.0, 10 * exp[~big].sum())
        pval = stats.chisquare(f_obs, f_exp * f_obs.sum() / f_exp.sum()).pvalue
        print(f"label {lab}: chi-square p = {pval:.4f}")
        assert pval > 1e-3


def test_out_of_range_codes_and_labels_are_clamped():
    c, _, m = _model("prior_ragged")
    codes, labels, _ = make_prior_inputs(c)
    x = torch.from_numpy(codes).cuda()
    lab = torch.from_numpy(labels).cuda()
    bad_x = x.clone()
    bad_x[0, 0, 0], bad_x[1, 2, 3], bad_x[2, 4, 4] = -7, c["K"], c["K"] + 100
    want_x = bad_x.clamp(0, c["K"] - 1)
    bad_l = torch.tensor([-1, c["n_classes"], 1], device="cuda")
    want_l = bad_l.clamp(0, c["n_classes"] - 1)
    assert torch.equal(m(bad_x, bad_l), m(want_x, want_l))
    u = torch.rand((3, c["size"], c["size"]), device="cuda")
    assert torch.equal(m._sample(bad_l, u), m._sample(want_l, u))


def test_generate_launch_count_and_graph_capture():
    from vqvae_b200 import ops
    c, _, m = _model("prior_default")
    B, S = 16, c["size"]
    labels = torch.arange(B, device="cuda") % 10
    u = torch.rand((B, S, S), device="cuda")
    x = torch.randint(0, c["K"], (B, S, S), device="cuda")
    ref_codes, ref_logits = m._sample(labels, u), m(x, labels)
    n0 = ops.launch_count()
    m._sample(labels, u)
    assert ops.launch_count() - n0 == S * (c["n_layers"] + S)
    n0 = ops.launch_count()
    m(x, labels)
    assert ops.launch_count() - n0 == 2 + 2 * c["n_layers"]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        codes_g = m._sample(labels, u)
        logits_g = m(x, labels)
    u.copy_(torch.rand_like(u))
    x.copy_(torch.randint(0, c["K"], x.shape, device="cuda"))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(codes_g, m._sample(labels, u)) and torch.equal(logits_g, m(x, labels))
    assert not torch.equal(codes_g, ref_codes) and not torch.equal(logits_g, ref_logits)


def test_standalone_layer_and_gate_match_torch():
    c, sd, m = _model("prior_ragged")
    torch.manual_seed(3)
    x = torch.randn((2, 2 * c["dim"], 5, 5), device="cuda")
    want = torch.tanh(x[:, :c["dim"]]) * torch.sigmoid(x[:, c["dim"]:])
    torch.testing.assert_close(m.layers[0].gate(x), want, atol=1e-6, rtol=0)
    for i in (0, 1):
        layer = m.layers[i]
        x_v, x_h = torch.randn((2, c["dim"], 5, 5), device="cuda"), torch.randn((2, c["dim"], 5, 5), device="cuda")
        h = torch.tensor([0, 2], device="cuda")
        out_v, out_h = layer(x_v, x_h, h)
        k = 7 if i == 0 else 3
        p = {n: t.detach().cpu().double() for n, t in layer.state_dict().items()}
        xv, xh = x_v.cpu().double(), x_h.cpu().double()
        e = p["class_cond_embedding.weight"][h.cpu()][:, :, None, None]
        hv = F.conv2d(xv, p["vert_stack.weight"], p["vert_stack.bias"], 1, k // 2)[:, :, :5]
        g = lambda t: torch.tanh(t[:, :c["dim"]]) * torch.sigmoid(t[:, c["dim"]:])   # noqa: E731
        hh = F.conv2d(xh, p["horiz_stack.weight"], p["horiz_stack.bias"], 1, (0, k // 2))[:, :, :, :5]
        o = g(F.conv2d(hv, p["vert_to_horiz.weight"], p["vert_to_horiz.bias"]) + hh + e)
        oh = F.conv2d(o, p["horiz_resid.weight"], p["horiz_resid.bias"]) + (xh if i else 0)
        torch.testing.assert_close(out_v.cpu().double(), g(hv + e), atol=1e-5, rtol=0)
        torch.testing.assert_close(out_h.cpu().double(), oh, atol=1e-5, rtol=0)


def test_generated_codes_decode_to_images():
    """Prior samples -> VQVAE.decode (fp32 mode) equals the C oracle's decoder on the codebook rows of the same codes."""
    from models.vqvae import VQVAE
    from oracle import cref
    from vqvae_b200.synth import make_state_dict
    c, _, m = _model("prior_default")
    hp = dict(h_dim=128, res_h_dim=32, n_res_layers=2, n_embeddings=512, embedding_dim=64)
    sd = make_state_dict(seed=0, codebook="normal", codebook_scale=0.05, **hp)
    vq = VQVAE(128, 32, 2, 512, 64, 0.25)
    vq.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    vq = vq.cuda().eval()
    torch.manual_seed(0)
    codes = m.generate(torch.arange(4, device="cuda"), shape=(8, 8), batch_size=4)
    x = vq.decode(codes.view(-1, 1), (8, 8))
    assert x.shape == (4, 3, 32, 32)
    E = np.asarray(sd["vector_quantization.embedding.weight"])
    zq = np.ascontiguousarray(E[codes.cpu().numpy()].transpose(0, 3, 1, 2))          # (4, 64, 8, 8)
    np.testing.assert_allclose(x.cpu().numpy(), cref.decoder(zq, sd, 2), atol=2e-6, rtol=0)

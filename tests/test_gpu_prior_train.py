"""Training the Gated PixelCNN prior on the H100: gradients against fp64 autograd of the differentiable restatement
(mask A's taps included), bitwise logits and launch counts in grad mode, deterministic backward, the reference's Adam
loop and an SGD trajectory against fp64, CUDA-graph capture of forward + backward, and a trained model's round trip."""
import numpy as np
import pytest
import torch

from oracle.prior_port import PRIOR_CASES, make_prior_inputs, make_prior_state_dict, prior_shapes
from oracle.prior_train_port import leaf_params, prior_logits, prior_loss

pytestmark = pytest.mark.gpu


def _setup(name):
    from pixelcnn.models import GatedPixelCNN
    c = PRIOR_CASES[name]
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"])
    m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    codes, labels, _ = make_prior_inputs(c)
    return c, sd, m.cuda(), torch.from_numpy(codes), torch.from_numpy(labels)


def _upstream(c, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((c["batch"], c["K"], c["size"], c["size"]), generator=g, dtype=torch.float64)


def _worst(got, want):
    """max over tensors of max|got - want| / max|want|"""
    return max(float((got[k].double().cpu() - want[k]).abs().max() / want[k].abs().max().clamp_min(1e-30))
               for k in want)


@pytest.mark.parametrize("kind", ["ce", "random"])
@pytest.mark.parametrize("name", ["prior_ragged", "prior_default", "prior_cfg3"])
def test_gradients_match_fp64_autograd_of_the_restatement(name, kind):
    c, sd, m, x, lab = _setup(name)
    with torch.enable_grad():
        g = leaf_params(sd, torch.float64)
        lg = prior_logits(g, x, lab, c["n_layers"])
        (prior_loss(lg, x) if kind == "ce" else (lg * _upstream(c, 9)).sum()).backward()
        want = {k: v.grad for k, v in g.items()}
        xc, lc = x.cuda(), lab.cuda()
        out = m(xc, lc)
        assert out.requires_grad
        if kind == "ce":
            prior_loss(out, xc).backward()
        else:
            out.backward(_upstream(c, 9).float().cuda())
    got = {k: p.grad for k, p in m.named_parameters()}
    assert all(got[k].shape == want[k].shape and got[k].dtype == torch.float32 for k in want)
    worst = _worst(got, want)
    masked = max(float((got[k].double().cpu() - want[k]).abs()[sl].max() / want[k].abs().max())
                 for k, sl in (("layers.0.vert_stack.weight", np.s_[:, :, -1]),
                               ("layers.0.horiz_stack.weight", np.s_[:, :, :, -1])))
    assert float(want["layers.0.vert_stack.weight"][:, :, -1].abs().max()) > 0
    print(f"{name} {kind}: worst |g - g64| / max|g64| = {worst:.2e} (mask A taps {masked:.2e})")
    assert worst <= (1e-4 if name == "prior_cfg3" else 2e-5)


def test_grad_mode_logits_are_the_inference_logits_with_the_same_launches():
    from vqvae_b200 import ops
    c, _, m, x, lab = _setup("prior_default")
    xc, lc = x.cuda(), lab.cuda()
    ref = m(xc, lc)
    with torch.enable_grad():
        n0 = ops.launch_count()
        out = m(xc, lc)
        assert ops.launch_count() - n0 == 2 + 2 * c["n_layers"]
    assert out.requires_grad and torch.equal(out.detach(), ref)


def test_backward_is_deterministic_and_its_launch_count_is_documented():
    from vqvae_b200 import ops
    c, _, m, x, lab = _setup("prior_default")
    xc, lc = x.cuda(), lab.cuda()
    G = _upstream(c, 3).float().cuda()
    runs = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        with torch.enable_grad():
            out = m(xc, lc)
            n0 = ops.launch_count()
            out.backward(G)
            assert ops.launch_count() - n0 == 7 + 10 * c["n_layers"]
        runs.append({k: p.grad.clone() for k, p in m.named_parameters()})
    assert all(torch.equal(runs[0][k], runs[1][k]) for k in runs[0])


def _train64(sd, c, x, lab, make_opt, steps):
    g = leaf_params(sd, torch.float64)
    opt = make_opt(list(g.values()))
    losses = []
    with torch.enable_grad():
        for _ in range(steps):
            loss = prior_loss(prior_logits(g, x, lab, c["n_layers"]), x)
            opt.zero_grad()
            loss.backward()
            opt.step()
            losses.append(loss.item())
    return losses, g


def test_reference_adam_loop_tracks_fp64():
    c, sd, m, x, lab = _setup("prior_ragged")
    want, _ = _train64(sd, c, x, lab, lambda p: torch.optim.Adam(p, lr=3e-4), 100)
    opt = torch.optim.Adam(m.parameters(), lr=3e-4)
    xc, lc = x.cuda(), lab.cuda()
    l0 = m.layers[0]
    got = []
    with torch.enable_grad():
        for _ in range(100):
            logits = m(xc, lc)
            assert l0.vert_stack.weight[:, :, -1].abs().sum() == 0 and l0.horiz_stack.weight[:, :, :, -1].abs().sum() == 0
            logits = logits.permute(0, 2, 3, 1).contiguous()
            loss = torch.nn.CrossEntropyLoss()(logits.view(-1, c["K"]), xc.view(-1))
            opt.zero_grad()
            loss.backward()
            opt.step()
            got.append(loss.item())
    rel = max(abs(a - b) / abs(b) for a, b in zip(got, want))
    print(f"adam: loss {got[0]:.5f} -> {got[50]:.5f} @50 -> {got[99]:.5f} @99; worst relative to fp64 {rel:.2e}")
    assert rel <= 1e-3


def test_sgd_trajectory_tracks_fp64():
    c, sd, m, x, lab = _setup("prior_ragged")
    _, g = _train64(sd, c, x, lab, lambda p: torch.optim.SGD(p, lr=0.05), 50)
    opt = torch.optim.SGD(m.parameters(), lr=0.05)
    xc, lc = x.cuda(), lab.cuda()
    with torch.enable_grad():
        for _ in range(50):
            loss = prior_loss(m(xc, lc), xc)
            opt.zero_grad()
            loss.backward()
            opt.step()
    worst = _worst(dict(m.named_parameters()), {k: v.detach() for k, v in g.items()})
    print(f"sgd: 50 steps, worst |p - p64| / max|p64| = {worst:.2e}")
    assert worst <= 1e-5


def test_forward_and_backward_capture_in_a_cuda_graph():
    c, _, m, x, lab = _setup("prior_ragged")
    xc, lc = x.cuda(), lab.cuda()
    G = _upstream(c, 5).float().cuda()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.enable_grad():
        for _ in range(2):
            m.zero_grad(set_to_none=True)
            m(xc, lc).backward(G)
    torch.cuda.current_stream().wait_stream(s)
    eager = {k: p.grad.clone() for k, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph), torch.enable_grad():
        logits = m(xc, lc)
        logits.backward(G)
    for p in m.parameters():
        p.grad.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(p.grad, eager[k]) for k, p in m.named_parameters())


def test_trained_prior_samples_decodes_and_keeps_the_reference_state_dict():
    from models.vqvae import VQVAE
    from oracle.prior_port import prior_forward
    from vqvae_b200.synth import make_state_dict
    c, _, m, x, lab = _setup("prior_default")
    opt = torch.optim.Adam(m.parameters(), lr=3e-4)
    xc, lc = x.cuda(), lab.cuda()
    with torch.enable_grad():
        for _ in range(3):
            loss = prior_loss(m(xc, lc), xc)
            opt.zero_grad()
            loss.backward()
            opt.step()
    sd = m.state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == \
        prior_shapes(c["K"], c["dim"], c["n_layers"], c["n_classes"])
    logits = m(xc, lc)                      # repacks (and re-zeroes mask A) after the last step
    trained = {k: v.cpu() for k, v in m.state_dict().items()}
    want = prior_forward(trained, x, lab, c["n_layers"])
    np.testing.assert_allclose(logits.cpu().numpy(), want.numpy(), atol=1e-4, rtol=0)
    hp = dict(h_dim=128, res_h_dim=32, n_res_layers=2, n_embeddings=512, embedding_dim=64)
    vq = VQVAE(128, 32, 2, 512, 64, 0.25)
    vq.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in make_state_dict(seed=0, **hp).items()})
    vq = vq.cuda().eval()
    torch.manual_seed(0)
    codes = m.generate(torch.arange(4, device="cuda"), shape=(8, 8), batch_size=4)
    img = vq.decode(codes.view(-1, 1), (8, 8))
    assert img.shape == (4, 3, 32, 32) and bool(torch.isfinite(img).all())

"""The masked restatement of the VQ-VAE (tests/vqvae_masked.py) without a GPU: fed the masks of its own fp64 forward,
built from the activations the GPU's training walk keeps in the order model_masks lays them out, its gradients equal
plain fp64 autograd of oracle/vqvae_train_port.py.  So the masks are consumed in the right order and each exactly
once, and the GPU tests that feed it the GPU's masks differentiate the function the GPU's backward does."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.prior_train_port import leaf_params
from oracle.torch_port import residual_stack
from oracle.vqvae_train_port import train_loss, vector_quantizer, vqvae_train_forward
from oracle.weights import make_state_dict
from tests.vqvae_masked import masked_relu, model_masks, stack_mask_list, vqvae64

HP = dict(h_dim=32, res_h_dim=8, n_res_layers=2, n_embeddings=16, embedding_dim=8)
VAR = 0.0625


def _params(sd):
    return leaf_params({k: sd[k] for k in sd if ".stack." not in k or ".stack.0." in k}, torch.float64)


def _kept(x, p, n, idx):
    """The activations the training walk keeps, from a plain fp64 forward: encoder (a1, a2, a3, e_out) with a3 the
    ReLU'd conv 4 output, decoder (d1, d_out, d2) with d1 the ReLU'd convT 0 output; and the stacks' weights."""
    e, d = "encoder.conv_stack.", "decoder.inverse_conv_stack."
    a1 = torch.relu(F.conv2d(x, p[e + "0.weight"], p[e + "0.bias"], 2, 1))
    a2 = torch.relu(F.conv2d(a1, p[e + "2.weight"], p[e + "2.bias"], 2, 1))
    h4 = F.conv2d(a2, p[e + "4.weight"], p[e + "4.bias"], 1, 1)
    ew = (p[e + "5.stack.0.res_block.1.weight"], p[e + "5.stack.0.res_block.3.weight"])
    e_out = residual_stack(h4, *ew, n)
    z_e = F.conv2d(e_out, p["pre_quantization_conv.weight"], p["pre_quantization_conv.bias"])
    _, z_q, _, _ = vector_quantizer(z_e, p["vector_quantization.embedding.weight"], 0.25, idx)
    h0 = F.conv_transpose2d(z_q, p[d + "0.weight"], p[d + "0.bias"], 1, 1)
    dw = (p[d + "1.stack.0.res_block.1.weight"], p[d + "1.stack.0.res_block.3.weight"])
    d_out = residual_stack(h0, *dw, n)
    d2 = torch.relu(F.conv_transpose2d(d_out, p[d + "2.weight"], p[d + "2.bias"], 2, 1))
    return (a1, a2, torch.relu(h4), e_out), (torch.relu(h0), d_out, d2), dict(enc=ew, dec=dw)


def _stack(weights, n):
    def masks(side, r0, out):
        w1, w2 = weights[side]
        mid = lambda r: torch.relu(F.conv2d(r, w1, None, 1, 1))                  # noqa: E731
        step = lambda r: torch.relu(r + F.conv2d(mid(r), w2))                    # noqa: E731
        return stack_mask_list(r0, out, n, mid, step)
    return masks


def _grads(p, x):
    return {k: v.grad.clone() for k, v in p.items()} | {"image": x.grad.clone()}


def _rel(got, want):
    return max(float((got[k] - want[k]).abs().max() / want[k].abs().max().clamp_min(1e-300)) for k in want)


def test_masked_restatement_at_its_own_masks_is_plain_fp64_autograd():
    n = HP["n_res_layers"]
    sd = make_state_dict(seed=3, codebook="normal", codebook_scale=0.1, **HP)
    x0 = torch.from_numpy(np.random.RandomState(4).uniform(-1, 1, (2, 3, 16, 24))).double()   # H != W
    with torch.enable_grad():
        p, x = _params(sd), x0.clone().requires_grad_()
        emb, x_hat, _, idx = vqvae_train_forward(x, p, n)
        train_loss(x, x_hat, emb, VAR)[0].backward()
        want = _grads(p, x)
    with torch.no_grad():
        enc, dec, weights = _kept(x0, {k: v.detach() for k, v in p.items()}, n, idx)
        masks = model_masks(enc, dec, _stack(weights, n))
    assert len(masks) == 2 + 2 * (2 * n + 1) + 1
    assert all(0 < float(m.double().mean()) < 1 for m in masks)          # every mask has both signs: none is trivial

    def masked(ms):
        relu, done = masked_relu(ms)
        with torch.enable_grad():
            q, xm = _params(sd), x0.clone().requires_grad_()
            emb, x_hat = vqvae64(xm, q, n, relu, idx)
            train_loss(xm, x_hat, emb, VAR)[0].backward()
        assert done()                                                    # every mask used, each once
        return _grads(q, xm)

    got = masked(masks)
    assert set(got) == set(want)
    worst = _rel(got, want)
    print(f"masked restatement vs plain fp64 autograd: {worst:.1e}")
    assert worst <= 1e-12
    # the check is sharp: the encoder stack's first two input masks swapped (same shape) move the gradients
    swapped = list(masks)
    swapped[2], swapped[4] = swapped[4], swapped[2]
    assert _rel(masked(swapped), want) > 1e-6

"""The VQ-VAE training step (VQVAE.forward in model.train(), main.py's loss, backward) at shapes where a latent image
does not fit one 128-pixel tile, against fp64 autograd of the restatement at the GPU's own ReLU masks and codes.

An fp64 forward flips ReLU masks against the GPU's forward, which is why the whole-model TF32 bar against a plain fp64
forward is 0.15 of max |g|.  Here the fp64 side (tests/vqvae_masked.py) multiplies by the masks the GPU's training walk
produced -- acts["enc"], acts["dec"] and the stack masks recomputed as _stack_backward does -- and quantizes to the
GPU's codes, so what is left is the backward's own arithmetic: every parameter gradient and the image gradient are
held to a fraction of the tensor's max |g64|.  The shapes reach 16 x 16 latents (two tiles per image, the fused
decoder tail declined in training), 12 x 20 latents (ragged tiles on both axes, H != W in every backward call), cfg3's
256 x 256 images (adjoint grids of more than one wave, a 32 768-position input-conv weight gradient) and main.py's
batch of 32 in TF32.  Needs an H100 (``-m gpu``).
"""
import numpy as np
import pytest
import torch

from oracle.prior_train_port import leaf_params
from oracle.vqvae_train_port import train_loss
from oracle.weights import make_state_dict
from tests.vqvae_masked import masked_relu, model_masks, nchw64, stack_masks, vqvae64

pytestmark = pytest.mark.gpu

VAR = 0.0625
CFG3 = dict(h_dim=128, res_h_dim=32, n_res_layers=2, embedding_dim=64)
SMALL_ODD = dict(h_dim=32, res_h_dim=8, n_res_layers=3, embedding_dim=16)
# name -> (architecture, K, B, H, W, codebook scale, seed)
CASES = {
    "s64": (CFG3, 1024, 3, 64, 64, 0.05, 1),              # 16 x 16 latents: no whole-image tile
    "s48x80": (CFG3, 512, 3, 48, 80, 0.05, 2),            # 12 x 20 latents: ragged tiles on both axes
    "s256": (CFG3, 1024, 2, 256, 256, 0.05, 3),           # cfg3's image size
    "main_py_b32": (CFG3, 512, 32, 32, 32, 0.05, 4),      # main.py's batch
    "small_odd_s64": (SMALL_ODD, 50, 3, 64, 64, 0.08, 5),  # Cin < 32 layers: the FFMA adjoints
}
CODEBOOK = "vector_quantization.embedding.weight"
# TF32 bars, of max |g64| per tensor, at most twice the worst tensor measured on an H100 80GB HBM3 (700 W power limit):
# s64 4.7e-3, s48x80 4.1e-3, s256 5.3e-3 (encoder residual W2), main_py_b32 4.3e-3, small_odd_s64 1.8e-3 (encoder
# conv 0), all in the encoder, whose gradients pass through every adjoint conv.  The fp32 mode is within 1e-6 on the
# same cases.  Against a plain fp64 forward, whose ReLU masks differ, TF32 steps at 32 x 32 are off by up to 0.09
# (tests/test_gpu_vqvae_train.py).
TF32_BAR = dict(s64=8e-3, s48x80=8e-3, s256=1e-2, main_py_b32=8e-3, small_odd_s64=3e-3)


def _model(name):
    from models.vqvae import VQVAE
    hp, K, B, H, W, scale, seed = CASES[name]
    sd = make_state_dict(seed=seed, n_embeddings=K, codebook="normal", codebook_scale=scale, **hp)
    m = VQVAE(hp["h_dim"], hp["res_h_dim"], hp["n_res_layers"], K, hp["embedding_dim"], 0.25)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    x = torch.from_numpy(np.random.RandomState(100 + seed).uniform(-1, 1, (B, 3, H, W)).astype(np.float32))
    return sd, m.cuda().train(), x


def _gpu_step(name, mode):
    """One training step in `mode` -> (gradients by parameter name and "image", the GPU's codes, the ReLU masks its
    backward read, NHWC; none in bf16 mode), and the state dict and images it ran on."""
    import vqvae_b200
    from vqvae_b200._lib import PRECISIONS
    sd, m, x = _model(name)
    n = m.encoder.conv_stack[5].n_res_layers
    layers = dict(enc=m.encoder.conv_stack[5].stack[0], dec=m.decoder.inverse_conv_stack[1].stack[0])
    xc = x.cuda()
    with vqvae_b200.precision(mode):
        masks = None
        if mode != "bf16":
            acts = {}
            m._walk(xc, False, acts)             # the training walk: the activations the backward reads
            prec = PRECISIONS[mode]
            masks = model_masks(acts["enc"], acts["dec"],
                                lambda side, r0, out: stack_masks(layers[side], r0, out, n, precision=prec))
            idx = acts["idx"].clone()
        xg = xc.clone().requires_grad_()
        m.zero_grad(set_to_none=True)
        with torch.enable_grad():
            embedding_loss, x_hat, _ = m(xg)
            (torch.mean((x_hat - xg) ** 2) / VAR + embedding_loss).backward()
    if masks is not None:
        assert torch.equal(m.last_min_encoding_indices.view(-1), idx)
    got = {k: p.grad.clone() for k, p in m.named_parameters()}
    got["image"] = xg.grad.clone()
    return got, m.last_min_encoding_indices.view(-1).clone(), masks, sd, x


def _fp64(name, sd, x, idx, masks):
    """fp64 autograd of the restatement at the GPU's masks and codes -> gradients by parameter name and "image"."""
    relu, done = masked_relu(nchw64(masks))
    with torch.enable_grad():
        p = leaf_params({k: sd[k] for k in sd if ".stack." not in k or ".stack.0." in k}, torch.float64)
        xt = x.double().requires_grad_()
        embedding_loss, x_hat = vqvae64(xt, p, CASES[name][0]["n_res_layers"], relu, idx.cpu())
        train_loss(xt, x_hat, embedding_loss, VAR)[0].backward()
    assert done()                                   # every mask used, each once
    want = {k: v.grad for k, v in p.items()}
    want["image"] = xt.grad
    return want


@pytest.fixture(scope="module")
def runs():
    """(name, mode) -> (GPU gradients, fp64 gradients or None in bf16 mode), each computed once per module: the
    256 x 256 case's fp64 reference is about 17 G multiply-adds per mode."""
    cache = {}

    def get(name, mode):
        if (name, mode) not in cache:
            got, idx, masks, sd, x = _gpu_step(name, mode)
            cache[(name, mode)] = (got, None if masks is None else _fp64(name, sd, x, idx, masks))
        return cache[(name, mode)]
    return get


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
@pytest.mark.parametrize("name", list(CASES))
def test_training_step_matches_fp64_at_the_gpu_masks(name, mode, runs):
    got, want = runs(name, mode)
    assert set(got) == set(want)
    per = {k: float((got[k].double().cpu() - want[k]).abs().max() / want[k].abs().max()) for k in want}
    print(f"{name} {mode} at the GPU's masks:",
          " ".join(f"{k}={v:.1e}" for k, v in sorted(per.items(), key=lambda kv: -kv[1])))
    bar = 1e-4 if mode == "fp32" else TF32_BAR[name]
    for k, v in per.items():
        assert v <= bar, (k, v, bar)


def test_bf16_mode_gradients_are_the_tf32_ones_at_256(runs):
    """bf16 mode trains on the TF32 kernels: every gradient bitwise TF32's, but the codebook's (float atomics)."""
    tf32, _ = runs("s256", "tf32")
    bf16, _ = runs("s256", "bf16")
    assert set(bf16) == set(tf32)
    for k in tf32:
        if k != CODEBOOK:
            assert torch.equal(bf16[k], tf32[k]), k

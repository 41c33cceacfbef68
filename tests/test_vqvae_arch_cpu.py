"""The VQ-VAE architectures of tests/vqvae_arch.py without a GPU: the C oracle and the fp64 restatement reproduce the
unmodified reference's outputs and gradients (tests/golden/arch_*.npz, made by oracle/make_arch_golden.py), and the
restated dispatch rules agree with every answer the library gives without a device."""
import numpy as np
import pytest
import torch

from oracle import cref
from oracle.prior_train_port import fingerprint, leaf_params
from oracle.vqvae_train_port import train_loss
from tests.helpers import load_golden
from tests.vqvae_arch import (ARCHS, GOLDEN_ARCHS, arch_inputs, bf16_covered, bf16_kind_ok, bf16_layers,
                              decoder_tail_shape, expected_kernels, fused_blocks, latent_block_shape, wg)
from tests.vqvae_masked import vqvae64


def _golden(name):
    g = load_golden("arch_" + name)
    hp, sd, x = arch_inputs(name)
    assert {k: g["case"][k] for k in hp} == hp and g["case"]["seed"] == ARCHS[name][8]
    return g, hp, sd, x


@pytest.mark.parametrize("name", GOLDEN_ARCHS)
def test_c_oracle_reproduces_the_reference(name):
    g, hp, sd, x = _golden(name)
    o = cref.vqvae_forward(x, sd, hp["n_res_layers"])
    # the oracle accumulates in double, the reference in fp32 over up to 512 * 9 products
    np.testing.assert_allclose(o["z_e"], g["z_e"], atol=1e-6, rtol=0)
    b = cref.vq_nchw(g["z_e"], sd["vector_quantization.embedding.weight"])
    assert np.array_equal(b["idx"], g["idx"])                   # same z_e in: the same codes
    assert np.array_equal(o["idx"], g["idx"])
    np.testing.assert_allclose(o["x_hat"], g["x_hat"], atol=1e-6, rtol=0)
    np.testing.assert_allclose(o["loss"], g["loss"], rtol=1e-5)
    np.testing.assert_allclose(o["perplexity"], g["perplexity"], rtol=2e-5)


@pytest.mark.parametrize("name", GOLDEN_ARCHS)
def test_fp64_restatement_reproduces_the_reference_forward_and_gradients(name):
    g, hp, sd, x = _golden(name)
    torch.set_num_threads(4)
    p = leaf_params({k: sd[k] for k in sd if ".stack." not in k or ".stack.0." in k}, torch.float64)
    xt = torch.from_numpy(x).double()
    with torch.enable_grad():
        emb, x_hat = vqvae64(xt, p, hp["n_res_layers"], torch.relu, torch.from_numpy(g["idx"].ravel()))
        loss, recon = train_loss(xt, x_hat, emb, g["case"]["x_train_var"])
        loss.backward()
    np.testing.assert_allclose(x_hat.detach().numpy(), g["x_hat"], atol=1e-6, rtol=0)
    np.testing.assert_allclose(loss.item(), float(g["train_loss"]), rtol=1e-5)
    keys = list(sd)
    for k, v in p.items():
        gr = v.grad.numpy()
        np.testing.assert_allclose(fingerprint(gr, keys.index(k)), g["grad/" + k], rtol=0, err_msg=k,
                                   atol=1e-4 * np.abs(gr).max() * np.sqrt(gr.size))


@pytest.mark.parametrize("name", list(ARCHS))
def test_dispatch_restatement_agrees_with_the_library_queries(name):
    import warnings
    import vqvae_b200
    from vqvae_b200 import _lib, ops
    lib = ops.lib()
    h, r, n, K, D, B, (H, W) = ARCHS[name][:7]
    H2, W2 = H // 4, W // 4
    assert bool(lib.vqb_latent_block_supported(h, H2, W2, h, r, D)) == latent_block_shape(h, h, r, H2, W2, D)
    assert bool(lib.vqb_latent_block_supported(D, H2, W2, h, r, 0)) == latent_block_shape(D, h, r, H2, W2, 0)
    assert bool(lib.vqb_decoder_tail_supported(h, H2, W2, h // 2, 3)) == decoder_tail_shape(h, H2, W2, h // 2, 3)
    kinds = dict(K1=_lib.CONV_K1, K3=_lib.CONV_K3, CONVT_K3=_lib.CONVT_K3, K4S2=_lib.CONV_K4S2,
                 CONVT_K4S2=_lib.CONVT_K4S2, CONVT_K4S2_OUT=_lib.CONVT_K4S2_OUT, RES_W2=_lib.RES_W2)
    for kind, cout, cin in bf16_layers(h, r, n, D):
        assert (lib.vqb_conv_bf16_packed_bytes(kinds[kind], cout, cin) != 0) == bf16_kind_ok(kind, cout, cin), kind
    m = vqvae_b200.VQVAE(h, r, n, K, D, 0.25)
    with vqvae_b200.precision("bf16"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        assert m._bf16_pipeline() is bf16_covered(name)


def test_every_row_reaches_a_kernel_the_cfg2_architecture_does_not():
    """Each row's restated kernels differ from the cfg2 architecture's (128, 32, 2, 512, 64 on 32 x 32 images) in some
    precision and walk."""
    from tests import vqvae_arch
    vqvae_arch.ARCHS["_cfg2"] = (128, 32, 2, 512, 64, 4, (32, 32), 0.05, 0)
    try:
        for name in ARCHS:
            if name != "_cfg2":
                assert any(expected_kernels(name, p, w) != expected_kernels("_cfg2", p, w)
                           for p in ("fp32", "tf32", "bf16") for w in ("eval", "train")), name
        assert fused_blocks("_cfg2") == (True, True, True) and bf16_covered("_cfg2")
    finally:
        del vqvae_arch.ARCHS["_cfg2"]


def test_restated_launches_of_the_rows_are_the_documented_paths():
    """A few of the row claims, read off the restatement."""
    k = expected_kernels
    assert k("h512", "tf32", "eval")["conv_in_k4s2_kernel"] == 1                 # Cout 256: 48 KB of weights
    assert k("h96", "tf32", "eval")["conv_small_cout_kernel"] == 4               # output layer from 48 channels
    assert k("h96", "tf32", "eval")["vq_exact_kernel"] == 1
    assert k("n6", "tf32", "eval")["res_scatter_kernel"] == 2                    # both latent blocks fused
    assert k("r64", "tf32", "eval")["wgconv_kernel<false, 64, 128, false>"] == 4  # res_wg per application
    assert k("r16", "bf16", "eval")["wgconv_kernel<true, 16, 128, false>"] == 6
    assert k("h160", "tf32", "eval")[wg(256)] == 6      # 160 live of N = 256: the k3 convs and 4 residual 1x1s

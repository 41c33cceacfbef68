"""CPU checks of VQ-VAE training: the differentiable restatement against the reference's gradient and trajectory
goldens, argument checks of the new entry points, and the training path's rejections that need no GPU."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle.make_golden import MODEL_CASES
from oracle.prior_train_port import fingerprint, leaf_params
from oracle.vqvae_train_port import train_loss, vqvae_train_forward
from oracle.weights import make_images, make_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HP = ("h_dim", "res_h_dim", "n_res_layers", "n_embeddings", "embedding_dim")


def _golden(name):
    with np.load(os.path.join(ROOT, "tests", "golden", name + ".npz")) as d:
        return {k: d[k] for k in d.files}


def _case(fixture):
    want = _golden(fixture)
    c = json.loads(str(want["case"]))
    base = {k: v for k, v in c.items() if k not in ("x_train_var", "steps")}
    name = next(n for n, v in MODEL_CASES.items() if v == base)
    sd = make_state_dict(seed=c["wseed"], codebook=c["codebook"], codebook_scale=c["codebook_scale"],
                         **{k: c[k] for k in HP})
    return c, name, sd, make_images(c["batch"], c["size"], c["xseed"]), want


def _single_thread(fn):
    threads = torch.get_num_threads()
    torch.set_num_threads(1)            # the goldens were made single-threaded
    try:
        with torch.enable_grad():
            return fn()
    finally:
        torch.set_num_threads(threads)


def _param_keys(sd):
    """The state-dict keys that are parameters: the shared ResidualLayer's key under stack.0 only."""
    return [k for k in sd if ".stack." not in k or ".stack.0." in k]


def _restated_grads(c, sd, x):
    def run():
        g = leaf_params({k: sd[k] for k in _param_keys(sd)})
        xt = torch.from_numpy(x)
        emb, x_hat, perp, idx = vqvae_train_forward(xt, g, c["n_res_layers"])
        loss, recon = train_loss(xt, x_hat, emb, c["x_train_var"])
        loss.backward()
        return loss.item(), recon.item(), perp.item(), idx.numpy(), {k: v.grad.numpy() for k, v in g.items()}
    return _single_thread(run)


def test_restatement_reproduces_the_reference_gradients_in_full():
    c, name, sd, x, want = _case("vqvae_grad_small_odd")
    assert name == "small_odd"
    loss, recon, perp, idx, grads = _restated_grads(c, sd, x)
    assert np.array_equal(idx, want["idx"])
    for got, key in ((loss, "loss"), (recon, "recon_error"), (perp, "perplexity")):
        assert abs(got - float(want[key])) <= 1e-5 * abs(float(want[key])), key
    assert sorted(k[5:] for k in want if k.startswith("grad/")) == sorted(grads)
    for k, v in grads.items():
        w = want["grad/" + k]
        assert v.shape == w.shape, k
        np.testing.assert_allclose(v, w, atol=1e-5 * np.abs(w).max(), rtol=0, err_msg=k)


def test_restatement_reproduces_the_reference_gradient_fingerprints():
    c, name, sd, x, want = _case("vqvae_grad_cifar_default")
    assert name == "cifar_default"
    loss, recon, perp, idx, grads = _restated_grads(c, sd, x)
    assert np.array_equal(idx, want["idx"])
    assert abs(loss - float(want["loss"])) <= 1e-5 * abs(float(want["loss"]))
    keys = list(sd)
    for k, v in grads.items():
        tol = 1e-5 * np.abs(v).max() * np.sqrt(v.size)
        np.testing.assert_allclose(fingerprint(v, keys.index(k)), want["grad/" + k], atol=tol, rtol=0, err_msg=k)


def test_restatement_reproduces_the_reference_adam_trajectory():
    c, name, sd, x, want = _case("vqvae_train_cifar_spread")
    assert name == "cifar_spread"

    def run():
        g = leaf_params({k: sd[k] for k in _param_keys(sd)})
        opt = torch.optim.Adam(list(g.values()), lr=3e-4, amsgrad=True)
        xt = torch.from_numpy(x)
        rows = []
        for _ in range(c["steps"]):
            opt.zero_grad()
            emb, x_hat, perp, _ = vqvae_train_forward(xt, g, c["n_res_layers"])
            loss, recon = train_loss(xt, x_hat, emb, c["x_train_var"])
            loss.backward()
            opt.step()
            rows.append([loss.item(), recon.item(), perp.item()])
        return np.array(rows)
    np.testing.assert_allclose(_single_thread(run), want["trajectory"], rtol=1e-4, atol=0)
    threads = torch.get_num_threads()
    torch.set_num_threads(4)            # the reference's second run
    try:
        with torch.enable_grad():
            got4 = run()
    finally:
        torch.set_num_threads(threads)
    np.testing.assert_allclose(got4, want["trajectory_threads4"], rtol=1e-4, atol=0)


def test_wgrad_entry_points_validate_arguments_without_a_gpu():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    wsb = lib.vqb_conv_wgrad_workspace_bytes
    assert wsb(0, 3, 8, 8, 16, 4, 4, 2, 1, 0) == 0
    assert wsb(2, 3, 8, 8, 16, 4, 4, 0, 1, 0) == 0
    assert wsb(2, 3, 8, 8, 16, 4, 4, 2, -1, 0) == 0
    assert wsb(2, 3, 2, 2, 16, 5, 5, 1, 0, 0) == 0               # empty output
    ws = wsb(2, 3, 8, 8, 16, 4, 4, 2, 1, 0)
    wst = wsb(2, 16, 4, 4, 3, 4, 4, 2, 1, 1)
    assert ws > 0 and wst > 0
    f = lib.vqb_conv_wgrad_f32
    args = (2, 3, 8, 8, 16, 4, 4, 2, 1, 0, 0, 1)
    assert f(None, p, p, p, *args, p, ws, None) == -1
    assert f(p, None, p, p, *args, p, ws, None) == -1
    assert f(p, p, None, p, *args, p, ws, None) == -1
    assert f(p, p, p, p, *args, None, ws, None) == -1
    assert f(p, p, p, p, 2, 3, 8, 8, 16, 4, 4, 2, 1, 0, 2, 1, p, ws, None) == -1      # bad layout
    assert f(p, p, p, p, 2, 3, 8, 8, 0, 4, 4, 2, 1, 0, 0, 1, p, ws, None) == -1
    assert f(p, p, p, p, *args, p, ws - 4, None) == -3
    assert f(p, p, p, p, 2, 16, 4, 4, 3, 4, 4, 2, 1, 1, 1, 0, p, wst - 4, None) == -3
    rb = lib.vqb_relu_backward_f32
    assert rb(None, p, p, 4, None) == -1
    assert rb(p, None, p, 4, None) == -1
    assert rb(p, p, None, 4, None) == -1
    assert rb(p, p, p, -1, None) == -1
    assert rb(p, p, p, 0, None) == 0


def test_wgrad_workspace_covers_the_plan_without_a_bias():
    """main.py's default shared 3x3 residual conv (128 -> 32, no bias) over its two applications at B = 32: 64 images
    of 8x8.  The size query must cover the plan without the bias column, and each call is checked against the
    partials of the plan it runs (every call below is rejected before any launch)."""
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    geom = (64, 128, 8, 8, 32, 3, 3, 1, 1, 0)
    q = lib.vqb_conv_wgrad_workspace_bytes(*geom)
    M, cols = 32, 9 * 128                       # rows: the 32 output channels; columns: 9 taps x 128 input channels
    splits = q // (4 * M * (cols + 1))
    assert q == 4 * splits * M * (cols + 1)     # the bias plan: the same splits, one more column
    no_bias = 4 * splits * M * cols
    assert no_bias >= 4 * 15 * M * cols         # 15 splits: what this geometry needs without the bias column
    f = lib.vqb_conv_wgrad_f32
    assert f(p, p, p, None, *geom, 1, 1, p, no_bias - 4, None) == -3
    assert f(p, p, p, p, *geom, 1, 1, p, no_bias, None) == -3      # with a bias the plan needs the ones column too


def _model():
    from models.vqvae import VQVAE
    return VQVAE(32, 8, 3, 50, 16, 0.25)


def test_training_rejects_a_process_group_before_any_launch():
    m = _model().train()
    m.process_group = object()
    with torch.enable_grad(), pytest.raises(RuntimeError, match="process_group"):
        m(torch.zeros((2, 3, 16, 16)))


def test_training_still_rejects_cpu_tensors():
    m = _model().train()
    with torch.enable_grad(), pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros((2, 3, 16, 16)))


def test_only_training_mode_with_grad_takes_the_differentiable_path():
    m = _model()
    x = torch.zeros((1, 3, 16, 16))
    with torch.enable_grad():
        assert m.training and m._trains(x)
        m.eval()
        assert not m._trains(x)                       # bench.py's pattern: eval() with grad enabled
        m.train()
        for p in m.parameters():
            p.requires_grad_(False)
        assert not m._trains(x)
        assert m._trains(x.requires_grad_())
    assert not m._trains(x)                          # no_grad

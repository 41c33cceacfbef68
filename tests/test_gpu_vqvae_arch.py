"""The VQ-VAE at the architectures main.py's flags build (tests/vqvae_arch.py): every layer's kernel path in fp32, TF32
and bf16, the forward against the reference and the C oracle, the training step against fp64 autograd of the
restatement at the GPU's own masks and codes, and the kernel names the profiler records against the restated dispatch
rules -- the check that each row reaches the path it is listed for, since a kernel that silently fell back to another
would pass every tolerance here.  Needs an H100 (``-m gpu``).
"""
import json
import os
import subprocess
import sys
import warnings
from collections import Counter

import numpy as np
import pytest
import torch

from oracle import cref
from oracle.prior_train_port import fingerprint, leaf_params
from oracle.vqvae_train_port import train_loss
from tests.helpers import load_golden
from tests.vqvae_arch import ARCHS, GOLDEN_ARCHS, arch_inputs, bf16_covered, expected_kernels, forward_kernels
from tests.vqvae_masked import masked_relu, model_masks, nchw64, stack_masks, vqvae64

pytestmark = pytest.mark.gpu

NAMES = list(ARCHS)
VAR = 0.0625
CODEBOOK = "vector_quantization.embedding.weight"
CONV_ATOL = 2e-6        # fp32 FFMA against the double-accumulated oracle, activations O(0.1 .. 1)
# TF32 training bars, of max |g64| per tensor: at most twice the worst tensor measured on an H100 80GB HBM3 (700 W
# power limit): h256 4.9e-3 (encoder residual W2), h64 4.2e-3, h96 1.9e-3, h160 3.5e-3, h512 9.2e-4, r64 4.3e-3,
# r16 4.0e-3, r48 4.8e-3, n0 3.7e-3, n6 5.5e-3, all in the encoder, whose gradients pass through every adjoint conv.
# The fp32 mode is within 2e-6 on every row.
TF32_BAR = dict(h256=9.5e-3, h64=8.5e-3, h96=3.8e-3, h160=7e-3, h512=1.8e-3, r64=8.5e-3, r16=8e-3, r48=9.5e-3,
                n0=7.4e-3, n6=1.1e-2)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _model(name, train=False):
    from models.vqvae import VQVAE
    hp, sd, x = arch_inputs(name)
    m = VQVAE(hp["h_dim"], hp["res_h_dim"], hp["n_res_layers"], hp["n_embeddings"], hp["embedding_dim"], 0.25)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    m = m.cuda()
    return (m.train() if train else m.eval()), hp, sd, x


def _rows(z_e, D):
    return z_e.reshape(-1, D).cpu().numpy()


@pytest.fixture(scope="module")
def oracle():
    """name -> the C oracle's fp32 forward (double-accumulated convs), computed once per module."""
    cache = {}

    def get(name):
        if name not in cache:
            hp, sd, x = arch_inputs(name)
            cache[name] = cref.vqvae_forward(x, sd, hp["n_res_layers"])
        return cache[name]
    return get


def _forward(name, mode):
    """One eval forward in `mode` -> (z_e rows, idx, x_hat, loss, perplexity) on the host, and the model."""
    import vqvae_b200
    m, hp, sd, x = _model(name)
    xc = _cuda(x)
    with vqvae_b200.precision(mode), torch.no_grad():
        z_e = m._encode_rows(xc, m._bf16_pipeline())[0]
        loss, x_hat, perp = m(xc)
    idx = m.last_min_encoding_indices.view(-1).cpu().numpy()
    return dict(z=_rows(z_e, hp["embedding_dim"]), idx=idx, x_hat=x_hat.cpu().numpy(), loss=loss.item(),
                perp=perp.item(), model=m, x=xc)


@pytest.fixture(scope="module")
def forwards():
    cache = {}

    def get(name, mode):
        if (name, mode) not in cache:
            cache[(name, mode)] = _forward(name, mode)
        return cache[(name, mode)]
    return get


def _nchw(rows, B, H, W):
    return np.ascontiguousarray(rows.reshape(B, H, W, -1).transpose(0, 3, 1, 2))


def _latent(name):
    B, (H, W) = ARCHS[name][5:7]
    return B, H // 4, W // 4


# --------------------------------------------------------------------------------------------------- fp32 forward
@pytest.mark.parametrize("name", NAMES)
def test_fp32_forward_matches_the_reference_and_the_oracle(name, forwards, oracle):
    hp, sd, x = arch_inputs(name)
    E = sd[CODEBOOK]
    f = forwards(name, "fp32")
    o = oracle(name)
    g = load_golden("arch_" + name) if name in GOLDEN_ARCHS else None
    want_z = g["z_e"] if g is not None else o["z_e"]
    B, H2, W2 = _latent(name)
    z = _nchw(f["z"], B, H2, W2)
    err_z = float(np.abs(z - want_z).max())
    np.testing.assert_allclose(z, want_z, atol=CONV_ATOL, rtol=0)
    v = cref.vq_rows(f["z"], E)
    assert np.array_equal(f["idx"], v["idx"])                    # bit-exact on the model's own z_e
    want_idx = (g["idx"] if g is not None else o["idx"]).ravel()
    bad = np.nonzero(f["idx"] != want_idx)[0]
    if bad.size:
        # a flip is only acceptable on a provable near-tie of the fp64 distances from the model's own z_e
        rows = f["z"].astype(np.float64)
        d = (rows ** 2).sum(1, keepdims=True) + (E.astype(np.float64) ** 2).sum(1) - 2 * rows @ E.astype(np.float64).T
        gap = np.abs(d[bad, f["idx"][bad]] - d[bad, want_idx[bad]])
        assert np.all(gap <= 4 * np.spacing(np.float32(np.abs(d[bad]).max()))), (bad.size, gap)
    assert bad.size <= max(1, f["idx"].size // 1000)
    # decoder: the oracle on the codes this forward chose, and the reference's x_hat when the codes agree
    xh_own = cref.decoder(_nchw(v["zq"], B, H2, W2), sd, hp["n_res_layers"])
    err_x = float(np.abs(f["x_hat"] - xh_own).max())
    np.testing.assert_allclose(f["x_hat"], xh_own, atol=CONV_ATOL, rtol=0)
    if bad.size == 0:
        np.testing.assert_allclose(f["x_hat"], g["x_hat"] if g is not None else o["x_hat"], atol=CONV_ATOL, rtol=0)
        np.testing.assert_allclose(f["loss"], float(g["loss"] if g is not None else o["loss"]), rtol=1e-5)
        np.testing.assert_allclose(f["perp"], float(g["perplexity"] if g is not None else o["perplexity"]), rtol=2e-5)
    print(f"{name} fp32: z_e {err_z:.1e}, x_hat {err_x:.1e}, flips {bad.size}")
    # encode / decode agree with forward
    import vqvae_b200
    m = f["model"]
    with vqvae_b200.precision("fp32"), torch.no_grad():
        idx = m.encode(f["x"])
        x_dec = m.decode(idx, (H2, W2))
    assert np.array_equal(idx.view(-1).cpu().numpy(), f["idx"])
    # decode feeds E[idx], forward z + (E[idx] - z): within 1 ulp of z_q
    np.testing.assert_allclose(x_dec.cpu().numpy(), f["x_hat"], atol=1e-6, rtol=0)


# --------------------------------------------------------------------------------------------------- TF32 forward
@pytest.mark.parametrize("name", NAMES)
def test_tf32_forward_against_fp32_and_the_training_walk(name, forwards):
    import vqvae_b200
    hp, sd, x = arch_inputs(name)
    B, H2, W2 = _latent(name)
    f32, t = forwards(name, "fp32"), forwards(name, "tf32")
    err_z = float(np.abs(t["z"] - f32["z"]).max())
    assert err_z <= 1e-3, err_z
    v = cref.vq_rows(t["z"], sd[CODEBOOK])
    assert np.array_equal(t["idx"], v["idx"])
    flips = int((t["idx"] != f32["idx"]).sum())
    # at most 0.5 %, or 3 flips: at 192 .. 640 rows one flip is 0.2 .. 0.5 % (test_tc_model_forward_tf32_tolerance)
    assert flips <= max(3, int(0.005 * t["idx"].size)), flips
    m = t["model"]
    with vqvae_b200.precision("fp32"), torch.no_grad():
        xh_ref = m.decode(_cuda(t["idx"]).view(-1, 1), (H2, W2)).cpu().numpy()
    err_x = float(np.abs(t["x_hat"] - xh_ref).max())
    assert err_x <= 1.5e-3, err_x
    print(f"{name} tf32: z_e {err_z:.1e}, flips {flips}/{t['idx'].size}, x_hat {err_x:.1e}")
    # the eval walk's fusions change launches, not bits
    lib = vqvae_b200.ops.lib()
    with vqvae_b200.precision("tf32"), torch.no_grad():
        torch.cuda.synchronize()
        n0 = lib.vqb_launch_count()
        loss_e, xh_e, perp_e = m._walk(t["x"], False)
        n1 = lib.vqb_launch_count()
        loss_t, xh_t, perp_t = m._walk(t["x"], False, acts={})
        n2 = lib.vqb_launch_count()
    assert torch.equal(xh_e, xh_t) and torch.equal(loss_e, loss_t) and torch.equal(perp_e, perp_t)
    assert np.array_equal(xh_e.cpu().numpy(), t["x_hat"])
    assert (n2 - n1) - (n1 - n0) == len(forward_kernels(name, "tf32", "train")) - \
        len(forward_kernels(name, "tf32", "eval"))


# --------------------------------------------------------------------------------------------------------- kernels
_PROFILE_SCRIPT = r"""
import json, re, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
import vqvae_b200
from models.vqvae import VQVAE
from tests.vqvae_arch import KERNELS, arch_inputs
BF16_ARG = {"convt_scatter_kernel": 0, "conv_in_k4s2_kernel": 1}

def norm(name):
    m = re.search(r"\b(" + "|".join(KERNELS) + r")\b(?:<([^<>]*)>)?", name)
    if m is None:
        return None
    base, args = m.group(1), [a.strip() for a in (m.group(2) or "").split(",")]
    if base == "wgconv_kernel":
        return f"{base}<{', '.join(args)}>"
    if base in BF16_ARG and args[BF16_ARG[base]] == "true":
        return base + "<bf16>"
    return base

def capture(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [norm(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return [n for n in names if n is not None]

def kernels(fn):
    # The profiler can lose activity records on a busy device (it never adds any), and fn launches the same kernels
    # every time: of three captures keep the fullest, and report how many came back short.
    caps = [capture(fn) for _ in range(3)]
    best = max(caps, key=len)
    return best, sum(len(c) < len(best) for c in caps)

out = {}
for name in json.loads(sys.argv[1]):
    hp, sd, x = arch_inputs(name)
    for mode in ("fp32", "tf32", "bf16"):
        m = VQVAE(hp["h_dim"], hp["res_h_dim"], hp["n_res_layers"], hp["n_embeddings"], hp["embedding_dim"], 0.25)
        m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
        m = m.cuda().eval()
        xc = torch.from_numpy(x).cuda()
        with vqvae_b200.precision(mode), torch.no_grad():
            m(xc)                                   # packs the weights outside the profiled window
            ev, ev_short = kernels(lambda: m(xc))
        m.train()
        xg = xc.clone().requires_grad_()

        def step():
            with vqvae_b200.precision(mode), torch.enable_grad():
                emb, x_hat, _ = m(xg)
                (torch.mean((x_hat - xg) ** 2) / 0.0625 + emb).backward()
        step()
        tr, tr_short = kernels(step)
        out[f"{name}/{mode}"] = dict(eval=ev, train=tr, short=ev_short + tr_short)
print(json.dumps(out))
"""


@pytest.fixture(scope="module")
def profiled():
    """name/mode -> the restated kernels the profiler saw in one eval forward and one training step, every row and
    precision read in one fresh interpreter, so that nothing earlier tests did to this process's profiling state plays
    a part."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    run = subprocess.run([sys.executable, "-c", _PROFILE_SCRIPT, json.dumps(NAMES)], cwd=root, capture_output=True,
                         text=True, timeout=1200)
    assert run.returncode == 0, run.stderr[-3000:]
    return json.loads(run.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("mode", ["fp32", "tf32", "bf16"])
@pytest.mark.parametrize("name", NAMES)
def test_profiled_kernels_are_the_restated_dispatch(name, mode, profiled):
    got = profiled[f"{name}/{mode}"]
    print(f"{name} {mode}: {got['short']} of 6 captures short")
    for walk in ("eval", "train"):
        seen = Counter(got[walk])
        print(f"{name} {mode} {walk}:", dict(sorted(seen.items())))
        assert seen == expected_kernels(name, mode, walk), (walk, seen - expected_kernels(name, mode, walk),
                                                            expected_kernels(name, mode, walk) - seen)


# ------------------------------------------------------------------------------------------------------------ bf16
@pytest.mark.parametrize("name", NAMES)
def test_bf16_forward(name, forwards, oracle):
    """Covered rows: the bars of test_bf16_model_forward_tolerance.  Other rows warn once and run the TF32 kernels."""
    hp, sd, x = arch_inputs(name)
    if not bf16_covered(name):
        import vqvae_b200
        m, _, _, _ = _model(name)
        t = forwards(name, "tf32")
        with vqvae_b200.precision("bf16"), torch.no_grad(), warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            _, x1, _ = m(t["x"])
            _, x2, _ = m(t["x"])
        assert len([i for i in w if "no bf16 kernels" in str(i.message)]) == 1
        assert np.array_equal(x1.cpu().numpy(), t["x_hat"]) and np.array_equal(x2.cpu().numpy(), t["x_hat"])
        return
    B, H2, W2 = _latent(name)
    E = sd[CODEBOOK]
    f = forwards(name, "bf16")
    o = oracle(name)
    z_ref = np.ascontiguousarray(o["z_e"].transpose(0, 2, 3, 1)).reshape(f["z"].shape)
    err_z = float(np.abs(f["z"] - z_ref).max())
    assert err_z <= 2.5e-3, err_z
    v = cref.vq_rows(f["z"], E)
    assert np.array_equal(f["idx"], v["idx"])
    xh_ref = cref.decoder(_nchw(v["zq"], B, H2, W2), sd, hp["n_res_layers"])
    err_x = float(np.abs(f["x_hat"] - xh_ref).max())
    assert err_x <= 3e-3, err_x
    print(f"{name} bf16: z_e {err_z:.1e}, x_hat {err_x:.1e}, flips vs oracle {int((f['idx'] != o['idx'].ravel()).sum())}")


# --------------------------------------------------------------------------------------------------- training step
def _gpu_step(name, mode, steps=1):
    """`steps` eager training steps in `mode` from the same weights -> (gradients of the last by parameter name and
    "image", every step's gradients, the codes, the ReLU masks the backward read (None in bf16 mode), the model)."""
    import vqvae_b200
    from vqvae_b200._lib import PRECISIONS
    m, hp, sd, x = _model(name, train=True)
    n = hp["n_res_layers"]
    xc = _cuda(x)
    masks = None
    with vqvae_b200.precision(mode):
        if mode != "bf16":
            acts = {}
            m._walk(xc, False, acts)
            if n:
                layers = dict(enc=m.encoder.conv_stack[5].stack[0], dec=m.decoder.inverse_conv_stack[1].stack[0])
                stack = lambda side, r0, out: stack_masks(layers[side], r0, out, n,  # noqa: E731
                                                          precision=PRECISIONS[mode])
            else:
                stack = lambda side, r0, out: [out > 0]  # noqa: E731
            masks = model_masks(acts["enc"], acts["dec"], stack)
        runs = []
        for _ in range(steps):
            xg = xc.clone().requires_grad_()
            m.zero_grad(set_to_none=True)
            with torch.enable_grad():
                emb, x_hat, _ = m(xg)
                (torch.mean((x_hat - xg) ** 2) / VAR + emb).backward()
            got = {k: p.grad.clone() for k, p in m.named_parameters()}
            got["image"] = xg.grad.clone()
            runs.append(got)
    return runs[-1], runs, m.last_min_encoding_indices.view(-1).clone(), masks, m


def _fp64(name, idx, masks):
    hp, sd, x = arch_inputs(name)
    relu, done = masked_relu(nchw64(masks))
    with torch.enable_grad():
        p = leaf_params({k: sd[k] for k in sd if ".stack." not in k or ".stack.0." in k}, torch.float64)
        xt = torch.from_numpy(x).double().requires_grad_()
        emb, x_hat = vqvae64(xt, p, hp["n_res_layers"], relu, idx.cpu())
        train_loss(xt, x_hat, emb, VAR)[0].backward()
    assert done()
    want = {k: v.grad for k, v in p.items()}
    want["image"] = xt.grad
    return want


@pytest.fixture(scope="module")
def steps():
    cache = {}

    def get(name, mode):
        if (name, mode) not in cache:
            got, runs, idx, masks, m = _gpu_step(name, mode, steps=2 if mode == "tf32" else 1)
            cache[(name, mode)] = (got, runs, idx, None if masks is None else _fp64(name, idx, masks), m)
        return cache[(name, mode)]
    return get


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
@pytest.mark.parametrize("name", NAMES)
def test_training_step_matches_fp64_at_the_gpu_masks(name, mode, steps):
    got, runs, idx, want, _ = steps(name, mode)
    assert set(got) == set(want)
    per = {k: float((got[k].double().cpu() - want[k]).abs().max() / want[k].abs().max().clamp_min(1e-30))
           for k in want}
    worst = max(per, key=per.get)
    print(f"{name} {mode}: worst {worst} {per[worst]:.1e};",
          " ".join(f"{k}={v:.1e}" for k, v in sorted(per.items(), key=lambda kv: -kv[1])[:4]))
    bar = 1e-4 if mode == "fp32" else TF32_BAR[name]
    for k, v in per.items():
        assert v <= bar, (k, v, bar)
    if mode == "tf32":                          # two eager steps: bitwise-equal conv gradients
        for k in got:
            if k != CODEBOOK:
                assert torch.equal(runs[0][k], runs[1][k]), k
    if mode == "fp32" and name in GOLDEN_ARCHS:
        g = load_golden("arch_" + name)
        if np.array_equal(idx.cpu().numpy(), g["idx"].ravel()):
            keys = list(arch_inputs(name)[1])
            for k, v in got.items():
                if k != "image":
                    v = v.double().cpu().numpy()
                    np.testing.assert_allclose(fingerprint(v, keys.index(k)), g["grad/" + k], rtol=0, err_msg=k,
                                               atol=1e-4 * np.abs(v).max() * np.sqrt(v.size))


@pytest.mark.parametrize("name", NAMES)
def test_bf16_mode_gradients_are_the_tf32_ones(name, steps):
    tf32 = steps(name, "tf32")[0]
    bf16 = steps(name, "bf16")[0]
    assert set(bf16) == set(tf32)
    for k in tf32:
        if k != CODEBOOK:
            assert torch.equal(bf16[k], tf32[k]), k


@pytest.mark.parametrize("name", NAMES)
def test_adam_step_refreshes_every_packing(name, steps):
    """After one vqvae_b200.optim.Adam step on the TF32 gradients, the next TF32 forward is bitwise that of a fresh
    model loaded with the stepped weights: every packing the forward and the backward read was refreshed."""
    import vqvae_b200
    from vqvae_b200.optim import Adam
    got, _, _, _, m = steps(name, "tf32")
    x = _cuda(arch_inputs(name)[2])
    for k, p in m.named_parameters():
        p.grad = got[k].clone()
    Adam(m.parameters(), lr=1e-2).step()
    fresh, _, _, _ = _model(name)
    fresh.load_state_dict(m.state_dict())
    m.eval()
    with vqvae_b200.precision("tf32"), torch.no_grad():
        a = m(x)
        b = fresh(x)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    # and the next training step's gradients, whose input gradients read the backward's own packings
    grads = []
    for model in (m, fresh):
        model.train()
        xg = x.clone().requires_grad_()
        model.zero_grad(set_to_none=True)
        with vqvae_b200.precision("tf32"), torch.enable_grad():
            emb, x_hat, _ = model(xg)
            (torch.mean((x_hat - xg) ** 2) / VAR + emb).backward()
        grads.append({k: p.grad for k, p in model.named_parameters()} | {"image": xg.grad})
    for k in grads[0]:
        if k != CODEBOOK:
            assert torch.equal(grads[0][k], grads[1][k]), k

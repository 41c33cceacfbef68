"""Training through the sub-modules on the H100: the notebook's piecewise walk under main.py's loss against the
reference's goldens, fp64 autograd and the fused training step; every VQ-VAE module alone in the fp32, TF32 and bf16
modes; the in-place ReLU's autograd semantics (Q2); GatedMaskedConv2d and GatedActivation against fp64 over the layer
grid; and the invariants (bitwise inference outputs, unchanged eval / no_grad launches, deterministic backward, CUDA
graph capture, the rejections)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import torch_port
from oracle.make_golden import MODEL_CASES
from oracle.piecewise_port import PRIOR_LAYER_KEYS, gate, gated_layer, residual_layer, residual_stack
from oracle.prior_train_port import fingerprint, leaf_params
from oracle.vqvae_train_port import train_loss, vqvae_train_forward
from oracle.weights import make_images, make_state_dict
from tests.vqvae_masked import dec64, enc64, masked_relu, nchw64, res64, stack_masks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HP = ("h_dim", "res_h_dim", "n_res_layers", "n_embeddings", "embedding_dim")
VAR = 0.0625
MAIN_PY = dict(h_dim=128, res_h_dim=32, n_res_layers=2, n_embeddings=512, embedding_dim=64, wseed=0, batch=32,
               size=32, xseed=7)


def _golden(name):
    with np.load(os.path.join(ROOT, "tests", "golden", name + ".npz")) as d:
        return {k: d[k] for k in d.files}


def _setup(name):
    from models.vqvae import VQVAE
    c = MAIN_PY if name == "main_py" else MODEL_CASES[name]
    sd = make_state_dict(seed=c["wseed"], **{k: c[k] for k in HP},
                         **({} if name == "main_py" else dict(codebook=c["codebook"],
                                                              codebook_scale=c["codebook_scale"])))
    m = VQVAE(*(c[k] for k in HP), 0.25)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    return c, sd, m.cuda().train(), torch.from_numpy(make_images(c["batch"], c["size"], c["xseed"]))


def _rel(got, want):
    return float((got.detach().double().cpu() - want).abs().max() / want.abs().max().clamp_min(1e-30))


def _grads(m):
    return {k: p.grad.clone() for k, p in m.named_parameters()}


def _walk(m, xc):
    """The notebook's piecewise forward (reconstruct / encode_data) under main.py's loss; gradients in .grad."""
    m.zero_grad(set_to_none=True)
    with torch.enable_grad():
        z_e = m.pre_quantization_conv(m.encoder(xc))
        embedding_loss, z_q, _, _, idx = m.vector_quantization(z_e)
        x_hat = m.decoder(z_q)
        loss = torch.mean((x_hat - xc) ** 2) / VAR + embedding_loss
        loss.backward()
    return idx


def _fp64(c, sd, x, idx):
    with torch.enable_grad():
        g = leaf_params({k: sd[k] for k in sd if ".stack." not in k or ".stack.0." in k}, torch.float64)
        emb, x_hat, _, _ = vqvae_train_forward(x.double(), g, c["n_res_layers"], idx=idx.cpu().reshape(-1))
        train_loss(x.double(), x_hat, emb, VAR)[0].backward()
    return {k: v.grad for k, v in g.items()}


@pytest.mark.parametrize("name", ["small_odd", "cifar_default", "main_py"])
def test_notebook_walk_trains_every_parameter(name):
    import vqvae_b200
    c, sd, m, x = _setup(name)
    xc = x.cuda()
    with vqvae_b200.precision("fp32"):
        idx = _walk(m, xc)
        got = _grads(m)
        m.zero_grad(set_to_none=True)
        with torch.enable_grad():
            embedding_loss, x_hat, _ = m(xc)
            (torch.mean((x_hat - xc) ** 2) / VAR + embedding_loss).backward()
        fused, fused_idx = _grads(m), m.last_min_encoding_indices
    assert all(g is not None and g.shape == p.shape for g, p in zip(got.values(), m.parameters()))
    assert torch.equal(idx, fused_idx)
    keys = list(sd)
    if name != "main_py":
        want = _golden("vqvae_grad_" + name)
        assert np.array_equal(idx.cpu().numpy().ravel(), want["idx"])
        for k, g in got.items():
            g, w = g.double().cpu().numpy(), want["grad/" + k]
            if w.shape == g.shape:
                np.testing.assert_allclose(g, w, atol=1e-4 * np.abs(w).max(), rtol=0, err_msg=k)
            else:
                np.testing.assert_allclose(fingerprint(g, keys.index(k)), w, rtol=0, err_msg=k,
                                           atol=1e-4 * np.abs(g).max() * np.sqrt(g.size))
    want64 = _fp64(c, sd, x, idx)
    conv = {k: _rel(got[k], want64[k]) for k in want64 if "embedding" not in k}
    vs_fused = max(_rel(got[k], fused[k].double().cpu()) for k in got)
    print(f"{name} walk fp32: worst conv rel {max(conv.values()):.2e}, codebook rel "
          f"{_rel(got['vector_quantization.embedding.weight'], want64['vector_quantization.embedding.weight']):.2e}, "
          f"vs fused {vs_fused:.2e}")
    assert max(conv.values()) <= 1e-5
    assert vs_fused <= 1e-5


def _module_cases(m, B, H, W):
    """(name, module, input shape, fp64 function of (input, params dict)) for every VQ-VAE module alone, on H x W
    images (H / 4 x W / 4 latents)."""
    e, d = "encoder.conv_stack.", "decoder.inverse_conv_stack."
    n = m.encoder.conv_stack[5].n_res_layers
    pq = m.pre_quantization_conv
    h, emb = pq.in_channels, pq.out_channels
    lat = (H // 4, W // 4)
    return [
        ("encoder", m.encoder, (B, 3, H, W), lambda x, p: torch_port.encoder(x, p, n, p=e)),
        ("decoder", m.decoder, (B, emb) + lat, lambda x, p: torch_port.decoder(x, p, n, p=d)),
        ("pre_quantization_conv", pq, (B, h) + lat,
         lambda x, p: F.conv2d(x, p["pre_quantization_conv.weight"], p["pre_quantization_conv.bias"])),
        ("residual_layer", m.encoder.conv_stack[5].stack[0], (B, h) + lat,
         lambda x, p: residual_layer(x, p[e + "5.stack.0.res_block.1.weight"], p[e + "5.stack.0.res_block.3.weight"])),
        ("residual_stack", m.decoder.inverse_conv_stack[1], (B, h) + lat,
         lambda x, p: residual_stack(x, [(p[d + "1.stack.0.res_block.1.weight"],
                                          p[d + "1.stack.0.res_block.3.weight"])] * n)),
    ]


def _module_prefix(m, mod):
    return next(k for k, v in m.named_modules() if v is mod)


def _run_module(mod, x, G):
    """Output and gradients (input first, then parameters by name) of one differentiable call."""
    for p in mod.parameters():
        p.grad = None
    xi = x.clone().requires_grad_()
    with torch.enable_grad():
        y = mod(xi * 1)
        y.backward(G)
    return y.detach(), dict(input=xi.grad, **{k: p.grad for k, p in mod.named_parameters()})


def _module_fp64(m, sd, fn, mod, x, G):
    with torch.enable_grad():
        p = leaf_params({k: sd[k] for k in sd if ".stack." not in k or ".stack.0." in k}, torch.float64)
        x64 = x.cpu().double().requires_grad_()
        (fn(x64 * 1, p) * G.cpu().double()).sum().backward()
    pre = _module_prefix(m, mod)
    out = dict(input=x64.grad)
    for k, _ in mod.named_parameters():
        key = pre + "." + k
        if key not in p:                             # a shared residual layer's weight: stored under stack.0
            key = key.replace(".stack.1.", ".stack.0.").replace(".stack.2.", ".stack.0.")
        out[k] = p[key].grad
    return out


# 32 x 32: every latent image inside one 128-pixel tile.  64 x 64: 16 x 16 latents, two tiles per image.  48 x 80:
# 12 x 20 latents, ragged tiles on both axes and H != W in every call.
IMAGE_SIZES = [(32, 32), (64, 64), (48, 80)]


def test_every_vqvae_module_alone_matches_fp64_in_every_mode():
    import vqvae_b200
    c, sd, m, _ = _setup("cifar_default")
    B = 4
    gen = torch.Generator().manual_seed(5)
    report = {}
    for (H, W), (name, mod, shape, fn) in [(hw, case) for hw in IMAGE_SIZES for case in _module_cases(m, B, *hw)]:
        name = f"{name} {H}x{W}"
        x = torch.randn(shape, generator=gen).cuda()
        with torch.no_grad():
            mod.eval()
            ref_out = mod(x.clone())
            mod.train()
        G = torch.randn(ref_out.shape, generator=gen).cuda()
        want = _module_fp64(m, sd, fn, mod, x, G)
        got = {}
        for mode in ("fp32", "tf32", "bf16"):
            with vqvae_b200.precision(mode):
                out, got[mode] = _run_module(mod, x, G)
            if mode != "bf16":
                with torch.no_grad(), vqvae_b200.precision(mode):
                    mod.eval()
                    inf = mod(x.clone())
                    mod.train()
                assert torch.equal(out, inf), (name, mode)            # the differentiable output is the inference one
        assert all(torch.equal(got["bf16"][k], got["tf32"][k]) for k in got["tf32"]), name
        for mode in ("fp32", "tf32"):
            report[(name, mode)] = {k: _rel(got[mode][k], want[k]) for k in want}
    for (name, mode), per in report.items():
        print(f"{name} {mode}:", " ".join(f"{k}={v:.1e}" for k, v in per.items()))
    # TF32 against an fp64 forward is printed only: its ReLU masks differ from the GPU's (up to 0.24 of max |g|,
    # DESIGN.md §10); test_tf32_modules_match_fp64_at_the_gpu_masks bounds the TF32 mode at the GPU's own masks.
    for (name, mode), per in report.items():
        if mode == "fp32":
            assert max(per.values()) <= 1e-5, (name, per)


def test_tf32_modules_match_fp64_at_the_gpu_masks():
    """Each VQ-VAE module alone in TF32 mode against fp64 autograd of the restatement whose ReLU masks are the ones
    the GPU's forward produced (the masks its backward reads): the TF32 error of the backward's own arithmetic, without
    the mask flips between a TF32 and an fp64 forward."""
    import vqvae_b200
    from vqvae_b200 import ops
    c, sd, m, _ = _setup("cifar_default")
    B, n = 4, m.encoder.conv_stack[5].n_res_layers
    gen = torch.Generator().manual_seed(12)
    report = {}
    for (H, W), (name, mod, shape, _) in [(hw, case) for hw in IMAGE_SIZES for case in _module_cases(m, B, *hw)]:
        x = torch.randn(shape, generator=gen).cuda()
        with vqvae_b200.precision("tf32"):
            with torch.no_grad():
                mod.eval()
                G = torch.randn(mod(x.clone()).shape, generator=gen).cuda()
                mod.train()
                if name == "encoder":
                    acts = {}
                    mod._forward_nhwc(x, False, acts)
                    a1, a2, a3, e_out = acts["enc"]
                    masks = [a1 > 0, a2 > 0] + stack_masks(mod.conv_stack[5].stack[0], a3, e_out, n)
                    fn = lambda t, p, relu: enc64(t, p, n, relu)                                   # noqa: E731
                elif name == "decoder":
                    acts = {}
                    mod._forward_from_nhwc(ops.nchw_to_nhwc(x), B, H // 4, W // 4, acts=acts)
                    d1, d_out, d2 = acts["dec"]
                    masks = stack_masks(mod.inverse_conv_stack[1].stack[0], d1, d_out, n) + [d2 > 0]
                    fn = lambda t, p, relu: dec64(t, p, n, relu)                                   # noqa: E731
                elif name == "pre_quantization_conv":
                    masks = []
                    fn = lambda t, p, relu: F.conv2d(t, p["pre_quantization_conv.weight"],        # noqa: E731
                                                     p["pre_quantization_conv.bias"])
                else:
                    layer = mod if name == "residual_layer" else mod.stack[0]
                    pre = _module_prefix(m, layer) + ".res_block."
                    out = ops.nchw_to_nhwc(mod(x.clone()))
                    masks = stack_masks(layer, ops.nchw_to_nhwc(torch.relu(x)), out, 1 if name == "residual_layer"
                                        else n, relu_out=name != "residual_layer")
                    k = 1 if name == "residual_layer" else n
                    fn = lambda t, p, relu, pre=pre, k=k, f=name != "residual_layer": res64(      # noqa: E731
                        t, p[pre + "1.weight"], p[pre + "3.weight"], k, relu, f)
            _, got = _run_module(mod, x, G)
        relu, done = masked_relu(nchw64(masks))                    # every mask is NHWC
        fn64 = lambda t, p: fn(t, p, relu)                                                          # noqa: E731
        want = _module_fp64(m, sd, fn64, mod, x, G)
        assert done(), (name, H, W)                                 # every mask used once
        report[(name, H, W)] = per = {k: _rel(got[k], want[k]) for k in want}
        print(f"{name} {H}x{W} tf32 at the GPU's masks:", " ".join(f"{k}={v:.1e}" for k, v in per.items()))
    for name, per in report.items():
        assert per["input"] <= 5e-3, (name, per)
        assert max(per.values()) <= 1e-2, (name, per)


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_residual_stacks_with_distinct_layers_and_none(mode):
    import vqvae_b200
    from models.residual import ResidualLayer, ResidualStack
    torch.manual_seed(3)
    C, Cmid, B, S = 64, 32, 3, 8
    st = ResidualStack(C, C, Cmid, 3).cuda().train()
    st.stack = torch.nn.ModuleList([ResidualLayer(C, C, Cmid) for _ in range(3)]).cuda()
    empty = ResidualStack(C, C, Cmid, 0).cuda().train()
    x = torch.randn((B, C, S, S), device="cuda")
    G = torch.randn((B, C, S, S), device="cuda")
    with vqvae_b200.precision(mode):
        _, got = _run_module(st, x, G)
        _, got0 = _run_module(empty, x, G)
    with torch.enable_grad():
        ws = [(l.res_block[1].weight.detach().cpu().double().requires_grad_(),
               l.res_block[3].weight.detach().cpu().double().requires_grad_()) for l in st.stack]
        x64 = x.cpu().double().requires_grad_()
        (residual_stack(x64 * 1, ws) * G.cpu().double()).sum().backward()
    per = {"input": _rel(got["input"], x64.grad)}
    for i, (w1, w2) in enumerate(ws):
        per[f"{i}.1"] = _rel(got[f"stack.{i}.res_block.1.weight"], w1.grad)
        per[f"{i}.3"] = _rel(got[f"stack.{i}.res_block.3.weight"], w2.grad)
    print(f"distinct layers {mode}:", " ".join(f"{k}={v:.1e}" for k, v in per.items()))
    assert max(per.values()) <= (1e-5 if mode == "fp32" else 0.3)       # TF32: measured 0.23, see above
    assert torch.equal(got0["input"], G * (x > 0))


def test_in_place_relu_semantics():
    from models.residual import ResidualLayer
    torch.manual_seed(4)
    layer = ResidualLayer(32, 32, 8).cuda().train()
    x0 = torch.randn((2, 32, 5, 5), device="cuda", requires_grad=True)
    G = torch.randn((2, 32, 5, 5), device="cuda")
    with torch.enable_grad():
        x = x0 * 1
        before, v0 = x.detach().clone(), x._version
        y = layer(x)
        assert torch.equal(x.detach(), torch.relu(before)) and x._version != v0
        y.backward(G)
        with torch.no_grad():
            layer.eval()
            assert torch.equal(y.detach(), layer(before.clone()))
            layer.train()
    w1, w2 = (layer.res_block[i].weight.detach().cpu().double().requires_grad_() for i in (1, 3))
    with torch.enable_grad():
        x64 = before.cpu().double().requires_grad_()
        (residual_layer(x64, w1, w2) * G.cpu().double()).sum().backward()
    assert _rel(x0.grad, x64.grad) <= 1e-5
    with torch.enable_grad(), pytest.raises(RuntimeError, match="leaf Variable that requires grad"):
        layer(x0)
    with torch.enable_grad():
        xs = x0 * 1
        st_out = layer(xs)
        xs.mul_(2)                         # the caller changes the ReLU'd tensor before the backward
        with pytest.raises(RuntimeError, match="modified by an inplace operation"):
            st_out.sum().backward()


def _gated(mask, kernel, residual, dim, size, seed):
    from pixelcnn.models import GatedMaskedConv2d
    torch.manual_seed(seed)
    layer = GatedMaskedConv2d(mask, dim, kernel, residual, n_classes=5).cuda()
    x_v = torch.randn((2, dim, size, size), device="cuda")
    x_h = torch.randn((2, dim, size, size), device="cuda")
    return layer, x_v, x_h, torch.tensor([4, 1], device="cuda")


def _gated_check(layer, x_v, x_h, h, mask, kernel, residual, with_v=True):
    gen = torch.Generator().manual_seed(kernel)
    Gv, Gh = (torch.randn(x_v.shape, generator=gen).cuda() for _ in range(2))
    with torch.no_grad():
        ref_v, ref_h = layer(x_v, x_h, h)
    xv, xh = x_v.clone().requires_grad_(), x_h.clone().requires_grad_()
    layer.zero_grad(set_to_none=True)
    with torch.enable_grad():
        out_v, out_h = layer(xv, xh, h)
        assert torch.equal(out_v.detach(), ref_v) and torch.equal(out_h.detach(), ref_h)
        loss = (out_h * Gh).sum() + ((out_v * Gv).sum() if with_v else 0)
        loss.backward()
    with torch.enable_grad():
        p = {k: v.detach().cpu().double().requires_grad_() for k, v in layer.named_parameters()}
        v64, h64 = x_v.cpu().double().requires_grad_(), x_h.cpu().double().requires_grad_()
        o_v, o_h = gated_layer(p, v64, h64, h.cpu(), mask, kernel, residual)
        ((o_h * Gh.cpu().double()).sum() + ((o_v * Gv.cpu().double()).sum() if with_v else 0)).backward()
    per = {"x_v": _rel(xv.grad, v64.grad), "x_h": _rel(xh.grad, h64.grad)}
    per.update({k: _rel(t.grad, p[k].grad) for k, t in layer.named_parameters() if p[k].grad.abs().max() > 0})
    assert set(dict(layer.named_parameters())) == set(PRIOR_LAYER_KEYS)
    return per


@pytest.mark.parametrize("size", [1, 7])
@pytest.mark.parametrize("dim", [32, 160, 256])
@pytest.mark.parametrize("residual", [True, False])
@pytest.mark.parametrize("kernel", [1, 3, 5, 15])
@pytest.mark.parametrize("mask", ["A", "B"])
def test_gated_layer_gradients_match_fp64(mask, kernel, residual, dim, size):
    layer, x_v, x_h, h = _gated(mask, kernel, residual, dim, size, 1000 * kernel + dim + size + (mask == "A"))
    per = _gated_check(layer, x_v, x_h, h, mask, kernel, residual)
    assert max(per.values()) <= 2e-5, per


@pytest.mark.parametrize("mask,kernel,residual", [("A", 7, False), ("B", 3, True)])
def test_gated_layer_without_a_vertical_gradient(mask, kernel, residual):
    layer, x_v, x_h, h = _gated(mask, kernel, residual, 64, 6, 7)
    per = _gated_check(layer, x_v, x_h, h, mask, kernel, residual, with_v=False)
    assert max(per.values()) <= 2e-5, per


def test_gated_activation_matches_fp64():
    from pixelcnn.models import GatedActivation
    torch.manual_seed(8)
    x = (torch.randn((3, 64, 7, 7), device="cuda") * 2).requires_grad_()
    G = torch.randn((3, 32, 7, 7), device="cuda")
    with torch.enable_grad():
        y = GatedActivation()(x)
        y.backward(G)
    with torch.no_grad():
        assert torch.equal(y.detach(), GatedActivation()(x))
    with torch.enable_grad():
        x64 = x.detach().cpu().double().requires_grad_()
        (gate(x64) * G.cpu().double()).sum().backward()
    worst = _rel(x.grad, x64.grad)
    print(f"GatedActivation: rel {worst:.2e}")
    assert worst <= 1e-6


def test_prior_stack_walked_module_by_module_matches_fp64():
    from oracle.prior_port import PRIOR_CASES, make_prior_inputs, make_prior_state_dict
    from pixelcnn.models import GatedPixelCNN
    c = PRIOR_CASES["prior_default"]
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"])
    m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    m = m.cuda()
    codes, labels, _ = make_prior_inputs(c)
    x, lab = torch.from_numpy(codes).cuda(), torch.from_numpy(labels).cuda()
    G = torch.randn((c["batch"], c["dim"], c["size"], c["size"]), generator=torch.Generator().manual_seed(2))
    with torch.enable_grad():
        x_v = x_h = m.embedding(x).permute(0, 3, 1, 2)
        for layer in m.layers:
            x_v, x_h = layer(x_v, x_h, lab)
        (x_h * G.cuda()).sum().backward()
    with torch.enable_grad():
        p = leaf_params(sd, torch.float64)
        xv = xh = F.embedding(x.cpu(), p["embedding.weight"]).permute(0, 3, 1, 2)
        for i, layer in enumerate(m.layers):
            pl = {k: p[f"layers.{i}.{k}"] for k in PRIOR_LAYER_KEYS}
            xv, xh = gated_layer(pl, xv, xh, lab.cpu(), layer.mask_type, layer.vert_stack.kernel_size[1],
                                 layer.residual)
        (xh * G.double()).sum().backward()
    per = {k: _rel(t.grad, p[k].grad) for k, t in m.named_parameters() if t.grad is not None}
    assert len(per) == 1 + 9 * c["n_layers"]
    print("prior stack walk: worst", max(per.items(), key=lambda kv: kv[1]))
    assert max(per.values()) <= 1e-4


def test_eval_and_no_grad_calls_keep_their_launches():
    """An eval-mode call with grad enabled is the no_grad inference call: same launches, same outputs, no graph.  The
    prior modules' inference calls keep their launch counts: two layouts in, two kernels, two layouts out; one gate."""
    from pixelcnn.models import GatedActivation
    from vqvae_b200 import ops
    c, sd, m, x = _setup("cifar_default")

    def count(mod, *args):
        n0 = ops.launch_count()
        out = mod(*[a.clone() for a in args])
        return ops.launch_count() - n0, out

    for name, mod, shape, _ in _module_cases(m, 4, 32, 32):
        xi = torch.randn(shape, device="cuda")
        with torch.no_grad():
            count(mod, xi)                       # packs the weights
            ref_n, ref = count(mod, xi)
        mod.eval()
        with torch.enable_grad():
            n, out = count(mod, xi)
        mod.train()
        assert n == ref_n and not out.requires_grad and torch.equal(out, ref), name
    layer, x_v, x_h, h = _gated("B", 3, True, 64, 6, 9)
    with torch.no_grad():
        count(layer, x_v, x_h, h)
        assert count(layer, x_v, x_h, h)[0] == 6
        assert count(GatedActivation(), torch.randn((2, 64, 5, 5), device="cuda"))[0] == 1


def test_piecewise_backward_is_deterministic_and_captures_in_a_cuda_graph():
    c, sd, m, x = _setup("cifar_default")
    xc = x.cuda()
    runs = []
    for _ in range(2):
        _walk(m, xc)
        runs.append(_grads(m))
    emb = "vector_quantization.embedding.weight"
    assert all(torch.equal(runs[0][k], runs[1][k]) for k in runs[0] if k != emb)

    G = torch.randn(xc.shape, generator=torch.Generator().manual_seed(6)).cuda()

    def step():
        m.zero_grad(set_to_none=True)
        with torch.enable_grad():
            (m.decoder(m.pre_quantization_conv(m.encoder(xc))) * G).sum().backward()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
        step()
    torch.cuda.current_stream().wait_stream(s)
    eager = {k: p.grad.clone() for k, p in m.named_parameters() if k != emb}
    m.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph), torch.enable_grad():
        (m.decoder(m.pre_quantization_conv(m.encoder(xc))) * G).sum().backward()
    for k, p in m.named_parameters():
        if k != emb:
            p.grad.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(p.grad, eager[k]) for k, p in m.named_parameters() if k != emb)


def test_rejections():
    c, sd, m, x = _setup("small_odd")
    xc = x.cuda()
    layer, x_v, x_h, h = _gated("A", 7, False, 32, 5, 10)
    with torch.enable_grad():
        z = torch.randn((2, m.vector_quantization.e_dim, 4, 4), device="cuda", requires_grad=True)
        for fwd in (lambda: m.encoder(xc), lambda: m.decoder(z), lambda: m.pre_quantization_conv(m.encoder(xc)),
                    lambda: m.encoder.conv_stack[5](z.new_ones(()) * m.encoder(xc)), lambda: layer(x_v, x_h, h)[1]):
            y = fwd()
            y.sum().backward(retain_graph=True)
            with pytest.raises(RuntimeError, match="twice"):
                y.sum().backward()
        y = m.decoder(m.pre_quantization_conv(m.encoder(xc)))
        with torch.no_grad():
            m.decoder.inverse_conv_stack[4].weight.mul_(2)
        with pytest.raises(RuntimeError, match="modified by an inplace operation"):
            y.sum().backward()
        y = layer(x_v, x_h, h)[1]
        with torch.no_grad():
            layer.horiz_resid.weight.mul_(2)
        with pytest.raises(RuntimeError, match="modified by an inplace operation"):
            y.sum().backward()


@pytest.mark.parametrize("mode", ["fp32", "tf32"])
def test_launch_counts_per_module(mode):
    """Library launches of each differentiable call, forward and backward (DESIGN.md).  The forward of a non-empty
    module is its inference call's launches; an empty stack is one ReLU."""
    import vqvae_b200
    from models.residual import ResidualStack
    from pixelcnn.models import GatedActivation
    from vqvae_b200 import ops
    c, sd, m, x = _setup("cifar_default")
    layer, x_v, x_h, h = _gated("B", 3, True, 64, 6, 11)
    cases = [(name, mod, (torch.randn(shape, device="cuda"),)) for name, mod, shape, _ in _module_cases(m, 4, 32, 32)]
    cases += [("empty_stack", ResidualStack(128, 128, 32, 0).cuda().train(), (torch.randn((4, 128, 8, 8), device="cuda"),)),
              ("gated_layer", layer, (x_v, x_h, h)),
              ("gated_activation", GatedActivation(), (torch.randn((2, 64, 6, 6), device="cuda"),))]
    counts = {}
    with vqvae_b200.precision(mode):
        for name, mod, args in cases:
            with torch.no_grad():
                mod(*[a.clone() for a in args])                      # packs the weights
                n0 = ops.launch_count()
                mod(*[a.clone() for a in args])
                inf = ops.launch_count() - n0
            ins = [a.clone().requires_grad_() if a.is_floating_point() else a for a in args]
            with torch.enable_grad():
                y = mod(*[a * 1 if a.is_floating_point() else a for a in ins])
                y = y[1] if isinstance(y, tuple) else y
                n0 = ops.launch_count()
                y.sum().backward()
                bwd = ops.launch_count() - n0
            with torch.enable_grad():
                n0 = ops.launch_count()
                mod(*[a * 1 if a.is_floating_point() else a for a in ins])
                fwd = ops.launch_count() - n0
            counts[name] = (inf, fwd, bwd)
            if name != "empty_stack":
                assert fwd == inf, (name, inf, fwd)
    print(f"launches {mode} (inference, differentiable forward, backward):",
          " ".join(f"{k}={v}" for k, v in counts.items()))
    want = {"fp32": dict(encoder=(8, 8, 37), decoder=(11, 11, 34), pre_quantization_conv=(1, 1, 4),
                         residual_layer=(5, 5, 11), residual_stack=(7, 7, 18), empty_stack=(3, 1, 1),
                         gated_layer=(6, 6, 13), gated_activation=(1, 1, 1)),
            "tf32": dict(encoder=(5, 5, 33), decoder=(5, 5, 33), pre_quantization_conv=(1, 1, 4),
                         residual_layer=(4, 4, 11), residual_stack=(4, 4, 17), empty_stack=(3, 1, 1),
                         gated_layer=(6, 6, 13), gated_activation=(1, 1, 1))}[mode]
    assert counts == want                                   # the table of DESIGN.md §10


def test_encoder_training_needs_sides_divisible_by_4_and_decoder_skips_an_unneeded_input_gradient():
    from vqvae_b200 import ops
    c, sd, m, x = _setup("cifar_default")
    x30 = torch.randn((2, 3, 30, 30), device="cuda")
    n0 = ops.launch_count()
    with torch.enable_grad(), pytest.raises(RuntimeError, match="divisible by 4"):
        m.encoder(x30)
    assert ops.launch_count() == n0
    with torch.no_grad():
        assert m.encoder(x30).shape == (2, 128, 7, 7)        # the inference call takes any size
    z = torch.randn((2, 64, 8, 8), device="cuda")
    with torch.enable_grad():
        m.decoder(z.clone().requires_grad_()).sum().backward()     # builds the input-gradient weight packings
    counts = []
    for needs in (True, False):
        zi = z.clone().requires_grad_(needs)
        with torch.enable_grad():
            y = m.decoder(zi)
            n0 = ops.launch_count()
            y.sum().backward()
            counts.append(ops.launch_count() - n0)
        assert (zi.grad is not None) == needs
    assert counts[1] == counts[0] - 1

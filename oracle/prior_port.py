"""The Gated PixelCNN prior restated functionally with torch CPU ops -- TEST INFRASTRUCTURE ONLY.

``prior_forward`` is the reference's GatedPixelCNN.forward (pixelcnn/models.py:121-130) on a state dict, op for op,
mask-A zeroing included; ``prior_generate`` its sampling loop (one full forward per position), which
tools/bench_prior.py times ("kind": "port") only when the verbatim copy of the reference (oracle/prior_ref.py) is
absent.  Pinned against the unmodified reference by tests/test_prior_cpu.py through the tests/golden/prior_*
vectors that ``python -m oracle.make_prior_golden`` writes.  The product (vqvae_b200/, models/, pixelcnn/) never
imports this module.
"""
import numpy as np
import torch
import torch.nn.functional as F

# name -> (K, dim, n_layers, n_classes, grid, batch, weight seed, input seed[, stored positions])
PRIOR_CASES = {
    "prior_default": dict(K=512, dim=64, n_layers=15, n_classes=10, size=8, batch=4, wseed=30, xseed=31),
    "prior_ragged": dict(K=37, dim=32, n_layers=4, n_classes=3, size=5, batch=3, wseed=32, xseed=33),
    # cfg3 latent (256x256 images): logits are stored at 64 seeded positions only
    "prior_cfg3": dict(K=1024, dim=64, n_layers=15, n_classes=10, size=64, batch=1, wseed=34, xseed=35,
                       positions=64),
}

A7, B3 = ["A", 7, False], ["B", 3, True]

# Cases over the documented shape range with their own layer stacks: `layers` lists (mask_type, kernel, residual)
# per layer, and the model is GatedPixelCNN(K, dim, n_layers, n_classes) with layers[i] replaced by
# GatedMaskedConv2d(mask_type, dim, kernel, residual, n_classes).  `parts` says what the GPU tests run on a case.
PRIOR_SHAPE_CASES = {
    # 2*dim = 512: both accumulators of every thread live; K = 8192: 256 codes per lane in the draw
    "wide": dict(K=8192, dim=256, n_layers=2, n_classes=10, size=6, batch=3, wseed=40, xseed=41, layers=[A7, B3]),
    # 2*dim = 320: the second accumulator partly live; K = 33: lanes 17..31 of the draw empty; 65 classes: 2 row tiles
    "mid": dict(K=33, dim=160, n_layers=3, n_classes=65, size=7, batch=5, wseed=42, xseed=43, layers=[A7, B3, B3]),
    # 2*dim = 192: ragged GEMM tiles; one class
    "narrow": dict(K=2, dim=96, n_layers=4, n_classes=1, size=4, batch=9, wseed=44, xseed=45,
                   layers=[A7, B3, B3, B3]),
    # every kernel path, mask A after layer 0 (kernel 1: no kept taps), a mask-B 15 reading 8 vertical rows of 9
    "kernels": dict(K=37, dim=32, n_layers=7, n_classes=3, size=9, batch=2, wseed=46, xseed=47,
                    layers=[["A", 15, False], ["B", 5, True], ["B", 1, True], ["A", 3, True], ["A", 1, True],
                            ["B", 15, False], B3]),
    # VQB_PRIOR_MAX_LAYERS layers
    "deep": dict(K=16, dim=32, n_layers=32, n_classes=10, size=6, batch=2, wseed=48, xseed=49,
                 layers=[A7] + [B3] * 31),
    "single": dict(K=1, dim=32, n_layers=1, n_classes=10, size=1, batch=1, wseed=50, xseed=51, layers=[A7]),
    "single3": dict(K=1, dim=32, n_layers=1, n_classes=10, size=3, batch=1, wseed=52, xseed=53, layers=[A7]),
    # 4608 positions: weight gradients over many chunks; 48 sampler rows
    "long": dict(K=512, dim=32, n_layers=2, n_classes=10, size=48, batch=2, wseed=54, xseed=55, layers=[A7, B3]),
    # residual on layer 0 (teacher-forced only: the sampler refuses it)
    "resid0": dict(K=37, dim=32, n_layers=2, n_classes=3, size=5, batch=2, wseed=56, xseed=57,
                   layers=[["A", 5, True], B3], parts=["forward", "backward"]),
    # 2523 positions, not a multiple of 32: every weight gradient in 5 to 79 position chunks, the last one ragged (27
    # to 475 positions) and ending in a short k-step; K = 300: three 128-wide N tiles of logits, the last 44 wide,
    # and a 300-deep head dgrad ending in a short k-step
    "chunks": dict(K=300, dim=64, n_layers=3, n_classes=10, size=29, batch=3, wseed=60, xseed=61,
                   layers=[A7, B3, B3], parts=["forward", "backward"]),
    # the cfg3 latent with the reference's stack: the sampler's vertical rings over 64 rows
    "cfg3_sampler": dict(K=1024, dim=64, n_layers=15, n_classes=10, size=64, batch=2, wseed=58, xseed=59,
                         layers=[A7] + [B3] * 14, parts=["sampler"]),
}

HIDDEN = 512


def reference_layers(n_layers):
    """(mask_type, kernel, residual) of every layer of the reference's GatedPixelCNN: mask A 7x7 without residual,
    then mask B 3x3 with residual."""
    return [A7] + [B3] * (n_layers - 1)


def _stack(n_layers, layers):
    layers = reference_layers(n_layers) if layers is None else [list(l) for l in layers]
    assert len(layers) == n_layers, (len(layers), n_layers)
    return layers


def prior_shapes(K, dim, n_layers, n_classes, layers=None):
    """(key, shape) of every tensor of GatedPixelCNN(K, dim, n_layers, n_classes).state_dict(), in order, with the
    layer stack `layers` ((mask_type, kernel, residual) per layer; default the reference's)."""
    out = [("embedding.weight", (K, dim))]
    for i, (_, k, _) in enumerate(_stack(n_layers, layers)):
        p = f"layers.{i}."
        out += [(p + "class_cond_embedding.weight", (n_classes, 2 * dim)),
                (p + "vert_stack.weight", (2 * dim, dim, k // 2 + 1, k)), (p + "vert_stack.bias", (2 * dim,)),
                (p + "vert_to_horiz.weight", (2 * dim, 2 * dim, 1, 1)), (p + "vert_to_horiz.bias", (2 * dim,)),
                (p + "horiz_stack.weight", (2 * dim, dim, 1, k // 2 + 1)), (p + "horiz_stack.bias", (2 * dim,)),
                (p + "horiz_resid.weight", (dim, dim, 1, 1)), (p + "horiz_resid.bias", (dim,))]
    out += [("output_conv.0.weight", (HIDDEN, dim, 1, 1)), ("output_conv.0.bias", (HIDDEN,)),
            ("output_conv.2.weight", (K, HIDDEN, 1, 1)), ("output_conv.2.bias", (K,))]
    return out


def make_prior_state_dict(K, dim, n_layers, n_classes, seed, layers=None):
    """Seeded float32 weights: Xavier-range conv weights (mask A's taps deliberately non-zero), small random biases,
    unit-normal embeddings."""
    rng = np.random.RandomState(seed)
    sd = {}
    for key, shape in prior_shapes(K, dim, n_layers, n_classes, layers):
        if key.endswith("bias"):
            v = rng.uniform(-0.1, 0.1, size=shape)
        elif len(shape) == 4:
            fan_in, fan_out = shape[1] * shape[2] * shape[3], shape[0] * shape[2] * shape[3]
            a = np.sqrt(6.0 / (fan_in + fan_out))
            v = rng.uniform(-a, a, size=shape)
        else:
            v = rng.standard_normal(shape)
        sd[key] = v.astype(np.float32)
    return sd


def make_prior_inputs(case):
    """(codes (B,H,W) int64, labels (B,) int64[, positions (P,2)]) of a case."""
    rng = np.random.RandomState(case["xseed"])
    B, S = case["batch"], case["size"]
    codes = rng.randint(0, case["K"], size=(B, S, S)).astype(np.int64)
    labels = rng.randint(0, case["n_classes"], size=(B,)).astype(np.int64)
    pos = None
    if case.get("positions"):
        flat = rng.choice(S * S, size=case["positions"], replace=False)
        pos = np.stack([flat // S, flat % S], axis=1).astype(np.int64)
    return codes, labels, pos


def _gate(t):
    a, b = t.chunk(2, dim=1)
    return torch.tanh(a) * torch.sigmoid(b)


@torch.no_grad()
def prior_forward(sd, x, label, n_layers, dtype=torch.float32, layers=None):
    """Logits (B, K, H, W) of codes x (B,H,W) int64 and labels (B,) int64; sd maps keys to tensors or arrays;
    layers: (mask_type, kernel, residual) per layer, default the reference's stack."""
    g = {k: torch.as_tensor(v).to(dtype) for k, v in sd.items()}
    x, label = torch.as_tensor(x), torch.as_tensor(label)
    h = F.embedding(x, g["embedding.weight"]).permute(0, 3, 1, 2)
    x_v = x_h = h
    for i, (mask, k, residual) in enumerate(_stack(n_layers, layers)):
        p = f"layers.{i}."
        wv, wh = g[p + "vert_stack.weight"], g[p + "horiz_stack.weight"]
        if mask == "A":                                   # mask A (models.py:61-63)
            wv, wh = wv.clone(), wh.clone()
            wv[:, :, -1] = 0
            wh[:, :, :, -1] = 0
        c = F.embedding(label, g[p + "class_cond_embedding.weight"])[:, :, None, None]
        hv = F.conv2d(x_v, wv, g[p + "vert_stack.bias"], 1, (k // 2, k // 2))[:, :, :x_v.size(-1), :]
        out_v = _gate(hv + c)
        hh = F.conv2d(x_h, wh, g[p + "horiz_stack.bias"], 1, (0, k // 2))[:, :, :, :x_h.size(-2)]
        v2h = F.conv2d(hv, g[p + "vert_to_horiz.weight"], g[p + "vert_to_horiz.bias"])
        out = _gate(v2h + hh + c)
        r = F.conv2d(out, g[p + "horiz_resid.weight"], g[p + "horiz_resid.bias"])
        x_h = r + x_h if residual else r
        x_v = out_v
    y = F.relu(F.conv2d(x_h, g["output_conv.0.weight"], g["output_conv.0.bias"]))
    return F.conv2d(y, g["output_conv.2.weight"], g["output_conv.2.bias"])


@torch.no_grad()
def prior_generate(sd, label, shape, batch_size, n_layers, device="cpu", rows=None):
    """The reference's sampling schedule (models.py:132-143): one full forward per position, softmax, multinomial.
    `rows` limits the loop to the first rows (timing a part of a large grid)."""
    g = {k: torch.as_tensor(v).to(device) for k, v in sd.items()}
    x = torch.zeros((batch_size,) + tuple(shape), dtype=torch.int64, device=device)
    for i in range(shape[0] if rows is None else rows):
        for j in range(shape[1]):
            logits = prior_forward(g, x, label, n_layers)
            probs = F.softmax(logits[:, :, i, j], -1)
            x[:, i, j].copy_(probs.multinomial(1).squeeze())
    return x

"""The sub-modules called on their own, restated differentiably with torch ops -- TEST INFRASTRUCTURE ONLY.

``residual_layer`` / ``residual_stack`` are the reference's models/residual.py on weight tensors (Q2: the in-place
ReLU makes a layer relu(x) + f(relu(x)); the restatement takes the ReLU on a new tensor, the tests check the caller's
tensor separately).  ``gated_layer`` is pixelcnn/models.py's GatedMaskedConv2d.forward with the reference's mask-A
semantics (the masked slices zeroed in place through ``.data``, then the full weight convolved, so the masked taps
get a gradient), ``gate`` its GatedActivation.  Pinned against the unmodified reference by
tests/test_piecewise_train_cpu.py through tests/golden/piecewise_grad.npz, which ``python -m
oracle.make_piecewise_grad_golden`` writes.  The product never imports this module.
"""
import numpy as np
import torch
import torch.nn.functional as F

# residual modules: ResidualLayer(C, C, CMID) and ResidualStack(C, C, CMID, n) on a (B, C, S, S) input
RES = dict(C=32, CMID=8, B=2, S=5, seed=60, stacks=[0, 1, 3])
# gated layers: (name, mask, kernel, residual) at dim DIM, N_CLASSES classes, (B, DIM, S, S) inputs
GATED = dict(DIM=32, N_CLASSES=3, B=2, S=5, seed=61, layers=[["A7", "A", 7, False], ["B3", "B", 3, True]])
GATE = dict(B=2, C=16, S=5, seed=62)
PRIOR_LAYER_KEYS = ("class_cond_embedding.weight", "vert_stack.weight", "vert_stack.bias", "vert_to_horiz.weight",
                    "vert_to_horiz.bias", "horiz_stack.weight", "horiz_stack.bias", "horiz_resid.weight",
                    "horiz_resid.bias")


def res_inputs():
    """{"w1", "w2", "x", "g/<n>"}: the residual weights (reference layout), the input and one upstream gradient per
    case ("g/layer" for the lone layer, "g/stack<n>" for the stacks), fp32 arrays."""
    c = RES
    rng = np.random.RandomState(c["seed"])
    f = lambda *s: rng.standard_normal(s).astype(np.float32)       # noqa: E731
    out = dict(w1=f(c["CMID"], c["C"], 3, 3) * np.float32(0.2), w2=f(c["C"], c["CMID"], 1, 1) * np.float32(0.3),
               x=f(c["B"], c["C"], c["S"], c["S"]))
    for name in ["layer"] + [f"stack{n}" for n in c["stacks"]]:
        out["g/" + name] = f(c["B"], c["C"], c["S"], c["S"])
    return out


def gated_inputs(name):
    """{param key: array} of one GATED layer plus "x_v", "x_h", "label", "g_v", "g_h"."""
    c = GATED
    _, mask, k, _ = next(l for l in c["layers"] if l[0] == name)
    rng = np.random.RandomState(c["seed"] + 7 * k + (mask == "A"))
    D, half = c["DIM"], k // 2
    f = lambda *s: rng.standard_normal(s).astype(np.float32)        # noqa: E731
    shapes = {"class_cond_embedding.weight": (c["N_CLASSES"], 2 * D), "vert_stack.weight": (2 * D, D, half + 1, k),
              "vert_stack.bias": (2 * D,), "vert_to_horiz.weight": (2 * D, 2 * D, 1, 1), "vert_to_horiz.bias": (2 * D,),
              "horiz_stack.weight": (2 * D, D, 1, half + 1), "horiz_stack.bias": (2 * D,),
              "horiz_resid.weight": (D, D, 1, 1), "horiz_resid.bias": (D,)}
    out = {key: f(*shapes[key]) * np.float32(0.1) for key in PRIOR_LAYER_KEYS}
    grid = (c["B"], D, c["S"], c["S"])
    out.update(x_v=f(*grid), x_h=f(*grid), g_v=f(*grid), g_h=f(*grid),
               label=rng.randint(0, c["N_CLASSES"], size=c["B"]).astype(np.int64))
    return out


def gate_inputs():
    c = GATE
    rng = np.random.RandomState(c["seed"])
    return dict(x=rng.standard_normal((c["B"], 2 * c["C"], c["S"], c["S"])).astype(np.float32) * np.float32(2),
                g=rng.standard_normal((c["B"], c["C"], c["S"], c["S"])).astype(np.float32))


def residual_layer(x, w1, w2):
    """residual.py:25-27 with Q2: relu(x) + W2 . relu(W1 (*) relu(x))."""
    r = F.relu(x)
    return r + F.conv2d(F.relu(F.conv2d(r, w1, None, 1, 1)), w2)


def residual_stack(x, layers):
    """residual.py:48-51: `layers` is a list of (w1, w2), one per application."""
    for w1, w2 in layers:
        x = residual_layer(x, w1, w2)
    return F.relu(x)


def gate(t):
    a, b = t.chunk(2, dim=1)
    return torch.tanh(a) * torch.sigmoid(b)


def gated_layer(p, x_v, x_h, label, mask, k, residual):
    """models.py:65-86 on the parameter dict p (leaf tensors keyed as in the layer's state dict)."""
    wv, wh = p["vert_stack.weight"], p["horiz_stack.weight"]
    if mask == "A":
        wv.data[:, :, -1].zero_()
        wh.data[:, :, :, -1].zero_()
    c = F.embedding(label, p["class_cond_embedding.weight"])[:, :, None, None]
    hv = F.conv2d(x_v, wv, p["vert_stack.bias"], 1, (k // 2, k // 2))[:, :, :x_v.size(-1), :]
    out_v = gate(hv + c)
    hh = F.conv2d(x_h, wh, p["horiz_stack.bias"], 1, (0, k // 2))[:, :, :, :x_h.size(-2)]
    out = gate(F.conv2d(hv, p["vert_to_horiz.weight"], p["vert_to_horiz.bias"]) + hh + c)
    r = F.conv2d(out, p["horiz_resid.weight"], p["horiz_resid.bias"])
    return out_v, (r + x_h if residual else r)

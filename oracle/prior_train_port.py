"""The Gated PixelCNN prior restated differentiably with torch ops -- TEST INFRASTRUCTURE ONLY.

``prior_logits`` is the reference's GatedPixelCNN.forward (pixelcnn/models.py:121-130) on a dict of leaf tensors,
with the reference's masking semantics: mask A zeroes the masked slices of its layer's weights IN PLACE (through
``.data``) and then convolves with the full weight, so autograd gives the masked taps a (non-zero) gradient, as the
reference's does.  (``oracle.prior_port.prior_forward`` masks a clone under no_grad, which would give them none.)
``prior_loss`` is the loss of the reference's ``gated_pixelcnn.py``.  Pinned against the unmodified reference by
tests/test_prior_train_cpu.py through the tests/golden/prior_grad_* vectors that ``python -m
oracle.make_prior_grad_golden`` writes.  The product never imports this module.
"""
import numpy as np
import torch
import torch.nn.functional as F

from .prior_port import _stack

# dot products of each gradient with this many seeded random tensors in the prior_grad_default fingerprint
N_PROBES = 4


def leaf_params(sd, dtype=torch.float32, device="cpu"):
    """{key: leaf tensor requiring grad} of a state dict (tensors or arrays)."""
    return {k: torch.tensor(np.asarray(v), dtype=dtype, device=device, requires_grad=True) for k, v in sd.items()}


def _gate(t):
    a, b = t.chunk(2, dim=1)
    return torch.tanh(a) * torch.sigmoid(b)


def prior_logits(g, x, label, n_layers, layers=None):
    """Logits (B, K, H, W) of codes x (B,H,W) int64 and labels (B,) int64; g maps keys to (leaf) tensors;
    layers: (mask_type, kernel, residual) per layer, default the reference's stack."""
    h = F.embedding(x, g["embedding.weight"]).permute(0, 3, 1, 2)
    x_v = x_h = h
    for i, (mask, k, residual) in enumerate(_stack(n_layers, layers)):
        p = f"layers.{i}."
        wv, wh = g[p + "vert_stack.weight"], g[p + "horiz_stack.weight"]
        if mask == "A":                                   # mask A (models.py:61-63): in place, on the parameter
            wv.data[:, :, -1].zero_()
            wh.data[:, :, :, -1].zero_()
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


def prior_loss(logits, x):
    """gated_pixelcnn.py's criterion: cross entropy of the logits at every position against the codes."""
    K = logits.shape[1]
    return F.cross_entropy(logits.permute(0, 2, 3, 1).contiguous().view(-1, K), x.reshape(-1))


def probes(shape, key_index):
    """The N_PROBES seeded fp64 random tensors the fingerprint dots a gradient with (seed from the key's index)."""
    rng = np.random.RandomState(1000 + key_index)
    return [rng.standard_normal(shape) for _ in range(N_PROBES)]


def fingerprint(grad, key_index):
    """[sum, L2 norm, dot with each probe] of a gradient, in fp64."""
    g = np.asarray(grad, dtype=np.float64)
    return np.array([g.sum(), np.sqrt((g * g).sum())] + [(g * q).sum() for q in probes(g.shape, key_index)])

"""The padding a Gated PixelCNN prior gets at a dim the kernels do not take, restated for the tests (the product never
imports this module): ``pad_prior_state_dict(sd, dim)`` is the state dict of the same prior at Cp = roundup(dim, 32)
channels, every added channel zero.  A gate axis (2*dim channels, tanh half then sigmoid half) is padded per half,
because the kernels pair channel c with channel c + Cp; a dim-wide axis is padded at its end; output_conv's 512 and K
axes and the embeddings' rows are kept.  ``split=False`` pads the gate axes at their end instead: the wrong padding,
which the tests use to show they can tell the two apart."""
import numpy as np
import torch

# axis kinds of each parameter's first two axes: 0 kept, 1 dim-wide, 2 gate (2*dim, padded per half)
KINDS = {"vert_stack.weight": (2, 1), "vert_stack.bias": (2, 0), "vert_to_horiz.weight": (2, 2),
         "vert_to_horiz.bias": (2, 0), "horiz_stack.weight": (2, 1), "horiz_stack.bias": (2, 0),
         "horiz_resid.weight": (1, 1), "horiz_resid.bias": (1, 0), "class_cond_embedding.weight": (0, 2),
         "embedding.weight": (0, 1), "output_conv.0.weight": (0, 1)}


def padded_dim(dim):
    return -(-dim // 32) * 32


def kinds(name):
    if name.startswith("layers."):
        name = name.split(".", 2)[2]
    return KINDS.get(name, (0, 0))


def _pad_axis(t, axis, kind, dim, cp, split):
    if kind == 0 or cp == dim:
        return t
    parts = torch.split(t, dim, dim=axis) if (kind == 2 and split) else [t]
    out = []
    for p in parts:
        shape = list(p.shape)
        shape[axis] = (cp if split or kind == 1 else 2 * cp) - p.shape[axis]
        out += [p, torch.zeros(shape, dtype=p.dtype)]
    return torch.cat(out, dim=axis)


def pad_prior_state_dict(sd, dim, split=True, dtype=torch.float64):
    """The state dict `sd` (keys to arrays or tensors) of a prior with `dim` channels, at Cp channels, in `dtype`."""
    cp = padded_dim(dim)
    out = {}
    for k, v in sd.items():
        t = torch.as_tensor(np.asarray(v) if not torch.is_tensor(v) else v).to(dtype)
        kout, kin = kinds(k)
        t = _pad_axis(t, 0, kout, dim, cp, split)
        if t.dim() > 1:
            t = _pad_axis(t, 1, kin, dim, cp, split)
        out[k] = t
    return out


def real_entries(t, name, dim):
    """The entries of the Cp-shaped tensor t (a parameter or its gradient) that are the dim-wide parameter's; the
    rest is padding."""
    cp = padded_dim(dim)

    def take(x, axis, kind):
        if kind == 0 or cp == dim:
            return x
        idx = torch.arange(dim) if kind == 1 else torch.cat([torch.arange(dim), cp + torch.arange(dim)])
        return x.index_select(axis, idx.to(x.device))
    kout, kin = kinds(name)
    t = take(t, 0, kout)
    return take(t, 1, kin) if t.dim() > 1 else t

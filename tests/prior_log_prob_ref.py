"""fp64 restatement of GatedPixelCNN.log_prob's contract on given logits (DESIGN.md §8, "Scoring code grids") --
TEST INFRASTRUCTURE ONLY.

lp[b, i, j] = log_softmax(logits[b, :, i, j])[clamp(codes[b, i, j], 0, K-1)]; the score of image b is the sum of lp
over the raster positions p = i*W + j >= n_given.  ``kahan32`` is the kernels' compensated fp32 sum in raster order.
"""
import numpy as np


def position_terms(logits, codes):
    """(B, H, W) fp64 lp of logits (B, K, H, W) at the clamped codes (B, H, W)."""
    z = np.asarray(logits, dtype=np.float64)
    K = z.shape[1]
    m = z.max(1, keepdims=True)
    ls = z - m - np.log(np.exp(z - m).sum(1, keepdims=True))
    c = np.clip(np.asarray(codes, dtype=np.int64), 0, K - 1)
    return np.take_along_axis(ls, c[:, None], 1)[:, 0]


def scored(B, H, W, n_given):
    """(B, H, W) bool: the positions p >= n_given."""
    return np.broadcast_to((np.arange(H * W) >= n_given).reshape(1, H, W), (B, H, W))


def log_prob(logits, codes, n_given=0):
    """(B,) fp64: the sum of position_terms over p >= n_given."""
    lp = position_terms(logits, codes)
    B, H, W = lp.shape
    return np.where(scored(B, H, W, n_given), lp, 0.0).reshape(B, -1).sum(-1)


def kahan32(terms, n_given=0):
    """(B,) fp32: the kernels' compensated sum of fp32 terms (B, H*W) over p >= n_given, in raster order."""
    t = np.asarray(terms, dtype=np.float32).reshape(len(terms), -1)
    out = np.zeros(len(t), dtype=np.float32)
    for b in range(len(t)):
        acc = comp = np.float32(0)
        for v in t[b, n_given:]:
            y = np.float32(v - comp)
            s = np.float32(acc + y)
            comp = np.float32(np.float32(s - acc) - y)
            acc = s
        out[b] = acc
    return out

"""fp64 restatement of the prior sampler's draw with temperature, top-k and top-p (DESIGN.md §8, "Sampling knobs"),
row-wise over (N, K) logits -- TEST INFRASTRUCTURE ONLY.

z = l / T in fp32 (saturated to +-FLT_MAX); key(z) the order-preserving map from fp32 to uint32; the kept set is
S = {k : key(z_k) >= max(t_k, t_p)} with t_k the largest threshold keeping at least top_k codes and t_p the largest
keeping at least top_p of the tempered softmax's mass (here in fp64); q is the softmax of z renormalized over S.
"""
import numpy as np

FLT_MAX = np.finfo(np.float32).max


def tempered(logits, T):
    """z = l / T in fp32, saturated to the finite range; l itself at T = 1."""
    l32 = np.asarray(logits, dtype=np.float32)
    if np.float32(T) == 1:
        return l32
    with np.errstate(over="ignore"):
        z = l32 / np.float32(T)
    return np.clip(z, -FLT_MAX, FLT_MAX).astype(np.float32)


def fkey(z32):
    """The order-preserving map from fp32 to uint32 (-0 below +0)."""
    bits = np.ascontiguousarray(z32, dtype=np.float32).view(np.uint32)
    return np.where(bits & np.uint32(0x80000000), ~bits, bits | np.uint32(0x80000000)).astype(np.uint32)


def softmax64(z32):
    z = np.asarray(z32, dtype=np.float64)
    e = np.exp(z - z.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def kept(logits, T=1.0, top_k=None, top_p=None):
    """(N, K) bool: the kept set S of each row."""
    z = np.atleast_2d(tempered(logits, T))
    N, K = z.shape
    key = fkey(z)
    t = np.zeros(N, dtype=np.uint32)
    if top_k is not None and top_k < K:
        t = np.maximum(t, -np.sort(-key.astype(np.int64), axis=-1)[:, top_k - 1].astype(np.uint32))
    if top_p is not None and top_p < 1:
        order = np.argsort(-key.astype(np.int64), axis=-1, kind="stable")
        ks = np.take_along_axis(key, order, -1)
        cum = np.cumsum(np.take_along_axis(softmax64(z), order, -1), -1)
        reach = cum >= np.float64(np.float32(top_p))
        first = np.argmax(reach, -1)
        t_p = np.where(reach.any(-1), ks[np.arange(N), first], 0).astype(np.uint32)
        t = np.maximum(t, t_p)
    return key >= t[:, None]


def probs(logits, T=1.0, top_k=None, top_p=None):
    """(N, K) fp64 q: the tempered softmax renormalized over S, 0 off S."""
    z = np.atleast_2d(tempered(logits, T)).astype(np.float64)
    S = kept(logits, T, top_k, top_p)
    e = np.where(S, np.exp(z - z.max(-1, keepdims=True)), 0.0)
    return e / e.sum(-1, keepdims=True)


def draw(logits, u, T=1.0, top_k=None, top_p=None):
    """(N,) int: the smallest k in S with u < CDF_k, else the last k in S with q_k > 0."""
    q = probs(logits, T, top_k, top_p)
    cdf = np.cumsum(q, -1)
    hit = (np.asarray(u, np.float64)[:, None] < cdf) & (q > 0)
    last = q.shape[1] - 1 - np.argmax((q > 0)[:, ::-1], -1)
    return np.where(hit.any(-1), np.argmax(hit, -1), last)


def log_softmax64(logits):
    z = np.asarray(logits, dtype=np.float64)
    m = z.max(-1, keepdims=True)
    return z - m - np.log(np.exp(z - m).sum(-1, keepdims=True))

"""Restatements of the EMA codebook update (VectorQuantizer(decay=...)) -- TEST INFRASTRUCTURE ONLY.

``segment_sums`` emulates in fp32 the fixed order in which vqb_vq_ema_update_f32 sums the rows of each code (rows of
a code by ascending row index, consecutive segments of SEG rows, one fp32 add chain per segment, the segment partials
added in segment order), so its result is the kernel's bit for bit.  ``ema_update_fp64`` is the update itself in fp64
(van den Oord et al. 2017, appendix A.1, with the Laplace smoothing of the cluster sizes).  ``commit_loss_fp64`` /
``commit_dz_fp64`` are the EMA quantizer's loss and input gradient.
"""
import numpy as np

SEG = 256          # rows per segment (vq_ema.cu EMA_SEG)


def clamp_codes(idx, K):
    return np.clip(np.asarray(idx, dtype=np.int64).reshape(-1), 0, K - 1)


def counts(idx, K):
    """n_k of the clamped codes (the VQ kernel's hist)."""
    return np.bincount(clamp_codes(idx, K), minlength=K).astype(np.int64)


def segment_sums(z, idx, K):
    """s_k (K, D) fp32 in the kernel's order."""
    z = np.ascontiguousarray(z, dtype=np.float32)
    N, D = z.shape
    codes = clamp_codes(idx, K)
    order = np.argsort(codes, kind="stable")                 # rows of each code by ascending row index
    sc = codes[order]
    first = np.searchsorted(sc, np.arange(K))
    rank = np.arange(N) - first[sc]
    seg_of = rank // SEG                                     # segment number within its code
    pos = rank % SEG
    nseg = (np.bincount(codes, minlength=K) + SEG - 1) // SEG
    seg_base = np.concatenate([[0], np.cumsum(nseg)])        # global segment id = seg_base[code] + seg_of
    gid = seg_base[sc] + seg_of
    table = np.full((int(seg_base[-1]), SEG), -1, dtype=np.int64)
    table[gid, pos] = order
    part = np.zeros((table.shape[0], D), dtype=np.float32)
    for r in range(SEG):                                     # one fp32 add chain per segment, in row order
        rows = table[:, r]
        live = rows >= 0
        part[live] = part[live] + z[rows[live]]
    s = np.zeros((K, D), dtype=np.float32)
    for j in range(int(nseg.max()) if K else 0):             # the partials of each code in segment order
        ks = np.nonzero(nseg > j)[0]
        s[ks] = s[ks] + part[seg_base[ks] + j]
    return s


def ema_update_fp64(cluster_size, embed_sum, n, s, decay, eps):
    """(N', m', e') in fp64 from the state (N, m), the counts n and the row sums s."""
    N0 = np.asarray(cluster_size, dtype=np.float64)
    m0 = np.asarray(embed_sum, dtype=np.float64)
    K = N0.shape[0]
    N1 = decay * N0 + (1.0 - decay) * np.asarray(n, dtype=np.float64)
    m1 = decay * m0 + (1.0 - decay) * np.asarray(s, dtype=np.float64)
    total = N1.sum()
    smoothed = (N1 + eps) / (total + K * eps) * total
    return N1, m1, m1 / smoothed[:, None]


def commit_loss_fp64(z, zq, beta):
    """beta * mean((sg[z_q] - z)^2)."""
    d = np.asarray(zq, dtype=np.float64) - np.asarray(z, dtype=np.float64)
    return beta * float(np.mean(d * d))


def commit_dz_fp64(z, zq, g_zq, g_loss, beta):
    """dz = g_zq + g_loss * 2 beta / (N D) * (z - z_q)."""
    z = np.asarray(z, dtype=np.float64)
    return np.asarray(g_zq, dtype=np.float64) + g_loss * 2.0 * beta / z.size * (z - np.asarray(zq, dtype=np.float64))

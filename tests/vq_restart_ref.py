"""Restatement of the EMA codebook's dead-code restart (VectorQuantizer.dead_code_threshold, vqb_vq_ema_restart_f32)
-- TEST INFRASTRUCTURE ONLY.

After an update, with threshold t (in fp32), rows z (N, D) fp32 and uniforms u (N,) fp32: the dead codes are those with
N_k < t (a NaN N_k is not dead), in ascending order; the rows are ordered by (u_i, i); for j < min(M, N) the j-th dead
code takes the j-th row: e <- z_row, m <- fl(t z_row), N <- t.  Exact in fp32, so the kernel must match it bit for bit.
"""
import numpy as np


def dead_codes(cluster_size, t):
    """Ascending indices k with N_k < t (strict; NaN compares false)."""
    return np.nonzero(np.asarray(cluster_size, dtype=np.float32) < np.float32(t))[0]


def row_order(u):
    """Row indices ordered by (u_i, i) ascending: a tie in u goes to the lower row."""
    u = np.asarray(u, dtype=np.float32)
    return np.lexsort((np.arange(u.shape[0]), u))


def restart(z, u, t, cluster_size, embed_sum, codebook):
    """(cluster_size, embed_sum, codebook, count) after the restart; the inputs are not modified."""
    z = np.asarray(z, dtype=np.float32)
    t32 = np.float32(t)
    Nk, m, e = (np.array(a, dtype=np.float32, copy=True) for a in (cluster_size, embed_sum, codebook))
    dead = dead_codes(Nk, t32)
    R = min(dead.shape[0], z.shape[0])
    ks, rows = dead[:R], row_order(u)[:R]
    e[ks] = z[rows]
    m[ks] = t32 * z[rows]                    # fp32 * fp32: one rounding, as __fmul_rn
    Nk[ks] = t32
    return Nk, m, e, R

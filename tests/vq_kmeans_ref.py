"""Restatement of the codebook's k-means initialisation (VectorQuantizer.init_codebook_kmeans, vqb_vq_kmeans_f32) --
TEST INFRASTRUCTURE ONLY.

Built from the restatements the kernels it reuses are checked against: the seed is the restart's row order
(vq_restart_ref.row_order), each step's assignment and SSE the C oracle's canonical fp32 VQ (oracle.cref.vq_rows), the
per-code sums the EMA update's fixed order (vq_ema_ref.segment_sums / counts), and the centroid one fp32 division.  So
the codebook must match the kernels bit for bit; the SSE is a double sum in another order.
"""
import numpy as np

from oracle import cref
from tests.vq_ema_ref import counts, segment_sums
from tests.vq_restart_ref import row_order


def seed(z, u, K):
    """Code j = the row of rank j by (u_i, i), copied exactly."""
    return np.array(np.asarray(z, dtype=np.float32)[row_order(u)[:K]], dtype=np.float32)


def lloyd_step(z, e):
    """(new codebook, sse before the step, n_k) of one step from the codebook e; e is not modified."""
    K = e.shape[0]
    v = cref.vq_rows(z, e)
    n = counts(v["idx"], K)
    s = segment_sums(z, v["idx"], K)
    out = e.copy()
    live = n > 0
    out[live] = s[live] / n[live].astype(np.float32)[:, None]        # fp32 / fp32: one rounding, as __fdiv_rn
    return out, v["sse"], n


def kmeans(z, u, K, iters):
    """(codebook (K, D) fp32, sse (iters,) float64) of vqb_vq_kmeans_f32 on rows z (N, D) and uniforms u (N,)."""
    z = np.ascontiguousarray(z, dtype=np.float32)
    e = seed(z, u, K)
    sse = np.zeros(iters, np.float64)
    for t in range(iters):
        e, sse[t], _ = lloyd_step(z, e)
    return e, sse

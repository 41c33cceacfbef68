"""The tensor-core VQ kernel (vq_tc_kernel in vq_exact.cu) against the exact FFMA kernel, the C oracle and
float64 scores.  Needs an H100: run with ``-m gpu``."""
import numpy as np
import pytest
import torch

from oracle import cref

pytestmark = pytest.mark.gpu

# The tensor-core kernel, the FFMA kernel and the oracle all add the (e - z)^2 terms in double, in different orders
# (per-thread row sums, per-CTA partials).  The tolerance leaves room for a per-row relative error of 16 * 2^-24 ~ 1e-6.
SSE_RTOL = 2e-6


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _inputs(N, K, kind, seed):
    rng = np.random.RandomState(seed)
    z = rng.standard_normal((N, 64)).astype(np.float32)
    if kind == "normal":
        E = rng.standard_normal((K, 64)).astype(np.float32)
    elif kind == "default":          # reference init: near-tie stress (SURVEY Q10)
        E = rng.uniform(-1.0 / K, 1.0 / K, size=(K, 64)).astype(np.float32)
        z *= np.float32(0.06)
    elif kind == "dups":             # heavily duplicated codebook: candidate-list overflow path
        base = rng.standard_normal((max(K // 32, 1), 64)).astype(np.float32)
        E = base[rng.randint(0, base.shape[0], size=K)]
    elif kind == "clustered":        # z sits on top of codes
        E = rng.standard_normal((K, 64)).astype(np.float32)
        z = E[rng.randint(0, K, size=N)] + 1e-4 * z
    elif kind == "nonfinite_z":
        E = rng.standard_normal((K, 64)).astype(np.float32)
        z[min(3, N - 1), 5] = np.nan
        z[min(70, N - 1), 9] = np.inf
    elif kind == "nonfinite_e":
        E = rng.standard_normal((K, 64)).astype(np.float32)
        E[K // 2, 3] = np.nan
    elif kind == "huge":
        E = (rng.standard_normal((K, 64)) * 1e15).astype(np.float32)
        z *= np.float32(1e15)
    return z, E


def _run(kernel, z, E):
    from vqvae_b200 import ops
    ops.set_vq_kernel(kernel)
    try:
        out = ops.vq_forward(_cuda(z), _cuda(E))
        torch.cuda.synchronize()
    finally:
        ops.set_vq_kernel("auto")
    return [t.cpu().numpy() for t in out]


def test_tf32_scores_match_float64():
    """Descriptor / layout check independent of the selection logic: the dumped
    scores must equal ||e||^2 - 2 z.e to TF32 accuracy for every (row, code)."""
    from vqvae_b200 import ops
    z, E = _inputs(300, 700, "normal", 1)
    idx, zq, sse, hist, scores = ops.vq_debug_scores(_cuda(z), _cuda(E))
    torch.cuda.synchronize()
    s = scores.cpu().numpy()
    ref = (E.astype(np.float64) ** 2).sum(1)[None, :] - 2.0 * z.astype(np.float64) @ E.astype(np.float64).T
    bound = 2.0 * 2.0 ** -9 * np.abs(z.astype(np.float64)) @ np.abs(E.astype(np.float64)).T + 1e-4
    assert np.all(np.isfinite(s[:, :700]))
    assert np.all(np.abs(s[:, :700] - ref) <= bound), float(np.abs(s[:, :700] - ref).max())
    assert np.all(np.isinf(s[:, 700:768]))          # padded codes score +inf


CASES = [(1, 1, "normal"), (100, 37, "normal"), (128, 256, "normal"), (129, 257, "normal"),
         (1000, 512, "normal"), (1000, 512, "default"), (777, 512, "dups"), (600, 300, "clustered"),
         (3000, 1024, "normal"), (2000, 1000, "default"), (1500, 8192, "normal"),
         (400, 512, "nonfinite_z"), (400, 512, "nonfinite_e"), (300, 600, "huge")]


@pytest.mark.parametrize("N,K,kind", CASES)
def test_tc_kernel_bit_exact_vs_exact_kernel_and_oracle(N, K, kind):
    z, E = _inputs(N, K, kind, N + K)
    o = cref.vq_rows(z, E)
    i_e, q_e, s_e, h_e = _run("exact", z, E)
    i_t, q_t, s_t, h_t = _run("tc", z, E)
    assert np.array_equal(i_e, o["idx"])
    assert np.array_equal(i_t, o["idx"]), int((i_t != o["idx"]).sum())
    assert np.array_equal(q_t, o["zq"], equal_nan=True)
    assert np.array_equal(h_t, o["hist"])
    np.testing.assert_allclose(s_t, s_e, rtol=SSE_RTOL, equal_nan=True)


@pytest.mark.parametrize("K,kind", [(512, "normal"), (512, "default"), (1024, "normal")])
def test_tc_kernel_large_n_matches_exact_kernel(K, kind):
    """BASELINE cfg4 scale (2^18 rows here): the selection bound must never drop the
    canonical winner -- identical indices, z_q and histogram to the exact kernel."""
    z, E = _inputs(1 << 18, K, kind, 7)
    i_e, q_e, s_e, h_e = _run("exact", z, E)
    i_t, q_t, s_t, h_t = _run("tc", z, E)
    assert np.array_equal(i_t, i_e), int((i_t != i_e).sum())
    assert np.array_equal(q_t, q_e)
    assert np.array_equal(h_t, h_e) and int(h_t.sum()) == 1 << 18
    np.testing.assert_allclose(s_t, s_e, rtol=SSE_RTOL)
    # oracle spot check on a slice
    o = cref.vq_rows(z[:4096], E)
    assert np.array_equal(i_t[:4096], o["idx"])

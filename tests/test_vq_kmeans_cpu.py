"""CPU-only checks of the codebook's k-means initialisation (init_codebook_kmeans, vqb_vq_kmeans_f32): the C ABI's two
entry points and their rejections before any CUDA call, the Python rejections, and the restatement in
tests/vq_kmeans_ref.py on cases small enough to work out by hand."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from vqvae_b200 import _lib
from tests.vq_kmeans_ref import kmeans, lloyd_step, seed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("vqb_vq_kmeans_workspace_bytes", "vqb_vq_kmeans_f32")


def test_new_symbols_are_declared_exported_and_typed_at_abi_3():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "vqvae_b200.h")).read(), flags=re.S)
    L = _lib.lib()
    for n in NEW:
        assert re.search(r"\b%s\s*\(" % n, src), n
        assert n in _lib.SIGNATURES and getattr(L, n).argtypes == _lib.SIGNATURES[n][1]
    assert L.vqb_abi_version() == 3


def test_workspace_covers_its_parts_and_is_zero_for_refused_shapes():
    L = _lib.lib()
    for N, K, D in ((1, 1, 4), (1000, 7, 4), (16384, 512, 64), (1 << 20, 8192, 64), (65536, 1024, 256)):
        ws = L.vqb_vq_kmeans_workspace_bytes(N, K, D)
        parts = (L.vqb_vq_ema_restart_workspace_bytes(N, K) + L.vqb_vq_ema_workspace_bytes(N, K, D) +
                 L.vqb_vq_workspace_bytes(N, K, D) + 8 * N + 4 * K + 4 * N * D)
        assert ws >= parts and ws % 16 == 0, (N, K, D)
        assert L.vqb_vq_kmeans_workspace_bytes(N, K, D) == ws
    for N, K, D in ((0, 1, 4), (4, 0, 4), (4, 4, 0), (-1, 1, 4), (4, 4, -4), (3, 4, 4), (16, 4, 6),
                    (9000, 8193, 4), (1 << 32, 4, 4)):
        assert L.vqb_vq_kmeans_workspace_bytes(N, K, D) == 0, (N, K, D)


def test_rejections_return_their_codes_before_any_cuda_call():
    L = _lib.lib()
    b = (ctypes.c_double * 4096)()
    p = ctypes.cast(b, ctypes.c_void_p).value
    assert p % 16 == 0
    ws = L.vqb_vq_kmeans_workspace_bytes(16, 4, 4)

    def km(N=16, K=4, D=4, iters=1, nbytes=ws, z=p, **null):
        a = {k: (None if k in null else p) for k in ("u", "e", "sse", "ws")}
        return L.vqb_vq_kmeans_f32(z, a["u"], N, K, D, iters, a["e"], a["sse"], a["ws"], nbytes, None)
    assert km(z=None) == -1
    for k in ("u", "e", "sse", "ws"):
        assert km(**{k: 1}) == -1, k
    assert km(N=0) == -1 and km(K=0) == -1 and km(D=0) == -1 and km(N=-5) == -1 and km(D=-4) == -1
    assert km(N=3) == -1                                        # fewer rows than codes
    assert km(iters=-1) == -1 and km(iters=-1, sse=1) == -1
    assert km(D=6) == -2
    assert km(N=9000, K=8193, nbytes=1 << 30) == -2
    assert km(N=1 << 32, nbytes=1 << 40) == -2
    assert km(D=1024, nbytes=1 << 30) == -2                    # the exact VQ kernel's tiles do not fit: a step is refused
    assert km(nbytes=ws - 1) == -3
    assert km(z=p + 4) == -5
    assert km(iters=0, nbytes=ws - 1, sse=1) == -3             # sse may be NULL when there is no step
    assert L.vqb_set_vq_kernel(2) == 0
    try:
        assert km() == -2                                       # D = 4 has no tensor-core kernel
    finally:
        assert L.vqb_set_vq_kernel(0) == 0


def test_python_rejections_come_before_any_launch():
    import vqvae_b200
    vq = vqvae_b200.VectorQuantizer(8, 4, 0.25)
    z = torch.zeros(2, 4, 2, 2)
    for bad in (-1, 1.0, 2.5, "3", None, True, [1]):
        with pytest.raises(ValueError, match="iters"):
            vq.init_codebook_kmeans(z, bad)
    with pytest.raises(ValueError, match="8192"):
        vqvae_b200.VectorQuantizer(8193, 4, 0.25).init_codebook_kmeans(z)
    with pytest.raises(ValueError, match="e_dim"):
        vqvae_b200.VectorQuantizer(8, 6, 0.25).init_codebook_kmeans(torch.zeros(2, 6, 2, 2))
    for bad in (z, torch.zeros(2, 5, 2, 2), torch.zeros(4, 2, 2)):            # CPU tensor, channels, rank
        with pytest.raises(RuntimeError):
            vq.init_codebook_kmeans(bad)
    m = vqvae_b200.VQVAE(32, 8, 1, 16, 8, 0.25)
    with pytest.raises(ValueError, match="iters"):
        m.init_codebook_kmeans(torch.zeros(2, 3, 8, 8), iters=-2)
    for bad in (torch.zeros(2, 3, 8, 8), torch.zeros(2, 4, 8, 8)):
        with pytest.raises(RuntimeError):
            m.init_codebook_kmeans(bad)


def test_the_drop_in_modules_inherit_the_method():
    from models.quantizer import VectorQuantizer
    from models.vqvae import VQVAE
    import vqvae_b200
    assert VectorQuantizer.init_codebook_kmeans is vqvae_b200.VectorQuantizer.init_codebook_kmeans
    assert VQVAE.init_codebook_kmeans is vqvae_b200.VQVAE.init_codebook_kmeans
    assert sorted(VectorQuantizer(8, 4, 0.25).state_dict()) == ["embedding.weight"]


# ---- the restatement ---------------------------------------------------------------------------------------------
def test_reference_two_clusters_by_hand():
    z = np.array([[0, 0, 0, 0], [1, 0, 0, 0], [10, 0, 0, 0], [11, 0, 0, 0], [0, 1, 0, 0]], np.float32)
    u = np.array([0.5, 0.25, 0.75, 0.125, 0.875], np.float32)                 # ranks: rows 3, 1, 0, 2, 4
    e, sse = kmeans(z, u, 2, 3)
    assert np.array_equal(seed(z, u, 2), z[[3, 1]])
    # step 0 from e = {11, 1}: rows 2, 3 -> code 0; rows 0, 1, 4 -> code 1; sse = 1 + 0 + 1 + 0 + 2
    assert sse[0] == 4.0
    want = np.array([[10.5, 0, 0, 0], [np.float32(1) / np.float32(3), np.float32(1) / np.float32(3), 0, 0]],
                    np.float32)
    assert np.array_equal(e, want)
    # a fixed point: the later steps change nothing and have equal inertia
    assert sse[1] == sse[2] and sse[1] < sse[0]


def test_reference_zero_iterations_only_seed():
    rng = np.random.default_rng(0)
    z = rng.standard_normal((50, 8)).astype(np.float32)
    u = rng.random(50, dtype=np.float32)
    e, sse = kmeans(z, u, 7, 0)
    assert sse.shape == (0,)
    assert np.array_equal(e, z[np.lexsort((np.arange(50), u))[:7]])


def test_reference_empty_clusters_keep_their_bits():
    # three copies of each of two rows: the seed takes two copies of one, and of two equal codes the first wins the rows
    z = np.array([[1, 2, 3, 4]] * 3 + [[5, 6, 7, 8]] * 3, np.float32)
    u = np.array([0.1, 0.2, 0.9, 0.3, 0.8, 0.7], np.float32)                  # ranks: rows 0, 1, 3, ...
    e0 = seed(z, u, 3)
    e1, sse, n = lloyd_step(z, e0)
    assert n.tolist() == [3, 0, 3]
    assert np.array_equal(e1[1], e0[1]) and np.array_equal(e1, e0) and sse == 0.0
    e, s = kmeans(z, u, 3, 2)
    assert np.array_equal(e, e0) and s.tolist() == [0.0, 0.0]


def test_reference_nan_row_takes_over():
    z = np.array([[0, 0, 0, 0], [1, 1, 1, 1], [np.nan, 0, 0, 0], [5, 5, 5, 5]], np.float32)
    u = np.array([0.1, 0.2, 0.9, 0.3], np.float32)
    e, _ = kmeans(z, u, 2, 1)
    assert np.isnan(e[0, 0]) and not np.isnan(e[1]).any()       # step 0: the NaN row's distances are NaN: code 0
    _, _, n = lloyd_step(z, e)
    assert n.tolist() == [4, 0]                                  # then every row's distance to code 0 is NaN

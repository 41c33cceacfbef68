"""CPU-only checks of the EMA codebook's dead-code restart (VectorQuantizer.dead_code_threshold): the C ABI's two entry
points and their rejections before any CUDA call, the validating property, the checkpoint entry and the restatement in
tests/vq_restart_ref.py."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

from vqvae_b200 import _lib
from tests.vq_restart_ref import dead_codes, restart, row_order

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("vqb_vq_ema_restart_workspace_bytes", "vqb_vq_ema_restart_f32")


def test_new_symbols_are_declared_exported_and_typed_at_abi_3():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "vqvae_b200.h")).read(), flags=re.S)
    L = _lib.lib()
    for n in NEW:
        assert re.search(r"\b%s\s*\(" % n, src), n
        assert n in _lib.SIGNATURES and getattr(L, n).argtypes == _lib.SIGNATURES[n][1]
    assert L.vqb_abi_version() == 3


def test_workspace_is_a_function_of_n_and_k():
    L = _lib.lib()
    for N, K in ((1, 1), (1000, 7), (16384, 512), (1 << 20, 8192), (524288, 1024)):
        ws = L.vqb_vq_ema_restart_workspace_bytes(N, K)
        assert ws >= 8 * K + 4 * K and ws % 16 == 0, (N, K)          # the selected keys and the dead list
        assert L.vqb_vq_ema_restart_workspace_bytes(N, K) == ws
    assert L.vqb_vq_ema_restart_workspace_bytes(1000, 8192) > L.vqb_vq_ema_restart_workspace_bytes(1000, 512)
    for N, K in ((0, 4), (4, 0), (-1, 4), (4, 8193), (1 << 32, 4)):
        assert L.vqb_vq_ema_restart_workspace_bytes(N, K) == 0, (N, K)


def test_rejections_return_their_codes_before_any_cuda_call():
    L = _lib.lib()
    b = (ctypes.c_float * 4096)()
    p = ctypes.cast(b, ctypes.c_void_p)
    ws = L.vqb_vq_ema_restart_workspace_bytes(16, 4)

    def rs(N=16, K=4, D=4, t=0.5, nbytes=ws, **null):
        a = {k: (None if k in null else p) for k in ("z", "u", "n", "m", "e", "cnt", "ws")}
        return L.vqb_vq_ema_restart_f32(a["z"], a["u"], N, K, D, t, a["n"], a["m"], a["e"], a["cnt"], a["ws"], nbytes,
                                        None)
    for k in ("z", "u", "n", "m", "e", "cnt", "ws"):
        assert rs(**{k: 1}) == -1, k
    assert rs(N=0) == -1 and rs(K=0) == -1 and rs(D=0) == -1 and rs(N=-5) == -1
    for t in (0.0, -0.5, math.inf, -math.inf, math.nan):
        assert rs(t=t) == -1, t
    assert rs(D=6) == -2
    assert rs(K=8193, nbytes=1 << 20) == -2
    assert rs(N=1 << 32, nbytes=1 << 20) == -2
    assert rs(nbytes=ws - 1) == -3
    assert L.vqb_vq_ema_update_f32(p, p, p, 16, 4, 4, 0.9, 1e-5, p, p, p, p, 0, None) == -3    # the update's own code


def test_threshold_property_validates():
    import vqvae_b200
    vq = vqvae_b200.VectorQuantizer(16, 8, 0.25, decay=0.99)
    assert vq.dead_code_threshold is None
    vq.dead_code_threshold = 0.5
    assert vq.dead_code_threshold == 0.5 and isinstance(vq.dead_code_threshold, float)
    vq.dead_code_threshold = 2
    assert vq.dead_code_threshold == 2.0
    vq.dead_code_threshold = np.float32(0.25)
    assert vq.dead_code_threshold == 0.25
    for bad in (0, 0.0, -1.0, math.inf, -math.inf, math.nan, "0.5", None.__class__, [0.5], True, 1j):
        with pytest.raises(ValueError):
            vq.dead_code_threshold = bad
        assert vq.dead_code_threshold == 0.25
    vq.dead_code_threshold = None
    assert vq.dead_code_threshold is None
    # not a state-dict entry, and last_restarts is not one either
    vq.dead_code_threshold = 1.0
    assert sorted(vq.state_dict()) == ["ema_cluster_size", "ema_embed_sum", "embedding.weight"]
    assert vq.last_restarts.dtype == torch.int32 and vq.last_restarts.shape == (1,)
    # restarts are an EMA feature, for codebooks the one-CTA sort holds
    plain = vqvae_b200.VectorQuantizer(16, 8, 0.25)
    with pytest.raises(ValueError):
        plain.dead_code_threshold = 0.5
    plain.dead_code_threshold = None
    assert plain.dead_code_threshold is None and plain.last_restarts is None
    big = vqvae_b200.VectorQuantizer(8193, 4, 0.25, decay=0.9)
    with pytest.raises(ValueError):
        big.dead_code_threshold = 0.5
    vqvae_b200.VectorQuantizer(8192, 4, 0.25, decay=0.9).dead_code_threshold = 0.5
    m = vqvae_b200.VQVAE(32, 8, 1, 16, 8, 0.25, ema_decay=0.9)
    m.vector_quantization.dead_code_threshold = 0.1
    assert "vector_quantization.last_restarts" not in m.state_dict()


def test_checkpoint_round_trip_adds_the_threshold_only_when_set(tmp_path):
    import vqvae_b200
    hp = dict(n_hiddens=32, n_residual_hiddens=8, n_residual_layers=1, n_embeddings=16, embedding_dim=8, beta=0.25)
    m = vqvae_b200.VQVAE(32, 8, 1, 16, 8, 0.25, ema_decay=0.95)
    path = str(tmp_path / "ema.pth")
    vqvae_b200.save_checkpoint(m, {}, hp, path)
    assert set(torch.load(path, map_location="cpu", weights_only=False)["vq_ema"]) == \
        {"decay", "eps", "cluster_size", "embed_sum"}
    assert vqvae_b200.load_checkpoint(path, device="cpu")[0].vector_quantization.dead_code_threshold is None
    m.vector_quantization.dead_code_threshold = 0.75
    vqvae_b200.save_checkpoint(m, {}, hp, path)
    data = torch.load(path, map_location="cpu", weights_only=False)
    assert set(data["vq_ema"]) == {"decay", "eps", "cluster_size", "embed_sum", "dead_code_threshold"}
    assert data["vq_ema"]["dead_code_threshold"] == 0.75
    assert not any("ema_" in k or "restart" in k for k in data["model"])
    m2, _ = vqvae_b200.load_checkpoint(path, device="cpu")
    assert m2.vector_quantization.dead_code_threshold == 0.75
    assert all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), m2.state_dict().values()))


def test_reference_ties_go_to_the_lower_row_and_dead_codes_are_strict():
    u = np.array([0.5, 0.25, 0.5, 0.25, 0.0, 0.5], np.float32)
    assert row_order(u).tolist() == [4, 1, 3, 0, 2, 5]
    Nk = np.array([0.5, 0.49, np.nan, 0.0, 1.0, 0.4999999], np.float32)
    assert dead_codes(Nk, 0.5).tolist() == [1, 3, 5]
    rng = np.random.default_rng(0)
    z = rng.standard_normal((6, 4)).astype(np.float32)
    m0, e0 = rng.standard_normal((6, 4)).astype(np.float32), rng.standard_normal((6, 4)).astype(np.float32)
    N1, m1, e1, R = restart(z, u, 0.5, Nk, m0, e0)
    assert R == 3
    assert np.array_equal(e1[[1, 3, 5]], z[[4, 1, 3]])
    assert np.array_equal(m1[[1, 3, 5]], np.float32(0.5) * z[[4, 1, 3]])
    assert N1[[1, 3, 5]].tolist() == [0.5] * 3
    keep = [0, 2, 4]
    assert np.array_equal(e1[keep], e0[keep]) and np.array_equal(m1[keep], m0[keep])
    assert np.array_equal(N1[keep], Nk[keep], equal_nan=True)


def test_reference_restarts_only_n_codes_when_more_are_dead():
    rng = np.random.default_rng(1)
    K, N, D = 10, 3, 4
    z = rng.standard_normal((N, D)).astype(np.float32)
    u = np.array([0.75, 0.125, 0.5], np.float32)
    Nk = np.zeros(K, np.float32)
    m0 = np.ones((K, D), np.float32)
    N1, m1, e1, R = restart(z, u, 0.3, Nk, m0, m0)
    assert R == N
    assert np.array_equal(e1[:3], z[[1, 2, 0]])
    assert np.array_equal(m1[:3], np.float32(0.3) * z[[1, 2, 0]])
    assert np.array_equal(N1, np.array([np.float32(0.3)] * 3 + [0.0] * 7, np.float32))
    assert np.array_equal(e1[3:], m0[3:])

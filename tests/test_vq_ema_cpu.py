"""CPU-only checks of the EMA codebook (VectorQuantizer(decay=...), VQVAE(ema_decay=...)): the C ABI's new entry points
and their rejections before any CUDA call, the constructors, the state dicts and the checkpoint layout."""
import ctypes
import inspect
import math
import os
import re

import numpy as np
import pytest
import torch

from vqvae_b200 import _lib
from tests.vq_ema_ref import SEG, counts, ema_update_fp64, segment_sums

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("vqb_vq_ema_workspace_bytes", "vqb_vq_ema_update_f32", "vqb_vq_commit_backward_f32", "vqb_vq_finish_ema_f32")


def _buf(n=64):
    b = (ctypes.c_float * n)()
    return b, ctypes.cast(b, ctypes.c_void_p)


def test_new_symbols_are_declared_exported_and_typed_at_abi_3():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "vqvae_b200.h")).read(), flags=re.S)
    L = _lib.lib()
    for n in NEW:
        assert re.search(r"\b%s\s*\(" % n, src), n
        assert n in _lib.SIGNATURES and getattr(L, n).argtypes == _lib.SIGNATURES[n][1]
    assert L.vqb_abi_version() == 3


def test_package_constructors_add_keyword_only_ema_after_the_reference_parameters():
    """vqvae_b200.VQVAE / VectorQuantizer take the reference's positional parameters, then the EMA knobs, keyword-only;
    the ``models`` drop-in classes are the same modules with the reference's constructors exactly."""
    import vqvae_b200
    from models.quantizer import VectorQuantizer
    from models.vqvae import VQVAE

    def sig(c):
        ps = list(inspect.signature(c.__init__).parameters.values())[1:]
        return [p.name for p in ps if p.kind != p.KEYWORD_ONLY], [p.name for p in ps if p.kind == p.KEYWORD_ONLY]

    ref_vqvae = ["h_dim", "res_h_dim", "n_res_layers", "n_embeddings", "embedding_dim", "beta", "save_img_embedding_map"]
    assert sig(vqvae_b200.VQVAE) == (ref_vqvae, ["ema_decay", "ema_eps"])
    assert sig(vqvae_b200.VectorQuantizer) == (["n_e", "e_dim", "beta"], ["decay", "eps"])
    assert sig(VQVAE) == (ref_vqvae, []) and sig(VectorQuantizer) == (["n_e", "e_dim", "beta"], [])
    assert issubclass(VQVAE, vqvae_b200.VQVAE) and issubclass(VectorQuantizer, vqvae_b200.VectorQuantizer)
    assert inspect.signature(vqvae_b200.VQVAE.__init__).parameters["ema_decay"].default is None
    assert inspect.signature(vqvae_b200.VectorQuantizer.__init__).parameters["eps"].default == 1e-5
    m = VQVAE(32, 8, 1, 16, 8, 0.25)
    assert m.vector_quantization.decay is None
    assert list(m.state_dict()) == list(vqvae_b200.VQVAE(32, 8, 1, 16, 8, 0.25).state_dict())
    with pytest.raises(TypeError):
        VQVAE(32, 8, 1, 16, 8, 0.25, ema_decay=0.99)


def test_workspace_query_from_shapes():
    L = _lib.lib()
    for N, K, D in ((1, 1, 4), (1000, 7, 64), (16384, 512, 64), (1 << 20, 8192, 64), (524288, 1024, 256)):
        ws = L.vqb_vq_ema_workspace_bytes(N, K, D)
        # at least the sorted row ids and one partial per possible segment
        assert ws >= 8 * N + 4 * (N // SEG + K + 1) * D, (N, K, D)
        assert ws % 16 == 0
        assert L.vqb_vq_ema_workspace_bytes(N, K, D) == ws                       # a function of the shape only
        assert L.vqb_vq_ema_workspace_bytes(4 * N, K, D) > ws
    for N, K, D in ((0, 4, 4), (4, 0, 4), (4, 4, 0), (4, 4, 6), (-1, 4, 4)):
        assert L.vqb_vq_ema_workspace_bytes(N, K, D) == 0


def test_rejections_return_their_codes_before_any_cuda_call():
    L = _lib.lib()
    _b, p = _buf(4096)
    ws = L.vqb_vq_ema_workspace_bytes(16, 4, 4)

    def upd(N=16, K=4, D=4, decay=0.99, eps=1e-5, nbytes=ws, **null):
        a = {k: (None if k in null else p) for k in ("z", "idx", "hist", "n", "m", "e", "ws")}
        return L.vqb_vq_ema_update_f32(a["z"], a["idx"], a["hist"], N, K, D, decay, eps, a["n"], a["m"], a["e"],
                                       a["ws"], nbytes, None)
    for k in ("z", "idx", "hist", "n", "m", "e", "ws"):
        assert upd(**{k: 1}) == -1, k
    assert upd(N=0) == -1 and upd(K=0) == -1 and upd(D=0) == -1
    for decay in (-0.1, 1.0, 1.5, math.nan):
        assert upd(decay=decay) == -1, decay
    for eps in (0.0, -1e-5, math.inf, math.nan):
        assert upd(eps=eps) == -1, eps
    assert upd(D=6) == -2
    assert upd(nbytes=ws - 1) == -3
    assert L.vqb_vq_commit_backward_f32(None, None, None, p, 16, 4, 0.25, p, None) == -1
    assert L.vqb_vq_commit_backward_f32(None, None, p, p, 0, 4, 0.25, p, None) == -1
    assert L.vqb_vq_commit_backward_f32(None, None, p, p, 16, 6, 0.25, p, None) == -2
    assert L.vqb_vq_finish_ema_f32(None, p, 16, 4, 4, 0.25, p, p, None) == -1
    assert L.vqb_vq_finish_ema_f32(p, p, 0, 4, 4, 0.25, p, p, None) == -1


@pytest.mark.parametrize("kw", [dict(decay=-0.01), dict(decay=1.0), dict(decay=float("nan")), dict(decay="0.9x"),
                                dict(decay=0.99, eps=0.0), dict(decay=0.99, eps=-1.0),
                                dict(decay=0.99, eps=float("inf")), dict(eps=float("nan"))])
def test_constructors_raise_value_error(kw):
    import vqvae_b200
    with pytest.raises(ValueError):
        vqvae_b200.VectorQuantizer(16, 8, 0.25, **kw)
    vkw = {"ema_" + k: v for k, v in kw.items()}
    with pytest.raises(ValueError):
        vqvae_b200.VQVAE(32, 8, 1, 16, 8, 0.25, **vkw)


def test_decay_none_keeps_todays_state_dict():
    import vqvae_b200
    from oracle.weights import state_dict_shapes
    m = vqvae_b200.VQVAE(128, 32, 2, 512, 64, 0.25)
    assert list(m.state_dict()) == [k for k, _, _ in state_dict_shapes(128, 32, 2, 512, 64)]
    vq = m.vector_quantization
    assert vq.decay is None and vq.embedding.weight.requires_grad
    assert list(vqvae_b200.VectorQuantizer(16, 8, 0.25).state_dict()) == ["embedding.weight"]


def test_ema_state_dict_keys_and_initial_values():
    import vqvae_b200
    from oracle.weights import state_dict_shapes
    torch.manual_seed(0)
    m = vqvae_b200.VQVAE(128, 32, 2, 512, 64, 0.25, ema_decay=0.99, ema_eps=1e-6)
    ref = [k for k, _, _ in state_dict_shapes(128, 32, 2, 512, 64)]
    sd = m.state_dict()
    extra = ["vector_quantization.ema_cluster_size", "vector_quantization.ema_embed_sum"]
    assert sorted(sd) == sorted(ref + extra)
    vq = m.vector_quantization
    assert vq.decay == 0.99 and vq.eps == 1e-6
    assert not vq.embedding.weight.requires_grad
    assert vq.ema_cluster_size.dtype == torch.float32 and torch.equal(vq.ema_cluster_size, torch.ones(512))
    assert torch.equal(vq.ema_embed_sum, vq.embedding.weight.detach())
    assert vq.ema_embed_sum.data_ptr() != vq.embedding.weight.data_ptr()
    # the same seed gives the same weights as a decay=None model: the buffers draw no random numbers
    torch.manual_seed(0)
    m0 = vqvae_b200.VQVAE(128, 32, 2, 512, 64, 0.25)
    assert all(torch.equal(v, sd[k]) for k, v in m0.state_dict().items())


def test_reference_state_dict_loads_into_an_ema_model_and_restarts_the_buffers():
    import vqvae_b200
    src = vqvae_b200.VQVAE(32, 8, 1, 16, 8, 0.25)
    m = vqvae_b200.VQVAE(32, 8, 1, 16, 8, 0.25, ema_decay=0.9)
    with torch.no_grad():
        m.vector_quantization.ema_cluster_size.fill_(7.0)
    res = m.load_state_dict(src.state_dict())                 # strict: nothing missing, nothing unexpected
    assert not res.missing_keys and not res.unexpected_keys
    vq = m.vector_quantization
    assert torch.equal(vq.embedding.weight, src.vector_quantization.embedding.weight)
    assert torch.equal(vq.ema_cluster_size, torch.ones(16))
    assert torch.equal(vq.ema_embed_sum, src.vector_quantization.embedding.weight.detach())
    # an EMA state dict restores its buffers as saved
    with torch.no_grad():
        vq.ema_cluster_size.fill_(3.0)
        vq.ema_embed_sum.mul_(2.0)
    m2 = vqvae_b200.VQVAE(32, 8, 1, 16, 8, 0.25, ema_decay=0.9)
    m2.load_state_dict(m.state_dict())
    assert torch.equal(m2.vector_quantization.ema_cluster_size, torch.full((16,), 3.0))
    assert torch.equal(m2.vector_quantization.ema_embed_sum, vq.ema_embed_sum)


def test_checkpoint_layout_keeps_the_reference_keys_and_adds_vq_ema(tmp_path):
    import vqvae_b200
    from oracle.weights import state_dict_shapes
    m = vqvae_b200.VQVAE(128, 32, 2, 512, 64, 0.25, ema_decay=0.95, ema_eps=2e-5)
    with torch.no_grad():
        m.vector_quantization.ema_cluster_size.uniform_(0.5, 2.0)
        m.vector_quantization.ema_embed_sum.normal_()
    hp = dict(n_hiddens=128, n_residual_hiddens=32, n_residual_layers=2, n_embeddings=512, embedding_dim=64,
              beta=0.25)
    path = str(tmp_path / "ema.pth")
    vqvae_b200.save_checkpoint(m, {"n_updates": 1}, hp, path)
    data = torch.load(path, map_location="cpu", weights_only=False)
    assert list(data["model"]) == [k for k, _, _ in state_dict_shapes(128, 32, 2, 512, 64)]     # 23 keys
    assert len(data["model"]) == 23
    ema = data["vq_ema"]
    assert set(ema) == {"decay", "eps", "cluster_size", "embed_sum"}
    assert ema["decay"] == 0.95 and ema["eps"] == 2e-5
    # the reference's notebook load_model: a decay=None model loads "model" strictly
    ref = vqvae_b200.VQVAE(128, 32, 2, 512, 64, 0.25)
    ref.load_state_dict(data["model"])
    m2, _ = vqvae_b200.load_checkpoint(path, device="cpu")
    vq, vq2 = m.vector_quantization, m2.vector_quantization
    assert vq2.decay == 0.95 and vq2.eps == 2e-5
    assert torch.equal(vq2.ema_cluster_size, vq.ema_cluster_size)
    assert torch.equal(vq2.ema_embed_sum, vq.ema_embed_sum)
    assert all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), m2.state_dict().values()))
    # a decay=None model's checkpoint has no vq_ema entry and loads as today
    vqvae_b200.save_checkpoint(ref, {}, hp, path)
    assert "vq_ema" not in torch.load(path, map_location="cpu", weights_only=False)
    assert vqvae_b200.load_checkpoint(path, device="cpu")[0].vector_quantization.decay is None


def test_reference_restatement_orders_the_sum_as_documented():
    """segment_sums: within fp32 rounding of the fp64 sums, equal to a plain loop over the documented order, and
    different in the last bits from one long add chain once a code takes more than one segment."""
    rng = np.random.default_rng(0)
    N, K, D = 3 * SEG + 17, 5, 4
    z = rng.standard_normal((N, D)).astype(np.float32)
    idx = rng.integers(-2, K + 2, N)
    idx[: 2 * SEG + 40] = 3                                  # one code over three segments
    s = segment_sums(z, idx, K)
    codes = np.clip(idx, 0, K - 1)
    for k in range(K):
        rows = np.nonzero(codes == k)[0]
        want = np.float32(0) * np.zeros(D, np.float32)
        for j0 in range(0, len(rows), SEG):
            acc = np.zeros(D, np.float32)
            for r in rows[j0:j0 + SEG]:
                acc = acc + z[r]
            want = want + acc
        assert np.array_equal(s[k], want), k
        np.testing.assert_allclose(s[k], z[rows].astype(np.float64).sum(0), rtol=1e-5, atol=1e-4)
    assert counts(idx, K).sum() == N
    n = counts(idx, K)
    N1, m1, e1 = ema_update_fp64(np.ones(K), np.zeros((K, D)), n, s, 0.0, 1e-12)
    used = n > 0
    np.testing.assert_allclose(e1[used], s[used] / n[used, None], rtol=1e-9)

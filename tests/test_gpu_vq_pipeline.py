"""The warp-specialised tensor-core VQ kernel (vq_tc_kernel: TMA ring, resident or streamed codebook, persistent CTAs,
two-launch calls) against the exact FFMA kernel, on the shapes where its structure changes.  Needs an H100: run with
``-m gpu``."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SSE_RTOL = 2e-6        # the two kernels add the (e - z)^2 terms in double in different orders


def _run(kernel, z, E, **kw):
    from vqvae_b200 import ops
    ops.set_vq_kernel(kernel)
    try:
        out = ops.vq_forward(z, E, **kw)
        torch.cuda.synchronize()
    finally:
        ops.set_vq_kernel("auto")
    return out


def _check(z, E, **kw):
    i_e, q_e, s_e, h_e = _run("exact", z, E, **kw)
    i_t, q_t, s_t, h_t = _run("tc", z, E, **kw)
    assert torch.equal(i_t, i_e), int((i_t != i_e).sum())
    assert torch.equal(q_t.view(torch.int16 if q_t.dtype == torch.bfloat16 else torch.int32),
                       q_e.view(torch.int16 if q_e.dtype == torch.bfloat16 else torch.int32))
    assert torch.equal(h_t, h_e) and int(h_t.sum()) == z.shape[0]
    np.testing.assert_allclose(s_t.item(), s_e.item(), rtol=SSE_RTOL, equal_nan=True)


def _normal(N, K, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    z = torch.randn((N, 64), generator=g) * scale
    E = torch.randn((K, 64), generator=g)
    return z.cuda(), E.cuda()


# 512 codes is the largest codebook that stays resident (4 chunks of 128); 513 streams through the ring
@pytest.mark.parametrize("K", [384, 511, 512, 513, 700, 1024, 8192])
def test_resident_and_streamed_codebooks(K):
    z, E = _normal(5000, K, K)
    _check(z, E)


@pytest.mark.parametrize("K", [512, 1024])
def test_several_tiles_per_cta_with_a_ragged_last_tile(K):
    N = 132 * 128 * 3 + 77              # every persistent CTA takes 3-4 tiles, the last one 77 rows
    z, E = _normal(N, K, 11)
    _check(z, E)


@pytest.mark.parametrize("K", [1, 5, 512, 1000])
def test_one_row(K):
    z, E = _normal(1, K, 3)
    _check(z, E)


def test_overflow_rows_mixed_with_normal_rows_in_one_tile():
    # 40 copies of one code (more than the candidate list holds) next to distinct codes: the rows near the copies
    # take the full scan, their tile neighbours the candidate list
    z, E = _normal(1000, 700, 5)
    E[100:140] = E[99]
    z[::2] = E[99] + 1e-3 * z[::2]
    _check(z, E)


def test_nonfinite_rows():
    z, E = _normal(1000, 1024, 9)
    z[3, 5] = float("nan")
    z[130, 9] = float("inf")
    z[131, 0] = -float("inf")
    z[999] = float("nan")
    _check(z, E)


@pytest.mark.parametrize("K", [512, 1000])
def test_bf16_zq_entry_point(K):
    """The bf16-z_q call gives the fp32 call's idx, hist and sse bitwise, and its z_q rounded to bf16."""
    z, E = _normal(3000, K, 21, scale=0.5)
    _check(z, E, zq_dtype=torch.bfloat16)
    i0, q0, s0, h0 = _run("tc", z, E)
    i1, q1, s1, h1 = _run("tc", z, E, zq_dtype=torch.bfloat16)
    assert torch.equal(i0, i1) and torch.equal(h0, h1) and s0.item() == s1.item()
    assert torch.equal(q1.view(torch.int16), q0.to(torch.bfloat16).view(torch.int16))


@pytest.mark.parametrize("K", [512, 1024])
def test_two_calls_are_bitwise_equal(K):
    z, E = _normal(70000, K, 13)
    a = _run("tc", z, E)
    b = _run("tc", z, E)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert a[2].item() == b[2].item()


def test_cuda_graph_capture_and_replay():
    from vqvae_b200 import ops
    z, E = _normal(20000, 1024, 17)
    ref = _run("tc", z, E)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.vq_forward(z, E)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.vq_forward(z, E)
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        for x, y in zip(out, ref):
            assert torch.equal(x, y)


def test_bench_cfg2_latents_match_the_exact_kernel():
    """bench.py's cfg2 model and images: the whole forward through the wgmma VQ kernel and through the exact kernel
    gives the same indices and the same x_hat."""
    import vqvae_b200
    from vqvae_b200 import ops
    from vqvae_b200.synth import make_images, make_state_dict
    from models.vqvae import VQVAE
    hp = dict(h_dim=128, res_h_dim=32, n_res_layers=2)
    sd = make_state_dict(seed=0, n_embeddings=512, embedding_dim=64, **hp)
    model = VQVAE(hp["h_dim"], hp["res_h_dim"], hp["n_res_layers"], 512, 64, 0.25)
    model.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    model = model.cuda().eval()
    x = torch.from_numpy(make_images(256, 32, seed=1)).cuda()
    vqvae_b200.set_precision("tf32")
    outs = {}
    for kernel in ("exact", "tc"):
        ops.set_vq_kernel(kernel)
        try:
            loss, x_hat, perp = model(x)
            torch.cuda.synchronize()
        finally:
            ops.set_vq_kernel("auto")
        outs[kernel] = (loss.item(), x_hat.clone(), perp.item(), model.last_min_encoding_indices.clone())
    (le, xe, pe, ie), (lt, xt, pt, it) = outs["exact"], outs["tc"]
    assert torch.equal(it, ie) and torch.equal(xt, xe) and pt == pe
    assert abs(lt - le) <= SSE_RTOL * abs(le)

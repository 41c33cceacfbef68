"""HostPipeline (vqvae_b200/pipeline.py): the streaming host-buffer front end returns, batch for
batch, exactly what a direct ``model(x.cuda())`` returns (same kernels, same order)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _state_dict(seed):
    from oracle import weights
    sd = weights.make_state_dict(128, 32, 2, 512, 64, seed=seed)
    return {k: torch.from_numpy(np.array(v)) for k, v in sd.items()}


def _model(prec, seed=5):
    import vqvae_b200
    m = vqvae_b200.VQVAE(128, 32, 2, 512, 64, 0.25)
    m.load_state_dict(_state_dict(seed))
    vqvae_b200.set_precision(prec)
    return m.cuda().eval()


def _batches(n, seed):
    rng = np.random.default_rng(seed)
    return [torch.from_numpy(rng.standard_normal((16, 3, 32, 32)).astype(np.float32)).pin_memory() for _ in range(n)]


def _direct(m, batches):
    with torch.no_grad():
        return [(float(loss), x_hat.cpu().clone(), float(perp)) for loss, x_hat, perp in (m(x.cuda()) for x in batches)]


def _assert_results_equal(want, got):
    assert len(want) == len(got)
    for (l0, xh0, p0), (l1, xh1, p1) in zip(want, got):
        assert l0 == l1 and p0 == p1
        assert torch.equal(xh0, xh1)


@pytest.mark.parametrize("use_graph", [True, False])
@pytest.mark.parametrize("prec", ["tf32", "fp32", "bf16"])
def test_pipeline_matches_direct_forward(use_graph, prec):
    import vqvae_b200
    try:
        m = _model(prec)
        rng = np.random.default_rng(11)
        batches = [torch.from_numpy(rng.standard_normal((16, 3, 32, 32)).astype(np.float32)).pin_memory()
                   for _ in range(7)]
        want = []
        with torch.no_grad():
            for x in batches:
                loss, x_hat, perp = m(x.cuda())
                want.append((float(loss), x_hat.cpu().clone(), float(perp)))
        pipe = vqvae_b200.HostPipeline(m, (16, 3, 32, 32), depth=3, use_graph=use_graph)
        got = []
        n = pipe.run(batches, lambda r: got.append((r.index, float(r.loss), r.x_hat.clone(), float(r.perplexity))))
        assert n == 7 and [g[0] for g in got] == list(range(7))
        for (l0, xh0, p0), (_, l1, xh1, p1) in zip(want, got):
            assert l0 == l1 and p0 == p1
            assert torch.equal(xh0, xh1)
    finally:
        vqvae_b200.set_precision("fp32")


def test_pipeline_rejects_wrong_input():
    import vqvae_b200
    m = _model("fp32")
    pipe = vqvae_b200.HostPipeline(m, (4, 3, 32, 32), depth=2, use_graph=False)
    with pytest.raises(ValueError):
        pipe.push(torch.zeros(4, 3, 16, 16))
    with pytest.raises(ValueError):
        pipe.push(torch.zeros(4, 3, 32, 32, dtype=torch.float64))
    assert pipe.drain() == []


@pytest.mark.parametrize("use_graph", [True, False])
@pytest.mark.parametrize("prec", ["tf32", "fp32", "bf16"])
def test_pipeline_follows_load_state_dict(use_graph, prec):
    """load_state_dict between pushes: the pipeline repacks, in place, every conv weight its captured graph reads, so
    each later result is bitwise what a direct forward with the new weights returns.  (Biases and the codebook are read
    where they lie: the pipeline is drained before the weights change.)"""
    import vqvae_b200
    try:
        m = _model(prec)
        old, new = _batches(4, 21), _batches(4, 22)
        want_old = _direct(m, old)
        pipe = vqvae_b200.HostPipeline(m, (16, 3, 32, 32), depth=2, use_graph=use_graph)

        def run(batches):
            got = []
            pipe.run(batches, lambda r: got.append((float(r.loss), r.x_hat.clone(), float(r.perplexity))))
            return got

        _assert_results_equal(want_old, run(old))
        m.load_state_dict(_state_dict(6))
        got_new = run(new)
        _assert_results_equal(_direct(_model(prec, seed=6), new), got_new)
    finally:
        vqvae_b200.set_precision("fp32")


@pytest.mark.parametrize("prec", ["tf32", "fp32", "bf16"])
def test_repack_packs_what_the_forward_reads(prec):
    """After repack() a forward finds every weight packing it reads in the cache, current: it adds no entry and
    refreshes none (an entry is replaced by a new (tag, buffer) pair whenever it is packed)."""
    import vqvae_b200
    try:
        m = _model(prec)
        m.repack()

        def entries():
            return {(name, key): entry for name, p in m.named_parameters()
                    for key, entry in getattr(p, "_vqb_packed", {}).items()}

        before = entries()
        assert before
        with torch.no_grad():
            m(torch.randn(4, 3, 32, 32, device="cuda"))
        after = entries()
        assert after.keys() == before.keys()
        assert all(after[k] is before[k] for k in before)
    finally:
        vqvae_b200.set_precision("fp32")

"""Time GatedPixelCNN.sample_completion with one prefix length per image on one GPU and print one JSON line.

  python tools/bench_prior_ragged.py [--iters N]

Two workloads (dim 64, 15 layers): B=100 on 8x8 with K=512, and B=16 on 64x64 with K=1024.  In each, image b's
n_given is drawn uniformly from [0, H*W] with a fixed seed.  Arms:
  ragged      one sample_completion call with the (B,) n_given tensor
  per_n       what a caller without per-image prefixes does: one scalar sample_completion call per distinct n_given,
              on the images that share it
  generate    generate on the same batch, the schedule the ragged call runs
Every arm is timed as a CUDA-graph replay of the private calls with fixed uniforms and eagerly through the public
methods (a fresh torch.rand per call); the arms take turns, one call each per round, and each reports the median over
--iters rounds, its launches per call and its ratio to generate's median in the same mode.  ragged_equals_per_n checks
that the two completions agree bitwise.  The GPU's name and power limit are read in the same run.  Nothing is written
to the tree.
"""
import argparse
import contextlib
import io
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_prior_sample import _card, _event_ms  # noqa: E402


def _arms(m, B, S, n):
    """name -> (private callable returning the codes, public callable); and the per_n groups."""
    labels = (torch.arange(10, device="cuda").repeat((B + 9) // 10))[:B]
    u = torch.rand((B, S, S), device="cuda")
    x = torch.randint(0, m.embedding.num_embeddings, (B, S, S), device="cuda")
    groups = [(v, torch.nonzero(n == v)[:, 0]) for v in sorted(set(n.tolist()))]
    sub = [(v, idx, labels[idx], u[idx], x[idx]) for v, idx in groups]

    def per_n_private():
        out = torch.empty_like(x)
        for v, idx, lab, uu, xx in sub:
            out[idx] = m._sample_with(lab, uu, xx, v, 1.0, None, None)[0]
        return out

    private = {"ragged": lambda: m._sample_with(labels, u, x, n, 1.0, None, None)[0],
               "per_n": per_n_private,
               "generate": lambda: m._sample(labels, u)}
    public = {"ragged": lambda: m.sample_completion(x, labels, n),
              "per_n": lambda: [m.sample_completion(x[idx], labels[idx], v) for v, idx in groups],
              "generate": lambda: m.generate(labels, shape=(S, S), batch_size=B)}
    return private, public, len(groups)


def bench(K, B, S, iters):
    from pixelcnn.models import GatedPixelCNN
    from vqvae_b200 import ops
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(K, 64, 15, 10).cuda().eval()
    g = torch.Generator().manual_seed(1234)
    n = torch.randint(0, S * S + 1, (B,), generator=g).cuda()
    private, public, distinct = _arms(m, B, S, n)
    equal = torch.equal(private["ragged"](), private["per_n"]())
    arms, launches = {}, {}
    for name, fn in private.items():
        fn()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            fn()
        graph.replay()
        n0 = ops.launch_count()
        public[name]()
        launches[name] = ops.launch_count() - n0
        arms[name] = (graph.replay, public[name])
    torch.cuda.synchronize()
    times = {name: {"graph": [], "eager": []} for name in arms}
    for _ in range(iters):
        for name, (replay, eager) in arms.items():
            times[name]["graph"].append(_event_ms(replay))
            times[name]["eager"].append(_event_ms(eager))
    res = dict(B=B, grid=S, K=K, dim=64, n_layers=15, iters=iters, distinct_n_given=distinct,
               ragged_equals_per_n=equal)
    gen = {mode: statistics.median(times["generate"][mode]) for mode in ("graph", "eager")}
    for name in arms:
        r = dict(launches=launches[name])
        for mode in ("graph", "eager"):
            med = statistics.median(times[name][mode])
            r[f"{mode}_ms"] = med
            r[f"{mode}_min_ms"] = min(times[name][mode])
            r[f"{mode}_vs_generate"] = med / gen[mode]
        res[name] = r
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = _card()
    res = dict(gpu=name, power_limit_w=power)
    with torch.no_grad():
        res["8x8_K512"] = bench(512, 100, 8, a.iters)
        res["64x64_K1024"] = bench(1024, 16, 64, a.iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

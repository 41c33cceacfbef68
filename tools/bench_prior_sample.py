"""Time GatedPixelCNN.sample's knobs against generate on one GPU and print one JSON line.

  python tools/bench_prior_sample.py [--iters N]

Three sizes: B=100 on 8x8 with K=512 and with K=8192, and B=16 on 64x64 with K=1024 (dim 64, 15 layers each).  Arms:
generate; sample with the default knobs; with temperature 0.8; with top_k=50; with top_p=0.9; with all three; and
sample_completion with all three and the top half of each grid given.  Every arm is timed as a CUDA-graph replay of
the private call with fixed uniforms and eagerly through the public method (a fresh torch.rand per call); the arms
take turns, one call each per round, and each reports the median over --iters rounds with its ratio to generate's
median in the same mode.  The GPU's name and power limit are read in the same run.  Nothing is written to the tree.
"""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ALL = dict(temperature=0.8, top_k=50, top_p=0.9)
KNOBS = {"sample": {}, "sample_T0.8": dict(temperature=0.8), "sample_topk50": dict(top_k=50),
         "sample_topp0.9": dict(top_p=0.9), "sample_all": ALL}


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(q.stdout.strip().splitlines()[0])
    except Exception:           # no nvidia-smi: the number is reported without it
        power = None
    return name, power


def _event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def _arms(m, B, S):
    """name -> (graph-replayed callable, eager callable)."""
    labels = (torch.arange(10, device="cuda").repeat((B + 9) // 10))[:B]
    u = torch.rand((B, S, S), device="cuda")
    x = torch.randint(0, m.embedding.num_embeddings, (B, S, S), device="cuda")
    n = S * S // 2
    k = lambda d: (d.get("temperature", 1.0), d.get("top_k"), d.get("top_p"))
    private = {"generate": lambda: m._sample(labels, u)}
    public = {"generate": lambda: m.generate(labels, shape=(S, S), batch_size=B)}
    for name, d in KNOBS.items():
        private[name] = (lambda d=d: m._sample_with(labels, u, None, 0, *k(d)))
        public[name] = (lambda d=d: m.sample(labels, shape=(S, S), batch_size=B, **d))
    private["sample_completion_all"] = lambda: m._sample_with(labels, u, x, n, *k(ALL))
    public["sample_completion_all"] = lambda: m.sample_completion(x, labels, n, **ALL)
    out = {}
    for name, fn in private.items():
        fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        out[name] = (g.replay, public[name])
    return out


def bench(K, B, S, iters):
    from pixelcnn.models import GatedPixelCNN
    from vqvae_b200 import ops
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(K, 64, 15, 10).cuda().eval()
    arms = _arms(m, B, S)
    times = {name: {"graph": [], "eager": []} for name in arms}
    launches = {}
    for name, (replay, eager) in arms.items():     # warm-up, and each arm's launches per call
        replay()
        n0 = ops.launch_count()
        eager()
        launches[name] = ops.launch_count() - n0
    torch.cuda.synchronize()
    for _ in range(iters):
        for name, (replay, eager) in arms.items():
            times[name]["graph"].append(_event_ms(replay))
            times[name]["eager"].append(_event_ms(eager))
    res = dict(B=B, grid=S, K=K, dim=64, n_layers=15, iters=iters)
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
        res["8x8_K8192"] = bench(8192, 100, 8, a.iters)
        res["64x64_K1024"] = bench(1024, 16, 64, a.iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

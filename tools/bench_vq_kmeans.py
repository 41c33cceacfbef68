"""Time the codebook's k-means initialisation (ops.vq_kmeans, vqb_vq_kmeans_f32) and print one JSON line.

  python tools/bench_vq_kmeans.py [--reps 10] [--quick]

D = 64, iters = 10, N in {16 384, 2^19, 2^20} x K in {512, 1024, 8192}, rows drawn around K random centres.  Each
timed call draws its uniforms with torch.rand, as the module does.  Arms, each timed with CUDA events around --reps
back-to-back calls, eagerly and as --reps replays of a graph holding one call:
  ours      vq_kmeans with iters = 10, and with iters = 0 (the seed alone): per_iter = (iters-10 - iters-0) / 10
  torch     the same algorithm restated with torch ops and no host synchronisation: stable sort of u, matmul distances
            (fp32, in row chunks of 2^18 so the N x K matrix fits), argmin, index_add_ of the rows and of ones, division
            where the count is > 0.  Its SSE before the last step is reported beside ours (sse[-1]).
  vq_ema    vq_forward plus vqb_vq_ema_update_f32 at the same N and K: one step's VQ and sums in the training loop.
The card's name and power limit are printed beside the numbers.  Nothing is written to the tree.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_vq_ema import as_graph, card, timed  # noqa: E402

SIZES = [(N, K) for N in (16384, 1 << 19, 1 << 20) for K in (512, 1024, 8192)]
D, ITERS, CHUNK = 64, 10, 1 << 18


def torch_kmeans(z, u, K, iters):
    """The baseline -> (codebook, sse (iters,) float64); graph-capturable."""
    N = z.shape[0]
    e = z[torch.sort(u, stable=True).indices[:K]].clone()
    sse = torch.empty(iters, dtype=torch.float64, device=z.device)
    ones = torch.ones(N, device=z.device)
    for t in range(iters):
        en = (e * e).sum(1)
        idx = torch.cat([torch.argmin(en[None, :] - 2.0 * (z[i:i + CHUNK] @ e.T), 1) for i in range(0, N, CHUNK)])
        sse[t] = ((z - e[idx]) ** 2).sum(dtype=torch.float64)
        n = torch.zeros(K, device=z.device).index_add_(0, idx, ones)
        s = torch.zeros_like(e).index_add_(0, idx, z)
        e = torch.where(n[:, None] > 0, s / n.clamp(min=1)[:, None], e)
    return e, sse


def point(ops, N, K, reps):
    g = torch.Generator().manual_seed(N + K)
    centres = 2.0 * torch.randn((K, D), generator=g)
    z = (centres[torch.randint(0, K, (N,), generator=g)] + 0.5 * torch.randn((N, D), generator=g)).cuda()
    cb = torch.empty((K, D), device="cuda")

    u = torch.rand((N,), device="cuda")                 # the final SSE of both on one u
    ours_sse = ops.vq_kmeans(z, u, ITERS, cb)
    _, torch_sse = torch_kmeans(z, u, K, ITERS)
    torch.cuda.synchronize()

    def ours():
        ops.vq_kmeans(z, torch.rand((N,), device="cuda"), ITERS, cb)

    def seed():
        ops.vq_kmeans(z, torch.rand((N,), device="cuda"), 0, cb)

    def base():
        torch_kmeans(z, torch.rand((N,), device="cuda"), K, ITERS)

    ust = [torch.ones(K, device="cuda"), cb.clone(), cb.clone()]

    def pair():
        idx, _, _, hist = ops.vq_forward(z, ust[2])
        ops.vq_ema_update(z, idx, hist, 0.99, 1e-5, *ust)
    for f in (ours, seed, base, pair):
        f(), f()
    r = {"N": N, "K": K, "D": D, "iters": ITERS,
         "ours_ms": timed(ours, reps), "ours_graph_ms": timed(as_graph(ours), reps),
         "seed_ms": timed(seed, reps), "seed_graph_ms": timed(as_graph(seed), reps),
         "torch_ms": timed(base, reps), "torch_graph_ms": timed(as_graph(base), reps),
         "vq_ema_ms": timed(pair, reps), "vq_ema_graph_ms": timed(as_graph(pair), reps),
         "ours_final_sse": float(ours_sse[-1]), "torch_final_sse": float(torch_sse[-1])}
    r["per_iter_graph_ms"] = (r["ours_graph_ms"] - r["seed_graph_ms"]) / ITERS
    r["per_iter_over_vq_ema"] = r["per_iter_graph_ms"] / r["vq_ema_graph_ms"]
    r["torch_over_ours"] = r["torch_ms"] / r["ours_ms"]
    r["torch_over_ours_graph"] = r["torch_graph_ms"] / r["ours_graph_ms"]
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--quick", action="store_true", help="first size only, few repetitions")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vq_kmeans.py needs a GPU")
    from vqvae_b200 import ops
    sizes = SIZES[:1] if a.quick else SIZES
    reps = 3 if a.quick else a.reps
    print(json.dumps({"card": card(), "kmeans": [point(ops, N, K, reps) for N, K in sizes]}))


if __name__ == "__main__":
    main()

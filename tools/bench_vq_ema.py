"""Time the EMA codebook update (ops.vq_ema_update, vqb_vq_ema_update_f32) and the VQ-VAE training step with it, and
print one JSON line.

  python tools/bench_vq_ema.py [--reps 50] [--steps 30] [--quick]

Update: N = 16 384, K = 512 (main.py's model at B = 256); N = 524 288, K = 1024 (cfg3's rows); N = 2^20 with K = 512
and K = 8192; all at D = 64, each with uniform codes and with every row on one code (the collapsed codebook).  Timed
with CUDA events around --reps back-to-back calls, eager and as --reps replays of a graph holding one call.  The
baseline is the same update restated in torch (index_add_ of the rows, lerp_ of both averages, the Laplace-smoothed
division), timed the same way.  Modelled bytes: z and idx read once, the EMA state and the codebook read and written
once; the roofline time is those bytes over the H100 SXM data-sheet HBM bandwidth (3.35 TB/s); the card's name and
power limit are printed beside the numbers.

Training step: main.py's model (h_dim 128, res_h_dim 32, 2 residual layers, K 512, D 64) on 32x32 images at B = 32 and
B = 256, TF32 mode, forward + loss + backward + vqvae_b200.optim.Adam(amsgrad, lr 3e-4), with the gradient-trained
codebook and with ema_decay=0.99; median of --steps eager steps (host clock around a synchronised step) and the mean
of --steps replays of the step captured as one CUDA graph.  Nothing is written to the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_GBS = 3350.0
SIZES = [(16384, 512), (524288, 1024), (1 << 20, 512), (1 << 20, 8192)]
D = 64


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:  # pragma: no cover - reported, not fatal
        return {"name": torch.cuda.get_device_name(), "error": repr(e)[:100]}


def torch_update(z, idx, hist, N_, m_, E_, decay, eps):
    """The baseline: the update restated with torch ops (float atomics in index_add_)."""
    K = E_.shape[0]
    s = torch.zeros_like(m_).index_add_(0, idx, z)
    N_.lerp_(hist.float(), 1.0 - decay)
    m_.lerp_(s, 1.0 - decay)
    n = N_.sum()
    E_.copy_(m_ / ((N_ + eps) / (n + K * eps) * n)[:, None])


def timed(fn, reps):
    """ms per call over `reps` back-to-back calls between two events."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    torch.cuda._sleep(20_000_000)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def as_graph(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def update_point(ops, N, K, kind, reps):
    g = torch.Generator().manual_seed(N + K)
    z = torch.randn((N, D), generator=g).cuda()
    idx = (torch.randint(0, K, (N,), generator=g) if kind == "uniform" else torch.full((N,), K // 2)).cuda()
    hist = torch.bincount(idx, minlength=K).to(torch.int32)
    st = [torch.ones(K, device="cuda"), torch.randn(K, D, device="cuda"), torch.randn(K, D, device="cuda")]
    tt = [t.clone() for t in st]

    def ours():
        ops.vq_ema_update(z, idx, hist, 0.99, 1e-5, *st)

    def base():
        torch_update(z, idx, hist, *tt, 0.99, 1e-5)
    for f in (ours, base):
        f(), f()
    out = {"N": N, "K": K, "D": D, "codes": kind,
           "ours_ms": timed(ours, reps), "ours_graph_ms": timed(as_graph(ours), reps),
           "torch_ms": timed(base, reps), "torch_graph_ms": timed(as_graph(base), reps)}
    nbytes = N * D * 4 + N * 8 + K * 4 * 3 + K * D * 4 * 3
    roof_ms = nbytes / (HBM_GBS * 1e9) * 1e3
    out.update(modelled_bytes=nbytes, roofline_ms=roof_ms, roofline_fraction=roof_ms / out["ours_graph_ms"],
               speedup_vs_torch=out["torch_ms"] / out["ours_ms"])
    return out


def train_point(B, ema, steps):
    import vqvae_b200
    from vqvae_b200.optim import Adam
    torch.manual_seed(0)
    m = vqvae_b200.VQVAE(128, 32, 2, 512, 64, 0.25, ema_decay=0.99 if ema else None).cuda().train()
    opt = Adam(m.parameters(), lr=3e-4, amsgrad=True)
    x = torch.rand((B, 3, 32, 32), device="cuda") - 0.5

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.enable_grad():
            embedding_loss, x_hat, _ = m(x)
            loss = torch.mean((x_hat - x) ** 2) / 0.0625 + embedding_loss
            loss.backward()
        opt.step()
        return loss
    for _ in range(3):
        step()
    times = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        step()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    replay = as_graph(step)
    return {"B": B, "codebook": "ema" if ema else "gradient", "eager_ms": statistics.median(times),
            "graph_ms": timed(replay, steps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--quick", action="store_true", help="first size only, few repetitions")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vq_ema.py needs a GPU")
    from vqvae_b200 import ops
    sizes = SIZES[:1] if a.quick else SIZES
    reps, steps = (5, 5) if a.quick else (a.reps, a.steps)
    update = [update_point(ops, N, K, kind, reps) for N, K in sizes for kind in ("uniform", "one")]
    train = []
    import vqvae_b200
    with vqvae_b200.precision("tf32"):
        for B in ((32,) if a.quick else (32, 256)):
            for rnd in range(2):                  # alternate the two arms to expose drift
                for ema in (False, True):
                    r = train_point(B, ema, steps)
                    r["round"] = rnd
                    train.append(r)
    print(json.dumps({"card": card(), "update": update, "train_step": train}))


if __name__ == "__main__":
    main()

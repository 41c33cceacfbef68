"""Time the fused VectorQuantizer call (ops.vq_forward, fp32 z_q) on its own, and print one JSON line.

Shapes: bench.py's cfg2 (16 384 rows, K = 512) and cfg3 (524 288 rows, K = 1024) latents, and the six vq_sweep points
(K in {512, 1024, 8192} x D in {64, 256}; 2^20 rows at D = 64, 2^18 at D = 256).  Each shape runs with two input
distributions: "bench_init" (the model's default codebook U(-1/K, 1/K), rows N(0, 0.06^2) like a trained encoder's
z_e) and "normal" (codebook and rows N(0, 1), what bench.py's vq_sweep uses).

Each call is timed with CUDA events behind a spin kernel (so host-side launch overhead is hidden), with L2 flushed
before it.  Roofline: max(bytes / HBM, FLOP / TF32) with the algorithmic bytes of bench.py (2 * D * 4 + 8 per row) and
the H100 SXM data-sheet peaks (3.35 TB/s, 495 TFLOP/s dense TF32); the card's name and power limit are printed beside
the numbers.

    python tools/bench_vq.py [--reps 20] [--quick]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_GBS, TF32_TFLOPS = 3350.0, 495.0


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:  # pragma: no cover - reported, not fatal
        return {"name": torch.cuda.get_device_name(), "error": repr(e)[:100]}


def inputs(N, K, D, init, dev, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    z = torch.randn((N, D), generator=g, dtype=torch.float32)
    if init == "bench_init":
        E = (torch.rand((K, D), generator=g, dtype=torch.float32) * 2 - 1) / K
        z *= 0.06
    else:
        E = torch.randn((K, D), generator=g, dtype=torch.float32)
    return z.to(dev), E.to(dev)


def point(ops, name, N, K, D, init, reps, flush, dev):
    z, E = inputs(N, K, D, init, dev, seed=N + K + D)
    for _ in range(3):
        ops.vq_forward(z, E)
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    torch.cuda._sleep(50_000_000)
    for e0, e1 in evs:
        flush.zero_()
        e0.record()
        ops.vq_forward(z, E)
        e1.record()
    torch.cuda.synchronize()
    t = sorted(a.elapsed_time(b) for a, b in evs)
    ms = float(np.median(t))
    byts = N * (2 * D * 4 + 8)
    flops = 2.0 * N * K * D
    t_hbm, t_tc = byts / (HBM_GBS * 1e9), flops / (TF32_TFLOPS * 1e12)
    return {"shape": name, "init": init, "rows": N, "K": K, "D": D, "ms": ms, "ms_min": t[0], "ms_max": t[-1],
            "GB_s": byts / (ms * 1e-3) / 1e9, "TFLOP_s": flops / (ms * 1e-3) / 1e12,
            "bound": "tensor" if t_tc > t_hbm else "hbm", "roofline_frac": max(t_hbm, t_tc) / (ms * 1e-3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--quick", action="store_true", help="cfg2 and cfg3 only")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_vq.py needs a GPU"
    import vqvae_b200  # noqa: F401  (builds / loads the library)
    from vqvae_b200 import ops
    dev = torch.device("cuda")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    shapes = [("cfg2", 16384, 512, 64), ("cfg3", 524288, 1024, 64)]
    if not args.quick:
        shapes += [(f"sweep_K{K}_D{D}", (1 << 20) if D == 64 else (1 << 18), K, D)
                   for K, D in ((512, 64), (1024, 64), (8192, 64), (512, 256), (1024, 256), (8192, 256))]
    rows = []
    for name, N, K, D in shapes:
        for init in ("bench_init", "normal"):
            rows.append(point(ops, name, N, K, D, init, args.reps, flush, dev))
            torch.cuda.empty_cache()
    print(json.dumps({"tool": "bench_vq", "card": card(), "reps": args.reps, "peaks": {"hbm_GB_s": HBM_GBS,
                      "tf32_TFLOP_s": TF32_TFLOPS, "source": "H100 SXM data sheet"}, "points": rows}), flush=True)


if __name__ == "__main__":
    main()

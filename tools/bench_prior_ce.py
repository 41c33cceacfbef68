"""Time one training step of the Gated PixelCNN prior with GatedPixelCNN.cross_entropy against forward plus torch's
cross-entropy on one GPU and print one JSON line.

  python tools/bench_prior_ce.py [--iters N]

Workloads (dim 64, 10 classes): the reference gated_pixelcnn.py's defaults (B=32 on 8x8, K=512, 15 layers), the cfg3
latent (B=16 on 64x64, K=1024, 15 layers), and the same grid with K=8192 (2 layers).  Arms, in fp32 and TF32:
  cross_entropy   loss = model.cross_entropy(x, label); loss.backward(); vqvae_b200.optim.Adam.step()
  forward_ce      the reference loop: model(x, label), permute / contiguous, nn.CrossEntropyLoss(), backward, step
Each arm reports the median over --iters rounds (arms alternate, after two warm-up steps) of device-event times of
the forward (through the loss), the backward and the optimizer step, the whole step, and the peak allocation above
what was allocated before the step (reset_peak_memory_stats).  The GPU's name and power limit are read in the same
run.  Nothing is written to the tree.
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

WORKLOADS = {"8x8_K512": (32, 8, 512, 15), "64x64_K1024": (16, 64, 1024, 15), "64x64_K8192": (16, 64, 8192, 2)}


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(q.stdout.strip().splitlines()[0])
    except Exception:           # no nvidia-smi: the number is reported without it
        power = None
    return name, power


def _step(m, opt, x, lab, arm):
    """One training step -> (forward ms, backward ms, step ms, peak GiB above the step's start)."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    opt.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ev[0].record()
    with torch.enable_grad():
        if arm == "cross_entropy":
            loss = m.cross_entropy(x, lab)
        else:
            lg = m(x, lab).permute(0, 2, 3, 1).contiguous()
            loss = torch.nn.CrossEntropyLoss()(lg.view(-1, lg.shape[-1]), x.view(-1))
        ev[1].record()
        loss.backward()
    ev[2].record()
    opt.step()
    ev[3].record()
    del loss
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3]), peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_prior_ce.py needs a GPU")
    from pixelcnn.models import GatedPixelCNN
    from vqvae_b200.optim import Adam
    name, power = _card()
    out = {"gpu": name, "power_limit_w": power, "iters": args.iters, "workloads": {}}
    for wl, (B, S, K, L) in WORKLOADS.items():
        gen = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randint(0, K, (B, S, S), device="cuda", generator=gen)
        lab = torch.randint(0, 10, (B,), device="cuda", generator=gen)
        for precision in ("fp32", "tf32"):
            torch.manual_seed(0)
            with contextlib.redirect_stdout(io.StringIO()):
                m = GatedPixelCNN(K, 64, L, 10).cuda()
            m.precision = precision
            opt = Adam(m.parameters(), lr=3e-4)
            arms = ("cross_entropy", "forward_ce")
            times = {a: [] for a in arms}
            for a in arms:
                for _ in range(2):
                    _step(m, opt, x, lab, a)
            for _ in range(args.iters):
                for a in arms:
                    times[a].append(_step(m, opt, x, lab, a))
            res = {}
            for a in arms:
                f, b, s, p = (statistics.median(t[i] for t in times[a]) for i in range(4))
                res[a] = {"forward_ms": round(f, 3), "backward_ms": round(b, 3), "step_ms": round(s, 3),
                          "total_ms": round(f + b + s, 3), "peak_gib": round(max(t[3] for t in times[a]), 3)}
            res["speedup"] = round(res["forward_ce"]["total_ms"] / res["cross_entropy"]["total_ms"], 3)
            out["workloads"][f"{wl}_{precision}"] = res
            print(f"{wl} {precision}: " + ", ".join(f"{a} {res[a]['total_ms']:.2f} ms ({res[a]['peak_gib']:.2f} GiB)"
                                                   for a in arms), file=sys.stderr)
            del m, opt
            torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

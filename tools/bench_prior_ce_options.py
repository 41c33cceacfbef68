"""Time one training step of the Gated PixelCNN prior with GatedPixelCNN.cross_entropy_ex (weight, ignore_index,
label_smoothing) against cross_entropy without them and against forward plus torch's cross-entropy with the same
options, on one GPU, and print one JSON line.

  python tools/bench_prior_ce_options.py [--iters N]

Workloads: tools/bench_prior_ce.py's (dim 64, 10 classes; B=32 on 8x8 with K=512 and 15 layers, B=16 on 64x64 with
K=1024 and 15 layers, and the same grid with K=8192 and 2 layers), in fp32 and TF32.  Arms, alternating:
  plain        loss = model.cross_entropy(x, label); backward; vqvae_b200.optim.Adam.step()
  options      model.cross_entropy_ex(x, label, ...) with weight (uniform in [0.1, 1.1)), ignore_index (a code
               present at about 1/K of the positions) and label_smoothing=0.1
  forward_ce   model(x, label), F.cross_entropy(..., same options) on the permuted logits, backward, step
Each arm reports the median over --iters rounds (after two warm-up steps) of device-event times of the forward
(through the loss), the backward and the optimizer step, their sum, the peak allocation above what was allocated
before the step, and the median of --iters replays of the whole step captured in one CUDA graph.  The GPU's name and
power limit are read in the same run.  forward_ce has no graph time: torch's cross-entropy with a weight and an
ignore_index synchronises with the host, which a capture does not allow.  Nothing is written to the tree.
"""
import argparse
import contextlib
import io
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_prior_ce import WORKLOADS, _card  # noqa: E402

ARMS = ("plain", "options", "forward_ce")


def _loss(m, x, lab, arm, opts):
    if arm == "plain":
        return m.cross_entropy(x, lab)
    if arm == "options":
        return m.cross_entropy_ex(x, lab, **opts)
    lg = m(x, lab).permute(0, 2, 3, 1).contiguous()
    K = lg.shape[-1]
    return F.cross_entropy(lg.view(-1, K), x.view(-1), weight=opts["weight"], ignore_index=opts["ignore_index"],
                           label_smoothing=opts["label_smoothing"])


def _step(m, opt, x, lab, arm, opts):
    """One training step -> (forward ms, backward ms, step ms, peak GiB above the step's start)."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    opt.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ev[0].record()
    with torch.enable_grad():
        loss = _loss(m, x, lab, arm, opts)
        ev[1].record()
        loss.backward()
    ev[2].record()
    opt.step()
    ev[3].record()
    del loss
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3]), peak


def _graph_ms(m, opt, x, lab, arm, opts, iters):
    """Median ms of replays of one whole step captured in a CUDA graph."""
    def step():
        opt.zero_grad(set_to_none=True)
        with torch.enable_grad():
            _loss(m, x, lab, arm, opts).backward()
        opt.step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    out = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    del g
    torch.cuda.synchronize()
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_prior_ce_options.py needs a GPU")
    from pixelcnn.models import GatedPixelCNN
    from vqvae_b200.optim import Adam
    name, power = _card()
    out = {"gpu": name, "power_limit_w": power, "iters": args.iters, "workloads": {}}
    met = True
    for wl, (B, S, K, L) in WORKLOADS.items():
        gen = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randint(0, K, (B, S, S), device="cuda", generator=gen)
        lab = torch.randint(0, 10, (B,), device="cuda", generator=gen)
        opts = dict(weight=torch.rand(K, device="cuda", generator=gen) + 0.1, ignore_index=int(x[0, 0, 0]),
                    label_smoothing=0.1)
        for precision in ("fp32", "tf32"):
            torch.manual_seed(0)
            with contextlib.redirect_stdout(io.StringIO()):
                m = GatedPixelCNN(K, 64, L, 10).cuda()
            m.precision = precision
            opt = Adam(m.parameters(), lr=3e-4)
            times = {a: [] for a in ARMS}
            for a in ARMS:
                for _ in range(2):
                    _step(m, opt, x, lab, a, opts)
            for _ in range(args.iters):
                for a in ARMS:
                    times[a].append(_step(m, opt, x, lab, a, opts))
            res = {}
            for a in ARMS:
                f, b, s, p = (statistics.median(t[i] for t in times[a]) for i in range(4))
                res[a] = {"forward_ms": round(f, 3), "backward_ms": round(b, 3), "step_ms": round(s, 3),
                          "total_ms": round(f + b + s, 3), "peak_gib": round(max(t[3] for t in times[a]), 3)}
            for a in ARMS[:2]:          # torch's cross-entropy with weight and ignore_index syncs: not capturable
                res[a]["graph_ms"] = round(_graph_ms(m, opt, x, lab, a, opts, args.iters), 3)
                torch.cuda.empty_cache()
            res["forward_ce"]["graph_ms"] = None
            res["options_over_plain"] = round(res["options"]["total_ms"] / res["plain"]["total_ms"], 3)
            res["options_over_plain_graph"] = round(res["options"]["graph_ms"] / res["plain"]["graph_ms"], 3)
            res["forward_ce_over_options"] = round(res["forward_ce"]["total_ms"] / res["options"]["total_ms"], 3)
            met &= res["options_over_plain"] <= 1.10
            if wl == "64x64_K8192":
                met &= res["options"]["peak_gib"] < 1.0
            out["workloads"][f"{wl}_{precision}"] = res
            print(f"{wl} {precision}: " + ", ".join(f"{a} {res[a]['total_ms']:.2f} ms (graph {res[a]['graph_ms']} ms, "
                                                   f"{res[a]['peak_gib']:.3f} GiB)" for a in ARMS), file=sys.stderr)
            del m, opt
            torch.cuda.empty_cache()
    out["targets_met"] = met
    print(json.dumps(out))


if __name__ == "__main__":
    main()

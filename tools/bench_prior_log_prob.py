"""Time GatedPixelCNN.log_prob against scoring through the logits on one GPU and print one JSON line.

  python tools/bench_prior_log_prob.py [--iters N]

Workloads (dim 64, 10 classes): the reference gated_pixelcnn.py's defaults (B=32 on 8x8, K=512, 15 layers), the cfg3
latent (B=16 on 64x64, K=1024, 15 layers), and the same grid with K=8192 (2 layers).  Arms, each returning per-image
sums of log p(x):
  log_prob_fp32, log_prob_tf32        GatedPixelCNN.log_prob in that precision
  forward_ce_fp32, forward_ce_tf32    our forward, then the reference test() loop's permute / contiguous and
                                      nn.CrossEntropyLoss(reduction='none') summed per image
  reference                           the same loss on the unmodified reference GatedPixelCNN (the copy in oracle/_ref,
                                      "kind": "reference"), or its torch restatement oracle/prior_port.py ("port")
Each arm reports the median of device-event times over --iters rounds (arms alternate, one call each per round,
after a warm-up call; our arms also as CUDA-graph replays, "graph_ms", which leaves out the host's time), the peak
allocation above what was allocated before the call (reset_peak_memory_stats), our
kernel launches per call, and the multiply-add FLOPs of the teacher-forced forward from shapes.  The GPU's name and
power limit are read in the same run.  Nothing is written to the tree.
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


def flops(B, S, K, dim, n_layers):
    """2 x multiply-adds of the teacher-forced forward (kept taps; layer 0 mask A 7x7, the rest mask B 3x3)."""
    C, ours = dim, 0
    for i in range(n_layers):
        k = 7 if i == 0 else 3
        a = i == 0
        ours += (k // 2 + 1 - a) * k * C * 2 * C + 4 * C * C + (k // 2 + 1 - a) * C * 2 * C + C * C
    return 2 * (ours + C * 512 + 512 * K) * B * S * S


def _ce_sum(logits, x):
    K = logits.shape[1]
    lg = logits.permute(0, 2, 3, 1).contiguous()
    ce = torch.nn.CrossEntropyLoss(reduction="none")(lg.view(-1, K), x.view(-1))
    return -ce.view(x.shape[0], -1).sum(-1)


def _reference(m, x, lab):
    from oracle.prior_ref import load_reference_prior
    Ref = load_reference_prior()
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    if Ref is None:
        from oracle.prior_port import prior_forward
        return (lambda: _ce_sum(prior_forward(sd, x, lab, len(m.layers)), x)), "port"
    with contextlib.redirect_stdout(io.StringIO()):
        ref = Ref(m.embedding.num_embeddings, m.dim, len(m.layers), 10)
    ref.load_state_dict(sd)
    ref = ref.cuda().eval()
    return (lambda: _ce_sum(ref(x, lab), x)), "reference"


def _event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def bench(B, S, K, L, iters):
    from pixelcnn.models import GatedPixelCNN
    from vqvae_b200 import ops
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(K, 64, L, 10).cuda().eval()
    x = torch.randint(0, K, (B, S, S), device="cuda")
    lab = torch.arange(B, device="cuda") % 10

    def ours(precision, fn):
        def call():
            m.precision = precision
            return fn()
        return call

    arms = {"log_prob_fp32": ours("fp32", lambda: m.log_prob(x, lab)),
            "log_prob_tf32": ours("tf32", lambda: m.log_prob(x, lab)),
            "forward_ce_fp32": ours("fp32", lambda: _ce_sum(m(x, lab), x)),
            "forward_ce_tf32": ours("tf32", lambda: _ce_sum(m(x, lab), x))}
    ref_fn, kind = _reference(m, x, lab)
    arms["reference"] = ref_fn
    res = dict(B=B, grid=S, K=K, dim=64, n_layers=L, iters=iters, flops=flops(B, S, K, 64, L),
               logits_bytes=B * K * S * S * 4)
    out = {}
    for name, fn in arms.items():               # warm-up, peak memory, launches and result of one call
        fn()
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        n0 = ops.launch_count()
        out[name] = fn().double()
        torch.cuda.synchronize()
        res[name] = dict(peak_bytes=torch.cuda.max_memory_allocated() - before,
                         launches=ops.launch_count() - n0 if name != "reference" else None)
    res["reference"]["kind"] = kind
    graphs = {}
    for name, fn in arms.items():               # our arms also as CUDA-graph replays: device time without the host
        if name == "reference":
            continue
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        g.replay()
        graphs[name] = g
    times = {name: [] for name in arms}
    gtimes = {name: [] for name in graphs}
    for _ in range(iters):
        for name, fn in arms.items():
            times[name].append(_event_ms(fn))
            if name in graphs:
                gtimes[name].append(_event_ms(graphs[name].replay))
    for name in arms:
        med = statistics.median(times[name])
        res[name].update(ms=med, min_ms=min(times[name]), tflops=res["flops"] / med / 1e9)
        if name in graphs:
            res[name]["graph_ms"] = statistics.median(gtimes[name])
        # the sums each arm returned, relative to forward_ce of the same precision (reference: to fp32)
        base = out["forward_ce_tf32" if name.endswith("tf32") else "forward_ce_fp32"]
        res[name]["max_rel_diff"] = float(((out[name] - base).abs() / base.abs()).max())
    for p in ("fp32", "tf32"):
        for t in ("ms", "graph_ms"):
            res[f"log_prob_{p}"][f"{t}_vs_forward_ce"] = res[f"log_prob_{p}"][t] / res[f"forward_ce_{p}"][t]
    del graphs
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = _card()
    res = dict(gpu=name, power_limit_w=power)
    with torch.no_grad():
        for w, (B, S, K, L) in WORKLOADS.items():
            res[w] = bench(B, S, K, L, a.iters)
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

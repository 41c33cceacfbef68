"""Time the Gated PixelCNN prior on one GPU and print one JSON line.

  python tools/bench_prior.py [--iters N]

Reports generate() for the reference's CIFAR settings (B=100, 8x8, K=512, dim=64, 15 layers, labels arange(10) x 10)
and for the cfg3 latent (B=16, 64x64, K=1024), eagerly and as a CUDA-graph replay; complete() of the same two
shapes with the top half of each grid given (n_given = 32 and 2048), the same ways, with launches per call and the
ratio of its graph replay to generate's ("vs_generate_graph"); the teacher-forced forward at
B=32, 8x8; algorithmic FLOPs of the incremental schedule and of the reference's one-forward-per-position schedule;
and the unmodified reference's GatedPixelCNN.generate in stock PyTorch eager on the same GPU ("kind": "reference",
from the copy oracle/prior_ref.py makes in oracle/_ref; without that copy the torch restatement
oracle/prior_port.py stands in, "kind": "port").  At 64x64 the reference is timed for one row of positions and
scaled by H ("extrapolated xH").  Nothing is written to the repository tree.
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(q.stdout.strip().splitlines()[0])
    except Exception:           # no nvidia-smi: the number is reported without it
        power = None
    return name, power


def _time(fn, iters, warmup=1):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def flops(H, W, K, dim, n_layers):
    """(incremental schedule, reference schedule) multiply-adds x 2 per image: the sampler computes every position
    once with mask A's taps dropped; the reference runs H*W whole-grid forwards with full kernels."""
    C = dim
    head = C * 512 + 512 * K
    ours = ref = 0
    for i in range(n_layers):
        k = 7 if i == 0 else 3
        kh, kw = k // 2 + 1, k // 2 + 1
        a = i == 0
        ours += (kh - a) * k * C * 2 * C + 4 * C * C + (kw - a) * C * 2 * C + C * C
        ref += kh * k * C * 2 * C + 4 * C * C + kw * C * 2 * C + C * C
    ours, ref = (ours + head) * H * W, (ref + head) * H * W
    return 2 * ours, 2 * ref * H * W


def bench_generate(m, B, S, iters, graph=True):
    from vqvae_b200 import ops
    labels = (torch.arange(10, device="cuda").repeat((B + 9) // 10))[:B]
    m.generate(labels, shape=(S, S), batch_size=B)
    n0 = ops.launch_count()
    m.generate(labels, shape=(S, S), batch_size=B)
    launches = ops.launch_count() - n0
    eager = _time(lambda: m.generate(labels, shape=(S, S), batch_size=B), iters)
    out = dict(B=B, grid=S, eager_ms=eager, launches=launches, samples_per_s_eager=B / eager * 1e3)
    if graph:
        u = torch.rand((B, S, S), device="cuda")
        m._sample(labels, u)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            m._sample(labels, u)
        ms = _time(g.replay, iters)
        out.update(graph_ms=ms, samples_per_s_graph=B / ms * 1e3)
    return out


def bench_complete(m, B, S, n_given, iters, ref_ms=None):
    """complete() of B grids of SxS from their first n_given positions: eager (a fresh torch.rand per call, as the public
    method draws) and as a CUDA-graph replay of _complete, with launches per call; ref_ms: generate's time at the same
    shape, for the ratio."""
    from vqvae_b200 import ops
    labels = (torch.arange(10, device="cuda").repeat((B + 9) // 10))[:B]
    x = torch.randint(0, m.embedding.num_embeddings, (B, S, S), device="cuda")
    m.complete(x, labels, n_given)
    n0 = ops.launch_count()
    m.complete(x, labels, n_given)
    launches = ops.launch_count() - n0
    eager = _time(lambda: m.complete(x, labels, n_given), iters)
    out = dict(B=B, grid=S, n_given=n_given, eager_ms=eager, launches=launches,
               samples_per_s_eager=B / eager * 1e3)
    u = torch.rand((B, S, S), device="cuda")
    m._complete(labels, u, x, n_given)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        m._complete(labels, u, x, n_given)
    ms = _time(g.replay, iters)
    out.update(graph_ms=ms, samples_per_s_graph=B / ms * 1e3)
    if ref_ms is not None:
        out["vs_generate_graph"] = ms / ref_ms
    return out


def _reference(m, labels, shape, B, rows=None):
    """(callable, kind) sampling with the reference: its own GatedPixelCNN ("reference", the verbatim copy made by
    oracle.prior_ref.build_prior_ref) holding m's weights, or the torch restatement ("port") when the copy is absent.
    rows: only the first rows of positions, each step one full forward, softmax and multinomial as in the
    reference's generate loop."""
    from oracle.prior_ref import load_reference_prior
    import torch.nn.functional as F
    Ref = load_reference_prior()
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    if Ref is None:
        from oracle.prior_port import prior_generate
        return (lambda: prior_generate(sd, labels, shape, B, len(m.layers), device="cuda", rows=rows)), "port"
    with contextlib.redirect_stdout(io.StringIO()):           # its init prints one line per layer
        ref = Ref(m.embedding.num_embeddings, m.dim, len(m.layers), m.layers[0].class_cond_embedding.num_embeddings)
    ref.load_state_dict(sd)
    ref = ref.cuda().eval()
    if rows is None:
        return (lambda: ref.generate(labels, shape=shape, batch_size=B)), "reference"

    def part():
        x = torch.zeros((B,) + tuple(shape), dtype=torch.int64, device="cuda")
        for i in range(rows):
            for j in range(shape[1]):
                logits = ref(x, labels)[:, :, i, j]
                x[:, i, j] = torch.multinomial(F.softmax(logits, -1), 1).view(-1)
        return x
    return part, "reference"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    from pixelcnn.models import GatedPixelCNN
    assert torch.cuda.is_available(), "needs a GPU"
    torch.manual_seed(0)
    name, power = _card()
    res = dict(gpu=name, power_limit_w=power)
    with torch.no_grad():
        m = GatedPixelCNN(512, 64, 15, 10).cuda().eval()
        res["generate_8x8"] = bench_generate(m, 100, 8, a.iters)
        res["generate_8x8"]["flops_incremental"], res["generate_8x8"]["flops_reference_schedule"] = \
            (f * 100 for f in flops(8, 8, 512, 64, 15))
        res["complete_8x8"] = bench_complete(m, 100, 8, 32, a.iters, res["generate_8x8"]["graph_ms"])
        x = torch.randint(0, 512, (32, 8, 8), device="cuda")
        lab = torch.arange(32, device="cuda") % 10
        res["forward_8x8_B32_ms"] = _time(lambda: m(x, lab), a.iters)
        labels = torch.arange(10, device="cuda").repeat(10)
        ref_fn, kind = _reference(m, labels, (8, 8), 100)
        ref = _time(ref_fn, max(1, a.iters // 2))
        res["reference_8x8"] = dict(kind=kind, eager_ms=ref, samples_per_s=100 / ref * 1e3)

        m3 = GatedPixelCNN(1024, 64, 15, 10).cuda().eval()
        res["generate_64x64"] = bench_generate(m3, 16, 64, max(1, a.iters // 2))
        res["generate_64x64"]["flops_incremental"], res["generate_64x64"]["flops_reference_schedule"] = \
            (f * 16 for f in flops(64, 64, 1024, 64, 15))
        res["complete_64x64"] = bench_complete(m3, 16, 64, 64 * 32, max(1, a.iters // 2),
                                               res["generate_64x64"]["graph_ms"])
        lab16 = torch.arange(10, device="cuda").repeat(2)[:16]
        row_fn, kind = _reference(m3, lab16, (64, 64), 16, rows=1)
        row = _time(row_fn, 1)
        res["reference_64x64"] = dict(kind=kind, one_row_ms=row, eager_ms=row * 64,
                                      note="extrapolated xH from one row of positions")
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Time one training step of the Gated PixelCNN prior on one GPU and print one JSON line.

  python tools/bench_prior_train.py [--iters N]

Workloads: the reference's prior defaults (B=32, 8x8, K=512, dim=64, 15 layers, 10 classes) and the cfg3 latent
(B=16, 64x64, K=1024).  Each step is gated_pixelcnn.py's: logits, cross entropy, backward, Adam (lr 3e-4); it is timed
split into forward (logits + loss), backward, and Adam with the repacking of the weights the next forward does.
Arms: "ours" (GatedPixelCNN.precision = "fp32", CUDA cores), "ours_tf32" (precision = "tf32", the wgmma TF32 GEMM)
and "baseline"; the arms of a workload are timed alternately, one step of each in turn.  Also reported: library
launches per step, and the forward's and the backward's FLOPs by shape (matrix products only; the one-hot sums of the
embedding and class gradients not counted) with the backward's achieved FLOP/s.  The baseline is the unmodified
reference's GatedPixelCNN in stock PyTorch eager on the same GPU ("kind": "reference", from the copy
oracle/prior_ref.py makes in oracle/_ref); without that copy the differentiable torch restatement
oracle/prior_train_port.py stands in ("kind": "port").  Nothing is written to the repository tree.
"""
import argparse
import contextlib
import io
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_prior import _card  # noqa: E402

WORKLOADS = {"default_8x8": dict(B=32, S=8, K=512), "cfg3_64x64": dict(B=16, S=64, K=1024)}
DIM, LAYERS, CLASSES = 64, 15, 10


def backward_flops(B, S, K, C=DIM, n_layers=LAYERS):
    """2 x multiply-adds of the backward's matrix products: dgrad over the taps the forward keeps, wgrad over all."""
    per = 2 * (K * 512 + 512 * C)                   # head: d_hidden and d x_h, then dW2 and dW1
    for i in range(n_layers):
        k, a = (7, 1) if i == 0 else (3, 0)
        h = k // 2 + 1
        per += C * C + C * C                                 # horiz_resid: dgrad, wgrad
        per += (h - a) * 2 * C * C + h * 2 * C * C          # horiz_stack: dgrad, wgrad
        per += 4 * C * C + 4 * C * C                        # vert_to_horiz: dgrad, wgrad
        per += (h - a) * k * 2 * C * C + h * k * 2 * C * C  # vert_stack: dgrad, wgrad
    return 2 * per * B * S * S


def forward_flops(B, S, K, C=DIM, n_layers=LAYERS):
    """2 x multiply-adds of the forward's matrix products over the taps each layer keeps."""
    per = K * 512 + 512 * C                         # head
    for i in range(n_layers):
        k, a = (7, 1) if i == 0 else (3, 0)
        h = k // 2 + 1
        per += (h - a) * k * 2 * C * C + 4 * C * C + (h - a) * 2 * C * C + C * C
    return 2 * per * B * S * S


def _split(arms, iters):
    """Median ms of each named phase of each arm over iters steps; arms: {arm: [(phase, fn), ...]}.  Each step runs
    one step of every arm in turn, so the arms see the same conditions."""
    times = {arm: {n: [] for n, _ in parts} for arm, parts in arms.items()}
    for it in range(iters + 1):
        for arm, parts in arms.items():
            for n, fn in parts:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                b.synchronize()
                if it:                              # step 0 warms up
                    times[arm][n].append(a.elapsed_time(b))
    res = {}
    for arm, phases in times.items():
        out = {}
        for n, ts in phases.items():
            ts.sort()
            out[n + "_ms"] = ts[len(ts) // 2]
        out["step_ms"] = sum(out[n + "_ms"] for n in phases)
        res[arm] = out
    return res


def _step_parts(model_fn, params, x, lab, K, repack=None):
    opt = torch.optim.Adam(params, lr=3e-4)
    crit = nn.CrossEntropyLoss()
    st = {}

    def fwd():
        with torch.enable_grad():
            logits = model_fn(x, lab).permute(0, 2, 3, 1).contiguous()
            st["loss"] = crit(logits.view(-1, K), x.view(-1))

    def bwd():
        opt.zero_grad()
        st.pop("loss").backward()

    def adam():
        opt.step()
        if repack:
            repack()
    return [("forward", fwd), ("backward", bwd), ("adam", adam)]


def ours(B, S, K, precision):
    """(step parts, launches per step) of our GatedPixelCNN in `precision`."""
    from pixelcnn.models import GatedPixelCNN
    from vqvae_b200 import ops
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(K, DIM, LAYERS, CLASSES).cuda()
    m.precision = precision
    x = torch.randint(0, K, (B, S, S), device="cuda")
    lab = torch.randint(0, CLASSES, (B,), device="cuda")
    parts = _step_parts(m, m.parameters(), x, lab, K, repack=lambda: m._net([]))
    for _, fn in parts:
        fn()
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    for _, fn in parts:
        fn()
    return parts, ops.launch_count() - n0


def reference(B, S, K):
    """(step parts, kind) of the baseline."""
    from oracle.prior_ref import load_reference_prior
    torch.manual_seed(0)
    x = torch.randint(0, K, (B, S, S), device="cuda")
    lab = torch.randint(0, CLASSES, (B,), device="cuda")
    Ref = load_reference_prior()
    if Ref is not None:
        with contextlib.redirect_stdout(io.StringIO()):           # its init prints one line per layer
            ref = Ref(K, DIM, LAYERS, CLASSES).cuda()
        parts, kind = _step_parts(ref, ref.parameters(), x, lab, K), "reference"
    else:
        from oracle.prior_port import make_prior_state_dict
        from oracle.prior_train_port import leaf_params, prior_logits
        g = leaf_params(make_prior_state_dict(K, DIM, LAYERS, CLASSES, 0), device="cuda")
        parts, kind = _step_parts(lambda a, b: prior_logits(g, a, b, LAYERS), g.values(), x, lab, K), "port"
    return parts, kind


def bench(B, S, K, iters):
    arms, launches = {}, {}
    for arm, precision in (("ours", "fp32"), ("ours_tf32", "tf32")):
        arms[arm], launches[arm] = ours(B, S, K, precision)
    arms["baseline"], kind = reference(B, S, K)
    res = _split(arms, iters)
    ff, fb = forward_flops(B, S, K), backward_flops(B, S, K)
    for arm in launches:
        res[arm].update(launches_per_step=launches[arm], forward_flops=ff, backward_flops=fb,
                        backward_tflops=fb / (res[arm]["backward_ms"] * 1e-3) / 1e12)
    res["baseline"]["kind"] = kind
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = _card()
    res = dict(gpu=name, power_limit_w=power)
    for w, cfg in WORKLOADS.items():
        res[w] = dict(cfg, **bench(cfg["B"], cfg["S"], cfg["K"], a.iters))
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

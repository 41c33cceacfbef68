"""Time one training step of the Gated PixelCNN prior on one GPU and print one JSON line.

  python tools/bench_prior_train.py [--iters N]

Workloads: the reference's prior defaults (B=32, 8x8, K=512, dim=64, 15 layers, 10 classes) and the cfg3 latent
(B=16, 64x64, K=1024).  Each step is gated_pixelcnn.py's: logits, cross entropy, backward, Adam (lr 3e-4); it is timed
split into forward (logits + loss), backward, and Adam with the repacking of the weights the next forward does.
Also reported: library launches per step, and the backward's achieved FLOP/s from the FLOPs its matrix products
need by shape (the one-hot sums of the embedding and class gradients not counted).  The baseline is the unmodified
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


def _split(step_parts, iters):
    """Median ms of each named phase over iters steps; step_parts: list of (name, fn) run in order per step."""
    times = {n: [] for n, _ in step_parts}
    for it in range(iters + 1):
        for n, fn in step_parts:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            if it:                                  # step 0 warms up
                times[n].append(a.elapsed_time(b))
    out = {}
    for n, ts in times.items():
        ts.sort()
        out[n + "_ms"] = ts[len(ts) // 2]
    out["step_ms"] = sum(out[n + "_ms"] for n, _ in step_parts)
    return out


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


def bench_ours(B, S, K, iters):
    from pixelcnn.models import GatedPixelCNN
    from vqvae_b200 import ops
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(K, DIM, LAYERS, CLASSES).cuda()
    x = torch.randint(0, K, (B, S, S), device="cuda")
    lab = torch.randint(0, CLASSES, (B,), device="cuda")
    parts = _step_parts(m, m.parameters(), x, lab, K, repack=lambda: m._net([]))
    for _, fn in parts:
        fn()
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    for _, fn in parts:
        fn()
    launches = ops.launch_count() - n0
    out = _split(parts, iters)
    fl = backward_flops(B, S, K)
    out.update(launches_per_step=launches, backward_flops=fl, backward_tflops=fl / (out["backward_ms"] * 1e-3) / 1e12)
    return out


def bench_reference(B, S, K, iters):
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
    out = _split(parts, iters)
    out["kind"] = kind
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = _card()
    res = dict(gpu=name, power_limit_w=power)
    for w, cfg in WORKLOADS.items():
        res[w] = dict(cfg, ours=bench_ours(cfg["B"], cfg["S"], cfg["K"], a.iters),
                      baseline=bench_reference(cfg["B"], cfg["S"], cfg["K"], a.iters))
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Time one training step of the notebook-style piecewise walk against the fused ``VQVAE.forward`` step.

main.py's model (h_dim 128, res_h_dim 32, 2 residual layers, 512 x 64 codebook) on a B x 3 x 32 x 32 batch, main.py's
loss, forward + backward (no optimizer step).  The piecewise step calls
``decoder(vector_quantization(pre_quantization_conv(encoder(x)))[1])`` as the reference's notebook does; it pays an
NCHW <-> NHWC copy and a separately saved input at each module boundary.  Median of --iters steps after a warm-up,
timed with CUDA events; library launches per step.  Prints one JSON line.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_prior import _card  # noqa: E402

HP = dict(h_dim=128, res_h_dim=32, n_res_layers=2, n_embeddings=512, embedding_dim=64)
X_TRAIN_VAR = 0.0625


def _fused(m, x):
    embedding_loss, x_hat, _ = m(x)
    return torch.mean((x_hat - x) ** 2) / X_TRAIN_VAR + embedding_loss


def _piecewise(m, x):
    embedding_loss, z_q, _, _, _ = m.vector_quantization(m.pre_quantization_conv(m.encoder(x)))
    x_hat = m.decoder(z_q)
    return torch.mean((x_hat - x) ** 2) / X_TRAIN_VAR + embedding_loss


def bench(m, x, fn, iters):
    from vqvae_b200 import ops

    def step():
        m.zero_grad(set_to_none=True)
        with torch.enable_grad():
            fn(m, x).backward()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    step()
    launches = ops.launch_count() - n0
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return dict(step_ms=statistics.median(times), launches_per_step=launches)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--batch", type=int, default=32)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    import vqvae_b200
    from models.vqvae import VQVAE
    name, power = _card()
    torch.manual_seed(0)
    m = VQVAE(*HP.values(), 0.25).cuda().train()
    x = torch.rand((a.batch, 3, 32, 32), device="cuda") - 0.5
    res = dict(gpu=name, power_limit_w=power, B=a.batch, S=32, iters=a.iters)
    for mode in ("fp32", "tf32"):
        with vqvae_b200.precision(mode):
            fused, piece = bench(m, x, _fused, a.iters), bench(m, x, _piecewise, a.iters)
        res[mode] = dict(fused=fused, piecewise=piece, piecewise_over_fused=piece["step_ms"] / fused["step_ms"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Time the Gated PixelCNN prior at dims that are not a multiple of 32 on one GPU and print one JSON line.

  python tools/bench_prior_anydim.py [--batch B] [--iters N] [--precisions fp32,tf32]

gated_pixelcnn.py builds GatedPixelCNN(512, img_dim**2, 15).  For img_dim 7, 14 and 28 (dim 49, 196 and 784, which
the kernels run at Cp = 64, 224 and 800 on zero-padded packings), at B = 32 on the img_dim x img_dim grid: the
teacher-forced forward and one training step (cross_entropy, its backward and a vqvae_b200.optim.Adam step), each
against GatedPixelCNN(512, Cp, 15) on the same grid, so the ratio is the padding machinery's own cost (the gradient
unpadding launch and the padded packings); the padded channels' arithmetic is in both.  Then generate() once at 7x7
for both.  Medians of --iters timed calls after one warm-up.  Nothing is written to the repository tree.
"""
import argparse
import contextlib
import io
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_prior import _card, _time  # noqa: E402


def _model(dim, precision, seed):
    from pixelcnn.models import GatedPixelCNN
    torch.manual_seed(seed)
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(512, dim, 15).cuda()
    m.precision = precision
    return m


def _times(m, x, lab, iters):
    from vqvae_b200.optim import Adam
    out = {}
    with torch.no_grad():
        out["forward_ms"] = _time(lambda: m(x, lab), iters)
    opt = Adam(m.parameters(), lr=3e-4)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.enable_grad():
            m.cross_entropy(x, lab).backward()
        opt.step()
    out["train_step_ms"] = _time(step, iters)
    return out


def bench_dim(img_dim, B, iters, precisions):
    dim = img_dim ** 2
    cp = -(-dim // 32) * 32
    x = torch.randint(0, 512, (B, img_dim, img_dim), device="cuda")
    lab = torch.arange(B, device="cuda") % 10
    out = dict(dim=dim, padded_to=cp, B=B, grid=img_dim, layers=15, K=512)
    for precision in precisions:
        res = {}
        for name, d in (("padded", dim), ("native", cp)):
            m = _model(d, precision, dim)
            res[name] = _times(m, x, lab, iters)
            del m
            torch.cuda.empty_cache()
        res["forward_ratio"] = res["padded"]["forward_ms"] / res["native"]["forward_ms"]
        res["train_step_ratio"] = res["padded"]["train_step_ms"] / res["native"]["train_step_ms"]
        out[precision] = res
    return out


def bench_generate(B, S):
    """generate() at SxS for dim S*S and for its Cp: one warm-up at 1x1 (weight packing) and one timed call each."""
    dim = S * S
    out = dict(B=B, grid=S, dim=dim)
    lab = torch.arange(B, device="cuda") % 10
    for name, d in (("padded", dim), ("native", -(-dim // 32) * 32)):
        m = _model(d, "fp32", dim).eval()
        with torch.no_grad():
            m.generate(lab, shape=(1, 1), batch_size=B)
            out[name + "_ms"] = _time(lambda: m.generate(lab, shape=(S, S), batch_size=B), 1, warmup=0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--precisions", default="fp32")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = _card()
    res = dict(gpu=name, power_limit_w=power)
    for img_dim in (7, 14, 28):
        res[f"img_dim_{img_dim}"] = bench_dim(img_dim, a.batch, a.iters, a.precisions.split(","))
    res["generate_7x7"] = bench_generate(a.batch, 7)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

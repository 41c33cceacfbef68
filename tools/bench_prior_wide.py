"""Time the Gated PixelCNN prior at the reference script's wide dims on one GPU and print one JSON line.

  python tools/bench_prior_wide.py [--batch B] [--iters N]

gated_pixelcnn.py builds GatedPixelCNN(512, img_dim**2, 15): dim = 576 for 24x24 latents and 1024 for 32x32.  For
both, at B = 32 (the script's batch size): the teacher-forced forward, and one training step (cross_entropy, its
backward and a vqvae_b200.optim.Adam step), in fp32 and TF32; the unmodified reference's GatedPixelCNN.forward in
stock PyTorch eager on the same GPU (from the copy oracle/prior_ref.py makes in oracle/_ref; without it the torch
restatement oracle/prior_port.py stands in, "kind": "port").  At 32x32: generate() once, whole, with the per-step
time it implies, and the reference's generate timed for one row of positions and scaled by H.  Medians of --iters
timed calls after one warm-up.  Nothing is written to the repository tree.
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

from bench_prior import _card, _reference, _time  # noqa: E402


def _model(dim, precision):
    from pixelcnn.models import GatedPixelCNN
    torch.manual_seed(dim)
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(512, dim, 15).cuda()
    m.precision = precision
    return m


def bench_dim(img_dim, B, iters):
    from vqvae_b200.optim import Adam
    from oracle.prior_ref import load_reference_prior
    dim = img_dim ** 2
    x = torch.randint(0, 512, (B, img_dim, img_dim), device="cuda")
    lab = torch.arange(B, device="cuda") % 10
    out = dict(dim=dim, B=B, grid=img_dim, layers=15, K=512)
    for precision in ("fp32", "tf32"):
        m = _model(dim, precision)
        with torch.no_grad():
            out[f"forward_{precision}_ms"] = _time(lambda: m(x, lab), iters)
        opt = Adam(m.parameters(), lr=3e-4)

        def step():
            opt.zero_grad(set_to_none=True)
            with torch.enable_grad():
                m.cross_entropy(x, lab).backward()
            opt.step()
        out[f"train_step_{precision}_ms"] = _time(step, iters)
        out[f"train_step_{precision}_peak_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
        del m, opt
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
    Ref = load_reference_prior()
    m = _model(dim, "fp32")
    if Ref is not None:
        with contextlib.redirect_stdout(io.StringIO()):
            ref = Ref(512, dim, 15)
        ref.load_state_dict(m.state_dict())
        ref = ref.cuda().eval()
        kind = "reference"
    else:
        from oracle.prior_port import prior_forward
        sd = {k: v.detach() for k, v in m.state_dict().items()}
        ref = (lambda a, b: prior_forward(sd, a, b, 15))
        kind = "port"
    with torch.no_grad():
        out["reference_forward"] = dict(kind=kind, ms=_time(lambda: ref(x, lab), iters),
                                        tf32_convs=torch.backends.cudnn.allow_tf32)
    return out, m


def bench_generate(m, B, S):
    """generate() at SxS, one warm-up at 1x1 (module load, weight packing) and one timed call of the whole grid."""
    from vqvae_b200 import ops
    lab = torch.arange(B, device="cuda") % 10
    with torch.no_grad():
        m.generate(lab, shape=(1, 1), batch_size=B)
        n0 = ops.launch_count()
        ms = _time(lambda: m.generate(lab, shape=(S, S), batch_size=B), 1, warmup=0)
        launches = ops.launch_count() - n0
        ref_fn, kind = _reference(m, lab, (S, S), B, rows=1)
        row = _time(ref_fn, 1)
    return dict(B=B, grid=S, ms=ms, ms_per_step=ms / (S * S), launches=launches,
                reference=dict(kind=kind, one_row_ms=row, ms=row * S, note="extrapolated xH from one row of positions"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=2)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = _card()
    res = dict(gpu=name, power_limit_w=power)
    res["img_dim_24"], _ = bench_dim(24, a.batch, a.iters)
    res["img_dim_32"], m = bench_dim(32, a.batch, a.iters)
    res["generate_32x32"] = bench_generate(m.eval(), a.batch, 32)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

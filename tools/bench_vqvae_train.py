"""Time one VQ-VAE training step (main.py's loop) on one GPU and print one JSON line.

  python tools/bench_vqvae_train.py [--iters N]

Workloads: main.py's defaults (h_dim 128, res_h_dim 32, 2 residual layers, K = 512, D = 64) on 32x32 images at
B = 32 (main.py's batch) and B = 256 (cfg2), each in the fp32 and tf32 modes.  A step is main.py:72-79: forward,
recon loss, backward, Adam(amsgrad=True, lr=3e-4) plus ``VQVAE.repack()``, which refreshes both packings of every
changed weight (the forward's, and the input-gradient one the backward reads) that the next forward and backward
would otherwise redo; it is timed split into forward (model + loss), backward, and optimizer, and the median of
--iters steps is reported.  Also: library launches per step; the weight-gradient FLOPs (2 x the multiply-adds of every conv
weight gradient, from the shapes) and the achieved TFLOP/s of the vqb_conv_wgrad_f32 launches (timed with CUDA
events in a separate step) against the 67 TFLOP/s FP32 data-sheet figure of the H100 SXM; and their share of the
step.  The baseline is the unmodified reference's VQVAE in stock PyTorch eager on the same GPU (cuDNN TF32 on, torch's
default), imported from the copy oracle.build_ref() makes in oracle/_ref ("kind": "reference"); without it the
differentiable restatement oracle/vqvae_train_port.py stands in ("kind": "port").  Nothing is written to the tree.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_prior import _card  # noqa: E402
from bench_prior_train import _split  # noqa: E402

HP = dict(h_dim=128, res_h_dim=32, n_res_layers=2, n_embeddings=512, embedding_dim=64)
S = 32
BATCHES = (32, 256)
FP32_PEAK_TFLOPS = 67.0
X_TRAIN_VAR = 0.0625


def wgrad_flops(B, S=S, h=HP["h_dim"], r=HP["res_h_dim"], n=HP["n_res_layers"], D=HP["embedding_dim"]):
    """2 x multiply-adds of every conv weight gradient: a conv reduces over its output pixels, a transposed conv over
    its input pixels, each tap of each (in, out) channel pair."""
    s1, s2 = (S // 2) ** 2, (S // 4) ** 2
    macs = 16 * 3 * (h // 2) * s1 + 16 * (h // 2) * h * s2 + 9 * h * h * s2     # encoder convs 0, 2, 4
    macs += n * (9 * h * r + r * h) * s2 * 2                                      # two stacks, n applications each
    macs += h * D * s2                                                             # pre-quantization 1x1
    macs += 9 * D * h * s2 + 16 * h * (h // 2) * s2 + 16 * (h // 2) * 3 * s1     # decoder convT 0, 2, 4
    return 2 * macs * B


def _step_parts(model, x):
    opt = torch.optim.Adam(model.parameters(), lr=3e-4, amsgrad=True)
    st = {}

    def fwd():
        with torch.enable_grad():
            embedding_loss, x_hat, perplexity = model(x)
            st["loss"] = torch.mean((x_hat - x) ** 2) / X_TRAIN_VAR + embedding_loss

    def bwd():
        opt.zero_grad()
        st.pop("loss").backward()

    def step():
        opt.step()
        if hasattr(model, "repack"):
            model.repack()
    return [("forward", fwd), ("backward", bwd), ("optimizer", step)]


def bench_ours(B, mode, iters):
    import vqvae_b200
    from models.vqvae import VQVAE
    from vqvae_b200 import ops
    torch.manual_seed(0)
    m = VQVAE(*HP.values(), 0.25).cuda().train()
    x = torch.rand((B, 3, S, S), device="cuda") - 0.5
    with vqvae_b200.precision(mode):
        parts = _step_parts(m, x)
        for _, fn in parts:
            fn()
        torch.cuda.synchronize()
        n0 = ops.launch_count()
        for _, fn in parts:
            fn()
        launches = ops.launch_count() - n0
        out = _split(parts, iters)
        ops.PROFILE = []                             # CUDA events around every library call of one more step
        try:
            for _, fn in parts:
                fn()
            torch.cuda.synchronize()
            wg_ms = sum(a.elapsed_time(b) for label, a, b in ops.PROFILE if label.startswith("wgrad"))
        finally:
            ops.PROFILE = None
    fl = wgrad_flops(B)
    tflops = fl / (wg_ms * 1e-3) / 1e12
    out.update(launches_per_step=launches, wgrad_flops=fl, wgrad_ms=wg_ms, wgrad_tflops=tflops,
               wgrad_share_of_fp32_peak=tflops / FP32_PEAK_TFLOPS, wgrad_share_of_step=wg_ms / out["step_ms"])
    return out


def _reference_model():
    import oracle
    ref_dir = oracle.ref_path()
    if not ref_dir:
        return None
    saved = {k: sys.modules.pop(k) for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]}
    sys.path.insert(0, ref_dir)
    try:
        from models.vqvae import VQVAE as RefVQVAE
    finally:
        sys.path.remove(ref_dir)
        for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
            del sys.modules[k]
        sys.modules.update(saved)                    # the product's own `models` package stays importable
    return RefVQVAE


def bench_reference(B, iters):
    torch.manual_seed(0)
    x = torch.rand((B, 3, S, S), device="cuda") - 0.5
    Ref = _reference_model()
    if Ref is not None:
        ref = Ref(*HP.values(), 0.25).cuda().train()
        out, kind = _split(_step_parts(ref, x), iters), "reference"
    else:
        from oracle.prior_train_port import leaf_params
        from oracle.vqvae_train_port import vqvae_train_forward
        from vqvae_b200.synth import make_state_dict
        sd = make_state_dict(seed=0, **HP)
        g = leaf_params({k: sd[k] for k in sd if ".stack." not in k or ".stack.0." in k}, device="cuda")

        class Port(torch.nn.Module):
            def __init__(self):
                super().__init__()
                self.p = torch.nn.ParameterList(list(g.values()))

            def forward(self, x):
                return vqvae_train_forward(x, g, HP["n_res_layers"])[:3]
        out, kind = _split(_step_parts(Port(), x), iters), "port"
    out["kind"] = kind
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    assert a.iters >= 10
    name, power = _card()
    res = dict(gpu=name, power_limit_w=power, iters=a.iters)
    for B in BATCHES:
        w = dict(B=B, S=S, baseline=bench_reference(B, a.iters))
        for mode in ("fp32", "tf32"):
            w[mode] = bench_ours(B, mode, a.iters)
            w[mode]["speedup_vs_baseline"] = w["baseline"]["step_ms"] / w[mode]["step_ms"]
        res[f"B{B}_{S}x{S}"] = w
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

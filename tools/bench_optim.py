"""Time the optimizer step of both models, torch's Adam against vqvae_b200.optim.Adam, and print one JSON line.

  python tools/bench_optim.py [--iters N]

Four arms per workload, timed alternately (one call of each in turn) with CUDA events and reported as medians:
  torch_phase  torch.optim.Adam.step() plus the repacking the next forward would do (VQVAE.repack(), or the prior's
               packing walk), on gradients of one real backward;
  fused_phase  vqvae_b200.optim.Adam.step() on the same kind of gradients;
  eager_step   a whole training step (forward, loss, backward, fused step), eager;
  graph_step   the same step captured as one CUDA graph after one eager step, replayed.
Each arm has its own model, so the arms do not share parameters.  launches_per_step counts library launches of one
call (for graph_step: the launches the captured step holds; a replay is one graph launch).
Workloads: the VQ-VAE at main.py's sizes (Adam amsgrad, lr 3e-4) at B = 32 and 256 on 32x32 images, in fp32 and tf32;
the prior (Adam, lr 3e-4) at B = 32 on 8x8 (K = 512) and B = 16 on 64x64 (K = 1024), in fp32 and tf32.
Nothing is written to the repository tree.
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_prior import _card  # noqa: E402
from bench_prior_train import _split  # noqa: E402

HP = dict(h_dim=128, res_h_dim=32, n_res_layers=2, n_embeddings=512, embedding_dim=64)
PRIOR = {"prior_8x8": dict(B=32, S=8, K=512), "prior_64x64": dict(B=16, S=64, K=1024)}
DIM, LAYERS, CLASSES = 64, 15, 10


def _vqvae_workload(B):
    from models.vqvae import VQVAE
    x = torch.rand((B, 3, 32, 32), device="cuda") - 0.5

    def make():
        torch.manual_seed(0)
        m = VQVAE(*HP.values(), 0.25).cuda().train()

        def loss():
            embedding_loss, x_hat, _ = m(x)
            return torch.mean((x_hat - x) ** 2) / 0.0625 + embedding_loss
        return m, loss, m.repack
    return make, dict(lr=3e-4, amsgrad=True)


def _prior_workload(B, S, K, precision):
    from pixelcnn.models import GatedPixelCNN
    x = torch.randint(0, K, (B, S, S), device="cuda")
    lab = torch.randint(0, CLASSES, (B,), device="cuda")

    def make():
        torch.manual_seed(0)
        with contextlib.redirect_stdout(io.StringIO()):
            m = GatedPixelCNN(K, DIM, LAYERS, CLASSES).cuda()
        m.precision = precision

        def loss():
            logits = m(x, lab).permute(0, 2, 3, 1).contiguous()
            return torch.nn.functional.cross_entropy(logits.view(-1, K), x.view(-1))
        return m, loss, lambda: m._net([])
    return make, dict(lr=3e-4)


def _arms(make, hp):
    from vqvae_b200 import ops
    from vqvae_b200.optim import Adam

    def backward(m, loss):
        for p in m.parameters():
            p.grad = None
        with torch.enable_grad():
            loss().backward()

    arms, launches = {}, {}
    m, loss, repack = make()
    backward(m, loss)
    opt = torch.optim.Adam(m.parameters(), **hp)
    arms["torch_phase"] = [("optimizer", lambda: (opt.step(), repack()))]
    m2, loss2, _ = make()
    backward(m2, loss2)
    opt2 = Adam(m2.parameters(), **hp)
    arms["fused_phase"] = [("optimizer", opt2.step)]
    m3, loss3, _ = make()
    opt3 = Adam(m3.parameters(), **hp)

    def eager():
        backward(m3, loss3)
        opt3.step()
    arms["eager_step"] = [("step", eager)]
    m4, loss4, _ = make()
    opt4 = Adam(m4.parameters(), **hp)

    def step4():
        backward(m4, loss4)
        opt4.step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step4()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    n0 = ops.launch_count()
    with torch.cuda.graph(graph):
        step4()
    launches["graph_step"] = ops.launch_count() - n0
    arms["graph_step"] = [("step", graph.replay)]
    for arm in ("torch_phase", "fused_phase", "eager_step"):
        fn = arms[arm][0][1]
        fn()                                # packings and state exist before counting
        torch.cuda.synchronize()
        n0 = ops.launch_count()
        fn()
        launches[arm] = ops.launch_count() - n0
    return arms, launches


def bench(make, hp, iters):
    arms, launches = _arms(make, hp)
    res = _split(arms, iters)
    out = {}
    for arm, r in res.items():
        out[arm] = dict(ms=r["step_ms"], launches_per_step=launches[arm])
    out["fused_phase_vs_torch_phase"] = out["torch_phase"]["ms"] / out["fused_phase"]["ms"]
    out["graph_vs_eager_step"] = out["eager_step"]["ms"] / out["graph_step"]["ms"]
    return out


def main():
    import vqvae_b200
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    name, power = _card()
    res = dict(gpu=name, power_limit_w=power, iters=a.iters)
    for B in (32, 256):
        for mode in ("fp32", "tf32"):
            with vqvae_b200.precision(mode):
                make, hp = _vqvae_workload(B)
                res[f"vqvae_B{B}_{mode}"] = bench(make, hp, a.iters)
            torch.cuda.empty_cache()
    for w, cfg in PRIOR.items():
        for mode in ("fp32", "tf32"):
            make, hp = _prior_workload(cfg["B"], cfg["S"], cfg["K"], mode)
            res[f"{w}_B{cfg['B']}_{mode}"] = bench(make, hp, a.iters)
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

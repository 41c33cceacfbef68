"""Time the EMA codebook's dead-code restart (ops.vq_ema_restart, vqb_vq_ema_restart_f32) and the VQ-VAE training step
with restarts on, and print one JSON line.

  python tools/bench_vq_restart.py [--reps 50] [--steps 30] [--quick]

Restart: D = 64, N in {16 384, 524 288, 2^20} x K in {512, 1024, 8192}, with no code dead, half the codes dead and
every code dead (t = 0.5).  A restarted code's cluster size becomes t, which is not below t, so each timed call first
resets the K cluster sizes (one K-float copy, timed on its own as reset_ms); each call also draws its uniforms with
torch.rand, as the module does.  Timed with CUDA events around --reps back-to-back calls, eager and as --reps replays of
a graph holding one call.  The baseline restates the restart in torch without a host synchronisation (stable sort of
u, cumsum of the dead flags, gathers and where); its outputs are compared with ours on the same u.  The EMA update at
the same shape (uniform codes) is timed beside it.

Training step: main.py's model (h_dim 128, res_h_dim 32, 2 residual layers, K 512, D 64, ema_decay 0.99) on 32x32
images at B = 32 and B = 256, TF32, forward + loss + backward + vqvae_b200.optim.Adam(amsgrad, lr 3e-4), with
restarts off, on with no code dead (t = 1e-6) and on with every code dead (t = 1e30); median of --steps eager steps
(host clock around a synchronised step) and the mean of --steps replays of the step captured as one CUDA graph; the
arms alternate over two rounds.  The card's name and power limit are printed beside the numbers.  Nothing is written
to the tree.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_vq_ema import as_graph, card, timed  # noqa: E402

SIZES = [(N, K) for N in (16384, 524288, 1 << 20) for K in (512, 1024, 8192)]
D = 64
T = 0.5


def torch_restart(z, u, t, Nk, m, e, cnt):
    """The baseline: the restart restated with torch ops, graph-capturable (no nonzero, no host sync)."""
    N = z.shape[0]
    order = torch.sort(u, stable=True).indices                  # rows by (u, i)
    dead = Nk < t
    rank = torch.cumsum(dead.to(torch.int32), 0) - 1            # j of each dead code
    sel = dead & (rank < N)
    rows = order[rank.clamp(0, N - 1)]
    zr = z[rows]
    e.copy_(torch.where(sel[:, None], zr, e))
    m.copy_(torch.where(sel[:, None], zr * t, m))
    Nk.copy_(torch.where(sel, torch.full_like(Nk, t), Nk))
    cnt.copy_(sel.sum().to(torch.int32).reshape(1))


def restart_point(ops, N, K, case, reps):
    g = torch.Generator().manual_seed(N + K)
    z = torch.randn((N, D), generator=g).cuda()
    kk = torch.arange(K, device="cuda")
    N0 = {"none": torch.ones(K, device="cuda"), "half": (kk % 2 == 0).float(),
          "all": torch.zeros(K, device="cuda")}[case]
    e0 = torch.randn(K, D, generator=g).cuda()
    ours_st = [N0.clone(), e0.clone(), e0.clone()]
    base_st = [N0.clone(), e0.clone(), e0.clone()]
    c_ours, c_base = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")

    # outputs compared on one u
    u = torch.rand((N,), device="cuda")
    ops.vq_ema_restart(z, u, T, *ours_st, c_ours)
    torch_restart(z, u, T, *base_st, c_base)
    torch.cuda.synchronize()
    same = all(torch.equal(a, b) for a, b in zip(ours_st + [c_ours], base_st + [c_base]))
    restarted = int(c_ours)

    def reset():
        ours_st[0].copy_(N0)

    def ours():
        ours_st[0].copy_(N0)
        ops.vq_ema_restart(z, torch.rand((N,), device="cuda"), T, *ours_st, c_ours)

    def base():
        base_st[0].copy_(N0)
        torch_restart(z, torch.rand((N,), device="cuda"), T, *base_st, c_base)

    idx = torch.randint(0, K, (N,), generator=g).cuda()
    hist = torch.bincount(idx, minlength=K).to(torch.int32)
    ust = [torch.ones(K, device="cuda"), e0.clone(), e0.clone()]

    def update():
        ops.vq_ema_update(z, idx, hist, 0.99, 1e-5, *ust)
    for f in (ours, base, update):
        f(), f()
    return {"N": N, "K": K, "D": D, "dead": case, "restarted": restarted, "outputs_equal_torch": same,
            "ours_ms": timed(ours, reps), "ours_graph_ms": timed(as_graph(ours), reps),
            "torch_ms": timed(base, reps), "torch_graph_ms": timed(as_graph(base), reps),
            "reset_graph_ms": timed(as_graph(reset), reps), "ema_update_graph_ms": timed(as_graph(update), reps)}


def train_point(B, threshold, steps):
    import vqvae_b200
    from vqvae_b200.optim import Adam
    torch.manual_seed(0)
    m = vqvae_b200.VQVAE(128, 32, 2, 512, 64, 0.25, ema_decay=0.99).cuda().train()
    m.vector_quantization.dead_code_threshold = threshold
    opt = Adam(m.parameters(), lr=3e-4, amsgrad=True)
    x = torch.rand((B, 3, 32, 32), device="cuda") - 0.5

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.enable_grad():
            embedding_loss, x_hat, _ = m(x)
            loss = torch.mean((x_hat - x) ** 2) / 0.0625 + embedding_loss
            loss.backward()
        opt.step()
        return loss
    for _ in range(3):
        step()
    times = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        step()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    replay = as_graph(step)
    return {"B": B, "threshold": threshold, "eager_ms": statistics.median(times), "graph_ms": timed(replay, steps),
            "last_restarts": int(m.vector_quantization.last_restarts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--quick", action="store_true", help="first size only, few repetitions")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vq_restart.py needs a GPU")
    from vqvae_b200 import ops
    sizes = SIZES[:1] if a.quick else SIZES
    reps, steps = (5, 5) if a.quick else (a.reps, a.steps)
    restart = [restart_point(ops, N, K, case, reps) for N, K in sizes for case in ("none", "half", "all")]
    train = []
    import vqvae_b200
    with vqvae_b200.precision("tf32"):
        for B in ((32,) if a.quick else (32, 256)):
            for rnd in range(2):                  # alternate the arms to expose drift
                for threshold in (None, 1e-6, 1e30):
                    r = train_point(B, threshold, steps)
                    r["round"] = rnd
                    train.append(r)
    print(json.dumps({"card": card(), "restart": restart, "train_step": train}))


if __name__ == "__main__":
    main()

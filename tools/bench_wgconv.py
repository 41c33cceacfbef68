"""Time every wgmma convolution launch (wgconv_kernel) of the benchmark's forwards alone, and set it against the
shared-memory traffic it needs.

  python tools/bench_wgconv.py [--iters N] [--reps R]

One eager VQVAE.forward per setting (cfg2 in tf32 and bf16, cfg3 in bf16; bench.py's shapes and seeded weights)
records every C-ABI call that runs on wgconv_kernel.  Each is then replayed on its own, back to back, `iters` times
between two CUDA events, `reps` times; the median per-launch time is reported.  The replays reuse the recorded device
pointers, which the caching allocator keeps mapped; only timing is read from them.

Beside each time: the modelled L2->SM bytes of the launch under two operand schemes -- "per-tap" (one 128-pixel A box
per k-step, what wgconv_kernel loads) and "halo" (each tile's input halo once per chunk, the alternative) -- both with
the N weight rows of every k-step, and the achieved bytes/s of each; the algorithmic FLOP/s; the card name and power
limit.  The output layer (convT to <= 4 channels) runs in scatter form, which loads each tile's halo once per chunk,
and so do the TF32 residual launches whose tiles hold whole images (res_scatter_kernel, which loads each tile once
for all applications): both columns give those launches' bytes.  A latent block (the k3 conv, the stack and the
encoder's 1x1 conv in one res_scatter_kernel launch) adds its head conv's per-tap boxes and the tail's weight.  The
decoder tail (the k4 s2 transposed conv and the output layer in one wgconv_kernel launch) is the transposed conv's
traffic with one CTA per tile for all four phases, plus the output layer's gathered weight once per CTA: its input h
stays in shared memory.  Prints one JSON line.  Nothing is written to the repository tree.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WGCONV_CALLS = {"vqb_conv2d_f32", "vqb_conv2d_bf16", "vqb_residual_layer_f32", "vqb_residual_stack_f32",
                "vqb_residual_layer_bf16", "vqb_latent_block_tf32", "vqb_decoder_tail_tf32"}


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = float(q.stdout.strip().splitlines()[0])
    except Exception:           # no nvidia-smi: the number is reported without it
        power = None
    return name, power


def _p2(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def layers(label):
    """The layer labels of one launch: a latent block's label ("res x2 128->32->128 8x8 +conv 128->128 k3s1 +conv
    128->64 k1s1") names its stack and, after each "+", a conv at the stack's resolution; a decoder tail's ("convT
    128->64 k4s2 8x8 +convT 64->3 k4s2") names the k4 s2 transposed conv and the output layer, which runs at that
    conv's output resolution."""
    parts = label.split(" +")
    hw = parts[0].split()[-1]
    if parts[0].split()[0] == "convT" and parts[0].split()[2] == "k4s2":
        h, w = (int(v) for v in hw.split("x"))
        hw = f"{2 * h}x{2 * w}"
    return [parts[0]] + [p + " " + hw for p in parts[1:]]


def traffic(label, B):
    """(CTAs, k-steps per CTA, per-tap bytes, halo bytes) of one wgconv launch, from its ops label.  Tile shape as
    launch_wgconv picks it; 128-byte rows; weights: N rows per k-step (+ the chained 1x1 weight once per CTA)."""
    bf = label.startswith("bf16 ")
    extra = [p.split() for p in layers(label)[1:]]
    parts = (label[5:] if bf else label).split(" +")[0].split()
    ck = 64 if bf else 32
    napps = 1
    if parts[0] == "res":
        if parts[1].startswith("x"):
            napps = int(parts[1][1:])
            parts = [parts[0]] + parts[2:]
        c, cm, _ = (int(v) for v in parts[1].split("->"))
        h, w = (int(v) for v in parts[2].split("x"))
        if not bf and cm == 32 and c in (64, 128) and w <= 16 and _p2(w) * _p2(h) <= 128:
            # scatter form (res_scatter_kernel): the whole-image tile once, then per application 3 passes x nc chunks
            # of 96 weight rows (one kernel row's taps), and the 1x1 weight once per CTA; both schemes alike
            nc = c // 32
            ctas = -(-B // (128 // (_p2(w) * _p2(h))))
            moved = ctas * (nc * 128 * 128 + napps * 3 * nc * 96 * 128 + c * 128)
            ksteps = napps * 3 * nc
            for conv in extra:
                cin_, cout_ = (int(v) for v in conv[1].split("->"))
                if conv[2] == "k3s1":
                    # the head conv (latent block): the separate launch's per-tap A boxes and C weight rows per k-step,
                    # in place of loading the tile
                    moved += ctas * (9 * (cin_ // 32) * (128 * 128 + cout_ * 128) - nc * 128 * 128)
                    ksteps += 9 * (cin_ // 32)
                else:                              # the 1x1 tail: its weight once per CTA
                    moved += ctas * cout_ * cin_ * 4
                    ksteps += cin_ // 32
            return ctas, ksteps, moved, moved
        cin, N, nph, taps, step, ext = c, _p2(max(cm, 16)), 1, 9, 1, 2
        w2 = c * 128 * (1 if bf else max(cm // 32, 1))
        grid = [(h, w)]
    else:
        transposed = parts[0] == "convT"
        cin, cout = (int(v) for v in parts[1].split("->"))
        k = int(parts[2][1:parts[2].index("s")])
        s = int(parts[2][parts[2].index("s") + 1:])
        h, w = (int(v) for v in parts[3].split("x"))
        w2 = 0
        if transposed and s == 2 and cout <= 4:
            # scatter-form output layer (convt_scatter_kernel): each tile's (TW + 2) x (TH + 2) halo once per chunk,
            # the 64 gathered weight rows once per persistent CTA (two per SM of a 132-SM H100); both schemes alike
            nc = (cin + ck - 1) // ck
            tx = -(-w // 16)
            tw = -(-w // tx)
            ty = -(-h // (128 // (tw + 2) - 2))
            th = -(-h // ty)
            tiles = tx * ty * B
            ctas = min(tiles, 2 * 132)
            moved = tiles * nc * (tw + 2) * (th + 2) * 128 + ctas * nc * 64 * 128
            return ctas, -(-tiles // ctas) * nc, moved, moved
        elif transposed and s == 2:                    # four sub-pixel phases of 2x2 taps
            N, nph, taps, step, ext, grid = _p2(max(cout, 16)), 4, 4, 1, 1, [(h, w)] * 4
        elif transposed or k == 3:
            N, nph, taps, step, ext, grid = _p2(max(cout, 16)), 1, 9, 1, 2, [(h, w)]
        elif k == 1:
            N, nph, taps, step, ext, grid = _p2(max(cout, 16)), 1, 1, 1, 0, [(h, w)]
        else:                                          # k4 s2 conv
            N, nph, taps, step, ext, grid = _p2(max(cout, 16)), 1, 16, 2, 3, [(h // 2, w // 2)]
    nc = (cin + ck - 1) // ck
    oh, ow = grid[0]
    BW = min(_p2(ow), 16)
    BH = min(_p2(oh), 128 // BW)
    BN = 128 // (BW * BH)
    ctas = -(-ow // BW) * -(-oh // BH) * -(-B // BN) * nph
    a = taps * nc
    halo_px = BN * ((BW - 1) * step + ext + 1) * ((BH - 1) * step + ext + 1)
    wbytes = ctas * (napps * a * N * 128 + w2)
    per_tap = ctas * napps * a * 128 * 128 + wbytes
    halo = ctas * napps * halo_px * nc * 128 + wbytes
    ksteps = napps * a
    if extra:
        # decoder tail: one CTA per tile runs the four phases, then gathers the output layer's 64 live weight rows per
        # 32-channel chunk of h once; h itself never leaves shared memory
        ctas //= nph
        ksteps *= nph
        per_tap += ctas * (cout // 32) * 64 * 128
        halo += ctas * (cout // 32) * 64 * 128
    return ctas, ksteps, per_tap, halo


def record(model, x):
    """The wgconv C-ABI calls of one eager forward: [(label, fn, args)] in call order."""
    from vqvae_b200 import ops
    real = ops.lib()
    calls, last = [], {}

    class Span(ops._Span):
        def __init__(self, label):
            super().__init__(label)
            last["label"] = label

    class Proxy:
        def __getattr__(self, name):
            fn = getattr(real, name)
            if name not in WGCONV_CALLS:
                return fn

            def rec(*args):
                label = last.get("label", name)
                if " 3->" not in label:                # the CUDA-core input conv
                    calls.append((label, fn, args))
                return fn(*args)
            return rec

    saved = ops.lib, ops._Span
    ops.lib, ops._Span = (lambda: Proxy()), Span
    try:
        with torch.no_grad():
            model(x)
        torch.cuda.synchronize()
    finally:
        ops.lib, ops._Span = saved
    return calls


def time_call(fn, args, iters, reps):
    for _ in range(10):
        fn(*args)
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn(*args)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / iters)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_wgconv.py needs a GPU"
    torch.cuda.set_device(0)
    import bench
    import vqvae_b200
    from vqvae_b200.synth import make_images

    card, power = _card()
    out = {"card": card, "power_limit_w": power, "iters": args.iters, "reps": args.reps, "settings": []}
    for wl_name, prec in (("cfg2", "tf32"), ("cfg2", "bf16"), ("cfg3", "bf16")):
        wl = bench.WORKLOADS[wl_name]
        model, _ = bench.build_model(wl, torch.device("cuda", 0))
        x = torch.from_numpy(make_images(wl["batch"], wl["size"], seed=1)).cuda()
        rows = []
        with vqvae_b200.precision(prec):
            with torch.no_grad():
                model(x)                               # packs weights, sizes workspaces
            torch.cuda.synchronize()
            for label, fn, cargs in record(model, x):
                ms = time_call(fn, cargs, args.iters, args.reps)
                ctas, ksteps, per_tap, halo = traffic(label, wl["batch"])
                flops = sum(bench.layer_model(part, wl["batch"], wl["K"], wl["D"])[0] for part in layers(label))
                rows.append(dict(launch=label, ms=round(ms, 5), ctas=ctas, ksteps_per_cta=ksteps,
                                 per_tap_MB=round(per_tap / 1e6, 1), halo_MB=round(halo / 1e6, 1),
                                 per_tap_TBps=round(per_tap / (ms * 1e-3) / 1e12, 2),
                                 halo_TBps=round(halo / (ms * 1e-3) / 1e12, 2),
                                 TFLOPps=round(flops / (ms * 1e-3) / 1e12, 1)))
        tot = sum(r["ms"] for r in rows)
        out["settings"].append(dict(workload=wl_name, precision=prec, wgconv_ms=round(tot, 4), launches=rows))
        for r in rows:
            print("%s %s  %-32s %8.4f ms  per-tap %6.1f MB %5.2f TB/s  halo %6.1f MB %5.2f TB/s  %6.1f TFLOP/s"
                  % (wl_name, prec, r["launch"], r["ms"], r["per_tap_MB"], r["per_tap_TBps"], r["halo_MB"],
                     r["halo_TBps"], r["TFLOPps"]), file=sys.stderr)
        print("%s %s wgconv total %.4f ms (%s, %s W)" % (wl_name, prec, tot, card, power), file=sys.stderr)
        del model
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

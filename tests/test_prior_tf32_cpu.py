"""CPU checks of the Gated PixelCNN prior's TF32 mode: the `precision` attribute, the TF32 entry points' declarations
and argument checks, and the emulated-TF32 restatement's helpers: its roundings, its evaluation at given activations,
and the decoder of the training forward's saved activations."""
import ctypes
import os
import re

import pytest
import torch

from tests.prior_tf32_port import (decode_saved, encode_saved, prior_logits_tf32, saved_offsets, saved_points,
                                   tf32_round, tf32_truncate)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAIRS = [("vqb_prior_forward_tf32", "vqb_prior_forward_f32"),
         ("vqb_prior_forward_train_tf32", "vqb_prior_forward_train_f32"),
         ("vqb_prior_backward_tf32", "vqb_prior_backward_f32"),
         ("vqb_prior_workspace_bytes_tf32", "vqb_prior_workspace_bytes")]


def test_precision_defaults_to_fp32_and_stays_out_of_the_state_dict():
    from pixelcnn.models import GatedPixelCNN
    m = GatedPixelCNN(37, 32, 2, 3)
    assert m.precision == "fp32"
    keys = list(m.state_dict())
    m.precision = "tf32"
    assert list(m.state_dict()) == keys and not any("precision" in k for k in keys)


@pytest.mark.parametrize("bad", ["bf16", "TF32", None, 32])
def test_other_precisions_raise_before_any_launch(bad):
    from pixelcnn.models import GatedPixelCNN
    m = GatedPixelCNN(37, 32, 2, 3)
    m.precision = bad
    for grad in (False, True):
        with torch.set_grad_enabled(grad), pytest.raises(ValueError, match="precision"):
            m(torch.zeros((2, 5, 5), dtype=torch.int64), torch.zeros(2, dtype=torch.int64))


def test_ops_take_a_precision_keyword_defaulting_to_fp32():
    import inspect
    from vqvae_b200 import ops
    for fn in (ops.prior_forward, ops.prior_forward_train, ops.prior_backward):
        assert inspect.signature(fn).parameters["precision"].default == "fp32"
    with pytest.raises(ValueError):
        ops._prior_precision("bf16")


def _prototype(src, name):
    m = re.search(r"\b(\w+\s*\*?)\s*\b" + name + r"\s*\(([^;]*)\)\s*;", src)
    assert m, name
    return m.group(1).strip(), [re.sub(r"\s+", " ", a).strip() for a in m.group(2).split(",")]


def test_tf32_entry_points_have_the_fp32_signatures():
    from vqvae_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "vqvae_b200.h")).read(), flags=re.S)
    for tf32, f32 in PAIRS:
        assert _prototype(src, tf32) == _prototype(src, f32), tf32
        assert _lib.SIGNATURES[tf32] == _lib.SIGNATURES[f32], tf32


def test_tf32_entry_points_validate_arguments_like_fp32_without_a_gpu():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.vqb_prior_workspace_bytes_tf32(0, 4, 4, 32, 2, 16) == 0
    assert lib.vqb_prior_workspace_bytes_tf32(2, 4, 4, 32, 2, 16) == 4 * 2 * 4 * 4 * (11 * 32 + 512)
    lw = _lib.PriorLayerWeights(*([p.value] * 9), 3, 0, 1)
    layers = (_lib.PriorLayerWeights * 2)(lw, lw)

    def net(**kw):
        a = dict(layers=layers, n_layers=2, embedding=p.value, out1_w=p.value, out1_b=p.value, out2_w=p.value,
                 out2_b=p.value, input_dim=16, dim=32, n_classes=2)
        a.update(kw)
        return ctypes.byref(_lib.PriorNet(**a))

    ws = lib.vqb_prior_workspace_bytes_tf32(1, 4, 4, 32, 2, 16)
    sv = lib.vqb_prior_train_saved_bytes(1, 4, 4, 32, 2)
    bws = lib.vqb_prior_backward_workspace_bytes(net(), 1, 4, 4)
    lg = _lib.PriorLayerGrads(*([p.value] * 9))
    grads = ctypes.byref(_lib.PriorGrads(layers=(_lib.PriorLayerGrads * 2)(lg, lg), n_layers=2,
                                         **{k: p.value for k in ("embedding", "out1_w", "out1_b", "out2_w", "out2_b")}))
    calls = {
        "forward": (lambda n, sfx, **kw: getattr(lib, "vqb_prior_forward_" + sfx)(
            n, kw.get("codes", p), p, 1, 4, kw.get("W", 4), p, p, kw.get("ws", ws if sfx == "tf32" else 1 << 20), None)),
        "forward_train": (lambda n, sfx, **kw: getattr(lib, "vqb_prior_forward_train_" + sfx)(
            n, kw.get("codes", p), p, 1, 4, kw.get("W", 4), p, p, kw.get("ws", sv), None)),
        "backward": (lambda n, sfx, **kw: getattr(lib, "vqb_prior_backward_" + sfx)(
            n, kw.get("codes", p), p, 1, 4, kw.get("W", 4), p, p, grads, p, kw.get("ws", bws), None)),
    }
    for what, call in calls.items():
        cases = [dict(n=None), dict(n=net(), codes=None), dict(n=net(), W=0), dict(n=net(), ws=4),
                 dict(n=net(dim=40)), dict(n=net(input_dim=8193)), dict(n=net(n_layers=33))]
        for kw in cases:
            n = kw.pop("n")
            got, want = call(n, "tf32", **kw), call(n, "f32", **kw)
            assert got == want and got != 0, (what, kw, got, want)


def test_tf32_rounding_of_chosen_bit_patterns():
    def bits(*u):
        return torch.tensor(u, dtype=torch.int64).to(torch.int32).view(torch.float32)

    x = bits(0x3F800000,          # 1.0: kept
             0x3F800FFF,          # just below half an ulp: down
             0x3F801000,          # exactly half, even kept bit: away from zero (up)
             0x3F803000,          # exactly half, odd kept bit: up
             0x3F801FFF,          # above half: up
             0xBF801000 - (1 << 32),   # -(half): away from zero
             0x3F9FF000,          # carry into the next ulp
             0x3FFFF000,          # carry into the exponent: 2.0
             0x00000FFF,          # subnormal: down to 0
             0x00001000,          # subnormal half: up
             0x80000000 - (1 << 32))   # -0.0 stays -0.0
    want = bits(0x3F800000, 0x3F800000, 0x3F802000, 0x3F804000, 0x3F802000, 0xBF802000 - (1 << 32), 0x3FA00000,
                0x40000000, 0x00000000, 0x00002000, 0x80000000 - (1 << 32))
    got = tf32_round(x)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    d = tf32_round(x.double())
    assert d.dtype == torch.float64 and torch.equal(d.float().view(torch.int32), want.view(torch.int32))
    assert int((tf32_round(torch.randn(1000)).view(torch.int32) & 0x1FFF).abs().sum()) == 0


def test_truncation_clears_the_low_13_bits():
    x = torch.tensor([0x3F801FFF, 0xBF803FFF - (1 << 32), 0x00001FFF], dtype=torch.int64).to(torch.int32)
    got = tf32_truncate(x.view(torch.float32).double()).float().view(torch.int32)
    assert got.tolist() == [0x3F800000, 0xBF802000 - (1 << 32), 0]


@pytest.mark.parametrize("kind", ["ce", "random"])
@pytest.mark.parametrize("name", ["prior_ragged", "kernels", "resid0", "single3", "narrow"])
def test_restatement_at_its_own_activations_is_the_plain_restatement(name, kind):
    """With `at` set to the activations it records itself, the straight-through evaluation changes no value and no
    gradient: logits and every gradient as without `at`."""
    from oracle.prior_port import PRIOR_CASES, PRIOR_SHAPE_CASES, make_prior_inputs, make_prior_state_dict
    from oracle.prior_train_port import leaf_params, prior_loss
    c = PRIOR_CASES.get(name) or PRIOR_SHAPE_CASES[name]
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], c.get("layers"))
    codes, labels, _ = make_prior_inputs(c)
    x, lab = torch.from_numpy(codes), torch.from_numpy(labels)
    up = torch.randn((c["batch"], c["K"], c["size"], c["size"]), generator=torch.Generator().manual_seed(3),
                     dtype=torch.float64)
    runs = []
    for at in (None, "own"):
        record = {}
        with torch.enable_grad():
            g = leaf_params(sd, torch.float64)
            if at == "own":
                prior_logits_tf32(leaf_params(sd, torch.float64), x, lab, c["n_layers"], c.get("layers"),
                                  record=record)
                at, record = record, {}
            lg = prior_logits_tf32(g, x, lab, c["n_layers"], c.get("layers"), at=at, record=record)
            (prior_loss(lg, x) if kind == "ce" else (lg * up).sum()).backward()
        assert list(record) == saved_points(c["n_layers"])
        runs.append((lg.detach(), {k: v.grad for k, v in g.items()}))
    (l0, g0), (l1, g1) = runs
    assert float((l1 - l0).abs().max()) <= 1e-12 * float(l0.abs().max())
    for k in g0:
        assert float((g1[k] - g0[k]).abs().max()) <= 1e-12 * max(float(g0[k].abs().max()), 1e-300), k


@pytest.mark.parametrize("B,H,W,dim,L", [(3, 5, 5, 32, 4), (1, 1, 1, 32, 1), (2, 6, 6, 96, 3), (3, 29, 29, 64, 3)])
def test_saved_decoder_round_trips_and_spans_the_library_buffer(B, H, W, dim, L):
    """Grids written at their offsets come back unchanged (no two overlap), the one grid left unnamed is the 2*dim
    scratch between a layer's launches, and the length is vqb_prior_train_saved_bytes."""
    from vqvae_b200 import _lib
    off, total = saved_offsets(B, H, W, dim, L)
    assert 4 * total == _lib.lib().vqb_prior_train_saved_bytes(B, H, W, dim, L)
    gen = torch.Generator().manual_seed(L)
    grids = {k: torch.randn((B, c, H, W), generator=gen).double() for k, (_, c) in off.items()}
    buf = encode_saved(grids, B, H, W, dim, L)
    assert buf.numel() == total and int(buf.isnan().sum()) == 2 * B * H * W * dim
    got = decode_saved(buf.view(torch.uint8), B, H, W, dim, L)
    assert set(got) == set(grids) >= set(saved_points(L)) | {"xv0"}
    assert all(got[k].dtype == torch.float64 and torch.equal(got[k], grids[k]) for k in grids)

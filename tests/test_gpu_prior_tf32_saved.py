"""The Gated PixelCNN prior's training forward and backward on the H100, checked at the activations the forward kept.

The module path (GatedPixelCNN.forward through _PriorFunction) runs with ops.prior_forward_train / ops.prior_backward
wrapped to keep the `saved` buffer and the d_logits the backward was given.  The restatement of
tests/prior_tf32_port.py is then evaluated at those activations (prior_logits_tf32(at=...)): each forward piece the GPU
kept is one product away from the GPU's own inputs, and the backward takes every gate and ReLU derivative at the GPU's
values, so the comparison does not drift with depth as the plain restatement's does (tests/test_gpu_prior_tf32.py).

Per case of PRIOR_CASES and of PRIOR_SHAPE_CASES with a backward part, for the cross-entropy loss and a random upstream
gradient:
  layout     xv0 is bitwise the embedding rows of the clamped codes, hid >= 0, the decoded length is
             vqb_prior_train_saved_bytes
  forward    every hv, ph, xv, xh, hid and the logits against the restatement at the GPU's inputs
  gradients  every parameter gradient, with bars graded by how many rounded products lie between the tensor and the
             upstream gradient (DESIGN.md section 8.2)
in TF32 against the TF32 restatement, and as a control of the harness and the decoder, in fp32 against the unrounded
restatement.  On one case, the forward pieces are closer to round-to-nearest TF32 operands than to truncated ones.
Each check prints its worst error over its bar."""
import contextlib
import io

import pytest
import torch
import torch.nn.functional as F

from oracle.prior_port import PRIOR_CASES, PRIOR_SHAPE_CASES, make_prior_inputs, make_prior_state_dict
from oracle.prior_train_port import leaf_params, prior_loss
from tests.prior_tf32_port import (decode_saved, no_rounding, prior_logits_tf32, saved_offsets, saved_points,
                                   tf32_round, tf32_truncate)

pytestmark = pytest.mark.gpu

CASES = list(PRIOR_CASES) + [n for n, c in PRIOR_SHAPE_CASES.items() if "backward" in c.get("parts", ["backward"])]

# Bars.
#   Forward pieces and output_conv.2's gradient: one product whose operands are the GPU's own (the saved activations,
#   the weights, d_logits), rounded alike on both sides, so only the fp32 accumulation separates them.  That error
#   scales with the terms, not with their sum: the tensor cores truncate as they accumulate, and a sum that cancels
#   (a logit of a 1x1 grid, a cross-entropy weight gradient) or runs over thousands of terms (a 7x7 layer of dim 256)
#   moves by more than 1e-5 of the result's max.  So these bars are relative to the tensor's largest sum of |terms|
#   (prior_logits_tf32(terms=...)).  xv (a gate of a saved value, no product) is relative to its max |.|.
#   One operand is not saved: xh{l+1} reads gate(ph{l}), which the GPU computes in fp32 with a few ulps of error, so
#   where that value lies within GATE_ULPS of a TF32 rounding midpoint either neighbour is right, and each such
#   operand adds its rounding step times |W| to the bar of the elements it enters (_gate_slack).
FORWARD = 1e-5
GATE_ULPS = 32
#   TF32 gradients other than output_conv.2, relative to the tensor's max |.|.  output_conv.0 reads W2^T d_logits,
#   which the GPU accumulates in fp32 and rounds to TF32 again: a different TF32 neighbour there moves a term by up to
#   2^-11 of it.  The layers and the embedding read upstream gradients that went through that re-rounding once per
#   product back from the head, and the saved activations hold none of them.
GRAD_OUT2, GRAD_OUT0, GRAD_LAYERS = 1e-5, 5e-4, 5e-3
#   fp32 gradients: the fp32 backward's bar against fp64 (tests/test_gpu_prior_train.py)
GRAD_FP32 = 2e-5


def _case(name):
    return PRIOR_CASES.get(name) or PRIOR_SHAPE_CASES[name]


def _model(c, precision):
    from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
    layers = c.get("layers")
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], layers)
    with contextlib.redirect_stdout(io.StringIO()):
        m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
        for i, (mask, k, residual) in enumerate(layers or []):
            m.layers[i] = GatedMaskedConv2d(mask, c["dim"], k, residual, c["n_classes"])
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    m.precision = precision
    codes, labels, _ = make_prior_inputs(c)
    return sd, m.cuda(), torch.from_numpy(codes), torch.from_numpy(labels)


def _upstream(c, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((c["batch"], c["K"], c["size"], c["size"]), generator=g, dtype=torch.float64)


def _capture(monkeypatch, c, precision, kind):
    """Run the module's training forward and backward -> (sd, codes, labels, logits, grads, saved, d_logits)."""
    from vqvae_b200 import ops
    sd, m, x, lab = _model(c, precision)
    kept = {}
    forward_train, backward = ops.prior_forward_train, ops.prior_backward

    def keep_saved(net, codes, labels, precision="fp32"):
        logits, saved = forward_train(net, codes, labels, precision)
        kept["saved"] = saved
        return logits, saved

    def keep_d_logits(net, codes, labels, d_logits, saved, grads, precision="fp32"):
        assert saved is kept["saved"]
        kept["d_logits"] = d_logits.clone()
        backward(net, codes, labels, d_logits, saved, grads, precision)

    monkeypatch.setattr(ops, "prior_forward_train", keep_saved)
    monkeypatch.setattr(ops, "prior_backward", keep_d_logits)
    xc, lc = x.cuda(), lab.cuda()
    with torch.enable_grad():
        out = m(xc, lc)
        if kind == "ce":
            prior_loss(out, xc).backward()
        else:
            out.backward(_upstream(c, 9).float().cuda())
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu() for k, p in m.named_parameters()}
    return sd, x, lab, out.detach().cpu(), grads, kept["saved"].cpu(), kept["d_logits"].double().cpu()


def _restate(c, sd, x, lab, at, d_logits, rounding, terms=None):
    """The restatement at the activations `at` -> (logits, {point: recomputed value}, {key: gradient})."""
    record = {}
    with torch.enable_grad():
        g = leaf_params(sd, torch.float64)
        lg = prior_logits_tf32(g, x, lab, c["n_layers"], c.get("layers"), at=at, record=record, rounding=rounding,
                               terms=terms)
        (lg * d_logits).sum().backward()
    return lg.detach(), record, {k: v.grad for k, v in g.items()}


def _decode(c, saved):
    from vqvae_b200 import _lib
    B, S, C, L = c["batch"], c["size"], c["dim"], c["n_layers"]
    _, total = saved_offsets(B, S, S, C, L)
    assert saved.numel() == 4 * total == _lib.lib().vqb_prior_train_saved_bytes(B, S, S, C, L)
    return decode_saved(saved, B, S, S, C, L)


def _gate_slack(c, sd, sv, l, rounding):
    """Per element of xh{l+1}: what the operand gate(ph{l}) can move it by when the GPU's fp32 gate and the fp64 one
    round to different neighbours: sum over inputs of |rounding step within GATE_ULPS| * |rounded W_resid|."""
    C, ph = c["dim"], sv[f"ph{l}"]
    g = torch.tanh(ph[:, :C]) * torch.sigmoid(ph[:, C:])
    d = g.abs() * GATE_ULPS * 2.0 ** -23
    step = (rounding(g + d) - rounding(g - d)).abs()
    w = rounding(torch.from_numpy(sd[f"layers.{l}.horiz_resid.weight"]).double()).abs()
    return F.conv2d(step, w)


def _rel_slack(got, want, scale, slack=0):
    """max (|got - want| - slack)^+ / max scale"""
    d = ((got.double().cpu() - want).abs() - slack).clamp_min(0)
    return float(d.max() / scale.abs().max().clamp_min(1e-30))


def _forward_errors(c, sd, sv, out, lg, rec, terms, rounding):
    """{piece: worst error over its scale} of every saved forward piece and the logits."""
    err = {}
    for k, v in rec.items():
        slack = _gate_slack(c, sd, sv, int(k[2:]) - 1, rounding) if k.startswith("xh") else 0
        err[k] = _rel_slack(sv[k], v, terms.get(k, v), slack)
    err["logits"] = _rel_slack(out, lg, terms["logits"])
    return err


def _out2_terms(dl, hid, rounding):
    """Sum of |terms| of each element of output_conv.2's gradients: |rnd(d_logits)|^T |rnd(hid)| and sum |rnd(d_logits)|"""
    a, h = rounding(dl).abs(), rounding(hid).abs()
    return {"output_conv.2.weight": torch.einsum("bkhw,bchw->kc", a, h)[:, :, None, None],
            "output_conv.2.bias": a.sum((0, 2, 3))}


def _grad_bar(key, tf32):
    if not tf32:
        return GRAD_FP32
    return GRAD_OUT2 if key.startswith("output_conv.2.") else GRAD_OUT0 if key.startswith("output_conv.0.") \
        else GRAD_LAYERS


def _check(monkeypatch, name, kind, precision):
    tf32 = precision == "tf32"
    c = _case(name)
    sd, x, lab, out, got, saved, dl = _capture(monkeypatch, c, precision, kind)
    sv = _decode(c, saved)
    # layout: the embedding gather and the hidden layer's ReLU
    emb = torch.from_numpy(sd["embedding.weight"]).double()
    assert torch.equal(sv["xv0"], emb[x.clamp(0, c["K"] - 1)].permute(0, 3, 1, 2)), "xv0 is not the embedding"
    assert bool((sv["hid"] >= 0).all()), "hid has negative values"
    at = {k: sv[k] for k in saved_points(c["n_layers"])}
    rounding = tf32_round if tf32 else no_rounding
    terms = {}
    lg, rec, want = _restate(c, sd, x, lab, at, dl, rounding, terms)
    fwd = _forward_errors(c, sd, sv, out, lg, rec, terms, rounding)
    worst_f = max(fwd, key=fwd.get)
    assert all(got[k].shape == want[k].shape and got[k].dtype == torch.float32 for k in want)
    if c["K"] == 1 and kind == "ce":                # log_softmax of one logit is 0: no gradient anywhere
        assert float(dl.abs().max()) == 0
        assert all(float(got[k].abs().max()) == 0 and float(want[k].abs().max()) == 0 for k in want)
        grad = {}
    else:
        scale = _out2_terms(dl, sv["hid"], rounding) if tf32 else {}
        grad = {k: _rel_slack(got[k], want[k], scale.get(k, want[k])) / _grad_bar(k, tf32) for k in want}
    groups = {"output_conv.2": [k for k in grad if k.startswith("output_conv.2.")],
              "output_conv.0": [k for k in grad if k.startswith("output_conv.0.")],
              "layers+embedding": [k for k in grad if not k.startswith("output_conv.")]}
    line = [f"forward {fwd[worst_f] / FORWARD:.3f} ({worst_f}: {fwd[worst_f]:.2e})"]
    for gname, keys in groups.items():
        if keys:
            k = max(keys, key=grad.get)
            line.append(f"{gname} {grad[k]:.3f} ({k}: {grad[k] * _grad_bar(k, tf32):.2e})")
    print(f"{name} {precision} {kind}: worst / bar: " + ", ".join(line))
    assert fwd[worst_f] <= FORWARD, (worst_f, fwd[worst_f])
    bad = {k: v for k, v in grad.items() if v > 1}
    assert not bad, {k: f"{v * _grad_bar(k, tf32):.2e}" for k, v in bad.items()}


@pytest.mark.parametrize("kind", ["ce", "random"])
@pytest.mark.parametrize("name", CASES)
def test_tf32_forward_and_gradients_at_the_saved_activations(monkeypatch, name, kind):
    _check(monkeypatch, name, kind, "tf32")


@pytest.mark.parametrize("kind", ["ce", "random"])
@pytest.mark.parametrize("name", CASES)
def test_fp32_forward_and_gradients_at_the_saved_activations(monkeypatch, name, kind):
    """The same harness on the fp32 kernels against the unrounded restatement: the decoder and the straight-through
    evaluation are right independently of TF32."""
    _check(monkeypatch, name, kind, "fp32")


def test_tf32_products_round_their_operands_to_nearest(monkeypatch):
    """Every forward product is nearer the restatement with round-to-nearest TF32 operands (cvt.rna, DESIGN.md
    section 8.2) than with truncated ones: mean |GPU - restatement| under half of truncation's, product by product."""
    c = _case("prior_default")
    sd, x, lab, out, _, saved, dl = _capture(monkeypatch, c, "tf32", "random")
    sv = _decode(c, saved)
    at = {k: sv[k] for k in saved_points(c["n_layers"])}
    err = {}
    for rounding in (tf32_round, tf32_truncate):
        lg, rec, _ = _restate(c, sd, x, lab, at, dl, rounding)
        rec = {k: v for k, v in rec.items() if not k.startswith("xv")}     # gates of saved values: no product
        err[rounding] = {k: float((sv[k] - v).abs().mean()) for k, v in rec.items()}
        err[rounding]["logits"] = float((out.double() - lg).abs().mean())
    ratio = {k: err[tf32_round][k] / err[tf32_truncate][k] for k in err[tf32_round]}
    worst = max(ratio, key=ratio.get)
    print(f"prior_default: mean error, round to nearest over truncation: worst {ratio[worst]:.2e} ({worst}), "
          f"logits {ratio['logits']:.2e}")
    assert ratio[worst] < 0.5, (worst, ratio[worst])

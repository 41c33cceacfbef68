"""An fp64 restatement of GatedPixelCNN.cross_entropy's options (weight, ignore_index, label_smoothing) -- TEST
INFRASTRUCTURE ONLY; the product never imports this module.

``ce_options`` is the per-position formula of DESIGN §8.3 written out on (N, K) logits and raw codes (N,):
y = clamp(code, 0, K - 1), lse the row's log-sum-exp, w the weights (ones for None), W = sum_k w_k, e the smoothing:
  loss_p = (1 - e) * w_y * (lse - l_y) + (e / K) * (W * lse - sum_k w_k * l_k), 0 where code == ignore_index;
"sum" adds loss_p, "mean" divides that by the sum of w_y over the positions not ignored (NaN when it is 0).
``torch_ce`` is torch's F.cross_entropy with the same conventions: targets clamped, ignore_index None meaning nothing
is ignored (the raw code compared, as the product does, by mapping ignored positions to torch's -100).
"""
import torch
import torch.nn.functional as F


def ce_options(logits, codes, weight=None, ignore_index=None, label_smoothing=0.0, reduction="mean"):
    l = logits.double()
    N, K = l.shape
    w = torch.ones(K, dtype=torch.float64) if weight is None else weight.double().cpu().to(l.device)
    y = codes.clamp(0, K - 1)
    ign = (codes == ignore_index) if ignore_index is not None else torch.zeros(N, dtype=torch.bool, device=l.device)
    lse = torch.logsumexp(l, dim=1)
    wy = w[y]
    e = float(label_smoothing)
    loss = (1 - e) * wy * (lse - l.gather(1, y[:, None])[:, 0]) + (e / K) * (w.sum() * lse - l @ w)
    loss = torch.where(ign, torch.zeros_like(loss), loss)
    if reduction == "none":
        return loss
    if reduction == "sum":
        return loss.sum()
    den = torch.where(ign, torch.zeros_like(wy), wy).sum()
    return loss.sum() / den if float(den) != 0.0 else torch.tensor(float("nan"), dtype=torch.float64)


def torch_ce(logits, codes, weight=None, ignore_index=None, label_smoothing=0.0, reduction="mean"):
    """F.cross_entropy on (N, K) logits with the product's target and ignore conventions"""
    K = logits.shape[1]
    target = codes.clamp(0, K - 1)
    if ignore_index is not None:
        target = torch.where(codes == ignore_index, torch.full_like(target, -100), target)
    return F.cross_entropy(logits, target, weight=weight, ignore_index=-100, label_smoothing=label_smoothing,
                           reduction=reduction)

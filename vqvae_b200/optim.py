"""On-device Adam for both models: a drop-in for the ``torch.optim.Adam`` that the reference's ``main.py`` and
``gated_pixelcnn.py`` construct.

``step()`` is two library launches per parameter group (csrc/optim.cu): ``vqb_adam_multi_f32`` updates every
parameter that has a gradient, with its moments, in the arithmetic of torch's single-tensor Adam; ``vqb_repack_multi``
then rebuilds every weight packing cached on those parameters (``_vqb_packed``, whatever its key: the forward's, the
input-gradient one a backward created, bf16 and the prior's kept-tap packings), zeroes a mask-A layer's excluded taps
in the parameter (what ``GatedMaskedConv2d.make_causal`` does before a repack) and advances each updated parameter's
step counter.  The packings are refilled in the buffers the forwards already read, and their cache tags set to the
parameters' new versions, so the next forward packs nothing.  Both launches take their tables by value: a forward,
loss, backward and ``step()`` capture into ONE CUDA graph after one eager step, and each replay is a whole training
step.  A replay runs with the hyper-parameters it was captured with (the step count, on the device, advances).

The state dict is torch's Adam format (per parameter ``step``, ``exp_avg``, ``exp_avg_sq`` and, with amsgrad,
``max_exp_avg_sq``; the steps are device fp32 tensors), so ``load_state_dict`` works in both directions with
``torch.optim.Adam``.  Parameters must be fp32 CUDA tensors on the current device, with dense gradients; a parameter
whose ``.grad`` is None is skipped and its step does not advance.  Tensor learning rates and torch's ``foreach``,
``fused``, ``capturable``, ``maximize``, ``differentiable`` and ``decoupled_weight_decay`` switches are not taken.
"""
import torch

from . import _lib, ops
from .modules import _param_tag, pack_spec

# torch.optim.Adam's group keys that this optimizer does not take; those that only choose torch's implementation
# are dropped from a loaded torch state dict, those that change the arithmetic must be False there
_IMPLEMENTATION_KEYS = ("foreach", "fused", "capturable", "differentiable")
_ARITHMETIC_KEYS = ("maximize", "decoupled_weight_decay")


def _layout_bytes(off, f):
    """End, in bytes from the buffer's start, of one vqb_repack_multi layout at byte offset `off` (pack_spec)."""
    layout = f["layout"]
    if layout in (_lib.PACK_F32, _lib.PACK_BF16):
        n = f["kh"] * f["kw"] * f["Cout"] * f["Cin_pad"]
    elif layout in (_lib.PACK_SHUFFLE_F32, _lib.PACK_SHUFFLE_BF16):
        n = 9 * 16 * f["Cin"]
    elif layout in (_lib.PACK_PRIOR_PAD_F32, _lib.PACK_PAD_F32):    # Cp in Cin_pad, the axis kinds in transposed
        cp, kout, kin = f["Cin_pad"], f["transposed"] & 3, f["transposed"] >> 2
        n = ops.pad_width(f["Cout"], kout, cp) * ops.pad_width(f["Cin"], kin, cp) * \
            (f["rows"] * f["cols"] if layout == _lib.PACK_PRIOR_PAD_F32 else f["kh"] * f["kw"])
    else:
        n = f["rows"] * f["cols"] * f["Cin"] * f["Cout"]
    return off + n * (2 if layout in (_lib.PACK_BF16, _lib.PACK_SHUFFLE_BF16) else 4)


class _Plan:
    """One group's tables: ctypes arrays of AdamTensor, PackDesc and step-counter pointers, the packing-cache entries
    they refresh, and the tensors they point into that nothing else holds."""
    __slots__ = ("tensors", "descs", "steps", "refreshed", "keep")

    def __init__(self, tensors, descs, steps, refreshed, keep):
        self.tensors, self.descs, self.steps, self.refreshed, self.keep = tensors, descs, steps, refreshed, keep


def _check_group(g):
    bad = [k for k in _IMPLEMENTATION_KEYS + _ARITHMETIC_KEYS if k in g]
    if bad:
        raise TypeError(f"vqvae_b200.optim.Adam does not take {bad}: it runs torch.optim.Adam's default arithmetic "
                        "in its own kernels")
    if torch.is_tensor(g["lr"]) or any(torch.is_tensor(b) for b in g["betas"]):
        raise TypeError("vqvae_b200.optim.Adam takes float hyper-parameters, not tensors")
    lr, (b1, b2), eps, wd = g["lr"], g["betas"], g["eps"], g["weight_decay"]
    if not 0.0 <= lr:
        raise ValueError(f"Invalid learning rate: {lr}")
    if not 0.0 <= eps:
        raise ValueError(f"Invalid epsilon value: {eps}")
    if not 0.0 <= b1 < 1.0 or not 0.0 <= b2 < 1.0:
        raise ValueError(f"Invalid beta parameters: {(b1, b2)}")
    if not 0.0 <= wd:
        raise ValueError(f"Invalid weight_decay value: {wd}")


class Adam(torch.optim.Optimizer):
    """torch.optim.Adam(params, lr, betas, eps, weight_decay, amsgrad) on the library's kernels (module docstring)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, **unsupported):
        if unsupported:
            raise TypeError(f"vqvae_b200.optim.Adam does not take {sorted(unsupported)}: it runs torch.optim.Adam's "
                            "default arithmetic in its own kernels")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad))

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        _check_group(self.param_groups[-1])

    def load_state_dict(self, state_dict):
        """Loads a state dict of this optimizer or of torch.optim.Adam (whose implementation switches are dropped;
        maximize or decoupled weight decay raise).  Steps move to their parameter's device as fp32 tensors."""
        for g in state_dict["param_groups"]:
            on = [k for k in _ARITHMETIC_KEYS if g.get(k)]
            if on:
                raise TypeError(f"vqvae_b200.optim.Adam cannot continue a run with {on}")
        super().load_state_dict(state_dict)
        self.__dict__.pop("_plans", None)   # the state tensors are new: so are the tables
        for g in self.param_groups:
            for k in _IMPLEMENTATION_KEYS + _ARITHMETIC_KEYS:
                g.pop(k, None)
            _check_group(g)
            for p in g["params"]:
                st = self.state.get(p)
                if st:
                    st["step"] = st["step"].to(device=p.device, dtype=torch.float32)
                    for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
                        if k in st:
                            st[k] = st[k].contiguous()

    def _state(self, p, amsgrad):
        st = self.state[p]
        if not st:
            st["step"] = torch.zeros((), dtype=torch.float32, device=p.device)
            st["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
            st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        if amsgrad and "max_exp_avg_sq" not in st:
            st["max_exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        if st["step"].device != p.device or st["step"].dtype != torch.float32:
            st["step"] = st["step"].to(device=p.device, dtype=torch.float32)
        return st

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            self._step_group(group)
        return loss

    def _step_group(self, group):
        params = [p for p in group["params"] if p.grad is not None]
        for p in params:                    # every check before any launch
            ops._require_cuda(p, "Adam parameter")
            if p.dtype != torch.float32 or p.grad.dtype != torch.float32:
                raise RuntimeError("vqvae_b200.optim.Adam: parameters and gradients must be fp32")
            if p.grad.is_sparse:
                raise RuntimeError("vqvae_b200.optim.Adam does not support sparse gradients")
            if not p.is_contiguous() or p.grad.device != p.device:
                raise RuntimeError("vqvae_b200.optim.Adam: parameters must be contiguous, with their gradient on "
                                   "their device")
        if not params:
            return
        amsgrad = bool(group["amsgrad"])
        plan = self._plan(group, params, amsgrad)
        beta1, beta2 = group["betas"]
        ops.adam_multi(plan.tensors, len(params), group["lr"], beta1, beta2, group["eps"], group["weight_decay"],
                       amsgrad)
        ops.repack_multi(plan.descs, len(plan.descs), plan.steps, len(plan.steps))
        plan.keep = None                    # (stream-ordered frees: safe once the launches are issued)
        # the update is an in-place change of every parameter: a forward saved before it raises in its backward,
        # as it does after torch's Adam; the packings refreshed from the new values are current at that version
        torch.autograd.graph.increment_version(params)
        tags = {}
        for p, cache, key, buf in plan.refreshed:
            tag = tags.get(id(p))
            if tag is None:
                tag = tags[id(p)] = _param_tag(p)
            cache[key] = (tag, buf)

    def _plan(self, group, params, amsgrad):
        """The group's two descriptor tables.  Rebuilt whenever a parameter, gradient or packing buffer moved or a
        packing appeared (the first backward's input-gradient packings), else the last step's, reused: building them
        costs host time only, but per parameter."""
        sig = [amsgrad]
        for p in params:
            g = p.grad
            if not g.is_contiguous():
                sig = None                  # a fresh contiguous copy every step: no reuse
                break
            cache = getattr(p, "_vqb_packed", None)
            sig.append((p.data_ptr(), g.data_ptr(), tuple(0 if b is None else b.data_ptr() for _, b in cache.values())
                        if cache else ()))
        sig = tuple(sig) if sig is not None else None
        plans = self.__dict__.setdefault("_plans", {})
        hit = plans.get(id(group))
        if sig is not None and hit is not None and hit[0] == sig and hit[1] is group:
            return hit[2]
        tensors, steps, descs, refreshed, keep = [], [], [], [], []
        for p in params:
            st = self._state(p, amsgrad)
            g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
            keep.append(g)
            tensors.append(_lib.AdamTensor(
                param=p.data_ptr(), grad=g.data_ptr(), exp_avg=st["exp_avg"].data_ptr(),
                exp_avg_sq=st["exp_avg_sq"].data_ptr(),
                max_exp_avg_sq=st["max_exp_avg_sq"].data_ptr() if amsgrad else None,
                step=st["step"].data_ptr(), numel=p.numel()))
            steps.append(st["step"].data_ptr())
            descs += self._packings(p, refreshed)
        plan = _Plan((_lib.AdamTensor * len(tensors))(*tensors), (_lib.PackDesc * len(descs))(*descs),
                     (_lib.C.c_void_p * len(steps))(*steps), refreshed, keep)
        plans[id(group)] = (sig, group, plan)
        return plan

    @staticmethod
    def _packings(p, refreshed):
        """vqb_repack_multi descriptors for every packing cached on `p` (appended to `refreshed` as (p, cache, key,
        buffer)) and, for a mask-A layer's weight, the zeroing of its excluded taps."""
        descs = []
        cache = getattr(p, "_vqb_packed", None) or {}
        for key, (_, buf) in cache.items():
            if buf is None or buf.device != p.device:
                continue                    # no packing (a bf16 shape without kernels), or one the next forward redoes
            _, layouts = pack_spec(p, key)
            if not layouts or buf.numel() * buf.element_size() < max(_layout_bytes(o, f) for o, f in layouts):
                continue
            descs += [_lib.PackDesc(dst=buf.data_ptr() + off, src=p.data_ptr(), **f) for off, f in layouts]
            refreshed.append((p, cache, key, buf))
        mask = getattr(p, "_vqb_mask_a", None)
        if mask is not None:
            cout, cin, kh, kw = p.shape
            descs.append(_lib.PackDesc(dst=p.data_ptr(), src=None, layout=_lib.PACK_MASK_ZERO, Cout=cout, Cin=cin,
                                       Cin_pad=cin, kh=kh, kw=kw, transposed=0, rows=mask[0], cols=mask[1]))
        return descs

"""CPU-only checks of the on-device Adam (vqvae_b200.optim): the new C entry points and their ctypes table, argument
validation before any CUDA call, the constructor's rejections and torch's state-dict layout."""
import ctypes
import os
import re

import pytest
import torch

from vqvae_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("vqb_adam_capacity", "vqb_adam_multi_f32", "vqb_repack_capacity", "vqb_repack_multi")


def _header():
    return open(os.path.join(ROOT, "include", "vqvae_b200.h")).read()


def test_new_symbols_are_declared_exported_and_typed():
    src = re.sub(r"/\*.*?\*/", "", _header(), flags=re.S)
    lib = _lib.lib()
    for name in NEW:
        assert re.search(r"\b" + name + r"\s*\(", src), name
        assert name in _lib.SIGNATURES and hasattr(lib, name)
    assert _lib.SIGNATURES["vqb_adam_multi_f32"][1] == [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_double] * 5 + \
        [ctypes.c_int, ctypes.c_void_p]
    assert _lib.SIGNATURES["vqb_repack_multi"][1] == [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                                      ctypes.c_void_p]
    assert lib.vqb_abi_version() == 3


def _fields(struct_name):
    body = re.search(r"typedef struct " + struct_name + r" \{(.*?)\}", _header(), flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            names += [re.sub(r"[^a-zA-Z0-9_]", "", part.split()[-1]) for part in decl.split(",")]
    return names


def test_descriptor_structs_match_the_header():
    assert [f for f, _ in _lib.AdamTensor._fields_] == _fields("vqb_adam_tensor")
    assert [f for f, _ in _lib.PackDesc._fields_] == _fields("vqb_pack_desc")
    assert ctypes.sizeof(_lib.AdamTensor) == 7 * 8
    assert ctypes.sizeof(_lib.PackDesc) == 2 * 8 + 9 * 4 + 4
    layouts = dict(re.findall(r"(VQB_PACK_[A-Z0-9_]+) = (\d+)", _header()))
    assert {k: int(v) for k, v in layouts.items()} == {
        "VQB_PACK_F32": _lib.PACK_F32, "VQB_PACK_SHUFFLE_F32": _lib.PACK_SHUFFLE_F32, "VQB_PACK_BF16": _lib.PACK_BF16,
        "VQB_PACK_SHUFFLE_BF16": _lib.PACK_SHUFFLE_BF16, "VQB_PACK_PRIOR_F32": _lib.PACK_PRIOR_F32,
        "VQB_PACK_MASK_ZERO": _lib.PACK_MASK_ZERO}


def test_argument_validation_without_a_gpu():
    lib = _lib.lib()
    assert lib.vqb_adam_capacity() == 480 and lib.vqb_repack_capacity() == 480
    buf = (ctypes.c_float * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p).value
    good = dict(param=p, grad=p, exp_avg=p, exp_avg_sq=p, max_exp_avg_sq=p, step=p, numel=4)
    hp = (1e-3, 0.9, 0.999, 1e-8, 0.0)

    def adam(n=1, hyper=hp, amsgrad=0, **kw):
        arr = (_lib.AdamTensor * 1)(_lib.AdamTensor(**dict(good, **kw)))
        return lib.vqb_adam_multi_f32(arr, n, *hyper, amsgrad, None)

    assert lib.vqb_adam_multi_f32(None, 1, *hp, 0, None) == -1
    assert lib.vqb_adam_multi_f32(None, 0, *hp, 0, None) == 0          # nothing to update: no launch
    assert adam(n=-1) == -1
    for k in ("param", "grad", "exp_avg", "exp_avg_sq", "step"):
        assert adam(**{k: None}) == -1, k
    assert adam(numel=-1) == -1
    assert adam(max_exp_avg_sq=None, amsgrad=1) == -1
    assert adam(numel=0) == 0                                           # an empty tensor: no launch
    for bad in ((-1e-3, 0.9, 0.999, 1e-8, 0.0), (1e-3, 1.0, 0.999, 1e-8, 0.0), (1e-3, 0.9, -0.1, 1e-8, 0.0),
                (1e-3, 0.9, 0.999, -1.0, 0.0), (1e-3, 0.9, 0.999, 1e-8, -1.0), (float("nan"), 0.9, 0.999, 1e-8, 0.0)):
        assert adam(hyper=bad) == -1, bad

    gd = dict(dst=p, src=p, layout=_lib.PACK_F32, Cout=2, Cin=3, Cin_pad=3, kh=3, kw=3, transposed=0, rows=0, cols=0)
    steps = (ctypes.c_void_p * 1)(p)

    def repack(n=1, n_steps=0, st=steps, **kw):
        arr = (_lib.PackDesc * 1)(_lib.PackDesc(**dict(gd, **kw)))
        return lib.vqb_repack_multi(arr, n, st, n_steps, None)

    assert lib.vqb_repack_multi(None, 1, None, 0, None) == -1
    assert lib.vqb_repack_multi(None, 0, None, 1, None) == -1          # step counters without their array
    assert lib.vqb_repack_multi(None, 0, None, 0, None) == 0
    assert repack(n=-1) == -1 and repack(n=0, n_steps=-1) == -1
    assert repack(n=0, n_steps=1, st=(ctypes.c_void_p * 1)(None)) == -1
    assert repack(layout=6) == -1 and repack(layout=-1) == -1          # unknown layouts
    assert repack(dst=None) == -1 and repack(src=None) == -1
    for k in ("Cout", "Cin", "kh", "kw"):
        assert repack(**{k: 0}) == -1, k
    assert repack(Cin_pad=2) == -1
    assert repack(layout=_lib.PACK_BF16, transposed=2) == -1
    assert repack(layout=_lib.PACK_SHUFFLE_F32) == -1                  # not a k4 transposed conv
    assert repack(layout=_lib.PACK_SHUFFLE_BF16, kh=4, kw=4, Cout=5) == -1
    assert repack(layout=_lib.PACK_PRIOR_F32, rows=4, cols=3) == -1
    assert repack(layout=_lib.PACK_MASK_ZERO, src=None, rows=2, cols=4) == -1
    assert repack(layout=_lib.PACK_PRIOR_F32, rows=0, cols=3) == 0     # no kept taps: nothing to write


def test_constructor_rejects_what_it_does_not_implement():
    from vqvae_b200.optim import Adam
    p = [torch.nn.Parameter(torch.zeros(4))]
    for kw in ("foreach", "fused", "capturable", "maximize", "differentiable", "decoupled_weight_decay"):
        with pytest.raises(TypeError, match=kw):
            Adam(p, **{kw: True})
    with pytest.raises(TypeError, match="tensors"):
        Adam(p, lr=torch.tensor(1e-3))
    with pytest.raises(TypeError, match="foreach"):
        Adam([{"params": p, "foreach": False}])
    with pytest.raises(ValueError, match="learning rate"):
        Adam(p, lr=-1.0)
    with pytest.raises(ValueError, match="beta"):
        Adam(p, betas=(0.9, 1.0))
    opt = Adam(p, lr=3e-4, amsgrad=True)
    assert isinstance(opt, torch.optim.Optimizer)
    assert opt.defaults == dict(lr=3e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=True)


def test_cpu_parameters_raise_before_any_launch():
    from vqvae_b200 import ops
    from vqvae_b200.optim import Adam
    p = torch.nn.Parameter(torch.zeros(4))
    p.grad = torch.ones(4)
    opt = Adam([p])
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match="CUDA"):
        opt.step()
    assert ops.launch_count() == n0 and not opt.state


def test_state_dict_layout_is_torchs_and_loads_both_ways():
    from vqvae_b200.optim import Adam
    ps = [torch.nn.Parameter(torch.zeros(3, 2)), torch.nn.Parameter(torch.zeros(5))]
    ref = torch.optim.Adam(ps, lr=2e-4, amsgrad=True)
    for p in ps:                        # torch's own state after a step, built by hand (no step runs on a CPU box here)
        ref.state[p] = dict(step=torch.tensor(3.0), exp_avg=torch.full_like(p, 0.5),
                            exp_avg_sq=torch.full_like(p, 0.25), max_exp_avg_sq=torch.full_like(p, 0.75))
    sd = ref.state_dict()
    ours = Adam(ps, lr=1e-3)
    ours.load_state_dict(sd)
    out = ours.state_dict()
    assert sorted(out["state"]) == sorted(sd["state"]) == [0, 1]
    for i in (0, 1):
        assert sorted(out["state"][i]) == ["exp_avg", "exp_avg_sq", "max_exp_avg_sq", "step"]
        for k, v in sd["state"][i].items():
            assert torch.equal(out["state"][i][k], v), k
        assert out["state"][i]["step"].dtype == torch.float32
    g = out["param_groups"][0]
    assert g["lr"] == 2e-4 and g["amsgrad"] is True and g["params"] == [0, 1]
    assert not any(k in g for k in ("foreach", "fused", "capturable", "maximize", "differentiable"))
    back = torch.optim.Adam(ps, lr=1.0)
    back.load_state_dict(out)
    assert back.param_groups[0]["lr"] == 2e-4 and back.param_groups[0]["maximize"] is False
    assert torch.equal(back.state[ps[1]]["max_exp_avg_sq"], torch.full((5,), 0.75))
    maxi = torch.optim.Adam(ps, maximize=True).state_dict()
    with pytest.raises(TypeError, match="maximize"):
        Adam(ps).load_state_dict(maxi)


def test_new_kernels_do_not_spill():
    from vqvae_b200.build import LIB_DIR, build
    build()
    log = open(os.path.join(LIB_DIR, "build.log")).read()
    part = log[log.index("== optim.cu"):]
    part = part[:part.index("\n== ")] if "\n== " in part else part
    props = re.findall(r"Function properties for \S*(adam_kernel|repack_kernel)\S*\n\s*(.*)", part)
    assert sorted(k for k, _ in props) == ["adam_kernel", "repack_kernel"]
    assert all("0 bytes spill stores, 0 bytes spill loads" in line for _, line in props), props

"""The Gated PixelCNN prior at every dim up to 1024, without a GPU.  A prior whose dim is not a multiple of 32 runs the
kernels at Cp = roundup(dim, 32) channels on zero-padded packings of its parameters, the gate axes padded per half.
Here: the fp64 restatement of that padding gives the unpadded model's logits (and the wrong, unsplit padding does not);
it reproduces the reference's goldens at the script's own dim = img_dim**2; the packing-cache keys become the padded
layouts with their byte sizes in Python integers; and the new entry points refuse bad arguments before any launch."""
import contextlib
import ctypes
import io
import json
import os
import re

import numpy as np
import pytest
import torch

from oracle.make_prior_anydim_golden import PRIOR_ANYDIM_CASES
from oracle.prior_port import A7, B3, make_prior_inputs, make_prior_state_dict, prior_forward, prior_shapes
from tests.prior_anydim_port import kinds, pad_prior_state_dict, padded_dim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAD = -1

# mask A and mask B layers, with and without residual, kernels 3 to 7
STACK = [A7, B3, ["A", 3, True], ["B", 5, False]]


@pytest.mark.parametrize("dim", [16, 49, 100, 784])
def test_padded_state_dict_gives_the_same_fp64_logits(dim):
    K, S, B = 37, 5, 2
    layers = STACK if dim < 784 else STACK[:2]
    sd = make_prior_state_dict(K, dim, len(layers), 3, 90 + dim, layers)
    rng = np.random.RandomState(dim)
    x = torch.from_numpy(rng.randint(0, K, size=(B, S, S)))
    lab = torch.from_numpy(rng.randint(0, 3, size=(B,)))
    want = prior_forward(sd, x, lab, len(layers), torch.float64, layers)
    pad = pad_prior_state_dict(sd, dim)
    cp = padded_dim(dim)
    assert pad["layers.0.vert_stack.weight"].shape[:2] == (2 * cp, cp)
    assert pad["embedding.weight"].shape == (K, cp) and pad["output_conv.0.weight"].shape[1] == cp
    got = prior_forward(pad, x, lab, len(layers), torch.float64, layers)
    err = float((got - want).abs().max() / want.abs().max())
    assert err <= 1e-12, err
    wrong = prior_forward(pad_prior_state_dict(sd, dim, split=False), x, lab, len(layers), torch.float64, layers)
    bad = float((wrong - want).abs().max() / want.abs().max())
    print(f"dim {dim} -> {cp}: split {err:.1e}, unsplit {bad:.1e}")
    assert bad > 1e-3, bad


@pytest.mark.parametrize("name", list(PRIOR_ANYDIM_CASES))
def test_padded_restatement_reproduces_the_anydim_goldens(name):
    """The reference's logits at the seeded positions, against the fp64 restatement at Cp of the padded weights."""
    c = PRIOR_ANYDIM_CASES[name]
    assert c["dim"] == c["size"] ** 2 and c["dim"] % 32
    with np.load(os.path.join(ROOT, "tests", "golden", name + ".npz")) as d:
        assert json.loads(str(d["case"])) == c
        gold = torch.from_numpy(d["logits_at"])
    sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"])
    codes, labels, pos = make_prior_inputs(c)
    want = prior_forward(pad_prior_state_dict(sd, c["dim"]), codes, labels, c["n_layers"], torch.float64)
    want = want[:, :, pos[:, 0], pos[:, 1]]
    assert gold.shape == (c["batch"], c["K"], c["positions"])
    err = float((gold.double() - want).abs().max() / want.abs().max())
    assert err <= 2e-5, err


def _model(K, dim, n_layers):
    from pixelcnn.models import GatedPixelCNN
    with contextlib.redirect_stdout(io.StringIO()):
        return GatedPixelCNN(K, dim, n_layers)


def _width(n, kind, cp):
    return kind * cp if kind else n


@pytest.mark.parametrize("dim", [49, 100, 1000])
def test_pack_spec_gives_the_padded_layouts_and_their_sizes(dim):
    """Every parameter the kernels read padded gets a padded key; pack_spec turns it into the padded layout, and
    _layout_bytes is the padded element count times 4, computed here in Python integers."""
    from vqvae_b200 import _lib
    from vqvae_b200.modules import pack_spec
    from vqvae_b200.optim import _layout_bytes
    from vqvae_b200.prior import _conv_key, _padded_dim
    cp = padded_dim(dim)
    assert _padded_dim(dim) == cp and _padded_dim(cp) == cp
    m = _model(512, dim, 2)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == \
        [(k, tuple(s)) for k, s in prior_shapes(512, dim, 2, 10)]
    for name, p in m.named_parameters():
        kout, kin = kinds(name)
        if not (kout or kin):
            continue
        shape = tuple(p.shape)
        cout, cin = shape[0], shape[1] if len(shape) > 1 else 1
        kh, kw = shape[2:] if len(shape) == 4 else (1, 1)
        geo = dict(Cout=cout, Cin=cin, Cin_pad=cp, kh=kh, kw=kw, transposed=kout + 4 * kin)
        keys = [("pad", cp, kout, kin)]
        if len(shape) == 4:
            keys.append(_conv_key(cp, dim, name.split(".", 2)[2] if name.startswith("layers.") else name, kh - 1, kw))
        for key in keys:
            _, layouts = pack_spec(p, key)
            assert len(layouts) == 1 and layouts[0][0] == 0
            f = layouts[0][1]
            if key[0] == "pad":
                assert f == dict(geo, layout=_lib.PACK_PAD_F32, rows=0, cols=0), (name, f)
                n = _width(cout, kout, cp) * _width(cin, kin, cp) * kh * kw
            else:
                assert key == ("prior_pad", key[1], key[2], cp, kout, kin)
                assert f == dict(geo, layout=_lib.PACK_PRIOR_PAD_F32, rows=key[1], cols=key[2]), (name, f)
                n = key[1] * key[2] * _width(cin, kin, cp) * _width(cout, kout, cp)
            assert _layout_bytes(0, f) == 4 * n and _layout_bytes(64, f) == 64 + 4 * n
    if dim == 1000:       # vert_stack of layer 0 at Cp = 1024: 4*7 taps of a 2048 x 1024 matrix
        f = pack_spec(m.layers[0].vert_stack.weight, ("prior_pad", 3, 7, 1024, 2, 1))[1][0][1]
        assert _layout_bytes(0, f) == 4 * 3 * 7 * 1024 * 2048


def test_multiples_of_32_keep_their_keys():
    from vqvae_b200.prior import _conv_key, _padded_dim
    for dim in (32, 64, 288, 1024):
        assert _padded_dim(dim) == dim
        assert _conv_key(dim, dim, "vert_stack.weight", 3, 7) == ("prior", 3, 7)


def test_the_padded_layouts_are_in_the_header():
    from vqvae_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vqvae_b200.h")).read()
    body = re.search(r"enum vqb_pack_layout \{(.*?)\};", src, flags=re.S).group(1)
    names = re.findall(r"^\s*(VQB_PACK_[A-Z0-9_]+)", re.sub(r"/\*.*?\*/", "", body, flags=re.S), flags=re.M)
    assert names[5:] == ["VQB_PACK_MASK_ZERO", "VQB_PACK_PRIOR_PAD_F32", "VQB_PACK_PAD_F32", "VQB_PACK_UNPAD_F32"]
    assert (_lib.PACK_PRIOR_PAD_F32, _lib.PACK_PAD_F32, _lib.PACK_UNPAD_F32) == (6, 7, 8)
    for name in ("vqb_nchw_to_nhwc_pad_f32", "vqb_nhwc_to_nchw_unpad_f32"):
        assert _lib.SIGNATURES[name][1] == [ctypes.c_void_p] * 2 + [ctypes.c_int] * 5 + [ctypes.c_void_p]


def test_padded_layouts_refuse_bad_descriptors_before_any_launch():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p).value
    # vert_stack of a dim-40 mask-B 3x3 layer at Cp = 64
    gd = dict(dst=p, src=p, layout=_lib.PACK_PRIOR_PAD_F32, Cout=80, Cin=40, Cin_pad=64, kh=2, kw=3, transposed=2 + 4,
              rows=2, cols=3)

    def repack(**kw):
        arr = (_lib.PackDesc * 1)(_lib.PackDesc(**dict(gd, **kw)))
        return lib.vqb_repack_multi(arr, 1, None, 0, None)

    for layout in (_lib.PACK_PRIOR_PAD_F32, _lib.PACK_PAD_F32, _lib.PACK_UNPAD_F32):
        assert repack(layout=layout, src=None) == BAD
        assert repack(layout=layout, dst=None) == BAD
        assert repack(layout=layout, Cin_pad=0) == BAD
        assert repack(layout=layout, transposed=0) == BAD           # nothing padded
        assert repack(layout=layout, transposed=3) == BAD           # kind 3
        assert repack(layout=layout, transposed=12 + 2) == BAD      # kind 3 on Cin
        assert repack(layout=layout, transposed=-1) == BAD
        assert repack(layout=layout, Cout=81) == BAD                # an odd gate axis
        assert repack(layout=layout, Cin_pad=39) == BAD             # fewer padded channels than real ones
        assert repack(layout=layout, Cout=0) == BAD and repack(layout=layout, kh=0) == BAD
    assert repack(rows=3) == BAD and repack(cols=4) == BAD and repack(rows=-1) == BAD
    assert repack(layout=9) == BAD


def test_padded_layout_changes_refuse_bad_arguments():
    from vqvae_b200 import _lib
    lib = _lib.lib()
    buf = (ctypes.c_float * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p).value
    for fn in (lib.vqb_nchw_to_nhwc_pad_f32, lib.vqb_nhwc_to_nchw_unpad_f32):
        assert fn(None, p, 1, 40, 64, 2, 2, None) == BAD
        assert fn(p, None, 1, 40, 64, 2, 2, None) == BAD
        assert fn(p, p, 1, 40, 39, 2, 2, None) == BAD               # Cp < C
        assert fn(p, p, 0, 40, 64, 2, 2, None) == BAD
        assert fn(p, p, 1, 0, 64, 2, 2, None) == BAD
        assert fn(p, p, 1, 40, 64, 0, 2, None) == BAD


def test_module_refusals_run_before_any_launch():
    from vqvae_b200 import ops
    from vqvae_b200.prior import GatedMaskedConv2d
    m = _model(16, 49, 2)
    n0 = ops.launch_count()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros((1, 4, 4), dtype=torch.int64), torch.zeros(1, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.cross_entropy(torch.zeros((1, 4, 4), dtype=torch.int64), torch.zeros(1, dtype=torch.int64))
    layer = GatedMaskedConv2d("B", 40, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        layer(torch.zeros((1, 40, 4, 4)), torch.zeros((1, 40, 4, 4)), torch.zeros(1, dtype=torch.int64))
    with pytest.raises(RuntimeError, match=r"\(B,40,H,W\)"):
        layer(torch.zeros((1, 64, 4, 4)), torch.zeros((1, 64, 4, 4)), torch.zeros(1, dtype=torch.int64))
    big = _model(16, 1025, 1)
    with pytest.raises(RuntimeError, match="1024"):
        big._net([])
    assert ops.launch_count() == n0

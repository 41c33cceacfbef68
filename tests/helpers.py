"""Shared helpers of the parity tests (test infrastructure; may import oracle/)."""
import json
import os
import subprocess
import sys

import numpy as np

from oracle.make_golden import MODEL_CASES, VQ_CASES, make_vq_inputs  # noqa: F401
from oracle.weights import make_images, make_state_dict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
HP_KEYS = ("h_dim", "res_h_dim", "n_res_layers", "n_embeddings", "embedding_dim")


def load_golden(name):
    with np.load(os.path.join(GOLDEN, name + ".npz")) as d:
        out = {k: d[k] for k in d.files}
    out["case"] = json.loads(str(out["case"]))
    return out


def model_case_inputs(case):
    hp = {k: case[k] for k in HP_KEYS}
    sd = make_state_dict(seed=case["wseed"], codebook=case["codebook"],
                         codebook_scale=case["codebook_scale"], **hp)
    x = make_images(case["batch"], case["size"], case["xseed"])
    return hp, sd, x


def build_model(hp, sd, device="cuda"):
    """The product model (drop-in import path) loaded with a numpy state dict."""
    import torch
    from models.vqvae import VQVAE
    m = VQVAE(hp["h_dim"], hp["res_h_dim"], hp["n_res_layers"], hp["n_embeddings"],
              hp["embedding_dim"], 0.25)
    m.load_state_dict({k: torch.from_numpy(np.array(v)) for k, v in sd.items()})
    return m.to(device).eval()


def expected_zq(g, E=None):
    """The reference's z_q (NCHW) of a golden case, or None when only its hash is stored.  Cases that drop z_q to
    stay small (cfg3_s256) hold z_e and idx, from which z_q = fl(z_e + fl(E[idx] - z_e)) follows (quantizer.py:60,67)."""
    if "z_q" in g:
        return g["z_q"]
    if "z_e" in g and E is not None:
        z = g["z_e"]
        B, D, H, W = z.shape
        rows = np.ascontiguousarray(z.transpose(0, 2, 3, 1)).reshape(-1, D)
        e = np.asarray(E, dtype=np.float32)[g["idx"].ravel()]
        zq = (rows + (e - rows).astype(np.float32)).astype(np.float32)
        return np.ascontiguousarray(zq.reshape(B, H, W, D).transpose(0, 3, 1, 2))
    return None


def assert_zq_matches(g, zq_nchw, E=None):
    """Bitwise comparison of a z_q (NCHW fp32 array) with the golden case, through the stored array, the
    reconstruction above, or the stored SHA-256 of the reference's bytes."""
    import hashlib
    zq_nchw = np.ascontiguousarray(zq_nchw, dtype=np.float32)
    want = expected_zq(g, E)
    if want is not None:
        assert np.array_equal(zq_nchw, want, equal_nan=True)
    else:
        assert hashlib.sha256(zq_nchw.tobytes()).hexdigest() == str(g["z_q_sha256"])


_CONV_PROFILE_SCRIPT = """
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
from vqvae_b200 import ops
from vqvae_b200._lib import TF32
out = []
for B, Cin, H, W, Cout, k, s, p, t, il, ol, relu, skip in json.loads(sys.argv[1]):
    oh, ow = ops.conv_out_hw(H, W, k, k, s, p, t)
    x = torch.rand((B * Cin * H * W,), device="cuda")
    w = ops.pack_conv_weight(torch.randn((Cin, Cout, k, k) if t else (Cout, Cin, k, k), device="cuda") * 0.05, t)
    b = torch.rand((Cout,), device="cuda")
    sk = torch.rand((B, oh, ow, Cout), device="cuda") if skip else None
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ops.conv2d(x, w, b, B=B, Cin=Cin, H=H, W=W, Cout=Cout, kh=k, kw=k, stride=s, pad=p, transposed=t,
                   in_layout=il, out_layout=ol, relu=relu, skip=sk, precision=TF32)
        torch.cuda.synchronize()
    out.append([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA])
print(json.dumps(out))
"""


def tf32_conv_kernels(cases):
    """The CUDA kernel names torch.profiler records for one vqb_conv2d_f32 call in TF32 mode per case (B, Cin, H, W,
    Cout, k, stride, pad, transposed, in_layout, out_layout, relu, skip), read in a fresh interpreter so that nothing
    earlier tests did to the process's profiling state plays a part."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    run = subprocess.run([sys.executable, "-c", _CONV_PROFILE_SCRIPT, json.dumps([list(c) for c in cases])], cwd=root,
                         capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-3000:]
    return [[n for n in names if not n.startswith("Memcpy") and not n.startswith("Memset")]
            for names in json.loads(run.stdout.strip().splitlines()[-1])]


def tf32_conv_kernel(case):
    """The kernel a TF32 vqb_conv2d_f32 call of `case` must run on, by name: the input conv (Cin = 3) its CUDA-core
    kernel in every mode, the k4 s2 transposed output conv to <= 4 channels in NCHW the scatter-form wgmma kernel,
    every other layer the wgmma convolution."""
    from vqvae_b200._lib import NCHW
    B, Cin, H, W, Cout, k, s, p, t, il, ol, relu, skip = case
    if Cin == 3 and k == 4 and s == 2 and not t:
        return "conv_in_k4s2_kernel"
    if t and k == 4 and s == 2 and Cout <= 4 and ol == NCHW:
        return "convt_scatter_kernel"
    return "wgconv_kernel"

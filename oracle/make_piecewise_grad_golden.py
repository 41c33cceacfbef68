"""Generate tests/golden/piecewise_grad.npz from the UNMODIFIED reference's modules called on their own.

TEST INFRASTRUCTURE ONLY.  Run from the repository root where a checkout of the reference exists
(``python -m oracle.make_piecewise_grad_golden [--ref DIR]``).  As in oracle.make_vqvae_grad_golden, the reference runs
in a subprocess with cwd = the reference root, CUDA hidden and one thread; weights and inputs come from the seeds of
oracle.piecewise_port.  Each module gets a random upstream gradient G and the loss (out * G).sum():
  res/layer, res/stack<n>   ResidualLayer and ResidualStack([layer] * n) on a NON-leaf input x = x0 * 1: x0's
                            gradient ("dx"), the two weight gradients ("dw1", "dw2") and x after the call ("x_after",
                            the in-place ReLU's mutation, Q2)
  gated/<name>              GatedMaskedConv2d: the gradients of x_v, x_h and all nine parameters (mask A's taps
                            included)
  gate                      GatedActivation: the input's gradient
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

from .build import REF_SRC
from .piecewise_port import GATE, GATED, PRIOR_LAYER_KEYS, RES, gate_inputs, gated_inputs, res_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "piecewise_grad.npz")

_SCRIPT = r"""
import sys, json, numpy as np, torch
sys.path.insert(0, %(ref)r)
from models.residual import ResidualLayer, ResidualStack
from pixelcnn.models import GatedActivation, GatedMaskedConv2d
torch.set_num_threads(1)
job = json.load(open(sys.argv[1]))
data = np.load(job["in"])
T = lambda k: torch.from_numpy(data[k])
out = {}
c = job["res"]
for n in [None] + c["stacks"]:
    name = "layer" if n is None else "stack%%d" %% n
    m = ResidualLayer(c["C"], c["C"], c["CMID"]) if n is None else ResidualStack(c["C"], c["C"], c["CMID"], n)
    layer = m if n is None else (m.stack[0] if n else None)
    if layer is not None:
        layer.res_block[1].weight.data.copy_(T("res/w1"))
        layer.res_block[3].weight.data.copy_(T("res/w2"))
    x0 = T("res/x").clone().requires_grad_()
    x = x0 * 1
    y = m(x)
    (y * T("res/g/" + name)).sum().backward()
    out["res/%%s/dx" %% name] = x0.grad.numpy()
    out["res/%%s/x_after" %% name] = x.detach().numpy()
    if layer is not None:
        out["res/%%s/dw1" %% name] = layer.res_block[1].weight.grad.numpy()
        out["res/%%s/dw2" %% name] = layer.res_block[3].weight.grad.numpy()
g = job["gated"]
for name, mask, k, residual in g["layers"]:
    p = "gated/%%s/" %% name
    m = GatedMaskedConv2d(mask, g["DIM"], k, residual, g["N_CLASSES"])
    m.load_state_dict({key: T(p + key) for key in m.state_dict()})
    x_v, x_h = T(p + "x_v").clone().requires_grad_(), T(p + "x_h").clone().requires_grad_()
    out_v, out_h = m(x_v, x_h, T(p + "label"))
    ((out_v * T(p + "g_v")).sum() + (out_h * T(p + "g_h")).sum()).backward()
    out[p + "dx_v"], out[p + "dx_h"] = x_v.grad.numpy(), x_h.grad.numpy()
    out.update({p + "d/" + key: t.grad.numpy() for key, t in m.named_parameters()})
x = T("gate/x").clone().requires_grad_()
(GatedActivation()(x) * T("gate/g")).sum().backward()
out["gate/dx"] = x.grad.numpy()
np.savez(job["out"], **out)
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default=REF_SRC)
    a = ap.parse_args()
    assert os.path.isdir(os.path.join(a.ref, "models")), "needs a checkout of the reference"
    inputs = {"res/" + k: v for k, v in res_inputs().items()}
    for name, _, _, _ in GATED["layers"]:
        inputs.update({f"gated/{name}/{k}": v for k, v in gated_inputs(name).items()})
    inputs.update({"gate/" + k: v for k, v in gate_inputs().items()})
    with tempfile.TemporaryDirectory() as td:
        job = dict(res=RES, gated=GATED, **{"in": os.path.join(td, "in.npz"), "out": os.path.join(td, "out.npz")})
        np.savez(job["in"], **inputs)
        path = os.path.join(td, "job.json")
        with open(path, "w") as f:
            json.dump(job, f)
        subprocess.run([sys.executable, "-c", _SCRIPT % dict(ref=a.ref), path], check=True, cwd=a.ref,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
        with np.load(job["out"]) as d:
            out = {k: d[k] for k in d.files}
    assert all(k in out for k in (f"gated/{n}/d/{key}" for n, *_ in GATED["layers"] for key in PRIOR_LAYER_KEYS))
    np.savez_compressed(OUT, case=json.dumps(dict(res=RES, gated=GATED, gate=GATE)), **out)
    print(OUT, len(out), "arrays")


if __name__ == "__main__":
    main()

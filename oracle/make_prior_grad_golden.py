"""Generate tests/golden/prior_grad_{ragged,default}.npz from the UNMODIFIED reference's pixelcnn package.

TEST INFRASTRUCTURE ONLY.  Run from the repository root where a checkout of the reference exists
(``python -m oracle.make_prior_grad_golden [--ref DIR] [fixture ...]``; only the named fixtures are regenerated, so
the others stay byte-identical).  As in oracle.make_prior_golden, the reference runs in a subprocess with cwd = the
reference root, CUDA hidden and one thread; weights and inputs come from the seeds in oracle.prior_port.PRIOR_CASES
and PRIOR_SHAPE_CASES.  The subprocess computes gated_pixelcnn.py's loss on the case and calls loss.backward().
prior_grad_ragged.npz keeps the loss and every gradient in full; prior_grad_default.npz keeps the loss and, per
gradient, oracle.prior_train_port.fingerprint (sum, L2 norm, dots with seeded probes), in fp64.
prior_grad_layers.npz (the PRIOR_SHAPE_CASES["kernels"] stack, built from the reference's own GatedMaskedConv2d)
keeps the loss, every gradient of at most FULL_MAX elements in full ("grad/" keys) and the fingerprint of the larger
ones, the two 15-wide vertical stacks ("fingerprint/" keys).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

from .build import REF_SRC
from .prior_port import PRIOR_CASES, PRIOR_SHAPE_CASES, make_prior_inputs, make_prior_state_dict
from .prior_train_port import fingerprint

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden")
CASES = {"prior_ragged": "prior_grad_ragged", "prior_default": "prior_grad_default", "kernels": "prior_grad_layers"}
FULL_MAX = 65536      # prior_grad_layers: larger gradients are stored as fingerprints

_SCRIPT = r"""
import sys, json, numpy as np, torch
import torch.nn as nn
sys.path.insert(0, %(ref)r)
from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
torch.set_num_threads(1)
job = json.load(open(sys.argv[1]))
c = job["case"]
data = np.load(job["in"])
model = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
for i, (mask, k, residual) in enumerate(c.get("layers", [])):
    model.layers[i] = GatedMaskedConv2d(mask, c["dim"], k, residual, c["n_classes"])
model.load_state_dict({k: torch.from_numpy(data[k]) for k in model.state_dict().keys()})
criterion = nn.CrossEntropyLoss()
x, label = torch.from_numpy(data["__codes"]), torch.from_numpy(data["__labels"])
logits = model(x, label)
logits = logits.permute(0, 2, 3, 1).contiguous()
loss = criterion(logits.view(-1, c["K"]), x.view(-1))
model.zero_grad()
loss.backward()
out = {"loss": np.array(loss.item(), dtype=np.float64)}
out.update({"grad/" + k: p.grad.numpy() for k, p in model.named_parameters()})
np.savez(job["out"], **out)
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default=REF_SRC)
    ap.add_argument("fixtures", nargs="*")
    a = ap.parse_args()
    assert os.path.isdir(os.path.join(a.ref, "pixelcnn")), "needs a checkout of the reference"
    for name, fixture in CASES.items():
        if a.fixtures and fixture not in a.fixtures:
            continue
        c = PRIOR_CASES[name] if name in PRIOR_CASES else PRIOR_SHAPE_CASES[name]
        sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], c.get("layers"))
        codes, labels, _ = make_prior_inputs(c)
        with tempfile.TemporaryDirectory() as td:
            job = dict(case=c, **{"in": os.path.join(td, "in.npz"), "out": os.path.join(td, "out.npz")})
            np.savez(job["in"], __codes=codes, __labels=labels, **sd)
            path = os.path.join(td, "job.json")
            with open(path, "w") as f:
                json.dump(job, f)
            subprocess.run([sys.executable, "-c", _SCRIPT % dict(ref=a.ref), path], check=True, cwd=a.ref,
                           env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
            with np.load(job["out"]) as d:
                out = {k: d[k] for k in d.files}
        keys = list(sd)
        if fixture == "prior_grad_default":
            out = {k: (fingerprint(v, keys.index(k[5:])) if k.startswith("grad/") else v) for k, v in out.items()}
        elif fixture == "prior_grad_layers":
            out = {("fingerprint/" + k[5:] if v.size > FULL_MAX else k):
                   (fingerprint(v, keys.index(k[5:])) if k.startswith("grad/") and v.size > FULL_MAX else v)
                   for k, v in out.items()}
        np.savez_compressed(os.path.join(OUT, fixture + ".npz"), case=json.dumps(c), **out)
        print(fixture, "loss %.7f" % float(out["loss"]), len(out) - 1, "gradients")


if __name__ == "__main__":
    main()

"""Generate tests/golden/prior_*.npz and prior_init_fingerprint.json from the UNMODIFIED reference's pixelcnn package.

TEST INFRASTRUCTURE ONLY.  Run from the repository root where a checkout of the reference exists
(``python -m oracle.make_prior_golden [--ref DIR] [prior_... ...]``; only the named cases are regenerated, so the
other fixtures stay byte-identical).  The reference is imported in a subprocess with cwd = the reference root and
CUDA hidden.  Weights and inputs are not stored: tests regenerate them from the seeds in
oracle.prior_port.PRIOR_CASES, so each fixture holds the reference's outputs only.  prior_layers.npz is the
PRIOR_SHAPE_CASES["kernels"] stack: the reference's GatedPixelCNN with each of its layers replaced by the reference's
own GatedMaskedConv2d(mask_type, dim, kernel, residual, n_classes).
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

OUT = os.path.join(ROOT, "tests", "golden")
LAYER_FIXTURES = {"prior_layers": "kernels"}          # fixture -> PRIOR_SHAPE_CASES entry

_SCRIPT = r"""
import sys, json, hashlib, numpy as np, torch
sys.path.insert(0, %(ref)r)
from pixelcnn.models import GatedMaskedConv2d, GatedPixelCNN
torch.set_num_threads(1)
job = json.load(open(sys.argv[1]))
if job["kind"] == "fingerprint":
    out = {}
    for name, c in job["configs"].items():
        torch.manual_seed(0)
        m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"])
        out[name] = [[k, list(v.shape), float(v.double().sum()), hashlib.sha256(v.contiguous().numpy().tobytes()).hexdigest()]
                     for k, v in m.state_dict().items()]
    json.dump(out, open(job["out"], "w"), indent=1)
else:
    c = job["case"]
    data = np.load(job["in"])
    m = GatedPixelCNN(c["K"], c["dim"], c["n_layers"], c["n_classes"]).eval()
    for i, (mask, k, residual) in enumerate(c.get("layers", [])):
        m.layers[i] = GatedMaskedConv2d(mask, c["dim"], k, residual, c["n_classes"])
    m.load_state_dict({k: torch.from_numpy(data[k]) for k in m.state_dict().keys()})
    with torch.no_grad():
        logits = m(torch.from_numpy(data["__codes"]), torch.from_numpy(data["__labels"]))
    out = dict(logits=logits.numpy())
    if "__pos" in data.files:
        p = data["__pos"]
        out = dict(logits_at=np.ascontiguousarray(logits.numpy()[:, :, p[:, 0], p[:, 1]]))
    np.savez(job["out"], **out)
"""


def _run(ref, job):
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "job.json")
        with open(path, "w") as f:
            json.dump(job, f)
        subprocess.run([sys.executable, "-c", _SCRIPT % dict(ref=ref), path], check=True, cwd=ref,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default=REF_SRC)
    ap.add_argument("cases", nargs="*")
    a = ap.parse_args()
    assert os.path.isdir(os.path.join(a.ref, "pixelcnn")), "needs a checkout of the reference"
    only = set(a.cases)
    if not only or "prior_init_fingerprint" in only:
        configs = {n: {k: PRIOR_CASES[n][k] for k in ("K", "dim", "n_layers", "n_classes")}
                   for n in ("prior_default", "prior_ragged")}
        _run(a.ref, dict(kind="fingerprint", configs=configs, out=os.path.join(OUT, "prior_init_fingerprint.json")))
        print("prior_init_fingerprint.json")
    cases = list(PRIOR_CASES.items()) + [(f, PRIOR_SHAPE_CASES[n]) for f, n in LAYER_FIXTURES.items()]
    for name, c in cases:
        if only and name not in only:
            continue
        sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"], c.get("layers"))
        codes, labels, pos = make_prior_inputs(c)
        arrays = dict(sd, __codes=codes, __labels=labels)
        if pos is not None:
            arrays["__pos"] = pos
        with tempfile.TemporaryDirectory() as td:
            job = dict(kind="case", case=c, **{"in": os.path.join(td, "in.npz"), "out": os.path.join(td, "out.npz")})
            np.savez(job["in"], **arrays)
            _run(a.ref, job)
            with np.load(job["out"]) as d:
                out = {k: d[k] for k in d.files}
        np.savez_compressed(os.path.join(OUT, name + ".npz"), case=json.dumps(c), **out)
        print(name, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()

"""Generate tests/golden/prior_wide_*.npz from the UNMODIFIED reference's pixelcnn package: the Gated PixelCNN prior at
dims above 256, as the reference's gated_pixelcnn.py builds it (``GatedPixelCNN(K, img_dim**2, n_layers)``: layer 0 a
7x7 mask A, the others 3x3 mask B with a residual).

TEST INFRASTRUCTURE ONLY.  Run from the repository root where a checkout of the reference exists
(``python -m oracle.make_prior_wide_golden [--ref DIR] [prior_wide_... ...]``; only the named cases are regenerated).
The reference runs on the CPU in a subprocess, through make_prior_golden's job script.  Weights and inputs are not
stored: tests regenerate them from the seeds in PRIOR_WIDE_CASES, so each fixture holds the reference's logits only.
"""
import argparse
import json
import os
import tempfile

import numpy as np

from .build import REF_SRC
from .make_prior_golden import OUT, _run
from .prior_port import make_prior_inputs, make_prior_state_dict

# name -> case, in PRIOR_CASES' format (K, dim, n_layers, n_classes, grid, batch, weight seed, input seed)
PRIOR_WIDE_CASES = {
    # dim = 24**2: 2*dim = 1152, 4.5 output channels per thread
    "prior_wide_576": dict(K=512, dim=576, n_layers=3, n_classes=10, size=6, batch=2, wseed=70, xseed=71),
    # dim = 32**2: 2*dim = 2048, the widest instantiation
    "prior_wide_1024": dict(K=512, dim=1024, n_layers=2, n_classes=10, size=4, batch=3, wseed=72, xseed=73),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default=REF_SRC)
    ap.add_argument("cases", nargs="*")
    a = ap.parse_args()
    assert os.path.isdir(os.path.join(a.ref, "pixelcnn")), "needs a checkout of the reference"
    for name, c in PRIOR_WIDE_CASES.items():
        if a.cases and name not in a.cases:
            continue
        sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"])
        codes, labels, _ = make_prior_inputs(c)
        with tempfile.TemporaryDirectory() as td:
            job = dict(kind="case", case=c, **{"in": os.path.join(td, "in.npz"), "out": os.path.join(td, "out.npz")})
            np.savez(job["in"], **sd, __codes=codes, __labels=labels)
            _run(a.ref, job)
            with np.load(job["out"]) as d:
                logits = d["logits"]
        np.savez_compressed(os.path.join(OUT, name + ".npz"), case=json.dumps(c), logits=logits)
        print(name, logits.shape)


if __name__ == "__main__":
    main()

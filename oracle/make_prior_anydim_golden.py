"""Generate tests/golden/prior_anydim_*.npz from the UNMODIFIED reference's pixelcnn package: the Gated PixelCNN prior at
dims that are not a multiple of 32, as the reference's gated_pixelcnn.py builds it (``GatedPixelCNN(K, img_dim**2,
n_layers)`` on its own img_dim x img_dim grid: layer 0 a 7x7 mask A, the others 3x3 mask B with a residual).

TEST INFRASTRUCTURE ONLY.  Run from the repository root where a checkout of the reference exists
(``python -m oracle.make_prior_anydim_golden [--ref DIR] [prior_anydim_... ...]``; only the named cases are
regenerated).  The reference runs on the CPU in a subprocess, through make_prior_golden's job script.  Weights and
inputs are not stored: tests regenerate them from the seeds in PRIOR_ANYDIM_CASES, so each fixture holds the
reference's logits only, at `positions` seeded grid positions (``logits_at``, (B, K, positions)).
"""
import argparse
import json
import os
import tempfile

import numpy as np

from .build import REF_SRC
from .make_prior_golden import OUT, _run
from .prior_port import make_prior_inputs, make_prior_state_dict

# name -> case, in PRIOR_CASES' format (K, dim, n_layers, n_classes, grid, batch, weight seed, input seed, stored
# positions); dim = size**2 throughout, the script's own prior for that latent grid
PRIOR_ANYDIM_CASES = {
    # 28x28 images (MNIST-sized) -> 7x7 latents: dim 49 runs at 64 channels
    "prior_anydim_49": dict(K=512, dim=49, n_layers=3, n_classes=10, size=7, batch=2, wseed=80, xseed=81,
                            positions=40),
    # 56x56 images -> 14x14 latents: dim 196 runs at 224
    "prior_anydim_196": dict(K=512, dim=196, n_layers=2, n_classes=10, size=14, batch=2, wseed=82, xseed=83,
                             positions=40),
    # 112x112 images -> 28x28 latents: dim 784 runs at 800
    "prior_anydim_784": dict(K=512, dim=784, n_layers=2, n_classes=10, size=28, batch=2, wseed=84, xseed=85,
                             positions=40),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default=REF_SRC)
    ap.add_argument("cases", nargs="*")
    a = ap.parse_args()
    assert os.path.isdir(os.path.join(a.ref, "pixelcnn")), "needs a checkout of the reference"
    for name, c in PRIOR_ANYDIM_CASES.items():
        if a.cases and name not in a.cases:
            continue
        sd = make_prior_state_dict(c["K"], c["dim"], c["n_layers"], c["n_classes"], c["wseed"])
        codes, labels, pos = make_prior_inputs(c)
        with tempfile.TemporaryDirectory() as td:
            job = dict(kind="case", case=c, **{"in": os.path.join(td, "in.npz"), "out": os.path.join(td, "out.npz")})
            np.savez(job["in"], **sd, __codes=codes, __labels=labels, __pos=pos)
            _run(a.ref, job)
            with np.load(job["out"]) as d:
                logits_at = d["logits_at"]
        np.savez_compressed(os.path.join(OUT, name + ".npz"), case=json.dumps(c), logits_at=logits_at)
        print(name, logits_at.shape)


if __name__ == "__main__":
    main()

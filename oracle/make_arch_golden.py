"""Generate tests/golden/arch_<name>.npz from the UNMODIFIED reference's models package, for the VQ-VAE
architectures of tests/vqvae_arch.py that main.py's flags build.

TEST INFRASTRUCTURE ONLY.  Run from the repository root where a checkout of the reference exists
(``python -m oracle.make_arch_golden [--ref DIR] [name ...]``).  As in oracle.make_vqvae_grad_golden, the reference runs
in a subprocess with cwd = the reference root, CUDA hidden and one thread; weights and images come from the row's
seed (tests.vqvae_arch.arch_inputs).  Each fixture holds the fp32 CPU forward -- z_e, idx, x_hat, loss, perplexity --
and, in training mode, main.py's loss (x_train_var fixed to X_TRAIN_VAR), its parts and every parameter gradient as
oracle.prior_train_port.fingerprint.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

from .build import REF_SRC
from .make_vqvae_grad_golden import X_TRAIN_VAR
from .prior_train_port import fingerprint

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden")

_SCRIPT = r"""
import sys, json, numpy as np, torch
sys.path.insert(0, %(ref)r)
import models.quantizer as Q
Q.device = torch.device("cpu")
from models.vqvae import VQVAE
torch.set_num_threads(1)
job = json.load(open(sys.argv[1]))
c = job["case"]
data = np.load(job["in"])
model = VQVAE(c["h_dim"], c["res_h_dim"], c["n_res_layers"], c["n_embeddings"], c["embedding_dim"], 0.25)
model.load_state_dict({k: torch.from_numpy(data[k]) for k in model.state_dict().keys()})
x = torch.from_numpy(data["__x"])
out = {}
model.eval()
with torch.no_grad():
    z_e = model.pre_quantization_conv(model.encoder(x.clone()))
    embedding_loss, x_hat, perplexity = model(x)
    out["z_e"] = z_e.numpy()
    out["idx"] = model.vector_quantization(z_e)[4].numpy()
    out["x_hat"] = x_hat.numpy()
    out["loss"] = np.array(embedding_loss.item(), dtype=np.float32)
    out["perplexity"] = np.array(perplexity.item(), dtype=np.float32)
model.train()
model.zero_grad()
embedding_loss, x_hat, perplexity = model(x)
recon_loss = torch.mean((x_hat - x)**2) / c["x_train_var"]
loss = recon_loss + embedding_loss
loss.backward()
out["train_loss"] = np.array(loss.item(), dtype=np.float64)
out["recon_error"] = np.array(recon_loss.item(), dtype=np.float64)
out.update({"grad/" + k: p.grad.numpy() for k, p in model.named_parameters()})
np.savez(job["out"], **out)
"""


def main():
    sys.path.insert(0, ROOT)
    from tests.vqvae_arch import ARCHS, GOLDEN_ARCHS, arch_inputs
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default=REF_SRC)
    ap.add_argument("names", nargs="*")
    a = ap.parse_args()
    assert os.path.isdir(os.path.join(a.ref, "models")), "needs a checkout of the reference"
    for name in a.names or GOLDEN_ARCHS:
        hp, sd, x = arch_inputs(name)
        B, (H, W), scale, seed = ARCHS[name][5:]
        c = dict(hp, batch=B, size=[H, W], codebook_scale=scale, seed=seed, x_train_var=X_TRAIN_VAR)
        with tempfile.TemporaryDirectory() as td:
            job = dict(case=c, **{"in": os.path.join(td, "in.npz"), "out": os.path.join(td, "out.npz")})
            np.savez(job["in"], __x=x, **sd)
            path = os.path.join(td, "job.json")
            with open(path, "w") as f:
                json.dump(job, f)
            subprocess.run([sys.executable, "-c", _SCRIPT % dict(ref=a.ref), path], check=True, cwd=a.ref,
                           env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
            with np.load(job["out"]) as d:
                out = {k: d[k] for k in d.files}
        keys = list(sd)
        out = {k: (fingerprint(v, keys.index(k[5:])) if k.startswith("grad/") else v) for k, v in out.items()}
        path = os.path.join(OUT, f"arch_{name}.npz")
        np.savez_compressed(path, case=json.dumps(c), **out)
        print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

"""Generate tests/golden/vqvae_grad_*.npz and vqvae_train_*.npz from the UNMODIFIED reference's models package.

TEST INFRASTRUCTURE ONLY.  Run from the repository root where a checkout of the reference exists
(``python -m oracle.make_vqvae_grad_golden [--ref DIR] [case ...]``).  As in oracle.make_prior_grad_golden, the
reference runs in a subprocess with cwd = the reference root, CUDA hidden and one thread; weights and images come from
the seeds of oracle.make_golden.MODEL_CASES.  The subprocess puts the model in training mode and runs main.py's loop
body (main.py:70-79) with the fixed x_train_var X_TRAIN_VAR, recorded in each case:
  small_odd       loss, recon error, perplexity, indices and every parameter gradient in full
  cifar_default   the same, with each gradient stored as oracle.prior_train_port.fingerprint
  cifar_spread    a STEPS-step Adam(amsgrad=True, lr=3e-4) trajectory on the fixed batch: loss, recon error and
                  perplexity per step, run with one thread ("trajectory") and again with TRAJECTORY_THREADS threads
                  ("trajectory_threads4"): the reference's own trajectory moves by 1.5e-4 of the loss with the thread
                  count (Adam turns last-bit differences of near-zero gradient elements into whole steps)
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

from .build import REF_SRC
from .make_golden import MODEL_CASES
from .prior_train_port import fingerprint
from .weights import make_images, make_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden")
X_TRAIN_VAR = 0.0625          # main.py divides the recon error by the training set's variance; fixed here
STEPS = 20
TRAJECTORY_THREADS = 4
CASES = {"small_odd": ("vqvae_grad_small_odd", "grads"), "cifar_default": ("vqvae_grad_cifar_default", "fingerprints"),
         "cifar_spread": ("vqvae_train_cifar_spread", "trajectory")}
HP = ("h_dim", "res_h_dim", "n_res_layers", "n_embeddings", "embedding_dim")

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
model.train()
x = torch.from_numpy(data["__x"])
out = {}
if job["kind"] == "trajectory":
    init = {k: v.clone() for k, v in model.state_dict().items()}
    for key, threads in (("trajectory", 1), ("trajectory_threads%%d" %% job["threads"], job["threads"])):
        torch.set_num_threads(threads)
        model.load_state_dict(init)
        optimizer = torch.optim.Adam(model.parameters(), lr=3e-4, amsgrad=True)
        rows = []
        for i in range(c["steps"]):
            optimizer.zero_grad()
            embedding_loss, x_hat, perplexity = model(x)
            recon_loss = torch.mean((x_hat - x)**2) / c["x_train_var"]
            loss = recon_loss + embedding_loss
            loss.backward()
            optimizer.step()
            rows.append([loss.item(), recon_loss.item(), perplexity.item()])
        out[key] = np.array(rows, dtype=np.float64)
else:
    model.zero_grad()
    embedding_loss, x_hat, perplexity = model(x)
    recon_loss = torch.mean((x_hat - x)**2) / c["x_train_var"]
    loss = recon_loss + embedding_loss
    loss.backward()
    out["loss"] = np.array(loss.item(), dtype=np.float64)
    out["recon_error"] = np.array(recon_loss.item(), dtype=np.float64)
    out["perplexity"] = np.array(perplexity.item(), dtype=np.float64)
    z_e = model.pre_quantization_conv(model.encoder(x.clone()))
    out["idx"] = model.vector_quantization(z_e)[4].numpy().ravel()
    out.update({"grad/" + k: p.grad.numpy() for k, p in model.named_parameters()})
np.savez(job["out"], **out)
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default=REF_SRC)
    ap.add_argument("cases", nargs="*")
    a = ap.parse_args()
    assert os.path.isdir(os.path.join(a.ref, "models")), "needs a checkout of the reference"
    for name, (fixture, kind) in CASES.items():
        if a.cases and name not in a.cases:
            continue
        c = dict(MODEL_CASES[name], x_train_var=X_TRAIN_VAR)
        if kind == "trajectory":
            c["steps"] = STEPS
        sd = make_state_dict(seed=c["wseed"], codebook=c["codebook"], codebook_scale=c["codebook_scale"],
                             **{k: c[k] for k in HP})
        x = make_images(c["batch"], c["size"], c["xseed"])
        with tempfile.TemporaryDirectory() as td:
            job = dict(case=c, kind=kind, threads=TRAJECTORY_THREADS,
                       **{"in": os.path.join(td, "in.npz"), "out": os.path.join(td, "out.npz")})
            np.savez(job["in"], __x=x, **sd)
            path = os.path.join(td, "job.json")
            with open(path, "w") as f:
                json.dump(job, f)
            subprocess.run([sys.executable, "-c", _SCRIPT % dict(ref=a.ref), path], check=True, cwd=a.ref,
                           env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
            with np.load(job["out"]) as d:
                out = {k: d[k] for k in d.files}
        if kind == "fingerprints":
            keys = list(sd)
            out = {k: (fingerprint(v, keys.index(k[5:])) if k.startswith("grad/") else v) for k, v in out.items()}
        np.savez_compressed(os.path.join(OUT, fixture + ".npz"), case=json.dumps(c), **out)
        print(fixture, {k: v.shape for k, v in out.items() if not k.startswith("grad/")})


if __name__ == "__main__":
    main()

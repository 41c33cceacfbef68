"""``from models.quantizer import VectorQuantizer`` -- reference models/quantizer.py:10-76."""
import torch

from vqvae_b200 import modules


class VectorQuantizer(modules.VectorQuantizer):
    """vqvae_b200.VectorQuantizer with the reference's constructor (quantizer.py:20) and nothing more: the EMA
    codebook's keywords (``decay``, ``eps``) are on vqvae_b200.VectorQuantizer."""

    def __init__(self, n_e, e_dim, beta):
        super().__init__(n_e, e_dim, beta)


# the reference binds a module-global device at import time (quantizer.py:7, SURVEY Q5);
# kept for callers that read it, unused by the kernels (buffers follow the input's device)
device = torch.device("cuda" if torch.cuda.is_available() else "cpu")

"""``from models.vqvae import VQVAE`` -- reference models/vqvae.py:10-44."""
from vqvae_b200 import modules
from models.encoder import Encoder  # noqa: F401
from models.quantizer import VectorQuantizer  # noqa: F401
from models.decoder import Decoder  # noqa: F401


class VQVAE(modules.VQVAE):
    """vqvae_b200.VQVAE with the reference's constructor (vqvae.py:11-12) and nothing more: the EMA codebook's keywords
    (``ema_decay``, ``ema_eps``) are on vqvae_b200.VQVAE."""

    def __init__(self, h_dim, res_h_dim, n_res_layers, n_embeddings, embedding_dim, beta,
                 save_img_embedding_map=False):
        super().__init__(h_dim, res_h_dim, n_res_layers, n_embeddings, embedding_dim, beta, save_img_embedding_map)

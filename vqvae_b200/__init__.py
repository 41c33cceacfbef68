"""vqvae_b200 -- H100-native (sm_90a) VQ-VAE inference hot path.

Hand-written CUDA kernels behind a C ABI (include/vqvae_b200.h), plus the host-side
mirror of the reference's nn.Module API (vqvae_b200.modules; re-exported by the
top-level ``models`` package so ``from models.vqvae import VQVAE`` drops in).
"""
from .modules import (Decoder, Encoder, ResidualLayer, ResidualStack, VectorQuantizer, VQVAE,  # noqa: F401
                      get_precision, invalidate_packed, packed_state, precision, set_precision)
from .pipeline import HostPipeline, HostResult  # noqa: F401
from .checkpoint import load_checkpoint, save_checkpoint  # noqa: F401
from .prior import GatedPixelCNN  # noqa: F401
from . import optim  # noqa: F401  (vqvae_b200.optim.Adam)

__all__ = ["VQVAE", "VectorQuantizer", "Encoder", "Decoder", "ResidualLayer", "ResidualStack",
           "set_precision", "get_precision", "precision", "invalidate_packed", "packed_state", "HostPipeline",
           "HostResult", "load_checkpoint", "save_checkpoint", "GatedPixelCNN"]

"""``from pixelcnn.models import GatedPixelCNN`` -- reference pixelcnn/models.py, on the sm_90a kernels."""
from vqvae_b200.prior import GatedActivation, GatedMaskedConv2d, GatedPixelCNN, weights_init  # noqa: F401

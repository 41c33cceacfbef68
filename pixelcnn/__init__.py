"""Drop-in for the reference's ``pixelcnn`` package (``from pixelcnn.models import GatedPixelCNN``)."""

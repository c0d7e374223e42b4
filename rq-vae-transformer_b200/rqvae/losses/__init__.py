"""rqvae.losses (reference: rqvae/losses/__init__.py).  Only the LPIPS forward is provided, on the native engine; the stage-1 training
losses (the PatchGAN discriminator, the GAN losses, create_vqgan_loss) and every backward are out of scope."""
from .vqgan import LPIPS

__all__ = ["LPIPS"]

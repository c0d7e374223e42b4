"""rqvae.losses.vqgan (reference: rqvae/losses/vqgan/__init__.py).  Exports LPIPS, whose forward runs on the native engine
(csrc/lpips_engine.cu).  create_vqgan_loss, the discriminator and the GAN losses are training helpers and are not provided."""
from .lpips import LPIPS

__all__ = ["LPIPS"]

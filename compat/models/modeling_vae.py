"""Drop-in for the reference's `models/modeling_vae.py` import path (cvvae_inference_video.py:1,
cvvae_sd3_inference_video.py:1): the same two public classes, backed by the sm_90a engine."""
from cvvae_b200.modeling_vae import (AutoencoderKLOutput, CVVAEModel, CVVAESD3Model, DecoderOutput,  # noqa: F401
                                     DiagonalGaussianDistribution)

__all__ = ["CVVAEModel", "CVVAESD3Model", "DiagonalGaussianDistribution", "DecoderOutput", "AutoencoderKLOutput"]

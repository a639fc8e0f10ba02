"""cvvae_b200 - H100-native (sm_90a) implementation of the CV-VAE encode()/decode() hot path.

Public surface (mirrors the reference's models/modeling_vae.py):
    CVVAEModel, CVVAESD3Model
"""
from .modeling_vae import (AutoencoderKLOutput, CVVAEModel, CVVAESD3Model, DecoderOutput,
                           DiagonalGaussianDistribution)

__all__ = ["CVVAEModel", "CVVAESD3Model", "DecoderOutput", "AutoencoderKLOutput", "DiagonalGaussianDistribution"]
__version__ = "0.1.0"

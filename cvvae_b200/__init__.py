"""cvvae_b200 - H100-native (sm_90a) implementation of the CV-VAE encode()/decode() hot path.

Public surface (mirrors the reference's models/modeling_vae.py):
    CVVAEModel, CVVAESD3Model
Streaming front end for clips of any length (cvvae_b200/streaming.py):
    StreamEncoder, StreamDecoder, reconstruct_frames
"""
from .modeling_vae import (AutoencoderKLOutput, CVVAEModel, CVVAESD3Model, DecoderOutput,
                           DiagonalGaussianDistribution)
from .streaming import StreamDecoder, StreamEncoder, reconstruct_frames

__all__ = ["CVVAEModel", "CVVAESD3Model", "DecoderOutput", "AutoencoderKLOutput", "DiagonalGaussianDistribution",
           "StreamEncoder", "StreamDecoder", "reconstruct_frames"]
__version__ = "0.1.0"

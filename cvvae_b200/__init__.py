"""cvvae_b200 - H100-native (sm_90a) implementation of the CV-VAE encode()/decode() hot path.

Public surface (mirrors the reference's models/modeling_vae.py):
    CVVAEModel, CVVAESD3Model
Streaming front end for clips of any length (cvvae_b200/streaming.py):
    StreamEncoder, StreamDecoder, reconstruct_frames
Reconstruction quality on the device (cvvae_b200/metrics.py): per-frame PSNR / SSIM of uint8 videos, and the
reconstruction stream with every frame scored:
    frame_metrics, FrameMetrics, evaluate_frames
"""
from .modeling_vae import (AutoencoderKLOutput, CVVAEModel, CVVAESD3Model, DecoderOutput,
                           DiagonalGaussianDistribution)
from .metrics import FrameMetrics, frame_metrics
from .streaming import StreamDecoder, StreamEncoder, evaluate_frames, reconstruct_frames

__all__ = ["CVVAEModel", "CVVAESD3Model", "DecoderOutput", "AutoencoderKLOutput", "DiagonalGaussianDistribution",
           "StreamEncoder", "StreamDecoder", "reconstruct_frames", "evaluate_frames", "frame_metrics", "FrameMetrics"]
__version__ = "0.1.0"

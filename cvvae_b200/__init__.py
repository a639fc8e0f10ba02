"""cvvae_b200 - H100-native (sm_90a) implementation of the CV-VAE encode()/decode() hot path.

Public surface (mirrors the reference's models/modeling_vae.py):
    CVVAEModel, CVVAESD3Model
Streaming front end for clips of any length (cvvae_b200/streaming.py):
    StreamEncoder, StreamDecoder, reconstruct_frames
Datasets of clips to latents, with the reference's training pre-processing (streaming.py, video_io.py):
    encode_clips, frames_to_training_input
Reconstruction quality on the device (cvvae_b200/metrics.py): per-frame PSNR / SSIM of uint8 videos, and the
reconstruction stream with every frame scored:
    frame_metrics, FrameMetrics, evaluate_frames
"""
from .modeling_vae import (AutoencoderKLOutput, CVVAEModel, CVVAESD3Model, DecoderOutput,
                           DiagonalGaussianDistribution)
from .metrics import FrameMetrics, frame_metrics
from .streaming import StreamDecoder, StreamEncoder, encode_clips, evaluate_frames, reconstruct_frames
from .video_io import frames_to_training_input

__all__ = ["CVVAEModel", "CVVAESD3Model", "DecoderOutput", "AutoencoderKLOutput", "DiagonalGaussianDistribution",
           "StreamEncoder", "StreamDecoder", "reconstruct_frames", "evaluate_frames",
           "encode_clips", "frames_to_training_input", "frame_metrics", "FrameMetrics"]
__version__ = "0.1.0"

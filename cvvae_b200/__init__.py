"""cvvae_b200 - H100-native (sm_90a) implementation of the CV-VAE encode()/decode() hot path.

Public surface (mirrors the reference's models/modeling_vae.py):
    CVVAEModel, CVVAESD3Model
Streaming front end for clips of any length (cvvae_b200/streaming.py):
    StreamEncoder, StreamDecoder, reconstruct_frames
Datasets of clips to latents, with the reference's training pre-processing (streaming.py, video_io.py):
    encode_clips, frames_to_training_input
Datasets of clip latents back to uint8 videos, batched, in float16, bfloat16 or float32 (streaming.py, video_io.py):
    decode_clips, batch_to_frames
Reconstruction quality on the device (cvvae_b200/metrics.py): per-frame PSNR / SSIM, multi-scale SSIM and LPIPS (VGG16 or,
with ``net="alex"``, AlexNet; weights from a state dict) of uint8 videos, and the reconstruction stream with every frame scored (MS-SSIM with
``ms_ssim=True``, LPIPS with ``lpips=LPIPS.from_state_dict(...)``), and where frames differ: per-position SSIM maps,
LPIPS maps (``LPIPS.map``) and ``evaluate_frames(..., maps=True)``:
    frame_metrics, FrameMetrics, frame_ms_ssim, ssim_map, LPIPS, evaluate_frames
Video sets scored by FVD (cvvae_b200/fvd.py): I3D embeddings on the device (weights from a state dict), a dataset of
clips embedded in batches, and the Fréchet distance of two sets of embeddings:
    I3D, embed_clips, frechet_distance
"""
from .modeling_vae import (AutoencoderKLOutput, CVVAEModel, CVVAESD3Model, DecoderOutput,
                           DiagonalGaussianDistribution)
from .fvd import I3D, frechet_distance
from .metrics import LPIPS, FrameMetrics, frame_metrics, frame_ms_ssim, ssim_map
from .streaming import (StreamDecoder, StreamEncoder, decode_clips, embed_clips, encode_clips, evaluate_frames,
                        reconstruct_frames)
from .video_io import batch_to_frames, frames_to_training_input

__all__ = ["CVVAEModel", "CVVAESD3Model", "DecoderOutput", "AutoencoderKLOutput", "DiagonalGaussianDistribution",
           "StreamEncoder", "StreamDecoder", "reconstruct_frames", "evaluate_frames",
           "encode_clips", "frames_to_training_input", "decode_clips", "batch_to_frames", "frame_metrics", "FrameMetrics",
           "frame_ms_ssim", "ssim_map", "LPIPS", "I3D", "embed_clips", "frechet_distance"]
__version__ = "0.1.0"

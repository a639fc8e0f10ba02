"""Reconstruction quality on the GPU: per-frame PSNR and SSIM of two uint8 videos.

    frame_metrics(a, b)  ->  FrameMetrics(psnr, ssim, sse), host tensors with one entry per frame

`a` and `b` are CUDA uint8 tensors [T, H, W, 3]: typically the frames the network saw (after the script's resize,
cvvae_inference_video.py:28) and the frames it gave back (:47-50).  One kernel (`csrc/metrics.cu`) reads both once and
leaves two 64-bit integers per frame: the exact sum of squared differences over the whole frame, and the sum of the
per-position SSIM values in units of 2^-32.  The scores are derived from them on the host in float64:

    psnr = 10 log10(255^2 * 3HW / sse)                      (+inf for identical frames)
    ssim = mean over channels and the positions whose 11 x 11 window lies inside the frame of
           (2 mu_a mu_b + C1)(2 s_ab + C2) / ((mu_a^2 + mu_b^2 + C1)(s_a^2 + s_b^2 + C2))

with Gaussian window weights (sigma 1.5), population (co)variances, C1 = (0.01 * 255)^2, C2 = (0.03 * 255)^2: Wang et
al. 2004 as the common libraries evaluate it (Gaussian weights, data range 255, 5-pixel border cropped, channels
averaged).  Integer accumulation makes the results bit-reproducible and independent of how the frames are batched.
"""
from __future__ import annotations

from typing import NamedTuple

import torch

from . import _lib as L

_WINDOW = 11


class FrameMetrics(NamedTuple):
    psnr: torch.Tensor   # float64 [T], dB
    ssim: torch.Tensor   # float64 [T]
    sse: torch.Tensor    # int64 [T], sum of squared differences over the frame


@L._on_tensor_device
def _launch(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """The kernel on the current stream of the frames' device: int64 [T, 2] (sse, sum of ssim * 2^32), on the device."""
    T, H, W, _ = a.shape
    acc = torch.empty((T, 2), dtype=torch.int64, device=a.device)
    L.check(L.load().cvvae_frame_metrics(a.data_ptr(), b.data_ptr(), T, H, W, acc.data_ptr(), L._stream(a)),
            "cvvae_frame_metrics")
    return acc


def _scores(acc: torch.Tensor, H: int, W: int) -> FrameMetrics:
    """Host int64 [T, 2] of the kernel -> scores."""
    sse = acc[:, 0].clone()
    psnr = 10.0 * torch.log10((65025.0 * 3 * H * W) / sse.double())
    ssim = acc[:, 1].double() / 4294967296.0 / (3 * (H - _WINDOW + 1) * (W - _WINDOW + 1))
    return FrameMetrics(psnr, ssim, sse)


def frame_metrics(a: torch.Tensor, b: torch.Tensor) -> FrameMetrics:
    """PSNR, SSIM and squared error of every frame of `b` against the same frame of `a` (both CUDA uint8 [T, H, W, 3])."""
    for name, x in (("a", a), ("b", b)):
        if not isinstance(x, torch.Tensor) or x.dtype != torch.uint8 or x.dim() != 4 or x.shape[-1] != 3 or not x.is_cuda:
            raise ValueError(f"frame_metrics expects CUDA uint8 tensors [T, H, W, 3]; `{name}` is "
                             f"{getattr(x, 'dtype', type(x))} {tuple(getattr(x, 'shape', ()))} on {getattr(x, 'device', 'the host')}")
    if a.shape != b.shape or a.device != b.device:
        raise ValueError(f"frame_metrics: `a` and `b` differ: {tuple(a.shape)} on {a.device} vs {tuple(b.shape)} on {b.device}")
    T, H, W, _ = a.shape
    if H < _WINDOW or W < _WINDOW:
        raise ValueError(f"frame_metrics: SSIM needs frames of at least {_WINDOW} x {_WINDOW} px; got {H} x {W}")
    if T == 0:
        return _scores(torch.empty((0, 2), dtype=torch.int64), H, W)
    return _scores(_launch(a.contiguous(), b.contiguous()).cpu(), H, W)

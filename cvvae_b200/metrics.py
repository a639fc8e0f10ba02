"""Reconstruction quality on the GPU: per-frame PSNR, SSIM and multi-scale SSIM of two uint8 videos.

    frame_metrics(a, b)  ->  FrameMetrics(psnr, ssim, sse), host tensors with one entry per frame
    frame_ms_ssim(a, b)  ->  float64 host tensor with one MS-SSIM per frame

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

MS-SSIM (Wang, Simoncelli and Bovik 2003) scores the same comparison at five scales, so that it also sees errors coarser
than the 11-pixel window: level 0 is the frames, level j+1 the 2 x 2 average pool of level j (an odd extent zero-padded
in front: ``F.avg_pool2d(x, 2, padding=(H % 2, W % 2))``).  At level j, per channel c and over the valid positions,

    cs_j(c) = mean of (2 s_ab + C2) / (s_a^2 + s_b^2 + C2),   s_j(c) = mean of the SSIM above   (data range 255 throughout)
    ms(c) = prod_{j<4} max(cs_j(c), 0)^w_j * max(s_4(c), 0)^w_4,   w = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)

and the frame's MS-SSIM is the mean of ms(c) over the three channels.  That is ``pytorch_msssim.ms_ssim(X, Y,
data_range=255, size_average=False)`` on [T, 3, H, W]; torchmetrics' MS-SSIM differs in two places: it floors odd sizes
instead of padding, and it averages the channels before taking the product.  Level 4 must hold the window, so frames
need at least 161 px on each side.  The pooled levels are kept as exact integer sums on the device, and one scoring
kernel per level leaves the sums of cs and SSIM per channel in units of 2^-32; the product is taken on the host in float64.
"""
from __future__ import annotations

from typing import NamedTuple

import torch

from . import _lib as L

_WINDOW = 11
MS_SSIM_WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)
MS_SSIM_MIN_SIZE = 161
MS_SSIM_LAUNCHES = 9          # per call: five levels scored, four pooling steps


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


def _check_frames(a: torch.Tensor, b: torch.Tensor, who: str) -> None:
    for name, x in (("a", a), ("b", b)):
        if not isinstance(x, torch.Tensor) or x.dtype != torch.uint8 or x.dim() != 4 or x.shape[-1] != 3 or not x.is_cuda:
            raise ValueError(f"{who} expects CUDA uint8 tensors [T, H, W, 3]; `{name}` is "
                             f"{getattr(x, 'dtype', type(x))} {tuple(getattr(x, 'shape', ()))} on {getattr(x, 'device', 'the host')}")
    if a.shape != b.shape or a.device != b.device:
        raise ValueError(f"{who}: `a` and `b` differ: {tuple(a.shape)} on {a.device} vs {tuple(b.shape)} on {b.device}")


def frame_metrics(a: torch.Tensor, b: torch.Tensor) -> FrameMetrics:
    """PSNR, SSIM and squared error of every frame of `b` against the same frame of `a` (both CUDA uint8 [T, H, W, 3])."""
    _check_frames(a, b, "frame_metrics")
    T, H, W, _ = a.shape
    if H < _WINDOW or W < _WINDOW:
        raise ValueError(f"frame_metrics: SSIM needs frames of at least {_WINDOW} x {_WINDOW} px; got {H} x {W}")
    if T == 0:
        return _scores(torch.empty((0, 2), dtype=torch.int64), H, W)
    return _scores(_launch(a.contiguous(), b.contiguous()).cpu(), H, W)


def _check_ms_ssim_size(H: int, W: int, who: str) -> None:
    if min(H, W) < MS_SSIM_MIN_SIZE:
        raise ValueError(f"{who}: MS-SSIM needs frames of at least {MS_SSIM_MIN_SIZE} x {MS_SSIM_MIN_SIZE} px (its coarsest "
                         f"of 5 levels, 1/16 of the size, must hold the 11 x 11 window); got {H} x {W}")


@L._on_tensor_device
def _launch_ms_ssim(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """The MS-SSIM kernels on the current stream of the frames' device: int64 [T, 5, 3, 2] (per level and channel, the
    sums of cs and of SSIM times 2^32), on the device.  The pooled levels live in a workspace freed on return."""
    T, H, W, _ = a.shape
    lib = L.load()
    n = lib.cvvae_ms_ssim_workspace_bytes(T, H, W)
    if n < 0:
        L.check(n, "cvvae_ms_ssim_workspace_bytes")
    workspace = torch.empty(n, dtype=torch.uint8, device=a.device)
    acc = torch.empty((T, len(MS_SSIM_WEIGHTS), 3, 2), dtype=torch.int64, device=a.device)
    L.check(lib.cvvae_frame_ms_ssim(a.data_ptr(), b.data_ptr(), T, H, W, workspace.data_ptr(), acc.data_ptr(), L._stream(a)),
            "cvvae_frame_ms_ssim")
    return acc


def _ms_ssim_levels(H: int, W: int) -> list:
    """(h, w) of the five levels: each is the previous one halved, rounded up."""
    sizes = [(H, W)]
    for _ in MS_SSIM_WEIGHTS[1:]:
        h, w = sizes[-1]
        sizes.append(((h + 1) // 2, (w + 1) // 2))
    return sizes


def _ms_ssim_scores(acc: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """Host int64 [T, 5, 3, 2] of the kernels -> MS-SSIM, float64 [T]."""
    n = torch.tensor([(h - _WINDOW + 1) * (w - _WINDOW + 1) for h, w in _ms_ssim_levels(H, W)], dtype=torch.float64)
    means = acc.double() / 4294967296.0 / n[:, None, None]          # [T, 5, 3, 2]: cs_j(c), s_j(c)
    w = torch.tensor(MS_SSIM_WEIGHTS, dtype=torch.float64)
    factors = torch.cat([means[:, :-1, :, 0], means[:, -1:, :, 1]], dim=1).clamp(min=0.0)   # [T, 5, 3]
    return factors.pow(w[:, None]).prod(dim=1).mean(dim=1)


def frame_ms_ssim(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Multi-scale SSIM of every frame of `b` against the same frame of `a` (both CUDA uint8 [T, H, W, 3], H, W >= 161):
    float64 [T] on the host.  The module docstring has the definition."""
    _check_frames(a, b, "frame_ms_ssim")
    T, H, W, _ = a.shape
    _check_ms_ssim_size(H, W, "frame_ms_ssim")
    if T == 0:
        return torch.empty(0, dtype=torch.float64)
    return _ms_ssim_scores(_launch_ms_ssim(a.contiguous(), b.contiguous()).cpu(), H, W)

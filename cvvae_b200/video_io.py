"""GPU pixel pre/post-processing of the reference's inference script, one fused pass each.

    frames_to_input(frames_u8)   ==  rearrange(frames, 't h w c -> c t h w').unsqueeze(0).half() / 127.5 - 1.0
    output_to_frames(x)          ==  rearrange(((clamp(x, -1, 1) + 1.0) * 127.5).to(uint8).squeeze(0), 'c t h w -> t h w c')

(cvvae_inference_video.py:30-38 and :47-50).  Bit-exact with those expressions.  The script's spatial resize
(`transforms.Resize(size=(height, width))` on the uint8 frames, :15-17,28) is available on the GPU as well:
`resize_frames(frames, size)` / `frames_to_input(frames, size=...)` (antialiased bilinear, within 1 LSB of torchvision's
fixed-point uint8 path, which differs from exact arithmetic on < 1 % of the pixels).
"""
from __future__ import annotations

import torch

from . import _lib as L
from .ops import dtype_code


def _check_frames(frames_u8: torch.Tensor, who: str) -> torch.Tensor:
    if frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4 or frames_u8.shape[-1] != 3 or not frames_u8.is_cuda:
        raise ValueError(f"{who} expects a CUDA uint8 tensor [T, H, W, 3]")
    return frames_u8.contiguous()


def resize_frames(frames_u8: torch.Tensor, size) -> torch.Tensor:
    """`transforms.Resize(size=(h, w))` of the script on the GPU: uint8 [T, H, W, 3] -> uint8 [T, h, w, 3]."""
    frames_u8 = _check_frames(frames_u8, "resize_frames")
    T, H, W, _ = frames_u8.shape
    oh, ow = int(size[0]), int(size[1])
    out = torch.empty((T, oh, ow, 3), dtype=torch.uint8, device=frames_u8.device)
    with torch.cuda.device(frames_u8.device):
        L.check(L.load().cvvae_video_resize_u8(frames_u8.data_ptr(), out.data_ptr(), None, T, H, W, oh, ow, L.F16,
                                               torch.cuda.current_stream(out.device).cuda_stream), "cvvae_video_resize_u8")
    return out


def frames_to_input(frames_u8: torch.Tensor, dtype: torch.dtype = torch.float16, size=None) -> torch.Tensor:
    """uint8 [T, H, W, 3] on the GPU -> [1, 3, T, H, W] in [-1, 1]; with `size=(h, w)` the frames are resized first
    (one fused pass: resize -> round to uint8 -> `.half() / 127.5 - 1.0`)."""
    return _to_input(frames_u8, dtype, size, False)[0]


def frames_to_input_and_u8(frames_u8: torch.Tensor, dtype: torch.dtype = torch.float16, size=None):
    """`frames_to_input` plus the uint8 frames the result was computed from, [T, h, w, 3]: the resized frames, written by
    the same launch, or `frames_u8` itself when nothing is resized."""
    return _to_input(frames_u8, dtype, size, True)


def _to_input(frames_u8: torch.Tensor, dtype: torch.dtype, size, want_u8: bool):
    frames_u8 = _check_frames(frames_u8, "frames_to_input")
    T, H, W, _ = frames_u8.shape
    if size is not None and (int(size[0]), int(size[1])) != (H, W):
        oh, ow = int(size[0]), int(size[1])
        out = torch.empty((1, 3, T, oh, ow), dtype=dtype, device=frames_u8.device)
        u8 = torch.empty((T, oh, ow, 3), dtype=torch.uint8, device=frames_u8.device) if want_u8 else None
        with torch.cuda.device(frames_u8.device):
            L.check(L.load().cvvae_video_resize_u8(frames_u8.data_ptr(), u8.data_ptr() if want_u8 else None, out.data_ptr(),
                                                   T, H, W, oh, ow, dtype_code(dtype),
                                                   torch.cuda.current_stream(out.device).cuda_stream), "cvvae_video_resize_u8")
        return out, u8
    out = torch.empty((1, 3, T, H, W), dtype=dtype, device=frames_u8.device)
    L.check(L.load().cvvae_video_u8_to_f16(frames_u8.data_ptr(), out.data_ptr(), T, H, W, dtype_code(dtype),
                                           torch.cuda.current_stream(out.device).cuda_stream), "cvvae_video_u8_to_f16")
    return out, frames_u8


def output_to_frames(x: torch.Tensor) -> torch.Tensor:
    """[1, 3, T, H, W] reconstruction -> uint8 [T, H, W, 3] (clamped to [-1, 1], scaled to 0..255)."""
    if x.dim() != 5 or x.shape[0] != 1 or x.shape[1] != 3 or not x.is_cuda:
        raise ValueError("output_to_frames expects a CUDA tensor [1, 3, T, H, W]")
    x = x.contiguous()
    _, _, T, H, W = x.shape
    out = torch.empty((T, H, W, 3), dtype=torch.uint8, device=x.device)
    L.check(L.load().cvvae_video_f16_to_u8(x.data_ptr(), out.data_ptr(), T, H, W, dtype_code(x.dtype),
                                           torch.cuda.current_stream(x.device).cuda_stream), "cvvae_video_f16_to_u8")
    return out

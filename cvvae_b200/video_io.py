"""GPU pixel pre/post-processing of the reference's inference script, one fused pass each.

    frames_to_input(frames_u8)   ==  rearrange(frames, 't h w c -> c t h w').unsqueeze(0).half() / 127.5 - 1.0
    output_to_frames(x)          ==  rearrange(((clamp(x, -1, 1) + 1.0) * 127.5).to(uint8).squeeze(0), 'c t h w -> t h w c')

(cvvae_inference_video.py:30-38 and :47-50).  Bit-exact with those expressions.  The script's spatial resize
(`transforms.Resize(size=(height, width))` on the uint8 frames, :15-17,28) is available on the GPU as well:
`resize_frames(frames, size)` / `frames_to_input(frames, size=...)` (antialiased bilinear, within 1 LSB of torchvision's
fixed-point uint8 path, which differs from exact arithmetic on < 1 % of the pixels).

The reference's *training* data path prepares frames differently (lvdm/data/decoder.py:99-109, transform.py): float
first, then CoverResize / Resize(short side) and CenterCrop, then `(x / 255 - 0.5) * 2`, never rounded to uint8.
`frames_to_training_input(frames, size, resize)` is that path as one kernel; `training_geometry` its resize and crop sizes.
"""
from __future__ import annotations

import numbers

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


RESIZE_MODES = ("cover", "short")


def _check_size(size) -> tuple:
    """(h, w) of a crop size given as an int (square, as the reference's `resolution`) or a pair."""
    if isinstance(size, numbers.Integral):
        size = (size, size)
    if (not isinstance(size, (tuple, list)) or len(size) != 2
            or not all(isinstance(v, numbers.Integral) and not isinstance(v, bool) and v > 0 for v in size)):
        raise ValueError(f"size must be a positive int or a pair (h, w) of positive ints; got {size!r}")
    return int(size[0]), int(size[1])


def _check_resize(resize) -> str:
    if resize not in RESIZE_MODES:
        raise ValueError(f"resize must be one of {RESIZE_MODES}; got {resize!r}")
    return resize


def training_geometry(H: int, W: int, size, resize: str = "cover") -> tuple:
    """(RH, RW, top, left): the size a [H, W] frame is resized to and the offset of its centre crop of `size`, computed as
    the reference's training transforms compute them (lvdm/data/transform.py):

      "cover":  CoverResize(size) + CenterCrop(size): scale s = max(h / H, w / W), (RH, RW) = (round(H s), round(W s));
      "short":  Resize(min(size)) + CenterCrop(size): the short side becomes min(size), the long side
                int(min(size) * long / short);

    then CenterCrop's top = int(round((RH - h) / 2.0)), left likewise (Python's round: half to even, as torchvision).
    Where CenterCrop would zero-pad (a crop larger than the resized frame: "short" with a non-square size) ValueError is
    raised; the padding is not reproduced."""
    h, w = _check_size(size)
    resize = _check_resize(resize)
    if resize == "cover":
        fh, fw = h / H, w / W
        f = fh if fh > fw else fw
        RH, RW = round(H * f), round(W * f)
    else:
        short, long = (W, H) if W <= H else (H, W)
        new_short, new_long = min(h, w), int(min(h, w) * long / short)
        RW, RH = (new_short, new_long) if W <= H else (new_long, new_short)
    if h > RH or w > RW:
        raise ValueError(f"a {H}x{W} frame resized ({resize!r}) to {RH}x{RW} is smaller than the crop {h}x{w}: "
                         "torchvision's CenterCrop would zero-pad it, which is not reproduced")
    return RH, RW, int(round((RH - h) / 2.0)), int(round((RW - w) / 2.0))


def frames_to_training_input(frames_u8: torch.Tensor, size, resize: str = "cover", dtype: torch.dtype = torch.float16,
                             out: torch.Tensor = None) -> torch.Tensor:
    """The reference's training pre-processing on the GPU: uint8 [T, H, W, 3] -> [1, 3, T, h, w], (h, w) = size.

    Equals, up to fp32 rounding order, ``(center_crop(resize(frames.permute(0, 3, 1, 2).float(), ...)) / 255 - 0.5) * 2``
    with torchvision's antialiased bilinear resize of float tensors and the geometry of ``training_geometry`` ("cover":
    the reference's CoverResize, "short": Resize(min(size))), rearranged to channels-first.  One kernel launch, fp32
    throughout, one rounding to `dtype` (float16, bfloat16 or float32); nothing is rounded to uint8 on the way.
    `out`, if given, is a contiguous [1, 3, T, h, w] tensor of `dtype` on the frames' device - for example one clip's
    slot ``batch[i:i + 1]`` of a batch - and is written in place and returned."""
    frames_u8 = _check_frames(frames_u8, "frames_to_training_input")
    T, H, W, _ = frames_u8.shape
    h, w = _check_size(size)
    RH, RW, top, left = training_geometry(H, W, (h, w), resize)
    if out is None:
        out = torch.empty((1, 3, T, h, w), dtype=dtype, device=frames_u8.device)
    elif (tuple(out.shape) != (1, 3, T, h, w) or out.dtype != dtype or out.device != frames_u8.device
          or not out.is_contiguous()):
        raise ValueError(f"frames_to_training_input: out must be a contiguous {dtype} tensor [1, 3, {T}, {h}, {w}] on "
                         f"{frames_u8.device}; got {out.dtype} {tuple(out.shape)} on {out.device}")
    with torch.cuda.device(frames_u8.device):
        L.check(L.load().cvvae_video_train_input(frames_u8.data_ptr(), out.data_ptr(), T, H, W, RH, RW, top, left, h, w,
                                                 dtype_code(dtype), torch.cuda.current_stream(out.device).cuda_stream),
                "cvvae_video_train_input")
    return out


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

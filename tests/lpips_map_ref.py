"""LPIPS maps (lpips v0.1, ``spatial=True``) restated with torch functional ops on the taps of lpips_ref.py (VGG16) and
lpips_alex_ref.py (AlexNet): per tap the head output sum_c w_k[c] (f^_a - f^_b)^2 at every position, upsampled to the
frame with ``F.interpolate(size=(H, W), mode="bilinear", align_corners=False)``, summed over the five taps.  In any
dtype and on any device; the tests compare the device kernels with it in fp64, and with the same restatement run in
fp32 on the GPU to size the error of a TF32 evaluation."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

import lpips_alex_ref as A
import lpips_ref as R

NETS = {"vgg": R, "alex": A}


def tap_map(f: torch.Tensor, w: torch.Tensor, T: int) -> torch.Tensor:
    """The head output per position of one tap f [2T, C, h, w] (frames of a, then of b) with head w [C]: [T, h, w] in f's
    dtype.  Its mean over positions is lpips_ref.tap_distance."""
    n = torch.sqrt((f * f).sum(1, keepdim=True) + 1e-10)
    fh = f / (n + 1e-10)
    return ((fh[:T] - fh[T:]) ** 2 * w.to(f)[None, :, None, None]).sum(1)


def upsample(m: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """[T, h, w] -> [T, H, W], as lpips' spatial mode upsamples a head output."""
    return F.interpolate(m[:, None], size=(H, W), mode="bilinear", align_corners=False)[:, 0]


def tap_maps(a: torch.Tensor, b: torch.Tensor, sd: dict, net: str = "vgg", dtype=torch.float64,
             tf32_first: bool = False) -> list:
    """The five tap maps [T, h_k, w_k] of uint8 [T, H, W, 3] videos a, b on their device, evaluated in `dtype`.
    `tf32_first`: the first convolution's operands rounded to TF32 (lpips_ref.taps / lpips_alex_ref.taps)."""
    T = a.shape[0]
    x = torch.cat([R.scaled_input(a), R.scaled_input(b)]).to(dtype)
    return [tap_map(f, sd[f"lin{k}.model.1.weight"].flatten(), T)
            for k, f in enumerate(NETS[net].taps(x, sd, tf32_first))]


def lpips_map(a: torch.Tensor, b: torch.Tensor, sd: dict, net: str = "vgg", dtype=torch.float64,
              tf32_first: bool = False) -> torch.Tensor:
    """LPIPS map [T, H, W] of uint8 [T, H, W, 3] videos a, b, evaluated in `dtype`: float64 on the host."""
    H, W = a.shape[1:3]
    return sum(upsample(m, H, W).double().cpu() for m in tap_maps(a, b, sd, net, dtype, tf32_first))


def bilinear_np(m: np.ndarray, H: int, W: int) -> np.ndarray:
    """An independent statement of the upsampling, for one map [h, w] in fp64: per axis, output i reads input
    src = max((i + 0.5) in / out - 0.5, 0), between floor(src) and the next input (the last one clamped)."""
    def axis(n_in, n_out):
        src = np.maximum((np.arange(n_out) + 0.5) * (n_in / n_out) - 0.5, 0.0)
        i0 = np.floor(src).astype(np.int64)
        i1 = np.minimum(i0 + 1, n_in - 1)
        return i0, i1, src - i0

    y0, y1, ly = axis(m.shape[0], H)
    x0, x1, lx = axis(m.shape[1], W)
    top = m[y0][:, x0] * (1 - lx) + m[y0][:, x1] * lx
    bot = m[y1][:, x0] * (1 - lx) + m[y1][:, x1] * lx
    return top * (1 - ly)[:, None] + bot * ly[:, None]

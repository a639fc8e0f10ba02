"""fp64 restatement of the reference's training pre-processing (lvdm/data/decoder.py:99-109, transform.py):
torchvision's antialiased bilinear resize of a float tensor, evaluated only at the centre-crop window, then
(v / 255 - 0.5) * 2.  Used by tests/test_clips_cpu.py (against torchvision itself) and tests/test_gpu_clips.py (against
the cvvae_video_train_input kernel).

The resize is defined by ATen's CPU kernel: scale = float32(in / out), centre c = float32(scale * (i + 0.5)), support
s = max(scale, 1), window [int(float32(c - s) + 0.5), int(float32(c + s) + 0.5)) clipped to the input and to
2 ceil(s) + 1 taps, triangle weights max(0, 1 - |j - c + 0.5| / max(scale, 1)) normalised per axis.  Those float32
centres and windows are part of the definition and are reproduced here; the weights, their normalisation, both sums
and the normalisation are evaluated in fp64.
"""
import math

import numpy as np

U32 = 2.0 ** -24   # unit round-off of fp32


def axis_weights(idx, in_size: int, out_size: int):
    """Normalised weights [len(idx), in_size] of output positions `idx` of a resize in_size -> out_size, plus the tap
    count and the sum of the unnormalised weights of each position (the error bound needs both)."""
    scale = np.float32(np.float32(in_size) / np.float32(out_size))
    support = scale if scale >= 1 else np.float32(1.0)
    inv = 1.0 / float(scale) if scale >= 1 else 1.0
    max_taps = int(math.ceil(float(support))) * 2 + 1
    Wm = np.zeros((len(idx), in_size))
    taps = np.zeros(len(idx), dtype=np.int64)
    sums = np.zeros(len(idx))
    for r, i in enumerate(idx):
        c = np.float32(float(scale) * (i + 0.5))
        lo = max(0, int(float(np.float32(c - support)) + 0.5))
        n = min(in_size, int(float(np.float32(c + support)) + 0.5)) - lo
        n = min(max(n, 0), max_taps)
        j = np.arange(lo, lo + n, dtype=np.float64)
        f = np.maximum(0.0, 1.0 - np.abs((j - float(c) + 0.5) * inv))
        S = f.sum()
        Wm[r, lo:lo + n] = f / S if S != 0 else f
        taps[r], sums[r] = n, S
    return Wm, taps, sums


def train_input_ref(frames_u8: np.ndarray, RH: int, RW: int, top: int, left: int, OH: int, OW: int):
    """uint8 [T, H, W, 3] -> (fp64 [3, T, OH, OW], E [OH, OW]): the crop of the frames resized to RH x RW, normalised,
    and the bound E on how far an fp32 evaluation of it may lie (see `error_bound`)."""
    T, H, W, _ = frames_u8.shape
    Wy, ny, Sy = axis_weights(range(top, top + OH), H, RH)
    Wx, nx, Sx = axis_weights(range(left, left + OW), W, RW)
    x = frames_u8.astype(np.float64)
    v = np.einsum("oh,thwc,pw->ctop", Wy, x, Wx, optimize=True)
    return (v / 255.0 - 0.5) * 2.0, error_bound(nx[None, :], Sx[None, :], ny[:, None], Sy[:, None])


def error_bound(nx, Sx, ny, Sy, sum_roundings: int = 1):
    """Largest |fp32 evaluation - fp64 value| of one normalised output, u = 2^-24, per axis with n taps whose unnormalised
    weights sum to S (first order in u):

      filter argument  fl(fl(j - c) + 0.5) * fl(1 / scale):  |dx| <= 3.5 u (|x| < 1 on every tap that counts)
      weight           fl(1 - |x|):                           |df| <= 4.5 u
      normalisation    fl(f / fl(sum f)):                     sum_j |dw_j| <= u (9 n / S + n)
      weighted sum     n fused multiply-adds over values <= 255:  <= 255 n u  (`sum_roundings` = 2 without FMA)
      -> each axis adds 255 u ((1 + sum_roundings) n + 9 n / S) to v in [0, 255] (the height pass averages the width
      pass's errors, it does not grow them);
      (v / 255 - 0.5) * 2:  2 dv / 255 + 3 u  (the IEEE division and the subtraction; * 2 is exact).
    """
    k = 1 + sum_roundings
    dv = k * nx + 9.0 * nx / Sx + k * ny + 9.0 * ny / Sy
    return U32 * (2.0 * dv + 3.0)


def ulp(ref: np.ndarray, mant_bits: int, min_exp: int) -> np.ndarray:
    """Spacing of a float format with `mant_bits` explicit mantissa bits and smallest normal exponent `min_exp` at the
    exact values `ref` (fp16: 10, -14; bf16: 7, -126; fp32: 23, -126)."""
    _, e = np.frexp(np.abs(ref))
    e = np.maximum(e - 1, min_exp)
    return np.ldexp(1.0, e - mant_bits)


FORMATS = {"fp16": (10, -14), "bf16": (7, -126), "fp32": (23, -126)}


def gate(got: np.ndarray, ref: np.ndarray, E: np.ndarray, fmt: str) -> np.ndarray:
    """Elementwise pass / fail: |got - ref| <= ulp(ref) / 2 + E for a 16-bit output (the final rounding plus the fp32
    evaluation), <= E for an fp32 output (its final rounding is inside E)."""
    half_ulp = 0.0 if fmt == "fp32" else 0.5 * ulp(ref, *FORMATS[fmt])
    return np.abs(got.astype(np.float64) - ref) <= half_ulp + E

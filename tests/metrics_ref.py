"""fp64 reference of the per-frame scores `cvvae_b200.metrics` computes on the GPU: a plain restatement of the definition.

SSIM: for each colour channel and each position whose 11 x 11 window lies inside the frame, means, variances and
covariance of the two frames under the window w = g (x) g, g = the 11-tap Gaussian (sigma 1.5) normalised to sum 1;

    ssim = (2 mu_a mu_b + C1)(2 s_ab + C2) / ((mu_a^2 + mu_b^2 + C1)(s_a^2 + s_b^2 + C2)),  C1 = 2.55^2, C2 = 7.65^2

and the frame's SSIM is the mean over those positions and the three channels.  PSNR = 10 log10(255^2 / mean squared
error) over the whole frame.
"""
import numpy as np
from scipy.ndimage import correlate1d

C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2


def weights() -> np.ndarray:
    k = np.arange(-5, 6, dtype=np.float64)
    g = np.exp(-k * k / (2 * 1.5 ** 2))
    return g / g.sum()


def _window_mean(x: np.ndarray) -> np.ndarray:
    """Weighted mean under the 11 x 11 window at every position whose window lies inside x ([H, W, ...] -> [H-10, W-10, ...])."""
    g = weights()
    y = correlate1d(correlate1d(x, g, axis=0, mode="constant"), g, axis=1, mode="constant")
    return y[5:-5, 5:-5]


def ssim_map(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """SSIM at every valid position of two frames [H, W, C] (any real dtype) -> float64 [H-10, W-10, C]."""
    a, b = a.astype(np.float64), b.astype(np.float64)
    mu_a, mu_b = _window_mean(a), _window_mean(b)
    var_a = _window_mean(a * a) - mu_a * mu_a
    var_b = _window_mean(b * b) - mu_b * mu_b
    cov = _window_mean(a * b) - mu_a * mu_b
    return (2 * mu_a * mu_b + C1) * (2 * cov + C2) / ((mu_a * mu_a + mu_b * mu_b + C1) * (var_a + var_b + C2))


def sse(a: np.ndarray, b: np.ndarray) -> int:
    d = a.astype(np.int64) - b.astype(np.int64)
    return int((d * d).sum())


def psnr_from_sse(s: int, n: int) -> float:
    """n = number of samples (3 H W)."""
    return float("inf") if s == 0 else 10.0 * np.log10(255.0 ** 2 * n / s)


def frame_scores(a: np.ndarray, b: np.ndarray):
    """Two uint8 videos [T, H, W, 3] -> (psnr float64 [T], ssim float64 [T], sse int64 [T])."""
    assert a.shape == b.shape and a.ndim == 4
    s = np.array([sse(x, y) for x, y in zip(a, b)], dtype=np.int64)
    p = np.array([psnr_from_sse(int(v), a[0].size) for v in s], dtype=np.float64)
    q = np.array([ssim_map(x, y).mean() for x, y in zip(a, b)], dtype=np.float64)
    return p, q, s

"""fp64 reference of `cvvae_b200.metrics.frame_ms_ssim`: a plain restatement of multi-scale SSIM (Wang, Simoncelli and
Bovik 2003) as pytorch_msssim evaluates it.

Level 0 is the frame as real numbers; level j+1 is the 2 x 2 average pool of level j, where an axis of odd length n
gets (n+1)/2 outputs out[i] = (x[2i-1] + x[2i]) / 2 with x[-1] = 0 (even length: (x[2i] + x[2i+1]) / 2).  At every
level, per colour channel, with the window and constants of `metrics_ref` (data range 255 at every level) and over the
positions whose 11 x 11 window lies inside the level:

    cs_j(c) = mean of (2 s_ab + C2) / (s_a^2 + s_b^2 + C2),   s_j(c) = mean of the full SSIM
    ms(c)   = prod_{j<4} max(cs_j(c), 0)^w_j * max(s_4(c), 0)^w_4,   w = WEIGHTS

and the frame's MS-SSIM is the mean of ms(c) over the channels.
"""
import numpy as np

import metrics_ref as R

WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)
LEVELS = len(WEIGHTS)


def pool(x: np.ndarray) -> np.ndarray:
    """One 2 x 2 average pool of [H, W, ...] (float64), odd extents zero-padded in front -> [(H+1)//2, (W+1)//2, ...]."""
    H, W = x.shape[:2]
    x = np.pad(x, [(H % 2, 0), (W % 2, 0)] + [(0, 0)] * (x.ndim - 2))
    return (x[0::2, 0::2] + x[1::2, 0::2] + x[0::2, 1::2] + x[1::2, 1::2]) / 4.0


def cs_and_ssim_maps(a: np.ndarray, b: np.ndarray):
    """cs and SSIM at every valid position of two images [H, W, C] (float64) -> two [H-10, W-10, C] maps."""
    mu_a, mu_b = R._window_mean(a), R._window_mean(b)
    var_a = R._window_mean(a * a) - mu_a * mu_a
    var_b = R._window_mean(b * b) - mu_b * mu_b
    cov = R._window_mean(a * b) - mu_a * mu_b
    cs = (2 * cov + R.C2) / (var_a + var_b + R.C2)
    return cs, (2 * mu_a * mu_b + R.C1) / (mu_a * mu_a + mu_b * mu_b + R.C1) * cs


def combine(cs: np.ndarray, s: np.ndarray) -> np.ndarray:
    """Per-level means cs, s [..., 5, 3] -> MS-SSIM [...]."""
    factors = np.concatenate([cs[..., :-1, :], s[..., -1:, :]], axis=-2).clip(min=0.0)
    return (factors ** np.asarray(WEIGHTS)[:, None]).prod(axis=-2).mean(axis=-1)


def frame(a: np.ndarray, b: np.ndarray):
    """Two frames [H, W, 3] -> cs [5, 3], s [5, 3] (means per level and channel) and the MS-SSIM."""
    a, b = a.astype(np.float64), b.astype(np.float64)
    cs, s = np.zeros((LEVELS, 3)), np.zeros((LEVELS, 3))
    for j in range(LEVELS):
        if j:
            a, b = pool(a), pool(b)
        cs_map, s_map = cs_and_ssim_maps(a, b)
        cs[j], s[j] = cs_map.mean(axis=(0, 1)), s_map.mean(axis=(0, 1))
    return cs, s, float(combine(cs, s))


def frame_scores(a: np.ndarray, b: np.ndarray):
    """Two uint8 videos [T, H, W, 3] -> cs [T, 5, 3], s [T, 5, 3], MS-SSIM [T] (float64)."""
    assert a.shape == b.shape and a.ndim == 4 and min(a.shape[1:3]) > 160
    per = [frame(x, y) for x, y in zip(a, b)]
    return (np.array([p[0] for p in per]), np.array([p[1] for p in per]), np.array([p[2] for p in per], dtype=np.float64))

"""Reconstruction scores without a GPU: the fp64 reference (tests/metrics_ref.py) against closed forms, and the refusals,
binding and exports of frame_metrics / evaluate_frames that need no device."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
from scipy.ndimage import gaussian_filter

import metrics_ref as R
from test_engine_wiring_cpu import CASES, build_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _noise(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def test_weights_are_the_common_gaussian():
    g = R.weights()
    assert g.shape == (11,) and abs(g.sum() - 1.0) < 1e-15 and np.array_equal(g, g[::-1])
    impulse = np.zeros(31)
    impulse[15] = 1.0
    theirs = gaussian_filter(impulse, sigma=1.5, truncate=3.5, mode="constant")   # radius int(3.5 * 1.5 + 0.5) = 5
    assert np.count_nonzero(theirs) == 11
    assert np.abs(theirs[10:21] - g).max() < 1e-15


def test_identical_frames():
    a = _noise((2, 20, 23, 3), 0)
    psnr, ssim, sse = R.frame_scores(a, a.copy())
    assert (sse == 0).all() and np.isinf(psnr).all() and (psnr > 0).all()
    assert np.abs(ssim - 1.0).max() < 1e-12
    assert np.abs(R.ssim_map(a[0], a[0]) - 1.0).max() < 1e-9


@pytest.mark.parametrize("c1,c2", [(0, 255), (10, 200), (128, 127), (255, 255)])
def test_constant_frames(c1, c2):
    a = np.full((1, 14, 17, 3), c1, dtype=np.uint8)
    b = np.full((1, 14, 17, 3), c2, dtype=np.uint8)
    _, ssim, sse = R.frame_scores(a, b)
    want = (2.0 * c1 * c2 + R.C1) / (c1 * c1 + c2 * c2 + R.C1)
    assert abs(ssim[0] - want) < 1e-9
    assert sse[0] == (c1 - c2) ** 2 * a.size


@pytest.mark.parametrize("sign", [1, -1])
def test_off_by_one_everywhere(sign):
    a = np.clip(_noise((1, 16, 16, 3), 1), 1, 254)
    b = (a.astype(np.int16) + sign).astype(np.uint8)
    psnr, ssim, sse = R.frame_scores(a, b)
    assert sse[0] == a.size
    assert abs(psnr[0] - 48.1308) < 1e-4        # 20 log10(255)
    assert 0.99 < ssim[0] < 1.0


def test_checkerboard_against_its_inverse_is_negative():
    yy, xx = np.mgrid[0:24, 0:24]
    a = np.repeat((((yy + xx) % 2) * 255).astype(np.uint8)[None, :, :, None], 3, axis=3)
    _, ssim, _ = R.frame_scores(a, 255 - a)
    assert ssim[0] < -0.9


def test_separable_passes_equal_the_dense_window():
    a, b = _noise((13, 16, 3), 2).astype(np.float64), _noise((13, 16, 3), 3).astype(np.float64)
    w = np.outer(R.weights(), R.weights())
    got = R.ssim_map(a, b)
    assert got.shape == (3, 6, 3)
    for y in range(3):
        for x in range(6):
            for c in range(3):
                pa, pb = a[y:y + 11, x:x + 11, c], b[y:y + 11, x:x + 11, c]
                ma, mb = (w * pa).sum(), (w * pb).sum()
                va, vb, vab = (w * pa * pa).sum() - ma * ma, (w * pb * pb).sum() - mb * mb, (w * pa * pb).sum() - ma * mb
                want = (2 * ma * mb + R.C1) * (2 * vab + R.C2) / ((ma * ma + mb * mb + R.C1) * (va + vb + R.C2))
                assert abs(got[y, x, c] - want) < 1e-10


def test_scores_from_the_kernel_sums():
    """The host side of frame_metrics: psnr from the exact integer, ssim from the 2^-32 fixed-point sum."""
    from cvvae_b200.metrics import _scores
    H, W = 20, 31
    n_valid = 3 * (H - 10) * (W - 10)
    acc = torch.tensor([[0, n_valid << 32], [3 * H * W, (n_valid << 32) // 2], [7, -(n_valid << 32) // 4]], dtype=torch.int64)
    m = _scores(acc, H, W)
    assert m.psnr.dtype == m.ssim.dtype == torch.float64 and m.sse.dtype == torch.int64
    assert m.sse.tolist() == [0, 3 * H * W, 7]
    assert m.psnr[0] == float("inf") and abs(m.psnr[1].item() - 20 * np.log10(255.0)) < 1e-12
    assert abs(m.psnr[2].item() - R.psnr_from_sse(7, 3 * H * W)) < 1e-12
    assert m.ssim.tolist() == [1.0, 0.5, -0.25]


def test_frame_metrics_refusals():
    from cvvae_b200 import frame_metrics
    u8 = torch.zeros((2, 16, 16, 3), dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA uint8"):
        frame_metrics(u8, u8)                                   # host tensors
    meta = torch.empty((2, 16, 16, 3), dtype=torch.uint8, device="meta")
    for bad in (u8.float(), u8[0], u8[..., :2], u8.numpy(), meta):
        with pytest.raises(ValueError, match="CUDA uint8"):
            frame_metrics(bad, bad)


@pytest.mark.parametrize("kwargs,match", [
    (dict(), "float16 / bfloat16 only"),                      # fp32 model
    (dict(half=True), "must be on a CUDA device"),             # 16-bit model on the host
])
def test_evaluate_frames_refuses_at_the_call(kwargs, match):
    from cvvae_b200 import evaluate_frames
    m, _ = build_model(CASES["sd21_w32_tiled"])
    if kwargs.get("half"):
        m = m.half()

    def frames():
        raise AssertionError("evaluate_frames read its input before refusing the model")
        yield

    with pytest.raises(ValueError, match="evaluate_frames: .*" + match):
        evaluate_frames(m, frames())


def test_evaluate_frames_needs_temporal_chunking():
    from cvvae_b200 import CVVAEModel, evaluate_frames
    plain = CVVAEModel(ch=32, en_de_n_frames_a_time=None, tile_spatial_size=None).half()
    plain.to("meta")
    with pytest.raises(ValueError):
        evaluate_frames(plain, [])


_CTYPES = {"const uint8_t*": ctypes.c_void_p, "int64_t*": ctypes.c_void_p, "void*": ctypes.c_void_p, "int32_t": ctypes.c_int32}


def test_header_prototype_matches_binding():
    from cvvae_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "cvvae_b200.h")).read(), flags=re.S)
    ret, args = re.search(r"(\w+)\s+cvvae_frame_metrics\s*\(([^)]*)\)\s*;", src).groups()
    types = [re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*") for a in args.split(",")]
    res, argtypes = _lib._SIGNATURES["cvvae_frame_metrics"]
    assert ret == "int" and res is ctypes.c_int
    assert [_CTYPES[t] for t in types] == argtypes
    assert "metrics.cu" in __import__("cvvae_b200._build", fromlist=["SOURCES"]).SOURCES
    assert _lib.ABI_VERSION == 3                                # an added entry point: the ABI version stays


def test_exports():
    import cvvae_b200
    for name in ("frame_metrics", "FrameMetrics", "evaluate_frames", "reconstruct_frames"):
        assert name in cvvae_b200.__all__ and hasattr(cvvae_b200, name)
    assert cvvae_b200.FrameMetrics._fields == ("psnr", "ssim", "sse")


def test_bench_metrics_fails_cleanly_without_a_device():
    import subprocess
    import sys
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    tool = os.path.join(ROOT, "tools", "bench_metrics.py")
    ok = subprocess.run([sys.executable, tool, "--help"], capture_output=True, text=True)
    assert ok.returncode == 0 and "--launches" in ok.stdout
    r = subprocess.run([sys.executable, tool, "--launches", "5"], capture_output=True, text=True)
    assert r.returncode != 0 and "needs a GPU" in r.stderr and "Traceback" not in r.stderr

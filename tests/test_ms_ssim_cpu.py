"""Multi-scale SSIM without a GPU: the fp64 reference (tests/ms_ssim_ref.py) against a second restatement in torch
(conv2d and avg_pool2d, as pytorch_msssim computes it), closed cases, the host combination of the kernel's sums, and
the refusals, binding and argument checks of frame_ms_ssim / evaluate_frames(ms_ssim=True) that need no device."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import metrics_ref as R
import ms_ssim_ref as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _noise(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def _pair(T, H, W, seed):
    """A picture and a noisy, slightly blurred copy of it: the kind of pair a codec gives."""
    a = _noise((T, H, W, 3), seed)
    blur = (a.astype(np.float64) + np.roll(a, 1, axis=2) + np.roll(a, 1, axis=1)) / 3.0
    b = np.clip(blur + np.random.default_rng(seed + 1).normal(0.0, 6.0, a.shape), 0, 255).astype(np.uint8)
    return a, b


def _torch_ms_ssim(a: np.ndarray, b: np.ndarray):
    """The procedure in torch float64 on [T, 3, H, W]: conv2d with the 11 x 11 window (no padding), avg_pool2d with
    padding (H % 2, W % 2) between the levels -> cs [T, 5, 3], s [T, 5, 3], MS-SSIM [T]."""
    x, y = (torch.from_numpy(v).permute(0, 3, 1, 2).double() for v in (a, b))
    g = torch.from_numpy(R.weights())
    win = torch.outer(g, g).expand(3, 1, 11, 11)
    mean = lambda z: F.conv2d(z, win, groups=3)   # noqa: E731
    cs_l, s_l = [], []
    for j in range(5):
        if j:
            x, y = (F.avg_pool2d(z, 2, padding=(z.shape[2] % 2, z.shape[3] % 2)) for z in (x, y))
        mx, my = mean(x), mean(y)
        vx, vy, cxy = mean(x * x) - mx * mx, mean(y * y) - my * my, mean(x * y) - mx * my
        cs = (2 * cxy + R.C2) / (vx + vy + R.C2)
        lum = (2 * mx * my + R.C1) / (mx * mx + my * my + R.C1)
        cs_l.append(cs.mean(dim=(2, 3)))
        s_l.append((lum * cs).mean(dim=(2, 3)))
    cs, s = torch.stack(cs_l, 1), torch.stack(s_l, 1)
    w = torch.tensor(M.WEIGHTS, dtype=torch.float64)
    ms = torch.cat([cs[:, :4], s[:, 4:]], 1).clamp(min=0.0).pow(w[:, None]).prod(1).mean(1)
    return cs.numpy(), s.numpy(), ms.numpy()


@pytest.mark.parametrize("H,W", [(8, 8), (9, 8), (8, 11), (11, 13), (161, 245), (1, 1)])
def test_pooling_is_avg_pool2d_with_front_padding(H, W):
    x = _noise((H, W, 3), H * W).astype(np.float64) * 4.0 + 1.0
    want = F.avg_pool2d(torch.from_numpy(x).permute(2, 0, 1)[None], 2, padding=(H % 2, W % 2))[0].permute(1, 2, 0)
    got = M.pool(x)
    assert got.shape == ((H + 1) // 2, (W + 1) // 2, 3)
    assert np.array_equal(got, want.numpy())           # exact: both add four values and divide by 4


def test_pooled_levels_are_exact_integer_sums():
    """A level-j pixel is a sum of at most 4^j bytes over 4^j: the kernel's uint16 sums hold it exactly."""
    x = _noise((161, 245, 3), 7).astype(np.float64)
    x[:] = 255.0
    for j in range(1, 5):
        x = M.pool(x)
        assert np.array_equal(x * 4 ** j, np.round(x * 4 ** j)) and (x * 4 ** j).max() <= 65280


@pytest.mark.parametrize("T,H,W", [(2, 161, 161), (1, 161, 245), (1, 176, 200), (1, 203, 171)])
def test_reference_equals_the_torch_restatement(T, H, W):
    a, b = _pair(T, H, W, H + W)
    cs, s, ms = M.frame_scores(a, b)
    tcs, ts, tms = _torch_ms_ssim(a, b)
    assert cs.shape == s.shape == (T, 5, 3) and ms.shape == (T,)
    np.testing.assert_allclose(cs, tcs, rtol=0, atol=1e-12)
    np.testing.assert_allclose(s, ts, rtol=0, atol=1e-12)
    np.testing.assert_allclose(ms, tms, rtol=0, atol=1e-12)
    assert 0.0 < ms.min() and ms.max() < 1.0
    # multi-scale is not the finest scale: level 0 alone is the plain SSIM of metrics_ref
    np.testing.assert_allclose(s[:, 0].mean(axis=1), R.frame_scores(a, b)[1], rtol=0, atol=1e-12)


def test_identical_frames_give_exactly_one():
    a = _noise((2, 165, 170, 3), 3)
    cs, s, ms = M.frame_scores(a, a.copy())
    assert (cs == 1.0).all() and (s == 1.0).all() and (ms == 1.0).all()


def test_inverted_checkerboard_gives_zero():
    yy, xx = np.mgrid[0:161, 0:177]
    a = np.repeat((((yy + xx) % 2) * 255).astype(np.uint8)[None, :, :, None], 3, axis=3)
    cs, _, ms = M.frame_scores(a, 255 - a)
    assert (cs[0, 0] < -0.9).all()           # level 0 anti-correlated: max(cs_0, 0) = 0 and the product is 0
    assert ms[0] == 0.0
    assert _torch_ms_ssim(a, 255 - a)[2][0] == 0.0


def test_scores_from_the_kernel_sums():
    """The host side of frame_ms_ssim: means from the 2^-32 fixed-point sums per level, the product in float64."""
    from cvvae_b200.metrics import _ms_ssim_levels, _ms_ssim_scores
    H, W = 161, 245
    sizes = _ms_ssim_levels(H, W)
    assert sizes == [(161, 245), (81, 123), (41, 62), (21, 31), (11, 16)]
    n = np.array([(h - 10) * (w - 10) for h, w in sizes], dtype=np.int64)
    rng = np.random.default_rng(0)
    cs = rng.uniform(-0.2, 1.0, (4, 5, 3))
    s = rng.uniform(-0.2, 1.0, (4, 5, 3))
    cs[0] = s[0] = 1.0                                           # identical frames: exactly 2^32 per position
    acc = np.stack([np.rint(cs * n[:, None] * 2.0 ** 32), np.rint(s * n[:, None] * 2.0 ** 32)], axis=-1).astype(np.int64)
    got = _ms_ssim_scores(torch.from_numpy(acc), H, W)
    assert got.dtype == torch.float64 and got.shape == (4,)
    assert got[0].item() == 1.0
    np.testing.assert_allclose(got.numpy(), M.combine(cs, s), rtol=0, atol=1e-12)


def test_frame_ms_ssim_refusals():
    from cvvae_b200 import frame_ms_ssim
    from cvvae_b200.metrics import _check_ms_ssim_size
    u8 = torch.zeros((2, 176, 176, 3), dtype=torch.uint8)
    with pytest.raises(ValueError, match="frame_ms_ssim expects CUDA uint8"):
        frame_ms_ssim(u8, u8)                                    # host tensors
    meta = torch.empty((2, 176, 176, 3), dtype=torch.uint8, device="meta")
    for bad in (u8.float(), u8[0], u8[..., :2], u8.numpy(), meta):
        with pytest.raises(ValueError, match="CUDA uint8"):
            frame_ms_ssim(bad, bad)
    _check_ms_ssim_size(161, 161, "x")
    for H, W in ((160, 161), (161, 160), (11, 11)):
        with pytest.raises(ValueError, match="x: MS-SSIM needs frames of at least 161 x 161 px"):
            _check_ms_ssim_size(H, W, "x")


class _Net:
    in_channels, z_channels = 3, 4


class _CudaModel:
    """Never reaches the device: the small frames are refused before anything is uploaded."""
    device = torch.device("cuda", 0)
    dtype = torch.float16
    encode_n_frames_a_time, decode_n_frames_a_time = 16, 4
    net = _Net()


@pytest.mark.parametrize("shape,size", [((3, 160, 200, 3), None), ((3, 200, 160, 3), None), ((3, 400, 400, 3), (176, 160)),
                                        ((3, 400, 400, 3), (150, 300))])
def test_evaluate_frames_refuses_small_frames_on_arrival(shape, size, monkeypatch):
    import cvvae_b200.streaming as S

    class NoTransfers:   # the copy stream needs a device; nothing may be uploaded before the refusal anyway
        def __init__(self, dev):
            pass

    monkeypatch.setattr(S, "_HostTransfers", NoTransfers)
    it = S.evaluate_frames(_CudaModel(), [np.zeros((0, 8, 8, 3), np.uint8), np.zeros(shape, np.uint8)], size=size,
                           ms_ssim=True)
    with pytest.raises(ValueError, match="evaluate_frames: MS-SSIM needs frames of at least 161 x 161"):
        next(it)


def test_evaluate_frames_ms_ssim_is_keyword_only():
    import inspect

    from cvvae_b200 import evaluate_frames
    p = inspect.signature(evaluate_frames).parameters["ms_ssim"]
    assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is False


_CTYPES = {"const uint8_t*": ctypes.c_void_p, "int64_t*": ctypes.c_void_p, "void*": ctypes.c_void_p, "int32_t": ctypes.c_int32}


def _header(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "cvvae_b200.h")).read(), flags=re.S)
    ret, args = re.search(rf"(\w+)\s+{name}\s*\(([^)]*)\)\s*;", src).groups()
    return ret, [_CTYPES[re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*")] for a in args.split(",")]


def test_header_prototypes_match_the_binding():
    from cvvae_b200 import _lib as L
    ret, args = _header("cvvae_frame_ms_ssim")
    assert ret == "int" and L._SIGNATURES["cvvae_frame_ms_ssim"] == (ctypes.c_int, args)
    assert args == [ctypes.c_void_p] * 2 + [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 3
    ret, args = _header("cvvae_ms_ssim_workspace_bytes")
    assert ret == "int64_t" and L._SIGNATURES["cvvae_ms_ssim_workspace_bytes"] == (ctypes.c_int64, args)
    assert {"cvvae_frame_ms_ssim", "cvvae_ms_ssim_workspace_bytes"} <= set(L.EXPORTS)
    assert L.ABI_VERSION == 3                                    # added entry points: the ABI version stays


def test_exports():
    import cvvae_b200
    assert "frame_ms_ssim" in cvvae_b200.__all__ and callable(cvvae_b200.frame_ms_ssim)


def test_library_exports_and_refuses_bad_arguments_before_any_launch():
    import __graft_entry__ as ge
    ge.build()
    from cvvae_b200 import _lib as L
    lib = L.load()
    assert hasattr(lib, "cvvae_frame_ms_ssim") and hasattr(lib, "cvvae_ms_ssim_workspace_bytes")
    # the workspace: levels 1-4 of both videos as uint16, each level's buffer rounded up to 256 bytes
    for T, H, W in ((1, 161, 161), (17, 576, 1024), (3, 721, 1279), (0, 200, 300)):
        want, h, w = 0, H, W
        for _ in range(4):
            h, w = (h + 1) // 2, (w + 1) // 2
            want += 2 * ((2 * T * h * w * 3 + 255) // 256 * 256)
        assert lib.cvvae_ms_ssim_workspace_bytes(T, H, W) == want
    for args in ((-1, 200, 200), (1, 0, 200), (1, 200, -5)):
        assert lib.cvvae_ms_ssim_workspace_bytes(*args) == -1
        assert lib.cvvae_last_error().startswith(b"cvvae_ms_ssim_workspace_bytes")
    fake = 256   # never dereferenced: every check precedes the first launch
    before = lib.cvvae_launch_count()
    for args, msg in (((None, fake, 1, 200, 200, fake, fake), b"null pointer"),
                      ((fake, None, 1, 200, 200, fake, fake), b"null pointer"),
                      ((fake, fake, 1, 200, 200, None, fake), b"null pointer"),
                      ((fake, fake, 1, 200, 200, fake, None), b"null pointer"),
                      ((fake, fake, -1, 200, 200, fake, fake), b"T=-1"),
                      ((fake, fake, 1, 160, 200, fake, fake), b"at least 161 x 161"),
                      ((fake, fake, 1, 200, 160, fake, fake), b"at least 161 x 161"),
                      ((fake, fake, 1, 30000, 30000, fake, fake), b"3*H*W < 2^31"),
                      ((fake, fake, 1, 200, 200, fake + 8, fake), b"16-byte aligned"),
                      ((fake, fake, 2 ** 27, 161, 161, fake, fake), b"too many frames")):
        assert lib.cvvae_frame_ms_ssim(*args, None) == -1, args
        assert lib.cvvae_last_error().startswith(b"cvvae_frame_ms_ssim") and msg in lib.cvvae_last_error(), args
    assert lib.cvvae_frame_ms_ssim(fake, fake, 0, 200, 200, fake, fake, None) == 0     # T = 0: nothing to do
    assert lib.cvvae_launch_count() == before

"""Error maps without a GPU: the fp64 LPIPS-map restatement (tests/lpips_map_ref.py) against an independent numpy
statement of the bilinear upsampling at interior and clamped edge positions, its closed cases (a constant map stays
constant, a tap map's mean is the tap distance), the binding against the header, the library's argument checks for the
new entry points, and the Python refusals of ssim_map, LPIPS.map and evaluate_frames(maps=...)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import lpips_alex_ref as A
import lpips_map_ref as M
import lpips_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_NEW = ("cvvae_frame_ssim_map", "cvvae_lpips_tap_map", "cvvae_lpips_upsample_sum")


def _frames(T, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (T, H, W, 3), generator=g, dtype=torch.uint8)


@pytest.mark.parametrize("h,w,H,W", [(1, 1, 16, 16), (2, 3, 16, 16), (4, 6, 64, 96), (23, 37, 23, 37), (7, 11, 31, 47),
                                     (36, 64, 576, 1024), (3, 5, 2, 4)])
def test_upsampling_is_the_independent_bilinear_formula(h, w, H, W):
    g = torch.Generator().manual_seed(h * w + H)
    m = torch.rand((2, h, w), generator=g, dtype=torch.float64)
    got = M.upsample(m, H, W).numpy()
    for t in range(2):
        want = M.bilinear_np(m[t].numpy(), H, W)
        np.testing.assert_allclose(got[t], want, rtol=1e-14, atol=1e-15)
    if H > h:   # upsampling: the first output row reads input row 0 alone (i0 clamped at 0), the last one row h - 1 alone
        np.testing.assert_allclose(got[:, 0, :], M.upsample(m[:, :1, :], 1, W).numpy()[:, 0, :], rtol=1e-14, atol=1e-15)
        np.testing.assert_allclose(got[:, -1, :], M.upsample(m[:, -1:, :], 1, W).numpy()[:, 0, :], rtol=1e-14, atol=1e-15)


def test_edge_positions_clamp_as_pytorch_does():
    """Explicit values at the clamped edges: with h = 2 -> H = 8 (scale 1/4), output row 0 has src = -0.375 -> 0 (row 0
    alone), row 7 has src = 1.375 -> i0 = 1 = h - 1, i1 clamped to 1 (row 1 alone); row 3 has src = 0.375 (interior)."""
    m = torch.tensor([[[1.0, 5.0], [3.0, 9.0]]], dtype=torch.float64)
    up = M.upsample(m, 8, 8)[0]
    assert up[0, 0] == 1.0 and up[0, 7] == 5.0 and up[7, 0] == 3.0 and up[7, 7] == 9.0
    assert up[3, 0] == 0.625 * 1.0 + 0.375 * 3.0
    assert up[0, 3] == 0.625 * 1.0 + 0.375 * 5.0
    np.testing.assert_array_equal(up.numpy(), M.bilinear_np(m[0].numpy(), 8, 8))


@pytest.mark.parametrize("h,w,H,W", [(1, 1, 16, 16), (3, 5, 31, 47), (36, 64, 576, 1024)])
def test_a_constant_map_stays_constant(h, w, H, W):
    m = torch.full((1, h, w), 0.3125, dtype=torch.float64)
    up = M.upsample(m, H, W)
    assert up.shape == (1, H, W)
    torch.testing.assert_close(up, torch.full_like(up, 0.3125), rtol=4e-16, atol=0)   # (1 - l) v + l v: one rounding


@pytest.mark.parametrize("net,H,W", [("vgg", 16, 16), ("vgg", 23, 37), ("alex", 31, 31), ("alex", 33, 47)])
def test_tap_map_means_are_the_tap_distances_and_the_map_is_their_upsampled_sum(net, H, W):
    ref = R if net == "vgg" else A
    sd = ref.make_state_dict(7)
    a, b = _frames(2, H, W, 1), _frames(2, H, W, 2)
    with torch.no_grad():
        maps = M.tap_maps(a, b, sd, net)
        x = torch.cat([R.scaled_input(a), R.scaled_input(b)]).double()
        for k, (m, f) in enumerate(zip(maps, ref.taps(x, sd))):
            assert m.shape == (2, *f.shape[2:])
            d = R.tap_distance(f, sd[f"lin{k}.model.1.weight"].flatten(), 2)
            torch.testing.assert_close(m.mean((1, 2)), d, rtol=1e-13, atol=0)
        full = M.lpips_map(a, b, sd, net)
        assert full.shape == (2, H, W) and full.dtype == torch.float64
        want = sum(torch.from_numpy(np.stack([M.bilinear_np(m[t].numpy(), H, W) for t in range(2)])) for m in maps)
        torch.testing.assert_close(full, want, rtol=1e-13, atol=1e-15)
        # the map's mean is close to, but in general not, the scalar: upsampling with clamped edges moves the mean
        scalar = ref.lpips(a, b, sd)
        assert ((full.mean((1, 2)) - scalar).abs() <= 0.5 * scalar).all()
        assert (M.lpips_map(a, a.clone(), sd, net) == 0).all()


_CTYPES = {"const uint8_t*": ctypes.c_void_p, "const float*": ctypes.c_void_p, "float*": ctypes.c_void_p,
           "int64_t*": ctypes.c_void_p, "void*": ctypes.c_void_p, "int32_t": ctypes.c_int32, "double*": ctypes.c_void_p,
           "const double*": ctypes.c_void_p, "const int32_t*": ctypes.POINTER(ctypes.c_int32)}


def _header(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "cvvae_b200.h")).read(), flags=re.S)
    ret, args = re.search(rf"(\w+)\s+{name}\s*\(([^)]*)\)\s*;", src).groups()
    return ret, [_CTYPES[re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*")] for a in args.split(",")]


def test_api_surface():
    import cvvae_b200
    from cvvae_b200 import _lib as L
    from cvvae_b200 import metrics
    for name in _NEW:
        ret, args = _header(name)
        assert ret == "int" and L._SIGNATURES[name] == (ctypes.c_int, args) and name in L.EXPORTS, name
    assert L.ABI_VERSION == 3
    assert "ssim_map" in cvvae_b200.__all__ and cvvae_b200.ssim_map is metrics.ssim_map
    assert callable(metrics.LPIPS.map)


def test_library_refuses_bad_arguments_before_any_launch():
    import __graft_entry__ as ge
    ge.build()
    from cvvae_b200 import _lib as L
    lib = L.load()
    fake = 256
    before = lib.cvvae_launch_count()
    for args, msg in (((None, fake, 1, 16, 16, fake, fake), b"null pointer"),
                      ((fake, fake, 1, 16, 16, None, fake), b"null pointer"),
                      ((fake, fake, 1, 16, 16, fake, None), b"null pointer"),
                      ((fake, fake, -1, 16, 16, fake, fake), b"T=-1"),
                      ((fake, fake, 1, 10, 16, fake, fake), b"H=10"),
                      ((fake, fake, 1, 16, 10, fake, fake), b"W=10"),
                      ((fake, fake, 1, 30000, 30000, fake, fake), b"3*H*W < 2^31"),
                      ((fake, fake, 1, 16, 16, fake, fake + 2), b"4-byte aligned")):
        assert lib.cvvae_frame_ssim_map(*args, None) == -1, args
        assert lib.cvvae_last_error().startswith(b"cvvae_frame_ssim_map") and msg in lib.cvvae_last_error(), args
    assert lib.cvvae_frame_ssim_map(fake, fake, 0, 16, 16, fake, fake, None) == 0
    for args, msg in (((fake, 1, 8, 8, 64, fake, fake, fake, fake, fake), b"at most one of pooled and copy"),
                      ((fake, 1, 8, 8, 64, fake, fake, None, None, None), b"null pointer"),
                      ((None, 1, 8, 8, 64, fake, fake, None, None, fake), b"null pointer"),
                      ((fake, 1, 8, 8, 64, fake, fake, None, None, fake + 4), b"8-byte aligned"),
                      ((fake, 1, 8, 8, 96, fake, fake, None, None, fake), b"C must be"),
                      ((fake, 1, 8, 8, 192, fake, fake, None, fake, fake), b"C must be 256 or 384"),
                      ((fake, 1, 1, 8, 64, fake, fake, fake, None, fake), b"pooling needs"),
                      ((fake, -1, 8, 8, 64, fake, fake, None, None, fake), b"T=-1"),
                      ((fake, 1, 4096, 4096, 64, fake, fake, None, None, fake), b"H*W <= 2^23"),
                      ((fake, 1, 8, 8, 256, fake, fake, None, fake + 8, fake), b"copy must be 16-byte aligned"),
                      ((fake, 2 ** 30, 64, 64, 64, fake, fake, None, None, fake), b"too many frames")):
        assert lib.cvvae_lpips_tap_map(*args, None) == -1, args
        assert lib.cvvae_last_error().startswith(b"cvvae_lpips_tap_map") and msg in lib.cvvae_last_error(), args
    assert lib.cvvae_lpips_tap_map(fake, 0, 8, 8, 384, fake, fake, None, fake, fake, None) == 0
    hw = (ctypes.c_int32 * 10)(16, 16, 8, 8, 4, 4, 2, 2, 1, 1)
    bad_hw = (ctypes.c_int32 * 10)(16, 16, 8, 8, 4, 0, 2, 2, 1, 1)
    for args, msg in (((None, 1, 16, 16, hw, fake), b"null pointer"), ((fake, 1, 16, 16, None, fake), b"null pointer"),
                      ((fake, 1, 16, 16, hw, None), b"null pointer"), ((fake, -1, 16, 16, hw, fake), b"T=-1"),
                      ((fake, 1, 0, 16, hw, fake), b"H=0"), ((fake + 4, 1, 16, 16, hw, fake), b"aligned"),
                      ((fake, 1, 16, 16, hw, fake + 2), b"aligned"), ((fake, 1, 16, 16, bad_hw, fake), b"tap 2 is 4 x 0"),
                      ((fake, 2 ** 30, 1024, 1024, hw, fake), b"too many positions")):
        assert lib.cvvae_lpips_upsample_sum(*args, None) == -1, args
        assert lib.cvvae_last_error().startswith(b"cvvae_lpips_upsample_sum") and msg in lib.cvvae_last_error(), args
    assert lib.cvvae_lpips_upsample_sum(fake, 0, 16, 16, hw, fake, None) == 0
    assert lib.cvvae_launch_count() == before


def test_python_refusals():
    from cvvae_b200 import metrics
    from cvvae_b200 import streaming as S
    from test_ms_ssim_cpu import _CudaModel
    a = torch.zeros((1, 16, 16, 3), dtype=torch.uint8)
    for x, y in ((a, a), (a.float(), a.float()), (a[..., :2], a[..., :2]), (a[0], a[0])):
        with pytest.raises(ValueError, match="ssim_map expects CUDA uint8"):
            metrics.ssim_map(x, y)
    m = object.__new__(metrics.LPIPS)
    m.device, m.net = torch.device("cuda", 0), "vgg"
    for x, y in ((a, a), (a.int(), a.int())):
        with pytest.raises(ValueError, match="LPIPS.map expects CUDA uint8"):
            m.map(x, y)
    for maps in (1, 0, "yes", None, np.bool_(True)):
        with pytest.raises(ValueError, match="`maps` must be a bool"):
            S.evaluate_frames(_CudaModel(), [], maps=maps)


def test_map_group_sizing_leaves_the_scalar_path_alone():
    from cvvae_b200 import metrics
    for net in ("vgg", "alex"):
        m = object.__new__(metrics.LPIPS)
        m.net, m._group_bytes = net, metrics.LPIPS_GROUP_BYTES
        spec = metrics._NETS[net]
        for H, W in ((576, 1024), (720, 1280), (2160, 3840)):
            assert m._group(H, W) == max(1, metrics.LPIPS_GROUP_BYTES // spec.pair_bytes(H, W))
            extra = 8 * sum(h * w for h, w in spec.tap_sizes(H, W)) + 4 * H * W
            # VGG16: about 15 B per pixel (its taps hold 4/3 of the frame's positions); AlexNet: under 5 B
            assert (14 * H * W <= extra <= 15 * H * W) if net == "vgg" else (4 * H * W < extra < 5 * H * W)
            assert m._group(H, W, maps=True) == max(1, metrics.LPIPS_GROUP_BYTES // (spec.pair_bytes(H, W) + extra))

"""LPIPS without a GPU: the fp64 restatement (tests/lpips_ref.py) against torchvision's VGG16, the weight loader's
layouts and refusals, the host combination of the tap sums, the binding against the header and the library's argument
checks, which must refuse before anything is launched."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lpips_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _frames(T, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (T, H, W, 3), generator=g, dtype=torch.uint8)


@pytest.mark.parametrize("H,W", [(16, 16), (23, 37), (64, 96)])
def test_restatement_equals_torchvision_vgg16(H, W):
    import torchvision
    sd = R.make_state_dict(1)
    vgg = torchvision.models.vgg16(weights=None).features[:30].double().eval()
    vgg.load_state_dict({k[len("features."):]: v for k, v in sd.items() if k.startswith("features.")})
    a, b = _frames(2, H, W, 2), _frames(2, H, W, 3)
    x = torch.cat([R.scaled_input(a), R.scaled_input(b)]).double()
    want = torch.zeros(2, dtype=torch.float64)
    k = 0
    with torch.no_grad():
        for i, layer in enumerate(vgg):
            x = layer(x)
            if i in (3, 8, 15, 22, 29):          # relu1_2 .. relu5_3
                fh = x / (torch.sqrt((x * x).sum(1, keepdim=True) + 1e-10) + 1e-10)
                head = sd[f"lin{k}.model.1.weight"].double()
                want += F.conv2d((fh[:2] - fh[2:]) ** 2, head).mean((1, 2, 3))
                k += 1
        got = R.lpips(a, b, sd)
    assert k == 5
    assert (got - want).abs().max().item() <= 1e-12 * want.abs().max().item(), (got, want)
    assert (R.lpips(a, a, sd) == 0).all()


def test_both_key_layouts_load_the_same_weights():
    from cvvae_b200.metrics import _lpips_weights
    sd = R.make_state_dict(5)
    c1, h1 = _lpips_weights((sd,))
    c2, h2 = _lpips_weights((R.to_reference_layout(sd),))
    assert len(c1) == 13 and len(h1) == 5
    for (w1, b1), (w2, b2) in zip(c1, c2):
        assert torch.equal(w1, w2) and torch.equal(b1, b2)
    assert all(torch.equal(x, y) for x, y in zip(h1, h2))
    # merged dicts: torchvision's VGG16 plus the lpips heads, unused keys ignored
    vgg = {k: v for k, v in sd.items() if k.startswith("features.")}
    vgg["classifier.0.weight"] = torch.zeros(3, 3)
    heads = {k: v for k, v in sd.items() if k.startswith("lin")}
    c3, h3 = _lpips_weights((vgg, heads))
    assert all(torch.equal(w1, w3) for (w1, _), (w3, _) in zip(c1, c3)) and all(torch.equal(x, y) for x, y in zip(h1, h3))


@pytest.mark.parametrize("edit,msg", [
    (lambda sd: sd.pop("features.0.weight"), "missing key 'features.0.weight'"),
    (lambda sd: sd.pop("features.28.bias"), "missing key 'features.28.bias'"),
    (lambda sd: sd.pop("lin3.model.1.weight"), "missing key 'lin3.model.1.weight'"),
    (lambda sd: sd.__setitem__("features.5.weight", torch.zeros(128, 64, 3, 2)), "'features.5.weight' has shape"),
    (lambda sd: sd.__setitem__("lin0.model.1.weight", torch.zeros(1, 32, 1, 1)), "'lin0.model.1.weight' has shape"),
    (lambda sd: sd.__setitem__("features.2.bias", torch.zeros(64, dtype=torch.int32)), "'features.2.bias' is torch.int32"),
    (lambda sd: sd.__setitem__("lin1.model.1.weight", torch.full((1, 128, 1, 1), 33.0)), "|w| > 32"),
    (lambda sd: sd.__setitem__("features.7.bias", torch.full((128,), float("nan"))), "non-finite"),
    (lambda sd: sd.__setitem__("scaling_layer.shift", torch.zeros(1, 3, 1, 1)), "'scaling_layer.shift' is"),
    (lambda sd: sd.__setitem__("scaling_layer.scale", torch.ones(1, 3)), "'scaling_layer.scale' has shape"),
])
def test_loader_refusals(edit, msg):
    from cvvae_b200 import LPIPS
    sd = R.make_state_dict(7)
    edit(sd)
    with pytest.raises(ValueError, match=re.escape(msg)):
        LPIPS.from_state_dict(sd)


def test_loader_refuses_a_host_device():
    from cvvae_b200 import LPIPS
    with pytest.raises(ValueError, match="must be a CUDA device"):
        LPIPS.from_state_dict(R.make_state_dict(7), device="cpu")


def test_metric_refuses_bad_frames_before_any_device_work():
    from cvvae_b200.metrics import LPIPS
    m = object.__new__(LPIPS)
    m.device = torch.device("cuda", 0)
    ok = torch.zeros((2, 16, 16, 3), dtype=torch.uint8)
    for a, b in ((ok, ok), (ok.float(), ok), (ok[..., :2], ok[..., :2]), (ok[0], ok[0])):
        with pytest.raises(ValueError, match="LPIPS expects CUDA uint8 tensors"):
            m(a, b)


def test_scores_from_the_tap_sums():
    from cvvae_b200.metrics import _lpips_scores, _lpips_tap_sizes
    assert _lpips_tap_sizes(23, 37) == [(23, 37), (11, 18), (5, 9), (2, 4), (1, 2)]
    acc = torch.tensor([[2 ** 32 * 23 * 37, 0], [0, 2 ** 31 * 11 * 18], [0, 0], [2 ** 32 * 8, 0], [0, -(2 ** 30) * 2]])
    got = _lpips_scores(acc, 23, 37)
    assert got.dtype == torch.float64 and got.tolist() == [2.0, 0.5 - 0.25]


@pytest.mark.parametrize("shape,size", [((3, 15, 40, 3), None), ((3, 40, 15, 3), None), ((3, 64, 64, 3), (8, 32))])
def test_evaluate_frames_refuses_small_frames_on_arrival(shape, size, monkeypatch):
    import cvvae_b200.streaming as S
    from cvvae_b200.metrics import LPIPS
    from test_ms_ssim_cpu import _CudaModel

    class NoTransfers:
        def __init__(self, dev):
            pass

    monkeypatch.setattr(S, "_HostTransfers", NoTransfers)
    m = object.__new__(LPIPS)
    m.device = torch.device("cuda", 0)
    it = S.evaluate_frames(_CudaModel(), [np.zeros((0, 8, 8, 3), np.uint8), np.zeros(shape, np.uint8)], size=size, lpips=m)
    with pytest.raises(ValueError, match="evaluate_frames: LPIPS needs frames of at least 16 x 16"):
        next(it)


def test_frames_beyond_the_fixed_point_range_are_refused_before_any_launch():
    from cvvae_b200.metrics import LPIPS_GROUP_BYTES, LPIPS_MAX_POSITIONS, _check_lpips_size
    _check_lpips_size(2160, 3840, "LPIPS")                       # 8.3 M px: 4K fits
    for H, W in ((2304, 4096), (2 ** 12 + 1, 2 ** 11)):
        with pytest.raises(ValueError, match="at most 2\\^23 px"):
            _check_lpips_size(H, W, "LPIPS")
    # one frame pair of the largest accepted size fits the group budget: conv1_2's input and output, 2 x 128 fp32 channels
    assert 2 * 128 * 4 * LPIPS_MAX_POSITIONS <= LPIPS_GROUP_BYTES


def test_evaluate_frames_refuses_an_lpips_on_another_device_at_the_call():
    import cvvae_b200.streaming as S
    from cvvae_b200.metrics import LPIPS
    from test_ms_ssim_cpu import _CudaModel
    m = object.__new__(LPIPS)
    m.device = torch.device("cuda", 1)
    with pytest.raises(ValueError, match="the LPIPS weights are on cuda:1, the model on cuda:0"):
        S.evaluate_frames(_CudaModel(), [], lpips=m)
    with pytest.raises(ValueError, match="must be a metrics.LPIPS"):
        S.evaluate_frames(_CudaModel(), [], lpips=object())


_CTYPES = {"const uint8_t*": ctypes.c_void_p, "const float*": ctypes.c_void_p, "float*": ctypes.c_void_p,
           "int64_t*": ctypes.c_void_p, "void*": ctypes.c_void_p, "int32_t": ctypes.c_int32}


def _header(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "cvvae_b200.h")).read(), flags=re.S)
    ret, args = re.search(rf"(\w+)\s+{name}\s*\(([^)]*)\)\s*;", src).groups()
    return ret, [_CTYPES[re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*")] for a in args.split(",")]


def test_header_prototypes_and_flag_match_the_binding():
    from cvvae_b200 import _lib as L
    from cvvae_b200 import metrics
    for name in ("cvvae_lpips_input", "cvvae_lpips_tap"):
        ret, args = _header(name)
        assert ret == "int" and L._SIGNATURES[name] == (ctypes.c_int, args) and name in L.EXPORTS
    hdr = open(os.path.join(ROOT, "include", "cvvae_b200.h")).read()
    assert int(re.search(r"CVVAE_CONV_RELU = (\d+)", hdr).group(1)) == L.CONV_RELU == 32
    assert int(re.search(r"CVVAE_CONV_TF32_OUT = (\d+)", hdr).group(1)) == L.CONV_TF32_OUT == 64
    assert L.ABI_VERSION == 3
    assert metrics.LPIPS_LAUNCHES == 1 + 13 + 5
    import cvvae_b200
    assert "LPIPS" in cvvae_b200.__all__ and cvvae_b200.LPIPS is metrics.LPIPS


def _desc(L, dtype, flags, cin=64, cout=64, **kw):
    fake = 256
    d = L.ConvDesc()
    d.x = L.Tensor5(fake, 2, 1, 8, 8, cin, 64 * cin, 64 * cin, 8 * cin, cin, 1)
    d.y = L.Tensor5(fake, 2, 1, 8, 8, cout, 64 * cout, 64 * cout, 8 * cout, cout, 1)
    d.w, d.Cout, d.KT, d.KH, d.KW = fake, cout, 1, 3, 3
    d.st = d.sh = d.sw = 1
    d.off_h = d.off_w = -1
    d.up_time, d.dtype, d.flags, d.alpha = 1, dtype, flags, 1.0
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_library_refuses_bad_arguments_before_any_launch():
    import __graft_entry__ as ge
    ge.build()
    from cvvae_b200 import _lib as L
    lib = L.load()
    fake = 256
    before = lib.cvvae_launch_count()
    for args, msg in (((None, fake, 1, 16, 16, fake), b"null pointer"), ((fake, fake, 1, 16, 16, None), b"null pointer"),
                      ((fake, fake, -1, 16, 16, fake), b"T=-1"), ((fake, fake, 1, 0, 16, fake), b"H=0"),
                      ((fake, fake, 1, 16, 16, fake + 4), b"16-byte aligned"),
                      ((fake, fake, 2 ** 30, 256, 256, fake), b"too many positions")):
        assert lib.cvvae_lpips_input(*args, None) == -1, args
        assert lib.cvvae_last_error().startswith(b"cvvae_lpips_input") and msg in lib.cvvae_last_error(), args
    assert lib.cvvae_lpips_input(fake, fake, 0, 16, 16, fake, None) == 0
    for args, msg in (((None, 1, 8, 8, 64, fake, fake, fake), b"null pointer"),
                      ((fake, 1, 8, 8, 64, None, fake, fake), b"null pointer"),
                      ((fake, 1, 8, 8, 64, fake, None, fake), b"null pointer"),
                      ((fake, 1, 8, 8, 96, fake, fake, fake), b"C must be"),
                      ((fake, -1, 8, 8, 64, fake, fake, fake), b"T=-1"),
                      ((fake, 1, 1, 8, 64, fake, fake, fake), b"pooling needs"),
                      ((fake, 1, 4096, 4096, 64, fake, fake, None), b"H*W <= 2^23"),
                      ((fake + 8, 1, 8, 8, 64, fake, fake, fake), b"16-byte aligned"),
                      ((fake, 1, 8, 8, 64, fake, fake, fake + 8), b"16-byte aligned"),
                      ((fake, 2 ** 30, 64, 64, 64, fake, fake, None), b"too many frames")):
        assert lib.cvvae_lpips_tap(*args, None) == -1, args
        assert lib.cvvae_last_error().startswith(b"cvvae_lpips_tap") and msg in lib.cvvae_last_error(), args
    assert lib.cvvae_lpips_tap(fake, 0, 8, 8, 64, fake, fake, fake, None) == 0
    # CVVAE_CONV_RELU: refused before any launch everywhere it is not the fp32 tensor-core register epilogue
    R_ = L.CONV_RELU
    refused = [(lib.cvvae_conv3d_tc, _desc(L, L.F16, R_)), (lib.cvvae_conv3d_tc, _desc(L, L.BF16, R_)),
               (lib.cvvae_conv3d, _desc(L, L.F16, R_)), (lib.cvvae_conv3d_direct, _desc(L, L.F32, R_)),
               (lib.cvvae_conv3d, _desc(L, L.F32, R_ | L.CONV_FORCE_DIRECT)),
               (lib.cvvae_conv3d, _desc(L, L.F32, R_, cin=3)),          # not eligible for the tensor-core path
               (lib.cvvae_conv3d_stacked, _desc(L, L.F16, R_, cout=3)),
               (lib.cvvae_conv3d_tc, _desc(L, L.F32, R_, residual=fake)),
               (lib.cvvae_conv3d_tc, _desc(L, L.F32, R_, gn_stats=fake, gn_groups=32)),
               (lib.cvvae_conv3d_tc, _desc(L, L.F32, R_, w2=fake)),
               (lib.cvvae_conv3d_tc, _desc(L, L.F32, R_, up_time=2)),
               (lib.cvvae_conv3d, _desc(L, L.F32, R_, residual=fake)),
               (lib.cvvae_conv3d_tc, _desc(L, L.F16, R_ | L.CONV_TF32_OUT)),
               (lib.cvvae_conv3d_direct, _desc(L, L.F32, R_ | L.CONV_TF32_OUT)),
               (lib.cvvae_conv3d_stacked, _desc(L, L.F16, R_ | L.CONV_TF32_OUT, cout=3))]
    for fn in (lib.cvvae_conv3d_tc, lib.cvvae_conv3d, lib.cvvae_conv3d_direct):   # the rounded store needs the ReLU epilogue
        d = _desc(L, L.F32, L.CONV_TF32_OUT)
        assert fn(ctypes.byref(d), None) == -1 and b"TF32_OUT" in lib.cvvae_last_error(), fn.__name__
    d = _desc(L, L.F16, L.CONV_TF32_OUT, cout=3)
    assert lib.cvvae_conv3d_stacked(ctypes.byref(d), None) == -1 and b"ReLU" in lib.cvvae_last_error()
    for flag in (L.CONV_OUT_F32, L.CONV_W_PER_BATCH, L.CONV_X_SHARED, L.CONV_BIAS_ALONG_M):
        refused += [(lib.cvvae_conv3d_tc, _desc(L, L.F32, R_ | flag)), (lib.cvvae_conv3d, _desc(L, L.F32, R_ | flag))]
    for fn, d in refused:
        assert fn(ctypes.byref(d), None) == -1, fn.__name__                 # CVVAE_E_ARG
        assert b"RELU" in lib.cvvae_last_error() or b"ReLU" in lib.cvvae_last_error(), (fn.__name__, lib.cvvae_last_error())
    assert lib.cvvae_launch_count() == before

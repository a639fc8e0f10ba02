"""LPIPS on AlexNet features without a GPU: the fp64 restatement (tests/lpips_alex_ref.py) against torchvision's AlexNet
sliced as lpips slices it, the tap sizes and the 31 px minimum, the loader's two key layouts and its refusals, the
unchanged VGG16 defaults, the binding against the header and the library's argument checks for the new entry points."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lpips_alex_ref as A
import lpips_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _frames(T, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (T, H, W, 3), generator=g, dtype=torch.uint8)


@pytest.mark.parametrize("H,W", [(31, 31), (33, 47), (64, 96)])
def test_restatement_equals_torchvision_alexnet_sliced_as_lpips(H, W):
    import torchvision
    sd = A.make_state_dict(1)
    features = torchvision.models.alexnet(weights=None).features.double().eval()
    features.load_state_dict({k[len("features."):]: v for k, v in sd.items() if k.startswith("features.")})
    a, b = _frames(2, H, W, 2), _frames(2, H, W, 3)
    x = torch.cat([R.scaled_input(a), R.scaled_input(b)]).double()
    want = torch.zeros(2, dtype=torch.float64)
    with torch.no_grad():
        got_taps = A.taps(x, sd)
        for k, (lo, hi) in enumerate(A.SLICES):
            x = features[lo:hi](x)
            assert torch.equal(x, got_taps[k]), k
            fh = x / (torch.sqrt((x * x).sum(1, keepdim=True) + 1e-10) + 1e-10)
            want += F.conv2d((fh[:2] - fh[2:]) ** 2, sd[f"lin{k}.model.1.weight"].double()).mean((1, 2, 3))
        got = A.lpips(a, b, sd)
    assert isinstance(features[12], torch.nn.MaxPool2d) and len(features) == 13     # the last pool is not part of LPIPS
    assert (got - want).abs().max().item() <= 1e-12 * want.abs().max().item(), (got, want)
    assert (A.lpips(a, a, sd) == 0).all()


@pytest.mark.parametrize("H,W", [(31, 31), (31, 38), (34, 35), (37, 42), (97, 161), (576, 1024), (720, 1280)])
def test_tap_sizes_are_torchvisions(H, W):
    from cvvae_b200.metrics import _lpips_alex_tap_sizes
    sd = A.make_state_dict(2)
    with torch.no_grad():
        shapes = [tuple(f.shape[2:]) for f in A.taps(torch.zeros((1, 3, H, W)), sd)]
    assert _lpips_alex_tap_sizes(H, W) == shapes


def test_31_px_is_the_smallest_frame():
    from cvvae_b200.metrics import LPIPS_ALEX_MIN_SIZE, _check_lpips_size, _lpips_alex_tap_sizes
    assert LPIPS_ALEX_MIN_SIZE == 31
    assert min(min(s) for s in _lpips_alex_tap_sizes(31, 31)) == 1
    assert _lpips_alex_tap_sizes(30, 31)[-1][0] == 0 and _lpips_alex_tap_sizes(31, 30)[-1][1] == 0
    with pytest.raises(RuntimeError):                  # torchvision agrees: nothing is left for the second pool
        A.taps(torch.zeros((1, 3, 30, 64)), A.make_state_dict(2))
    _check_lpips_size(31, 31, "LPIPS", "alex")
    _check_lpips_size(2160, 3840, "LPIPS", "alex")
    for H, W in ((30, 64), (64, 30), (16, 16)):
        with pytest.raises(ValueError, match="LPIPS \\(AlexNet\\) needs frames of at least 31 x 31 px"):
            _check_lpips_size(H, W, "LPIPS", "alex")
    with pytest.raises(ValueError, match="at most 2\\^23 px"):
        _check_lpips_size(2304, 4096, "LPIPS", "alex")
    # VGG16 keeps its limit and message
    _check_lpips_size(16, 16, "LPIPS")
    _check_lpips_size(16, 16, "LPIPS", "vgg")
    with pytest.raises(ValueError, match="LPIPS: LPIPS needs frames of at least 16 x 16 px \\(its last tap, relu5_3"):
        _check_lpips_size(15, 16, "LPIPS", "vgg")


def test_scores_from_the_tap_sums():
    from cvvae_b200.metrics import _lpips_alex_tap_sizes, _lpips_scores
    sizes = _lpips_alex_tap_sizes(64, 96)          # [(15, 23), (7, 11), (3, 5), (3, 5), (3, 5)]
    assert sizes == [(15, 23), (7, 11), (3, 5), (3, 5), (3, 5)]
    acc = torch.tensor([[2 ** 32 * 15 * 23, 0], [0, 2 ** 31 * 7 * 11], [2 ** 32 * 15, 0], [0, 0], [0, -(2 ** 30) * 15]])
    got = _lpips_scores(acc, 64, 96, "alex")
    assert got.dtype == torch.float64 and got.tolist() == [2.0, 0.5 - 0.25]


def test_both_key_layouts_load_the_same_weights():
    from cvvae_b200.metrics import _lpips_weights
    sd = A.make_state_dict(5)
    c1, h1 = _lpips_weights((sd,), "alex")
    c2, h2 = _lpips_weights((A.to_lpips_layout(sd),), "alex")
    assert len(c1) == 5 and len(h1) == 5
    assert [tuple(w.shape) for w, _ in c1] == [(64, 3, 11, 11), (192, 64, 5, 5), (384, 192, 3, 3), (256, 384, 3, 3),
                                               (256, 256, 3, 3)]
    assert [h.numel() for h in h1] == [64, 192, 384, 256, 256]
    for (w1, b1), (w2, b2) in zip(c1, c2):
        assert torch.equal(w1, w2) and torch.equal(b1, b2)
    assert all(torch.equal(x, y) for x, y in zip(h1, h2))
    # merged dicts: torchvision's AlexNet (classifier included) plus the lpips heads, unused keys ignored
    net = {k: v for k, v in sd.items() if k.startswith("features.")}
    net["classifier.1.weight"] = torch.zeros(4096, 9216)
    heads = {k: v for k, v in sd.items() if k.startswith("lin")}
    c3, h3 = _lpips_weights((net, heads), "alex")
    assert all(torch.equal(w1, w3) for (w1, _), (w3, _) in zip(c1, c3)) and all(torch.equal(x, y) for x, y in zip(h1, h3))


@pytest.mark.parametrize("edit,msg", [
    (lambda sd: sd.pop("features.0.weight"), "missing key 'features.0.weight' (or 'net.slice1.0.weight')"),
    (lambda sd: sd.pop("features.10.bias"), "missing key 'features.10.bias' (or 'net.slice5.10.bias')"),
    (lambda sd: sd.pop("lin2.model.1.weight"), "missing key 'lin2.model.1.weight'"),
    (lambda sd: sd.__setitem__("features.0.weight", torch.zeros(64, 3, 3, 3)), "'features.0.weight' has shape"),
    (lambda sd: sd.__setitem__("features.3.weight", torch.zeros(192, 64, 3, 3)), "'features.3.weight' has shape"),
    (lambda sd: sd.__setitem__("lin1.model.1.weight", torch.zeros(1, 128, 1, 1)), "'lin1.model.1.weight' has shape"),
    (lambda sd: sd.__setitem__("features.6.bias", torch.zeros(384, dtype=torch.int64)), "'features.6.bias' is torch.int64"),
    (lambda sd: sd.__setitem__("lin4.model.1.weight", torch.full((1, 256, 1, 1), -33.0)), "|w| > 32"),
    (lambda sd: sd.__setitem__("features.8.weight", torch.full((256, 384, 3, 3), float("inf"))), "non-finite"),
    (lambda sd: sd.__setitem__("scaling_layer.shift", torch.zeros(1, 3, 1, 1)), "'scaling_layer.shift' is"),
    (lambda sd: sd.__setitem__("scaling_layer.scale", torch.ones(1, 3)), "'scaling_layer.scale' has shape"),
])
def test_loader_refusals(edit, msg):
    from cvvae_b200 import LPIPS
    sd = A.make_state_dict(7)
    edit(sd)
    with pytest.raises(ValueError, match=re.escape(msg)):
        LPIPS.from_state_dict(sd, net="alex")


def test_loader_refuses_an_unknown_net_and_a_host_device():
    from cvvae_b200 import LPIPS
    for net in ("squeeze", "VGG", None):
        with pytest.raises(ValueError, match="`net` must be one of \\('vgg', 'alex'\\)"):
            LPIPS.from_state_dict(A.make_state_dict(7), net=net)
    with pytest.raises(ValueError, match="must be a CUDA device"):
        LPIPS.from_state_dict(A.make_state_dict(7), device="cpu", net="alex")
    # each network's state dict is refused by the other's loader: the shapes differ at features.0
    with pytest.raises(ValueError, match="'features.0.weight' has shape \\(64, 3, 3, 3\\), expected \\(64, 3, 11, 11\\)"):
        LPIPS.from_state_dict(R.make_state_dict(7), net="alex")
    with pytest.raises(ValueError, match="'features.0.weight' has shape \\(64, 3, 11, 11\\), expected \\(64, 3, 3, 3\\)"):
        LPIPS.from_state_dict(A.make_state_dict(7))


def test_vgg_stays_the_default():
    from cvvae_b200 import metrics
    from cvvae_b200.metrics import LPIPS, _lpips_scores, _lpips_weights
    assert (metrics.LPIPS_MIN_SIZE, metrics.LPIPS_LAUNCHES, metrics.LPIPS_GROUP_BYTES) == (16, 19, 8 << 30)
    assert (metrics.LPIPS_ALEX_MIN_SIZE, metrics.LPIPS_ALEX_LAUNCHES) == (31, 14)
    sd = R.make_state_dict(5)
    c1, h1 = _lpips_weights((sd,))
    c2, h2 = _lpips_weights((sd,), "vgg")
    assert len(c1) == 13 and all(torch.equal(x, y) for (x, _), (y, _) in zip(c1, c2))
    assert all(torch.equal(x, y) for x, y in zip(h1, h2))
    acc = torch.arange(10, dtype=torch.int64).reshape(5, 2) * 2 ** 30
    assert torch.equal(_lpips_scores(acc, 23, 37), _lpips_scores(acc, 23, 37, "vgg"))
    m = object.__new__(LPIPS)                              # no network named: VGG16
    assert (m.net, m.min_size, m.launches) == ("vgg", 16, 19)
    m._group_bytes = 8 << 30
    assert m._group(576, 1024) == (8 << 30) // (2 * 128 * 4 * 576 * 1024) == 14
    m.net = "alex"
    assert (m.min_size, m.launches) == (31, 14)


def test_group_budget_holds_a_frame_pair_at_the_largest_size():
    from cvvae_b200.metrics import LPIPS, LPIPS_GROUP_BYTES, _lpips_alex_tap_sizes
    m = object.__new__(LPIPS)
    m.net, m._group_bytes = "alex", LPIPS_GROUP_BYTES
    for H, W in ((2048, 4096), (2896, 2896), (31, 2 ** 23 // 31)):
        (h1, w1), (h2, w2) = _lpips_alex_tap_sizes(H, W)[:2]
        pair = 2 * 4 * max(448 * h1 * w1, 1792 * h2 * w2)      # conv1's or conv2's packed input and output, fp32
        assert pair <= LPIPS_GROUP_BYTES and m._group(H, W) == LPIPS_GROUP_BYTES // pair
        # within one image the packing kernels' 32-bit indices suffice (the entry points check it)
        assert 25 * 64 * h2 * w2 < 2 ** 31 and 384 * h1 * w1 < 2 ** 31
    (h1, w1), (h2, w2) = _lpips_alex_tap_sizes(576, 1024)[:2]
    assert m._group(576, 1024) == LPIPS_GROUP_BYTES // (8 * max(448 * h1 * w1, 1792 * h2 * w2))


def test_metric_refuses_bad_frames_before_any_device_work():
    from cvvae_b200.metrics import LPIPS
    m = object.__new__(LPIPS)
    m.device, m.net = torch.device("cuda", 0), "alex"
    ok = torch.zeros((2, 31, 31, 3), dtype=torch.uint8)
    for a, b in ((ok, ok), (ok.float(), ok), (ok[..., :2], ok[..., :2]), (ok[0], ok[0])):
        with pytest.raises(ValueError, match="LPIPS expects CUDA uint8 tensors"):
            m(a, b)


@pytest.mark.parametrize("shape,size", [((3, 30, 40, 3), None), ((3, 40, 30, 3), None), ((3, 64, 64, 3), (24, 64))])
def test_evaluate_frames_refuses_small_frames_on_arrival(shape, size, monkeypatch):
    import cvvae_b200.streaming as S
    from cvvae_b200.metrics import LPIPS
    from test_ms_ssim_cpu import _CudaModel

    class NoTransfers:
        def __init__(self, dev):
            pass

    monkeypatch.setattr(S, "_HostTransfers", NoTransfers)
    m = object.__new__(LPIPS)
    m.device, m.net = torch.device("cuda", 0), "alex"
    it = S.evaluate_frames(_CudaModel(), [np.zeros((0, 8, 8, 3), np.uint8), np.zeros(shape, np.uint8)], size=size, lpips=m)
    with pytest.raises(ValueError, match="evaluate_frames: LPIPS \\(AlexNet\\) needs frames of at least 31 x 31"):
        next(it)


_CTYPES = {"const uint8_t*": ctypes.c_void_p, "const float*": ctypes.c_void_p, "float*": ctypes.c_void_p,
           "int64_t*": ctypes.c_void_p, "void*": ctypes.c_void_p, "int32_t": ctypes.c_int32}
_NEW = ("cvvae_lpips_alex_input", "cvvae_lpips_max_pool3s2", "cvvae_lpips_pack5x5", "cvvae_lpips_tap_copy")


def _header(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "cvvae_b200.h")).read(), flags=re.S)
    ret, args = re.search(rf"(\w+)\s+{name}\s*\(([^)]*)\)\s*;", src).groups()
    return ret, [_CTYPES[re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*")] for a in args.split(",")]


def test_header_prototypes_match_the_binding():
    from cvvae_b200 import _lib as L
    for name in _NEW + ("cvvae_lpips_input", "cvvae_lpips_tap"):
        ret, args = _header(name)
        assert ret == "int" and L._SIGNATURES[name] == (ctypes.c_int, args) and name in L.EXPORTS, name
    assert L.ABI_VERSION == 3


def test_library_refuses_bad_arguments_before_any_launch():
    import __graft_entry__ as ge
    ge.build()
    from cvvae_b200 import _lib as L
    lib = L.load()
    fake = 256
    before = lib.cvvae_launch_count()
    for args, msg in (((None, fake, 1, 31, 31, fake), b"null pointer"), ((fake, fake, 1, 31, 31, None), b"null pointer"),
                      ((fake, fake, -1, 31, 31, fake), b"T=-1"), ((fake, fake, 1, 6, 31, fake), b"H=6"),
                      ((fake, fake, 1, 31, 6, fake), b"W=6"), ((fake, fake, 1, 31, 31, fake + 4), b"16-byte aligned"),
                      ((fake, fake, 1, 2 ** 16, 2 ** 16, fake), b"too large")):
        assert lib.cvvae_lpips_alex_input(*args, None) == -1, args
        assert lib.cvvae_last_error().startswith(b"cvvae_lpips_alex_input") and msg in lib.cvvae_last_error(), args
    assert lib.cvvae_lpips_alex_input(fake, fake, 0, 31, 31, fake, None) == 0
    for fn, name, small in ((lib.cvvae_lpips_max_pool3s2, b"cvvae_lpips_max_pool3s2", 2),
                            (lib.cvvae_lpips_pack5x5, b"cvvae_lpips_pack5x5", 0)):
        for args, msg in (((None, 1, 8, 8, 64, fake), b"null pointer"), ((fake, 1, 8, 8, 64, None), b"null pointer"),
                          ((fake, -1, 8, 8, 64, fake), b"N=-1"), ((fake, 1, small, 8, 64, fake), b"H=%d" % small),
                          ((fake, 1, 8, 8, 66, fake), b"C=66"), ((fake, 1, 8, 8, 0, fake), b"C=0"),
                          ((fake + 4, 1, 8, 8, 64, fake), b"16-byte aligned"), ((fake, 1, 8, 8, 64, fake + 8), b"16-byte aligned"),
                          ((fake, 1, 4096, 4096, 256, fake), b"too large")):
            assert fn(*args, None) == -1, (name, args)
            assert lib.cvvae_last_error().startswith(name) and msg in lib.cvvae_last_error(), (name, args, lib.cvvae_last_error())
        assert fn(fake, 0, 8, 8, 64, fake, None) == 0
    for args, msg in (((None, 1, 8, 8, 256, fake, fake, fake), b"null pointer"),
                      ((fake, 1, 8, 8, 256, fake, fake, None), b"null pointer"),
                      ((fake, 1, 8, 8, 192, fake, fake, fake), b"C must be 256 or 384"),
                      ((fake, 1, 8, 8, 512, fake, fake, fake), b"C must be 256 or 384"),
                      ((fake, -1, 8, 8, 256, fake, fake, fake), b"T=-1"),
                      ((fake, 1, 4096, 4096, 256, fake, fake, fake), b"H*W <= 2^23"),
                      ((fake, 1, 8, 8, 256, fake, fake, fake + 8), b"f, lin_w and copy must be 16-byte aligned"),
                      ((fake, 2 ** 30, 64, 64, 384, fake, fake, fake), b"too many frames")):
        assert lib.cvvae_lpips_tap_copy(*args, None) == -1, args
        assert lib.cvvae_last_error().startswith(b"cvvae_lpips_tap_copy") and msg in lib.cvvae_last_error(), args
    assert lib.cvvae_lpips_tap_copy(fake, 0, 1, 1, 384, fake, fake, fake, None) == 0
    # the tap kernel now takes AlexNet's 192 and 384 channels too, and still refuses others
    for C in (96, 320, 768):
        assert lib.cvvae_lpips_tap(fake, 1, 8, 8, C, fake, fake, None, None) == -1
        assert b"C must be 64, 128, 192, 256, 384 or 512" in lib.cvvae_last_error()
    assert lib.cvvae_lpips_tap(fake, 0, 8, 8, 192, fake, fake, fake, None) == 0
    assert lib.cvvae_lpips_tap(fake, 0, 8, 8, 384, fake, fake, fake, None) == 0
    assert lib.cvvae_launch_count() == before

"""FVD without a GPU: the SAME-padding rule and the output shapes of the plan (against the restatement in
tests/i3d_ref.py on meta tensors), the plan's launch count and group budget, the stem's weight layout, BN folding, the
loader's key layout and refusals, frechet_distance against closed forms and an independent restatement, the public
surface, the binding against the header and the library's argument checks for the new entry points."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import scipy.linalg
import torch
import torch.nn.functional as F

import i3d_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fvd():
    from cvvae_b200 import fvd
    return fvd


@pytest.mark.parametrize("n,k,s,want", [(16, 7, 2, (2, 3, 8)), (17, 7, 2, (3, 3, 9)), (9, 7, 2, (3, 3, 5)),
                                        (224, 7, 2, (2, 3, 112)), (112, 3, 2, (0, 1, 56)), (7, 3, 2, (1, 1, 4)),
                                        (8, 3, 1, (1, 1, 8)), (8, 1, 1, (0, 0, 8)), (4, 2, 2, (0, 0, 2)),
                                        (5, 2, 2, (0, 1, 3)), (3, 3, 2, (1, 1, 2)), (1, 3, 1, (1, 1, 1))])
def test_same_padding_table(n, k, s, want):
    """pad = max(k - s, 0) if n % s == 0 else max(k - n % s, 0), front = pad // 2, output ceil(n / s)."""
    fvd = _fvd()
    assert fvd.same_padding(n, k, s) == want
    x = torch.zeros((1, 1, n, 1, 1))
    assert R.same_pad(x, (k, 1, 1), (s, 1, 1)).shape[2] == n + want[0] + want[1]
    assert F.max_pool3d(R.same_pad(x, (k, 1, 1), (s, 1, 1)), (k, 1, 1), (s, 1, 1)).shape[2] == want[2]


@pytest.mark.parametrize("T,T5", [(9, 2), (16, 2), (17, 3), (24, 3), (33, 5)])
def test_plan_shapes_match_the_restatement(T, T5):
    """Every buffer the plan writes has the shape the restatement computes (on meta tensors): Mixed_5c is
    [1024, 2, 7, 7] at 16 x 224^2 and [1024, 3, 7, 7] at 17 frames."""
    fvd = _fvd()
    plan = fvd.i3d_plan(T)
    assert plan.buffers[plan.steps[-1].src] == (T5, 7, 7, 1024)
    sd = {k: v.to("meta") for k, v in R.make_state_dict(0).items()}
    f = R.trunk(torch.empty((1, 3, T, 224, 224), device="meta", dtype=torch.float64), sd)
    assert tuple(f.shape) == (1, 1024, T5, 7, 7)
    assert tuple(R.head(f, sd).shape) == (1, 400)
    # the stem's conv output and the trunk pools' outputs against the restatement's layers
    stem = plan.buffers[plan.steps[1].dst]
    assert stem == (-(-T // 2), 112, 112, 64)
    assert plan.buffers[plan.steps[1].src] == (stem[0] + 2, 112, 112, fvd.I3D_STEM_CHANNELS)
    trunk_pools = [plan.buffers[s.dst] for s in plan.steps if s.op == "pool" and s.name.startswith("MaxPool3d")]
    assert trunk_pools == [(stem[0], 56, 56, 64), (stem[0], 28, 28, 192), (-(-stem[0] // 2), 14, 14, 480),
                           (T5, 7, 7, 832)]


def test_plan_counts_and_units():
    fvd = _fvd()
    plan = fvd.i3d_plan(16)
    ops = [s.op for s in plan.steps]
    assert ops.count("conv") == 57 and ops.count("pool") == 13 and ops[0] == "stem" and ops[-1] == "head"
    assert fvd.I3D_LAUNCHES == len(plan.steps) == 72 and fvd.I3D.launches == 72
    assert [u[:3] for u in fvd.I3D_UNITS] == [u[:3] for u in R.units()]
    assert [u[3] for u in fvd.I3D_UNITS] == [u[3] for u in R.units()]
    # only Mixed_5c's branches leave fp32 for the head; every other convolution output is read by convolutions
    assert {s.name.split(".")[0] for s in plan.steps if s.op == "conv" and not s.tf32_out} == {"Mixed_5c"}
    # branch outputs tile their block's channels exactly
    for name, o in R.BLOCKS.items():
        slices = sorted((s.c0, s.c0 + s.cout) for s in plan.steps if s.op == "conv" and s.name in
                        (f"{name}.b0", f"{name}.b1b", f"{name}.b2b", f"{name}.b3b"))
        assert slices[0][0] == 0 and all(a[1] == b[0] for a, b in zip(slices, slices[1:]))
        assert slices[-1][1] == o[0] + o[2] + o[4] + o[5]


def test_minimum_frames():
    fvd = _fvd()
    assert fvd.i3d_plan(9).buffers[fvd.i3d_plan(9).steps[-1].src][0] == 2
    assert fvd.i3d_plan(8).buffers[fvd.i3d_plan(8).steps[-1].src][0] == 1   # no position left after the [2, 7, 7] pool
    fvd._check_frames_count(9, "I3D")
    with pytest.raises(ValueError, match="at least 9 frames.*got 8"):
        fvd._check_frames_count(8, "I3D")


def test_group_budget_from_the_plan():
    """The group holds as many clips as the budget allows for the plan's largest live set: at 16 x 224^2 that is the
    prepared clip (held by the caller throughout), the packed stem input and the stem's output, 260 MB per clip."""
    fvd = _fvd()
    plan = fvd.i3d_plan(16)
    stem_in, stem_out = plan.buffers[1], plan.buffers[2]
    assert plan.clip_bytes() == 4 * (math.prod(stem_in) + math.prod(stem_out) + 3 * 16 * 224 * 224)
    assert fvd.I3D_GROUP_BYTES // plan.clip_bytes() >= 32
    assert fvd.i3d_plan(64).clip_bytes() > 3 * plan.clip_bytes()


def test_stem_weight_layout():
    """The 3 x 1 x 1 convolution over the packed channels equals the 7 x 7 x 7 stride-2 SAME convolution."""
    fvd = _fvd()
    g = torch.Generator().manual_seed(3)
    w = torch.randn((8, 3, 7, 7, 7), generator=g, dtype=torch.float64)
    x = torch.randn((1, 3, 11, 15, 13), generator=g, dtype=torch.float64)
    want = F.conv3d(R.same_pad(x, (7, 7, 7), (2, 2, 2)), w, stride=2)
    ft, _, to = fvd.same_padding(11, 7, 2)
    fh, _, ho = fvd.same_padding(15, 7, 2)
    fw, _, wo = fvd.same_padding(13, 7, 2)
    xp = F.pad(x, (fw, 13, fh, 13, ft, 2 * (to + 2) + 1 - 11 - ft))
    packed = torch.zeros((to + 2, ho, wo, 448), dtype=torch.float64)
    for u in range(to + 2):
        for j in range(3):
            patch = xp[0, :, 2 * u + j].unfold(1, 7, 2).unfold(2, 7, 2)[:, :ho, :wo]   # [3, ho, wo, 7, 7]
            packed[u, :, :, j * 147:(j + 1) * 147] = patch.permute(1, 2, 3, 4, 0).reshape(ho, wo, 147)
    got = F.conv3d(packed.permute(3, 0, 1, 2)[None], fvd.stem_weight(w))
    assert got.shape == want.shape and torch.allclose(got, want, rtol=0, atol=1e-12)


def test_bn_folding_is_conv_then_bn():
    fvd = _fvd()
    sd = R.make_state_dict(5)
    name = "Mixed_3b.b1b"
    sd[f"{name}.bn.running_var"] = sd[f"{name}.bn.running_var"] * 10 ** torch.linspace(-3, 1, 128)   # a wide range of scales
    w, b = fvd.i3d_weights(sd)[0][name]
    x = torch.randn((2, 96, 3, 9, 9), generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    want = R.unit(x, sd, name, (3, 3, 3))
    got = F.relu(F.conv3d(R.same_pad(x, (3, 3, 3), (1, 1, 1)), w, b))
    assert (got - want).abs().max().item() <= 1e-12 * max(1.0, want.abs().max().item())


def test_round_tf32_rounds_once():
    fvd = _fvd()
    v = torch.tensor([1.0, 1 + 2 ** -11, 1 + 3 * 2 ** -11, 1 + 2 ** -11 + 2 ** -40, -(1 + 2 ** -11), 0.0, 3e-30, 1e30],
                     dtype=torch.float64)
    got = fvd.round_tf32(v)
    assert got.tolist() == pytest.approx([1.0, 1.0, 1 + 4 * 2 ** -11, 1 + 2 ** -10, -1.0, 0.0, got[6].item(), got[7].item()],
                                         rel=0, abs=0)
    # 10 explicit mantissa bits and at most half a TF32 ulp away
    bits = got.view(torch.int32)
    assert ((bits & 0x1FFF) == 0).all()
    x = torch.randn(10000, dtype=torch.float64)
    r = fvd.round_tf32(x).double()
    assert ((r - x).abs() <= 2.0 ** (torch.floor(torch.log2(x.abs())) - 11)).all()
    assert torch.equal(fvd.round_tf32(x), R.tf32(fvd.round_tf32(x)))


def test_loader_reads_the_port_layout():
    fvd = _fvd()
    sd = R.make_state_dict(7)
    units, (w, b) = fvd.i3d_weights(sd)
    assert len(units) == 57 and w.shape == (400, 1024) and b.shape == (400,) and w.dtype == torch.float64
    for name, cin, cout, k in R.units():
        uw, ub = units[name]
        assert uw.shape == (cout, cin, *k) and ub.shape == (cout,)
    # the number of classes comes from the logits' weight; unrelated keys are ignored
    sd10 = dict(R.make_state_dict(7, classes=10), unrelated=torch.zeros(3))
    assert fvd.i3d_weights(sd10)[1][0].shape == (10, 1024)


def _edit(sd, key, value):
    sd = dict(sd)
    if value is None:
        del sd[key]
    else:
        sd[key] = value(sd[key]) if callable(value) else value
    return sd


@pytest.mark.parametrize("key,value,msg", [
    ("Conv3d_1a_7x7.conv3d.weight", None, "missing key 'Conv3d_1a_7x7.conv3d.weight'"),
    ("Mixed_4e.b2a.bn.running_mean", None, "missing key 'Mixed_4e.b2a.bn.running_mean'"),
    ("logits.conv3d.bias", None, "missing key 'logits.conv3d.bias'"),
    ("Mixed_3b.b1b.conv3d.weight", lambda v: v[:, :, :1], "'Mixed_3b.b1b.conv3d.weight' has shape"),
    ("Mixed_5c.b0.bn.weight", lambda v: v[:-1], "'Mixed_5c.b0.bn.weight' has shape"),
    ("logits.conv3d.weight", lambda v: v[:, :512], "'logits.conv3d.weight' has shape"),
    ("logits.conv3d.bias", lambda v: v[:-1], "'logits.conv3d.bias' has shape"),
    ("Conv3d_2c_3x3.conv3d.weight", lambda v: v.to(torch.int32), "'Conv3d_2c_3x3.conv3d.weight' is torch.int32"),
    ("Mixed_4b.b3b.bn.bias", lambda v: torch.where(torch.arange(len(v)) == 3, float("nan"), v),
     "'Mixed_4b.b3b.bn.bias' has non-finite values"),
    ("logits.conv3d.weight", lambda v: v * float("inf"), "'logits.conv3d.weight' has non-finite values"),
    ("Mixed_3c.b2b.bn.running_var", lambda v: torch.where(torch.arange(len(v)) == 0, -1e-3, v),
     "'Mixed_3c.b2b.bn.running_var' \\+ eps must be > 0"),
    ("Conv3d_2b_1x1.bn.running_var", lambda v: v - v - 5.0, "'Conv3d_2b_1x1.bn.running_var' \\+ eps must be > 0"),
])
def test_loader_refusals(key, value, msg):
    fvd = _fvd()
    with pytest.raises(ValueError, match=msg):
        fvd.i3d_weights(_edit(R.make_state_dict(8), key, value))


def test_loader_ignores_num_batches_tracked_and_refuses_a_host_device():
    fvd = _fvd()
    sd = {k: v for k, v in R.make_state_dict(9).items() if not k.endswith("num_batches_tracked")}
    fvd.i3d_weights(sd)
    with pytest.raises(ValueError, match="CUDA device"):
        fvd.I3D.from_state_dict(sd, device="cpu")


def _fd_restated(a, b):
    """Independent restatement: covariances by hand, the square root by eigendecomposition of the symmetric product
    sqrt(Sa) Sb sqrt(Sa), whose trace of square root equals tr(sqrtm(Sa Sb))."""
    ma, mb = a.mean(0), b.mean(0)
    sa = (a - ma).T @ (a - ma) / (len(a) - 1)
    sb = (b - mb).T @ (b - mb) / (len(b) - 1)
    ea, va = np.linalg.eigh(sa)
    ra = (va * np.sqrt(np.clip(ea, 0, None))) @ va.T
    ev = np.linalg.eigvalsh(ra @ sb @ ra)
    return float(((ma - mb) ** 2).sum() + np.trace(sa) + np.trace(sb) - 2 * np.sqrt(np.clip(ev, 0, None)).sum())


def test_frechet_identical_sets_give_zero():
    from cvvae_b200 import frechet_distance
    a = np.random.default_rng(0).normal(size=(300, 40)) * np.linspace(0.1, 3, 40)
    tr = np.trace(np.cov(a, rowvar=False))
    assert abs(frechet_distance(a, a)) <= 1e-9 * tr


def test_frechet_shift_gives_the_squared_norm():
    from cvvae_b200 import frechet_distance
    rng = np.random.default_rng(1)
    a = rng.normal(size=(200, 16))
    delta = rng.normal(size=16)
    assert frechet_distance(a, a + delta) == pytest.approx(float((delta ** 2).sum()), rel=1e-8, abs=1e-8)


def test_frechet_diagonal_covariances():
    """Axis-aligned sets: the distance is sum (sqrt(var_a) - sqrt(var_b))^2 + |dmu|^2 per axis."""
    from cvvae_b200 import frechet_distance
    rng = np.random.default_rng(2)
    # a 2^k-point design with exactly zero sample covariance between axes
    signs = np.array([[(i >> j) & 1 for j in range(6)] for i in range(64)], dtype=np.float64) * 2 - 1
    sa, sb = rng.uniform(0.2, 3, 6), rng.uniform(0.2, 3, 6)
    ma, mb = rng.normal(size=6), rng.normal(size=6)
    a, b = ma + signs * sa, mb + signs[::-1] * sb
    va, vb = np.var(a, axis=0, ddof=1), np.var(b, axis=0, ddof=1)
    want = float(((np.sqrt(va) - np.sqrt(vb)) ** 2).sum() + ((a.mean(0) - b.mean(0)) ** 2).sum())
    assert frechet_distance(a, b) == pytest.approx(want, rel=1e-9, abs=1e-10)


@pytest.mark.parametrize("n,m,d", [(50, 80, 8), (500, 300, 400), (3, 2, 5)])
def test_frechet_agrees_with_an_independent_restatement(n, m, d):
    from cvvae_b200 import frechet_distance
    rng = np.random.default_rng(n + d)
    mix = rng.normal(size=(d, d)) / np.sqrt(d)
    a = rng.normal(size=(n, d)) @ mix
    b = rng.normal(size=(m, d)) @ (mix + 0.3 * np.eye(d)) + 0.5
    got = frechet_distance(a, b)
    assert got == pytest.approx(_fd_restated(a, b), rel=1e-7, abs=1e-7 * np.trace(np.cov(a, rowvar=False)))
    # the formula as written: sqrtm of the product
    s = scipy.linalg.sqrtm(np.cov(a, rowvar=False) @ np.cov(b, rowvar=False))
    s = s[0] if isinstance(s, tuple) else s
    ref = np.real(((a.mean(0) - b.mean(0)) ** 2).sum() + np.trace(np.cov(a, rowvar=False) + np.cov(b, rowvar=False) - 2 * s))
    assert got == ref
    assert frechet_distance(torch.from_numpy(a), torch.from_numpy(b)) == got


@pytest.mark.parametrize("a,b,msg", [
    (np.zeros((4, 3)), np.zeros((4, 2)), "D = 3.*D = 2"),
    (np.zeros((1, 3)), np.zeros((4, 3)), "N >= 2"),
    (np.zeros((4, 3)), np.zeros((1, 3)), "N >= 2"),
    (np.zeros((4, 3), dtype=np.float32), np.zeros((4, 3)), "float64"),
    (np.zeros(4), np.zeros(4), "float64 \\[N, D\\]"),
    (np.full((4, 3), np.nan), np.zeros((4, 3)), "`a` has non-finite"),
    (np.zeros((4, 3)), np.full((4, 3), np.inf), "`b` has non-finite"),
])
def test_frechet_refusals(a, b, msg):
    from cvvae_b200 import frechet_distance
    with pytest.raises(ValueError, match=msg):
        frechet_distance(a, b)


def test_public_surface():
    import cvvae_b200
    from cvvae_b200 import fvd, streaming
    for name in ("I3D", "embed_clips", "frechet_distance"):
        assert name in cvvae_b200.__all__ and hasattr(cvvae_b200, name)
    assert cvvae_b200.I3D is fvd.I3D and cvvae_b200.embed_clips is streaming.embed_clips


def test_embed_clips_refusals_at_the_call():
    from cvvae_b200 import embed_clips
    with pytest.raises(ValueError, match="fvd.I3D"):
        embed_clips(object(), [])
    fake = object.__new__(_fvd().I3D)
    for bs in (0, -1, 1.5, True):
        with pytest.raises(ValueError, match="batch_size"):
            embed_clips(fake, [], batch_size=bs)


@pytest.mark.parametrize("item,msg", [(np.zeros((8, 32, 32, 3), np.uint8), "T >= 9"),
                                      (np.zeros((9, 32, 32, 3), np.float32), "uint8"),
                                      (np.zeros((9, 32, 32, 4), np.uint8), "uint8 clips"),
                                      (np.zeros((9, 32, 32), np.uint8), "uint8 clips")])
def test_embed_clips_refuses_bad_items(item, msg):
    from cvvae_b200.streaming import _embed_clip
    with pytest.raises(ValueError, match=msg):
        _embed_clip(item, torch.device("cuda", 0))


_NEW = ("cvvae_i3d_stem_input", "cvvae_i3d_max_pool3d", "cvvae_i3d_head")
_CTYPES = {"const float*": ctypes.c_void_p, "float*": ctypes.c_void_p, "int32_t": ctypes.c_int32, "void*": ctypes.c_void_p,
           "const int32_t*": ctypes.POINTER(ctypes.c_int32), "double*": ctypes.c_void_p}


def _header(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "cvvae_b200.h")).read(), flags=re.S)
    ret, args = re.search(rf"(\w+)\s+{name}\s*\(([^)]*)\)\s*;", src).groups()
    return ret, [_CTYPES[re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*")] for a in args.split(",")]


def test_header_prototypes_match_the_binding():
    from cvvae_b200 import _lib as L
    for name in _NEW:
        ret, args = _header(name)
        assert ret == "int" and L._SIGNATURES[name] == (ctypes.c_int, args) and name in L.EXPORTS, name
    assert L.ABI_VERSION == 3


def _lib():
    import __graft_entry__ as ge
    ge.build()
    from cvvae_b200 import _lib as L
    return L.load()


def test_library_refuses_bad_arguments_before_any_launch():
    lib = _lib()
    fake = 256
    before = lib.cvvae_launch_count()

    def refused(fn, name, args, msg):
        assert fn(*args, None) == -1, (name, args)
        err = lib.cvvae_last_error()
        assert err.startswith(name) and msg in err, (name, args, err)

    for args, msg in (((None, 1, 16, 224, 224, fake), b"null pointer"), ((fake, 1, 16, 224, 224, None), b"null pointer"),
                      ((fake, -1, 16, 224, 224, fake), b"N=-1"), ((fake, 1, 0, 224, 224, fake), b"T=0"),
                      ((fake, 1, 16, 0, 224, fake), b"H=0"), ((fake + 2, 1, 16, 224, 224, fake), b"4-byte"),
                      ((fake, 1, 16, 224, 224, fake + 4), b"16-byte aligned"),
                      ((fake, 1, 1024, 4096, 4096, fake), b"too large")):
        refused(lib.cvvae_i3d_stem_input, b"cvvae_i3d_stem_input", args, msg)
    assert lib.cvvae_i3d_stem_input(fake, 0, 16, 224, 224, fake, None) == 0

    k3, s2 = (ctypes.c_int32 * 3)(3, 3, 3), (ctypes.c_int32 * 3)(2, 2, 2)
    bad_k, bad_s = (ctypes.c_int32 * 3)(1, 0, 3), (ctypes.c_int32 * 3)(1, 2, 8)
    for args, msg in (((None, 1, 8, 28, 28, 480, k3, s2, fake), b"null pointer"),
                      ((fake, 1, 8, 28, 28, 480, None, s2, fake), b"null pointer"),
                      ((fake, -1, 8, 28, 28, 480, k3, s2, fake), b"N=-1"), ((fake, 1, 8, 28, 28, 482, k3, s2, fake), b"C=482"),
                      ((fake, 1, 0, 28, 28, 480, k3, s2, fake), b"T=0"),
                      ((fake + 4, 1, 8, 28, 28, 480, k3, s2, fake), b"16-byte aligned"),
                      ((fake, 1, 8, 28, 28, 480, bad_k, s2, fake), b"k=0 s=2 on axis 1"),
                      ((fake, 1, 8, 28, 28, 480, k3, bad_s, fake), b"k=3 s=8 on axis 2"),
                      ((fake, 1, 1024, 512, 512, 64, k3, s2, fake), b"too large")):
        refused(lib.cvvae_i3d_max_pool3d, b"cvvae_i3d_max_pool3d", args, msg)
    assert lib.cvvae_i3d_max_pool3d(fake, 0, 8, 28, 28, 480, k3, s2, fake, None) == 0

    for args, msg in (((None, 1, 2, 7, 7, 1024, fake, fake, 400, fake), b"null pointer"),
                      ((fake, 1, 2, 7, 7, 1024, fake, None, 400, fake), b"null pointer"),
                      ((fake, 1, 1, 7, 7, 1024, fake, fake, 400, fake), b"T=1"),
                      ((fake, 1, 2, 8, 7, 1024, fake, fake, 400, fake), b"H=8"),
                      ((fake, -1, 2, 7, 7, 1024, fake, fake, 400, fake), b"N=-1"),
                      ((fake, 1, 2, 7, 7, 8192, fake, fake, 400, fake), b"C=8192"),
                      ((fake, 1, 2, 7, 7, 1024, fake, fake, 0, fake), b"K=0"),
                      ((fake, 1, 2, 7, 7, 1024, fake, fake, 400, fake + 4), b"8-byte aligned")):
        refused(lib.cvvae_i3d_head, b"cvvae_i3d_head", args, msg)
    assert lib.cvvae_i3d_head(fake, 0, 2, 7, 7, 1024, fake, fake, 400, fake, None) == 0
    assert lib.cvvae_launch_count() == before


def _desc(x_shape, y_shape, kernel, stride, offset):
    """A conv descriptor of the plan's geometry over a fake aligned address (cvvae_conv3d_is_tc reads only the
    descriptor): contiguous channels-last x and y, packed weights, fp32 with the ReLU / TF32-store flags."""
    from cvvae_b200 import _lib as L

    def t5(shape):
        st, acc = [0] * 5, 1
        for i in range(4, -1, -1):
            st[i], acc = acc, acc * shape[i]
        return L.Tensor5(1 << 20, *shape, *st)
    d = L.ConvDesc()
    d.x, d.y, d.w, d.Cout = t5(x_shape), t5(y_shape), 1 << 30, y_shape[-1]
    d.KT, d.KH, d.KW = kernel
    d.st, d.sh, d.sw = stride
    d.off_t, d.off_h, d.off_w = offset
    d.up_time, d.dtype, d.flags, d.alpha = 1, L.F32, L.CONV_RELU | L.CONV_TF32_OUT, 1.0
    return d


def test_every_convolution_is_tensor_core_eligible_and_the_unpacked_stem_is_not():
    """The eligibility check of conv_tc on the plan's descriptors: every one of the 57 runs on the tensor cores.  A stem
    left as a 7 x 7 x 7 stride-2 convolution (or with its spatial taps packed and seven temporal ones) would not: conv_tc
    takes kernel extents up to 3, which is why three frames' taps are packed into the stem's channels."""
    fvd = _fvd()
    lib = _lib()
    plan = fvd.i3d_plan(16)
    for s in plan.steps:
        if s.op != "conv":
            continue
        offset = (0, 0, 0) if s.src == 1 else tuple(-((k - 1) // 2) for k in s.kernel)
        d = _desc((1, *plan.buffers[s.src]), (1, *plan.buffers[s.dst][:3], s.cout), s.kernel, (1, 1, 1), offset)
        assert lib.cvvae_conv3d_is_tc(ctypes.byref(d)) == 1, s.name
    d = _desc((1, 16, 112, 112, 152), (1, 8, 112, 112, 64), (7, 1, 1), (2, 1, 1), (-2, 0, 0))
    assert lib.cvvae_conv3d_is_tc(ctypes.byref(d)) == 0
    d = _desc((1, 16, 224, 224, 8), (1, 8, 112, 112, 64), (7, 7, 7), (2, 2, 2), (-2, -2, -2))
    assert lib.cvvae_conv3d_is_tc(ctypes.byref(d)) == 0

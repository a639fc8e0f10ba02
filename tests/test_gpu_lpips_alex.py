"""LPIPS on AlexNet features on the H100: the conv1 packing, the 3 x 3 stride-2 pool and the conv2 packing bit for bit
against torch, the tap kernel at C = 192 and 384 and its TF32 copy, the whole metric against the fp64 restatement
(tests/lpips_alex_ref.py) gated by the error of PyTorch's own TF32 evaluation, its exact properties, and
evaluate_frames(lpips=...) against the metric of the aligned input."""
import pytest
import torch
import torch.nn.functional as F

import lpips_alex_ref as A
import lpips_ref as R
from test_gpu_lpips import _lpips_contents
from test_gpu_metrics import CASES, _build, _contents, _items, _peak

pytestmark = pytest.mark.gpu
_WORST = {}


def _bits(x):
    return x.contiguous().view(torch.int32)


def _lib():
    from cvvae_b200 import _lib as L
    return L, L.load()


def _ops():
    from cvvae_b200.ops import CudaOps
    return CudaOps()


def _conv1_input(a, b):
    """torch's step 1 on the device (the scaled input, TF32-rounded), unfolded as conv1 reads it: [2T, h1, w1, 384] with
    channel (c * 11 + kh) * 11 + kw, channels 363.. zero."""
    s = R.tf32(torch.cat([R.scaled_input(a), R.scaled_input(b)]))
    H, W = s.shape[2:]
    h1, w1 = (H - 7) // 4 + 1, (W - 7) // 4 + 1
    cols = F.unfold(s, 11, padding=2, stride=4)                       # [2T, 363, h1 * w1], (c, kh, kw) order
    return F.pad(cols.transpose(1, 2).reshape(s.shape[0], h1, w1, 363), (0, 21))


@pytest.mark.parametrize("T,H,W", [(2, 31, 31), (1, 33, 47), (1, 34, 38), (2, 97, 161), (1, 577, 1023)])
def test_conv1_packing_is_torch_bit_for_bit(T, H, W):
    L, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(H * W)
    a = torch.randint(0, 256, (T, H, W, 3), generator=g, device="cuda", dtype=torch.uint8)
    b = torch.randint(0, 256, (T, H, W, 3), generator=g, device="cuda", dtype=torch.uint8)
    a.view(-1, 3)[:256] = torch.arange(256, device="cuda", dtype=torch.uint8)[:, None]   # every byte in every channel
    b.view(-1, 3)[-256:] = torch.arange(255, -1, -1, device="cuda", dtype=torch.uint8)[:, None]
    h1, w1 = (H - 7) // 4 + 1, (W - 7) // 4 + 1
    out = torch.full((2 * T, h1, w1, 384), float("nan"), device="cuda")
    L.check(lib.cvvae_lpips_alex_input(a.data_ptr(), b.data_ptr(), T, H, W, out.data_ptr(), L._stream(a)), "alex input")
    assert torch.equal(_bits(out), _bits(_conv1_input(a, b)))
    # the frame border: row 0 and column 0 read two rows / columns of padding, channels 363.. are zero
    assert (out[:, 0, :, :363].reshape(2 * T, w1, 3, 11, 11)[:, :, :, :2, :] == 0).all()
    assert (out[:, :, 0, :363].reshape(2 * T, h1, 3, 11, 11)[..., :2] == 0).all() and (out[..., 363:] == 0).all()


@pytest.mark.parametrize("N,H,W,C", [(4, 143, 255, 64), (2, 7, 7, 64), (3, 8, 10, 64), (2, 71, 127, 192), (1, 3, 5, 192),
                                     (2, 44, 79, 64)])
def test_pool_and_conv2_packing_are_torch_bit_for_bit(N, H, W, C):
    L, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(N * H * W + C)
    f = torch.relu(torch.randn((N, H, W, C), generator=g, device="cuda"))
    f[0, 0, 0, :4] = torch.tensor([0.0, 1.0 + 2 ** -11, 1.0 + 2 ** -10 + 2 ** -11, 3.0 + 2 ** -22], device="cuda")  # ties
    oh, ow = (H - 3) // 2 + 1, (W - 3) // 2 + 1
    p = torch.full((N, oh, ow, C), float("nan"), device="cuda")
    L.check(lib.cvvae_lpips_max_pool3s2(f.data_ptr(), N, H, W, C, p.data_ptr(), L._stream(f)), "pool")
    want = R.tf32(F.max_pool2d(f.permute(0, 3, 1, 2), 3, 2).permute(0, 2, 3, 1))
    assert torch.equal(_bits(p), _bits(want))
    if C != 64:
        return
    x = torch.full((N, oh, ow, 25 * C), float("nan"), device="cuda")
    L.check(lib.cvvae_lpips_pack5x5(p.data_ptr(), N, oh, ow, C, x.data_ptr(), L._stream(p)), "pack5x5")
    cols = F.unfold(want.permute(0, 3, 1, 2), 5, padding=2)                     # [N, C * 25, oh * ow], (c, kh, kw)
    cols = cols.reshape(N, C, 25, oh, ow).permute(0, 3, 4, 2, 1).reshape(N, oh, ow, 25 * C)   # -> (kh, kw, c)
    assert torch.equal(_bits(x), _bits(cols))


def _tap(f, T, H, W, C, w, side=None, copy=False):
    L, lib = _lib()
    acc = torch.full((T,), -7, dtype=torch.int64, device="cuda")
    if copy:
        L.check(lib.cvvae_lpips_tap_copy(f.data_ptr(), T, H, W, C, w.data_ptr(), acc.data_ptr(), side.data_ptr(),
                                         L._stream(f)), "tap copy")
    else:
        L.check(lib.cvvae_lpips_tap(f.data_ptr(), T, H, W, C, w.data_ptr(), acc.data_ptr(),
                                    None if side is None else side.data_ptr(), L._stream(f)), "tap")
    return acc


@pytest.mark.parametrize("C,H,W,mode", [(192, 71, 127, "pool"), (192, 9, 13, "none"), (384, 35, 63, "copy"),
                                        (384, 5, 7, "none"), (256, 35, 63, "copy"), (256, 1, 1, "copy"),
                                        (384, 44, 79, "copy")])
def test_tap_kernel_against_fp64_and_its_side_output(C, H, W, mode):
    T = 3
    g = torch.Generator(device="cuda").manual_seed(C + H)
    fa = torch.relu(torch.randn((T, H, W, C), generator=g, device="cuda"))
    near = torch.relu(fa + 1e-2 * torch.randn(fa.shape, generator=g, device="cuda"))
    far = torch.relu(torch.randn((T, H, W, C), generator=g, device="cuda"))
    w = torch.rand(C, generator=g, device="cuda")
    worst = 0.0
    for fb in (near, far):
        f = torch.cat([fa, fb]).contiguous()
        side = None
        if mode == "pool":
            side = torch.full((2 * T, H // 2, W // 2, C), float("nan"), device="cuda")
        elif mode == "copy":
            side = torch.full_like(f, float("nan"))
        acc = _tap(f, T, H, W, C, w, side, mode == "copy")
        got = acc.double().cpu() / 2.0 ** 32 / (H * W)
        want = R.tap_distance(f.double().permute(0, 3, 1, 2), w.double(), T).cpu()
        worst = max(worst, ((got - want).abs() / want.abs()).max().item())
        ctas = -(-((H + 1) // 2) * ((W + 1) // 2) // 32)                      # the existing bound: CTA sum rounding
        bound = ctas * 2.0 ** -33 / (H * W) + 1e-12 * want.abs()
        assert ((got - want).abs() <= bound).all(), (got, want)
        if mode == "pool":
            mp = F.max_pool2d(f.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
            assert torch.equal(_bits(side), _bits(R.tf32(mp)))
        elif mode == "copy":
            assert torch.equal(_bits(side), _bits(R.tf32(f)))          # the next convolution's input
            assert not torch.equal(side, f)                            # ... while the tap was read in fp32
    _WORST[f"tap C={C} {H}x{W} {mode}"] = worst


def test_tap_copy_is_the_plain_tap():
    T, H, W, C = 2, 17, 19, 384
    g = torch.Generator(device="cuda").manual_seed(5)
    f = torch.relu(torch.randn((2 * T, H, W, C), generator=g, device="cuda"))
    w = torch.rand(C, generator=g, device="cuda")
    plain = _tap(f, T, H, W, C, w)
    assert torch.equal(_tap(f, T, H, W, C, w, torch.empty_like(f), copy=True), plain)
    swapped = torch.cat([f[T:], f[:T]])
    assert torch.equal(_tap(swapped, T, H, W, C, w, torch.empty_like(f), copy=True), plain)


@pytest.fixture(scope="module")
def sd():
    return A.make_state_dict(2025)


@pytest.fixture(scope="module")
def metric(sd):
    from cvvae_b200 import LPIPS
    return LPIPS.from_state_dict(sd, net="alex")


def test_metric_attributes(metric):
    from cvvae_b200 import LPIPS
    assert (metric.net, metric.min_size, metric.launches) == ("alex", 31, 14)
    assert metric.device == torch.device("cuda", torch.cuda.current_device())
    vgg = LPIPS.from_state_dict(R.make_state_dict(1))
    assert (vgg.net, vgg.min_size, vgg.launches) == ("vgg", 16, 19)
    same = LPIPS.from_state_dict(A.to_lpips_layout(A.make_state_dict(2025)), net="alex")
    a, b = (torch.from_numpy(x).cuda() for x in _contents(2, 40, 56, 1)["reconstruction"])
    assert torch.equal(same(a, b), metric(a, b))


def _torch_tf32(a, b, sd):
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        sd32 = {k: v.cuda() for k, v in sd.items()}
        with torch.no_grad():
            return torch.cat([A.lpips(a[i:i + 4], b[i:i + 4], sd32, torch.float32, tf32_conv1=True)
                              for i in range(0, a.shape[0], 4)])
    finally:
        torch.backends.cudnn.allow_tf32 = prev


def _fp64(a, b, sd):
    sd64 = {k: v.cuda().double() for k, v in sd.items()}
    with torch.no_grad():
        return torch.cat([A.lpips(a[i:i + 2], b[i:i + 2], sd64) for i in range(0, a.shape[0], 2)])


GATE = 3


def _gate(name, ours, ref, torch_tf32):
    err = (ours - ref).abs().max().item()
    t = (torch_tf32 - ref).abs().max().item()
    bound = GATE * t + 1e-6 * ref.abs().max().item()
    _WORST[name] = err / max(t, 1e-300)
    print(f"{name}: max|ours - ref| {err:.3e}, max|torch_tf32 - ref| {t:.3e}, ratio {err / max(t, 1e-300):.3f}")
    assert err <= bound, (name, err, bound)


@pytest.mark.parametrize("T,H,W", [(3, 31, 31), (2, 33, 47), (2, 97, 161), (2, 256, 448), (2, 576, 1024)])
def test_metric_against_fp64_gated_by_torch_tf32(T, H, W, sd, metric):
    for name, (a, b) in _lpips_contents(T, H, W, H * W + 1).items():
        da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        ours = metric(da, db)
        assert ours.dtype == torch.float64 and ours.shape == (T,) and ours.device.type == "cpu"
        _gate(f"{name} {H}x{W}", ours, _fp64(da, db, sd), _torch_tf32(da, db, sd))


def test_exact_properties_grouping_and_determinism(metric):
    a, b = (torch.from_numpy(x).cuda() for x in _contents(7, 48, 80, 3)["reconstruction"])
    first = metric(a, b)
    assert (first > 0).all()
    assert (metric(a, a.clone()) == 0.0).all()
    assert torch.equal(metric(b, a), first) and torch.equal(metric(a, b), first)
    assert torch.equal(torch.cat([metric(a[:3], b[:3]), metric(a[3:], b[3:])]), first)
    saved = metric._group_bytes
    try:
        per_pair = saved // metric._group(48, 80)
        for g in (1, 2, 3):
            metric._group_bytes = g * per_pair
            assert metric._group(48, 80) == g
            assert torch.equal(metric(a, b), first), g
    finally:
        metric._group_bytes = saved


def test_launches_per_group(metric):
    a, b = (torch.from_numpy(x).cuda() for x in _contents(5, 40, 56, 3)["noise"])
    ops = _ops()
    saved = metric._group_bytes
    try:
        metric._group_bytes = 2 * (saved // metric._group(40, 56))      # 2 frames a group: 3 groups
        assert metric._group(40, 56) == 2
        before = ops.launch_count()
        metric(a, b)
        assert ops.launch_count() - before == 3 * metric.launches == 42
    finally:
        metric._group_bytes = saved


def test_frames_elsewhere_or_too_small_are_refused(metric):
    L, lib = _lib()
    a = torch.zeros((1, 31, 31, 3), dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA uint8"):
        metric(a, a)
    before = lib.cvvae_launch_count()
    with pytest.raises(ValueError, match="at least 31 x 31"):
        metric(a[:, :30].cuda(), a[:, :30].cuda())
    assert lib.cvvae_launch_count() == before


SIZE = (96, 128)


def _frames(T):
    frames = torch.from_numpy(_contents(T, 100, 140, T)["reconstruction"][0])
    frames[T // 2:] = frames[T // 2:].flip(1)
    return frames


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_evaluate_frames_lpips_is_the_metric_of_the_aligned_input(dtype, graphs, metric):
    from cvvae_b200 import evaluate_frames
    from cvvae_b200.video_io import resize_frames
    m = _build("sd21", 32, CASES["sd21_w32_tiled"]["wrap"], dtype)
    m.enable_cuda_graphs(graphs)
    try:
        for T in (1, 17):
            frames = _frames(T)
            plain = list(evaluate_frames(m, _items(frames), size=SIZE))
            pieces = list(evaluate_frames(m, _items(frames), size=SIZE, lpips=metric))
            assert len(pieces) == len(plain) and all(len(p) == 4 for p in pieces)
            for k in range(3):
                assert torch.equal(torch.cat([p[k] for p in pieces]), torch.cat([p[k] for p in plain])), (T, k)
            rec = torch.cat([p[0] for p in pieces])
            lp = torch.cat([p[-1] for p in pieces])
            assert lp.dtype == torch.float64 and (lp > 0).all()
            assert torch.equal(lp, metric(resize_frames(frames[:rec.shape[0]].cuda(), SIZE), rec.cuda())), T
    finally:
        m.enable_cuda_graphs(False)


def test_evaluate_frames_lpips_adds_its_launches_per_piece(metric):
    from cvvae_b200 import _lib as L
    from cvvae_b200 import evaluate_frames
    m = _build("sd21", 32, CASES["sd21_w32_tiled"]["wrap"], torch.float16)
    frames = _frames(33)

    def launches(**kw):
        before = L.load().cvvae_launch_count()
        pieces = list(evaluate_frames(m, _items(frames), size=SIZE, **kw))
        return L.load().cvvae_launch_count() - before, len(pieces)

    launches()
    plain, n = launches()
    scored, n_scored = launches(lpips=metric)
    assert n == n_scored == 8
    assert scored - plain == metric.launches * n, (plain, scored)        # each piece is one group at this size


def test_evaluate_frames_lpips_memory_is_flat_in_clip_length(metric):
    from cvvae_b200 import evaluate_frames
    m = _build("sd21", 128, {}, torch.float16)
    S, H, W = m.encode_n_frames_a_time, 256, 256
    clips = {T: torch.randint(0, 256, (T, H, W, 3), generator=torch.Generator().manual_seed(T), dtype=torch.uint8)
             for T in (33, 129)}

    def run(clip):
        pieces = evaluate_frames(m, (clip[a:a + 8] for a in range(0, clip.shape[0], 8)), lpips=metric)
        assert sum(p[0].shape[0] for p in pieces) == clip.shape[0]

    for clip in clips.values():
        run(clip)
    peak = {T: _peak(lambda: run(clip)) for T, clip in clips.items()}
    chunk_io = 2 * (S + 1) * 3 * H * W * 2
    assert peak[129] - peak[33] <= chunk_io, (peak, chunk_io)


def test_evaluate_frames_refuses_small_frames_at_the_first_piece(metric):
    from cvvae_b200 import evaluate_frames
    m = _build("sd21", 32, CASES["sd21_w32_tiled"]["wrap"], torch.float16)
    frames = _frames(9)
    it = evaluate_frames(m, _items(frames), size=(24, 64), lpips=metric)
    with pytest.raises(ValueError, match="evaluate_frames: LPIPS \\(AlexNet\\) needs frames of at least 31 x 31"):
        next(it)


def test_evaluate_frames_refuses_an_lpips_on_another_device(metric):
    from cvvae_b200 import evaluate_frames
    m = _build("sd21", 32, CASES["sd21_w32_tiled"]["wrap"], torch.float16)
    other = object.__new__(type(metric))
    other.device, other.net = torch.device("cuda", m.device.index + 1), "alex"
    with pytest.raises(ValueError, match="LPIPS weights are on"):
        evaluate_frames(m, [], lpips=other)


def test_report_largest_ratio():
    if _WORST:
        print("largest error ratios / relative errors observed:", {k: f"{v:.3g}" for k, v in _WORST.items()})

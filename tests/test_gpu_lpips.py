"""LPIPS on the H100: conv_tc's ReLU epilogue at the thirteen VGG16 layer shapes, the input and tap kernels bit for bit or
against fp64, the whole metric against the fp64 restatement (tests/lpips_ref.py) gated by the error of PyTorch's own
TF32 evaluation, its exact properties, and evaluate_frames(lpips=...) against the metric of the aligned input."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lpips_ref as R
from test_gpu_metrics import CASES, _build, _contents, _items, _peak

pytestmark = pytest.mark.gpu
LAYERS = [(32, 64, True), (64, 64, False), (64, 128, False), (128, 128, False), (128, 256, False), (256, 256, False),
          (256, 512, False), (512, 512, False)]   # (Cin, Cout, conv1_1 as its tap-packed 1 x 1): every distinct shape
_WORST = {}


def _ops():
    from cvvae_b200.ops import CudaOps
    return CudaOps()


def _bits(x):
    return x.contiguous().view(torch.int32)


@pytest.mark.parametrize("H,W", [(23, 37), (9, 130), (64, 96)])
@pytest.mark.parametrize("cin,cout,packed", LAYERS)
def test_relu_epilogue_is_the_unfused_launch_clamped(cin, cout, packed, H, W):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(cin * cout + H)
    x = torch.randn((2, 1, H, W, cin), generator=g, device="cuda")
    k = (1, 1, 1) if packed else (1, 3, 3)
    w = ops.pack_weight(torch.randn((cout, cin, *k), generator=g, device="cuda") * (2.0 / (cin * 9)) ** 0.5)
    b = torch.randn(cout, generator=g, device="cuda") * 0.1
    kw = dict(kernel=k, offset=(0, 0, 0) if packed else (0, -1, -1))
    plain = torch.empty((2, 1, H, W, cout), device="cuda")
    fused, fused_tf32 = torch.empty_like(plain), torch.empty_like(plain)
    ops.conv(x, w, b, out=plain, **kw)
    ops.conv(x, w, b, out=fused, relu=True, **kw)
    ops.conv(x, w, b, out=fused_tf32, relu=True, tf32_out=True, **kw)
    plan = ops.conv_tc_plan(x, w, b, out=plain, **kw)
    assert ops.conv_tc_plan(x, w, b, out=fused, relu=True, **kw) == plan
    assert ops.conv_tc_plan(x, w, b, out=fused, relu=True, tf32_out=True, **kw) == plan
    assert torch.equal(_bits(fused), _bits(plain.clamp_min(0) + 0.0))          # -0 stored as +0
    assert torch.equal(_bits(fused_tf32), _bits(_tf32(plain.clamp_min(0) + 0.0)))
    assert (fused > 0).any() and (fused == 0).any() and not torch.equal(fused, fused_tf32)


def test_relu_epilogue_first_block_at_full_size():
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn((2, 1, 576, 1024, 32), generator=g, device="cuda")
    for cin, cout, packed in LAYERS[:2]:
        k = (1, 1, 1) if packed else (1, 3, 3)
        w = ops.pack_weight(torch.randn((cout, cin, *k), generator=g, device="cuda") * 0.1)
        b = torch.randn(cout, generator=g, device="cuda") * 0.1
        kw = dict(kernel=k, offset=(0, 0, 0) if packed else (0, -1, -1))
        plain = torch.empty((2, 1, 576, 1024, cout), device="cuda")
        fused = torch.empty_like(plain)
        ops.conv(x, w, b, out=plain, **kw)
        ops.conv(x, w, b, out=fused, relu=True, **kw)
        assert torch.equal(_bits(fused), _bits(plain.clamp_min(0) + 0.0))
        ops.conv(x, w, b, out=fused, relu=True, tf32_out=True, **kw)
        assert torch.equal(_bits(fused), _bits(_tf32(plain.clamp_min(0) + 0.0)))
        x = fused


def test_relu_refusals_launch_nothing():
    from cvvae_b200 import _lib as L
    ops = _ops()
    x = torch.randn((1, 1, 8, 8, 64), device="cuda")
    w = ops.pack_weight(torch.randn((64, 64, 1, 3, 3), device="cuda"))
    y = torch.empty((1, 1, 8, 8, 64), device="cuda")
    kw = dict(kernel=(1, 3, 3), offset=(0, -1, -1))
    xh, wh, yh = x.half(), ops.pack_weight(torch.randn((64, 64, 1, 3, 3), device="cuda").half()), y.half()
    torch.cuda.synchronize()
    before = ops.launch_count()
    for extra in (dict(residual=y.clone()), dict(gn_stats=torch.zeros((1, 32, 2), dtype=torch.int64, device="cuda")),
                  dict(force="direct"), dict(bias_along_m=True), dict(force="direct", tf32_out=True)):
        with pytest.raises(L.CvvaeError, match="RELU|ReLU"):
            ops.conv(x, w, None, out=y, relu=True, **kw, **extra)
    for force in (None, "tc", "direct"):                                       # the rounded store needs the ReLU epilogue
        with pytest.raises(L.CvvaeError, match="TF32_OUT"):
            ops.conv(x, w, None, out=y, tf32_out=True, force=force, **kw)
    for force in (None, "tc"):
        with pytest.raises(L.CvvaeError, match="RELU"):
            ops.conv(xh, wh, None, out=yh, relu=True, force=force, **kw)
    assert ops.launch_count() == before


_tf32 = R.tf32


def _packed_input(a, b):
    """torch's step 1 on the device, zero-padded and tap-packed as cvvae_lpips_input lays it out, TF32-rounded."""
    s = torch.cat([R.scaled_input(a), R.scaled_input(b)])            # [2T, 3, H, W]
    H, W = s.shape[2:]
    p = F.pad(s, (1, 1, 1, 1))
    taps = [p[:, :, kh:kh + H, kw:kw + W] for kh in range(3) for kw in range(3)]
    out = torch.stack(taps, 1).permute(0, 3, 4, 1, 2).reshape(s.shape[0], H, W, 27)
    return R.tf32(F.pad(out, (0, 5)))


@pytest.mark.parametrize("T,H,W", [(2, 16, 16), (1, 17, 31), (3, 64, 65), (1, 577, 1023)])
def test_input_kernel_is_torch_bit_for_bit(T, H, W):
    from cvvae_b200 import _lib as L
    g = torch.Generator(device="cuda").manual_seed(H * W)
    a = torch.randint(0, 256, (T, H, W, 3), generator=g, device="cuda", dtype=torch.uint8)
    b = torch.randint(0, 256, (T, H, W, 3), generator=g, device="cuda", dtype=torch.uint8)
    a.view(-1, 3)[:256] = torch.arange(256, device="cuda", dtype=torch.uint8)[:, None]   # every byte in every channel
    b.view(-1, 3)[-256:] = torch.arange(255, -1, -1, device="cuda", dtype=torch.uint8)[:, None]
    out = torch.full((2 * T, H, W, 32), float("nan"), device="cuda")
    L.check(L.load().cvvae_lpips_input(a.data_ptr(), b.data_ptr(), T, H, W, out.data_ptr(), L._stream(a)), "input")
    want = _packed_input(a, b)
    assert torch.equal(_bits(out), _bits(want))
    assert (out[:, 0, :, :9] == 0).all() and (out[:, :, -1, 6:9] == 0).all() and (out[..., 27:] == 0).all()


def _tap(f, T, H, W, C, w, pooled=True):
    from cvvae_b200 import _lib as L
    acc = torch.full((T,), -7, dtype=torch.int64, device="cuda")
    p = torch.full((2 * T, H // 2, W // 2, C), float("nan"), device="cuda") if pooled else None
    L.check(L.load().cvvae_lpips_tap(f.data_ptr(), T, H, W, C, w.data_ptr(), acc.data_ptr(),
                                     None if p is None else p.data_ptr(), L._stream(f)), "tap")
    return acc, p


@pytest.mark.parametrize("C,H,W", [(64, 33, 47), (128, 16, 24), (256, 9, 13), (512, 5, 7), (512, 36, 64), (64, 288, 512)])
def test_tap_kernel_against_fp64_and_max_pool(C, H, W):
    T = 3
    g = torch.Generator(device="cuda").manual_seed(C + H)
    fa = torch.relu(torch.randn((T, H, W, C), generator=g, device="cuda"))
    near = torch.relu(fa + 1e-2 * torch.randn(fa.shape, generator=g, device="cuda"))        # a close reconstruction
    far = torch.relu(torch.randn((T, H, W, C), generator=g, device="cuda"))
    w = torch.rand(C, generator=g, device="cuda")
    worst = 0.0
    for fb in (near, far):
        f = torch.cat([fa, fb]).contiguous()
        acc, pooled = _tap(f, T, H, W, C, w)
        got = acc.double().cpu() / 2.0 ** 32 / (H * W)
        f64 = f.double().permute(0, 3, 1, 2)
        want = R.tap_distance(f64, w.double(), T).cpu()
        rel = ((got - want).abs() / want.abs()).max().item()
        worst = max(worst, rel)
        # Each CTA's fp64 sum (128 positions) is rounded once to 2^-32, an error of at most 2^-33 per CTA; the fp64
        # arithmetic itself stays far below 1e-12 relative.  fp32 normalisation would be ~1e-7 / |f^_a - f^_b| relative.
        ctas = -(-((H + 1) // 2) * ((W + 1) // 2) // 32)
        bound = ctas * 2.0 ** -33 / (H * W) + 1e-12 * want.abs()
        assert ((got - want).abs() <= bound).all(), (rel, got, want)
        mp = F.max_pool2d(f.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
        assert torch.equal(_bits(pooled), _bits(_tf32(mp)))                    # the next convolution's input: TF32
    _WORST[f"tap C={C} {H}x{W}"] = worst
    print(f"largest relative tap error at C={C}, {H}x{W}: {worst:.2e}")


def test_tap_kernel_properties():
    T, H, W, C = 4, 17, 19, 128
    g = torch.Generator(device="cuda").manual_seed(11)
    fa = torch.relu(torch.randn((T, H, W, C), generator=g, device="cuda"))
    fb = torch.relu(torch.randn((T, H, W, C), generator=g, device="cuda"))
    w = torch.rand(C, generator=g, device="cuda")
    acc_ab, _ = _tap(torch.cat([fa, fb]), T, H, W, C, w, pooled=False)
    acc_ba, _ = _tap(torch.cat([fb, fa]), T, H, W, C, w, pooled=False)
    acc_aa, _ = _tap(torch.cat([fa, fa]), T, H, W, C, w, pooled=False)
    assert torch.equal(acc_ab, acc_ba) and (acc_aa == 0).all() and (acc_ab > 0).all()
    acc_1, _ = _tap(torch.cat([fa[2:3], fb[2:3]]), 1, H, W, C, w, pooled=False)     # the other frames change nothing
    assert torch.equal(acc_1, acc_ab[2:3])


@pytest.fixture(scope="module")
def sd():
    return R.make_state_dict(2024)


@pytest.fixture(scope="module")
def metric(sd):
    from cvvae_b200 import LPIPS
    return LPIPS.from_state_dict(sd)


def _torch_tf32(a, b, sd, tf32: bool):
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = tf32
    try:
        sd32 = {k: v.cuda() for k, v in sd.items()}
        with torch.no_grad():
            # with TF32 on, conv1_1 is made a TF32 convolution at every size (lpips_ref.taps)
            return torch.cat([R.lpips(a[i:i + 4], b[i:i + 4], sd32, torch.float32, tf32_conv1_1=tf32)
                              for i in range(0, a.shape[0], 4)])
    finally:
        torch.backends.cudnn.allow_tf32 = prev


def _lpips_contents(T, H, W, seed):
    cases = {k: v for k, v in _contents(T, H, W, seed).items() if k in ("noise", "reconstruction", "saturated_halves")}
    smooth = cases["reconstruction"][0]
    t = torch.from_numpy(smooth).permute(0, 3, 1, 2).float()
    blurred = F.avg_pool2d(F.pad(t, (1, 1, 1, 1), mode="replicate"), 3, 1).round().clamp(0, 255).byte()
    cases["blurred"] = (smooth, blurred.permute(0, 2, 3, 1).contiguous().numpy())
    cases["shifted"] = (smooth, np.roll(smooth, 2, axis=2))
    cases["quantised"] = (smooth, (smooth // 16 * 16 + 8).astype(np.uint8))
    return cases


GATE = 3


def _gate(name, ours, ref, torch_err_ref):
    err = (ours - ref).abs().max().item()
    t = (torch_err_ref - ref).abs().max().item()
    bound = GATE * t + 1e-6 * ref.abs().max().item()
    _WORST[name] = err / max(t, 1e-300)
    print(f"{name}: max|ours - ref| {err:.3e}, max|torch_tf32 - ref| {t:.3e}, ratio {err / max(t, 1e-300):.3f}")
    assert err <= bound, (name, err, bound)


@pytest.mark.parametrize("T,H,W", [(3, 16, 16), (2, 23, 37), (2, 64, 96), (2, 256, 448)])
def test_metric_against_fp64_gated_by_torch_tf32(T, H, W, sd, metric):
    for name, (a, b) in _lpips_contents(T, H, W, H * W).items():
        da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        ours = metric(da, db)
        assert ours.dtype == torch.float64 and ours.shape == (T,) and ours.device.type == "cpu"
        ref = R.lpips(da.cpu(), db.cpu(), sd)
        _gate(f"{name} {H}x{W}", ours, ref, _torch_tf32(da, db, sd, True))


@pytest.mark.parametrize("variant", ["sd21", "sd3"])
def test_metric_on_real_reconstructions(variant, sd, metric):
    from cvvae_b200 import reconstruct_frames
    m = _build(variant, 32, CASES[f"{variant}_w32_tiled"]["wrap"], torch.float16)
    frames = torch.from_numpy(_contents(9, 96, 128, 5)["reconstruction"][0])
    rec = torch.cat(list(reconstruct_frames(m, _items(frames))))
    a, b = frames[:rec.shape[0]].cuda(), rec.cuda()
    _gate(f"{variant} reconstruction", metric(a, b), R.lpips(a.cpu(), b.cpu(), sd), _torch_tf32(a, b, sd, True))


def test_metric_at_full_size_against_torch_fp32(sd, metric):
    a, b = (torch.from_numpy(x).cuda() for x in _contents(17, 576, 1024, 9)["reconstruction"])
    ref = _torch_tf32(a, b, sd, False)
    _gate("reconstruction 17x576x1024 (ref: torch fp32)", metric(a, b), ref, _torch_tf32(a, b, sd, True))


def test_exact_properties_and_grouping(metric):
    a, b = (torch.from_numpy(x).cuda() for x in _contents(7, 48, 80, 3)["reconstruction"])
    first = metric(a, b)
    assert (metric(a, a.clone()) == 0.0).all()
    assert torch.equal(metric(b, a), first) and torch.equal(metric(a, b), first)
    assert torch.equal(torch.cat([metric(a[:3], b[:3]), metric(a[3:], b[3:])]), first)
    saved = metric._group_bytes
    try:
        for g in (1, 2, 3):
            metric._group_bytes = g * 2 * 128 * 4 * 48 * 80
            assert metric._group(48, 80) == g
            assert torch.equal(metric(a, b), first), g
    finally:
        metric._group_bytes = saved


def test_launches_per_group(metric):
    from cvvae_b200.metrics import LPIPS_LAUNCHES
    a, b = (torch.from_numpy(x).cuda() for x in _contents(5, 32, 48, 3)["noise"])
    ops = _ops()
    saved = metric._group_bytes
    try:
        metric._group_bytes = 2 * 2 * 128 * 4 * 32 * 48       # 2 frames a group: 3 groups
        before = ops.launch_count()
        metric(a, b)
        assert ops.launch_count() - before == 3 * LPIPS_LAUNCHES == 57
    finally:
        metric._group_bytes = saved


def test_frames_on_another_device_are_refused(metric):
    a = torch.zeros((1, 16, 16, 3), dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA uint8"):
        metric(a, a)
    with pytest.raises(ValueError, match="at least 16 x 16"):
        metric(a[:, :15].cuda(), a[:, :15].cuda())


SIZE = (96, 128)


def _frames(T):
    frames = torch.from_numpy(_contents(T, 100, 140, T)["reconstruction"][0])
    frames[T // 2:] = frames[T // 2:].flip(1)
    return frames


def _expected(metric, frames, rec):
    from cvvae_b200.video_io import resize_frames
    return metric(resize_frames(frames[:rec.shape[0]].cuda(), SIZE), rec.cuda())


@pytest.mark.parametrize("ms_ssim", [False, True], ids=["alone", "with_ms_ssim"])
@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("variant", ["sd21", "sd3"])
def test_evaluate_frames_lpips_is_the_metric_of_the_aligned_input(variant, dtype, graphs, ms_ssim, metric):
    from cvvae_b200 import evaluate_frames
    size = SIZE if not ms_ssim else (176, 176)
    m = _build(variant, 32, CASES[f"{variant}_w32_tiled"]["wrap"], dtype)
    m.enable_cuda_graphs(graphs)
    for T in (1, 17):
        frames = _frames(T) if not ms_ssim else torch.from_numpy(_contents(T, 184, 200, T)["reconstruction"][0])
        plain = list(evaluate_frames(m, _items(frames), size=size, ms_ssim=ms_ssim))
        pieces = list(evaluate_frames(m, _items(frames), size=size, ms_ssim=ms_ssim, lpips=metric))
        n = 5 if ms_ssim else 4
        assert len(pieces) == len(plain) and all(len(p) == n for p in pieces)
        for k in range(n - 1):
            assert torch.equal(torch.cat([p[k] for p in pieces]), torch.cat([p[k] for p in plain])), (T, k)
        rec = torch.cat([p[0] for p in pieces])
        lp = torch.cat([p[-1] for p in pieces])
        assert lp.dtype == torch.float64
        from cvvae_b200.video_io import resize_frames
        assert torch.equal(lp, metric(resize_frames(frames[:rec.shape[0]].cuda(), size), rec.cuda())), T
    m.enable_cuda_graphs(False)


def test_evaluate_frames_lpips_adds_its_launches_per_piece(metric):
    from cvvae_b200 import _lib as L
    from cvvae_b200 import evaluate_frames
    from cvvae_b200.metrics import LPIPS_LAUNCHES
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
    assert scored - plain == LPIPS_LAUNCHES * n, (plain, scored)        # each piece is one group at this size


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


def test_evaluate_frames_refuses_an_lpips_on_another_device(metric):
    from cvvae_b200 import evaluate_frames
    m = _build("sd21", 32, CASES["sd21_w32_tiled"]["wrap"], torch.float16)
    other = object.__new__(type(metric))
    other.device = torch.device("cuda", m.device.index + 1)
    with pytest.raises(ValueError, match="LPIPS weights are on"):
        evaluate_frames(m, [], lpips=other)


def test_report_largest_ratio():
    if _WORST:
        print("largest error ratios / relative errors observed:", {k: f"{v:.3g}" for k, v in _WORST.items()})

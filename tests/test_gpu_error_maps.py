"""Error maps on the H100: ssim_map per position against the fp64 reference (tests/metrics_ref.py) and tied bit for bit
to frame_metrics' sums; LPIPS.map (VGG16 and AlexNet) against the fp64 restatement (tests/lpips_map_ref.py) gated by the
error of PyTorch's own TF32 evaluation, its tap maps through the C ABI, its exact properties, grouping and launch count;
evaluate_frames(maps=True) against the maps of the aligned input, with unchanged frames and scores and flat memory."""
import numpy as np
import pytest
import torch

import lpips_alex_ref as A
import lpips_map_ref as M
import lpips_ref as R
import metrics_ref as MR
from test_gpu_lpips import _lpips_contents
from test_gpu_metrics import CASES, SSIM_ATOL, _build, _contents, _items, _peak

pytestmark = pytest.mark.gpu
_WORST = {}


def _bits(x):
    return x.contiguous().view(torch.int32)


def _lib():
    from cvvae_b200 import _lib as L
    return L, L.load()


def _ssim_contents(T, H, W, seed):
    """name -> (a, b) uint8 [T, H, W, 3]: noise, a smooth gradient with small noise, flat 255 against 254, a one-pixel
    shift of the gradient and small noise on noise."""
    c = _contents(T, H, W, seed)
    smooth = c["reconstruction"][0]
    rng = np.random.default_rng(seed + 1)
    noise = c["noise"][0]
    small = np.clip(noise.astype(np.int32) + rng.integers(-2, 3, noise.shape), 0, 255).astype(np.uint8)
    return {"noise": c["noise"], "gradient": c["reconstruction"], "flat_255_254": c["flat_255_254"],
            "shifted": (smooth, np.roll(smooth, 1, axis=2)), "small_noise": (noise, small)}


def _fix(m):
    """Per frame, the sum of round_half_even(v * 2^32) over the map: what frame_metrics accumulates."""
    return (m.double() * 2.0 ** 32).round().to(torch.int64).flatten(1).sum(1)


@pytest.mark.parametrize("T,H,W", [(3, 11, 11), (3, 12, 13), (2, 45, 129), (2, 55, 139), (2, 97, 161), (1, 256, 448),
                                   (1, 576, 1024)])
def test_ssim_map_against_fp64_per_position(T, H, W):
    from cvvae_b200 import metrics, ssim_map
    worst = {}
    for name, (a, b) in _ssim_contents(T, H, W, H * W + T).items():
        da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        got = ssim_map(da, db)
        assert got.shape == (T, H - 10, W - 10, 3) and got.dtype == torch.float32 and got.device == da.device
        want = np.stack([MR.ssim_map(x, y) for x, y in zip(a, b)])
        worst[name] = float(np.abs(got.cpu().double().numpy() - want).max())
        assert worst[name] <= SSIM_ATOL, (name, worst)
        assert torch.equal(_fix(got).cpu(), metrics._launch(da, db)[:, 1].cpu()), name     # the exact tie
    _WORST[f"ssim map {H}x{W}"] = max(worst.values())
    print(f"largest |ssim map - fp64| at {T}x{H}x{W}: {max(worst.values()):.3e} ({worst})")


def test_ssim_map_exact_ties():
    from cvvae_b200 import _lib as L
    from cvvae_b200 import metrics, ssim_map
    a, b = (torch.from_numpy(x).cuda() for x in _contents(9, 67, 141, 4)["reconstruction"])
    acc, first = metrics._launch(a, b, maps=True)
    assert torch.equal(acc, metrics._launch(a, b))                       # the map launch's SSE and SSIM sums
    assert torch.equal(_fix(first), acc[:, 1])
    assert (ssim_map(a, a.clone()) == 1.0).all()
    assert torch.equal(_bits(ssim_map(b, a)), _bits(first))
    assert torch.equal(_bits(ssim_map(a, b)), _bits(first))
    assert torch.equal(_bits(torch.cat([ssim_map(a[:4], b[:4]), ssim_map(a[4:], b[4:])])), _bits(first))
    assert a[1:].data_ptr() % 16 != 0                                    # frames off a 16-byte boundary
    assert torch.equal(_bits(ssim_map(a[1:], b[1:])), _bits(first[1:]))
    assert ssim_map(a[:0], b[:0]).shape == (0, 57, 131, 3)
    lib = L.load()
    before = lib.cvvae_launch_count()
    ssim_map(a, b)
    assert lib.cvvae_launch_count() - before == 1
    before = lib.cvvae_launch_count()
    with pytest.raises(ValueError, match="at least 11"):
        ssim_map(a[:, :10], b[:, :10])
    with pytest.raises(ValueError, match="differ"):
        ssim_map(a, b[:2])
    with pytest.raises(ValueError, match="CUDA uint8"):
        ssim_map(a.cpu(), b.cpu())
    assert lib.cvvae_launch_count() == before


@pytest.fixture(scope="module")
def metrics_by_net():
    from cvvae_b200 import LPIPS
    sds = {"vgg": R.make_state_dict(2024), "alex": A.make_state_dict(2025)}
    return {net: (sd, LPIPS.from_state_dict(sd, net=net)) for net, sd in sds.items()}


def _torch_tf32_map(a, b, sd, net):
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        sd32 = {k: v.cuda() for k, v in sd.items()}
        with torch.no_grad():
            return torch.cat([M.lpips_map(a[i:i + 1], b[i:i + 1], sd32, net, torch.float32, tf32_first=True)
                              for i in range(a.shape[0])])
    finally:
        torch.backends.cudnn.allow_tf32 = prev


def _fp64_map(a, b, sd, net):
    sd64 = {k: v.cuda().double() for k, v in sd.items()}
    with torch.no_grad():
        return torch.cat([M.lpips_map(a[i:i + 1], b[i:i + 1], sd64, net) for i in range(a.shape[0])])


@pytest.mark.parametrize("net,T,H,W", [("vgg", 2, 16, 16), ("vgg", 2, 23, 37), ("vgg", 2, 33, 47), ("vgg", 2, 97, 161),
                                       ("vgg", 1, 256, 448), ("vgg", 1, 576, 1024), ("alex", 2, 31, 31),
                                       ("alex", 2, 33, 47), ("alex", 2, 97, 161), ("alex", 1, 256, 448),
                                       ("alex", 1, 576, 1024)])
def test_lpips_map_against_fp64_gated_by_torch_tf32(net, T, H, W, metrics_by_net):
    sd, metric = metrics_by_net[net]
    names = ("reconstruction", "blurred", "shifted") if H * W > 256 * 448 else None
    for name, (a, b) in _lpips_contents(T, H, W, H * W + 2).items():
        if names and name not in names:
            continue
        da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        ours = metric.map(da, db)
        assert ours.shape == (T, H, W) and ours.dtype == torch.float32 and ours.device == da.device
        ours = ours.double().cpu()
        ref, t32 = _fp64_map(da, db, sd, net), _torch_tf32_map(da, db, sd, net)
        for t in range(T):
            err = (ours[t] - ref[t]).abs().max().item()
            terr = (t32[t] - ref[t]).abs().max().item()
            bound = 3 * terr + 1e-6 * ref[t].abs().max().item()
            key = f"{net} {name} {H}x{W}"
            _WORST[key] = max(_WORST.get(key, 0.0), err / max(terr, 1e-300))
            print(f"{key} frame {t}: max|ours - fp64| {err:.3e}, max|torch_tf32 - fp64| {terr:.3e}, "
                  f"ratio {err / max(terr, 1e-300):.3f}")
            assert err <= bound, (key, t, err, bound)


@pytest.mark.parametrize("C,H,W,side", [(64, 33, 47, "pool"), (128, 16, 24, "pool"), (192, 9, 13, None), (256, 35, 63, "copy"),
                                        (384, 17, 19, "copy"), (384, 5, 7, None), (512, 36, 64, None), (64, 1, 1, None)])
def test_tap_maps_through_the_abi(C, H, W, side):
    L, lib = _lib()
    T = 3
    g = torch.Generator(device="cuda").manual_seed(C + H)
    fa = torch.relu(torch.randn((T, H, W, C), generator=g, device="cuda"))
    fb = torch.relu(fa + 1e-2 * torch.randn(fa.shape, generator=g, device="cuda"))
    f = torch.cat([fa, fb]).contiguous()
    w = torch.rand(C, generator=g, device="cuda")
    shape = {"pool": (2 * T, H // 2, W // 2, C), "copy": f.shape, None: None}[side]
    plain_side = None if shape is None else torch.full(shape, float("nan"), device="cuda")
    map_side = None if shape is None else torch.full(shape, float("nan"), device="cuda")
    acc = torch.full((T,), -7, dtype=torch.int64, device="cuda")
    fn = lib.cvvae_lpips_tap_copy if side == "copy" else lib.cvvae_lpips_tap
    L.check(fn(f.data_ptr(), T, H, W, C, w.data_ptr(), acc.data_ptr(), None if shape is None else plain_side.data_ptr(),
               L._stream(f)), "tap")
    acc_map = torch.full((T,), -7, dtype=torch.int64, device="cuda")
    tap = torch.full((T, H, W), float("nan"), dtype=torch.float64, device="cuda")
    ptr = None if shape is None else map_side.data_ptr()
    before = lib.cvvae_launch_count()
    L.check(lib.cvvae_lpips_tap_map(f.data_ptr(), T, H, W, C, w.data_ptr(), acc_map.data_ptr(),
                                    ptr if side == "pool" else None, ptr if side == "copy" else None, tap.data_ptr(),
                                    L._stream(f)), "tap map")
    assert lib.cvvae_launch_count() - before == 1
    assert torch.equal(acc_map, acc)                                       # the scalar's sums are untouched
    if shape is not None:
        assert torch.equal(_bits(map_side), _bits(plain_side))
    want = M.tap_map(f.double().permute(0, 3, 1, 2), w.double(), T)
    assert ((tap - want).abs() <= 1e-12 * want.abs().max()).all()
    d = acc.double().cpu() / 2.0 ** 32 / (H * W)
    ctas = -(-((H + 1) // 2) * ((W + 1) // 2) // 32)                       # the scalar's bound: CTA sum rounding
    bound = ctas * 2.0 ** -33 / (H * W) + 1e-12 * d.abs()
    assert ((tap.mean((1, 2)).cpu() - d).abs() <= bound).all()


def test_lpips_map_invariants_grouping_and_launches(metrics_by_net):
    from cvvae_b200 import _lib as L
    lib = L.load()
    for net, (_, metric) in metrics_by_net.items():
        a, b = (torch.from_numpy(x).cuda() for x in _contents(7, 48, 80, 3)["reconstruction"])
        acc, first = metric._launch(a, b, maps=True)
        assert torch.equal(acc, metric._launch(a, b)), net                  # scalar sums with and without maps
        assert torch.equal(_bits(metric.map(a, b)), _bits(first)), net     # across calls
        assert (first > 0).any() and (first >= 0).all()
        assert (metric.map(a, a.clone()) == 0).all(), net
        assert torch.equal(_bits(metric.map(b, a)), _bits(first)), net
        assert torch.equal(_bits(torch.cat([metric.map(a[:3], b[:3]), metric.map(a[3:], b[3:])])), _bits(first)), net
        saved = metric._group_bytes
        try:
            per_frame = saved // metric._group(48, 80, maps=True)
            for g in (1, 2, 3):
                metric._group_bytes = g * per_frame
                assert metric._group(48, 80, maps=True) == g
                assert torch.equal(_bits(metric.map(a, b)), _bits(first)), (net, g)
            metric._group_bytes = 3 * per_frame                              # 7 frames: 3 groups
            before = lib.cvvae_launch_count()
            metric.map(a, b)
            assert lib.cvvae_launch_count() - before == 3 * (metric.launches + 1), net
        finally:
            metric._group_bytes = saved
        before = lib.cvvae_launch_count()
        with pytest.raises(ValueError, match="at least"):
            metric.map(a[:, :15], b[:, :15])
        with pytest.raises(ValueError, match="CUDA uint8"):
            metric.map(a.cpu(), b.cpu())
        assert metric.map(a[:0], b[:0]).shape == (0, 48, 80)
        assert lib.cvvae_launch_count() == before


SIZE = (96, 128)


def _frames(T):
    frames = torch.from_numpy(_contents(T, 100, 140, T)["reconstruction"][0])
    frames[T // 2:] = frames[T // 2:].flip(1)
    return frames


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("variant", ["sd21", "sd3"])
def test_evaluate_frames_maps_are_the_maps_of_the_aligned_input(variant, dtype, metrics_by_net):
    from cvvae_b200 import evaluate_frames, ssim_map
    from cvvae_b200.video_io import resize_frames
    m = _build(variant, 32, CASES[f"{variant}_w32_tiled"]["wrap"], dtype)
    metric = metrics_by_net["vgg" if dtype == torch.float16 else "alex"][1]
    for T in (1, 17):
        frames = _frames(T)
        for lp in (None, metric):
            plain = list(evaluate_frames(m, _items(frames), size=SIZE, lpips=lp))
            pieces = list(evaluate_frames(m, _items(frames), size=SIZE, lpips=lp, maps=True))
            n = len(plain[0])
            assert len(pieces) == len(plain) and all(len(p) == n + 1 + (lp is not None) for p in pieces)
            for k in range(n):                                             # frames and every score unchanged
                assert torch.equal(torch.cat([p[k] for p in pieces]), torch.cat([p[k] for p in plain])), (T, k)
            rec = torch.cat([p[0] for p in pieces])
            seen = resize_frames(frames[:rec.shape[0]].cuda(), SIZE)
            sm = torch.cat([p[n] for p in pieces])
            assert sm.dtype == torch.float32 and sm.device.type == "cpu" and sm.shape == (rec.shape[0], 86, 118, 3)
            assert torch.equal(_bits(sm), _bits(ssim_map(seen, rec.cuda()).cpu())), T
            if lp is not None:
                lm = torch.cat([p[n + 1] for p in pieces])
                assert lm.dtype == torch.float32 and lm.shape == (rec.shape[0], *SIZE)
                assert torch.equal(_bits(lm), _bits(lp.map(seen, rec.cuda()).cpu())), T


def test_evaluate_frames_maps_keep_the_launch_count(metrics_by_net):
    from cvvae_b200 import _lib as L
    from cvvae_b200 import evaluate_frames
    m = _build("sd21", 32, CASES["sd21_w32_tiled"]["wrap"], torch.float16)
    metric = metrics_by_net["alex"][1]
    frames = _frames(33)

    def launches(**kw):
        before = L.load().cvvae_launch_count()
        pieces = list(evaluate_frames(m, _items(frames), size=SIZE, **kw))
        return L.load().cvvae_launch_count() - before, len(pieces)

    launches()
    plain, n = launches(lpips=metric)
    mapped, n_mapped = launches(lpips=metric, maps=True)
    assert n == n_mapped == 8
    assert mapped - plain == n, (plain, mapped)        # the SSIM map is the same one launch; LPIPS one upsample per group


def test_evaluate_frames_maps_memory_is_flat_in_clip_length(metrics_by_net):
    from cvvae_b200 import evaluate_frames
    m = _build("sd21", 128, {}, torch.float16)
    metric = metrics_by_net["alex"][1]
    S, H, W = m.encode_n_frames_a_time, 256, 256
    clips = {T: torch.randint(0, 256, (T, H, W, 3), generator=torch.Generator().manual_seed(T), dtype=torch.uint8)
             for T in (33, 129)}

    def run(clip):
        pieces = evaluate_frames(m, (clip[a:a + 8] for a in range(0, clip.shape[0], 8)), lpips=metric, maps=True)
        assert sum(p[0].shape[0] for p in pieces) == clip.shape[0]

    for clip in clips.values():
        run(clip)
    peak = {T: _peak(lambda: run(clip)) for T, clip in clips.items()}
    chunk_io = 2 * (S + 1) * 3 * H * W * 2
    chunk_maps = (S + 1) * (4 * 3 * (H - 10) * (W - 10) + 4 * H * W)
    assert peak[129] - peak[33] <= chunk_io + chunk_maps, (peak, chunk_io, chunk_maps)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_frames_on_another_device_than_the_current_one():
    from cvvae_b200 import LPIPS, ssim_map
    a, b = _contents(2, 64, 80, 3)["reconstruction"]
    want = ssim_map(torch.from_numpy(a).cuda(0), torch.from_numpy(b).cuda(0))
    sd = A.make_state_dict(2025)
    lp0, lp1 = LPIPS.from_state_dict(sd, net="alex", device="cuda:0"), LPIPS.from_state_dict(sd, net="alex", device="cuda:1")
    want_lp = lp0.map(torch.from_numpy(a).cuda(0), torch.from_numpy(b).cuda(0))
    with torch.cuda.device(0):
        a1, b1 = torch.from_numpy(a).to("cuda:1"), torch.from_numpy(b).to("cuda:1")
        got = ssim_map(a1, b1)
        got_lp = lp1.map(a1, b1)
    assert got.device == a1.device and torch.equal(_bits(got.cpu()), _bits(want.cpu()))
    assert got_lp.device == a1.device and torch.equal(_bits(got_lp.cpu()), _bits(want_lp.cpu()))
    with pytest.raises(ValueError, match="differ"):
        ssim_map(torch.from_numpy(a).cuda(0), b1)


def test_report_largest_ratio():
    if _WORST:
        print("largest ssim-map errors / LPIPS-map error ratios observed:", {k: f"{v:.3g}" for k, v in _WORST.items()})

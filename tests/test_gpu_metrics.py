"""frame_metrics / evaluate_frames on the H100: the kernel against the fp64 reference (tests/metrics_ref.py) over frame
sizes from one valid position to 721x1279 and contents from noise to flat and saturated frames; exact integers, exact 1.0
for identical frames, bit-identical however the frames are batched; evaluate_frames equal to reconstruct_frames plus
frame_metrics of the aligned input, bit for bit, at flat device memory and one extra launch per piece."""
import json
import os

import numpy as np
import pytest
import torch

import metrics_ref as R
from oracle import cvvae_oracle as O

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
with open(os.path.join(GOLD, "manifest.json")) as f:
    MANIFEST = json.load(f)
CASES = {c["name"]: c for c in MANIFEST["cases"]}
SSIM_ATOL = 1e-5


def _contents(T, H, W, seed):
    """name -> (a, b) uint8 [T, H, W, 3]."""
    rng = np.random.default_rng(seed)
    shape = (T, H, W, 3)
    noise = lambda: rng.integers(0, 256, shape, dtype=np.uint8)   # noqa: E731
    near = lambda x, k: np.clip(x.astype(np.int32) + rng.integers(-k, k + 1, shape), 0, 255).astype(np.uint8)   # noqa: E731
    yy, xx = np.mgrid[0:H, 0:W]
    ramp = (xx * (153.0 / max(W - 1, 1)) + yy * (102.0 / max(H - 1, 1)))[None, :, :, None] + np.array([0.0, 20.0, -20.0])
    smooth = np.clip(ramp + rng.normal(0.0, 4.0, shape), 0, 255).astype(np.uint8)
    halves = np.zeros(shape, dtype=np.uint8)
    halves[:, :, W // 2:] = 255
    halves[:, H // 2:, :, 1] = 255 - halves[:, H // 2:, :, 1]
    checker = np.broadcast_to((((yy + xx) % 2) * 255).astype(np.uint8)[None, :, :, None], shape).copy()
    flat = lambda v: np.full(shape, v, dtype=np.uint8)   # noqa: E731
    return {
        "noise": (noise(), noise()),
        "reconstruction": (smooth, near(smooth, 3)),      # smooth picture + small clipped noise: what a codec returns
        "flat_0_255": (flat(0), flat(255)),
        "flat_255_254": (flat(255), flat(254)),
        "flat_0_1": (flat(0), flat(1)),
        "saturated_halves": (halves, near(halves, 2)),
        "checkerboard_inverse": (checker, 255 - checker),
    }


@pytest.mark.parametrize("T,H,W", [(17, 11, 11), (3, 12, 37), (17, 64, 65), (3, 272, 384), (1, 576, 1024), (3, 721, 1279)])
def test_kernel_against_reference(T, H, W):
    from cvvae_b200 import frame_metrics
    worst = {}
    for name, (a, b) in _contents(T, H, W, H * W + T).items():
        da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        got = frame_metrics(da, db)
        want_psnr, want_ssim, want_sse = R.frame_scores(a, b)
        assert got.psnr.shape == got.ssim.shape == got.sse.shape == (T,)
        assert got.psnr.device.type == got.ssim.device.type == got.sse.device.type == "cpu"
        assert np.array_equal(got.sse.numpy(), want_sse), name
        np.testing.assert_allclose(got.psnr.numpy(), want_psnr, rtol=1e-13, atol=1e-12, err_msg=name)   # 0 dB at flat 0 / 255
        worst[name] = float(np.abs(got.ssim.numpy() - want_ssim).max())
        assert worst[name] <= SSIM_ATOL, (name, worst)
        assert torch.equal(da.cpu(), torch.from_numpy(a)) and torch.equal(db.cpu(), torch.from_numpy(b)), "inputs modified"
        # identical inputs: exactly 1.0 and +inf, whatever the content
        same = frame_metrics(da, da.clone())
        assert (same.ssim == 1.0).all() and (same.psnr == float("inf")).all() and (same.sse == 0).all(), name
    print(f"largest |ssim - fp64 reference| at {T}x{H}x{W}: {max(worst.values()):.3e} ({worst})")


def test_bit_identical_across_calls_and_batching():
    from cvvae_b200 import frame_metrics
    a, b = (torch.from_numpy(x).cuda() for x in _contents(17, 123, 211, 5)["reconstruction"])
    first = frame_metrics(a, b)
    for _ in range(20):
        again = frame_metrics(a, b)
        assert all(torch.equal(x, y) for x, y in zip(first, again))
    singles = [frame_metrics(a[i:i + 1], b[i:i + 1]) for i in range(17)]
    for k in range(3):
        assert torch.equal(torch.cat([s[k] for s in singles]), first[k])
    # frames that do not start on a 16-byte boundary (123 * 211 * 3 is odd): a view into the clip, not a copy
    assert a[1:].data_ptr() % 16 != 0
    tail = frame_metrics(a[1:], b[1:])
    assert all(torch.equal(x[1:], y) for x, y in zip(first, tail))
    empty = frame_metrics(a[:0], b[:0])
    assert all(x.shape == (0,) for x in empty) and empty.sse.dtype == torch.int64


def test_canaries_and_doctored_pixel():
    from cvvae_b200 import _lib as L
    from cvvae_b200 import frame_metrics
    T, H, W = 3, 40, 53
    a, b = (torch.from_numpy(x).cuda() for x in _contents(T, H, W, 9)["noise"])
    canary = -0x0123456789ABCDEF
    buf = torch.full((T + 2, 2), canary, dtype=torch.int64, device="cuda")
    before = L.load().cvvae_launch_count()
    L.check(L.load().cvvae_frame_metrics(a.data_ptr(), b.data_ptr(), T, H, W, buf[1:].data_ptr(),
                                         torch.cuda.current_stream().cuda_stream), "cvvae_frame_metrics")
    assert L.load().cvvae_launch_count() - before == 1          # squared error and SSIM come from one kernel
    host = buf.cpu()
    assert (host[0] == canary).all() and (host[-1] == canary).all()
    base = frame_metrics(a, b)
    assert torch.equal(host[1:-1, 0], base.sse)
    for (t, y, x, c) in ((0, 0, 0, 0), (1, 20, 26, 1), (2, H - 1, W - 1, 2), (1, 4, W - 1, 0)):   # corners, interior, border
        doctored = b.clone()
        old = int(b[t, y, x, c])
        new = old + 1 if old < 255 else old - 1
        doctored[t, y, x, c] = new
        ref = int(a[t, y, x, c])
        got = frame_metrics(a, doctored)
        delta = torch.zeros(T, dtype=torch.int64)
        delta[t] = (ref - new) ** 2 - (ref - old) ** 2
        assert torch.equal(got.sse, base.sse + delta), (t, y, x, c)
    # refusals of the entry point, before any launch
    before = L.load().cvvae_launch_count()
    for args in ((a.data_ptr(), b.data_ptr(), -1, H, W, buf.data_ptr()), (a.data_ptr(), b.data_ptr(), T, 10, W, buf.data_ptr()),
                 (a.data_ptr(), b.data_ptr(), T, H, 10, buf.data_ptr()), (None, b.data_ptr(), T, H, W, buf.data_ptr()),
                 (a.data_ptr(), b.data_ptr(), T, H, W, None), (a.data_ptr(), b.data_ptr(), 1, 30000, 30000, buf.data_ptr())):
        assert L.load().cvvae_frame_metrics(*args, None) == -1
        assert L.load().cvvae_last_error().decode().startswith("cvvae_frame_metrics")
    assert L.load().cvvae_launch_count() == before
    with pytest.raises(ValueError, match="at least 11"):
        frame_metrics(a[:, :10], b[:, :10])
    with pytest.raises(ValueError, match="differ"):
        frame_metrics(a, b[:2])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_frames_on_another_device_than_the_current_one():
    from cvvae_b200 import frame_metrics
    a, b = _contents(2, 64, 80, 3)["reconstruction"]
    want = frame_metrics(torch.from_numpy(a).cuda(0), torch.from_numpy(b).cuda(0))
    with torch.cuda.device(0):
        got = frame_metrics(torch.from_numpy(a).to("cuda:1"), torch.from_numpy(b).to("cuda:1"))
    assert all(torch.equal(x, y) for x, y in zip(want, got))
    with pytest.raises(ValueError, match="differ"):
        frame_metrics(torch.from_numpy(a).cuda(0), torch.from_numpy(b).to("cuda:1"))


def _build(variant, ch, wrap, dtype):
    from cvvae_b200 import CVVAEModel, CVVAESD3Model
    if variant == "sd21":
        m = CVVAEModel(ch=ch, **wrap)
        cfg = O.VAEConfig(variant="sd21", ch=ch, **wrap)
    else:
        m = CVVAESD3Model(block_out_channels=[ch * k for k in (1, 2, 4, 4)], **wrap)
        cfg = O.VAEConfig(variant="sd3", ch=ch, z_channels=16, **wrap)
    m.load_state_dict(O.make_state_dict(cfg, MANIFEST["weight_seed"]), strict=True)
    return m.to(dtype).cuda()


def _items(frames):
    """Ragged host items, numpy and torch alternating, an empty one among them."""
    lens, items, t = [7, 1, 20, 13, 0, 5], [], 0
    while t < frames.shape[0]:
        k = lens[len(items) % len(lens)]
        items.append(frames[t:t + k].numpy() if len(items) % 2 else frames[t:t + k])
        t += k
    return items


def _expected_scores(frames, rec, size):
    from cvvae_b200 import frame_metrics
    from cvvae_b200.video_io import resize_frames
    seen = frames[:rec.shape[0]].cuda()
    if size is not None:
        seen = resize_frames(seen, size)
    return frame_metrics(seen, rec.cuda())


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("variant", ["sd21", "sd3"])
def test_evaluate_frames_is_reconstruct_frames_plus_aligned_scores(variant, dtype, graphs):
    from cvvae_b200 import evaluate_frames, reconstruct_frames
    m = _build(variant, 32, CASES[f"{variant}_w32_tiled"]["wrap"], dtype)
    m.enable_cuda_graphs(graphs)
    for T in (1, 5, 17, 18, 33, 49):
        frames = torch.from_numpy(_contents(T, 80, 104, T)["reconstruction"][0])
        frames[T // 2:] = frames[T // 2:].flip(1)       # a cut in the middle: neighbouring frames score differently
        for size in (None, (72, 88)):
            want_rec = torch.cat(list(reconstruct_frames(m, _items(frames), size=size)))
            pieces = list(evaluate_frames(m, _items(frames), size=size))
            assert all(p.shape[0] == s.shape[0] == q.shape[0] and s.dtype == q.dtype == torch.float64
                       and s.device.type == q.device.type == "cpu" for p, s, q in pieces)
            rec = torch.cat([p for p, _, _ in pieces])
            assert rec.shape[0] == 1 + (T - 1) // 4 * 4           # the trailing frames are neither returned nor scored
            assert torch.equal(rec, want_rec), (T, size)
            want = _expected_scores(frames, rec, size)
            assert torch.equal(torch.cat([s for _, s, _ in pieces]), want.psnr), (T, size)
            assert torch.equal(torch.cat([q for _, _, q in pieces]), want.ssim), (T, size)
            if T > 1:                                             # the alignment check has teeth: a one-frame slip differs
                slipped = _expected_scores(frames[1:], rec[:-1], size)
                assert not torch.equal(slipped.ssim, want.ssim[:-1])
    m.enable_cuda_graphs(False)


def test_evaluate_frames_refuses_sizes_the_networks_do_not_return():
    """80 x 100 is not a multiple of the spatial stride: reconstruct_frames returns another size, and evaluate_frames has
    nothing to score that against."""
    from cvvae_b200 import evaluate_frames, reconstruct_frames
    m = _build("sd21", 32, CASES["sd21_w32_tiled"]["wrap"], torch.float16)
    frames = torch.from_numpy(_contents(9, 80, 100, 2)["noise"][0])
    assert torch.cat(list(reconstruct_frames(m, [frames]))).shape[1:3] != (80, 100)
    with pytest.raises(ValueError, match="for an input of 80 x 100"):
        list(evaluate_frames(m, [frames]))
    pieces = list(evaluate_frames(m, [frames], size=(80, 104)))
    assert sum(p.shape[0] for p, _, _ in pieces) == 9


def test_evaluate_frames_sample_posterior_is_seeded():
    from cvvae_b200 import evaluate_frames
    m = _build("sd21", 32, {}, torch.bfloat16)
    frames = [np.full((9, 32, 48, 3), v, dtype=np.uint8) for v in (10, 200, 90)]
    runs = [list(evaluate_frames(m, frames, sample_posterior=True, generator=torch.Generator(device="cuda").manual_seed(5)))
            for _ in range(2)]
    for k in range(3):
        x, y = (torch.cat([p[k] for p in run]) for run in runs)
        assert x.shape[0] == 25 and torch.equal(x, y)


def test_scoring_adds_one_launch_per_piece_and_nothing_to_the_unscored_path():
    from cvvae_b200 import _lib as L
    from cvvae_b200 import evaluate_frames, reconstruct_frames
    m = _build("sd21", 32, CASES["sd21_w32_tiled"]["wrap"], torch.float16)
    frames = torch.from_numpy(_contents(33, 80, 104, 1)["reconstruction"][0])

    def launches(fn, size):
        before = L.load().cvvae_launch_count()
        pieces = list(fn(m, _items(frames), size=size))
        return L.load().cvvae_launch_count() - before, len(pieces)

    for size in (None, (72, 88)):
        launches(reconstruct_frames, size)                          # packed weights, engine
        plain, n = launches(reconstruct_frames, size)
        scored, n_scored = launches(evaluate_frames, size)
        assert n == n_scored == 8                                   # 4-frame chunks: [0, 5), then 4 frames at a time
        # one metrics kernel (squared error and SSIM together) per piece; with `size`, the resize that also writes the
        # uint8 frames is still the one launch per host item it was
        assert scored - plain == n, (size, plain, scored)


def _peak(fn) -> int:
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_evaluate_frames_memory_is_flat_in_clip_length():
    from cvvae_b200 import evaluate_frames
    m = _build("sd21", 128, {}, torch.float16)
    S, H, W = m.encode_n_frames_a_time, 256, 256
    clips = {T: torch.randint(0, 256, (T, H, W, 3), generator=torch.Generator().manual_seed(T), dtype=torch.uint8)
             for T in (33, 129)}

    def run(clip):
        n = sum(p.shape[0] for p, _, _ in evaluate_frames(m, (clip[a:a + 8] for a in range(0, clip.shape[0], 8))))
        assert n == clip.shape[0]

    for clip in clips.values():
        run(clip)
    peak = {T: _peak(lambda: run(clip)) for T, clip in clips.items()}
    chunk_io = 2 * (S + 1) * 3 * H * W * 2          # one chunk's fp16 input plus output
    assert peak[129] - peak[33] <= chunk_io, (peak, chunk_io)

"""frame_ms_ssim / evaluate_frames(ms_ssim=True) on the H100: every level's cs and SSIM against the fp64 reference
(tests/ms_ssim_ref.py) over sizes from the 161-px minimum to 721x1279 (odd at several levels) and contents from noise to
flat, saturated and anti-correlated frames; exact 1.0 for identical frames; bit-identical however the frames are batched
or aligned; nothing written outside the outputs; evaluate_frames' MS-SSIM equal to frame_ms_ssim of the aligned input,
bit for bit, with its other outputs unchanged, a documented number of extra launches and flat device memory."""
import numpy as np
import pytest
import torch

import ms_ssim_ref as M
from test_gpu_metrics import CASES, _build, _contents, _items, _peak

pytestmark = pytest.mark.gpu
ATOL = 1e-5


def _ms_contents(T, H, W, seed):
    """The SSIM test contents plus a picture against its copy shifted by one pixel."""
    cases = _contents(T, H, W, seed)
    smooth = cases["reconstruction"][0]
    cases["shifted_1px"] = (smooth, np.roll(smooth, 1, axis=2))
    return cases


def _level_means(acc: torch.Tensor, H: int, W: int) -> np.ndarray:
    """Kernel sums int64 [T, 5, 3, 2] -> means float64 [T, 5, 3, 2] (cs, SSIM)."""
    from cvvae_b200.metrics import _ms_ssim_levels
    n = np.array([(h - 10) * (w - 10) for h, w in _ms_ssim_levels(H, W)], dtype=np.float64)
    return acc.numpy().astype(np.float64) / 2.0 ** 32 / n[None, :, None, None]


@pytest.mark.parametrize("T,H,W", [(3, 161, 161), (2, 161, 245), (3, 176, 176), (2, 256, 256), (1, 576, 1024), (1, 721, 1279)])
def test_kernel_against_reference(T, H, W):
    from cvvae_b200 import frame_ms_ssim
    from cvvae_b200.metrics import _launch_ms_ssim
    worst_level, worst_ms = {}, {}
    for name, (a, b) in _ms_contents(T, H, W, H * W + T).items():
        da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        got = frame_ms_ssim(da, db)
        assert got.shape == (T,) and got.dtype == torch.float64 and got.device.type == "cpu"
        means = _level_means(_launch_ms_ssim(da, db).cpu(), H, W)
        cs, s, ms = M.frame_scores(a, b)
        worst_level[name] = max(np.abs(means[..., 0] - cs).max(), np.abs(means[..., 1] - s).max())
        assert worst_level[name] <= ATOL, (name, worst_level)
        # the product jumps at the max(., 0) kink ((1e-9)^0.0448 = 0.40): gate frames whose factors all keep off zero
        factors = np.concatenate([cs[:, :4], s[:, 4:]], axis=1)
        clear = (np.abs(factors) >= 1e-3).all(axis=(1, 2))
        err = np.abs(got.numpy() - ms)[clear]
        worst_ms[name] = float(err.max()) if err.size else None
        assert (err <= ATOL).all(), (name, worst_ms)
        assert torch.equal(da.cpu(), torch.from_numpy(a)) and torch.equal(db.cpu(), torch.from_numpy(b)), "inputs modified"
        same = frame_ms_ssim(da, da.clone())
        assert (same == 1.0).all(), name                        # identical inputs: exactly 1.0, whatever the content
    print(f"largest |cs or ssim - fp64| per level at {T}x{H}x{W}: {max(worst_level.values()):.3e}; "
          f"largest |ms-ssim - fp64|: {max(v for v in worst_ms.values() if v is not None):.3e} ({worst_ms})")


def test_checkerboard_against_its_inverse_is_zero_and_identical_frames_are_one():
    from cvvae_b200 import frame_ms_ssim
    a, b = (torch.from_numpy(x).cuda() for x in _contents(2, 161, 245, 1)["checkerboard_inverse"])
    assert (frame_ms_ssim(a, b) == 0.0).all()
    assert (frame_ms_ssim(b, b.clone()) == 1.0).all()


def test_bit_identical_across_calls_batching_and_alignment():
    from cvvae_b200 import frame_ms_ssim
    from cvvae_b200.metrics import _launch_ms_ssim
    a, b = (torch.from_numpy(x).cuda() for x in _ms_contents(17, 161, 245, 5)["reconstruction"])
    first, sums = frame_ms_ssim(a, b), _launch_ms_ssim(a, b).cpu()
    for _ in range(10):
        assert torch.equal(frame_ms_ssim(a, b), first) and torch.equal(_launch_ms_ssim(a, b).cpu(), sums)
    for cuts in ([0, 1, 17], [0, 5, 6, 16, 17], list(range(18))):
        parts = [_launch_ms_ssim(a[i:j], b[i:j]).cpu() for i, j in zip(cuts, cuts[1:])]
        assert torch.equal(torch.cat(parts), sums), cuts
    # frames that do not start on a 16-byte boundary (161 * 245 * 3 is odd): a view into the clip, not a copy
    assert a[1:].data_ptr() % 16 != 0 and b[3:].data_ptr() % 16 != 0
    assert torch.equal(frame_ms_ssim(a[1:], b[1:]), first[1:])
    assert torch.equal(_launch_ms_ssim(a[3:], b[3:]).cpu(), sums[3:])
    assert frame_ms_ssim(a[:0], b[:0]).shape == (0,)


def test_canaries_and_launch_count():
    from cvvae_b200 import _lib as L
    from cvvae_b200 import frame_ms_ssim
    T, H, W = 3, 163, 199
    a, b = (torch.from_numpy(x).cuda() for x in _contents(T, H, W, 9)["noise"])
    lib = L.load()
    n = lib.cvvae_ms_ssim_workspace_bytes(T, H, W)
    canary = -0x0123456789ABCDEF
    acc = torch.full((T + 2, 5, 3, 2), canary, dtype=torch.int64, device="cuda")
    ws = torch.full((n + 512,), 0xA5, dtype=torch.uint8, device="cuda")
    before = lib.cvvae_launch_count()
    L.check(lib.cvvae_frame_ms_ssim(a.data_ptr(), b.data_ptr(), T, H, W, ws[256:].data_ptr(), acc[1:].data_ptr(),
                                    torch.cuda.current_stream().cuda_stream), "cvvae_frame_ms_ssim")
    from cvvae_b200.metrics import MS_SSIM_LAUNCHES, _ms_ssim_scores
    assert lib.cvvae_launch_count() - before == MS_SSIM_LAUNCHES == 9
    host, hws = acc.cpu(), ws.cpu()
    assert (host[0] == canary).all() and (host[-1] == canary).all()
    assert (hws[:256] == 0xA5).all() and (hws[256 + n:] == 0xA5).all()
    assert torch.equal(_ms_ssim_scores(host[1:-1], H, W), frame_ms_ssim(a, b))
    with pytest.raises(ValueError, match="differ"):
        frame_ms_ssim(a, b[:2])
    for small in (a[:, :160], a[:, :, :160]):
        with pytest.raises(ValueError, match="frame_ms_ssim: MS-SSIM needs frames of at least 161 x 161 px"):
            frame_ms_ssim(small, small)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_frames_on_another_device_than_the_current_one():
    from cvvae_b200 import frame_ms_ssim
    a, b = _ms_contents(2, 170, 190, 3)["reconstruction"]
    want = frame_ms_ssim(torch.from_numpy(a).cuda(0), torch.from_numpy(b).cuda(0))
    with torch.cuda.device(0):
        got = frame_ms_ssim(torch.from_numpy(a).to("cuda:1"), torch.from_numpy(b).to("cuda:1"))
    assert torch.equal(want, got)


SIZE = (176, 176)


def _frames(T):
    frames = torch.from_numpy(_contents(T, 184, 200, T)["reconstruction"][0])
    frames[T // 2:] = frames[T // 2:].flip(1)       # a cut in the middle: neighbouring frames score differently
    return frames


def _expected_ms(frames, rec):
    from cvvae_b200 import frame_ms_ssim
    from cvvae_b200.video_io import resize_frames
    return frame_ms_ssim(resize_frames(frames[:rec.shape[0]].cuda(), SIZE), rec.cuda())


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("variant", ["sd21", "sd3"])
def test_evaluate_frames_ms_ssim_is_frame_ms_ssim_of_the_aligned_input(variant, dtype, graphs):
    from cvvae_b200 import evaluate_frames
    m = _build(variant, 32, CASES[f"{variant}_w32_tiled"]["wrap"], dtype)
    m.enable_cuda_graphs(graphs)
    for T in (1, 5, 17, 33):
        frames = _frames(T)
        plain = list(evaluate_frames(m, _items(frames), size=SIZE))
        pieces = list(evaluate_frames(m, _items(frames), size=SIZE, ms_ssim=True))
        assert len(pieces) == len(plain) and all(len(p) == 4 for p in pieces)
        for k in range(3):                                   # frames, PSNR and SSIM: the default call's, bit for bit
            assert torch.equal(torch.cat([p[k] for p in pieces]), torch.cat([p[k] for p in plain])), (T, k)
        assert all(p[3].shape == (p[0].shape[0],) and p[3].dtype == torch.float64 and p[3].device.type == "cpu"
                   for p in pieces)
        rec = torch.cat([p[0] for p in pieces])
        ms = torch.cat([p[3] for p in pieces])
        assert torch.equal(ms, _expected_ms(frames, rec)), T
        if T > 1:                                            # the alignment check has teeth: a one-frame slip differs
            slipped = _expected_ms(frames[1:], rec[:-1])
            assert not torch.equal(slipped, ms[:-1])
    m.enable_cuda_graphs(False)


def test_ms_ssim_adds_a_fixed_number_of_launches_per_piece():
    from cvvae_b200 import _lib as L
    from cvvae_b200 import evaluate_frames
    from cvvae_b200.metrics import MS_SSIM_LAUNCHES
    m = _build("sd21", 32, CASES["sd21_w32_tiled"]["wrap"], torch.float16)
    frames = _frames(33)

    def launches(**kw):
        before = L.load().cvvae_launch_count()
        pieces = list(evaluate_frames(m, _items(frames), size=SIZE, **kw))
        return L.load().cvvae_launch_count() - before, len(pieces)

    launches()                                                      # packed weights, engine
    plain, n = launches()
    scored, n_scored = launches(ms_ssim=True)
    assert n == n_scored == 8                                       # 4-frame chunks: [0, 5), then 4 frames at a time
    assert scored - plain == MS_SSIM_LAUNCHES * n, (plain, scored)


def test_evaluate_frames_ms_ssim_memory_is_flat_in_clip_length():
    from cvvae_b200 import evaluate_frames
    m = _build("sd21", 128, {}, torch.float16)
    S, H, W = m.encode_n_frames_a_time, 256, 256
    clips = {T: torch.randint(0, 256, (T, H, W, 3), generator=torch.Generator().manual_seed(T), dtype=torch.uint8)
             for T in (33, 129)}

    def run(clip):
        pieces = evaluate_frames(m, (clip[a:a + 8] for a in range(0, clip.shape[0], 8)), ms_ssim=True)
        assert sum(p.shape[0] for p, _, _, _ in pieces) == clip.shape[0]

    for clip in clips.values():
        run(clip)
    peak = {T: _peak(lambda: run(clip)) for T, clip in clips.items()}
    chunk_io = 2 * (S + 1) * 3 * H * W * 2          # one chunk's fp16 input plus output
    assert peak[129] - peak[33] <= chunk_io, (peak, chunk_io)

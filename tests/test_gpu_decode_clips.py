"""The batched pixel conversion (cvvae_video_output_u8, video_io.batch_to_frames) against PyTorch's own evaluation of the
reference expression on the device, and decode_clips against per-clip tiled_decode calls: bit-identical in every dtype,
eager and with CUDA graphs, in order, owned by the caller, in device memory that does not grow with the number of clips,
and on a device other than the current one.

NaN inputs are left out of the kernel tests: `.to(torch.uint8)` of NaN is undefined behaviour in PyTorch (a float to
integer conversion out of range), so there is no reference byte to compare with."""
import math

import numpy as np
import pytest
import torch

from test_gpu_clips import DTYPES, WRAPS, _build, _peak

pytestmark = pytest.mark.gpu
INF = float("inf")


def _torch_frames(x: torch.Tensor) -> torch.Tensor:
    """The reference's line, evaluated by PyTorch in x's dtype on x's device: [B, 3, T, H, W] -> [B, T, H, W, 3]."""
    return ((x.clamp(-1, 1) + 1.0) * 127.5).to(torch.uint8).permute(0, 2, 3, 4, 1)


def _all_16bit(dtype) -> torch.Tensor:
    """Every bit pattern of a 16-bit type but the NaNs: all finite values, both zeros and both infinities."""
    v = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dtype)
    return v[~torch.isnan(v)]


def _fp32_cases() -> torch.Tensor:
    f = torch.float32
    special = torch.tensor([0.0, -0.0, INF, -INF], dtype=f)
    den = torch.tensor([1, 2, 3, 0x1234, 0x400000, 0x7FFFFE, 0x7FFFFF], dtype=torch.int32).view(f)   # denormals
    # each k/127.5 - 1 is where ((x + 1) * 127.5) crosses the integer k, i.e. where the truncation steps; and +-1, the
    # clamp's bounds.  Every fp32 value within 4 ulps of them:
    edges = torch.tensor([k / 127.5 - 1 for k in range(256)] + [1.0, -1.0], dtype=torch.float64).to(f)
    near, up, down = [edges], edges, edges
    for _ in range(4):
        up, down = torch.nextafter(up, torch.tensor(INF)), torch.nextafter(down, torch.tensor(-INF))
        near += [up, down]
    rnd = torch.rand(2 ** 24, generator=torch.Generator().manual_seed(7), dtype=f) * 3 - 1.5
    return torch.cat([special, den, -den, *near, rnd])


def _as_batch(values: torch.Tensor, B: int, H: int = 37) -> torch.Tensor:
    """`values`, shuffled and repeated to fill a CUDA [B, 3, 1, H, W] tensor, W odd and not a multiple of 8."""
    W = math.ceil(values.numel() / (3 * B * H)) | 1
    n = B * 3 * H * W
    perm = torch.randperm(values.numel(), generator=torch.Generator().manual_seed(B))
    reps = math.ceil(n / values.numel())
    return values[perm].repeat(reps)[:n].reshape(B, 3, 1, H, W).cuda()


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("fmt", sorted(DTYPES))
def test_kernel_matches_torch(fmt, B):
    from cvvae_b200.video_io import batch_to_frames
    dtype = DTYPES[fmt]
    values = _fp32_cases() if fmt == "fp32" else _all_16bit(dtype)
    x = _as_batch(values, B)
    assert x.numel() >= values.numel() and x.shape[-1] % 8 and x.shape[-2] % 8
    got = batch_to_frames(x)
    want = _torch_frames(x)
    assert got.shape == want.shape and got.dtype == torch.uint8 and got.is_contiguous()
    bad = got != want
    assert not bad.any(), (int(bad.sum()), x.permute(0, 2, 3, 4, 1)[bad][:8].tolist())
    assert got.min() == 0 and got.max() == 255


@pytest.mark.parametrize("fmt", ["bf16", "fp16"])
def test_batch_slots_equal_output_to_frames(fmt):
    from cvvae_b200.video_io import batch_to_frames, output_to_frames
    dtype = DTYPES[fmt]
    g = torch.Generator(device="cuda").manual_seed(3)
    x = (torch.randn((3, 3, 5, 37, 43), generator=g, device="cuda") * 0.8).to(dtype)
    got = batch_to_frames(x)
    for b in range(3):
        assert torch.equal(got[b], output_to_frames(x[b:b + 1])), b
    # a strided view is converted as its values, and `out` is written in place
    assert torch.equal(batch_to_frames(x.transpose(3, 4)), batch_to_frames(x.transpose(3, 4).contiguous()))
    out = torch.full((3, 5, 37, 43, 3), 7, dtype=torch.uint8, device="cuda")
    assert batch_to_frames(x, out=out).data_ptr() == out.data_ptr() and torch.equal(out, got)
    for bad in (out[:2],                                                                        # shape
                torch.empty(out.shape, dtype=torch.float32, device="cuda"),                     # dtype
                torch.empty((3, 5, 43, 37, 3), dtype=torch.uint8, device="cuda").transpose(2, 3),   # not contiguous
                torch.empty(out.shape, dtype=torch.uint8)):                                     # device
        with pytest.raises(ValueError, match="out must be"):
            batch_to_frames(x, out=bad)


def _per_clip(m, latents):
    """Each clip through the route decode_clips reproduces: tiled_decode of the clip alone, then the pixel conversion."""
    from cvvae_b200.video_io import output_to_frames
    out = []
    for z in latents:
        x = m.tiled_decode(torch.as_tensor(z)[None].to(m.device))
        f = _torch_frames(x)[0] if m.dtype == torch.float32 else output_to_frames(x)
        out.append(f.cpu())
    return out


def _mixed_latents(z_channels, dtype, seed):
    """11 clips of t' in {1, 2, 3, 5}, runs of equal shape broken and resumed, one clip of another size; numpy arrays
    (CPU tensors for bfloat16, which numpy lacks), CPU tensors and device tensors in turn."""
    g = torch.Generator().manual_seed(seed)
    shapes = [(2, 13, 15), (2, 13, 15), (5, 13, 15), (1, 13, 15), (1, 13, 15), (1, 13, 15), (3, 13, 15), (2, 9, 11),
              (2, 13, 15), (5, 13, 15), (5, 13, 15)]
    out = []
    for i, s in enumerate(shapes):
        z = torch.randn((z_channels, *s), generator=g).to(dtype)
        kind = i % 3
        out.append(z.numpy() if kind == 0 and dtype != torch.bfloat16 else z.cuda() if kind == 2 else z)
    return out


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
@pytest.mark.parametrize("fmt", sorted(DTYPES))
@pytest.mark.parametrize("variant", ["sd21", "sd3"])
def test_decode_clips_bit_identical(variant, fmt, graphs):
    """Tiled fixtures (72-pixel tiles, 4 frames a chunk) at 13 x 15 latents: every batch is tiled and chunked."""
    from cvvae_b200 import decode_clips
    m = _build(variant, 32, WRAPS[f"{variant}_w32_tiled"], DTYPES[fmt])
    latents = _mixed_latents(m.net.z_channels, m.dtype, 17)
    want = _per_clip(m, latents)
    m.enable_cuda_graphs(graphs)
    for bs in (1, 3, 8):
        for rep in range(2 if graphs else 1):      # with graphs: the first pass captures, the second replays
            got = list(decode_clips(m, latents, batch_size=bs))
            assert len(got) == len(want)
            for i, (g, w, z) in enumerate(zip(got, want, latents)):
                T = m._engine().decoded_frames(z.shape[1])
                assert g.device.type == "cpu" and g.dtype == torch.uint8, (i, g.device, g.dtype)
                assert g.shape == w.shape == (T, 8 * z.shape[2], 8 * z.shape[3], 3), (i, g.shape, w.shape)
                assert torch.equal(g, w), (variant, fmt, graphs, bs, rep, i)
    if graphs:
        assert m._graph_cache
    m.enable_cuda_graphs(False)


def test_decode_clips_full_width():
    """sd21 at full width, default tiling and chunking: 8 clips of [4, 5, 32, 32] (17 x 256 x 256 each) in one batch."""
    from cvvae_b200 import decode_clips
    m = _build("sd21", 128, {}, torch.float16)
    g = torch.Generator().manual_seed(5)
    latents = [torch.randn((4, 5, 32, 32), generator=g).half() for _ in range(8)]
    want = _per_clip(m, latents)
    got = list(decode_clips(m, latents, batch_size=8))
    assert len(got) == 8 and got[0].shape == (17, 256, 256, 3)
    assert all(torch.equal(a, b) for a, b in zip(got, want))


def test_encode_then_decode_clips_round_trip():
    """encode_clips -> the posterior's mode -> decode_clips equals the per-clip chain encode -> mode -> decode."""
    from cvvae_b200 import DiagonalGaussianDistribution, decode_clips, encode_clips
    from cvvae_b200.video_io import frames_to_training_input, output_to_frames
    m = _build("sd21", 32, {}, torch.float16)
    g = np.random.default_rng(4)
    clips = [g.integers(0, 256, (t, 72, 96, 3), dtype=np.uint8) for t in (9, 9, 1, 9, 5)]
    size = (64, 80)
    modes = [DiagonalGaussianDistribution(mo[None]).mode()[0] for mo in encode_clips(m, clips, size, batch_size=4)]
    got = list(decode_clips(m, modes, batch_size=4))
    for i, c in enumerate(clips):
        z = m.encode(frames_to_training_input(torch.from_numpy(c).cuda(), size, "cover", m.dtype)).latent_dist.mode()
        want = output_to_frames(m.decode(z).sample).cpu()
        assert got[i].shape == want.shape == (c.shape[0], *size, 3) and torch.equal(got[i], want), i


def test_decode_clips_yields_are_owned_and_ordered():
    """Every clip has its own constant latent, so a clip out of order or a slot overwritten later shows."""
    from cvvae_b200 import decode_clips
    m = _build("sd21", 32, {}, torch.float16)
    latents = [np.full((4, 2, 6, 8), -1.5 + 0.4 * i, dtype=np.float16) for i in range(7)]
    want = _per_clip(m, latents)
    assert len({w.double().sum().item() for w in want}) == len(want)
    kept, snapshots = [], []
    for y in decode_clips(m, latents, batch_size=2):
        kept.append(y)
        snapshots.append(y.clone())
    assert all(torch.equal(a, b) for a, b in zip(kept, snapshots))   # later yields left the earlier ones alone
    assert all(torch.equal(a, b) for a, b in zip(kept, want))        # and each is its own clip's


def test_decode_clips_refuses_bad_items_on_arrival():
    from cvvae_b200 import decode_clips
    m = _build("sd21", 32, {}, torch.float16)
    good = np.zeros((4, 2, 6, 8), np.float16)
    for bad, match in ((np.zeros((4, 2, 6, 8), np.float32), "float32"),
                       (torch.zeros((4, 2, 6, 8), dtype=torch.bfloat16, device="cuda"), "bfloat16"),
                       (np.zeros((16, 2, 6, 8), np.float16), "latents \\[4"),
                       (np.zeros((1, 4, 2, 6, 8), np.float16), "latents \\[4"),
                       (np.zeros((4, 0, 6, 8), np.float16), "t', h, w >= 1"),
                       (torch.zeros((4, 2, 6, 8), dtype=torch.float16, device="meta"), "meta")):
        with pytest.raises(ValueError, match=match):
            list(decode_clips(m, [good, bad], batch_size=1))


def test_decode_clips_memory_does_not_grow_with_clip_count():
    from cvvae_b200 import decode_clips
    m = _build("sd21", 128, {}, torch.float16)
    z = torch.randn((4, 5, 16, 16), generator=torch.Generator().manual_seed(2)).half()
    clip_bytes = 17 * 128 * 128 * 3
    bs = 4

    def run(n):
        for y in decode_clips(m, (z for _ in range(n)), batch_size=bs):
            assert y.shape == (17, 128, 128, 3)

    run(8)                                  # warm-up: engine, packed weights, allocator
    p8, p32 = _peak(lambda: run(8)), _peak(lambda: run(32))
    assert p32 - p8 <= bs * clip_bytes, (p8, p32, bs * clip_bytes)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_decode_clips_on_another_device_than_the_current_one():
    from cvvae_b200 import decode_clips
    from cvvae_b200.video_io import batch_to_frames
    g = torch.Generator().manual_seed(9)
    latents = [torch.randn((4, t, 8, 10), generator=g).half() for t in (2, 2, 1)]

    def calls(dev):
        m = _build("sd21", 32, {}, torch.float16).to(dev)
        x = torch.randn((2, 3, 3, 24, 40), generator=g.manual_seed(1)).half().to(dev)
        return [batch_to_frames(x).cpu(), *decode_clips(m, [latents[0], latents[1].to(dev), latents[2]], batch_size=2)]

    want = calls("cuda:0")
    with torch.cuda.device(0):
        got = calls("cuda:1")
    assert len(got) == len(want) == 4
    assert all(torch.equal(a, b) for a, b in zip(got, want))

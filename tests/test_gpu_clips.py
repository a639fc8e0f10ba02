"""The training pre-processing kernel (cvvae_video_train_input) against the fp64 restatement and torchvision, its in-place
batch-slot writes, and encode_clips against per-clip model.encode calls: bit-identical, in order, owned by the caller,
and in device memory that does not grow with the number of clips."""
import json
import os

import numpy as np
import pytest
import torch

import clip_ref as R
from oracle import cvvae_oracle as O
from test_clips_cpu import CASES, IDS, frames, shifted_crop, torchvision_train_input

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
with open(os.path.join(GOLD, "manifest.json")) as f:
    MANIFEST = json.load(f)
WRAPS = {c["name"]: c["wrap"] for c in MANIFEST["cases"]}
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": torch.float32}


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


def _next_beyond(value: float, dtype) -> float:
    """The smallest `dtype` value above `value`: one ulp beyond a bound that ends at `value`."""
    t = torch.tensor(value, dtype=torch.float64).to(dtype)
    if float(t) <= value:
        t = torch.nextafter(t, torch.tensor(float("inf"), dtype=dtype))
    return float(t)


@pytest.mark.parametrize("fmt", sorted(DTYPES))
@pytest.mark.parametrize("T,H,W,size,resize", CASES, ids=IDS)
def test_kernel_matches_reference(T, H, W, size, resize, fmt):
    from cvvae_b200.video_io import frames_to_training_input, training_geometry
    dtype = DTYPES[fmt]
    x = frames(T, H, W, H * W + 1)
    got_t = frames_to_training_input(torch.from_numpy(x).cuda(), size, resize, dtype)
    assert got_t.shape == (1, 3, T, *size) and got_t.dtype == dtype
    got = got_t[0].double().cpu().numpy()
    RH, RW, top, left = training_geometry(H, W, size, resize)
    ref, E = R.train_input_ref(x, RH, RW, top, left, *size)
    ok = R.gate(got, ref, E, fmt)
    assert ok.all(), (np.abs(got - ref)[~ok].max(), int((~ok).sum()))

    # the gate catches one element one ulp beyond it, and a crop one pixel off
    k = np.unravel_index(np.argmax(np.abs(got - ref)), got.shape)
    bound = (0.0 if fmt == "fp32" else 0.5 * R.ulp(ref[k], *R.FORMATS[fmt])) + E[k[-2:]]
    bad = got.copy()
    bad[k] = _next_beyond(ref[k] + bound, dtype)
    assert not R.gate(bad, ref, E, fmt).all()
    shifted, _ = R.train_input_ref(x, RH, RW, *shifted_crop(RH, RW, top, left, size), *size)
    assert not R.gate(got, shifted, E, fmt).all()

    if fmt != "fp32":
        # torchvision's float result rounded to the 16-bit type.  Both fp32 evaluations lie within their bound of the
        # exact value (E here, E_tv with unfused products), so wherever the exact value is farther than E + E_tv from a
        # rounding midpoint of the type they must round alike, and everywhere they differ by at most ulp + E + E_tv.
        # (Plain equality on a fixed share of elements is not implied: (v / 255 - 0.5) * 2 cancels near 0, where the
        # 16-bit types resolve far finer steps than any fp32 evaluation's absolute error.)
        Wy, ny, Sy = R.axis_weights(range(top, top + size[0]), H, RH)
        Wx, nx, Sx = R.axis_weights(range(left, left + size[1]), W, RW)
        E_tv = R.error_bound(nx[None, :], Sx[None, :], ny[:, None], Sy[:, None], sum_roundings=2)
        tv = torchvision_train_input(x, size, resize).to(dtype).double().numpy()
        u = R.ulp(ref, *R.FORMATS[fmt])
        to_midpoint = np.abs(ref / u - np.floor(ref / u) - 0.5) * u
        clear = to_midpoint > E + E_tv
        assert np.all(got[clear] == tv[clear]), int((got[clear] != tv[clear]).sum())
        assert np.all(np.abs(got - tv) <= u + E + E_tv), np.abs(got - tv).max()


def test_out_writes_one_batch_slot():
    from cvvae_b200.video_io import frames_to_training_input
    x = torch.from_numpy(frames(5, 120, 160, 3)).cuda()
    want = frames_to_training_input(x, (64, 96), "cover", torch.bfloat16)
    batch = torch.full((3, 3, 5, 64, 96), float("nan"), dtype=torch.bfloat16, device="cuda")
    got = frames_to_training_input(x, (64, 96), "cover", torch.bfloat16, out=batch[1:2])
    assert got.data_ptr() == batch[1:2].data_ptr()
    assert torch.equal(batch[1:2], want)
    assert torch.isnan(batch[0]).all() and torch.isnan(batch[2]).all()
    with pytest.raises(ValueError, match="out must be"):
        frames_to_training_input(x, (64, 96), "cover", torch.float16, out=batch[1:2])
    with pytest.raises(ValueError, match="out must be"):
        frames_to_training_input(x, (64, 96), "cover", torch.bfloat16, out=batch[:, :, :, :, :48])


def _per_clip(m, clips, size, resize):
    from cvvae_b200.video_io import frames_to_training_input
    return [m.encode(frames_to_training_input(torch.as_tensor(c).cuda(), size, resize, m.dtype))
            .latent_dist.parameters[0].cpu() for c in clips]


def _mixed_clips(hw, seed):
    """Clips of T in {1, 5, 9, 17} from sources of several sizes, numpy and torch, runs of equal T broken and resumed."""
    g = np.random.default_rng(seed)
    sources = [(hw[0], hw[1]), (hw[0] + 16, hw[1] + 40), (2 * hw[0], 3 * hw[1]), (hw[0] - 9, 2 * hw[1] + 1)]
    ts = [17, 17, 5, 1, 1, 1, 1, 9, 9, 9, 9, 5, 17]
    out = []
    for i, t in enumerate(ts):
        H, W = sources[i % len(sources)]
        c = g.integers(0, 256, (t, H, W, 3), dtype=np.uint8)
        out.append(c if i % 2 else torch.from_numpy(c))
    return out


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
@pytest.mark.parametrize("fmt", sorted(DTYPES))
@pytest.mark.parametrize("variant", ["sd21", "sd3"])
def test_encode_clips_bit_identical(variant, fmt, graphs):
    """Tiled fixtures (72-pixel tiles, 4 frames a chunk) at 104 x 120 crops: every batch is tiled and chunked."""
    from cvvae_b200 import encode_clips
    m = _build(variant, 32, WRAPS[f"{variant}_w32_tiled"], DTYPES[fmt])
    size = (104, 120)
    clips = _mixed_clips(size, 11)
    want = _per_clip(m, clips, size, "cover")
    m.enable_cuda_graphs(graphs)
    for bs in (1, 3, 8):
        for rep in range(2 if graphs else 1):      # with graphs: the first pass captures, the second replays
            got = list(encode_clips(m, clips, size, "cover", batch_size=bs))
            assert len(got) == len(want)
            for i, (g, w) in enumerate(zip(got, want)):
                assert g.device.type == "cpu" and g.dtype == m.dtype and g.shape == w.shape, (i, g.shape, w.shape)
                assert torch.equal(g, w), (variant, fmt, graphs, bs, i)
    if graphs:
        assert m._graph_cache
    m.enable_cuda_graphs(False)


def test_encode_clips_full_width_720p():
    """sd21 at full width, default tiling and chunking: 8 clips of 17 x 256^2 cropped from 720p, one batch of 8."""
    from cvvae_b200 import encode_clips
    m = _build("sd21", 128, {}, torch.float16)
    g = np.random.default_rng(5)
    clips = [g.integers(0, 256, (17, 720, 1280, 3), dtype=np.uint8) for _ in range(8)]
    want = _per_clip(m, clips, (256, 256), "cover")
    got = list(encode_clips(m, clips, (256, 256), batch_size=8))
    assert len(got) == 8 and got[0].shape == (8, 5, 32, 32)
    assert all(torch.equal(a, b) for a, b in zip(got, want))


def test_encode_clips_yields_are_owned_and_ordered():
    """Every clip has its own constant value, so a clip out of order or a slot overwritten later shows."""
    from cvvae_b200 import encode_clips
    m = _build("sd21", 32, {}, torch.float16)
    clips = [np.full((5, 40, 56, 3), 10 + 20 * i, dtype=np.uint8) for i in range(7)]
    want = _per_clip(m, clips, (32, 48), "cover")
    assert len({w.float().sum().item() for w in want}) == len(want)
    kept, snapshots = [], []
    for y in encode_clips(m, clips, (32, 48), batch_size=2):
        kept.append(y)
        snapshots.append(y.clone())
    assert all(torch.equal(a, b) for a, b in zip(kept, snapshots))   # later yields left the earlier ones alone
    assert all(torch.equal(a, b) for a, b in zip(kept, want))        # and each is its own clip's


def test_encode_clips_refuses_bad_items_on_arrival():
    from cvvae_b200 import encode_clips
    m = _build("sd21", 32, {}, torch.float16)
    good = np.zeros((1, 40, 56, 3), np.uint8)
    for bad, match in ((np.zeros((1, 40, 56, 3), np.float32), "host uint8"), (np.zeros((40, 56, 3), np.uint8), "host uint8"),
                       (np.zeros((0, 40, 56, 3), np.uint8), "host uint8"), (torch.zeros((1, 40, 56, 3), dtype=torch.uint8,
                                                                                      device="cuda"), "host uint8"),
                       (np.zeros((1, 480, 640, 3), np.uint8), "pad")):
        it = encode_clips(m, [good, bad], (32, 48) if match != "pad" else (320, 512), "short" if match == "pad" else "cover")
        with pytest.raises(ValueError, match=match):
            list(it)


def _peak(fn) -> int:
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_encode_clips_memory_does_not_grow_with_clip_count():
    from cvvae_b200 import encode_clips
    m = _build("sd21", 128, {}, torch.float16)
    g = np.random.default_rng(2)
    clip = g.integers(0, 256, (17, 180, 320, 3), dtype=np.uint8)
    bs = 4

    def run(n):
        for y in encode_clips(m, (clip for _ in range(n)), (128, 128), batch_size=bs):
            assert y.shape == (8, 5, 16, 16)

    run(8)                                  # warm-up: engine, packed weights, allocator
    p8, p32 = _peak(lambda: run(8)), _peak(lambda: run(32))
    assert p32 - p8 <= bs * clip.nbytes, (p8, p32, bs * clip.nbytes)

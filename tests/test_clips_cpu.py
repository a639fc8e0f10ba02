"""The training pre-processing on the CPU: the fp64 restatement (tests/clip_ref.py) against torchvision's float path, the
resize / crop geometry of video_io.training_geometry against torchvision's, the batching schedule of encode_clips, and
every refusal that needs no GPU."""
import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
from torchvision import transforms

import clip_ref as R
from cvvae_b200.streaming import clip_batches, encode_clips
from cvvae_b200.video_io import frames_to_training_input, training_geometry

# (T, H, W, size, resize): down-scale x2.8, up-scale, the short-side resize at 16:10, crop only, odd margins whose crop
# offsets are x.5 (rounded half to even), and one image
CASES = [
    (2, 720, 1280, (256, 256), "cover"),
    (2, 240, 320, (256, 256), "cover"),
    (1, 1080, 1920, (320, 512), "short"),
    (2, 256, 263, (256, 256), "cover"),
    (2, 100, 151, (64, 64), "cover"),
    (1, 37, 29, (24, 16), "cover"),
]
IDS = ["720p-256", "240p-256-up", "1080p-320x512-short", "crop-only", "odd-margins", "image"]


def frames(T, H, W, seed):
    return np.random.default_rng(seed).integers(0, 256, (T, H, W, 3), dtype=np.uint8)


def cover_size(H, W, size):
    """CoverResize (lvdm/data/transform.py:14-59): the smallest scale at which the frame covers `size`, sizes rounded."""
    f = max(size[0] / H, size[1] / W)
    return round(H * f), round(W * f)


def shifted_crop(RH, RW, top, left, size):
    """The crop offsets moved by one pixel, along an axis that has a margin."""
    return (top, left + 1) if RW > size[1] else (top + 1, left)


def torchvision_train_input(frames_u8, size, resize):
    """The reference's data path in torchvision, float32 throughout: [T, H, W, 3] -> [3, T, h, w]."""
    x = torch.from_numpy(frames_u8).permute(0, 3, 1, 2).float()
    if resize == "cover":
        x = F.resize(x, list(cover_size(x.shape[-2], x.shape[-1], size)), transforms.InterpolationMode.BILINEAR,
                     antialias=True)
    else:
        x = transforms.Resize(min(size))(x)
    x = F.center_crop(x, list(size))
    return ((x / 255 - 0.5) * 2).permute(1, 0, 2, 3)


@pytest.mark.parametrize("T,H,W,size,resize", CASES, ids=IDS)
def test_reference_matches_torchvision(T, H, W, size, resize):
    """clip_ref (fp64) and torchvision (fp32, no fused multiply-add assumed) agree within the fp32 error bound."""
    x = frames(T, H, W, H * W)
    RH, RW, top, left = training_geometry(H, W, size, resize)
    ref, _ = R.train_input_ref(x, RH, RW, top, left, *size)
    Wy, ny, Sy = R.axis_weights(range(top, top + size[0]), H, RH)
    Wx, nx, Sx = R.axis_weights(range(left, left + size[1]), W, RW)
    E = R.error_bound(nx[None, :], Sx[None, :], ny[:, None], Sy[:, None], sum_roundings=2)
    tv = torchvision_train_input(x, size, resize).double().numpy()
    assert tv.shape == ref.shape == (3, T, *size)
    assert np.all(np.abs(tv - ref) <= E), np.abs(tv - ref).max()
    # the bound is not vacuous: a crop one pixel off fails it
    shifted, _ = R.train_input_ref(x, RH, RW, *shifted_crop(RH, RW, top, left, size), *size)
    assert not np.all(np.abs(tv - shifted) <= E)


HS = [1, 17, 64, 99, 100, 240, 255, 256, 257, 263, 480, 720, 1080]
SIZES = [(256, 256), (320, 512), (64, 64), (100, 37), 48]


@pytest.mark.parametrize("size", SIZES, ids=str)
def test_geometry_matches_torchvision(size):
    """training_geometry gives torchvision's resized shape and CenterCrop's offsets, or refuses where CenterCrop pads."""
    hw = (size, size) if isinstance(size, int) else size
    for H in HS:
        for W in HS:
            for resize in ("cover", "short"):
                if resize == "cover":
                    RH, RW = cover_size(H, W, hw)
                else:
                    RH, RW = transforms.Resize(min(hw))(torch.zeros(1, H, W)).shape[-2:]
                if hw[0] > RH or hw[1] > RW:
                    with pytest.raises(ValueError, match="pad"):
                        training_geometry(H, W, size, resize)
                    continue
                grid = torch.arange(RH * RW, dtype=torch.float64).reshape(1, RH, RW)
                corner = int(F.center_crop(grid, list(hw))[0, 0, 0])
                assert training_geometry(H, W, size, resize) == (RH, RW, corner // RW, corner % RW), (H, W, size, resize)


def test_schedule_order_and_grouping():
    ts = [17, 17, 17, 5, 5, 1, 17, 17, 9, 9, 9, 9, 9]
    clips = list(enumerate(ts))
    for bs in (1, 2, 3, 8):
        batches = list(clip_batches(clips, bs, length=lambda c: c[1]))
        assert [c for b in batches for c in b] == clips                 # every clip once, in input order
        assert all(len(b) <= bs and len({c[1] for c in b}) == 1 for b in batches)
        # batches are maximal: a batch ends only when full, when T changes, or at the end
        for b, nxt in zip(batches, batches[1:]):
            assert len(b) == bs or b[0][1] != nxt[0][1]
    assert [[c[0] for c in b] for b in clip_batches(clips, 3, length=lambda c: c[1])] == \
        [[0, 1, 2], [3, 4], [5], [6, 7], [8, 9, 10], [11, 12]]
    assert list(clip_batches([], 4)) == []


def test_schedule_yields_a_full_batch_before_reading_on():
    read = []

    def source():
        for i in range(5):
            read.append(i)
            yield np.zeros((4, 2, 2, 3), np.uint8)

    it = clip_batches(source(), 2)
    assert len(next(it)) == 2 and read == [0, 1]
    assert len(next(it)) == 2 and read == [0, 1, 2, 3]
    assert len(next(it)) == 1 and read == [0, 1, 2, 3, 4]


class _CpuModel:
    device = torch.device("cpu")
    dtype = torch.float16


class _CudaModel:
    device = torch.device("cuda", 0)
    dtype = torch.float16


@pytest.mark.parametrize("kw,match", [
    (dict(batch_size=0), "batch_size"), (dict(batch_size=2.0), "batch_size"), (dict(batch_size=True), "batch_size"),
    (dict(size=(256,)), "size"), (dict(size=(0, 256)), "size"), (dict(size="256"), "size"), (dict(size=(256.0, 256)), "size"),
    (dict(resize="crop"), "resize"),
])
def test_encode_clips_refuses_at_the_call(kw, match):
    read = []

    def source():
        read.append(1)
        yield np.zeros((1, 8, 8, 3), np.uint8)

    args = dict(size=(256, 256), resize="cover", batch_size=4)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        encode_clips(_CudaModel(), source(), **args)
    assert read == []
    with pytest.raises(ValueError, match="CUDA"):
        encode_clips(_CpuModel(), source(), (256, 256))
    assert read == []


def test_geometry_and_binding_refusals():
    with pytest.raises(ValueError, match="pad"):
        training_geometry(480, 640, (320, 512), "short")       # 4:3 source, short side 320 -> 320 x 426 < 512
    with pytest.raises(ValueError, match="pad"):
        training_geometry(1920, 1080, (320, 512), "short")     # portrait source, 320 wide
    with pytest.raises(ValueError, match="resize"):
        training_geometry(480, 640, (256, 256), "area")
    with pytest.raises(ValueError, match="CUDA uint8"):
        frames_to_training_input(torch.zeros((2, 8, 8, 3), dtype=torch.uint8), (4, 4))
    with pytest.raises(ValueError, match="CUDA uint8"):
        frames_to_training_input(torch.zeros((2, 8, 8, 4), dtype=torch.uint8), (4, 4))

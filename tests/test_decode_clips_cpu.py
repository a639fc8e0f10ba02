"""decode_clips and the batched pixel conversion without a GPU: every refusal at the call and on arrival, the batching
schedule with a latent-shape key, the ctypes binding of cvvae_video_output_u8 against the header, and the library's
argument checks, which come before any launch."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from cvvae_b200.streaming import clip_batches, decode_clips

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPE = lambda z: tuple(z.shape)   # noqa: E731  (the key decode_clips batches by)


class _Net:
    z_channels = 4


class _CpuModel:
    device = torch.device("cpu")
    dtype = torch.float16
    net = _Net()


class _CudaModel:
    """Never reaches the device: every item refused with it is refused before the first batch is complete."""
    device = torch.device("cuda", 0)
    dtype = torch.float16
    net = _Net()


@pytest.mark.parametrize("batch_size", [0, -1, 2.0, True, "8", None])
def test_refuses_at_the_call(batch_size):
    read = []

    def source():
        read.append(1)
        yield np.zeros((4, 1, 2, 2), np.float16)

    with pytest.raises(ValueError, match="batch_size"):
        decode_clips(_CudaModel(), source(), batch_size=batch_size)
    with pytest.raises(ValueError, match="CUDA"):
        decode_clips(_CpuModel(), source())
    assert read == []


@pytest.mark.parametrize("bad,match", [
    (np.zeros((4, 2, 8), np.float16), "latents \\[4, t', h, w\\]"),                  # rank 3
    (np.zeros((1, 4, 2, 8, 8), np.float16), "latents \\[4, t', h, w\\]"),            # rank 5: a batch, not a clip
    (np.zeros((16, 2, 8, 8), np.float16), "latents \\[4, t', h, w\\]"),              # sd3's channel count
    (np.zeros((4, 0, 8, 8), np.float16), "t', h, w >= 1"),                           # t' = 0
    (np.zeros((4, 2, 0, 8), np.float16), "t', h, w >= 1"),
    (np.zeros((4, 2, 8, 8), np.float32), "float32, the model is torch.float16"),     # never cast
    (torch.zeros((4, 2, 8, 8), dtype=torch.bfloat16), "bfloat16, the model is torch.float16"),
    (torch.zeros((4, 2, 8, 8), dtype=torch.float16, device="meta"), "meta"),         # neither host nor the model's device
], ids=["rank3", "rank5", "channels", "t0", "h0", "fp32", "bf16", "device"])
def test_refuses_bad_items_on_arrival(bad, match, monkeypatch):
    import cvvae_b200.streaming as S

    class NoTransfers:   # the copy stream needs a device; nothing may be uploaded before the refusal anyway
        def __init__(self, dev):
            pass

    monkeypatch.setattr(S, "_HostTransfers", NoTransfers)
    good = np.zeros((4, 2, 8, 8), np.float16)
    it = decode_clips(_CudaModel(), [good, torch.from_numpy(good), bad], batch_size=8)
    with pytest.raises(ValueError, match=match):
        next(it)


def test_schedule_closes_on_shape_changes():
    shapes = [(4, 5, 32, 32), (4, 5, 32, 32), (4, 2, 32, 32), (4, 2, 32, 32), (4, 2, 32, 48), (4, 5, 32, 32),
              (4, 5, 32, 32), (4, 5, 32, 32), (4, 1, 16, 16)]
    clips = [torch.zeros(s) for s in shapes]
    for bs in (1, 2, 3, 8):
        batches = list(clip_batches(clips, bs, length=SHAPE))
        assert [c for b in batches for c in b] == clips                  # every clip once, in input order
        assert all(len(b) <= bs and len({tuple(c.shape) for c in b}) == 1 for b in batches)
        for b, nxt in zip(batches, batches[1:]):                         # maximal: full, a new shape, or the end
            assert len(b) == bs or b[0].shape != nxt[0].shape
    idx = {id(c): i for i, c in enumerate(clips)}
    assert [[idx[id(c)] for c in b] for b in clip_batches(clips, 2, length=SHAPE)] == \
        [[0, 1], [2, 3], [4], [5, 6], [7], [8]]


def test_schedule_yields_a_full_batch_before_reading_on():
    read = []

    def source():
        for i in range(5):
            read.append(i)
            yield torch.zeros((4, 2, 8, 8))

    it = clip_batches(source(), 2, length=SHAPE)
    assert len(next(it)) == 2 and read == [0, 1]
    assert len(next(it)) == 2 and read == [0, 1, 2, 3]
    assert len(next(it)) == 1 and read == [0, 1, 2, 3, 4]


def _header_args(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "cvvae_b200.h")).read(), flags=re.S)
    m = re.search(rf"\bint\s+{name}\s*\(([^)]*)\)", src)
    assert m, name
    ctype = {"int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64}
    return [ctypes.c_void_p if "*" in a else ctype[a.split()[-2]] for a in m.group(1).split(",")]


def test_output_u8_is_bound_with_the_header_signature():
    from cvvae_b200 import _lib as L
    res, args = L._SIGNATURES["cvvae_video_output_u8"]
    assert res is ctypes.c_int
    assert args == _header_args("cvvae_video_output_u8") == [ctypes.c_void_p] * 2 + [ctypes.c_int32] * 5 + [ctypes.c_void_p]
    assert "cvvae_video_output_u8" in L.EXPORTS


def test_output_u8_refuses_bad_arguments_before_any_launch():
    import __graft_entry__ as ge
    ge.build()
    from cvvae_b200 import _lib as L
    lib = L.load()
    fake = 256   # never dereferenced: every check precedes the launch
    big = 2 ** 31 - 1
    for args, msg in (((fake, fake, 1, 1, 2, 2, 7, None), b"unsupported dtype 7"),
                      ((fake, fake, 1, 1, 2, 2, -1, None), b"unsupported dtype -1"),
                      ((fake, fake, 0, 1, 2, 2, L.F16, None), b"B=0"),
                      ((fake, fake, -3, 1, 2, 2, L.F32, None), b"B=-3"),
                      ((fake, fake, 1, 0, 2, 2, L.BF16, None), b"T=0"),
                      ((fake, fake, 1, 1, 2, -2, L.F16, None), b"W=-2"),
                      ((None, fake, 1, 1, 2, 2, L.F16, None), b"bad argument"),
                      ((fake, None, 1, 1, 2, 2, L.F32, None), b"bad argument"),
                      ((fake, fake, big, big, big, big, L.F16, None), b"overflow"),
                      ((fake, fake, 2, 2 ** 21, 2 ** 20, 2 ** 20, L.F32, None), b"overflow")):
        assert lib.cvvae_video_output_u8(*args) == -1, args
        assert msg in lib.cvvae_last_error(), (args, lib.cvvae_last_error())
        assert b"cvvae_video_output_u8" in lib.cvvae_last_error() or msg.startswith(b"unsupported")


def test_batch_to_frames_refuses_without_a_launch():
    from cvvae_b200.video_io import batch_to_frames
    for x in (torch.zeros((1, 3, 1, 4, 4), dtype=torch.float16),            # host tensor
              torch.zeros((3, 1, 4, 4), dtype=torch.float16, device="meta"),  # rank 4
              torch.zeros((1, 4, 1, 4, 4), dtype=torch.float16, device="meta"),
              torch.zeros((1, 3, 1, 4, 4), dtype=torch.float64, device="meta")):
        with pytest.raises(ValueError, match="batch_to_frames expects"):
            batch_to_frames(x)

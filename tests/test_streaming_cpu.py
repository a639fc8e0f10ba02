"""StreamEncoder / StreamDecoder without a GPU: the product code driven through the torch restatement of the operator set
(tests/fake_ops.py), as in test_engine_wiring_cpu.py, on the tiled fixtures (72-px tiles, 4 pixel / 1 latent frames a
chunk, ragged edge tiles at 104x120).

The streams must reproduce the whole-clip encode() / decode() bit for bit however the clip is split across feeds, run
each chunk in the feed that delivers its last frame, and refuse inconsistent input before running anything.
"""
import random

import pytest
import torch

from cvvae_b200 import CVVAEModel, StreamDecoder, StreamEncoder, reconstruct_frames
from oracle import cvvae_oracle as O
from test_engine_wiring_cpu import CASES, build_model

HW = (104, 120)


def _splits(T, seed):
    """The three feed patterns: one feed, one frame per feed, a seeded random split (empty feeds included)."""
    rng = random.Random(seed)
    ragged, t = [], 0
    while t < T:
        k = rng.randint(0, 3)
        ragged.append((t, min(T, t + k)))
        t += k
    return {"whole": [(0, T)], "frames": [(i, i + 1) for i in range(T)], "random": ragged}


def _stream(stream, x, pieces):
    out = []
    for a, b in pieces:
        out += stream.feed(x[:, :, a:b])
    return out + stream.close()


@pytest.mark.parametrize("name", ["sd21_w32_tiled", "sd3_w32_tiled"])
@pytest.mark.parametrize("direction", ["encode", "decode"])
def test_stream_equals_whole_clip(name, direction):
    m, _ = build_model(CASES[name])
    S = m.encode_n_frames_a_time if direction == "encode" else m.decode_n_frames_a_time
    assert S == (4 if direction == "encode" else 1)
    zc = m.net.z_channels
    lat_hw = (m._engine().encoded_hw(HW[0]), m._engine().encoded_hw(HW[1]))
    for T in (0, 1, 2, S, S + 1, S + 2, 2 * S + 1, 2 * S + 2, 3 * S - 1):
        if direction == "encode":
            x = O.synthetic_video((1, 3, T, *HW), 4 + T) if T else torch.zeros((1, 3, 0, *HW))
            want = m.encode(x).latent_dist.parameters if T else None
        else:
            x = torch.randn((1, zc, T, *lat_hw), generator=torch.Generator().manual_seed(T))
            want = m.decode(x).sample if T else None
        for pattern, pieces in _splits(T, T).items():
            stream = StreamEncoder(m) if direction == "encode" else StreamDecoder(m)
            chunks = _stream(stream, x, pieces)
            if T == 0:
                assert chunks == [], pattern
                continue
            if direction == "encode":
                chunks = [c.parameters for c in chunks]
            got = torch.cat(chunks, dim=2)
            assert got.shape == want.shape and torch.equal(got, want), (T, pattern)


@pytest.mark.parametrize("direction", ["encode", "decode"])
def test_chunk_comes_back_from_the_feed_that_completes_it(direction):
    m, _ = build_model(CASES["sd21_w32_tiled"])
    S = m.encode_n_frames_a_time if direction == "encode" else m.decode_n_frames_a_time
    C = 3 if direction == "encode" else m.net.z_channels
    hw = HW if direction == "encode" else (13, 15)
    T = 3 * S + 1
    x = torch.randn((1, C, T, *hw), generator=torch.Generator().manual_seed(1))
    stream = StreamEncoder(m) if direction == "encode" else StreamDecoder(m)
    for i in range(T):
        got = stream.feed(x[:, :, i:i + 1])
        # chunk n covers frames [S*n, S*n + S + 1): it runs once frame S*n + S is in
        assert len(got) == (1 if i >= S and i % S == 0 else 0), (i, len(got))
    assert stream.close() == []        # T == S*m + 1: the last chunk ended on the clip's last frame
    assert stream.close() == []        # a second close() has nothing either

    make = StreamEncoder if direction == "encode" else StreamDecoder
    stream = make(m)
    assert stream.feed(x[:, :, :1]) == [] and len(stream.close()) == 1     # T == 1: one 1-frame round, as _chunks
    if S > 1:                                                                 # a partial chunk runs at close()
        stream = make(m)
        assert len(stream.feed(x[:, :, :S + 2])) == 1 and len(stream.close()) == 1 and stream.close() == []


def test_errors():
    m, _ = build_model(CASES["sd21_w32_tiled"])
    x = O.synthetic_video((1, 3, 2, 32, 40), 1)
    plain = CVVAEModel(ch=32, en_de_n_frames_a_time=None, tile_spatial_size=None)
    for cls in (StreamEncoder, StreamDecoder):
        with pytest.raises(ValueError, match="temporal chunking"):
            cls(plain)
    enc = StreamEncoder(m)
    enc.feed(x[:, :, :1])
    for bad, what in ((x.expand(2, -1, -1, -1, -1), "batch"), (x[:, :, :, :24], "height"), (x[..., :32], "width")):
        with pytest.raises(ValueError, match=what):
            enc.feed(bad)
    with pytest.raises(ValueError, match=r"\[B, 3, t, H, W\]"):
        enc.feed(x[:, :2])
    with pytest.raises(ValueError, match=r"\[B, 4, t, H, W\]"):
        StreamDecoder(m).feed(x)
    # mismatches against the model: the wrapper's own errors
    with pytest.raises(RuntimeError, match="Input type"):
        enc.feed(x.double())
    closed = StreamEncoder(m)
    closed.feed(x)
    closed.close()
    with pytest.raises(ValueError, match="after close"):
        closed.feed(x)
    # dtype / device changed between feeds (the model was converted mid-clip)
    m.double()
    with pytest.raises(ValueError, match="dtype changed"):
        enc.feed(x.double())
    m.float()
    m.to("meta")
    with pytest.raises(ValueError, match="device changed"):
        enc.feed(torch.empty(x.shape, device="meta"))


def test_reconstruct_frames_refuses_float32():
    m, _ = build_model(CASES["sd21_w32_tiled"])
    frames = [torch.zeros((5, 16, 16, 3), dtype=torch.uint8)]
    with pytest.raises(ValueError, match="float16 / bfloat16 only"):
        reconstruct_frames(m, frames)          # raises at the call, before anything is read or launched

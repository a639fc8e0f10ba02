"""StreamEncoder / StreamDecoder / reconstruct_frames on the H100: bit-exact against the whole-clip calls in every dtype,
eager and with CUDA graphs, at the fixtures' sizes and at 49x576x1024; device memory flat in the clip length; the
host-to-host reconstruction chain equal to the reference script's whole-clip chain, also for a model on a device other
than the current one."""
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import cvvae_oracle as O

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
with open(os.path.join(GOLD, "manifest.json")) as f:
    MANIFEST = json.load(f)
CASES = {c["name"]: c for c in MANIFEST["cases"]}
TILED = {
    "sd21_w32": dict(variant="sd21", ch=32, wrap=CASES["sd21_w32_tiled"]["wrap"], hw=(104, 120)),
    "sd3_w32": dict(variant="sd3", ch=32, wrap=CASES["sd3_w32_tiled"]["wrap"], hw=(104, 120)),
    "sd21_w128": dict(variant="sd21", ch=128, wrap=CASES["sd21_w128_tiled"]["wrap"], hw=(96, 112)),
    "sd3_w128": dict(variant="sd3", ch=128, wrap=CASES["sd21_w128_tiled"]["wrap"], hw=(96, 112)),
}


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


def _random_split(T, seed):
    rng = random.Random(seed)
    out, t = [], 0
    while t < T:
        k = rng.randint(0, 6)
        out.append((t, min(T, t + k)))
        t += k
    return out


def _stream(stream, x, pieces):
    out = []
    for a, b in pieces:
        out += stream.feed(x[:, :, a:b])
    return out + stream.close()


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32], ids=["fp16", "bf16", "fp32"])
@pytest.mark.parametrize("name", sorted(TILED))
def test_stream_bit_exact(name, dtype, graphs):
    """The fixture's chunking (4 frames a chunk: two full chunks), and 8 frames a chunk with a final partial chunk of 5
    frames / 2 latents.  (A partial chunk that adds no frame, e.g. the last 2 or 3 frames at 4 a chunk, is not compared:
    the whole-clip call refuses the empty copy of its result on the GPU; the streams emit it as an empty chunk.)"""
    from cvvae_b200 import StreamDecoder, StreamEncoder
    c = TILED[name]
    for frames_a_time, T in ((c["wrap"]["en_de_n_frames_a_time"], 9), (8, 21)):
        m = _build(c["variant"], c["ch"], dict(c["wrap"], en_de_n_frames_a_time=frames_a_time), dtype)
        x = O.synthetic_video((1, 3, T, *c["hw"]), 21).to(dtype).cuda()
        want_mom = m.encode(x).latent_dist.parameters
        z = want_mom[:, :m.net.z_channels]
        want_rec = m.decode(z).sample
        m.enable_cuda_graphs(graphs)
        for rep in range(2 if graphs else 1):      # with graphs: the first pass captures, the second replays
            for pieces in ([(0, T)], _random_split(T, rep)):
                got = torch.cat([p.parameters for p in _stream(StreamEncoder(m), x, pieces)], dim=2)
                assert torch.equal(got, want_mom), (name, frames_a_time, pieces)
            for pieces in ([(0, z.shape[2])], [(i, i + 1) for i in range(z.shape[2])]):
                got = torch.cat(_stream(StreamDecoder(m), z, pieces), dim=2)
                assert torch.equal(got, want_rec), (name, frames_a_time, pieces)
        if graphs:
            assert m._graph_cache
        m.enable_cuda_graphs(False)


def test_stream_bit_exact_full_size():
    """49x576x1024 fp16, full-width sd21 at the default tiling: 3 chunks x 2 tiles each way."""
    from cvvae_b200 import StreamDecoder, StreamEncoder
    m = _build("sd21", 128, {}, torch.float16)
    x = O.synthetic_video((1, 3, 49, 576, 1024), 3).half().cuda()
    post = m.encode(x).latent_dist
    want_rec = m.decode(post.mode()).sample
    pieces = _random_split(49, 7)
    enc_chunks = _stream(StreamEncoder(m), x, pieces)
    assert len(enc_chunks) == 3
    assert torch.equal(torch.cat([p.parameters for p in enc_chunks], dim=2), post.parameters)
    dec = StreamDecoder(m)
    rec_chunks = [r for p in enc_chunks for r in dec.feed(p.mode())] + dec.close()
    assert len(rec_chunks) == 3
    assert torch.equal(torch.cat(rec_chunks, dim=2), want_rec)


def _peak(fn) -> int:
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_stream_memory_is_flat_in_clip_length():
    from cvvae_b200 import StreamDecoder, StreamEncoder
    m = _build("sd21", 128, {}, torch.float16)
    S, H, W = m.encode_n_frames_a_time, 256, 256
    clips = {T: O.synthetic_video((1, 3, T, H, W), T).half() for T in (33, 129)}

    def stream(x_host):
        enc, dec, kept = StreamEncoder(m), StreamDecoder(m), []
        for a in range(0, x_host.shape[2], 8):
            for p in enc.feed(x_host[:, :, a:a + 8].cuda()):
                kept += [r.cpu() for r in dec.feed(p.mode())]
        for p in enc.close():
            kept += [r.cpu() for r in dec.feed(p.mode())]
        kept += [r.cpu() for r in dec.close()]
        assert sum(r.shape[2] for r in kept) == x_host.shape[2]

    def whole(x_host):
        x = x_host.cuda()
        rec = m.decode(m.encode(x).latent_dist.mode()).sample
        assert rec.shape == x.shape

    for T, x in clips.items():          # warm-up: engine, packed weights, allocator
        stream(x)
    s = {T: _peak(lambda: stream(x)) for T, x in clips.items()}
    w = {T: _peak(lambda: whole(x)) for T, x in clips.items()}
    frame = 3 * H * W * 2               # one fp16 frame, input or reconstruction
    chunk_io = 2 * (S + 1) * frame      # one chunk's input plus output
    assert s[129] - s[33] <= chunk_io, (s, chunk_io)
    assert w[129] - w[33] >= 96 * 2 * frame, (w, 96 * 2 * frame)


def _script_chain(m, frames_u8, size):
    """The reference script's body on the whole clip: trim, upload, convert, encode, mode, decode, convert, download."""
    from cvvae_b200.video_io import frames_to_input, output_to_frames
    T = frames_u8.shape[0]
    frame_end = 1 + (T - 1) // 4 * 4
    x = frames_to_input(frames_u8[:frame_end].cuda(), dtype=m.dtype, size=size)
    return output_to_frames(m.decode(m.encode(x).latent_dist.mode()).sample).cpu()


@pytest.mark.parametrize("size", [None, (72, 88)], ids=["native", "resized"])
@pytest.mark.parametrize("T", [41, 44])
@pytest.mark.parametrize("name", ["sd21_w32_tiled", "sd21_w32_default"])
def test_reconstruct_frames_bit_exact(name, T, size):
    from cvvae_b200 import reconstruct_frames
    wrap = {} if name == "sd21_w32_default" else CASES[name]["wrap"]
    m = _build("sd21", 32, wrap, torch.float16)
    g = torch.Generator().manual_seed(T)
    frames = torch.randint(0, 256, (T, 80, 100, 3), generator=g, dtype=torch.uint8)
    lens, items, t = [7, 1, 20, 13, 0, 5], [], 0
    while t < T:
        k = lens[len(items) % len(lens)]
        items.append(frames[t:t + k].numpy() if len(items) % 2 else frames[t:t + k])
        t += k
    pieces = list(reconstruct_frames(m, items, size=size))        # every piece kept to the end
    want = _script_chain(m, frames, size)
    assert all(p.dtype == torch.uint8 and p.device.type == "cpu" for p in pieces)
    got = torch.cat(pieces, dim=0)
    assert got.shape == want.shape and torch.equal(got, want)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_model_on_another_device_than_the_current_one():
    """A model on cuda:1 while cuda:0 is current: the host-facing streams and the pixel conversions launch on the model's
    device, and give the bits the same calls give on cuda:0."""
    from cvvae_b200 import encode_clips, evaluate_frames, reconstruct_frames
    from cvvae_b200.video_io import frames_to_input, output_to_frames
    frames = torch.randint(0, 256, (9, 64, 80, 3), generator=torch.Generator().manual_seed(9), dtype=torch.uint8)
    items = [frames[:4], frames[4:].numpy()]

    def calls(dev):
        m = _build("sd21", 32, {}, torch.float16).to(dev)
        x = frames_to_input(frames.to(dev), dtype=m.dtype)
        scored = list(evaluate_frames(m, items))
        return [x.cpu(), output_to_frames(x).cpu(), torch.cat(list(reconstruct_frames(m, items))),
                *(torch.cat(parts) for parts in zip(*scored)), *encode_clips(m, [frames[:5], frames.numpy()], (64, 80))]

    want = calls("cuda:0")
    with torch.cuda.device(0):
        got = calls("cuda:1")
    assert len(got) == len(want) == 8
    assert all(torch.equal(a, b) for a, b in zip(got, want))


def test_reconstruct_frames_sample_posterior_is_seeded():
    from cvvae_b200 import reconstruct_frames
    m = _build("sd21", 32, {}, torch.bfloat16)
    frames = [np.full((9, 32, 48, 3), v, dtype=np.uint8) for v in (10, 200, 90)]
    runs = [torch.cat(list(reconstruct_frames(m, frames, sample_posterior=True,
                                              generator=torch.Generator(device="cuda").manual_seed(5))))
            for _ in range(2)]
    mode = torch.cat(list(reconstruct_frames(m, frames)))
    assert runs[0].shape == mode.shape == (25, 32, 48, 3)
    assert torch.equal(runs[0], runs[1])

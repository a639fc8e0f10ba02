"""Streaming encode / decode: a clip of any length, fed and returned one temporal chunk at a time.

``model.encode(x)`` / ``model.decode(z)`` take the whole clip as one device tensor and build the whole result as one
tensor, so device memory grows with the clip.  The networks themselves already run one chunk at a time: chunk n covers
frames [S*n, S*n + S + 1) (S = ``encode_n_frames_a_time`` / ``decode_n_frames_a_time``) and depends on the rest of
the clip only through its first frame, which it shares with chunk n-1 (``_CVVAEBase._chunks``; the same coupling
``parallel.FrameShardedVAE`` exchanges between ranks).  The streams here keep that one carried frame plus the frames
of the open chunk in a staging buffer of S+1 frames, run each chunk through ``model.tiled_encode`` /
``model.tiled_decode`` as soon as its last frame arrives, and hand the result back.  Device memory is bounded by one
chunk however long the clip is, and the concatenated chunks are bit-identical to the whole-clip call.

``reconstruct_frames`` chains pixel upload, encoder, posterior, decoder and pixel download over host uint8 frames:
the body of the reference's ``cvvae_inference_video.py`` as a stream.  ``evaluate_frames`` is the same stream with every
reconstructed frame scored (PSNR, SSIM) on the device against the input frame the network saw.
"""
from __future__ import annotations

from collections import deque
from typing import Iterable, Iterator, Optional

import torch

from .modeling_vae import DiagonalGaussianDistribution


class _ChunkStream:
    """Chunk schedule shared by StreamEncoder and StreamDecoder; `_which` selects the network."""

    _which = ""

    def __init__(self, model):
        stride = model.encode_n_frames_a_time if self._which == "encode" else model.decode_n_frames_a_time
        if stride is None:
            raise ValueError(f"streaming {self._which} needs temporal chunking: the model was built with "
                             "en_de_n_frames_a_time=None")
        self.model = model
        self.stride = stride
        self._channels = model.net.in_channels if self._which == "encode" else model.net.z_channels
        self._buf: Optional[torch.Tensor] = None   # [B, C, S+1, H, W]: carried frame | frames of the open chunk
        self._fill = 0                             # frames held in _buf
        self._chunks_run = 0
        self._closed = False

    def _check(self, x: torch.Tensor) -> None:
        if self._closed:
            raise ValueError(f"{type(self).__name__}.feed() after close()")
        self.model._maybe_offload_hook()
        if x.dim() != 5 or x.shape[1] != self._channels:
            raise ValueError(f"{type(self).__name__}.feed() expects [B, {self._channels}, t, H, W]; got {tuple(x.shape)}")
        self.model._check_input(x)
        if self._buf is None:
            B, C, _, H, W = x.shape
            self._buf = torch.empty((B, C, self.stride + 1, H, W), dtype=x.dtype, device=x.device)
            return
        b = self._buf
        for what, got, want in (("batch", x.shape[0], b.shape[0]), ("height", x.shape[3], b.shape[3]),
                                ("width", x.shape[4], b.shape[4]), ("dtype", x.dtype, b.dtype),
                                ("device", x.device, b.device)):
            if got != want:
                raise ValueError(f"{type(self).__name__}.feed(): {what} changed between feeds ({want} -> {got})")

    def _run(self, n_frames: int) -> torch.Tensor:
        """The chunk held in the first `n_frames` staged frames; chunk n > 0 drops its first (carried) output frame."""
        src = self._buf[:, :, :n_frames]
        out = self.model.tiled_encode(src) if self._which == "encode" else self.model.tiled_decode(src)
        if self._chunks_run:
            out = out[:, :, 1:]
        self._chunks_run += 1
        return out

    def _wrap(self, out: torch.Tensor):
        return out

    @torch.no_grad()
    def feed(self, x: torch.Tensor) -> list:
        """Append frames `x` ([B, C, t, H, W], t >= 0) to the clip; returns the chunks this feed completed."""
        self._check(x)
        done = []
        t, pos, full = x.shape[2], 0, self.stride + 1
        while pos < t:
            k = min(full - self._fill, t - pos)
            self._buf[:, :, self._fill:self._fill + k].copy_(x[:, :, pos:pos + k])
            self._fill += k
            pos += k
            if self._fill == full:
                done.append(self._wrap(self._run(full)))
                self._buf[:, :, :1].copy_(self._buf[:, :, full - 1:])   # last frame of this chunk opens the next one
                self._fill = 1
        return done

    @torch.no_grad()
    def close(self) -> list:
        """End of the clip: runs the final partial chunk, if there is one, and returns it ([] when nothing is left).
        Later calls return []."""
        if self._closed:
            return []
        self._closed = True
        done = []
        # the staged frames are the clip's frames [S*m, T) with m = chunks already run: a partial chunk is left when it
        # holds more than the carried frame, or when it is the 1-frame clip (one round for T = 1, as in _chunks)
        if self._fill > 1 or (self._fill == 1 and self._chunks_run == 0):
            self.model._maybe_offload_hook()
            done.append(self._wrap(self._run(self._fill)))
        self._buf = None
        return done


class StreamEncoder(_ChunkStream):
    """Encode a clip fed in pieces of any length.

    ``feed(x)`` takes pixel frames ``[B, 3, t, H, W]`` on the model's device in the model's dtype and returns the chunks
    it completed, each a ``DiagonalGaussianDistribution`` over that chunk's moments; ``close()`` returns the rest.
    Concatenated along dim 2, the chunks' ``parameters`` (and so ``mode()``) are bit-identical to
    ``model.encode(whole_clip).latent_dist.parameters``, however the clip was split across feeds.  ``sample(generator)``
    draws its noise chunk by chunk, so it does not reproduce a whole-clip ``sample()`` with the same generator.

    With the defaults (16 frames a chunk) chunk 0 holds latents [0, 5) and chunk n > 0 latents [4n+1, 4n+5), which is
    what ``StreamDecoder`` needs to run its chunk n.  A final partial chunk of 2 to 4 frames adds no latent frame beyond
    its carried one and comes back with 0 frames.
    """

    _which = "encode"

    def _wrap(self, out: torch.Tensor) -> DiagonalGaussianDistribution:
        return DiagonalGaussianDistribution(out)


class StreamDecoder(_ChunkStream):
    """Decode latents fed in pieces of any length.

    ``feed(z)`` takes latents ``[B, z, t, h, w]`` and returns the pixel chunks ``[B, 3, t', H, W]`` it completed;
    ``close()`` returns the rest.  Concatenated along dim 2 they are bit-identical to ``model.decode(z).sample`` of
    the whole 5-D latent (with ``reshape_x_dim_to_4=False``), however the latents were split across feeds.
    """

    _which = "decode"


def _pinned(shape, like: torch.Tensor) -> torch.Tensor:
    return torch.empty(shape, dtype=like.dtype, pin_memory=True)


def reconstruct_frames(model, frames: Iterable, size=None, sample_posterior: bool = False,
                       generator: Optional[torch.Generator] = None) -> Iterator[torch.Tensor]:
    """Encode and decode a video given as host uint8 frames, one chunk at a time.

    `frames` is an iterable of uint8 batches ``[t, H, W, 3]`` (numpy arrays or CPU tensors, any t per item).  Yields
    the reconstruction as host uint8 ``[t', h, w, 3]`` pieces (``(h, w) = size`` if given, else ``(H, W)``).  Like the
    reference script, the trailing frames past ``1 + (T-1)//4*4`` are dropped (4 = the model's time compression), so
    the concatenated pieces equal::

        output_to_frames(model.decode(model.encode(frames_to_input(all_frames[:frame_end].cuda(), size=size))
                                      .latent_dist.mode()).sample)

    bit for bit.  ``sample_posterior=True`` decodes ``sample(generator)`` instead of ``mode()``, drawn chunk by chunk.

    Uploads and downloads run on a side stream, overlapped with the networks on the device's current stream.  A piece
    is yielded once the next chunk has been enqueued, so the GPU keeps working while the caller consumes it; device
    memory holds about one chunk.  Yielded tensors are the caller's: later pieces never overwrite them.  Only float16
    and bfloat16 models are supported (the pixel conversion kernels are 16-bit).
    """
    enc, dec = _open(model, "reconstruct_frames")
    return _reconstruct(model, enc, dec, iter(frames), size, sample_posterior, generator, False)


def evaluate_frames(model, frames: Iterable, size=None, sample_posterior: bool = False,
                    generator: Optional[torch.Generator] = None) -> Iterator[tuple]:
    """``reconstruct_frames`` with a score for every frame: yields ``(frames_u8, psnr, ssim)`` per piece.

    Same inputs and refusals as ``reconstruct_frames``, and ``frames_u8`` is what it yields.  ``psnr`` and ``ssim`` are
    float64 host tensors with one entry per frame of the piece (``cvvae_b200.metrics`` has the definitions).  Output
    frame i is scored against input frame i as the network saw it: after the resize to `size`, as uint8, before
    ``/ 127.5 - 1``.  The trailing frames past ``1 + (T-1)//4*4`` are not reconstructed and so not scored.
    The networks reproduce frame sizes that are a multiple of their spatial stride; when the reconstruction's size differs
    from the input's there is nothing to score it against and ``ValueError`` is raised: pass such a `size`.

    The scores are computed on the device, one kernel per piece right after the pixel conversion, and travel to the
    host with the frames.  The uint8 input of a chunk stays on the device until its reconstruction appears, so the
    stream holds at most two chunks' uint8 frames more than ``reconstruct_frames``, whatever the clip's length.
    """
    enc, dec = _open(model, "evaluate_frames")
    return _reconstruct(model, enc, dec, iter(frames), size, sample_posterior, generator, True)


def _open(model, who: str):
    if model.dtype not in (torch.float16, torch.bfloat16):
        raise ValueError(f"{who}: the pixel conversion is float16 / bfloat16 only; model dtype is {model.dtype}")
    if model.device.type != "cuda":
        raise ValueError(f"{who}: the model must be on a CUDA device")
    return StreamEncoder(model), StreamDecoder(model)   # raise for models without temporal chunking


def _reconstruct(model, enc: StreamEncoder, dec: StreamDecoder, frames: Iterator, size, sample_posterior: bool,
                 generator, score: bool) -> Iterator:
    """The stream behind reconstruct_frames (`score` False: yields frames) and evaluate_frames (True: yields
    (frames, psnr, ssim))."""
    from . import metrics
    from .video_io import frames_to_input, frames_to_input_and_u8, output_to_frames

    # No device context is held across the yields (it would leak into the caller's code): every allocation, stream and
    # launch below names the model's device, and the networks run on that device's current stream.
    dev = model.device
    time_compress = model.encode_n_frames_a_time // model.decode_n_frames_a_time
    copy = torch.cuda.Stream(device=dev)
    staging: Optional[torch.Tensor] = None   # pinned upload buffer, refilled once its last upload has completed
    staged = torch.cuda.Event()
    pending: deque = deque()    # input frames on the device, not yet fed: the clip may end before they are kept
    refs: deque = deque()       # score only: uint8 input frames as the network saw them, from the first frame not yet scored
    fed = received = 0
    downloads: deque = deque()  # (host frames, host int64 sums of their scores or None, event of their download), oldest first

    def take_refs(n: int) -> torch.Tensor:
        """The next `n` input frames: decoder chunks return the clip's frames in order, [0, 17) then 16 at a time."""
        parts = []
        while n:
            r = refs.popleft()
            if r.shape[0] > n:
                refs.appendleft(r[n:])
                r = r[:n]
            parts.append(r)
            n -= r.shape[0]
        return parts[0] if len(parts) == 1 else torch.cat(parts)

    def download(x: torch.Tensor) -> None:
        u8 = output_to_frames(x)
        host = _pinned(u8.shape, u8)
        acc = None
        if score:
            ref = take_refs(u8.shape[0])
            if ref.shape != u8.shape:
                raise ValueError(f"evaluate_frames: the networks return {u8.shape[1]} x {u8.shape[2]} frames for an input of "
                                 f"{ref.shape[1]} x {ref.shape[2]}, and frames of different sizes cannot be scored; pass "
                                 "`size=` with a size the networks reproduce (a multiple of their spatial stride)")
            acc = metrics._launch(ref, u8)
        sums = _pinned(acc.shape, acc) if score else None
        copy.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(copy):
            host.copy_(u8, non_blocking=True)
            if score:
                sums.copy_(acc, non_blocking=True)
            done = torch.cuda.Event()
            done.record(copy)
        u8.record_stream(copy)
        if score:
            acc.record_stream(copy)
        downloads.append((host, sums, done))

    def piece():
        host, sums, done = downloads.popleft()
        done.synchronize()
        if not score:
            return host
        m = metrics._scores(sums, host.shape[1], host.shape[2])
        return host, m.psnr, m.ssim

    def decode_chunks(latent_chunks) -> None:
        for post in latent_chunks:
            z = post.sample(generator=generator) if sample_posterior else post.mode()
            for x in dec.feed(z):
                download(x)

    for item in frames:
        item = torch.as_tensor(item)
        if item.dtype != torch.uint8 or item.dim() != 4 or item.shape[-1] != 3 or item.device.type != "cpu":
            raise ValueError(f"{'evaluate_frames' if score else 'reconstruct_frames'} expects host uint8 frames "
                             f"[t, H, W, 3]; got {item.dtype} {tuple(item.shape)} on {item.device}")
        t = item.shape[0]
        if t == 0:
            continue
        # host -> pinned staging -> device on the copy stream; the compute stream waits for that upload only
        staged.synchronize()
        if staging is None or staging.shape[0] < t or staging.shape[1:] != item.shape[1:]:
            staging = _pinned(item.shape, item)
        staging[:t].copy_(item)
        with torch.cuda.stream(copy):
            dev_u8 = torch.empty(item.shape, dtype=torch.uint8, device=dev)
            dev_u8.copy_(staging[:t], non_blocking=True)
            staged.record(copy)
        compute = torch.cuda.current_stream(dev)
        compute.wait_event(staged)
        dev_u8.record_stream(compute)
        if score:
            x, ref = frames_to_input_and_u8(dev_u8, dtype=model.dtype, size=size)
            pending.append(x)
            refs.append(ref)
        else:
            pending.append(frames_to_input(dev_u8, dtype=model.dtype, size=size))
        received += t
        # feed up to the last frame the script keeps so far (1 + (T-1)//4*4): frames past it wait for more input, and
        # are dropped if the clip ends first
        keep = 1 + (received - 1) // time_compress * time_compress
        while fed < keep:
            x = pending.popleft()
            k = min(x.shape[2], keep - fed)
            if k < x.shape[2]:
                pending.appendleft(x[:, :, k:])
            decode_chunks(enc.feed(x[:, :, :k]))
            fed += k
        # one-chunk lag: a piece goes to the caller only once a later chunk is enqueued behind it
        while len(downloads) > 1:
            yield piece()
    pending.clear()
    decode_chunks(enc.close())
    for x in dec.close():
        download(x)
    refs.clear()   # the trailing frames that were never reconstructed
    while downloads:
        yield piece()

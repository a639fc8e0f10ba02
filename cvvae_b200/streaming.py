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
reconstructed frame scored (PSNR, SSIM, optionally MS-SSIM and LPIPS) on the device against the input frame the network
saw.

``encode_clips`` turns a dataset of clips into latents: each clip goes through the reference's training pre-processing
(``video_io.frames_to_training_input``) straight into its slot of a batch, and batches of clips with equal length run
through one ``model.encode`` call each.  ``decode_clips`` is the way back: batches of clip latents of equal shape run
through one ``model.tiled_decode`` call and one pixel conversion each, and come back as uint8 videos.  ``embed_clips``
scores such sets: each clip's I3D embedding for FVD (``fvd.py``), batched the same way.
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


def _pinned(shape, dtype: torch.dtype) -> torch.Tensor:
    return torch.empty(shape, dtype=dtype, pin_memory=True)


class _HostTransfers:
    """The host <-> device copies of one host-facing stream: on a side copy stream of `dev`, overlapped with the kernels
    on that device's current (compute) stream.  Every allocation and stream names `dev`, so no device context is held
    between calls, and the callers may yield between them."""

    def __init__(self, dev: torch.device):
        self._dev = dev
        self._copy = torch.cuda.Stream(device=dev)
        self._staging: Optional[torch.Tensor] = None   # pinned uint8, flat, grown on demand; reused once its upload is done
        self._staged = torch.cuda.Event()
        self._downloads: deque = deque()               # (host tensors, event of their download), oldest first

    def __len__(self) -> int:
        """Downloads queued and not yet taken."""
        return len(self._downloads)

    def upload(self, host: torch.Tensor) -> torch.Tensor:
        """host -> pinned staging -> device on the copy stream; the compute stream waits for that upload only.  The
        staging buffer holds bytes: it is viewed as `host`'s dtype, whatever that is."""
        n = host.numel() * host.element_size()
        self._staged.synchronize()
        if self._staging is None or self._staging.numel() < n:
            self._staging = _pinned(n, torch.uint8)
        pinned = self._staging[:n].view(host.dtype).view(host.shape)
        pinned.copy_(host)
        with torch.cuda.stream(self._copy):
            out = torch.empty(host.shape, dtype=host.dtype, device=self._dev)
            out.copy_(pinned, non_blocking=True)
            self._staged.record(self._copy)
        compute = torch.cuda.current_stream(self._dev)
        compute.wait_event(self._staged)
        out.record_stream(compute)
        return out

    def download(self, *tensors: torch.Tensor) -> None:
        """Queue copies of `tensors` into fresh pinned host tensors, made after everything already enqueued on the
        compute stream."""
        hosts = tuple(_pinned(t.shape, t.dtype) for t in tensors)
        self._copy.wait_stream(torch.cuda.current_stream(self._dev))
        with torch.cuda.stream(self._copy):
            for host, t in zip(hosts, tensors):
                host.copy_(t, non_blocking=True)
            done = torch.cuda.Event()
            done.record(self._copy)
        for t in tensors:
            t.record_stream(self._copy)
        self._downloads.append((hosts, done))

    def take(self) -> tuple:
        """The host tensors of the oldest queued download, as passed to ``download``, once its copies have completed."""
        hosts, done = self._downloads.popleft()
        done.synchronize()
        return hosts


def _host_frames(item, who: str, min_t: int) -> torch.Tensor:
    """A host item (numpy array or tensor) as a host uint8 tensor [t, H, W, 3] with t >= `min_t`; ValueError otherwise."""
    item = torch.as_tensor(item)
    if (item.dtype != torch.uint8 or item.dim() != 4 or item.shape[0] < min_t or item.shape[-1] != 3
            or item.device.type != "cpu"):
        expects = f"clips [T, H, W, 3] with T >= {min_t}" if min_t else "frames [t, H, W, 3]"
        raise ValueError(f"{who} expects host uint8 {expects}; got {item.dtype} {tuple(item.shape)} on {item.device}")
    return item


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
    return _reconstruct(model, enc, dec, iter(frames), size, sample_posterior, generator, [])


def evaluate_frames(model, frames: Iterable, size=None, sample_posterior: bool = False,
                    generator: Optional[torch.Generator] = None, *, ms_ssim: bool = False, lpips=None,
                    maps: bool = False) -> Iterator[tuple]:
    """``reconstruct_frames`` with a score for every frame: yields ``(frames_u8, psnr, ssim)`` per piece,
    ``(frames_u8, psnr, ssim, ms_ssim)`` with ``ms_ssim=True``, and the per-frame LPIPS as one more last element when
    `lpips` is given.

    Same inputs and refusals as ``reconstruct_frames``, and ``frames_u8`` is what it yields.  ``psnr`` and ``ssim`` are
    float64 host tensors with one entry per frame of the piece (``cvvae_b200.metrics`` has the definitions).  Output
    frame i is scored against input frame i as the network saw it: after the resize to `size`, as uint8, before
    ``/ 127.5 - 1``.  The trailing frames past ``1 + (T-1)//4*4`` are not reconstructed and so not scored.
    The networks reproduce frame sizes that are a multiple of their spatial stride; when the reconstruction's size differs
    from the input's there is nothing to score it against and ``ValueError`` is raised: pass such a `size`.

    The scores are computed on the device, one kernel per piece right after the pixel conversion, and travel to the
    host with the frames.  The uint8 input of a chunk stays on the device until its reconstruction appears, so the
    stream holds at most two chunks' uint8 frames more than ``reconstruct_frames``, whatever the clip's length.

    With ``ms_ssim=True`` each piece is also scored by multi-scale SSIM (``metrics.frame_ms_ssim``, float64 per frame):
    ``metrics.MS_SSIM_LAUNCHES`` more kernels per piece on the same stream, right after the PSNR / SSIM kernel, on the
    same aligned input frames, and their sums ride in the same download.  MS-SSIM needs frames of at least 161 x 161 px
    as the network sees them; smaller ones raise ``ValueError`` when the first of them arrives.

    `lpips`: a ``metrics.LPIPS`` on the model's device (another device raises ``ValueError`` at the call), on VGG16 or
    AlexNet features (``lpips.net``).  Each piece is then also scored by LPIPS (float64 per frame): ``lpips.launches``
    kernels per group of frames on the same stream, right after the other metric kernels, on the same aligned input
    frames; its sums ride in the same download.  The activations of one group are freed before the next, so device
    memory stays flat in the clip's length.  LPIPS needs frames of at least ``lpips.min_size`` px on each side as the
    network sees them (16 for VGG16, 31 for AlexNet); smaller ones raise ``ValueError`` when the first of them arrives.

    ``maps=True`` says where each frame lost, not only how much: after every element above, each piece also carries the
    SSIM map (``metrics.ssim_map``, host float32 ``[t', h - 10, w - 10, 3]``) and, when `lpips` is given, the LPIPS map
    (``LPIPS.map``, host float32 ``[t', h, w]``), scored against the same aligned input frames.  The PSNR / SSIM launch
    becomes the kernel's map instantiation (still one launch, the same sums bit for bit) and LPIPS runs its network once
    for both score and map; the maps ride in the same download, so device memory stays flat in the clip's length.  The
    download grows accordingly: at 576 x 1024 the maps are 6.9 MB (SSIM) and 2.4 MB (LPIPS) per frame, against 1.8 MB for
    the uint8 frame.  Anything but a bool for `maps` raises ``ValueError``.
    """
    from . import metrics
    if not isinstance(maps, bool):
        raise ValueError(f"evaluate_frames: `maps` must be a bool; got {maps!r}")
    if lpips is not None:
        if not isinstance(lpips, metrics.LPIPS):
            raise ValueError(f"evaluate_frames: `lpips` must be a metrics.LPIPS or None; got {type(lpips).__name__}")
        if lpips.device != model.device:
            raise ValueError(f"evaluate_frames: the LPIPS weights are on {lpips.device}, the model on {model.device}")
    enc, dec = _open(model, "evaluate_frames")
    mapped = metrics._with_maps if maps else (lambda scorer: scorer)
    scorers = ([mapped(metrics._PSNR_SSIM)] + ([metrics._MS_SSIM] if ms_ssim else []) +
               ([mapped(lpips)] if lpips is not None else []))
    return _reconstruct(model, enc, dec, iter(frames), size, sample_posterior, generator, scorers)


def _open(model, who: str):
    if model.dtype not in (torch.float16, torch.bfloat16):
        raise ValueError(f"{who}: the pixel conversion is float16 / bfloat16 only; model dtype is {model.dtype}")
    if model.device.type != "cuda":
        raise ValueError(f"{who}: the model must be on a CUDA device")
    return StreamEncoder(model), StreamDecoder(model)   # raise for models without temporal chunking


def _reconstruct(model, enc: StreamEncoder, dec: StreamDecoder, frames: Iterator, size, sample_posterior: bool,
                 generator, scorers: list) -> Iterator:
    """The stream behind reconstruct_frames (no `scorers`: yields frames) and evaluate_frames (yields the frames, then
    what each of `scorers`, metrics' scorers, finishes for them, then the maps they leave, in the same order)."""
    from .video_io import frames_to_input, frames_to_input_and_u8, output_to_frames

    # No device context is held across the yields (it would leak into the caller's code): every allocation, stream and
    # launch below names the model's device or switches to it for its own duration, and the networks run on that
    # device's current stream.
    time_compress = model.encode_n_frames_a_time // model.decode_n_frames_a_time
    io = _HostTransfers(model.device)
    pending: deque = deque()    # input frames on the device, not yet fed: the clip may end before they are kept
    refs: deque = deque()       # score only: uint8 input frames as the network saw them, from the first frame not yet scored
    fed = received = 0

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
        if not scorers:
            return io.download(u8)
        ref = take_refs(u8.shape[0])
        if ref.shape != u8.shape:
            raise ValueError(f"evaluate_frames: the networks return {u8.shape[1]} x {u8.shape[2]} frames for an input of "
                             f"{ref.shape[1]} x {ref.shape[2]}, and frames of different sizes cannot be scored; pass "
                             "`size=` with a size the networks reproduce (a multiple of their spatial stride)")
        left = [out if isinstance(out, tuple) else (out,) for out in (m._launch(ref, u8) for m in scorers)]
        io.download(u8, *[out[0] for out in left], *[v for out in left for v in out[1:]])   # the sums, then the maps

    def piece(host: torch.Tensor, *outs: torch.Tensor):
        if not scorers:
            return host
        H, W = host.shape[1], host.shape[2]
        sums, maps = outs[:len(scorers)], outs[len(scorers):]
        return (host,) + tuple(v for m, s in zip(scorers, sums) for v in m._finish(s, H, W)) + maps

    def decode_chunks(latent_chunks) -> None:
        for post in latent_chunks:
            z = post.sample(generator=generator) if sample_posterior else post.mode()
            for x in dec.feed(z):
                download(x)

    for item in frames:
        item = _host_frames(item, "evaluate_frames" if scorers else "reconstruct_frames", 0)
        t = item.shape[0]
        if t == 0:
            continue
        seen = (int(size[0]), int(size[1])) if size is not None else tuple(item.shape[1:3])   # as the network sees them
        for m in scorers:
            m._check(*seen, "evaluate_frames")
        dev_u8 = io.upload(item)
        if scorers:
            x, ref = frames_to_input_and_u8(dev_u8, dtype=model.dtype, size=size)
            refs.append(ref)
        else:
            x = frames_to_input(dev_u8, dtype=model.dtype, size=size)
        pending.append(x)
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
        while len(io) > 1:
            yield piece(*io.take())
    pending.clear()
    decode_chunks(enc.close())
    for x in dec.close():
        download(x)
    refs.clear()   # the trailing frames that were never reconstructed
    while io:
        yield piece(*io.take())


def clip_batches(clips: Iterable, batch_size: int, length=len) -> Iterator[list]:
    """The batching schedule of ``encode_clips`` and ``decode_clips``: consecutive clips of equal ``length(clip)`` (for
    ``decode_clips``, a clip's latent shape) in batches of at most `batch_size`, in input order.  A batch closes as soon
    as it is full, when a clip of another length arrives, or at the end of the input; it is yielded then, before the next
    clip is read."""
    batch: list = []
    for clip in clips:
        if batch and length(clip) != length(batch[0]):
            yield batch
            batch = []
        batch.append(clip)
        if len(batch) == batch_size:
            yield batch
            batch = []
    if batch:
        yield batch


def encode_clips(model, clips: Iterable, size, resize: str = "cover", batch_size: int = 8) -> Iterator[torch.Tensor]:
    """Encode a dataset of clips to latent moments, batched on the GPU.

    `clips` is an iterable of host uint8 clips ``[T, H, W, 3]`` (numpy arrays or CPU tensors; T >= 1, a 1-frame clip is
    an image; T and the source size may differ from clip to clip).  Yields, for each clip in input order, a host tensor
    ``[2 z, t', h', w']`` in the model's dtype equal bit for bit to::

        model.encode(frames_to_training_input(clip.cuda(), size, resize, model.dtype)).latent_dist.parameters[0]

    that is, the clip prepared as the reference's training data path prepares it (``video_io.training_geometry``:
    "cover" = CoverResize + CenterCrop, "short" = Resize(min(size)) + CenterCrop), then encoded.
    ``DiagonalGaussianDistribution(moments[None])`` gives ``mode()`` / ``sample()``.

    Consecutive clips of equal T are stacked into one ``[B, 3, T, h, w]`` input (B <= `batch_size`, see
    ``clip_batches``), each clip written into its slot by one kernel launch, and the batch runs through one
    ``model.encode`` call, with the model's chunking, tiling and CUDA graphs.  Batching does not change any clip's
    moments: the engine's tile plans and GroupNorm statistics are per sample.

    Uploads and downloads run on a side stream, overlapped with the kernels on the device's current stream, and a batch's
    moments are yielded once the next batch has been enqueued.  Device memory holds one batch's input, activations and
    moments plus the source frames of the clips in flight, however many clips there are.  Yielded tensors are the
    caller's: later yields never overwrite them.

    Raises ValueError at the call for a model that is not on CUDA, `batch_size` < 1 or a malformed `size` / `resize`,
    and when an item arrives that is not a host uint8 ``[T, H, W, 3]`` clip with T >= 1, or whose centre crop torchvision
    would pad.
    """
    from .video_io import _check_resize, _check_size
    if model.device.type != "cuda":
        raise ValueError("encode_clips: the model must be on a CUDA device")
    if isinstance(batch_size, bool) or not isinstance(batch_size, int) or batch_size < 1:
        raise ValueError(f"encode_clips: batch_size must be an int >= 1; got {batch_size!r}")
    size = _check_size(size)
    _check_resize(resize)
    return _encode_clips(model, iter(clips), size, resize, batch_size)


def _encode_clips(model, clips: Iterator, size: tuple, resize: str, batch_size: int) -> Iterator[torch.Tensor]:
    from .video_io import frames_to_training_input, training_geometry

    def checked(items):
        for item in items:
            item = _host_frames(item, "encode_clips", 1)
            training_geometry(item.shape[1], item.shape[2], size, resize)   # refuses a crop torchvision would pad
            yield item

    # As in _reconstruct, no device context is held across the yields.  The `del`s free a clip's source frames once its
    # slot is written and the batch's input once it is encoded, so device memory stays one batch deep.
    io = _HostTransfers(model.device)
    for batch in clip_batches(checked(clips), batch_size):
        x = torch.empty((len(batch), 3, batch[0].shape[0], *size), dtype=model.dtype, device=model.device)
        for i, clip in enumerate(batch):
            src = io.upload(clip)
            frames_to_training_input(src, size, resize, model.dtype, out=x[i:i + 1])
            del src
        moments = model.encode(x).latent_dist.parameters
        del x
        io.download(moments)
        del moments
        # one-batch lag: a batch's moments go to the caller only once the next batch is enqueued behind it
        while len(io) > 1:
            yield from io.take()[0].unbind(0)
    while io:
        yield from io.take()[0].unbind(0)


def embed_clips(i3d, clips: Iterable, batch_size: int = 16) -> Iterator[torch.Tensor]:
    """FVD's I3D embedding of every clip of a dataset, batched on the GPU (``fvd.I3D``, ``fvd.frechet_distance``).

    `clips` is an iterable of uint8 clips ``[T, H, W, 3]`` with T >= 9: numpy arrays, CPU tensors or tensors on the
    network's device; T and the source size may differ from clip to clip.  Yields, for each clip in input order, a host
    float64 tensor ``[K]`` (K = 400 for Kinetics-400) equal bit for bit to ``i3d(clip[None])[0]``.

    Consecutive clips of equal ``(T, H, W)`` are stacked into one batch of at most `batch_size` (``clip_batches``); host
    clips are uploaded through a side stream, each clip is prepared into its slot of the batch by one
    ``frames_to_training_input(..., size=224, resize="short", dtype=torch.float32, out=...)`` launch, and the batch runs
    through the network in groups of ``i3d.group(T)`` clips.  A batch's embeddings are yielded once the next batch has
    been enqueued.  Device memory holds one batch's prepared clips and one group's activations plus the clips in flight,
    however many clips there are.

    Raises ValueError at the call for anything but an ``I3D`` or a `batch_size` that is not an int >= 1, and when an item
    arrives that is not a uint8 ``[T, H, W, 3]`` clip with T >= 9 on the host or the network's device."""
    from .fvd import I3D
    if not isinstance(i3d, I3D):
        raise ValueError(f"embed_clips: `i3d` must be an fvd.I3D; got {type(i3d).__name__}")
    if isinstance(batch_size, bool) or not isinstance(batch_size, int) or batch_size < 1:
        raise ValueError(f"embed_clips: batch_size must be an int >= 1; got {batch_size!r}")
    return _embed_clips(i3d, iter(clips), batch_size)


def _embed_clip(item, device: torch.device) -> torch.Tensor:
    """One clip (numpy array or tensor) as a host or `device` uint8 tensor [T, H, W, 3] with T >= 9; ValueError otherwise."""
    from .fvd import I3D_MIN_FRAMES
    item = torch.as_tensor(item)
    if (item.dtype != torch.uint8 or item.dim() != 4 or item.shape[0] < I3D_MIN_FRAMES or item.shape[-1] != 3
            or min(item.shape[1:3]) < 1):
        raise ValueError(f"embed_clips expects uint8 clips [T, H, W, 3] with T >= {I3D_MIN_FRAMES}; got {item.dtype} "
                         f"{tuple(item.shape)}")
    if item.device.type != "cpu" and item.device != device:
        raise ValueError(f"embed_clips: a clip on {item.device} for a network on {device}; pass host tensors or tensors "
                         "on the network's device")
    return item


def _embed_clips(i3d, clips: Iterator, batch_size: int) -> Iterator[torch.Tensor]:
    from .fvd import I3D_SIZE
    from .video_io import frames_to_training_input

    dev = i3d.device
    checked = (_embed_clip(item, dev) for item in clips)
    # As in _encode_clips, no device context is held across the yields, and the `del`s keep device memory one batch deep.
    io = _HostTransfers(dev)
    for batch in clip_batches(checked, batch_size, length=lambda clip: tuple(clip.shape[:3])):
        x = torch.empty((len(batch), 3, batch[0].shape[0], I3D_SIZE, I3D_SIZE), dtype=torch.float32, device=dev)
        for i, clip in enumerate(batch):
            src = io.upload(clip) if clip.device.type == "cpu" else clip
            frames_to_training_input(src, I3D_SIZE, "short", torch.float32, out=x[i:i + 1])
            del src
        emb = i3d._embed(x)
        del x
        io.download(emb)
        del emb
        # one-batch lag: a batch's embeddings go to the caller only once the next batch is enqueued behind it
        while len(io) > 1:
            yield from io.take()[0].unbind(0)
    while io:
        yield from io.take()[0].unbind(0)


def decode_clips(model, latents: Iterable, batch_size: int = 8) -> Iterator[torch.Tensor]:
    """Decode a dataset of clip latents to uint8 videos, batched on the GPU: the mirror of ``encode_clips``.

    `latents` is an iterable of one clip's latents each, ``[z, t', h, w]`` with t' >= 1, in the model's dtype: numpy
    arrays, CPU tensors or tensors on the model's device (a posterior's ``mode()[0]``, or a diffusion model's sample,
    scaled as ``model.decode`` expects).  Yields, for each clip in input order, a host uint8 ``[T, H, W, 3]`` tensor,
    T = ``model._engine().decoded_frames(t')``, equal bit for bit to::

        x = model.tiled_decode(z[None].to(model.device))     # what model.decode(z[None]).sample runs on 5-D latents
        output_to_frames(x)                                   # float16 / bfloat16 models
        ((x.clamp(-1, 1) + 1.0) * 127.5).to(torch.uint8)[0].permute(1, 2, 3, 0)   # float32 models, evaluated by torch

    Consecutive clips of equal ``(t', h, w)`` are stacked into one ``[B, z, t', h, w]`` batch (B <= `batch_size`, see
    ``clip_batches``), which runs through one ``model.tiled_decode`` call, with the model's chunking, tiling and CUDA
    graphs, and one ``video_io.batch_to_frames`` launch.  Batching changes no clip's frames: nothing in the engine mixes
    samples.

    Uploads and downloads run on a side stream, overlapped with the kernels on the device's current stream, and a batch's
    frames are yielded once the next batch has been enqueued.  Device memory holds one batch's latents, activations,
    decoded pixels and uint8 frames plus the download in flight, however many clips there are.  Yielded tensors are the
    caller's: later yields never overwrite them.

    Raises ValueError at the call for a model that is not on CUDA or a `batch_size` that is not an int >= 1, and when an
    item arrives that is not ``[z, t', h, w]`` with t', h, w >= 1, or whose dtype or device is not the model's (nothing is
    cast).
    """
    if model.device.type != "cuda":
        raise ValueError("decode_clips: the model must be on a CUDA device")
    if isinstance(batch_size, bool) or not isinstance(batch_size, int) or batch_size < 1:
        raise ValueError(f"decode_clips: batch_size must be an int >= 1; got {batch_size!r}")
    return _decode_clips(model, iter(latents), batch_size)


def _clip_latents(item, z_channels: int, dtype: torch.dtype, device: torch.device) -> torch.Tensor:
    """One clip's latents (numpy array or tensor) as a host or `device` tensor [z, t', h, w]; ValueError otherwise."""
    item = torch.as_tensor(item)
    if item.dim() != 4 or item.shape[0] != z_channels or min(item.shape[1:]) < 1:
        raise ValueError(f"decode_clips expects latents [{z_channels}, t', h, w] with t', h, w >= 1; got {tuple(item.shape)}")
    if item.dtype != dtype:
        raise ValueError(f"decode_clips: latents are {item.dtype}, the model is {dtype}; cast them first")
    if item.device.type != "cpu" and item.device != device:
        raise ValueError(f"decode_clips: latents on {item.device} for a model on {device}; pass host tensors or tensors "
                         "on the model's device")
    return item


def _decode_clips(model, latents: Iterator, batch_size: int) -> Iterator[torch.Tensor]:
    from .video_io import batch_to_frames

    dev, dtype, z_channels = model.device, model.dtype, model.net.z_channels
    checked = (_clip_latents(item, z_channels, dtype, dev) for item in latents)
    # As in _encode_clips, no device context is held across the yields, and the `del`s keep device memory one batch deep.
    io = _HostTransfers(dev)
    for batch in clip_batches(checked, batch_size, length=lambda z: tuple(z.shape)):
        z = torch.empty((len(batch), *batch[0].shape), dtype=dtype, device=dev)
        for i, item in enumerate(batch):
            if item.device.type == "cpu":
                src = io.upload(item)
                z[i].copy_(src)
                del src
            else:
                z[i].copy_(item)
        model._maybe_offload_hook()
        x = model.tiled_decode(z)
        del z
        frames = batch_to_frames(x)
        del x
        io.download(frames)
        del frames
        # one-batch lag: a batch's frames go to the caller only once the next batch is enqueued behind it
        while len(io) > 1:
            yield from io.take()[0].unbind(0)
    while io:
        yield from io.take()[0].unbind(0)

"""Fréchet Video Distance on the GPU: I3D embeddings of video clips, and the distance between two sets of them.

    I3D.from_state_dict(sd)(clips)             ->  float64 host [N, 400], one embedding per clip
    streaming.embed_clips(i3d, clips)          ->  the same, one [400] per clip of a dataset, batched
    frechet_distance(emb_a, emb_b)             ->  FVD, a Python float

FVD (Unterthiner et al. 2018) as VideoGPT and the common video-metrics scripts compute it: the Fréchet distance between
Gaussians fitted to the clips' Kinetics-400 I3D embeddings.  The network is ``InceptionI3d`` of the widely used PyTorch
port (``rgb_imagenet.pt`` / ``i3d_pretrained_400.pt``), in eval mode, and the embedding is its 400 logits averaged over
time.  rFVD of a video VAE is the FVD between real clips and their reconstructions.

Input: a clip is uint8 [T, H, W, 3] with T >= 9 (the smallest T for which the final pool has a temporal position).  It
is prepared as ``frames_to_training_input(clip, size=(224, 224), resize="short", dtype=torch.float32)``: torchvision's
antialiased ``Resize(224)`` of the float frames, ``CenterCrop(224)``, ``(x / 255 - 0.5) * 2``.  A 224 x 224 clip passes
unresized, so its network input is exactly ``(x / 255 - 0.5) * 2``.  VideoGPT resizes with non-antialiased
``F.interpolate`` instead (and other scripts resize uint8 frames, or to 224 x 224 without a crop), so FVD values are
comparable only between numbers computed by one pipeline.

Network: every convolution ``Unit3D`` is conv3d without bias, eval-mode ``BatchNorm3d(eps=1e-3)``, ReLU.  TF "SAME"
padding applies to every convolution and every max pool, per axis of extent n, kernel k, stride s: pad = max(k - s, 0)
if n % s == 0 else max(k - n % s, 0), front = pad // 2, back = pad - front, zeros (for the pools the same as -inf: they
read ReLU outputs); the output extent is ceil(n / s).  Layers: Conv3d_1a_7x7 (7^3, stride 2, 3 -> 64), MaxPool3d_2a_3x3
(1 x 3 x 3, stride (1, 2, 2)), Conv3d_2b_1x1 (64), Conv3d_2c_3x3 (3^3, 192), MaxPool3d_3a_3x3 (as 2a), Mixed_3b, 3c,
MaxPool3d_4a_3x3 (3^3, stride 2), Mixed_4b .. 4f, MaxPool3d_5a_2x2 (2^3, stride 2), Mixed_5b, 5c.  An Inception block of
widths (o0 .. o5) concatenates b0 = 1^3 -> o0; b1 = 1^3 -> o1, 3^3 -> o2; b2 = 1^3 -> o3, 3^3 -> o4; b3 = 3^3 stride-1
max pool, 1^3 -> o5.  Head: ``AvgPool3d([2, 7, 7], stride 1)`` without padding, the ``logits`` 1^3 convolution
1024 -> 400 with bias (no BN, no ReLU), the mean over the remaining temporal positions (Mixed_5c is [1024, 2, 7, 7] at
16 x 224^2, leaving one; [1024, 3, 7, 7] at 17 frames, leaving two).  Implementations differ here: some take the
pre-logits 1024-d pool or the softmax, or resize differently; this one follows VideoGPT's logits.

Computation: the 57 convolutions are BN-folded (in float64, then rounded once: the weights to TF32, the biases to fp32)
and run on the tensor-core convolution in fp32 with TF32 products and the ReLU in the epilogue, which is how PyTorch
evaluates an fp32 I3D on this GPU by default; every activation whose only consumers are convolutions is stored rounded
to TF32.  Each Inception branch writes straight into its channel slice of the block's output.  The stem's 7 x 7 spatial
taps of three consecutive frames are packed into 448 channels (``cvvae_i3d_stem_input``), so it runs as a 3 x 1 x 1
convolution.  The head is fp64.  A clip's embedding is bit-reproducible and independent of the other clips in the call.

``frechet_distance`` is the formula of StyleGAN-V / StyleGAN2-ADA, on the host in float64.
"""
from __future__ import annotations

import ctypes
import math
from typing import NamedTuple

import torch

from . import _lib as L

I3D_MIN_FRAMES = 9
I3D_SIZE = 224
I3D_BN_EPS = 1e-3
I3D_FEATURES = 1024           # channels of Mixed_5c, the logits' input
I3D_GROUP_BYTES = 8 << 30     # device bytes of activations one group of clips may take
I3D_STEM_CHANNELS = 448       # 3 frames x 7 x 7 taps x 3 channels = 441, padded to a multiple of 8
_BLOCKS = (("Mixed_3b", (64, 96, 128, 16, 32, 32)), ("Mixed_3c", (128, 128, 192, 32, 96, 64)), "MaxPool3d_4a_3x3",
           ("Mixed_4b", (192, 96, 208, 16, 48, 64)), ("Mixed_4c", (160, 112, 224, 24, 64, 64)),
           ("Mixed_4d", (128, 128, 256, 24, 64, 64)), ("Mixed_4e", (112, 144, 288, 32, 64, 64)),
           ("Mixed_4f", (256, 160, 320, 32, 128, 128)), "MaxPool3d_5a_2x2",
           ("Mixed_5b", (256, 160, 320, 32, 128, 128)), ("Mixed_5c", (384, 192, 384, 48, 128, 128)))
_TRUNK_POOLS = {"MaxPool3d_2a_3x3": ((1, 3, 3), (1, 2, 2)), "MaxPool3d_3a_3x3": ((1, 3, 3), (1, 2, 2)),
                "MaxPool3d_4a_3x3": ((3, 3, 3), (2, 2, 2)), "MaxPool3d_5a_2x2": ((2, 2, 2), (2, 2, 2))}


def same_padding(n: int, k: int, s: int) -> tuple:
    """TF "SAME" padding of an axis of extent n for kernel k and stride s: (front, back, output extent)."""
    pad = max(k - s, 0) if n % s == 0 else max(k - n % s, 0)
    return pad // 2, pad - pad // 2, -(-n // s)


class _Step(NamedTuple):
    """One kernel launch of the plan.  op "stem": cvvae_i3d_stem_input; "conv": the BN-folded Unit3D `name` (ReLU, then
    rounded to TF32 if `tf32_out`), into channels [c0, c0 + cout) of `dst`; "pool": SAME max pool; "head": the logits.
    `src` / `dst` index the plan's buffers."""
    op: str
    name: str
    src: int
    dst: int
    kernel: tuple = (1, 1, 1)
    stride: tuple = (1, 1, 1)
    cin: int = 0
    cout: int = 0
    c0: int = 0
    tf32_out: bool = True


class _Plan(NamedTuple):
    """The network on clips of T frames: its steps and the per-clip shape (T, H, W, C) of every buffer they read or write
    (buffer 0 is the prepared clip, channels-first [3, T, 224, 224], the others channels-last).  The forward pass, the
    launch count and the group size all read it."""
    steps: tuple
    buffers: tuple

    def lifetimes(self) -> list:
        """(first, last) step index of every buffer: the step that first writes it and the last that reads it.  The input
        belongs to the caller and is live throughout."""
        span = [[-1, len(self.steps) - 1] if b == 0 else [None, -1] for b in range(len(self.buffers))]
        for i, s in enumerate(self.steps):
            if s.dst >= 0 and span[s.dst][0] is None:
                span[s.dst][0] = i
            span[s.src][1] = max(span[s.src][1], i)
        return [tuple(v) for v in span]

    def clip_bytes(self) -> int:
        """Device bytes of the activations live at once for one clip, at the plan's largest point (fp32)."""
        spans = self.lifetimes()
        sizes = [4 * math.prod(shape) for shape in self.buffers]
        return max(sum(n for n, (a, b) in zip(sizes, spans) if a <= i <= b) for i in range(len(self.steps)))


def i3d_plan(T: int) -> _Plan:
    """The plan of I3D on clips of T frames at 224 x 224."""
    bufs, steps = [(T, I3D_SIZE, I3D_SIZE, 3)], []

    def new(shape) -> int:
        bufs.append(tuple(shape))
        return len(bufs) - 1

    def conv(name, src, cout, k, dst=None, c0=0, tf32_out=True) -> int:
        t, h, w, c = bufs[src]
        dst = new((t, h, w, cout)) if dst is None else dst
        steps.append(_Step("conv", name, src, dst, kernel=k, cin=c, cout=cout, c0=c0, tf32_out=tf32_out))
        return dst

    def pool(name, src, k, s) -> int:
        t, h, w, c = bufs[src]
        dst = new((*(same_padding(n, kk, ss)[2] for n, kk, ss in zip((t, h, w), k, s)), c))
        steps.append(_Step("pool", name, src, dst, kernel=k, stride=s))
        return dst

    t1, h1 = same_padding(T, 7, 2)[2], same_padding(I3D_SIZE, 7, 2)[2]
    packed = new((t1 + 2, h1, h1, I3D_STEM_CHANNELS))
    steps.append(_Step("stem", "Conv3d_1a_7x7", 0, packed))
    x = conv("Conv3d_1a_7x7", packed, 64, (3, 1, 1), new((t1, h1, h1, 64)))
    x = pool("MaxPool3d_2a_3x3", x, *_TRUNK_POOLS["MaxPool3d_2a_3x3"])
    x = conv("Conv3d_2b_1x1", x, 64, (1, 1, 1))
    x = conv("Conv3d_2c_3x3", x, 192, (3, 3, 3))
    x = pool("MaxPool3d_3a_3x3", x, *_TRUNK_POOLS["MaxPool3d_3a_3x3"])
    for block in _BLOCKS:
        if isinstance(block, str):
            x = pool(block, x, *_TRUNK_POOLS[block])
            continue
        name, o = block
        tf32_out = name != "Mixed_5c"   # the head reads Mixed_5c as data
        t, h, w, _ = bufs[x]
        y = new((t, h, w, o[0] + o[2] + o[4] + o[5]))
        conv(f"{name}.b0", x, o[0], (1, 1, 1), y, 0, tf32_out)
        conv(f"{name}.b1b", conv(f"{name}.b1a", x, o[1], (1, 1, 1)), o[2], (3, 3, 3), y, o[0], tf32_out)
        conv(f"{name}.b2b", conv(f"{name}.b2a", x, o[3], (1, 1, 1)), o[4], (3, 3, 3), y, o[0] + o[2], tf32_out)
        conv(f"{name}.b3b", pool(f"{name}.b3a", x, (3, 3, 3), (1, 1, 1)), o[5], (1, 1, 1), y, o[0] + o[2] + o[4],
             tf32_out)
        x = y
    steps.append(_Step("head", "logits", x, -1))
    return _Plan(tuple(steps), tuple(bufs))


_PLAN16 = i3d_plan(16)
I3D_LAUNCHES = len(_PLAN16.steps)   # per group of clips: the stem packing, 57 convolutions, 13 max pools, the head
# (name, Cin, Cout, kernel) of the 57 Unit3D as the state dict holds them, in order (the stem: 3 -> 64, 7 x 7 x 7)
I3D_UNITS = tuple((s.name, 3, s.cout, (7, 7, 7)) if s.name == "Conv3d_1a_7x7" else (s.name, s.cin, s.cout, s.kernel)
                  for s in _PLAN16.steps if s.op == "conv")


def _check_frames_count(T: int, who: str) -> None:
    if T < I3D_MIN_FRAMES:
        raise ValueError(f"{who}: I3D needs clips of at least {I3D_MIN_FRAMES} frames (Mixed_5c must keep 2 temporal "
                         f"positions for the [2, 7, 7] average pool); got {T}")


def _tensor(sd: dict, key: str, shape) -> torch.Tensor:
    """sd[key] as a float64 host tensor of `shape` (None: any 1-d or more); ValueError naming the key otherwise."""
    if key not in sd:
        raise ValueError(f"I3D.from_state_dict: missing key {key!r}")
    v = sd[key]
    v = v.detach() if isinstance(v, torch.Tensor) else torch.as_tensor(v)
    if shape is not None and tuple(v.shape) != tuple(shape):
        raise ValueError(f"I3D.from_state_dict: {key!r} has shape {tuple(v.shape)}, expected {tuple(shape)}")
    if not v.is_floating_point():
        raise ValueError(f"I3D.from_state_dict: {key!r} is {v.dtype}, expected a floating-point tensor")
    v = v.to("cpu", torch.float64)
    if not torch.isfinite(v).all():
        raise ValueError(f"I3D.from_state_dict: {key!r} has non-finite values")
    return v


def fold_bn(w: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, mean: torch.Tensor, var: torch.Tensor,
            eps: float = I3D_BN_EPS) -> tuple:
    """conv3d (no bias) then eval-mode BatchNorm3d as one convolution with bias, in the inputs' precision:
    w' = w * gamma / sqrt(var + eps), b' = beta - mean * gamma / sqrt(var + eps)."""
    scale = gamma / torch.sqrt(var + eps)
    return w * scale.reshape(-1, *([1] * (w.dim() - 1))), beta - mean * scale


def i3d_weights(sd: dict) -> tuple:
    """The checked, BN-folded weights of ``I3D.from_state_dict`` on the host in float64: ({name: (w [Cout, Cin, kt, kh,
    kw], b [Cout])} of the 57 Unit3D, (w [K, 1024], b [K]) of the logits)."""
    units = {}
    for name, cin, cout, k in I3D_UNITS:
        w = _tensor(sd, f"{name}.conv3d.weight", (cout, cin, *k))
        bn = [_tensor(sd, f"{name}.bn.{p}", (cout,)) for p in ("weight", "bias", "running_mean", "running_var")]
        if not (bn[3] + I3D_BN_EPS > 0).all():
            raise ValueError(f"I3D.from_state_dict: {name + '.bn.running_var'!r} + eps must be > 0")
        units[name] = fold_bn(w, *bn)
    key = "logits.conv3d.weight"
    w = _tensor(sd, key, None)
    if w.dim() != 5 or w.shape[0] < 1 or tuple(w.shape[1:]) != (I3D_FEATURES, 1, 1, 1):
        raise ValueError(f"I3D.from_state_dict: {key!r} has shape {tuple(w.shape)}, expected (K, {I3D_FEATURES}, 1, 1, 1)")
    b = _tensor(sd, "logits.conv3d.bias", (w.shape[0],))
    return units, (w.reshape(w.shape[0], I3D_FEATURES), b)


def round_tf32(v: torch.Tensor) -> torch.Tensor:
    """float64 -> the nearest TF32 value (10 explicit mantissa bits, ties to even) as float32: one rounding."""
    m, e = torch.frexp(v.double())
    return torch.ldexp(torch.round(m * 2048.0) / 2048.0, e.double()).float()


def stem_weight(w: torch.Tensor) -> torch.Tensor:
    """Conv3d_1a_7x7's weight [64, 3, 7, 7, 7] as the 3 x 1 x 1 convolution over cvvae_i3d_stem_input's 448 channels:
    [64, 448, 3, 1, 1], tap k channel ((j * 7 + kh) * 7 + kw) * 3 + c = w[:, c, 2k + j, kh, kw] for the temporal taps
    tap k carries (k = 0: j = 0, 1, 2; k = 1, 2: j = 1, 2), zero elsewhere."""
    out = torch.zeros((w.shape[0], I3D_STEM_CHANNELS, 3), dtype=w.dtype)
    for k in range(3):
        for j in range(0 if k == 0 else 1, 3):
            out[:, j * 147:(j + 1) * 147, k] = w[:, :, 2 * k + j].permute(0, 2, 3, 1).reshape(w.shape[0], 147)
    return out[..., None, None]


class I3D:
    """The Kinetics-400 I3D of FVD on the GPU; the module docstring has the definition.  Build it with
    ``I3D.from_state_dict``; ``i3d(clips)`` takes CUDA uint8 ``[N, T, H, W, 3]`` on ``i3d.device`` (T >= 9, any size)
    and returns float64 ``[N, K]`` on the host (K = 400 for Kinetics-400).

    Clips are prepared one launch each, then run in groups whose activations stay within ``I3D_GROUP_BYTES``
    (``i3d.group(T)`` clips); each group is ``i3d.launches`` kernel launches on the current stream of the device.  A clip's
    embedding is the same, bit for bit, whatever the grouping and whatever other clips share its call."""

    launches = I3D_LAUNCHES

    def __init__(self, units: dict, logits: tuple, device: torch.device):   # as i3d_weights returns them
        from .ops import CudaOps
        self._ops = CudaOps()
        self._units = {}
        for name, (w, b) in units.items():
            w = round_tf32(stem_weight(w) if name == "Conv3d_1a_7x7" else w)
            self._units[name] = (self._ops.pack_weight(w.to(device).contiguous()), b.float().to(device))
        self._logits = tuple(v.float().contiguous().to(device) for v in logits)   # fp32 [K, 1024], [K]
        self.classes = logits[0].shape[0]
        self.device = device
        self._group_bytes = I3D_GROUP_BYTES

    @classmethod
    def from_state_dict(cls, sd: dict, device=None) -> "I3D":
        """Weights from the PyTorch port's state dict: ``{unit}.conv3d.weight`` and ``{unit}.bn.{weight, bias,
        running_mean, running_var}`` of every Unit3D (``Conv3d_1a_7x7``, ``Conv3d_2b_1x1``, ``Conv3d_2c_3x3``,
        ``Mixed_3b.b0`` / ``.b1a`` / ``.b1b`` / ``.b2a`` / ``.b2b`` / ``.b3b`` .. ``Mixed_5c.*``), ``logits.conv3d.weight``
        ``[K, 1024, 1, 1, 1]`` and ``logits.conv3d.bias``; ``num_batches_tracked`` and every other key are ignored.  A
        missing key, a wrong shape, a non-float or non-finite value or ``running_var + 1e-3 <= 0`` raises ValueError
        naming the key.  `device`: a CUDA device (default: the current one).  Nothing is downloaded."""
        units, logits = i3d_weights(sd)
        dev = torch.device(device) if device is not None else None
        if dev is not None and dev.type != "cuda":
            raise ValueError(f"I3D.from_state_dict: the device must be a CUDA device, got {dev}")
        if dev is None or dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        return cls(units, logits, dev)

    def group(self, T: int) -> int:
        """Clips per group at T frames: the budget over one clip's largest live activations in the plan."""
        return max(1, self._group_bytes // i3d_plan(T).clip_bytes())

    def _check(self, clips: torch.Tensor, who: str) -> None:
        if (not isinstance(clips, torch.Tensor) or clips.dtype != torch.uint8 or clips.dim() != 5 or clips.shape[-1] != 3
                or not clips.is_cuda):
            raise ValueError(f"{who} expects a CUDA uint8 tensor [N, T, H, W, 3]; got {getattr(clips, 'dtype', type(clips))} "
                             f"{tuple(getattr(clips, 'shape', ()))} on {getattr(clips, 'device', 'the host')}")
        if clips.device != self.device:
            raise ValueError(f"{who}: the clips are on {clips.device}, the weights on {self.device}")
        _check_frames_count(clips.shape[1], who)

    def __call__(self, clips: torch.Tensor) -> torch.Tensor:
        from .video_io import frames_to_training_input
        self._check(clips, "I3D")
        N, T = clips.shape[:2]
        x = torch.empty((N, 3, T, I3D_SIZE, I3D_SIZE), dtype=torch.float32, device=self.device)
        for i in range(N):
            frames_to_training_input(clips[i], I3D_SIZE, "short", torch.float32, out=x[i:i + 1])
        return self._embed(x).cpu()

    @L._on_tensor_device
    def _embed(self, x: torch.Tensor) -> torch.Tensor:
        """Prepared clips, fp32 [N, 3, T, 224, 224] on the device -> their embeddings, float64 [N, K] on the device."""
        N, T = x.shape[0], x.shape[2]
        out = torch.empty((N, self.classes), dtype=torch.float64, device=x.device)
        plan, g = i3d_plan(T), self.group(T)
        for n0 in range(0, N, g):
            self._run_group(plan, x[n0:n0 + g], out[n0:n0 + g])
        return out

    def _run_group(self, plan: _Plan, x: torch.Tensor, out: torch.Tensor) -> None:
        """The plan on one group of prepared clips.  A buffer is allocated at its first write and dropped after its
        last read, so only what later steps read stays alive."""
        G = x.shape[0]
        lib, stream, dev = self._ops.lib, L._stream(x), x.device
        last = [b for _, b in plan.lifetimes()]
        bufs = {0: x}
        for i, s in enumerate(plan.steps):
            if s.dst >= 0 and s.dst not in bufs:
                bufs[s.dst] = torch.empty((G, *plan.buffers[s.dst]), dtype=torch.float32, device=dev)
            src = bufs[s.src]
            if s.op == "stem":
                L.check(lib.cvvae_i3d_stem_input(src.data_ptr(), G, *src.shape[2:], bufs[s.dst].data_ptr(), stream),
                        "cvvae_i3d_stem_input")
            elif s.op == "conv":
                w, b = self._units[s.name]
                y = bufs[s.dst][..., s.c0:s.c0 + s.cout]
                # SAME at stride 1 pads (k - 1) // 2 in front; the packed stem input already holds its padding
                offset = (0, 0, 0) if s.src == 1 else tuple(-((k - 1) // 2) for k in s.kernel)
                self._ops.conv(src, w, b, kernel=s.kernel, offset=offset, out=y, relu=True, tf32_out=s.tf32_out,
                               force="tc")
            elif s.op == "pool":
                k, st = (ctypes.c_int32 * 3)(*s.kernel), (ctypes.c_int32 * 3)(*s.stride)
                L.check(lib.cvvae_i3d_max_pool3d(src.data_ptr(), G, *src.shape[1:], k, st, bufs[s.dst].data_ptr(), stream),
                        "cvvae_i3d_max_pool3d")
            else:
                w, b = self._logits
                L.check(lib.cvvae_i3d_head(src.data_ptr(), G, *src.shape[1:], w.data_ptr(), b.data_ptr(), self.classes,
                                           out.data_ptr(), stream), "cvvae_i3d_head")
            for n, end in enumerate(last):
                if end == i and n in bufs and n != 0:
                    del bufs[n]


def frechet_distance(a, b) -> float:
    """The Fréchet distance between Gaussians fitted to two sets of embeddings, a Python float.  `a` and `b` are float64
    ``[N, D]`` host arrays or tensors (N >= 2 each, equal D), e.g. the I3D embeddings of real and of generated or
    reconstructed clips (FVD):

        mu = mean over rows, Sigma = np.cov(rowvar=False) (divisor N - 1)
        s = scipy.linalg.sqrtm(Sigma_a @ Sigma_b)
        FVD = real(|mu_a - mu_b|^2 + tr(Sigma_a + Sigma_b - 2 s))

    which is the formula of StyleGAN-V / StyleGAN2-ADA (they call ``sqrtm(..., disp=False)``; the matrix is the same).
    Host float64: a D x D matrix square root is not GPU work.  Mismatched D, N < 2, a non-float64 or non-finite input
    raises ValueError."""
    import numpy as np
    import scipy.linalg

    def rows(v, name):
        v = v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
        if v.dtype != np.float64 or v.ndim != 2 or v.shape[0] < 2 or v.shape[1] < 1:
            raise ValueError(f"frechet_distance expects float64 [N, D] with N >= 2; `{name}` is {v.dtype} {v.shape}")
        if not np.isfinite(v).all():
            raise ValueError(f"frechet_distance: `{name}` has non-finite values")
        return v

    a, b = rows(a, "a"), rows(b, "b")
    if a.shape[1] != b.shape[1]:
        raise ValueError(f"frechet_distance: `a` has D = {a.shape[1]}, `b` has D = {b.shape[1]}")
    mu_a, mu_b = a.mean(axis=0), b.mean(axis=0)
    sa, sb = np.atleast_2d(np.cov(a, rowvar=False)), np.atleast_2d(np.cov(b, rowvar=False))
    s = scipy.linalg.sqrtm(sa @ sb)
    return float(np.real(np.sum((mu_a - mu_b) ** 2) + np.trace(sa + sb - 2.0 * s)))

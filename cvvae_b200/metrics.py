"""Reconstruction quality on the GPU: per-frame PSNR, SSIM, multi-scale SSIM and LPIPS of two uint8 videos.

    frame_metrics(a, b)  ->  FrameMetrics(psnr, ssim, sse), host tensors with one entry per frame
    frame_ms_ssim(a, b)  ->  float64 host tensor with one MS-SSIM per frame
    LPIPS.from_state_dict(*state_dicts)(a, b)  ->  float64 host tensor with one LPIPS per frame
    ssim_map(a, b), LPIPS.map(a, b)  ->  where they differ: per-position maps on the device (see the end)

`a` and `b` are CUDA uint8 tensors [T, H, W, 3]: typically the frames the network saw (after the script's resize,
cvvae_inference_video.py:28) and the frames it gave back (:47-50).  One kernel (`csrc/metrics.cu`) reads both once and
leaves two 64-bit integers per frame: the exact sum of squared differences over the whole frame, and the sum of the
per-position SSIM values in units of 2^-32.  The scores are derived from them on the host in float64:

    psnr = 10 log10(255^2 * 3HW / sse)                      (+inf for identical frames)
    ssim = mean over channels and the positions whose 11 x 11 window lies inside the frame of
           (2 mu_a mu_b + C1)(2 s_ab + C2) / ((mu_a^2 + mu_b^2 + C1)(s_a^2 + s_b^2 + C2))

with Gaussian window weights (sigma 1.5), population (co)variances, C1 = (0.01 * 255)^2, C2 = (0.03 * 255)^2: Wang et
al. 2004 as the common libraries evaluate it (Gaussian weights, data range 255, 5-pixel border cropped, channels
averaged).  Integer accumulation makes the results bit-reproducible and independent of how the frames are batched.

MS-SSIM (Wang, Simoncelli and Bovik 2003) scores the same comparison at five scales, so that it also sees errors coarser
than the 11-pixel window: level 0 is the frames, level j+1 the 2 x 2 average pool of level j (an odd extent zero-padded
in front: ``F.avg_pool2d(x, 2, padding=(H % 2, W % 2))``).  At level j, per channel c and over the valid positions,

    cs_j(c) = mean of (2 s_ab + C2) / (s_a^2 + s_b^2 + C2),   s_j(c) = mean of the SSIM above   (data range 255 throughout)
    ms(c) = prod_{j<4} max(cs_j(c), 0)^w_j * max(s_4(c), 0)^w_4,   w = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)

and the frame's MS-SSIM is the mean of ms(c) over the three channels.  That is ``pytorch_msssim.ms_ssim(X, Y,
data_range=255, size_average=False)`` on [T, 3, H, W]; torchmetrics' MS-SSIM differs in two places: it floors odd sizes
instead of padding, and it averages the channels before taking the product.  Level 4 must hold the window, so frames
need at least 161 px on each side.  The pooled levels are kept as exact integer sums on the device, and one scoring
kernel per level leaves the sums of cs and SSIM per channel in units of 2^-32; the product is taken on the host in float64.

LPIPS (Zhang et al. 2018; the VGG16 variant, lpips v0.1) is the learned perceptual distance the reference adds to its
reconstruction loss, per frame.  Per frame pair: s = ((frame / 127.5 - 1) - shift) / scale (fp32, shift = (-0.030,
-0.088, -0.188), scale = (0.458, 0.448, 0.450)); VGG16 ``features[0:30]``, thirteen 3 x 3 convolutions (zero padding 1)
each followed by ReLU, with a 2 x 2 max pool after convolutions 2, 4, 7 and 10; at the five taps relu1_2 .. relu5_3
(C = 64, 128, 256, 512, 512), f^ = f / (sqrt(sum_c f^2 + 1e-10) + 1e-10) and d_k = mean over positions of
sum_c w_k[c] (f^_a - f^_b)^2 with the 1 x 1 head lin{k}; LPIPS = sum_k d_k.  The convolutions run on the tensor-core
convolution with fp32 activations and TF32 products, which is how PyTorch computes an fp32 LPIPS on this GPU by default
(cuDNN with TF32 on); every activation that only a convolution reads is stored rounded to the nearest TF32 value, the
taps stay fp32.  The normalisation and the weighted difference are fp64 and their per-frame sums integer fixed
point, so results are bit-reproducible, independent of how frames are grouped, exactly 0 for identical frames and
symmetric in a and b.  Frames need at least 16 x 16 px (relu5_3 is H/16 x W/16) and at most 2^23 px (the range of the
fixed-point sums).  No weights ship with the package:
``LPIPS.from_state_dict`` takes torchvision's VGG16 state dict (or the reference module's) and the lpips heads.

``LPIPS.from_state_dict(..., net='alex')`` is the same metric on AlexNet features, the lpips package's default network
(``lpips.LPIPS()``, and the LPIPS column of most published reconstruction tables; the two networks give different
numbers).  Only the trunk differs: torchvision's ``alexnet().features[0:12]``, i.e. conv1 (11 x 11, stride 4, padding 2)
-> relu1, a 3 x 3 stride-2 max pool (floor), conv2 (5 x 5, padding 2) -> relu2, the same pool, conv3 .. conv5 (3 x 3,
padding 1) -> relu3 .. relu5, with C = 64, 192, 384, 256, 256 at the taps (``features[12]``, the last pool, is not
part of LPIPS).  conv1 and conv2 run as 1 x 1 tensor-core convolutions over their taps packed into channels; the taps
are h1 = (H - 7) // 4 + 1, p1 = (h1 - 3) // 2 + 1 for relu2, p2 = (p1 - 3) // 2 + 1 for relu3 .. relu5 (likewise W), so
frames need at least 31 x 31 px.

Maps say where two frames differ, not only how much:

    ssim_map(a, b)  ->  CUDA float32 [T, H - 10, W - 10, 3], entry [t, y, x, c] the SSIM of channel c at pixel (y+5, x+5)
    LPIPS.map(a, b)  ->  CUDA float32 [T, H, W], lpips' ``spatial=True``

The SSIM map is written by the map instantiation of the PSNR / SSIM kernel: its entries are the fp32 values whose sum (in
units of 2^-32) is the frame's SSIM, and the same launch leaves the same sums bit for bit.  The LPIPS map is each tap's
head output sum_c w_k[c] (f^_a - f^_b)^2 per position (fp64), upsampled to H x W as ``nn.Upsample(size=(H, W),
mode="bilinear", align_corners=False)`` upsamples an fp32 tensor, summed over the five taps in fp64 and rounded to fp32
once.  Its mean is not exactly the scalar LPIPS (bilinear upsampling with clamped edges does not preserve the mean; the
same holds for lpips).  Both are bit-reproducible and independent of how frames are grouped.
"""
from __future__ import annotations

import ctypes
import functools
from types import SimpleNamespace
from typing import NamedTuple, Optional

import torch

from . import _lib as L

_WINDOW = 11
MS_SSIM_WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)
MS_SSIM_MIN_SIZE = 161
MS_SSIM_LAUNCHES = 9          # per call: five levels scored, four pooling steps
LPIPS_MIN_SIZE = 16
LPIPS_ALEX_MIN_SIZE = 31      # AlexNet: relu3 .. relu5 have (p1 - 3) // 2 + 1 >= 1 rows, p1 = ((H - 7) // 4 - 2) // 2 + 1
LPIPS_MAX_POSITIONS = 1 << 23   # H * W: the range of the tap kernel's fixed-point sums (include/cvvae_b200.h)
LPIPS_GROUP_BYTES = 8 << 30   # device bytes of activations one group may take: one frame pair at the largest size
LPIPS_SHIFT = (-0.030, -0.088, -0.188)
LPIPS_SCALE = (0.458, 0.448, 0.450)
LPIPS_MAX_HEAD = 32.0         # |w| bound of the heads that keeps the tap kernel's fixed-point sums in range


class FrameMetrics(NamedTuple):
    psnr: torch.Tensor   # float64 [T], dB
    ssim: torch.Tensor   # float64 [T]
    sse: torch.Tensor    # int64 [T], sum of squared differences over the frame


@L._on_tensor_device
def _launch(a: torch.Tensor, b: torch.Tensor, maps: bool = False):
    """The kernel on the current stream of the frames' device: int64 [T, 2] (sse, sum of ssim * 2^32), on the device.
    `maps`: the map instantiation of the same kernel, one launch, which also leaves the SSIM map: (sums, map fp32
    [T, H - 10, W - 10, 3])."""
    T, H, W, _ = a.shape
    acc = torch.empty((T, 2), dtype=torch.int64, device=a.device)
    if not maps:
        L.check(L.load().cvvae_frame_metrics(a.data_ptr(), b.data_ptr(), T, H, W, acc.data_ptr(), L._stream(a)),
                "cvvae_frame_metrics")
        return acc
    out = torch.empty((T, H - _WINDOW + 1, W - _WINDOW + 1, 3), dtype=torch.float32, device=a.device)
    L.check(L.load().cvvae_frame_ssim_map(a.data_ptr(), b.data_ptr(), T, H, W, acc.data_ptr(), out.data_ptr(), L._stream(a)),
            "cvvae_frame_ssim_map")
    return acc, out


def _scores(acc: torch.Tensor, H: int, W: int) -> FrameMetrics:
    """Host int64 [T, 2] of the kernel -> scores."""
    sse = acc[:, 0].clone()
    psnr = 10.0 * torch.log10((65025.0 * 3 * H * W) / sse.double())
    ssim = acc[:, 1].double() / 4294967296.0 / (3 * (H - _WINDOW + 1) * (W - _WINDOW + 1))
    return FrameMetrics(psnr, ssim, sse)


def _check_frames(a: torch.Tensor, b: torch.Tensor, who: str) -> None:
    for name, x in (("a", a), ("b", b)):
        if not isinstance(x, torch.Tensor) or x.dtype != torch.uint8 or x.dim() != 4 or x.shape[-1] != 3 or not x.is_cuda:
            raise ValueError(f"{who} expects CUDA uint8 tensors [T, H, W, 3]; `{name}` is "
                             f"{getattr(x, 'dtype', type(x))} {tuple(getattr(x, 'shape', ()))} on {getattr(x, 'device', 'the host')}")
    if a.shape != b.shape or a.device != b.device:
        raise ValueError(f"{who}: `a` and `b` differ: {tuple(a.shape)} on {a.device} vs {tuple(b.shape)} on {b.device}")


# A scorer is a metric as evaluate_frames runs it on every piece, and _sums for the per-frame functions (LPIPS is one):
#   _check(H, W, who)     refuses a frame size before any device work (ValueError naming `who`)
#   _launch(a, b)         the kernels on the frames' device and current stream: the int64 sums, on the device; or
#                         (sums, *maps) for a scorer that also leaves maps, device tensors a piece carries as they are
#   _finish(sums, H, W)   those sums on the host -> the float64 [T] tensors a piece of evaluate_frames carries
#   _empty                the host sums of no frames
# _with_maps(scorer) is the scorer whose _launch(a, b, maps=True) leaves its maps too.


def _with_maps(scorer):
    return SimpleNamespace(_check=scorer._check, _launch=functools.partial(scorer._launch, maps=True),
                           _finish=scorer._finish, _empty=scorer._empty)


def _sums(metric, a: torch.Tensor, b: torch.Tensor, who: str) -> torch.Tensor:
    """`metric`'s size refusal, then its sums of the checked frames `a` and `b`, on the host (no frames: no device work)."""
    T, H, W, _ = a.shape
    metric._check(H, W, who)
    return metric._launch(a.contiguous(), b.contiguous()).cpu() if T else metric._empty


def _check_ssim_size(H: int, W: int, who: str) -> None:
    if H < _WINDOW or W < _WINDOW:
        raise ValueError(f"{who}: SSIM needs frames of at least {_WINDOW} x {_WINDOW} px; got {H} x {W}")


def frame_metrics(a: torch.Tensor, b: torch.Tensor) -> FrameMetrics:
    """PSNR, SSIM and squared error of every frame of `b` against the same frame of `a` (both CUDA uint8 [T, H, W, 3])."""
    _check_frames(a, b, "frame_metrics")
    _, H, W, _ = a.shape
    _check_ssim_size(H, W, "frame_metrics")
    return _scores(_sums(_PSNR_SSIM, a, b, "frame_metrics"), H, W)


def ssim_map(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """The SSIM map of every frame of `b` against the same frame of `a` (both CUDA uint8 [T, H, W, 3], H, W >= 11): CUDA
    float32 [T, H - 10, W - 10, 3] on the frames' device, entry [t, y, x, c] the SSIM of channel c under the 11 x 11
    window centred on pixel (y + 5, x + 5).  Each entry is the fp32 value ``frame_metrics`` rounds to 2^-32 and sums, so
    the frame's SSIM is the mean of the map up to that rounding.  One kernel launch."""
    _check_frames(a, b, "ssim_map")
    T, H, W, _ = a.shape
    _check_ssim_size(H, W, "ssim_map")
    if not T:
        return torch.empty((0, H - _WINDOW + 1, W - _WINDOW + 1, 3), dtype=torch.float32, device=a.device)
    return _launch(a.contiguous(), b.contiguous(), maps=True)[1]


# evaluate_frames refuses no size for PSNR / SSIM on arrival: frame_metrics checks the 11 px itself, and in the stream
# the kernel's entry point refuses smaller frames at the launch
_PSNR_SSIM = SimpleNamespace(_check=lambda H, W, who: None, _launch=_launch,
                             _finish=lambda sums, H, W: _scores(sums, H, W)[:2], _empty=torch.empty((0, 2), dtype=torch.int64))


def _check_ms_ssim_size(H: int, W: int, who: str) -> None:
    if min(H, W) < MS_SSIM_MIN_SIZE:
        raise ValueError(f"{who}: MS-SSIM needs frames of at least {MS_SSIM_MIN_SIZE} x {MS_SSIM_MIN_SIZE} px (its coarsest "
                         f"of 5 levels, 1/16 of the size, must hold the 11 x 11 window); got {H} x {W}")


@L._on_tensor_device
def _launch_ms_ssim(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """The MS-SSIM kernels on the current stream of the frames' device: int64 [T, 5, 3, 2] (per level and channel, the
    sums of cs and of SSIM times 2^32), on the device.  The pooled levels live in a workspace freed on return."""
    T, H, W, _ = a.shape
    lib = L.load()
    n = lib.cvvae_ms_ssim_workspace_bytes(T, H, W)
    if n < 0:
        L.check(n, "cvvae_ms_ssim_workspace_bytes")
    workspace = torch.empty(n, dtype=torch.uint8, device=a.device)
    acc = torch.empty((T, len(MS_SSIM_WEIGHTS), 3, 2), dtype=torch.int64, device=a.device)
    L.check(lib.cvvae_frame_ms_ssim(a.data_ptr(), b.data_ptr(), T, H, W, workspace.data_ptr(), acc.data_ptr(), L._stream(a)),
            "cvvae_frame_ms_ssim")
    return acc


def _ms_ssim_levels(H: int, W: int) -> list:
    """(h, w) of the five levels: each is the previous one halved, rounded up."""
    sizes = [(H, W)]
    for _ in MS_SSIM_WEIGHTS[1:]:
        h, w = sizes[-1]
        sizes.append(((h + 1) // 2, (w + 1) // 2))
    return sizes


def _ms_ssim_scores(acc: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """Host int64 [T, 5, 3, 2] of the kernels -> MS-SSIM, float64 [T]."""
    n = torch.tensor([(h - _WINDOW + 1) * (w - _WINDOW + 1) for h, w in _ms_ssim_levels(H, W)], dtype=torch.float64)
    means = acc.double() / 4294967296.0 / n[:, None, None]          # [T, 5, 3, 2]: cs_j(c), s_j(c)
    w = torch.tensor(MS_SSIM_WEIGHTS, dtype=torch.float64)
    factors = torch.cat([means[:, :-1, :, 0], means[:, -1:, :, 1]], dim=1).clamp(min=0.0)   # [T, 5, 3]
    return factors.pow(w[:, None]).prod(dim=1).mean(dim=1)


_MS_SSIM = SimpleNamespace(_check=_check_ms_ssim_size, _launch=_launch_ms_ssim,
                           _finish=lambda sums, H, W: (_ms_ssim_scores(sums, H, W),),
                           _empty=torch.empty((0, len(MS_SSIM_WEIGHTS), 3, 2), dtype=torch.int64))


def frame_ms_ssim(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Multi-scale SSIM of every frame of `b` against the same frame of `a` (both CUDA uint8 [T, H, W, 3], H, W >= 161):
    float64 [T] on the host.  The module docstring has the definition."""
    _check_frames(a, b, "frame_ms_ssim")
    return _ms_ssim_scores(_sums(_MS_SSIM, a, b, "frame_ms_ssim"), a.shape[1], a.shape[2])


def _lpips_tap_sizes(H: int, W: int) -> list:
    """(h, w) of VGG16's five taps: each block after the first starts with a 2 x 2 max pool, floor."""
    return [(H >> k, W >> k) for k in range(5)]


def _lpips_alex_tap_sizes(H: int, W: int) -> list:
    """(h, w) of AlexNet's five taps: relu1 after conv1 (11 x 11, stride 4, padding 2), relu2 after a 3 x 3 stride-2 max
    pool (floor) and the 'same' conv2, relu3 .. relu5 after a second such pool and 'same' 3 x 3 convolutions."""
    def sizes(n: int) -> tuple:
        c1 = (n - 7) // 4 + 1
        p1 = (c1 - 3) // 2 + 1
        return c1, p1, (p1 - 3) // 2 + 1
    (h1, hp1, hp2), (w1, wp1, wp2) = sizes(H), sizes(W)
    return [(h1, w1), (hp1, wp1)] + [(hp2, wp2)] * 3


class _Conv(NamedTuple):
    """One convolution (then ReLU) of an LPIPS trunk.  `pack` None: 'same' 3 x 3; ``(order, Cp)``: 1 x 1 over its taps,
    which the step before packs into Cp channels, zero-padded, in (kh, kw, c) ("hwc") or (c, kh, kw) ("chw") order."""
    slice: int           # lpips' net.slice{slice + 1} holds it
    index: int           # its torchvision ``features`` index
    cin: int
    cout: int
    extent: int          # kernel extent
    pack: Optional[tuple] = None


class _LpipsNet(NamedTuple):
    """Everything that differs between the LPIPS networks.  `plan`: one kernel launch per step, each reading what the
    one before left: ("input", fn) packs the scaled frames for conv 0; ("conv", n, tf32_out) is conv n, its output
    rounded to TF32 if only a convolution reads it; ("tap", k, side) is tap k, also writing the 2 x 2 max pool ("pool2")
    or a TF32 copy ("copy") for the next convolution; ("max_pool3s2",); ("pack5x5",) packs 5 x 5 taps, (kh, kw, c)."""
    convs: tuple         # _Conv, in order
    channels: tuple      # C_k of the taps; their number sizes the accumulator
    tap_sizes: object    # (H, W) -> [(h, w)] of the taps
    min_size: int
    too_small: str       # the refusal of frames under min_size, formatted with who, n = min_size, H and W
    plan: tuple

    def shapes(self, H: int, W: int) -> list:
        """(h, w, C) of the activation each step of the plan leaves for the next, for H x W frames."""
        out, h, w, c = [], H, W, 3
        for op, *arg in self.plan:
            if op == "input":
                (h, w), c = self.tap_sizes(H, W)[0], self.convs[0].pack[1]
            elif op == "conv":
                c = self.convs[arg[0]].cout
            elif op == "tap" and arg[1] == "pool2":
                h, w = h // 2, w // 2
            elif op == "max_pool3s2":
                h, w = (h - 3) // 2 + 1, (w - 3) // 2 + 1
            elif op == "pack5x5":
                c *= 25
            out.append((h, w, c))
        return out

    def pair_bytes(self, H: int, W: int) -> int:
        """Device bytes of the largest activations live at once for a frame pair: a convolution's fp32 input and output."""
        shapes = self.shapes(H, W)
        return 2 * 4 * max((shapes[n - 1][2] + c) * h * w
                           for n, ((op, *_), (h, w, c)) in enumerate(zip(self.plan, shapes)) if op == "conv")


def _vgg16() -> _LpipsNet:
    """VGG16 ``features[0:30]``: lpips' five slices of 3 x 3 convolutions, each ending in a tap, 2 x 2 max pools between
    them.  conv1_1 runs as a 1 x 1 convolution over the 27 taps cvvae_lpips_input packs into 32 channels."""
    blocks = ((0, 2), (5, 7), (10, 12, 14), (17, 19, 21), (24, 26, 28))   # features indices of the convolutions
    channels = (64, 128, 256, 512, 512)
    convs, plan, cin = [], [("input", "cvvae_lpips_input")], 3
    for k, (block, c) in enumerate(zip(blocks, channels)):
        for j, i in enumerate(block):
            # a slice's last convolution is its tap, read as data in fp32; the others only feed the next convolution
            plan.append(("conv", len(convs), j + 1 < len(block)))
            convs.append(_Conv(k, i, cin, c, 3, None if convs else ("hwc", 32)))
            cin = c
        plan.append(("tap", k, "pool2" if k + 1 < len(blocks) else None))
    return _LpipsNet(tuple(convs), channels, _lpips_tap_sizes, LPIPS_MIN_SIZE,
                     "{who}: LPIPS needs frames of at least {n} x {n} px (its last tap, relu5_3, is 1/16 of the size); "
                     "got {H} x {W}", tuple(plan))


_VGG16 = _vgg16()
# AlexNet features[0:12], one convolution (a tap) per lpips slice.  conv1 and conv2 run as 1 x 1 convolutions over their
# taps packed into channels; relu3 and relu4 reach the next convolution through the tap kernel's TF32 copy.
_ALEXNET = _LpipsNet(
    convs=(_Conv(0, 0, 3, 64, 11, ("chw", 384)), _Conv(1, 3, 64, 192, 5, ("hwc", 1600)), _Conv(2, 6, 192, 384, 3),
           _Conv(3, 8, 384, 256, 3), _Conv(4, 10, 256, 256, 3)),
    channels=(64, 192, 384, 256, 256),
    tap_sizes=_lpips_alex_tap_sizes,
    min_size=LPIPS_ALEX_MIN_SIZE,
    too_small="{who}: LPIPS (AlexNet) needs frames of at least {n} x {n} px (its last taps, relu3 .. relu5, follow the "
              "stride-4 conv1 and two 3 x 3 stride-2 pools); got {H} x {W}",
    plan=(("input", "cvvae_lpips_alex_input"), ("conv", 0, False), ("tap", 0, None), ("max_pool3s2",), ("pack5x5",),
          ("conv", 1, False), ("tap", 1, None), ("max_pool3s2",), ("conv", 2, False), ("tap", 2, "copy"),
          ("conv", 3, False), ("tap", 3, "copy"), ("conv", 4, False), ("tap", 4, None)))
_NETS = {"vgg": _VGG16, "alex": _ALEXNET}
LPIPS_NETS = tuple(_NETS)
LPIPS_LAUNCHES = len(_VGG16.plan)          # per group of frames: the input kernel, 13 convolutions, 5 taps
LPIPS_ALEX_LAUNCHES = len(_ALEXNET.plan)   # the input kernel, 5 convolutions, 5 taps, 2 pools, conv2's packing


def _check_lpips_size(H: int, W: int, who: str, net: str = "vgg") -> None:
    spec = _NETS[net]
    if min(H, W) < spec.min_size:
        raise ValueError(spec.too_small.format(who=who, n=spec.min_size, H=H, W=W))
    if H * W > LPIPS_MAX_POSITIONS:
        raise ValueError(f"{who}: LPIPS takes frames of at most 2^23 px (the range of its fixed-point sums); got {H} x {W}")


def _lpips_scores(acc: torch.Tensor, H: int, W: int, net: str = "vgg") -> torch.Tensor:
    """Host int64 [5, T] of the tap kernels (per tap and frame, the sum over positions times 2^32) -> LPIPS, float64 [T]."""
    d = torch.zeros(acc.shape[1], dtype=torch.float64)
    for k, (h, w) in enumerate(_NETS[net].tap_sizes(H, W)):
        d += acc[k].double() / 4294967296.0 / (h * w)
    return d


def _lpips_weights(state_dicts: tuple, net: str = "vgg") -> tuple:
    """The checked weights of ``LPIPS.from_state_dict`` on the host, fp32: ([(weight, bias)] of the convolutions
    (VGG16: thirteen, AlexNet: five), [head [C_k]] of the five taps)."""
    sd: dict = {}
    for d in state_dicts:
        sd.update(d)

    def get(keys: tuple, shape: tuple) -> torch.Tensor:
        key = next((k for k in keys if k in sd), None)
        if key is None:
            raise ValueError(f"LPIPS.from_state_dict: missing key {keys[0]!r}" +
                             (f" (or {keys[1]!r})" if len(keys) > 1 else ""))
        v = sd[key]
        v = torch.as_tensor(v) if not isinstance(v, torch.Tensor) else v.detach()
        if tuple(v.shape) != shape:
            raise ValueError(f"LPIPS.from_state_dict: {key!r} has shape {tuple(v.shape)}, expected {shape}")
        if not v.is_floating_point():
            raise ValueError(f"LPIPS.from_state_dict: {key!r} is {v.dtype}, expected a floating-point tensor")
        v = v.to("cpu", torch.float32)
        if not torch.isfinite(v).all():
            raise ValueError(f"LPIPS.from_state_dict: {key!r} has non-finite values")
        return v

    for name, want in (("shift", LPIPS_SHIFT), ("scale", LPIPS_SCALE)):
        key = f"scaling_layer.{name}"
        if key in sd:
            v = get((key,), (1, 3, 1, 1))
            if not torch.equal(v.flatten(), torch.tensor(want, dtype=torch.float32)):
                raise ValueError(f"LPIPS.from_state_dict: {key!r} is {v.flatten().tolist()}, expected {list(want)}")
    convs = []
    for c in _NETS[net].convs:
        keys = lambda s: (f"features.{c.index}.{s}", f"net.slice{c.slice + 1}.{c.index}.{s}")   # noqa: E731
        convs.append((get(keys("weight"), (c.cout, c.cin, c.extent, c.extent)), get(keys("bias"), (c.cout,))))
    heads = []
    for k, c in enumerate(_NETS[net].channels):
        key = f"lin{k}.model.1.weight"
        v = get((key,), (1, c, 1, 1))
        if v.abs().max().item() > LPIPS_MAX_HEAD:
            raise ValueError(f"LPIPS.from_state_dict: {key!r} has |w| > {LPIPS_MAX_HEAD:g}, outside the range of the "
                             "fixed-point sums")
        heads.append(v.flatten())

    return convs, heads


def _conv_tc_weight(w: torch.Tensor, pack: Optional[tuple]) -> torch.Tensor:
    """A weight as conv_tc runs it (see _Conv): unchanged, or [Cout, Cp, 1, 1], the taps in the packing order, zeros after."""
    if pack is None:
        return w
    order, cp = pack
    taps = (w.permute(0, 2, 3, 1) if order == "hwc" else w).reshape(w.shape[0], -1)
    out = torch.zeros((w.shape[0], cp), dtype=torch.float32)
    out[:, :taps.shape[1]] = taps
    return out[:, :, None, None]


class LPIPS:
    """LPIPS (lpips v0.1, VGG16 or AlexNet features) of every frame of `b` against the same frame of `a` on the GPU; the
    module docstring has the definition.  Build it with ``LPIPS.from_state_dict``; ``metric(a, b)`` takes two CUDA uint8
    ``[T, H, W, 3]`` videos on ``metric.device`` (H, W >= ``metric.min_size``, H * W <= 2^23) and returns float64 ``[T]``
    on the host.  ``metric.net`` is ``'vgg'`` or ``'alex'``.

    Frames are scored in groups whose activations stay within ``LPIPS_GROUP_BYTES``; each group is ``metric.launches``
    kernel launches on the current stream of the device.  The result is the same, bit for bit, whatever the grouping."""

    net = "vgg"   # the network of an instance built without naming one

    def __init__(self, convs: list, heads: list, device: torch.device, net: str = "vgg"):   # as _lpips_weights returns them
        from .ops import CudaOps
        self._ops = CudaOps()
        self._convs = [(self._ops.pack_weight(_conv_tc_weight(w, c.pack).to(device).contiguous()), b.to(device))
                       for (w, b), c in zip(convs, _NETS[net].convs)]   # the weights as conv_tc reads them
        self._heads = [h.to(device) for h in heads]                      # fp32 [C_k] per tap
        self.device = device
        self.net = net
        self._group_bytes = LPIPS_GROUP_BYTES

    @property
    def min_size(self) -> int:
        """The smallest frame side the network accepts: 16 px for VGG16, 31 px for AlexNet."""
        return _NETS[self.net].min_size

    @property
    def launches(self) -> int:
        """Kernel launches per group of frames."""
        return len(_NETS[self.net].plan)

    @classmethod
    def from_state_dict(cls, *state_dicts, device=None, net: str = "vgg") -> "LPIPS":
        """Weights from one or more state dicts, merged (later ones win).  ``net="vgg"`` (the default): the thirteen
        convolutions under torchvision's keys ``features.{i}.weight`` / ``.bias`` (``vgg16-397923af.pth``) or the
        reference module's ``net.slice{k}.{i}.*`` (same i), the heads under ``lin{k}.model.1.weight`` ``[1, C_k, 1, 1]``
        (lpips v0.1 ``vgg.pth``, or the reference's ``LPIPS().state_dict()``).  ``net='alex'``, the lpips package's
        default network: the five convolutions ``features.{0,3,6,8,10}.*`` of torchvision's AlexNet
        (``alexnet-owt-7be5be79.pth``) or the lpips module's ``net.slice{k}.{i}.*``, and the heads of lpips v0.1
        ``alex.pth`` (C_k = 64, 192, 384, 256, 256).  ``scaling_layer.shift`` / ``.scale``, if present, must be the
        constants above; every other key is ignored.  A missing key, a wrong shape, a non-float or non-finite value, a
        head with |w| > 32 or an unknown `net` raises ValueError.  `device`: a CUDA device (default: the current one).
        The weights are packed once, the convolutions' rounded to TF32."""
        if net not in LPIPS_NETS:
            raise ValueError(f"LPIPS.from_state_dict: `net` must be one of {LPIPS_NETS}, got {net!r}")
        convs, heads = _lpips_weights(state_dicts, net)
        dev = torch.device(device) if device is not None else None
        if dev is not None and dev.type != "cuda":
            raise ValueError(f"LPIPS.from_state_dict: the device must be a CUDA device, got {dev}")
        if dev is None or dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device() if dev is None or dev.index is None else dev.index)
        return cls(convs, heads, dev, net)

    def _group(self, H: int, W: int, maps: bool = False) -> int:
        """Frames per group: the budget over a frame pair's largest live activations (VGG16: conv1_2's input and output;
        AlexNet: conv1's or conv2's), plus with `maps` the frame's fp64 tap maps and its fp32 map."""
        net = _NETS[self.net]
        per_frame = net.pair_bytes(H, W)
        if maps:
            per_frame += 8 * sum(h * w for h, w in net.tap_sizes(H, W)) + 4 * H * W
        return max(1, self._group_bytes // per_frame)

    def _check(self, H: int, W: int, who: str) -> None:
        _check_lpips_size(H, W, who, self.net)

    @L._on_tensor_device
    def _launch(self, a: torch.Tensor, b: torch.Tensor, maps: bool = False):
        """The kernels on the current stream of the frames' device: int64 [5, T] (per tap and frame, the sum over
        positions of the weighted squared difference times 2^32), on the device.  `maps`: the same sums and the LPIPS
        map, (sums, map fp32 [T, H, W]), from the same pass of the network."""
        T, H, W, _ = a.shape
        acc = torch.empty((len(_NETS[self.net].channels), T), dtype=torch.int64, device=a.device)
        out = torch.empty((T, H, W), dtype=torch.float32, device=a.device) if maps else None
        g = self._group(H, W, maps)
        for t0 in range(0, T, g):
            self._run_group(a[t0:t0 + g], b[t0:t0 + g], acc[:, t0:t0 + g], None if out is None else out[t0:t0 + g])
        return acc if out is None else (acc, out)

    def _finish(self, sums: torch.Tensor, H: int, W: int) -> tuple:
        return (_lpips_scores(sums, H, W, self.net),)

    @property
    def _empty(self) -> torch.Tensor:
        return torch.empty((len(_NETS[self.net].channels), 0), dtype=torch.int64)

    def _run_group(self, a: torch.Tensor, b: torch.Tensor, acc: torch.Tensor, out: Optional[torch.Tensor] = None) -> None:
        """The network's plan on one group of frame pairs, both videos as one batch of 2G images.  Only the activation
        the next step reads stays alive: each step's output replaces it, a tap without a side output leaves it.
        `out` (fp32 [G, H, W]): the taps also leave their maps, fp64 and back to back, and one launch after the plan
        upsamples and sums them into it."""
        G, H, W, _ = a.shape
        net, lib, stream = _NETS[self.net], self._ops.lib, L._stream(a)
        sizes = net.tap_sizes(H, W)
        if out is not None:
            taps = torch.empty(G * sum(h * w for h, w in sizes), dtype=torch.float64, device=a.device)
            offsets = [G * sum(h * w for h, w in sizes[:k]) for k in range(len(sizes))]
        x = None
        for (op, *arg), shape in zip(net.plan, net.shapes(H, W)):
            y = (None if op == "tap" and arg[1] is None else
                 torch.empty((2 * G, 1, *shape), dtype=torch.float32, device=a.device))
            if op == "input":
                L.check(getattr(lib, arg[0])(a.data_ptr(), b.data_ptr(), G, H, W, y.data_ptr(), stream), arg[0])
            elif op == "conv":
                (wp, bias), same3x3 = self._convs[arg[0]], net.convs[arg[0]].pack is None
                kw = dict(kernel=(1, 3, 3), offset=(0, -1, -1)) if same3x3 else {}
                self._ops.conv(x, wp, bias, out=y, relu=True, tf32_out=arg[1], **kw)
            elif op == "tap":
                k, side = arg
                y_ptr = None if y is None else y.data_ptr()
                args = (x.data_ptr(), G, *x.shape[2:], self._heads[k].data_ptr(), acc[k].data_ptr())
                if out is not None:
                    fn = "cvvae_lpips_tap_map"
                    sides = (None, y_ptr) if side == "copy" else (y_ptr, None)
                    L.check(lib.cvvae_lpips_tap_map(*args, *sides, taps[offsets[k]:].data_ptr(), stream), fn)
                else:
                    fn = "cvvae_lpips_tap_copy" if side == "copy" else "cvvae_lpips_tap"
                    L.check(getattr(lib, fn)(*args, y_ptr, stream), fn)
            else:   # max_pool3s2, pack5x5: image by image
                fn = "cvvae_lpips_" + op
                L.check(getattr(lib, fn)(x.data_ptr(), 2 * G, *x.shape[2:], y.data_ptr(), stream), fn)
            if y is not None:
                x = y
        if out is not None:
            hw = (ctypes.c_int32 * (2 * len(sizes)))(*(n for size in sizes for n in size))
            L.check(lib.cvvae_lpips_upsample_sum(taps.data_ptr(), G, H, W, hw, out.data_ptr(), stream),
                    "cvvae_lpips_upsample_sum")

    def map(self, a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
        """The LPIPS map of every frame of `b` against the same frame of `a`, lpips' ``spatial=True``: CUDA float32
        [T, H, W] on ``metric.device``, with the inputs and limits of ``metric(a, b)``.  Each tap's head output
        sum_c w_k[c] (f^_a - f^_b)^2 is kept per position (fp64), upsampled to H x W as ``nn.Upsample(size=(H, W),
        mode="bilinear", align_corners=False)`` does for fp32 tensors, and the five are summed in fp64 and rounded to
        fp32 once.  The map's mean is close to, but not exactly, the scalar LPIPS: bilinear upsampling with the edges
        clamped does not preserve the mean (lpips' spatial maps behave the same way).  One pass of the network gives both:
        ``metric.launches + 1`` launches per group of frames, and the map is the same, bit for bit, whatever the grouping."""
        _check_frames(a, b, "LPIPS.map")
        if a.device != self.device:
            raise ValueError(f"LPIPS.map: the frames are on {a.device}, the weights on {self.device}")
        T, H, W, _ = a.shape
        self._check(H, W, "LPIPS.map")
        if not T:
            return torch.empty((0, H, W), dtype=torch.float32, device=a.device)
        return self._launch(a.contiguous(), b.contiguous(), maps=True)[1]

    def __call__(self, a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
        _check_frames(a, b, "LPIPS")
        if a.device != self.device:
            raise ValueError(f"LPIPS: the frames are on {a.device}, the weights on {self.device}")
        return _lpips_scores(_sums(self, a, b, "LPIPS"), a.shape[1], a.shape[2], self.net)

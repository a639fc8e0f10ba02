"""LPIPS on AlexNet features (lpips v0.1, net='alex') restated from its definition with torch functional ops, in any
dtype and on any device, and seeded weights in torchvision's and the lpips module's state-dict layouts.  The scaling
layer, the normalisation and the heads are those of lpips_ref.py; only the trunk, ``alexnet().features[0:12]``, differs.
The tests compare the device kernels with it in fp64, and with the same restatement run in fp32 on the GPU (cuDNN with
TF32) to size the error of a TF32 evaluation."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from lpips_ref import SCALE, SHIFT, scaled_input, tap_distance, tf32

# alexnet.features index, Cin, Cout, kernel extent, stride, padding of the five convolutions; lpips' slice k holds the
# k-th of them with its ReLU, slices 2 and 3 start with a 3 x 3 stride-2 max pool
CONVS = ((0, 3, 64, 11, 4, 2), (3, 64, 192, 5, 1, 2), (6, 192, 384, 3, 1, 1), (8, 384, 256, 3, 1, 1), (10, 256, 256, 3, 1, 1))
CHANNELS = tuple(c[2] for c in CONVS)
SLICES = ((0, 2), (2, 5), (5, 8), (8, 10), (10, 12))   # lpips.pretrained_networks.alexnet: features[a:b] per slice


def make_state_dict(seed: int) -> dict:
    """torchvision's AlexNet feature keys plus the lpips heads: He-normal convolutions, small biases, non-negative heads."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for i, cin, cout, k, _, _ in CONVS:
        sd[f"features.{i}.weight"] = torch.randn((cout, cin, k, k), generator=g) * (2.0 / (k * k * cin)) ** 0.5
        sd[f"features.{i}.bias"] = torch.randn((cout,), generator=g) * 0.05
    for k, c in enumerate(CHANNELS):
        sd[f"lin{k}.model.1.weight"] = torch.rand((1, c, 1, 1), generator=g) * (4.0 / c)
    return sd


def to_lpips_layout(sd: dict) -> dict:
    """The same weights under the lpips module's keys (net.slice{k}.{i}.*), with its scaling layer."""
    out = {}
    for k, (i, *_) in enumerate(CONVS):
        for s in ("weight", "bias"):
            out[f"net.slice{k + 1}.{i}.{s}"] = sd[f"features.{i}.{s}"]
    for k in range(5):
        out[f"lin{k}.model.1.weight"] = sd[f"lin{k}.model.1.weight"]
    out["scaling_layer.shift"] = torch.tensor(SHIFT)[None, :, None, None]
    out["scaling_layer.scale"] = torch.tensor(SCALE)[None, :, None, None]
    return out


def taps(x: torch.Tensor, sd: dict, tf32_conv1: bool = False) -> list:
    """The five ReLU outputs relu1 .. relu5 of AlexNet features[0:12] on x [N, 3, H, W] (x's dtype and device).
    `tf32_conv1` (fp32 only): conv1's input and weights rounded to TF32 first, as a TF32 convolution reads them, in case
    cuDNN runs the 3-channel convolution in plain fp32."""
    out = []
    for k, (i, _, _, _, stride, pad) in enumerate(CONVS):
        if k in (1, 2):
            x = F.max_pool2d(x, 3, 2)
        w = sd[f"features.{i}.weight"].to(x)
        if tf32_conv1 and k == 0:
            x, w = tf32(x), tf32(w)
        x = F.relu(F.conv2d(x, w, sd[f"features.{i}.bias"].to(x), stride=stride, padding=pad))
        out.append(x)
    return out


def lpips(a: torch.Tensor, b: torch.Tensor, sd: dict, dtype=torch.float64, tf32_conv1: bool = False) -> torch.Tensor:
    """LPIPS (AlexNet) per frame of uint8 [T, H, W, 3] videos a, b on their device, evaluated in `dtype`: float64 [T] on
    the host."""
    T = a.shape[0]
    x = torch.cat([scaled_input(a), scaled_input(b)]).to(dtype)
    d = torch.zeros(T, dtype=torch.float64)
    for k, f in enumerate(taps(x, sd, tf32_conv1)):
        d += tap_distance(f, sd[f"lin{k}.model.1.weight"].flatten(), T).double().cpu()
    return d

"""LPIPS (VGG16, lpips v0.1) restated from its definition with torch functional ops, in any dtype and on any device,
and seeded weights in the real state-dict layout.  The tests compare the device kernels with it in fp64, and with the
same restatement run in fp32 on the GPU (cuDNN, TF32 on or off) to size the error of a TF32 evaluation."""
from __future__ import annotations

import torch
import torch.nn.functional as F

SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)
BLOCKS = ((0, 2), (5, 7), (10, 12, 14), (17, 19, 21), (24, 26, 28))   # vgg16.features indices of the convolutions
CHANNELS = (64, 128, 256, 512, 512)


def make_state_dict(seed: int) -> dict:
    """torchvision's VGG16 feature keys plus the lpips heads: He-normal convolutions, small biases, non-negative heads
    (lpips clamps its heads to w >= 0 while training)."""
    g = torch.Generator().manual_seed(seed)
    sd, cin = {}, 3
    for block, c in zip(BLOCKS, CHANNELS):
        for i in block:
            sd[f"features.{i}.weight"] = torch.randn((c, cin, 3, 3), generator=g) * (2.0 / (9 * cin)) ** 0.5
            sd[f"features.{i}.bias"] = torch.randn((c,), generator=g) * 0.05
            cin = c
    for k, c in enumerate(CHANNELS):
        sd[f"lin{k}.model.1.weight"] = torch.rand((1, c, 1, 1), generator=g) * (4.0 / c)
    return sd


def to_reference_layout(sd: dict) -> dict:
    """The same weights under the reference module's keys (net.slice{k}.{i}.*), with its scaling layer."""
    out = {}
    for k, block in enumerate(BLOCKS):
        for i in block:
            for s in ("weight", "bias"):
                out[f"net.slice{k + 1}.{i}.{s}"] = sd[f"features.{i}.{s}"]
    for k in range(5):
        out[f"lin{k}.model.1.weight"] = sd[f"lin{k}.model.1.weight"]
    out["scaling_layer.shift"] = torch.tensor(SHIFT)[None, :, None, None]
    out["scaling_layer.scale"] = torch.tensor(SCALE)[None, :, None, None]
    return out


def scaled_input(u8: torch.Tensor) -> torch.Tensor:
    """uint8 [T, H, W, 3] -> fp32 [T, 3, H, W]: (frame / 127.5 - 1 - shift) / scale, in fp32 as PyTorch evaluates it."""
    x = u8.permute(0, 3, 1, 2).float() / 127.5 - 1.0
    shift = torch.tensor(SHIFT, dtype=torch.float32, device=u8.device)[None, :, None, None]
    scale = torch.tensor(SCALE, dtype=torch.float32, device=u8.device)[None, :, None, None]
    return (x - shift) / scale


def tf32(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> the nearest TF32 value, ties to even, as the library rounds (common.cuh tf32_rn)."""
    u = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    u = torch.where((u & 0x7F800000) != 0x7F800000, u + 0xFFF + ((u >> 13) & 1), u) & 0xFFFFE000
    return torch.where(u >= 2 ** 31, u - 2 ** 32, u).to(torch.int32).view(torch.float32)


def taps(x: torch.Tensor, sd: dict, tf32_conv1_1: bool = False) -> list:
    """The five ReLU outputs relu1_2 .. relu5_3 of VGG16 features[0:30] on x [N, 3, H, W] (x's dtype and device).
    `tf32_conv1_1` (fp32 only): conv1_1's input and weights rounded to TF32 first, as a TF32 convolution reads them.
    cuDNN picks a plain fp32 kernel for this 3-channel convolution at small sizes even with TF32 allowed, and this makes
    the restatement a TF32 evaluation at every size."""
    out = []
    if tf32_conv1_1:
        x = tf32(x)
    for k, block in enumerate(BLOCKS):
        if k:
            x = F.max_pool2d(x, 2, 2)
        for i in block:
            w = sd[f"features.{i}.weight"].to(x)
            if tf32_conv1_1 and i == 0:
                w = tf32(w)
            b = sd[f"features.{i}.bias"].to(x)
            x = F.relu(F.conv2d(x, w, b, padding=1))
        out.append(x)
    return out


def tap_distance(f: torch.Tensor, w: torch.Tensor, T: int) -> torch.Tensor:
    """d_k per frame of one tap f [2T, C, h, w] (frames of a, then of b) with head w [C], in f's dtype."""
    n = torch.sqrt((f * f).sum(1, keepdim=True) + 1e-10)
    fh = f / (n + 1e-10)
    d = (fh[:T] - fh[T:]) ** 2
    return (d * w.to(f)[None, :, None, None]).sum(1).mean((1, 2))


def lpips(a: torch.Tensor, b: torch.Tensor, sd: dict, dtype=torch.float64, tf32_conv1_1: bool = False) -> torch.Tensor:
    """LPIPS per frame of uint8 [T, H, W, 3] videos a, b on their device, evaluated in `dtype`: float64 [T] on the host."""
    T = a.shape[0]
    x = torch.cat([scaled_input(a), scaled_input(b)]).to(dtype)
    d = torch.zeros(T, dtype=torch.float64)
    for k, f in enumerate(taps(x, sd, tf32_conv1_1)):
        d += tap_distance(f, sd[f"lin{k}.model.1.weight"].flatten(), T).double().cpu()
    return d

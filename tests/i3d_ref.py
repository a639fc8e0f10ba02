"""FVD's I3D restated in torch, from its definition (cvvae_b200/fvd.py, DESIGN §5c "FVD"), unfolded: every Unit3D is
F.pad (TF "SAME", zeros) + F.conv3d without bias + ``nn.BatchNorm3d(eps=1e-3).eval()`` + ReLU, every max pool F.pad +
F.max_pool3d, the head ``F.avg_pool3d([2, 7, 7], stride 1)`` + the logits convolution with bias + the mean over time.

``embed(x, sd)`` takes prepared clips [N, 3, T, 224, 224] (frames_to_training_input's output) and returns [N, K]:
  - in float64 (``tf32=False``), the accuracy reference;
  - with ``tf32=True``, PyTorch's default fp32 evaluation on the GPU (cuDNN with TF32 on), with the stem's operands
    rounded to TF32 by hand: cuDNN runs a 3-channel convolution in plain fp32, which no TF32 evaluation would.

``make_state_dict(seed)`` is a seeded state dict in the PyTorch port's layout: He-scaled weights and random BN
statistics that keep the activations O(1) through the 20 layers."""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

BLOCKS = {"Mixed_3b": (64, 96, 128, 16, 32, 32), "Mixed_3c": (128, 128, 192, 32, 96, 64),
          "Mixed_4b": (192, 96, 208, 16, 48, 64), "Mixed_4c": (160, 112, 224, 24, 64, 64),
          "Mixed_4d": (128, 128, 256, 24, 64, 64), "Mixed_4e": (112, 144, 288, 32, 64, 64),
          "Mixed_4f": (256, 160, 320, 32, 128, 128), "Mixed_5b": (256, 160, 320, 32, 128, 128),
          "Mixed_5c": (384, 192, 384, 48, 128, 128)}


def units():
    """(name, Cin, Cout, kernel) of every Unit3D, in order."""
    out = [("Conv3d_1a_7x7", 3, 64, (7, 7, 7)), ("Conv3d_2b_1x1", 64, 64, (1, 1, 1)), ("Conv3d_2c_3x3", 64, 192, (3, 3, 3))]
    cin = 192
    for name, o in BLOCKS.items():
        out += [(f"{name}.b0", cin, o[0], (1, 1, 1)), (f"{name}.b1a", cin, o[1], (1, 1, 1)),
                (f"{name}.b1b", o[1], o[2], (3, 3, 3)), (f"{name}.b2a", cin, o[3], (1, 1, 1)),
                (f"{name}.b2b", o[3], o[4], (3, 3, 3)), (f"{name}.b3b", cin, o[5], (1, 1, 1))]
        cin = o[0] + o[2] + o[4] + o[5]
    return out


def make_state_dict(seed: int, classes: int = 400) -> dict:
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, cin, cout, k in units():
        fan_in = cin * math.prod(k)
        sd[f"{name}.conv3d.weight"] = torch.randn((cout, cin, *k), generator=g) * math.sqrt(2.0 / fan_in)
        sd[f"{name}.bn.weight"] = 0.8 + 0.4 * torch.rand(cout, generator=g)
        sd[f"{name}.bn.bias"] = 0.1 * torch.randn(cout, generator=g)
        sd[f"{name}.bn.running_mean"] = 0.1 * torch.randn(cout, generator=g)
        sd[f"{name}.bn.running_var"] = 0.5 + torch.rand(cout, generator=g)
        sd[f"{name}.bn.num_batches_tracked"] = torch.tensor(1000)
    sd["logits.conv3d.weight"] = torch.randn((classes, 1024, 1, 1, 1), generator=g) / 32.0
    sd["logits.conv3d.bias"] = 0.1 * torch.randn(classes, generator=g)
    return sd


def tf32(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> the nearest TF32 value (ties to even), as fp32."""
    u = x.contiguous().view(torch.int32)
    keep = (u & 0x7F800000) != 0x7F800000
    r = torch.where(keep, u + 0xFFF + ((u >> 13) & 1), u) & ~0x1FFF
    return r.view(torch.float32)


def same_pad(x: torch.Tensor, k, s) -> torch.Tensor:
    """TF "SAME" zero padding of [N, C, T, H, W] for kernel k and stride s (per axis t, h, w)."""
    pads = []
    for n, kk, ss in reversed(list(zip(x.shape[2:], k, s))):
        pad = max(kk - ss, 0) if n % ss == 0 else max(kk - n % ss, 0)
        pads += [pad // 2, pad - pad // 2]
    return F.pad(x, pads)


def unit(x, sd, name, k, s=(1, 1, 1), round_stem=False):
    w = sd[f"{name}.conv3d.weight"].to(x)
    x = same_pad(x, k, s)
    if round_stem:
        x, w = tf32(x), tf32(w)
    y = F.conv3d(x, w, stride=s)
    bn = nn.BatchNorm3d(w.shape[0], eps=1e-3).eval()
    bn.load_state_dict({p: sd[f"{name}.bn.{p}"] for p in ("weight", "bias", "running_mean", "running_var")}, strict=False,
                       assign=True)
    return F.relu(bn.to(x)(y))


def max_pool(x, k, s):
    return F.max_pool3d(same_pad(x, k, s), k, s)


def trunk(x: torch.Tensor, sd: dict, tf32_mode: bool = False) -> torch.Tensor:
    """Prepared clips [N, 3, T, 224, 224] -> Mixed_5c [N, 1024, T5, 7, 7]."""
    x = unit(x, sd, "Conv3d_1a_7x7", (7, 7, 7), (2, 2, 2), round_stem=tf32_mode)
    x = max_pool(x, (1, 3, 3), (1, 2, 2))
    x = unit(x, sd, "Conv3d_2b_1x1", (1, 1, 1))
    x = unit(x, sd, "Conv3d_2c_3x3", (3, 3, 3))
    x = max_pool(x, (1, 3, 3), (1, 2, 2))
    for name in BLOCKS:
        if name == "Mixed_4b":
            x = max_pool(x, (3, 3, 3), (2, 2, 2))
        if name == "Mixed_5b":
            x = max_pool(x, (2, 2, 2), (2, 2, 2))
        b0 = unit(x, sd, f"{name}.b0", (1, 1, 1))
        b1 = unit(unit(x, sd, f"{name}.b1a", (1, 1, 1)), sd, f"{name}.b1b", (3, 3, 3))
        b2 = unit(unit(x, sd, f"{name}.b2a", (1, 1, 1)), sd, f"{name}.b2b", (3, 3, 3))
        b3 = unit(max_pool(x, (3, 3, 3), (1, 1, 1)), sd, f"{name}.b3b", (1, 1, 1))
        x = torch.cat([b0, b1, b2, b3], dim=1)
    return x


def head(f: torch.Tensor, sd: dict) -> torch.Tensor:
    """Mixed_5c [N, 1024, T5, 7, 7] -> [N, K]: average pool, logits, mean over time."""
    x = F.avg_pool3d(f, (2, 7, 7), stride=1)
    x = F.conv3d(x, sd["logits.conv3d.weight"].to(x), sd["logits.conv3d.bias"].to(x))
    return x.mean(dim=2).flatten(1)


@torch.no_grad()
def embed(x: torch.Tensor, sd: dict, tf32: bool = False) -> torch.Tensor:
    """With ``tf32``, cuDNN's TF32 switch is set to PyTorch's default (on) for the call and restored after it, so the
    mode does not depend on what ran before in the process."""
    if not tf32:
        return head(trunk(x.double(), sd), sd)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        return head(trunk(x.float(), sd, True), sd)
    finally:
        torch.backends.cudnn.allow_tf32 = prev

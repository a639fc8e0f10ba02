"""The weights the engine rewrites before a kernel sees them, in fp16 and bf16, without a GPU.

Two folds turn one checkpoint weight into another:
  * prepack_params folds the decoder's up-sampler (nearest x2, then a 3x3x3 conv) into four 3x2x2 phase kernels on the
    input that is not up-sampled (Engine.upsample runs one conv per phase into a (ph::2, pw::2) lattice of the output);
  * on a one-frame input (the image path) Engine._single_frame_weights sums the time taps of a 3x3x3 conv (replicate
    time padding) or selects one (zero padding), and of an up_time = 2 conv keeps only the half of the output channels
    that lands on the kept frame.
a. The geometry of both folds, independent of rounding: folded exactly in fp64 and run through FakeOps(torch.float64),
   the engine's layers equal the oracle's layers run in fp64 on the same 16-bit checkpoint weights.
b. Every stored folded weight is the exact sum of the checkpoint's 16-bit weights rounded once to the compute dtype,
   bit for bit - the multi-frame phase weights, every single-frame fold (3x3x3 convs, the tap-packed conv_in, the
   up-sampler phases).
"""
import pytest
import torch

from cvvae_b200.engine import Act, Engine, NetConfig, prepack_params
from fake_ops import FakeOps
from oracle import cvvae_oracle as O

F64 = torch.float64
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
SEED = 1234
WIDTH = 64
# the decoder's up-samplers: (oracle prefix, up_time)
UPSAMPLERS = {
    "sd21": [("decoder.up.3.upsample", 2), ("decoder.up.2.upsample", 1), ("decoder.up.1.upsample", 2)],
    "sd3": [("decoder.up_blocks.0.upsamplers.0", 2), ("decoder.up_blocks.1.upsamplers.0", 1),
            ("decoder.up_blocks.2.upsamplers.0", 2)],
}
CONV3 = {"sd21": "decoder.up.3.block.0.conv1", "sd3": "decoder.up_blocks.0.resnets.0.conv1"}


def _configs(variant, causal_decoder=False):
    cfg = O.VAEConfig(variant=variant, ch=WIDTH, z_channels=4 if variant == "sd21" else 16, causal_decoder=causal_decoder)
    net = NetConfig(variant=variant, z_channels=cfg.z_channels, widths=tuple(cfg.widths), causal_decoder=causal_decoder)
    return cfg, net


_SD = {}


def _checkpoint(variant, dtype):
    """The synthetic state dict stored in the 16-bit model dtype (what prepack_params receives from a .half() model)."""
    if (variant, dtype) not in _SD:
        cfg, _ = _configs(variant)
        _SD[variant, dtype] = {k: v.to(dtype) for k, v in O.make_state_dict(cfg, SEED).items()}
    return _SD[variant, dtype]


def _engine64(variant, dtype, causal_decoder=False):
    """Engine on the checkpoint's 16-bit weights widened to fp64: folds exact, every operator evaluated in fp64."""
    sd64 = {k: v.to(F64) for k, v in _checkpoint(variant, dtype).items()}
    ops = FakeOps(F64)
    _, net = _configs(variant, causal_decoder)
    return Engine(net, prepack_params(sd64, ops, F64), ops, F64), sd64


def _rand(shape, seed):
    """fp32 values in fp64 (the oracle's sd21 causal conv pads in fp32, as the reference does)."""
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(shape, generator=g) * 2 - 1).to(F64)


def _assert_fp64_equal(got, want, tag):
    err = (got - want).abs().max().item()
    scale = want.abs().max().item()
    assert got.shape == want.shape and err <= 1e-12 * scale, f"{tag}: max |err| {err:.3e} vs max |ref| {scale:.3e}"


def _round_once(r, dtype):
    """fp64 -> the nearest `dtype` value, ties to even, in one step (a cast through fp32 would round twice)."""
    p, emin = (11, -14) if dtype == torch.float16 else (8, -126)
    e = ((r.view(torch.int64) >> 52) & 0x7FF) - 1023
    ulp = (((e.clamp_min(emin) - (p - 1)) + 1023) << 52).view(F64)
    return (torch.round(r / ulp) * ulp).to(dtype)


# --------------------------------------------------------------------------------------- a. geometry in fp64
@pytest.mark.parametrize("T", [1, 2, 3])
@pytest.mark.parametrize("variant,causal", [("sd21", False), ("sd3", False), ("sd3", True)])
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_upsample_phase_fold_equals_reference_in_fp64(dt, variant, causal, T):
    """Four phase convs into lattice views (and at T = 1 the single-frame fold with its up_time half) == nearest x2 +
    3x3x3 conv + interleave of the oracle.  sd21 never forwards `causal` to its up-sampler (always replicate (1, 1))."""
    eng, sd64 = _engine64(variant, DTYPES[dt], causal)
    for i, (p, up_time) in enumerate(UPSAMPLERS[variant]):
        ci = sd64[p + ".conv.weight"].shape[1]
        x = _rand((1, ci, T, 5, 6), 10 + i)
        y = eng.upsample(Act(x.permute(0, 2, 3, 4, 1)), p + ".conv", up_time, causal).t.permute(0, 4, 1, 2, 3)
        if variant == "sd21":
            want = O.sd21_upsample(x, sd64, p, up_time=up_time == 2)
        else:
            want = O.sd3_upsample(x, sd64, p, up_time=up_time == 2, causal=causal)
        _assert_fp64_equal(y, want, f"{p} T={T}")


@pytest.mark.parametrize("variant,causal", [("sd21", False), ("sd21", True), ("sd3", False), ("sd3", True)])
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_single_frame_conv_fold_equals_reference_in_fp64(dt, variant, causal):
    """T = 1: a 3x3x3 conv with replicate time padding sums its taps, with zero padding (sd21 non-causal) keeps the centre
    tap; the tap-packed network-input conv folds the same way."""
    eng, sd64 = _engine64(variant, DTYPES[dt], causal)
    p = CONV3[variant]
    x = _rand((1, sd64[p + ".weight"].shape[1], 1, 7, 5), 20)
    y = eng.conv3(Act(x.permute(0, 2, 3, 4, 1)), p, causal).t.permute(0, 4, 1, 2, 3)
    want = O.sd21_conv(x, sd64, p, causal, 1) if variant == "sd21" else O.sd3_conv3d(x, sd64, p, causal, 1)
    _assert_fp64_equal(y, want, p)
    assert any(k.startswith(p + ".weight.t1.") for k in eng.p), "the single-frame fold did not run"
    # the network-input conv (3 real channels, NCDHW input): spatial taps packed into channels, then the time fold
    z = _rand((1, 3, 1, 7, 5), 21)
    y = eng.conv3(Act(z.permute(0, 2, 3, 4, 1)), "encoder.conv_in", causal).t.permute(0, 4, 1, 2, 3)
    want = (O.sd21_conv(z, sd64, "encoder.conv_in", causal, 1) if variant == "sd21"
            else O.sd3_conv3d(z, sd64, "encoder.conv_in", causal, 1))
    _assert_fp64_equal(y, want, "encoder.conv_in")
    assert any(k.startswith("encoder.conv_in.weight.hwpack.t1.") for k in eng.p), "the tap-packed fold did not run"


# --------------------------------------------------------------------------------------- b. one rounding
def _single_frame_exact(w64, key):
    """Exact single-frame fold of a packed fp64 weight [3 * khw, Co, Ci] for the key f"{wkey}.t1.{tl}.{pad_t}.{up_time}"."""
    tl, pad_t, up_time = (int(s) for s in key.rsplit(".", 3)[1:])
    w4 = w64.view(3, -1, w64.shape[1], w64.shape[2])
    wf = w4.sum(0) if pad_t == 1 else (w4[tl] if 0 <= tl < 3 else torch.zeros_like(w4[0]))
    return wf[:, w64.shape[1] // 2:] if up_time == 2 else wf


@pytest.mark.parametrize("variant", ["sd21", "sd3"])
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_every_folded_weight_is_rounded_once(dt, variant):
    dtype = DTYPES[dt]
    sd = _checkpoint(variant, dtype)
    cfg, net = _configs(variant)
    ops = FakeOps()
    eng = Engine(net, prepack_params(sd, ops, dtype), ops, dtype)
    # one image through encoder and decoder creates the single-frame fold of every 3x3x3 conv the network runs
    eng.decode(eng.encode(_rand((1, 3, 1, 16, 16), 30).to(dtype))[:, : cfg.z_channels])
    exact, _ = _engine64(variant, dtype)
    checked, failures = {"phase": 0, "t1": 0, "phase.t1": 0, "hwpack": 0}, []
    for k, v in eng.p.items():
        if ".phase" in k and k.endswith(".weight"):
            kind, want = "phase", exact.p[k]
        elif ".t1." in k and not k.endswith(".bias"):
            wkey = k.split(".t1.")[0]
            kind = "phase.t1" if ".phase" in wkey else ("hwpack" if wkey.endswith(".hwpack") else "t1")
            want = _single_frame_exact(exact.p[wkey], k)
        else:
            continue
        checked[kind] += 1
        want = _round_once(want, dtype)
        if not torch.equal(v, want):
            failures.append(f"{k}: {(v == want).double().mean().item():.4f} of the weights rounded once")
    assert checked["phase"] == 12 and checked["phase.t1"] == 12 and checked["hwpack"] >= 1 and checked["t1"] > 20, checked
    assert not failures, "\n".join(failures)

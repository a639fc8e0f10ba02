"""conv_tc's TMA epilogue (output staged in shared memory and written by TMA stores, residual prefetched by TMA into the
activation ring) against the register epilogue it replaces, fp16 and bf16.

Each case runs twice on the same inputs: as planned, and with CVVAE_TMA_EPILOGUE=0, which restores the register
epilogue (the interior-tile and general loops that tests/test_gpu_conv_plans.py checks against fp64).  The plan query
proves which path each run took.  Outputs and fused GroupNorm statistics must be equal bit for bit.  The cases cover what
the TMA path handles without per-element tests: edge tiles (H and W not multiples of TH and TW), Cout below the CTA's
channel count, the up_time = 2 interleave with its first half skipped at t = 0, residual together with fused statistics,
batch > 1, a flat (H = 1, 1x1x1) problem, and an output that is a window of a larger buffer filled with a canary: nothing
outside the window may change.
"""
import pytest
import torch

import test_gpu_conv_plans as CP
from fake_ops import PAD_REPLICATE, PAD_ZERO

pytestmark = pytest.mark.gpu
DEV = "cuda"
CANARY = -7.75   # exact in fp16 and bf16

# name: input [B, T, H, W, Cin], Cout, kernel, stride, pads ((t), (h), (w)), pad_t, up_time, extras, expected N_cta
# extras: residual, gn (groups), alpha, shortcut (Cin2), window (output and residual are views into larger buffers)
CASES = {
    "residual_gn": ((1, 3, 45, 75, 128), 128, (3, 3, 3), (1, 1, 1), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1,
                    {"residual": True, "gn": 32}, 128),
    "up_time_gn": ((1, 2, 45, 75, 128), 128, (3, 3, 3), (1, 1, 1), ((1, 1), (1, 1), (1, 1)), PAD_REPLICATE, 2,
                   {"gn": 32}, 128),
    "up_time_bn256": ((1, 2, 30, 45, 256), 512, (3, 3, 3), (1, 1, 1), ((1, 1), (1, 1), (1, 1)), PAD_REPLICATE, 2,
                      {"gn": 32}, 256),
    "bn256_residual_gn": ((1, 2, 30, 45, 512), 512, (3, 3, 3), (1, 1, 1), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1,
                          {"residual": True, "gn": 32}, 256),
    "cout8": ((1, 3, 37, 37, 512), 8, (3, 3, 3), (1, 1, 1), ((2, 0), (1, 1), (1, 1)), PAD_REPLICATE, 1, {}, 64),
    "bn64_alpha_gn": ((1, 3, 45, 75, 64), 64, (3, 3, 3), (1, 1, 1), ((2, 0), (1, 1), (1, 1)), PAD_REPLICATE, 1,
                      {"gn": 32, "alpha": 0.5}, 64),
    "shortcut_gn": ((1, 2, 45, 75, 128), 128, (3, 3, 3), (1, 1, 1), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1,
                    {"shortcut": 256, "gn": 32}, 128),
    "batch2_residual_gn": ((2, 2, 45, 75, 128), 128, (3, 3, 3), (1, 1, 1), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1,
                           {"residual": True, "gn": 32}, 128),
    "flat_residual": ((1, 2, 1, 1000, 128), 256, (1, 1, 1), (1, 1, 1), ((0, 0), (0, 0), (0, 0)), PAD_ZERO, 1,
                      {"residual": True}, 256),
    "window_residual_gn": ((1, 2, 45, 75, 128), 128, (3, 3, 3), (1, 1, 1), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1,
                           {"residual": True, "gn": 32, "window": True}, 128),
}
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
# window: the output sits at (h, w, c) = (2, 3, 8) of a buffer 5 rows, 7 columns and 24 channels larger (the channel
# offset and the row pitch stay 16-byte multiples, as the TMA path needs)
WIN_OFF, WIN_PAD = (2, 3, 8), (5, 7, 24)


def _window_buffer(yshape, dtype, fill):
    B, T, H, W, Cc = yshape
    buf = torch.full((B, T, H + WIN_PAD[0], W + WIN_PAD[1], Cc + WIN_PAD[2]), fill, dtype=dtype, device=DEV)
    h, w, c = WIN_OFF
    return buf, buf[:, :, h:h + H, w:w + W, c:c + Cc]


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("name", list(CASES))
def test_conv_tc_tma_epilogue_matches_register_epilogue(name, dt, monkeypatch):
    from cvvae_b200.ops import CudaOps
    ops, dtype = CudaOps(), DTYPES[dt]
    case = CASES[name]
    xs, co, kernel, stride, pads, pad_t, up_time, ex, n_cta = case
    B, T, H, W, Ci = xs
    taps = kernel[0] * kernel[1] * kernel[2]
    To, Ho, Wo, yshape = CP._geometry(case)
    x = CP._rand(xs, dtype, 3)
    w = CP._rand((taps, co, Ci), dtype, 4, scale=(taps * Ci) ** -0.5 * 2)
    bias = CP._rand((co,), torch.float32, 5, 0.3)
    (tl, _), (hl, _), (wl, _) = pads
    kw = dict(kernel=kernel, stride=stride, offset=(-tl, -hl, -wl), pad_t=pad_t, pad_hw=PAD_ZERO, up_time=up_time,
              alpha=ex.get("alpha", 1.0))
    window = ex.get("window", False)
    if ex.get("residual"):
        r = CP._rand(yshape, dtype, 6)
        if window:   # the residual is read on the output's strides
            _, rv = _window_buffer(yshape, dtype, 0.0)
            rv.copy_(r)
            r = rv
        kw["residual"] = r
    if ex.get("shortcut"):
        c2 = ex["shortcut"]
        kw["sc_x"] = CP._rand(yshape[:4] + (c2,), dtype, 7)
        kw["sc_w"] = CP._rand((co, c2), dtype, 8, scale=c2 ** -0.5)
    groups = ex.get("gn")

    runs = {}
    for switch in ("1", "0"):
        monkeypatch.setenv("CVVAE_TMA_EPILOGUE", switch)
        if window:
            buf, y = _window_buffer(yshape, dtype, CANARY)
        else:
            buf, y = None, torch.zeros(yshape, dtype=dtype, device=DEV)
        st = ops.new_stats(B, groups, DEV) if groups else None
        skw = dict(gn_stats=st, gn_groups=groups) if groups else {}
        plan = ops.conv_tc_plan(x, w, bias, out=y, epilogue=True, **kw, **skw)
        ops.conv(x, w, bias, out=y, force="tc", **kw, **skw)
        runs[switch] = (plan, y, st, buf)
    torch.cuda.synchronize()

    (p_on, y_on, st_on, buf_on), (p_off, y_off, st_off, _) = runs["1"], runs["0"]
    assert p_on["eligible"] == 1 and p_on["N_cta"] == n_cta, p_on
    assert p_on["tma_epilogue"] == 1 and p_off["tma_epilogue"] == 0, (p_on, p_off)
    assert {k: v for k, v in p_on.items() if k != "tma_epilogue"} == {k: v for k, v in p_off.items() if k != "tma_epilogue"}
    if not p_on["flat"]:   # edge tiles in both H and W
        assert Ho % p_on["TH"] and Wo % p_on["TW"], (p_on, Ho, Wo)
    assert torch.equal(y_on, y_off), f"{int((y_on != y_off).sum().item())} of {y_on.numel()} elements differ"
    if groups:
        assert torch.equal(st_on, st_off), "fused GroupNorm statistics differ"
    if window:
        outside = torch.ones(buf_on.shape, dtype=torch.bool, device=DEV)
        h, w_, c = WIN_OFF
        outside[:, :, h:h + Ho, w_:w_ + Wo, c:c + yshape[4]] = False
        assert bool((buf_on[outside] == CANARY).all()), "the TMA store wrote outside the output view"

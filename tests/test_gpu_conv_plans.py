"""conv_tc at the tile plans of the network's expensive layers, fp16 and bf16, against the convolution spec in fp64.

The op-level conv cases (tests/test_gpu_ops.py) are small enough that the planner drops to NACC = 1.  Here every case is
large enough that each CTA keeps its full set of accumulators (NACC = 256 / N_cta), so the kernel runs the branch-free
wgmma chain, addresses sub-tiles s > 0 and, on tiles whose rows and channels are all valid, the interior epilogue (its own
bias / residual / pack / store code and GroupNorm sums).  Each case proves its plan through cvvae_conv_tc_plan() and has
interior and edge tiles; it holds at least 2 x 132 CTAs per sample, so the plan is the same on H100 SXM (132 SMs) and
PCIe (114 SMs).  Shapes are the network's own layers (tools/bench_conv.py P, the engine's residual / fused shortcut /
GroupNorm-statistics calls) with T and H x W cut down.

Reference: FakeOps(torch.float64).conv on the same 16-bit inputs (the written-down spec evaluated in fp64), and the
condition sum S = |alpha| sum |x w| + |bias| + |residual| (the same spec on absolute values).  Gates, one per class of
defect:
  1. per element  |y - r| <= 1/2 ulp_dt(r) + C_ACC * 2^-24 * sqrt(K) * S            (rounding; accumulation)
  2. share of elements equal to r correctly rounded to the output dtype           (truncating / mis-rounding pack)
  3. |mean((y - r) / ulp_dt(r))| <= 0.05                                          (directed rounding, scaled alpha / bias)
  4. the interior epilogue equals the general one bit for bit, statistics included: the case runs again into a view
     whose pointer is odd in elements, which turns off word stores (vec2) and with them the interior loop
  5. fused GroupNorm statistics equal fp64 sums of the stored tensor, and GroupNorm fed with them equals GroupNorm
     computing its own
Measured values go to conv_plans.json in the directory where the GPU tests record their measurements
(test_gpu_ops.OUT).
"""
import json
import math
import os

import pytest
import torch

import test_gpu_ops
from fake_ops import PAD_REPLICATE, PAD_ZERO, FakeOps

pytestmark = pytest.mark.gpu
DEV = "cuda"
OUT = test_gpu_ops.OUT   # the record directory shared by the GPU tests
MIN_CTAS_PER_SAMPLE = 2 * 132

# Gate 1.  The products of two 16-bit values are exact in fp32.  Each wgmma (K = 16) adds its products to the fp32
# accumulator with at most one truncation, |err| <= 2^-23 * S, so a chain of K / 16 MMAs is off by at most
# (K / 16) * 2^-23 * S = 2^-24 * sqrt(K) * S * sqrt(K) / 8: C_ACC = 16 covers K <= 16384 (the largest case here has
# K = 27 * 512 = 13824, sqrt(K) / 8 = 14.7).  The epilogue's fma(acc, alpha, bias) and residual add are two more fp32
# roundings, 2 * 2^-24 * S, inside the remaining 1.3 * sqrt(K) >= 40.
C_ACC = 16.0
# Gate 2.  fp32 accumulation error is about 2^-17 |y| at K ~ 3.5e3 (it grows like sqrt(K)); a mismatch needs r within
# that distance of a rounding midpoint, so the expected share of mismatches is about 2^-17 / ulp_rel: ~1-2 % for fp16
# (ulp 2^-11..2^-10 relative), 8x fewer for bf16 (3 fewer mantissa bits).  The gate allows 5x the upper estimate, which
# leaves room for the 4x larger K of the 512-channel case; a truncating pack mismatches ~50 %.
MISMATCH_EST = {torch.float16: 0.02, torch.bfloat16: 0.02 / 8}
MISMATCH_MARGIN = 5.0
# Gate 3.  Correct rounding has mean signed error ~0 +- 0.3 / sqrt(n) ulp; directed rounding gives +-0.5 ulp.
MAX_MEAN_ULP = 0.05

# name: input [B, T, H, W, Cin], Cout, kernel, stride, pads ((t), (h), (w)), pad_t, up_time, extras, expected N_cta
# extras: residual, shortcut (Cin2), gn (groups), alpha, ncdhw (NCDHW output view: s_c != 1, no word stores)
CASES = {
    # BN = 128, NACC = 2 (E/D 128->128 @17x576, 256->128, the encoder's down-sampling)
    "e128_causal333": ((1, 3, 116, 172, 128), 128, (3, 3, 3), (1, 1, 1), ((2, 0), (1, 1), (1, 1)), PAD_REPLICATE, 1,
                       {"gn": 32}, 128),
    "e128_zero133": ((1, 3, 116, 172, 128), 128, (1, 3, 3), (1, 1, 1), ((0, 0), (1, 1), (1, 1)), PAD_ZERO, 1, {}, 128),
    "e128_down222": ((1, 5, 228, 324, 128), 128, (3, 3, 3), (2, 2, 2), ((2, 0), (0, 1), (0, 1)), PAD_REPLICATE, 1, {}, 128),
    "d128_up_time": ((1, 2, 140, 212, 128), 128, (3, 3, 3), (1, 1, 1), ((1, 1), (1, 1), (1, 1)), PAD_REPLICATE, 2,
                     {"gn": 32}, 128),
    "d128_residual": ((2, 3, 116, 172, 128), 128, (3, 3, 3), (1, 1, 1), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1,
                      {"residual": True, "gn": 32}, 128),
    "d256_128_shortcut": ((1, 3, 116, 172, 128), 128, (3, 3, 3), (1, 1, 1), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1,
                          {"shortcut": 256, "gn": 32}, 128),
    "d256_128": ((1, 3, 116, 172, 256), 128, (3, 3, 3), (1, 1, 1), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1, {"gn": 32}, 128),
    # BN = 64, NACC = 4; Cout = 32 never has a channel-interior tile
    "n64_alpha": ((1, 3, 196, 196, 64), 64, (3, 3, 3), (1, 1, 1), ((2, 0), (1, 1), (1, 1)), PAD_REPLICATE, 1,
                  {"gn": 32, "alpha": 0.5}, 64),
    "n32_cpg1": ((1, 3, 196, 196, 64), 32, (3, 3, 3), (1, 1, 1), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1, {"gn": 32}, 64),
    # BN = 256 (one 128-position sub-tile per CTA: always full)
    "e512_333": ((1, 3, 68, 68, 512), 512, (3, 3, 3), (1, 1, 1), ((2, 0), (1, 1), (1, 1)), PAD_REPLICATE, 1, {"gn": 32}, 256),
    "d256_512_up_time": ((1, 2, 84, 84, 256), 512, (3, 3, 3), (1, 1, 1), ((1, 1), (1, 1), (1, 1)), PAD_REPLICATE, 2,
                         {"gn": 16}, 256),
    # the general epilogue at full NACC: NCDHW output (channel stride != 1)
    "n128_ncdhw": ((1, 3, 116, 172, 128), 128, (3, 3, 3), (1, 1, 1), ((2, 0), (1, 1), (1, 1)), PAD_REPLICATE, 1,
                   {"ncdhw": True}, 128),
}
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
_RECORD = {}


def _rand(shape, dtype, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(shape, generator=g) * 2 - 1) * scale).to(dtype).to(DEV)


def _ulp(r, dtype):
    """Spacing of `dtype` numbers at |r| (r float64; subnormal spacing below the smallest normal).

    Built from the exponent bits: torch.ldexp / pow on the GPU are not exact powers of two."""
    p, emin = (11, -14) if dtype == torch.float16 else (8, -126)
    e = ((r.view(torch.int64) >> 52) & 0x7FF) - 1023         # binade of |r| (0 and fp64 subnormals: -1023)
    e = e.clamp_min(emin) - (p - 1)
    return ((e + 1023) << 52).view(torch.float64)


def _geometry(case):
    xs, co, kernel, stride, pads, pad_t, up_time, ex, _ = case
    B, T, H, W, Ci = xs
    (tl, th), (hl, hh), (wl, wh) = pads
    To = (T + tl + th - kernel[0]) // stride[0] + 1
    Ho = (H + hl + hh - kernel[1]) // stride[1] + 1
    Wo = (W + wl + wh - kernel[2]) // stride[2] + 1
    yshape = (B, 2 * To - 1, Ho, Wo, co // 2) if up_time == 2 else (B, To, Ho, Wo, co)
    return To, Ho, Wo, yshape


def _out(yshape, dtype, layout):
    """An output tensor of the logical [B,T,H,W,C] shape: channels last, NCDHW, or channels last at an odd element offset."""
    if layout == "ncdhw":
        B, T, H, W, Cc = yshape
        return torch.zeros((B, Cc, T, H, W), dtype=dtype, device=DEV).permute(0, 2, 3, 4, 1)
    if layout == "odd":
        n = math.prod(yshape)
        return torch.zeros(n + 1, dtype=dtype, device=DEV)[1:].view(yshape)
    return torch.zeros(yshape, dtype=dtype, device=DEV)


def _check_plan(plan, case, To, Ho, Wo):
    """Full accumulators on every CTA, interior and edge tiles, enough CTAs per sample for either H100."""
    xs, co, kernel, stride, pads, pad_t, up_time, ex, n_cta = case
    B = xs[0]
    assert plan["eligible"] == 1 and plan["flat"] == 0, plan
    assert plan["N_cta"] == n_cta and plan["NACC"] == 256 // n_cta, plan
    assert plan["TH"] == plan["ROWS"] * plan["NACC"] and plan["TW"] * plan["ROWS"] == 128, plan
    assert plan["tiles_w"] == -(-Wo // plan["TW"]) and plan["tiles_h"] == -(-Ho // plan["TH"]), plan
    assert plan["n_tiles_n"] == -(-co // n_cta), plan
    assert plan["grid"] == plan["n_tiles_n"] * To * plan["tiles_w"] * plan["tiles_h"] * B, plan
    assert plan["grid"] // B >= MIN_CTAS_PER_SAMPLE, plan
    full_w, full_h = Wo // plan["TW"], Ho // plan["TH"]
    interior = full_w * full_h                                     # tiles with every row valid
    edge = plan["tiles_w"] * plan["tiles_h"] - interior
    assert interior > 0 and edge > 0, (plan, Ho, Wo)
    return {"interior_tiles_per_frame": interior, "edge_tiles_per_frame": edge,
            "channel_interior": co >= n_cta}


def _dump():
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "conv_plans.json"), "w") as f:
        json.dump(_RECORD, f, indent=1, sort_keys=True)


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("name", list(CASES))
def test_conv_tc_full_accumulator_plans(name, dt):
    from cvvae_b200.ops import CudaOps
    ops, dtype = CudaOps(), DTYPES[dt]
    case = CASES[name]
    xs, co, kernel, stride, pads, pad_t, up_time, ex, n_cta = case
    B, T, H, W, Ci = xs
    taps = kernel[0] * kernel[1] * kernel[2]
    To, Ho, Wo, yshape = _geometry(case)
    yC = yshape[4]
    x = _rand(xs, dtype, 3)
    w = _rand((taps, co, Ci), dtype, 4, scale=(taps * Ci) ** -0.5 * 2)
    bias = _rand((co,), torch.float32, 5, 0.3)
    (tl, _), (hl, _), (wl, _) = pads
    kw = dict(kernel=kernel, stride=stride, offset=(-tl, -hl, -wl), pad_t=pad_t, pad_hw=PAD_ZERO, up_time=up_time,
              alpha=ex.get("alpha", 1.0))
    if ex.get("residual"):
        kw["residual"] = _rand(yshape, dtype, 6)
    if ex.get("shortcut"):
        c2 = ex["shortcut"]
        kw["sc_x"] = _rand(yshape[:4] + (c2,), dtype, 7)
        kw["sc_w"] = _rand((co, c2), dtype, 8, scale=c2 ** -0.5)
    groups = ex.get("gn")

    # two runs: the case's layout, and one that flips word stores (vec2) and with them the epilogue loop
    layouts = ("ncdhw", "last") if ex.get("ncdhw") else ("last", "odd")
    ys, stats, plans = [], [], []
    for layout in layouts:
        y = _out(yshape, dtype, layout)   # a residual shares the strides of both (contiguous) channels-last outputs
        st = ops.new_stats(B, groups, DEV) if groups else None
        skw = dict(gn_stats=st, gn_groups=groups) if groups else {}
        plans.append(ops.conv_tc_plan(x, w, bias, out=y, **kw, **skw))
        ops.conv(x, w, bias, out=y, force="tc", **kw, **skw)
        ys.append(y)
        stats.append(st)
    torch.cuda.synchronize()
    rec = {"plan": plans[0]}
    rec.update(_check_plan(plans[0], case, To, Ho, Wo))
    p_alt = dict(plans[1])
    assert p_alt.pop("vec2") != plans[0]["vec2"] and p_alt == {k: v for k, v in plans[0].items() if k != "vec2"}, plans
    y = ys[0]
    failed = []   # every gate is evaluated and recorded; the test fails on any of them

    # gate 4: interior loop == general loop, bit for bit (outputs and fused statistics)
    rec["epilogues_bit_equal"] = torch.equal(ys[0], ys[1]) and (not groups or torch.equal(stats[0], stats[1]))
    if not rec["epilogues_bit_equal"]:
        failed.append("4: interior and general epilogues differ"
                      f" ({int((ys[0] != ys[1]).sum().item())} elements, statistics equal: {groups and torch.equal(stats[0], stats[1])})")
    del ys

    # fp64 spec and condition sum
    f64 = FakeOps(torch.float64)
    r = f64.conv(x, w, bias, out=torch.zeros(yshape, dtype=torch.float64, device=DEV), **kw)
    abs_kw = dict(kw, alpha=abs(kw["alpha"]))
    for k in ("residual", "sc_x", "sc_w"):
        if kw.get(k) is not None:
            abs_kw[k] = kw[k].abs()
    S = f64.conv(x.abs(), w.abs(), bias.abs(), out=torch.zeros(yshape, dtype=torch.float64, device=DEV), **abs_kw)
    K = taps * Ci + (ex.get("shortcut") or 0)
    yd = y.double()
    ulp = _ulp(r, dtype)
    err = yd - r

    # gate 1: per-element bound
    bound = 0.5 * ulp + C_ACC * 2.0 ** -24 * math.sqrt(K) * S
    ratio = (err.abs() / bound).max().item()
    if not ratio <= 1.0:
        failed.append(f"1: |y - r| exceeds the bound by {ratio:.3f}x")
    # gate 2: correctly rounded share (r / ulp is exact in fp64; round half to even)
    rn = torch.round(r / ulp) * ulp
    share = (yd == rn).double().mean().item()
    min_share = 1.0 - MISMATCH_MARGIN * MISMATCH_EST[dtype]
    if not share >= min_share:
        failed.append(f"2: {share:.4f} correctly rounded < {min_share:.4f}")
    # gate 3: mean signed error in ulps
    mean_ulp = (err / ulp).mean().item()
    if not abs(mean_ulp) <= MAX_MEAN_ULP:
        failed.append(f"3: mean signed error {mean_ulp:+.4f} ulp")
    rec.update({"K": K, "numel": y.numel(), "worst_bound_ratio": ratio, "correctly_rounded_share": share,
                "min_share": min_share, "mean_signed_ulp": mean_ulp})
    del r, S, yd, ulp, err, bound, rn

    # gate 5: fused statistics vs fp64 sums of the stored tensor; GroupNorm fed with them vs computing its own
    if groups:
        v = y.double().reshape(B, -1, groups, yC // groups)
        want = torch.stack([v.sum(dim=(1, 3)), (v * v).sum(dim=(1, 3))], dim=-1)
        got = torch.stack([stats[0][..., 0].double() / 2.0 ** 20, stats[0][..., 1].double() / 2.0 ** 18], dim=-1)
        del v
        rec["stats_max_abs_err"] = (got - want).abs().max().item()
        try:
            torch.testing.assert_close(got, want, rtol=1e-5, atol=2e-2)
        except AssertionError as e:
            failed.append(f"5: fused statistics vs fp64 sums of y: {str(e).splitlines()[0:4]}")
        g = _rand((yC,), torch.float32, 21) * 0.5 + 1.0
        b = _rand((yC,), torch.float32, 22, 0.2)
        tol = dict(rtol=1e-3, atol=1e-4) if dtype == torch.float16 else dict(rtol=8e-3, atol=1e-3)
        try:
            torch.testing.assert_close(ops.groupnorm(y, g, b, groups, 1e-5, stats=stats[0]).float(),
                                       ops.groupnorm(y, g, b, groups, 1e-5).float(), **tol)
        except AssertionError as e:
            failed.append(f"5: GroupNorm with the fused statistics: {str(e).splitlines()[0:4]}")
    rec["failed_gates"] = failed
    _RECORD[f"{name}/{dt}"] = rec
    _dump()
    assert not failed, f"{name}/{dt}: " + "; ".join(failed)

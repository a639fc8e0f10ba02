"""The kernels around the convolution in fp16 and bf16, against the operation in fp64 on the same 16-bit inputs.

tests/test_gpu_ops.py checks these entry points in fp16 at rtol 1e-3 / atol 1e-4 against an fp32 torch restatement: one
fp16 ulp is 4.9e-4 .. 9.8e-4 relative, so a round-toward-zero store or an off-by-one-ulp affine passes there, and bf16 is
reached only end to end.  Here every kernel the SD3 model in bf16 runs outside conv_tc is checked in both 16-bit dtypes, on
the branches the network takes: GroupNorm with 2, 4, 8 and 16 channels per group, per frame or per sample, SiLU on and off,
statistics computed by the kernel or handed in, dense and framed (non-dense) views, position counts that leave a tail
in the 4-way unrolled loops; LayerNorm at C = 512 (norm_t) and 128; softmax_rows at the mid-block token counts, ragged,
misaligned (scalar path) and above 12 288 columns (the > 48 KB shared-memory opt-in); temporal attention in each of its
MAXT = 32 / 128 / 512 instantiations; the tap-stacked conv_out kernel on plain and on framed (SD3) inputs, partial
64-channel blocks, Cout 1 / 3 / 4; pack_taps_hw with the KT x 1 x 1 conv_in; the data movers; the block cases in bf16.

Reference: the operation in fp64 (torch on the GPU) on the same 16-bit inputs.  Gates, one per class of defect:
  1. per element  |y - r| <= 1/2 ulp_dt(r) + E, E the kernel's fp32 computation error bound, derived next to each
     kernel below                                                             (wrong value, lost term, bad statistics)
  2. share of elements equal to r rounded once to the dtype >= 1 - MISMATCH_MARGIN * mean(min(1, E / ulp_dt(r)))
                                                                              (truncating or mis-rounding store)
  3. |mean((y - r) / ulp_dt(r))| <= MAX_MEAN_ULP                             (directed rounding, biased shift or scale)
Data movers are compared bit for bit with tests/fake_ops.py instead, and the block cases against the fp32 oracle block.
Measured values go to kernels16.json in the directory where the GPU tests record their measurements (test_gpu_ops.OUT).
"""
import json
import math
import os

import pytest
import torch
import torch.nn.functional as F

import block_cases as BC
import kernel_bounds as KB
import test_gpu_conv_plans as CP
import test_gpu_ops
from fake_ops import PAD_REPLICATE, PAD_ZERO, FakeOps

pytestmark = pytest.mark.gpu
DEV = "cuda"
OUT = test_gpu_ops.OUT
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
U32 = KB.U32
_RECORD = {}


def _ops():
    from cvvae_b200.ops import CudaOps
    return CudaOps()


def _rand(shape, dtype, seed, scale=1.0, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) * scale + offset).to(dtype).to(DEV)


def _dump():
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "kernels16.json"), "w") as f:
        json.dump(_RECORD, f, indent=1, sort_keys=True)


def _gates(tag, y, r, E, dtype, **extra):
    """Gates 1-3 (kernel_bounds._gates) on a 16-bit result; records under `tag`, returns the failures."""
    rec, failed = KB._gates(y, r, E, dtype)
    _RECORD[tag] = {**rec, **extra}
    _dump()
    return [f"{tag}: {f}" for f in failed]


# ------------------------------------------------------------------------------------------------------------ GroupNorm
# The statistics and apply kernels' bound: kernel_bounds.gn_pointwise.
# name: (shape [B,T,H,W,C], per_frame, silu, layout, offset of the input's mean); C in {64, 128, 256, 512} with 32 groups
GN_CASES = {
    "c64_cpg2": ((1, 5, 24, 20, 64), False, True, "dense", 0.3),
    "c64_cpg2_frames_strided": ((2, 3, 10, 14, 64), True, False, "strided", 0.3),
    "c128_cpg4_frames": ((2, 3, 18, 22, 128), True, True, "dense", 0.3),
    "c128_cpg4_strided": ((1, 3, 20, 30, 128), False, False, "strided", 0.3),
    "c256_cpg8_strided": ((1, 4, 20, 27, 256), False, True, "strided", 0.3),
    "c512_cpg16_frames": ((1, 3, 14, 18, 512), True, True, "dense", 0.3),
    "c512_cpg16": ((1, 3, 14, 18, 512), False, False, "dense", 0.3),
    "c128_cpg4_large_mean": ((1, 3, 16, 21, 128), False, True, "dense", 3.0),
}


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("name", list(GN_CASES))
def test_groupnorm16(name, dt):
    ops, dtype = _ops(), DTYPES[dt]
    shape, per_frame, silu, layout, offset = GN_CASES[name]
    B, T, H, W, Cc = shape
    G, eps = 32, 1e-6
    cpg = Cc // G
    # the case reaches the branches it is named for
    pix, ppb, lanes, nblocks, n_last = KB.gn_geometry(shape, per_frame)
    assert n_last % (4 * lanes) != 0, "positions of the last CTA leave no tail after the 4-way unrolled loop"
    assert name.split("_")[1] == f"cpg{cpg}" and ((cpg < 8) == (Cc < 256))
    scale = 1.0 if offset > 1 else 2.0
    x = _rand(shape, dtype, 20, scale, offset)
    if layout == "strided":
        pad, inner = ops.empty_padded(*shape, dtype, DEV)
        inner.copy_(x)
        x = inner
        assert not x.is_contiguous() and x.stride(2) == (W + 2) * Cc, "the input view is not framed"
    gam = _rand((Cc,), torch.float32, 21, 0.5, 1.0)
    bet = _rand((Cc,), torch.float32, 22, 0.2)
    failed = []

    # statistics computed by the kernel
    eps_sum, fix, _ = KB.gn_sum_terms(shape, per_frame, G)
    y = ops.groupnorm(x, gam, bet, G, eps, per_frame=per_frame, silu=silu)
    r, E, k = KB.gn_reference(x, gam, bet, G, eps, per_frame, silu, eps_sum, fix)
    if offset > 1:
        assert k > 4.0, k                                   # mean several standard deviations from zero
    failed += _gates(f"groupnorm/{name}/kernel_stats/{dt}", y, r, E, dtype, max_mean_over_std=k, eps_sum=eps_sum)

    # statistics handed in (exact fp64 sums in the fixed-point format), as a conv epilogue would
    if not per_frame:
        st = ops.new_stats(B, G, DEV)
        v = x.double().reshape(B, -1, G, cpg)
        st[..., 0] = torch.round(v.sum(dim=(1, 3)) * 2.0 ** 20).long()
        st[..., 1] = torch.round((v * v).sum(dim=(1, 3)) * 2.0 ** 18).long()
        y2 = ops.groupnorm(x, gam, bet, G, eps, per_frame=False, silu=silu, stats=st)
        r2, E2, _ = KB.gn_reference(x, gam, bet, G, eps, False, silu, None, None)
        failed += _gates(f"groupnorm/{name}/exact_stats/{dt}", y2, r2, E2, dtype)

    # framed output (SD3 conv_norm_out): the interior equals the dense result bit for bit, the frame replicates it
    pad, inner = ops.empty_padded(*shape, dtype, DEV)
    ops.groupnorm(x, gam, bet, G, eps, per_frame=per_frame, silu=silu, out=inner)
    ops.replicate_border(pad)
    want = F.pad(inner.permute(0, 4, 1, 2, 3).float(), (1, 1, 1, 1, 0, 0), mode="replicate").permute(0, 2, 3, 4, 1)
    torch.cuda.synchronize()
    assert torch.equal(inner, y), "framed output differs from the dense one"
    assert torch.equal(pad.float(), want), "replicate_border"
    assert not failed, "; ".join(failed)


# ------------------------------------------------------------------------------------------------------------ LayerNorm
# Bound: kernel_bounds.layernorm_reference (|mean| <= sigma here: the 2^-16 (|gamma| (1 + |z|) + |beta|) form).
@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("shape", [(2, 3, 5, 7, 512), (1, 3, 7, 9, 128)])
def test_layernorm16(shape, dt):
    ops, dtype = _ops(), DTYPES[dt]
    B, T, H, W, Cc = shape
    assert (B * T * H * W) % 8 != 0, "tokens fill every 8-warp CTA"
    x = _rand(shape, dtype, 30, 2.0, 0.3)
    gam = _rand((Cc,), torch.float32, 31, 0.5, 1.0)
    bet = _rand((Cc,), torch.float32, 32, 0.2)
    y = ops.layernorm(x, gam, bet, 1e-5)
    r, E, _ = KB.layernorm_reference(x, gam, bet, 1e-5)
    failed = _gates(f"layernorm/C{Cc}/{dt}", y, r, E, dtype)
    assert not failed, "; ".join(failed)


# ---------------------------------------------------------------------------------------------------------- softmax_rows
# Bound: kernel_bounds.softmax_reference, E = 2^-18 r (4 + |s - m|).
# Gate 3 in fp16 at 20 000 columns: 17 % of the probabilities lie below half the subnormal spacing, and within each ulp
# step they are denser toward zero, so r rounded once is itself off by -0.025 ulp on average (-0.008 at 5184 columns).
# name: (rows, cols, ld_s, ld_p, misaligned).  1024 / 4096 / 5184: mid-block tokens of 256- / 512- / 576-px tiles.
SOFTMAX_CASES = {
    "cols1024": (64, 1024, 1024, 1024, False),
    "cols4096": (24, 4096, 4096, 4104, False),
    "cols5184": (20, 5184, 5184, 5192, False),
    "ragged1001": (48, 1001, 1008, 1016, False),
    "misaligned_scalar": (40, 1003, 1009, 1013, True),
    "optin_cols20000": (6, 20000, 20004, 20008, False),
}


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("name", list(SOFTMAX_CASES))
def test_softmax_rows16(name, dt):
    ops, dtype = _ops(), DTYPES[dt]
    rows, cols, ld_s, ld_p, misaligned = SOFTMAX_CASES[name]
    sentinel = -3.0
    s_buf = _rand((rows * ld_s + 1,), torch.float32, 33, 6.0)
    p_buf = torch.full((rows * ld_p + 1,), sentinel, dtype=dtype, device=DEV)
    o = 1 if misaligned else 0                          # one element past an aligned start
    s, p = s_buf[o:o + rows * ld_s].view(rows, ld_s), p_buf[o:o + rows * ld_p].view(rows, ld_p)
    vec = ld_s % 4 == 0 and ld_p % 4 == 0 and s.data_ptr() % 16 == 0 and p.data_ptr() % 8 == 0
    if misaligned:
        assert not vec and s.data_ptr() % 16 != 0, "the scalar (vec = 0) path is not taken"
    else:
        assert vec, "the vector path is not taken"
    if name.startswith("ragged"):
        assert cols % 4 != 0 and ld_s > cols and ld_p > cols
    if name.startswith("optin"):
        assert cols > 12288 and 4 * cols > 48 * 1024, "the row fits the default 48 KB of shared memory"
    ops.softmax_rows(s, cols, p)
    torch.cuda.synchronize()
    r, E = KB.softmax_reference(s, cols)
    failed = _gates(f"softmax_rows/{name}/{dt}", p[:, :cols], r, E, dtype)
    # columns between cols and ld, and the buffer outside the rows, are left untouched
    untouched = torch.cat([p[:, cols:].flatten(), p_buf[:o], p_buf[o + rows * ld_p:]])
    assert (untouched == sentinel).all(), "softmax_rows wrote outside its columns"
    assert not failed, "; ".join(failed)


# -------------------------------------------------------------------------------------------------- temporal attention
# Bound: kernel_bounds.attn_temporal_reference, E = u ((2 n1 + 19) A_i + 2 T + 5) sum_j p_ij |v_j|.
# name: (shape [B,T,H,W,C], MAXT of the instantiation that runs it)
ATTN_CASES = {
    "T5_C512": ((1, 5, 3, 5, 512), 32),
    "T5_C128": ((2, 5, 3, 5, 128), 32),
    "T40_C512": ((1, 40, 3, 5, 512), 128),
    "T40_C128": ((1, 40, 3, 5, 128), 128),
    "T200_C512": ((1, 200, 3, 5, 512), 512),
    "T200_C128": ((1, 200, 3, 5, 128), 512),
}


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("name", list(ATTN_CASES))
def test_attn_temporal16(name, dt):
    ops, dtype = _ops(), DTYPES[dt]
    shape, maxt = ATTN_CASES[name]
    B, T, H, W, Cc = shape
    assert maxt == (32 if T <= 32 else 128 if T <= 128 else 512), "T misses its MAXT bracket"
    # q.k / sqrt(C) has standard deviation s^2 / 3 for q, k uniform in [-s, s]: s^2 = 4.5 -> 1.5
    s = 4.5 ** 0.5
    q, k = (_rand(shape, dtype, 34 + i, s) for i in range(2))
    v = _rand(shape, dtype, 36, 1.0, 0.5)
    o = ops.attn_temporal(q, k, v)
    r, E, pmax = KB.attn_temporal_reference(q, k, v)
    assert 2.0 / T < pmax < 0.9, f"softmax is flat or one-hot (mean max p {pmax:.3f})"
    failed = _gates(f"attn_temporal/{name}/{dt}", o, r, E, dtype, mean_max_p=pmax)
    assert not failed, "; ".join(failed)


# ------------------------------------------------------------------------------------------ tap-stacked conv_out kernel
# Bound: kernel_bounds.conv_stacked_bound, E = u (2 KT ceil(Cin / 16) + 10) S,  S = sum |x w| + |bias|.
# name: (input [B,T,H,W,Cin], Cout, KT, time offset, pad_t, form); "framed": the SD3 decoder's call - the
# empty_padded buffer after replicate_border, offset (-tl, 0, 0) - against the conv of the interior with replicate padding
STK_CASES = {
    "causal_c3": ((1, 3, 23, 47, 128), 3, 3, -2, PAD_REPLICATE, "plain"),
    "noncausal_c4_b2": ((2, 3, 21, 37, 128), 4, 3, -1, PAD_ZERO, "plain"),
    "cin96_c3": ((1, 2, 17, 33, 96), 3, 3, -2, PAD_REPLICATE, "plain"),
    "cout1": ((1, 2, 13, 31, 128), 1, 3, -1, PAD_ZERO, "plain"),
    "sd3_framed_causal_c3": ((1, 3, 23, 47, 128), 3, 3, -2, PAD_REPLICATE, "framed"),
    "sd3_framed_noncausal_c3_b2": ((2, 3, 19, 41, 128), 3, 3, -1, PAD_REPLICATE, "framed"),
    "sd3_framed_cin96_c4": ((1, 2, 11, 62, 96), 4, 3, -2, PAD_REPLICATE, "framed"),
}


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("name", list(STK_CASES))
def test_conv_stacked16(name, dt):
    ops, dtype = _ops(), DTYPES[dt]
    shape, cout, kt, off_t, pad_t, form = STK_CASES[name]
    B, T, H, W, Ci = shape
    assert H % 10 and W % 30, "the output fills whole 10 x 30 tiles"
    x = _rand(shape, dtype, 50)
    w = _rand((kt * 9, cout, Ci), dtype, 51, (kt * 9 * Ci) ** -0.5 * 2)
    stk = torch.zeros((kt, 80, Ci), dtype=dtype, device=DEV)
    stk[:, :72].view(kt, 9, 8, Ci)[:, :, :cout] = w.view(kt, 9, cout, Ci)
    bias = _rand((cout,), torch.float32, 52, 0.3)
    ys = []
    if form == "framed":
        pad, inner = ops.empty_padded(B, T, H, W, Ci, dtype, DEV)
        inner.copy_(x)
        ops.replicate_border(pad)
        off = (off_t, 0, 0)
        assert off[1] >= 0 and off[2] >= 0 and pad.shape[2:4] == (H + 2, W + 2), "input is not framed"
        # PAD_ZERO as the engine passes it, and PAD_REPLICATE, which runs the host's framed-input check: same launch
        for pad_hw in (PAD_ZERO, PAD_REPLICATE):
            y = torch.zeros((B, cout, T, H, W), dtype=dtype, device=DEV)
            ops.conv_stacked(pad, stk, bias, kt=kt, cout=cout, offset=off, pad_t=pad_t, pad_hw=pad_hw, out=y.permute(0, 2, 3, 4, 1))
            ys.append(y)
    else:
        y = torch.zeros((B, cout, T, H, W), dtype=dtype, device=DEV)
        ops.conv_stacked(x, stk, bias, kt=kt, cout=cout, offset=(off_t, -1, -1), pad_t=pad_t, out=y.permute(0, 2, 3, 4, 1))
        ys.append(y)
    torch.cuda.synchronize()
    if len(ys) == 2:
        assert torch.equal(ys[0], ys[1]), "framed input: PAD_ZERO and PAD_REPLICATE launches differ"
    y = ys[0].permute(0, 2, 3, 4, 1)
    kw = dict(kernel=(kt, 3, 3), offset=(off_t, -1, -1), pad_t=pad_t, pad_hw=PAD_REPLICATE if form == "framed" else PAD_ZERO)
    f64 = FakeOps(torch.float64)
    r = f64.conv(x, w, bias, out=torch.zeros(y.shape, dtype=torch.float64, device=DEV), **kw)
    S = f64.conv(x.abs(), w.abs(), bias.abs(), out=torch.zeros(y.shape, dtype=torch.float64, device=DEV), **kw)
    E = KB.conv_stacked_bound(S, kt, Ci)
    failed = _gates(f"conv_stacked/{name}/{dt}", y, r, E, dtype)
    assert not failed, "; ".join(failed)


# ------------------------------------------------------------------------------------- pack_taps_hw + KT x 1 x 1 conv_in
@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("cin,cp,pad_hw", [(3, 32, PAD_ZERO), (3, 32, PAD_REPLICATE), (4, 64, PAD_ZERO)])
def test_pack_taps_hw_conv_in16(cin, cp, pad_hw, dt):
    """The gather bit for bit; the conv over the packed tensor under gate 1 of test_gpu_conv_plans.py (K = 3 cp)."""
    ops, dtype = _ops(), DTYPES[dt]
    fake, f64 = FakeOps(), FakeOps(torch.float64)
    x = _rand((2, cin, 5, 21, 30), dtype, 100).permute(0, 2, 3, 4, 1)
    got = torch.full((2, 5, 21, 30, cp), float("nan"), dtype=dtype, device=DEV)
    want = torch.empty_like(got)
    ops.pack_taps_hw(x, got, 3, 3, offset=(-1, -1), pad_hw=pad_hw)
    fake.pack_taps_hw(x, want, 3, 3, offset=(-1, -1), pad_hw=pad_hw)
    torch.cuda.synchronize()
    assert torch.equal(got, want), "pack_taps_hw"
    co = 128
    w5 = _rand((co, cin, 3, 3, 3), dtype, 101, 0.2)
    b = _rand((co,), torch.float32, 102, 0.1)
    wp = torch.zeros((3, co, cp), dtype=dtype, device=DEV)
    wp[:, :, :9 * cin] = w5.permute(2, 0, 3, 4, 1).reshape(3, co, 9 * cin)
    y = torch.zeros((2, 5, 21, 30, co), dtype=dtype, device=DEV)
    ops.conv(got, wp, b, kernel=(3, 1, 1), offset=(-2, 0, 0), pad_t=PAD_REPLICATE, out=y, force="tc")
    kw = dict(kernel=(3, 3, 3), offset=(-2, -1, -1), pad_t=PAD_REPLICATE, pad_hw=pad_hw)
    r = f64.conv(x, f64.pack_weight(w5), b, out=torch.zeros(y.shape, dtype=torch.float64, device=DEV), **kw)
    S = f64.conv(x.abs(), f64.pack_weight(w5).abs(), b.abs(), out=torch.zeros(y.shape, dtype=torch.float64, device=DEV), **kw)
    E = CP.C_ACC * U32 * math.sqrt(3 * cp) * S
    failed = _gates(f"conv_in_packed/cin{cin}_cp{cp}_pad{pad_hw}/{dt}", y, r, E, dtype)
    assert not failed, "; ".join(failed)


# ----------------------------------------------------------------------------------------------------------- data movers
@pytest.mark.parametrize("dt", sorted(DTYPES))
def test_movers16_bit_exact(dt):
    ops, fake, dtype = _ops(), FakeOps(), DTYPES[dt]
    a = _rand((1, 8, 3, 20, 24), dtype, 41)           # NCDHW tiles as the wrapper holds them
    b = _rand((1, 8, 3, 20, 24), dtype, 42)
    for axis in (0, 1):
        got, want = b.clone(), b.clone()
        ops.blend(a.permute(0, 2, 3, 4, 1), got.permute(0, 2, 3, 4, 1), 6, axis)
        fake.blend(a.permute(0, 2, 3, 4, 1), want.permute(0, 2, 3, 4, 1), 6, axis)
        torch.cuda.synchronize()
        assert torch.equal(got, want), f"blend axis {axis}"
    pad = _rand((2, 2, 12, 17, 24), dtype, 43)
    want = pad.clone()
    ops.replicate_border(pad)
    fake.replicate_border(want)
    torch.cuda.synchronize()
    assert torch.equal(pad, want), "replicate_border"
    # NCDHW -> NCDHW window (the wrapper's tile assembly): 16-byte row path and element path
    for w0, d0 in ((0, 16), (3, 5)):
        src = _rand((1, 3, 4, 16, 48), dtype, 44)
        dst = torch.zeros((1, 3, 4, 32, 64), dtype=dtype, device=DEV)
        ops.copy(src[..., w0:w0 + 40].permute(0, 2, 3, 4, 1), dst[:, :, :, 8:24, d0:d0 + 40].permute(0, 2, 3, 4, 1))
        want = torch.zeros_like(dst)
        want[:, :, :, 8:24, d0:d0 + 40] = src[..., w0:w0 + 40]
        torch.cuda.synchronize()
        assert torch.equal(dst, want), f"copy window {w0} -> {d0}"
    # strided channels-last copy, and a channels-first gather into a wider channel-padded buffer
    cl = _rand((1, 2, 10, 12, 64), dtype, 45)[:, :, 1:9, 2:10]
    out = torch.empty(cl.shape, dtype=dtype, device=DEV)
    ops.copy(cl, out)
    x = _rand((1, 3, 2, 10, 12), dtype, 46).permute(0, 2, 3, 4, 1)
    g = torch.full((1, 2, 10, 12, 8), float("nan"), dtype=dtype, device=DEV)
    ops.copy(x, g)
    torch.cuda.synchronize()
    assert torch.equal(out, cl), "strided copy"
    assert torch.equal(g[..., :3], x) and (g[..., 3:] == 0).all(), "channel gather"


# ----------------------------------------------------------------------------------------------------------- blocks bf16
@pytest.mark.parametrize("name", sorted(BC.cases()))
def test_block_bf16(name):
    """The block cases against the fp32 oracle block: the fp16 gate of test_gpu_blocks.py (mean 6e-4, max 1e-2) times
    2^-8 / 2^-11 = 8, bf16's larger rounding after each kernel."""
    got, want = BC.run_case(name, _ops(), torch.bfloat16, DEV)
    assert got.shape == want.shape and torch.isfinite(got).all()
    err = (got - want).abs()
    scale = want.abs().mean().item()
    rec = {"max_abs_err": err.max().item(), "mean_abs_err": err.mean().item(), "mean_abs_ref": scale}
    _RECORD[f"block_bf16/{name}"] = rec
    _dump()
    assert rec["mean_abs_err"] <= 8 * 6e-4 * max(scale, 1.0) and rec["max_abs_err"] <= 8 * 1e-2 * max(scale, 1.0), rec

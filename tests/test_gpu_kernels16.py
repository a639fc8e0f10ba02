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
import test_gpu_conv_plans as CP
import test_gpu_ops
from fake_ops import PAD_REPLICATE, PAD_ZERO, FakeOps
from test_gpu_fp32 import _ulp as _ulp_p

pytestmark = pytest.mark.gpu
DEV = "cuda"
OUT = test_gpu_ops.OUT
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
U32 = 2.0 ** -24   # unit roundoff of fp32

# Gate 2.  The kernel's fp32 value c is within E of r, so it rounds to a different 16-bit number than r only when a
# rounding midpoint lies between them: for r placed at random on the 16-bit grid that happens with probability
# |c - r| / ulp <= E / ulp.  mean(min(1, E / ulp)) therefore over-estimates the mismatch rate (E is a worst case); the
# margin covers the sampling noise of cases with few elements.  A truncating store mismatches ~50 %.  Where E is far
# above the typical error (a sum of n roundings is typically sqrt(n) times below its bound: conv_stacked's 58-term
# bound puts the estimate at 0.3-0.45 for fp16), the estimate says little, so the gate never asks for less than
# SHARE_FLOOR, which a truncating store still misses by half.
MISMATCH_MARGIN = 2.0
SHARE_FLOOR = 0.75
# Gate 3.  Correct rounding has mean signed error ~0 +- 0.3 / sqrt(n) ulp; directed rounding gives +-0.5 ulp.
MAX_MEAN_ULP = 0.05
_RECORD = {}


def _ops():
    from cvvae_b200.ops import CudaOps
    return CudaOps()


def _rand(shape, dtype, seed, scale=1.0, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) * scale + offset).to(dtype).to(DEV)


def _ulp(r, dtype):
    """Spacing of `dtype` numbers at |r| (r float64), from the exponent bits (test_gpu_fp32._ulp)."""
    return _ulp_p(r, 11, -14) if dtype == torch.float16 else _ulp_p(r, 8, -126)


def _dump():
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "kernels16.json"), "w") as f:
        json.dump(_RECORD, f, indent=1, sort_keys=True)


def _gates(tag, y, r, E, dtype, **extra):
    """Gates 1-3 on a 16-bit result y against its fp64 reference r and fp32 error bound E; records, returns failures."""
    yd = y.double()
    ulp = _ulp(r, dtype)
    err = yd - r
    ratio = (err.abs() / (0.5 * ulp + E)).max().item()
    rn = torch.round(r / ulp) * ulp                     # r / ulp is exact in fp64; round half to even
    share = (yd == rn).double().mean().item()
    est = (E / ulp).clamp(max=1.0).mean().item()
    min_share = max(1.0 - MISMATCH_MARGIN * est, SHARE_FLOOR)
    mean_ulp = (err / ulp).mean().item()
    failed = []
    if not ratio <= 1.0:
        failed.append(f"1: |y - r| exceeds the bound by {ratio:.3f}x")
    if not share >= min_share:
        failed.append(f"2: {share:.4f} correctly rounded < {min_share:.4f}")
    if not abs(mean_ulp) <= MAX_MEAN_ULP:
        failed.append(f"3: mean signed error {mean_ulp:+.4f} ulp")
    _RECORD[tag] = {"numel": y.numel(), "worst_bound_ratio": ratio, "correctly_rounded_share": share,
                    "mismatch_est": est, "min_share": min_share, "mean_signed_ulp": mean_ulp, "failed_gates": failed, **extra}
    _dump()
    return [f"{tag}: {f}" for f in failed]


# ------------------------------------------------------------------------------------------------------------ GroupNorm
# Statistics pass (gn_stats_kernel): each thread sums its 8 channels over P_t = ceil(ppb / lanes) positions in fp32
# (lanes = 256 / (C / 8) positions per sweep, ppb positions per CTA: pick_grid), then folds min(cpg, 8) channel sums into
# each of its groups; the square of a 16-bit value is exact in fp32.  Recursive summation of n terms is off by at most
# n u sum|x_i|, so with eps_sum = (P_t + 7) u the sums are off by eps_sum sum|x| and eps_sum sum x^2.  Each partial is then
# rounded to the fixed point (1/2 * 2^-20 for the sum, 1/2 * 2^-18 for the squares); a group receives nblocks * lanes *
# ceil(cpg / 8) partials, N_c per element (fix below).  The block and device sums are exact integers, and the apply
# kernel turns them into mean and variance in fp64:
#     dm   = eps_sum E|x|  + 2^-21 N_c            dsq = eps_sum E[x^2] + 2^-19 N_c
#     var  = E[x^2] - mean^2  ->  dvar = dsq + 2 |mean| dm + dm^2
#     z = (x - mean) rstd     ->  dz   = 1/2 dvar / (var + eps) |z| (1.01: second order) + dm rstd
# For an input whose mean is k standard deviations, dvar ~ eps_sum sigma^2 (1 + k^2 + 2 k sqrt(1 + k^2)) ~ 3 k^2 eps_sum
# sigma^2: z is off by ~1.5 k^2 eps_sum |z|, 2^-14 |z| at k = 5 and C = 128 (P_t = 16): the large-mean case checks it.
# Statistics handed in through stats= (exact fp64 sums rounded once to the fixed point): dm = 2^-21 / cnt,
# dsq = 2^-19 / cnt.
# The apply kernel rounds rstd and mean to fp32, forms a = rstd gamma and b = beta - mean a in fp32 and stores
# fma(x, a, b): at most 6 roundings of terms of size |gamma| (|z| + k) or |beta| + |gamma| k, under
# 2^-21 (|gamma| (|z| + 2k + 1) + |beta|).  SiLU has slope in [-0.1, 1.1] and __expf / __fdividef / the add cost under
# 2^-18 |y| for |pre| <= 10.  E = |gamma| dz + 2^-21 (...), times 1.1 plus 2^-18 |r| with SiLU; then the 16-bit store.
def _gn_reference(x, gamma, beta, G, eps, per_frame, silu, eps_sum, fix):
    B, T, H, W, Cc = x.shape
    cpg = Cc // G
    xd = x.double()
    v = xd.reshape(B * T, H * W, G, cpg) if per_frame else xd.reshape(B, T * H * W, G, cpg)
    mean = v.mean(dim=(1, 3), keepdim=True)
    var = v.var(dim=(1, 3), unbiased=False, keepdim=True)
    sd = torch.sqrt(var + eps)
    z = (v - mean) / sd
    if eps_sum is None:                                    # exact statistics through stats=
        cnt = v.shape[1] * cpg
        dm, dsq = 2.0 ** -21 / cnt, 2.0 ** -19 / cnt
    else:
        dm = eps_sum * v.abs().mean(dim=(1, 3), keepdim=True) + 2.0 ** -21 * fix
        dsq = eps_sum * (v * v).mean(dim=(1, 3), keepdim=True) + 2.0 ** -19 * fix
    dvar = dsq + 2 * mean.abs() * dm + dm * dm
    k = mean.abs() / sd
    dz = 0.5 * 1.01 * dvar / (var + eps) * z.abs() + dm / sd
    gam = gamma.double().view(1, 1, G, cpg)
    bet = beta.double().view(1, 1, G, cpg)
    pre = z * gam + bet
    E = gam.abs() * dz + 2.0 ** -21 * (gam.abs() * (z.abs() + 2 * k + 1) + bet.abs())
    r = pre
    if silu:
        r = pre * torch.sigmoid(pre)
        E = 1.1 * E + 2.0 ** -18 * r.abs()
    return r.reshape(x.shape), E.reshape(x.shape), k.max().item()


def _gn_geometry(shape, per_frame):
    """pick_grid / gn_*_kernel: positions per CTA, positions per sweep, CTAs, positions in the last CTA."""
    B, T, H, W, Cc = shape
    pix = H * W if per_frame else T * H * W
    ppb = max(256, -(-pix // 1184))
    lanes = 256 // (Cc // 8)
    nblocks = -(-pix // ppb)
    return pix, ppb, lanes, nblocks, pix - (nblocks - 1) * ppb


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
    pix, ppb, lanes, nblocks, n_last = _gn_geometry(shape, per_frame)
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
    eps_sum = (-(-ppb // lanes) + 7) * U32
    fix = nblocks * lanes * -(-cpg // 8) / (pix * cpg)
    y = ops.groupnorm(x, gam, bet, G, eps, per_frame=per_frame, silu=silu)
    r, E, k = _gn_reference(x, gam, bet, G, eps, per_frame, silu, eps_sum, fix)
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
        r2, E2, _ = _gn_reference(x, gam, bet, G, eps, False, silu, None, None)
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
# One warp per token, two-pass fp32 statistics: the sum over C is off by (C / 32 + 5) u sum|x|, mean = sum / C exact (C a
# power of two), the squared deviations by (C / 32 + 7) u, rsqrtf 2 ulp, then (x - mean) rstd gamma + beta in <= 4
# roundings: for inputs with |mean| <= sigma, E <= 2^-19 (|gamma| (1 + |z|) + |beta|).  The fp32 form of
# test_gpu_fp32._norm_bound, 2^-16 (|gamma| (1 + |z|) + |beta|), covers it.
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
    xd = x.double()
    z = (xd - xd.mean(-1, keepdim=True)) / torch.sqrt(xd.var(-1, unbiased=False, keepdim=True) + 1e-5)
    r = z * gam.double() + bet.double()
    E = 2.0 ** -16 * (gam.double().abs() * (1 + z.abs()) + bet.double().abs())
    failed = _gates(f"layernorm/C{Cc}/{dt}", y, r, E, dtype)
    assert not failed, "; ".join(failed)


# ---------------------------------------------------------------------------------------------------------- softmax_rows
# test_gpu_fp32's softmax bound: __expf(s - m) is within 2^-22 + 2.5 u |s - m| relative; the row sum adds at most
# cols / 1024 + 2 (vector path) or cols / 256 (scalar path) terms per thread plus 13 in the warp and block reductions, under
# 92 u = 2^-17.5 at 20 000 columns; 1 / sum and the product two more roundings:  E = 2^-18 r (4 + |s - m|).
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
    sd = s[:, :cols].double()
    r = torch.softmax(sd, dim=-1)
    E = 2.0 ** -18 * r * (4 + (sd - sd.max(-1, keepdim=True).values).abs())
    failed = _gates(f"softmax_rows/{name}/{dt}", p[:, :cols], r, E, dtype)
    # columns between cols and ld, and the buffer outside the rows, are left untouched
    untouched = torch.cat([p[:, cols:].flatten(), p_buf[:o], p_buf[o + rows * ld_p:]])
    assert (untouched == sentinel).all(), "softmax_rows wrote outside its columns"
    assert not failed, "; ".join(failed)


# -------------------------------------------------------------------------------------------------- temporal attention
# One warp per position, fp32 throughout.  Scores: each lane adds n1 = 8 ceil(C / 256) products, then 5 shuffle adds, the
# scale and its own rounding: |ds| <= (n1 + 7) u A_i, A_i = max_j C^-0.5 sum_c |q_ic k_jc|.  A probability is off by
# 2 |ds| (its score and the max), 2.5 u |s - m| <= 5 u A_i (subtraction, __expf's argument scaling), 2^-22 (ex2.approx),
# (T - 1) u (the sum over T) and 2 u (1 / sum, the product); the value sum is an fma chain over T frames, T u sum p |v|:
#     E = u ((2 n1 + 19) A_i + 2 T + 5) sum_j p_ij |v_j|.
# At T = 5, C = 512 this is the fp32 file's 2^-16 (1 + A_i) sum p |v| to within 20 %; it grows with T.
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
    qd, kd, vd = (t.double().permute(0, 2, 3, 1, 4).reshape(B * H * W, T, Cc) for t in (q, k, v))
    a = torch.softmax(qd @ kd.transpose(1, 2) * Cc ** -0.5, dim=-1)
    pmax = a.amax(-1).mean().item()
    assert 2.0 / T < pmax < 0.9, f"softmax is flat or one-hot (mean max p {pmax:.3f})"
    A = ((qd.abs() @ kd.abs().transpose(1, 2)) * Cc ** -0.5).amax(-1, keepdim=True)
    n1 = 8 * -(-Cc // 256)
    E = U32 * ((2 * n1 + 19) * A + 2 * T + 5) * (a @ vd.abs())
    back = lambda t: t.reshape(B, H, W, T, Cc).permute(0, 3, 1, 2, 4)
    failed = _gates(f"attn_temporal/{name}/{dt}", o, back(a @ vd), back(E), dtype, mean_max_p=pmax)
    assert not failed, "; ".join(failed)


# ------------------------------------------------------------------------------------------ tap-stacked conv_out kernel
# conv_stk accumulates, per tap column, KT ceil(Cin / 16) wgmmas of K = 16 (each adds exact 16-bit products with at most
# one truncation, 2^-23 S: gate 1 of test_gpu_conv_plans.py), then sums the 9 shifted tap partials in fp32 (9 u S) and adds
# the bias (u S):  E = u (2 KT ceil(Cin / 16) + 10) S,  S = sum |x w| + |bias|.  (A single chain over all 9 KT Cin
# products would need gate 1's 16 sqrt(K) = 940 u S at KT = 3, Cin = 128; the split keeps it at 58 u S.)
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
    E = U32 * (2 * kt * -(-Ci // 16) + 10) * S
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

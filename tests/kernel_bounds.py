"""fp32 error bounds of the kernels around the convolution, and the gates that apply them to a 16-bit result.

Shared by tests/test_gpu_kernels16.py (each kernel at picked shapes), tests/test_gpu_attention16.py (the launches of the
attention blocks) and tests/network_audit.py (every launch of a network pass).  The conv_tc GEMM bounds, the gates
accumulated over pieces of a result and the fused-statistics gate live in tests/attention_gates.py and are re-exported.

Reference: the operation in fp64 on the same 16-bit inputs.  Gates, one per class of defect:
  1. per element  |y - r| <= 1/2 ulp_dt(r) + E, E the kernel's fp32 computation error bound, derived next to each
     kernel below                                                             (wrong value, lost term, bad statistics)
  2. share of elements equal to r rounded once to the dtype >= 1 - MISMATCH_MARGIN * mean(min(1, E / ulp_dt(r)))
                                                                              (truncating or mis-rounding store)
  3. |mean((y - r) / ulp_dt(r))| <= MAX_MEAN_ULP                             (directed rounding, biased shift or scale)
"""
import torch

from attention_gates import TF32, Gates, gemm_bound, logit_bound, softmax_bound, stats_gate  # noqa: F401  (re-exported)
from test_gpu_fp32 import _ulp as _ulp_p

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


def _ulp(r, dtype):
    """Spacing of `dtype` numbers at |r| (r float64), from the exponent bits (test_gpu_fp32._ulp); dtype TF32: the
    store format of fp32 outputs read only by tensor-core products (p = 11, e_min = -126)."""
    if dtype == TF32:
        return _ulp_p(r, 11, -126)
    return _ulp_p(r, 11, -14) if dtype == torch.float16 else _ulp_p(r, 8, -126)


def _gates(y, r, E, dtype):
    """Gates 1-3 on a 16-bit result y against its fp64 reference r and fp32 error bound E: ({measured values}, [failures])."""
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
    rec = {"numel": y.numel(), "worst_bound_ratio": ratio, "correctly_rounded_share": share, "mismatch_est": est,
           "min_share": min_share, "mean_signed_ulp": mean_ulp, "failed_gates": failed}
    return rec, failed


# ------------------------------------------------------------------------------------------------------------ GroupNorm
# Statistics pass (gn_stats_kernel): each thread sums its 8 channels over P_t = ceil(ppb / lanes) positions in fp32
# (lanes = 256 / (C / 8) positions per sweep, ppb positions per CTA: pick_grid), then folds min(cpg, 8) channel sums into
# each of its groups; the square is exact: a 16-bit value's square fits in fp32, and for fp32 inputs q = fmaf(f, f, q)
# forms it exactly inside the fma, so in either case each term costs one rounding of the running sum.  Recursive summation of n terms is off by at most
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
def gn_pointwise(v, mean, var, absmean, sqmean, gamma, beta, eps, silu, eps_sum, fix):
    """The bound above on v [units, positions, G, cpg] (fp64) with its group moments ([units, 1, G, 1]: mean, variance,
    E|x|, E[x^2]; the last two unused for handed-in statistics, eps_sum None).  Returns (r, E, max k) in v's shape."""
    G, cpg = v.shape[2], v.shape[3]
    sd = torch.sqrt(var + eps)
    z = (v - mean) / sd
    if eps_sum is None:                                    # exact statistics through stats=
        cnt = fix
        dm, dsq = 2.0 ** -21 / cnt, 2.0 ** -19 / cnt
    else:
        dm = eps_sum * absmean + 2.0 ** -21 * fix
        dsq = eps_sum * sqmean + 2.0 ** -19 * fix
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
    return r, E, k.max().item()


def gn_reference(x, gamma, beta, G, eps, per_frame, silu, eps_sum, fix):
    """GroupNorm (+ SiLU) of x [B,T,H,W,C] in fp64 and the bound E above; eps_sum None: statistics handed in.
    Returns (r, E, max k) in x's shape."""
    B, T, H, W, Cc = x.shape
    cpg = Cc // G
    xd = x.double()
    v = xd.reshape(B * T, H * W, G, cpg) if per_frame else xd.reshape(B, T * H * W, G, cpg)
    mean = v.mean(dim=(1, 3), keepdim=True)
    var = v.var(dim=(1, 3), unbiased=False, keepdim=True)
    if eps_sum is None:
        absmean = sqmean = None
        fix = v.shape[1] * cpg
    else:
        absmean = v.abs().mean(dim=(1, 3), keepdim=True)
        sqmean = (v * v).mean(dim=(1, 3), keepdim=True)
    r, E, k = gn_pointwise(v, mean, var, absmean, sqmean, gamma, beta, eps, silu, eps_sum, fix)
    return r.reshape(x.shape), E.reshape(x.shape), k


def gn_geometry(shape, per_frame):
    """pick_grid / gn_*_kernel: positions per CTA, positions per sweep, CTAs, positions in the last CTA."""
    B, T, H, W, Cc = shape
    pix = H * W if per_frame else T * H * W
    ppb = max(256, -(-pix // 1184))
    lanes = 256 // (Cc // 8)
    nblocks = -(-pix // ppb)
    return pix, ppb, lanes, nblocks, pix - (nblocks - 1) * ppb


def gn_sum_terms(shape, per_frame, groups):
    """(eps_sum, fix, P_t) of the kernel-statistics bound for a launch on `shape`: P_t fp32 terms per thread."""
    pix, ppb, lanes, nblocks, _ = gn_geometry(shape, per_frame)
    cpg = shape[4] // groups
    p_t = -(-ppb // lanes)
    return (p_t + 7) * U32, nblocks * lanes * -(-cpg // 8) / (pix * cpg), p_t


# ------------------------------------------------------------------------------------------------------------ LayerNorm
# One warp per token, two-pass fp32 statistics: the sum over C is off by (C / 32 + 5) u sum|x|, mean = sum / C exact (C a
# power of two), the squared deviations by (C / 32 + 7) u, rsqrtf 2 ulp, then (x - mean) rstd gamma + beta in <= 4
# roundings: for inputs with |mean| <= sigma, E <= 2^-19 (|gamma| (1 + |z|) + |beta|).  The fp32 form of
# test_gpu_fp32._norm_bound, 2^-16 (|gamma| (1 + |z|) + |beta|), covers it.
# A token whose mean is k = |mean| / sigma > 1 standard deviations (norm_t's inputs need not be centred): the mean is the
# only statistic whose error grows with k.  dm = (C / 32 + 5) u E|x| <= (C / 32 + 5) u sigma sqrt(1 + k^2), and it shifts
# z by dm / sigma <= 21 u (1 + k) at C = 512.  The second pass sums (x - mean~)^2 = (x - mean)^2 + dm^2 on average (the
# cross term sums to zero), so the variance gains only dm^2, and the terms the store rounds, |gamma z| and |beta|, do not
# depend on k.  The 2^-16 |gamma| term (256 u |gamma|) holds the k <= 1 terms with room; replacing it by
# 2^-16 |gamma| max(1, k) covers 21 u (1 + k) + 2^-19 for every k >= 1 (256 k >= 29.7 k + 32).
def layernorm_reference(x, gamma, beta, eps):
    """LayerNorm over the channels of x in fp64, and the bound above.  Returns (r, E, max k)."""
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    sd = torch.sqrt(xd.var(-1, unbiased=False, keepdim=True) + eps)
    z = (xd - mean) / sd
    k = mean.abs() / sd
    r = z * gamma.double() + beta.double()
    E = 2.0 ** -16 * (gamma.double().abs() * (k.clamp_min(1.0) + z.abs()) + beta.double().abs())
    return r, E, k.max().item()


# ---------------------------------------------------------------------------------------------------------- softmax_rows
# test_gpu_fp32's softmax bound: __expf(s - m) is within 2^-22 + 2.5 u |s - m| relative; the row sum adds at most
# cols / 1024 + 2 (vector path) or cols / 256 (scalar path) terms per thread plus 13 in the warp and block reductions, under
# 92 u = 2^-17.5 at 20 000 columns; 1 / sum and the product two more roundings:  E = 2^-18 r (4 + |s - m|)
# (attention_gates.softmax_bound).
def softmax_reference(s, cols):
    """softmax over the first `cols` columns of the fp32 rows s, in fp64, and its bound.  Returns (r, E)."""
    sd = s[:, :cols].double()
    r = torch.softmax(sd, dim=-1)
    return r, softmax_bound(sd, r)


# -------------------------------------------------------------------------------------------------- temporal attention
# One warp per position, fp32 throughout.  Scores: each lane adds n1 = 8 ceil(C / 256) products, then 5 shuffle adds, the
# scale and its own rounding: |ds| <= (n1 + 7) u A_i, A_i = max_j C^-0.5 sum_c |q_ic k_jc|.  A probability is off by
# 2 |ds| (its score and the max), 2.5 u |s - m| <= 5 u A_i (subtraction, __expf's argument scaling), 2^-22 (ex2.approx),
# (T - 1) u (the sum over T) and 2 u (1 / sum, the product); the value sum is an fma chain over T frames, T u sum p |v|:
#     E = u ((2 n1 + 19) A_i + 2 T + 5) sum_j p_ij |v_j|.
# At T = 5, C = 512 this is the fp32 file's 2^-16 (1 + A_i) sum p |v| to within 20 %; it grows with T.
def attn_temporal_reference(q, k, v):
    """softmax(C^-1/2 q k^T) v over the frames of each position, q / k / v [B,T,H,W,C], in fp64, and the bound above.
    Returns (r, E, mean max probability) in q's shape."""
    B, T, H, W, Cc = q.shape
    qd, kd, vd = (t.double().permute(0, 2, 3, 1, 4).reshape(B * H * W, T, Cc) for t in (q, k, v))
    a = torch.softmax(qd @ kd.transpose(1, 2) * Cc ** -0.5, dim=-1)
    pmax = a.amax(-1).mean().item()
    A = ((qd.abs() @ kd.abs().transpose(1, 2)) * Cc ** -0.5).amax(-1, keepdim=True)
    n1 = 8 * -(-Cc // 256)
    E = U32 * ((2 * n1 + 19) * A + 2 * T + 5) * (a @ vd.abs())
    back = lambda t: t.reshape(B, H, W, T, Cc).permute(0, 3, 1, 2, 4)
    return back(a @ vd), back(E), pmax


# ------------------------------------------------------------------------------------------ tap-stacked conv_out kernel
# conv_stk accumulates, per tap column, KT ceil(Cin / 16) wgmmas of K = 16 (each adds exact 16-bit products with at most
# one truncation, 2^-23 S: gate 1 of test_gpu_conv_plans.py), then sums the 9 shifted tap partials in fp32 (9 u S) and adds
# the bias (u S):  E = u (2 KT ceil(Cin / 16) + 10) S,  S = sum |x w| + |bias|.  (A single chain over all 9 KT Cin
# products would need gate 1's 16 sqrt(K) = 940 u S at KT = 3, Cin = 128; the split keeps it at 58 u S.)
def conv_stacked_bound(S, kt, cin):
    return U32 * (2 * kt * -(-cin // 16) + 10) * S


def unstack_weight(w_stk, kt, cout):
    """[KT][80][Cin] (row (kh*3+kw)*8 + c) -> packed [KT*9][Cout][Cin] (fake_ops.FakeOps.conv_stacked)."""
    ci = w_stk.shape[2]
    return w_stk[:, :72].reshape(kt, 9, 8, ci)[:, :, :cout].reshape(kt * 9, cout, ci)

"""Error bounds and gates of the mid-block spatial attention (Engine.spatial_attention), shared by
tests/test_gpu_attention16.py (the kernels on the GPU) and tests/test_attention_gates_cpu.py (a CPU emulation of the
kernels' arithmetic, which checks the bounds themselves: a correctly rounded emulation passes, doctored outputs fail).

The attention runs as three batched conv_tc GEMMs and one softmax_rows per group of frames:
  v^T = W_v hn^T + b_v   (K = C, 16-bit out)      S = alpha q k^T   (K = C, fp32 out)
  P = softmax_rows(S)    (16-bit out)             O = P v           (K = N, 16-bit out)
Each wgmma adds 16 exact products of 16-bit values to the fp32 accumulator with at most one truncation, 2^-23 of the
running condition sum (test_gpu_conv_plans.py, gate 1), so a chain of ceil(K / 16) MMAs is off by at most
(K / 16) 2^-23 S.  This is the linear form from which that file's C_ACC = 16 sqrt(K) form is derived; unlike the sqrt(K)
form, it holds at any K (the attention reaches K = N = 14400).  The epilogue's fma(acc, alpha, bias) adds one fp32
rounding, and the bound allows a second one.

Gates, evaluated over a result that may arrive in pieces (row chunks, frames), as in tests/test_gpu_kernels16.py:
  1. per element  |y - r| <= 1/2 ulp_dt(r) + E          (the fp32 logits and end to end: |y - r| <= E, E complete)
  2. share of y equal to r rounded once >= max(1 - MISMATCH_MARGIN * mean(min(1, E / ulp)), SHARE_FLOOR)
  3. |mean(clamp((y - r) / ulp_dt(r), -1, 1)) - D| <= MAX_MEAN_ULP,  D = DRIFT_PER_K[dt] * K * mean(sign(r))
     (each element counts at most one ulp: where a sum cancels to nearly zero, E is many ulps of the result and its
     error in ulps says nothing about the store; a correctly rounded element is within 1/2 ulp + E)
Gate 3 is after a directed store.  The accumulators' truncations are directed too, toward zero, and over a long chain
they shift a result of one sign by a measured amount in proportion to K: O (positive, K = N) by -6.0e-6 N fp16 ulps
(-0.031 at N = 5184, -0.055 at 9216, -0.086 at 14400) and -6e-7 N bf16 ulps, on an H100 SXM (the same coefficient at
every N and at C = 128 and 512).  The gate takes that expected drift D off the mean and keeps MAX_MEAN_ULP for the rest,
so a store biased by a tenth of an ulp fails at any K.  For results of mixed sign (v^T, the block's convolutions) and
for short chains D is a few thousandths of an ulp.
Fused GroupNorm statistics (the blocks' proj_out / to_out.0): gate 5 of test_gpu_conv_plans.py against fp64 sums of the
stored output, and bit for bit equality with the register epilogue's, which is what sees one unit of the fixed-point
format (a single partial sum rounded the other way is already inside gate 5's tolerance).
"""
import torch

from test_gpu_conv_plans import MAX_MEAN_ULP, _ulp
from test_gpu_fp32 import _ulp as _ulp_p

U = 2.0 ** -24            # unit roundoff of fp32
MISMATCH_MARGIN = 2.0     # gate 2 of tests/test_gpu_kernels16.py
SHARE_FLOOR = 0.75
DRIFT_PER_K = {torch.float16: -6.0e-6, torch.bfloat16: -6.0e-7}   # gate 3: mean signed ulps per unit of K, measured
GN_SUM_SCALE, GN_SQ_SCALE = 2.0 ** 20, 2.0 ** 18                   # fixed point of the fused statistics
TF32 = "tf32"   # store format of fp32 outputs read only by tensor-core products: fp32 storage, rounded to nearest TF32

# fp32 models (TF32 products).  Each wgmma adds K = 8 exact products of two 11-bit significands (22 bits, exact in
# fp32), so the linear bound above holds with ceil(K / 8) MMAs.  A full-precision fp32 result (a conv or GEMM output, the
# temporal attention) is checked under gate 1 with 1/2 ulp_fp32 and two more gates:
#   F. the share of stored values whose low 13 mantissa bits are all zero is <= FULL_SHARE_MAX.  Generic fp32 values
#      give 2^-13; a store rounded or truncated to TF32 gives 100 %.
#   R. how the operands are read.  r is the fp64 product of the operands as the tensor core reads them (low 13 bits
#      truncated), r_rn the same with operands rounded to nearest.  Where the two readings differ by
#      sep = rms(r_rn - r) >= SEP_MIN rms(r), the result must be at least twice as close to r: rms(y - r) <= R_FRACTION
#      sep.  Gate 1 is a worst case ~10^3 x above the typical error and cannot see a systematic operand error; this can.
#      An operand with all its low bits set moves by one TF32 ulp (2^-11..2^-10 of its size) half the time, so
#      sep ~ 0.5 * 2^-10 rms(r) = 5e-4 rms(r) (5.0e-4 on the CPU doubles).  A kernel that reads the operands rounded to
#      nearest has rms(y - r) = sep.  A correct kernel: every wgmma truncates the accumulator toward zero, so the error
#      of a chain is a directed drift, linear in the number of MMAs rather than sqrt: rms(y - r) / rms(r) measured on
#      an H100 80GB HBM3 at 0.3 * 2^-24 ceil(K / 8) for convolutions (1.6e-5 at K = 6912, 3.0e-5 at K = 13824) and
#      0.93 * 2^-24 ceil(K / 8) for O = P v (3.6e-5 at K = N = 5184).  A fixed bound on rms(y - r) / rms(r) cannot
#      separate that drift from a wrong operand reading at the largest K (R_MAX = 2^-16, derived for a sqrt(K) error,
#      is exceeded by a correct kernel from K ~ 7000 on); the ratio to sep can: at SEP_MIN the gate allows
#      R_FRACTION SEP_MIN = 1.2e-4 rms(r), 3.4x the largest drift measured, and a rounding reader fails it by 2x at any
#      K.  Measured over the fp32 network audit (tests/test_gpu_network_audit32.py, H100 80GB HBM3): sep 2.4e-4 - 1.0e-3
#      on the gated launches, rms(y - r) / sep <= 0.103, 4.9x inside the gate.  A launch whose operands have (almost) no low bits has nothing to tell apart: sep and rms(y - r) / rms(r) are
#      recorded, not gated, and a TF32 store is gate F's (2^-11 / sqrt(12) rms(r) there).
# An MMA-only producer (GroupNorm, LayerNorm, softmax_rows) stores TF32 values: gates 1-3 with TF32 (p = 11,
# e_min = -126) as the store format, sharp there (the fp32 compute error, <~ 2^-16 relative, is far below the TF32 half
# ulp, 2^-12), and
#   T. every stored value has its low 13 mantissa bits zero.
SEP_MIN = 2.0 ** -12
R_FRACTION = 0.5
FULL_SHARE_MAX = 0.01


def kstep(dtype):
    """Products per wgmma of the operand dtype: 8 for fp32 storage (TF32), 16 for 16-bit operands."""
    return 8 if dtype == torch.float32 else 16


def n_mma(K, kstep=16):
    """MMAs of a chain over K, kstep products each (a ragged last block still costs one MMA per started kstep)."""
    return -(-K // kstep)


def gemm_bound(K, S, kstep=16):
    """fp32 error of a conv_tc GEMM over K before the store; S = sum |x w| + |bias| (fp64)."""
    return (2 * n_mma(K, kstep) + 2) * U * S


def logit_bound(K, alpha32, qk_abs, r, kstep=16):
    """|S - r| for the fp32 logits S = fma(acc, alpha32, 0), r = alpha32 q k^T, qk_abs = |q| |k|^T."""
    return (2 * n_mma(K, kstep) + 1) * U * alpha32 * qk_abs + U * r.abs()


def store_ulp(r, fmt):
    """Spacing of the store format at |r|: a 16-bit dtype, TF32 or torch.float32."""
    if fmt == TF32:
        return _ulp_p(r, 11, -126)
    if fmt == torch.float32:
        return _ulp_p(r, 24, -126)
    return _ulp(r, fmt)


def low13(y):
    """The low 13 mantissa bits of the fp32 tensor y (any strides), as int32: what a TF32 operand read drops."""
    return y.view(torch.int32) & 0x1FFF


def softmax_bound(s, r):
    """softmax_rows' fp32 error on rows s (fp64 copy of the fp32 logits), r = softmax(s) (tests/test_gpu_kernels16.py)."""
    return 2.0 ** -18 * r * (4 + (s - s.amax(-1, keepdim=True)).abs())


def stored_bound(r, E, dtype):
    """|y - r| for y the 16-bit store of a value within E of r: the rounding of a value up to |r| + E, plus E."""
    return E + 0.5 * _ulp(r.abs() + E, dtype)


def attention_reference(q, k, v, dv, alpha32, dtype):
    """softmax(C^-1/2 q k^T) v in fp64 for a chunk of query rows, and the bound E_i of the pipeline's 16-bit output.

    q [R, C] and k [N, C] are the 16-bit operands (as fp64), v [N, C] = hn W_v^T + b_v exactly, dv [N, C] bounds the
    stored v^T against v.  With delta_i the largest logit error of row i (the stage bound plus the rounding of alpha to
    fp32), the kernel's probabilities of the computed logits are within p (e^(2 delta) - 1) of p; softmax_rows adds
    2^-18 p~ (4 + |s~ - m~|) and the store 1/2 ulp:  |dP| <= p (e^(2 delta) - 1) + E_sm + 1/2 ulp(p e^(2 delta) + E_sm).
    Then  O - o = sum_j dP_ij (v_j + dv_j) + p_ij dv_j  plus the chain over K = N and the final store:
      E_i = sum_j |dP_ij| (|v_j| + dv_j) + sum_j p_ij dv_j + (N / 16) 2^-23 sum_j P_ij (|v_j| + dv_j) + 1/2 ulp(o_i)."""
    C, N = q.shape[1], k.shape[0]
    alpha = C ** -0.5
    qk = q @ k.T
    s = alpha * qk
    p = torch.softmax(s, dim=-1)
    o = p @ v
    d = (logit_bound(C, alpha32, q.abs() @ k.abs().T, alpha32 * qk) + abs(alpha32 - alpha) * qk.abs()).amax(-1, keepdim=True)
    del qk
    p_hi = p * torch.exp(2 * d)
    e_sm = 2.0 ** -18 * p_hi * (4 + (s - s.amax(-1, keepdim=True)).abs() + 2 * d)
    del s
    dP = p * torch.expm1(2 * d) + e_sm + 0.5 * _ulp(p_hi + e_sm, dtype)
    del p_hi, e_sm
    vabs = v.abs() + dv
    E = dP @ vabs + p @ dv + gemm_bound(N, (p + dP) @ vabs)
    return o, stored_bound(o, E, dtype)


class Gates:
    """Gates accumulated over pieces of one result.  dtype: the store format - a 16-bit dtype or TF32 (gates 1-3; TF32
    also gate T), torch.float32 (a full-precision fp32 result: gate 1 with 1/2 ulp_fp32, gates F and R, R only with
    rms), None (an fp32 result, gate 1 only, E complete).  half_ulp False: E already contains the final rounding (end to
    end), gates 2-3 are recorded but not applied.  K: the length of the accumulation chain, for gate 3's expected drift."""

    def __init__(self, dtype, half_ulp=True, K=0, rms=True):
        self.dtype, self.half_ulp, self.K, self.rms = dtype, half_ulp, K, rms
        self.n = self.n_rn = 0
        self.sum_ulp = self.sum_est = self.sum_sign = 0.0
        self.ratio = 0.0
        self.n_low_zero = self.n_low_set = 0
        self.sq_err = self.sq_ref = self.sq_sep = 0.0

    def add(self, y, r, E, r_rn=None):
        """r_rn (torch.float32 only): the reference with the operands rounded to nearest instead of truncated, where
        an operand has low bits (gate R)."""
        yd = y.double()
        err = yd - r
        if self.dtype is None:
            lim = E
        elif self.dtype == torch.float32:
            lim = 0.5 * store_ulp(r, self.dtype) + E
            self.n_low_zero += int((low13(y) == 0).sum().item())
            self.sq_err += (err * err).sum().item()
            self.sq_ref += (r * r).sum().item()
            if r_rn is not None:
                self.sq_sep += ((r_rn - r) ** 2).sum().item()
        else:
            ulp = store_ulp(r, self.dtype)
            lim = 0.5 * ulp + E if self.half_ulp else E
            self.n_rn += int((yd == torch.round(r / ulp) * ulp).sum().item())   # r / ulp exact; half to even
            self.sum_ulp += (err / ulp).clamp(-1.0, 1.0).sum().item()
            self.sum_est += (E / ulp).clamp(max=1.0).sum().item()
            self.sum_sign += torch.sign(r).sum().item()
            if self.dtype == TF32:
                self.n_low_set += int((low13(y) != 0).sum().item())
        m = (err.abs() / lim).max().item()
        if not m <= self.ratio:       # NaN sticks
            self.ratio = m
        self.n += r.numel()
        return self

    def result(self):
        """({measured values}, [failed gates])"""
        rec = {"numel": self.n, "worst_bound_ratio": self.ratio}
        failed = []
        if not self.ratio <= 1.0:
            failed.append(f"1: |y - r| exceeds the bound by {self.ratio:.3f}x")
        if self.dtype == torch.float32:
            share = self.n_low_zero / self.n
            rec["tf32_valued_share"] = share
            if not share <= FULL_SHARE_MAX:
                failed.append(f"F: {share:.4f} of the stored values have their low 13 bits zero")
            if self.rms:
                ref = self.sq_ref if self.sq_ref > 0 else float("nan")
                rr, sep = (self.sq_err / ref) ** 0.5, (self.sq_sep / ref) ** 0.5
                rec.update({"rms_error_ratio": rr, "rn_separation": sep})
                if sep >= SEP_MIN:
                    rec["error_over_separation"] = rr / sep
                    if not rr <= R_FRACTION * sep:
                        failed.append(f"R: rms(y - r) = {rr:.3g} rms(r), not below {R_FRACTION} x the "
                                      f"round-to-nearest reading's {sep:.3g}")
                elif rr != rr:
                    failed.append("R: rms(y - r) is NaN")
        elif self.dtype is not None:
            share = self.n_rn / self.n
            est = self.sum_est / self.n
            min_share = max(1.0 - MISMATCH_MARGIN * est, SHARE_FLOOR)
            mean_ulp = self.sum_ulp / self.n
            drift = DRIFT_PER_K.get(self.dtype, 0.0) * self.K * self.sum_sign / self.n
            rec.update({"correctly_rounded_share": share, "mismatch_est": est, "min_share": min_share,
                        "mean_signed_ulp": mean_ulp, "expected_drift_ulp": drift})
            if self.half_ulp and not share >= min_share:
                failed.append(f"2: {share:.4f} correctly rounded < {min_share:.4f}")
            if self.half_ulp and not abs(mean_ulp - drift) <= MAX_MEAN_ULP:
                failed.append(f"3: mean signed error {mean_ulp:+.4f} ulp, expected drift {drift:+.4f}")
            if self.dtype == TF32:
                rec["low_bits_set"] = self.n_low_set
                if self.n_low_set:
                    failed.append(f"T: {self.n_low_set} stored values have low 13 bits set (not TF32)")
        rec["failed_gates"] = failed
        return rec, failed


def row_chunks(n, rows):
    return [slice(i, min(n, i + rows)) for i in range(0, n, rows)]


def truncate(r, dtype):
    """r rounded toward zero to dtype (a doctored store), as fp64."""
    ulp = _ulp(r, dtype)
    return torch.trunc(r / ulp) * ulp


def branches(N):
    """What a token count reaches in the attention GEMMs (ld = ceil8(N) is the row stride of S, P and v^T)."""
    return {"ld_gt_n": N % 8 != 0, "odd_n": N % 2 == 1, "ragged_k_block": N % 64 != 0,
            "guarded_k_block": 0 < N % 64 <= 48,          # last K block of O has fewer than 4 MMAs
            "partial_channel_tile": N % 256 != 0}


def stats_gate(y, st, groups):
    """Gate 5 of test_gpu_conv_plans.py: fused statistics st [B, groups, 2] (fixed point) against fp64 sums of the
    stored y [B, ..., C].  Returns (max abs error, [failures])."""
    v = y.double().reshape(y.shape[0], -1, groups, y.shape[-1] // groups)
    return stats_compare(torch.stack([v.sum(dim=(1, 3)), (v * v).sum(dim=(1, 3))], dim=-1), st)


def stats_compare(want, st):
    """stats_gate against sums computed by the caller: want [B, groups, 2] (fp64 sum, sum of squares)."""
    got = torch.stack([st[..., 0].double() / GN_SUM_SCALE, st[..., 1].double() / GN_SQ_SCALE], dim=-1)
    try:
        torch.testing.assert_close(got, want, rtol=1e-5, atol=2e-2)
        failed = []
    except AssertionError as e:
        failed = [f"5: fused statistics vs fp64 sums of y: {str(e).splitlines()[0:4]}"]
    return (got - want).abs().max().item(), failed


def same_bits(a, b):
    """Two runs that must perform the same operations in the same order: equal outputs and statistics, bit for bit."""
    return all(torch.equal(x, z) for x, z in zip(a, b)) and len(a) == len(b)

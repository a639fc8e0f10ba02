"""Every launch of a network pass against its operation in fp64, one row per launch.

AuditOps wraps an operator set (cvvae_b200.ops.CudaOps on the GPU, a test double on the CPU); the model wrapper's
`_ops_factory` hook injects it, which also keeps CUDA graphs off.  For every call it
  1. snapshots what the call mutates: blend's b, the replicate_border buffer, the gn_stats accumulator, and any argument
     that shares storage with `out`;
  2. runs the call and synchronises;
  3. evaluates the same call in fp64 on the same 16-bit inputs and views, with the semantics of tests/fake_ops.py;
  4. applies that op's gates, records one row and frees everything, so memory stays bounded by one launch.

Gates per call (bounds in tests/kernel_bounds.py and tests/attention_gates.py):
  conv, 16-bit out      gates 1-3 (attention_gates.Gates) with E = gemm_bound(K, S); K = taps x Cin (+ C2 of a fused
                        shortcut, N for the P v GEMM), S the same conv on absolute values (+ |bias| + |residual|)
  conv, out_f32         gate 1 with logit_bound
  conv with gn_stats    also stats_gate on this launch's delta of the accumulator against fp64 sums over the view it
                        stored (chained launches add one lattice at a time)
  groupnorm             kernel statistics: gn_pointwise with this launch's geometry; handed-in stats=: normalised with
                        the fp64 mean and variance of the handed-in fixed-point sums (the apply kernel alone)
  layernorm, softmax_rows, attn_temporal, conv_stacked   their kernel_bounds references
  copy, replicate_border, pack_taps_hw, blend, pack_weight   bit for bit against fake_ops.FakeOps
fp32 models (TF32 products) pick their gates by output dtype (the fp32 block of tests/attention_gates.py):
  conv, GEMM, logits    every tensor-core operand (x, w, sc_x; both operands of a batched GEMM) read with its low 13
                        mantissa bits truncated, as wgmma .tf32 reads it; bias and residual as they are.  Gate 1 with
                        1/2 ulp_fp32 and K = 8 per MMA, F (the store stays full fp32), R (closer to the truncating
                        reading than the round-to-nearest one is, where an operand has low bits)
  groupnorm, layernorm, softmax_rows   gates 1-3 with TF32 as the store format, and T (low 13 bits zero)
  attn_temporal         gates 1 and F
  pack_weight, pack_taps_hw, the channels-first -> channels-last gather   bit for bit against tf32_rn of FakeOps'
  result; the other movers bit for bit as above.  Each GroupNorm row also records the headroom of the largest 64-bit
  fixed-point sum of squares below 2^63.
A conv reference is evaluated on the output frames {0, 1, To/2, To-2, To-1} (all of them when To <= 5; for up_time 2 the
output frames those conv frames produce) at every H x W position and channel, as a sum over taps of
[H W, Cin] @ [Cin, Cout] fp64 GEMMs; the batched attention GEMMs are checked in full.
`empty` / `empty_padded` return NaN-filled buffers, so a launch that leaves part of its output unwritten, or reads a
border nobody filled, fails gate 1.  Any operator-set method outside AUDITED fails the audit, and
`launch_identity()` proves that every library launch happened inside an audited call.
"""
import math
import time

import torch

import kernel_bounds as KB
from attention_gates import (GN_SQ_SCALE, GN_SUM_SCALE, TF32, Gates, gemm_bound, kstep, logit_bound, low13,
                             stats_compare)
from fake_ops import PAD_REPLICATE, PAD_ZERO, FakeOps
from test_gpu_fp32 import tf32_rn, tf32_trunc

F64 = torch.float64
AUDITED = ("empty", "empty_padded", "new_stats", "launch_count", "pack_weight", "conv", "conv_stacked", "groupnorm",
           "layernorm", "softmax_rows", "attn_temporal", "replicate_border", "copy", "pack_taps_hw", "blend")
PLAN_FIELDS = ("eligible", "N_cta", "NACC", "vec2", "tma_epilogue")
_DESC_KW = ("kernel", "stride", "offset", "pad_t", "pad_hw", "up_time", "residual", "alpha", "out", "out_f32",
            "bias_along_m", "w_ld", "cout", "gn_stats", "gn_groups", "w_per_batch", "x_shared", "sc_x", "sc_w")


def sample_frames(n):
    """Conv frames whose outputs are checked: {0, 1, n/2, n-2, n-1}, or all of them when n <= 5."""
    return list(range(n)) if n <= 5 else sorted({0, 1, n // 2, n - 2, n - 1})


def view_kind(t):
    """dense, ncdhw (channel stride != 1), lattice (every other W position), framed (interior of a padded buffer)."""
    if t.is_contiguous():
        return "dense"
    if t.stride(4) != 1:
        return "ncdhw"
    if t.dim() == 5 and t.stride(3) == 2 * t.shape[4]:
        return "lattice"
    if t.dim() == 5 and t.stride(3) == t.shape[4] and t.stride(2) == (t.shape[3] + 2) * t.shape[4]:
        return "framed"
    return "strided"


def same_bits(a, b):
    """Bit-for-bit equality (NaN equals the same NaN)."""
    it = {2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(it), b.view(it))


def store_format(dtype):
    """What the MMA-only producers store: the dtype itself, or TF32 values in fp32 storage."""
    return TF32 if dtype == torch.float32 else dtype


def rounding_copy(x, out):
    """Whether cvvae_copy5 rounds to TF32: fp32, not the row path, channels-first -> channels-last (the gather of a
    network input into the channel-padded buffer of the first convolution, its only reader)."""
    rows = x.stride(3) == 1 and out.stride(3) == 1 and x.shape[4] == out.shape[4] and out.shape[3] > 1
    return out.dtype == torch.float32 and not rows and x.stride(4) != 1 and out.stride(4) == 1


def low_bits_share(t):
    """Share of the elements of the fp32 tensor t whose low 13 mantissa bits are not all zero (what a TF32 operand read
    drops), counted in pieces of at most 2^26 elements."""
    def count(u):
        if u.numel() <= 1 << 26:
            return int((low13(u) != 0).sum().item())
        d = max(range(u.dim()), key=lambda i: u.shape[i])
        step = max(1, u.shape[d] * (1 << 26) // u.numel())
        return sum(count(u.narrow(d, a, min(step, u.shape[d] - a))) for a in range(0, u.shape[d], step))
    return count(t) / max(t.numel(), 1)


def _shares(a, b):
    return a is not None and b is not None and a.untyped_storage().data_ptr() == b.untyped_storage().data_ptr()


def _taps(n_out, k, s, off, n_in, mode, device):
    """Input index of each tap and output position [k, n_out] (clamped), and where zero padding applies (or None)."""
    idx = (torch.arange(n_out, device=device) * s + off).view(1, -1) + torch.arange(k, device=device).view(-1, 1)
    valid = (idx >= 0) & (idx < n_in)
    return idx.clamp(0, n_in - 1), (None if mode == PAD_REPLICATE or bool(valid.all()) else valid)


def conv_reference(x, w, bias, out_shape, frames, *, kernel=(1, 1, 1), stride=(1, 1, 1), offset=(0, 0, 0),
                   pad_t=PAD_ZERO, pad_hw=PAD_ZERO, up_time=1, alpha=1.0, residual=None, sc_x=None, sc_w=None,
                   cout=None, operand=None):
    """FakeOps.conv in fp64 on the conv frames `frames`: (output frame indices, r, S) with r, S [B, frames, Ho, Wo, C]
    and S the same sum on absolute values.  Out-of-range taps are clamped (replicate) or contribute zero.  operand: how
    the tensor cores read x, w and sc_x (tf32_trunc for fp32 storage), applied before the products."""
    op = operand or (lambda t: t)
    kt, kh, kw = kernel
    st, sh, sw = stride
    B, T, H, W, Ci = x.shape
    Co = cout if cout is not None else w.shape[1]
    Ho, Wo = out_shape[2], out_shape[3]
    dev = x.device
    wt = op(w[:, :Co, :Ci]).double()
    wa = wt.abs()
    hi, hv = _taps(Ho, kh, sh, offset[1], H, pad_hw, dev)
    wi, wv = _taps(Wo, kw, sw, offset[2], W, pad_hw, dev)
    r = torch.zeros((B, len(frames), Ho, Wo, Co), dtype=F64, device=dev)
    S = torch.zeros_like(r)
    for fi, t in enumerate(frames):
        for j in range(kt):
            ti = t * st + j + offset[0]
            if not 0 <= ti < T:
                if pad_t != PAD_REPLICATE:
                    continue
                ti = min(max(ti, 0), T - 1)
            for a in range(kh):
                xa = x[:, ti].index_select(1, hi[a])
                if hv is not None:
                    xa = torch.where(hv[a].view(1, -1, 1, 1), xa, torch.zeros((), dtype=xa.dtype, device=dev))
                for b in range(kw):
                    xab = xa.index_select(2, wi[b])
                    if wv is not None:
                        xab = torch.where(wv[b].view(1, 1, -1, 1), xab, torch.zeros((), dtype=xab.dtype, device=dev))
                    X = op(xab.reshape(-1, Ci)).double()
                    tap = (j * kh + a) * kw + b
                    r[:, fi] += (X @ wt[tap].T).view(B, Ho, Wo, Co)
                    S[:, fi] += (X.abs() @ wa[tap].T).view(B, Ho, Wo, Co)
                    del X, xab
    r *= alpha
    S *= abs(alpha)
    if bias is not None:
        r += bias.double()
        S += bias.double().abs()
    if up_time == 2:
        # conv frame t, channel half n -> output frame 2t + n - 1 ("b (n c) t h w -> b c (t n) h w", frame 0 dropped)
        c = Co // 2
        of, rs, ss = [], [], []
        for fi, t in enumerate(frames):
            for n in (0, 1):
                if 2 * t + n >= 1:
                    of.append(2 * t + n - 1)
                    rs.append(r[:, fi, ..., n * c:(n + 1) * c])
                    ss.append(S[:, fi, ..., n * c:(n + 1) * c])
        r, S = torch.stack(rs, 1), torch.stack(ss, 1)
    else:
        of = list(frames)
    if sc_w is not None:
        xs = op(sc_x[:, of]).double()
        r += xs @ op(sc_w).double().T
        S += xs.abs() @ op(sc_w).double().abs().T
    if residual is not None:
        rr = residual[:, of].double()
        r += rr
        S += rr.abs()
    return of, r, S


def group_sums(y, groups):
    """fp64 (sum, sum of squares) per (sample, group) of y [B, T, H, W, C], one frame at a time: [B, groups, 2]."""
    B, C = y.shape[0], y.shape[-1]
    acc = torch.zeros((B, groups, 2), dtype=F64, device=y.device)
    for t in range(y.shape[1]):
        v = y[:, t].double().reshape(B, -1, groups, C // groups)
        acc[..., 0] += v.sum(dim=(1, 3))
        acc[..., 1] += (v * v).sum(dim=(1, 3))
    return acc


class AuditOps:
    """An operator set that checks every call of the one it wraps (module docstring); `rows` holds one row per call."""

    def __init__(self, inner):
        self.inner = inner
        self.rows = []
        self.params = {}        # the engine's parameter table, for the layer names (set once the engine exists)
        self._count = {}
        self._last_layer = None
        self._base = inner.launch_count()
        self._fake = FakeOps()

    # ---------------------------------------------------------------- bookkeeping
    def launch_identity(self):
        """(library launches since this set was created, sum of the per-call launches of the rows)."""
        return self.inner.launch_count() - self._base, sum(r["launches"] for r in self.rows)

    def failures(self):
        return [r for r in self.rows if r["failed"]]

    def _layer(self, *tensors):
        ptrs = {v.data_ptr(): k for k, v in self.params.items() if isinstance(v, torch.Tensor)}
        for t in tensors:
            if isinstance(t, torch.Tensor) and t.data_ptr() in ptrs:
                self._last_layer = ptrs[t.data_ptr()]
                return self._last_layer
        return f"(after {self._last_layer})" if self._last_layer else "(start of the pass)"

    @staticmethod
    def _sync():
        if torch.cuda.is_available():
            torch.cuda.synchronize()

    def _run(self, fn, *a, **kw):
        n0 = self.inner.launch_count()
        y = fn(*a, **kw)
        self._sync()
        return y, self.inner.launch_count() - n0

    def _row(self, op, launches, layer, failed, t0, **fields):
        i = self._count.get(op, 0)
        self._count[op] = i + 1
        row = {"i": len(self.rows), "op": op, "op_index": i, "layer": layer, "launches": launches,
               "failed": list(failed), "audit_s": round(time.perf_counter() - t0, 4)}
        row.update(fields)
        self.rows.append(row)
        return row

    def _gate_fields(self, gates):
        rec, failed = gates.result()
        keep = ("worst_bound_ratio", "correctly_rounded_share", "mean_signed_ulp", "numel", "tf32_valued_share",
                "rms_error_ratio", "rn_separation", "error_over_separation", "low_bits_set")
        return {k: rec[k] for k in keep if k in rec}, failed

    # ---------------------------------------------------------------- memory (NaN-filled)
    def empty(self, shape, dtype, device):
        return torch.full(tuple(shape), float("nan"), dtype=dtype, device=device)

    def empty_padded(self, B, T, H, W, Cc, dtype, device):
        p = torch.full((B, T, H + 2, W + 2, Cc), float("nan"), dtype=dtype, device=device)
        return p, p[:, :, 1:-1, 1:-1, :]

    def new_stats(self, B, groups, device):
        return self.inner.new_stats(B, groups, device)

    def launch_count(self):
        return self.inner.launch_count()

    def __getattr__(self, name):
        attr = getattr(self.inner, name)     # AttributeError for what the wrapped set lacks, too
        if not callable(attr):
            return attr

        def unaudited(*a, **kw):
            t0 = time.perf_counter()
            y, n = self._run(attr, *a, **kw)
            self._row(name, n, self._layer(*a), [f"unaudited operator {name!r}"], t0)
            return y
        return unaudited

    # ---------------------------------------------------------------- bit-exact movers
    def pack_weight(self, w):
        t0 = time.perf_counter()
        y, n = self._run(self.inner.pack_weight, w)
        ref = self._fake.pack_weight(w)
        ok = same_bits(y, tf32_rn(ref) if w.dtype == torch.float32 else ref)
        self._row("pack_weight", n, self._layer(w), [] if ok else ["bits differ from FakeOps.pack_weight"], t0,
                  shape_in=list(w.shape))
        return y

    def copy(self, x, out):
        t0 = time.perf_counter()
        xs = x.clone() if _shares(x, out) else x
        y, n = self._run(self.inner.copy, x, out)
        ref = torch.full(out.shape, float("nan"), dtype=out.dtype, device=out.device)
        self._fake.copy(xs, ref)
        rounded = rounding_copy(x, out)
        ok = same_bits(out, tf32_rn(ref) if rounded else ref)
        self._row("copy", n, self._layer(), [] if ok else ["bits differ from FakeOps.copy"], t0,
                  shape_in=list(x.shape), shape_out=list(out.shape), view=view_kind(out), view_in=view_kind(x),
                  tf32_rounded=rounded)
        return y

    def replicate_border(self, xpad):
        t0 = time.perf_counter()
        ref = xpad.clone()
        _, n = self._run(self.inner.replicate_border, xpad)
        self._fake.replicate_border(ref)
        ok = same_bits(xpad, ref)
        self._row("replicate_border", n, self._layer(), [] if ok else ["bits differ from FakeOps.replicate_border"], t0,
                  shape_out=list(xpad.shape))

    def pack_taps_hw(self, x, out, kh, kw, offset=(0, 0), pad_hw=PAD_ZERO):
        t0 = time.perf_counter()
        y, n = self._run(self.inner.pack_taps_hw, x, out, kh, kw, offset=offset, pad_hw=pad_hw)
        ref = torch.full(out.shape, float("nan"), dtype=out.dtype, device=out.device)
        self._fake.pack_taps_hw(x, ref, kh, kw, offset=offset, pad_hw=pad_hw)
        ok = same_bits(out, tf32_rn(ref) if out.dtype == torch.float32 else ref)
        self._row("pack_taps_hw", n, self._layer(), [] if ok else ["bits differ from FakeOps.pack_taps_hw"], t0,
                  shape_in=list(x.shape), shape_out=list(out.shape), view_in=view_kind(x))
        return y

    def blend(self, a, b, overlap, axis):
        t0 = time.perf_counter()
        ref = b.clone()
        y, n = self._run(self.inner.blend, a, b, overlap, axis)
        self._fake.blend(a, ref, overlap, axis)
        ok = same_bits(b, ref)
        self._row("blend", n, "wrapper", [] if ok else ["bits differ from FakeOps.blend"], t0,
                  shape_out=list(b.shape), overlap=overlap, axis=axis)
        return y

    # ---------------------------------------------------------------- convolution
    def conv(self, x, w, bias, **kw):
        t0 = time.perf_counter()
        out = kw["out"]
        st = kw.get("gn_stats")
        before = st.clone() if st is not None else None
        snap = {k: (v.clone() if _shares(v, out) else v) for k, v in (("x", x), ("residual", kw.get("residual")),
                                                                          ("sc_x", kw.get("sc_x")))}
        y, n = self._run(self.inner.conv, x, w, bias, **kw)
        x = snap["x"]
        ref_kw = {k: v for k, v in kw.items() if k in _DESC_KW and k not in ("out", "gn_stats", "gn_groups", "w_ld")}
        ref_kw["residual"], ref_kw["sc_x"] = snap["residual"], snap["sc_x"]
        batched = kw.get("w_per_batch") or kw.get("x_shared")
        kernel = kw.get("kernel", (1, 1, 1))
        K = x.shape[4] * kernel[0] * kernel[1] * kernel[2] + (kw["sc_x"].shape[4] if kw.get("sc_w") is not None else 0)
        dtype = out.dtype
        fields = {"shape_in": list(x.shape), "shape_out": list(out.shape), "view": view_kind(out), "K": K,
                  "kernel": list(kernel), "stride": list(kw.get("stride", (1, 1, 1))), "up_time": kw.get("up_time", 1),
                  "shortcut": kw.get("sc_w") is not None, "residual": kw.get("residual") is not None,
                  "out_f32": bool(kw.get("out_f32")), "batched": bool(batched)}
        plan_fn = getattr(self.inner, "conv_tc_plan", None)
        plan = None
        if plan_fn is not None:
            plan = plan_fn(x, w, bias, epilogue=True, **{k: v for k, v in kw.items() if k in _DESC_KW})
            fields["plan"] = {k: plan[k] for k in PLAN_FIELDS}
        f32 = x.dtype == torch.float32     # an fp32 model (the logits of a 16-bit one are fp32 too)
        tc = plan is None or bool(plan["eligible"])     # the operator sets without a plan query stand for conv_tc
        # fp32: the tensor cores read x, w and sc_x truncated to TF32, K = 8 products per MMA; the CUDA-core conv reads
        # them whole, one fma rounding per product (the linear bound with one product per step)
        ks = (8 if tc else 1) if f32 else kstep(x.dtype)
        op = tf32_trunc if f32 and tc else None
        rn = False       # gate R: also the reference with operands rounded to nearest, where an operand has low bits
        if f32:
            fields["x_low_bits_share"] = low_bits_share(x)
            if batched:
                fields["w_low_bits_share"] = low_bits_share(w)
            if kw.get("sc_w") is not None:
                fields["sc_x_low_bits_share"] = low_bits_share(ref_kw["sc_x"])
            rn = tc and max(v for k, v in fields.items() if k.endswith("low_bits_share")) > 0
        if kw.get("out_f32"):
            gates = Gates(torch.float32 if f32 else None)
        else:
            gates = Gates(dtype, K=K)
        if batched:
            alpha = float(kw.get("alpha", 1.0))
            a32 = float(torch.tensor(alpha, dtype=torch.float32))
            Co = kw.get("cout") or w.shape[1]
            for bi in range(out.shape[0]):
                X = x[0 if kw.get("x_shared") else bi].reshape(-1, x.shape[4])
                Wm = w[bi if kw.get("w_per_batch") else 0][:Co, :x.shape[4]]
                r_rn = (tf32_rn(X).double() @ tf32_rn(Wm).double().T) if rn else None
                X, Wm = (op(X), op(Wm)) if op else (X, Wm)
                X, Wm = X.double(), Wm.double()
                yb = out[bi].reshape(X.shape[0], Co)
                if kw.get("out_f32"):
                    r = a32 * (X @ Wm.T)
                    gates.add(yb, r, logit_bound(x.shape[4], a32, X.abs() @ Wm.abs().T, r, ks),
                              r_rn=a32 * r_rn if rn else None)
                    continue
                r, S = alpha * (X @ Wm.T), abs(alpha) * (X.abs() @ Wm.abs().T)
                if bias is not None:
                    bb = bias.double().view(-1, 1) if kw.get("bias_along_m") else bias.double().view(1, -1)
                    r, S = r + bb, S + bb.abs()
                    r_rn = alpha * r_rn + bb if rn else None
                elif rn:
                    r_rn = alpha * r_rn
                gates.add(yb, r, gemm_bound(K, S, ks), r_rn=r_rn)
                del X, Wm, r, S
        else:
            To = (out.shape[1] + 1) // 2 if kw.get("up_time", 1) == 2 else out.shape[1]
            of, r, S = conv_reference(x, w, bias, tuple(out.shape), sample_frames(To), operand=op, **ref_kw)
            r_rn = None
            if rn:
                r_rn = conv_reference(x, w, bias, tuple(out.shape), sample_frames(To), operand=tf32_rn, **ref_kw)[1]
            fields["frames_checked"] = of
            gates.add(out[:, of], r, gemm_bound(K, S, ks), r_rn=r_rn)
            del r_rn
            del r, S
        vals, failed = self._gate_fields(gates)
        fields.update(vals)
        if st is not None:
            groups = kw.get("gn_groups", 32)
            fields["stats_chained"] = bool(before.abs().sum().item() > 0)
            err, f_st = stats_compare(group_sums(out, groups), st - before)
            fields["stats_max_abs_err"] = err
            failed = failed + f_st
        self._row("conv", n, self._layer(w, x, bias), failed, t0, **fields)
        return y

    def conv_stacked(self, x, w_stk, bias, *, kt, cout, offset=(0, -1, -1), pad_t=PAD_ZERO, pad_hw=PAD_ZERO, out=None):
        t0 = time.perf_counter()
        y, n = self._run(self.inner.conv_stacked, x, w_stk, bias, kt=kt, cout=cout, offset=offset, pad_t=pad_t,
                         pad_hw=pad_hw, out=out)
        w = KB.unstack_weight(w_stk, kt, cout)
        of, r, S = conv_reference(x, w, bias, tuple(out.shape), sample_frames(out.shape[1]), kernel=(kt, 3, 3),
                                  offset=offset, pad_t=pad_t, pad_hw=pad_hw)
        gates = Gates(out.dtype).add(out[:, of], r, KB.conv_stacked_bound(S, kt, x.shape[4]))
        vals, failed = self._gate_fields(gates)
        self._row("conv_stacked", n, self._layer(w_stk, bias), failed, t0, shape_in=list(x.shape),
                  shape_out=list(out.shape), view=view_kind(out), view_in=view_kind(x), frames_checked=of, **vals)
        return y

    # ---------------------------------------------------------------- normalisation and attention
    def groupnorm(self, x, gamma, beta, groups, eps, *, per_frame=False, silu=True, out=None, stats=None):
        t0 = time.perf_counter()
        y, n = self._run(self.inner.groupnorm, x, gamma, beta, groups, eps, per_frame=per_frame, silu=silu, out=out,
                         stats=stats)
        vals, failed, fields = self._groupnorm_gates(x, y, gamma, beta, groups, eps, per_frame, silu, stats)
        fields.update(vals)
        if stats is not None:
            # the network hands every per-sample GroupNorm its producer's sums, so the statistics kernel would never run
            # at tile size (hundreds of fp32 terms per thread): the same input once more with the kernel's own statistics,
            # inside this audited call
            y2, n2 = self._run(self.inner.groupnorm, x, gamma, beta, groups, eps, per_frame=False, silu=silu)
            v2, f2, fl2 = self._groupnorm_gates(x, y2, gamma, beta, groups, eps, False, silu, None)
            fields["kernel_stats_twin"] = dict(v2, P_t=fl2["P_t"], max_mean_over_std=fl2["max_mean_over_std"])
            failed = failed + [f"kernel-statistics twin: {f}" for f in f2]
            n += n2
            del y2
        self._row("groupnorm", n, self._layer(gamma), failed, t0, **fields)
        return y

    def _groupnorm_gates(self, x, y, gamma, beta, groups, eps, per_frame, silu, stats):
        B, T, H, W, Cc = x.shape
        cpg = Cc // groups
        gates = Gates(store_format(y.dtype))
        sq_max = 0.0        # the largest fixed-point sum of squares of a statistics unit (a sample, or a frame)
        fields = {"shape_in": list(x.shape), "view_in": view_kind(x), "view": view_kind(y), "per_frame": per_frame,
                  "silu": silu, "handed_in_stats": stats is not None}
        if per_frame:
            eps_sum, fix, fields["P_t"] = KB.gn_sum_terms(tuple(x.shape), True, groups)
            for t in range(T):
                r, E, _ = KB.gn_reference(x[:, t:t + 1], gamma, beta, groups, eps, True, silu, eps_sum, fix)
                gates.add(y[:, t:t + 1], r, E)
                v = x[:, t].double().reshape(B, -1, groups, cpg)
                sq_max = max(sq_max, (v * v).sum(dim=(1, 3)).max().item())
        else:
            cnt = T * H * W * cpg
            if stats is None:
                eps_sum, fix, fields["P_t"] = KB.gn_sum_terms(tuple(x.shape), False, groups)
                s1 = torch.zeros((B, 1, groups, 1), dtype=F64, device=x.device)
                s2, sa = torch.zeros_like(s1), torch.zeros_like(s1)
                for t in range(T):
                    v = x[:, t].double().reshape(B, -1, groups, cpg)
                    s1 += v.sum(dim=(1, 3), keepdim=True)
                    s2 += (v * v).sum(dim=(1, 3), keepdim=True)
                    sa += v.abs().sum(dim=(1, 3), keepdim=True)
                mean, sqmean, absmean = s1 / cnt, s2 / cnt, sa / cnt
                var = (sqmean - mean * mean).clamp_min(0)
                sq_max = s2.max().item()
            else:
                st = stats.double()
                mean = (st[:, :, 0] / GN_SUM_SCALE / cnt).view(B, 1, groups, 1)
                var = (st[:, :, 1] / GN_SQ_SCALE / cnt).view(B, 1, groups, 1) - mean * mean
                var = var.clamp_min(0)
                absmean = sqmean = None
                eps_sum, fix = None, cnt
                sq_max = st[:, :, 1].max().item() / GN_SQ_SCALE
            kmax = 0.0
            for t in range(T):
                v = x[:, t].double().reshape(B, -1, groups, cpg)
                r, E, k = KB.gn_pointwise(v, mean, var, absmean, sqmean, gamma, beta, eps, silu, eps_sum, fix)
                kmax = max(kmax, k)
                gates.add(y[:, t].reshape(r.shape), r, E)
                del v, r, E
            fields["max_mean_over_std"] = kmax
        # DESIGN section 6: the sums are 64-bit fixed point (sum of squares * 2^18); bits left below 2^63 (recorded only)
        fields["sq_headroom_bits"] = math.log2(2.0 ** 63 / max(sq_max * GN_SQ_SCALE, 1.0))
        vals, failed = self._gate_fields(gates)
        return vals, failed, fields

    def layernorm(self, x, gamma, beta, eps):
        t0 = time.perf_counter()
        y, n = self._run(self.inner.layernorm, x, gamma, beta, eps)
        r, E, k = KB.layernorm_reference(x, gamma, beta, eps)
        vals, failed = self._gate_fields(Gates(store_format(y.dtype)).add(y, r, E))
        self._row("layernorm", n, self._layer(gamma), failed, t0, shape_in=list(x.shape), max_mean_over_std=k, **vals)
        return y

    def softmax_rows(self, s, cols, out):
        t0 = time.perf_counter()
        y, n = self._run(self.inner.softmax_rows, s, cols, out)
        r, E = KB.softmax_reference(s, cols)
        vals, failed = self._gate_fields(Gates(store_format(out.dtype)).add(out[:, :cols], r, E))
        self._row("softmax_rows", n, self._layer(), failed, t0, shape_in=list(s.shape), cols=cols, **vals)
        return y

    def attn_temporal(self, q, k, v):
        t0 = time.perf_counter()
        y, n = self._run(self.inner.attn_temporal, q, k, v)
        r, E, _ = KB.attn_temporal_reference(q, k, v)
        # fp32: CUDA cores, no operand truncation; the store is full fp32 (gates 1 and F)
        vals, failed = self._gate_fields(Gates(y.dtype, rms=False).add(y, r, E))
        self._row("attn_temporal", n, self._layer(), failed, t0, shape_in=list(q.shape), **vals)
        return y


def summary(ops):
    """Per-op launch counts and the failing rows, for assertion messages."""
    counts = {}
    for r in ops.rows:
        counts[r["op"]] = counts.get(r["op"], 0) + 1
    bad = [{k: r.get(k) for k in ("i", "op", "op_index", "layer", "shape_out", "view", "failed")} for r in ops.failures()]
    return {"calls": counts, "failures": bad}

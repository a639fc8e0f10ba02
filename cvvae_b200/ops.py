"""Torch-tensor facing wrappers of the C ABI (device pointers + the current CUDA stream in, nothing else).

Every activation is a torch tensor viewed as logical ``[B, T, H, W, C]`` with arbitrary strides
(channels-last buffers are contiguous in that view; a caller's NCDHW tensor is passed as
``x.permute(0, 2, 3, 4, 1)`` without a copy).  PyTorch is used for memory and streams only.

``CudaOps`` is the one production backend.  The engine takes the backend as an argument so that the
CPU test-suite can drive the same graph code with a torch restatement of each operator
(``tests/fake_ops.py``); the product never selects anything but ``CudaOps``.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Tuple

import torch

from . import _lib as L

_DT = {torch.float16: L.F16, torch.bfloat16: L.BF16, torch.float32: L.F32}


def dtype_code(dt: torch.dtype) -> int:
    try:
        return _DT[dt]
    except KeyError:
        raise L.CvvaeError(f"cvvae_b200 computes in float16, bfloat16 or float32 (TF32 tensor-core products), got {dt}")


def _t5(t: torch.Tensor) -> L.Tensor5:
    assert t.dim() == 5, t.shape
    s = t.stride()
    return L.Tensor5(t.data_ptr(), t.shape[0], t.shape[1], t.shape[2], t.shape[3], t.shape[4], s[0], s[1], s[2], s[3], s[4])


def _stream(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _on_tensor_device(fn):
    """Run a CudaOps method with the CUDA device of its first tensor argument current.

    The C ABI launches on the current device (kernel attributes, SM count and the stream handle are per device), so
    a model living on cuda:1 while cuda:0 is current - single-process multi-GPU, diffusers device placement - must
    switch for the duration of the call, exactly as a PyTorch operator would."""
    import functools

    @functools.wraps(fn)
    def wrapper(self, *args, **kwargs):
        dev = None
        for a in args:
            if isinstance(a, torch.Tensor):
                dev = a.device
                break
        if dev is None or dev.type != "cuda" or dev.index == torch.cuda.current_device():
            return fn(self, *args, **kwargs)
        with torch.cuda.device(dev):
            return fn(self, *args, **kwargs)

    return wrapper


class CudaOps:
    """The production operator set: every method is one (or two) hand-written sm_90a kernels."""

    name = "cuda"

    def __init__(self):
        self.lib = L.load()
        # optional instrumentation (bench.py): algorithmic FLOPs and CUDA-event time per convolution path
        self.profile = None  # None | {"flops": {path: int}, "events": {path: [(start, end), ...]}}

    def start_profile(self):
        self.profile = {"flops": {"conv_tc": 0, "conv_direct": 0}, "ref_flops": {"conv_tc": 0, "conv_direct": 0},
                        "bytes": {"conv_tc": 0, "conv_direct": 0},
                        "events": {"conv_tc": [], "conv_direct": []}, "launches": {"conv_tc": 0, "conv_direct": 0}}

    def stop_profile(self):
        """Returns {path: {"flops": F, "ms": T, "launches": n}} (synchronises)."""
        prof, self.profile = self.profile, None
        torch.cuda.synchronize()
        out = {}
        for path in prof["flops"]:
            ms = sum(s.elapsed_time(e) for s, e in prof["events"][path])
            out[path] = {"flops": prof["flops"][path], "ref_flops": prof["ref_flops"][path], "bytes": prof["bytes"][path], "ms": ms,
                         "launches": prof["launches"][path]}
        return out

    # ------------------------------------------------------------------ memory (plumbing)
    @staticmethod
    def empty(shape: Sequence[int], dtype, device) -> torch.Tensor:
        return torch.empty(tuple(shape), dtype=dtype, device=device)

    def empty_padded(self, B, T, H, W, Cc, dtype, device) -> Tuple[torch.Tensor, torch.Tensor]:
        """A buffer with a 1-position frame in H and W; returns (padded, interior view)."""
        p = torch.empty((B, T, H + 2, W + 2, Cc), dtype=dtype, device=device)
        return p, p[:, :, 1:-1, 1:-1, :]

    # ------------------------------------------------------------------ convolution / GEMM
    @_on_tensor_device
    def pack_weight(self, w: torch.Tensor) -> torch.Tensor:
        """[Cout, Cin, *k] (PyTorch) -> [taps, Cout, Cin] in the same dtype (fp32: rounded to the nearest TF32 value)."""
        w = w.contiguous()
        co, ci = w.shape[0], w.shape[1]
        taps = 1
        for k in w.shape[2:]:
            taps *= k
        out = torch.empty((taps, co, ci), dtype=w.dtype, device=w.device)
        L.check(self.lib.cvvae_pack_conv_weight(w.data_ptr(), out.data_ptr(), co, ci, taps, dtype_code(w.dtype), _stream(w)),
                "cvvae_pack_conv_weight")
        return out

    @_on_tensor_device
    def conv(self, x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], *, kernel=(1, 1, 1),
             stride=(1, 1, 1), offset=(0, 0, 0), pad_t=L.PAD_ZERO, pad_hw=L.PAD_ZERO, up_time=1,
             residual: Optional[torch.Tensor] = None, alpha: float = 1.0, out: Optional[torch.Tensor] = None,
             out_f32: bool = False, bias_along_m: bool = False, w_ld: int = 0, cout: Optional[int] = None,
             force: Optional[str] = None, ref_taps: Optional[int] = None, gn_stats: Optional[torch.Tensor] = None,
             gn_groups: int = 32, w_per_batch: bool = False, x_shared: bool = False,
             k_alg: Optional[int] = None, sc_x: Optional[torch.Tensor] = None, sc_w: Optional[torch.Tensor] = None) -> torch.Tensor:
        """y = alpha * conv(x, w) + bias + residual.  ``w`` is packed [taps, Cout, Cin(ld)].

        Batched GEMM (attention): ``w_per_batch`` - w is [B, Cout, Cin(ld)], one matrix per batch item of y;
        ``x_shared`` - x has batch 1 and is the left operand of every batch item.
        Fused 1x1 shortcut: ``sc_x`` [B,T,H,W,C2] (the output's extents) times ``sc_w`` [Cout, C2] is accumulated into the
        same fp32 accumulators as the taps (``bias`` then carries the sum of both biases)."""
        d = self._conv_desc(x, w, bias, kernel=kernel, stride=stride, offset=offset, pad_t=pad_t, pad_hw=pad_hw,
                            up_time=up_time, residual=residual, alpha=alpha, out=out, out_f32=out_f32,
                            bias_along_m=bias_along_m, w_ld=w_ld, cout=cout, gn_stats=gn_stats, gn_groups=gn_groups,
                            w_per_batch=w_per_batch, x_shared=x_shared, sc_x=sc_x, sc_w=sc_w)
        B, T, H, W, Ci = x.shape
        if x_shared:
            B = out.shape[0]
        kt, kh, kw = kernel
        Co = d.Cout
        fn = {None: self.lib.cvvae_conv3d, "tc": self.lib.cvvae_conv3d_tc, "direct": self.lib.cvvae_conv3d_direct}[force]
        if self.profile is None:
            L.check(fn(C.byref(d), _stream(x)), "cvvae_conv3d")
            return out
        path = "conv_tc" if (force == "tc" or (force is None and self.lib.cvvae_conv3d_is_tc(C.byref(d)))) else "conv_direct"
        t_conv = (out.shape[1] + 1) // 2 if up_time == 2 else out.shape[1]
        # executed: 2 * M * N * K of this launch (zero-padded taps included).  reference-dense: the same output
        # positions at the tap count the reference issues (27 for the folded up-sample phases, ref_taps)
        mn = 2 * B * t_conv * out.shape[2] * out.shape[3] * Co * Ci
        if k_alg is not None:   # tap-packed network-input conv: count the algorithmic K (taps x real channels), not the padded one
            mn, kt, kh, kw, ref_taps = 2 * B * t_conv * out.shape[2] * out.shape[3] * Co, k_alg, 1, 1, None
        self.profile["flops"][path] += mn * kt * kh * kw
        self.profile["ref_flops"][path] += mn * (ref_taps if ref_taps is not None else kt * kh * kw)
        if sc_w is not None:   # the fused 1x1 shortcut's MACs (a separate conv in the reference) and its input bytes
            sc = 2 * B * t_conv * out.shape[2] * out.shape[3] * Co * sc_x.shape[4]
            self.profile["flops"][path] += sc
            self.profile["ref_flops"][path] += sc
            self.profile["bytes"][path] += sc_x.numel() * sc_x.element_size() + sc_w.numel() * sc_w.element_size()
        # algorithmic bytes: every operand once (input, weights, residual, output)
        self.profile["bytes"][path] += (x.numel() * x.element_size() + w.numel() * w.element_size() +
                                        out.numel() * out.element_size() * (2 if residual is not None else 1))
        self.profile["launches"][path] += 1
        s_ev, e_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s_ev.record()
        L.check(fn(C.byref(d), _stream(x)), "cvvae_conv3d")
        e_ev.record()
        self.profile["events"][path].append((s_ev, e_ev))
        return out

    @_on_tensor_device
    def conv_tc_plan(self, x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], *, epilogue: bool = False,
                     **kw) -> dict:
        """The tile plan ``conv(..., force="tc")`` launches for the same arguments on the current device
        ({name: value} over ``_lib.CONV_TC_PLAN_FIELDS``; ``eligible`` 0 when the tensor-core path refuses them).
        ``epilogue``: also report ``tma_epilogue``, whether the output goes through shared memory and TMA stores
        (it depends on the output's alignment and on CVVAE_TMA_EPILOGUE, the tiling does not).  Launches nothing."""
        d = self._conv_desc(x, w, bias, **kw)
        fields = L.CONV_TC_PLAN_EPILOGUE_FIELDS if epilogue else L.CONV_TC_PLAN_FIELDS
        n = len(fields)
        vals = (C.c_int32 * n)()
        rc = self.lib.cvvae_conv_tc_plan(C.byref(d), vals, n)
        if rc < 0:
            L.check(rc, "cvvae_conv_tc_plan")
        return dict(zip(fields, list(vals)))

    @staticmethod
    def _conv_desc(x, w, bias, *, kernel=(1, 1, 1), stride=(1, 1, 1), offset=(0, 0, 0), pad_t=L.PAD_ZERO, pad_hw=L.PAD_ZERO,
                   up_time=1, residual=None, alpha=1.0, out=None, out_f32=False, bias_along_m=False, w_ld=0, cout=None,
                   gn_stats=None, gn_groups=32, w_per_batch=False, x_shared=False, sc_x=None, sc_w=None) -> L.ConvDesc:
        kt, kh, kw = kernel
        st, sh, sw = stride
        ot, oh, ow = offset
        Co = cout if cout is not None else w.shape[1]
        if out is None:
            # PyTorch conv arithmetic with the padding implied by the offsets: out = floor((in + pad - k)/s) + 1,
            # where the engine always passes offsets so that the reference's output extents result.
            raise ValueError("conv(): the caller provides `out` (the engine knows the reference's output extents)")
        assert w.shape[0] == (out.shape[0] if w_per_batch else kt * kh * kw), (w.shape, kernel)
        d = L.ConvDesc()
        d.x = _t5(x)
        d.y = _t5(out)
        d.w = w.data_ptr()
        d.w_ld = w_ld
        d.bias = _ptr(bias)
        d.residual = _ptr(residual)
        d.Cout = Co
        d.KT, d.KH, d.KW = kt, kh, kw
        d.st, d.sh, d.sw = st, sh, sw
        d.off_t, d.off_h, d.off_w = ot, oh, ow
        d.pad_t, d.pad_hw = pad_t, pad_hw
        d.up_time = up_time
        d.dtype = dtype_code(x.dtype)
        d.flags = ((L.CONV_BIAS_ALONG_M if bias_along_m else 0) | (L.CONV_OUT_F32 if out_f32 else 0) |
                   (L.CONV_W_PER_BATCH if w_per_batch else 0) | (L.CONV_X_SHARED if x_shared else 0))
        d.alpha = alpha
        if gn_stats is not None:  # int64 fixed point [B, groups, 2], zeroed by the caller; the epilogue accumulates into it
            assert gn_stats.dtype == torch.int64 and gn_stats.is_contiguous()
            d.gn_stats = gn_stats.data_ptr()
            d.gn_groups = gn_groups
        if residual is not None:
            assert residual.shape == out.shape and residual.stride() == out.stride(), "residual must share y's geometry"
        if sc_w is not None:
            assert sc_x is not None and tuple(sc_x.shape[:4]) == tuple(out.shape[:4]) and tuple(sc_w.shape) == (Co, sc_x.shape[4])
            assert sc_w.is_contiguous() and sc_w.dtype == x.dtype
            d.x2 = _t5(sc_x)
            d.w2 = sc_w.data_ptr()
        return d

    @_on_tensor_device
    def conv_stacked(self, x: torch.Tensor, w_stk: torch.Tensor, bias: Optional[torch.Tensor], *, kt: int, cout: int,
                     offset=(0, -1, -1), pad_t=L.PAD_ZERO, pad_hw=L.PAD_ZERO, out: torch.Tensor = None) -> torch.Tensor:
        """(KT x) 3 x 3 stride-1 convolution with Cout <= 4 through the tap-stacked kernel; w_stk is [KT, 80, Cin]."""
        assert w_stk.shape[0] == kt and w_stk.shape[1] == 80 and w_stk.is_contiguous()
        d = L.ConvDesc()
        d.x = _t5(x)
        d.y = _t5(out)
        d.w = w_stk.data_ptr()
        d.bias = _ptr(bias)
        d.Cout = cout
        d.KT, d.KH, d.KW = kt, 3, 3
        d.st = d.sh = d.sw = 1
        d.off_t, d.off_h, d.off_w = offset
        d.pad_t, d.pad_hw = pad_t, pad_hw
        d.up_time = 1
        d.dtype = dtype_code(x.dtype)
        d.alpha = 1.0
        if self.profile is not None:
            B, T, H, W, Ci = x.shape
            fl = 2 * B * out.shape[1] * out.shape[2] * out.shape[3] * cout * Ci * kt * 9
            self.profile["flops"]["conv_tc"] += fl
            self.profile["ref_flops"]["conv_tc"] += fl
            self.profile["bytes"]["conv_tc"] += x.numel() * x.element_size() + out.numel() * out.element_size()
            self.profile["launches"]["conv_tc"] += 1
            s_ev, e_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s_ev.record()
            L.check(self.lib.cvvae_conv3d_stacked(C.byref(d), _stream(x)), "cvvae_conv3d_stacked")
            e_ev.record()
            self.profile["events"]["conv_tc"].append((s_ev, e_ev))
        else:
            L.check(self.lib.cvvae_conv3d_stacked(C.byref(d), _stream(x)), "cvvae_conv3d_stacked")
        return out

    # ------------------------------------------------------------------ normalisation
    def new_stats(self, B: int, groups: int, device) -> torch.Tensor:
        """Zeroed int64 fixed-point [B, groups, 2] accumulator (sum * 2^20, sum^2 * 2^18) for conv-epilogue statistics."""
        return torch.zeros((B, groups, 2), dtype=torch.int64, device=device)

    @_on_tensor_device
    def groupnorm(self, x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int, eps: float, *,
                  per_frame: bool = False, silu: bool = True, out: Optional[torch.Tensor] = None,
                  stats: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`stats`: sums already produced by the conv that wrote x (skips the statistics pass)."""
        B, T = x.shape[0], x.shape[1]
        units = B * T if per_frame else B
        if out is None:
            out = torch.empty(x.shape, dtype=x.dtype, device=x.device)
        dt = dtype_code(x.dtype)
        xs, ys = _t5(x), _t5(out)
        if stats is None:
            stats = torch.empty((units, groups, 2), dtype=torch.int64, device=x.device)
            L.check(self.lib.cvvae_groupnorm_stats(C.byref(xs), groups, int(per_frame), stats.data_ptr(), dt, _stream(x)),
                    "cvvae_groupnorm_stats")
        else:
            assert not per_frame and tuple(stats.shape) == (units, groups, 2)
        L.check(self.lib.cvvae_groupnorm_apply(C.byref(xs), C.byref(ys), groups, int(per_frame), stats.data_ptr(),
                                               gamma.data_ptr(), beta.data_ptr(), eps, int(silu), dt, _stream(x)),
                "cvvae_groupnorm_apply")
        return out

    @_on_tensor_device
    def layernorm(self, x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float) -> torch.Tensor:
        out = torch.empty(x.shape, dtype=x.dtype, device=x.device)
        xs, ys = _t5(x), _t5(out)
        L.check(self.lib.cvvae_layernorm(C.byref(xs), C.byref(ys), gamma.data_ptr(), beta.data_ptr(), eps,
                                         dtype_code(x.dtype), _stream(x)), "cvvae_layernorm")
        return out

    # ------------------------------------------------------------------ attention helpers
    @_on_tensor_device
    def softmax_rows(self, s: torch.Tensor, cols: int, out: torch.Tensor) -> torch.Tensor:
        """s: fp32 [rows, ld_s]; out: activation dtype [rows, ld_p]; softmax over the first `cols` of each row."""
        assert s.dtype == torch.float32 and s.dim() == 2 and out.dim() == 2 and s.stride(1) == 1 and out.stride(1) == 1
        L.check(self.lib.cvvae_softmax_rows(s.data_ptr(), s.stride(0), out.data_ptr(), out.stride(0), s.shape[0], cols,
                                            dtype_code(out.dtype), _stream(s)), "cvvae_softmax_rows")
        return out

    @_on_tensor_device
    def attn_temporal(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
        out = torch.empty(q.shape, dtype=q.dtype, device=q.device)
        a, b, c, o = _t5(q), _t5(k), _t5(v), _t5(out)
        L.check(self.lib.cvvae_attn_temporal(C.byref(a), C.byref(b), C.byref(c), C.byref(o), dtype_code(q.dtype), _stream(q)),
                "cvvae_attn_temporal")
        return out

    # ------------------------------------------------------------------ data movement
    @_on_tensor_device
    def replicate_border(self, xpad: torch.Tensor) -> None:
        xs = _t5(xpad)
        L.check(self.lib.cvvae_replicate_border(C.byref(xs), dtype_code(xpad.dtype), _stream(xpad)), "cvvae_replicate_border")

    @_on_tensor_device
    def copy(self, x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
        xs, ys = _t5(x), _t5(out)
        L.check(self.lib.cvvae_copy5(C.byref(xs), C.byref(ys), dtype_code(x.dtype), _stream(x)), "cvvae_copy5")
        return out

    @_on_tensor_device
    def pack_taps_hw(self, x: torch.Tensor, out: torch.Tensor, kh: int, kw: int, offset=(0, 0), pad_hw=L.PAD_ZERO) -> torch.Tensor:
        """out[..., (a*kw+b)*Cx + c] = x[.., h+a+off_h, w+b+off_w, c] (zero / clamped outside), remaining channels zero."""
        xs, ys = _t5(x), _t5(out)
        L.check(self.lib.cvvae_pack_taps_hw(C.byref(xs), C.byref(ys), kh, kw, offset[0], offset[1], pad_hw, dtype_code(out.dtype),
                                            _stream(x)), "cvvae_pack_taps_hw")
        return out

    @_on_tensor_device
    def blend(self, a: torch.Tensor, b: torch.Tensor, overlap: int, axis: int) -> torch.Tensor:
        """In place on b (logical [B,T,H,W,C] views): axis 0 = width (blend_h), 1 = height (blend_v)."""
        xs, ys = _t5(a), _t5(b)
        L.check(self.lib.cvvae_blend(C.byref(xs), C.byref(ys), overlap, axis, dtype_code(b.dtype), _stream(b)), "cvvae_blend")
        return b

    def launch_count(self) -> int:
        return int(self.lib.cvvae_launch_count())

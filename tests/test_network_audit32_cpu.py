"""The launch audit (tests/network_audit.py) of float32 models on the CPU, proving its fp32 gates can fail.

The tiny golden models (w32) run in fp32 through an honest test double of the TF32 engine: the fp64 spec of
tests/fake_ops.py on tensor-core operands truncated to TF32 (as wgmma .tf32 reads them), each convolution, GEMM and
temporal-attention output rounded once to fp32, each output of an MMA-only producer (GroupNorm, LayerNorm, softmax, the
packed weights, pack_taps_hw and the network-input gather) rounded once to the nearest TF32 value.  It must pass with
every launch audited.  Each doctored double must then fail, at the launch it doctored and on the gate it targets.
"""
import pytest
import torch

from attention_gates import TF32, store_ulp
from fake_ops import GN_SQ_SCALE, GN_SUM_SCALE, FakeOps
from network_audit import rounding_copy, summary
from test_gpu_fp32 import tf32_rn, tf32_trunc
from test_network_audit_cpu import TARGET, _assert_complete, run_audit

F32 = torch.float32


def tf32_once(y64):
    """fp64 -> the nearest TF32 value (ties to even), rounded once, in fp32 storage."""
    ulp = store_ulp(y64, TF32)
    return (torch.round(y64 / ulp) * ulp).float()      # y64 / ulp exact; the result is a TF32 value, exact in fp32


class HonestOps32(FakeOps):
    """FakeOps evaluated in fp64 on TF32-truncated tensor-core operands, each result rounded once to what its kernel
    stores."""

    def __init__(self):
        super().__init__(torch.float64)
        self.n_conv = 0

    # how the tensor cores read an operand, and how each kind of output is stored
    def _operand(self, t):
        return tf32_trunc(t) if t.dtype == F32 else t

    def _store_conv(self, y64, out):
        out.copy_(y64.to(out.dtype))

    def _store_mma_only(self, y64):
        return tf32_once(y64)

    def pack_weight(self, w):
        self.launches += 1
        return tf32_rn(super().pack_weight(w))

    def conv(self, x, w, bias, *, out=None, gn_stats=None, gn_groups=32, sc_x=None, **kw):
        self.n_conv += 1
        y64 = torch.empty(out.shape, dtype=torch.float64)
        super().conv(self._operand(x), self._operand(w), bias, out=y64,
                     sc_x=self._operand(sc_x) if sc_x is not None else None, **kw)
        self._store_conv(y64, out)
        if gn_stats is not None:   # sums of the stored values, as FakeOps.conv
            v = out.double().reshape(out.shape[0], -1, gn_groups, out.shape[-1] // gn_groups)
            gn_stats[:, :, 0] += torch.round(v.sum(dim=(1, 3)) * GN_SUM_SCALE).to(torch.int64)
            gn_stats[:, :, 1] += torch.round((v * v).sum(dim=(1, 3)) * GN_SQ_SCALE).to(torch.int64)
        return out

    def groupnorm(self, x, gamma, beta, groups, eps, *, per_frame=False, silu=True, out=None, stats=None):
        y64 = torch.empty(x.shape, dtype=torch.float64)
        super().groupnorm(x, gamma, beta, groups, eps, per_frame=per_frame, silu=silu, out=y64, stats=stats)
        if out is None:
            out = torch.empty(x.shape, dtype=x.dtype)
        out.copy_(self._store_mma_only(y64))
        return out

    def layernorm(self, x, gamma, beta, eps):
        return tf32_once(super().layernorm(x.double(), gamma, beta, eps))

    def softmax_rows(self, s, cols, out):
        self.launches += 1
        out[:, :cols] = self._store_softmax(torch.softmax(s[:, :cols].double(), dim=-1))
        return out

    def _store_softmax(self, p64):
        return tf32_once(p64)

    def attn_temporal(self, q, k, v):
        return super().attn_temporal(q.double(), k.double(), v.double()).float()

    def pack_taps_hw(self, x, out, kh, kw, offset=(0, 0), pad_hw=0):
        super().pack_taps_hw(x, out, kh, kw, offset=offset, pad_hw=pad_hw)
        out.copy_(tf32_rn(out))
        return out

    def copy(self, x, out):
        super().copy(x, out)
        if self._round_copy(x, out):
            out.copy_(tf32_rn(out))
        return out

    def _round_copy(self, x, out):
        return rounding_copy(x, out)


class ConvStoreTf32(HonestOps32):
    """The doctored convolution stores its result rounded to TF32 instead of full fp32."""

    def _store_conv(self, y64, out):
        if self.n_conv != TARGET:
            return super()._store_conv(y64, out)
        out.copy_(tf32_once(y64))


class ConvReadsRoundedOperands(HonestOps32):
    """Every tensor-core operand read rounded to the nearest TF32 value instead of truncated."""

    def _operand(self, t):
        return tf32_rn(t) if t.dtype == F32 else t


class GroupNormFullFp32(HonestOps32):
    """The first GroupNorm stores its fp32 result without rounding it to TF32."""
    done = False

    def _store_mma_only(self, y64):
        if self.done:
            return super()._store_mma_only(y64)
        self.done = True
        return y64.float()


class SoftmaxTruncatedTf32(HonestOps32):
    """softmax_rows stores its probabilities truncated to TF32 instead of rounded to nearest."""

    def _store_softmax(self, p64):
        ulp = store_ulp(p64, TF32)
        return (torch.trunc(p64 / ulp) * ulp).float()


class GatherNotRounded(HonestOps32):
    """The network-input gather copies fp32 values without rounding them to TF32."""

    def _round_copy(self, x, out):
        return False


class LastFrameUnwritten32(HonestOps32):
    def _store_conv(self, y64, out):
        if self.n_conv != TARGET:
            return super()._store_conv(y64, out)
        out[:, :-1].copy_(y64[:, :-1].to(out.dtype))


@pytest.mark.parametrize("name", ["sd21_w32_plain", "sd3_w32_plain", "sd21_w32_image", "sd3_w32_tiled"])
def test_honest_fp32_double_passes(name):
    ops = run_audit(name, F32, HonestOps32)
    s = summary(ops)
    assert not s["failures"], s
    _assert_complete(ops)
    ops_seen = set(s["calls"])
    assert {"conv", "groupnorm", "pack_weight", "softmax_rows"} <= ops_seen, s["calls"]
    assert "conv_stacked" not in ops_seen, "an fp32 conv_out runs through the general tensor-core convolution"
    if name.endswith("tiled"):
        assert {"copy", "blend"} <= ops_seen, s["calls"]
    convs = [r for r in ops.rows if r["op"] == "conv"]
    assert all("rms_error_ratio" in r and "tf32_valued_share" in r for r in convs)
    assert any(r["x_low_bits_share"] > 0.5 for r in convs), "no conv reads an operand with low bits"
    assert any(r["view"] == "ncdhw" for r in convs), "the conv_out views are not audited"
    if not name.endswith("image"):
        assert any(r["shortcut"] and r["sc_x_low_bits_share"] > 0.5 for r in convs), "no fused shortcut with low bits"
        assert any(r["up_time"] == 2 for r in convs)
    norms = [r for r in ops.rows if r["op"] in ("groupnorm", "layernorm", "softmax_rows")]
    assert norms and all(r["low_bits_set"] == 0 for r in norms)
    assert all(r["sq_headroom_bits"] > 0 for r in ops.rows if r["op"] == "groupnorm")


def test_honest_fp32_double_passes_through_the_gather():
    """The channel-padded gather of the network input (the engine's path without the tap-packed conv_in) rounds to
    TF32."""
    ops = run_audit("sd21_w32_plain", F32, HonestOps32, drop_hwpack=True)
    assert not ops.failures(), summary(ops)
    _assert_complete(ops)
    assert any(r["op"] == "copy" and r["tf32_rounded"] for r in ops.rows)


# name: (double, gate or message the first failing row must carry, op of that row, tap packing dropped)
DOCTORED = {
    "conv_store_tf32": (ConvStoreTf32, "F:", "conv", False),
    "conv_reads_rounded_operands": (ConvReadsRoundedOperands, "R:", "conv", False),
    "groupnorm_full_fp32": (GroupNormFullFp32, "T:", "groupnorm", False),
    "softmax_truncated_tf32": (SoftmaxTruncatedTf32, ("2:", "3:"), "softmax_rows", False),
    "gather_not_rounded": (GatherNotRounded, "bits differ from FakeOps.copy", "copy", True),
    "last_frame_unwritten": (LastFrameUnwritten32, "1:", "conv", False),
}


@pytest.mark.parametrize("doctor", list(DOCTORED))
def test_doctored_fp32_double_fails_at_its_launch(doctor):
    cls, gate, op, drop = DOCTORED[doctor]
    ops = run_audit("sd21_w32_plain", F32, cls, drop_hwpack=drop)
    bad = ops.failures()
    assert bad, f"{doctor}: the audit passed"
    first = bad[0]
    assert first["op"] == op and first["layer"], first
    assert any(f.startswith(gate) for f in first["failed"]), first
    if cls in (ConvStoreTf32, LastFrameUnwritten32):
        assert first["op_index"] == TARGET - 1, first
    if cls is ConvStoreTf32:        # a wrong store format, finite values: nothing downstream fails
        assert len(bad) == 1, summary(ops)["failures"]
    if cls is ConvReadsRoundedOperands:
        # the launches whose operands are all TF32 values read them the same either way and pass; the first to fail
        # reads an operand with low bits
        assert max(first["x_low_bits_share"], first.get("sc_x_low_bits_share", 0.0),
                   first.get("w_low_bits_share", 0.0)) > 0, first
        assert all(max(r["x_low_bits_share"], r.get("sc_x_low_bits_share", 0.0), r.get("w_low_bits_share", 0.0)) > 0
                   for r in bad if r["op"] == "conv"), summary(ops)["failures"]
    if cls is GroupNormFullFp32:
        assert first["op_index"] == 0 and len(bad) == 1, summary(ops)["failures"]
    _assert_complete(ops)

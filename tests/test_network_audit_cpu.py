"""The launch audit (tests/network_audit.py) on the CPU, proving it can fail.

The tiny golden models (w32) run in fp16 and bf16 through an honest test double - the fp64 spec of tests/fake_ops.py,
every store rounded once to the dtype - and must pass with every launch audited.  Each doctored double must then fail,
at the launch it doctored and on the gate it targets.
"""
import pytest
import torch

from attention_gates import truncate
from cvvae_b200.engine import Act, Engine, _round_once
from fake_ops import GN_SQ_SCALE, GN_SUM_SCALE, FakeOps
from network_audit import AUDITED, AuditOps, summary
from oracle import cvvae_oracle as O
from test_engine_wiring_cpu import CASES, MANIFEST, build_model

DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}


class HonestOps(FakeOps):
    """FakeOps evaluated in fp64, each result rounded once to the output dtype."""

    def __init__(self):
        super().__init__(torch.float64)
        self.n_conv = 0

    def _store_conv(self, y64, out):
        out.copy_(_round_once(y64, out.dtype))

    def conv(self, x, w, bias, *, out=None, gn_stats=None, gn_groups=32, **kw):
        self.n_conv += 1
        y64 = torch.empty(out.shape, dtype=torch.float64)
        super().conv(x, w, bias, out=y64, **kw)
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
        out.copy_(_round_once(y64, out.dtype))
        return out

    def layernorm(self, x, gamma, beta, eps):
        return _round_once(super().layernorm(x.double(), gamma, beta, eps), x.dtype)

    def softmax_rows(self, s, cols, out):
        self.launches += 1
        out[:, :cols] = _round_once(torch.softmax(s[:, :cols].double(), dim=-1), out.dtype)
        return out

    def attn_temporal(self, q, k, v):
        return _round_once(super().attn_temporal(q.double(), k.double(), v.double()), q.dtype)


TARGET = 3   # the doctored convolution: the encoder's third launch (first block's conv2), before any batched GEMM


class TruncatingStore(HonestOps):
    def _store_conv(self, y64, out):
        if self.n_conv != TARGET:
            return super()._store_conv(y64, out)
        out.copy_(truncate(y64, out.dtype))


class ZeroInLastRow(HonestOps):
    def _store_conv(self, y64, out):
        super()._store_conv(y64, out)
        if self.n_conv == TARGET:
            row = out[0, 0, -1]
            j = int(row.abs().argmax())
            row.view(-1)[j] = 0


class LastFrameUnwritten(HonestOps):
    def _store_conv(self, y64, out):
        if self.n_conv != TARGET:
            return super()._store_conv(y64, out)
        out[:, :-1].copy_(_round_once(y64[:, :-1], out.dtype))


class StatsOff(HonestOps):
    """The first fused statistics off by 2^-10 of one group's sum."""
    done = False

    def conv(self, x, w, bias, *, gn_stats=None, **kw):
        before = gn_stats.clone() if gn_stats is not None else None
        out = super().conv(x, w, bias, gn_stats=gn_stats, **kw)
        if gn_stats is not None and not self.done:
            self.done = True
            d = gn_stats[0, :, 0] - before[0, :, 0]
            g = int(d.abs().argmax())
            gn_stats[0, g, 0] += int(round(float(d[g]) * 2.0 ** -10))
        return out


class CornerSkipped(HonestOps):
    """replicate_border leaves one corner of its first buffer as it found it."""
    done = False

    def replicate_border(self, xpad):
        corner = xpad[:, :, 0, 0].clone()
        super().replicate_border(xpad)
        if not self.done:
            self.done = True
            xpad[:, :, 0, 0] = corner


class CopyKeepsPadding(HonestOps):
    """copy leaves the channel padding of a wider destination as it found it."""

    def copy(self, x, out):
        self.launches += 1
        out[..., :x.shape[-1]] = x
        return out


class ExtraKernel(HonestOps):
    def groupnorm_v2(self, *a, **kw):
        return self.groupnorm(*a, **kw)


def run_audit(name, dtype, inner, drop_hwpack=False):
    """Encode and decode the golden case's input through AuditOps(inner()); returns the audit."""
    case = CASES[name]
    made = []
    m, _ = build_model(case, lambda: made.append(AuditOps(inner())) or made[-1])
    m = m.to(dtype)
    eng = m._engine()
    ops = made[-1]
    ops.params = eng.p
    if drop_hwpack:   # network inputs through the channel-padded copy instead of the tap-packed conv_in
        for k in [k for k in eng.p if k.endswith(".hwpack")]:
            del eng.p[k]
    x = O.synthetic_video(case["shape"], MANIFEST["input_seed"]).to(dtype)
    post = m.encode(x).latent_dist
    m.decode(post.mode())
    return ops


def _assert_complete(ops):
    total, per_call = ops.launch_identity()
    assert total == per_call and total > 0, (total, per_call)
    assert {r["op"] for r in ops.rows} <= set(AUDITED), summary(ops)


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("name", ["sd21_w32_plain", "sd3_w32_plain", "sd21_w32_image", "sd3_w32_tiled"])
def test_honest_double_passes(name, dt):
    ops = run_audit(name, DTYPES[dt], HonestOps)
    s = summary(ops)
    assert not s["failures"], s
    _assert_complete(ops)
    ops_seen = set(s["calls"])
    assert {"conv", "groupnorm", "pack_weight", "softmax_rows"} <= ops_seen, s["calls"]
    if name.startswith("sd3"):
        assert {"replicate_border", "conv_stacked"} <= ops_seen, s["calls"]
    if name.endswith("tiled"):
        assert {"copy", "blend"} <= ops_seen, s["calls"]
    convs = [r for r in ops.rows if r["op"] == "conv"]
    assert any(r["shortcut"] for r in convs) and any(r["up_time"] == 2 for r in convs) or name.endswith("image")
    assert any(r.get("stats_chained") and r["view"] == "lattice" for r in convs), "no chained statistics on a lattice"
    assert any(r["view"] == "ncdhw" for r in convs), "the encoder's conv_out view is not audited"


def test_honest_double_passes_without_tap_packing():
    """The channel-padded copy of the network input (the engine's path without the tap-packed conv_in)."""
    ops = run_audit("sd21_w32_plain", torch.float16, HonestOps, drop_hwpack=True)
    assert not ops.failures(), summary(ops)
    _assert_complete(ops)
    assert any(r["op"] == "copy" and r["shape_out"][-1] > r["shape_in"][-1] for r in ops.rows)


# name: (double, gate or message the failing row must carry, the rows that may fail after it, tap packing dropped)
DOCTORED = {
    "truncating_store": (TruncatingStore, "2:", False, False),
    "zero_in_last_row": (ZeroInLastRow, "1:", False, False),
    "last_frame_unwritten": (LastFrameUnwritten, "1:", True, False),
    "stats_off": (StatsOff, "5:", False, False),
    "corner_skipped": (CornerSkipped, "bits differ from FakeOps.replicate_border", True, False),
    "copy_keeps_padding": (CopyKeepsPadding, "bits differ from FakeOps.copy", True, True),
}


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("doctor", list(DOCTORED))
def test_doctored_double_fails_at_its_launch(doctor, dt):
    cls, gate, spreads, drop = DOCTORED[doctor]
    name = "sd3_w32_plain" if doctor == "corner_skipped" else "sd21_w32_plain"
    ops = run_audit(name, DTYPES[dt], cls, drop_hwpack=drop)
    bad = ops.failures()
    assert bad, f"{doctor}: the audit passed"
    first = bad[0]
    assert any(f.startswith(gate) for f in first["failed"]), first
    if cls in (TruncatingStore, ZeroInLastRow, LastFrameUnwritten):
        assert first["op"] == "conv" and first["op_index"] == TARGET - 1, first
    if cls is StatsOff:
        assert first["op"] == "conv" and first["layer"], first
    assert first["layer"], first
    if not spreads:   # a wrong value that stays finite: the launches that read it check against the same input
        assert len(bad) == 1, summary(ops)["failures"]
    _assert_complete(ops)


def test_unknown_operator_fails(monkeypatch):
    """An engine that calls a kernel the audit does not know fails, with the call named."""
    orig = Engine.gn

    def gn(self, a, name, *, silu=True, per_frame=False, framed=False):
        if name != "encoder.norm_out":
            return orig(self, a, name, silu=silu, per_frame=per_frame, framed=framed)
        g, b = self.p[name + ".weight"], self.p[name + ".bias"]
        return Act(self.ops.groupnorm_v2(a.t, g, b, self.cfg.groups, self.cfg.eps, silu=silu))

    monkeypatch.setattr(Engine, "gn", gn)
    ops = run_audit("sd21_w32_plain", torch.float16, ExtraKernel)
    bad = ops.failures()
    assert len(bad) == 1 and bad[0]["op"] == "groupnorm_v2" and "unaudited" in bad[0]["failed"][0], summary(ops)
    assert bad[0]["layer"] == "encoder.norm_out.weight", bad[0]
    total, per_call = ops.launch_identity()
    assert total == per_call

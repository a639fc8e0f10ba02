"""The decoder's up-sampler as the engine runs it, fp16 and bf16, against fp64: the kernel against its own spec and the
layer against the reference.

Upsample3D (nearest x2, then a 3x3x3 conv, then for up_time = 2 the channel -> time interleave that drops frame 0) never
runs in that form.  prepack_params folds it into four 3x2x2 phase kernels; Engine.upsample runs one conv per phase into
the (ph::2, pw::2) lattice view of the output, with the interleave and the dropped half in the store, the four launches
adding into one GroupNorm statistics accumulator, and (sd3) on a replicate-framed copy of the input.  At T = 1 the
engine also folds the time taps (Engine._single_frame_weights); the T = 1 cases cover that for the up-sampler and for
the 3x3x3 convs.  Cases are the network's up-samplers with T and H x W cut down, plus the 128-channel plan of the small
models.  Per case:
  1. y against FakeOps(torch.float64) running the same Engine call on the stored weights: gates 1-3 of
     tests/test_gpu_conv_plans.py with K = taps x Cin per launch
  2. y against the oracle's layer in fp64 on the checkpoint's 16-bit weights: gate 1 plus E_w, the fp64 engine on |x|
     with |stored - exact| folded weights and no bias; E_w is at most one weight rounding, u * sum |x| |w_fold|
  3. the plan of every launch: N_cta, full accumulators, interior and edge tiles, the TMA epilogue on the lattice views
  4. the TMA epilogue equals the register one (CVVAE_TMA_EPILOGUE=0) bit for bit, statistics included
  5. lattice canary: phase by phase into a canary-filled buffer with one spare frame in front, each launch changes its
     own lattice only, none leaves a canary in y, and nothing lands in the spare frame (the dropped half of up_time = 2)
  6. the statistics chained over the four launches equal fp64 sums of y, and GroupNorm fed with them equals GroupNorm
     computing its own
Measured values go to upsample16.json in test_gpu_ops.OUT.
"""
import json
import math
import os

import pytest
import torch

import test_gpu_conv_plans as CP
from cvvae_b200.engine import Act, Engine, NetConfig, prepack_params
from fake_ops import FakeOps
from oracle import cvvae_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64
CANARY = -7.75   # exact in fp16 and bf16, far outside the outputs
U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}   # unit roundoff
DTYPES = CP.DTYPES
_RECORD = {}

# name: variant, layer (oracle prefix; an up-sampler when up_time is set), Cin, Cout of the conv, up_time (None: conv3),
# causal, input [T, H, W], expected N_cta
CASES = {
    "sd21_up3": ("sd21", "decoder.up.3.upsample", 512, 1024, 2, False, (2, 20, 44), 256),
    "sd21_up2": ("sd21", "decoder.up.2.upsample", 512, 512, 1, False, (3, 20, 44), 256),
    "sd21_up1": ("sd21", "decoder.up.1.upsample", 256, 512, 2, False, (3, 36, 52), 256),
    "sd3_up0": ("sd3", "decoder.up_blocks.0.upsamplers.0", 512, 1024, 2, False, (2, 20, 44), 256),
    "sd3_up1_causal": ("sd3", "decoder.up_blocks.1.upsamplers.0", 512, 512, 1, True, (3, 20, 44), 256),
    "sd3_up2": ("sd3", "decoder.up_blocks.2.upsamplers.0", 256, 512, 2, False, (3, 36, 52), 256),
    # BN = 128 with NACC = 2 and >= 2 x 132 CTAs per sample and phase: the plan of the width-32 / 64 models
    "sd21_c128": ("sd21", "decoder.up.2.upsample", 128, 128, 1, False, (3, 150, 170), 128),
    # single frame: the time taps folded, of up_time = 2 only the kept half of the channels computed
    "sd21_up3_t1": ("sd21", "decoder.up.3.upsample", 512, 1024, 2, False, (1, 20, 44), 256),
    "sd21_up2_t1": ("sd21", "decoder.up.2.upsample", 512, 512, 1, False, (1, 20, 44), 256),
    "sd3_up0_t1": ("sd3", "decoder.up_blocks.0.upsamplers.0", 512, 1024, 2, False, (1, 20, 44), 256),
    "sd21_conv3_causal_t1": ("sd21", "decoder.up.2.block.0.conv1", 512, 512, None, True, (1, 40, 44), 256),
    "sd21_conv3_t1": ("sd21", "decoder.up.2.block.0.conv1", 512, 512, None, False, (1, 40, 44), 256),
    "sd3_conv3_t1": ("sd3", "decoder.up_blocks.1.resnets.0.conv1", 512, 512, None, False, (1, 40, 44), 256),
}


class _Recording:
    """CudaOps that keeps the arguments of every conv launch (for the plan query and the per-phase replay)."""

    def __init__(self):
        from cvvae_b200.ops import CudaOps
        self.inner, self.calls = CudaOps(), []

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def conv(self, x, w, bias, **kw):
        self.calls.append((x, w, bias, kw))
        return self.inner.conv(x, w, bias, **kw)


def _setup(name, dt):
    variant, p, ci, co, up_time, causal, (T, H, W), _ = CASES[name]
    dtype = DTYPES[dt]
    wkey = p + (".conv" if up_time else "")
    taps = (co, ci, 3, 3, 3)
    sd16 = {wkey + ".weight": O.synth_param(wkey + ".weight", taps, 1234).to(dtype).to(DEV),
            wkey + ".bias": O.synth_param(wkey + ".bias", (co,), 1234).to(dtype).to(DEV)}
    net = NetConfig(variant=variant, z_channels=4 if variant == "sd21" else 16, causal_decoder=causal)
    g = torch.Generator().manual_seed(list(CASES).index(name))
    x = ((torch.rand((1, T, H, W, ci), generator=g) * 2 - 1)).to(dtype).to(DEV)
    return variant, p, wkey, up_time, causal, dtype, sd16, net, x


def _run(eng, wkey, up_time, causal, x):
    """Engine.upsample, or the conv3 with its single-frame fold; returns (y, chained statistics or None)."""
    if up_time:
        a = eng.upsample(Act(x), wkey, up_time, causal)
    else:
        a = eng.conv3(Act(x), wkey, causal)
    return a.t, a.stats


def _engine64(net, params):
    ops = FakeOps(F64)
    return Engine(net, params, ops, F64)


def _dump():
    os.makedirs(CP.OUT, exist_ok=True)
    with open(os.path.join(CP.OUT, "upsample16.json"), "w") as f:
        json.dump(_RECORD, f, indent=1, sort_keys=True)


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("name", list(CASES))
def test_upsample_folds_fp64(name, dt, monkeypatch):
    variant, p, wkey, up_time, causal, dtype, sd16, net, x = _setup(name, dt)
    n_cta = CASES[name][7]
    ci = x.shape[4]
    B = x.shape[0]
    failed, rec = [], {}

    # the production run, and the same run through the register epilogue
    runs = {}
    for switch in ("1", "0"):
        monkeypatch.setenv("CVVAE_TMA_EPILOGUE", switch)
        ops = _Recording()
        eng = Engine(net, prepack_params(sd16, ops.inner, dtype), ops, dtype)
        y, st = _run(eng, wkey, up_time, causal, x)
        plans = []
        for (xi, wi, bi, kw) in ops.calls:
            qkw = {k: v for k, v in kw.items() if k not in ("ref_taps", "k_alg", "force")}
            plans.append(ops.conv_tc_plan(xi, wi, bi, epilogue=True, **qkw))
        runs[switch] = (y, st, plans, ops, eng)
    torch.cuda.synchronize()
    y, st, plans, ops, eng = runs["1"]
    monkeypatch.setenv("CVVAE_TMA_EPILOGUE", "1")

    # 3: the plan of every launch
    n_launch = 4 if up_time else 1
    assert len(ops.calls) == n_launch, len(ops.calls)
    Ho, Wo = ops.calls[0][3]["out"].shape[2:4]
    for pl in plans:
        assert pl["eligible"] == 1 and pl["flat"] == 0 and pl["N_cta"] == n_cta and pl["NACC"] == 256 // n_cta, pl
        assert pl["tma_epilogue"] == 1, pl
        interior = (Wo // pl["TW"]) * (Ho // pl["TH"])
        assert interior > 0 and pl["tiles_w"] * pl["tiles_h"] > interior, (pl, Ho, Wo)
        if n_cta == 128:
            assert pl["grid"] // B >= CP.MIN_CTAS_PER_SAMPLE, pl
    assert all(pl0["tma_epilogue"] == 0 for pl0 in runs["0"][2]), runs["0"][2]
    rec["plan"] = plans[0]

    # 4: TMA epilogue == register epilogue, bit for bit
    y0, st0 = runs["0"][0], runs["0"][1]
    rec["tma_equals_register"] = torch.equal(y, y0) and (st is None or torch.equal(st, st0))
    if not rec["tma_equals_register"]:
        failed.append(f"4: TMA and register epilogues differ ({int((y != y0).sum().item())} elements)")

    # 1: against the same Engine call in fp64 on the stored weights (single-frame folds included)
    stored = {k: v.to(F64) for k, v in eng.p.items()}
    xd = x.to(F64)
    r, _ = _run(_engine64(net, stored), wkey, up_time, causal, xd)
    S, _ = _run(_engine64(net, {k: v.abs() for k, v in stored.items()}), wkey, up_time, causal, xd.abs())
    w_launch = ops.calls[0][1]
    K = w_launch.shape[0] * ci
    yd = y.to(F64)
    ulp = CP._ulp(r, dtype)
    err = yd - r
    bound = 0.5 * ulp + CP.C_ACC * 2.0 ** -24 * math.sqrt(K) * S
    ratio = (err.abs() / bound).max().item()
    if not ratio <= 1.0:
        failed.append(f"1: |y - r| exceeds the bound by {ratio:.3f}x")
    share = (yd == torch.round(r / ulp) * ulp).double().mean().item()
    min_share = 1.0 - CP.MISMATCH_MARGIN * CP.MISMATCH_EST[dtype]
    if not share >= min_share:
        failed.append(f"2: {share:.4f} correctly rounded < {min_share:.4f}")
    mean_ulp = (err / ulp).mean().item()
    if not abs(mean_ulp) <= CP.MAX_MEAN_ULP:
        failed.append(f"3: mean signed error {mean_ulp:+.4f} ulp")
    rec.update({"K": K, "numel": y.numel(), "worst_bound_ratio": ratio, "correctly_rounded_share": share,
                "min_share": min_share, "mean_signed_ulp": mean_ulp})

    # 2: against the oracle's layer in fp64 on the checkpoint's weights; E_w from |stored - exact| folded weights
    sd64 = {k: v.to(F64) for k, v in sd16.items()}
    exact_eng = _engine64(net, prepack_params(sd64, FakeOps(F64), F64))
    _run(exact_eng, wkey, up_time, causal, xd)          # creates the exact single-frame folds
    exact = exact_eng.p
    dw = {k: ((v - exact[k]).abs() if k in exact and not k.endswith("bias") else torch.zeros_like(v))
          for k, v in stored.items()}
    Ew, _ = _run(_engine64(net, dw), wkey, up_time, causal, xd.abs())
    Sw, _ = _run(_engine64(net, {k: (exact[k].abs() if not k.endswith("bias") else torch.zeros_like(v))
                                 for k, v in stored.items()}), wkey, up_time, causal, xd.abs())
    ncdhw = xd.permute(0, 4, 1, 2, 3)
    if not up_time:
        want = (O.sd21_conv(ncdhw, sd64, wkey, causal, 1) if variant == "sd21"
                else O.sd3_conv3d(ncdhw, sd64, wkey, causal, 1))
    elif variant == "sd21":
        want = O.sd21_upsample(ncdhw, sd64, p, up_time=up_time == 2)
    else:
        want = O.sd3_upsample(ncdhw, sd64, p, up_time=up_time == 2, causal=causal)
    want = want.permute(0, 2, 3, 4, 1)
    assert want.shape == y.shape, (want.shape, y.shape)
    layer_ratio = ((yd - want).abs() / (bound + Ew)).max().item()
    ew_ratio = (Ew / (U[dtype] * Sw).clamp_min(1e-300)).max().item()
    rec.update({"layer_bound_ratio": layer_ratio, "Ew_over_one_rounding": ew_ratio})
    if not layer_ratio <= 1.0:
        failed.append(f"layer: |y - oracle| exceeds gate 1 + E_w by {layer_ratio:.3f}x")
    if not ew_ratio <= 1.0:
        failed.append(f"layer: E_w is {ew_ratio:.3f}x one weight rounding")
    del r, S, err, bound, Ew, Sw, want, dw, exact, stored

    # 5: phase by phase into a canary buffer with a spare frame in front of y
    if up_time:
        Bq, Tq, Hq, Wq, Cq = y.shape
        buf = torch.full((Bq, Tq + 1, Hq, Wq, Cq), CANARY, dtype=dtype, device=DEV)
        yc = buf[:, 1:]
        done = torch.zeros((Hq, Wq), dtype=torch.bool, device=DEV)
        for i, (xi, wi, bi, kw) in enumerate(ops.calls):
            ph, pw = divmod(i, 2)
            ops.inner.conv(xi, wi, bi, **dict(kw, out=yc[:, :, ph::2, pw::2], gn_stats=None))
            torch.cuda.synchronize()
            changed = (yc != CANARY).all(dim=4).all(dim=1).all(dim=0)
            untouched = (yc == CANARY).all(dim=4).all(dim=1).all(dim=0)
            done[ph::2, pw::2] = True
            if not (torch.equal(changed, done) and torch.equal(untouched, ~done)):
                failed.append(f"5: phase {ph}{pw} wrote outside its lattice or left part of it unwritten")
                break
        if not bool((buf[:, 0] == CANARY).all()):
            failed.append("5: a launch wrote the frame in front of y (the dropped half of the interleave)")
        if not torch.equal(yc, y):
            failed.append("5: the phase-by-phase replay differs from Engine.upsample")
        del buf

    # 6: statistics chained over the four launches
    if up_time:
        groups = net.groups
        yC = y.shape[4]
        v = yd.reshape(B, -1, groups, yC // groups)
        want_st = torch.stack([v.sum(dim=(1, 3)), (v * v).sum(dim=(1, 3))], dim=-1)
        got = torch.stack([st[..., 0].double() / 2.0 ** 20, st[..., 1].double() / 2.0 ** 18], dim=-1)
        rec["stats_max_abs_err"] = (got - want_st).abs().max().item()
        try:
            torch.testing.assert_close(got, want_st, rtol=1e-5, atol=2e-2)
        except AssertionError as e:
            failed.append(f"6: chained statistics vs fp64 sums of y: {str(e).splitlines()[0:4]}")
        gam = CP._rand((yC,), torch.float32, 21) * 0.5 + 1.0
        bet = CP._rand((yC,), torch.float32, 22, 0.2)
        tol = dict(rtol=1e-3, atol=1e-4) if dtype == torch.float16 else dict(rtol=8e-3, atol=1e-3)
        try:
            torch.testing.assert_close(ops.groupnorm(y, gam, bet, groups, 1e-5, stats=st).float(),
                                       ops.groupnorm(y, gam, bet, groups, 1e-5).float(), **tol)
        except AssertionError as e:
            failed.append(f"6: GroupNorm with the chained statistics: {str(e).splitlines()[0:4]}")
    rec["failed_gates"] = failed
    _RECORD[f"{name}/{dt}"] = rec
    _dump()
    assert not failed, f"{name}/{dt}: " + "; ".join(failed)

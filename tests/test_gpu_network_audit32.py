"""Every launch of full-tile encode and decode passes of float32 models (TF32 products) against its operation in fp64.

The harness, weights and inputs of tests/test_gpu_network_audit.py, in fp32, where network_audit.AuditOps picks the
fp32 gates (tests/attention_gates.py): every tensor-core operand read truncated to TF32, convolution / GEMM outputs
under gate 1 with K = 8 per MMA, full-precision stores (F) and truncated, not rounded, operand reads (R); the MMA-only
producers under gates
1-3 with TF32 as the store format and T; the gather, pack_taps_hw and the packed weights bit for bit against RN-TF32.
These reach fp32 paths that run at network shapes only inside a full pass: the NCDHW decoder conv_out through conv_tc
(no tap-stacked kernel in fp32), the spatial attention with an fp32 P (twice the scratch per frame, its own frame
grouping) at N = 5184 / 4096 and on the ragged clip's tiles, and the truncated reads of block outputs by the re-sampling
convolutions, the fused shortcuts, q / k / v^T and proj_out.

Each case asserts zero failed gates, launch identity and only audited operators; the 17-frame cases also PLANS32 and the
coverage of _covered32.  Rows, wall time and peak memory go to network_audit32.json in test_gpu_ops.OUT.
"""
import json
import os
import time

import pytest
import torch

import test_gpu_ops
from network_audit import AUDITED, AuditOps, summary
from oracle import cvvae_oracle as O
from test_gpu_network_audit import _model, _plan_set

pytestmark = pytest.mark.gpu
OUT = test_gpu_ops.OUT
_RECORD = {}

# name: variant, input [B, C, T, H, W]
CASES = {
    "sd21_576_fp32": ("sd21", (1, 3, 17, 576, 576)),
    "sd3_512_fp32": ("sd3", (1, 3, 17, 512, 512)),
    "sd21_image_576_fp32": ("sd21", (1, 3, 1, 576, 576)),
    "sd21_tiled_576x704_fp32": ("sd21", (1, 3, 9, 576, 704)),
}

# (N_cta, NACC, vec2, tma_epilogue) of the tensor-core convolutions of one fp32 pass, read off the first recorded run on
# an H100 80GB HBM3 (the same set for sd21 at 576^2 and sd3 at 512^2).  fp32 has no TMA epilogue; BN = 64 is the NCDHW
# conv_out, NACC 1 in the encoder (Cout = 8 / 32) and NACC 4 in the decoder (Cout = 3).  Measured on that run: about
# 21 s and 28.5 GB peak for sd21 at 17x576x576, 17 s and 22.9 GB for sd3 at 17x512x512.
PLANS32 = [(64, 1, 0, 0), (64, 4, 0, 0), (128, 2, 1, 0), (256, 1, 1, 0)]


def _low_bits(r):
    return max(r.get("x_low_bits_share", 0.0), r.get("sc_x_low_bits_share", 0.0), r.get("w_low_bits_share", 0.0))


def _covered32(rows):
    """What a full 17-frame fp32 pass is meant to reach."""
    convs = [r for r in rows if r["op"] == "conv"]
    plans = [r["plan"] for r in convs if r["plan"]["eligible"]]
    return {
        "N_cta_128_NACC_2": any(p["N_cta"] == 128 and p["NACC"] == 2 for p in plans),
        "N_cta_256": any(p["N_cta"] == 256 for p in plans),
        "register_epilogue_only": bool(plans) and all(p["tma_epilogue"] == 0 for p in plans),
        "every_conv_on_tensor_cores": all(r["plan"]["eligible"] for r in convs),
        "fused_shortcut": any(r["shortcut"] for r in convs),
        "lattice_chained_stats": any(r["view"] == "lattice" and r.get("stats_chained") for r in convs),
        "up_time_2": any(r["up_time"] == 2 for r in convs),
        "ncdhw_conv_out_on_conv_tc": sum(r["view"] == "ncdhw" and r["plan"]["eligible"] for r in convs) >= 2,
        "no_conv_stacked": not any(r["op"] == "conv_stacked" for r in rows),
        "truncated_operand": any(_low_bits(r) > 0.5 for r in convs if not r["batched"]),
        "o_equals_p_v_K_4096": any(r["batched"] and r["K"] >= 4096 and r.get("w_low_bits_share", 0.0) > 0.5
                                   for r in convs),
        "groupnorm_P_t_200": any(r["op"] == "groupnorm" and max(r.get("P_t", 0), r.get("kernel_stats_twin", {}).get("P_t", 0))
                                 >= 200 for r in rows),
    }


def _extremes(rows):
    """The measured values the fp32 gates are judged by, over all launches of a pass."""
    convs = [r for r in rows if r["op"] == "conv"]
    producers = [r for r in rows if r["op"] in ("groupnorm", "layernorm", "softmax_rows")]
    gn = [r for r in rows if r["op"] == "groupnorm"]
    out = {
        "max_rms_error_ratio": max((r["rms_error_ratio"] for r in convs), default=None),
        "tf32_valued_share_min_max": [min((r["tf32_valued_share"] for r in convs), default=None),
                                      max((r["tf32_valued_share"] for r in convs), default=None)],
        "max_conv_bound_ratio": max((r["worst_bound_ratio"] for r in convs), default=None),
        "min_producer_correctly_rounded_share": min((r["correctly_rounded_share"] for r in producers), default=None),
        "min_sq_headroom_bits": min((r["sq_headroom_bits"] for r in gn), default=None),
    }
    worst = max(convs, key=lambda r: r["rms_error_ratio"], default=None)
    if worst is not None:
        out["max_rms_error_ratio_at"] = {k: worst.get(k) for k in ("i", "layer", "K", "batched", "x_low_bits_share")}
    return out


def _dump():
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "network_audit32.json"), "w") as f:
        json.dump(_RECORD, f, indent=1, sort_keys=True)


@pytest.mark.parametrize("name", list(CASES))
def test_network_audit_fp32(name):
    from cvvae_b200.ops import CudaOps
    variant, shape = CASES[name]
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    made = []
    m = _model(variant, torch.float32, lambda: made.append(AuditOps(CudaOps())) or made[-1])
    eng = m._engine()
    ops = made[-1]
    ops.params = eng.p
    x = O.synthetic_video(shape, 21).float().cuda()
    post = m.encode(x).latent_dist
    rec = m.decode(post.mode()).sample
    torch.cuda.synchronize()
    assert rec.shape == x.shape and rec.dtype == torch.float32
    total, per_call = ops.launch_identity()
    s = summary(ops)
    entry = {"wall_s": time.perf_counter() - t0, "peak_memory_gb": torch.cuda.max_memory_allocated() / 2 ** 30,
             "launches": total, "launches_in_audited_calls": per_call, "calls": s["calls"], "failures": s["failures"],
             "plans": _plan_set(ops.rows), "extremes": _extremes(ops.rows), "rows": ops.rows}
    if shape[2] == 17:
        entry["coverage"] = _covered32(ops.rows)
    _RECORD[name] = entry
    _dump()
    assert not s["failures"], s["failures"][:20]
    assert total == per_call and total > 0, (total, per_call)
    assert set(s["calls"]) <= set(AUDITED), s["calls"]
    if shape[2] == 17:
        missing = [k for k, v in entry["coverage"].items() if not v]
        assert not missing, f"the pass is smaller than intended: {missing}"
        assert [tuple(p) for p in entry["plans"]] == PLANS32, entry["plans"]
    if name.startswith("sd21_tiled"):
        assert s["calls"].get("copy", 0) >= 2 and s["calls"].get("blend", 0) >= 2, s["calls"]

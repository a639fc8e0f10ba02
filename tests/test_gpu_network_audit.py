"""Every launch of full-tile encode and decode passes against its operation in fp64, fp16 and bf16.

The end-to-end statistics (tests/test_gpu_fullsize.py, tests/test_gpu_e2e.py) absorb a defect confined to one layer, and
the bit-equality tests (tiling, streaming, graphs, batching) reproduce it on both sides.  Here tests/network_audit.py
checks each launch of a pass on the tensors the network actually passes, under that op's gates: sd21 at the 576^2 pixel
tile every full-size configuration runs (the 5184-token mid-block), sd3 at C3's 512^2 tile, the image path (T = 1) and
two overlapping tiles of which one is ragged, so the tiler's copy and blend run on their real buffers.  Weights are
make_state_dict's with randomised norm parameters and biases (as tests/test_gpu_fullsize.py), inputs synthetic_video's.

Each case asserts zero failed gates and that every library launch happened inside an audited call; the 17-frame cases
also that the pass reached what it is meant to reach (PLANS, the frozen set of conv_tc plans a pass runs, and the
coverage of _covered).  Rows, wall time and peak memory go to network_audit.json in test_gpu_ops.OUT.
"""
import json
import os
import time

import pytest
import torch

import test_gpu_ops
from network_audit import AUDITED, AuditOps, summary
from oracle import cvvae_oracle as O

pytestmark = pytest.mark.gpu
OUT = test_gpu_ops.OUT
_RECORD = {}

# name: variant, dtype, input [B, C, T, H, W]
CASES = {
    "sd21_576_fp16": ("sd21", torch.float16, (1, 3, 17, 576, 576)),
    "sd21_576_bf16": ("sd21", torch.bfloat16, (1, 3, 17, 576, 576)),
    "sd3_512_fp16": ("sd3", torch.float16, (1, 3, 17, 512, 512)),
    "sd3_512_bf16": ("sd3", torch.bfloat16, (1, 3, 17, 512, 512)),
    "sd21_image_576_fp16": ("sd21", torch.float16, (1, 3, 1, 576, 576)),
    "sd3_image_512_bf16": ("sd3", torch.bfloat16, (1, 3, 1, 512, 512)),
    "sd21_tiled_576x704_bf16": ("sd21", torch.bfloat16, (1, 3, 9, 576, 704)),
}


# (N_cta, NACC, vec2, tma_epilogue) of the tensor-core convolutions of one pass, read off the first recorded run on an H100
# (the same set for sd21 at 576^2 and sd3 at 512^2, fp16 and bf16): BN = 64 is the NCDHW conv_out
PLANS = [(64, 1, 0, 0), (128, 2, 1, 1), (256, 1, 1, 0), (256, 1, 1, 1)]


def _model(variant, dtype, ops_factory):
    from cvvae_b200 import CVVAEModel, CVVAESD3Model
    cfg = O.VAEConfig(variant=variant) if variant == "sd21" else O.VAEConfig(variant="sd3", z_channels=16)
    sd = O.make_state_dict(cfg, 4242)
    g = torch.Generator().manual_seed(8)
    for k, v in sd.items():
        if v.dim() == 1:
            bias = k.endswith("bias")
            v.copy_(torch.rand(v.shape, generator=g) * (0.4 if bias else 1.0) + (-0.2 if bias else 0.5))
    m = CVVAEModel() if variant == "sd21" else CVVAESD3Model()
    m.load_state_dict(sd, strict=True)
    m._ops_factory = ops_factory
    return m.to(dtype).cuda()


def _plan_set(rows):
    return sorted({tuple(r["plan"][k] for k in ("N_cta", "NACC", "vec2", "tma_epilogue"))
                   for r in rows if r["op"] == "conv" and r.get("plan", {}).get("eligible")})


def _covered(rows):
    """What a full 17-frame pass is meant to reach."""
    convs = [r for r in rows if r["op"] == "conv"]
    plans = [r["plan"] for r in convs if r["plan"]["eligible"]]
    return {
        "N_cta_128_NACC_2": any(p["N_cta"] == 128 and p["NACC"] == 2 for p in plans),
        "N_cta_256": any(p["N_cta"] == 256 for p in plans),
        "tma_epilogue": any(p["tma_epilogue"] == 1 for p in plans),
        "register_epilogue": any(p["tma_epilogue"] == 0 for p in plans),
        "fused_shortcut": any(r["shortcut"] for r in convs),
        "lattice_chained_stats": any(r["view"] == "lattice" and r.get("stats_chained") for r in convs),
        "up_time_2": any(r["up_time"] == 2 for r in convs),
        "ncdhw_conv_out": any(r["view"] == "ncdhw" for r in convs),
        "groupnorm_P_t_200": any(r["op"] == "groupnorm" and max(r.get("P_t", 0), r.get("kernel_stats_twin", {}).get("P_t", 0))
                                 >= 200 for r in rows),
    }


def _dump():
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "network_audit.json"), "w") as f:
        json.dump(_RECORD, f, indent=1, sort_keys=True)


@pytest.mark.parametrize("name", list(CASES))
def test_network_audit(name):
    from cvvae_b200.ops import CudaOps
    variant, dtype, shape = CASES[name]
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    made = []
    m = _model(variant, dtype, lambda: made.append(AuditOps(CudaOps())) or made[-1])
    eng = m._engine()
    ops = made[-1]
    ops.params = eng.p
    x = O.synthetic_video(shape, 21).to(dtype).cuda()
    post = m.encode(x).latent_dist
    rec = m.decode(post.mode()).sample
    torch.cuda.synchronize()
    assert rec.shape == x.shape
    total, per_call = ops.launch_identity()
    s = summary(ops)
    entry = {"wall_s": time.perf_counter() - t0, "peak_memory_gb": torch.cuda.max_memory_allocated() / 2 ** 30,
             "launches": total, "launches_in_audited_calls": per_call, "calls": s["calls"], "failures": s["failures"],
             "plans": _plan_set(ops.rows), "rows": ops.rows}
    if shape[2] == 17:
        entry["coverage"] = _covered(ops.rows)
    _RECORD[name] = entry
    _dump()
    assert not s["failures"], s["failures"][:20]
    assert total == per_call and total > 0, (total, per_call)
    assert set(s["calls"]) <= set(AUDITED), s["calls"]
    if shape[2] == 17:
        missing = [k for k, v in entry["coverage"].items() if not v]
        assert not missing, f"the pass is smaller than intended: {missing}"
        assert [tuple(p) for p in entry["plans"]] == PLANS, entry["plans"]
    if name.startswith("sd21_tiled"):
        assert s["calls"].get("copy", 0) >= 2 and s["calls"].get("blend", 0) >= 2, s["calls"]

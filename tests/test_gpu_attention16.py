"""The mid-block spatial attention at the tiler's token counts, fp16 and bf16, stage by stage and end to end against fp64.

Engine.spatial_attention runs three batched conv_tc GEMMs on the flat plan (v^T = W_v hn^T + b_v with a shared left
operand and the bias along M; S = alpha q k^T into fp32; O = P v with K = N and weight row stride ld = ceil8(N)) and one
softmax_rows, over groups of fg frames whose [fg, N, ld] buffers stay under attn_scratch_bytes.  The token counts are
those the tiler produces (see CASES); C = 512 is the mid-block width of both full models, C = 128 that of the small ones.
Per case and dtype:
  A. each GEMM on the engine's buffer layout, written through the [:n, :, :N] views, against fp64 on the same 16-bit
     inputs under gates 1-3 of tests/attention_gates.py (the fp32 logits: gate 1); the batched logits equal per-frame
     launches bit for bit; the plans (flat, N_cta, NACC, TMA epilogue) through cvvae_conv_tc_plan()
  B. softmax_rows over S[:n].view(n N, ld) under its bound; canaries in the padding columns N..ld of S, P and v^T and in
     the frames n..fg of a partial last group stay untouched, and NaN in the padding columns of P and v^T does not reach O
  C. Engine.spatial_attention against softmax(C^-1/2 q k^T)(hn W_v^T + b_v) in fp64 (attention_gates.attention_reference);
     bit for bit equal to the staged run, to runs with fg = 1 and fg = 2, to the register epilogue, to per-sample runs
     (B = 2), and to a run whose scratch buffers start as NaN
  D. the three attention blocks (attn_sd21 encoder and spatial-temporal decoder, attn_sd3) at N = 2295 / 3060 and 5184 on
     oracle.synth_param weights: every launch replayed on its recorded inputs against fp64 - the per-frame GroupNorm
     (tests/test_gpu_kernels16.py's bound, several CTAs per frame), the flat 1x1 convolutions (TMA epilogue, residual),
     LayerNorm, temporal attention and the spatial attention end to end; the last conv's fused GroupNorm statistics
     (a flat plan with statistics) against fp64 sums of its output, and bit for bit against the register epilogue
  E. negative controls: a store rounding toward zero fails gates 2-3, O without its last K block fails gate 1, O with a
     token shifted or two frames swapped fails the end-to-end gate, statistics with one group's sum off by one unit of
     the fixed-point format fail the bit-for-bit comparison
Peak device memory stays under 16 GB per case.  Measured values go to attention16.json in test_gpu_ops.OUT.
"""
import json
import os

import pytest
import torch

import attention_gates as AG
import kernel_bounds as KB
import test_gpu_ops
from cvvae_b200.engine import Engine, NetConfig, _round_once
from test_gpu_upsample16 import _Recording

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
CANARY = -7.75            # exact in fp16, bf16 and fp32, far outside every output
MAX_PEAK = 16 << 30
ROWS = 2048               # query rows per fp64 reference chunk
_RECORD = {}

# name: (H, W) of the latent tile, C, T, B, the branches the token count reaches (attention_gates.branches)
CASES = {
    # 800x600 corner tile (sd21 and sd3): ld > N, ragged K block of 4 tokens (one MMA), partial 256-token tile; B = 2
    "n836_corner_b2": ((19, 44), 512, 5, 2, dict(ld_gt_n=True, odd_n=False, ragged_k_block=True, guarded_k_block=True,
                                               partial_channel_tile=True)),
    # SD3 at 854x360, right tile: odd N, N % 64 = 55.  S and v^T have Cout = N odd, so their last channel goes through the
    # single-element (c1ok) store.  That depends on the parity of Cout alone, so N's parity is the proof; a paired store
    # that overran would hit the canary in column N
    "n2295_odd": ((45, 51), 512, 5, 1, dict(ld_gt_n=True, odd_n=True, ragged_k_block=True, guarded_k_block=False,
                                          partial_channel_tile=True)),
    # SD3 at 854x480, right tile: N % 8 = 4, N % 64 = 52
    "n3060": ((60, 51), 512, 5, 1, dict(ld_gt_n=True, odd_n=False, ragged_k_block=True, guarded_k_block=False,
                                      partial_channel_tile=True)),
    # 854x480 / 640x480, left tile: N % 64 = 32 (two MMAs in the last K block), N % 256 = 224
    "n4320": ((60, 72), 512, 5, 1, dict(ld_gt_n=False, odd_n=False, ragged_k_block=True, guarded_k_block=True,
                                      partial_channel_tile=True)),
    # every full 576-px tile (the default): N % 256 = 64
    "n5184_tile": ((72, 72), 512, 5, 1, dict(ld_gt_n=False, odd_n=False, ragged_k_block=False, guarded_k_block=False,
                                           partial_channel_tile=True)),
    # 1024x576 untiled
    "n9216_untiled": ((72, 128), 512, 3, 1, dict(ld_gt_n=False, odd_n=False, ragged_k_block=False, guarded_k_block=False,
                                               partial_channel_tile=False)),
    # 1280x720 untiled: the largest K here
    "n14400_720p": ((90, 160), 512, 2, 1, dict(ld_gt_n=False, odd_n=False, ragged_k_block=False, guarded_k_block=False,
                                             partial_channel_tile=True)),
    # the small models' 128-channel mid-block: O runs on the 128-channel tile
    "c128_n4320": ((60, 72), 128, 5, 1, dict(ld_gt_n=False, odd_n=False, ragged_k_block=True, guarded_k_block=True,
                                           partial_channel_tile=True)),
}


def _rand(shape, dtype, seed, scale=1.0, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(shape, generator=g, dtype=F64) * 2 - 1) * scale + offset).to(dtype).to(DEV)


def _dump():
    os.makedirs(test_gpu_ops.OUT, exist_ok=True)
    with open(os.path.join(test_gpu_ops.OUT, "attention16.json"), "w") as f:
        json.dump(_RECORD, f, indent=1, sort_keys=True)


class _NanEmpty(_Recording):
    """Scratch and output buffers of the engine start as NaN."""

    @staticmethod
    def empty(shape, dtype, device):
        return torch.full(tuple(shape), float("nan"), dtype=dtype, device=device)


def _engine(ops, wv, bv, dtype):
    return Engine(NetConfig(), {"a.v.weight": wv, "a.v.bias": bv}, ops, dtype)


def _attention_refs(hf, qf, kf, wv64, bv64, alpha32, dtype):
    """(frame, query rows, fp64 attention o, end-to-end bound E) over [F, N, C] operands, in row chunks."""
    C = hf.shape[2]
    for f in range(hf.shape[0]):
        h64, q64, k64 = hf[f].double(), qf[f].double(), kf[f].double()
        v = h64 @ wv64.T + bv64
        dv = AG.stored_bound(v, AG.gemm_bound(C, h64.abs() @ wv64.abs().T + bv64.abs()), dtype)
        for rows in AG.row_chunks(hf.shape[1], ROWS):
            o, E = AG.attention_reference(q64[rows], k64, v, dv, alpha32, dtype)
            yield f, rows, o, E


def _plan(ops, call):
    x, w, b, kw = call
    return ops.conv_tc_plan(x, w, b, epilogue=True, **{k: v for k, v in kw.items() if k not in ("force", "ref_taps", "k_alg")})


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("name", list(CASES))
def test_spatial_attention16(name, dt, monkeypatch):
    (H, W), C, T, B, want_br = CASES[name]
    dtype = DTYPES[dt]
    torch.cuda.reset_peak_memory_stats()
    t_start = torch.cuda.Event(enable_timing=True)
    t_start.record()
    N, F = H * W, B * T
    ld = (N + 7) // 8 * 8
    br = AG.branches(N)
    assert br == want_br, (br, want_br)
    alpha = float(C) ** -0.5
    alpha32 = torch.tensor(alpha, dtype=torch.float32).item()     # what the kernel receives (C^-1/2 is not exact)
    s = 4.5 ** 0.5                                                 # logits with standard deviation 1.5
    hn = _rand((B, T, H, W, C), dtype, 1, 1.7)
    q = _rand((B, T, H, W, C), dtype, 2, s)
    k = _rand((B, T, H, W, C), dtype, 3, s)
    wv = _rand((1, C, C), dtype, 4, C ** -0.5)                    # packed [taps, Cout, Cin]
    bv = _rand((C,), torch.float32, 5, 0.2, 0.5)                  # O stays positive: gate 3 sees a directed rounding
    failed, rec = [], {"N": N, "ld": ld, "C": C, "T": T, "B": B, "branches": br}

    # ---------------------------------------------------------------- the engine (C), recorded
    monkeypatch.setenv("CVVAE_TMA_EPILOGUE", "1")
    ops = _Recording()
    y = _engine(ops, wv, bv, dtype).spatial_attention(hn, q, k, "a.v")
    assert len(ops.calls) == 3, "the default scratch cap holds every frame in one group"
    plans = {st: _plan(ops.inner, c) for st, c in zip(("vT", "S", "O"), ops.calls)}
    rec["plans"] = plans
    n_cta_o = 256 if C >= 256 else 128
    for st, pl in plans.items():
        n_cta = n_cta_o if st == "O" else 256
        m_rows = C if st == "vT" else N                        # positions of the flat problem: rows of the GEMM
        cout = C if st == "O" else N
        assert pl["eligible"] == 1 and pl["flat"] == 1, (st, pl)
        assert pl["N_cta"] == n_cta and pl["NACC"] == 1, (st, pl)       # too few CTAs per frame for NACC = 2
        assert pl["n_tiles_n"] == -(-cout // n_cta) and pl["tiles_w"] == -(-m_rows // 128), (st, pl)
        assert pl["grid"] == pl["n_tiles_n"] * pl["tiles_w"] * F, (st, pl)
        assert pl["tma_epilogue"] == (1 if st == "O" else 0), (st, pl)  # fp32 logits and bias along M: registers
    if br["ragged_k_block"]:
        assert ops.calls[2][0].shape[4] == N and N % 64, "O's K is N with a ragged last 64-channel block"

    # ---------------------------------------------------------------- A / B: the stages on the engine's layout
    hf, qf, kf = (t.reshape(F, N, C) for t in (hn, q, k))
    fg = F - 1 if F > 2 else 1                                    # a partial last group wherever F > 2
    vT = torch.empty((fg, C, ld), dtype=dtype, device=DEV)
    S = torch.empty((fg, N, ld), dtype=torch.float32, device=DEV)
    P = torch.empty((fg, N, ld), dtype=dtype, device=DEV)
    S1 = torch.empty((N, ld), dtype=torch.float32, device=DEV)
    o_st = torch.empty((F, N, C), dtype=dtype, device=DEV)
    wv64, bv64 = wv[0].double(), bv.double()
    g = {"vT": AG.Gates(dtype, K=C), "S": AG.Gates(None), "P": AG.Gates(dtype), "O": AG.Gates(dtype, K=N)}
    canaries_ok, s_batched_equal, neg = True, True, {}
    for f0 in range(0, F, fg):
        n = min(fg, F - f0)
        for t in (vT, S, P):
            t.fill_(CANARY)
        ops.inner.conv(wv.view(1, 1, 1, C, C), hf[f0:f0 + n], bv, bias_along_m=True, x_shared=True, w_per_batch=True,
                       cout=N, out=vT[:n, :, :N].unsqueeze(1).unsqueeze(1))
        ops.inner.conv(qf[f0:f0 + n].view(n, 1, 1, N, C), kf[f0:f0 + n], None, alpha=alpha, out_f32=True, w_per_batch=True,
                       cout=N, out=S[:n, :, :N].unsqueeze(1).unsqueeze(1))
        ops.inner.softmax_rows(S[:n].view(n * N, ld), N, P[:n].view(n * N, ld))
        torch.cuda.synchronize()
        for t in (vT, S, P):
            canaries_ok &= bool((t[:n, :, N:] == CANARY).all()) and bool((t[n:] == CANARY).all())
        for i in range(n):
            f = f0 + i
            h64, q64, k64 = hf[f].double(), qf[f].double(), kf[f].double()
            g["vT"].add(vT[i, :, :N], wv64 @ h64.T + bv64[:, None],
                        AG.gemm_bound(C, wv64.abs() @ h64.abs().T + bv64.abs()[:, None]))
            ops.inner.conv(qf[f:f + 1].view(1, 1, 1, N, C), kf[f:f + 1], None, alpha=alpha, out_f32=True, w_per_batch=True,
                           cout=N, out=S1[:, :N].unsqueeze(0).unsqueeze(0).unsqueeze(0))
            torch.cuda.synchronize()
            s_batched_equal &= torch.equal(S1[:, :N], S[i, :, :N])
            for rows in AG.row_chunks(N, ROWS):
                r = alpha32 * (q64[rows] @ k64.T)
                g["S"].add(S[i, rows, :N], r, AG.logit_bound(C, alpha32, q64[rows].abs() @ k64.abs().T, r))
                sd = S[i, rows, :N].double()
                rp = torch.softmax(sd, dim=-1)
                g["P"].add(P[i, rows, :N], rp, AG.softmax_bound(sd, rp))
                del r, sd, rp
        if ld > N:                                                # NaN past N in both operands of O
            P[:n, :, N:] = float("nan")
            vT[:n, :, N:] = float("nan")
        ops.inner.conv(P[:n, :, :N].unsqueeze(1).unsqueeze(1), vT[:n], None, w_ld=ld, cout=C, w_per_batch=True,
                       out=o_st[f0:f0 + n].view(n, 1, 1, N, C))
        torch.cuda.synchronize()
        for i in range(n):
            v64 = vT[i, :, :N].double()
            for rows in AG.row_chunks(N, ROWS):
                p64 = P[i, rows, :N].double()
                r = p64 @ v64.T
                E = AG.gemm_bound(N, p64 @ v64.abs().T)
                g["O"].add(o_st[f0 + i, rows], r, E)
                if f0 + i == 0 and rows.start == 0:
                    # E: a store rounding toward zero; O without its last K block (64 tokens)
                    neg["O_truncated"] = AG.Gates(dtype, K=N).add(AG.truncate(r, dtype), r, E).result()[1]
                    if br["ragged_k_block"]:
                        kk = N - N % 64
                        short = _round_once(p64[:, :kk] @ v64[:, :kk].T, dtype)
                        neg["O_without_last_k_block"] = AG.Gates(dtype, K=N).add(short, r, E).result()[1]
                del p64, r, E
    del vT, S, P, S1
    for st, gt in g.items():
        rec[st], f_st = gt.result()
        failed += [f"{st} {x}" for x in f_st]
    rec["canaries_untouched"] = canaries_ok
    rec["logits_batched_equal_per_frame"] = s_batched_equal
    if not canaries_ok:
        failed.append("B: a launch wrote a padding column or a frame past its group")
    if not s_batched_equal:
        failed.append("A: batched logits differ from per-frame launches")
    if not bool(torch.isfinite(o_st).all()):
        failed.append("B: NaN in the padding columns of P / v^T reached O")

    # ---------------------------------------------------------------- C: end to end against fp64 attention
    yf = y.reshape(F, N, C)
    e2e = AG.Gates(dtype, half_ulp=False)
    y_shift = torch.roll(yf[0], 1, 0)
    for f, rows, o, E in _attention_refs(hf, qf, kf, wv64, bv64, alpha32, dtype):
        e2e.add(yf[f, rows], o, E)
        if f == 0:
            neg.setdefault("e2e_token_shift", AG.Gates(dtype, half_ulp=False))
            neg["e2e_token_shift"].add(y_shift[rows], o, E)
            if F > 1:
                neg.setdefault("e2e_frames_swapped", AG.Gates(dtype, half_ulp=False))
                neg["e2e_frames_swapped"].add(yf[1, rows], o, E)
        del o, E
    rec["e2e"], f_e = e2e.result()
    failed += [f"end to end {x}" for x in f_e]

    # bit-for-bit identities of the engine's output
    same = {"staged_fg%d" % fg: torch.equal(o_st, yf)}
    Fb = N * ld * 4                                               # scratch per frame (fp32 logits)
    if F > 2:
        for fgx in (1, 2):
            e = _engine(ops.inner, wv, bv, dtype)
            e.attn_scratch_bytes = fgx * Fb
            same[f"fg{fgx}"] = torch.equal(e.spatial_attention(hn, q, k, "a.v"), y)
    same["nan_scratch"] = torch.equal(_engine(_NanEmpty(), wv, bv, dtype).spatial_attention(hn, q, k, "a.v"), y)
    if B > 1:
        e = _engine(ops.inner, wv, bv, dtype)
        same["per_sample"] = all(torch.equal(e.spatial_attention(hn[b:b + 1], q[b:b + 1], k[b:b + 1], "a.v"), y[b:b + 1])
                                 for b in range(B))
    monkeypatch.setenv("CVVAE_TMA_EPILOGUE", "0")
    ops0 = _Recording()
    same["register_epilogue"] = torch.equal(_engine(ops0, wv, bv, dtype).spatial_attention(hn, q, k, "a.v"), y)
    assert _plan(ops0.inner, ops0.calls[2])["tma_epilogue"] == 0
    monkeypatch.setenv("CVVAE_TMA_EPILOGUE", "1")
    rec["bit_equal"] = same
    failed += [f"C: output differs from the {k_} run" for k_, ok in same.items() if not ok]

    # ---------------------------------------------------------------- E: the gates reject doctored outputs
    neg = {k_: (v_.result()[1] if isinstance(v_, AG.Gates) else v_) for k_, v_ in neg.items()}
    rec["negative_controls"] = neg
    if not (any(x.startswith("2:") for x in neg["O_truncated"]) and any(x.startswith("3:") for x in neg["O_truncated"])):
        failed.append("E: gates 2-3 accept a store rounding toward zero")
    for k_ in ("O_without_last_k_block", "e2e_token_shift", "e2e_frames_swapped"):
        if k_ in neg and not any(x.startswith("1:") for x in neg[k_]):
            failed.append(f"E: gate 1 accepts {k_}")
    assert ("O_without_last_k_block" in neg) == br["ragged_k_block"] and ("e2e_frames_swapped" in neg) == (F > 1)

    t_end = torch.cuda.Event(enable_timing=True)
    t_end.record()
    torch.cuda.synchronize()
    rec["peak_bytes"] = torch.cuda.max_memory_allocated()
    rec["seconds"] = t_start.elapsed_time(t_end) / 1000
    if not rec["peak_bytes"] <= MAX_PEAK:
        failed.append(f"peak device memory {rec['peak_bytes'] / 2 ** 30:.2f} GB")
    rec["failed"] = failed
    _RECORD[f"{name}/{dt}"] = rec
    _dump()
    assert not failed, f"{name}/{dt}: " + "; ".join(failed)


# ------------------------------------------------------------------------------------------------- D: the three blocks
# name: variant, attention type (sd21) or None (sd3), parameter prefix, (H, W), T.  C = 512, the full models' mid-block.
BLOCK_CASES = {
    "sd21_encoder_n3060": ("sd21", "vanilla-xformers", "encoder.mid.attn_1", (60, 51), 3),
    "sd21_encoder_n5184": ("sd21", "vanilla-xformers", "encoder.mid.attn_1", (72, 72), 3),
    "sd21_decoder_st_n3060": ("sd21", "spatial-temporal-xformer", "decoder.mid.attn_1", (60, 51), 3),
    "sd21_decoder_st_n5184": ("sd21", "spatial-temporal-xformer", "decoder.mid.attn_1", (72, 72), 3),
    "sd3_n2295": ("sd3", None, "encoder.mid_block.attentions.0", (45, 51), 3),
    "sd3_n5184": ("sd3", None, "encoder.mid_block.attentions.0", (72, 72), 3),
}
BLOCK_C = 512


def _block_params(variant, attn_type, p, C, dtype):
    """The block's checkpoint entries (oracle.synth_param) in the dtype, as prepack_params receives them."""
    from oracle import cvvae_oracle as O
    shapes = {}
    if variant == "sd21":
        shapes.update({p + ".norm.weight": (C,), p + ".norm.bias": (C,)})
        for n in ("q", "k", "v", "proj_out"):
            shapes.update({f"{p}.{n}.weight": (C, C, 1, 1), f"{p}.{n}.bias": (C,)})
        if attn_type == "spatial-temporal-xformer":
            shapes.update({p + ".norm_t.weight": (C,), p + ".norm_t.bias": (C,)})
            for n in ("q_t", "k_t", "v_t", "proj_out_t"):
                shapes.update({f"{p}.{n}.weight": (C, C), f"{p}.{n}.bias": (C,)})
    else:
        shapes.update({p + ".group_norm.weight": (C,), p + ".group_norm.bias": (C,)})
        for n in ("to_q", "to_k", "to_v", "to_out.0"):
            shapes.update({f"{p}.{n}.weight": (C, C), f"{p}.{n}.bias": (C,)})
    return {k: O.synth_param(k, sh, 1234).to(dtype).to(DEV) for k, sh in shapes.items()}


class _BlockRecording(_Recording):
    """_Recording that also keeps the normalisation and temporal-attention launches with their outputs."""

    def __init__(self):
        super().__init__()
        self.other = []

    def groupnorm(self, x, gamma, beta, groups, eps, **kw):
        y = self.inner.groupnorm(x, gamma, beta, groups, eps, **kw)
        self.other.append(("groupnorm", (x, gamma, beta, groups, eps, kw), y))
        return y

    def layernorm(self, x, gamma, beta, eps):
        y = self.inner.layernorm(x, gamma, beta, eps)
        self.other.append(("layernorm", (x, gamma, beta, eps), y))
        return y

    def attn_temporal(self, q, k, v):
        y = self.inner.attn_temporal(q, k, v)
        self.other.append(("attn_temporal", (q, k, v), y))
        return y


def _run_block(variant, attn_type, p, params, x, dtype):
    from cvvae_b200.engine import Act
    ops = _BlockRecording()
    eng = Engine(NetConfig(variant=variant, z_channels=4 if variant == "sd21" else 16), params, ops, dtype)
    a = eng.attn_sd21(Act(x), p, attn_type) if variant == "sd21" else eng.attn_sd3(Act(x), p)
    torch.cuda.synchronize()
    return a, ops


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("name", list(BLOCK_CASES))
def test_attention_block16(name, dt, monkeypatch):
    """Every launch of the block replayed against its spec in fp64 on its recorded inputs; proj_out's fused statistics
    (flat plan, residual, TMA epilogue) against fp64 sums and bit for bit against the register epilogue."""
    variant, attn_type, p, (H, W), T = BLOCK_CASES[name]
    dtype, C, G = DTYPES[dt], BLOCK_C, 32
    torch.cuda.reset_peak_memory_stats()
    N = H * W
    sd16 = _block_params(variant, attn_type, p, C, dtype)
    x = _rand((1, T, H, W, C), dtype, 11, 1.5, 0.2)
    failed, rec = [], {"N": N, "T": T}
    monkeypatch.setenv("CVVAE_TMA_EPILOGUE", "1")
    from cvvae_b200.engine import prepack_params
    params = prepack_params(sd16, _Recording().inner, dtype)
    out, ops = _run_block(variant, attn_type, p, params, x, dtype)
    monkeypatch.setenv("CVVAE_TMA_EPILOGUE", "0")
    out0, ops0 = _run_block(variant, attn_type, p, params, x, dtype)
    pl0 = _plan(ops0.inner, ops0.calls[-1])                  # the plan reads the switch: query it under the same setting
    monkeypatch.setenv("CVVAE_TMA_EPILOGUE", "1")

    # per-frame GroupNorm over N positions per frame, many CTAs per frame
    kinds = [o[0] for o in ops.other]
    assert kinds == (["groupnorm", "layernorm", "attn_temporal"] if attn_type == "spatial-temporal-xformer"
                     else ["groupnorm"]), kinds
    for kind, args, y in ops.other:
        if kind == "groupnorm":
            xi, gam, bet, groups, eps, kw = args
            assert kw == dict(per_frame=True, silu=False), kw
            pix, ppb, lanes, nblocks, _ = KB.gn_geometry(tuple(xi.shape), True)
            assert pix == N and nblocks > 1, (pix, nblocks)
            eps_sum, fix, _ = KB.gn_sum_terms(tuple(xi.shape), True, groups)
            r, E, _ = KB.gn_reference(xi, gam, bet, groups, eps, True, False, eps_sum, fix)
            gt = AG.Gates(dtype).add(y, r, E)
        elif kind == "layernorm":
            xi, gam, bet, eps = args
            r, E, rec["layernorm_max_mean_over_std"] = KB.layernorm_reference(xi, gam, bet, eps)
            gt = AG.Gates(dtype).add(y, r, E)
        else:
            r, E, _ = KB.attn_temporal_reference(*args)
            gt = AG.Gates(dtype).add(y, r, E)
        rec[kind], f_k = gt.result()
        failed += [f"{kind} {f}" for f in f_k]

    # the 1x1 convolutions (flat plans) and the spatial attention
    attn = [c for c in ops.calls if c[3].get("w_per_batch")]
    convs = [c for c in ops.calls if not c[3].get("w_per_batch")]
    # q, k, proj_out (+ q_t, k_t, v_t, proj_out_t); v is the first attention GEMM
    assert len(attn) == 3 and len(convs) == (7 if attn_type == "spatial-temporal-xformer" else 3), len(ops.calls)
    with_stats = [c for c in convs if c[3].get("gn_stats") is not None]
    assert len(with_stats) == 1 and with_stats[0] is convs[-1] and convs[-1][3].get("residual") is not None
    rec["convs"] = []
    for i, (xi, w, b, kw) in enumerate(convs):
        pl = _plan(ops.inner, (xi, w, b, kw))
        assert pl["eligible"] == 1 and pl["flat"] == 1 and pl["N_cta"] == 256 and pl["NACC"] == 1, pl
        assert pl["tma_epilogue"] == 1, pl                   # 16-bit channels-last outputs: the flat TMA epilogue
        yi, res = kw["out"], kw.get("residual")
        x2, y2 = xi.reshape(-1, C).double(), yi.reshape(-1, C)
        w64, b64 = w[0].double(), b.double()
        r = x2 @ w64.T + b64
        S = x2.abs() @ w64.abs().T + b64.abs()
        if res is not None:
            r = r + res.reshape(-1, C).double()
            S = S + res.reshape(-1, C).double().abs()
        c_rec, f_c = AG.Gates(dtype, K=C).add(y2, r, AG.gemm_bound(C, S)).result()
        c_rec.update(plan=pl, residual=res is not None, stats=kw.get("gn_stats") is not None)
        rec["convs"].append(c_rec)
        failed += [f"conv {i} {f}" for f in f_c]
    assert pl0["flat"] == 1 and pl0["tma_epilogue"] == 0, pl0

    # fused statistics of the last conv (proj_out / proj_out_t / to_out.0): gate 5, and the TMA epilogue's equal the
    # register epilogue's bit for bit
    assert out.stats is not None and out.stats is with_stats[0][3]["gn_stats"]
    rec["stats_max_abs_err"], f_s = AG.stats_gate(out.t, out.stats, G)
    failed += f_s
    rec["tma_equals_register"] = AG.same_bits((out.t, out.stats), (out0.t, out0.stats))
    if not rec["tma_equals_register"]:
        failed.append("TMA and register epilogues differ (output or statistics)")
    # E: one group's sum off by one unit of the fixed-point format is seen by the bit-for-bit comparison
    bad = out.stats.clone()
    bad[0, G // 2, 0] += 1
    if AG.same_bits((out.t, bad), (out0.t, out0.stats)):
        failed.append("E: statistics off by one fixed-point unit pass the bit-for-bit comparison")

    # the spatial attention inside the block, end to end
    (wv_act, hfw, bv, _), (qv, kfw, _, kw_s), _ = attn
    yf = attn[2][3]["out"].reshape(T, N, C)
    alpha32 = torch.tensor(kw_s["alpha"], dtype=torch.float32).item()
    e2e = AG.Gates(dtype, half_ulp=False)
    for f, rows, o, E in _attention_refs(hfw, qv.reshape(T, N, C), kfw, wv_act.reshape(C, C).double(), bv.double(),
                                         alpha32, dtype):
        e2e.add(yf[f, rows], o, E)
    rec["e2e"], f_e = e2e.result()
    failed += [f"spatial attention end to end {f}" for f in f_e]

    rec["peak_bytes"] = torch.cuda.max_memory_allocated()
    if not rec["peak_bytes"] <= MAX_PEAK:
        failed.append(f"peak device memory {rec['peak_bytes'] / 2 ** 30:.2f} GB")
    rec["failed"] = failed
    _RECORD[f"block/{name}/{dt}"] = rec
    _dump()
    assert not failed, f"{name}/{dt}: " + "; ".join(failed)

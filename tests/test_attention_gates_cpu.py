"""The bounds of tests/attention_gates.py against a CPU emulation of the attention kernels' arithmetic.

The emulation does what the tensor cores and epilogues do, with every rounding correct: 16-bit operands, fp32
accumulation in K = 16 steps that each add an exact partial sum with one truncation toward zero, fma(acc, alpha, bias) in
fp32, round-to-nearest 16-bit stores and a 16-bit P.  Every gate must pass it, and every doctored output of
tests/test_gpu_attention16.py's negative controls must fail: so the bounds are sound and sharp before any GPU runs them.
Token counts 836 (19 x 44, N % 8 = 4, N % 64 = 4) and 2295 (45 x 51, odd), C = 512.
"""
import pytest
import torch

import attention_gates as AG
from cvvae_b200.engine import _round_once

F64 = torch.float64
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}


def _rand(shape, dtype, seed, scale=1.0, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(shape, generator=g, dtype=F64) * 2 - 1) * scale + offset).to(dtype).to(F64)


def _trunc32(t):
    """fp64 -> fp32 toward zero (as fp64)."""
    f = t.float()
    f = torch.where(f.double().abs() > t.abs(), torch.nextafter(f, torch.zeros_like(f)), f)
    return f.double()


def _mma_chain(a, b):
    """a [M, K] @ b[N, K]^T in fp32 accumulators: K = 16 exact partial sums, each added with one truncation."""
    acc = torch.zeros((a.shape[0], b.shape[0]), dtype=F64)
    for k0 in range(0, a.shape[1], 16):
        acc = _trunc32(acc + a[:, k0:k0 + 16] @ b[:, k0:k0 + 16].T)
    return acc


def _store(acc, alpha32, bias, dtype):
    """fma(acc, alpha, bias) in fp32, then the 16-bit store (fp32 -> 16 bit rounds once)."""
    return (acc * alpha32 + bias).float().to(dtype).to(F64)


@pytest.mark.parametrize("dt", sorted(DTYPES))
@pytest.mark.parametrize("hw,F", [((19, 44), 2), ((45, 51), 1)])
def test_emulated_attention_passes_and_doctored_fails(hw, F, dt):
    dtype = DTYPES[dt]
    N, C = hw[0] * hw[1], 512
    br = AG.branches(N)
    assert br["ld_gt_n"] or br["odd_n"]
    alpha32 = torch.tensor(C ** -0.5, dtype=torch.float32).item()
    s = 4.5 ** 0.5                                            # logits with standard deviation 1.5
    hn, q, k = _rand((F, N, C), dtype, 1, 1.7), _rand((F, N, C), dtype, 2, s), _rand((F, N, C), dtype, 3, s)
    wv = _rand((C, C), dtype, 4, C ** -0.5)
    bv = _rand((C,), torch.float32, 5, 0.2, 0.5)
    g = {"vT": AG.Gates(dtype, K=C), "S": AG.Gates(None), "P": AG.Gates(dtype), "O": AG.Gates(dtype, K=N)}
    e2e = AG.Gates(dtype, half_ulp=False)
    ys, refs = [], []
    for f in range(F):
        vT = _store(_mma_chain(wv, hn[f]), 1.0, bv[:, None], dtype)
        g["vT"].add(vT, wv @ hn[f].T + bv[:, None], AG.gemm_bound(C, wv.abs() @ hn[f].abs().T + bv.abs()[:, None]))
        S = _store(_mma_chain(q[f], k[f]), alpha32, 0.0, torch.float32)
        r = alpha32 * (q[f] @ k[f].T)
        g["S"].add(S, r, AG.logit_bound(C, alpha32, q[f].abs() @ k[f].abs().T, r))
        rp = torch.softmax(S, dim=-1)
        P = _round_once(rp, dtype).to(F64)
        g["P"].add(P, rp, AG.softmax_bound(S, rp))
        O = _store(_mma_chain(P, vT), 1.0, 0.0, dtype)
        r = P @ vT.T
        E = AG.gemm_bound(N, P @ vT.abs().T)
        g["O"].add(O, r, E)
        # negative controls of the stage gates: a store rounding toward zero; the last K block dropped
        rec, failed = AG.Gates(dtype, K=N).add(AG.truncate(r, dtype), r, E).result()
        assert any(x.startswith("2:") for x in failed) and any(x.startswith("3:") for x in failed), rec
        if br["ragged_k_block"]:
            kk = N - N % 64
            short = _round_once(P[:, :kk] @ vT[:, :kk].T, dtype).to(F64)
            rec, failed = AG.Gates(dtype, K=N).add(short, r, E).result()
            assert any(x.startswith("1:") for x in failed), rec
        # end to end against softmax(C^-1/2 q k^T) v in fp64
        v = hn[f] @ wv.T + bv
        dv = AG.stored_bound(v, AG.gemm_bound(C, hn[f].abs() @ wv.abs().T + bv.abs()), dtype)
        o, Eo = AG.attention_reference(q[f], k[f], v, dv, alpha32, dtype)
        e2e.add(O, o, Eo)
        ys.append(O)
        refs.append((o, Eo))
    for name, gt in list(g.items()) + [("e2e", e2e)]:
        rec, failed = gt.result()
        assert not failed, (name, rec)
    # end-to-end negative controls: one token shifted; two frames swapped
    o, Eo = refs[0]
    rec, failed = AG.Gates(dtype, half_ulp=False).add(torch.roll(ys[0], 1, 0), o, Eo).result()
    assert failed, rec
    if F > 1:
        rec, failed = AG.Gates(dtype, half_ulp=False).add(ys[1], o, Eo).result()
        assert failed, rec


def test_statistics_gate_and_one_unit_control():
    """Gate 5 accepts the exact fixed-point sums of a stored tensor and rejects a wrong group; one unit of the fixed-point
    format in one group is inside its tolerance, and the bit-for-bit comparison with the register epilogue sees it."""
    y = _rand((2, 3, 10, 12, 512), torch.bfloat16, 6, 1.5, 0.2)
    v = y.reshape(2, -1, 32, 16)
    st = torch.stack([torch.round(v.sum(dim=(1, 3)) * AG.GN_SUM_SCALE),
                      torch.round((v * v).sum(dim=(1, 3)) * AG.GN_SQ_SCALE)], dim=-1).to(torch.int64)
    assert not AG.stats_gate(y, st, 32)[1] and AG.same_bits((y, st), (y.clone(), st.clone()))
    off = st.clone()
    off[1, 16, 0] += 1
    assert not AG.stats_gate(y, off, 32)[1]
    assert not AG.same_bits((y, off), (y, st))
    wrong = st.clone()
    wrong[0, 3, 0] += int(AG.GN_SUM_SCALE)          # one group's sum off by 1.0
    assert AG.stats_gate(y, wrong, 32)[1]

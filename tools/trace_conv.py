#!/usr/bin/env python
"""Per-CTA phase timing of conv_tc_kernel (uses cvvae_conv_tc_set_trace).  Prints medians in microseconds.

    python tools/trace_conv.py [--only substring]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_conv import P  # noqa: E402
from cvvae_b200._lib import PAD_ZERO  # noqa: E402
from cvvae_b200.ops import CudaOps  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="")
    ap.add_argument("--n", type=int, default=8192)
    args = ap.parse_args()
    ops = CudaOps()
    dt = torch.float16
    for name, ci, co, k, s, (T, H, W), pads, pad_t, up in P:
        if args.only and args.only not in name:
            continue
        (tl, th), (hl, hh), (wl, wh) = pads
        To = (T + tl + th - k[0]) // s[0] + 1
        Ho = (H + hl + hh - k[1]) // s[1] + 1
        Wo = (W + wl + wh - k[2]) // s[2] + 1
        x = (torch.rand((1, T, H, W, ci), device="cuda") - 0.5).to(dt)
        w = ((torch.rand((k[0] * k[1] * k[2], co, ci), device="cuda") - 0.5) * 0.05).to(dt)
        b = torch.zeros(co, device="cuda")
        if up == 2:
            y = torch.empty((1, 2 * To - 1, Ho, Wo, co // 2), dtype=dt, device="cuda")
        elif co < 16:
            y = torch.empty((1, co, To, Ho, Wo), dtype=dt, device="cuda").permute(0, 2, 3, 4, 1)
        else:
            y = torch.empty((1, To, Ho, Wo, co), dtype=dt, device="cuda")
        kw = dict(kernel=k, stride=s, offset=(-tl, -hl, -wl), pad_t=pad_t, pad_hw=PAD_ZERO, up_time=up, out=y, force="tc")
        ops.conv(x, w, b, **kw)
        torch.cuda.synchronize()
        buf = torch.zeros((args.n, 8), dtype=torch.int64, device="cuda")
        ops.lib.cvvae_conv_tc_set_trace(buf.data_ptr(), args.n)
        s_ev, e_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s_ev.record()
        ops.conv(x, w, b, **kw)
        e_ev.record()
        torch.cuda.synchronize()
        ops.lib.cvvae_conv_tc_set_trace(None, 0)
        t = buf.cpu().numpy().astype(np.uint64)
        t = t[t[:, 0] > 0]
        if len(t) == 0:  # persistent kernel: no per-CTA stamps
            print(json.dumps({"layer": name, "kernel_ms": round(s_ev.elapsed_time(e_ev), 3), "ctas_traced": 0}), flush=True)
            continue
        smid = (t[:, 7] >> np.uint64(48)).astype(np.int64)
        t7 = (t[:, 7] & np.uint64(0xFFFFFFFFFFFF)).astype(np.int64)
        tt = t.astype(np.int64)
        tt[:, 7] = (tt[:, 0] & ~np.int64(0xFFFFFFFFFFFF)) | t7
        def d(a, b_):
            # phase stamps may be missing (untraced CTAs): use the rows that have both
            rows = tt[(t[:, a] > 0) & (t[:, b_] > 0)]
            return float(np.median(rows[:, b_] - rows[:, a])) / 1e3 if len(rows) else None
        # idle gap between consecutive CTAs on the same SM
        gaps = []
        for sm in np.unique(smid):
            rows = tt[smid == sm]
            rows = rows[np.argsort(rows[:, 0])]
            if len(rows) > 1:
                gaps.extend((rows[1:, 0] - rows[:-1, 7]).tolist())
        print(json.dumps({"layer": name, "kernel_ms": round(s_ev.elapsed_time(e_ev), 3), "ctas_traced": int(len(tt)),
                          "us_setup": d(0, 1), "us_first_A": d(1, 2), "us_first_B_after_A": d(2, 3), "us_mainloop_issue": d(3, 4),
                          "us_acc_ready_after_issue": d(4, 5), "us_epilogue": d(5, 6), "us_exit": d(6, 7), "us_total": d(0, 7),
                          "us_gap_between_ctas_same_sm": float(np.median(gaps)) / 1e3 if gaps else None}), flush=True)


if __name__ == "__main__":
    main()

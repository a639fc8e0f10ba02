#!/usr/bin/env python
"""Per-layer microbenchmark of the tensor-core convolution on the distinct conv problems of one
17x576x576 tile (SURVEY.md section 3.6).  Prints one JSON line per problem: ms, TFLOP/s, fraction of the peak bench.py
uses (MEASURED_PEAKS.json when present, else the H100 SXM data-sheet 989 TFLOP/s); with --dtype fp32 (TF32 products) the
H100 SXM data-sheet dense TF32 figure, 495 TFLOP/s, labelled as such.  L2 is flushed between timed
launches (256 MB memset) and each timing is the median of `reps`.

    python tools/bench_conv.py [--reps 5] [--only substring] [--dtype fp16|bf16|fp32]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402  (the same peak source as the benchmark)
from cvvae_b200._lib import PAD_REPLICATE, PAD_ZERO  # noqa: E402
from cvvae_b200.ops import CudaOps  # noqa: E402

# name, Cin, Cout, kernel, stride, in T,H,W, pads, pad_t, up_time
P = [
    ("E 128->128 333 @17x576", 128, 128, (3, 3, 3), (1, 1, 1), (17, 576, 576), ((2, 0), (1, 1), (1, 1)), PAD_REPLICATE, 1),
    ("E 128->128 133 @17x576", 128, 128, (1, 3, 3), (1, 1, 1), (17, 576, 576), ((0, 0), (1, 1), (1, 1)), PAD_ZERO, 1),
    ("E 128->128 333 s222", 128, 128, (3, 3, 3), (2, 2, 2), (17, 576, 576), ((2, 0), (0, 1), (0, 1)), PAD_REPLICATE, 1),
    ("E 128->256 333 @9x288", 128, 256, (3, 3, 3), (1, 1, 1), (9, 288, 288), ((2, 0), (1, 1), (1, 1)), PAD_REPLICATE, 1),
    ("E 256->256 333 @9x288", 256, 256, (3, 3, 3), (1, 1, 1), (9, 288, 288), ((2, 0), (1, 1), (1, 1)), PAD_REPLICATE, 1),
    ("E 256->256 133 @9x288", 256, 256, (1, 3, 3), (1, 1, 1), (9, 288, 288), ((0, 0), (1, 1), (1, 1)), PAD_ZERO, 1),
    ("E 128->256 111 @9x288", 128, 256, (1, 1, 1), (1, 1, 1), (9, 288, 288), ((0, 0), (0, 0), (0, 0)), PAD_ZERO, 1),
    ("E 256->512 333 @9x144", 256, 512, (3, 3, 3), (1, 1, 1), (9, 144, 144), ((2, 0), (1, 1), (1, 1)), PAD_REPLICATE, 1),
    ("E 512->512 333 @9x144", 512, 512, (3, 3, 3), (1, 1, 1), (9, 144, 144), ((2, 0), (1, 1), (1, 1)), PAD_REPLICATE, 1),
    ("E 512->512 333 @5x72", 512, 512, (3, 3, 3), (1, 1, 1), (5, 72, 72), ((2, 0), (1, 1), (1, 1)), PAD_REPLICATE, 1),
    ("E 512->512 133 @5x72", 512, 512, (1, 3, 3), (1, 1, 1), (5, 72, 72), ((0, 0), (1, 1), (1, 1)), PAD_ZERO, 1),
    ("E 512->8 333 @5x72", 512, 8, (3, 3, 3), (1, 1, 1), (5, 72, 72), ((2, 0), (1, 1), (1, 1)), PAD_REPLICATE, 1),
    ("D 512->1024 333 up @5x144", 512, 1024, (3, 3, 3), (1, 1, 1), (5, 144, 144), ((1, 1), (1, 1), (1, 1)), PAD_REPLICATE, 2),
    ("D 512->512 333 @9x144", 512, 512, (3, 3, 3), (1, 1, 1), (9, 144, 144), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1),
    ("D 512->512 333 @9x288", 512, 512, (3, 3, 3), (1, 1, 1), (9, 288, 288), ((1, 1), (1, 1), (1, 1)), PAD_REPLICATE, 1),
    ("D 512->256 333 @9x288", 512, 256, (3, 3, 3), (1, 1, 1), (9, 288, 288), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1),
    ("D 256->512 333 up @9x576", 256, 512, (3, 3, 3), (1, 1, 1), (9, 576, 576), ((1, 1), (1, 1), (1, 1)), PAD_REPLICATE, 2),
    ("D 256->128 333 @17x576", 256, 128, (3, 3, 3), (1, 1, 1), (17, 576, 576), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1),
    ("D 128->128 333 @17x576", 128, 128, (3, 3, 3), (1, 1, 1), (17, 576, 576), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1),
    ("D 128->3 333 @17x576", 128, 3, (3, 3, 3), (1, 1, 1), (17, 576, 576), ((1, 1), (1, 1), (1, 1)), PAD_ZERO, 1),
]


DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": torch.float32}
TF32_PEAK_DATASHEET = 495.0   # TFLOP/s: H100 SXM data sheet, dense TF32 tensor-core rate


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default="")
    ap.add_argument("--dtype", choices=sorted(DTYPES), default="fp16")
    args = ap.parse_args()
    dt = DTYPES[args.dtype]
    if dt == torch.float32:
        peak, peak_src = TF32_PEAK_DATASHEET, "H100 SXM data sheet, dense TF32"
    else:
        peak, peak_src = bench.peaks()[0], "bench.peaks()"
    ops = CudaOps()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
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
        times = []
        for _ in range(args.reps):
            flush.zero_()
            s_ev, e_ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s_ev.record()
            ops.conv(x, w, b, **kw)
            e_ev.record()
            torch.cuda.synchronize()
            times.append(s_ev.elapsed_time(e_ev))
        times.sort()
        ms = times[len(times) // 2]
        flops = 2.0 * To * Ho * Wo * co * k[0] * k[1] * k[2] * ci
        tf = flops / (ms * 1e-3) / 1e12
        print(json.dumps({"layer": name, "ms": round(ms, 3), "tflops": round(tf, 1), "frac_of_peak": round(tf / peak, 3),
                          "gflop": round(flops / 1e9, 1), "dtype": args.dtype, "peak_source": peak_src}), flush=True)
        del x, w, y


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""What scoring costs: the frame-metrics and MS-SSIM kernels on their own, and evaluate_frames against reconstruct_frames.

    python tools/bench_metrics.py [--launches 200] [--frames 129] [--reps 3] [--skip-stream]

  kernel   cvvae_frame_metrics on two resident uint8 clips of 17 frames (one decoder chunk) at 576x1024 and 720x1280:
           CUDA events around `--launches` back-to-back launches after 20 untimed ones; time per frame, and the achieved
           bytes/s against the 2 * 3 * H * W bytes per frame the algorithm has to read (one read of each frame).
  ms_ssim  cvvae_frame_ms_ssim (4 pooling steps and 5 scoring launches) on the same clips, timed the same way and
           reported against the same 2 * 3 * H * W bytes per frame.
  stream   evaluate_frames (with and without ms_ssim=True) against reconstruct_frames over one seeded host clip of `--frames` frames at 576x1024 in
           16-frame items, SD2.1 model at full width (seeded random weights, as bench.py), fp16, default tiling.  Each arm
           runs once untimed, then `--reps` times alternating with the others; a time is a host clock around the call that
           ends in a device synchronise; the line reports the median and the spread (min, max).

The card's name, power limit and SM clock are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNEL_SHAPES = ((17, 576, 1024), (17, 720, 1280))
H, W, ITEM = 576, 1024, 16


def _clip_pair(torch, T: int, h: int, w: int):
    g = torch.Generator(device="cuda").manual_seed(h)
    a = torch.randint(0, 256, (T, h, w, 3), generator=g, dtype=torch.uint8, device="cuda")
    b = (a.int() + torch.randint(-3, 4, a.shape, generator=g, device="cuda")).clamp_(0, 255).to(torch.uint8)
    return a, b


def _us_per_frame(torch, launch, a, b, launches: int) -> float:
    for _ in range(20):
        launch(a, b)
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        launch(a, b)
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) * 1e3 / launches / a.shape[0]


def bench_kernel(torch, launches: int) -> list:
    from cvvae_b200 import frame_metrics
    from cvvae_b200.metrics import _launch
    rows = []
    for T, h, w in KERNEL_SHAPES:
        a, b = _clip_pair(torch, T, h, w)
        us_frame = _us_per_frame(torch, _launch, a, b, launches)
        m = frame_metrics(a, b)
        rows.append({"shape": f"{T}x{h}x{w}x3", "launches": launches, "us_per_frame": round(us_frame, 2),
                     "algorithmic_bytes_per_frame": 2 * 3 * h * w,
                     "achieved_GB_per_s": round(2 * 3 * h * w / us_frame / 1e3, 1),
                     "psnr_frame0": round(m.psnr[0].item(), 3), "ssim_frame0": round(m.ssim[0].item(), 6)})
    return rows


def bench_ms_ssim_kernel(torch, launches: int) -> list:
    from cvvae_b200 import frame_ms_ssim
    from cvvae_b200.metrics import MS_SSIM_LAUNCHES, _launch_ms_ssim
    rows = []
    for T, h, w in KERNEL_SHAPES:
        a, b = _clip_pair(torch, T, h, w)
        us_frame = _us_per_frame(torch, _launch_ms_ssim, a, b, launches)
        rows.append({"shape": f"{T}x{h}x{w}x3", "calls": launches, "kernel_launches_per_call": MS_SSIM_LAUNCHES,
                     "us_per_frame": round(us_frame, 2), "algorithmic_bytes_per_frame": 2 * 3 * h * w,
                     "achieved_GB_per_s": round(2 * 3 * h * w / us_frame / 1e3, 1),
                     "ms_ssim_frame0": round(frame_ms_ssim(a[:1], b[:1])[0].item(), 6)})
    return rows


def bench_stream(torch, frames: int, reps: int) -> dict:
    from bench import CONFIGS, build_model
    from cvvae_b200 import evaluate_frames, reconstruct_frames
    m = build_model(CONFIGS["c2"], torch.float16)
    clip = torch.randint(0, 256, (frames, H, W, 3), generator=torch.Generator().manual_seed(frames), dtype=torch.uint8)
    arms = {"reconstruct_frames": reconstruct_frames, "evaluate_frames": evaluate_frames,
            "evaluate_frames_ms_ssim": lambda model, items: evaluate_frames(model, items, ms_ssim=True)}

    def run(fn) -> float:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in fn(m, (clip[a:a + ITEM] for a in range(0, frames, ITEM))):
            pass
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for fn in arms.values():
        run(fn)
    times = {name: [] for name in arms}
    for _ in range(reps):
        for name, fn in arms.items():
            times[name].append(run(fn))
    out = {"shape": f"{frames}x{H}x{W}x3", "reps": reps, "model": "sd21 full width, fp16, seeded random weights, default tiling"}
    for name, ts in times.items():
        fps = sorted(frames / s for s in ts)
        out[name] = {"frames_per_s": round(fps[len(fps) // 2], 2), "frames_per_s_spread": [round(fps[0], 2), round(fps[-1], 2)]}
    return out


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--launches", type=int, default=200, help="timed kernel launches per shape (after 20 untimed)")
    ap.add_argument("--frames", type=int, default=129, help="clip length of the stream comparison")
    ap.add_argument("--reps", type=int, default=3, help="timed runs per arm of the stream comparison")
    ap.add_argument("--skip-stream", action="store_true", help="kernel timing only")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        print("bench_metrics.py needs a GPU: no CUDA device is available", file=sys.stderr)
        return 2
    import __graft_entry__ as ge
    from tools.bench_stream import card
    ge.build()
    result = {"card": card(), "kernel": bench_kernel(torch, args.launches),
              "ms_ssim_kernel": bench_ms_ssim_kernel(torch, args.launches)}
    print(json.dumps(result), flush=True)
    if not args.skip_stream:
        stream = bench_stream(torch, args.frames, args.reps)
        stream["card_after_runs"] = card()
        print(json.dumps({"stream": stream}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())

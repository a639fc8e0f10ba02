#!/usr/bin/env python
"""What error maps cost: the SSIM map against the PSNR / SSIM kernel, LPIPS.map against the scalar LPIPS, and
evaluate_frames with and without maps.

    python tools/bench_error_maps.py [--launches 200] [--reps 10] [--frames 129] [--stream-reps 3] [--skip-stream]

  kernel   cvvae_frame_metrics against cvvae_frame_ssim_map on two resident uint8 clips of 17 frames (one decoder chunk)
           at 576x1024 and 720x1280: CUDA events around `--launches` back-to-back launches after 20 untimed ones, the
           two arms alternated three times; the median time per frame.
  lpips    LPIPS scalar (``metric(a, b)`` without the host copy) against ``metric.map(a, b)`` on 4 resident frame pairs
           at 576x1024, for VGG16 and AlexNet (seeded random weights, as tools/bench_lpips.py): CUDA events around each
           call after 3 untimed ones, arms alternated for `--reps` rounds; the median time per frame pair.
  stream   evaluate_frames over one seeded host clip of `--frames` frames at 576x1024 in 16-frame items, SD2.1 model at
           full width (seeded random weights, as bench.py), fp16, default tiling, in three arms: without maps, with
           maps, and with maps plus AlexNet LPIPS.  Each arm runs once untimed, then `--stream-reps` times alternating
           with the others; a time is a host clock around the call that ends in a device synchronise; the line reports
           the median and the spread (min, max).

The card's name, power limit and SM clock are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

KERNEL_SHAPES = ((17, 576, 1024), (17, 720, 1280))
H, W, ITEM, PAIRS = 576, 1024, 16, 4


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
    from cvvae_b200.metrics import _launch
    arms = {"frame_metrics": lambda a, b: _launch(a, b), "ssim_map": lambda a, b: _launch(a, b, maps=True)}
    rows = []
    for T, h, w in KERNEL_SHAPES:
        a, b = _clip_pair(torch, T, h, w)
        times = {name: [] for name in arms}
        for _ in range(3):
            for name, fn in arms.items():
                times[name].append(_us_per_frame(torch, fn, a, b, launches))
        row = {"shape": f"{T}x{h}x{w}x3", "launches": launches, "rounds": 3}
        for name, ts in times.items():
            row[f"{name}_us_per_frame"] = round(statistics.median(ts), 2)
            row[f"{name}_spread"] = [round(min(ts), 2), round(max(ts), 2)]
        row["map_bytes_per_frame"] = 4 * 3 * (h - 10) * (w - 10)
        rows.append(row)
    return rows


def bench_lpips(torch, reps: int) -> list:
    import lpips_alex_ref as A
    import lpips_ref as R
    from cvvae_b200 import LPIPS
    a, b = _clip_pair(torch, PAIRS, H, W)
    rows = []
    for net, ref in (("vgg", R), ("alex", A)):
        metric = LPIPS.from_state_dict(ref.make_state_dict(0), net=net)
        arms = {"scalar": lambda: metric._launch(a, b), "map": lambda: metric._launch(a, b, maps=True)}
        for fn in arms.values():
            for _ in range(3):
                fn()
        times = {name: [] for name in arms}
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(reps):
            for name, fn in arms.items():
                start.record()
                fn()
                stop.record()
                stop.synchronize()
                times[name].append(start.elapsed_time(stop) / PAIRS)
        row = {"net": net, "shape": f"{PAIRS}x{H}x{W}x3", "reps": reps,
               "launches_per_group": {"scalar": metric.launches, "map": metric.launches + 1}}
        for name, ts in times.items():
            row[f"{name}_ms_per_pair"] = round(statistics.median(ts), 3)
            row[f"{name}_spread"] = [round(min(ts), 3), round(max(ts), 3)]
        rows.append(row)
    return rows


def bench_stream(torch, frames: int, reps: int) -> dict:
    import lpips_alex_ref as A
    from bench import CONFIGS, build_model
    from cvvae_b200 import LPIPS, evaluate_frames
    m = build_model(CONFIGS["c2"], torch.float16)
    alex = LPIPS.from_state_dict(A.make_state_dict(0), net="alex")
    clip = torch.randint(0, 256, (frames, H, W, 3), generator=torch.Generator().manual_seed(frames), dtype=torch.uint8)
    arms = {"evaluate_frames": {}, "evaluate_frames_maps": {"maps": True},
            "evaluate_frames_maps_lpips_alex": {"maps": True, "lpips": alex}}

    def run(kw) -> float:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in evaluate_frames(m, (clip[a:a + ITEM] for a in range(0, frames, ITEM)), **kw):
            pass
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for kw in arms.values():
        run(kw)
    times = {name: [] for name in arms}
    for _ in range(reps):
        for name, kw in arms.items():
            times[name].append(run(kw))
    out = {"shape": f"{frames}x{H}x{W}x3", "reps": reps, "model": "sd21 full width, fp16, seeded random weights, default tiling",
           "download_bytes_per_frame": {"frame": 3 * H * W, "ssim_map": 4 * 3 * (H - 10) * (W - 10), "lpips_map": 4 * H * W}}
    for name, ts in times.items():
        fps = sorted(frames / s for s in ts)
        out[name] = {"frames_per_s": round(fps[len(fps) // 2], 2), "frames_per_s_spread": [round(fps[0], 2), round(fps[-1], 2)],
                     "ms_per_frame": round(1e3 / fps[len(fps) // 2], 2)}
    return out


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--launches", type=int, default=200, help="timed kernel launches per shape and round (after 20 untimed)")
    ap.add_argument("--reps", type=int, default=10, help="timed rounds of the LPIPS comparison (after 3 untimed calls)")
    ap.add_argument("--frames", type=int, default=129, help="clip length of the stream comparison")
    ap.add_argument("--stream-reps", type=int, default=3, help="timed runs per arm of the stream comparison")
    ap.add_argument("--skip-stream", action="store_true", help="kernel and LPIPS timing only")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        print("bench_error_maps.py needs a GPU: no CUDA device is available", file=sys.stderr)
        return 2
    import __graft_entry__ as ge
    from tools.bench_stream import card
    ge.build()
    print(json.dumps({"card": card(), "kernel": bench_kernel(torch, args.launches), "lpips": bench_lpips(torch, args.reps)}),
          flush=True)
    if not args.skip_stream:
        stream = bench_stream(torch, args.frames, args.stream_reps)
        stream["card_after_runs"] = card()
        print(json.dumps({"stream": stream}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())

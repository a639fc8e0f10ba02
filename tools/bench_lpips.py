#!/usr/bin/env python
"""What LPIPS costs: the metric's kernels on resident frames, PyTorch's own fp32 evaluation, and evaluate_frames with it.

    python tools/bench_lpips.py [--reps 20] [--frames 129] [--stream-reps 3] [--skip-stream]

  kernels  LPIPS.__call__'s device work (metrics.LPIPS._launch) on 4 resident frame pairs at 576x1024 and 720x1280,
           seeded weights in the real layout (tests/lpips_ref.py): CUDA events around every launch of `--reps` calls
           after 3 untimed ones, summed per part (input kernel, the 13 convolutions, the 5 tap kernels); us per frame
           pair, and the convolutions' executed TF32 rate.  Executed MACs per image pixel: conv1_1 as its 32-channel
           1 x 1 (64 x 32) plus, for the other twelve, Cin x Cout x 9 at their resolution; the algorithmic count is the
           same with conv1_1 at 27 input channels (305,856 MAC per pixel).  Both are computed from the shapes below.
  torch    the same metric restated in PyTorch (tests/lpips_ref.py, fp32, default flags: cuDNN with TF32), alternated
           call by call with ours in the same process; median us per frame pair.
  stream   evaluate_frames over one seeded host clip of `--frames` frames at 576x1024 in 16-frame items, SD2.1 model at
           full width (seeded weights, as bench.py), fp16, default tiling, without and with lpips=, alternated, each
           arm once untimed and `--stream-reps` times timed (host clock around the call, ending in a synchronise).

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

SHAPES = ((576, 1024), (720, 1280))
PAIRS = 4
CONVS = [(3, 64, 0), (64, 64, 0), (64, 128, 1), (128, 128, 1), (128, 256, 2), (256, 256, 2), (256, 256, 2),
         (256, 512, 3), (512, 512, 3), (512, 512, 3), (512, 512, 4), (512, 512, 4), (512, 512, 4)]   # Cin, Cout, level


def macs_per_pixel(executed: bool) -> float:
    """MACs per image pixel of the thirteen convolutions (a level-j layer runs on 4^-j of the pixels)."""
    first = 64 * 32 if executed else 64 * 27
    return first + sum(ci * co * 9 / 4 ** j for ci, co, j in CONVS[1:])


def bench_kernels(torch, metric, sd, reps: int) -> list:
    import lpips_ref as R
    from cvvae_b200 import _lib as L
    rows = []
    for H, W in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(H)
        a = torch.randint(0, 256, (PAIRS, H, W, 3), generator=g, dtype=torch.uint8, device="cuda")
        b = (a.int() + torch.randint(-3, 4, a.shape, generator=g, device="cuda")).clamp_(0, 255).to(torch.uint8)
        assert metric._group(H, W) >= PAIRS
        lib = L.load()
        events = {"input": [], "conv": [], "tap": []}
        fns = {"cvvae_lpips_input": "input", "cvvae_conv3d": "conv", "cvvae_lpips_tap": "tap"}
        real = {name: getattr(lib, name) for name in fns}

        def timed(name):
            fn = real[name]

            def call(*args):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                rc = fn(*args)
                e.record()
                events[fns[name]].append((s, e))
                return rc
            call.__name__ = name
            return call

        sd32 = {k: v.cuda() for k, v in sd.items()}
        with torch.no_grad():
            for _ in range(3):
                metric._launch(a, b)
                R.lpips(a, b, sd32, torch.float32)
            torch_us = []
            for name in fns:
                setattr(lib, name, timed(name))
            try:
                for _ in range(reps):
                    metric._launch(a, b)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    R.lpips(a, b, sd32, torch.float32)
                    torch.cuda.synchronize()
                    torch_us.append((time.perf_counter() - t0) * 1e6 / PAIRS)
            finally:
                for name in fns:
                    setattr(lib, name, real[name])
        torch.cuda.synchronize()
        us = {k: sum(s.elapsed_time(e) for s, e in v) * 1e3 / reps / PAIRS for k, v in events.items()}
        assert len(events["conv"]) == 13 * reps and len(events["tap"]) == 5 * reps
        flops_pair = 2 * 2 * H * W                     # two images, 2 FLOP per MAC
        total = sum(us.values())
        ours = metric(a, b)
        rows.append({
            "shape": f"{PAIRS} frame pairs x {H}x{W}", "reps": reps,
            "us_per_frame_pair": round(total, 1), "split_us": {k: round(v, 1) for k, v in us.items()},
            "conv_executed_TFLOP_per_pair": round(flops_pair * macs_per_pixel(True) / 1e12, 4),
            "conv_algorithmic_TFLOP_per_pair": round(flops_pair * macs_per_pixel(False) / 1e12, 4),
            "conv_executed_TFLOP_per_s": round(flops_pair * macs_per_pixel(True) / us["conv"] / 1e6, 1),
            "torch_fp32_default_us_per_frame_pair": round(statistics.median(torch_us), 1),
            "lpips_frame0": round(ours[0].item(), 6),
        })
    return rows


def bench_stream(torch, metric, frames: int, reps: int) -> dict:
    from bench import CONFIGS, build_model
    from cvvae_b200 import evaluate_frames
    m = build_model(CONFIGS["c2"], torch.float16)
    H, W, ITEM = 576, 1024, 16
    clip = torch.randint(0, 256, (frames, H, W, 3), generator=torch.Generator().manual_seed(frames), dtype=torch.uint8)
    arms = {"evaluate_frames": {}, "evaluate_frames_lpips": {"lpips": metric}}

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
    out = {"shape": f"{frames}x{H}x{W}x3", "reps": reps, "model": "sd21 full width, fp16, seeded random weights, default tiling"}
    for name, ts in times.items():
        fps = sorted(frames / s for s in ts)
        out[name] = {"frames_per_s": round(fps[len(fps) // 2], 2), "frames_per_s_spread": [round(fps[0], 2), round(fps[-1], 2)],
                     "ms_per_frame": round(1e3 / fps[len(fps) // 2], 2)}
    return out


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=20, help="timed calls per shape (after 3 untimed)")
    ap.add_argument("--frames", type=int, default=129, help="clip length of the stream comparison")
    ap.add_argument("--stream-reps", type=int, default=3, help="timed runs per arm of the stream comparison")
    ap.add_argument("--skip-stream", action="store_true", help="kernel timing only")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        print("bench_lpips.py needs a GPU: no CUDA device is available", file=sys.stderr)
        return 2
    import __graft_entry__ as ge
    import lpips_ref as R
    from tools.bench_stream import card
    ge.build()
    from cvvae_b200 import LPIPS
    sd = R.make_state_dict(0)
    metric = LPIPS.from_state_dict(sd)
    print(json.dumps({"card": card(), "kernels": bench_kernels(torch, metric, sd, args.reps)}), flush=True)
    if not args.skip_stream:
        stream = bench_stream(torch, metric, args.frames, args.stream_reps)
        stream["card_after_runs"] = card()
        print(json.dumps({"stream": stream}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())

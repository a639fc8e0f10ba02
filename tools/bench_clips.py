#!/usr/bin/env python
"""What turning clips into latents costs: the training pre-processing kernel on its own, encode_clips at several batch
sizes, and the route a user has without it.

    python tools/bench_clips.py [--launches 200] [--clips 32] [--baseline-clips 8] [--reps 3]

  kernel     cvvae_video_train_input on one resident 17 x 720 x 1280 uint8 clip -> 17 x 256 x 256 ("cover": resize to
             256 x 455, centre crop), fp16: CUDA events around `--launches` back-to-back launches after 20 untimed ones.
  encode     encode_clips over `--clips` seeded host clips of 17 x 720 x 1280 (8 distinct clips, cycled), size 256 x 256,
             SD2.1 model at full width (seeded random weights, as bench.py), fp16, default tiling and chunking, at
             batch_size 1 / 8 / 32, eager and with CUDA graphs (a second model with the same weights, whose graphs stay
             captured from the untimed run on).
  baseline   today's route on the first `--baseline-clips` of the same clips: torchvision's CPU float transform per clip
             (float32, resize, centre crop, (x / 255 - 0.5) * 2), cast to fp16, host -> device, model.encode at B = 1, moments
             back to the host.

Every arm runs once untimed, then `--reps` times, the arms alternating; a time is a host clock around the whole run,
ending in a device synchronise.  Each line reports clips/s as the median and spread (min, max), and the arm's peak
device memory above what was allocated before it (torch.cuda.max_memory_allocated).  The card's name, power limit and
SM clock are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T, SRC_H, SRC_W, SIZE = 17, 720, 1280, (256, 256)


def bench_kernel(torch, launches: int) -> dict:
    from cvvae_b200.video_io import frames_to_training_input, training_geometry
    clip = torch.randint(0, 256, (T, SRC_H, SRC_W, 3), generator=torch.Generator(device="cuda").manual_seed(0),
                         dtype=torch.uint8, device="cuda")
    out = torch.empty((1, 3, T, *SIZE), dtype=torch.float16, device="cuda")
    for _ in range(20):
        frames_to_training_input(clip, SIZE, "cover", torch.float16, out=out)
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        frames_to_training_input(clip, SIZE, "cover", torch.float16, out=out)
    stop.record()
    stop.synchronize()
    us = start.elapsed_time(stop) * 1e3 / launches
    RH, RW, top, left = training_geometry(SRC_H, SRC_W, SIZE, "cover")
    return {"arm": "kernel", "shape": f"{T}x{SRC_H}x{SRC_W}x3 -> {T}x{SIZE[0]}x{SIZE[1]} (resize {RH}x{RW}, crop at "
            f"{top},{left}), fp16", "launches": launches, "us_per_clip": round(us, 1), "us_per_frame": round(us / T, 2)}


def torchvision_route(torch, m, clips):
    import torchvision.transforms.functional as F
    from torchvision.transforms import InterpolationMode
    out = []
    for c in clips:
        x = torch.from_numpy(c).permute(0, 3, 1, 2).float()
        f = max(SIZE[0] / SRC_H, SIZE[1] / SRC_W)
        x = F.resize(x, [round(SRC_H * f), round(SRC_W * f)], InterpolationMode.BILINEAR, antialias=True)
        x = (F.center_crop(x, list(SIZE)) / 255 - 0.5) * 2
        x = x.permute(1, 0, 2, 3).unsqueeze(0).half().cuda()
        out.append(m.encode(x).latent_dist.parameters[0].cpu())
    return out


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--launches", type=int, default=200, help="timed kernel launches (after 20 untimed)")
    ap.add_argument("--clips", type=int, default=32, help="clips per encode_clips run")
    ap.add_argument("--baseline-clips", type=int, default=8, help="clips per run of today's route")
    ap.add_argument("--reps", type=int, default=3, help="timed runs per arm")
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        print("bench_clips.py needs a GPU: no CUDA device is available", file=sys.stderr)
        return 2
    import __graft_entry__ as ge
    from bench import CONFIGS, build_model
    from cvvae_b200 import encode_clips
    from tools.bench_stream import card
    ge.build()
    print(json.dumps({"card": card(), **bench_kernel(torch, args.launches)}), flush=True)

    m = build_model(CONFIGS["c5"], torch.float16)
    mg = build_model(CONFIGS["c5"], torch.float16).enable_cuda_graphs(True)   # its own model: disabling graphs drops them
    g = np.random.default_rng(1)
    distinct = [g.integers(0, 256, (T, SRC_H, SRC_W, 3), dtype=np.uint8) for _ in range(8)]
    clips = [distinct[i % len(distinct)] for i in range(args.clips)]
    base_clips = clips[:args.baseline_clips]

    def encode_arm(bs, graphs):
        return lambda: sum(1 for _ in encode_clips(mg if graphs else m, clips, SIZE, "cover", batch_size=bs))

    arms = {f"encode_clips bs={bs} {'graphs' if gr else 'eager'}": encode_arm(bs, gr) for bs in (1, 8, 32) for gr in (False, True)}
    arms["torchvision CPU transform + encode B=1"] = lambda: len(torchvision_route(torch, m, base_clips))

    # the two routes compute the same moments up to the fp32 rounding order of the transform: their distance is reported
    a = list(encode_clips(m, base_clips[:2], SIZE, batch_size=2))
    b = torchvision_route(torch, m, base_clips[:2])
    max_diff = max((x.float() - y.float()).abs().max().item() for x, y in zip(a, b))

    def timed(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        before = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        n = fn()
        torch.cuda.synchronize()
        return n / (time.perf_counter() - t0), torch.cuda.max_memory_allocated() - before

    for fn in arms.values():
        timed(fn)
    rates = {name: [] for name in arms}
    peaks = {name: 0 for name in arms}
    for _ in range(args.reps):
        for name, fn in arms.items():
            r, p = timed(fn)
            rates[name].append(r)
            peaks[name] = max(peaks[name], p)
    model = "sd21 full width, fp16, seeded random weights, default tiling and chunking"
    for name, rs in rates.items():
        rs = sorted(rs)
        print(json.dumps({"arm": name, "model": model, "clips": args.baseline_clips if name.startswith("torchvision") else args.clips,
                          "clip": f"{T}x{SRC_H}x{SRC_W}x3 -> {SIZE[0]}x{SIZE[1]}", "reps": args.reps,
                          "clips_per_s": round(rs[len(rs) // 2], 2), "clips_per_s_spread": [round(rs[0], 2), round(rs[-1], 2)],
                          "peak_device_MiB": round(peaks[name] / 2 ** 20, 1)}), flush=True)
    print(json.dumps({"moments_max_abs_diff_vs_torchvision_route": max_diff, "card_after_runs": card()}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())

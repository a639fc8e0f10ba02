#!/usr/bin/env python
"""What turning clip latents back into uint8 videos costs: the batched pixel conversion on its own, decode_clips at
several batch sizes, and the route a user has without it.

    python tools/bench_decode_clips.py [--launches 200] [--clips 32] [--baseline-clips 8] [--reps 3]

  kernel     cvvae_video_output_u8 (video_io.batch_to_frames) on one resident fp16 [1, 3, 17, 576, 1024] batch: CUDA events
             around `--launches` back-to-back launches after 20 untimed ones; bytes per second against 2 * 3 * N bytes read
             and 3 * N bytes written (N = pixels).
  decode     decode_clips over `--clips` seeded host latents [4, 5, 32, 32] (17 x 256 x 256 out), SD2.1 model at full width
             (seeded random weights, as bench.py), fp16, default tiling and chunking, at batch_size 1 / 8 / 32 eager, and
             at 1 / 8 with CUDA graphs (a second model with the same weights, whose graphs stay captured from the untimed
             run on).  A graph keeps its activations in a private memory pool for as long as it is cached: at batch_size
             32 the decoder's full-resolution layers alone are 9 GB per tensor, and capturing that graph next to the other
             arms ran out of the H100's 80 GB, so it is not an arm.
  baseline   today's route on the first `--baseline-clips` of the same latents: per clip, host -> device, model.decode at
             B = 1, output_to_frames, .cpu().

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

LATENT = (4, 5, 32, 32)
KERNEL_SHAPE = (1, 3, 17, 576, 1024)


def bench_kernel(torch, launches: int) -> dict:
    from cvvae_b200.video_io import batch_to_frames
    x = torch.randn(KERNEL_SHAPE, generator=torch.Generator(device="cuda").manual_seed(0), device="cuda").half()
    out = torch.empty((1, *KERNEL_SHAPE[2:], 3), dtype=torch.uint8, device="cuda")
    for _ in range(20):
        batch_to_frames(x, out=out)
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(launches):
        batch_to_frames(x, out=out)
    stop.record()
    stop.synchronize()
    s = start.elapsed_time(stop) * 1e-3 / launches
    n = KERNEL_SHAPE[2] * KERNEL_SHAPE[3] * KERNEL_SHAPE[4]
    return {"arm": "kernel", "shape": "fp16 [1,3,17,576,1024] -> uint8 [1,17,576,1024,3]", "launches": launches,
            "us_per_launch": round(s * 1e6, 1), "GB_per_s": round((2 * 3 * n + 3 * n) / s / 1e9, 1)}


def today_route(torch, m, latents):
    from cvvae_b200.video_io import output_to_frames
    return [output_to_frames(m.decode(z[None].to(m.device)).sample).cpu() for z in latents]


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--launches", type=int, default=200, help="timed kernel launches (after 20 untimed)")
    ap.add_argument("--clips", type=int, default=32, help="clips per decode_clips run")
    ap.add_argument("--baseline-clips", type=int, default=8, help="clips per run of today's route")
    ap.add_argument("--reps", type=int, default=3, help="timed runs per arm")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        print("bench_decode_clips.py needs a GPU: no CUDA device is available", file=sys.stderr)
        return 2
    import __graft_entry__ as ge
    from bench import CONFIGS, build_model
    from cvvae_b200 import decode_clips
    from tools.bench_stream import card
    ge.build()
    print(json.dumps({"card": card(), **bench_kernel(torch, args.launches)}), flush=True)

    m = build_model(CONFIGS["c5"], torch.float16)
    mg = build_model(CONFIGS["c5"], torch.float16).enable_cuda_graphs(True)   # its own model: disabling graphs drops them
    g = torch.Generator().manual_seed(1)
    latents = [torch.randn(LATENT, generator=g).half() for _ in range(args.clips)]
    base = latents[:args.baseline_clips]

    def decode_arm(bs, graphs):
        return lambda: sum(1 for _ in decode_clips(mg if graphs else m, latents, batch_size=bs))

    arms = {f"decode_clips bs={bs} {'graphs' if gr else 'eager'}": decode_arm(bs, gr)
            for bs in (1, 8, 32) for gr in (False, True) if not (gr and bs > 8)}
    arms["per-clip decode + output_to_frames + .cpu()"] = lambda: len(today_route(torch, m, base))

    # the two routes must agree bit for bit
    same = all(torch.equal(a, b) for a, b in zip(decode_clips(m, base[:2], batch_size=2), today_route(torch, m, base[:2])))

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
        print(json.dumps({"arm": name, "model": model, "clips": args.baseline_clips if name.startswith("per-clip") else args.clips,
                          "clip": f"latents {list(LATENT)} -> 17x256x256x3", "reps": args.reps,
                          "clips_per_s": round(rs[len(rs) // 2], 2), "clips_per_s_spread": [round(rs[0], 2), round(rs[-1], 2)],
                          "peak_device_MiB": round(peaks[name] / 2 ** 20, 1)}), flush=True)
    print(json.dumps({"routes_bit_identical": same, "card_after_runs": card()}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())

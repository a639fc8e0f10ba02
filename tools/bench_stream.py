#!/usr/bin/env python
"""Streaming vs whole-clip encode -> mode -> decode: frames/s and peak device memory as the clip grows.

    python tools/bench_stream.py [--frames 33 129 257] [--reps 3]

SD2.1 model at full width (seeded random weights, as bench.py), fp16, 576x1024, default tiling (576-px tiles, 16-frame
chunks).  The input is one seeded uint8 clip.  Two comparisons per clip length T:

  device   whole:  model.decode(model.encode(x).latent_dist.mode()).sample on the clip resident on the device
           stream: StreamEncoder -> mode() -> StreamDecoder over the same resident clip fed 16 frames at a time,
                   each reconstructed chunk dropped as it arrives
           peak = torch.cuda.max_memory_allocated() above what was allocated before the call (weights, resident clip)
  host     script: host uint8 clip -> H2D -> frames_to_input -> whole-clip encode/mode/decode -> output_to_frames -> D2H
                   (cvvae_inference_video.py's chain)
           stream: reconstruct_frames over the host clip in 16-frame items, each yielded piece dropped
           peak as above (nothing resident but the weights)

Each arm runs once untimed per T, then `--reps` times alternating with its partner; a time is a host clock around the
call that ends in a device synchronise.  The line reports the median and the spread (min, max) of the reps.  The card's
name, power limit and SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import CONFIGS, build_model  # noqa: E402
from cvvae_b200 import StreamDecoder, StreamEncoder, reconstruct_frames  # noqa: E402
from cvvae_b200.video_io import frames_to_input, output_to_frames  # noqa: E402

H, W, ITEM = 576, 1024, 16


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), (v.strip() for v in out.strip().split(","))))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name()}


def measure(fn):
    """(seconds, peak bytes above the allocation at the start) of one call, ending in a device synchronise."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[33, 129, 257])
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_stream.py needs a GPU"
    import __graft_entry__ as ge
    ge.build()
    m = build_model(CONFIGS["c2"], torch.float16)

    def whole_device(x):
        m.decode(m.encode(x).latent_dist.mode()).sample

    def stream_device(x):
        enc, dec = StreamEncoder(m), StreamDecoder(m)
        for a in range(0, x.shape[2], ITEM):
            for post in enc.feed(x[:, :, a:a + ITEM]):
                dec.feed(post.mode())
        for post in enc.close():
            dec.feed(post.mode())
        dec.close()

    def script_host(frames_u8):
        T = frames_u8.shape[0]
        x = frames_to_input(frames_u8[:1 + (T - 1) // 4 * 4].cuda())
        output_to_frames(m.decode(m.encode(x).latent_dist.mode()).sample).cpu()

    def stream_host(frames_u8):
        for _ in reconstruct_frames(m, (frames_u8[a:a + ITEM] for a in range(0, frames_u8.shape[0], ITEM))):
            pass

    rows = []
    for T in args.frames:
        frames_u8 = torch.randint(0, 256, (T, H, W, 3), generator=torch.Generator().manual_seed(T), dtype=torch.uint8)
        x = frames_to_input(frames_u8.cuda())
        pairs = {"device": (("whole", lambda: whole_device(x)), ("stream", lambda: stream_device(x))),
                 "host": (("script", lambda: script_host(frames_u8)), ("stream", lambda: stream_host(frames_u8)))}
        row = {"frames": T, "shape": f"1x3x{T}x{H}x{W}"}
        for kind, arms in pairs.items():
            for _, fn in arms:                       # warm-up: every shape the timed calls use, graphs off
                fn()
            res = {name: [] for name, _ in arms}
            for _ in range(args.reps):
                for name, fn in arms:
                    res[name].append(measure(fn))
            for name, runs in res.items():
                fps = sorted(T / s for s, _ in runs)
                row[f"{kind}_{name}"] = {"frames_per_s": round(fps[len(fps) // 2], 2),
                                         "frames_per_s_spread": [round(fps[0], 2), round(fps[-1], 2)],
                                         "peak_gb": round(max(p for _, p in runs) / 1e9, 3)}
        row["card_after_runs"] = card()              # SM clock sampled right after the timed calls
        del x
        torch.cuda.empty_cache()
        rows.append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"card": card(), "model": "sd21 full width, fp16, seeded random weights, default tiling",
                      "reps": args.reps, "results": rows}), flush=True)


if __name__ == "__main__":
    main()

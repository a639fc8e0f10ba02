#!/usr/bin/env python
"""What FVD's I3D embedding costs on the GPU, against PyTorch's own fp32 evaluation of the same network.

    python tools/bench_fvd.py [--clips 64] [--frames 16] [--groups 4,8,16,32,64] [--reps 10] [--stream-clips 128]
                              [--skip-stream]

  network  `--clips` resident prepared clips of `--frames` x 224 x 224 (seeded weights in the PyTorch port's layout,
           tests/i3d_ref.py), embedded by the network (I3D._embed: the packing, 57 convolutions, 13 pools and the head per
           group) at each group size of `--groups`; one untimed call, then `--reps` timed calls between CUDA events.  Clips
           per second, and the convolutions' executed and algorithmic TF32 rates (MACs from the plan's shapes: the stem
           at 448 x 3 packed channels executed, 3 x 7^3 algorithmic).
  torch    the restatement (tests/i3d_ref.py) in fp32 with PyTorch's defaults (cuDNN, TF32 on) on the same prepared
           clips, 16 at a time, alternated rep by rep with ours at the largest group size.
  stream   embed_clips over `--stream-clips` host uint8 clips of 16 x 720 x 1280 (batch 16): upload, preparation
           (resize and crop to 224), network, download; host clock around the whole iteration, after one untimed pass.

The card's name, power limit and SM clock are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [v.strip() for v in out.stdout.splitlines()[0].split(",")])) if out.returncode == 0 else {}


def conv_macs(T: int, executed: bool) -> int:
    """MACs of the 57 convolutions on one clip of T x 224 x 224, from the plan's shapes."""
    from cvvae_b200.fvd import i3d_plan
    plan = i3d_plan(T)
    total = 0
    for s in plan.steps:
        if s.op != "conv":
            continue
        k = s.cin * math.prod(s.kernel) if executed or s.src != 1 else 3 * 7 ** 3
        total += math.prod(plan.buffers[s.dst][:3]) * s.cout * k
    return total


def timed(torch, fn, reps: int) -> float:
    """Seconds per call: CUDA events around `reps` calls, after the device is idle."""
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3 / reps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--groups", default="4,8,16,32,64")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--stream-clips", type=int, default=128)
    ap.add_argument("--skip-stream", action="store_true")
    args = ap.parse_args()

    import torch

    import i3d_ref as R
    from cvvae_b200 import I3D, embed_clips, frames_to_training_input
    from cvvae_b200.fvd import I3D_GROUP_BYTES, i3d_plan

    assert torch.cuda.is_available(), "bench_fvd measures on the GPU"
    info = card()
    print(json.dumps({"card": info}), flush=True)
    sd = R.make_state_dict(0)
    i3d = I3D.from_state_dict(sd)
    N, T = args.clips, args.frames
    g = torch.Generator(device="cuda").manual_seed(0)
    clips = torch.randint(0, 256, (N, T, 224, 224, 3), generator=g, device="cuda", dtype=torch.uint8)
    x = torch.empty((N, 3, T, 224, 224), device="cuda")
    for i in range(N):
        frames_to_training_input(clips[i], 224, "short", torch.float32, out=x[i:i + 1])
    clip_bytes = i3d_plan(T).clip_bytes()
    executed, algorithmic = conv_macs(T, True), conv_macs(T, False)
    rows = []
    for group in [int(v) for v in args.groups.split(",")]:
        i3d._group_bytes = group * clip_bytes
        i3d._embed(x)
        s = timed(torch, lambda: i3d._embed(x), args.reps)
        rows.append({"group": group, "clips_per_s": N / s, "ms_per_clip": 1e3 * s / N,
                     "executed_tflops": 2 * executed * N / s / 1e12, "algorithmic_tflops": 2 * algorithmic * N / s / 1e12})
        print(json.dumps({"network": rows[-1], "frames": T, "clips": N}), flush=True)

    # ours at the largest group, alternated rep by rep with PyTorch's fp32 evaluation (16 clips per call)
    torch_batch = 16
    ref = lambda: [R.embed(x[n:n + torch_batch], sd, tf32=True) for n in range(0, N, torch_batch)]   # noqa: E731
    ref()
    ours_s, torch_s = [], []
    for _ in range(args.reps):
        ours_s.append(timed(torch, lambda: i3d._embed(x), 1))
        torch_s.append(timed(torch, ref, 1))
    ours_best, torch_best = min(ours_s), min(torch_s)
    print(json.dumps({"alternated": {"group": i3d._group_bytes // clip_bytes, "ours_clips_per_s": N / ours_best,
                                     "torch_fp32_clips_per_s": N / torch_best, "speedup": torch_best / ours_best,
                                     "ours_s": ours_s, "torch_s": torch_s}}), flush=True)
    del x, clips
    torch.cuda.empty_cache()

    if not args.skip_stream:
        gen = torch.Generator().manual_seed(1)
        base = torch.randint(0, 256, (16, 720, 1280, 3), generator=gen, dtype=torch.uint8)
        distinct = [base.roll(n, dims=2) for n in range(8)]
        host = [distinct[n % 8] for n in range(args.stream_clips)]
        i3d._group_bytes = I3D_GROUP_BYTES
        list(embed_clips(i3d, host[:16], batch_size=16))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = list(embed_clips(i3d, host, batch_size=16))
        torch.cuda.synchronize()
        s = time.perf_counter() - t0
        assert len(out) == len(host)
        print(json.dumps({"embed_clips_720p": {"clips": len(host), "clips_per_s": len(host) / s, "s": s}}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()

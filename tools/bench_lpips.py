#!/usr/bin/env python
"""What LPIPS costs: the metric's kernels on resident frames, PyTorch's own fp32 evaluation, and evaluate_frames with it.

    python tools/bench_lpips.py [--net vgg|alex] [--reps 20] [--frames 129] [--stream-reps 3] [--skip-stream]

  kernels  LPIPS.__call__'s device work (metrics.LPIPS._launch) on 4 resident frame pairs at 576x1024 and 720x1280,
           seeded weights in the real layout (tests/lpips_ref.py, tests/lpips_alex_ref.py): CUDA events around every
           launch of `--reps` calls after 3 untimed ones, summed per part; us per frame pair, and the convolutions'
           executed TF32 rate.  VGG16 (the default): the input kernel, the 13 convolutions, the 5 tap kernels; executed
           MACs per image pixel: conv1_1 as its 32-channel 1 x 1 (64 x 32) plus, for the other twelve, Cin x Cout x 9 at
           their resolution; the algorithmic count is the same with conv1_1 at 27 input channels (305,856 MAC per
           pixel).  AlexNet (--net alex): the conv1 input kernel, the two pools, the conv2 packing (the three summed as
           "packing_us"), the 5 convolutions and the 5 tap kernels; executed MACs from the tap sizes with conv1 at 384 input channels and
           conv2 at 1600, algorithmic with conv1 at 363.  Also the whole call between two events ("call_us"), which
           includes any time the GPU waits for the host's launches.
  torch    the same metric restated in PyTorch (tests/lpips_ref.py or tests/lpips_alex_ref.py, fp32, default flags:
           cuDNN with TF32), alternated call by call with ours in the same process; median us per frame pair.
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


def alex_macs_per_image(H: int, W: int, executed: bool) -> int:
    """MACs of AlexNet's five convolutions on one H x W image, from the tap sizes."""
    from cvvae_b200.metrics import _lpips_alex_tap_sizes
    (h1, w1), (h2, w2), (h3, w3) = _lpips_alex_tap_sizes(H, W)[:3]
    return (h1 * w1 * 64 * (384 if executed else 363) + h2 * w2 * 192 * 1600 +
            h3 * w3 * 9 * (192 * 384 + 384 * 256 + 256 * 256))


def bench_kernels(torch, metric, sd, reps: int) -> list:
    import lpips_alex_ref as A
    import lpips_ref as R
    from cvvae_b200 import _lib as L
    alex = metric.net == "alex"
    ref = A if alex else R
    rows = []
    for H, W in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(H)
        a = torch.randint(0, 256, (PAIRS, H, W, 3), generator=g, dtype=torch.uint8, device="cuda")
        b = (a.int() + torch.randint(-3, 4, a.shape, generator=g, device="cuda")).clamp_(0, 255).to(torch.uint8)
        assert metric._group(H, W) >= PAIRS
        lib = L.load()
        if alex:
            events = {"input": [], "pool": [], "pack5x5": [], "conv": [], "tap": []}
            fns = {"cvvae_lpips_alex_input": "input", "cvvae_lpips_max_pool3s2": "pool", "cvvae_lpips_pack5x5": "pack5x5",
                   "cvvae_conv3d": "conv", "cvvae_lpips_tap": "tap", "cvvae_lpips_tap_copy": "tap"}
        else:
            events = {"input": [], "conv": [], "tap": []}
            fns = {"cvvae_lpips_input": "input", "cvvae_conv3d": "conv", "cvvae_lpips_tap": "tap"}
        calls = []
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
                ref.lpips(a, b, sd32, torch.float32)
            torch_us = []
            for name in fns:
                setattr(lib, name, timed(name))
            try:
                for _ in range(reps):
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s.record()
                    metric._launch(a, b)
                    e.record()
                    calls.append((s, e))
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    ref.lpips(a, b, sd32, torch.float32)
                    torch.cuda.synchronize()
                    torch_us.append((time.perf_counter() - t0) * 1e6 / PAIRS)
            finally:
                for name in fns:
                    setattr(lib, name, real[name])
        torch.cuda.synchronize()
        us = {k: sum(s.elapsed_time(e) for s, e in v) * 1e3 / reps / PAIRS for k, v in events.items()}
        assert len(events["conv"]) == (5 if alex else 13) * reps and len(events["tap"]) == 5 * reps
        if alex:
            executed, algorithmic = (2 * 2 * alex_macs_per_image(H, W, x) for x in (True, False))
        else:
            executed, algorithmic = (2 * 2 * H * W * macs_per_pixel(x) for x in (True, False))   # two images, 2 FLOP/MAC
        total = sum(us.values())
        ours = metric(a, b)
        rows.append({
            "net": metric.net, "shape": f"{PAIRS} frame pairs x {H}x{W}", "reps": reps,
            "us_per_frame_pair": round(total, 1), "split_us": {k: round(v, 1) for k, v in us.items()},
            **({"packing_us": round(us["input"] + us["pool"] + us["pack5x5"], 1)} if alex else {}),
            "call_us_per_frame_pair": round(statistics.median(s.elapsed_time(e) for s, e in calls) * 1e3 / PAIRS, 1),
            "conv_executed_TFLOP_per_pair": round(executed / 1e12, 4),
            "conv_algorithmic_TFLOP_per_pair": round(algorithmic / 1e12, 4),
            "conv_executed_TFLOP_per_s": round(executed / us["conv"] / 1e6, 1),
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
    out = {"net": metric.net, "shape": f"{frames}x{H}x{W}x3", "reps": reps, "model": "sd21 full width, fp16, seeded random weights, default tiling"}
    for name, ts in times.items():
        fps = sorted(frames / s for s in ts)
        out[name] = {"frames_per_s": round(fps[len(fps) // 2], 2), "frames_per_s_spread": [round(fps[0], 2), round(fps[-1], 2)],
                     "ms_per_frame": round(1e3 / fps[len(fps) // 2], 2)}
    return out


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--net", choices=("vgg", "alex"), default="vgg", help="the LPIPS network")
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
    import lpips_alex_ref as A
    import lpips_ref as R
    from tools.bench_stream import card
    ge.build()
    from cvvae_b200 import LPIPS
    sd = (A if args.net == "alex" else R).make_state_dict(0)
    metric = LPIPS.from_state_dict(sd, net=args.net)
    print(json.dumps({"card": card(), "kernels": bench_kernels(torch, metric, sd, args.reps)}), flush=True)
    if not args.skip_stream:
        stream = bench_stream(torch, metric, args.frames, args.stream_reps)
        stream["card_after_runs"] = card()
        print(json.dumps({"stream": stream}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())

#!/usr/bin/env python
"""float32 models through the public API: encode + decode step time of the engine in fp32 against the engine in the
configuration's 16-bit dtype (alternated in one process), and against the reference algorithm on torch-CUDA in fp32
with PyTorch's default flags (cuDNN TF32 on, matmul TF32 off).  Reports peak memory per arm and the card name and power
limit read in the same run.  One JSON line per configuration.

    python tools/bench_fp32.py [--configs c2,c3] [--rounds 3] [--torch-reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

DT = {"fp16": torch.float16, "bf16": torch.bfloat16}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:  # the query is informational
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unavailable ({e.__class__.__name__})"}


def time_engine(m, x, reps):
    def step():
        with torch.no_grad():
            return m.decode(m.encode(x).latent_dist.mode()).sample
    step()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        step()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c2,c3")
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the two engine arms")
    ap.add_argument("--reps", type=int, default=2, help="timed steps per arm and round")
    ap.add_argument("--torch-reps", type=int, default=3)
    args = ap.parse_args()
    for name in args.configs.split(","):
        cfg = bench.CONFIGS[name]
        shape = (cfg["batch"], 3, cfg["frames"], cfg["height"], cfg["width"])
        zc = 4 if cfg["variant"] == "sd21" else 16
        from oracle import cvvae_oracle as O
        x32 = O.synthetic_video(shape, 1).cuda()
        arms = {"engine_fp32": torch.float32, "engine_" + cfg["dtype"]: DT[cfg["dtype"]]}
        models = {k: bench.build_model(cfg, dt) for k, dt in arms.items()}
        xs = {k: x32.to(dt) for k, dt in arms.items()}
        times = {k: [] for k in arms}
        peak = {}
        for _ in range(args.rounds):
            for k in arms:
                torch.cuda.reset_peak_memory_stats()
                times[k] += time_engine(models[k], xs[k], args.reps)
                peak[k] = max(peak.get(k, 0), torch.cuda.max_memory_allocated())
        sd = {k: v.detach().float() for k, v in models["engine_fp32"].state_dict().items()}
        del models
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        ref = bench.TorchCudaReference(cfg, sd)
        flags = {"cudnn.allow_tf32": torch.backends.cudnn.allow_tf32, "matmul.allow_tf32": torch.backends.cuda.matmul.allow_tf32}
        tc = bench.time_torch_cuda(ref, x32, zc, warmup=1, reps=args.torch_reps)
        peak["torch_cuda_fp32_default_flags"] = torch.cuda.max_memory_allocated()
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        frames = shape[0] * shape[2]
        t_ref = min(a["ms_per_step_median"] for a in tc.values())
        line = {"config": name, "shape": shape, "card": card(),
                "engine_ms_per_step_median": med, "engine_ms_all": times,
                "engine_frames_per_s": {k: frames / (v * 1e-3) for k, v in med.items()},
                "fp32_over_16bit": med["engine_fp32"] / med["engine_" + cfg["dtype"]],
                "torch_cuda_fp32": tc, "torch_cuda_flags": flags,
                "engine_fp32_speedup_vs_torch_cuda_fp32": t_ref / med["engine_fp32"],
                "peak_memory_gib": {k: v / 2 ** 30 for k, v in peak.items()}}
        print(json.dumps(line), flush=True)
        del ref, xs, x32
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

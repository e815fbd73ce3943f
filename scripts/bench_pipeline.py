#!/usr/bin/env python
"""Keyframe interpolation pipeline on full-size synthetic weights: 320 x 512, DDIM-50, CFG 7.5 (scripts/run.sh).

For K = 2 and K = 5 keyframes it times, alternating in one process, two ways to get the same storyboard:
  batched:  ToonCrafterPipeline.interpolate(K keyframes)  (the S = K-1 segments as the rows of one fused sample())
  pairs:    S separate one-pair interpolate() calls (one sample() + the two decodes per pair, bench.py's run_clip order)
Each arm is warmed up once at DDIM-2 (plans, graphs), then timed `--reps` times with the device synchronised.
Prints the GPU name and power limit (nvidia-smi) and one JSON line.

    python scripts/bench_pipeline.py [--reps 2] [--ddim-steps 50]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def full_pipeline_config():
    """configs/inference_512_v1.0.yaml with the OpenCLIP towers and the Resampler of this repository."""
    from tiny_config import FULL_DDCONFIG, FULL_UNET, model_config
    cfg = model_config(FULL_UNET, FULL_DDCONFIG)
    p = cfg["params"]
    p["cond_stage_config"] = {"target": "tooncrafter_b200.modules.FrozenOpenCLIPEmbedder",
                              "params": {"freeze": True, "layer": "penultimate"}}
    p["img_cond_stage_config"] = {"target": "tooncrafter_b200.modules.FrozenOpenCLIPImageEmbedderV2",
                                  "params": {"freeze": True}}
    p["image_proj_stage_config"] = {"target": "lvdm.modules.encoders.resampler.Resampler",
                                    "params": dict(dim=1024, depth=4, dim_head=64, heads=12, num_queries=16,
                                                   embedding_dim=1280, output_dim=1024, ff_mult=4, video_length=16)}
    return cfg


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return dict(name=name, power_limit=power)
    except Exception as e:  # noqa: BLE001 - the measurement stands without it, but say why it is missing
        return dict(name=torch.cuda.get_device_name(), power_limit=f"unavailable ({type(e).__name__})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--ddim-steps", type=int, default=50)
    args = ap.parse_args()
    from tooncrafter_b200 import synthetic
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    if not torch.cuda.is_available():
        raise SystemExit("bench_pipeline.py measures the GPU; no CUDA device found")
    dev = torch.device("cuda")
    info = gpu_info()
    print(f"GPU: {info['name']}, power limit {info['power_limit']}", flush=True)
    torch.backends.cuda.matmul.allow_tf32 = False
    t0 = time.perf_counter()
    model = synthetic.synthetic_model(full_pipeline_config(), dev)
    model.perframe_ae = True
    build_s = time.perf_counter() - t0
    pipe = ToonCrafterPipeline(model)
    g = torch.Generator().manual_seed(0)
    results = []
    for K in (2, 5):
        kf = (torch.rand(K, 320, 512, 3, generator=g) * 255).to(torch.uint8)
        S = K - 1

        def batched(steps):
            return pipe.interpolate(kf, steps=steps, seed=123)

        def pairs(steps):
            return [pipe.interpolate(kf[k:k + 2], steps=steps, seed=123 + k) for k in range(S)]

        arms = dict(batched=batched, pairs=pairs)
        for fn in arms.values():
            fn(2)
        torch.cuda.synchronize()
        times = {name: [] for name in arms}
        for _ in range(args.reps):
            for name, fn in arms.items():
                torch.cuda.synchronize()
                t = time.perf_counter()
                fn(args.ddim_steps)
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t)
        F = 15 * S + 1
        row = dict(K=K, segments=S, frames=F)
        for name, ts in times.items():
            best = min(ts)
            row[name] = dict(sec_per_video=best, frames_per_s=F / best, all_s=[round(x, 3) for x in ts])
        row["batched_over_pairs_time"] = row["batched"]["sec_per_video"] / row["pairs"]["sec_per_video"]
        results.append(row)
        print(json.dumps(row), flush=True)
    out = dict(metric="keyframe interpolation: seconds per video (320x512, DDIM-%d, CFG 7.5, eta 1, synthetic weights)"
               % args.ddim_steps, gpu=info, reps=args.reps, model_build_s=build_s, configs=results,
               note="sec_per_video = best of the timed reps, host clock around work ending in a device synchronise; "
                    "frames counts the joined video (15 * segments + 1)")
    print(json.dumps(out), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())

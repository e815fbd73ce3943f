#!/usr/bin/env python
"""DDIM against DPM-Solver++(2M) on full-size synthetic weights: K = 2 keyframes at 320 x 512, CFG 7.5, the
pipeline's defaults otherwise (scripts/run.sh).

For eta 0 and 1 and each step count it times ToonCrafterPipeline.interpolate(sampler="ddim") and
interpolate(sampler="dpmpp_2m"), alternating, `--reps` times each after a warm-up of both at DDIM-4 (plans, graphs),
and reports seconds per video.  Both samplers run the same UNet evaluations per step, so their difference is the
update kernel's.  That kernel is also timed alone at the same shape (one row of 4 x 16 x 40 x 64 latents): CUDA events
around `--kernel-reps` launches of tc_ddim_step and of tc_dpm_step with a non-zero correction weight, alternating.
Prints the GPU name and power limit (nvidia-smi) and one JSON line.

    python scripts/bench_samplers.py [--reps 2] [--steps 10 15 20 25 50]
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "scripts"))
sys.path.insert(0, str(ROOT / "tests"))


def update_kernel_us(reps: int) -> dict:
    """Microseconds per call of ops.ddim_step and ops.dpm_step (guidance rescale on, c = 0.3) at B = 1, n = 163840."""
    from tooncrafter_b200 import ops
    B, n = 1, 4 * 16 * 40 * 64
    g = torch.Generator().manual_seed(0)
    r = lambda: torch.randn(B, n, generator=g).cuda()
    e_c, e_uc = r().half(), r().half()
    x, noise, prev = r(), r(), r()
    x_prev, pred = torch.empty_like(x), torch.empty_like(x)
    head = [7.5, 0.7, 0.6, 0.8, 0.98, 0.7, 0.3, 0.5]
    coef_ddim = torch.tensor(head, device="cuda")
    coef_dpm = torch.tensor(head + [0.3], device="cuda")
    ws = torch.empty(4 * B * ops.DDIM_PARTIALS, dtype=torch.float64, device="cuda")
    arms = {"tc_ddim_step": lambda: ops.ddim_step(e_c, e_uc, x, noise, x_prev, pred, coef_ddim, ws, B=B, n=n),
            "tc_dpm_step": lambda: ops.dpm_step(e_c, e_uc, x, noise, prev, x_prev, pred, coef_dpm, ws, B=B, n=n)}
    for fn in arms.values():
        for _ in range(20):
            fn()
    out = {name: [] for name in arms}
    for _ in range(5):
        for name, fn in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                fn()
            b.record()
            b.synchronize()
            out[name].append(1e3 * a.elapsed_time(b) / reps)
    return {name: min(v) for name, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--steps", type=int, nargs="+", default=[10, 15, 20, 25, 50])
    ap.add_argument("--kernel-reps", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_samplers.py measures the GPU; no CUDA device found")
    from bench_pipeline import full_pipeline_config, gpu_info
    from tooncrafter_b200 import synthetic
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    info = gpu_info()
    print(f"GPU: {info['name']}, power limit {info['power_limit']}", flush=True)
    torch.backends.cuda.matmul.allow_tf32 = False
    size = (320, 512)
    kernel = update_kernel_us(args.kernel_reps)
    print(f"update kernel pair per step: tc_ddim_step {kernel['tc_ddim_step']:.1f} us, "
          f"tc_dpm_step {kernel['tc_dpm_step']:.1f} us", flush=True)
    model = synthetic.synthetic_model(full_pipeline_config(size), torch.device("cuda"))
    model.perframe_ae = True
    pipe = ToonCrafterPipeline(model)
    kf = (torch.rand(2, size[0], size[1], 3, generator=torch.Generator().manual_seed(0)) * 255).to(torch.uint8)
    call = lambda sampler, steps, eta: pipe.interpolate(kf, steps=steps, eta=eta, seed=123, size=size,
                                                        sampler=sampler)
    for sampler in ("ddim", "dpmpp_2m"):
        call(sampler, 4, 1.0)
    results = []
    for eta in (0.0, 1.0):
        for steps in args.steps:
            times = {"ddim": [], "dpmpp_2m": []}
            for _ in range(args.reps):
                for sampler in times:
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    call(sampler, steps, eta)
                    torch.cuda.synchronize()
                    times[sampler].append(time.perf_counter() - t)
            row = dict(eta=eta, steps=steps, **{f"{k}_s": [round(v, 3) for v in vs] for k, vs in times.items()})
            print(f"eta {eta:.0f}, {steps:2d} steps: DDIM {min(times['ddim']):.3f} s, "
                  f"DPM++(2M) {min(times['dpmpp_2m']):.3f} s per video", flush=True)
            results.append(row)
    print(json.dumps(dict(gpu=info["name"], power_limit=info["power_limit"], size=list(size), K=2, cfg_scale=7.5,
                          update_kernel_us=kernel, seconds_per_video=results)))
    return 0


if __name__ == "__main__":
    sys.exit(main())

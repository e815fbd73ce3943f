#!/usr/bin/env python
"""Keyframe interpolation pipeline on full-size synthetic weights: 320 x 512, DDIM-50, CFG 7.5 (scripts/run.sh).

For K = 2 and K = 5 keyframes it times, alternating in one process, two ways to get the same storyboard:
  batched:  ToonCrafterPipeline.interpolate(K keyframes)  (the S = K-1 segments as the rows of one fused sample())
  pairs:    S separate one-pair interpolate() calls (one sample() + the two decodes per pair, bench.py's run_clip order)
Each arm is warmed up once at DDIM-2 (plans, graphs), then timed `--reps` times with the device synchronised.
Prints the GPU name and power limit (nvidia-smi) and one JSON line.

    python scripts/bench_pipeline.py [--reps 2] [--ddim-steps 50] [--first-stage plain|dualref] [--size H W]

--animate measures the single-image path instead, at --size with --first-stage: seconds per video and frames/s of
ToonCrafterPipeline.animate and of a K = 2 interpolate() (warm-up, then `--reps` timed runs each, alternating), the
peak device memory of each, the peak of a default K = 5 interpolate() call (segments_per_batch 4, DDIM-2: memory does
not depend on the step count), and the first-stage decode of 16 latents, plain against dual-reference decoder (CUDA
events, 10 replays after a warm-up):

    python scripts/bench_pipeline.py --animate --first-stage plain --size 576 1024

--video-length T [T ...] measures a K = 2 interpolate() with T frames per segment at --size with --first-stage, for
each T in turn: seconds per video and frames/s (warm-up at DDIM-2, then `--reps` timed calls) and the peak device
memory of a timed call.  Each T starts from freshly built engines, so its peak holds its own plans only:

    python scripts/bench_pipeline.py --video-length 8 16 24 32 64

--gpus N measures ToonCrafterPipeline sharded over N GPUs, one process per GPU under torchrun (--gpus 1: the same
workload on one GPU, without torchrun): a K = 5 interpolate() at --size, or with --animate one animate() call, with
--latency-mode one clip per GPU pair.  Warm-up at DDIM-2, then `--reps` timed calls, each between a barrier and a
device synchronise; the time reported is the maximum over ranks.

    python scripts/bench_pipeline.py --gpus 1
    torchrun --nproc-per-node 2 scripts/bench_pipeline.py --gpus 2 [--latency-mode]
    torchrun --nproc-per-node 2 scripts/bench_pipeline.py --gpus 2 --latency-mode --animate --first-stage plain \
        --size 576 1024

--n-samples N [N ...] measures variants of a K = 2 interpolate() at --size, for each n in turn: one batched call
(interpolate(n_samples=n), the variants as rows of the same sample() calls) against n separate single-sample calls,
alternating; seconds per call and per sample, and the peak device memory of each arm (warm-up at DDIM-2):

    python scripts/bench_pipeline.py --n-samples 1 2 4 8

--pairs P measures interpolate_pairs() on P synthetic keyframe pairs (--n-samples n, default 1), sharded over --gpus
N as above (the maximum over ranks): seconds per call and per clip:

    python scripts/bench_pipeline.py --pairs 8 --gpus 1
    torchrun --nproc-per-node 2 scripts/bench_pipeline.py --pairs 8 --gpus 2

--refine S [S ...] measures ToonCrafterPipeline.refine on a synthetic 16-frame clip at --size: interpolate() of the
clip's first and last frames (K = 2), refine() at each strength S (int(S * steps) DDIM steps plus the encode of the
16 frames), and refine(0.5, keep=[0, 1, 14, 15]) (the masked fused sampler), alternating; seconds per call and the
peak device memory of each arm (warm-up at DDIM-4, so that every strength runs a step):

    python scripts/bench_pipeline.py --refine 0.25 0.5 1.0
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def full_pipeline_config(size=(320, 512)):
    """configs/inference_512_v1.0.yaml with the OpenCLIP towers and the Resampler of this repository (image_size:
    the latent of `size`, as configs/training_1024_v1.0 sets [72, 128] for 576 x 1024)."""
    from tiny_config import FULL_DDCONFIG, FULL_UNET, model_config
    cfg = model_config(FULL_UNET, FULL_DDCONFIG)
    cfg["params"]["image_size"] = [size[0] // 8, size[1] // 8]
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


def _timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, torch.cuda.max_memory_allocated()


def decode_ms(size, reps=10):
    """ms per decode of 16 latents at `size`, plain AutoencoderKL vs AutoencoderKL_Dualref (full width, synthetic
    weights, the dual-reference decoder with its reference-frame maps), each engine's program replayed as a graph."""
    from tiny_config import FULL_DDCONFIG
    from tooncrafter_b200 import diffusion, synthetic
    h, w = size[0] // 8, size[1] // 8
    z = torch.randn(16, 4, h, w, generator=torch.Generator().manual_seed(1)).cuda() * 3.0
    out = {}
    for name, cls in (("plain", diffusion.AutoencoderKL), ("dualref", diffusion.AutoencoderKL_Dualref)):
        with torch.device("meta"):
            sk = cls(ddconfig=FULL_DDCONFIG, embed_dim=4)
        ae = sk.to_empty(device="cuda")
        with torch.no_grad():
            for k, p in ae.named_parameters():
                p.copy_(synthetic.synthetic_tensor("first_stage_model." + k, tuple(p.shape), 0).cuda())
        eng = ae.decoder_engine()
        if name == "plain":
            run = lambda: eng.decode(z)                                                      # noqa: E731
        else:
            ref = [r.cuda() for r in synthetic.synthetic_ref_context(FULL_DDCONFIG["ch"], FULL_DDCONFIG["ch_mult"],
                                                                     size[0], size[1])]
            run = lambda: eng.decode(z, ref)                                                 # noqa: E731
        run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            run()
        e1.record()
        torch.cuda.synchronize()
        out[name] = e0.elapsed_time(e1) / reps
        del eng, ae
        torch.cuda.empty_cache()
    return out


def bench_animate(args, model, info, build_s, decode16):
    """animate and K = 2 interpolate at args.size (see the module docstring)."""
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    size = tuple(args.size)
    pipe = ToonCrafterPipeline(model)
    g = torch.Generator().manual_seed(0)
    kf = (torch.rand(5, size[0], size[1], 3, generator=g) * 255).to(torch.uint8)
    arms = dict(animate=(lambda st: pipe.animate(kf[0], steps=st, seed=123, size=size), 16),
                interpolate_k2=(lambda st: pipe.interpolate(kf[:2], steps=st, seed=123, size=size), 16))
    for fn, _ in arms.values():
        fn(2)
    times = {name: [] for name in arms}
    peaks = {name: 0 for name in arms}
    for _ in range(args.reps):
        for name, (fn, _) in arms.items():
            t, peak = _timed(lambda: fn(args.ddim_steps))
            times[name].append(t)
            peaks[name] = max(peaks[name], peak)
    row = {}
    for name, (_, F) in arms.items():
        best = min(times[name])
        row[name] = dict(frames=F, sec_per_video=best, frames_per_s=F / best, all_s=[round(x, 3) for x in times[name]],
                         peak_mem_gib=peaks[name] / 2 ** 30)
    _, peak5 = _timed(lambda: pipe.interpolate(kf, steps=2, seed=123, size=size))
    row["interpolate_k5_default_peak_mem_gib"] = peak5 / 2 ** 30
    row["decode16_ms"] = decode16
    out = dict(metric="single-image animate and K=2 interpolation: seconds per video (%dx%d, DDIM-%d, CFG 7.5, eta 1, "
               "synthetic weights, %s first stage)" % (size[0], size[1], args.ddim_steps, args.first_stage),
               gpu=info, reps=args.reps, model_build_s=build_s, first_stage=args.first_stage, size=list(size), **row,
               note="sec_per_video = best of the timed reps, host clock around work ending in a device synchronise; "
                    "peak_mem = torch.cuda.max_memory_allocated over the call (model and cached plans included); "
                    "decode16_ms = CUDA events over 10 graph replays of one 16-latent decode")
    print(json.dumps(out), flush=True)
    return 0


def bench_video_length(args, model, info, build_s):
    """K = 2 interpolate at each T of args.video_length (see the module docstring)."""
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    size = tuple(args.size)
    pipe = ToonCrafterPipeline(model)
    kf = (torch.rand(2, size[0], size[1], 3, generator=torch.Generator().manual_seed(0)) * 255).to(torch.uint8)
    rows = []
    for T in args.video_length:
        model.model.diffusion_model._engine = None                  # this T's plans only in the peak
        model.first_stage_model._dec_engine = None
        torch.cuda.empty_cache()
        run = lambda st: pipe.interpolate(kf, steps=st, seed=123, size=size, video_length=T)   # noqa: E731
        run(2)
        times, peak = [], 0
        for _ in range(args.reps):
            dt, pk = _timed(lambda: run(args.ddim_steps))
            times.append(dt)
            peak = max(peak, pk)
        best = min(times)
        row = dict(video_length=T, frames=T, sec_per_video=best, frames_per_s=T / best,
                   all_s=[round(x, 3) for x in times], peak_gib=peak / 2 ** 30)
        rows.append(row)
        print(json.dumps(row), flush=True)
    out = dict(metric="K = 2 interpolation by frames per segment: seconds per video (%dx%d, DDIM-%d, CFG 7.5, eta 1, "
               "synthetic weights, %s first stage)" % (size[0], size[1], args.ddim_steps, args.first_stage), gpu=info,
               reps=args.reps, model_build_s=build_s, configs=rows,
               note="sec_per_video = best of the timed reps, host clock around work ending in a device synchronise; "
                    "peak_gib = torch.cuda.max_memory_allocated over a timed call")
    print(json.dumps(out), flush=True)
    return 0


def bench_n_samples(args, model, info, build_s):
    """K = 2 interpolate with n variants, batched against n single-sample calls (see the module docstring)."""
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    size = tuple(args.size)
    pipe = ToonCrafterPipeline(model)
    kf = (torch.rand(2, size[0], size[1], 3, generator=torch.Generator().manual_seed(0)) * 255).to(torch.uint8)
    rows = []
    for n in args.n_samples:
        arms = dict(batched=lambda st: pipe.interpolate(kf, steps=st, seed=123, size=size, n_samples=n),
                    separate=lambda st: [pipe.interpolate(kf, steps=st, seed=123 + v, size=size) for v in range(n)])
        for fn in arms.values():
            fn(2)
        times, peaks = {a: [] for a in arms}, {a: 0 for a in arms}
        for _ in range(args.reps):
            for name, fn in arms.items():
                dt, pk = _timed(lambda: fn(args.ddim_steps))
                times[name].append(dt)
                peaks[name] = max(peaks[name], pk)
        row = dict(n_samples=n)
        for name in arms:
            best = min(times[name])
            row[name] = dict(sec_per_call=best, sec_per_sample=best / n, all_s=[round(x, 3) for x in times[name]],
                             peak_gib=peaks[name] / 2 ** 30)
        row["batched_over_separate_time"] = row["batched"]["sec_per_call"] / row["separate"]["sec_per_call"]
        rows.append(row)
        print(json.dumps(row), flush=True)
    out = dict(metric="K = 2 interpolation, n variants: seconds per call and per sample, batched vs n single-sample "
               "calls (%dx%d, DDIM-%d, CFG 7.5, eta 1, synthetic weights, %s first stage)"
               % (size[0], size[1], args.ddim_steps, args.first_stage), gpu=info, reps=args.reps,
               model_build_s=build_s, configs=rows,
               note="sec_per_call = best of the timed reps, host clock around work ending in a device synchronise; "
                    "peak_gib = torch.cuda.max_memory_allocated over a timed call (model and cached plans included)")
    print(json.dumps(out), flush=True)
    return 0


def bench_refine(args, model, info, build_s):
    """interpolate against refine at each strength of args.refine and one keep case (see the module docstring)."""
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    size = tuple(args.size)
    pipe = ToonCrafterPipeline(model)
    clip = (torch.rand(16, size[0], size[1], 3, generator=torch.Generator().manual_seed(0)) * 255).to(torch.uint8)
    arms = {"interpolate": lambda st: pipe.interpolate(clip[[0, 15]], steps=st, seed=123, size=size)}
    for strength in args.refine:
        arms[f"refine_{strength:g}"] = lambda st, s_=strength: pipe.refine(clip, s_, steps=st, seed=123, size=size)
    arms["refine_0.5_keep"] = lambda st: pipe.refine(clip, 0.5, keep=[0, 1, 14, 15], steps=st, seed=123, size=size)
    for fn in arms.values():
        fn(4)
    times, peaks = {a: [] for a in arms}, {a: 0 for a in arms}
    for _ in range(args.reps):
        for name, fn in arms.items():
            dt, pk = _timed(lambda: fn(args.ddim_steps))
            times[name].append(dt)
            peaks[name] = max(peaks[name], pk)
    rows = []
    for name in arms:
        best = min(times[name])
        row = dict(arm=name, sec_per_call=best, all_s=[round(x, 3) for x in times[name]],
                   peak_gib=peaks[name] / 2 ** 30, gpu=info)
        rows.append(row)
        print(json.dumps(row), flush=True)
    out = dict(metric="refine a 16-frame clip: seconds per call (%dx%d, DDIM-%d, CFG 7.5, eta 1, synthetic weights, "
               "%s first stage)" % (size[0], size[1], args.ddim_steps, args.first_stage), gpu=info, reps=args.reps,
               model_build_s=build_s, configs=rows,
               note="sec_per_call = best of the timed reps, host clock around work ending in a device synchronise; "
                    "peak_gib = torch.cuda.max_memory_allocated over a timed call (model and cached plans included)")
    print(json.dumps(out), flush=True)
    return 0


def bench_sharded(args, model, info, build_s, group):
    """--gpus N: K = 5 interpolate (or animate) sharded over `group` (None: one GPU); see the module docstring."""
    import torch.distributed as dist

    from tooncrafter_b200.distributed import max_over_ranks
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    size = tuple(args.size)
    pipe = ToonCrafterPipeline(model, group, latency=args.latency_mode)
    g = torch.Generator().manual_seed(0)
    kf = (torch.rand(5, size[0], size[1], 3, generator=g) * 255).to(torch.uint8)
    if args.pairs is not None:
        n = args.n_samples[0] if args.n_samples else 1
        kp = (torch.rand(2 * args.pairs, size[0], size[1], 3, generator=g) * 255).to(torch.uint8)
        pairs = [(kp[2 * i], kp[2 * i + 1]) for i in range(args.pairs)]
        fn = lambda st: pipe.interpolate_pairs(pairs, n_samples=n, steps=st, seed=123, size=size)   # noqa: E731
        frames, what = 16 * n * args.pairs, f"interpolate_pairs P={args.pairs} n={n}"
    elif args.animate:
        fn, frames, what = (lambda st: pipe.animate(kf[0], steps=st, seed=123, size=size)), 16, "animate"
    else:
        fn, frames, what = (lambda st: pipe.interpolate(kf, steps=st, seed=123, size=size)), 15 * 4 + 1, "K=5"
    fn(2)
    times = []
    for _ in range(args.reps):
        torch.cuda.synchronize()
        if group is not None:
            dist.barrier(group)
        t = time.perf_counter()
        fn(args.ddim_steps)
        torch.cuda.synchronize()
        times.append(max_over_ranks(time.perf_counter() - t, model.device))
    if group is not None and dist.get_rank() != 0:
        return 0
    best = min(times)
    out = dict(metric="%s %s: seconds per video over %d GPU%s (%dx%d, DDIM-%d, CFG 7.5, eta 1, synthetic weights, %s "
               "first stage)" % (what, "latency mode" if args.latency_mode else "sharded", args.gpus,
                                 "s" if args.gpus > 1 else "", size[0], size[1], args.ddim_steps, args.first_stage),
               gpu=info, gpus=args.gpus, latency_mode=args.latency_mode, reps=args.reps, model_build_s=build_s,
               frames=frames, sec_per_video=best, frames_per_s=frames / best, all_s=[round(x, 3) for x in times],
               **(dict(pairs=args.pairs, sec_per_clip=best * 16 / frames) if args.pairs is not None else {}),
               note="sec_per_video = best of the timed reps; each rep is the maximum over ranks of a host clock "
                    "started after a barrier and stopped after a device synchronise")
    print(json.dumps(out), flush=True)
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--ddim-steps", type=int, default=50)
    ap.add_argument("--first-stage", choices=("dualref", "plain"), default="dualref",
                    help="AutoencoderKL_Dualref (ToonCrafter) or the plain AutoencoderKL (DynamiCrafter / training configs)")
    ap.add_argument("--size", type=int, nargs=2, default=(320, 512), metavar=("H", "W"))
    ap.add_argument("--animate", action="store_true", help="measure animate and K = 2 interpolation (docstring)")
    ap.add_argument("--gpus", type=int, default=None,
                    help="measure the pipeline sharded over N GPUs, under torchrun when N > 1 (docstring)")
    ap.add_argument("--latency-mode", action="store_true", help="with --gpus: one clip per GPU pair")
    ap.add_argument("--video-length", type=int, nargs="+", default=None, metavar="T",
                    help="measure K = 2 interpolation at each of these frames-per-segment counts (docstring)")
    ap.add_argument("--n-samples", type=int, nargs="+", default=None, metavar="N",
                    help="measure K = 2 interpolation with each of these numbers of variants (docstring); with "
                         "--pairs, the variants per pair")
    ap.add_argument("--pairs", type=int, default=None, metavar="P",
                    help="measure interpolate_pairs on P synthetic pairs over --gpus N (default 1)")
    ap.add_argument("--refine", type=float, nargs="+", default=None, metavar="S",
                    help="measure refine of a 16-frame clip at each of these strengths, against interpolate "
                         "(docstring)")
    args = ap.parse_args()
    if args.refine is not None and any(not 0.0 < x <= 1.0 for x in args.refine):
        ap.error("--refine strengths lie in (0, 1]")
    if args.pairs is not None and args.gpus is None:
        args.gpus = 1
    if args.video_length is not None:
        from tooncrafter_b200.pipeline import check_video_length
        try:
            for T in args.video_length:
                check_video_length(T)
        except ValueError as e:
            ap.error(str(e))
    from tooncrafter_b200 import synthetic
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    if not torch.cuda.is_available():
        raise SystemExit("bench_pipeline.py measures the GPU; no CUDA device found")
    dev, group = torch.device("cuda"), None
    if args.gpus is not None and args.gpus > 1:
        import torch.distributed as dist
        if int(os.environ.get("WORLD_SIZE", "1")) != args.gpus:
            raise SystemExit(f"--gpus {args.gpus}: run under torchrun --nproc-per-node {args.gpus}")
        dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
        torch.cuda.set_device(dev)
        dist.init_process_group("nccl", device_id=dev)
        group = dist.group.WORLD
    elif args.latency_mode:
        raise SystemExit("--latency-mode pairs GPUs: give --gpus N with an even N, under torchrun")
    info = gpu_info()
    print(f"GPU: {info['name']}, power limit {info['power_limit']}", flush=True)
    torch.backends.cuda.matmul.allow_tf32 = False
    size = tuple(args.size)
    decode16 = decode_ms(size) if args.animate and args.gpus is None else None   # before the model: the decoders alone
    torch.cuda.empty_cache()
    t0 = time.perf_counter()
    model = synthetic.synthetic_model(full_pipeline_config(size), dev, first_stage=args.first_stage)
    model.perframe_ae = True
    build_s = time.perf_counter() - t0
    if args.gpus is not None:
        try:
            return bench_sharded(args, model, info, build_s, group)
        finally:
            if group is not None:
                torch.distributed.destroy_process_group()
    if args.animate:
        return bench_animate(args, model, info, build_s, decode16)
    if args.video_length is not None:
        return bench_video_length(args, model, info, build_s)
    if args.n_samples is not None:
        return bench_n_samples(args, model, info, build_s)
    if args.refine is not None:
        return bench_refine(args, model, info, build_s)
    pipe = ToonCrafterPipeline(model)
    g = torch.Generator().manual_seed(0)
    results = []
    for K in (2, 5):
        kf = (torch.rand(K, size[0], size[1], 3, generator=g) * 255).to(torch.uint8)
        S = K - 1

        def batched(steps):
            return pipe.interpolate(kf, steps=steps, seed=123, size=size)

        def pairs(steps):
            return [pipe.interpolate(kf[k:k + 2], steps=steps, seed=123 + k, size=size) for k in range(S)]

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
    out = dict(metric="keyframe interpolation: seconds per video (%dx%d, DDIM-%d, CFG 7.5, eta 1, synthetic weights, "
               "%s first stage)" % (size[0], size[1], args.ddim_steps, args.first_stage), gpu=info, reps=args.reps, model_build_s=build_s, configs=results,
               note="sec_per_video = best of the timed reps, host clock around work ending in a device synchronise; "
                    "frames counts the joined video (15 * segments + 1)")
    print(json.dumps(out), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())

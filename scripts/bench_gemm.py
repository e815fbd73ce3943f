#!/usr/bin/env python
"""Per-shape timing of tc_conv_gemm, the implicit-GEMM conv / linear kernel, at the shapes of bench.py's clip.

Plans the programs of one clip on the meta device (pure host logic, as bench.py:gemm_roofline and
tests/test_engine_host_cpu.py do): the UNet forward at B = 2, 16 x 40 x 64 latents, 77 + 256 context tokens, and the
decoder at T = 16 and T = 14.  Every distinct tc_conv_gemm call (shape, tap table, epilogue, forced block_n) is
collected with its launch count per program, then one call of each is replayed on the GPU with seeded synthetic
operands of the recorded shapes and strides.  Each shape is timed with CUDA events around replays of a CUDA graph of
back-to-back launches, at least --min-ms of GPU time per shape.

    python scripts/bench_gemm.py --out DIR [--min-ms 100] [--sweep] [--top 15] [--fixed-cost [--fixed-cost-shape MxNxK]]

Reports per shape: microseconds per launch, TFLOP/s, launches per program and the (block_n, k-slices, stages) the
library chose; per program the launch-weighted GEMM time and its TFLOP/s.  --sweep also times the --top shapes by
FLOP share of a clip (50 UNet forwards + both decodes) under every legal block_n and k-slice cap.  Card name, power
limit and SM clocks (query-only nvidia-smi) are recorded with the numbers.  Writes DIR/bench_gemm.json.

Every shape whose epilogue reads a residual or a per-sample bias (bias2) is timed a second time without those operands,
at the block_n and k-slices of the recorded call, so both runs use the same tiling.  The difference is what reading
them costs; it is reported per shape ("operand_us") and summed over a clip ("epilogue_operands").

--fixed-cost measures what a tile costs besides its k-blocks, for 1x1 shapes whose tiles have only a few k-blocks: the
same M, N and epilogue timed at K = 64 .. 640, at the recorded block_n and one k-slice, fitted as
time = waves x (c0 + c1 x k-blocks).  c0 is reported in microseconds and in SM cycles at the sampled clock ("fixed_cost").
"""
from __future__ import annotations

import argparse
import json
import math
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

DDIM_STEPS = 50
H, W, T = 40, 64, 16
CTX_TOKENS = 77 + 16 * T


def plan_programs():
    """{program: [(args, kwargs) of every tc_conv_gemm call]} for one clip's programs, planned on the meta device."""
    from tiny_config import FULL_DDCONFIG, FULL_UNET
    from tooncrafter_b200 import engine, modules, ops, vae_engine
    with torch.device("meta"):
        unet = modules.UNetModel(**FULL_UNET)
        dec = modules.VideoDecoder(**FULL_DDCONFIG)
    gemms = lambda calls: [(a, kw) for fn, a, kw in calls if fn is ops.conv_gemm]
    uplan = engine.UNetEngine(unet, device="meta", plan_only=True).plan_for(2, T, H, W, CTX_TOKENS)
    deng = vae_engine.DecoderEngine(dec, device="meta", plan_only=True)
    progs = {"unet": gemms(uplan.main.calls), "unet_ctx": gemms(uplan.ctx.calls)}
    for t in (16, 14):
        dplan = deng.plan_for(t, H, W)
        progs[f"decode{t}"] = gemms(list(dplan.ctx.calls) + list(dplan.main.calls))
    return progs


# how often each program runs per clip: 50 UNet forwards (one per DDIM step, cond + uncond batched), the context
# program once per sample(), each decode once
RUNS_PER_CLIP = {"unet": DDIM_STEPS, "unet_ctx": 1, "decode16": 1, "decode14": 1}


def shape_key(a, kw):
    a_dims, taps, out_dims, n_cols = a[1], a[4], a[6], a[7]
    M = out_dims[0] * out_dims[1] * out_dims[2]
    epi = dict(geglu=bool(kw.get("geglu")), res=kw.get("res") is not None, bias2=kw.get("bias2") is not None,
               ln=kw.get("ln_stats") is not None, ln_nslots=kw.get("ln_nslots", 0),
               row_stats=kw.get("row_stats") is not None, block_n=kw.get("block_n", 0))
    return (M, n_cols, a_dims[3], len(taps), tuple(out_dims), tuple(tuple(t) for t in taps), tuple(sorted(epi.items())))


def collect(progs):
    shapes = {}
    for prog, calls in progs.items():
        for a, kw in calls:
            k = shape_key(a, kw)
            d = shapes.setdefault(k, dict(call=(a, kw), launches={p: 0 for p in progs}))
            d["launches"][prog] += 1
    for k, d in shapes.items():
        M, N, C, taps = k[:4]
        d["flop"] = 2.0 * M * N * taps * C
        d["clip_flop"] = d["flop"] * sum(n * RUNS_PER_CLIP[p] for p, n in d["launches"].items())
    return shapes


def materialize(call, dev, seed):
    """The recorded call with every meta tensor replaced by a seeded device tensor of the same dtype, shape and strides
    (a tensor that appears twice in the call stays one tensor)."""
    a, kw = call
    g = torch.Generator(device=dev).manual_seed(seed)
    real = {}

    def conv(x):
        if not isinstance(x, torch.Tensor):
            return x
        if id(x) not in real:
            n = 1 + sum((s - 1) * st for s, st in zip(x.shape, x.stride()))
            buf = torch.zeros(n, dtype=x.dtype, device=dev)
            if x.dtype.is_floating_point:
                buf.copy_(torch.randn(n, generator=g, device=dev) * 0.25)
            real[id(x)] = buf.as_strided(x.shape, x.stride())
        return real[id(x)]

    return [conv(x) for x in a], {k: conv(v) for k, v in kw.items()}


def time_call(fn, min_ms):
    """(us per launch, launches timed): CUDA events around replays of a graph of back-to-back launches."""
    ev = lambda: torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = ev(), ev()
    e0.record()
    for _ in range(5):
        fn()
    e1.record()
    torch.cuda.synchronize()
    est_ms = max(e0.elapsed_time(e1) / 5, 1e-3)
    inner = max(1, min(64, math.ceil(min_ms / 4 / est_ms)))
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
        with torch.cuda.graph(graph, stream=side):
            for _ in range(inner):
                fn()
    torch.cuda.current_stream().wait_stream(side)
    graph.replay()
    torch.cuda.synchronize()
    replays = max(2, math.ceil(min_ms / (inner * est_ms)))
    e0.record()
    for _ in range(replays):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    n = replays * inner
    return 1e3 * e0.elapsed_time(e1) / n, n


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # noqa: BLE001 - the measurement stands without it, but say why it is missing
        return dict(name=torch.cuda.get_device_name(), error=f"nvidia-smi unavailable ({type(e).__name__})")


class ClockSampler:
    """SM clock under load: query-only nvidia-smi sampling while the shapes run (median of the samples)."""

    def __init__(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits",
                                          "-lms", "500", "-i", "0"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                                         text=True)
        except OSError as e:
            self.proc, self.error = None, f"nvidia-smi unavailable ({type(e).__name__})"

    def stop(self):
        if self.proc is None:
            return dict(sm_mhz_median=None, error=self.error)
        self.proc.terminate()
        out, _ = self.proc.communicate(timeout=30)
        mhz = sorted(float(x) for x in out.split() if x.replace(".", "", 1).isdigit())
        return dict(sm_mhz_median=mhz[len(mhz) // 2] if mhz else None, sm_mhz_min=mhz[0] if mhz else None,
                    samples=len(mhz))


def describe(k, d):
    M, N, C, taps, out_dims, _, epi = k
    return dict(M=M, N=N, K=C * taps, C=C, taps=taps, out_dims=list(out_dims), epilogue=dict(epi),
                gflop=round(d["flop"] / 1e9, 3), launches=d["launches"])


def sweep_options(kw, n_cols):
    """(block_n, k-slice cap) pairs to try: block_n is free only where the call does not fix it (GEGLU and row-statistics
    calls pack / index by their block_n); k-slices only for epilogues that can split."""
    if kw.get("block_n", 0):
        bns = [kw["block_n"]]
    else:
        n16 = -(-n_cols // 16) * 16
        bns = sorted({bn for bn in range(64, 257, 32) if n_cols % bn == 0} | ({n16} if n16 <= 256 else set()))
    splittable = not (kw.get("geglu") or kw.get("ln_stats") is not None or kw.get("row_stats") is not None)
    caps = [1, 2, 3, 4] if splittable else [1]
    return [(bn, cap) for bn in bns for cap in caps]


def m_tiles(out_dims):
    """Output tiles along M: the (TW, TH, TN) box of <= 128 output pixels with the fewest tiles (tc_conv_gemm's search)."""
    N, H, W = out_dims
    best = None
    for tw in range(1, min(W, 128) + 1):
        for th in range(1, min(128 // tw, H) + 1):
            tn = min(128 // (tw * th), N)
            t = -(-W // tw) * -(-H // th) * -(-N // tn)
            best = t if best is None else min(best, t)
    return best


def fixed_cost(call, block_n, dev, seed, min_ms, kblocks=range(1, 11)):
    """Fixed per-tile cost of one 1x1 (linear) shape: the same M, N and epilogue at K = 64 k, k = kblocks, one k-slice,
    the given block_n; least-squares fit of  time = waves x (c0 + c1 k)  (waves = tiles / SMs, rounded up).  c0 is
    what a tile costs besides its k-blocks: launch share, pipeline fill, epilogue and output stores."""
    import numpy as np
    from tooncrafter_b200 import _lib, ops
    lib = _lib.load()
    a, kw = materialize(call, dev, seed)
    a_dims, out_dims, n_cols, w = a[1], a[6], a[7], a[3]
    g = torch.Generator(device=dev).manual_seed(seed)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    tiles = m_tiles(out_dims) * -(-n_cols // block_n)
    waves = -(-tiles // sms)
    pts = []
    lib.tc_debug_set_gemm_mode(1 << 8)                 # one k-slice
    try:
        for k in kblocks:
            C = 64 * k
            N, H, W = a_dims[0], a_dims[1], a_dims[2]
            x = torch.randn(N * H * W * C, generator=g, device=dev).mul_(0.25).half()
            wk = torch.randn(w.shape[0], C, generator=g, device=dev).mul_(C ** -0.5).half()
            args = (x, (N, H, W, C), (H * W * C, W * C, C), wk) + tuple(a[4:])
            kwk = dict(kw, block_n=block_n, a_offset=0)
            fn = lambda: ops.conv_gemm(*args, **kwk)
            us, _ = time_call(fn, min_ms)
            cfg = ops.last_gemm_config()
            assert (cfg["block_n"], cfg["ksplit"]) == (block_n, 1), cfg
            pts.append(dict(kblocks=k, us=round(us, 2)))
            del x, wk
    finally:
        lib.tc_debug_set_gemm_mode(0)
    ks = np.array([p["kblocks"] for p in pts], dtype=np.float64)
    per_wave = np.array([p["us"] for p in pts]) / waves
    c1, c0 = np.polyfit(ks, per_wave, 1)
    resid = per_wave - (c0 + c1 * ks)
    return dict(block_n=block_n, tiles=tiles, waves=waves, points=pts, c0_us=round(float(c0), 3),
                c1_us_per_kblock=round(float(c1), 3), fit_rms_us=round(float(np.sqrt((resid ** 2).mean())), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory (bench_gemm.json)")
    ap.add_argument("--min-ms", type=float, default=100.0, help="GPU time per timed shape (and per sweep point)")
    ap.add_argument("--sweep", action="store_true", help="also time the --top shapes under every block_n / k-slice cap")
    ap.add_argument("--top", type=int, default=15)
    ap.add_argument("--fixed-cost", action="store_true",
                    help="also fit the fixed per-tile cost c0 of the clip's 1x1 GEGLU shapes with K <= 640 and of every "
                         "--fixed-cost-shape (K = 64 .. 640, the recorded block_n, one k-slice)")
    ap.add_argument("--fixed-cost-shape", action="append", default=None, metavar="MxNxK",
                    help="1x1 shape for --fixed-cost (repeatable; default 81920x960x320)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm.py measures the GPU; no CUDA device found")
    from tooncrafter_b200 import _lib, ops
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    t0 = time.perf_counter()
    progs = plan_programs()
    shapes = collect(progs)
    plan_s = time.perf_counter() - t0
    clip_flop = sum(d["clip_flop"] for d in shapes.values())
    order = sorted(shapes, key=lambda k: -shapes[k]["clip_flop"])
    info = gpu_info()
    print(f"GPU: {info.get('name')}, power limit {info.get('power.limit')}; {len(shapes)} distinct shapes", flush=True)
    clocks = ClockSampler()
    rows = []
    try:
        for i, k in enumerate(order):
            d = shapes[k]
            a, kw = materialize(d["call"], dev, seed=i)
            fn = lambda: ops.conv_gemm(*a, **kw)
            lib.tc_debug_set_gemm_mode(0)
            us, n = time_call(fn, args.min_ms)
            cfg = ops.last_gemm_config()
            row = describe(k, d)
            row.update(rank=i, clip_flop_share=round(d["clip_flop"] / clip_flop, 4), us=round(us, 2),
                       tflops=round(d["flop"] / us / 1e6, 1), timed_launches=n,
                       config=dict(block_n=cfg["block_n"], ksplit=cfg["ksplit"], stages=cfg["stages"]))
            if kw.get("res") is not None or kw.get("bias2") is not None:
                # same tiling, no residual / bias2: block_n forced, k-slices capped at the recorded count
                lib.tc_debug_set_gemm_mode(cfg["ksplit"] << 8)
                kw0 = dict(kw, block_n=cfg["block_n"], res=None, bias2=None)
                fn0 = lambda: ops.conv_gemm(*a, **kw0)
                us0, _ = time_call(fn0, args.min_ms)
                c0 = ops.last_gemm_config()
                lib.tc_debug_set_gemm_mode(0)
                assert (c0["block_n"], c0["ksplit"]) == (cfg["block_n"], cfg["ksplit"]), (c0, cfg)
                row.update(us_without_operands=round(us0, 2), operand_us=round(us - us0, 2),
                           config_without_operands=dict(block_n=c0["block_n"], ksplit=c0["ksplit"], stages=c0["stages"]))
            if args.sweep and i < args.top:
                pts = []
                for bn, cap in sweep_options(kw, k[1]):
                    lib.tc_debug_set_gemm_mode(cap << 8)
                    kw2 = dict(kw, block_n=bn)
                    fn2 = lambda: ops.conv_gemm(*a, **kw2)
                    us2, _ = time_call(fn2, args.min_ms / 2)
                    c2 = ops.last_gemm_config()
                    pts.append(dict(block_n=c2["block_n"], ksplit=c2["ksplit"], stages=c2["stages"], cap=cap,
                                    us=round(us2, 2)))
                lib.tc_debug_set_gemm_mode(0)
                best = min(p["us"] for p in pts)
                row["sweep"] = pts
                row["chosen_over_best"] = round(us / best, 3)
            rows.append(row)
            print(json.dumps({x: row[x] for x in ("rank", "M", "N", "K", "taps", "us", "tflops", "config")}
                             | {x: row[x] for x in ("operand_us", "config_without_operands") if x in row}
                             | ({"chosen_over_best": row["chosen_over_best"]} if "sweep" in row else {})), flush=True)
            del a, kw
            torch.cuda.empty_cache()
        if args.fixed_cost:
            extra = {tuple(int(v) for v in x.split("x")) for x in (args.fixed_cost_shape or ["81920x960x320"])}
            for r in rows:
                k = order[r["rank"]]
                if r["taps"] != 1 or not (r["epilogue"]["geglu"] and r["K"] <= 640 or (r["M"], r["N"], r["K"]) in extra):
                    continue
                r["fixed_cost"] = fixed_cost(shapes[k]["call"], r["config"]["block_n"], dev, r["rank"], args.min_ms / 2)
                print(json.dumps({x: r[x] for x in ("rank", "M", "N", "K", "us")} | {"fixed_cost": r["fixed_cost"]}),
                      flush=True)
                torch.cuda.empty_cache()
    finally:
        lib.tc_debug_set_gemm_mode(0)
        clk = clocks.stop()
    programs = {}
    for p in progs:
        ms = sum(r["us"] * r["launches"][p] for r in rows) / 1e3
        fl = sum(shapes[k]["flop"] * shapes[k]["launches"][p] for k in order)
        programs[p] = dict(launches=len(progs[p]), gemm_ms=round(ms, 3), tflop=round(fl / 1e12, 3),
                           tflops=round(fl / ms / 1e9, 1) if ms else None)
    clip_ms = sum(programs[p]["gemm_ms"] * RUNS_PER_CLIP[p] for p in programs)
    clip_launches = lambda r: sum(n * RUNS_PER_CLIP[p] for p, n in r["launches"].items())
    abl = [r for r in rows if "operand_us" in r]
    op_ms = sum(r["operand_us"] * clip_launches(r) for r in abl) / 1e3
    epi_ops = dict(shapes=len(abl), clip_launches=sum(clip_launches(r) for r in abl),
                   clip_ms_with=round(sum(r["us"] * clip_launches(r) for r in abl) / 1e3, 1),
                   clip_ms_without=round(sum(r["us_without_operands"] * clip_launches(r) for r in abl) / 1e3, 1),
                   clip_operand_ms=round(op_ms, 1), share_of_clip_gemm=round(op_ms / clip_ms, 4) if clip_ms else None)
    out = dict(metric="tc_conv_gemm per-shape time at the shapes of one clip (synthetic fp16 operands, CUDA graph of "
                      "back-to-back launches, CUDA events)",
               gpu=info, clocks_during_run=clk, min_ms_per_shape=args.min_ms, plan_s=round(plan_s, 1),
               programs=programs, runs_per_clip=RUNS_PER_CLIP,
               clip=dict(gemm_ms=round(clip_ms, 1), tflop=round(clip_flop / 1e12, 1),
                         tflops=round(clip_flop / clip_ms / 1e9, 1)),
               epilogue_operands=epi_ops, shapes=rows)
    fits = [r for r in rows if "fixed_cost" in r]
    if fits:
        mhz = clk.get("sm_mhz_median")
        out["fixed_cost"] = [dict(M=r["M"], N=r["N"], K=r["K"], epilogue=r["epilogue"], us=r["us"],
                                  c0_us=r["fixed_cost"]["c0_us"], c1_us_per_kblock=r["fixed_cost"]["c1_us_per_kblock"],
                                  c0_sm_cycles=round(r["fixed_cost"]["c0_us"] * mhz) if mhz else None,
                                  block_n=r["fixed_cost"]["block_n"], waves=r["fixed_cost"]["waves"]) for r in fits]
    od = Path(args.out)
    od.mkdir(parents=True, exist_ok=True)
    (od / "bench_gemm.json").write_text(json.dumps(out, indent=1))
    print(json.dumps(dict(gpu=info, clocks_during_run=clk, programs=programs, clip=out["clip"],
                           epilogue_operands=epi_ops) | ({"fixed_cost": out["fixed_cost"]} if fits else {})), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())

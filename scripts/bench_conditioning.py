"""Time the conditioning stage of one clip at the shapes image_guided_synthesis uses (reference
scripts/evaluation/inference.py:186-214), ViT-H-14 encoders and the Resampler of configs/inference_512_v1.0.yaml with
seeded synthetic weights:
  text encode   B = 2 (prompt token ids and the empty prompt), "penultimate" layer
  image encode  B = 2 (a 320 x 512 frame and its zero image), preprocessing included
  Resampler     B = 2 (257 CLIP image tokens each)
Each is timed warm with CUDA events on this library's engines and on the fp32 oracle under torch.autocast(fp16) with
SDPA attention (what the reference runs), on the same GPU.  Prints one JSON line with the device name, power limit and
SM clock read in the same run.

    python scripts/bench_conditioning.py [--iters 20] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import clip_oracle, resampler_oracle  # noqa: E402
from tooncrafter_b200 import modules, synthetic  # noqa: E402

RESAMPLER = dict(dim=1024, depth=4, dim_head=64, heads=12, num_queries=16, embedding_dim=1280, output_dim=1024,
                 ff_mult=4, video_length=16)            # configs/inference_512_v1.0.yaml: image_proj_stage_config


def _gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, sm, smax = [s.strip() for s in out.split(",")]
        return dict(gpu=name, power_limit=plim, sm_clock=sm, sm_clock_max=smax)
    except Exception as e:  # the timing does not depend on it; say why it is missing
        return dict(gpu=torch.cuda.get_device_name(0), power_limit=f"unavailable ({e})")


def _time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_conditioning.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.backends.cuda.matmul.allow_tf32 = False

    text = modules.FrozenOpenCLIPEmbedder(layer="penultimate")
    synthetic.fill_module_(text, seed=0, prefix="cond_stage_model.")
    image = modules.FrozenOpenCLIPImageEmbedderV2()
    synthetic.fill_module_(image, seed=0, prefix="embedder.")
    rs = modules.Resampler(**RESAMPLER).eval()
    synthetic.fill_module_(rs, seed=0, prefix="image_proj_model.")
    text, image, rs = text.to(dev), image.to(dev), rs.to(dev)

    tokens = modules.clip_tokenize(["", ""])
    tokens[0, 1:12] = torch.randint(1, 49400, (11,), generator=synthetic._gen("bench.prompt", 0))
    tokens[0, 12] = modules.CLIP_EOT                        # an 11-token prompt, then the empty prompt
    tokens = tokens.to(dev)
    frame = torch.rand(1, 3, 320, 512, generator=synthetic._gen("bench.frame", 0)) * 2 - 1
    imgs = torch.cat([frame, torch.zeros_like(frame)]).to(dev)
    clip_tok = torch.randn(2, 257, 1280, generator=synthetic._gen("bench.tokens", 0)).to(dev)
    sd_t, sd_i, sd_r = text.state_dict(), image.state_dict(), rs.state_dict()

    def ac(fn):
        def run():
            with torch.autocast("cuda", dtype=torch.float16):
                fn()
        return run

    res = {}
    with torch.no_grad():
        res["text_ms"] = _time_ms(lambda: text(tokens), args.iters, args.warmup)
        res["image_ms"] = _time_ms(lambda: image(imgs), args.iters, args.warmup)
        res["resampler_ms"] = _time_ms(lambda: rs(clip_tok), args.iters, args.warmup)
        res["text_autocast_oracle_ms"] = _time_ms(ac(lambda: clip_oracle.encode_text(sd_t, tokens, 16, 1, "model.")),
                                                  args.iters, args.warmup)
        res["image_autocast_oracle_ms"] = _time_ms(
            ac(lambda: clip_oracle.encode_image(sd_i, modules.clip_preprocess(imgs), 16, "model.")), args.iters,
            args.warmup)
        res["resampler_autocast_oracle_ms"] = _time_ms(
            ac(lambda: resampler_oracle.resampler_forward(sd_r, clip_tok, heads=RESAMPLER["heads"])), args.iters,
            args.warmup)
    res["total_ms"] = res["text_ms"] + res["image_ms"] + res["resampler_ms"]
    res["total_autocast_oracle_ms"] = (res["text_autocast_oracle_ms"] + res["image_autocast_oracle_ms"]
                                       + res["resampler_autocast_oracle_ms"])
    out = dict(metric="conditioning_stage", B=2, iters=args.iters, **{k: round(v, 3) for k, v in res.items()})
    out.update(_gpu_info())
    print(json.dumps(out))


if __name__ == "__main__":
    main()

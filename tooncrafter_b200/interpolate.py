"""Command line: keyframe PNGs -> one interpolated video, on the CUDA library (tooncrafter_b200.pipeline).

    python -m tooncrafter_b200.interpolate --config configs/inference_512_v1.0.yaml --ckpt model.ckpt \
        --frames a.png b.png c.png --prompt "an anime scene" --out results/storyboard

With a single --frames image the image is animated instead (ToonCrafterPipeline.animate, image-to-video):

    python -m tooncrafter_b200.interpolate --config configs/training_1024_v1.0/config.yaml --ckpt model.ckpt \
        --frames still.png --height 576 --width 1024 --out results/clip

Writes DIR/frame_%04d.png, DIR/video.npy (uint8 [F, H, W, 3]) and, when OpenCV can open an mp4 writer,
DIR/video.mp4.  The sampling defaults are those of the reference's scripts/run.sh.  --video-length T sets the frames
of each segment (the reference's --video_length; any even T from 4 to 64, default the config's temporal_length):

    python -m tooncrafter_b200.interpolate --config ... --frames a.png b.png --video-length 32 --out results/long

Under torchrun (WORLD_SIZE > 1) every process drives the GPU LOCAL_RANK over NCCL, builds the model (the checkpoint,
or the same synthetic seed) and the segments are sharded over the processes (ToonCrafterPipeline's `group`);
--latency-mode shards them over GPU pairs instead, one guidance branch per GPU.  Rank 0 writes the outputs:

    torchrun --nproc-per-node 8 -m tooncrafter_b200.interpolate --config ... --frames a.png b.png c.png --out DIR

The config is the reference-style YAML (read with PyYAML; only its `model:` section is used, so the training
configs, whose first stage is the plain AutoencoderKL, work as well).  Its two OpenCLIP conditioning targets
(lvdm.modules.encoders.condition.FrozenOpenCLIP*) are pointed at this repository's classes unless
--keep-config-targets is given.  --synthetic-weights replaces the checkpoint by seeded synthetic weights (smoke runs).
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import torch

OPENCLIP_TARGETS = {
    "lvdm.modules.encoders.condition.FrozenOpenCLIPEmbedder": "tooncrafter_b200.modules.FrozenOpenCLIPEmbedder",
    "lvdm.modules.encoders.condition.FrozenOpenCLIPImageEmbedderV2":
        "tooncrafter_b200.modules.FrozenOpenCLIPImageEmbedderV2",
}


def get_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m tooncrafter_b200.interpolate", description=__doc__.split("\n\n")[0])
    ap.add_argument("--config", required=True, help="reference-style model YAML (configs/inference_512_v1.0.yaml)")
    ap.add_argument("--ckpt", default=None, help="checkpoint with a state_dict (loaded strictly)")
    ap.add_argument("--synthetic-weights", action="store_true", help="seeded synthetic weights instead of --ckpt")
    ap.add_argument("--keep-config-targets", action="store_true",
                    help="keep the YAML's OpenCLIP targets instead of this repository's classes")
    ap.add_argument("--frames", nargs="+", required=True,
                    help="K >= 2 keyframe images, in order; one image: animate it")
    ap.add_argument("--prompt", default="", help="prompt of every segment")
    ap.add_argument("--prompts-file", default=None, help="one prompt per segment, one per non-empty line")
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--height", type=int, default=320)
    ap.add_argument("--width", type=int, default=512)
    ap.add_argument("--ddim-steps", type=int, default=50)
    ap.add_argument("--ddim-eta", type=float, default=1.0)
    ap.add_argument("--cfg-scale", type=float, default=7.5, help="classifier-free guidance scale")
    ap.add_argument("--cfg-img", type=float, default=None, help="image guidance scale (three-way guidance)")
    ap.add_argument("--frame-stride", type=int, default=10, help="fs conditioning (smaller: larger motion)")
    ap.add_argument("--guidance-rescale", type=float, default=0.7)
    ap.add_argument("--timestep-spacing", default="uniform_trailing")
    ap.add_argument("--segments-per-batch", type=int, default=None,
                    help="segments sampled together (default: 4 at 320x512, 1 at 576x1024)")
    ap.add_argument("--video-length", type=int, default=None,
                    help="frames per segment, an even number from 4 to 64 (default: the config's temporal_length)")
    ap.add_argument("--loop", action="store_true", help="add a closing segment from the last keyframe to the first")
    ap.add_argument("--seed", type=int, default=123)
    ap.add_argument("--latency-mode", action="store_true",
                    help="under torchrun: one clip per GPU pair, one guidance branch per GPU (even world size)")
    ap.add_argument("--fps", type=int, default=8, help="frame rate of the mp4")
    return ap


def rewrite_targets(node, keep: bool = False):
    """The config with every OpenCLIP target of the reference replaced by this repository's class (unless keep)."""
    if isinstance(node, dict):
        out = {k: rewrite_targets(v, keep) for k, v in node.items()}
        if not keep and out.get("target") in OPENCLIP_TARGETS:
            out["target"] = OPENCLIP_TARGETS[out["target"]]
        return out
    if isinstance(node, list):
        return [rewrite_targets(v, keep) for v in node]
    return node


def load_model_config(path: str, keep_targets: bool = False) -> dict:
    import yaml
    with open(path) as f:
        cfg = yaml.safe_load(f)
    if "model" not in cfg:
        raise ValueError(f"{path}: no top-level `model` section")
    return rewrite_targets(cfg["model"], keep_targets)


def load_checkpoint(model, path: str) -> None:
    """load_state_dict(ckpt["state_dict"]) with strict key checking and a readable report of mismatches."""
    sd = torch.load(path, map_location="cpu", weights_only=True)
    sd = sd.get("state_dict", sd)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    if missing or unexpected:
        def show(keys):
            return "\n".join(f"    {k}" for k in keys[:20]) + (f"\n    ... {len(keys) - 20} more" if len(keys) > 20 else "")
        msg = [f"{path} does not match the model built from the config:"]
        if missing:
            msg.append(f"  {len(missing)} missing keys:\n{show(missing)}")
        if unexpected:
            msg.append(f"  {len(unexpected)} unexpected keys:\n{show(unexpected)}")
        raise RuntimeError("\n".join(msg))


def read_prompts(args, n_segments: int):
    if args.prompts_file is None:
        return args.prompt
    with open(args.prompts_file) as f:
        lines = [ln.strip() for ln in f if ln.strip()]
    if len(lines) != n_segments:
        raise SystemExit(f"{args.prompts_file}: {len(lines)} prompts for {n_segments} segments")
    return lines


def write_video(video: np.ndarray, out_dir: str, fps: int) -> None:
    from PIL import Image
    os.makedirs(out_dir, exist_ok=True)
    for i, fr in enumerate(video):
        Image.fromarray(fr).save(os.path.join(out_dir, f"frame_{i:04d}.png"))
    np.save(os.path.join(out_dir, "video.npy"), video)
    try:
        import cv2
        path = os.path.join(out_dir, "video.mp4")
        wr = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), fps, (video.shape[2], video.shape[1]))
        opened = wr.isOpened()
    except ImportError:
        opened = False
    if opened:
        for fr in video:
            wr.write(np.ascontiguousarray(fr[..., ::-1]))
        wr.release()
        print(f"wrote {path}")
    else:
        print("mp4 skipped: no OpenCV video writer could be opened")


def main(argv=None) -> int:
    ap = get_parser()
    args = ap.parse_args(argv)
    if args.video_length is not None:
        from .pipeline import check_video_length
        try:
            check_video_length(args.video_length)
        except ValueError as e:
            ap.error(str(e))
    if not args.synthetic_weights and args.ckpt is None:
        raise SystemExit("give --ckpt, or --synthetic-weights for a run without a checkpoint")
    cfg = load_model_config(args.config, args.keep_config_targets)
    if not torch.cuda.is_available():
        raise SystemExit("a CUDA device is required")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.latency_mode and world == 1:
        raise SystemExit("--latency-mode pairs GPUs: run under torchrun with an even number of processes")
    if world == 1:
        return run(args, cfg, torch.device("cuda"), None)
    import torch.distributed as dist
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    try:
        return run(args, cfg, dev, dist.group.WORLD)
    finally:
        dist.destroy_process_group()


def run(args, cfg, dev, group) -> int:
    """Build the model on `dev`, make the video (sharded over `group` when given) and write it from rank 0."""
    from PIL import Image

    from . import diffusion, synthetic
    from .pipeline import ToonCrafterPipeline
    if args.synthetic_weights:
        model = synthetic.synthetic_model(cfg, dev, seed=0)
    else:
        model = diffusion.instantiate_from_config(cfg)
        load_checkpoint(model, args.ckpt)
        model = model.to(dev).eval()
    model.perframe_ae = True
    frames = [np.asarray(Image.open(p).convert("RGB")) for p in args.frames]
    pipe = ToonCrafterPipeline(model, group, latency=args.latency_mode)
    common = dict(steps=args.ddim_steps, cfg_scale=args.cfg_scale, eta=args.ddim_eta, fs=args.frame_stride,
                  guidance_rescale=args.guidance_rescale, timestep_spacing=args.timestep_spacing, cfg_img=args.cfg_img,
                  seed=args.seed, size=(args.height, args.width), video_length=args.video_length)
    if len(frames) == 1:
        if args.loop:
            raise SystemExit("--loop needs at least two keyframes")
        video = pipe.animate(frames[0], prompt=read_prompts(args, 1), **common)
    else:
        n_seg = len(frames) if args.loop else len(frames) - 1
        video = pipe.interpolate(frames, prompts=read_prompts(args, n_seg), loop=args.loop,
                                 segments_per_batch=args.segments_per_batch, **common)
    if group is not None and torch.distributed.get_rank() != 0:
        return 0
    v = video.cpu().numpy()
    write_video(v, args.out, args.fps)
    print(f"{len(frames)} {'image' if len(frames) == 1 else 'keyframes'} -> {v.shape[0]} frames of "
          f"{v.shape[1]}x{v.shape[2]} in {args.out}")
    return 0


if __name__ == "__main__":
    sys.exit(main())

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

--n-samples N makes N variants (the reference's --n_samples; ToonCrafterPipeline's n_samples) and writes variant v to
DIR/sample{v}/.  --prompt-dir SRC instead of --frames runs a directory of independent keyframe pairs as the
reference's --prompt_dir with --interp does (read_prompt_dir): pair i is the sorted images 2i and 2i+1 with line i of
the directory's first .txt file (or "" without --text-input), and variant v of pair i goes to
DIR/<name of image 2i>_sample{v}/ (ToonCrafterPipeline.interpolate_pairs, pair i seeded seed + i):

    python -m tooncrafter_b200.interpolate --config ... --ckpt ... --prompt-dir prompts/512_interp --n-samples 4 \
        --out results/

--init-video SRC instead refines an existing clip (ToonCrafterPipeline.refine): SRC is a directory of frame images, a
uint8 [T, H, W, 3] .npy (what this command writes) or a video file OpenCV can read.  --strength S (required) re-runs
int(S * steps) DDIM steps from the clip's latents; --keep-frames 0-3,12-15 holds those frames to the clip and
regenerates the ones between:

    python -m tooncrafter_b200.interpolate --config ... --ckpt ... --init-video out/video.npy --strength 0.5 \
        --keep-frames 0-1,14-15 --out results/refined

The config is the reference-style YAML (read with PyYAML; only its `model:` section is used, so the training
configs, whose first stage is the plain AutoencoderKL, work as well).  Its two OpenCLIP conditioning targets
(lvdm.modules.encoders.condition.FrozenOpenCLIP*) are pointed at this repository's classes unless
--keep-config-targets is given.  --synthetic-weights replaces the checkpoint by seeded synthetic weights (smoke runs).
"""
from __future__ import annotations

import argparse
import glob
import os
import re
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
    src = ap.add_mutually_exclusive_group()        # one of them is required: main() checks
    src.add_argument("--frames", nargs="+", help="K >= 2 keyframe images, in order; one image: animate it")
    src.add_argument("--prompt-dir", default=None,
                     help="a directory of keyframe pairs and a prompt file, laid out as the reference's --prompt_dir")
    src.add_argument("--init-video", default=None,
                     help="refine this clip (ToonCrafterPipeline.refine): a directory of frame images, a uint8 "
                          "[T, H, W, 3] .npy, or a video file OpenCV can read")
    ap.add_argument("--strength", type=float, default=None,
                    help="with --init-video (required there): share of the DDIM steps re-run, in (0, 1]")
    ap.add_argument("--keep-frames", default=None,
                    help="with --init-video: frames held to the clip, e.g. 0-3,12-15 (the frames between are "
                         "regenerated)")
    ap.add_argument("--text-input", action="store_true",
                    help="with --prompt-dir: pair i gets line i of the prompt file (default: every pair gets \"\")")
    ap.add_argument("--n-samples", type=int, default=None,
                    help="variants per video, written to OUT/sample{v}/ (OUT/<name>_sample{v}/ with --prompt-dir)")
    ap.add_argument("--pairs-per-batch", type=int, default=None,
                    help="with --prompt-dir: pairs sampled together (default: as many as the rows budget allows)")
    ap.add_argument("--prompt", default="", help="prompt of every segment")
    ap.add_argument("--prompts-file", default=None, help="one prompt per segment, one per non-empty line")
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--height", type=int, default=320)
    ap.add_argument("--width", type=int, default=512)
    ap.add_argument("--ddim-steps", type=int, default=50)
    ap.add_argument("--ddim-eta", type=float, default=1.0)
    ap.add_argument("--sampler", default="ddim",
                    help="ddim (the reference's sampler) or dpmpp_2m (DPM-Solver++(2M), --ddim-eta 0 or 1)")
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


IMAGE_SUFFIXES = ("jpg", "png", "jpeg", "JPEG", "PNG")


def _filelist(data_dir: str, postfixes) -> list:
    """get_filelist (inference.py:19-25): the files matching each `*.{postfix}`, collected and then sorted."""
    files = []
    for postfix in postfixes:
        files.extend(glob.glob(os.path.join(data_dir, f"*.{postfix}")))
    files.sort()
    return files


def read_prompt_dir(data_dir: str, text_input: bool = False):
    """A --prompt_dir of the reference for interpolation (load_data_prompts with interp, inference.py:54-106).

    Prompts: the non-empty stripped lines of the first `.txt` file by name; P = their number.  Images: the files
    `*.jpg|png|jpeg|JPEG|PNG`, sorted as get_filelist sorts them; pair i is images 2i and 2i+1.  A pair's prompt is its
    line with text_input and "" without (inference.py:186-187).  Its output name is image 2i's file name up to the
    first dot, as save_results_seperate names `<name>_sample{v}.mp4`.  Returns ([(image a, image b)], prompts, names);
    ValueError for a missing directory or prompt file, no prompts, or fewer than 2P images."""
    if not os.path.isdir(data_dir):
        raise ValueError(f"{data_dir}: not a directory")
    txt = _filelist(data_dir, ["txt"])
    if not txt:
        raise ValueError(f"{data_dir}: no prompt file (*.txt)")
    with open(txt[0]) as f:
        lines = [ln.strip() for ln in f if ln.strip()]
    if not lines:
        raise ValueError(f"{txt[0]}: no prompts")
    images = _filelist(data_dir, IMAGE_SUFFIXES)
    P = len(lines)
    if len(images) < 2 * P:
        raise ValueError(f"{data_dir}: {len(images)} images for {P} prompts; pair i is images 2i and 2i+1, so "
                         f"{2 * P} are needed")
    pairs = [(images[2 * i], images[2 * i + 1]) for i in range(P)]
    names = [os.path.basename(a).split(".")[0] for a, _ in pairs]
    return pairs, (lines if text_input else [""] * P), names


def read_init_video(path: str) -> np.ndarray:
    """The clip of --init-video as uint8 [T, H, W, 3] RGB: a directory of images (sorted as get_filelist sorts them,
    what write_video writes as frame_%04d.png), a .npy array (write_video's video.npy), or any other file through
    OpenCV's VideoCapture.  ValueError for a missing or unreadable source, or frames of different sizes."""
    if os.path.isdir(path):
        from PIL import Image
        files = _filelist(path, IMAGE_SUFFIXES)
        if not files:
            raise ValueError(f"{path}: no images (*.{'|'.join(IMAGE_SUFFIXES)})")
        frames = [np.asarray(Image.open(f).convert("RGB")) for f in files]
        if len({f.shape for f in frames}) != 1:
            raise ValueError(f"{path}: the images differ in size")
        return np.stack(frames)
    if not os.path.isfile(path):
        raise ValueError(f"{path}: no such file or directory")
    if path.endswith(".npy"):
        v = np.load(path)
        if v.dtype != np.uint8 or v.ndim != 4 or v.shape[-1] != 3:
            raise ValueError(f"{path}: expected a uint8 [T, H, W, 3] array, got {v.dtype} {v.shape}")
        return v
    try:
        import cv2
    except ImportError:
        raise ValueError(f"{path}: reading a video file needs OpenCV (cv2)") from None
    cap = cv2.VideoCapture(path)
    frames = []
    while cap.isOpened():
        ok, fr = cap.read()
        if not ok:
            break
        frames.append(np.ascontiguousarray(fr[..., ::-1]))
    cap.release()
    if not frames:
        raise ValueError(f"{path}: OpenCV read no frames")
    return np.stack(frames)


def parse_frame_ranges(spec: str, T: int) -> list:
    """--keep-frames: comma-separated frame indices and inclusive ranges a-b ("0-3,12-15"), each within 0 .. T-1 and
    listed once (ToonCrafterPipeline.refine's keep, sorted).  ValueError otherwise."""
    from .pipeline import check_keep
    out = []
    for part in spec.split(","):
        part = part.strip()
        if not re.fullmatch(r"\d+(-\d+)?", part):
            raise ValueError(f"--keep-frames: {part!r} is not a frame index or a range a-b")
        a, _, b = part.partition("-")
        if int(a) > int(b or a):
            raise ValueError(f"--keep-frames: {part!r} is not a range a-b with a <= b")
        out.extend(range(int(a), int(b or a) + 1))
    return check_keep(out, T)


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
    if args.frames is None and args.prompt_dir is None and args.init_video is None:
        ap.error("one of the arguments --frames --prompt-dir is required (or --init-video to refine a clip)")
    from .pipeline import check_count, check_n_samples, check_strength, check_video_length
    from .sampler import check_sampler
    try:
        check_sampler(args.sampler, args.ddim_eta)
        if args.video_length is not None:
            check_video_length(args.video_length)
        if args.n_samples is not None:
            check_n_samples(args.n_samples)
        for name in ("segments_per_batch", "pairs_per_batch"):
            if getattr(args, name) is not None:
                check_count(getattr(args, name), name)
    except ValueError as e:
        ap.error(str(e))
    if args.prompt_dir is not None:
        if args.loop:
            ap.error("--loop does not apply to --prompt-dir")
        if args.prompt or args.prompts_file:
            ap.error("--prompt-dir reads its prompts from the directory's .txt file (--prompt / --prompts-file)")
        try:
            read_prompt_dir(args.prompt_dir, args.text_input)
        except ValueError as e:
            ap.error(str(e))
    elif args.text_input or args.pairs_per_batch is not None:
        ap.error("--text-input and --pairs-per-batch apply to --prompt-dir")
    args.clip = args.keep = None
    if args.init_video is not None:
        if args.strength is None:
            ap.error("--init-video needs --strength")
        if args.loop:
            ap.error("--loop does not apply to --init-video")
        try:
            args.clip = read_init_video(args.init_video)
            T = check_video_length(len(args.clip))
            if args.video_length is not None and args.video_length != T:
                raise ValueError(f"--video-length {args.video_length}: the clip has {T} frames")
            check_strength(args.strength, args.ddim_steps)
            if args.keep_frames is not None:
                args.keep = parse_frame_ranges(args.keep_frames, T)
        except ValueError as e:
            ap.error(str(e))
    elif args.strength is not None or args.keep_frames is not None:
        ap.error("--strength and --keep-frames apply to --init-video")
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
    pipe = ToonCrafterPipeline(model, group, latency=args.latency_mode)
    common = dict(steps=args.ddim_steps, cfg_scale=args.cfg_scale, eta=args.ddim_eta, fs=args.frame_stride,
                  guidance_rescale=args.guidance_rescale, timestep_spacing=args.timestep_spacing, cfg_img=args.cfg_img,
                  size=(args.height, args.width), video_length=args.video_length, sampler=args.sampler)
    writes = group is None or torch.distributed.get_rank() == 0
    if args.prompt_dir is not None:
        return run_prompt_dir(args, pipe, common, group, writes)
    if args.clip is not None:
        common.pop("video_length")
        video = pipe.refine(args.clip, args.strength, prompt=read_prompts(args, 1), keep=args.keep, seed=args.seed,
                            n_samples=args.n_samples, segments_per_batch=args.segments_per_batch, **common)
        frames = args.clip
    elif len(args.frames) == 1:
        frames = [np.asarray(Image.open(args.frames[0]).convert("RGB"))]
        if args.loop:
            raise SystemExit("--loop needs at least two keyframes")
        video = pipe.animate(frames[0], prompt=read_prompts(args, 1), seed=args.seed, n_samples=args.n_samples,
                             **common)
    else:
        frames = [np.asarray(Image.open(p).convert("RGB")) for p in args.frames]
        n_seg = len(frames) if args.loop else len(frames) - 1
        video = pipe.interpolate(frames, prompts=read_prompts(args, n_seg), loop=args.loop, seed=args.seed,
                                 segments_per_batch=args.segments_per_batch, n_samples=args.n_samples, **common)
    if not writes:
        return 0
    v = video.cpu().numpy()
    if args.n_samples is None:
        write_video(v, args.out, args.fps)
    else:
        for i, variant in enumerate(v):
            write_video(variant, os.path.join(args.out, f"sample{i}"), args.fps)
    what = "frames refined" if args.clip is not None else ("image" if len(frames) == 1 else "keyframes")
    print(f"{len(frames)} {what} -> "
          f"{'' if args.n_samples is None else f'{v.shape[0]} x '}{v.shape[-4]} frames of {v.shape[-3]}x{v.shape[-2]} "
          f"in {args.out}")
    return 0


def run_prompt_dir(args, pipe, common, group, writes: bool) -> int:
    """--prompt-dir: the directory's pairs through interpolate_pairs in chunks of (blocks x pairs per batch) pairs,
    each chunk written before the next is read, so host and device memory hold one chunk; pair i is seeded seed + i
    whatever chunk holds it.  Every pair runs (the reference drops the P % ranks pairs left over)."""
    from PIL import Image

    from .pipeline import check_video_length, default_pairs_per_batch
    pairs, prompts, names = read_prompt_dir(args.prompt_dir, args.text_input)
    n = 1 if args.n_samples is None else args.n_samples
    T = check_video_length(pipe.model.temporal_length if args.video_length is None else args.video_length)
    per_batch = args.pairs_per_batch or default_pairs_per_batch(common["size"], T, n)
    blocks = 1 if group is None else torch.distributed.get_world_size(group) // (2 if args.latency_mode else 1)
    chunk = blocks * per_batch
    for c0 in range(0, len(pairs), chunk):
        idx = range(c0, min(c0 + chunk, len(pairs)))
        images = [[np.asarray(Image.open(p).convert("RGB")) for p in pairs[i]] for i in idx]
        video = pipe.interpolate_pairs(images, prompts=[prompts[i] for i in idx], n_samples=n, seed=args.seed + c0,
                                       pairs_per_batch=per_batch, **common)
        if not writes:
            continue
        v = video.cpu().numpy()
        for j, i in enumerate(idx):
            for s in range(n):
                write_video(v[j, s], os.path.join(args.out, f"{names[i]}_sample{s}"), args.fps)
    if writes:
        print(f"{len(pairs)} pairs x {n} samples from {args.prompt_dir} -> {args.out}")
    return 0


if __name__ == "__main__":
    sys.exit(main())

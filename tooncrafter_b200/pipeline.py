"""Keyframe interpolation end to end: K >= 2 keyframes -> one joined uint8 video.

The reference turns ONE pair of keyframes into a 16-frame clip with its evaluation glue (scripts/evaluation/inference.py:
load_data_prompts :64-106, image_guided_synthesis :180-277, save_results_seperate :135-155).  `ToonCrafterPipeline`
restates that glue on this library for a storyboard of K keyframes: S = K - 1 segments (S = K with `loop`, the last
one running from keyframe K-1 back to keyframe 0), sampled together and joined into one video.

Per call:
  * preprocessing of load_data_prompts (shorter side resized to min(size) with anti-aliasing, centre crop, [-1, 1]) as
    torchvision tensor ops on the model's device;
  * ONE VAE encode of the K distinct keyframes (the reference encodes 8 copies of each frame of a pair); segment k
    gets c_concat = z_k at frame 0, z_{k+1} at frame T-1, zeros elsewhere (inference.py:197-200), and the decoder
    reference maps [h_k, h_{k+1}] per level (inference.py:164-178);
  * ONE image-tower pass over the first keyframe of every segment plus the zero image, ONE text-tower pass over the
    distinct prompts plus "" (inference.py:186-216);
  * the segments as the batch rows of one fused DDIM sample() per group of `segments_per_batch`;
  * per segment the T and T - 2 decodes (inference.py:262-270; one decode with a plain first stage, see below), each
    in chunks of en_and_decode_n_samples_a_time (default temporal_length) frames as decode_core runs them, read by one
    tc_video_u8 launch that applies the middle-frame splice and the uint8 conversion of the save path and writes the
    segment's frames into the joined video at frame (T-1)*k.

RNG contract: keyframe j's posterior noise is drawn from a CPU generator seeded `seed + j`; segment k's x_T and
DDIM step noise come from a generator on the model's device seeded `seed + k` (DDIMSampler's `noise_generators`).
So segment k of a K-keyframe run is the same computation as a 2-keyframe run on (keyframe k, keyframe k+1) with
`seed + k`, whatever batch it runs in (up to the batch tiling of the kernels).

Variants (`n_samples`, the reference's --n_samples, image_guided_synthesis's loop at inference.py:234-274): n videos
that share the keyframe latents (the posterior noise above, drawn once), the tower outputs and the decoder reference
maps, and differ only in their DDIM noise: variant v of segment k draws from a device generator seeded
`seed + k + v * VARIANT_SEED_STRIDE` (2**32 + 0x9E3779B9), so variant 0 is the single-sample video and the seed of
(k, v) depends neither on n, S, the batch nor the rank.  A sampled row is one (segment, variant); rows run in variant-major order r = v * S + k, so
`segments_per_batch` consecutive rows share a sample() call and a contiguous block of rows writes a contiguous range
of the flattened [n * F] video (of [n * S] segments for float output).

Pair directories (`interpolate_pairs`, the reference's --prompt_dir with --interp, inference.py:64-106 and 280-340):
P independent pairs, pair i being the call interpolate([a_i, b_i], prompts=p_i, seed=seed + i, n_samples=n,
segments_per_batch=n).  Pairs are taken `pairs_per_batch` at a time, each group encoded, conditioned and sampled on
its own (pair-major rows, pair i's variant v being row i * n + v); with one pair per group the call is therefore
bit for bit that sequence of interpolate calls, and memory does not grow with P.

Seam rule: neighbouring segments share a keyframe; the earlier segment's last frame is kept and the later segment's
frame 0 is dropped.  With `loop`, the closing segment's last frame (keyframe 0 again) is dropped as well, so the
video has (T-1)*S + 1 frames, or (T-1)*K with `loop`.

`ToonCrafterPipeline.animate` is the same glue for one image (image_guided_synthesis with interp=False): one segment
whose c_concat is the image's latent repeated over the T frames.

Clip length: `video_length` T (the reference's --video_length, inference.py:93-100, 197-203), any even T from 4 to 64,
default the model's temporal_length.  The UNet gives each frame its own 16 image tokens only when the context holds
77 + 16 T tokens; the pipeline's 77 + 256 tokens give every frame all of them at any other T (openaimodel3d.py:556-562).

First stage: with the dual-reference AutoencoderKL_Dualref each segment is decoded twice (T and T - 2 frames, then
spliced, as above), every chunk of frames with the segment's two reference maps.  The plain AutoencoderKL of the
DynamiCrafter / training configs decodes every frame on its own, so each segment is decoded once, without reference
maps, and tc_video_u8 runs without a splice.

Several GPUs (`ToonCrafterPipeline(model, group)`, one process per GPU): the n * S rows are split into contiguous
blocks by distributed.shard_clips, one block per rank, or one per GPU pair with `latency` (the pair samples its block
with DDIMSampler.latency_group, one guidance branch per GPU, and pair-rank 0 decodes).  Every rank still encodes all
K keyframes and runs the two conditioning towers over the inputs of the single-process call, then takes its own
rows: the batch sizes, and with them the kernels' tiling, are those of the single-process call.  By the RNG contract a
row is then the same computation whichever rank runs it; each block writes its contiguous range of the flattened
video, and the blocks are broadcast so that every rank returns the full result.  interpolate_pairs splits the P pairs
the same way (each rank encoding only its own groups) and broadcasts each block's pairs.
"""
from __future__ import annotations

from typing import NamedTuple, Optional, Sequence, Union

import numpy as np
import torch
import torch.distributed as dist

from . import distributed, ops, runtime
from .modules import VideoDecoder, clip_tokenize
from .sampler import SAMPLERS, check_sampler, randn_rows


def preprocess(keyframes, size=(320, 512), device="cpu") -> torch.Tensor:
    """uint8 HWC RGB images -> [K, 3, size[0], size[1]] float32 in [-1, 1] on `device`.

    load_data_prompts's transform (inference.py:65-69): Resize(min(size)) (shorter side, bilinear, anti-aliased),
    CenterCrop(size) (zero padding where the image is smaller), ToTensor, Normalize(0.5, 0.5).  The resize runs on the
    uint8 tensor, like PIL's; an image whose shorter side already is min(size) is not resampled."""
    from torchvision.transforms.v2 import functional as TF
    if isinstance(keyframes, (torch.Tensor, np.ndarray)) and keyframes.ndim == 4:
        keyframes = list(keyframes)
    out = []
    for im in keyframes:
        t = im if isinstance(im, torch.Tensor) else torch.from_numpy(np.array(im))
        if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[-1] != 3:
            raise ValueError(f"keyframes must be uint8 [H, W, 3] RGB images, got {t.dtype} {tuple(t.shape)}")
        t = t.to(device).permute(2, 0, 1)
        if min(t.shape[1:]) != min(size):
            t = TF.resize(t, min(size), antialias=True)
        if tuple(t.shape[1:]) != tuple(size):
            t = TF.center_crop(t, list(size))
        out.append(t)
    return torch.stack(out).float().div(255).sub(0.5).div(0.5)


MIN_VIDEO_LENGTH, MAX_VIDEO_LENGTH = 4, 64


def check_video_length(T) -> int:
    """The clip lengths the pipeline runs: even (the interpolation video is T/2 copies of each keyframe,
    inference.py:93-94), at least 4 (the middle-frame splice of the T - 2 decode), at most 64 (tc_temporal_attention)."""
    if (isinstance(T, bool) or not isinstance(T, (int, np.integer)) or T % 2
            or not MIN_VIDEO_LENGTH <= T <= MAX_VIDEO_LENGTH):
        raise ValueError(f"video_length must be an even integer from {MIN_VIDEO_LENGTH} to {MAX_VIDEO_LENGTH}, got {T!r}")
    return int(T)


def default_segments_per_batch(size, T: int = 16) -> int:
    """Segments sampled together by default: as many as keep the UNet program at the activation budget of 4 segments
    of 16 frames at 320 x 512 (8 rows of 16 frames of a 40 x 64 latent, an arena of about 8 GB; it grows with rows x
    frames x latent pixels).  At 576 x 1024 and T = 16 that is 1 segment: with 4 the UNet arena alone would take 28 GiB,
    and a default call after an animate call (whose plans stay cached) no longer fits on an 80 GB H100."""
    return max(1, (4 * 16 * 320 * 512) // (T * size[0] * size[1]))


def default_pairs_per_batch(size, T: int, n_samples: int) -> int:
    """interpolate_pairs' default group: as many pairs as keep its pairs x n_samples rows within
    default_segments_per_batch(size, T), and at least one (a pair's variants always share one sample() call)."""
    return max(1, default_segments_per_batch(size, T) // n_samples)


# Variant v of a row whose single-sample noise seed is s draws from a generator seeded s + v * VARIANT_SEED_STRIDE: far
# from the seeds seed + k of the other segments (and pairs), and independent of the number of variants or rows.  The
# stride is 2**32 plus the 32-bit golden-ratio constant, so that variants differ in the low 32 bits as well: a CUDA
# generator keeps all 64 bits of its seed, a CPU generator (mt19937) only the low 32.
VARIANT_SEED_STRIDE = 2 ** 32 + 0x9E3779B9


def check_count(value, name: str) -> int:
    """n_samples, segments_per_batch, pairs_per_batch: an integer >= 1 (numpy integers too); bools are refused."""
    if isinstance(value, bool) or not isinstance(value, (int, np.integer)) or value < 1:
        raise ValueError(f"{name} must be an integer >= 1, got {value!r}")
    return int(value)


def check_n_samples(n) -> int:
    """Variants per input (the reference's --n_samples): an integer >= 1; bools are refused."""
    return check_count(n, "n_samples")


def check_strength(strength, steps: int) -> int:
    """refine's DDIM steps: k = int(strength * steps) for a strength in (0, 1]; ValueError when k < 1."""
    if (isinstance(strength, bool) or not isinstance(strength, (int, float, np.integer, np.floating))
            or not 0.0 < strength <= 1.0):
        raise ValueError(f"strength must be a number in (0, 1], got {strength!r}")
    k = int(strength * steps)
    if k < 1:
        raise ValueError(f"strength {strength} x steps {steps} runs no DDIM step (int(strength * steps) < 1)")
    return k


def check_keep(keep, T: int) -> Optional[list]:
    """refine's kept frames: None, or frame indices from 0 to T - 1, each listed once.  Returns them sorted (None for
    an empty list)."""
    if keep is None:
        return None
    keep = list(keep)
    if any(isinstance(j, bool) or not isinstance(j, (int, np.integer)) or not 0 <= j < T for j in keep):
        raise ValueError(f"keep must hold frame indices from 0 to {T - 1}, got {keep!r}")
    if len(set(int(j) for j in keep)) != len(keep):
        raise ValueError(f"keep lists a frame twice: {keep!r}")
    return sorted(int(j) for j in keep) or None


class _Call(NamedTuple):
    T: int                      # frames per segment
    n: int                      # variants per input
    per_batch: int              # segments_per_batch (rows per sample() call), or interpolate_pairs' pairs_per_batch
    variant_axis: bool          # the result keeps its leading variant axis (n_samples was given)
    size: tuple
    output: str
    steps: int
    cfg_scale: float
    eta: float
    fs: int
    guidance_rescale: float
    timestep_spacing: str
    cfg_img: Optional[float]
    sampler: str                # a key of sampler.SAMPLERS


class _Row(NamedTuple):
    """One sampled row: a (segment, variant), or a (pair, variant) of interpolate_pairs."""
    seg: int                    # its segment: an index into the first / last keyframe lists of the call that samples it
    seed: int                   # the seed of its device generator (x_T and step noise)
    index: int                  # float output: its clip in the flattened [rows, 3, T, H, W] video
    f_begin: int                # uint8 output: its frames f_begin .. f_end - 1 (the seam rule) go to frames out_frame ..
    f_end: int                  # of the flattened [frames, H, W, 3] video
    out_frame: int


class _Refine(NamedTuple):
    """refine's start: one segment whose keyframes 0 and 1 are the clip's first and last frames."""
    frames: torch.Tensor        # the preprocessed frames 1 .. T-2
    seeds: list                 # their posterior-noise seeds
    k: int                      # DDIM steps to run
    keep: Optional[list]        # frame indices held to the clip, or None


def _check_prompts(prompts, count: int, what: str) -> None:
    """One string, a list of `count` strings, or token ids [count, 77]: one prompt per segment or pair (`what`)."""
    if isinstance(prompts, torch.Tensor):
        if prompts.dim() != 2 or prompts.shape[0] != count:
            raise ValueError(f"token ids must be [{count} {what}, 77], got {tuple(prompts.shape)}")
    elif not isinstance(prompts, str) and len(prompts) != count:
        raise ValueError(f"{len(prompts)} prompts for {count} {what}")


def _span(rows, output: str) -> tuple:
    """[begin, end) of the flattened output that the consecutive `rows` write."""
    a, b = rows[0], rows[-1]
    if output == "float":
        return a.index, b.index + 1
    return a.out_frame, b.out_frame + b.f_end - b.f_begin


def _posterior_sample(m, post, seeds) -> torch.Tensor:
    """First-stage latents of an encoded batch, frame i's posterior noise from a CPU generator seeded seeds[i]."""
    noise = torch.stack([torch.randn(tuple(post.mean.shape[1:]), generator=torch.Generator().manual_seed(s))
                         for s in seeds])
    return m.get_first_stage_encoding(post, noise=noise)


def _decode_chunks(dec, lat, n: int, ref, ex):
    """decode_core's loop (ddpm3d.py:656-675): lat [T, 4, h, w] decoded n frames at a time (a dual-reference decoder
    with timesteps = the chunk's length and the same reference maps `ref`).  One chunk returns the plan's output view
    as it is; several are copied into one [T, 3, H, W] tensor, since chunks of one length share a plan."""
    args = () if ref is None else (ref,)
    if lat.shape[0] <= n:
        return dec.decode(lat.float(), *args, executor=ex)
    out = None
    for i in range(0, lat.shape[0], n):
        y = dec.decode(lat[i:i + n].float(), *args, executor=ex)
        if out is None:
            out = torch.empty((lat.shape[0],) + tuple(y.shape[1:]), dtype=y.dtype, device=y.device)
        out[i:i + y.shape[0]].copy_(y)
    return out


class ToonCrafterPipeline:
    """K keyframes -> one interpolated video, on a LatentVisualDiffusion of this library (see the module docstring).

    group: None (one process; torch.distributed is not touched even when initialised), or a torch.distributed process
    group whose ranks all construct the pipeline and make the same calls: the segments are sharded over its ranks and
    every rank returns the full result of the single-process call.  latency: shard over GPU pairs (adjacent ranks of
    `group`) instead, each pair sampling one block with one classifier-free-guidance branch per GPU; needs an even
    group size, and refuses cfg_img and cfg_scale 1.0.  With `latency` every rank of the world must construct the
    pipeline (the pair groups are created collectively)."""

    def __init__(self, model, group=None, latency: bool = False):
        self.model = model
        self.group = group
        self.latency = latency
        self._pair = None
        if latency:
            if group is None:
                raise ValueError("latency mode needs a process group of GPU pairs")
            self._pair, self._block, self._pair_rank = distributed.latency_pairs(group)
            self._n_blocks = dist.get_world_size(group) // 2
        elif group is not None:
            self._block, self._n_blocks = dist.get_rank(group), dist.get_world_size(group)

    @torch.no_grad()
    def interpolate(self, keyframes, prompts: Union[str, Sequence[str], torch.Tensor] = "", steps: int = 50,
                    cfg_scale: float = 7.5, eta: float = 1.0, fs: int = 10, guidance_rescale: float = 0.7,
                    timestep_spacing: str = "uniform_trailing", cfg_img=None, loop: bool = False, seed: int = 123,
                    size=(320, 512), segments_per_batch: Optional[int] = None, output: str = "uint8",
                    video_length: Optional[int] = None, n_samples: Optional[int] = None,
                    sampler: str = "ddim") -> torch.Tensor:
        """keyframes: K >= 2 uint8 RGB images (tensor [K, H, W, 3], ndarray, or a list of [H, W, 3] arrays of any
        size).  prompts: one string for every segment, a list of S strings, or token ids [S, 77] (strings other than
        "" need open_clip's tokenizer).  cfg_img not None: three-way guidance (DDIMSamplerMultiCond).  Defaults are
        those of the reference's scripts/run.sh.

        video_length: T frames per segment, an even number from 4 to 64 (ValueError otherwise); None: the model's
        temporal_length.  n_samples: None, or n >= 1 variants of the whole video (the reference's --n_samples), which
        share the keyframe latents, the conditioning and the decoder reference maps and differ in their DDIM noise
        only (module docstring).  segments_per_batch: sampled rows, one (segment, variant) each, per sample() call;
        None: default_segments_per_batch(size, T), 4 at 320 x 512 and 1 at 576 x 1024 for T = 16.

        Returns uint8 [F, size[0], size[1], 3] on the model's device, F = (T-1)*S + 1 (or (T-1)*K with `loop`); with
        output="float", the spliced per-segment videos before quantisation, float32 [S, 3, T, size[0], size[1]].
        With an integer n_samples both gain a leading variant axis, [n, F, H, W, 3] / [n, S, 3, T, H, W], and
        video[v] is a complete single-sample result (video[0] is the n_samples=None result).

        sampler: "ddim" (the reference's sampler) or "dpmpp_2m" (DPM-Solver++(2M), eta 0 or 1: the same UNet
        evaluations per step, second order; INTEGRATION.md).  Every method takes it; ValueError for an unknown name or
        dpmpp_2m with another eta, before any work."""
        c = self._checked(video_length, n_samples, segments_per_batch, size, output, steps, cfg_scale, eta, fs,
                          guidance_rescale, timestep_spacing, cfg_img, sampler)
        frames = preprocess(keyframes, c.size, self.model.device)
        K = frames.shape[0]
        if K < 2:
            raise ValueError("interpolation needs at least two keyframes")
        S = K if loop else K - 1
        return self._generate(frames, prompts, list(range(S)), [(k + 1) % K for k in range(S)], True, loop, seed, c)

    @torch.no_grad()
    def animate(self, image, prompt: Union[str, torch.Tensor] = "", steps: int = 50, cfg_scale: float = 7.5,
                eta: float = 1.0, fs: int = 10, guidance_rescale: float = 0.7,
                timestep_spacing: str = "uniform_trailing", cfg_img=None, seed: int = 123, size=(320, 512),
                output: str = "uint8", video_length: Optional[int] = None, n_samples: Optional[int] = None,
                segments_per_batch: Optional[int] = None, sampler: str = "ddim") -> torch.Tensor:
        """One image -> one T-frame video: image_guided_synthesis with interp=False, loop=False (inference.py:
        180-277; c_concat is the image's latent repeated over the T frames, :201-203), the image-to-video mode of
        the DynamiCrafter checkpoints.  image: a uint8 [H, W, 3] RGB image of any size; prompt: a string or token
        ids [1, 77].  The image's posterior noise comes from a CPU generator seeded `seed`, x_T and the DDIM step
        noise from a generator on the model's device seeded `seed` (keyframe 0 / segment 0 of `interpolate`); a
        dual-reference first stage gets the image's encoder maps as both reference frames.  video_length: T, and
        n_samples / segments_per_batch (variants sampled per call), as for interpolate.

        Returns uint8 [T, size[0], size[1], 3] on the model's device; with output="float", the spliced video before
        quantisation, float32 [3, T, size[0], size[1]]; with an integer n_samples, [n, T, H, W, 3] / [n, 3, T, H, W].
        sampler: as for interpolate."""
        c = self._checked(video_length, n_samples, segments_per_batch, size, output, steps, cfg_scale, eta, fs,
                          guidance_rescale, timestep_spacing, cfg_img, sampler)
        frames = preprocess([image], c.size, self.model.device)
        return self._generate(frames, prompt, [0], [0], False, False, seed, c, segment_axis=False)

    @torch.no_grad()
    def refine(self, clip, strength: float, prompt: Union[str, torch.Tensor] = "", keep: Optional[Sequence[int]] = None,
               steps: int = 50, cfg_scale: float = 7.5, eta: float = 1.0, fs: int = 10, guidance_rescale: float = 0.7,
               timestep_spacing: str = "uniform_trailing", cfg_img=None, seed: int = 123, size=(320, 512),
               output: str = "uint8", n_samples: Optional[int] = None,
               segments_per_batch: Optional[int] = None, sampler: str = "ddim") -> torch.Tensor:
        """Re-render an existing clip (SDEdit: DDIMSampler.stochastic_encode, then the last k DDIM steps), conditioned
        on its own first and last frames exactly as interpolate([clip[0], clip[T-1]], video_length=T) is.

        clip: T uint8 RGB frames (tensor [T, H, W, 3], ndarray, or a list of [H, W, 3] arrays), T even from 4 to 64.
        strength in (0, 1]: k = int(strength * steps) >= 1 DDIM steps run, from the clip's latents noised to DDIM
        index k - 1 (the noise level of the first step that runs); strength 1.0 is full sampling.  keep: None, or
        frame indices whose latents are held to the clip's (the sampler's mask / x0: at every step those frames are
        replaced by the clip's latents noised to the step's level), so only the frames between are regenerated.
        Kept frames are decoded again with the rest, not pasted back, so they are close to, not equal to, the input.

        First stage: frames 0 and T-1 are encoded as interpolate encodes its two keyframes (one N = 2 call, posterior
        noise seeds `seed` and `seed + 1`), frames 1 .. T-2 in chunks of en_and_decode_n_samples_a_time (default
        temporal_length) frames, frame j with posterior noise seed `seed + 1 + j`.  Variant v draws, from its device
        generator seeded seed + v * VARIANT_SEED_STRIDE, first the encode noise (where interpolate draws x_T), then each
        step's q_sample noise of the kept frames (with keep) and DDIM noise.  Under a zero-terminal-SNR schedule
        (sqrt(alphas_cumprod[999]) = 0) refine(clip, 1.0) is therefore interpolate([clip[0], clip[-1]],
        video_length=T) bit for bit.

        Returns what a one-segment interpolate returns: uint8 [T, size[0], size[1], 3], or float32 [3, T, size[0],
        size[1]] with output="float"; an integer n_samples adds a leading variant axis.  ValueError for a bad clip
        length, strength, keep, n_samples, segments_per_batch, output or sampler before any work.  sampler: as for
        interpolate; the last k steps run with it."""
        c = self._checked(len(clip), n_samples, segments_per_batch, size, output, steps, cfg_scale, eta, fs,
                          guidance_rescale, timestep_spacing, cfg_img, sampler)
        T = c.T
        k, keep = check_strength(strength, steps), check_keep(keep, T)
        frames = preprocess(clip, c.size, self.model.device)
        start = _Refine(frames[1:T - 1], [seed + 1 + j for j in range(1, T - 1)], k, keep)
        return self._generate(frames[[0, T - 1]], prompt, [0], [1], True, False, seed, c, segment_axis=False,
                              refine=start)

    @torch.no_grad()
    def interpolate_pairs(self, pairs, prompts: Union[str, Sequence[str], torch.Tensor] = "", n_samples: int = 1,
                          steps: int = 50, cfg_scale: float = 7.5, eta: float = 1.0, fs: int = 10,
                          guidance_rescale: float = 0.7, timestep_spacing: str = "uniform_trailing", cfg_img=None,
                          seed: int = 123, size=(320, 512), pairs_per_batch: Optional[int] = None,
                          output: str = "uint8", video_length: Optional[int] = None,
                          sampler: str = "ddim") -> torch.Tensor:
        """P independent keyframe pairs -> n_samples T-frame clips each: the reference's --prompt_dir --interp run
        (module docstring).  pairs: P pairs of uint8 RGB images (a sequence of (a, b), or a tensor [P, 2, H, W, 3]);
        prompts: one string for every pair, a list of P strings, or token ids [P, 77].

        Pair i is the call interpolate([a_i, b_i], prompts=p_i, seed=seed + i, n_samples=n, segments_per_batch=n):
        bit for bit with pairs_per_batch=1, on any number of ranks; to the kernels' batch tiling with larger groups.
        pairs_per_batch: pairs whose keyframes are encoded, conditioned and sampled together (pairs_per_batch x n rows
        per sample() call); None: default_pairs_per_batch(size, T, n).

        Returns uint8 [P, n, T, size[0], size[1], 3] on the model's device, every pair's whole clip; with
        output="float", float32 [P, n, 3, T, size[0], size[1]].  sampler: as for interpolate."""
        P = len(pairs)
        if P < 1 or any(len(p) != 2 for p in pairs):
            raise ValueError("pairs must be a non-empty sequence of (image, image) pairs")
        _check_prompts(prompts, P, "pairs")
        c = self._checked(video_length, n_samples, pairs_per_batch, size, output, steps, cfg_scale, eta, fs,
                          guidance_rescale, timestep_spacing, cfg_img, sampler, pairs=True)
        n, T = c.n, c.T
        # pair-major rows: pair i's variant v is row i * n + v, its whole clip (frames 0 .. T-1, no seam)
        rows = [_Row(i, seed + i + v * VARIANT_SEED_STRIDE, i * n + v, 0, T, (i * n + v) * T)
                for i in range(P) for v in range(n)]
        video = self._empty(rows, c)
        mine = self._mine(P)
        for g0 in range(0, len(mine), c.per_batch):
            group = mine[g0:g0 + c.per_batch]
            frames = preprocess([im for i in group for im in pairs[i]], c.size, self.model.device)
            text = prompts if isinstance(prompts, str) else (prompts[group] if isinstance(prompts, torch.Tensor)
                                                             else [prompts[i] for i in group])
            batch = [r._replace(seg=r.seg - group[0]) for r in rows[group[0] * n:(group[-1] + 1) * n]]
            G = len(group)
            self._render(frames, text, [2 * k for k in range(G)], [2 * k + 1 for k in range(G)], True,
                         [seed + i + j for i in group for j in (0, 1)], batch, len(batch), video, c)
        self._broadcast(video, rows, n, c.output)
        return (video.view(P, n, T, *c.size, 3) if c.output == "uint8" else video.view(P, n, 3, T, *c.size))

    def _checked(self, video_length, n_samples, per_batch, size, output, steps, cfg_scale, eta, fs, guidance_rescale,
                 timestep_spacing, cfg_img, sampler, pairs: bool = False) -> _Call:
        """The argument checks the public methods share, all before any work; returns the normalised arguments.
        video_length None: the model's temporal_length.  per_batch: segments_per_batch, or pairs_per_batch with
        `pairs` (where n_samples must be an integer); None: its default."""
        T = check_video_length(self.model.temporal_length if video_length is None else video_length)
        n = check_n_samples(n_samples) if pairs or n_samples is not None else 1
        if per_batch is not None:
            per_batch = check_count(per_batch, "pairs_per_batch" if pairs else "segments_per_batch")
        else:
            per_batch = default_pairs_per_batch(size, T, n) if pairs else default_segments_per_batch(size, T)
        if output not in ("uint8", "float"):
            raise ValueError(f"output must be 'uint8' or 'float', got {output!r}")
        check_sampler(sampler, eta)
        if size[0] % 16 or size[1] % 16:
            raise ValueError(f"size {tuple(size)} must be a multiple of 16")
        if self.model.model.conditioning_key != "hybrid":
            raise NotImplementedError("image-conditioned synthesis needs the hybrid (concat + cross-attention) model")
        if self.latency and cfg_img is not None:
            raise NotImplementedError("latency mode splits two guidance branches over a GPU pair; three-way "
                                      "guidance (cfg_img) is not supported")
        if self.latency and cfg_scale == 1.0:
            raise ValueError("latency mode splits the conditional and unconditional branches over a GPU pair; "
                             "cfg_scale 1.0 has no unconditional branch")
        return _Call(T, n, per_batch, pairs or n_samples is not None, tuple(size), output, steps, cfg_scale, eta, fs,
                     guidance_rescale, timestep_spacing, cfg_img, sampler)

    def _mine(self, n_items: int):
        """The items (rows, pairs) of this rank's block: all of them without a group."""
        return list(range(n_items)) if self.group is None else distributed.shard_clips(n_items, self._block,
                                                                                       self._n_blocks)

    def _empty(self, rows, c: _Call) -> torch.Tensor:
        """The flattened output that all of the call's `rows` fill."""
        if c.output == "float":
            return torch.empty(len(rows), 3, c.T, *c.size, dtype=torch.float32, device=self.model.device)
        return torch.empty(_span(rows, "uint8")[1], *c.size, 3, dtype=torch.uint8, device=self.model.device)

    def _broadcast(self, video, rows, per_item: int, output: str) -> None:
        """With a group: give every rank the whole `video`.  The items _mine shards are the groups of `per_item`
        consecutive `rows` (all of the call's rows); block b's rows write their span of the rank that computed them."""
        if self.group is None:
            return
        blocks = []
        for b in range(self._n_blocks):
            items = distributed.shard_clips(len(rows) // per_item, b, self._n_blocks)
            if items:                               # held by the rank, or pair-rank 0 of the pair, that computed it
                owner = dist.get_global_rank(self.group, 2 * b if self.latency else b)
                blocks.append((owner,) + _span(rows[items[0] * per_item:(items[-1] + 1) * per_item], output))
        distributed.broadcast_blocks(video, blocks, self.group)

    def _generate(self, frames, prompts, first, last, interp: bool, loop, seed, c: _Call, segment_axis: bool = True,
                  refine: Optional[_Refine] = None) -> torch.Tensor:
        """c.n variants of S = len(first) segments of c.T frames; segment k runs from keyframe first[k] to keyframe
        last[k] (interp), or animates keyframe first[k] (not interp).  Row r = v * S + k is variant v of segment k.
        With a group, this rank computes its block of rows and the blocks are then broadcast.
        Returns uint8 [n, F, H, W, 3] or float [n, S, 3, T, H, W], without the variant axis unless c.variant_axis,
        and without the float segment axis unless segment_axis."""
        S, T, n = len(first), c.T, c.n
        F = (T - 1) * S + (0 if loop else 1)
        rows = []
        for r in range(n * S):
            v, k = divmod(r, S)
            f_begin, f_end = (1 if k else 0), (T - 1 if (loop and k == S - 1) else T)
            rows.append(_Row(k, seed + k + v * VARIANT_SEED_STRIDE, r, f_begin, f_end, v * F + (T - 1) * k + f_begin))
        video = self._empty(rows, c)
        mine = [rows[r] for r in self._mine(len(rows))]
        if mine:
            self._render(frames, prompts, first, last, interp, [seed + j for j in range(frames.shape[0])], mine,
                         c.per_batch, video, c, refine)
        self._broadcast(video, rows, 1, c.output)
        if c.output == "uint8":
            video = video.view(n, F, *c.size, 3)
        else:
            video = video.view(n, S, 3, T, *c.size)
            if not segment_axis:
                video = video[:, 0]
        return video if c.variant_axis else video[0]

    def _render(self, frames, prompts, first, last, interp: bool, key_seeds, rows, rows_per_batch, video, c: _Call,
                refine: Optional[_Refine] = None) -> None:
        """Sample and decode `rows` (consecutive, rows_per_batch per sample() call) into `video`.  Segment k of S =
        len(first) runs from keyframe first[k] to keyframe last[k] (interp), or animates keyframe first[k]; keyframe
        j's posterior noise is seeded key_seeds[j].  refine: every row starts from the clip's latents (_refine_start)."""
        m = self.model
        T = c.T
        emb = self._conditioning(frames, prompts, first)
        post, hidden = m.first_stage_model.encode(frames, return_hidden_states=True)
        z = _posterior_sample(m, post, key_seeds)                                    # [K, 4, h, w]
        if interp:
            c_concat = torch.zeros(len(first), z.shape[1], T, *z.shape[-2:], dtype=z.dtype, device=m.device)
            c_concat[:, :, 0] = z[first]
            c_concat[:, :, -1] = z[last]
        else:
            c_concat = z[first][:, :, None].expand(-1, -1, T, -1, -1).contiguous()
        x0 = None if refine is None else self._clip_latents(z, refine.frames, refine.seeds)   # [1, 4, T, h, w]

        two_way, three_way = SAMPLERS[c.sampler]
        sampler = two_way(m) if c.cfg_img is None else three_way(m)
        sampler.latency_group = self._pair
        decodes = not (self.latency and self._pair_rank)          # in a latency pair, pair-rank 0 decodes
        dec = m.first_stage_model.decoder_engine() if decodes else None
        dual_ref = isinstance(m.first_stage_model.decoder, VideoDecoder)
        for g0 in range(0, len(rows), rows_per_batch):
            batch = rows[g0:g0 + rows_per_batch]
            gens = [torch.Generator(device=m.device).manual_seed(r.seed) for r in batch]
            start = {} if refine is None else self._refine_start(sampler, x0, refine, gens, c)
            samples = self._sample(sampler, emb, c_concat, [r.seg for r in batch], gens, start, c)
            if not decodes:
                continue
            for row, sample in zip(batch, samples):
                ref = ([torch.stack([hd[first[row.seg]], hd[last[row.seg]]], 1).unsqueeze(0) for hd in hidden]
                       if dual_ref else None)
                self._write_row(dec, video, row, sample, ref, T)

    def _conditioning(self, frames, prompts, first):
        """(text, unconditional text, image, unconditional image) embeddings of the S = len(first) segments: one text-
        tower pass over the distinct prompts + "", one image-tower pass over each segment's first keyframe + the zero
        image.  Over all S segments whatever rows are sampled: the towers' batch size stays that of the single-process
        call, and the variants of a segment share its conditioning."""
        m = self.model
        S = len(first)
        _check_prompts(prompts, S, "segments")
        if isinstance(prompts, torch.Tensor):
            uniq, inv = torch.unique(prompts.long().cpu(), dim=0, return_inverse=True)
            emb = m.get_learned_conditioning(torch.cat([uniq, clip_tokenize([""], prompts.shape[1])]).to(m.device))
            cond_emb, empty_emb = emb[inv.to(emb.device)], emb[-1:]
        else:
            texts = [prompts] * S if isinstance(prompts, str) else list(prompts)
            distinct = list(dict.fromkeys(texts + [""]))
            emb = m.get_learned_conditioning(distinct)
            idx = torch.tensor([distinct.index(t) for t in texts], device=emb.device)
            cond_emb, empty_emb = emb[idx], emb[distinct.index("")][None]
        if m.uncond_type == "empty_seq":
            uc_emb = empty_emb.expand_as(cond_emb)
        elif m.uncond_type == "zero_embed":
            uc_emb = torch.zeros_like(cond_emb)
        else:
            raise NotImplementedError(f"uncond_type {m.uncond_type!r}")
        img = torch.cat([frames[first], torch.zeros_like(frames[:1])])
        img_all = m.image_proj_model(m.embedder(img))
        return cond_emb, uc_emb, img_all[:S], img_all[S:].expand(S, -1, -1)

    def _clip_latents(self, z_ends, interior, seeds) -> torch.Tensor:
        """[1, 4, T, h, w] latents of a clip: frames 0 and T-1 from z_ends [2, 4, h, w], frames 1 .. T-2 encoded from
        `interior` in chunks of decode_core's chunk length (the encoder is per frame, so chunking changes only its
        batch tiling), frame j's posterior noise from a CPU generator seeded seeds[j - 1]."""
        m = self.model
        n_enc = m.en_and_decode_n_samples_a_time or m.temporal_length
        T = interior.shape[0] + 2
        x0 = torch.empty((1, z_ends.shape[1], T) + tuple(z_ends.shape[-2:]), dtype=z_ends.dtype, device=z_ends.device)
        x0[0, :, 0], x0[0, :, T - 1] = z_ends[0], z_ends[1]
        for i in range(0, T - 2, n_enc):
            post = m.first_stage_model.encode(interior[i:i + n_enc])
            x0[0, :, 1 + i:1 + i + post.mean.shape[0]] = _posterior_sample(m, post, seeds[i:i + n_enc]).transpose(0, 1)
        return x0

    def _refine_start(self, sampler, x0, refine: _Refine, gens, c: _Call) -> dict:
        """sample()'s keywords that start a batch of len(gens) rows from the clip's latents x0, stochastic_encode'd to
        DDIM index k - 1 with noise drawn first from each row's generator, and run the last k steps (with keep: mask
        and x0 on the kept frames)."""
        dev = self.model.device
        shape = (len(gens),) + tuple(x0.shape[1:])
        sampler.make_schedule(c.steps, c.timestep_spacing, c.eta, verbose=False)
        x_k = sampler.stochastic_encode(x0.expand(shape), torch.full((len(gens),), refine.k - 1, device=dev),
                                        noise=randn_rows(shape, dev, gens))
        start = dict(x_T=x_k, t_start=refine.k)
        if refine.keep is not None:
            mask = torch.zeros(1, 1, c.T, 1, 1, dtype=torch.float32, device=dev)
            mask[:, :, refine.keep] = 1.0
            start.update(mask=mask, x0=x0.expand(shape).contiguous())
        return start

    def _sample(self, sampler, emb, c_concat, seg, gens, start: dict, c: _Call) -> torch.Tensor:
        cond_emb, uc_emb, img_emb, uc_img_emb = emb
        b = len(seg)
        cc = [c_concat[seg]]
        cond = {"c_crossattn": [torch.cat([cond_emb[seg], img_emb[seg]], 1)], "c_concat": cc}
        uc = ({"c_crossattn": [torch.cat([uc_emb[seg], uc_img_emb[seg]], 1)], "c_concat": cc}
              if c.cfg_scale != 1.0 else None)
        if c.cfg_img is not None:
            start = dict(start, cfg_img=c.cfg_img, unconditional_conditioning_img_nonetext={
                "c_crossattn": [torch.cat([uc_emb[seg], img_emb[seg]], 1)], "c_concat": cc})
        samples, _ = sampler.sample(S=c.steps, conditioning=cond, batch_size=b, shape=list(c_concat.shape[1:]),
                                    verbose=False, unconditional_guidance_scale=c.cfg_scale,
                                    unconditional_conditioning=uc, eta=c.eta,
                                    fs=torch.tensor([c.fs] * b, dtype=torch.long, device=self.model.device),
                                    timestep_spacing=c.timestep_spacing, guidance_rescale=c.guidance_rescale,
                                    noise_generators=gens, **start)
        return samples

    def _write_row(self, dec, video, row: _Row, sample, ref, T: int) -> None:
        """Decode one row's latents [4, T, h, w] and write it into `video` at its place: the spliced clip in float
        output, its seam-rule frames through tc_video_u8 in uint8 output.  ref: the dual-reference decoder's maps, None
        with a plain first stage."""
        m = self.model
        n_dec = m.en_and_decode_n_samples_a_time or m.temporal_length                # decode_core's chunk
        ex = runtime.TEST_EXECUTOR
        keep = [t for t in range(T) if t not in (1, T - 2)]                           # inference.py:264-267
        lat = (1.0 / m.scale_factor * sample).permute(1, 0, 2, 3)                    # decode_core order
        if ref is not None:
            y16 = _decode_chunks(dec, lat, n_dec, ref, ex)          # a view of the plan's output for T <= n_dec
            y14 = _decode_chunks(dec, lat[keep], n_dec, ref, ex)
        else:
            # A frame-independent decoder turns each latent into the same frame whichever chunk holds it, so the
            # reference's T - 2 pass is y16[keep] and the T - 2 decode is skipped.  For T >= 6 the two spliced frames
            # (keep[T/2-2], keep[T/2-1] = latents T/2-1, T/2) are the frames already in place: no splice at all
            # (tc_video_u8 with x14 = NULL).
            y16 = _decode_chunks(dec, lat, n_dec, None, ex)
            y14 = None if T >= 6 else y16[keep]
        if video.dtype == torch.float32:
            v = y16.float()
            if y14 is not None:
                v[T // 2 - 1:T // 2 + 1] = y14[T // 2 - 2:T // 2].float()
            video[row.index] = v.permute(1, 0, 2, 3)
            return
        args, kw = (y16, y14, video), dict(f_begin=row.f_begin, f_end=row.f_end, out_frame=row.out_frame)
        if ex is not None:
            ex(ops.video_u8, args, kw)
        else:
            ops.video_u8(*args, **kw)

"""Multi-GPU plumbing.  Throughput mode — the clip-parallel path: the reference shards prompts across ranks with no
collective on the data path (scripts/evaluation/inference.py:314-320, scripts/evaluation/ddp_wrapper.py:8-46).

One process per GPU; the only collectives are ONE broadcast of the weights at init and the max-over-ranks of the
timed region.  Backend "nccl" on GPUs (NVLink 5 / NVSwitch), "gloo" in the CPU tests.

Latency mode: pairs of adjacent ranks share ONE clip.  Classifier-free guidance needs two UNet
evaluations per step (ddim.py:217-232); pair-rank 0 runs the conditional branch, pair-rank 1 the unconditional one
(B = 1 each instead of one B = 2 forward), and one NCCL all-gather of the two fp16 predictions (2 x 327 KB at 320x512x16)
per DDIM step is the only exchange: both ranks then apply the identical fused DDIM update.  `latency_pairs()` builds the
groups, `DDIMSampler.latency_group` switches the sampler over.
"""
from __future__ import annotations

from typing import List

import torch
import torch.distributed as dist


def shard_clips(n_clips: int, rank: int, world: int) -> List[int]:
    """Clip indices of `rank`: contiguous blocks like the reference (inference.py:314-320) when n_clips divides
    evenly, and the remainder spread one-per-rank from rank 0 (the reference silently drops it)."""
    base, rem = divmod(n_clips, world)
    start = rank * base + min(rank, rem)
    return list(range(start, start + base + (1 if rank < rem else 0)))


def clip_seed(base_seed: int, clip_index: int) -> int:
    """Per-clip RNG seed: results do not depend on the world size."""
    return base_seed + clip_index


def broadcast_parameters(module: torch.nn.Module, src: int = 0, bucket_bytes: int = 1 << 30) -> int:
    """Broadcast every parameter and buffer of `module` from `src` in flat buckets; returns bytes sent."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return 0
    tensors = [p.data for p in module.parameters()] + [b.data for b in module.buffers()]
    total = 0
    by_dtype = {}
    for t in tensors:
        by_dtype.setdefault((t.dtype, t.device), []).append(t)
    for (_, _), group in by_dtype.items():
        bucket, size = [], 0
        def flush():
            nonlocal bucket, size, total
            if not bucket:
                return
            flat = torch._utils._flatten_dense_tensors(bucket)
            dist.broadcast(flat, src=src)
            for t, s in zip(bucket, torch._utils._unflatten_dense_tensors(flat, bucket)):
                t.copy_(s)
            total += flat.numel() * flat.element_size()
            bucket, size = [], 0
        for t in group:
            bucket.append(t)
            size += t.numel() * t.element_size()
            if size >= bucket_bytes:
                flush()
        flush()
    return total


def max_over_ranks(value: float, device="cpu") -> float:
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def latency_pairs(group=None):
    """Process groups of adjacent rank pairs (0,1), (2,3), ... of `group` (default: the world); returns (group of this
    rank, pair index, rank in pair).  Every rank of the world must call this (new_group is collective).  The size of
    `group` must be even."""
    ranks = list(range(dist.get_world_size())) if group is None else dist.get_process_group_ranks(group)
    if len(ranks) % 2:
        raise ValueError("latency mode pairs GPUs: the world size must be even")
    me = ranks.index(dist.get_rank())
    mine = None
    for p in range(len(ranks) // 2):
        g = dist.new_group(ranks=ranks[2 * p:2 * p + 2])
        if me // 2 == p:
            mine = g
    return mine, me // 2, me % 2


def _device_collectives(group) -> bool:
    """NCCL moves device tensors directly (NVLink); any other backend (gloo: two ranks time-sharing ONE GPU in the
    single-GPU test, or CPU tests) is staged through host memory."""
    return dist.get_backend(group) == "nccl"


def pair_broadcast(t: torch.Tensor, src: int, group) -> None:
    if _device_collectives(group) or t.device.type == "cpu":
        dist.broadcast(t, src=src, group=group)
        return
    h = t.cpu()
    dist.broadcast(h, src=src, group=group)
    t.copy_(h)


def pair_all_gather(out: torch.Tensor, inp: torch.Tensor, group) -> None:
    """out[r * n:(r + 1) * n] = inp of pair-rank r (the per-step exchange of latency mode: 2 x 327 KB of fp16)."""
    if _device_collectives(group) or inp.device.type == "cpu":
        dist.all_gather_into_tensor(out, inp, group=group)
        return
    parts = [torch.empty(inp.shape, dtype=inp.dtype) for _ in range(dist.get_world_size(group))]
    dist.all_gather(parts, inp.cpu().contiguous(), group=group)
    out.copy_(torch.cat(parts, 0))


def sync_pair_state(x: torch.Tensor, group, rng_state: bool = True) -> None:
    """Make the start latent and the CUDA RNG stream of a latency pair identical (pair-rank 0 wins), so that both ranks
    draw the same per-step noise (ddim.py:273) and apply the same update.  rng_state=False: the start latent only, for
    a sampler whose rows draw their noise from per-row generators seeded alike on both ranks (the global RNG is then
    not used, and is left alone)."""
    src = dist.get_global_rank(group, 0)
    pair_broadcast(x, src, group)
    if not rng_state:
        return
    state = torch.cuda.get_rng_state(x.device)              # a CPU byte tensor
    if _device_collectives(group):
        dstate = state.to(x.device)
        dist.broadcast(dstate, src=src, group=group)
        state = dstate.cpu()
    else:
        dist.broadcast(state, src=src, group=group)
    torch.cuda.set_rng_state(state, x.device)


def broadcast_blocks(t: torch.Tensor, blocks, group) -> None:
    """Assemble `t` on every rank of `group` from contiguous blocks along dim 0: blocks = [(src, begin, end), ...],
    t[begin:end] of global rank `src` is copied to every other rank.  One broadcast per non-empty block, so blocks may
    differ in size; device tensors go over NCCL directly, anything else through host memory (pair_broadcast)."""
    for src, begin, end in blocks:
        if end > begin:
            pair_broadcast(t[begin:end], src, group)

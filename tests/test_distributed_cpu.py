"""world_size-2 gloo tests (CPU) of the N>1 path: clip sharding, the single weight broadcast, max-over-ranks."""
import sys
from pathlib import Path

import torch
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from distributed_harness import spawn  # noqa: E402
from tooncrafter_b200 import distributed as D  # noqa: E402


def test_shard_clips_partition():
    for n in (0, 1, 3, 8, 17):
        for world in (1, 2, 4, 8):
            shards = [D.shard_clips(n, r, world) for r in range(world)]
            flat = [i for s in shards for i in s]
            assert flat == list(range(n))                      # disjoint, complete, ordered
            assert max(len(s) for s in shards) - min(len(s) for s in shards) <= 1
    assert D.shard_clips(8, 3, 4) == [6, 7]                      # reference-style contiguous blocks
    assert D.clip_seed(123, 5) == 128


def _worker(rank, world):
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.manual_seed(100 + rank)                            # different random weights per rank before the broadcast
        m = torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.GroupNorm(4, 32), torch.nn.Linear(32, 8))
        m.register_buffer("sched", torch.arange(5, dtype=torch.float32) * (rank + 1))
        sent = D.broadcast_parameters(m, src=0, bucket_bytes=1024)   # several buckets
        sig = torch.cat([p.detach().flatten() for p in m.parameters()] + [m.sched]).double().sum().item()
        gathered = [None] * world
        dist.all_gather_object(gathered, sig)
        mx = D.max_over_ranks(10.0 + rank)
        clips = D.shard_clips(5, rank, world)
        allc = [None] * world
        dist.all_gather_object(allc, clips)
        return dict(sent=sent, sigs=gathered, mx=mx, clips=allc)
    finally:
        dist.destroy_process_group()


def test_two_rank_broadcast_and_timing_reduction():
    res = spawn(_worker, world=2, timeout=120)[0]
    assert res["sent"] > 0
    assert res["sigs"][0] == res["sigs"][1]                     # every rank holds rank 0's weights and buffers
    assert res["mx"] == 11.0                                     # max over ranks, not the local value
    assert res["clips"] == [[0, 1, 2], [3, 4]]


def _pair_worker(rank, world):
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        group, pair, in_pair = D.latency_pairs()
        # the per-step exchange of latency mode: all-gather of the two guidance branches inside the pair
        mine = torch.full((1, 4, 2, 3, 3), float(10 * pair + in_pair))
        both = torch.empty(2 * mine.shape[0], *mine.shape[1:])            # concatenated along dim 0: [cond | uncond]
        dist.all_gather_into_tensor(both, mine, group=group)
        x = torch.full((3,), float(rank))
        dist.broadcast(x, src=dist.get_global_rank(group, 0), group=group)      # what sync_pair_state does for x_T
        res = [None] * world
        dist.all_gather_object(res, dict(pair=pair, in_pair=in_pair, e_c=float(both[0].mean()), e_uc=float(both[1].mean()),
                                         x=float(x[0])))
        return res
    finally:
        dist.destroy_process_group()


def test_latency_pairs_two_rank_exchange():
    """Latency mode plumbing on gloo: pair groups, the branch all-gather, the start-state broadcast."""
    res = spawn(_pair_worker, world=2, timeout=120)[0]
    assert [r["pair"] for r in res] == [0, 0] and [r["in_pair"] for r in res] == [0, 1]
    assert all(r["e_c"] == 0.0 and r["e_uc"] == 1.0 for r in res)        # slot 0 = conditional rank, slot 1 = unconditional
    assert all(r["x"] == 0.0 for r in res)                               # pair-rank 0's start latent wins

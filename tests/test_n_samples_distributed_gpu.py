"""interpolate_pairs and interpolate(n_samples) with a process group on the GPU, in the two variants of
test_pipeline_distributed_gpu.py: two ranks sharing one GPU over gloo, and two GPUs over NCCL (skipped with fewer than
two).  Every rank compares its result with the single-process call made in the same process afterwards: bit for bit
with one pair (or row) per sample() call, within test_latency_gpu.py's bound in latency mode."""
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from distributed_harness import LATENCY_BOUND  # noqa: E402
from test_pipeline_distributed_gpu import VARIANTS, _init, _spawn  # noqa: E402


def _worker(rank, world, one_gpu):
    dist, dev = _init(rank, world, one_gpu)
    try:
        from test_pipeline import TINY_SIZE, keyframes, tiny_model
        from tooncrafter_b200.pipeline import ToonCrafterPipeline
        m = tiny_model(dev)
        kf = keyframes(6, seed=52)
        pairs = [(kf[2 * i], kf[2 * i + 1]) for i in range(3)]
        kw = dict(steps=3, seed=61, size=TINY_SIZE, n_samples=2)
        calls = {"pairs_uint8": lambda p: p.interpolate_pairs(pairs, pairs_per_batch=1, **kw),
                 "pairs_float": lambda p: p.interpolate_pairs(pairs, pairs_per_batch=1, output="float", **kw),
                 "variants_uint8": lambda p: p.interpolate(kf[:3], segments_per_batch=1, **kw)}
        group = ToonCrafterPipeline(m, dist.group.WORLD)
        got = {name: fn(group) for name, fn in calls.items()}
        lat = ToonCrafterPipeline(m, dist.group.WORLD, latency=True).interpolate_pairs(
            pairs, pairs_per_batch=1, output="float", **kw)
        single = ToonCrafterPipeline(m)
        ref = {name: fn(single) for name, fn in calls.items()}
        res = {f"equal_{k}": bool(got[k].shape == ref[k].shape and torch.equal(got[k], ref[k])) for k in got}
        r = ref["pairs_float"]
        res.update(latency_err=float((lat - r).abs().max()), scale=float(r.abs().max()),
                   latency_finite=bool(torch.isfinite(lat).all()), latency_sum=float(lat.double().sum()))
        return res
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize(**VARIANTS)
def test_sharded_pairs_and_variants_equal_single_process(one_gpu):
    """P = 3 pairs (blocks [0, 1] / [2]) with n = 2, uint8 and float, and K = 3 with n = 2 (four rows, blocks of
    two), one pair or row per call: bit for bit; latency mode (one GPU pair) within the bound, same on both ranks."""
    res = _spawn(_worker, one_gpu, 900)
    for r in range(2):
        assert all(v for k, v in res[r].items() if k.startswith("equal_")), res[r]
        assert res[r]["latency_finite"] and res[r]["latency_err"] <= LATENCY_BOUND * res[r]["scale"], res[r]
    assert res[0]["latency_sum"] == res[1]["latency_sum"]

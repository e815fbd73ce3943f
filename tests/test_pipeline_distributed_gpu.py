"""ToonCrafterPipeline with a process group on the GPU, in the two variants of test_latency_gpu.py: two ranks sharing
one GPU over gloo (collectives staged through host memory), and two GPUs over NCCL (skipped with fewer than two).
Every rank compares its returned video with the single-process pipeline run in the same process afterwards: equal bit
for bit with segments_per_batch=1, within test_latency_gpu.py's bound in latency mode.  The full-size case runs on two
GPUs only."""
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from distributed_harness import LATENCY_BOUND, spawn  # noqa: E402

VARIANTS = dict(argnames="one_gpu", argvalues=[True, False], ids=["two_ranks_on_one_gpu_gloo", "two_gpus_nccl"])


def _init(rank, world, one_gpu):
    import torch.distributed as dist
    dev = torch.device("cuda", 0 if one_gpu else rank)
    torch.cuda.set_device(dev)
    if one_gpu:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    else:
        dist.init_process_group("nccl", device_id=dev)
    torch.backends.cuda.matmul.allow_tf32 = False
    return dist, dev


def _tiny_worker(rank, world, one_gpu):
    dist, dev = _init(rank, world, one_gpu)
    try:
        from test_pipeline import TINY_SIZE, keyframes, tiny_model
        from tooncrafter_b200.pipeline import ToonCrafterPipeline
        m = tiny_model(dev)
        kf = keyframes(3, seed=51)
        kw = dict(steps=3, seed=60, size=TINY_SIZE, segments_per_batch=1)
        pipe = ToonCrafterPipeline(m, dist.group.WORLD)
        got = {o: pipe.interpolate(kf, output=o, **kw) for o in ("uint8", "float")}
        lat = ToonCrafterPipeline(m, dist.group.WORLD, latency=True).interpolate(kf, output="float", **kw)
        single = ToonCrafterPipeline(m)
        ref = {o: single.interpolate(kf, output=o, **kw) for o in ("uint8", "float")}
        res = {f"equal_{o}": bool(got[o].shape == ref[o].shape and torch.equal(got[o], ref[o])) for o in got}
        res.update(latency_err=float((lat - ref["float"]).abs().max()), scale=float(ref["float"].abs().max()),
                   latency_finite=bool(torch.isfinite(lat).all()), latency_sum=float(lat.double().sum()))
        return res
    finally:
        dist.destroy_process_group()


def _full_size_worker(rank, world, one_gpu):
    dist, dev = _init(rank, world, one_gpu)
    try:
        from test_pipeline import keyframes
        from tiny_config import FULL_DDCONFIG, FULL_UNET, model_config
        from tooncrafter_b200 import synthetic
        from tooncrafter_b200.interpolate import rewrite_targets
        from tooncrafter_b200.pipeline import ToonCrafterPipeline
        cfg = model_config(FULL_UNET, FULL_DDCONFIG)
        p = cfg["params"]
        p["cond_stage_config"] = {"target": "lvdm.modules.encoders.condition.FrozenOpenCLIPEmbedder",
                                  "params": {"freeze": True, "layer": "penultimate"}}
        p["img_cond_stage_config"] = {"target": "lvdm.modules.encoders.condition.FrozenOpenCLIPImageEmbedderV2",
                                      "params": {"freeze": True}}
        p["image_proj_stage_config"] = {"target": "lvdm.modules.encoders.resampler.Resampler",
                                        "params": dict(dim=1024, depth=4, dim_head=64, heads=12, num_queries=16,
                                                       embedding_dim=1280, output_dim=1024, ff_mult=4,
                                                       video_length=16)}
        m = synthetic.synthetic_model(rewrite_targets(cfg), dev)
        m.perframe_ae = True
        kf = [keyframes(1, (320, 512), seed=s)[0].numpy() for s in (4, 5, 6)]
        kw = dict(steps=2, segments_per_batch=1, output="float")
        got = ToonCrafterPipeline(m, dist.group.WORLD).interpolate(kf, **kw)
        ref = ToonCrafterPipeline(m).interpolate(kf, **kw)
        return dict(equal=bool(got.shape == ref.shape and torch.equal(got, ref)),
                    finite=bool(torch.isfinite(got).all()), shape=tuple(got.shape))
    finally:
        dist.destroy_process_group()


def _spawn(worker, one_gpu, timeout):
    """Run worker(rank, 2, one_gpu) on two ranks; {rank: its result dict}."""
    if not one_gpu and torch.cuda.device_count() < 2:
        pytest.skip("the NCCL variant shards over two GPUs")
    res = spawn(worker, one_gpu, world=2, timeout=timeout)
    print(worker.__name__, res)
    return res


@pytest.mark.gpu
@pytest.mark.parametrize(**VARIANTS)
def test_sharded_pipeline_equals_single_process(one_gpu):
    """Tiny model, K = 3 (blocks [0] / [1]), segments_per_batch=1: uint8 and float bit for bit; latency mode (one pair
    samples both segments) within the bound of the pair's sampler test, and the same on both ranks."""
    res = _spawn(_tiny_worker, one_gpu, 900)
    for r in range(2):
        assert res[r]["equal_uint8"] and res[r]["equal_float"], res[r]
        assert res[r]["latency_finite"] and res[r]["latency_err"] <= LATENCY_BOUND * res[r]["scale"], res[r]
    assert res[0]["latency_sum"] == res[1]["latency_sum"]


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_sharded_pipeline_full_size_k3_ddim2_on_two_gpus():
    """Full-size synthetic weights at 320 x 512, K = 3, DDIM-2, segments_per_batch=1: bit for bit the one-GPU run.
    Two GPUs only: two full-size models and their plans do not fit on one 80 GB card together."""
    res = _spawn(_full_size_worker, False, 1700)
    for r in range(2):
        assert res[r]["shape"] == (2, 3, 16, 320, 512) and res[r]["finite"] and res[r]["equal"], res[r]

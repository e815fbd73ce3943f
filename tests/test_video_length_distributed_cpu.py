"""ToonCrafterPipeline with a process group at a clip length other than the model's temporal_length, on the CPU
program interpreter: two gloo ranks run the tiny model of test_pipeline.py at T = 8 frames per segment, and every
rank's returned video is compared with the single-process call that rank 0 makes afterwards.

Sharding with segments_per_batch=1 is the single-process computation segment by segment, so it must be equal bit for
bit.  Latency mode samples each guidance branch as its own B = 1 program (the single-process call batches them), so it
is held to the bound test_pipeline_distributed_cpu.py applies to that mode."""
import os
import sys
import traceback
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from test_pipeline import TINY_SIZE, _scale_close, keyframes, tiny_model  # noqa: E402
from tooncrafter_b200 import runtime  # noqa: E402
from tooncrafter_b200.pipeline import ToonCrafterPipeline  # noqa: E402

T = 8
CASES = {"k3_loop_u8": (3, dict(segments_per_batch=1, loop=True))}      # blocks [0, 1] / [2], the closing seam
LATENCY_BOUND = 3e-2


def _interpolate(pipe, K, kw):
    return pipe.interpolate(keyframes(K), steps=2, seed=123, size=TINY_SIZE, video_length=T, **kw)


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    import pipeline_emulator
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        runtime.TEST_EXECUTOR = pipeline_emulator.executor
        m = tiny_model()
        res = {}
        pipe = ToonCrafterPipeline(m, dist.group.WORLD)
        for name, (K, kw) in CASES.items():
            res[name] = _interpolate(pipe, K, kw).numpy()
        lat = ToonCrafterPipeline(m, dist.group.WORLD, latency=True)
        res["latency_k4_float"] = _interpolate(lat, 4, dict(segments_per_batch=1, output="float")).numpy()
        if rank == 0:
            single = ToonCrafterPipeline(m)
            for name, (K, kw) in CASES.items():
                res["single_" + name] = _interpolate(single, K, kw).numpy()
            res["single_k4_float"] = _interpolate(single, 4, dict(segments_per_batch=1, output="float")).numpy()
        out.put((rank, res))
    except BaseException:
        out.put((rank, traceback.format_exc()))
        raise
    finally:
        runtime.TEST_EXECUTOR = None
        dist.destroy_process_group()


def _free_port():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.fixture(scope="module")
def sharded():
    """{case: [rank 0's result, rank 1's result]}; "single_<case>": [the single-process call]."""
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = dict(q.get(timeout=2400) for _ in range(world))
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    for r in range(world):
        assert isinstance(got[r], dict), f"rank {r} failed:\n{got[r]}"
    assert all(p.exitcode == 0 for p in procs)
    return {name: [torch.from_numpy(got[r][name]) for r in range(world) if name in got[r]] for name in got[0]}


@pytest.mark.parametrize("case", list(CASES))
def test_sharded_video_length_equals_single_process(sharded, case):
    ref, = sharded["single_" + case]
    K, kw = CASES[case]
    S = K if kw.get("loop") else K - 1
    expect = (S, 3, T, *TINY_SIZE) if kw.get("output") == "float" else ((T - 1) * S + (0 if kw.get("loop") else 1),
                                                                         *TINY_SIZE, 3)
    assert tuple(ref.shape) == expect
    for r, got in enumerate(sharded[case]):
        assert got.shape == ref.shape and got.dtype == ref.dtype, (case, r)
        assert torch.equal(got, ref), f"{case}: rank {r} differs from the single-process call"


def test_latency_mode_video_length_matches_single_process(sharded):
    ref, = sharded["single_k4_float"]
    a, b = sharded["latency_k4_float"]
    assert torch.equal(a, b), "the two ranks of the pair returned different videos"
    assert a.shape == ref.shape == (3, 3, T, *TINY_SIZE)
    _scale_close(a, ref, "latency mode K=4, T=8 vs single process", rel=LATENCY_BOUND)

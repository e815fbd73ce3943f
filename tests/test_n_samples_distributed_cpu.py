"""Variants and keyframe-pair directories with a process group, on the CPU program interpreter: two gloo ranks run
the tiny model of test_pipeline.py, and every rank's returned tensor is compared with the single-process call that
rank 0 makes afterwards (in a process with the same thread count: CPU matmuls round differently at other counts).

interpolate(n_samples=3) on K = 2 has three rows, split into blocks [0, 1] / [2]; interpolate_pairs on P = 3 pairs
splits them into [0, 1] / [2].  With one row (or pair) per sample() call that is the single-process computation row by
row, so it must be equal bit for bit.  Latency mode samples each guidance branch as its own program (the
single-process call batches them), so it is held to the bound test_pipeline_distributed_cpu.py applies to that mode;
both ranks of the pair must still return the same bits."""
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

LATENCY_BOUND = 3e-2


def _variants(pipe, output):
    return pipe.interpolate(keyframes(2, seed=8), steps=1, seed=21, size=TINY_SIZE, n_samples=3,
                            segments_per_batch=1, output=output)


def _pairs(pipe, output):
    kf = keyframes(6, seed=9)
    return pipe.interpolate_pairs([(kf[2 * i], kf[2 * i + 1]) for i in range(3)], n_samples=2, steps=1, seed=33,
                                  size=TINY_SIZE, pairs_per_batch=1, output=output)


CASES = {"variants_u8": (_variants, "uint8"), "variants_float": (_variants, "float"),
         "pairs_u8": (_pairs, "uint8"), "pairs_float": (_pairs, "float")}


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
        for name, (fn, output) in CASES.items():
            res[name] = fn(pipe, output).numpy()
        lat = ToonCrafterPipeline(m, dist.group.WORLD, latency=True)
        res["latency_variants_float"] = _variants(lat, "float").numpy()
        res["latency_pairs_float"] = _pairs(lat, "float").numpy()
        if rank == 0:
            single = ToonCrafterPipeline(m)
            for name, (fn, output) in CASES.items():
                res["single_" + name] = fn(single, output).numpy()
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
def test_sharded_rows_and_pairs_equal_single_process(sharded, case):
    ref, = sharded["single_" + case]
    expect = {"variants_u8": (3, 4, *TINY_SIZE, 3), "variants_float": (3, 1, 3, 4, *TINY_SIZE),
              "pairs_u8": (3, 2, 4, *TINY_SIZE, 3), "pairs_float": (3, 2, 3, 4, *TINY_SIZE)}[case]
    assert tuple(ref.shape) == expect
    for r, got in enumerate(sharded[case]):
        assert got.shape == ref.shape and got.dtype == ref.dtype, (case, r)
        assert torch.equal(got, ref), f"{case}: rank {r} differs from the single-process call"


@pytest.mark.parametrize("case", ["variants_float", "pairs_float"])
def test_latency_mode_rows_and_pairs_match_single_process(sharded, case):
    ref, = sharded["single_" + case]
    a, b = sharded["latency_" + case]
    assert torch.equal(a, b), "the two ranks of the pair returned different results"
    assert a.shape == ref.shape
    _scale_close(a, ref, f"latency mode {case} vs single process", rel=LATENCY_BOUND)

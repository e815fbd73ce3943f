"""refine with a process group, on the CPU program interpreter: two gloo ranks run the tiny model of test_pipeline.py,
and every rank's result is compared with the single-process call that rank 0 makes afterwards (in a process with the
same thread count: CPU matmuls round differently at other counts).

refine(n_samples=3, keep=...) has three rows, split into blocks [0, 1] / [2]; with one row per sample() call that is the
single-process computation row by row, so it must be equal bit for bit.  Latency mode samples each guidance branch as
its own program, so it is held to the bound test_pipeline_distributed_cpu.py applies to that mode."""
import os
import sys
import traceback
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from test_n_samples_distributed_cpu import LATENCY_BOUND, _free_port  # noqa: E402
from test_pipeline import TINY_SIZE, _scale_close, keyframes, tiny_model  # noqa: E402
from tooncrafter_b200 import runtime  # noqa: E402
from tooncrafter_b200.pipeline import ToonCrafterPipeline  # noqa: E402


def _refine(pipe, output):
    return pipe.refine(keyframes(8, seed=12), 0.5, keep=[0, 1, 7], steps=2, seed=21, size=TINY_SIZE, n_samples=3,
                       segments_per_batch=1, output=output)


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    import refine_emulator
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        runtime.TEST_EXECUTOR = refine_emulator.executor
        m = tiny_model()
        pipe = ToonCrafterPipeline(m, dist.group.WORLD)
        res = {"u8": _refine(pipe, "uint8").numpy(), "float": _refine(pipe, "float").numpy(),
               "latency": _refine(ToonCrafterPipeline(m, dist.group.WORLD, latency=True), "float").numpy()}
        if rank == 0:
            single = ToonCrafterPipeline(m)
            res["single_u8"], res["single_float"] = _refine(single, "uint8").numpy(), _refine(single, "float").numpy()
        out.put((rank, res))
    except BaseException:
        out.put((rank, traceback.format_exc()))
        raise
    finally:
        runtime.TEST_EXECUTOR = None
        dist.destroy_process_group()


@pytest.fixture(scope="module")
def sharded():
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


@pytest.mark.parametrize("case", ["u8", "float"])
def test_sharded_refine_equals_single_process(sharded, case):
    ref, = sharded["single_" + case]
    assert tuple(ref.shape) == ((3, 8, *TINY_SIZE, 3) if case == "u8" else (3, 3, 8, *TINY_SIZE))
    for r, got in enumerate(sharded[case]):
        assert torch.equal(got, ref), f"{case}: rank {r} differs from the single-process call"


def test_latency_mode_refine_matches_single_process(sharded):
    ref, = sharded["single_float"]
    a, b = sharded["latency"]
    assert torch.equal(a, b), "the two ranks of the pair returned different results"
    _scale_close(a, ref, "latency mode refine vs single process", rel=LATENCY_BOUND)

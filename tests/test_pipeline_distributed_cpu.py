"""ToonCrafterPipeline with a process group, on the CPU program interpreter: two gloo ranks spawned by this file run the
tiny model of test_pipeline.py, and every rank's returned video is compared with the single-process call, which rank 0
makes afterwards (in a process with the same thread count: CPU matmuls round differently at other thread counts).

With segments_per_batch=1 a sharded call is the single-process computation segment by segment (same per-segment
generators, same tower and encoder batches, same B = 1 sampling), so its output must be equal bit for bit.  Other
batchings and latency mode change the batch rows of the UNet program and are held to the bounds the single-process
tests apply to those."""
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

# name -> (K, interpolate kwargs); K = 4 splits S = 3 segments into blocks [0, 1] / [2], as does K = 3 with loop
CASES = {
    "k4_u8": (4, dict(segments_per_batch=1)),
    "k4_float": (4, dict(segments_per_batch=1, output="float")),
    "k3_loop_u8": (3, dict(segments_per_batch=1, loop=True)),
    "k3_loop_float": (3, dict(segments_per_batch=1, loop=True, output="float")),
    "k4_default_batch_float": (4, dict(output="float")),
}
LATENCY_BOUND = 3e-2          # of the output scale: test_latency_gpu.py's bound for the pair against the fused path


def _interpolate(pipe, K, kw):
    return pipe.interpolate(keyframes(K), steps=2, seed=123, size=TINY_SIZE, **kw)


def _animate(pipe):
    return pipe.animate(keyframes(1, seed=5)[0], steps=2, seed=77, size=TINY_SIZE)


def _refusal(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001 - the type and message are what the test checks
        return type(e).__name__, str(e)
    return None


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist

    import pipeline_emulator
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        runtime.TEST_EXECUTOR = pipeline_emulator.executor
        m = tiny_model()
        group = dist.group.WORLD
        res = {}
        pipe = ToonCrafterPipeline(m, group)
        for name, (K, kw) in CASES.items():
            res[name] = _interpolate(pipe, K, kw).numpy()
        res["animate"] = _animate(pipe).numpy()
        lat = ToonCrafterPipeline(m, group, latency=True)
        res["latency_k4_float"] = _interpolate(lat, 4, dict(segments_per_batch=1, output="float")).numpy()
        res["latency_animate"] = _animate(lat).numpy()
        res["refuse_cfg_img"] = _refusal(lambda: _interpolate(lat, 3, dict(cfg_img=5.0)))
        res["refuse_cfg_scale_1"] = _refusal(lambda: _interpolate(lat, 3, dict(cfg_scale=1.0)))
        res["refuse_no_group"] = _refusal(lambda: ToonCrafterPipeline(m, latency=True))
        one = dist.new_group(ranks=[0])                       # a group of odd size (collective: every rank calls it)
        if rank == 0:
            res["refuse_odd_world"] = _refusal(lambda: ToonCrafterPipeline(m, one, latency=True))
        # group=None with torch.distributed initialised: the single-process call, no collective
        res["no_group"] = _interpolate(ToonCrafterPipeline(m), 4, dict(segments_per_batch=1, output="float")).numpy()
        if rank == 0:
            single = ToonCrafterPipeline(m)
            for name, (K, kw) in CASES.items():
                res["single_" + name] = _interpolate(single, K, kw).numpy()
            res["single_animate"] = _animate(single).numpy()
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
    """{case: [rank 0's result, rank 1's result]} of one world-2 session; "single_<case>": [the single-process call]."""
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
    return {name: [torch.from_numpy(got[r][name]) if hasattr(got[r][name], "dtype") else got[r][name]
                   for r in range(world) if name in got[r]] for name in got[0]}


@pytest.mark.parametrize("case", [c for c in CASES if "default" not in c])
def test_sharded_segments_equal_single_process(sharded, case):
    ref, = sharded["single_" + case]
    for r, got in enumerate(sharded[case]):
        assert got.shape == ref.shape and got.dtype == ref.dtype, (case, r)
        assert torch.equal(got, ref), f"{case}: rank {r} differs from the single-process call"


def test_sharded_default_batching_matches_single_process(sharded):
    """Default segments_per_batch (4): the single-process call samples the 3 segments as one batch, the ranks as
    batches of 2 and 1 (the bound of the RNG-contract tests)."""
    ref, = sharded["single_k4_default_batch_float"]
    a, b = sharded["k4_default_batch_float"]
    assert torch.equal(a, b)
    _scale_close(a, ref, "K=4 default batching, world 2 vs single process")


def test_sharded_animate_equals_single_process(sharded):
    ref, = sharded["single_animate"]
    for r, got in enumerate(sharded["animate"]):
        assert torch.equal(got, ref), f"animate: rank {r} differs from the single-process call"


def test_latency_mode_matches_single_process(sharded):
    """One GPU pair samples all 3 segments, one guidance branch per rank; pair-rank 0 decodes and broadcasts."""
    ref, = sharded["single_k4_float"]
    a, b = sharded["latency_k4_float"]
    assert torch.equal(a, b), "the two ranks of the pair returned different videos"
    _scale_close(a, ref, "latency mode K=4 vs single process", rel=LATENCY_BOUND)
    ref, = sharded["single_animate"]
    a, b = sharded["latency_animate"]
    assert torch.equal(a, b) and a.shape == ref.shape
    _scale_close(a, ref, "latency mode animate vs single process", rel=LATENCY_BOUND)


def test_latency_mode_refusals(sharded):
    for r in range(2):
        kind, msg = sharded["refuse_cfg_img"][r]
        assert kind == "NotImplementedError" and "cfg_img" in msg
        kind, msg = sharded["refuse_cfg_scale_1"][r]
        assert kind == "ValueError" and "cfg_scale 1.0" in msg
        kind, msg = sharded["refuse_no_group"][r]
        assert kind == "ValueError" and "process group" in msg
    kind, msg = sharded["refuse_odd_world"][0]
    assert kind == "ValueError" and "even" in msg


def test_no_group_is_the_single_process_call(sharded):
    """group=None with torch.distributed initialised makes no collective and gives the single-process result."""
    ref, = sharded["single_k4_float"]
    for got in sharded["no_group"]:
        assert torch.equal(got, ref)

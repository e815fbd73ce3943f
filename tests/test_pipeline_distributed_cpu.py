"""ToonCrafterPipeline with a process group, on the CPU program interpreter: one session of two gloo ranks runs the tiny
model of test_pipeline.py through interpolate (also at T = 8 frames per segment), animate, variants, interpolate_pairs
and refine, and every rank's result is compared with the single-process call, which rank 0 makes afterwards (in a
process with the same thread count: CPU matmuls round differently at other thread counts).

With one row (or pair) per sample() call a sharded call is the single-process computation row by row (same per-row
generators, same tower and encoder batches, same B = 1 sampling), so its output must be equal bit for bit.  Other
batchings change the batch rows of the UNet program and are held to the bound the single-process tests apply to those;
latency mode samples each guidance branch as its own program and is held to LATENCY_BOUND, both ranks of the pair
returning the same bits."""
import os
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from distributed_harness import LATENCY_BOUND, spawn  # noqa: E402
from test_pipeline import TINY_SIZE, _scale_close, keyframes, tiny_model  # noqa: E402
from tooncrafter_b200 import runtime  # noqa: E402
from tooncrafter_b200.pipeline import ToonCrafterPipeline  # noqa: E402

T8 = 8


def _interpolate(K, **kw):
    return lambda pipe: pipe.interpolate(keyframes(K), steps=2, seed=123, size=TINY_SIZE, **kw)


def _animate(pipe):
    return pipe.animate(keyframes(1, seed=5)[0], steps=2, seed=77, size=TINY_SIZE)


def _variants(output):
    """n_samples=3 on K = 2: three rows, blocks [0, 1] / [2]."""
    return lambda pipe: pipe.interpolate(keyframes(2, seed=8), steps=1, seed=21, size=TINY_SIZE, n_samples=3,
                                         segments_per_batch=1, output=output)


def _pairs(output):
    """P = 3 pairs, blocks [0, 1] / [2]."""
    def call(pipe):
        kf = keyframes(6, seed=9)
        return pipe.interpolate_pairs([(kf[2 * i], kf[2 * i + 1]) for i in range(3)], n_samples=2, steps=1, seed=33,
                                      size=TINY_SIZE, pairs_per_batch=1, output=output)
    return call


def _refine(output):
    """n_samples=3 with keep: three rows, blocks [0, 1] / [2]."""
    return lambda pipe: pipe.refine(keyframes(8, seed=12), 0.5, keep=[0, 1, 7], steps=2, seed=21, size=TINY_SIZE,
                                    n_samples=3, segments_per_batch=1, output=output)


# name -> call, made on the sharded pipeline and by rank 0 on the single-process one; K = 4 splits S = 3 segments into
# blocks [0, 1] / [2], as does K = 3 with loop (with the closing seam)
CASES = {
    "k4_u8": _interpolate(4, segments_per_batch=1),
    "k4_float": _interpolate(4, segments_per_batch=1, output="float"),
    "k3_loop_u8": _interpolate(3, segments_per_batch=1, loop=True),
    "k3_loop_float": _interpolate(3, segments_per_batch=1, loop=True, output="float"),
    "k4_default_batch_float": _interpolate(4, output="float"),
    "animate": _animate,
    "t8_k3_loop_u8": _interpolate(3, segments_per_batch=1, loop=True, video_length=T8),
    "variants_u8": _variants("uint8"), "variants_float": _variants("float"),
    "pairs_u8": _pairs("uint8"), "pairs_float": _pairs("float"),
    "refine_u8": _refine("uint8"), "refine_float": _refine("float"),
}
# name -> call, made on the latency-mode pipeline; its single-process reference is CASES[name] or SINGLE[name]
LATENCY = {"k4_float": CASES["k4_float"], "animate": _animate,
           "t8_k4_float": _interpolate(4, segments_per_batch=1, output="float", video_length=T8),
           "variants_float": CASES["variants_float"], "pairs_float": CASES["pairs_float"],
           "refine_float": CASES["refine_float"]}
SINGLE = {"t8_k4_float": LATENCY["t8_k4_float"]}


def _refusal(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001 - the type and message are what the test checks
        return type(e).__name__, str(e)
    return None


def _worker(rank, world):
    import torch.distributed as dist

    import clip_emulator
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        runtime.TEST_EXECUTOR = clip_emulator.executor
        m = tiny_model()
        group = dist.group.WORLD
        pipe = ToonCrafterPipeline(m, group)
        res = {name: fn(pipe).numpy() for name, fn in CASES.items()}
        lat = ToonCrafterPipeline(m, group, latency=True)
        res.update({"latency_" + name: fn(lat).numpy() for name, fn in LATENCY.items()})
        res["refuse_cfg_img"] = _refusal(lambda: _interpolate(3, cfg_img=5.0)(lat))
        res["refuse_cfg_scale_1"] = _refusal(lambda: _interpolate(3, cfg_scale=1.0)(lat))
        res["refuse_no_group"] = _refusal(lambda: ToonCrafterPipeline(m, latency=True))
        one = dist.new_group(ranks=[0])                       # a group of odd size (collective: every rank calls it)
        if rank == 0:
            res["refuse_odd_world"] = _refusal(lambda: ToonCrafterPipeline(m, one, latency=True))
        # group=None with torch.distributed initialised: the single-process call, no collective
        res["no_group"] = CASES["k4_float"](ToonCrafterPipeline(m)).numpy()
        if rank == 0:
            single = ToonCrafterPipeline(m)
            res.update({"single_" + name: fn(single).numpy() for name, fn in {**CASES, **SINGLE}.items()})
        return res
    finally:
        runtime.TEST_EXECUTOR = None
        dist.destroy_process_group()


@pytest.fixture(scope="module")
def sharded():
    """{case: [rank 0's result, rank 1's result]} of one world-2 session; "single_<case>": [the single-process call]."""
    got = spawn(_worker, world=2)
    return {name: [torch.from_numpy(got[r][name]) if hasattr(got[r][name], "dtype") else got[r][name]
                   for r in range(2) if name in got[r]] for name in got[0]}


def _check_equal(sharded, case, shape=None):
    ref, = sharded["single_" + case]
    assert shape is None or tuple(ref.shape) == shape, (case, tuple(ref.shape))
    for r, got in enumerate(sharded[case]):
        assert got.shape == ref.shape and got.dtype == ref.dtype, (case, r)
        assert torch.equal(got, ref), f"{case}: rank {r} differs from the single-process call"


def _check_latency(sharded, case):
    ref, = sharded["single_" + case]
    a, b = sharded["latency_" + case]
    assert torch.equal(a, b), "the two ranks of the pair returned different results"
    assert a.shape == ref.shape
    _scale_close(a, ref, f"latency mode {case} vs single process", rel=LATENCY_BOUND)


@pytest.mark.parametrize("case", ["k4_u8", "k4_float", "k3_loop_u8", "k3_loop_float"])
def test_sharded_segments_equal_single_process(sharded, case):
    _check_equal(sharded, case)


def test_sharded_default_batching_matches_single_process(sharded):
    """Default segments_per_batch (4): the single-process call samples the 3 segments as one batch, the ranks as
    batches of 2 and 1 (the bound of the RNG-contract tests)."""
    ref, = sharded["single_k4_default_batch_float"]
    a, b = sharded["k4_default_batch_float"]
    assert torch.equal(a, b)
    _scale_close(a, ref, "K=4 default batching, world 2 vs single process")


def test_sharded_animate_equals_single_process(sharded):
    _check_equal(sharded, "animate")


def test_latency_mode_matches_single_process(sharded):
    """One GPU pair samples all 3 segments, one guidance branch per rank; pair-rank 0 decodes and broadcasts."""
    _check_latency(sharded, "k4_float")
    _check_latency(sharded, "animate")


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


@pytest.mark.parametrize("case", ["k3_loop_u8"])
def test_sharded_video_length_equals_single_process(sharded, case):
    """At a clip length other than the model's temporal_length."""
    _check_equal(sharded, "t8_" + case, ((T8 - 1) * 3, *TINY_SIZE, 3))


def test_latency_mode_video_length_matches_single_process(sharded):
    _check_latency(sharded, "t8_k4_float")
    assert sharded["latency_t8_k4_float"][0].shape == (3, 3, T8, *TINY_SIZE)


@pytest.mark.parametrize("case", ["variants_u8", "variants_float", "pairs_u8", "pairs_float"])
def test_sharded_rows_and_pairs_equal_single_process(sharded, case):
    expect = {"variants_u8": (3, 4, *TINY_SIZE, 3), "variants_float": (3, 1, 3, 4, *TINY_SIZE),
              "pairs_u8": (3, 2, 4, *TINY_SIZE, 3), "pairs_float": (3, 2, 3, 4, *TINY_SIZE)}[case]
    _check_equal(sharded, case, expect)


@pytest.mark.parametrize("case", ["variants_float", "pairs_float"])
def test_latency_mode_rows_and_pairs_match_single_process(sharded, case):
    _check_latency(sharded, case)


@pytest.mark.parametrize("case", ["u8", "float"])
def test_sharded_refine_equals_single_process(sharded, case):
    _check_equal(sharded, "refine_" + case, (3, 8, *TINY_SIZE, 3) if case == "u8" else (3, 3, 8, *TINY_SIZE))


def test_latency_mode_refine_matches_single_process(sharded):
    _check_latency(sharded, "refine_float")

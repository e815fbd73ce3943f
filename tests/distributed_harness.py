"""TEST INFRASTRUCTURE — spawned process groups for the distributed tests.

`spawn` runs a worker function on every rank of a fresh world, each in its own spawned process, and returns what the
workers returned; the workers initialise and destroy their own process group (gloo on CPU, gloo or NCCL on the GPU).
"""
from __future__ import annotations

import os
import socket
import traceback

# Bound of latency mode against the single-process call, as a share of the output scale: test_latency_gpu.py's bound
# for the pair against the fused path (the pair samples each guidance branch as its own program).
LATENCY_BOUND = 3e-2


def _free_port() -> int:
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(worker, rank, world, port, out, args):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    try:
        out.put((rank, worker(rank, world, *args), None))
    except BaseException:
        out.put((rank, None, traceback.format_exc()))
        raise


def spawn(worker, *args, world: int = 2, timeout: float = 2400) -> dict:
    """worker(rank, world, *args) on `world` spawned ranks (MASTER_ADDR, MASTER_PORT, RANK and WORLD_SIZE set);
    {rank: its return value}.  A rank that raised fails the caller with its traceback."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_run, args=(worker, r, world, port, q, args)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = [q.get(timeout=timeout) for _ in procs]
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    for rank, _, error in got:
        assert error is None, f"rank {rank} failed:\n{error}"
    assert all(p.exitcode == 0 for p in procs)
    return {rank: res for rank, res, _ in got}

"""Host runtime shared by the network engines: activation pool, activation views, recorded programs, and the engine
lifecycle (weight fingerprint, plan cache, execution).

Design (H100-first): every network is executed as a STATIC program — a flat list of C-ABI kernel launches over
pre-allocated channels-last fp16 buffers carved out of one HBM arena — built once per input geometry and then
replayed, either launch-by-launch or as a captured CUDA graph (no per-step Python/allocator work, no
`rearrange().contiguous()` copies: spatial tokens, temporal tokens and conv pixels are all views of the same
[B][T][H][W][C] buffer).
"""
from __future__ import annotations

import bisect
from dataclasses import dataclass
from typing import Callable, List, Optional

import torch

# TESTS ONLY.  tests/ops_emulator.executor is installed here by host-logic tests that drive the public API (samplers,
# UNetModel.forward, AutoencoderKL.encode / decode) without a GPU: engines are then built plan-only and their recorded
# programs are interpreted in PyTorch instead of launched.  The product never sets it; with it unset a CPU module still
# raises ("CUDA only, no CPU fallback").
TEST_EXECUTOR: Optional[Callable] = None


class Arena:
    """First-fit allocator with coalescing over one device buffer (used only while a program is being built)."""

    ALIGN = 1024

    def __init__(self, nbytes: int, device):
        self.buf = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self.free_blocks = [(0, nbytes)]       # sorted (offset, size)
        self.live = {}
        self.high_water = 0
        self.in_use = 0

    def alloc(self, nbytes: int) -> int:
        nbytes = (max(nbytes, 1) + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        for i, (off, size) in enumerate(self.free_blocks):
            if size >= nbytes:
                if size == nbytes:
                    self.free_blocks.pop(i)
                else:
                    self.free_blocks[i] = (off + nbytes, size - nbytes)
                self.live[off] = nbytes
                self.in_use += nbytes
                self.high_water = max(self.high_water, off + nbytes)
                return off
        raise MemoryError(f"activation arena exhausted: need {nbytes} bytes, in use {self.in_use} of "
                          f"{self.buf.numel()}")

    def free(self, off: int) -> None:
        size = self.live.pop(off)
        self.in_use -= size
        i = bisect.bisect_left(self.free_blocks, (off, 0))
        self.free_blocks.insert(i, (off, size))
        # coalesce with neighbours
        if i + 1 < len(self.free_blocks) and self.free_blocks[i][0] + self.free_blocks[i][1] == self.free_blocks[i + 1][0]:
            o, s = self.free_blocks[i]
            self.free_blocks[i] = (o, s + self.free_blocks[i + 1][1])
            self.free_blocks.pop(i + 1)
        if i > 0 and self.free_blocks[i - 1][0] + self.free_blocks[i - 1][1] == self.free_blocks[i][0]:
            o, s = self.free_blocks[i - 1]
            self.free_blocks[i - 1] = (o, s + self.free_blocks[i][1])
            self.free_blocks.pop(i)

    def tensor(self, off: int, numel: int, dtype=torch.float16) -> torch.Tensor:
        esize = torch.empty((), dtype=dtype).element_size()
        return self.buf[off:off + numel * esize].view(dtype)


@dataclass
class Act:
    """A channels-last activation view: rows = N*H*W pixels, C channels at element offset `off`, row stride `ld`."""
    t: torch.Tensor          # backing fp16 tensor (flat)
    N: int
    H: int
    W: int
    C: int
    ld: int
    off: int = 0             # element offset of channel 0 inside the backing tensor
    arena_off: Optional[int] = None
    arena: Optional[Arena] = None

    @property
    def rows(self) -> int:
        return self.N * self.H * self.W

    def slice(self, c0: int, c: int) -> "Act":
        return Act(self.t, self.N, self.H, self.W, c, self.ld, self.off + c0)

    def free(self) -> None:
        if self.arena is not None and self.arena_off is not None:
            self.arena.free(self.arena_off)
            self.arena_off = None

    def as_torch(self) -> torch.Tensor:
        """[N, H, W, C] strided torch view (debug / tests only)."""
        return torch.as_strided(self.t, (self.N, self.H, self.W, self.C), (self.H * self.W * self.ld, self.W * self.ld,
                                                                         self.ld, 1),
                                self.t.storage_offset() + self.off)


class Program:
    """Recorded list of kernel launches; `run()` replays them on the current stream, `graph()` captures them."""

    def __init__(self):
        self.calls: List = []
        self._graph: Optional[torch.cuda.CUDAGraph] = None

    def add(self, fn: Callable, *args, **kw) -> None:
        self.calls.append((fn, args, kw))

    def run(self, executor: Optional[Callable] = None) -> None:
        """Issue every recorded launch; `executor(fn, args, kw)` lets tests interpret the program instead."""
        if executor is not None:
            for fn, args, kw in self.calls:
                executor(fn, args, kw)
            return
        for fn, args, kw in self.calls:
            fn(*args, **kw)

    def __len__(self):
        return len(self.calls)

    def replay(self, use_graph: bool) -> None:
        if not use_graph:
            self.run()
            return
        if self._graph is None:
            # warm up on a side stream, then capture
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                self.run()
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self.run()
            self._graph = g
        self._graph.replay()


class Builder:
    """Allocation + recording context handed to the layer builders."""

    def __init__(self, arena: Arena, prog: Program):
        self.arena = arena
        self.prog = prog

    def act(self, N: int, H: int, W: int, C: int) -> Act:
        off = self.arena.alloc(N * H * W * C * 2)
        return Act(self.arena.tensor(off, N * H * W * C), N, H, W, C, C, 0, off, self.arena)

    def raw(self, numel: int, dtype=torch.float16):
        off = self.arena.alloc(numel * torch.empty((), dtype=dtype).element_size())
        return self.arena.tensor(off, numel, dtype), off

    def free_raw(self, off: int) -> None:
        self.arena.free(off)

    def op(self, fn: Callable, *args, **kw) -> None:
        self.prog.add(fn, *args, **kw)


def weights_signature(*modules: torch.nn.Module):
    """Fingerprint of EVERY parameter and buffer (storage address + in-place version counter).  The modules keep their
    tensors alive, so an address cannot be recycled while the signature is current; a partial load_state_dict, a LoRA
    merge or an edit of a late block all bump a version counter and force a re-pack."""
    return tuple((t.data_ptr(), t._version) for m in modules for t in list(m.parameters()) + list(m.buffers()))


class Engine:
    """Lifecycle shared by the network engines: weights packed once from a holder module, one recorded program per
    input geometry (`plan_for(*key)` -> the subclass's `_build(*key)`, cached in `_plans`), executed by `_execute`.

    plan_only=True builds programs without a GPU (host-logic tests interpret them through an executor); such an engine
    cannot launch anything."""

    def __init__(self, holder: torch.nn.Module, device=None, use_graph: bool = False, plan_only: bool = False):
        modules = self._weights(holder)
        self.dev = torch.device(device) if device is not None else next(modules[0].parameters()).device
        self.plan_only = plan_only
        if self.dev.type != "cuda" and not plan_only:
            raise RuntimeError("tooncrafter_b200 runs on CUDA only (no CPU fallback); move the model to a GPU")
        self._sig = weights_signature(*modules)
        self.use_graph = use_graph
        self._plans: dict = {}

    @staticmethod
    def _weights(holder: torch.nn.Module):
        """The modules whose weights the engine packs from `holder`."""
        return (holder,)

    def matches(self, holder: torch.nn.Module) -> bool:
        """True while no weight of `holder` was replaced, moved or written in place since packing."""
        modules = self._weights(holder)
        return next(modules[0].parameters()).device == self.dev and self._sig == weights_signature(*modules)

    @classmethod
    def cached(cls, holder: torch.nn.Module, attr: str, executor: Optional[Callable] = None,
               module: Optional[torch.nn.Module] = None):
        """The engine of `module` (default: `holder`) stored in `holder.<attr>`, (re)built when missing or stale;
        plan-only when an executor will interpret its programs."""
        module = holder if module is None else module
        eng = getattr(holder, attr)
        if eng is None or not eng.matches(module):
            eng = cls(module, plan_only=executor is not None)
            setattr(holder, attr, eng)
        return eng

    def plan_for(self, *key):
        if key not in self._plans:
            self._plans[key] = self._build(*key)
        return self._plans[key]

    def _execute(self, prog: Program, executor: Optional[Callable] = None, use_graph: bool = False) -> None:
        """Interpret `prog` through `executor` (tests), or launch it: as a captured CUDA graph when `use_graph`."""
        if executor is not None:
            prog.run(executor)
        elif self.plan_only:
            raise RuntimeError("plan_only engine cannot execute")
        else:
            prog.replay(use_graph)

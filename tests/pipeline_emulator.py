"""TEST INFRASTRUCTURE — the CPU program interpreter of clip_emulator, extended to `ops.video_u8`, the one launch of the
keyframe pipeline (tooncrafter_b200/pipeline.py) that no engine program records.  Every other op goes to
clip_emulator unchanged.  Like ops_emulator it validates host logic only.
"""
from __future__ import annotations

import torch

import clip_emulator


def video_u8(x16, x14, out, *, f_begin, f_end, out_frame):
    """Middle-frame splice (inference.py:270), frame window, then the save path of inference.py:148-153 in torch."""
    T = x16.shape[0]
    v = x16.clone()
    if x14 is not None:
        v[T // 2 - 1:T // 2 + 1] = x14[T // 2 - 2:T // 2]
    v = torch.clamp(v[f_begin:f_end].float(), -1.0, 1.0)
    v = (v + 1.0) / 2.0
    out[out_frame:out_frame + f_end - f_begin] = (v * 255).to(torch.uint8).permute(0, 2, 3, 1)


def executor(fn, args, kw):
    """Program.run(executor=...) hook: clip_emulator.executor plus video_u8."""
    if fn.__name__ == "video_u8":
        video_u8(*args, **kw)
    else:
        clip_emulator.executor(fn, args, kw)


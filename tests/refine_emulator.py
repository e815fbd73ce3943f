"""TEST INFRASTRUCTURE — the CPU program interpreter of pipeline_emulator, extended to `ops.q_sample`, the forward-
diffusion launch of the sampler's masked blend and of stochastic_encode.  Every other op goes to pipeline_emulator
unchanged.  Like ops_emulator it validates host logic only.
"""
from __future__ import annotations

import pipeline_emulator


def q_sample(x, x0, noise, mask, coef, *, B, n, clean=False):
    """torch's fp32 arithmetic of ddpm3d.py:306-309 and ddim.py:172-180, in the reference's op order."""
    xv = x.reshape(B, n)
    x0v = x0.reshape(B, n)
    if clean:
        q = x0v.clone()
    else:
        c = coef[:2 * B].reshape(B, 2)
        q = c[:, :1] * x0v + c[:, 1:] * noise.reshape(B, n)
    if mask is not None:
        m = mask.reshape(B, n)
        q = q * m + (1.0 - m) * xv
    xv.copy_(q)


def executor(fn, args, kw):
    """Program.run(executor=...) hook: pipeline_emulator.executor plus q_sample."""
    if fn.__name__ == "q_sample":
        q_sample(*args, **kw)
    else:
        pipeline_emulator.executor(fn, args, kw)

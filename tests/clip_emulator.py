"""TEST INFRASTRUCTURE — the CPU program interpreter of ops_emulator, extended to the head-dim-80 and causal forms of
`ops.attention` that the OpenCLIP engines record (keywords head_dim / causal).  Every other op, and attention calls
without those keywords, go to ops_emulator unchanged.  Like ops_emulator it validates host logic only.
"""
from __future__ import annotations

import torch

import ops_emulator


def attention(q, segs, out, *, q_batches, Lq, heads, scale, ldq, ldo, q_offset=0, out_offset=0, head_dim=64,
              causal=False):
    """fp32 math on the fp16 operands, one softmax per segment, outputs summed; causal masks key j for query i > j."""
    d = head_dim
    C = heads * d
    st = ops_emulator._strided
    sp = lambda t: t.reshape(t.shape[0], t.shape[1], heads, d).transpose(1, 2)
    Q = st(q, (q_batches, Lq, C), (Lq * ldq, ldq, 1), q_offset).float()
    total = torch.zeros(q_batches, Lq, C)
    for s in segs:
        Lk, div = s["Lk"], s.get("kv_div", 1)
        kvb = (q_batches + div - 1) // div
        K = st(s["k"], (kvb, Lk, C), (Lk * s["ldk"], s["ldk"], 1), s.get("k_offset", 0)).float()
        V = st(s["v"], (kvb, Lk, C), (Lk * s["ldv"], s["ldv"], 1), s.get("v_offset", 0)).float()
        idx = torch.arange(q_batches) // div
        sc = (sp(Q) @ sp(K[idx]).transpose(-1, -2)) * scale
        if causal:
            sc = sc.masked_fill(torch.ones(Lq, Lk, dtype=torch.bool).triu(1), float("-inf"))
        total += (sc.softmax(-1) @ sp(V[idx])).transpose(1, 2).reshape(q_batches, Lq, C)
    st(out, (q_batches, Lq, C), (Lq * ldo, ldo, 1), out_offset).copy_(total.half())


def executor(fn, args, kw):
    """Program.run(executor=...) hook: ops_emulator.executor plus the attention forms above."""
    if fn.__name__ == "attention" and ("head_dim" in kw or "causal" in kw):
        attention(*args, **kw)
    else:
        ops_emulator.executor(fn, args, kw)

"""ResamplerEngine: the image-conditioning Resampler as a recorded program of C-ABI launches.

Reference: lvdm/modules/encoders/resampler.py:96-145 (Resampler.forward), :49-93 (PerceiverAttention: LayerNorm of the
image tokens and of the latents, q from the latents, k/v from their concatenation, ONE softmax over all keys, scale
dim_head^-1/4 on q and k), :27-34 (FeedForward: LayerNorm -> Linear -> GELU -> Linear, no biases).  Runs once per clip
on a few hundred tokens; it reuses the hot path's GEMM / LayerNorm / attention kernels, no new design.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn as nn

from . import ops
from .engine import _P, _f, _h, linear, pack_linear, weights_signature
from .runtime import Act, Arena, Builder, Program


class ResamplerEngine:
    def __init__(self, rs: nn.Module, device=None, use_graph: bool = False, plan_only: bool = False):
        p0 = rs.latents
        self.dev = torch.device(device) if device is not None else p0.device
        self.plan_only = plan_only
        if self.dev.type != "cuda" and not plan_only:
            raise RuntimeError("tooncrafter_b200 runs on CUDA only (no CPU fallback); move the model to a GPU")
        self._sig = weights_signature(rs)
        self.use_graph = use_graph
        self.dim, self.heads, self.inner = rs.dim, rs.heads, rs.heads * rs.dim_head
        self.n_lat = rs.latents.shape[1]
        self.emb = rs.proj_in.weight.shape[1]
        self.out_dim = rs.proj_out.weight.shape[0]
        for n in (self.dim, self.emb, self.inner, self.out_dim):
            if n % 64:
                raise NotImplementedError("Resampler widths must be multiples of 64 (GEMM K granularity)")
        self._pack(rs)
        self._plans: Dict = {}

    def matches(self, rs) -> bool:
        return rs.latents.device == self.dev and self._sig == weights_signature(rs)

    def _pack(self, rs):
        dev = self.dev
        ln = lambda m: _P(g=_f(m.weight, dev), b=_f(m.bias, dev), eps=m.eps)
        self.latents = _h(rs.latents[0], dev)                                  # [n_lat, dim]
        self.p_in = _P(w=pack_linear(rs.proj_in.weight, dev), b=_f(rs.proj_in.bias, dev))
        self.p_out = _P(w=pack_linear(rs.proj_out.weight, dev), b=_f(rs.proj_out.bias, dev), norm=ln(rs.norm_out))
        self.layers = []
        for attn, ff in rs.layers:
            self.layers.append(_P(n1=ln(attn.norm1), n2=ln(attn.norm2), q=pack_linear(attn.to_q.weight, dev),
                                  kv=pack_linear(attn.to_kv.weight, dev), o=pack_linear(attn.to_out.weight, dev),
                                  ffn=ln(ff[0]), w1=pack_linear(ff[1].weight, dev), w2=pack_linear(ff[3].weight, dev)))

    def _build(self, B: int, n1: int):
        dev, dim, inner, n2 = self.dev, self.dim, self.inner, self.n_lat
        hid = self.layers[0].w1.shape[0] if self.layers else dim
        rows_x, rows_l, rows_kv = B * n1, B * n2, B * (n1 + n2)
        arena = Arena(2 * (rows_x * (self.emb + dim) + rows_l * (4 * dim + 2 * inner + hid + self.out_dim * 2)
                           + rows_kv * (dim + 2 * inner)) + (8 << 20), dev)
        main = Program()
        bld = Builder(arena, main)
        plan = _P(B=B, n1=n1, arena=arena, main=main)
        plan.x_in = torch.zeros(rows_x * self.emb, dtype=torch.float16, device=dev)           # flat, like arena tensors
        plan.lat0 = self.latents.repeat(B, 1).reshape(-1).contiguous()        # [B*n2, dim], constant
        ln = lambda x, y, n, rows, C: bld.op(ops.layernorm, x, y, n.g, n.b, rows=rows, C=C, eps=n.eps, ldx=C, ldy=C)

        xp = bld.act(1, 1, rows_x, dim)
        linear(bld, Act(plan.x_in, 1, 1, rows_x, self.emb, self.emb), self.p_in.w, xp, bias=self.p_in.b)
        lat = Act(plan.lat0, 1, 1, rows_l, dim, dim)
        for p in self.layers:
            kvin = bld.act(1, 1, rows_kv, dim)                                # per sample: [x tokens | latents], normed
            nl = bld.act(1, 1, rows_l, dim)
            ln(lat.t, nl.t, p.n2, rows_l, dim)
            for b in range(B):
                ln(xp.t[b * n1 * dim:], kvin.t[b * (n1 + n2) * dim:], p.n1, n1, dim)
                ln(lat.t[b * n2 * dim:], kvin.t[(b * (n1 + n2) + n1) * dim:], p.n2, n2, dim)
            q = bld.act(1, 1, rows_l, inner)
            linear(bld, nl, p.q, q)
            nl.free()
            kv = bld.act(1, 1, rows_kv, 2 * inner)
            linear(bld, kvin, p.kv, kv)
            kvin.free()
            att = bld.act(1, 1, rows_l, inner)
            # (q s)(k s)^T with s = dim_head^-1/4  ==  q k^T * dim_head^-1/2   (resampler.py:84-86)
            bld.op(ops.attention, q.t, [dict(k=kv.t, v=kv.t, ldk=2 * inner, ldv=2 * inner, Lk=n1 + n2, v_offset=inner)],
                   att.t, q_batches=B, Lq=n2, heads=self.heads, scale=64 ** -0.5, ldq=inner, ldo=inner)
            q.free()
            kv.free()
            lat2 = bld.act(1, 1, rows_l, dim)
            linear(bld, att, p.o, lat2, res=lat)
            att.free()
            hn = bld.act(1, 1, rows_l, dim)
            ln(lat2.t, hn.t, p.ffn, rows_l, dim)
            g = bld.act(1, 1, rows_l, hid)
            linear(bld, hn, p.w1, g)
            hn.free()
            bld.op(ops.gelu2d, g.t, g.t, rows=rows_l, cols=hid, ldx=hid, ldy=hid)
            lat3 = bld.act(1, 1, rows_l, dim)
            linear(bld, g, p.w2, lat3, res=lat2)
            g.free()
            lat2.free()
            if lat.t is not plan.lat0:
                lat.free()
            lat = lat3
        po = bld.act(1, 1, rows_l, self.out_dim)
        linear(bld, lat, self.p_out.w, po, bias=self.p_out.b)
        plan.out = torch.zeros(rows_l * self.out_dim, dtype=torch.float16, device=dev)
        ln(po.t, plan.out, self.p_out.norm, rows_l, self.out_dim)
        return plan

    def plan_for(self, B: int, n1: int):
        key = (B, n1)
        if key not in self._plans:
            self._plans[key] = self._build(B, n1)
        return self._plans[key]

    def forward(self, x: torch.Tensor, executor=None) -> torch.Tensor:
        B, n1, E = x.shape
        assert E == self.emb, f"expected {self.emb}-wide image tokens"
        plan = self.plan_for(B, n1)
        plan.x_in.copy_(x.reshape(-1))
        if executor is not None:
            plan.main.run(executor)
        else:
            plan.main.replay(self.use_graph)
        return plan.out.view(B, self.n_lat, self.out_dim).float()

"""Conditioning engines: the image-conditioning Resampler and the OpenCLIP text / image towers as recorded programs
of C-ABI launches.

ResamplerEngine:

Reference: lvdm/modules/encoders/resampler.py:96-145 (Resampler.forward), :49-93 (PerceiverAttention: LayerNorm of the
image tokens and of the latents, q from the latents, k/v from their concatenation, ONE softmax over all keys, scale
dim_head^-1/4 on q and k), :27-34 (FeedForward: LayerNorm -> Linear -> GELU -> Linear, no biases).  Runs once per clip
on a few hundred tokens; it reuses the hot path's GEMM / LayerNorm / attention kernels, no new design.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops
from .engine import RowStats, _P, _f, _h, fold_layernorm, linear, ln_linear, pack_linear
from .runtime import Act, Arena, Builder, Engine, Program


class ResamplerEngine(Engine):
    def __init__(self, rs: nn.Module, device=None, use_graph: bool = False, plan_only: bool = False):
        super().__init__(rs, device, use_graph, plan_only)
        self.dim, self.heads, self.inner = rs.dim, rs.heads, rs.heads * rs.dim_head
        self.n_lat = rs.latents.shape[1]
        self.emb = rs.proj_in.weight.shape[1]
        self.out_dim = rs.proj_out.weight.shape[0]
        for n in (self.dim, self.emb, self.inner, self.out_dim):
            if n % 64:
                raise NotImplementedError("Resampler widths must be multiples of 64 (GEMM K granularity)")
        self._pack(rs)

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

    def forward(self, x: torch.Tensor, executor=None) -> torch.Tensor:
        B, n1, E = x.shape
        assert E == self.emb, f"expected {self.emb}-wide image tokens"
        plan = self.plan_for(B, n1)
        plan.x_in.copy_(x.reshape(-1))
        self._execute(plan.main, executor, self.use_graph)
        return plan.out.view(B, self.n_lat, self.out_dim).float()


# ------------------------------------------------------------------------------------------------ OpenCLIP towers
CLIP_LN_EPS = 1e-5            # open_clip LayerNorm
PATCH_K_PAD = 64              # GEMM K granularity: the 3 * patch^2 patch vector is zero-padded to a multiple of it


class _ClipTowerEngine(Engine):
    """Shared part of the two OpenCLIP tower engines: the residual attention blocks of open_clip.transformer
    (reference condition.py:214-231, :369; open_clip ResidualAttentionBlock: x += attn(ln_1(x)); x += mlp(ln_2(x)),
    nn.MultiheadAttention with a fused in_proj, MLP c_fc -> GELU (erf) -> c_proj).

    ln_1 / ln_2 are folded into the in_proj / c_fc GEMMs; their row statistics ride the epilogue of the GEMM that
    writes the residual stream.  Attention reads q / k / v as channel slices of the in_proj output."""

    causal = False

    def __init__(self, m: nn.Module, device=None, use_graph: bool = False, plan_only: bool = False):
        super().__init__(m, device, use_graph, plan_only)
        self.heads = m.heads

    def _pack_blocks(self, blocks):
        dev = self.dev
        self.width = blocks[0].ln_1.weight.shape[0]
        if self.width % 64 or self.width % self.heads:
            raise NotImplementedError("OpenCLIP width must be a multiple of 64 (GEMM K granularity)")
        self.d_head = self.width // self.heads
        if self.d_head not in (64, 80):
            raise NotImplementedError(f"head dim {self.d_head}: the attention kernel takes 64 or 80")
        self.layers = []
        for r in blocks:
            self.layers.append(_P(
                qkv=fold_layernorm(r.attn.in_proj_weight, r.attn.in_proj_bias, _LN(r.ln_1), dev),
                o_w=pack_linear(r.attn.out_proj.weight, dev), o_b=_f(r.attn.out_proj.bias, dev),
                fc=fold_layernorm(r.mlp.c_fc.weight, r.mlp.c_fc.bias, _LN(r.ln_2), dev),
                pj_w=pack_linear(r.mlp.c_proj.weight, dev), pj_b=_f(r.mlp.c_proj.bias, dev)))
        self.hid = self.layers[0].fc.w.shape[0] if self.layers else 4 * self.width

    def _blocks(self, bld: Builder, x: Act, B: int, L: int, last_out: Act = None) -> Act:
        """Record the residual blocks over x [B * L tokens][width]; returns the residual stream after the last block
        (written into `last_out` when given).  Frees x unless it is the input."""
        W, rows = self.width, B * L
        st = None                                  # row statistics of x: from the producing GEMM after block 0
        x_in = x
        for i, p in enumerate(self.layers):
            qkv = bld.act(1, 1, rows, 3 * W)
            ln_linear(bld, x, p.qkv, qkv, stats=st)
            att = bld.act(1, 1, rows, W)
            bld.op(ops.attention, qkv.t, [dict(k=qkv.t, v=qkv.t, ldk=3 * W, ldv=3 * W, Lk=L, k_offset=W, v_offset=2 * W)],
                   att.t, q_batches=B, Lq=L, heads=self.heads, scale=self.d_head ** -0.5, ldq=3 * W, ldo=W,
                   head_dim=self.d_head, causal=self.causal)
            qkv.free()
            s1 = RowStats(bld, rows, W)
            x1 = bld.act(1, 1, rows, W)
            linear(bld, att, p.o_w, x1, bias=p.o_b, res=x, **s1.producer_kw())
            att.free()
            h = bld.act(1, 1, rows, self.hid)
            ln_linear(bld, x1, p.fc, h, stats=s1)
            s1.free()
            bld.op(ops.gelu2d, h.t, h.t, rows=rows, cols=self.hid, ldx=self.hid, ldy=self.hid)
            last = i == len(self.layers) - 1
            s2 = None if last else RowStats(bld, rows, W)
            x2 = last_out if (last and last_out is not None) else bld.act(1, 1, rows, W)
            linear(bld, h, p.pj_w, x2, bias=p.pj_b, res=x1, **({} if s2 is None else s2.producer_kw()))
            h.free()
            x1.free()
            if x is not x_in:
                x.free()
            if st is not None:
                st.free()
            x, st = x2, s2
        return x


class _LN:
    """LayerNorm view of an open_clip LayerNorm parameter pair (what fold_layernorm reads)."""

    def __init__(self, n):
        self.weight, self.bias, self.eps = n.weight, n.bias, CLIP_LN_EPS


class ClipTextEngine(_ClipTowerEngine):
    """OpenCLIP text tower (reference condition.py:214-231): token embedding + positional embedding (torch gather into
    the plan's input buffer), the first n - layer_idx residual blocks with the causal mask, ln_final."""

    causal = True

    def __init__(self, m: nn.Module, device=None, use_graph: bool = False, plan_only: bool = False):
        super().__init__(m, device, use_graph, plan_only)
        dev = self.dev
        md = m.model
        blocks = list(md.transformer.resblocks)
        blocks = blocks[:len(blocks) - m.layer_idx]        # "penultimate": the last block is never run
        self._pack_blocks(blocks)
        self.ctx = md.positional_embedding.shape[0]
        self.tok = _h(md.token_embedding.weight, dev)
        self.pos = _f(md.positional_embedding, dev)
        self.ln_final = _P(g=_f(md.ln_final.weight, dev), b=_f(md.ln_final.bias, dev))

    def _build(self, B: int):
        W, L, dev = self.width, self.ctx, self.dev
        rows = B * L
        arena = Arena(2 * rows * (6 * W + self.hid) + 64 * rows + (8 << 20), dev)
        main = Program()
        bld = Builder(arena, main)
        plan = _P(B=B, arena=arena, main=main)
        plan.x_in = torch.zeros(rows * W, dtype=torch.float16, device=dev)
        x = self._blocks(bld, Act(plan.x_in, 1, 1, rows, W, W), B, L)
        plan.out = torch.zeros(rows * W, dtype=torch.float16, device=dev)
        bld.op(ops.layernorm, x.t, plan.out, self.ln_final.g, self.ln_final.b, rows=rows, C=W, eps=CLIP_LN_EPS,
               ldx=W, ldy=W)
        return plan

    def forward(self, tokens: torch.Tensor, executor=None) -> torch.Tensor:
        """tokens [B, ctx] int64 -> [B, ctx, width] fp32."""
        B, L = tokens.shape
        assert L == self.ctx, f"expected {self.ctx} token ids per prompt"
        plan = self.plan_for(B)
        ids = tokens.to(self.dev)
        plan.x_in.view(B, L, self.width).copy_(self.tok[ids].float() + self.pos)
        self._execute(plan.main, executor, self.use_graph)
        return plan.out.view(B, L, self.width).float()


class ClipImageEngine(_ClipTowerEngine):
    """OpenCLIP vision tower without ln_post / proj (reference condition.py:342-372): patch embedding conv1 as one GEMM
    over the patches of every image, the class token and positional embedding in its epilogue, ln_pre, the residual
    blocks.  Input: preprocessed pixels [B, 3, image, image]."""

    def __init__(self, m: nn.Module, device=None, use_graph: bool = False, plan_only: bool = False):
        super().__init__(m, device, use_graph, plan_only)
        dev = self.dev
        vis = m.model.visual
        self._pack_blocks(list(vis.transformer.resblocks))
        self.patch = vis.conv1.weight.shape[-1]
        self.n_tok = vis.positional_embedding.shape[0]          # 1 + grid^2
        self.grid = int(round((self.n_tok - 1) ** 0.5))
        kp = 3 * self.patch * self.patch
        self.kpad = -(-kp // PATCH_K_PAD) * PATCH_K_PAD          # 588 -> 640 (like conv_in's cpad)
        w = vis.conv1.weight.detach().reshape(self.width, kp)     # [width, (c, py, px)]
        self.conv_w = _h(torch.nn.functional.pad(w, (0, self.kpad - kp)), dev)
        # per token row: class_embedding + pos[0] for the class token, pos[1 + p] for patch p (added in the epilogue)
        pos = vis.positional_embedding.detach().float().clone()
        pos[0] += vis.class_embedding.detach().float()
        self.tok_bias = _h(pos, dev)
        self.ln_pre = _P(g=_f(vis.ln_pre.weight, dev), b=_f(vis.ln_pre.bias, dev))

    def _build(self, B: int):
        W, L, dev = self.width, self.n_tok, self.dev
        rows = B * L
        arena = Arena(2 * rows * (6 * W + self.hid) + 64 * rows + (8 << 20), dev)
        main = Program()
        bld = Builder(arena, main)
        plan = _P(B=B, arena=arena, main=main)
        # im2col of the patches; row b * L of each image (the class token) stays zero, so the GEMM writes the bias there
        plan.x_in = torch.zeros(rows * self.kpad, dtype=torch.float16, device=dev)
        plan.bias = self.tok_bias.repeat(B, 1).contiguous()                           # [B * L, W], constant
        x0 = bld.act(1, 1, rows, W)
        linear(bld, Act(plan.x_in, 1, 1, rows, self.kpad, self.kpad), self.conv_w, x0, bias2=plan.bias,
               bias2_rows_per=1)
        x = bld.act(1, 1, rows, W)
        bld.op(ops.layernorm, x0.t, x.t, self.ln_pre.g, self.ln_pre.b, rows=rows, C=W, eps=CLIP_LN_EPS, ldx=W, ldy=W)
        x0.free()
        plan.out = torch.zeros(rows * W, dtype=torch.float16, device=dev)
        self._blocks(bld, x, B, L, last_out=Act(plan.out, 1, 1, rows, W, W))
        return plan

    def forward(self, pixels: torch.Tensor, executor=None) -> torch.Tensor:
        """pixels [B, 3, image, image] (CLIP-normalised) -> [B, 1 + grid^2, width] fp32."""
        B = pixels.shape[0]
        g, P = self.grid, self.patch
        assert pixels.shape[1:] == (3, g * P, g * P), f"expected [B, 3, {g * P}, {g * P}] pixels"
        plan = self.plan_for(B)
        patches = pixels.to(self.dev).float().reshape(B, 3, g, P, g, P).permute(0, 2, 4, 1, 3, 5)
        xin = plan.x_in.view(B, self.n_tok, self.kpad)
        xin[:, 1:, :3 * P * P].copy_(patches.reshape(B, g * g, 3 * P * P))
        self._execute(plan.main, executor, self.use_graph)
        return plan.out.view(B, self.n_tok, self.width).float()

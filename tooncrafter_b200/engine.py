"""CUDA execution engines for the denoising UNet (this file) — weights packed once into fp16 GEMM layouts, the
forward pass built once per input geometry as a static program of C-ABI launches (see runtime.py).

Reference semantics restated by the builders (paths relative to /root/reference):
  UNetModel.forward                      lvdm/modules/networks/openaimodel3d.py:548-603
  ResBlock / TemporalConvBlock           openaimodel3d.py:210-236, 272-279
  SpatialTransformer / TemporalTransformer / BasicTransformerBlock / CrossAttention / GEGLU-FF
                                         lvdm/modules/attention.py:81-144, 242-246, 294-310, 365-412, 415-442
H100-first departures (results identical up to fp16 rounding):
  * channels-last [B][T][H][W][C] fp16 activations; no layout copies, skip "cat" realised by writing producers
    straight into channel slices of the concat buffer;
  * cond / uncond batched as B = 2 through one forward; context K/V projections computed once per
    conditioning (they are step-invariant; the reference recomputes them 100x per clip);
  * per-ResBlock timestep-embedding Linear layers evaluated by ONE stacked GEMV per step;
  * q/k/v projections fused into one GEMM; GEGLU fused into its GEMM epilogue.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from . import ops
from .layout import Layer, UNetLayout
from .runtime import Act, Arena, Builder, Engine, Program

GEGLU_BN = 256


# ------------------------------------------------------------------------------------------------ weight packing
def _h(t: torch.Tensor, dev) -> torch.Tensor:
    return t.detach().to(device=dev, dtype=torch.float16).contiguous()


def _f(t: torch.Tensor, dev) -> torch.Tensor:
    return t.detach().to(device=dev, dtype=torch.float32).contiguous()


def pack_conv(w: torch.Tensor, dev, cin_pad: Optional[int] = None) -> torch.Tensor:
    """[Co, Ci, *k] conv weight -> [Co, taps * Ci_pad] (tap-major, channel-minor) fp16."""
    co, ci = w.shape[0], w.shape[1]
    w = w.detach().reshape(co, ci, -1).permute(0, 2, 1)            # [Co, taps, Ci]
    if cin_pad is not None and cin_pad != ci:
        w = torch.nn.functional.pad(w, (0, cin_pad - ci))
    return _h(w.reshape(co, -1), dev)


def pack_linear(w: torch.Tensor, dev) -> torch.Tensor:
    return _h(w.reshape(w.shape[0], -1), dev)


def geglu_perm(n2: int, bn: int = GEGLU_BN) -> torch.Tensor:
    """Row permutation of GEGLU.proj [2*inner, dim] (rows: value half then gate half, attention.py:421) into the
    per-N-tile interleave [value(bn/2) | gate(bn/2)], so one accumulator tile holds matching value/gate columns."""
    inner = n2 // 2
    hb = bn // 2
    assert inner % hb == 0, f"GEGLU inner dim {inner} must be a multiple of {hb}"
    a = torch.arange(inner).reshape(inner // hb, hb)
    return torch.cat([a, a + inner], dim=1).reshape(-1)


def fold_layernorm(w: torch.Tensor, b: Optional[torch.Tensor], norm, dev, perm: Optional[torch.Tensor] = None):
    """LN(x) @ W^T + b  ==  rstd * (x @ Wg^T - mean * u) + c  with Wg = W * gamma (fp16), u = rowsum(Wg) computed from
    the ROUNDED fp16 weights (so the subtraction cancels exactly what the tensor core accumulated), c = W beta + b."""
    w32 = w.detach().float().reshape(w.shape[0], -1)
    wg16 = (w32 * norm.weight.detach().float()[None, :]).half()
    u = wg16.float().sum(dim=1)
    c = w32 @ norm.bias.detach().float()
    if b is not None:
        c = c + b.detach().float()
    if perm is not None:
        wg16, u, c = wg16[perm], u[perm], c[perm]
    return _P(w=wg16.to(dev).contiguous(), u=_f(u, dev), c=_f(c, dev), eps=float(norm.eps))


class _P:
    """Attribute bag for packed tensors."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def pack_norm(m, dev):
    return _P(g=_f(m.weight, dev), b=_f(m.bias, dev), eps=float(m.eps))


def pack_transformer_block(tb, dev, cross: bool):
    """LayerNorms are folded into the GEMM that consumes them (fold_layernorm); q/k/v projections fused."""
    inner = tb.attn1.to_q.weight.shape[0]
    p = _P(inner=inner)

    def attn(a, norm, qkv: bool):
        w = torch.cat([a.to_q.weight, a.to_k.weight, a.to_v.weight], 0) if qkv else a.to_q.weight
        return _P(proj=fold_layernorm(w, None, norm, dev), o_w=pack_linear(a.to_out[0].weight, dev),
                  o_b=_f(a.to_out[0].bias, dev))
    a2 = tb.attn2
    p.attn1, p.attn2 = attn(tb.attn1, tb.norm1, True), attn(a2, tb.norm2, not cross)
    if cross:
        p.kv_txt = _h(torch.cat([a2.to_k.weight, a2.to_v.weight], 0), dev)
        p.kv_img = (_h(torch.cat([a2.to_k_ip.weight, a2.to_v_ip.weight], 0), dev) if hasattr(a2, "to_k_ip") else None)
    proj = tb.ff.net[0].proj
    p.ff1 = fold_layernorm(proj.weight, proj.bias, tb.norm3, dev, perm=geglu_perm(proj.weight.shape[0]))
    p.ff2_w, p.ff2_b = pack_linear(tb.ff.net[2].weight, dev), _f(tb.ff.net[2].bias, dev)
    return p


# ------------------------------------------------------------------------------------------------ shared builders
def gemm(bld: Builder, a: Act, w: torch.Tensor, taps, out: Act, *, a_dims=None, a_strides=None, out_dims=None,
         bias=None, bias2=None, bias2_rows_per=0, res: Optional[Act] = None, acc_scale=1.0, geglu=False,
         n_cols=None, block_n=0, ln_stats=None, ln_u=None, ln_nslots=0, ln_eps=1e-5, row_stats=None,
         row_stats_slots=0):
    """Record one tc_conv_gemm launch: out = epilogue(im2col(a) @ w.T)."""
    if a_dims is None:
        a_dims = (a.N, a.H, a.W, a.C)
        a_strides = (a.H * a.W * a.ld, a.W * a.ld, a.ld)
    if out_dims is None:
        out_dims = (out.N, out.H, out.W)
    n_cols = n_cols if n_cols is not None else (out.C * 2 if geglu else out.C)
    bld.op(ops.conv_gemm, a.t, a_dims, a_strides, w, taps, out.t, out_dims, n_cols, ldc=out.ld, bias=bias,
           bias2=bias2, bias2_rows_per=bias2_rows_per, res=None if res is None else res.t,
           ldr=None if res is None else res.ld, acc_scale=acc_scale, geglu=geglu, block_n=block_n, a_offset=a.off,
           out_offset=out.off, res_offset=0 if res is None else res.off, ln_stats=ln_stats, ln_u=ln_u,
           ln_nslots=ln_nslots, ln_eps=ln_eps, row_stats=row_stats, row_stats_slots=row_stats_slots)


def linear(bld: Builder, a: Act, w, out: Act, **kw):
    """Row-wise linear over all pixels/tokens of `a` (token order is irrelevant)."""
    rows = a.rows
    gemm(bld, a, w, ops.TAPS_1x1, out, a_dims=(1, 1, rows, a.C), a_strides=(rows * a.ld, rows * a.ld, a.ld),
         out_dims=(1, 1, rows), **kw)


def temporal_conv(bld: Builder, a: Act, w, out: Act, B: int, **kw):
    """(3,1,1) conv over the frame axis: view [B][T][HW][C], taps along T."""
    T, HW = a.N // B, a.H * a.W
    gemm(bld, a, w, ops.TAPS_T3, out, a_dims=(B, T, HW, a.C), a_strides=(T * HW * a.ld, HW * a.ld, a.ld),
         out_dims=(B, T, HW), **kw)


def groupnorm(bld: Builder, x: Act, y: Act, n: _P, *, frames_per_stat=1, silu=False, eps=None):
    bld.op(ops.groupnorm, x.t, y.t, n.g, n.b, frames=x.N, frames_per_stat=frames_per_stat, hw=x.H * x.W, C=x.C,
           eps=n.eps if eps is None else eps, silu=silu, ldx=x.ld, ldy=y.ld, x_offset=x.off, y_offset=y.off)


class RowStats:
    """Partial LayerNorm statistics of an activation, written by the epilogue of the GEMM that produces it
    ([rows][slots] {sum, sumsq}; tc_conv_gemm row_stats) and finished by the epilogue of the GEMM that consumes it."""

    def __init__(self, bld: Builder, rows: int, width: int):
        self.bn = 160 if width in (320, 640) else (256 if width % 256 == 0 else 0)   # producer tile (fixes the slot count)
        self.slots = -(-width // self.bn) if self.bn else 0
        self.bld = bld
        self.buf, self.off = bld.raw(2 * self.slots * rows, torch.float32) if self.bn else (None, None)

    def producer_kw(self):
        return dict(block_n=self.bn, row_stats=self.buf, row_stats_slots=self.slots) if self.bn else {}

    def free(self):
        if self.bn:
            self.bld.free_raw(self.off)


def ln_linear(bld: Builder, x: Act, f: _P, out: Act, stats: Optional[RowStats] = None, **kw):
    """out = LN(x) @ W^T (+ ...) with the LayerNorm folded into the GEMM epilogue.  The row statistics come from the
    producer of x (`stats`, no extra pass over x) or from one tc_row_stats pass; either way the LayerNorm kernel and
    its normalised fp16 copy of x are gone."""
    assert x.off == 0
    if stats is not None and stats.bn:
        linear(bld, x, f.w, out, bias=f.c, ln_stats=stats.buf, ln_u=f.u, ln_nslots=stats.slots, ln_eps=f.eps, **kw)
        return
    buf, off = bld.raw(2 * x.rows, torch.float32)
    bld.op(ops.row_stats, x.t, buf, rows=x.rows, C=x.C, eps=f.eps, ldx=x.ld)
    linear(bld, x, f.w, out, bias=f.c, ln_stats=buf, ln_u=f.u, **kw)
    bld.free_raw(off)


def feed_forward(bld: Builder, x: Act, p: _P, out: Act, stats: Optional[RowStats] = None):
    """x + W2 (a * gelu(g)), with (a, g) = W1 LN(x)   (attention.py:245, 415-442)."""
    hid = bld.act(x.N, x.H, x.W, 4 * x.C)
    ln_linear(bld, x, p.ff1, hid, stats=stats, geglu=True, block_n=GEGLU_BN)
    linear(bld, hid, p.ff2_w, out, bias=p.ff2_b, res=x)
    hid.free()


def attention_sublayer(bld: Builder, x: Act, a: _P, record, out: Act, s_in: RowStats, s_out: RowStats):
    """out = x + Wo attention(LN(x) Wproj), with the LayerNorm folded into the projection (statistics `s_in`) and the
    row statistics of out (`s_out`) written by the output projection; `record(proj, att)` records the attention
    launch from the projection's output into att."""
    proj = bld.act(x.N, x.H, x.W, a.proj.w.shape[0])
    ln_linear(bld, x, a.proj, proj, stats=s_in)
    att = bld.act(x.N, x.H, x.W, x.C)
    record(proj, att)
    proj.free()
    linear(bld, att, a.o_w, out, bias=a.o_b, res=x, **s_out.producer_kw())
    att.free()


def pack_resblock(dev, norm1, conv1, norm2, conv2, skip=None, time=(), alpha: float = 1.0) -> _P:
    """ResNet block (UNet ResBlock, VAE ResnetBlock / VideoResBlock): norm1, conv1 (3x3), norm2, conv2 (3x3), the
    optional 1x1 `skip` conv, and the optional temporal stages `time` [(GroupNorm, (3,1,1) conv)], whose last one
    blends in the residual with `alpha` (see resblock)."""
    p = _P(cin=conv1.weight.shape[1], cout=conv1.weight.shape[0], n1=pack_norm(norm1, dev), n2=pack_norm(norm2, dev),
           c1_w=pack_conv(conv1.weight, dev), c1_b=_f(conv1.bias, dev),
           c2_w=pack_conv(conv2.weight, dev), c2_b=_f(conv2.bias, dev), skip_w=None, alpha=alpha)
    if skip is not None:
        p.skip_w, p.skip_b = pack_linear(skip.weight, dev), _f(skip.bias, dev)
    p.time = [_P(gn=pack_norm(gn, dev), w=pack_conv(conv.weight, dev), b=_f(conv.bias, dev)) for gn, conv in time]
    return p


def resblock(bld: Builder, p: _P, x: Act, dst: Act, *, B: int = 1, T: int = 1, emb=None) -> None:
    """GN+SiLU -> 3x3 conv (+ per-sample timestep embedding `emb` [B, cout]) -> GN+SiLU -> 3x3 conv + x (through the
    1x1 skip when the width changes).  Then, when p.time is set, the temporal stack over the [B][T] frames:
    [GN over (C/32, T, H, W) -> SiLU -> (3,1,1) conv] per stage, the last one writing dst = s + alpha * conv(...) with s
    the spatial part's output (UNet TemporalConvBlock: alpha 1, openaimodel3d.py:272-279; VideoResBlock: alpha =
    sigmoid(mix_factor), autoencoder_dualref.py:892-911)."""
    N, H, W = x.N, x.H, x.W
    g1 = bld.act(N, H, W, p.cin)
    groupnorm(bld, x, g1, p.n1, silu=True)
    h1 = bld.act(N, H, W, p.cout)
    gemm(bld, g1, p.c1_w, ops.TAPS_3x3, h1, bias=p.c1_b, bias2=emb, bias2_rows_per=0 if emb is None else T * H * W)
    g1.free()
    g2 = bld.act(N, H, W, p.cout)
    groupnorm(bld, h1, g2, p.n2, silu=True)
    h1.free()
    xs = x
    if p.skip_w is not None:
        xs = bld.act(N, H, W, p.cout)
        linear(bld, x, p.skip_w, xs, bias=p.skip_b)
    s = bld.act(N, H, W, p.cout) if p.time else dst
    gemm(bld, g2, p.c2_w, ops.TAPS_3x3, s, bias=p.c2_b, res=xs)
    g2.free()
    if xs is not x:
        xs.free()
    if not p.time:
        return
    cur = s
    for i, tc in enumerate(p.time):
        g = bld.act(N, H, W, p.cout)
        groupnorm(bld, cur, g, tc.gn, frames_per_stat=T, silu=True)
        if cur is not s:
            cur.free()
        last = i == len(p.time) - 1
        nxt = dst if last else bld.act(N, H, W, p.cout)
        temporal_conv(bld, g, tc.w, nxt, B, bias=tc.b, res=s if last else None, acc_scale=p.alpha if last else 1.0)
        g.free()
        cur = nxt
    s.free()


# ------------------------------------------------------------------------------------------------ the UNet engine
class UNetEngine(Engine):
    def __init__(self, unet: nn.Module, device=None, arena_bytes: int = 0, use_graph: bool = True,
                 plan_only: bool = False):
        super().__init__(unet, device, use_graph, plan_only)
        self.lay: UNetLayout = unet.layout
        self.arena_bytes = arena_bytes
        self._pack(unet)

    # ---------------------------------------------------------------------------------- packing
    def _pack(self, u: nn.Module):
        dev, lay = self.dev, self.lay
        emb_w, emb_b = [], []
        self.emb_cols = 0

        def pack_res(m, l: Layer):
            time = ()
            if hasattr(m, "temopral_conv"):
                tc = m.temopral_conv
                time = [(getattr(tc, n)[0], getattr(tc, n)[ci])
                        for n, ci in (("conv1", 2), ("conv2", 3), ("conv3", 3), ("conv4", 3))]
            p = pack_resblock(dev, m.in_layers[0], m.in_layers[2], m.out_layers[0], m.out_layers[3],
                              m.skip_connection if l.cin != l.cout else None, time)
            p.emb_off = self.emb_cols
            self.emb_cols += l.cout
            emb_w.append(m.emb_layers[1].weight.detach())
            emb_b.append(m.emb_layers[1].bias.detach())
            return p

        def pack_tf(m, l: Layer, spatial: bool):
            assert l.d_head == 64, "attention kernels are specialised for head dim 64"
            p = _P(heads=l.heads, inner=l.heads * l.d_head, C=l.cin, spatial=spatial)
            p.norm = pack_norm(m.norm, dev)
            p.in_w, p.in_b = pack_linear(m.proj_in.weight, dev), _f(m.proj_in.bias, dev)
            p.out_w, p.out_b = pack_linear(m.proj_out.weight, dev), _f(m.proj_out.bias, dev)
            p.tb = pack_transformer_block(m.transformer_blocks[0], dev, cross=spatial)
            return p

        def pack_layers(node, layers):
            out = []
            for i, l in enumerate(layers):
                m = getattr(node, str(i))
                if l.kind == "conv_in":
                    cpad = (l.cin + 63) // 64 * 64
                    out.append(_P(kind="conv_in", w=pack_conv(m.weight, dev, cpad), b=_f(m.bias, dev), cpad=cpad,
                                  cout=l.cout))
                elif l.kind == "res":
                    q = pack_res(m, l)
                    q.kind = "res"
                    out.append(q)
                elif l.kind in ("st", "tt"):
                    q = pack_tf(m, l, l.kind == "st")
                    q.kind = l.kind
                    out.append(q)
                elif l.kind == "down":
                    out.append(_P(kind="down", w=pack_conv(m.op.weight, dev), b=_f(m.op.bias, dev), C=l.cout))
                elif l.kind == "up":
                    out.append(_P(kind="up", w=pack_conv(m.conv.weight, dev), b=_f(m.conv.bias, dev), C=l.cout))
            return out

        self.p_input = [pack_layers(getattr(u.input_blocks, pref.split(".")[1]), layers)
                        for pref, layers in lay.input_blocks]
        self.p_init = pack_layers(u.init_attn, lay.init_attn) if lay.init_attn else []
        self.p_middle = pack_layers(u.middle_block, lay.middle_block)
        self.p_output = [pack_layers(getattr(u.output_blocks, pref.split(".")[1]), layers)
                         for pref, layers in lay.output_blocks]
        self.emb_w = _h(torch.cat(emb_w, 0), dev)
        self.emb_b = _f(torch.cat(emb_b, 0), dev)

        def mlp(m):
            return _P(w1=pack_linear(m[0].weight, dev), b1=_f(m[0].bias, dev), w2=pack_linear(m[2].weight, dev),
                      b2=_f(m[2].bias, dev))
        self.p_time = mlp(u.time_embed)
        self.p_fps = mlp(u.fps_embedding) if lay.fs_condition else None
        self.p_out = _P(gn=pack_norm(u.out[0], dev), w=pack_conv(u.out[2].weight, dev), b=_f(u.out[2].bias, dev))

    # ---------------------------------------------------------------------------------- layer builders
    def _transformer(self, bld: Builder, p: _P, x: Act, dst: Act, B: int, T: int, kv=None) -> None:
        """SpatialTransformer (p.spatial: self-attention over the H*W tokens of each frame, cross-attention to the
        context K/V `kv`) or TemporalTransformer (two self-attentions over the T frames of each pixel)."""
        N, H, W = x.N, x.H, x.W
        heads, tb = p.heads, p.tb
        n = bld.act(N, H, W, p.C)
        groupnorm(bld, x, n, p.norm, frames_per_stat=1 if p.spatial else T)
        # LayerNorm statistics of t0 / t1 / t2 ride the epilogues of the GEMMs that write them
        rows = N * H * W
        s0, s1, s2 = (RowStats(bld, rows, p.inner) for _ in range(3))
        t0 = bld.act(N, H, W, p.inner)
        linear(bld, n, p.in_w, t0, bias=p.in_b, **s0.producer_kw())
        n.free()

        def self_attn(qkv: Act, att: Act):
            C = att.C
            if p.spatial:
                L = att.H * att.W
                bld.op(ops.attention, qkv.t, [dict(k=qkv.t, v=qkv.t, ldk=3 * C, ldv=3 * C, Lk=L, k_offset=C,
                                                   v_offset=2 * C)],
                       att.t, q_batches=att.N, Lq=L, heads=heads, scale=64 ** -0.5, ldq=3 * C, ldo=C)
            else:
                bld.op(ops.temporal_attention, qkv.t, qkv.t, qkv.t, att.t, ld=3 * C, ldo=C, B=B, T=T,
                       P=att.H * att.W, heads=heads, scale=64 ** -0.5, k_offset=C, v_offset=2 * C)

        def cross_attn(q: Act, att: Act):
            C = att.C
            segs = [dict(k=kv["txt"], v=kv["txt"], ldk=2 * C, ldv=2 * C, Lk=kv["n_txt"], kv_div=T, v_offset=C)]
            if kv["img"] is not None:
                segs.append(dict(k=kv["img"], v=kv["img"], ldk=2 * C, ldv=2 * C, Lk=kv["n_img"], kv_div=kv["img_div"],
                                 v_offset=C))
            bld.op(ops.attention, q.t, segs, att.t, q_batches=att.N, Lq=att.H * att.W, heads=heads, scale=64 ** -0.5,
                   ldq=C, ldo=C)

        t1 = bld.act(N, H, W, p.inner)
        attention_sublayer(bld, t0, tb.attn1, self_attn, t1, s0, s1)
        t0.free()
        t2 = bld.act(N, H, W, p.inner)
        attention_sublayer(bld, t1, tb.attn2, cross_attn if p.spatial else self_attn, t2, s1, s2)
        t1.free()
        t3 = bld.act(N, H, W, p.inner)
        feed_forward(bld, t2, tb, t3, stats=s2)
        t2.free()
        for r in (s0, s1, s2):
            r.free()
        linear(bld, t3, p.out_w, dst, bias=p.out_b, res=x)
        t3.free()

    def _down(self, bld: Builder, p: _P, x: Act, dst: Act) -> None:
        N, H, W, C = x.N, x.H, x.W, x.C
        src = x
        if x.ld != C or x.off != 0:            # phase split needs a dense tensor
            src = bld.act(N, H, W, C)
            bld.op(ops.copy2d, x.t, src.t, rows=x.rows, cols=C, lds=x.ld, ldd=C, src_offset=x.off)
        ph = bld.act(4 * N, H // 2, W // 2, C)
        bld.op(ops.phase_split2, src.t, ph.t, N=N, H=H, W=W, C_=C)
        if src is not x:
            src.free()
        gemm(bld, ph, p.w, ops.taps_3x3_stride2(N), dst, bias=p.b)
        ph.free()

    def _up(self, bld: Builder, p: _P, x: Act, dst: Act) -> None:
        assert x.off == 0 and x.ld == x.C
        up = bld.act(x.N, 2 * x.H, 2 * x.W, x.C)
        bld.op(ops.upsample2x, x.t, up.t, N=x.N, H=x.H, W=x.W, C_=x.C)
        gemm(bld, up, p.w, ops.TAPS_3x3, dst, bias=p.b)
        up.free()

    # ---------------------------------------------------------------------------------- plan construction
    def _build(self, B: int, T: int, H: int, W: int, n_ctx: int):
        lay, dev = self.lay, self.dev
        N = B * T
        if n_ctx <= 77:
            raise NotImplementedError("context must hold 77 text tokens and at least one image token")
        # openaimodel3d.py:556-562: a context of exactly 77 + 16 T tokens gives frame t its own 16 image tokens (image
        # K/V rows per frame); any other length gives every frame the whole context (image K/V rows per sample, shared
        # by its T frames like the text rows)
        per_frame = n_ctx == 77 + 16 * T
        n_img, img_rows, img_div = (16, N * 16, 1) if per_frame else (n_ctx - 77, B * (n_ctx - 77), T)
        # arena: generous static budget (activations of one B-sample forward)
        px = N * H * W
        arena_bytes = self.arena_bytes or int(px * lay.model_channels * 2 * 40 + (256 << 20))
        arena = Arena(arena_bytes, dev)
        main, ctxp = Program(), Program()
        bld = Builder(arena, main)
        plan = _P(B=B, T=T, H=H, W=W, arena=arena, main=main, ctx=ctxp)

        # static inputs
        plan.x_in = torch.zeros(B, lay.in_channels, T, H, W, dtype=torch.float32, device=dev)
        plan.t_in = torch.zeros(B, dtype=torch.float32, device=dev)
        plan.fs_in = torch.zeros(B, dtype=torch.float32, device=dev)
        plan.ctx_txt = torch.zeros(B * 77, lay.context_dim, dtype=torch.float16, device=dev)
        plan.ctx_img = torch.zeros(img_rows, lay.context_dim, dtype=torch.float16, device=dev)
        plan.emb = torch.zeros(B, lay.time_dim, dtype=torch.float32, device=dev)
        plan.emb_ws = torch.zeros(B * (lay.model_channels + lay.time_dim), dtype=torch.float32, device=dev)
        plan.emb_all = torch.zeros(B, self.emb_cols, dtype=torch.float16, device=dev)
        plan.y_out = torch.zeros(B, lay.out_channels, T, H, W, dtype=torch.float16, device=dev)

        # --- timestep / fps embeddings -> stacked per-ResBlock embedding vectors
        pt = self.p_time
        main.add(ops.time_embed, plan.t_in, pt.w1, pt.b1, pt.w2, pt.b2, plan.emb, plan.emb_ws,
                 dim=lay.model_channels, hidden=lay.time_dim, accumulate=False)
        if self.p_fps is not None:
            pf = self.p_fps
            main.add(ops.time_embed, plan.fs_in, pf.w1, pf.b1, pf.w2, pf.b2, plan.emb, plan.emb_ws,
                     dim=lay.model_channels, hidden=lay.time_dim, accumulate=True)
        main.add(ops.small_linear, plan.emb, self.emb_w, self.emb_b, plan.emb_all, silu_in=True)

        # --- context K/V for every spatial transformer (own program: re-run only when the conditioning changes)
        kvs = {}
        cb = Builder(arena, ctxp)
        txt = Act(plan.ctx_txt, 1, 1, B * 77, lay.context_dim, lay.context_dim)
        img = Act(plan.ctx_img, 1, 1, img_rows, lay.context_dim, lay.context_dim)

        def make_kv(p: _P):
            C = p.inner
            kt = torch.zeros(B * 77, 2 * C, dtype=torch.float16, device=dev)
            linear(cb, txt, p.tb.kv_txt, Act(kt, 1, 1, B * 77, 2 * C, 2 * C))
            ki = None
            if p.tb.kv_img is not None:
                ki = torch.zeros(img_rows, 2 * C, dtype=torch.float16, device=dev)
                linear(cb, img, p.tb.kv_img, Act(ki, 1, 1, img_rows, 2 * C, 2 * C))
            kvs[id(p)] = dict(txt=kt, img=ki, n_txt=77, n_img=n_img, img_div=img_div)

        for blk in self.p_input + [self.p_middle] + self.p_output:
            for p in blk:
                if p.kind == "st":
                    make_kv(p)

        # --- concat buffers for the skip connections: output block k reads cat[h | skip]
        skip_ch = list(lay.skip_channels)
        # geometry of each skip tensor
        geo = []
        h_, w_ = H, W
        for pref, layers in lay.input_blocks:
            if layers[0].kind == "down":
                h_, w_ = h_ // 2, w_ // 2
            geo.append((h_, w_))
        cats = []          # per output block: Act of the concat buffer (never freed: live for the whole program)
        ch = lay.middle_block[-1].cout
        for k, (pref, layers) in enumerate(lay.output_blocks):
            ich = skip_ch[len(skip_ch) - 1 - k]
            gh, gw = geo[len(geo) - 1 - k]
            cats.append(bld.act(N, gh, gw, ch + ich))
            ch = layers[0].cout
        plan.cats = cats

        def skip_dst(j: int) -> Act:
            """Destination slice for the output of input block j (its skip is consumed by output block n-1-j)."""
            k = len(lay.input_blocks) - 1 - j
            c = cats[k]
            ich = skip_ch[j]
            return c.slice(c.C - ich, ich)

        def head_dst(k: int) -> Act:
            c = cats[k]
            ich = skip_ch[len(skip_ch) - 1 - k]
            return c.slice(0, c.C - ich)

        def run_layers(packed, x: Act, final_dst: Optional[Act]) -> Act:
            for i, p in enumerate(packed):
                last = i == len(packed) - 1
                if p.kind == "down":
                    oh, ow, oc = x.H // 2, x.W // 2, p.C
                elif p.kind == "up":
                    oh, ow, oc = x.H * 2, x.W * 2, p.C
                elif p.kind in ("res", "conv_in"):
                    oh, ow, oc = x.H, x.W, p.cout
                else:
                    oh, ow, oc = x.H, x.W, p.C
                dst = final_dst if (last and final_dst is not None) else bld.act(x.N, oh, ow, oc)
                if last and final_dst is not None:
                    assert (dst.N, dst.H, dst.W, dst.C) == (x.N, oh, ow, oc), "destination geometry mismatch"
                if p.kind == "conv_in":
                    gemm(bld, x, p.w, ops.TAPS_3x3, dst, bias=p.b)
                elif p.kind == "res":
                    resblock(bld, p, x, dst, B=B, T=T, emb=plan.emb_all[:, p.emb_off:p.emb_off + p.cout])
                elif p.kind in ("st", "tt"):
                    self._transformer(bld, p, x, dst, B, T, kvs.get(id(p)))
                elif p.kind == "down":
                    self._down(bld, p, x, dst)
                elif p.kind == "up":
                    self._up(bld, p, x, dst)
                x.free()           # no-op for slices / static inputs
                x = dst
            return x

        # --- input: NCTHW fp32 -> channels-last fp16, zero-padded to 64 channels
        cpad = self.p_input[0][0].cpad
        x0_t = torch.zeros(N * H * W * cpad, dtype=torch.float16, device=dev)
        x0 = Act(x0_t, N, H, W, cpad, cpad)
        main.add(ops.ncthw_to_cl, plan.x_in, x0_t, B=B, C_=lay.in_channels, T=T, H=H, W=W, Cpad=cpad, coff=0,
                 scale=1.0)

        plan.marks = []        # (launch count, name, Act): block boundaries, for debugging / tests

        def mark(name, a):
            plan.marks.append((len(main), name, a))

        nin = len(self.p_input)
        h = x0
        for j in range(nin):
            if j == 0 and self.p_init:
                h = run_layers(self.p_input[0], h, None)
                mark("conv_in", h)
                h = run_layers(self.p_init, h, skip_dst(0))
            else:
                h = run_layers(self.p_input[j], h, skip_dst(j))
            mark(f"input_blocks.{j}", h)
        h = run_layers(self.p_middle, h, head_dst(0))
        mark("middle_block", h)
        nout = len(self.p_output)
        for k in range(nout):
            dst = head_dst(k + 1) if k + 1 < nout else None
            h = run_layers(self.p_output[k], cats[k], dst)
            mark(f"output_blocks.{k}", h)
        # --- out: GN + SiLU + conv3x3 -> NCTHW fp16
        g = bld.act(N, H, W, h.C)
        groupnorm(bld, h, g, self.p_out.gn, silu=True)
        yo = bld.act(N, H, W, 16)
        gemm(bld, g, self.p_out.w, ops.TAPS_3x3, yo, bias=self.p_out.b, n_cols=lay.out_channels)
        main.add(ops.cl_to_ncthw, yo.t, plan.y_out, B=B, C_=lay.out_channels, T=T, H=H, W=W, ldx=16)
        plan.n_ctx = n_ctx
        return plan

    # ---------------------------------------------------------------------------------- execution
    def set_context(self, plan, context: torch.Tensor, executor=None) -> None:
        """Copy the conditioning in and re-run the context K/V program — unconditionally.  Nothing about a caller's
        tensor (address, version counter, shape) identifies its CONTENT once an earlier tensor has been freed: the
        caching allocator hands the next `torch.cat` temporary the same block.  The program is 32 small GEMMs
        (< 0.2 ms) per call, against 50 denoising steps per `sample()`."""
        B = plan.B
        if tuple(context.shape[:2]) != (B, plan.n_ctx):
            raise ValueError(f"context {tuple(context.shape)} does not fit the plan ({B}, {plan.n_ctx}, ...)")
        plan.ctx_txt.copy_(context[:, :77].reshape(B * 77, -1))
        plan.ctx_img.copy_(context[:, 77:].reshape(plan.ctx_img.shape[0], -1))   # (b t) x 16 or b x (n_ctx - 77) rows
        self._execute(plan.ctx, executor)

    def load_inputs(self, plan, x, timesteps, fs) -> None:
        B = plan.B
        plan.x_in.copy_(x)
        plan.t_in.copy_(timesteps.to(torch.float32))
        if self.lay.fs_condition:
            if fs is None:
                plan.fs_in.fill_(float(self.lay.default_fs))
            else:
                plan.fs_in.copy_(torch.as_tensor(fs, device=self.dev).to(torch.float32).reshape(-1).expand(B))

    @torch.no_grad()
    def forward(self, x: torch.Tensor, timesteps: torch.Tensor, context: torch.Tensor, fs=None,
                executor=None) -> torch.Tensor:
        """`executor` (tests only) interprets the recorded program instead of launching it."""
        B, _, T, H, W = x.shape
        plan = self.plan_for(B, T, H, W, context.shape[1])
        self.set_context(plan, context, executor)
        self.load_inputs(plan, x, timesteps, fs)
        self._execute(plan.main, executor, self.use_graph)
        return plan.y_out

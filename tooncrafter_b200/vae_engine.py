"""CUDA execution engines for the first stage: the dual-reference video decoder (AutoencoderKL_Dualref /
VideoDecoder, `DecoderEngine`), the plain per-frame decoder of AutoencoderKL (`PlainDecoderEngine`) and the shared
encoder (`EncoderEngine`).

Reference semantics restated (paths relative to /root/reference):
  Decoder.forward                     lvdm/models/autoencoder_dualref.py:489-527
  VideoResBlock / ResnetBlock / 3-D ResBlock (skip_t_emb)         :72-92, 672-698, 892-911
  MemoryEfficientAttnBlock (mid, 1 head, d = C)                   :172-206
  MemoryEfficientCrossAttentionWrapperFusion (levels 2, 3)        :270-341
  Combiner (levels 0, 1 and before conv_out)                      :357-368
  AE3DConv (conv_out + time_mix_conv)                             :929-935
  AutoencoderKL.decode skips post_quant_conv when kwargs are given  lvdm/models/autoencoder.py:112-116
One call decodes ONE chunk of T latents of ONE clip (the only case in which the reference is well defined);
the T = 16 and T = 14 passes of scripts/evaluation/inference.py:262-270 use two plans.

H100-first notes: the learned alpha-blend of VideoResBlock is folded into the last temporal conv's epilogue
(out = s + sigmoid(mix) * h), the Combiner's add is the residual of its own 1x1-conv GEMM written in place,
reference-frame K/V projections are computed once per clip, and the mid-block softmax bias trick
(P (V + 1 b^T) = P V + b^T) lets V^T be produced directly by a GEMM.
"""
from __future__ import annotations

from typing import List

import torch
import torch.nn as nn

from . import ops
from .engine import (_P, _f, _h, gemm, groupnorm, linear, pack_conv, pack_linear, pack_norm, pack_resblock, resblock,
                     temporal_conv)
from .layout import DecoderLayout
from .runtime import Act, Arena, Builder, Engine, Program


def pack_vae_resnet(m, dev) -> _P:
    """ResnetBlock, or VideoResBlock when it has a time_stack (alpha = sigmoid(mix_factor))."""
    skip = getattr(m, "nin_shortcut", None)
    ts = getattr(m, "time_stack", None)
    if ts is None:
        return pack_resblock(dev, m.norm1, m.conv1, m.norm2, m.conv2, skip)
    mf = m.mix_factor.detach().float()
    alpha = 0.5 if mf.is_meta else float(torch.sigmoid(mf).item())    # meta: planning-only engines (host tests)
    return pack_resblock(dev, m.norm1, m.conv1, m.norm2, m.conv2, skip,
                         ((ts.in_layers[0], ts.in_layers[2]), (ts.out_layers[0], ts.out_layers[3])), alpha)


def pack_mid_attention(a, C: int, dev) -> _P:
    return _P(C=C, norm=pack_norm(a.norm, dev),
              qkv_w=_h(torch.cat([a.q.weight.reshape(C, C), a.k.weight.reshape(C, C), a.v.weight.reshape(C, C)], 0), dev),
              qkv_b=_f(torch.cat([a.q.bias, a.k.bias, a.v.bias], 0), dev),
              o_w=pack_linear(a.proj_out.weight, dev), o_b=_f(a.proj_out.bias, dev))


def mid_attention(bld: Builder, p: _P, x: Act, dst: Act) -> None:
    """AttnBlock (autoencoder_dualref.py:172-206, ae_modules.py:28-75): GroupNorm -> fused q/k/v 1x1 convs -> one fused
    single-head attention kernel per call (head dim = C, scores never leave the SM) -> proj_out + residual."""
    N, H, W, C = x.N, x.H, x.W, p.C
    if C % 64 or C > 512 or (C > 256 and C % 128):
        raise NotImplementedError(f"mid-block attention: {C} channels (tc_attention_wide takes multiples of 64 up to 512, "
                                  f"of 128 above 256)")
    n = bld.act(N, H, W, C)
    groupnorm(bld, x, n, p.norm)
    qkv = bld.act(N, H, W, 3 * C)
    linear(bld, n, p.qkv_w, qkv, bias=p.qkv_b)
    n.free()
    att = bld.act(N, H, W, C)
    bld.op(ops.attention_wide, qkv.t, att.t, batches=N, L=H * W, D=C, scale=C ** -0.5, ld=3 * C, ldo=C,
           q_offset=0, k_offset=C, v_offset=2 * C)
    qkv.free()
    linear(bld, att, p.o_w, dst, bias=p.o_b, res=x)
    att.free()


class DecoderEngine(Engine):
    def __init__(self, decoder: nn.Module, device=None, arena_bytes: int = 0, use_graph: bool = True,
                 plan_only: bool = False):
        super().__init__(decoder, device, use_graph, plan_only)
        self.lay: DecoderLayout = decoder.layout
        self.arena_bytes = arena_bytes
        self._pack(decoder)

    # ---------------------------------------------------------------------------------- packing
    def _pack(self, d: nn.Module):
        dev, lay = self.dev, self.lay
        self.cpad_in = (lay.z_channels + 63) // 64 * 64
        self.p_conv_in = _P(w=pack_conv(d.conv_in.weight, dev, self.cpad_in), b=_f(d.conv_in.bias, dev))
        self.p_mid1, self.p_mid2 = pack_vae_resnet(d.mid.block_1, dev), pack_vae_resnet(d.mid.block_2, dev)
        self.p_attn = pack_mid_attention(d.mid.attn_1, lay.block_in, dev)
        self.p_levels: List[_P] = []
        for i, lv in enumerate(lay.levels):
            up = d.up[i]
            p = _P(channels=lv["channels"], refine=lv["refine"], upsample=lv["upsample"])
            p.blocks = [pack_vae_resnet(up.block[j], dev) for j in range(len(lv["blocks"]))]
            r = d.attn_refinement[i]
            if lv["refine"] == "fusion":
                heads = r.to_q.weight.shape[0] // 64
                p.fus = _P(heads=heads, norm=pack_norm(r.norm, dev), q_w=pack_linear(r.to_q.weight, dev),
                           kv_w=_h(torch.cat([r.to_k.weight, r.to_v.weight], 0), dev),
                           o_w=pack_linear(r.to_out[0].weight, dev), o_b=_f(r.to_out[0].bias, dev))
            else:
                p.comb = _P(w=pack_linear(r.conv.weight, dev), b=_f(r.conv.bias, dev))
            if lv["upsample"]:
                p.up_w, p.up_b = pack_conv(up.upsample.conv.weight, dev), _f(up.upsample.conv.bias, dev)
            self.p_levels.append(p)
        rf = d.attn_refinement[lay.num_resolutions]
        self.p_final = _P(norm=pack_norm(d.norm_out, dev), comb_w=pack_linear(rf.conv.weight, dev),
                          comb_b=_f(rf.conv.bias, dev), out_w=pack_conv(d.conv_out.weight, dev),
                          out_b=_f(d.conv_out.bias, dev),
                          tmix_w=pack_conv(d.conv_out.time_mix_conv.weight, dev, 64),
                          tmix_b=_f(d.conv_out.time_mix_conv.bias, dev))

    # ---------------------------------------------------------------------------------- builders
    def _fusion(self, bld: Builder, p: _P, x: Act, dst: Act, kv: torch.Tensor, n_kv: int) -> None:
        N, H, W, C = x.N, x.H, x.W, x.C
        n = bld.act(N, H, W, C)
        groupnorm(bld, x, n, p.norm)
        inner = p.heads * 64
        q = bld.act(N, H, W, inner)
        linear(bld, n, p.q_w, q)
        n.free()
        att = bld.act(N, H, W, inner)
        bld.op(ops.attention, q.t, [dict(k=kv, v=kv, ldk=2 * inner, ldv=2 * inner, Lk=n_kv, kv_div=N, v_offset=inner)],
               att.t, q_batches=N, Lq=H * W, heads=p.heads, scale=64 ** -0.5, ldq=inner, ldo=inner)
        q.free()
        linear(bld, att, p.o_w, dst, bias=p.o_b, res=x)
        att.free()

    @staticmethod
    def _combine(bld: Builder, w, b, x: Act, ctx_tokens: torch.Tensor, C: int) -> None:
        """x[frame 0] += conv1x1(ctx[0]); x[frame -1] += conv1x1(ctx[1])  (in place: out aliases the residual)."""
        HW = x.H * x.W
        for which, frame in ((0, 0), (1, x.N - 1)):
            src = Act(ctx_tokens, 1, 1, HW, C, C, which * HW * C)
            tgt = Act(x.t, 1, 1, HW, x.C, x.ld, x.off + frame * HW * x.ld)
            linear(bld, src, w, tgt, bias=b, res=tgt)

    # ---------------------------------------------------------------------------------- plan
    def _build(self, T: int, h: int, w: int):
        lay, dev = self.lay, self.dev
        nlev = lay.num_resolutions
        H0, W0 = h * 2 ** (nlev - 1), w * 2 ** (nlev - 1)
        biggest = T * H0 * W0 * max(lay.levels[0]["channels"], 2 * lay.levels[0]["channels"]) * 2
        arena_bytes = self.arena_bytes or int(biggest * 7 + T * (h * w) ** 2 * 2 + (512 << 20))
        arena = Arena(arena_bytes, dev)
        main, ctxp = Program(), Program()
        bld, cb = Builder(arena, main), Builder(arena, ctxp)
        plan = _P(T=T, h=h, w=w, arena=arena, main=main, ctx=ctxp)
        plan.z_in = torch.zeros(T, lay.z_channels, 1, h, w, dtype=torch.float32, device=dev)   # (frames as batch)
        z_cl = torch.zeros(T * h * w * self.cpad_in, dtype=torch.float16, device=dev)
        main.add(ops.ncthw_to_cl, plan.z_in, z_cl, B=T, C_=lay.z_channels, T=1, H=h, W=w, Cpad=self.cpad_in, coff=0,
                 scale=1.0)
        # reference-frame context: static NCTHW fp32 inputs -> channels-last tokens (+ fused K/V for fusion levels)
        plan.ref_in, plan.ref_tok, plan.kv = [], [], {}
        for i in range(nlev + 1):
            lv = i if i < nlev else 0
            c = lay.levels[lv]["channels"] if i < nlev else lay.levels[0]["channels"]
            hh, ww = (h * 2 ** (nlev - 1 - lv), w * 2 ** (nlev - 1 - lv))
            rin = torch.zeros(1, c, 2, hh, ww, dtype=torch.float32, device=dev)
            tok = torch.zeros(2 * hh * ww * c, dtype=torch.float16, device=dev)
            ctxp.add(ops.ncthw_to_cl, rin, tok, B=1, C_=c, T=2, H=hh, W=ww, Cpad=c, coff=0, scale=1.0)
            plan.ref_in.append(rin)
            plan.ref_tok.append(tok)
            if i < nlev and self.p_levels[i].refine == "fusion":
                p = self.p_levels[i].fus
                inner = p.heads * 64
                kv = torch.zeros(2 * hh * ww, 2 * inner, dtype=torch.float16, device=dev)
                linear(cb, Act(tok, 1, 1, 2 * hh * ww, c, c), p.kv_w, Act(kv, 1, 1, 2 * hh * ww, 2 * inner, 2 * inner))
                plan.kv[i] = (kv, 2 * hh * ww)

        x = Act(z_cl, T, h, w, self.cpad_in, self.cpad_in)
        cur = bld.act(T, h, w, lay.block_in)
        gemm(bld, x, self.p_conv_in.w, ops.TAPS_3x3, cur, bias=self.p_conv_in.b)
        plan.marks = []

        nxt = bld.act(T, h, w, lay.block_in)
        resblock(bld, self.p_mid1, cur, nxt, T=T); cur.free(); cur = nxt
        nxt = bld.act(T, h, w, lay.block_in)
        mid_attention(bld, self.p_attn, cur, nxt); cur.free(); cur = nxt
        nxt = bld.act(T, h, w, lay.block_in)
        resblock(bld, self.p_mid2, cur, nxt, T=T); cur.free(); cur = nxt
        plan.marks.append((len(main), "mid", cur))
        for i in reversed(range(nlev)):
            p = self.p_levels[i]
            for rb in p.blocks:
                nxt = bld.act(T, cur.H, cur.W, rb.cout)
                resblock(bld, rb, cur, nxt, T=T); cur.free(); cur = nxt
            if p.refine == "fusion":
                nxt = bld.act(T, cur.H, cur.W, cur.C)
                kv, n_kv = plan.kv[i]
                self._fusion(bld, p.fus, cur, nxt, kv, n_kv); cur.free(); cur = nxt
            else:
                self._combine(bld, p.comb.w, p.comb.b, cur, plan.ref_tok[i], cur.C)
            if p.upsample:
                up = bld.act(T, 2 * cur.H, 2 * cur.W, cur.C)
                bld.op(ops.upsample2x, cur.t, up.t, N=T, H=cur.H, W=cur.W, C_=cur.C)
                cur.free()
                nxt = bld.act(T, up.H, up.W, up.C)
                gemm(bld, up, p.up_w, ops.TAPS_3x3, nxt, bias=p.up_b)
                up.free()
                cur = nxt
            plan.marks.append((len(main), f"level{i}", cur))
        pf = self.p_final
        g = bld.act(T, cur.H, cur.W, cur.C)
        groupnorm(bld, cur, g, pf.norm, silu=True)
        cur.free()
        self._combine(bld, pf.comb_w, pf.comb_b, g, plan.ref_tok[nlev], g.C)
        # conv_out (C -> out_ch) into a zero-initialised 64-channel buffer, then the (3,1,1) time-mix conv
        Hf, Wf = g.H, g.W
        co_t = torch.zeros(T * Hf * Wf * 64, dtype=torch.float16, device=dev)
        co = Act(co_t, T, Hf, Wf, 64, 64)
        gemm(bld, g, pf.out_w, ops.TAPS_3x3, co, bias=pf.out_b, n_cols=lay.out_ch)
        g.free()
        fin = bld.act(T, Hf, Wf, 16)
        temporal_conv(bld, co, pf.tmix_w, fin, 1, bias=pf.tmix_b, n_cols=lay.out_ch)
        plan.y_out = torch.zeros(T, lay.out_ch, 1, Hf, Wf, dtype=torch.float16, device=dev)
        main.add(ops.cl_to_ncthw, fin.t, plan.y_out, B=T, C_=lay.out_ch, T=1, H=Hf, W=Wf, ldx=16)
        return plan

    def set_ref_context(self, plan, ref_context, executor=None) -> None:
        """Copy the reference-frame maps in and re-run the packing / fusion-K/V program on EVERY decode: tensor
        addresses recycle between clips (the maps are per-clip temporaries), so no pointer-derived key may skip it.
        Cost: ~0.6 GB of traffic + 2 GEMMs, ~0.2 ms against a 50 ms decode."""
        if len(ref_context) != len(plan.ref_in):
            raise ValueError(f"ref_context must hold {len(plan.ref_in)} maps")
        for dst, src in zip(plan.ref_in, ref_context):
            if tuple(src.shape) != tuple(dst.shape):
                raise ValueError(f"ref_context map {tuple(src.shape)} != expected {tuple(dst.shape)} "
                                 "(one clip per decode call: batch must be 1)")
            dst.copy_(src)
        self._execute(plan.ctx, executor)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, ref_context, executor=None) -> torch.Tensor:
        """z [T, z_channels, h, w] (already divided by scale_factor), ref_context: 5 maps [1, C, 2, H_l, W_l]
        -> [T, 3, 8h, 8w] fp16."""
        if ref_context is None:
            raise NotImplementedError("VideoDecoder without ref_context is outside the supported hot path")
        T, _, h, w = z.shape
        plan = self.plan_for(T, h, w)
        self.set_ref_context(plan, ref_context, executor)
        plan.z_in.copy_(z.reshape(plan.z_in.shape))
        self._execute(plan.main, executor, self.use_graph)
        return plan.y_out.reshape(T, self.lay.out_ch, plan.y_out.shape[-2], plan.y_out.shape[-1])


class PlainDecoderEngine(Engine):
    """AutoencoderKL.decode(z) without kwargs for the plain per-frame Decoder: post_quant_conv + Decoder.forward.

    Reference: lvdm/models/autoencoder.py:112-116 (post_quant_conv), lvdm/modules/networks/ae_modules.py:538-575
    (Decoder.forward), :153-213 (ResnetBlock, temb None), :28-75 (AttnBlock), :78-89 (Upsample, nearest + 3x3 conv).
    Every frame is decoded independently, so one plan serves any number of frames N and chunking does not change the
    result."""

    def __init__(self, ae: nn.Module, device=None, arena_bytes: int = 0, use_graph: bool = True,
                 plan_only: bool = False):
        super().__init__(ae, device, use_graph, plan_only)
        self.lay: DecoderLayout = ae.decoder.layout
        self.arena_bytes = arena_bytes
        self._pack(ae)

    @staticmethod
    def _weights(ae):
        return (ae.decoder, ae.post_quant_conv)

    def _pack(self, ae):
        dev, lay, d = self.dev, self.lay, ae.decoder
        self.cpad_in = (lay.z_channels + 63) // 64 * 64
        pq = ae.post_quant_conv.weight.detach()
        self.p_pq = _P(w=_h(torch.nn.functional.pad(pq.reshape(pq.shape[0], -1), (0, self.cpad_in - pq.shape[1])), dev),
                       b=_f(ae.post_quant_conv.bias, dev))
        self.p_conv_in = _P(w=pack_conv(d.conv_in.weight, dev, self.cpad_in), b=_f(d.conv_in.bias, dev))
        self.p_mid1, self.p_mid2 = pack_vae_resnet(d.mid.block_1, dev), pack_vae_resnet(d.mid.block_2, dev)
        self.p_attn = pack_mid_attention(d.mid.attn_1, lay.block_in, dev)
        self.p_levels: List[_P] = []
        for i, lv in enumerate(lay.levels):
            up = d.up[i]
            p = _P(blocks=[pack_vae_resnet(up.block[j], dev) for j in range(len(lv["blocks"]))], upsample=lv["upsample"])
            if lv["upsample"]:
                p.up_w, p.up_b = pack_conv(up.upsample.conv.weight, dev), _f(up.upsample.conv.bias, dev)
            self.p_levels.append(p)
        self.p_final = _P(norm=pack_norm(d.norm_out, dev), out_w=pack_conv(d.conv_out.weight, dev),
                          out_b=_f(d.conv_out.bias, dev))

    def arena_size(self, N: int, h: int, w: int) -> int:
        """Bytes of activation arena a plan for N frames of an h x w latent takes: 3.5 maps of the widest
        full-resolution activation (level 1's channels after its upsampling; the program peaks at 3.25 of them in
        level 0's first ResnetBlock) plus 64 MiB of slack for the low-resolution levels."""
        lay = self.lay
        nlev = lay.num_resolutions
        H0, W0 = h * 2 ** (nlev - 1), w * 2 ** (nlev - 1)
        widest = max(lv["channels"] for lv in lay.levels[:2])
        return self.arena_bytes or int(3.5 * N * H0 * W0 * widest * 2 + (64 << 20))

    def _build(self, N: int, h: int, w: int):
        lay, dev = self.lay, self.dev
        arena = Arena(self.arena_size(N, h, w), dev)
        main = Program()
        bld = Builder(arena, main)
        plan = _P(N=N, h=h, w=w, arena=arena, main=main)
        plan.z_in = torch.zeros(N, lay.z_channels, 1, h, w, dtype=torch.float32, device=dev)
        # the padding channels of both buffers stay zero: conv_in and post_quant_conv read all cpad_in of them
        z_cl = torch.zeros(N * h * w * self.cpad_in, dtype=torch.float16, device=dev)
        pq_t = torch.zeros(N * h * w * self.cpad_in, dtype=torch.float16, device=dev)
        main.add(ops.ncthw_to_cl, plan.z_in, z_cl, B=N, C_=lay.z_channels, T=1, H=h, W=w, Cpad=self.cpad_in, coff=0,
                 scale=1.0)
        pq = Act(pq_t, N, h, w, self.cpad_in, self.cpad_in)
        linear(bld, Act(z_cl, N, h, w, self.cpad_in, self.cpad_in), self.p_pq.w, pq, bias=self.p_pq.b,
               n_cols=lay.z_channels)
        cur = bld.act(N, h, w, lay.block_in)
        gemm(bld, pq, self.p_conv_in.w, ops.TAPS_3x3, cur, bias=self.p_conv_in.b)

        nxt = bld.act(N, h, w, lay.block_in)
        resblock(bld, self.p_mid1, cur, nxt); cur.free(); cur = nxt
        nxt = bld.act(N, h, w, lay.block_in)
        mid_attention(bld, self.p_attn, cur, nxt); cur.free(); cur = nxt
        nxt = bld.act(N, h, w, lay.block_in)
        resblock(bld, self.p_mid2, cur, nxt); cur.free(); cur = nxt
        for i in reversed(range(lay.num_resolutions)):
            p = self.p_levels[i]
            for rb in p.blocks:
                nxt = bld.act(N, cur.H, cur.W, rb.cout)
                resblock(bld, rb, cur, nxt); cur.free(); cur = nxt
            if p.upsample:
                up = bld.act(N, 2 * cur.H, 2 * cur.W, cur.C)
                bld.op(ops.upsample2x, cur.t, up.t, N=N, H=cur.H, W=cur.W, C_=cur.C)
                cur.free()
                nxt = bld.act(N, up.H, up.W, up.C)
                gemm(bld, up, p.up_w, ops.TAPS_3x3, nxt, bias=p.up_b)
                up.free()
                cur = nxt
        pf = self.p_final
        g = bld.act(N, cur.H, cur.W, cur.C)
        groupnorm(bld, cur, g, pf.norm, silu=True)
        cur.free()
        # conv_out (C -> out_ch) into a 64-channel buffer, read back as NCHW
        Hf, Wf = g.H, g.W
        co_t = torch.zeros(N * Hf * Wf * 64, dtype=torch.float16, device=dev)
        gemm(bld, g, pf.out_w, ops.TAPS_3x3, Act(co_t, N, Hf, Wf, 64, 64), bias=pf.out_b, n_cols=lay.out_ch)
        g.free()
        plan.y_out = torch.zeros(N, lay.out_ch, 1, Hf, Wf, dtype=torch.float16, device=dev)
        main.add(ops.cl_to_ncthw, co_t, plan.y_out, B=N, C_=lay.out_ch, T=1, H=Hf, W=Wf, ldx=64)
        return plan

    @torch.no_grad()
    def decode(self, z: torch.Tensor, executor=None) -> torch.Tensor:
        """z [N, z_channels, h, w] (already divided by scale_factor) -> [N, 3, 8h, 8w] fp16, a view of the plan's
        static output buffer (valid until the next decode of the same geometry)."""
        N, _, h, w = z.shape
        plan = self.plan_for(N, h, w)
        plan.z_in.copy_(z.reshape(plan.z_in.shape))
        self._execute(plan.main, executor, self.use_graph)
        return plan.y_out.reshape(N, self.lay.out_ch, plan.y_out.shape[-2], plan.y_out.shape[-1])


class EncoderEngine(Engine):
    """AutoencoderKL.encode(x, return_hidden_states=True): Encoder + quant_conv.

    Reference: lvdm/modules/networks/ae_modules.py:432-475 (Encoder.forward), :153-213 (ResnetBlock), :28-75
    (AttnBlock), :92-108 (Downsample, asymmetric pad); lvdm/models/autoencoder.py:100-105 (quant_conv)."""

    def __init__(self, ae: nn.Module, device=None, arena_bytes: int = 0, use_graph: bool = False,
                 plan_only: bool = False):
        super().__init__(ae, device, use_graph, plan_only)
        self.lay = ae.encoder.layout
        self.arena_bytes = arena_bytes
        self._pack(ae)

    @staticmethod
    def _weights(ae):
        return (ae.encoder, ae.quant_conv)

    def _pack(self, ae):
        dev, lay, e = self.dev, self.lay, ae.encoder
        self.cpad_in = (lay.in_channels + 63) // 64 * 64
        self.p_conv_in = _P(w=pack_conv(e.conv_in.weight, dev, self.cpad_in), b=_f(e.conv_in.bias, dev))
        self.p_levels = []
        for i, lv in enumerate(lay.levels):
            d = e.down[i]
            p = _P(blocks=[pack_vae_resnet(d.block[j], dev) for j in range(len(lv["blocks"]))], down=lv["downsample"],
                   channels=lv["channels"])
            if lv["downsample"]:
                p.down_w, p.down_b = pack_conv(d.downsample.conv.weight, dev), _f(d.downsample.conv.bias, dev)
            self.p_levels.append(p)
        self.p_mid1, self.p_mid2 = pack_vae_resnet(e.mid.block_1, dev), pack_vae_resnet(e.mid.block_2, dev)
        self.p_attn = pack_mid_attention(e.mid.attn_1, lay.block_in, dev)
        self.zc2 = e.conv_out.weight.shape[0]
        self.p_out = _P(norm=pack_norm(e.norm_out, dev), w=pack_conv(e.conv_out.weight, dev), b=_f(e.conv_out.bias, dev),
                        q_w=_h(torch.nn.functional.pad(ae.quant_conv.weight.detach().reshape(ae.quant_conv.weight.shape[0], -1),
                                                       (0, 64 - self.zc2)), dev),
                        q_b=_f(ae.quant_conv.bias, dev), q_out=ae.quant_conv.weight.shape[0])

    def _build(self, N: int, H: int, W: int):
        lay, dev = self.lay, self.dev
        biggest = N * H * W * lay.ch * 2
        arena = Arena(self.arena_bytes or int(biggest * 10 + N * ((H // 8) * (W // 8)) ** 2 * 2 + (256 << 20)), dev)
        main = Program()
        bld = Builder(arena, main)
        plan = _P(N=N, H=H, W=W, arena=arena, main=main)
        plan.x_in = torch.zeros(N, lay.in_channels, 1, H, W, dtype=torch.float32, device=dev)
        x_cl = torch.zeros(N * H * W * self.cpad_in, dtype=torch.float16, device=dev)
        main.add(ops.ncthw_to_cl, plan.x_in, x_cl, B=N, C_=lay.in_channels, T=1, H=H, W=W, Cpad=self.cpad_in, coff=0,
                 scale=1.0)
        plan.hidden = []

        def export(a: Act):
            out = torch.zeros(N, a.C, 1, a.H, a.W, dtype=torch.float16, device=dev)
            main.add(ops.cl_to_ncthw, a.t, out, B=N, C_=a.C, T=1, H=a.H, W=a.W, ldx=a.ld, x_offset=a.off)
            return out

        first = bld.act(N, H, W, lay.ch)
        gemm(bld, Act(x_cl, N, H, W, self.cpad_in, self.cpad_in), self.p_conv_in.w, ops.TAPS_3x3, first,
             bias=self.p_conv_in.b)
        first_out = export(first)
        cur = first
        for p in self.p_levels:
            for rb in p.blocks:
                nxt = bld.act(N, cur.H, cur.W, rb.cout)
                resblock(bld, rb, cur, nxt)
                cur.free()
                cur = nxt
            plan.hidden.append(export(cur))
            if p.down:
                ph = bld.act(4 * N, cur.H // 2, cur.W // 2, cur.C)
                bld.op(ops.phase_split2, cur.t, ph.t, N=N, H=cur.H, W=cur.W, C_=cur.C)
                nxt = bld.act(N, cur.H // 2, cur.W // 2, cur.C)
                gemm(bld, ph, p.down_w, ops.taps_3x3_stride2(N, pad=0), nxt, bias=p.down_b)
                ph.free()
                cur.free()
                cur = nxt
        plan.hidden.append(first_out)
        nxt = bld.act(N, cur.H, cur.W, cur.C)
        resblock(bld, self.p_mid1, cur, nxt); cur.free(); cur = nxt
        nxt = bld.act(N, cur.H, cur.W, cur.C)
        mid_attention(bld, self.p_attn, cur, nxt); cur.free(); cur = nxt
        nxt = bld.act(N, cur.H, cur.W, cur.C)
        resblock(bld, self.p_mid2, cur, nxt); cur.free(); cur = nxt
        g = bld.act(N, cur.H, cur.W, cur.C)
        groupnorm(bld, cur, g, self.p_out.norm, silu=True)
        cur.free()
        co_t = torch.zeros(N * g.H * g.W * 64, dtype=torch.float16, device=dev)
        co = Act(co_t, N, g.H, g.W, 64, 64)
        gemm(bld, g, self.p_out.w, ops.TAPS_3x3, co, bias=self.p_out.b, n_cols=self.zc2)
        g.free()
        mo = bld.act(N, co.H, co.W, 16)
        linear(bld, co, self.p_out.q_w, mo, bias=self.p_out.q_b, n_cols=self.p_out.q_out)
        plan.moments = torch.zeros(N, self.p_out.q_out, 1, co.H, co.W, dtype=torch.float32, device=dev)
        main.add(ops.cl_to_ncthw, mo.t, plan.moments, B=N, C_=self.p_out.q_out, T=1, H=co.H, W=co.W, ldx=16)
        return plan

    @torch.no_grad()
    def encode(self, x: torch.Tensor, executor=None):
        """x [N, 3, H, W] in [-1, 1] -> (moments [N, 2*embed, H/8, W/8] fp32, [5 hidden maps [N, C, H_l, W_l] fp16])."""
        N, _, H, W = x.shape
        plan = self.plan_for(N, H, W)
        plan.x_in.copy_(x.reshape(plan.x_in.shape))
        self._execute(plan.main, executor, self.use_graph)
        sq = lambda t: t.reshape(t.shape[0], t.shape[1], t.shape[3], t.shape[4]).clone()
        return sq(plan.moments), [sq(h) for h in plan.hidden]

"""TEST INFRASTRUCTURE ONLY — CPU fp32 restatement of the image-conditioning Resampler.

Follows lvdm/modules/encoders/resampler.py of the reference: Resampler.forward :132-145 (latents repeated per sample,
proj_in, depth x [PerceiverAttention + latents, FeedForward + latents], proj_out, norm_out), PerceiverAttention.forward
:65-93 (norm1 on the image tokens, norm2 on the latents, q from the latents, k/v from cat(image tokens, latents), both
scaled by dim_head^-1/4, fp32 softmax over ALL keys), FeedForward :27-34 (LayerNorm, Linear, exact GELU, Linear; no biases).
Pinned against the unmodified reference through tests/golden/resampler_tiny.npz (tests/golden/make_golden_resampler.py).
Only tests/ may import this module.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def resampler_forward(sd: dict, x: torch.Tensor, heads: int, prefix: str = "") -> torch.Tensor:
    """sd: state dict with the reference's keys (optionally under `prefix`), x [B, n1, embedding_dim] fp32."""
    g = lambda k: sd[prefix + k].float()
    depth = 1 + max(int(k[len(prefix):].split(".")[1]) for k in sd if k.startswith(prefix + "layers."))
    B = x.shape[0]
    lat = g("latents").repeat(B, 1, 1)
    xp = F.linear(x.float(), g("proj_in.weight"), g("proj_in.bias"))
    dim = lat.shape[-1]
    for i in range(depth):
        a = f"layers.{i}.0."
        xn = F.layer_norm(xp, (dim,), g(a + "norm1.weight"), g(a + "norm1.bias"))
        ln = F.layer_norm(lat, (dim,), g(a + "norm2.weight"), g(a + "norm2.bias"))
        q = F.linear(ln, g(a + "to_q.weight"))
        k, v = F.linear(torch.cat([xn, ln], dim=1), g(a + "to_kv.weight")).chunk(2, dim=-1)
        split = lambda t: t.view(B, t.shape[1], heads, -1).transpose(1, 2)
        q, k, v = split(q), split(k), split(v)
        s = 1.0 / math.sqrt(math.sqrt(q.shape[-1]))
        w = torch.softmax((q * s) @ (k * s).transpose(-2, -1), dim=-1)
        o = (w @ v).permute(0, 2, 1, 3).reshape(B, lat.shape[1], -1)
        lat = F.linear(o, g(a + "to_out.weight")) + lat
        f = f"layers.{i}.1."
        h = F.layer_norm(lat, (dim,), g(f + "0.weight"), g(f + "0.bias"))
        h = F.linear(F.gelu(F.linear(h, g(f + "1.weight"))), g(f + "3.weight"))
        lat = h + lat
    out = F.linear(lat, g("proj_out.weight"), g("proj_out.bias"))
    return F.layer_norm(out, (out.shape[-1],), g("norm_out.weight"), g("norm_out.bias"))

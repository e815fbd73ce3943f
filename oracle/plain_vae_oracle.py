"""TEST INFRASTRUCTURE ONLY — CPU fp32 restatement of the plain AutoencoderKL decoder (post_quant_conv + the per-frame
2-D Decoder), reusing the ResnetBlock / AttnBlock restatements of vae_oracle.  Pinned against the unmodified reference
by tests/golden/plain_decoder_tiny.npz (tests/golden/make_golden_plain_vae.py).  Paths cited are relative to the
reference repository.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .unet_oracle import SD, group_norm
from .vae_oracle import mid_attention, resnet2d, swish


@torch.no_grad()
def decode_plain(sd, lay, z, prefix="first_stage_model."):
    """lvdm/models/autoencoder.py:112-116 (decode without kwargs: post_quant_conv first) +
    lvdm/modules/networks/ae_modules.py:538-575 (Decoder.forward, attn_resolutions = []).
    z [N, embed_dim, h, w] (already divided by scale_factor) -> [N, out_ch, 8h, 8w]."""
    q = SD(sd, prefix)
    p = q.sub("decoder.")
    h = F.conv2d(z.float(), q("post_quant_conv.weight"), q("post_quant_conv.bias"))
    h = F.conv2d(h, p("conv_in.weight"), p("conv_in.bias"), padding=1)
    h = resnet2d(p.sub("mid.block_1."), h)
    h = mid_attention(p.sub("mid.attn_1."), h)
    h = resnet2d(p.sub("mid.block_2."), h)
    for i_level in reversed(range(lay.num_resolutions)):
        lv = lay.levels[i_level]
        for j in range(len(lv["blocks"])):
            h = resnet2d(p.sub(f"up.{i_level}.block.{j}."), h)
        if lv["upsample"]:
            u = p.sub(f"up.{i_level}.upsample.")
            h = F.conv2d(F.interpolate(h, scale_factor=2, mode="nearest"), u("conv.weight"), u("conv.bias"), padding=1)
    h = swish(group_norm(h, p.sub("norm_out."), 1e-6))
    return F.conv2d(h, p("conv_out.weight"), p("conv_out.bias"), padding=1)


@torch.no_grad()
def decode_first_stage_plain(sd, lay, z, scale_factor=0.18215, prefix="first_stage_model."):
    """ddpm3d.py:647-683 (decode_core) for a plain first stage: z [B, 4, T, h, w] -> [B, 3, T, 8h, 8w].  Every frame
    is decoded on its own, so the perframe_ae chunking does not change the result."""
    b, c, t, hh, ww = z.shape
    zz = z.permute(0, 2, 1, 3, 4).reshape(b * t, c, hh, ww) * (1.0 / scale_factor)
    out = decode_plain(sd, lay, zz, prefix)
    return out.reshape(b, t, *out.shape[1:]).permute(0, 2, 1, 3, 4)

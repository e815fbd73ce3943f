"""TEST INFRASTRUCTURE ONLY — CPU fp32 restatement of the two OpenCLIP conditioning encoders.

Reads a state dict with open_clip's CLIP key names (optionally under `prefix`, e.g. "cond_stage_model.model." or
"embedder.model.").  Follows lvdm/modules/encoders/condition.py of the reference:
  FrozenOpenCLIPEmbedder.encode_with_transformer :214-221 (token_embedding + positional_embedding, the residual blocks
      with the causal attn_mask, ln_final) and text_transformer_forward :223-231 (the last `layer_idx` blocks are not
      run: 1 for "penultimate");
  FrozenOpenCLIPImageEmbedderV2.encode_with_vision_transformer :342-372 (conv1 patch embedding, class token,
      positional embedding, ln_pre, the residual blocks; no ln_post / proj).  Preprocessing (:322-330) is not part of
      this module: tests pass pixels through tooncrafter_b200.modules.clip_preprocess first.
open_clip's residual block: x = x + attn(ln_1(x)); x = x + c_proj(gelu(c_fc(ln_2(x)))), exact-erf GELU, LayerNorm eps
1e-5, nn.MultiheadAttention with a fused in_proj (rows q | k | v), scale head_dim^-1/2.
Pinned against an independent implementation of the same architecture (transformers' CLIPTextModel /
CLIPVisionModel) through tests/golden/clip_tiny.npz (tests/golden/make_golden_clip.py).  Only tests/ may import this
module.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

LN_EPS = 1e-5


def _n_blocks(sd, prefix):
    return 1 + max(int(k[len(prefix):].split(".")[2]) for k in sd if k.startswith(prefix + "transformer.resblocks."))


def _blocks(sd, prefix, x, heads, n, causal):
    """open_clip Transformer over x [B, L, W] (batch-first here; the reference permutes to LND and back)."""
    g = lambda k: sd[prefix + k].float()
    B, L, W = x.shape
    for i in range(n):
        a = f"transformer.resblocks.{i}."
        h = F.layer_norm(x, (W,), g(a + "ln_1.weight"), g(a + "ln_1.bias"), LN_EPS)
        q, k, v = F.linear(h, g(a + "attn.in_proj_weight"), g(a + "attn.in_proj_bias")).chunk(3, dim=-1)
        split = lambda t: t.reshape(B, L, heads, W // heads).transpose(1, 2)
        o = F.scaled_dot_product_attention(split(q), split(k), split(v), is_causal=causal)
        x = x + F.linear(o.transpose(1, 2).reshape(B, L, W), g(a + "attn.out_proj.weight"), g(a + "attn.out_proj.bias"))
        h = F.layer_norm(x, (W,), g(a + "ln_2.weight"), g(a + "ln_2.bias"), LN_EPS)
        h = F.gelu(F.linear(h, g(a + "mlp.c_fc.weight"), g(a + "mlp.c_fc.bias")))
        x = x + F.linear(h, g(a + "mlp.c_proj.weight"), g(a + "mlp.c_proj.bias"))
    return x


def encode_text(sd: dict, tokens: torch.Tensor, heads: int, layer_idx: int = 1, prefix: str = "") -> torch.Tensor:
    """tokens [B, 77] int64 -> [B, 77, width] after ln_final; layer_idx 0 = "last", 1 = "penultimate"."""
    g = lambda k: sd[prefix + k].float()
    x = F.embedding(tokens.to(sd[prefix + "token_embedding.weight"].device), g("token_embedding.weight"))
    x = x + g("positional_embedding")
    x = _blocks(sd, prefix, x, heads, _n_blocks(sd, prefix) - layer_idx, causal=True)
    return F.layer_norm(x, (x.shape[-1],), g("ln_final.weight"), g("ln_final.bias"), LN_EPS)


def encode_image(sd: dict, pixels: torch.Tensor, heads: int, prefix: str = "") -> torch.Tensor:
    """pixels [B, 3, 224, 224] (CLIP-normalised) -> [B, 1 + grid^2, width], the transformer output."""
    vp = prefix + "visual."
    g = lambda k: sd[vp + k].float()
    w = g("conv1.weight")
    x = F.conv2d(pixels.float(), w, stride=w.shape[-1])                   # [B, W, grid, grid]
    x = x.reshape(x.shape[0], x.shape[1], -1).permute(0, 2, 1)
    cls = g("class_embedding").expand(x.shape[0], 1, -1)
    x = torch.cat([cls.to(x.dtype), x], dim=1) + g("positional_embedding")
    x = F.layer_norm(x, (x.shape[-1],), g("ln_pre.weight"), g("ln_pre.bias"), LN_EPS)
    return _blocks(sd, vp, x, heads, _n_blocks(sd, vp), causal=False)

"""Seeded synthetic weights and inputs (there is no checkpoint and no network in this environment).

Every tensor is drawn from its own generator seeded by crc32(key) ^ seed, so the values do not depend on
iteration order or on which other tensors exist, and the GPU box regenerates bit-identical weights.

A freshly constructed reference model is useless for parity: every block's last layer is zero-initialised
(openaimodel3d.py:179,269-270,381-382,545; attention.py:288-290,360-362; autoencoder_dualref.py:261-262,348-349,
640), so the UNet output is identically 0 and every transformer/temporal block is the identity.  Here all of
them get non-zero values.
"""
from __future__ import annotations

import zlib
from typing import Dict, Iterable, Tuple

import torch


def _gen(key: str, seed: int) -> torch.Generator:
    return torch.Generator(device="cpu").manual_seed((zlib.crc32(key.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)


def synthetic_tensor(key: str, shape: Tuple[int, ...], seed: int = 0, gain: float = 1.0) -> torch.Tensor:
    g = _gen(key, seed)
    shape = tuple(shape)
    if key.endswith("mix_factor"):
        return torch.zeros(shape)                       # sigmoid(0) = 0.5 blend, as the released config's alpha=0
    if len(shape) <= 1:
        n = torch.randn(shape, generator=g)
        if key.endswith("weight"):                      # GroupNorm / LayerNorm scale
            return 1.0 + 0.1 * n
        return 0.05 * n                                 # biases
    fan_in = 1
    for s in shape[1:]:
        fan_in *= s
    return torch.randn(shape, generator=g) * (gain / fan_in ** 0.5)


def synthetic_state_dict(named_shapes: Iterable[Tuple[str, Tuple[int, ...]]], seed: int = 0,
                         prefix: str = "") -> Dict[str, torch.Tensor]:
    return {k: synthetic_tensor(prefix + k, s, seed) for k, s in named_shapes}


def fill_module_(module: torch.nn.Module, seed: int = 0, prefix: str = "") -> None:
    """In-place synthetic init of every parameter of `module` (keys = prefix + state-dict key)."""
    with torch.no_grad():
        for k, p in module.named_parameters():
            p.copy_(synthetic_tensor(prefix + k, tuple(p.shape), seed).to(p.dtype))


FIRST_STAGE_TARGETS = {"plain": "lvdm.models.autoencoder.AutoencoderKL",
                       "dualref": "lvdm.models.autoencoder.AutoencoderKL_Dualref"}


def with_first_stage(config, first_stage: str):
    """A copy of a LatentVisualDiffusion config whose first stage is the plain AutoencoderKL ("plain": the DynamiCrafter
    and training configs) or AutoencoderKL_Dualref ("dualref": the ToonCrafter inference configs), same ddconfig."""
    import copy
    if first_stage not in FIRST_STAGE_TARGETS:
        raise ValueError(f"first_stage must be one of {sorted(FIRST_STAGE_TARGETS)}, got {first_stage!r}")
    cfg = copy.deepcopy(config)
    cfg["params"]["first_stage_config"]["target"] = FIRST_STAGE_TARGETS[first_stage]
    return cfg


def synthetic_model(config, device, seed: int = 0, first_stage=None) -> torch.nn.Module:
    """instantiate_from_config(config) with the weights fill_module_(model, seed) gives, built straight on `device`
    (meta skeleton, each tensor drawn on the host and copied over), so a full-size model needs no host-side copy.
    first_stage "plain" / "dualref" replaces the config's first-stage class (with_first_stage)."""
    from . import diffusion, modules
    if first_stage is not None:
        config = with_first_stage(config, first_stage)
    with torch.device("meta"):
        skeleton = diffusion.instantiate_from_config(config)
    m = skeleton.to_empty(device=device)
    m.reset_schedule_buffers()
    with torch.no_grad():
        for k, p in m.named_parameters():
            p.copy_(synthetic_tensor(k, tuple(p.shape), seed).to(p.dtype))
        for mod in m.modules():                 # constructor-made buffers that to_empty() left uninitialised
            if isinstance(mod, modules.FrozenOpenCLIPEmbedder):
                mod.model.attn_mask.fill_(float("-inf")).triu_(1)
            elif isinstance(mod, modules.FrozenOpenCLIPImageEmbedderV2):
                mod.mean.copy_(torch.tensor(modules.CLIP_MEAN))
                mod.std.copy_(torch.tensor(modules.CLIP_STD))
    return m.eval()


def synthetic_inputs(B: int, T: int, h: int, w: int, context_dim: int = 1024, seed: int = 123,
                     latent_channels: int = 4):
    """x_T, cond / uncond dicts in the shapes scripts/evaluation/inference.py:189-216 builds."""
    def r(name, *shape):
        return torch.randn(*shape, generator=_gen(name, seed))
    x_T = r("x_T", B, latent_channels, T, h, w)
    z = r("z_ref", B, latent_channels, T, h, w) * 0.18215 * 5.0     # ~ scale_factor * typical latent std
    c_concat = torch.zeros_like(z)
    c_concat[:, :, 0] = z[:, :, 0]
    c_concat[:, :, -1] = z[:, :, -1]
    ctx_c = r("ctx_cond", B, 77 + 16 * T, context_dim)
    ctx_u = r("ctx_uncond", B, 77 + 16 * T, context_dim)
    cond = {"c_crossattn": [ctx_c], "c_concat": [c_concat]}
    uncond = {"c_crossattn": [ctx_u], "c_concat": [c_concat]}
    return x_T, cond, uncond


def synthetic_ref_context(dd_ch: int, ch_mult, H: int, W: int, seed: int = 123):
    """Five encoder hidden-state maps (first+last frame) in the shapes the VideoDecoder consumes
    (ae_modules.py:432-460; scripts/evaluation/inference.py:164-178): levels 0..3 then the conv_in features."""
    out = []
    for i, m in enumerate(ch_mult):
        s = 2 ** i
        out.append(torch.randn(1, dd_ch * m, 2, H // s, W // s, generator=_gen(f"ref_context.{i}", seed)))
    out.append(torch.randn(1, dd_ch, 2, H, W, generator=_gen("ref_context.in", seed)))
    return out

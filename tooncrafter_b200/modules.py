"""Parameter holders for the hot-path networks.

These nn.Modules own parameters under EXACTLY the reference checkpoint's names (so
`load_state_dict(sd, strict=True)` of the public ToonCrafter checkpoint works, typos such as `temopral_conv`
included), but contain no arithmetic: `forward` hands the tensors to the CUDA engine (`engine.py`).

Reference constructors mirrored (names/shapes only): lvdm/modules/networks/openaimodel3d.py:109-195,239-270,
311-546; lvdm/modules/attention.py:42-78,212-229,249-291,313-363,415-439; lvdm/models/autoencoder_dualref.py
:35-70,145-170,256-262,343-349,371-487,846-880,914-927; lvdm/modules/networks/ae_modules.py:92-108,366-430,478-536;
lvdm/modules/attention_svd.py:347-371.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .layout import Layer, decoder_layout, encoder_layout, plain_decoder_layout, unet_layout


class Node(nn.Module):
    """Anonymous container; children are attached under arbitrary (also numeric) names."""

    def __init__(self, **children):
        super().__init__()
        for k, v in children.items():
            self.add_module(k, v)

    def put(self, name, module):
        self.add_module(str(name), module)
        return module

    def __getitem__(self, idx):
        return getattr(self, str(idx))


def _numbered(entries: dict) -> Node:
    n = Node()
    for k, v in entries.items():
        n.put(k, v)
    return n


def _gn(c, eps=1e-5):
    return nn.GroupNorm(32, c, eps=eps)


# ----------------------------------------------------------------------------------------------------- UNet parts
def _temporal_conv_block(c):
    def stage(first):
        return _numbered({0: _gn(c), (2 if first else 3): nn.Conv3d(c, c, (3, 1, 1), padding=(1, 0, 0))})
    return Node(conv1=stage(True), conv2=stage(False), conv3=stage(False), conv4=stage(False))


def _res_block(cin, cout, time_dim, temporal_conv):
    n = Node(
        in_layers=_numbered({0: _gn(cin), 2: nn.Conv2d(cin, cout, 3, padding=1)}),
        emb_layers=_numbered({1: nn.Linear(time_dim, cout)}),
        out_layers=_numbered({0: _gn(cout), 3: nn.Conv2d(cout, cout, 3, padding=1)}),
        skip_connection=nn.Identity() if cin == cout else nn.Conv2d(cin, cout, 1),
    )
    if temporal_conv:
        n.put("temopral_conv", _temporal_conv_block(cout))   # sic: checkpoint key (openaimodel3d.py:190)
    return n


def _attention(query_dim, context_dim, heads, d_head, image_branch):
    inner = heads * d_head
    ctx = context_dim if context_dim is not None else query_dim
    n = Node(to_q=nn.Linear(query_dim, inner, bias=False), to_k=nn.Linear(ctx, inner, bias=False),
             to_v=nn.Linear(ctx, inner, bias=False), to_out=_numbered({0: nn.Linear(inner, query_dim)}))
    if image_branch:
        n.put("to_k_ip", nn.Linear(ctx, inner, bias=False))
        n.put("to_v_ip", nn.Linear(ctx, inner, bias=False))
    return n


def _transformer_block(dim, heads, d_head, context_dim, image_branch):
    ff = Node(net=_numbered({0: Node(proj=nn.Linear(dim, 8 * dim)), 2: nn.Linear(4 * dim, dim)}))
    return Node(attn1=_attention(dim, None, heads, d_head, False), ff=ff,
                attn2=_attention(dim, context_dim, heads, d_head, image_branch),
                norm1=nn.LayerNorm(dim), norm2=nn.LayerNorm(dim), norm3=nn.LayerNorm(dim))


def _spatial_transformer(l: Layer, context_dim, image_branch):
    inner = l.heads * l.d_head
    if l.use_linear:
        pin, pout = nn.Linear(l.cin, inner), nn.Linear(inner, l.cin)
    else:
        pin, pout = nn.Conv2d(l.cin, inner, 1), nn.Conv2d(inner, l.cin, 1)
    return Node(norm=_gn(l.cin, 1e-6), proj_in=pin,
                transformer_blocks=_numbered({0: _transformer_block(inner, l.heads, l.d_head, context_dim,
                                                                    image_branch)}),
                proj_out=pout)


def _temporal_transformer(l: Layer):
    inner = l.heads * l.d_head
    if l.use_linear:
        pin, pout = nn.Linear(l.cin, inner), nn.Linear(inner, l.cin)
    else:
        pin, pout = nn.Conv1d(l.cin, inner, 1), nn.Conv1d(inner, l.cin, 1)
    return Node(norm=_gn(l.cin, 1e-6), proj_in=pin,
                transformer_blocks=_numbered({0: _transformer_block(inner, l.heads, l.d_head, None, False)}),
                proj_out=pout)


class UNetModel(nn.Module):
    """Drop-in for lvdm.modules.networks.openaimodel3d.UNetModel (same ctor kwargs, same state-dict keys)."""

    def __init__(self, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions,
                 dropout=0.0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, context_dim=None,
                 use_scale_shift_norm=False, resblock_updown=False, num_heads=-1, num_head_channels=-1,
                 transformer_depth=1, use_linear=False, use_checkpoint=False, temporal_conv=False,
                 tempspatial_aware=False, temporal_attention=True, use_relative_position=True,
                 use_causal_attention=False, temporal_length=None, use_fp16=False, addition_attention=False,
                 temporal_selfatt_only=True, image_cross_attention=False,
                 image_cross_attention_scale_learnable=False, default_fs=4, fs_condition=False):
        super().__init__()
        if image_cross_attention_scale_learnable:
            raise NotImplementedError("image_cross_attention_scale_learnable=True is outside the supported hot path")
        params = dict(locals())
        params.pop("self")
        params.pop("__class__", None)
        self.params = params
        lay = self.layout = unet_layout(params)
        self.in_channels, self.model_channels, self.out_channels = in_channels, model_channels, out_channels
        self.temporal_length = temporal_length
        self.default_fs, self.fs_condition = default_fs, fs_condition
        self.addition_attention = addition_attention
        self.use_checkpoint = use_checkpoint
        self.dtype = torch.float16 if use_fp16 else torch.float32
        mc, td = model_channels, lay.time_dim

        def mlp():
            return _numbered({0: nn.Linear(mc, td), 2: nn.Linear(td, td)})

        self.time_embed = mlp()
        if fs_condition:
            self.fps_embedding = mlp()

        def build(layers):
            blk = Node()
            for i, l in enumerate(layers):
                if l.kind == "conv_in":
                    m = nn.Conv2d(l.cin, l.cout, 3, padding=1)
                elif l.kind == "res":
                    m = _res_block(l.cin, l.cout, td, lay.temporal_conv)
                elif l.kind == "st":
                    m = _spatial_transformer(l, lay.context_dim, lay.image_cross_attention)
                elif l.kind == "tt":
                    m = _temporal_transformer(l)
                elif l.kind == "down":
                    m = Node(op=nn.Conv2d(l.cin, l.cout, 3, stride=2, padding=1))
                elif l.kind == "up":
                    m = Node(conv=nn.Conv2d(l.cin, l.cout, 3, padding=1))
                else:
                    raise ValueError(l.kind)
                blk.put(i, m)
            return blk

        self.input_blocks = Node()
        for prefix, layers in lay.input_blocks:
            self.input_blocks.put(prefix.split(".")[1], build(layers))
        if lay.init_attn:
            self.init_attn = build(lay.init_attn)
        self.middle_block = build(lay.middle_block)
        self.output_blocks = Node()
        for prefix, layers in lay.output_blocks:
            self.output_blocks.put(prefix.split(".")[1], build(layers))
        self.out = _numbered({0: _gn(mc), 2: nn.Conv2d(mc, out_channels, 3, padding=1)})
        self._engine = None

    def forward(self, x, timesteps, context=None, features_adapter=None, fs=None, **kwargs):
        """x [B, in_channels, T, H, W] fp32, timesteps [B], context [B, 77+16*T, context_dim] -> [B, out, T, H, W] fp16.

        Extra kwargs are tolerated and ignored exactly like the reference (openaimodel3d.py:548)."""
        if features_adapter is not None:
            raise NotImplementedError("features_adapter is outside the supported hot path")
        from . import runtime
        from .engine import UNetEngine
        ex = runtime.TEST_EXECUTOR
        return UNetEngine.cached(self, "_engine", ex).forward(x, timesteps, context, fs, executor=ex).clone()


# ----------------------------------------------------------------------------------------------------- VAE parts
def _vae_resnet(cin, cout):
    n = Node(norm1=_gn(cin, 1e-6), conv1=nn.Conv2d(cin, cout, 3, padding=1), norm2=_gn(cout, 1e-6),
             conv2=nn.Conv2d(cout, cout, 3, padding=1))
    if cin != cout:
        n.put("nin_shortcut", nn.Conv2d(cin, cout, 1))
    return n


def _video_res_block(cin, cout):
    n = _vae_resnet(cin, cout)
    n.put("time_stack", Node(
        in_layers=_numbered({0: _gn(cout), 2: nn.Conv3d(cout, cout, (3, 1, 1), padding=(1, 0, 0))}),
        out_layers=_numbered({0: _gn(cout), 3: nn.Conv3d(cout, cout, (3, 1, 1), padding=(1, 0, 0))})))
    n.register_parameter("mix_factor", nn.Parameter(torch.zeros(1)))
    return n


def _attn_block(c):
    return Node(norm=_gn(c, 1e-6), q=nn.Conv2d(c, c, 1), k=nn.Conv2d(c, c, 1), v=nn.Conv2d(c, c, 1),
                proj_out=nn.Conv2d(c, c, 1))


def _fusion_attn(c, heads=8, d_head=64):
    inner = heads * d_head
    return Node(to_q=nn.Linear(c, inner, bias=False), to_k=nn.Linear(c, inner, bias=False),
                to_v=nn.Linear(c, inner, bias=False), to_out=_numbered({0: nn.Linear(inner, c)}), norm=_gn(c, 1e-6))


class VideoDecoder(nn.Module):
    """Parameter holder for lvdm.models.autoencoder_dualref.VideoDecoder (time_mode 'conv-only')."""

    def __init__(self, **ddconfig):
        super().__init__()
        lay = self.layout = decoder_layout(ddconfig)
        self.conv_in = nn.Conv2d(lay.z_channels, lay.block_in, 3, padding=1)
        self.mid = Node(block_1=_video_res_block(lay.block_in, lay.block_in), attn_1=_attn_block(lay.block_in),
                        block_2=_video_res_block(lay.block_in, lay.block_in))
        self.up = Node()
        self.attn_refinement = Node()
        for i, lv in enumerate(lay.levels):
            up = Node(block=_numbered({j: _video_res_block(a, b) for j, (a, b) in enumerate(lv["blocks"])}),
                      attn=Node())
            if lv["upsample"]:
                up.put("upsample", Node(conv=nn.Conv2d(lv["channels"], lv["channels"], 3, padding=1)))
            self.up.put(i, up)
            c = lv["channels"]
            self.attn_refinement.put(i, _fusion_attn(c) if lv["refine"] == "fusion" else Node(conv=nn.Conv2d(c, c, 1)))
        c0 = lay.levels[0]["channels"]
        self.norm_out = _gn(c0, 1e-6)
        self.attn_refinement.put(lay.num_resolutions, Node(conv=nn.Conv2d(c0, c0, 1)))
        conv_out = nn.Conv2d(c0, lay.out_ch, 3, padding=1)
        conv_out.add_module("time_mix_conv", nn.Conv3d(lay.out_ch, lay.out_ch, (3, 1, 1), padding=(1, 0, 0)))
        self.conv_out = conv_out


class Decoder(nn.Module):
    """Parameter holder for lvdm.modules.networks.ae_modules.Decoder, the per-frame 2-D decoder of the plain
    AutoencoderKL (attn_resolutions = [])."""

    def __init__(self, **ddconfig):
        super().__init__()
        lay = self.layout = plain_decoder_layout(ddconfig)
        self.conv_in = nn.Conv2d(lay.z_channels, lay.block_in, 3, padding=1)
        self.mid = Node(block_1=_vae_resnet(lay.block_in, lay.block_in), attn_1=_attn_block(lay.block_in),
                        block_2=_vae_resnet(lay.block_in, lay.block_in))
        self.up = Node()
        for i, lv in enumerate(lay.levels):
            up = Node(block=_numbered({j: _vae_resnet(a, b) for j, (a, b) in enumerate(lv["blocks"])}), attn=Node())
            if lv["upsample"]:
                up.put("upsample", Node(conv=nn.Conv2d(lv["channels"], lv["channels"], 3, padding=1)))
            self.up.put(i, up)
        c0 = lay.levels[0]["channels"]
        self.norm_out = _gn(c0, 1e-6)
        self.conv_out = nn.Conv2d(c0, lay.out_ch, 3, padding=1)


class Encoder(nn.Module):
    """Parameter holder for lvdm.modules.networks.ae_modules.Encoder (attn_resolutions = [])."""

    def __init__(self, **ddconfig):
        super().__init__()
        lay = self.layout = encoder_layout(ddconfig)
        self.conv_in = nn.Conv2d(lay.in_channels, lay.ch, 3, padding=1)
        self.down = Node()
        for i, lv in enumerate(lay.levels):
            d = Node(block=_numbered({j: _vae_resnet(a, b) for j, (a, b) in enumerate(lv["blocks"])}), attn=Node())
            if lv["downsample"]:
                d.put("downsample", Node(conv=nn.Conv2d(lv["channels"], lv["channels"], 3, stride=2, padding=0)))
            self.down.put(i, d)
        c = lay.block_in
        self.mid = Node(block_1=_vae_resnet(c, c), attn_1=_attn_block(c), block_2=_vae_resnet(c, c))
        self.norm_out = _gn(c, 1e-6)
        self.conv_out = nn.Conv2d(c, 2 * lay.z_channels if lay.double_z else lay.z_channels, 3, padding=1)


# ------------------------------------------------------------------------------------ conditioning: image Resampler
class Resampler(nn.Module):
    """Drop-in for lvdm.modules.encoders.resampler.Resampler (same ctor kwargs, same state-dict keys): the perceiver
    resampler that turns CLIP image tokens into the 16 x T image-context tokens of the UNet's cross-attention
    (reference resampler.py:96-145, PerceiverAttention :49-93, FeedForward :27-34)."""

    def __init__(self, dim=1024, depth=8, dim_head=64, heads=16, num_queries=8, embedding_dim=768, output_dim=1024,
                 ff_mult=4, video_length=None):
        super().__init__()
        if dim_head != 64:
            raise NotImplementedError("the attention kernel is specialised for 64-wide heads")
        self.num_queries, self.video_length = num_queries, video_length
        self.dim, self.depth, self.heads, self.dim_head = dim, depth, heads, dim_head
        nq = num_queries * video_length if video_length is not None else num_queries
        self.latents = nn.Parameter(torch.randn(1, nq, dim) / dim ** 0.5)
        self.proj_in = nn.Linear(embedding_dim, dim)
        self.proj_out = nn.Linear(dim, output_dim)
        self.norm_out = nn.LayerNorm(output_dim)
        inner = dim_head * heads
        self.layers = nn.ModuleList()
        for _ in range(depth):
            attn = Node(norm1=nn.LayerNorm(dim), norm2=nn.LayerNorm(dim), to_q=nn.Linear(dim, inner, bias=False),
                        to_kv=nn.Linear(dim, 2 * inner, bias=False), to_out=nn.Linear(inner, dim, bias=False))
            ff = nn.Sequential(nn.LayerNorm(dim), nn.Linear(dim, int(dim * ff_mult), bias=False), nn.GELU(),
                               nn.Linear(int(dim * ff_mult), dim, bias=False))
            self.layers.append(nn.ModuleList([attn, ff]))
        self._engine = None

    def forward(self, x):
        """x [B, n_tokens, embedding_dim] (CLIP image tokens) -> [B, num_queries (* video_length), output_dim] fp32."""
        from . import runtime
        from .cond_engine import ResamplerEngine
        ex = runtime.TEST_EXECUTOR
        return ResamplerEngine.cached(self, "_engine", ex).forward(x, executor=ex).clone()


# ------------------------------------------------------------------------- conditioning: OpenCLIP text / image towers
# Geometry of the OpenCLIP architectures the reference configs name (configs/inference_512_v1.0.yaml: "ViT-H-14").
# `arch` may also be a dict of the same form (width-reduced test models).
CLIP_ARCHS = {
    "ViT-H-14": dict(embed_dim=1024,
                     text=dict(width=1024, heads=16, layers=24, ctx=77, vocab=49408),
                     vision=dict(width=1280, heads=16, layers=32, patch=14, image=224)),
}
CLIP_SOT, CLIP_EOT = 49406, 49407                    # open_clip's <start_of_text> / <end_of_text> token ids
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)      # reference condition.py:318-319
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def _clip_arch(arch):
    if isinstance(arch, dict):
        return arch
    if arch not in CLIP_ARCHS:
        raise NotImplementedError(f"OpenCLIP arch {arch!r} is not supported (supported: {sorted(CLIP_ARCHS)})")
    return CLIP_ARCHS[arch]


def _param(*shape):
    return nn.Parameter(torch.empty(shape), requires_grad=False)


def _clip_linear(cin, cout, bias=True):
    n = Node()
    n.register_parameter("weight", _param(cout, cin))
    if bias:
        n.register_parameter("bias", _param(cout))
    return n


def _clip_ln(c):
    n = Node()
    n.register_parameter("weight", _param(c))
    n.register_parameter("bias", _param(c))
    return n


def _clip_transformer(width, layers):
    """open_clip.transformer.Transformer: pre-LayerNorm residual attention blocks (nn.MultiheadAttention with a fused
    in_proj, MLP c_fc -> GELU (erf) -> c_proj, 4x wide)."""
    blocks = nn.ModuleList()
    for _ in range(layers):
        attn = Node(out_proj=_clip_linear(width, width))
        attn.register_parameter("in_proj_weight", _param(3 * width, width))
        attn.register_parameter("in_proj_bias", _param(3 * width))
        blocks.append(Node(ln_1=_clip_ln(width), attn=attn, ln_2=_clip_ln(width),
                           mlp=Node(c_fc=_clip_linear(width, 4 * width), c_proj=_clip_linear(4 * width, width))))
    return Node(resblocks=blocks)


def _clip_text_top(model: Node, a) -> None:
    """Text-side top-level tensors of open_clip's CLIP module (the transformer itself is added by the text class)."""
    t = a["text"]
    model.put("token_embedding", Node())
    model.token_embedding.register_parameter("weight", _param(t["vocab"], t["width"]))
    model.register_parameter("positional_embedding", _param(t["ctx"], t["width"]))
    model.put("ln_final", _clip_ln(t["width"]))
    model.register_parameter("text_projection", _param(t["width"], a["embed_dim"]))
    model.register_parameter("logit_scale", _param())
    # causal mask of the text tower (open_clip CLIP.build_attention_mask); non-persistent, as in open_clip
    model.register_buffer("attn_mask", torch.full((t["ctx"], t["ctx"]), float("-inf")).triu_(1), persistent=False)


def clip_tokenize(text, ctx: int = 77) -> torch.Tensor:
    """Token ids [B, ctx] of a list of strings.  Uses open_clip.tokenize when open_clip imports; without it only the
    empty prompt is known (<start_of_text> <end_of_text> then zeros: what image_guided_synthesis feeds the
    unconditional branch and every prompt when text input is off)."""
    if isinstance(text, str):
        text = [text]
    try:
        import open_clip
    except ImportError:
        open_clip = None
    if open_clip is not None:
        return open_clip.tokenize(list(text), context_length=ctx)
    out = torch.zeros(len(text), ctx, dtype=torch.long)
    for i, s in enumerate(text):
        if s != "":
            raise RuntimeError(f"tokenizing {s!r} needs open_clip's BPE tokenizer (open_clip.tokenize), which is not "
                               "installed; without it only the empty prompt \"\" is supported, or pass token ids [B, 77]")
        out[i, 0], out[i, 1] = CLIP_SOT, CLIP_EOT
    return out


def _gaussian_blur_reflect(x: torch.Tensor, sigma, ksize) -> torch.Tensor:
    """Separable Gaussian blur with reflect borders (kornia.filters.gaussian_blur2d)."""
    for axis, (s, k) in enumerate(zip(sigma, ksize)):
        r = torch.arange(k, dtype=torch.float32, device=x.device) - (k - 1) / 2
        w = torch.exp(-r * r / (2.0 * s * s))
        w = (w / w.sum()).to(x.dtype)
        C = x.shape[1]
        if axis == 0:      # along H
            x = torch.nn.functional.pad(x, (0, 0, k // 2, k // 2), mode="reflect")
            x = torch.nn.functional.conv2d(x, w.view(1, 1, k, 1).repeat(C, 1, 1, 1), groups=C)
        else:              # along W
            x = torch.nn.functional.pad(x, (k // 2, k // 2, 0, 0), mode="reflect")
            x = torch.nn.functional.conv2d(x, w.view(1, 1, 1, k).repeat(C, 1, 1, 1), groups=C)
    return x


def clip_preprocess(x: torch.Tensor, size: int = 224, antialias: bool = True) -> torch.Tensor:
    """Reference condition.py:322-330: kornia.geometry.resize(x, (size, size), interpolation="bicubic",
    align_corners=True, antialias) -> (x + 1) / 2 -> CLIP mean / std normalisation; x in [-1, 1], [B, 3, H, W].

    The resize is restated from kornia's published algorithm (kornia is not a dependency here, so it is not checked
    against kornia itself): when an axis is downscaled by `factor` and antialias is on, a Gaussian blur with
    sigma = max((factor - 1) / 2, 0.001) per axis, a kernel of int(max(4 sigma, 3)) taps (made odd) and reflect
    borders on both axes, then bicubic interpolation with align_corners=True."""
    x = x.float()
    H, W = x.shape[-2:]
    if antialias and max(H / size, W / size) > 1:
        sig = (max((H / size - 1.0) / 2.0, 0.001), max((W / size - 1.0) / 2.0, 0.001))
        ks = tuple(k + 1 if k % 2 == 0 else k for k in (int(max(4.0 * s, 3)) for s in sig))
        x = _gaussian_blur_reflect(x, sig, ks)
    x = torch.nn.functional.interpolate(x, size=(size, size), mode="bicubic", align_corners=True)
    x = (x + 1.0) / 2.0
    mean = torch.tensor(CLIP_MEAN, device=x.device).view(1, 3, 1, 1)
    std = torch.tensor(CLIP_STD, device=x.device).view(1, 3, 1, 1)
    return (x - mean) / std


class FrozenOpenCLIPEmbedder(nn.Module):
    """Drop-in for lvdm.modules.encoders.condition.FrozenOpenCLIPEmbedder (same ctor kwargs; state-dict keys those of
    open_clip's CLIP after `del model.visual`, reference condition.py:184-202).  Downloads nothing: the parameters
    are empty until the checkpoint's cond_stage_model.* tensors are loaded.  forward / encode run the text tower on
    the CUDA engine (reference :209-231) and return [B, 77, width] fp32 after ln_final."""

    LAYERS = ["last", "penultimate"]

    def __init__(self, arch="ViT-H-14", version="laion2b_s32b_b79k", device="cuda", max_length=77, freeze=True,
                 layer="last"):
        super().__init__()
        if layer not in self.LAYERS:
            raise NotImplementedError(f"layer must be one of {self.LAYERS}, got {layer!r}")
        a = _clip_arch(arch)
        t = a["text"]
        self.arch, self.version, self.device, self.max_length = arch, version, device, max_length
        self.heads = t["heads"]
        self.layer = layer
        self.layer_idx = 0 if layer == "last" else 1
        self.model = Node()
        _clip_text_top(self.model, a)
        self.model.put("transformer", _clip_transformer(t["width"], t["layers"]))
        self._engine = None
        if freeze:
            self.freeze()

    def freeze(self):
        self.eval()
        for p in self.parameters():
            p.requires_grad = False

    def tokenize(self, text) -> torch.Tensor:
        return clip_tokenize(text, self.model.positional_embedding.shape[0])

    def forward(self, text):
        """text: list of strings (or one string), or token ids [B, 77] -> [B, 77, width] fp32."""
        tokens = text if isinstance(text, torch.Tensor) else self.tokenize(text)
        from . import runtime
        from .cond_engine import ClipTextEngine
        ex = runtime.TEST_EXECUTOR
        return ClipTextEngine.cached(self, "_engine", ex).forward(tokens, executor=ex).clone()

    def encode(self, text):
        return self(text)


class FrozenOpenCLIPImageEmbedderV2(nn.Module):
    """Drop-in for lvdm.modules.encoders.condition.FrozenOpenCLIPImageEmbedderV2 (same ctor kwargs; state-dict keys
    those of open_clip's CLIP after `del model.transformer`, reference condition.py:300-320).  Downloads nothing.
    forward: images [B, 3, H, W] in [-1, 1] -> the vision transformer's [B, 1 + grid^2, width] tokens, fp32, without
    ln_post or proj (reference :337-372), on the CUDA engine."""

    def __init__(self, arch="ViT-H-14", version="laion2b_s32b_b79k", device="cuda", freeze=True, layer="pooled",
                 antialias=True):
        super().__init__()
        if layer != "pooled":
            raise NotImplementedError(f"layer must be 'pooled', got {layer!r}")    # reference condition.py:312-314
        a = _clip_arch(arch)
        v = a["vision"]
        self.arch, self.version, self.device, self.layer, self.antialias = arch, version, device, layer, antialias
        self.heads, self.patch, self.image_size = v["heads"], v["patch"], v["image"]
        grid, w = v["image"] // v["patch"], v["width"]
        self.model = Node()
        _clip_text_top(self.model, a)
        visual = Node(conv1=Node(), ln_pre=_clip_ln(w), transformer=_clip_transformer(w, v["layers"]),
                      ln_post=_clip_ln(w))
        visual.register_parameter("class_embedding", _param(w))
        visual.register_parameter("positional_embedding", _param(grid * grid + 1, w))
        visual.register_parameter("proj", _param(w, a["embed_dim"]))
        visual.conv1.register_parameter("weight", _param(w, 3, v["patch"], v["patch"]))
        self.model.put("visual", visual)
        self.register_buffer("mean", torch.tensor(CLIP_MEAN), persistent=False)
        self.register_buffer("std", torch.tensor(CLIP_STD), persistent=False)
        self._engine = None
        if freeze:
            self.freeze()

    def freeze(self):
        self.eval()
        for p in self.model.parameters():
            p.requires_grad = False

    def preprocess(self, x):
        return clip_preprocess(x, self.image_size, self.antialias)

    def forward(self, image, no_dropout=False):
        from . import runtime
        from .cond_engine import ClipImageEngine
        ex = runtime.TEST_EXECUTOR
        return ClipImageEngine.cached(self, "_engine", ex).forward(self.preprocess(image), executor=ex).clone()

    def encode(self, image):
        return self(image)

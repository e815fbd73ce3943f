"""Static structure of the two networks on the hot path, derived from the reference's YAML params.

`unet_layout` / `decoder_layout` return plain-data descriptions (lists of layer tuples) that drive three things
with ONE source of truth: the parameter holders in `modules.py` (state-dict keys identical to the reference
checkpoint), the CUDA engine's execution plan, and the CPU oracle's walk over the state dict.

Reference: lvdm/modules/networks/openaimodel3d.py:311-546 (UNetModel.__init__),
           lvdm/models/autoencoder_dualref.py:371-487,1121-1176 (Decoder / VideoDecoder).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Tuple


@dataclass
class Layer:
    kind: str            # conv_in | res | st | tt | down | up
    cin: int = 0
    cout: int = 0
    heads: int = 0
    d_head: int = 64
    use_linear: bool = True   # tt only: Linear vs Conv1d(k=1) projections


@dataclass
class UNetLayout:
    in_channels: int
    out_channels: int
    model_channels: int
    time_dim: int
    context_dim: int
    temporal_length: int
    fs_condition: bool
    default_fs: int
    temporal_conv: bool
    image_cross_attention: bool
    # each block: (state-dict prefix, [Layer, ...]); prefix e.g. "input_blocks.3"
    input_blocks: List[Tuple[str, List[Layer]]] = field(default_factory=list)
    init_attn: List[Layer] = field(default_factory=list)
    middle_block: List[Layer] = field(default_factory=list)
    output_blocks: List[Tuple[str, List[Layer]]] = field(default_factory=list)
    skip_channels: List[int] = field(default_factory=list)   # channels pushed by each input block


def _get(p, name, default=None):
    if isinstance(p, dict):
        return p.get(name, default)
    return getattr(p, name, default)


def unet_layout(p) -> UNetLayout:
    mc = _get(p, "model_channels")
    mult = list(_get(p, "channel_mult", (1, 2, 4, 8)))
    nres = _get(p, "num_res_blocks")
    attn_res = set(_get(p, "attention_resolutions"))
    nhc = _get(p, "num_head_channels", -1)
    nheads = _get(p, "num_heads", -1)
    use_linear = bool(_get(p, "use_linear", False))
    t_attn = bool(_get(p, "temporal_attention", True))
    if nhc == -1 and nheads == -1:
        raise ValueError("Either num_heads or num_head_channels has to be set")
    for unsupported in ("use_scale_shift_norm", "resblock_updown", "use_relative_position", "use_causal_attention",
                        "tempspatial_aware"):
        if _get(p, unsupported, False):
            raise NotImplementedError(f"UNetModel option {unsupported}=True is outside the supported hot path")
    if _get(p, "dims", 2) != 2 or not _get(p, "conv_resample", True) or _get(p, "transformer_depth", 1) != 1:
        raise NotImplementedError("only dims=2, conv_resample=True, transformer_depth=1 are supported")

    def heads_for(ch):
        return (ch // nheads, nheads)[::-1] if nhc == -1 else (ch // nhc, nhc)   # (heads, d_head)

    lay = UNetLayout(
        in_channels=_get(p, "in_channels"), out_channels=_get(p, "out_channels"), model_channels=mc,
        time_dim=4 * mc, context_dim=_get(p, "context_dim"), temporal_length=_get(p, "temporal_length"),
        fs_condition=bool(_get(p, "fs_condition", False)), default_fs=_get(p, "default_fs", 4),
        temporal_conv=bool(_get(p, "temporal_conv", False)),
        image_cross_attention=bool(_get(p, "image_cross_attention", False)))

    def attn_layers(ch):
        h, d = heads_for(ch)
        out = [Layer("st", ch, ch, heads=h, d_head=d, use_linear=use_linear)]
        if t_attn:
            out.append(Layer("tt", ch, ch, heads=h, d_head=d, use_linear=use_linear))
        return out

    lay.input_blocks.append(("input_blocks.0", [Layer("conv_in", lay.in_channels, mc)]))
    lay.skip_channels.append(mc)
    if _get(p, "addition_attention", False):
        lay.init_attn = [Layer("tt", mc, mc, heads=8, d_head=nhc, use_linear=False)]
    ch, ds, idx = mc, 1, 1
    for level, m in enumerate(mult):
        for _ in range(nres):
            layers = [Layer("res", ch, m * mc)]
            ch = m * mc
            if ds in attn_res:
                layers += attn_layers(ch)
            lay.input_blocks.append((f"input_blocks.{idx}", layers))
            lay.skip_channels.append(ch)
            idx += 1
        if level != len(mult) - 1:
            lay.input_blocks.append((f"input_blocks.{idx}", [Layer("down", ch, ch)]))
            lay.skip_channels.append(ch)
            idx += 1
            ds *= 2
    lay.middle_block = [Layer("res", ch, ch)] + attn_layers(ch) + [Layer("res", ch, ch)]
    skips = list(lay.skip_channels)
    oidx = 0
    for level, m in list(enumerate(mult))[::-1]:
        for i in range(nres + 1):
            ich = skips.pop()
            layers = [Layer("res", ch + ich, m * mc)]
            ch = m * mc
            if ds in attn_res:
                layers += attn_layers(ch)
            if level and i == nres:
                layers.append(Layer("up", ch, ch))
                ds //= 2
            lay.output_blocks.append((f"output_blocks.{oidx}", layers))
            oidx += 1
    return lay


@dataclass
class DecoderLayout:
    z_channels: int
    ch: int
    out_ch: int
    num_resolutions: int
    num_res_blocks: int
    block_in: int                       # channels at the lowest resolution
    # per level (index = i_level): list of (cin, cout) res blocks, has_upsample, refinement kind
    levels: List[dict] = field(default_factory=list)


def decoder_layout(dd) -> DecoderLayout:
    ch = _get(dd, "ch")
    ch_mult = list(_get(dd, "ch_mult"))
    nres = _get(dd, "num_res_blocks")
    if list(_get(dd, "attn_resolutions", [])):
        raise NotImplementedError("VideoDecoder with attn_resolutions != [] is outside the supported hot path")
    nlev = len(ch_mult)
    block_in = ch * ch_mult[-1]
    lay = DecoderLayout(z_channels=_get(dd, "z_channels"), ch=ch, out_ch=_get(dd, "out_ch"), num_resolutions=nlev,
                        num_res_blocks=nres, block_in=block_in)
    attn_level = [2, 3]   # Decoder default (autoencoder_dualref.py:388)
    levels = [None] * nlev
    cur = block_in
    for i_level in reversed(range(nlev)):
        cout = ch * ch_mult[i_level]
        blocks = []
        for _ in range(nres + 1):
            blocks.append((cur, cout))
            cur = cout
        levels[i_level] = dict(blocks=blocks, upsample=(i_level != 0), channels=cur,
                               refine="fusion" if i_level in attn_level else "combiner")
    lay.levels = levels
    return lay


def plain_decoder_layout(dd) -> DecoderLayout:
    """lvdm/modules/networks/ae_modules.py:478-536 (the per-frame AutoencoderKL Decoder): num_res_blocks + 1
    ResnetBlocks per level, an upsampling conv on every level but 0, no reference-frame refinement.  Only the options
    the reference's configs use are accepted."""
    if list(_get(dd, "attn_resolutions", [])):
        raise NotImplementedError("Decoder with attn_resolutions != [] is outside the supported hot path")
    for flag in ("give_pre_end", "tanh_out", "use_linear_attn"):
        if _get(dd, flag, False):
            raise NotImplementedError(f"Decoder option {flag}=True is outside the supported hot path")
    if _get(dd, "attn_type", "vanilla") != "vanilla":
        raise NotImplementedError(f"Decoder attn_type={_get(dd, 'attn_type')!r} is outside the supported hot path")
    if not _get(dd, "resamp_with_conv", True):
        raise NotImplementedError("Decoder resamp_with_conv=False is outside the supported hot path")
    ch = _get(dd, "ch")
    ch_mult = list(_get(dd, "ch_mult"))
    nres = _get(dd, "num_res_blocks")
    nlev = len(ch_mult)
    block_in = ch * ch_mult[-1]
    lay = DecoderLayout(z_channels=_get(dd, "z_channels"), ch=ch, out_ch=_get(dd, "out_ch"), num_resolutions=nlev,
                        num_res_blocks=nres, block_in=block_in)
    levels = [None] * nlev
    cur = block_in
    for i_level in reversed(range(nlev)):
        cout = ch * ch_mult[i_level]
        blocks = []
        for _ in range(nres + 1):
            blocks.append((cur, cout))
            cur = cout
        levels[i_level] = dict(blocks=blocks, upsample=(i_level != 0), channels=cur)
    lay.levels = levels
    return lay


@dataclass
class EncoderLayout:
    in_channels: int
    ch: int
    z_channels: int
    double_z: bool
    levels: List[dict] = field(default_factory=list)
    block_in: int = 0


def encoder_layout(dd) -> EncoderLayout:
    """lvdm/modules/networks/ae_modules.py:366-430 (Encoder.__init__), attn_resolutions=[] only."""
    ch = _get(dd, "ch")
    ch_mult = list(_get(dd, "ch_mult"))
    nres = _get(dd, "num_res_blocks")
    lay = EncoderLayout(in_channels=_get(dd, "in_channels"), ch=ch, z_channels=_get(dd, "z_channels"),
                        double_z=bool(_get(dd, "double_z", True)))
    in_mult = [1] + ch_mult
    for i_level in range(len(ch_mult)):
        cin = ch * in_mult[i_level]
        cout = ch * ch_mult[i_level]
        blocks = []
        for _ in range(nres):
            blocks.append((cin, cout))
            cin = cout
        lay.levels.append(dict(blocks=blocks, downsample=(i_level != len(ch_mult) - 1), channels=cout))
    lay.block_in = ch * ch_mult[-1]
    return lay

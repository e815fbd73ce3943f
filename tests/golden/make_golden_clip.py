"""Generate tests/golden/clip_tiny.npz and tests/golden/state_dict_manifest_clip.json:
    python tests/golden/make_golden_clip.py

open_clip (which the reference's encoders wrap) cannot run offline, so the golden comes from an independent
implementation of the same architecture: transformers' CLIPTextModel / CLIPVisionModel, constructed from a config (no
download), eager attention, exact GELU, LayerNorm eps 1e-5, fp32 on CPU.  The width-reduced encoders of
tooncrafter_b200.modules are filled with the seeded synthetic weights and those weights are mapped into the HF models
(in_proj split into q / k / v).  Stored: the token ids, the low-resolution source of the two test images (the model
sees its bicubic upsample to 224 x 224), the text output hidden_states[n - 1] through final_layer_norm ("penultimate"
layer), and the rows IMAGE_ROWS (class token and every 8th patch token) of the image output last_hidden_state (no
post_layernorm).

The manifest is the full-size (ViT-H-14) key list of open_clip's CLIP module after the reference's `del model.visual`
(text encoder) or `del model.transformer` (image encoder), restated from open_clip's module structure (open_clip.model
.CLIP, open_clip.transformer.{Transformer, VisionTransformer}); it has not been checked against the public checkpoint.
"""
import json
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path.insert(0, str(ROOT))

from tooncrafter_b200 import modules, synthetic  # noqa: E402

TEXT_TINY = dict(embed_dim=64, text=dict(width=128, heads=2, layers=3, ctx=77, vocab=49408))
VISION_TINY = dict(embed_dim=64, text=dict(width=128, heads=2, layers=3, ctx=77, vocab=49408),
                   vision=dict(width=320, heads=4, layers=2, patch=14, image=224))
SEED = 11


def tiny_text():
    m = modules.FrozenOpenCLIPEmbedder(arch=TEXT_TINY, layer="penultimate", device="cpu")
    synthetic.fill_module_(m, seed=SEED, prefix="cond_stage_model.")
    return m


def tiny_image():
    m = modules.FrozenOpenCLIPImageEmbedderV2(arch=VISION_TINY, device="cpu")
    synthetic.fill_module_(m, seed=SEED, prefix="embedder.")
    return m


def tiny_tokens():
    """Two prompts: the empty prompt and a random one of 9 tokens, each <sot> ... <eot> then zeros."""
    ids = torch.zeros(2, 77, dtype=torch.long)
    ids[0, :2] = torch.tensor([modules.CLIP_SOT, modules.CLIP_EOT])
    body = torch.randint(1, 49400, (9,), generator=synthetic._gen("clip.tokens", 1))
    ids[1, 0], ids[1, 1:10], ids[1, 10] = modules.CLIP_SOT, body, modules.CLIP_EOT
    return ids


def tiny_pixels_lowres():
    """Seeded 56 x 56 source of the test images; fp16-representable, so the fixture stores it exactly as float16."""
    return torch.randn(2, 3, 56, 56, generator=synthetic._gen("clip.pixels", 2)).half().float()


def tiny_pixels():
    """The two 224 x 224 test images: bicubic 4x upsample of tiny_pixels_lowres (values vary inside every patch)."""
    return torch.nn.functional.interpolate(tiny_pixels_lowres(), size=(224, 224), mode="bicubic", align_corners=False)


# token rows of the image output kept in the fixture: the class token and every 8th patch token, the last one included
IMAGE_ROWS = torch.arange(0, 257, 8)


def manifest(a=None):
    """Key -> shape of open_clip's CLIP state dict for the two reference encoders (relative to `model.`)."""
    a = a or modules.CLIP_ARCHS["ViT-H-14"]
    t, v, e = a["text"], a["vision"], a["embed_dim"]

    def blocks(pre, w, n):
        out = {}
        for i in range(n):
            b = f"{pre}transformer.resblocks.{i}."
            out.update({b + "ln_1.weight": [w], b + "ln_1.bias": [w],
                        b + "attn.in_proj_weight": [3 * w, w], b + "attn.in_proj_bias": [3 * w],
                        b + "attn.out_proj.weight": [w, w], b + "attn.out_proj.bias": [w],
                        b + "ln_2.weight": [w], b + "ln_2.bias": [w],
                        b + "mlp.c_fc.weight": [4 * w, w], b + "mlp.c_fc.bias": [4 * w],
                        b + "mlp.c_proj.weight": [w, 4 * w], b + "mlp.c_proj.bias": [w]})
        return out

    top = {"positional_embedding": [t["ctx"], t["width"]], "text_projection": [t["width"], e], "logit_scale": [],
           "token_embedding.weight": [t["vocab"], t["width"]],
           "ln_final.weight": [t["width"]], "ln_final.bias": [t["width"]]}
    grid, w = v["image"] // v["patch"], v["width"]
    visual = {"visual.class_embedding": [w], "visual.positional_embedding": [grid * grid + 1, w],
              "visual.proj": [w, e], "visual.conv1.weight": [w, 3, v["patch"], v["patch"]],
              "visual.ln_pre.weight": [w], "visual.ln_pre.bias": [w],
              "visual.ln_post.weight": [w], "visual.ln_post.bias": [w]}
    visual.update(blocks("visual.", w, v["layers"]))
    text = dict(top)
    text.update(blocks("", t["width"], t["layers"]))
    image = dict(top)
    image.update(visual)
    return {"text": {"model." + k: s for k, s in text.items()}, "image": {"model." + k: s for k, s in image.items()}}


def _hf_layers(sd, pre, n, w):
    out = {}
    for i in range(n):
        a, h = f"{pre}transformer.resblocks.{i}.", f"encoder.layers.{i}."
        qw, kw, vw = sd[a + "attn.in_proj_weight"].chunk(3, 0)
        qb, kb, vb = sd[a + "attn.in_proj_bias"].chunk(3, 0)
        out.update({h + "self_attn.q_proj.weight": qw, h + "self_attn.k_proj.weight": kw, h + "self_attn.v_proj.weight": vw,
                    h + "self_attn.q_proj.bias": qb, h + "self_attn.k_proj.bias": kb, h + "self_attn.v_proj.bias": vb,
                    h + "self_attn.out_proj.weight": sd[a + "attn.out_proj.weight"],
                    h + "self_attn.out_proj.bias": sd[a + "attn.out_proj.bias"],
                    h + "layer_norm1.weight": sd[a + "ln_1.weight"], h + "layer_norm1.bias": sd[a + "ln_1.bias"],
                    h + "layer_norm2.weight": sd[a + "ln_2.weight"], h + "layer_norm2.bias": sd[a + "ln_2.bias"],
                    h + "mlp.fc1.weight": sd[a + "mlp.c_fc.weight"], h + "mlp.fc1.bias": sd[a + "mlp.c_fc.bias"],
                    h + "mlp.fc2.weight": sd[a + "mlp.c_proj.weight"], h + "mlp.fc2.bias": sd[a + "mlp.c_proj.bias"]})
    return out


def _load(hf, sd):
    missing, unexpected = hf.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all(k.endswith("position_ids") for k in missing), missing


def hf_text(m, tokens):
    from transformers import CLIPTextConfig, CLIPTextModel
    t = TEXT_TINY["text"]
    cfg = CLIPTextConfig(vocab_size=t["vocab"], hidden_size=t["width"], intermediate_size=4 * t["width"],
                         num_hidden_layers=t["layers"], num_attention_heads=t["heads"], max_position_embeddings=t["ctx"],
                         hidden_act="gelu", layer_norm_eps=1e-5, attn_implementation="eager")
    hf = CLIPTextModel(cfg).eval()
    sd = {k[len("model."):]: v for k, v in m.state_dict().items()}
    hsd = {"embeddings.token_embedding.weight": sd["token_embedding.weight"],
           "embeddings.position_embedding.weight": sd["positional_embedding"],
           "final_layer_norm.weight": sd["ln_final.weight"], "final_layer_norm.bias": sd["ln_final.bias"]}
    hsd.update(_hf_layers(sd, "", t["layers"], t["width"]))
    _load(hf.text_model, hsd)
    with torch.no_grad():
        o = hf(input_ids=tokens, output_hidden_states=True)
        return hf.text_model.final_layer_norm(o.hidden_states[t["layers"] - 1])


def hf_vision(m, pixels):
    from transformers import CLIPVisionConfig, CLIPVisionModel
    v = VISION_TINY["vision"]
    cfg = CLIPVisionConfig(hidden_size=v["width"], intermediate_size=4 * v["width"], num_hidden_layers=v["layers"],
                           num_attention_heads=v["heads"], image_size=v["image"], patch_size=v["patch"], num_channels=3,
                           hidden_act="gelu", layer_norm_eps=1e-5, attn_implementation="eager")
    hf = CLIPVisionModel(cfg).eval()
    sd = {k[len("model.visual."):]: v for k, v in m.state_dict().items() if k.startswith("model.visual.")}
    hsd = {"embeddings.class_embedding": sd["class_embedding"], "embeddings.patch_embedding.weight": sd["conv1.weight"],
           "embeddings.position_embedding.weight": sd["positional_embedding"],
           "pre_layrnorm.weight": sd["ln_pre.weight"], "pre_layrnorm.bias": sd["ln_pre.bias"],
           "post_layernorm.weight": sd["ln_post.weight"], "post_layernorm.bias": sd["ln_post.bias"]}
    hsd.update(_hf_layers(sd, "", v["layers"], v["width"]))
    _load(hf.vision_model, hsd)
    with torch.no_grad():
        return hf(pixel_values=pixels).last_hidden_state


def main():
    torch.manual_seed(0)
    tokens, pixels = tiny_tokens(), tiny_pixels()
    yt = hf_text(tiny_text(), tokens)
    yi = hf_vision(tiny_image(), pixels)
    np.savez_compressed(HERE / "clip_tiny.npz", tokens=tokens.int().numpy(),
                        pixels_lowres=tiny_pixels_lowres().half().numpy(), image_rows=IMAGE_ROWS.int().numpy(),
                        text=yt.numpy(), image=yi[:, IMAGE_ROWS].numpy())
    (HERE / "state_dict_manifest_clip.json").write_text(json.dumps(manifest(), indent=0, sort_keys=True))
    print("clip golden:", tuple(yt.shape), tuple(yi.shape), float(yt.abs().max()), float(yi.abs().max()))


if __name__ == "__main__":
    main()

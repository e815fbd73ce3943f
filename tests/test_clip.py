"""OpenCLIP conditioning encoders (text tower, image tower): oracle pinned to an independent CLIP implementation,
state-dict keys pinned to the manifest, engine programs checked on the CPU emulator and (gpu) on the H100 kernels,
plus the head-dim-80 and causal forms of tc_attention they use."""
import json
import socket
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from make_golden_clip import (SEED, TEXT_TINY, VISION_TINY, tiny_image, tiny_pixels, tiny_pixels_lowres,  # noqa: E402
                              tiny_text, tiny_tokens)
from oracle import clip_oracle, resampler_oracle  # noqa: E402
from tooncrafter_b200 import modules, synthetic  # noqa: E402

GOLD = HERE / "golden" / "clip_tiny.npz"
EMPTY_IDS = [49406, 49407] + [0] * 75


def _sd(m):
    return {k: v.detach().cpu() for k, v in m.state_dict().items()}


def _emu_tol(y, ref):
    """The Resampler test's bound for fp16 storage between the launches."""
    return (y - ref).abs().max().item() < 3e-3 * ref.abs().max().item() + 4e-3


# ------------------------------------------------------------------------------------------------------------ CPU
def test_oracle_matches_independent_clip_golden():
    gold = np.load(GOLD)
    tokens = torch.from_numpy(gold["tokens"]).long()
    assert torch.equal(tokens, tiny_tokens())
    assert torch.equal(torch.from_numpy(gold["pixels_lowres"]).float(), tiny_pixels_lowres())
    pixels = tiny_pixels()
    rows = torch.from_numpy(gold["image_rows"]).long()
    with torch.no_grad():
        yt = clip_oracle.encode_text(_sd(tiny_text()), tokens, TEXT_TINY["text"]["heads"], layer_idx=1, prefix="model.")
        yi = clip_oracle.encode_image(_sd(tiny_image()), pixels, VISION_TINY["vision"]["heads"], prefix="model.")
    assert (yt - torch.from_numpy(gold["text"])).abs().max().item() < 2e-5
    assert (yi[:, rows] - torch.from_numpy(gold["image"])).abs().max().item() < 2e-5


def test_clip_emulator_attention_matches_ops_emulator():
    """The emulator extension reproduces ops_emulator.attention for head dim 64 without a mask."""
    import clip_emulator
    import ops_emulator
    g = synthetic._gen("clip.emu", 9)
    qkv = torch.randn(2 * 70 * 384, generator=g).half()
    outs = []
    for fn, extra in ((ops_emulator.attention, {}), (clip_emulator.attention, dict(head_dim=64, causal=False))):
        out = torch.zeros(2 * 70 * 128, dtype=torch.float16)
        fn(qkv, [dict(k=qkv, v=qkv, ldk=384, ldv=384, Lk=70, k_offset=128, v_offset=256)], out, q_batches=2, Lq=70,
           heads=2, scale=0.125, ldq=384, ldo=128, **extra)
        outs.append(out)
    assert torch.equal(outs[0], outs[1])


def test_state_dict_keys_match_manifest():
    ref = json.loads((HERE / "golden" / "state_dict_manifest_clip.json").read_text())
    with torch.device("meta"):
        t = modules.FrozenOpenCLIPEmbedder(layer="penultimate")
        i = modules.FrozenOpenCLIPImageEmbedderV2()
    assert {k: list(v.shape) for k, v in t.state_dict().items()} == ref["text"]
    assert {k: list(v.shape) for k, v in i.state_dict().items()} == ref["image"]
    assert "model.attn_mask" not in t.state_dict() and "model.attn_mask" in dict(t.named_buffers())


def test_empty_prompt_tokenizes_natively():
    ids = modules.clip_tokenize(["", ""])
    assert ids.dtype == torch.long and ids.tolist() == [EMPTY_IDS, EMPTY_IDS]


def test_other_prompts_need_the_tokenizer():
    try:
        import open_clip  # noqa: F401
        pytest.skip("open_clip is installed")
    except ImportError:
        pass
    with pytest.raises(RuntimeError, match="open_clip"):
        modules.clip_tokenize(["a cartoon cat"])


def test_unsupported_layers_raise():
    with pytest.raises(NotImplementedError):
        modules.FrozenOpenCLIPEmbedder(arch=TEXT_TINY, layer="pooled")
    with pytest.raises(NotImplementedError):
        modules.FrozenOpenCLIPImageEmbedderV2(arch=VISION_TINY, layer="penultimate")
    with pytest.raises(NotImplementedError):
        modules.FrozenOpenCLIPEmbedder(arch="ViT-bigG-14")


def test_text_engine_program_on_emulator():
    import clip_emulator
    from tooncrafter_b200.cond_engine import ClipTextEngine
    m = tiny_text()
    eng = ClipTextEngine(m, device="cpu", plan_only=True)
    tokens = tiny_tokens()
    y = eng.forward(tokens, executor=clip_emulator.executor)
    assert len(eng.layers) == TEXT_TINY["text"]["layers"] - 1          # "penultimate": the last block is not packed
    with torch.no_grad():
        ref = clip_oracle.encode_text(_sd(m), tokens, TEXT_TINY["text"]["heads"], layer_idx=1, prefix="model.")
    assert _emu_tol(y, ref)


def test_image_engine_program_on_emulator():
    import clip_emulator
    from tooncrafter_b200.cond_engine import ClipImageEngine
    m = tiny_image()
    eng = ClipImageEngine(m, device="cpu", plan_only=True)
    px = tiny_pixels()
    y = eng.forward(px, executor=clip_emulator.executor)
    with torch.no_grad():
        ref = clip_oracle.encode_image(_sd(m), px, VISION_TINY["vision"]["heads"], prefix="model.")
    assert y.shape == (2, 257, VISION_TINY["vision"]["width"])
    assert _emu_tol(y, ref)


def test_public_classes_on_emulator():
    """forward() of the public classes, string prompts and [-1, 1] images, through the test executor hook."""
    import clip_emulator
    from tooncrafter_b200 import runtime
    t, i = tiny_text(), tiny_image()
    img = torch.rand(1, 3, 40, 64, generator=synthetic._gen("clip.img", 3)) * 2 - 1
    runtime.TEST_EXECUTOR = clip_emulator.executor
    try:
        yt = t([""])
        yi = i(img)
    finally:
        runtime.TEST_EXECUTOR = None
    with torch.no_grad():
        rt = clip_oracle.encode_text(_sd(t), torch.tensor([EMPTY_IDS]), TEXT_TINY["text"]["heads"], 1, "model.")
        ri = clip_oracle.encode_image(_sd(i), modules.clip_preprocess(img), VISION_TINY["vision"]["heads"], "model.")
    assert _emu_tol(yt, rt) and _emu_tol(yi, ri)


def test_preprocess_matches_plain_resize_when_upscaling():
    """Upscaling needs no anti-alias blur (sigma 0.001 is a delta kernel): the restatement reduces to bicubic."""
    x = torch.rand(2, 3, 100, 150, generator=synthetic._gen("clip.pre", 4)) * 2 - 1
    ref = F.interpolate(x, size=(224, 224), mode="bicubic", align_corners=True)
    ref = ((ref + 1) / 2 - torch.tensor(modules.CLIP_MEAN).view(1, 3, 1, 1)) / torch.tensor(modules.CLIP_STD).view(1, 3, 1, 1)
    assert (modules.clip_preprocess(x) - ref).abs().max().item() < 1e-5


def test_full_config_instantiates_without_open_clip_or_network(monkeypatch):
    from tiny_config import FULL_DDCONFIG, FULL_UNET, model_config
    from tooncrafter_b200 import diffusion

    def no_network(*a, **k):
        raise AssertionError("network access")
    monkeypatch.setattr(socket.socket, "connect", no_network)
    cfg = model_config(FULL_UNET, FULL_DDCONFIG)
    p = cfg["params"]
    p["cond_stage_config"] = {"target": "tooncrafter_b200.modules.FrozenOpenCLIPEmbedder",
                              "params": {"freeze": True, "layer": "penultimate"}}
    p["img_cond_stage_config"] = {"target": "tooncrafter_b200.modules.FrozenOpenCLIPImageEmbedderV2",
                                  "params": {"freeze": True}}
    p["image_proj_stage_config"] = {"target": "lvdm.modules.encoders.resampler.Resampler",
                                    "params": dict(dim=1024, depth=4, dim_head=64, heads=12, num_queries=16,
                                                   embedding_dim=1280, output_dim=1024, ff_mult=4, video_length=16)}
    with torch.device("meta"):
        m = diffusion.instantiate_from_config(cfg)
    assert "open_clip" not in sys.modules
    ref = json.loads((HERE / "golden" / "state_dict_manifest_clip.json").read_text())
    sd = m.state_dict()
    for pre, key in (("cond_stage_model.", "text"), ("embedder.", "image")):
        ours = {k[len(pre):]: list(v.shape) for k, v in sd.items() if k.startswith(pre)}
        assert ours == ref[key]


def test_engines_refuse_cpu():
    from tooncrafter_b200.cond_engine import ClipImageEngine, ClipTextEngine
    with pytest.raises(RuntimeError):
        ClipTextEngine(tiny_text())
    with pytest.raises(RuntimeError):
        ClipImageEngine(tiny_image())


# ------------------------------------------------------------------------------------------------------------ GPU
def _rand(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).cuda()


def _sdpa_ref(q, k, v, heads, d, causal=False):
    """fp32 attention of fp16 q [B, Lq, h*d], k / v [B, Lk, h*d] -> [B, Lq, h*d]."""
    B, Lq, _ = q.shape
    sp = lambda t: t.float().reshape(B, -1, heads, d).transpose(1, 2)
    o = F.scaled_dot_product_attention(sp(q), sp(k), sp(v), is_causal=causal)
    return o.transpose(1, 2).reshape(B, Lq, heads * d)


def _close(out, ref, what):
    """The bounds of the existing attention tests (tests/test_kernels_gpu.py): max-norm 3e-3 * max|ref| + 1e-3, and at
    most 0.1 % of the outputs outside rtol 1e-3 / atol 1e-4."""
    out, ref = out.float(), ref.float()
    assert torch.isfinite(out).all(), what
    diff = (out - ref).abs()
    err, bound = diff.max().item(), 3e-3 * ref.abs().max().item() + 1e-3
    viol = (diff > 1e-4 + 1e-3 * ref.abs()).float().mean().item()
    print(f"{what}: max err {err:.3e} (bound {bound:.3e}); outside rtol 1e-3/atol 1e-4: {100 * viol:.4f} %")
    assert err <= bound, what
    assert viol <= 1e-3, what


@pytest.fixture(scope="module")
def ops():
    from tooncrafter_b200 import ops as _ops
    torch.backends.cuda.matmul.allow_tf32 = False
    return _ops


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [1, 16])
@pytest.mark.parametrize("L", [1, 64, 65, 77, 257, 600])
def test_attention_head_dim_80_ragged(ops, L, heads):
    B, d = 2, 80
    C = heads * d
    q, k, v = (_rand(B, L, C, seed=s).half() for s in (801, 802, 803))
    out = torch.zeros_like(q)
    ops.attention(q, [dict(k=k, v=v, ldk=C, ldv=C, Lk=L)], out, q_batches=B, Lq=L, heads=heads, scale=d ** -0.5,
                  ldq=C, ldo=C, head_dim=80)
    _close(out, _sdpa_ref(q, k, v, heads, d), f"attention d=80 L={L} heads={heads}")


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [1, 16])
def test_attention_head_dim_80_fused_qkv(ops, heads):
    """q / k / v as channel slices of one [tokens][3C] in_proj output (the vision tower's layout), output written into
    a channel slice of a wider tensor."""
    B, L, d = 2, 257, 80
    C = heads * d
    qkv = _rand(B, L, 3 * C, seed=804).half()
    out = torch.zeros(B, L, 2 * C, dtype=torch.float16, device="cuda")
    ops.attention(qkv, [dict(k=qkv, v=qkv, ldk=3 * C, ldv=3 * C, Lk=L, k_offset=C, v_offset=2 * C)], out,
                  q_batches=B, Lq=L, heads=heads, scale=d ** -0.5, ldq=3 * C, ldo=2 * C, out_offset=C, head_dim=80)
    ref = _sdpa_ref(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], heads, d)
    _close(out[..., C:], ref, f"attention d=80 fused qkv heads={heads}")
    assert out[..., :C].abs().max().item() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("d", [64, 80])
@pytest.mark.parametrize("L", [77, 200])
def test_attention_causal(ops, d, L):
    B, heads = 2, 4
    C = heads * d
    qkv = _rand(B, L, 3 * C, seed=805).half()
    out = torch.zeros(B, L, C, dtype=torch.float16, device="cuda")
    ops.attention(qkv, [dict(k=qkv, v=qkv, ldk=3 * C, ldv=3 * C, Lk=L, k_offset=C, v_offset=2 * C)], out,
                  q_batches=B, Lq=L, heads=heads, scale=d ** -0.5, ldq=3 * C, ldo=C, head_dim=d, causal=True)
    ref = _sdpa_ref(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], heads, d, causal=True)
    _close(out, ref, f"causal attention d={d} L={L}")


@pytest.mark.gpu
def test_attention_rejects_unsupported_forms(ops):
    from tooncrafter_b200._lib import TcError
    q = torch.zeros(1, 64, 96, dtype=torch.float16, device="cuda")
    seg = dict(k=q, v=q, ldk=96, ldv=96, Lk=64)
    with pytest.raises(TcError):
        ops.attention(q, [seg], q, q_batches=1, Lq=64, heads=1, scale=1.0, ldq=96, ldo=96, head_dim=96)
    with pytest.raises(TcError):
        ops.attention(q, [seg, seg], q, q_batches=1, Lq=64, heads=1, scale=1.0, ldq=96, ldo=96, causal=True)


def _check(name, out, ref32, ref16):
    """The yardstick of tests/test_fullsize_gpu.py: at most 3x as far from the fp32 oracle as the oracle under fp16
    autocast (+ 2e-3 of the scale) in max error, 2x (+ 2e-4 of the scale) in rms, and at most 1.5x the autocast
    fraction (+ 2 %) of the elements outside rtol 1e-3 / atol 1e-4."""
    out, ref32, ref16 = out.float().flatten().cpu(), ref32.float().flatten().cpu(), ref16.float().flatten().cpu()
    viol = lambda a: ((a - ref32).abs() > 1e-4 + 1e-3 * ref32.abs()).float().mean().item()
    assert torch.isfinite(out).all(), name + ": non-finite"
    scale = ref32.abs().max().item()
    err, e16 = (out - ref32).abs().max().item(), (ref16 - ref32).abs().max().item()
    rms, rms16 = (out - ref32).pow(2).mean().sqrt().item(), (ref16 - ref32).pow(2).mean().sqrt().item()
    v, v16 = viol(out), viol(ref16)
    print(f"{name}: max err {err:.3e} (autocast {e16:.3e}, scale {scale:.3e}); rms {rms:.3e} (autocast {rms16:.3e}); "
          f"outside rtol 1e-3/atol 1e-4: {100 * v:.2f} % (autocast {100 * v16:.2f} %)")
    assert err <= 3 * e16 + 2e-3 * scale, name
    assert rms <= 2 * rms16 + 2e-4 * scale, name
    assert v <= 1.5 * v16 + 0.02, name


@pytest.mark.gpu
def test_full_size_text_tower_on_gpu():
    """ViT-H-14 text tower, "penultimate": 23 of 24 blocks of width 1024, causal, against the fp32 oracle."""
    torch.manual_seed(0)
    m = modules.FrozenOpenCLIPEmbedder(layer="penultimate")
    synthetic.fill_module_(m, seed=SEED, prefix="cond_stage_model.")
    m = m.cuda()
    tokens = torch.cat([tiny_tokens()[1:], modules.clip_tokenize([""])])
    sd = m.state_dict()
    with torch.no_grad():
        y = m(tokens)
        ref = clip_oracle.encode_text(sd, tokens.cuda(), 16, 1, "model.")
        with torch.autocast("cuda", dtype=torch.float16):
            ref16 = clip_oracle.encode_text(sd, tokens.cuda(), 16, 1, "model.")
    assert y.shape == (2, 77, 1024)
    _check("text tower ViT-H-14", y, ref, ref16)


@pytest.mark.gpu
def test_full_size_image_tower_on_gpu():
    """ViT-H-14 vision tower: 32 blocks of width 1280, 16 heads of 80, 257 tokens, a 320 x 512 frame and its zero
    image, against the fp32 oracle."""
    torch.manual_seed(0)
    m = modules.FrozenOpenCLIPImageEmbedderV2()
    synthetic.fill_module_(m, seed=SEED, prefix="embedder.")
    m = m.cuda()
    img = torch.rand(1, 3, 320, 512, generator=synthetic._gen("clip.full.img", 5)) * 2 - 1
    img = torch.cat([img, torch.zeros_like(img)]).cuda()
    sd = m.state_dict()
    with torch.no_grad():
        y = m(img)
        px = modules.clip_preprocess(img)
        ref = clip_oracle.encode_image(sd, px, 16, "model.")
        with torch.autocast("cuda", dtype=torch.float16):
            ref16 = clip_oracle.encode_image(sd, px, 16, "model.")
    assert y.shape == (2, 257, 1280)
    _check("image tower ViT-H-14", y, ref, ref16)


@pytest.mark.gpu
def test_reference_glue_order_on_tiny_model():
    """image_guided_synthesis's order (reference scripts/evaluation/inference.py:186-214) through the public classes:
    embedder -> image_proj_model -> get_learned_conditioning -> DDIM sample -> decode_first_stage."""
    from tiny_config import TINY_CONTEXT_DIM, TINY_DDCONFIG, TINY_LATENT_HW, TINY_T, model_config
    from tooncrafter_b200 import diffusion
    from tooncrafter_b200.sampler import DDIMSampler

    cfg = model_config()
    p = cfg["params"]
    p["cond_stage_config"] = {"target": "tooncrafter_b200.modules.FrozenOpenCLIPEmbedder",
                              "params": dict(arch=TEXT_TINY, layer="penultimate")}
    p["img_cond_stage_config"] = {"target": "tooncrafter_b200.modules.FrozenOpenCLIPImageEmbedderV2",
                                  "params": dict(arch=VISION_TINY)}
    rs = dict(dim=128, depth=1, dim_head=64, heads=2, num_queries=16, embedding_dim=VISION_TINY["vision"]["width"],
              output_dim=TINY_CONTEXT_DIM, ff_mult=4, video_length=TINY_T)
    p["image_proj_stage_config"] = {"target": "lvdm.modules.encoders.resampler.Resampler", "params": rs}
    m = diffusion.instantiate_from_config(cfg)
    synthetic.fill_module_(m, seed=SEED)
    m = m.cuda().eval()
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    h, w = TINY_LATENT_HW
    g = synthetic._gen("clip.glue", 6)
    frames = [(torch.rand(1, 3, 8 * h, 8 * w, generator=g) * 2 - 1).cuda() for _ in range(2)]
    conds = []
    with torch.no_grad():
        for img in frames:
            img_emb = m.image_proj_model(m.embedder(img))
            cond_emb = m.get_learned_conditioning([""])
            c = torch.cat([cond_emb, img_emb], dim=1)
            # oracle of the same chain
            t_ref = clip_oracle.encode_text(sd, torch.tensor([EMPTY_IDS]).cuda(), TEXT_TINY["text"]["heads"], 1,
                                            "cond_stage_model.model.")
            i_ref = clip_oracle.encode_image(sd, modules.clip_preprocess(img), VISION_TINY["vision"]["heads"],
                                             "embedder.model.")
            r_ref = resampler_oracle.resampler_forward(sd, i_ref, heads=rs["heads"], prefix="image_proj_model.")
            ref = torch.cat([t_ref, r_ref], dim=1)
            assert c.shape == (1, 77 + 16 * TINY_T, TINY_CONTEXT_DIM)
            err = (c - ref).abs().max().item()
            assert err < 2e-2 * ref.abs().max().item() + 1e-2, err
            conds.append(c)
        assert (conds[0] - conds[1]).abs().max().item() > 1e-2, "two different images gave the same conditioning"
        x_T, cond, uncond = synthetic.synthetic_inputs(1, TINY_T, h, w, TINY_CONTEXT_DIM, seed=7)
        cond = {"c_crossattn": [conds[0]], "c_concat": [cond["c_concat"][0].cuda()]}
        uc_img = m.image_proj_model(m.embedder(torch.zeros_like(frames[0])))
        uncond = {"c_crossattn": [torch.cat([m.get_learned_conditioning([""]), uc_img], 1)],
                  "c_concat": cond["c_concat"]}
        samples, _ = DDIMSampler(m).sample(S=2, batch_size=1, shape=[4, TINY_T, h, w], conditioning=cond,
                                           unconditional_conditioning=uncond, eta=1.0, unconditional_guidance_scale=7.5,
                                           x_T=x_T.cuda(), fs=torch.tensor([10], device="cuda"),
                                           timestep_spacing="uniform_trailing", guidance_rescale=0.7, verbose=False)
        ref_ctx = [r.cuda() for r in synthetic.synthetic_ref_context(TINY_DDCONFIG["ch"], TINY_DDCONFIG["ch_mult"],
                                                                     8 * h, 8 * w, seed=7)]
        video = m.decode_first_stage(samples, ref_context=ref_ctx)
    assert torch.isfinite(samples).all() and torch.isfinite(video).all()
    assert video.shape[2] == TINY_T

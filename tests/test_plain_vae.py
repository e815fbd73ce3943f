"""The plain AutoencoderKL first stage (per-frame 2-D Decoder of the DynamiCrafter / training configs) and the
single-image `animate` entry point, on the CPU: parameter holder and checkpoint keys, the plain decode program
interpreted by tests/ops_emulator.py against the unmodified reference (tests/golden/plain_decoder_tiny.npz), launch
arguments of the full-size programs at the 512 and 1024 geometries, and the pipeline / CLI glue."""
import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

import ops_emulator  # noqa: E402
from make_golden_plain_vae import SEED, plain_inputs  # noqa: E402
from test_engine_host_cpu import _check_program  # noqa: E402
from test_pipeline import TINY_SIZE, _scale_close, keyframes, save_path_u8, tiny_config  # noqa: E402
from tiny_config import FULL_DDCONFIG, TINY_DDCONFIG, TINY_LATENT_HW, TINY_T, model_config  # noqa: E402
from tooncrafter_b200 import diffusion, layout, modules, ops, runtime, synthetic, vae_engine  # noqa: E402
from tooncrafter_b200.pipeline import ToonCrafterPipeline  # noqa: E402

GOLD = np.load(HERE / "golden" / "plain_decoder_tiny.npz")
T = TINY_T


def tiny_plain_ae():
    ae = diffusion.AutoencoderKL(ddconfig=TINY_DDCONFIG, embed_dim=4).eval()
    synthetic.fill_module_(ae, seed=SEED, prefix="first_stage_model.")
    return ae


def _close(got, gold, what):
    """The bound of the emulator's dual-ref decoder test: 3e-2 of the output scale + 1e-2 (fp16 storage)."""
    err, scale = (got.float() - gold).abs().max().item(), gold.abs().max().item()
    print(f"{what}: max diff {err:.3e}, scale {scale:.3e}")
    assert err < 3e-2 * scale + 1e-2, what


class _Emulated:
    def __enter__(self):
        runtime.TEST_EXECUTOR = ops_emulator.executor

    def __exit__(self, *exc):
        runtime.TEST_EXECUTOR = None


# ------------------------------------------------------------------------------------------ holder, layout, checkpoint
@pytest.mark.parametrize("option", [dict(attn_resolutions=[32]), dict(give_pre_end=True), dict(tanh_out=True),
                                    dict(use_linear_attn=True), dict(attn_type="none"),
                                    dict(resamp_with_conv=False)])
def test_plain_decoder_refuses_options_outside_the_configs(option):
    with pytest.raises(NotImplementedError, match="outside the supported hot path"):
        diffusion.AutoencoderKL(ddconfig=dict(TINY_DDCONFIG, **option), embed_dim=4)


def test_plain_decoder_layout():
    lay = layout.plain_decoder_layout(FULL_DDCONFIG)
    assert [lv["channels"] for lv in lay.levels] == [128, 256, 512, 512]
    assert [len(lv["blocks"]) for lv in lay.levels] == [3, 3, 3, 3]
    assert [lv["upsample"] for lv in lay.levels] == [False, True, True, True]
    assert lay.levels[3]["blocks"][0] == (512, 512) and lay.levels[0]["blocks"][0] == (256, 128)


@pytest.mark.parametrize("res", [512, 1024])
def test_training_configs_load_a_checkpoint_with_the_reference_first_stage_keys(res):
    """LatentVisualDiffusion from the `model:` section of the reference's configs/training_{res}_v1.0/config.yaml (first
    stage lvdm.models.autoencoder.AutoencoderKL) loads, strictly, a state dict whose first-stage keys and shapes are
    those of the reference's plain AutoencoderKL (tests/golden/state_dict_manifest_plain_vae.json)."""
    from tooncrafter_b200.interpolate import rewrite_targets
    cfg = rewrite_targets(json.loads((HERE / "golden" / f"reference_model_config_training_{res}.json").read_text()))
    assert cfg["params"]["first_stage_config"]["target"] == "lvdm.models.autoencoder.AutoencoderKL"
    manifest = json.loads((HERE / "golden" / "state_dict_manifest_plain_vae.json").read_text())
    with torch.device("meta"):
        m = diffusion.instantiate_from_config(cfg)
    assert type(m.first_stage_model) is diffusion.AutoencoderKL
    assert isinstance(m.first_stage_model.decoder, modules.Decoder)
    own = m.state_dict()
    fs = {k: list(v.shape) for k, v in own.items() if k.startswith("first_stage_model.")}
    assert fs == manifest
    sd = {k: v for k, v in own.items() if not k.startswith("first_stage_model.")}
    sd.update({k: torch.empty(s, device="meta") for k, s in manifest.items()})
    m.load_state_dict(sd, strict=True)
    assert m.image_size == ([40, 64] if res == 512 else [72, 128]) and m.perframe_ae


# ------------------------------------------------------------------------------------------ decode program vs golden
def test_plain_decode_program_on_emulator_matches_reference_golden():
    """AutoencoderKL.decode(z): post_quant_conv + Decoder.forward, interpreted on the CPU, against the reference."""
    ae = tiny_plain_ae()
    with _Emulated():
        y = ae.decode(torch.from_numpy(GOLD["z"]))
    assert y.dtype == torch.float16 and tuple(y.shape) == GOLD["decode"].shape
    _close(y, torch.from_numpy(GOLD["decode"]), "plain decode(z) vs reference")
    with pytest.raises(NotImplementedError, match="no decode kwargs"):
        ae.decode(torch.from_numpy(GOLD["z"]), timesteps=2)


@pytest.mark.parametrize("perframe_ae", [True, False])
def test_decode_first_stage_on_plain_model_applies_post_quant_conv_without_kwargs(perframe_ae):
    """decode_core (ddpm3d.py:647-683) on a 5-frame latent with temporal_length 4: two chunks with perframe_ae (no
    kwargs reach decode, so post_quant_conv runs, autoencoder.py:112-116), one call without; both equal the reference."""
    m = diffusion.instantiate_from_config(synthetic.with_first_stage(model_config(), "plain"))
    synthetic.fill_module_(m, seed=SEED)
    m.eval().perframe_ae = perframe_ae
    calls = []
    orig = m.first_stage_model.decode
    m.first_stage_model.decode = lambda z, **kw: (calls.append((z.shape[0], kw)), orig(z, **kw))[1]
    with _Emulated():
        y = m.decode_first_stage(torch.from_numpy(GOLD["z5"]))
    assert calls == ([(4, {}), (1, {})] if perframe_ae else [(5, {})])
    _close(y, torch.from_numpy(GOLD["decode_first_stage"]), f"decode_first_stage perframe_ae={perframe_ae}")


def test_plain_inputs_are_the_fixture_inputs():
    gi = plain_inputs()
    assert torch.equal(gi["z"], torch.from_numpy(GOLD["z"])) and torch.equal(gi["z5"], torch.from_numpy(GOLD["z5"]))


def test_plain_decoder_programs_plan_at_512_and_1024_with_valid_launch_arguments():
    """The full-width plain decode program for 16 frames at latent 40 x 64 and 72 x 128 (the training_1024 config),
    planned on the meta device: every GEMM / GroupNorm call passes the kernels' documented refusal rules, the mid
    block is one fused tc_attention_wide launch, and the activation arena holds the program."""
    with torch.device("meta"):
        ae = diffusion.AutoencoderKL(ddconfig=FULL_DDCONFIG, embed_dim=4)
    eng = vae_engine.PlainDecoderEngine(ae, device="meta", plan_only=True)
    for (N, h, w) in ((16, 40, 64), (16, 72, 128)):
        plan = eng.plan_for(N, h, w)
        calls = list(plan.main.calls)
        assert _check_program(calls) == {"groupnorm"}
        wide = [kw for fn, a, kw in calls if fn is ops.attention_wide]
        assert len(wide) == 1 and (wide[0]["D"], wide[0]["batches"], wide[0]["L"]) == (512, N, h * w)
        assert (wide[0]["ld"], wide[0]["ldo"]) == (3 * 512, 512)
        ups = [kw for fn, a, kw in calls if fn is ops.upsample2x]
        assert len(ups) == 3 and all(kw["C_"] % 8 == 0 for kw in ups)
        assert not any(fn in (ops.temporal_attention, ops.attention, ops.softmax_rows) for fn, a, kw in calls)
        assert plan.arena.in_use == 0 and plan.arena.high_water <= plan.arena.buf.numel()
        assert tuple(plan.y_out.shape) == (N, 3, 1, 8 * h, 8 * w)
        print(f"plain decoder N={N} latent {h}x{w}: arena {plan.arena.buf.numel() / 2 ** 30:.2f} GiB, "
              f"high water {plan.arena.high_water / 2 ** 30:.2f} GiB, {len(plan.main)} launches")


# ------------------------------------------------------------------------------------------ pipeline and CLI glue
_MODELS = {}


def tiny_model(first_stage):
    """tests/test_pipeline.py's tiny model with the given first stage (cached)."""
    if first_stage not in _MODELS:
        from tooncrafter_b200.interpolate import rewrite_targets
        m = diffusion.instantiate_from_config(rewrite_targets(synthetic.with_first_stage(tiny_config(), first_stage)))
        synthetic.fill_module_(m, seed=SEED)
        m.perframe_ae = True
        _MODELS[first_stage] = m.eval()
    return _MODELS[first_stage]


def _recording(executor, log):
    def run(fn, args, kw):
        log.append((fn, args, kw))
        executor(fn, args, kw)
    return run


def restated_animate(m, image, seed, steps, cfg_scale=7.5):
    """scripts/evaluation/inference.py:180-277 with interp=False, loop=False, restated from the public classes: the
    image as T frames encoded together (frame 0's posterior noise from the seeded CPU generator; the other frames'
    noise is irrelevant, c_concat repeats frame 0's latent), x_T and the step noise from the seeded device generator,
    then the T and T - 2 decodes and the middle-frame splice, returned as float [3, T, H, W]."""
    from tooncrafter_b200.sampler import DDIMSampler
    dev, T = m.device, m.temporal_length
    fr = image.to(dev).permute(2, 0, 1)[None].float().div(255).sub(0.5).div(0.5)
    videos = fr.expand(T, -1, -1, -1)                                            # (b t) c h w
    post, hs = m.first_stage_model.encode(videos, return_hidden_states=True)
    noise = torch.randn(post.mean.shape, generator=torch.Generator().manual_seed(99))
    noise[0] = torch.randn(noise.shape[1:], generator=torch.Generator().manual_seed(seed))
    z = m.get_first_stage_encoding(post, noise=noise)
    z = z.reshape(1, T, *z.shape[1:]).permute(0, 2, 1, 3, 4)
    hs = [hd.reshape(1, T, *hd.shape[1:]).permute(0, 2, 1, 3, 4)[:, :, [0, -1]] for hd in hs]
    img_emb = m.image_proj_model(m.embedder(fr))
    img_cat_cond = z[:, :, :1].repeat(1, 1, T, 1, 1)
    cond = {"c_crossattn": [torch.cat([m.get_learned_conditioning([""]), img_emb], 1)], "c_concat": [img_cat_cond]}
    uc_img_emb = m.image_proj_model(m.embedder(torch.zeros_like(fr)))
    uc = {"c_crossattn": [torch.cat([m.get_learned_conditioning([""]), uc_img_emb], 1)], "c_concat": [img_cat_cond]}
    samples, _ = DDIMSampler(m).sample(S=steps, conditioning=cond, batch_size=1, shape=[4, T, *z.shape[-2:]],
                                       verbose=False, unconditional_guidance_scale=cfg_scale,
                                       unconditional_conditioning=uc, eta=1.0, fs=torch.tensor([10], device=dev),
                                       timestep_spacing="uniform_trailing", guidance_rescale=0.7,
                                       noise_generators=[torch.Generator(device=dev).manual_seed(seed)])
    kw = {} if isinstance(m.first_stage_model.decoder, modules.Decoder) else {"ref_context": hs}
    ref = m.decode_first_stage(samples, **kw)
    index = list(range(T))
    del index[1]
    del index[-2]
    mid = m.decode_first_stage(samples[:, :, index], **kw)
    ref[:, :, T // 2 - 1:T // 2 + 1] = mid[:, :, T // 2 - 2:T // 2]
    return ref[0]


@pytest.mark.parametrize("first_stage", ["plain", "dualref"])
def test_animate_on_emulator_follows_image_guided_synthesis_and_its_rng_contract(first_stage):
    m = tiny_model(first_stage)
    image = keyframes(1, seed=5)[0]
    pipe = ToonCrafterPipeline(m)
    runtime.TEST_EXECUTOR = __import__("clip_emulator").executor
    try:
        u8 = pipe.animate(image, steps=2, seed=77, size=TINY_SIZE)
        vf = pipe.animate(image, steps=2, seed=77, size=TINY_SIZE, output="float")
        again = pipe.animate(image, steps=2, seed=77, size=TINY_SIZE, output="float")
        other = pipe.animate(image, steps=2, seed=78, size=TINY_SIZE, output="float")
        ref = restated_animate(m, image, 77, 2)
    finally:
        runtime.TEST_EXECUTOR = None
    assert u8.shape == (T, *TINY_SIZE, 3) and u8.dtype == torch.uint8
    assert vf.shape == (3, T, *TINY_SIZE) and vf.dtype == torch.float32
    assert torch.equal(u8, save_path_u8(vf))
    assert torch.equal(vf, again), "same seed, different video"
    assert (vf - other).abs().max().item() > 1e-2, "the seed does not reach the video"
    # 3e-2 of the scale: the interpreter stores every activation in fp16, and the two sides encode a different
    # number of frames (1 vs T) and embed the images in different batches, so roundings differ through two DDIM steps
    # and the decoder (measured 1.1e-2); a wrong seed, c_concat or splice is an O(1) difference
    _scale_close(vf, ref, f"animate ({first_stage} first stage) vs restated image_guided_synthesis(interp=False)",
                 rel=3e-2)


def test_interpolate_with_plain_first_stage_decodes_each_segment_once():
    """K = 3 on the plain first stage: one T-frame decode per segment and no T - 2 frame decode (recorded launches),
    and the joined video follows the seam rule of the float output."""
    import clip_emulator
    m = tiny_model("plain")
    kf = keyframes(3, seed=8)
    pipe = ToonCrafterPipeline(m)
    m.first_stage_model._dec_engine = None                # drop plans other tests made on the shared model
    log = []
    runtime.TEST_EXECUTOR = _recording(clip_emulator.executor, log)
    try:
        u8 = pipe.interpolate(kf, steps=2, seed=5, size=TINY_SIZE)
        vf = pipe.interpolate(kf, steps=2, seed=5, size=TINY_SIZE, output="float")
    finally:
        runtime.TEST_EXECUTOR = None
    dec = m.first_stage_model.decoder_engine()
    assert isinstance(dec, vae_engine.PlainDecoderEngine) and list(dec._plans) == [(T, *TINY_LATENT_HW)]
    outs = [a[1] for fn, a, kw in log if fn is ops.cl_to_ncthw and kw["C_"] == 3]
    assert len(outs) == 2 * 2 and all(o.shape[0] == T for o in outs)      # 2 segments x 2 calls, T frames each
    assert not any(fn is ops.ncthw_to_cl and kw["B"] == T - 2 for fn, a, kw in log)
    u8_calls = [kw for fn, a, kw in log if fn is ops.video_u8]
    assert len(u8_calls) == 2
    from test_pipeline import joined_from_segments
    assert u8.shape == (2 * (T - 1) + 1, *TINY_SIZE, 3)
    assert torch.equal(u8, joined_from_segments(vf, loop=False))


def test_cli_animates_one_frame_and_reads_a_training_config(tmp_path):
    import yaml

    from tooncrafter_b200 import interpolate
    cfg = json.loads((HERE / "golden" / "reference_model_config_training_1024.json").read_text())
    path = tmp_path / "training_1024.yaml"
    path.write_text(yaml.safe_dump({"model": cfg, "data": {"target": "utils_data.DataModuleFromConfig"},
                                    "lightning": {"precision": 16}}))
    args = interpolate.get_parser().parse_args(["--config", str(path), "--frames", "still.png", "--out", "o",
                                                "--height", "576", "--width", "1024", "--synthetic-weights"])
    assert args.frames == ["still.png"] and (args.height, args.width) == (576, 1024)
    model_cfg = interpolate.load_model_config(str(path))
    p = model_cfg["params"]
    assert p["first_stage_config"]["target"] == "lvdm.models.autoencoder.AutoencoderKL"
    assert p["cond_stage_config"]["target"] == "tooncrafter_b200.modules.FrozenOpenCLIPEmbedder"
    assert p["image_size"] == [72, 128]
    with torch.device("meta"):
        m = diffusion.instantiate_from_config(model_cfg)
    assert isinstance(m.first_stage_model.decoder, modules.Decoder)


def test_grown_groupnorm_workspace_stays_allocated_for_captured_graphs():
    """A CUDA graph bakes in the GroupNorm workspace's address.  animate (UNet at 2 rows) followed by a K >= 3
    interpolate (4 rows and more) grows the workspace after the plain decoder's graph was captured: the old workspace
    must stay allocated, or the decoder's next replay writes into memory the allocator has handed out again."""
    dev = torch.device("cpu")
    ops._GN_WS.pop(dev, None)
    small = ops._gn_ws(dev, 2 * 32 * 32 * ops.GN_MAX_PARTIALS)          # 32 frames: the 1 Mi-float minimum
    assert ops._gn_ws(dev, 10) is small
    big = ops._gn_ws(dev, 2 * 64 * 32 * ops.GN_MAX_PARTIALS)            # 64 frames: grows
    assert big is not small and big.numel() >= 2 * 64 * 32 * ops.GN_MAX_PARTIALS
    assert any(t is small for t in ops._GN_WS_RETIRED)
    ops._GN_WS.pop(dev)


def test_default_segments_per_batch_keeps_the_unet_budget():
    from tooncrafter_b200.pipeline import default_segments_per_batch
    assert default_segments_per_batch((320, 512)) == 4 and default_segments_per_batch((576, 1024)) == 1

"""Keyframe interpolation pipeline (tooncrafter_b200.pipeline, tooncrafter_b200.interpolate) and its output kernel
tc_video_u8: frame counts, seams and the RNG contract on the CPU program interpreter; the kernel, the pipeline against
the reference glue restated from the public classes, and the command line on the H100."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from make_golden_clip import SEED, TEXT_TINY, VISION_TINY  # noqa: E402
from tiny_config import TINY_CONTEXT_DIM, TINY_LATENT_HW, TINY_T, model_config  # noqa: E402
from tooncrafter_b200 import diffusion, runtime, synthetic  # noqa: E402
from tooncrafter_b200.pipeline import ToonCrafterPipeline, preprocess  # noqa: E402

TINY_SIZE = (8 * TINY_LATENT_HW[0], 8 * TINY_LATENT_HW[1])
T = TINY_T


def tiny_config():
    """tests/tiny_config.py's model with the tiny OpenCLIP towers of test_clip.py and a one-layer Resampler, under the
    reference's target strings."""
    cfg = model_config()
    p = cfg["params"]
    p["cond_stage_config"] = {"target": "lvdm.modules.encoders.condition.FrozenOpenCLIPEmbedder",
                              "params": dict(arch=TEXT_TINY, layer="penultimate")}
    p["img_cond_stage_config"] = {"target": "lvdm.modules.encoders.condition.FrozenOpenCLIPImageEmbedderV2",
                                  "params": dict(arch=VISION_TINY)}
    p["image_proj_stage_config"] = {"target": "lvdm.modules.encoders.resampler.Resampler",
                                    "params": dict(dim=128, depth=1, dim_head=64, heads=2, num_queries=16,
                                                   embedding_dim=VISION_TINY["vision"]["width"],
                                                   output_dim=TINY_CONTEXT_DIM, ff_mult=4, video_length=TINY_T)}
    return cfg


def tiny_model(device="cpu"):
    from tooncrafter_b200.interpolate import rewrite_targets
    m = diffusion.instantiate_from_config(rewrite_targets(tiny_config()))
    synthetic.fill_module_(m, seed=SEED)
    m.perframe_ae = True
    return m.to(device).eval()


def keyframes(K, size=TINY_SIZE, seed=11):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(K, size[0], size[1], 3, generator=g) * 255).to(torch.uint8)


def save_path_u8(video):
    """scripts/evaluation/inference.py:148-153 on one [3, T, H, W] video -> [T, H, W, 3] uint8."""
    v = torch.clamp(video.float(), -1.0, 1.0)
    v = (v + 1.0) / 2.0
    return (v * 255).to(torch.uint8).permute(1, 2, 3, 0)


def joined_from_segments(vf, loop):
    """The seam rule by Python slicing: segment k supplies frames [1 if k else 0, T - 1 if closing loop else T)."""
    S, T = vf.shape[0], vf.shape[2]
    parts = []
    for k in range(S):
        f_end = T - 1 if (loop and k == S - 1) else T
        parts.append(save_path_u8(vf[k].cpu())[(1 if k else 0):f_end])
    return torch.cat(parts)


def _scale_close(a, b, what, rel=1e-2):
    """The bound of test_unet_engine_batch_independence: 1e-2 of the output scale."""
    a, b = a.float().cpu(), b.float().cpu()
    err, scale = (a - b).abs().max().item(), b.abs().max().item()
    print(f"{what}: max diff {err:.3e}, scale {scale:.3e}")
    assert torch.isfinite(a).all() and err <= rel * scale, what


# ------------------------------------------------------------------------------------------------------------ CPU
_RUNS = {}


def _emulated(K, loop=False, output="uint8", seed=123, frames=None, **kw):
    """One pipeline run on the tiny model through the CPU program interpreter (cached per argument set)."""
    import clip_emulator
    key = (K, loop, output, seed, None if frames is None else tuple(frames), tuple(sorted(kw.items())))
    if key not in _RUNS:
        if "model" not in _RUNS:
            _RUNS["model"] = tiny_model()
        kf = keyframes(4 if frames is not None else K)
        kf = kf[list(frames)] if frames is not None else kf
        runtime.TEST_EXECUTOR = clip_emulator.executor
        try:
            _RUNS[key] = ToonCrafterPipeline(_RUNS["model"]).interpolate(kf, steps=2, loop=loop, seed=seed,
                                                                         size=TINY_SIZE, output=output, **kw)
        finally:
            runtime.TEST_EXECUTOR = None
    return _RUNS[key]


@pytest.mark.parametrize("K,loop", [(2, False), (4, False), (2, True), (3, True)])
def test_frame_count_and_seams_on_emulator(K, loop):
    u8 = _emulated(K, loop)
    S = K if loop else K - 1
    assert u8.shape == ((T - 1) * (K if loop else S) + (0 if loop else 1), *TINY_SIZE, 3) and u8.dtype == torch.uint8
    vf = _emulated(K, loop, output="float")
    assert vf.shape == (S, 3, T, *TINY_SIZE) and vf.dtype == torch.float32
    assert torch.equal(u8, joined_from_segments(vf, loop))
    for k in range(1, S):          # the frame a seam shares is the earlier segment's last frame
        assert torch.equal(u8[(T - 1) * k], save_path_u8(vf[k - 1].cpu())[T - 1])


def test_rng_contract_on_emulator():
    """Segment 2 of a K = 4 run with `seed` is the K = 2 run on (keyframe 2, keyframe 3) with seed + 2."""
    four = _emulated(4, output="float")
    pair = _emulated(2, output="float", seed=125, frames=(2, 3))
    _scale_close(four[2], pair[0], "segment 2 of K=4 vs K=2 on its pair (emulator)")
    assert (four[1] - pair[0]).abs().max().item() > 1e-2, "different segments gave the same video"


def test_rng_contract_on_the_general_sampler_path():
    """Without guidance (cfg_scale 1) sample() takes the general path (_ddim_update): per-row draws there too."""
    three = _emulated(3, output="float", cfg_scale=1.0)
    pair = _emulated(2, output="float", seed=124, frames=(1, 2), cfg_scale=1.0)
    _scale_close(three[1], pair[0], "segment 1 of K=3 vs K=2 on its pair, general path (emulator)")


def test_emulator_video_u8_matches_save_path_on_every_finite_half():
    import ops_emulator
    h = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16)
    h = h[torch.isfinite(h)]
    H, W = 16, 88
    n = 16 * 3 * H * W
    x16 = h.repeat(-(-n // h.numel()))[:n].reshape(16, 3, H, W)
    x14 = h.flip(0)[:14 * 3 * H * W].reshape(14, 3, H, W).contiguous()
    spliced = x16.clone()
    spliced[7:9] = x14[6:8]
    for xi, src in ((None, x16), (x14, spliced)):
        for f0, f1 in ((0, 16), (1, 16), (1, 15)):
            out = torch.full((20, H, W, 3), 77, dtype=torch.uint8)
            ops_emulator.video_u8(x16, xi, out, f_begin=f0, f_end=f1, out_frame=3)
            assert torch.equal(out[3:3 + f1 - f0], save_path_u8(src.permute(1, 0, 2, 3))[f0:f1])
            assert (out[:3] == 77).all() and (out[3 + f1 - f0:] == 77).all()


def test_preprocess_matches_torchvision_pil_path():
    """load_data_prompts's PIL transform (inference.py:65-69) on a synthetic 600 x 900 image and its transpose.
    Measured: at most one uint8 level (2/255) apart, on 1.7 % / 1.1 % of the values (bilinear resample of PIL vs
    torchvision's tensor kernel; both round to uint8)."""
    import torchvision.transforms as transforms
    from PIL import Image
    size = (320, 512)
    tf = transforms.Compose([transforms.Resize(min(size)), transforms.CenterCrop(size), transforms.ToTensor(),
                             transforms.Normalize(mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5))])
    for H, W in ((600, 900), (900, 600)):
        yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
        base = torch.stack([torch.sin(7 * xx + 3 * yy), torch.cos(5 * yy - 2 * xx), torch.sin(11 * xx * yy)], -1)
        noise = torch.rand(H, W, 3, generator=torch.Generator().manual_seed(5))
        img = ((base * 0.35 + 0.5 + 0.15 * noise).clamp(0, 1) * 255).round().to(torch.uint8).numpy()
        ref = tf(Image.fromarray(img))
        d = (preprocess([img], size)[0] - ref).abs()
        print(f"{H}x{W}: max diff {d.max().item():.3e}, differing {100 * (d > 1e-6).float().mean().item():.2f} %")
        assert d.max().item() <= 2 / 255 + 1e-6
        assert (d > 1e-6).float().mean().item() <= 0.02


def test_preprocess_passes_matching_sizes_through_exactly():
    kf = keyframes(2, (320, 512))
    x = preprocess(kf, (320, 512))
    assert torch.equal(x, kf.permute(0, 3, 1, 2).float().div(255).sub(0.5).div(0.5))


def test_library_exports_video_u8():
    from tooncrafter_b200 import _lib
    lib = _lib.load()
    assert hasattr(lib, "tc_video_u8")
    assert lib.tc_version() == 102


def test_cli_parses_arguments_loads_yaml_and_rewrites_targets(tmp_path):
    import yaml

    from tooncrafter_b200 import interpolate
    path = tmp_path / "tiny.yaml"
    path.write_text(yaml.safe_dump({"model": tiny_config()}))
    args = interpolate.get_parser().parse_args(["--config", str(path), "--frames", "a.png", "b.png", "c.png",
                                                "--out", "o", "--loop", "--cfg-img", "7.5", "--synthetic-weights"])
    assert args.frames == ["a.png", "b.png", "c.png"] and args.loop and args.cfg_img == 7.5
    assert (args.ddim_steps, args.cfg_scale, args.ddim_eta, args.frame_stride, args.guidance_rescale,
            args.timestep_spacing, args.seed) == (50, 7.5, 1.0, 10, 0.7, "uniform_trailing", 123)
    cfg = interpolate.load_model_config(str(path))
    p = cfg["params"]
    assert p["cond_stage_config"]["target"] == "tooncrafter_b200.modules.FrozenOpenCLIPEmbedder"
    assert p["img_cond_stage_config"]["target"] == "tooncrafter_b200.modules.FrozenOpenCLIPImageEmbedderV2"
    assert p["cond_stage_config"]["params"]["arch"] == TEXT_TINY
    kept = interpolate.load_model_config(str(path), keep_targets=True)
    assert kept["params"]["cond_stage_config"]["target"] == "lvdm.modules.encoders.condition.FrozenOpenCLIPEmbedder"
    with torch.device("meta"):
        m = diffusion.instantiate_from_config(cfg)
    assert type(m.cond_stage_model).__name__ == "FrozenOpenCLIPEmbedder"


def test_cli_reports_checkpoint_key_mismatch(tmp_path):
    from tooncrafter_b200 import interpolate
    m = tiny_model()
    sd = m.state_dict()
    sd.pop("model.diffusion_model.out.2.bias")
    sd["extra.weight"] = torch.zeros(1)
    torch.save({"state_dict": sd}, tmp_path / "bad.ckpt")
    with pytest.raises(RuntimeError, match=r"1 missing keys:\n    model.diffusion_model.out.2.bias"):
        interpolate.load_checkpoint(m, str(tmp_path / "bad.ckpt"))


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def gpu_model():
    torch.backends.cuda.matmul.allow_tf32 = False
    return tiny_model("cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(16, 88), (5, 7)])
def test_video_u8_kernel_is_exact(H, W):
    """Every finite fp16 value (with 16 x 88 pixels; 5 x 7 is the ragged, scalar path), the splice and the frame
    window against the save path by Python slicing, written at an output offset."""
    from tooncrafter_b200 import ops
    h = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16)
    h = h[torch.isfinite(h)]
    n = 16 * 3 * H * W
    x16 = h.repeat(-(-n // h.numel()))[:n].reshape(16, 3, H, W)
    x14 = h.flip(0)[:14 * 3 * H * W].reshape(14, 3, H, W).contiguous()
    spliced = x16.clone()
    spliced[7:9] = x14[6:8]
    covered = 0
    for xi, src in ((None, x16), (x14, spliced)):
        for f0, f1 in ((0, 16), (1, 16), (1, 15), (7, 9)):
            out = torch.full((20, H, W, 3), 77, dtype=torch.uint8, device="cuda")
            ops.video_u8(x16.cuda(), None if xi is None else xi.cuda(), out, f_begin=f0, f_end=f1, out_frame=3)
            ref = save_path_u8(src.permute(1, 0, 2, 3))[f0:f1]
            got = out.cpu()
            assert torch.equal(got[3:3 + f1 - f0], ref), (H, W, xi is None, f0, f1)
            assert (got[:3] == 77).all() and (got[3 + f1 - f0:] == 77).all()
            covered += 1
    assert covered == 8
    assert (H, W) == (5, 7) or x16.numel() >= h.numel()        # 16 x 88: every finite half went through the kernel


@pytest.mark.gpu
def test_video_u8_kernel_refuses_bad_windows():
    from tooncrafter_b200 import _lib, ops
    x = torch.zeros(16, 3, 8, 8, dtype=torch.float16, device="cuda")
    out = torch.zeros(16, 8, 8, 3, dtype=torch.uint8, device="cuda")
    with pytest.raises(_lib.TcError):
        ops.video_u8(x, None, out, f_begin=3, f_end=3, out_frame=0)
    x3 = torch.zeros(3, 3, 8, 8, dtype=torch.float16, device="cuda")
    with pytest.raises(_lib.TcError):
        ops.video_u8(x3, x3[:1].contiguous(), out, f_begin=0, f_end=3, out_frame=0)


@pytest.mark.gpu
def test_pipeline_k2_matches_restated_image_guided_synthesis(gpu_model):
    """inference.py:180-277 restated from the public classes: the pair as T frames (T/2 copies of each keyframe)
    encoded together, rows 0 and T-1 of the posterior noise from the pipeline's keyframe generators, x_T and the step
    noise from its segment generator; then the two decodes and the splice."""
    from tooncrafter_b200.sampler import DDIMSampler
    m, seed, steps = gpu_model, 321, 3
    kf = keyframes(2, seed=21)
    got = ToonCrafterPipeline(m).interpolate(kf, steps=steps, seed=seed, size=TINY_SIZE, output="float")[0]
    with torch.no_grad():
        fr = kf.cuda().permute(0, 3, 1, 2).float().div(255).sub(0.5).div(0.5)
        videos = torch.cat([fr[0:1].expand(T // 2, -1, -1, -1), fr[1:2].expand(T // 2, -1, -1, -1)])   # (b t) c h w
        post, hs = m.first_stage_model.encode(videos, return_hidden_states=True)
        noise = torch.randn(post.mean.shape, generator=torch.Generator().manual_seed(7))
        noise[0] = torch.randn(noise.shape[1:], generator=torch.Generator().manual_seed(seed))
        noise[-1] = torch.randn(noise.shape[1:], generator=torch.Generator().manual_seed(seed + 1))
        z = m.get_first_stage_encoding(post, noise=noise)
        z = z.reshape(1, T, *z.shape[1:]).permute(0, 2, 1, 3, 4)
        hs = [hd.reshape(1, T, *hd.shape[1:]).permute(0, 2, 1, 3, 4)[:, :, [0, -1]] for hd in hs]
        img = videos[0:1]
        img_emb = m.image_proj_model(m.embedder(img))
        cond_emb = m.get_learned_conditioning([""])
        img_cat_cond = torch.zeros_like(z)
        img_cat_cond[:, :, 0], img_cat_cond[:, :, -1] = z[:, :, 0], z[:, :, -1]
        cond = {"c_crossattn": [torch.cat([cond_emb, img_emb], 1)], "c_concat": [img_cat_cond]}
        uc_img_emb = m.image_proj_model(m.embedder(torch.zeros_like(img)))
        uc = {"c_crossattn": [torch.cat([m.get_learned_conditioning([""]), uc_img_emb], 1)], "c_concat": [img_cat_cond]}
        samples, _ = DDIMSampler(m).sample(S=steps, conditioning=cond, batch_size=1, shape=[4, T, *TINY_LATENT_HW],
                                           verbose=False, unconditional_guidance_scale=7.5, unconditional_conditioning=uc,
                                           eta=1.0, fs=torch.tensor([10], device="cuda"),
                                           timestep_spacing="uniform_trailing", guidance_rescale=0.7,
                                           noise_generators=[torch.Generator(device="cuda").manual_seed(seed)])
        ref = m.decode_first_stage(samples, ref_context=hs)
        index = list(range(T))
        del index[1]
        del index[-2]
        mid = m.decode_first_stage(samples[:, :, index], ref_context=hs)
        ref[:, :, T // 2 - 1:T // 2 + 1] = mid[:, :, T // 2 - 2:T // 2]
    _scale_close(got, ref[0], "pipeline K=2 vs restated image_guided_synthesis")


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_img,per_batch", [(None, 4), (5.0, 2)])
def test_pipeline_segments_match_pair_runs(gpu_model, cfg_img, per_batch):
    """K = 4: each segment against a K = 2 run on its pair with seed + k (three-way guidance and two batches of
    segments in the second case)."""
    kf = keyframes(4, seed=31)
    pipe = ToonCrafterPipeline(gpu_model)
    kw = dict(steps=3, size=TINY_SIZE, output="float", cfg_img=cfg_img)
    four = pipe.interpolate(kf, seed=40, segments_per_batch=per_batch, **kw)
    for k in range(3):
        pair = pipe.interpolate(kf[k:k + 2], seed=40 + k, **kw)
        _scale_close(four[k], pair[0], f"cfg_img={cfg_img}: segment {k} of K=4 vs K=2 on its pair")
    assert (four[0] - four[1]).abs().max().item() > 1e-2


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_pipeline_full_size_k3_ddim2():
    """Full-size synthetic weights at 320 x 512, K = 3, DDIM-2: shape, finiteness, and the seams by Python slicing of
    the float output."""
    from tiny_config import FULL_DDCONFIG, FULL_UNET
    from tooncrafter_b200.interpolate import rewrite_targets
    cfg = model_config(FULL_UNET, FULL_DDCONFIG)
    p = cfg["params"]
    p["cond_stage_config"] = {"target": "lvdm.modules.encoders.condition.FrozenOpenCLIPEmbedder",
                              "params": {"freeze": True, "layer": "penultimate"}}
    p["img_cond_stage_config"] = {"target": "lvdm.modules.encoders.condition.FrozenOpenCLIPImageEmbedderV2",
                                  "params": {"freeze": True}}
    p["image_proj_stage_config"] = {"target": "lvdm.modules.encoders.resampler.Resampler",
                                    "params": dict(dim=1024, depth=4, dim_head=64, heads=12, num_queries=16,
                                                   embedding_dim=1280, output_dim=1024, ff_mult=4, video_length=16)}
    m = synthetic.synthetic_model(rewrite_targets(cfg), torch.device("cuda"))
    m.perframe_ae = True
    kf = [keyframes(1, (300, 480), seed=s)[0].numpy() for s in (1, 2, 3)]       # resized + cropped to 320 x 512
    pipe = ToonCrafterPipeline(m)
    u8 = pipe.interpolate(kf, steps=2)
    assert u8.shape == (31, 320, 512, 3) and u8.dtype == torch.uint8 and u8.is_cuda
    vf = pipe.interpolate(kf, steps=2, output="float")
    assert vf.shape == (2, 3, 16, 320, 512) and torch.isfinite(vf).all()
    assert torch.equal(u8.cpu(), joined_from_segments(vf, loop=False))


@pytest.mark.gpu
def test_cli_writes_frames_and_video_npy(tmp_path):
    import yaml
    from PIL import Image

    from tooncrafter_b200 import interpolate
    cfg_path = tmp_path / "tiny.yaml"
    cfg_path.write_text(yaml.safe_dump({"model": tiny_config()}))
    frames = []
    for i, kf in enumerate(keyframes(3, (100, 140), seed=41)):
        frames.append(str(tmp_path / f"kf{i}.png"))
        Image.fromarray(kf.numpy()).save(frames[-1])
    out = tmp_path / "out"
    rc = interpolate.main(["--config", str(cfg_path), "--synthetic-weights", "--frames", *frames, "--out", str(out),
                           "--height", str(TINY_SIZE[0]), "--width", str(TINY_SIZE[1]), "--ddim-steps", "2"])
    assert rc == 0
    v = np.load(out / "video.npy")
    F = 2 * (T - 1) + 1
    assert v.shape == (F, *TINY_SIZE, 3) and v.dtype == np.uint8
    assert sorted(p.name for p in out.glob("frame_*.png")) == [f"frame_{i:04d}.png" for i in range(F)]
    assert np.array_equal(np.asarray(Image.open(out / "frame_0003.png")), v[3])

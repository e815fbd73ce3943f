"""Clips of any even length T from 4 to 64 frames (the reference's --video_length): the oracle and the UNet engine's
shared-context layout against the unmodified reference (tests/golden/make_golden_video_length.py), the recorded
programs, argument checks of the pipeline and the command line; on the H100 the UNet engine, both samplers, the
pipeline with either first stage, and the full-size programs at T = 8, 24 and 64.

Layouts (openaimodel3d.py:556-562): a context of exactly 77 + 16 T tokens gives frame t the image tokens
16 t .. 16 t + 15 (per-frame layout); any other length gives every frame the whole context (shared layout), which is
what the pipeline's 77 + 256 tokens become at T != 16."""
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

import ops_emulator  # noqa: E402
from make_golden import SEED  # noqa: E402
from make_golden_video_length import HW, N_CTX, video_length_inputs  # noqa: E402
from tiny_config import FULL_UNET, TINY_UNET  # noqa: E402

from tooncrafter_b200 import engine, layout, modules, ops, synthetic  # noqa: E402
from tooncrafter_b200.pipeline import ToonCrafterPipeline, check_video_length, default_segments_per_batch  # noqa: E402

GOLD = np.load(HERE / "golden" / "video_length_tiny.npz")
PFX = "model.diffusion_model."


def _tiny_unet(dev="cpu"):
    m = modules.UNetModel(**TINY_UNET)
    synthetic.fill_module_(m, seed=SEED, prefix=PFX)
    return m.to(dev).eval()


def _oracle(m, u, dev="cpu", autocast=False):
    from oracle import unet_oracle
    sd = {PFX + k: v for k, v in m.state_dict().items()}
    with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
        return unet_oracle.unet_forward(sd, layout.unet_layout(TINY_UNET), u["x"].to(dev), u["t"].to(dev),
                                        u["ctx"].to(dev), u["fs"].to(dev), prefix=PFX)


def _cross_attention_segments(plan):
    return [a[1] for fn, a, kw in plan.main.calls if fn is ops.attention and len(a[1]) == 2]


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("T", [8, 24])
def test_oracle_matches_reference_golden(T):
    """The oracle's shared-context branch against the reference UNet at T = 8 and T = 24."""
    y = _oracle(_tiny_unet(), video_length_inputs(T))
    gold = torch.from_numpy(GOLD[f"unet_y_T{T}"])
    assert y.shape == gold.shape
    assert (y - gold).abs().max().item() < 1e-3


@pytest.mark.parametrize("T", [8, 24, 40, 64])
def test_unet_program_interpreted_on_cpu_matches_oracle(T):
    """The engine's shared-context plan on the CPU program interpreter: image K/V rows per sample, shared by its T
    frames (kv_div = T), against the fp32 oracle and, at T = 8 and 24, the reference golden."""
    m = _tiny_unet()
    eng = engine.UNetEngine(m, device="cpu", plan_only=True)
    u = video_length_inputs(T) if T in (8, 24) else dict(video_length_inputs(8), x=torch.randn(
        2, 8, T, *HW, generator=torch.Generator().manual_seed(T)))
    y = eng.forward(u["x"], u["t"], u["ctx"], u["fs"], executor=ops_emulator.executor).float()
    ref = GOLD[f"unet_y_T{T}"] if T in (8, 24) else _oracle(m, u).numpy()
    ref = torch.from_numpy(ref)
    err = (y - ref).abs().max().item()
    assert err < 2e-2 * ref.abs().max().item(), err       # the bound of test_unet_program_interpreted_on_cpu
    plan = eng.plan_for(2, T, *HW, N_CTX)
    assert tuple(plan.ctx_img.shape) == (2 * 256, TINY_UNET["context_dim"])
    segs = _cross_attention_segments(plan)
    assert len(segs) == 16
    for txt, img in segs:
        assert (txt["Lk"], txt["kv_div"], img["Lk"], img["kv_div"]) == (77, T, 256, T)


def test_per_frame_layout_at_t16_keeps_its_program():
    """At T = 16 a 77 + 256-token context keeps the per-frame layout (16 image rows per frame, kv_div 1); the shared
    layout of another context length records the same launches in the same order, only the image K/V differ."""
    m = _tiny_unet()
    eng = engine.UNetEngine(m, device="cpu", plan_only=True)
    per_frame = eng.plan_for(2, 16, *HW, 77 + 16 * 16)
    shared = eng.plan_for(2, 16, *HW, 77 + 64)
    assert tuple(per_frame.ctx_img.shape) == (2 * 16 * 16, TINY_UNET["context_dim"])
    assert tuple(shared.ctx_img.shape) == (2 * 64, TINY_UNET["context_dim"])
    for txt, img in _cross_attention_segments(per_frame):
        assert (txt["Lk"], txt["kv_div"], img["Lk"], img["kv_div"]) == (77, 16, 16, 1)
    for plan_a, plan_b in ((per_frame.main, shared.main), (per_frame.ctx, shared.ctx)):
        assert [fn.__name__ for fn, a, kw in plan_a.calls] == [fn.__name__ for fn, a, kw in plan_b.calls]
    assert len(per_frame.ctx) == 32
    with pytest.raises(NotImplementedError):
        eng.plan_for(2, 8, *HW, 77)


@pytest.mark.parametrize("T", [8, 16, 24, 64])
def test_full_size_programs_plan_with_valid_launch_arguments(T):
    """The full-size UNet programs on the meta device at 320 x 512 with the pipeline's 77 + 256 tokens: the launch count
    of the T = 16 program, and every tc_conv_gemm / attention / norm call within the C ABI's preconditions (temporal
    attention up to T = 64)."""
    from test_engine_host_cpu import _check_conv_gemm_call, _check_norm_attention_call
    with torch.device("meta"):
        unet = modules.UNetModel(**FULL_UNET)
    eng = engine.UNetEngine(unet, device="meta", plan_only=True)
    plan = eng.plan_for(2, T, 40, 64, 77 + 256)
    assert len(plan.main) == 664 and len(plan.ctx) == 32
    seen = set()
    for fn, a, kw in list(plan.ctx.calls) + list(plan.main.calls):
        if fn is ops.conv_gemm:
            _check_conv_gemm_call(a, kw)
        elif fn is ops.temporal_attention:
            assert kw["T"] == T and 0 < T <= 64 and kw["ld"] % 8 == 0 and kw["ldo"] % 8 == 0
            seen.add(fn.__name__)
        elif fn in (ops.groupnorm, ops.attention):
            _check_norm_attention_call(fn, a, kw)
            seen.add(fn.__name__)
    assert seen == {"groupnorm", "attention", "temporal_attention"}
    print(f"T={T}: UNet arena high water {plan.arena.high_water / 2 ** 30:.2f} GiB")


@pytest.mark.parametrize("T", [3, 5, 2, 0, 66, 65, 128, 16.0, True, "16", None])
def test_unsupported_video_lengths_are_refused(T):
    with pytest.raises(ValueError, match="video_length"):
        check_video_length(T)


def test_pipeline_refuses_unsupported_lengths_before_any_work():
    """interpolate and animate check T first: a model object with nothing but temporal_length is enough."""
    pipe = ToonCrafterPipeline(SimpleNamespace(temporal_length=16))
    for T in (7, 66, 2):
        with pytest.raises(ValueError, match="video_length"):
            pipe.interpolate(None, video_length=T)
        with pytest.raises(ValueError, match="video_length"):
            pipe.animate(None, video_length=T)
    assert [check_video_length(T) for T in (4, 8, 16, 24, 64)] == [4, 8, 16, 24, 64]


def test_cli_video_length_argument(capsys):
    from tooncrafter_b200 import interpolate
    base = ["--config", "c.yaml", "--frames", "a.png", "b.png", "--out", "o"]
    assert interpolate.get_parser().parse_args(base).video_length is None
    assert interpolate.get_parser().parse_args(base + ["--video-length", "24"]).video_length == 24
    with pytest.raises(SystemExit):
        interpolate.main(base + ["--synthetic-weights", "--video-length", "15"])
    assert "video_length must be an even integer from 4 to 64" in capsys.readouterr().err


def test_default_segments_per_batch_follows_video_length():
    """The default batch keeps rows x frames x latent pixels at 4 segments of 16 frames at 320 x 512."""
    assert default_segments_per_batch((320, 512)) == default_segments_per_batch((320, 512), 16) == 4
    assert [default_segments_per_batch((320, 512), T) for T in (4, 8, 24, 32, 64)] == [16, 8, 2, 2, 1]
    assert default_segments_per_batch((576, 1024), 8) == 2 and default_segments_per_batch((576, 1024), 64) == 1


# ------------------------------------------------------------------------------------------------------------ GPU
DEV = "cuda"


@pytest.fixture(scope="module")
def gpu_unet():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return _tiny_unet(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [8, 24, 40, 64])
def test_unet_engine_at_video_length(gpu_unet, T):
    """The CUDA program against the fp32 oracle, with the oracle's own autocast error as yardstick (test_engine_gpu's
    bound), and the fp32 oracle against the reference golden at T = 8 and 24."""
    from test_engine_gpu import _report
    u = video_length_inputs(T) if T in (8, 24) else dict(video_length_inputs(8), x=torch.randn(
        2, 8, T, *HW, generator=torch.Generator().manual_seed(T)))
    y = gpu_unet(u["x"].to(DEV), u["t"].to(DEV), context=u["ctx"].to(DEV), fs=u["fs"].to(DEV))
    assert tuple(y.shape) == (2, 4, T, *HW)
    y32, y16 = _oracle(gpu_unet, u, DEV), _oracle(gpu_unet, u, DEV, autocast=True)
    if T in (8, 24):
        assert (y32.cpu() - torch.from_numpy(GOLD[f"unet_y_T{T}"])).abs().max().item() < 1e-3
    _report(f"tiny unet T={T}, 77 + 256 shared tokens", y, y32, y16)


def _pipeline_config(first_stage):
    from test_pipeline import tiny_config
    from tooncrafter_b200.interpolate import rewrite_targets
    return rewrite_targets(synthetic.with_first_stage(tiny_config(), first_stage))


@pytest.fixture(scope="module", params=["dualref", "plain"])
def gpu_model(request):
    from test_pipeline import SEED as PSEED
    from tooncrafter_b200 import diffusion
    torch.backends.cuda.matmul.allow_tf32 = False
    m = diffusion.instantiate_from_config(_pipeline_config(request.param))
    synthetic.fill_module_(m, seed=PSEED)
    m.perframe_ae = True
    return m.to(DEV).eval()


def _conditioning(m, frames, first):
    """Text "" and the first keyframe's image tokens per segment, as the pipeline builds them (inference.py:186-216)."""
    S = len(first)
    img_emb = m.image_proj_model(m.embedder(frames[first]))
    uc_img = m.image_proj_model(m.embedder(torch.zeros_like(frames[:1]))).expand(S, -1, -1)
    txt = m.get_learned_conditioning([""]).expand(S, -1, -1)
    return img_emb, uc_img, txt


@pytest.mark.gpu
@pytest.mark.parametrize("T", [8, 24])
@pytest.mark.parametrize("three_way", [False, True])
def test_fused_sampler_matches_per_branch_path(gpu_model, T, three_way):
    """The fused DDIM path (guidance branches as the batch rows of one UNet program) against the per-branch path
    (_fast_path_ok False), same per-row generators, at T != 16 with the shared-context layout."""
    from test_pipeline import _scale_close
    from tooncrafter_b200.sampler import DDIMSampler, DDIMSamplerMultiCond
    m = gpu_model
    h, w = 16, 16
    g = torch.Generator().manual_seed(T)
    S = 2
    ctx = lambda: torch.randn(S, N_CTX, TINY_UNET["context_dim"], generator=g).to(DEV)       # noqa: E731
    cc = [torch.randn(S, 4, T, h, w, generator=g).to(DEV)]
    cond, uc = {"c_crossattn": [ctx()], "c_concat": cc}, {"c_crossattn": [ctx()], "c_concat": cc}
    base = DDIMSamplerMultiCond if three_way else DDIMSampler
    extra = dict(cfg_img=4.0, unconditional_conditioning_img_nonetext={"c_crossattn": [ctx()], "c_concat": cc}) \
        if three_way else {}

    class PerBranch(base):
        def _fast_path_ok(self, *a, **k):
            return False

    out = []
    for cls in (base, PerBranch):
        gens = [torch.Generator(device=DEV).manual_seed(50 + k) for k in range(S)]
        x, _ = cls(m).sample(S=3, conditioning=cond, batch_size=S, shape=[4, T, h, w], verbose=False,
                             unconditional_guidance_scale=7.5, unconditional_conditioning=uc, eta=1.0,
                             fs=torch.tensor([10] * S, device=DEV), timestep_spacing="uniform_trailing",
                             guidance_rescale=0.7, noise_generators=gens, **extra)
        out.append(x)
    keys = list(m.model.diffusion_model._engine._plans.keys())
    assert ((3 if three_way else 2) * S, T, h, w, N_CTX) in keys, keys
    # the per-branch programs run B = 2 rows, the fused one 4 or 6: tiles and split-K slices differ, and three free DDIM
    # steps amplify the fp16 roundings that flip; test_latency_gpu.py bounds the same B = 1 / B = 2 difference by 3 %
    _scale_close(out[0], out[1], f"T={T} {'three' if three_way else 'two'}-way: fused vs per-branch", rel=3e-2)


def _composed(m, kf, T, seed, steps, loop=False, interp=True):
    """The pipeline restated from DDIMSampler.sample and model.decode_first_stage (decode_core's chunks): keyframe j's
    posterior noise seeded seed + j, segment k's generator seed + k, the T and T - 2 decodes, the middle-frame splice
    (inference.py:262-270).  Returns float [S, 3, T, H, W]."""
    from test_pipeline import TINY_SIZE
    from tooncrafter_b200.pipeline import preprocess
    from tooncrafter_b200.sampler import DDIMSampler
    K = kf.shape[0]
    S = (K if loop else K - 1) if interp else 1
    first = list(range(S))
    last = [(k + 1) % K for k in range(S)] if interp else [0]
    frames = preprocess(kf, TINY_SIZE, DEV)
    post, hidden = m.first_stage_model.encode(frames, return_hidden_states=True)
    noise = torch.stack([torch.randn(tuple(post.mean.shape[1:]), generator=torch.Generator().manual_seed(seed + j))
                         for j in range(K)])
    z = m.get_first_stage_encoding(post, noise=noise)
    h, w = z.shape[-2:]
    if interp:
        c_concat = torch.zeros(S, 4, T, h, w, device=DEV)
        c_concat[:, :, 0], c_concat[:, :, -1] = z[first], z[last]
    else:
        c_concat = z[first][:, :, None].expand(-1, -1, T, -1, -1).contiguous()
    img_emb, uc_img, txt = _conditioning(m, frames, first)
    cond = {"c_crossattn": [torch.cat([txt, img_emb], 1)], "c_concat": [c_concat]}
    uc = {"c_crossattn": [torch.cat([txt, uc_img], 1)], "c_concat": [c_concat]}
    samples, _ = DDIMSampler(m).sample(S=steps, conditioning=cond, batch_size=S, shape=[4, T, h, w], verbose=False,
                                       unconditional_guidance_scale=7.5, unconditional_conditioning=uc, eta=1.0,
                                       fs=torch.tensor([10] * S, device=DEV), timestep_spacing="uniform_trailing",
                                       guidance_rescale=0.7,
                                       noise_generators=[torch.Generator(device=DEV).manual_seed(seed + k)
                                                         for k in range(S)])
    dual = isinstance(m.first_stage_model.decoder, modules.VideoDecoder)
    out = []
    index = [t for t in range(T) if t not in (1, T - 2)]
    for k in range(S):
        kw = dict(ref_context=[torch.stack([hd[first[k]], hd[last[k]]], 1).unsqueeze(0) for hd in hidden]) if dual else {}
        y = m.decode_first_stage(samples[k:k + 1], **kw)
        mid = m.decode_first_stage(samples[k:k + 1, :, index], **kw)
        y[:, :, T // 2 - 1:T // 2 + 1] = mid[:, :, T // 2 - 2:T // 2]
        out.append(y[0].float())
    return torch.stack(out)


@pytest.mark.gpu
@pytest.mark.parametrize("T,loop", [(8, False), (8, True), (24, False), (24, True)])
def test_interpolate_at_video_length_matches_composed_reference(gpu_model, T, loop):
    """K = 3 at T frames per segment: frame count, the uint8 video as the seam rule and save path of the float output,
    and the float output against the composition of the public classes.  The tiny model's temporal_length is 4, so
    every decode runs in chunks of 4 frames."""
    from test_pipeline import TINY_SIZE, _scale_close, joined_from_segments, keyframes
    m = gpu_model
    assert m.temporal_length == 4 and m.en_and_decode_n_samples_a_time is None
    kf = keyframes(3, seed=61)
    pipe = ToonCrafterPipeline(m)
    kw = dict(steps=3, seed=70, size=TINY_SIZE, loop=loop, video_length=T)
    u8 = pipe.interpolate(kf, **kw)
    S = 3 if loop else 2
    assert u8.shape == ((T - 1) * S + (0 if loop else 1), *TINY_SIZE, 3) and u8.dtype == torch.uint8
    vf = pipe.interpolate(kf, output="float", **kw)
    assert vf.shape == (S, 3, T, *TINY_SIZE)
    assert torch.equal(u8.cpu(), joined_from_segments(vf, loop))
    ref = _composed(m, kf, T, 70, 3, loop=loop)
    _scale_close(vf, ref, f"interpolate K=3 T={T} loop={loop} vs composed DDIMSampler + decode_first_stage")


@pytest.mark.gpu
def test_animate_at_video_length_matches_composed_reference(gpu_model):
    from test_pipeline import TINY_SIZE, _scale_close, keyframes, save_path_u8
    m = gpu_model
    T = 24
    kf = keyframes(1, seed=62)
    pipe = ToonCrafterPipeline(m)
    u8 = pipe.animate(kf[0], steps=3, seed=80, size=TINY_SIZE, video_length=T)
    vf = pipe.animate(kf[0], steps=3, seed=80, size=TINY_SIZE, video_length=T, output="float")
    assert u8.shape == (T, *TINY_SIZE, 3) and vf.shape == (3, T, *TINY_SIZE)
    assert torch.equal(u8.cpu(), save_path_u8(vf.cpu()))
    _scale_close(vf, _composed(m, kf, T, 80, 3, interp=False)[0], "animate T=24 vs composed reference")
    with pytest.raises(ValueError, match="video_length"):
        pipe.animate(kf[0], steps=3, size=TINY_SIZE, video_length=66)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_full_size_unet_at_video_lengths():
    """320 x 512 (40 x 64 latent), B = 2 (a conditional and an unconditional row), 77 + 256 tokens: the programs at
    T = 8, 24 and 64 build and give finite outputs; the peak device memory of each is printed."""
    with torch.device("meta"):
        skeleton = modules.UNetModel(**FULL_UNET)
    m = skeleton.to_empty(device=DEV)
    with torch.no_grad():
        for k, p in m.named_parameters():
            p.copy_(synthetic.synthetic_tensor(PFX + k, tuple(p.shape), SEED).to(DEV))
    m.eval()
    g = torch.Generator().manual_seed(12)
    ctx = torch.randn(2, 77 + 256, 1024, generator=g).to(DEV)
    for T in (8, 24, 64):
        m._engine = None                                       # this length's plan only
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        x = torch.randn(2, 8, T, 40, 64, generator=g).to(DEV)
        y = m(x, torch.tensor([901, 901], device=DEV), context=ctx, fs=torch.tensor([10, 10], device=DEV))
        torch.cuda.synchronize()
        assert tuple(y.shape) == (2, 4, T, 40, 64) and torch.isfinite(y).all()
        print(f"full-size UNet B=2 T={T}: max_memory_allocated {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")

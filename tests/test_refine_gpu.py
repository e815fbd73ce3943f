"""Refining a clip on the H100: tc_q_sample against torch's fp32 arithmetic bit for bit, decode and the masked sampler
on the fused path against the per-branch path, and ToonCrafterPipeline.refine's equalities with the CUDA library, on
the tiny model and with full-size synthetic weights at 320 x 512."""
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from test_pipeline import _scale_close, keyframes  # noqa: E402

DEV = torch.device("cuda")
FUSED_BOUND = 3e-2        # test_video_length.py's fused vs per-branch bound (batch tiling amplified by free DDIM steps)


@pytest.fixture(scope="module")
def cuda_tf32_off():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


@pytest.mark.gpu
@pytest.mark.parametrize("B,n", [(1, 1001), (3, 40961), (3, 7)])
@pytest.mark.parametrize("mask_kind", [None, "binary", "fractional"])
@pytest.mark.parametrize("clean", [False, True])
def test_q_sample_is_torch_fp32_bit_for_bit(B, n, mask_kind, clean):
    from tooncrafter_b200 import ops
    g = torch.Generator().manual_seed(B * 7 + n)
    r = lambda: torch.randn(B, n, generator=g).to(DEV)           # noqa: E731
    x, x0, noise = r(), r(), r()
    coef = torch.rand(2 * B, generator=g).to(DEV)
    mask = None
    if mask_kind == "binary":
        mask = (torch.rand(B, n, generator=g) < 0.5).float().to(DEV)
    elif mask_kind == "fractional":
        mask = torch.rand(B, n, generator=g).to(DEV)
    a, c = coef.view(B, 2)[:, :1], coef.view(B, 2)[:, 1:]
    q = x0 if clean else a * x0 + c * noise
    want = q if mask is None else q * mask + (1.0 - mask) * x
    got = x.clone()
    ptr = got.data_ptr()
    ops.q_sample(got, x0, None if clean else noise, mask, None if clean else coef, B=B, n=n, clean=clean)
    torch.cuda.synchronize()
    assert got.data_ptr() == ptr
    assert torch.equal(got, want), (got - want).abs().max().item()


@pytest.mark.gpu
def test_stochastic_encode_kernel_is_the_torch_formula(cuda_tf32_off):
    """DDIMSampler.stochastic_encode on CUDA fp32 (tc_q_sample) against ddim.py:309-318's torch expression over the
    sampler's own tables, per-row DDIM indices and DDPM timesteps."""
    from test_n_samples import model
    from tooncrafter_b200.sampler import DDIMSampler
    s = DDIMSampler(model("dualref", "cuda"))
    s.make_schedule(50, "uniform_trailing", 1.0, verbose=False)
    g = torch.Generator().manual_seed(3)
    x0, noise = torch.randn(3, 4, 8, 16, 16, generator=g).to(DEV), torch.randn(3, 4, 8, 16, 16, generator=g).to(DEV)
    for t, orig in ((torch.tensor([0, 24, 49]), False), (torch.tensor([0, 500, 999]), True)):
        t = t.to(DEV)
        sa, s1 = ((s.sqrt_alphas_cumprod, s.sqrt_one_minus_alphas_cumprod) if orig
                  else (torch.sqrt(s.ddim_alphas), s.ddim_sqrt_one_minus_alphas))
        want = sa.gather(-1, t).view(3, 1, 1, 1, 1) * x0 + s1.gather(-1, t).view(3, 1, 1, 1, 1) * noise
        got = s.stochastic_encode(x0, t, use_original_steps=orig, noise=noise)
        assert torch.equal(got, want), (orig, (got - want).abs().max().item())


def _fused_vs_general(m, dim, h, w, T, three_way, steps=3):
    """decode (two-way), t_start and masked sample (with and without clean_cond) on the fused path against the
    per-branch path, the same per-row generators; dim: the UNet's context width."""
    from tooncrafter_b200.sampler import DDIMSampler, DDIMSamplerMultiCond
    n_ctx = 77 + 256
    g = torch.Generator().manual_seed(T + h)
    ctx = lambda: torch.randn(2, n_ctx, dim, generator=g).to(DEV)                  # noqa: E731
    cc = [torch.randn(2, 4, T, h, w, generator=g).to(DEV)]
    cond, uc = {"c_crossattn": [ctx()], "c_concat": cc}, {"c_crossattn": [ctx()], "c_concat": cc}
    base = DDIMSamplerMultiCond if three_way else DDIMSampler
    extra = dict(cfg_img=4.0, unconditional_conditioning_img_nonetext={"c_crossattn": [ctx()], "c_concat": cc}) \
        if three_way else {}
    x0 = torch.randn(2, 4, T, h, w, generator=g).to(DEV)
    x_T = torch.randn(2, 4, T, h, w, generator=g).to(DEV)
    mask = torch.zeros(1, 1, T, 1, 1, device=DEV)
    mask[:, :, [0, 1, T - 1]] = 1.0

    class PerBranch(base):
        def _fast_path_ok(self, *a, **k):
            return False

    runs = {"masked": dict(mask=mask, x0=x0), "masked_clean": dict(mask=mask, x0=x0, clean_cond=True),
            "t_start": dict(t_start=2)}
    for name, kw in runs.items():
        out = []
        for cls in (base, PerBranch):
            gens = [torch.Generator(device=DEV).manual_seed(70 + k) for k in range(2)]
            x, _ = cls(m).sample(S=steps, conditioning=cond, batch_size=2, shape=[4, T, h, w], verbose=False,
                                 unconditional_guidance_scale=7.5, unconditional_conditioning=uc, eta=1.0,
                                 fs=torch.tensor([10, 10], device=DEV), timestep_spacing="uniform_trailing",
                                 guidance_rescale=0.7, noise_generators=gens, x_T=x_T, **kw, **extra)
            out.append(x)
        _scale_close(out[0], out[1], f"{name} {h}x{w} T={T} three_way={three_way}: fused vs per-branch",
                     rel=FUSED_BOUND)
    if not three_way:
        out = []
        for cls in (base, PerBranch):
            s = cls(m)
            s.make_schedule(steps, "uniform_trailing", 1.0, verbose=False)
            torch.manual_seed(5)
            z = s.stochastic_encode(x0, torch.tensor([1, 1], device=DEV))
            out.append(s.decode(z, cond, 2, unconditional_guidance_scale=7.5, unconditional_conditioning=uc))
        _scale_close(out[0], out[1], f"decode {h}x{w}: fused vs per-branch", rel=FUSED_BOUND)


@pytest.mark.gpu
@pytest.mark.parametrize("three_way", [False, True])
def test_decode_and_masked_sample_fused_vs_per_branch_tiny(cuda_tf32_off, three_way):
    from test_n_samples import model
    from tiny_config import TINY_UNET
    _fused_vs_general(model("dualref", "cuda"), TINY_UNET["context_dim"], 16, 16, 8, three_way)


@pytest.fixture(scope="module")
def full_models():
    sys.path.insert(0, str(HERE.parent / "scripts"))
    from bench_pipeline import full_pipeline_config
    from tooncrafter_b200 import synthetic
    cache = {}

    def get(first_stage):
        if first_stage not in cache:
            cache.clear()
            torch.cuda.empty_cache()
            m = synthetic.synthetic_model(full_pipeline_config(), DEV, first_stage=first_stage)
            m.perframe_ae = True
            cache[first_stage] = m
        return cache[first_stage]
    return get


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_decode_and_masked_sample_fused_vs_per_branch_full_width(cuda_tf32_off, full_models):
    from tiny_config import FULL_UNET
    _fused_vs_general(full_models("dualref"), FULL_UNET["context_dim"], 40, 64, 16, False, steps=2)


@pytest.mark.gpu
@pytest.mark.parametrize("first_stage", ["dualref", "plain"])
def test_refine_equalities_on_gpu_tiny(cuda_tf32_off, first_stage):
    from test_n_samples import model
    from test_refine import Emulated, check_refine_is_interpolate, check_variants_and_keep
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    p = Emulated(ToonCrafterPipeline(model(first_stage, "cuda")), "cuda")
    check_refine_is_interpolate(p, steps=3)
    check_refine_is_interpolate(p, steps=3, T_=12)
    check_variants_and_keep(p, steps=4)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("first_stage", ["dualref", "plain"])
def test_refine_full_size(cuda_tf32_off, full_models, first_stage):
    """320 x 512, full-size synthetic weights, T = 16: refine(clip, 1.0) is interpolate bit for bit; a keep run at
    strength 0.5 has the right shape; variant 0 of n_samples=2 is the single-sample result."""
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    p = ToonCrafterPipeline(full_models(first_stage))
    size, T = (320, 512), 16
    clip = keyframes(T, size=size, seed=81)
    a = p.refine(clip, 1.0, steps=3, seed=9, size=size)
    b = p.interpolate(clip[[0, T - 1]], steps=3, seed=9, size=size, video_length=T)
    assert a.shape == (T, *size, 3) and torch.equal(a, b)
    keep = p.refine(clip, 0.5, keep=[0, 1, T - 2, T - 1], steps=4, seed=9, size=size)
    assert keep.shape == (T, *size, 3) and keep.dtype == torch.uint8
    one = p.refine(clip, 0.5, steps=4, seed=9, size=size)
    two = p.refine(clip, 0.5, steps=4, seed=9, size=size, n_samples=2, segments_per_batch=1)
    assert two.shape == (2, T, *size, 3) and torch.equal(two[0], one) and not torch.equal(two[1], one)
    assert not torch.equal(keep, one)


def _worker(rank, world, one_gpu):
    from test_pipeline_distributed_gpu import _init
    dist, dev = _init(rank, world, one_gpu)
    try:
        from test_pipeline import TINY_SIZE, tiny_model
        from tooncrafter_b200.pipeline import ToonCrafterPipeline
        m = tiny_model(dev)
        clip = keyframes(8, seed=91)
        kw = dict(steps=4, seed=61, size=TINY_SIZE, n_samples=3, keep=[0, 7], segments_per_batch=1)
        got = ToonCrafterPipeline(m, dist.group.WORLD).refine(clip, 0.75, **kw)
        got_f = ToonCrafterPipeline(m, dist.group.WORLD).refine(clip, 0.75, output="float", **kw)
        lat = ToonCrafterPipeline(m, dist.group.WORLD, latency=True).refine(clip, 0.75, output="float", **kw)
        single = ToonCrafterPipeline(m)
        ref, ref_f = single.refine(clip, 0.75, **kw), single.refine(clip, 0.75, output="float", **kw)
        return dict(equal=bool(torch.equal(got, ref)), equal_float=bool(torch.equal(got_f, ref_f)),
                    latency_err=float((lat - ref_f).abs().max()), scale=float(ref_f.abs().max()),
                    latency_sum=float(lat.double().sum()))
    finally:
        dist.destroy_process_group()


@pytest.mark.gpu
def test_refine_two_ranks_on_one_gpu_equal_single_process():
    """n_samples=3 with keep over two gloo ranks (rows [0, 1] / [2]): bit for bit; latency mode within its bound and
    the same on both ranks."""
    from distributed_harness import LATENCY_BOUND
    from test_pipeline_distributed_gpu import _spawn
    res = _spawn(_worker, True, 900)
    for r in range(2):
        assert res[r]["equal"] and res[r]["equal_float"], res[r]
        assert res[r]["latency_err"] <= LATENCY_BOUND * res[r]["scale"], res[r]
    assert res[0]["latency_sum"] == res[1]["latency_sum"]

"""End-to-end parity of the CUDA engines (through the C ABI) against the oracle and the reference goldens.

Tolerance: the product path computes in fp16 with fp32 accumulation, like the reference under
torch.cuda.amp.autocast (scripts/evaluation/inference.py:323).  The yardstick is therefore the reference
algorithm's OWN fp16-autocast error: the oracle is evaluated twice on the GPU (fp32, and under autocast fp16),
and the engine must be as close to the fp32 result as the autocast evaluation is, up to a factor 3
(plus 2e-3 of the output scale).  Goldens from the unmodified reference pin the fp32 oracle itself.
"""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

pytestmark = pytest.mark.gpu

from tiny_config import (FULL_UNET, TINY_CONTEXT_DIM, TINY_DDCONFIG, TINY_LATENT_HW, TINY_T, TINY_UNET)  # noqa: E402
from make_golden import SEED, golden_inputs  # noqa: E402

DEV = "cuda"
GOLD = np.load(HERE / "golden" / "tiny_reference_outputs.npz")


def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _report(name, out, ref32, ref16=None):
    out, ref32 = out.float().cpu(), ref32.float().cpu()
    scale = ref32.abs().max().item()
    err = (out - ref32).abs().max().item()
    msg = f"{name}: engine-vs-fp32 max err {err:.3e} (scale {scale:.3e})"
    bound = 2e-3 * scale
    if ref16 is not None:
        e16 = (ref16.float().cpu() - ref32).abs().max().item()
        msg += f", autocast-vs-fp32 {e16:.3e}"
        bound += 3 * e16
    print(msg)
    assert torch.isfinite(out).all(), name + ": non-finite"
    assert err <= bound, msg + f" > bound {bound:.3e}"


@pytest.fixture(scope="module")
def tiny_unet():
    from tooncrafter_b200 import modules, synthetic
    m = modules.UNetModel(**TINY_UNET)
    synthetic.fill_module_(m, seed=SEED, prefix="model.diffusion_model.")
    return m.to(DEV).eval()


def test_unet_engine_matches_reference_golden_and_oracle(tiny_unet):
    from oracle import unet_oracle
    from tooncrafter_b200 import layout
    _no_tf32()
    gi = golden_inputs()["unet"]
    x, t, ctx, fs = gi["x"].to(DEV), gi["t"].to(DEV), gi["ctx"].to(DEV), gi["fs"].to(DEV)
    y = tiny_unet(x, t, context=ctx, fs=fs)
    assert y.dtype == torch.float16 and tuple(y.shape) == (2, 4, TINY_T, *TINY_LATENT_HW)
    sd = {"model.diffusion_model." + k: v for k, v in tiny_unet.state_dict().items()}
    lay = layout.unet_layout(TINY_UNET)
    y32 = unet_oracle.unet_forward(sd, lay, x, t, ctx, fs, prefix="model.diffusion_model.")
    with torch.autocast("cuda", dtype=torch.float16):
        y16 = unet_oracle.unet_forward(sd, lay, x, t, ctx, fs, prefix="model.diffusion_model.")
    # the GPU fp32 oracle agrees with the unmodified reference (CPU golden)
    assert (y32.cpu() - torch.from_numpy(GOLD["unet_y"])).abs().max().item() < 1e-3
    _report("tiny unet", y, torch.from_numpy(GOLD["unet_y"]), y16)
    # replay (CUDA graph) gives the same answer, and a new timestep / context is picked up
    y_again = tiny_unet(x, t, context=ctx, fs=fs).clone()
    assert torch.equal(y_again, y)
    t2 = torch.tensor([100, 900], device=DEV)
    ctx2 = ctx.flip(0).contiguous()
    y2 = tiny_unet(x, t2, context=ctx2, fs=fs)
    y2_32 = unet_oracle.unet_forward(sd, lay, x, t2, ctx2, fs, prefix="model.diffusion_model.")
    with torch.autocast("cuda", dtype=torch.float16):
        y2_16 = unet_oracle.unet_forward(sd, lay, x, t2, ctx2, fs, prefix="model.diffusion_model.")
    _report("tiny unet (new t, ctx)", y2, y2_32, y2_16)


def test_unet_engine_batch_independence(tiny_unet):
    """B=2 batched CFG evaluation == two B=1 evaluations (the reference makes two B=1 calls, ddim.py:221-222)."""
    gi = golden_inputs()["unet"]
    x, t, ctx, fs = gi["x"].to(DEV), gi["t"].to(DEV), gi["ctx"].to(DEV), gi["fs"].to(DEV)
    y = tiny_unet(x, t, context=ctx, fs=fs).clone()
    for b in range(2):
        yb = tiny_unet(x[b:b + 1], t[b:b + 1], context=ctx[b:b + 1].contiguous(), fs=fs[b:b + 1])
        # different M tiling / accumulation order -> fp16 rounding noise only (a real cross-sample coupling is O(1))
        assert (yb[0].float() - y[b].float()).abs().max().item() <= 1e-2 * y.float().abs().max().item()


@pytest.mark.timeout(1200)
def test_unet_engine_full_size_one_forward():
    """inference_512_v1.0 UNet (1.44 G params), B=1, T=16, latent 40x64: engine vs the fp32 oracle on the GPU."""
    from oracle import unet_oracle
    from tooncrafter_b200 import layout, modules, synthetic
    _no_tf32()
    with torch.device("meta"):
        skeleton = modules.UNetModel(**FULL_UNET)
    m = skeleton.to_empty(device=DEV)
    with torch.no_grad():
        for k, p in m.named_parameters():
            p.copy_(synthetic.synthetic_tensor("model.diffusion_model." + k, tuple(p.shape), SEED).to(DEV))
    m.eval()
    g = torch.Generator().manual_seed(11)
    x = torch.randn(1, 8, 16, 40, 64, generator=g).to(DEV)
    ctx = torch.randn(1, 77 + 256, 1024, generator=g).to(DEV)
    t = torch.tensor([601], device=DEV)
    fs = torch.tensor([10], device=DEV)
    y = m(x, t, context=ctx, fs=fs)
    sd = {"model.diffusion_model." + k: v for k, v in m.state_dict().items()}
    lay = layout.unet_layout(FULL_UNET)
    y32 = unet_oracle.unet_forward(sd, lay, x, t, ctx, fs, prefix="model.diffusion_model.")
    with torch.autocast("cuda", dtype=torch.float16):
        y16 = unet_oracle.unet_forward(sd, lay, x, t, ctx, fs, prefix="model.diffusion_model.")
    _report("full-size unet", y, y32, y16)


# ------------------------------------------------------------------------------------------------ VAE
@pytest.fixture(scope="module")
def tiny_ae():
    from tooncrafter_b200 import diffusion, synthetic
    ae = diffusion.AutoencoderKL_Dualref(ddconfig=TINY_DDCONFIG, embed_dim=4)
    synthetic.fill_module_(ae, seed=SEED, prefix="first_stage_model.")
    return ae.to(DEV).eval()


def test_vae_encoder_and_decoder_engines_match_reference_golden(tiny_ae):
    from oracle import vae_oracle
    from tooncrafter_b200 import layout
    _no_tf32()
    gi = golden_inputs()
    frames = gi["frames"].to(DEV)
    post, hidden = tiny_ae.encode(frames, return_hidden_states=True)
    sd = {"first_stage_model." + k: v for k, v in tiny_ae.state_dict().items()}
    qw, qb = sd["first_stage_model.quant_conv.weight"], sd["first_stage_model.quant_conv.bias"]
    h32, hid32 = vae_oracle.encode_hidden(sd, layout.encoder_layout(TINY_DDCONFIG), frames)
    with torch.autocast("cuda", dtype=torch.float16):
        h16, hid16 = vae_oracle.encode_hidden(sd, layout.encoder_layout(TINY_DDCONFIG), frames)
        m16 = torch.nn.functional.conv2d(h16, qw, qb)
    m32 = torch.nn.functional.conv2d(h32, qw, qb)
    assert (m32.cpu() - torch.from_numpy(GOLD["enc_moments"])).abs().max().item() < 1e-3
    _report("encoder moments", post.parameters, torch.from_numpy(GOLD["enc_moments"]), m16)
    for i, h in enumerate(hidden):
        assert (hid32[i].flatten()[::97].cpu() - torch.from_numpy(GOLD[f"enc_hidden{i}_sub"])).abs().max() < 1e-3
        _report(f"encoder hidden {i}", h, hid32[i], hid16[i])
    # decoder: reference frames' hidden states from the fp32 oracle so the two engines are checked independently
    ref_ctx = [h.reshape(1, 2, *h.shape[1:]).permute(0, 2, 1, 3, 4).contiguous() for h in hid32]
    z = gi["z"].to(DEV)
    zz = (z.permute(0, 2, 1, 3, 4).reshape(TINY_T, 4, *TINY_LATENT_HW) / 0.18215).contiguous()
    y = tiny_ae.decode(zz, ref_context=ref_ctx, timesteps=TINY_T)
    dlay = layout.decoder_layout(TINY_DDCONFIG)
    y32 = vae_oracle.decode(sd, dlay, zz, ref_ctx)
    with torch.autocast("cuda", dtype=torch.float16):
        y16 = vae_oracle.decode(sd, dlay, zz, ref_ctx)
    gold = torch.from_numpy(GOLD["decode"])[0].permute(1, 0, 2, 3)
    assert (y32.cpu() - gold).abs().max().item() < 2e-3
    _report("decoder", y, gold, y16)
    # a 3-frame chunk (the reference decodes T=14 in its second pass: any T must work)
    y3 = tiny_ae.decode(zz[:3].contiguous(), ref_context=ref_ctx, timesteps=3)
    y3_32 = vae_oracle.decode(sd, dlay, zz[:3], ref_ctx)
    with torch.autocast("cuda", dtype=torch.float16):
        y3_16 = vae_oracle.decode(sd, dlay, zz[:3], ref_ctx)
    _report("decoder T=3", y3, y3_32, y3_16)


# ------------------------------------------------------------------------------------------------ sampler
def _tiny_model():
    from tiny_config import model_config
    from tooncrafter_b200 import diffusion, synthetic
    cfg = model_config()
    m = diffusion.instantiate_from_config(cfg)
    synthetic.fill_module_(m, seed=SEED)
    m.perframe_ae = True
    return m.to(DEV).eval()


def test_ddim_sampler_fused_path_matches_reference_golden():
    """DDIMSampler.sample() (reference API) on the fused H100 path vs the reference's own 4-step sample."""
    from oracle import ddim_oracle, unet_oracle
    from tooncrafter_b200 import layout
    from tooncrafter_b200.sampler import DDIMSampler
    _no_tf32()
    m = _tiny_model()
    gi = golden_inputs()
    to = lambda c: {k: [t.to(DEV) for t in v] for k, v in c.items()}
    cond, uncond = to(gi["cond"]), to(gi["uncond"])
    x_T = gi["x_T"].to(DEV)
    noises = [n.to(DEV) for n in gi["noises"]]
    # teacher-forced noise: make torch.randn return the golden draws, exactly like make_golden.py did for the reference
    it = iter(noises)
    import tooncrafter_b200.sampler as smod
    real_randn = torch.randn
    smod.torch.randn = lambda *a, **k: next(it)
    try:
        s = DDIMSampler(m)
        samples, inter = s.sample(S=gi["S"], batch_size=1, shape=list(x_T.shape[1:]), conditioning=cond,
                                  unconditional_conditioning=uncond, eta=1.0, unconditional_guidance_scale=7.5,
                                  x_T=x_T, fs=gi["fs"].to(DEV), timestep_spacing="uniform_trailing",
                                  guidance_rescale=0.7, verbose=False)
    finally:
        smod.torch.randn = real_randn
    # yardstick: the oracle's sampler on the GPU in fp32 and under autocast
    sd = {k: v for k, v in m.state_dict().items()}
    ulay = layout.unet_layout(TINY_UNET)

    def apply_model(x, t, c, fs):
        xc = torch.cat([x] + c["c_concat"], dim=1)
        return unet_oracle.unet_forward(sd, ulay, xc, t, torch.cat(c["c_crossattn"], 1), fs, "model.diffusion_model.")

    sched = {k: v.to(DEV) for k, v in ddim_oracle.model_schedule().items()}
    sched_cpu = ddim_oracle.model_schedule()
    x32, _ = ddim_oracle.sample(apply_model, sched_cpu, x_T, cond, uncond, gi["S"], noises=noises, fs=gi["fs"].to(DEV))

    def apply_model16(x, t, c, fs):
        with torch.autocast("cuda", dtype=torch.float16):
            return apply_model(x, t, c, fs)

    x16, _ = ddim_oracle.sample(apply_model16, sched_cpu, x_T, cond, uncond, gi["S"], noises=noises, fs=gi["fs"].to(DEV))
    gold = torch.from_numpy(GOLD["ddim_samples"])
    assert (x32.cpu() - gold).abs().max().item() < 5e-3
    _report("ddim 4-step sample", samples, gold, x16)
    assert len(inter["x_inter"]) >= 2


def test_general_sampler_path_and_decode_first_stage():
    """Non-fused option combination (no CFG) runs through apply_model; decode_first_stage through the decoder."""
    from tooncrafter_b200.sampler import DDIMSampler
    m = _tiny_model()
    gi = golden_inputs()
    to = lambda c: {k: [t.to(DEV) for t in v] for k, v in c.items()}
    s = DDIMSampler(m)
    torch.manual_seed(3)
    samples, _ = s.sample(S=2, batch_size=1, shape=list(gi["x_T"].shape[1:]), conditioning=to(gi["cond"]), eta=0.0,
                          x_T=gi["x_T"].to(DEV), fs=gi["fs"].to(DEV), timestep_spacing="uniform_trailing",
                          verbose=False)
    assert torch.isfinite(samples).all() and tuple(samples.shape) == tuple(gi["x_T"].shape)
    frames = gi["frames"].to(DEV)
    post, hidden = m.first_stage_model.encode(frames, return_hidden_states=True)
    z0 = m.get_first_stage_encoding(post)
    assert tuple(z0.shape) == (2, 4, *TINY_LATENT_HW)
    ref_ctx = [h.reshape(1, 2, *h.shape[1:]).permute(0, 2, 1, 3, 4).contiguous() for h in hidden]
    m.temporal_length = TINY_T
    img = m.decode_first_stage(samples, ref_context=ref_ctx)
    assert tuple(img.shape) == (1, 3, TINY_T, 8 * TINY_LATENT_HW[0], 8 * TINY_LATENT_HW[1])
    assert torch.isfinite(img).all()


def test_multicond_sampler_fused_path_matches_reference_golden():
    """DDIMSampler_multicond (ddim_multiplecond.py:214-234) on the fused H100 path — the three guidance branches as ONE
    B = 3 UNet program per step + tc_ddim_step3 — vs the reference's own 4-step sample (golden) with the autocast oracle
    as yardstick, and vs the general three-pass path on the same GPU."""
    from make_golden_multicond import CFG_IMG, multicond_inputs
    from oracle import ddim_oracle, unet_oracle
    from tooncrafter_b200 import layout
    from tooncrafter_b200.sampler import DDIMSamplerMultiCond
    import tooncrafter_b200.sampler as smod
    _no_tf32()
    m = _tiny_model()
    gi = multicond_inputs()
    to = lambda c: {k: [t.to(DEV) for t in v] for k, v in c.items()}
    cond, uncond, uimg = to(gi["cond"]), to(gi["uncond"]), to(gi["uncond_img"])
    x_T, fs = gi["x_T"].to(DEV), gi["fs"].to(DEV)
    noises = [n.to(DEV) for n in gi["noises"]]
    real_randn = torch.randn

    def run(sampler):
        it = iter(noises)
        smod.torch.randn = lambda *a, **k: next(it)
        try:
            out, _ = sampler.sample(S=gi["S"], batch_size=1, shape=list(x_T.shape[1:]), conditioning=cond,
                                    unconditional_conditioning=uncond, eta=1.0, unconditional_guidance_scale=7.5,
                                    cfg_img=CFG_IMG, x_T=x_T, fs=fs, timestep_spacing="uniform_trailing",
                                    guidance_rescale=0.7, verbose=False, unconditional_conditioning_img_nonetext=uimg)
        finally:
            smod.torch.randn = real_randn
        return out

    s = DDIMSamplerMultiCond(m)
    fused = run(s)
    plan_keys = list(m.model.diffusion_model._engine._plans.keys())
    assert any(k[0] == 3 for k in plan_keys), f"the fused multi-cond path must batch the 3 branches (plans: {plan_keys})"

    class General(DDIMSamplerMultiCond):
        def _fast_path_ok(self, *a, **k):
            return False
    general = run(General(m))

    # yardstick: the reference algorithm (oracle) under autocast with the three-way combine
    sd = {k: v for k, v in m.state_dict().items()}
    ulay = layout.unet_layout(TINY_UNET)
    sched = ddim_oracle.model_schedule()
    tab = ddim_oracle.ddim_tables(sched, gi["S"], 1.0)

    def oracle_sample(autocast):
        x = x_T
        for i, step in enumerate(np.flip(tab["timesteps"])):
            index = gi["S"] - i - 1
            ts = torch.full((1,), int(step), dtype=torch.long, device=DEV)
            es = []
            for c in (cond, uncond, uimg):
                xc = torch.cat([x] + c["c_concat"], 1)
                with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
                    es.append(unet_oracle.unet_forward(sd, ulay, xc, ts, torch.cat(c["c_crossattn"], 1), fs,
                                                       "model.diffusion_model."))
            e_c, e_uc, e_img = es
            v = e_uc + CFG_IMG * (e_img - e_uc) + 7.5 * (e_c - e_img)
            v = ddim_oracle.rescale_noise_cfg(v, e_c, 0.7).float()
            co = ddim_oracle.step_coefficients(sched, tab, index)
            eps = co["sqrt_ac"] * v + co["sqrt_1mac"] * x
            x0 = (co["sqrt_ac"] * x - co["sqrt_1mac"] * v) * co["rescale"]
            x = co["sqrt_aprev"] * x0 + co["dir_coef"] * eps + co["sigma"] * noises[i]
        return x

    x32, x16 = oracle_sample(False), oracle_sample(True)
    gold = torch.from_numpy(np.load(HERE / "golden" / "multicond_tiny.npz")["ddim_samples"])
    assert (x32.cpu() - gold).abs().max().item() < 5e-3, "fp32 oracle disagrees with the reference's multi-cond sample"
    _report("multi-cond 4-step sample (fused, B = 3 program)", fused, gold, x16)
    _report("multi-cond 4-step sample (general path)", general, gold, x16)

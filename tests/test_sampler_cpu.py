"""CPU tests of the sampler's general path (host logic): schedule tables, CFG / rescale / v-parameterisation update
and the 3-way multi-cond guidance, driven by a cheap stand-in denoiser, against the oracle's restatement of
lvdm/models/samplers/ddim.py (pinned to the reference by tests/golden)."""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from tiny_config import TINY_T, model_config  # noqa: E402

from oracle import ddim_oracle  # noqa: E402
from tooncrafter_b200 import diffusion  # noqa: E402
from tooncrafter_b200.sampler import DDIMSampler, DDIMSamplerMultiCond  # noqa: E402


def _model():
    with torch.device("meta"):
        m = diffusion.instantiate_from_config(model_config())
    m = m.to_empty(device="cpu")
    m.reset_schedule_buffers()
    return m


def _denoiser(x, t, c, fs=None, **kw):
    """Stand-in for the UNet: deterministic, depends on x, t and the conditioning."""
    ctx = torch.cat(c["c_crossattn"], 1).mean() if isinstance(c, dict) else c.mean()
    return 0.3 * x + 0.05 * ctx + 1e-3 * t.float().view(-1, 1, 1, 1, 1) * torch.tanh(x)


def test_general_path_matches_oracle_sampler():
    m = _model()
    m.apply_model = lambda x, t, c, **kw: _denoiser(x, t, c, **kw)
    g = torch.Generator().manual_seed(0)
    x_T = torch.randn(1, 4, TINY_T, 8, 8, generator=g)
    cond = {"c_crossattn": [torch.randn(1, 77, 16, generator=g)], "c_concat": [torch.zeros_like(x_T)]}
    uc = {"c_crossattn": [torch.randn(1, 77, 16, generator=g)], "c_concat": [torch.zeros_like(x_T)]}
    S = 5
    noises = [torch.randn(x_T.shape, generator=g) for _ in range(S)]
    it = iter(noises)
    import tooncrafter_b200.sampler as smod
    real = torch.randn
    smod.torch.randn = lambda *a, **k: next(it)
    try:
        out, inter = DDIMSampler(m).sample(S=S, batch_size=1, shape=list(x_T.shape[1:]), conditioning=cond,
                                           unconditional_conditioning=uc, eta=1.0, unconditional_guidance_scale=7.5,
                                           x_T=x_T, timestep_spacing="uniform_trailing", guidance_rescale=0.7,
                                           verbose=False)
    finally:
        smod.torch.randn = real
    ref, _ = ddim_oracle.sample(lambda x, t, c, fs: _denoiser(x, t, c), ddim_oracle.model_schedule(), x_T, cond, uc, S,
                                noises=noises)
    assert (out - ref).abs().max().item() < 1e-4
    assert len(inter["x_inter"]) == 2 + 1 or len(inter["x_inter"]) >= 2


def test_fused_step_coefficients_match_oracle_tables():
    m = _model()
    s = DDIMSampler(m)
    sched = ddim_oracle.model_schedule()
    for S in (10, 50):
        s.make_schedule(S, "uniform_trailing", 1.0, verbose=False)
        tab = ddim_oracle.ddim_tables(sched, S, 1.0)
        for index in (0, S // 2, S - 1):
            co = ddim_oracle.step_coefficients(sched, tab, index)
            got = s.step_coefficients(index, 7.5, 0.7)
            want = [7.5, 0.7, co["sqrt_ac"], co["sqrt_1mac"], co["rescale"], co["sqrt_aprev"], co["dir_coef"], co["sigma"]]
            assert np.allclose(got, want, rtol=0, atol=0), (S, index, got, want)


def test_multicond_guidance_formula():
    m = _model()
    calls = []

    def apply_model(x, t, c, **kw):
        calls.append(c["tag"])
        return {"c": 1.0, "uc": 0.25, "img": 0.5}[c["tag"]] * torch.ones_like(x)

    m.apply_model = apply_model
    s = DDIMSamplerMultiCond(m)
    s.make_schedule(10, "uniform_trailing", 0.0, verbose=False)
    x = torch.zeros(1, 4, TINY_T, 4, 4)
    t = torch.full((1,), int(s.ddim_timesteps[3]), dtype=torch.long)
    captured = {}
    orig = s._ddim_update
    s._ddim_update = lambda x_, t_, index, mo, *a: (captured.setdefault("v", mo), orig(x_, t_, index, mo, *a))[1]
    s.p_sample_ddim(x, {"tag": "c"}, t, index=3, unconditional_guidance_scale=7.5,
                    unconditional_conditioning={"tag": "uc"}, cfg_img=2.0,
                    unconditional_conditioning_img_nonetext={"tag": "img"})
    # e_uc + cfg_img (e_img - e_uc) + s (e_c - e_img)   (ddim_multiplecond.py:229-234)
    assert calls == ["c", "uc", "img"]
    assert torch.allclose(captured["v"], torch.full_like(x, 0.25 + 2.0 * (0.5 - 0.25) + 7.5 * (1.0 - 0.5)))


def test_fused_path_on_the_emulator_matches_reference_golden():
    """The fused sampler path (cond+uncond batched through the UNet program, context set once, device coefficient table,
    fused DDIM update) with the recorded programs interpreted on CPU, against the REFERENCE's own 4-step sample."""
    import numpy as np
    import ops_emulator
    from make_golden import SEED, golden_inputs
    from tooncrafter_b200 import synthetic
    from tooncrafter_b200.engine import UNetEngine
    m = diffusion.instantiate_from_config(model_config())
    synthetic.fill_module_(m, seed=SEED)
    m = m.eval()
    unet = m.model.diffusion_model
    unet._engine = UNetEngine(unet, device="cpu", plan_only=True)
    gi = golden_inputs()
    it = iter(gi["noises"])
    import tooncrafter_b200.sampler as smod
    real = torch.randn
    smod.torch.randn = lambda *a, **k: next(it)
    try:
        s = DDIMSampler(m)
        s._test_executor = ops_emulator.executor
        out, inter = s.sample(S=gi["S"], batch_size=1, shape=list(gi["x_T"].shape[1:]), conditioning=gi["cond"],
                              unconditional_conditioning=gi["uncond"], eta=1.0, unconditional_guidance_scale=7.5,
                              x_T=gi["x_T"], fs=gi["fs"], timestep_spacing="uniform_trailing", guidance_rescale=0.7,
                              verbose=False)
    finally:
        smod.torch.randn = real
    gold = torch.from_numpy(np.load(HERE / "golden" / "tiny_reference_outputs.npz")["ddim_samples"])
    err = (out - gold).abs().max().item()
    assert err < 3e-2 * gold.abs().max().item(), err      # fp16 activations in the interpreted UNet, 4 steps
    assert len(inter["x_inter"]) >= 2 and out.dtype == torch.float32


def test_fused_multicond_path_on_the_emulator_matches_reference_golden():
    """DDIMSampler_multicond on the fused path — one B = 3 UNet program per step + tc_ddim_step3 — with the
    recorded programs interpreted on CPU, against the reference's own 4-step three-way-guidance sample
    (tests/golden/make_golden_multicond.py), and against the general (three-pass) path."""
    import numpy as np
    import ops_emulator
    from make_golden import SEED
    from make_golden_multicond import CFG_IMG, multicond_inputs
    from tooncrafter_b200 import synthetic
    from tooncrafter_b200.engine import UNetEngine
    m = diffusion.instantiate_from_config(model_config())
    synthetic.fill_module_(m, seed=SEED)
    m = m.eval()
    unet = m.model.diffusion_model
    unet._engine = UNetEngine(unet, device="cpu", plan_only=True)
    gi = multicond_inputs()
    import tooncrafter_b200.sampler as smod
    real = torch.randn

    def run(fused):
        it = iter(gi["noises"])
        smod.torch.randn = lambda *a, **k: next(it)
        try:
            s = DDIMSamplerMultiCond(m)
            if fused:
                s._test_executor = ops_emulator.executor
            else:
                # general path: apply_model through the emulator-backed engine
                m.model.diffusion_model.forward = lambda x, t, context=None, fs=None, **kw: unet._engine.forward(
                    x, t, context, fs, executor=ops_emulator.executor).clone()
            out, _ = s.sample(S=gi["S"], batch_size=1, shape=list(gi["x_T"].shape[1:]), conditioning=gi["cond"],
                              unconditional_conditioning=gi["uncond"], eta=1.0, unconditional_guidance_scale=7.5,
                              cfg_img=CFG_IMG, x_T=gi["x_T"], fs=gi["fs"], timestep_spacing="uniform_trailing",
                              guidance_rescale=0.7, verbose=False,
                              unconditional_conditioning_img_nonetext=gi["uncond_img"])
            return out
        finally:
            smod.torch.randn = real

    fused = run(True)
    gold = torch.from_numpy(np.load(HERE / "golden" / "multicond_tiny.npz")["ddim_samples"])
    err = (fused - gold).abs().max().item()
    assert err < 3e-2 * gold.abs().max().item(), err      # fp16 activations in the interpreted UNet, 4 steps
    general = run(False)
    assert (fused - general).abs().max().item() < 3e-2 * gold.abs().max().item()

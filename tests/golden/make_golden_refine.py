"""Golden for refining a clip: the UNMODIFIED reference samplers (lvdm/models/samplers/ddim.py and
ddim_multiplecond.py) on the tiny configuration, with teacher-forced noise — run in the authoring container:

    python tests/golden/make_golden_refine.py

Covers `stochastic_encode` (per-row DDIM indices, and DDPM timesteps with use_original_steps), `decode` (t_start 3 of a
4-step uniform_trailing eta-1 schedule, cfg 7.5) and a 4-step `sample(mask=..., x0=...)` with and without clean_cond,
for both samplers (the multi-condition `decode` raises KeyError in the reference and is not run).  Every N(0, 1) draw
comes from refine_inputs(): the DDIM noise through ddim.noise_like, the q_sample noise through torch.randn_like.
"""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))

from oracle import ref_shims  # noqa: E402
from tiny_config import TINY_LATENT_HW, TINY_T, model_config  # noqa: E402
from make_golden import SEED  # noqa: E402
from make_golden_multicond import CFG_IMG, multicond_inputs  # noqa: E402
from tooncrafter_b200 import synthetic  # noqa: E402

S, T_START = 4, 3


def refine_inputs():
    """make_golden_multicond's conditioning plus the clip latents, masks and teacher-forced noise of this golden."""
    gi = multicond_inputs()
    T = TINY_T
    h, w = TINY_LATENT_HW
    g = lambda name: synthetic._gen(name, 123)
    gi["x0"] = torch.randn(1, 4, T, h, w, generator=g("refine.x0"))
    gi["x0_rows"] = torch.randn(3, 4, T, h, w, generator=g("refine.x0_rows"))
    gi["enc_noise_rows"] = torch.randn(3, 4, T, h, w, generator=g("refine.enc_noise_rows"))
    gi["t_ddim"] = torch.tensor([0, 2, 3])
    gi["t_ddpm"] = torch.tensor([0, 499, 999])
    gi["enc_noise"] = torch.randn(1, 4, T, h, w, generator=g("refine.enc_noise"))
    # frames 0 and T-1 kept, frame 1 half kept (a fractional mask exercises the blend arithmetic), the rest sampled
    mask = torch.zeros(1, 1, T, 1, 1)
    mask[:, :, [0, T - 1]] = 1.0
    mask[:, :, 1] = 0.5
    gi["mask"] = mask
    gi["q_noises"] = [torch.randn(1, 4, T, h, w, generator=g(f"refine.q_noise.{i}")) for i in range(S)]
    return gi


def _sampler(module):
    class Sampler(module.DDIMSampler):
        def register_buffer(self, name, attr):
            if isinstance(attr, torch.Tensor):
                attr = attr.to(self.model.device)
            setattr(self, name, attr)
    return Sampler


def run_reference(module, model, gi, multicond: bool):
    """{name: array} of every run the reference sampler in `module` supports."""
    out = {}
    sampler = _sampler(module)(model)
    sampler.make_schedule(S, "uniform_trailing", ddim_eta=1.0, verbose=False)
    out["enc_ddim"] = sampler.stochastic_encode(gi["x0_rows"], gi["t_ddim"], noise=gi["enc_noise_rows"])
    out["enc_ddpm"] = sampler.stochastic_encode(gi["x0_rows"], gi["t_ddpm"], use_original_steps=True,
                                                noise=gi["enc_noise_rows"])
    z_enc = sampler.stochastic_encode(gi["x0"], torch.tensor([T_START - 1]), noise=gi["enc_noise"])
    orig_nl, orig_rl = module.noise_like, torch.randn_like
    try:
        if not multicond:
            it = iter(gi["noises"])
            module.noise_like = lambda shape, device, repeat=False: next(it)
            out["decode"] = sampler.decode(z_enc, gi["cond"], T_START, unconditional_guidance_scale=7.5,
                                           unconditional_conditioning=gi["uncond"])
        extra = dict(cfg_img=CFG_IMG, unconditional_conditioning_img_nonetext=gi["uncond_img"]) if multicond else {}
        for clean in (False, True):
            it, qit = iter(gi["noises"]), iter(gi["q_noises"])
            module.noise_like = lambda shape, device, repeat=False: next(it)
            torch.randn_like = lambda x, *a, **k: next(qit)
            samples, _ = sampler.sample(S=S, batch_size=1, shape=list(gi["x_T"].shape[1:]), conditioning=gi["cond"],
                                        unconditional_conditioning=gi["uncond"], eta=1.0,
                                        unconditional_guidance_scale=7.5, x_T=gi["x_T"], fs=gi["fs"],
                                        timestep_spacing="uniform_trailing", guidance_rescale=0.7, verbose=False,
                                        mask=gi["mask"], x0=gi["x0"], clean_cond=clean, **extra)
            out["masked_clean" if clean else "masked"] = samples
    finally:
        module.noise_like, torch.randn_like = orig_nl, orig_rl
    return {k: v.numpy() for k, v in out.items()}


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    model = ref_shims.build_reference_model(model_config()).eval()
    synthetic.fill_module_(model, seed=SEED)
    gi = refine_inputs()
    ref_shims.install()
    import lvdm.models.samplers.ddim as ref_ddim
    import lvdm.models.samplers.ddim_multiplecond as ref_mc
    with torch.no_grad():
        out = run_reference(ref_ddim, model, gi, False)
        out.update({f"mc_{k}": v for k, v in run_reference(ref_mc, model, gi, True).items()})
        try:
            mc = _sampler(ref_mc)(model)
            mc.make_schedule(S, "uniform_trailing", ddim_eta=1.0, verbose=False)
            mc.decode(gi["x0"], gi["cond"], T_START, unconditional_guidance_scale=7.5,
                      unconditional_conditioning=gi["uncond"])
            raise SystemExit("the reference's multi-condition decode was expected to raise KeyError")
        except KeyError as e:
            assert e.args == ("unconditional_conditioning_img_nonetext",), e
    np.savez_compressed(HERE / "refine_tiny.npz", **out)
    print("wrote refine_tiny.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()

"""Golden for the multi-condition sampler: the UNMODIFIED reference
lvdm/models/samplers/ddim_multiplecond.py::DDIMSampler on the tiny configuration, 4 teacher-forced steps, three-way
guidance (cfg 7.5, cfg_img 4.0, guidance_rescale 0.7) — run in the authoring container:

    python tests/golden/make_golden_multicond.py
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
from tiny_config import TINY_CONTEXT_DIM, TINY_LATENT_HW, TINY_T, model_config  # noqa: E402
from make_golden import SEED, golden_inputs  # noqa: E402
from tooncrafter_b200 import synthetic  # noqa: E402

CFG_IMG = 4.0


def multicond_inputs():
    """The third conditioning (image without text) on top of make_golden.golden_inputs()."""
    gi = golden_inputs()
    h, w = TINY_LATENT_HW
    ctx = torch.randn(1, 77 + 16 * TINY_T, TINY_CONTEXT_DIM, generator=synthetic._gen("ctx_uncond_img", 123))
    gi["uncond_img"] = {"c_crossattn": [ctx], "c_concat": gi["uncond"]["c_concat"]}
    return gi


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    model = ref_shims.build_reference_model(model_config()).eval()
    synthetic.fill_module_(model, seed=SEED)
    gi = multicond_inputs()
    ref_shims.install()
    import lvdm.models.samplers.ddim_multiplecond as ref_mc

    class Sampler(ref_mc.DDIMSampler):
        def register_buffer(self, name, attr):
            if isinstance(attr, torch.Tensor):
                attr = attr.to(self.model.device)
            setattr(self, name, attr)

    it = iter(gi["noises"])
    orig = ref_mc.noise_like
    ref_mc.noise_like = lambda shape, device, repeat=False: next(it)
    try:
        with torch.no_grad():
            samples, _ = Sampler(model).sample(S=gi["S"], batch_size=1, shape=list(gi["x_T"].shape[1:]),
                                               conditioning=gi["cond"], unconditional_conditioning=gi["uncond"],
                                               eta=1.0, unconditional_guidance_scale=7.5, cfg_img=CFG_IMG, x_T=gi["x_T"],
                                               fs=gi["fs"], timestep_spacing="uniform_trailing", guidance_rescale=0.7,
                                               verbose=False,
                                               unconditional_conditioning_img_nonetext=gi["uncond_img"])
    finally:
        ref_mc.noise_like = orig
    np.savez_compressed(HERE / "multicond_tiny.npz", ddim_samples=samples.numpy())
    print("wrote multicond_tiny.npz", samples.shape, float(samples.abs().max()))


if __name__ == "__main__":
    main()

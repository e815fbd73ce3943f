"""Generate tests/golden/full_reference_outputs.npz from the UNMODIFIED reference at FULL width — run in the
authoring container (CPU, fp32, ~10 min, peak RSS ~20 GB):

    python tests/golden/make_golden_full.py

What is pinned (the benchmark geometry: inference_512_v1.0 UNet + VAE, T = 16, latent 40 x 64):
  * three teacher-forced DDIM steps of the reference's own `DDIMSampler.p_sample_ddim` (ddim.py:206-279) at
    S = 50 indices 49 (first, t = 999), 25 (middle) and 0 (last, the sqrt(5.96e-8) step), CFG 7.5, rescale 0.7,
    eta 1: the two UNet outputs (cond / uncond = the B = 2 program the bench times), x_prev and pred_x0;
  * `decode_first_stage` (ddpm3d.py:647-683 -> autoencoder_dualref.py:489-527) of the T = 16 pass and of the
    T = 14 pass of scripts/evaluation/inference.py:262-270.
Weights and inputs are regenerated from seeds by the tests (tooncrafter_b200/synthetic.py); only strided
subsamples + moments of the reference's OUTPUTS are stored (the full tensors are 2.6 MB and 94 MB).
"""
import sys
import time
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(HERE.parent))

from oracle import ref_shims  # noqa: E402
from tiny_config import FULL_DDCONFIG, FULL_UNET, model_config  # noqa: E402
from tooncrafter_b200 import synthetic  # noqa: E402

SEED = 0
T, LH, LW = 16, 40, 64
DDIM_S = 50
DDIM_INDICES = (49, 25, 0)
UNET_STRIDE = 37          # 655 360 outputs -> 17 713 samples
DEC_STRIDE = 997          # 7 864 320 (T = 16) -> 7 888 samples


def full_inputs():
    """Deterministic full-size inputs shared with the GPU tests."""
    g = lambda name: synthetic._gen(name, 321)
    x_T, cond, uncond = synthetic.synthetic_inputs(1, T, LH, LW, 1024, seed=123)
    xs = {49: x_T}
    for idx in DDIM_INDICES[1:]:
        xs[idx] = torch.randn(1, 4, T, LH, LW, generator=g(f"full.x.{idx}"))
    noises = {idx: torch.randn(1, 4, T, LH, LW, generator=g(f"full.noise.{idx}")) for idx in DDIM_INDICES}
    z = torch.randn(1, 4, T, LH, LW, generator=g("full.z")) * 0.18215 * 3
    ref = synthetic.synthetic_ref_context(FULL_DDCONFIG["ch"], FULL_DDCONFIG["ch_mult"], 8 * LH, 8 * LW, seed=123)
    return dict(cond=cond, uncond=uncond, xs=xs, noises=noises, z=z, ref=ref, fs=torch.tensor([10]))


def middle_pass_indices(t=T):
    """scripts/evaluation/inference.py:264-267: drop latents 1 and -2 for the second decode."""
    idx = list(range(t))
    del idx[1]
    del idx[-2]
    return idx


def sub(t, stride):
    f = t.flatten().float()
    return f[::stride].numpy(), np.array([f.mean().item(), f.std().item(), f.abs().max().item()])


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    t0 = time.time()
    model = ref_shims.build_reference_model(model_config(FULL_UNET, FULL_DDCONFIG)).eval()
    synthetic.fill_module_(model, seed=SEED)
    model.perframe_ae = True
    model.temporal_length = T
    gi = full_inputs()
    out = {}
    print(f"model built in {time.time() - t0:.0f} s")
    with torch.no_grad():
        sampler = ref_shims.make_sampler(model)
        sampler.make_schedule(ddim_num_steps=DDIM_S, ddim_discretize="uniform_trailing", ddim_eta=1.0, verbose=False)
        import lvdm.models.samplers.ddim as ref_ddim
        rec = []
        real_apply = model.apply_model
        model.apply_model = lambda *a, **k: (rec.append(real_apply(*a, **k)) or rec[-1])
        orig_noise = ref_ddim.noise_like
        for idx in DDIM_INDICES:
            t1 = time.time()
            rec.clear()
            ref_ddim.noise_like = lambda shape, device, repeat=False, _n=gi["noises"][idx]: _n
            step = int(sampler.ddim_timesteps[idx])
            ts = torch.full((1,), step, dtype=torch.long)
            x_prev, pred_x0 = sampler.p_sample_ddim(gi["xs"][idx], gi["cond"], ts, index=idx,
                                                    unconditional_guidance_scale=7.5,
                                                    unconditional_conditioning=gi["uncond"], fs=gi["fs"],
                                                    guidance_rescale=0.7)
            assert len(rec) == 2
            for name, ten in (("e_c", rec[0]), ("e_uc", rec[1]), ("x_prev", x_prev), ("pred_x0", pred_x0)):
                out[f"ddim{idx}_{name}_sub"], out[f"ddim{idx}_{name}_stats"] = sub(ten, UNET_STRIDE)
            out[f"ddim{idx}_t"] = np.array([step])
            print(f"ddim index {idx} (t={step}): {time.time() - t1:.0f} s, |e_c|max {rec[0].abs().max():.3f}")
        ref_ddim.noise_like = orig_noise
        model.apply_model = real_apply

        t1 = time.time()
        vid16 = model.decode_first_stage(gi["z"], ref_context=gi["ref"])
        out["dec16_sub"], out["dec16_stats"] = sub(vid16, DEC_STRIDE)
        print(f"decode T=16: {time.time() - t1:.0f} s, shape {tuple(vid16.shape)}")
        t1 = time.time()
        vid14 = model.decode_first_stage(gi["z"][:, :, middle_pass_indices()], ref_context=gi["ref"])
        out["dec14_sub"], out["dec14_stats"] = sub(vid14, DEC_STRIDE)
        print(f"decode T=14: {time.time() - t1:.0f} s, shape {tuple(vid14.shape)}")
    np.savez_compressed(HERE / "full_reference_outputs.npz", **out)
    for k, v in out.items():
        if k.endswith("stats"):
            print(k, v)
    print(f"total {time.time() - t0:.0f} s")


if __name__ == "__main__":
    main()

"""Generate the plain-AutoencoderKL fixtures from the UNMODIFIED reference — run where the reference is importable:

    python tests/golden/make_golden_plain_vae.py

  * plain_decoder_tiny.npz: the reference's lvdm.models.autoencoder.AutoencoderKL (ae_modules.Decoder) at the tiny
    width of tests/tiny_config.py, with the seeded synthetic weights of tooncrafter_b200/synthetic.py (key prefix
    "first_stage_model."), on CPU in fp32: decode(z) on seeded latents, and LatentDiffusion.decode_first_stage on a
    seeded 5-D latent of 5 frames with temporal_length 4 (two perframe_ae chunks).  Inputs are stored with outputs.
  * state_dict_manifest_plain_vae.json: keys and shapes of the reference's plain AutoencoderKL at full width (meta
    device), prefixed "first_stage_model." as in a checkpoint.
  * reference_model_config_training_{512,1024}.json: the parsed `model` sections of the reference's
    configs/training_{512,1024}_v1.0/config.yaml, whose first stage is the plain AutoencoderKL.
"""
import json
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(HERE.parent))

from oracle import ref_shims  # noqa: E402
from tiny_config import FULL_DDCONFIG, TINY_DDCONFIG, TINY_T, model_config  # noqa: E402
from tooncrafter_b200 import synthetic  # noqa: E402

SEED = 0
PLAIN_TARGET = "lvdm.models.autoencoder.AutoencoderKL"


def plain_model_config(unet=None, ddconfig=None):
    """tests/tiny_config.model_config with the plain AutoencoderKL as first stage."""
    cfg = model_config(unet, ddconfig)
    cfg["params"]["first_stage_config"]["target"] = PLAIN_TARGET
    return cfg


def plain_inputs():
    """Seeded latents: z [2, 4, 8, 12] for decode(z) (already divided by scale_factor), z5 [1, 4, 5, 8, 8] for
    decode_first_stage (scaled like a sampler output)."""
    g = lambda name: synthetic._gen(name, 123)
    z = torch.randn(2, 4, 8, 12, generator=g("plain.z")) * 3.0
    z5 = torch.randn(1, 4, 5, 8, 8, generator=g("plain.z5")) * 0.18215 * 3.0
    return dict(z=z, z5=z5)


def main():
    torch.set_num_threads(8)
    ref_shims.install()
    from lvdm.models.autoencoder import AutoencoderKL
    model = ref_shims.build_reference_model(plain_model_config()).eval()
    assert type(model.first_stage_model) is AutoencoderKL
    synthetic.fill_module_(model, seed=SEED)
    model.perframe_ae = True
    model.temporal_length = TINY_T
    gi = plain_inputs()
    with torch.no_grad():
        dec = model.first_stage_model.decode(gi["z"])
        dfs = model.decode_first_stage(gi["z5"])
    out = dict(z=gi["z"].numpy(), decode=dec.numpy(), z5=gi["z5"].numpy(), decode_first_stage=dfs.numpy())
    np.savez_compressed(HERE / "plain_decoder_tiny.npz", **out)

    with torch.device("meta"):
        vae = AutoencoderKL(ddconfig=dict(FULL_DDCONFIG), lossconfig={"target": "torch.nn.Identity"}, embed_dim=4)
    manifest = {"first_stage_model." + k: list(v.shape) for k, v in vae.state_dict().items()}
    (HERE / "state_dict_manifest_plain_vae.json").write_text(json.dumps(manifest, indent=0))

    import yaml
    for res in (512, 1024):
        with open(ref_shims.REFERENCE_ROOT / "configs" / f"training_{res}_v1.0" / "config.yaml") as f:
            cfg = yaml.safe_load(f)["model"]
        (HERE / f"reference_model_config_training_{res}.json").write_text(json.dumps(cfg, indent=1, sort_keys=True)
                                                                          + "\n")
    for k, v in out.items():
        print(k, v.shape, float(np.abs(v).max()))
    print(len(manifest), "first-stage keys")


if __name__ == "__main__":
    main()

"""Generate tests/golden/live_reference_unet.npz and tests/golden/reference_model_config_512.json from the UNMODIFIED
original project (its checkout given as the first argument):

    python tests/golden/make_golden_live_reference.py <original project checkout>

  * live_reference_unet.npz: the original UNetModel on the tiny configuration (weights seed 5, inputs seed 3), the output
    tests/test_oracle_cpu.py::test_oracle_matches_live_reference_unet compares the oracle against;
  * reference_model_config_512.json: the `model` section of the original's configs/inference_512_v1.0.yaml, parsed, for
    tests/test_oracle_cpu.py::test_reference_yaml_config_builds_our_classes_with_checkpoint_keys.
"""
import json
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE.parent))


def main():
    src = Path(sys.argv[1]).resolve()
    import yaml
    cfg = yaml.safe_load((src / "configs" / "inference_512_v1.0.yaml").read_text())["model"]
    (HERE / "reference_model_config_512.json").write_text(json.dumps(cfg, indent=1, sort_keys=True) + "\n")

    from oracle import ref_shims
    ref_shims.REFERENCE_ROOT = src
    from tiny_config import TINY_CONTEXT_DIM, TINY_T, TINY_UNET
    from tooncrafter_b200 import synthetic
    ref = ref_shims.build_reference_unet(TINY_UNET).eval()
    synthetic.fill_module_(ref, seed=5, prefix="model.diffusion_model.")
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 8, TINY_T, 16, 16, generator=g)
    t = torch.tensor([250])
    ctx = torch.randn(1, 77 + 16 * TINY_T, TINY_CONTEXT_DIM, generator=g)
    fs = torch.tensor([7])
    with torch.no_grad():
        a = ref(x, t, context=ctx, fs=fs)
    np.savez_compressed(HERE / "live_reference_unet.npz", out=a.numpy().astype(np.float32))
    print("wrote", a.shape)


if __name__ == "__main__":
    main()

"""Golden for clip lengths other than the training length: the UNMODIFIED reference UNet
(lvdm/modules/networks/openaimodel3d.py) on the tiny configuration at T = 8 and T = 24 frames with a 77 + 256-token
context, which takes the shared-context branch of UNetModel.forward (:556-562: every frame sees all 77 + 256 tokens)
— run in the authoring container:

    python tests/golden/make_golden_video_length.py

Weights come from tooncrafter_b200/synthetic.py (seed make_golden.SEED) and the inputs from
video_length_inputs(), so only the reference's outputs are stored (tests/golden/video_length_tiny.npz).
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

from tiny_config import TINY_CONTEXT_DIM, TINY_UNET  # noqa: E402
from make_golden import SEED  # noqa: E402
from tooncrafter_b200 import synthetic  # noqa: E402

LENGTHS = (8, 24)
HW = (8, 8)
N_CTX = 77 + 256


def video_length_inputs(T: int):
    """Deterministic UNet inputs at T frames, shared by this generator and the tests."""
    g = lambda name: synthetic._gen(f"video_length.{name}.{T}", 123)
    return dict(x=torch.randn(2, 8, T, *HW, generator=g("x")), t=torch.tensor([999, 301]),
                ctx=torch.randn(2, N_CTX, TINY_CONTEXT_DIM, generator=g("ctx")), fs=torch.tensor([10, 24]))


def main():
    from oracle import ref_shims
    torch.manual_seed(0)
    torch.set_num_threads(8)
    unet = ref_shims.build_reference_unet(TINY_UNET).eval()
    synthetic.fill_module_(unet, seed=SEED, prefix="model.diffusion_model.")
    out = {}
    with torch.no_grad():
        for T in LENGTHS:
            u = video_length_inputs(T)
            out[f"unet_y_T{T}"] = unet(u["x"], u["t"], context=u["ctx"], fs=u["fs"]).numpy()
    np.savez_compressed(HERE / "video_length_tiny.npz", **out)
    for k, v in out.items():
        print(k, v.shape, float(np.abs(v).max()))


if __name__ == "__main__":
    main()

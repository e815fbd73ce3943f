"""Image-conditioning Resampler: oracle pinned to the reference golden, state-dict keys pinned to the
reference manifest, engine program checked on the CPU emulator and (gpu) on the H100 kernels."""
import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from make_golden_resampler import FULL, SEED, TINY, tiny_input  # noqa: E402
from oracle import resampler_oracle  # noqa: E402
from tooncrafter_b200 import modules, synthetic  # noqa: E402


def _tiny_module():
    torch.manual_seed(0)
    m = modules.Resampler(**TINY).eval()
    synthetic.fill_module_(m, seed=SEED, prefix="image_proj_model.")
    return m


def test_oracle_matches_reference_golden():
    m = _tiny_module()
    gold = torch.from_numpy(np.load(HERE / "golden" / "resampler_tiny.npz")["out"])
    with torch.no_grad():
        y = resampler_oracle.resampler_forward(m.state_dict(), tiny_input(), heads=TINY["heads"])
    assert y.shape == gold.shape
    assert (y - gold).abs().max().item() < 2e-5, "oracle restatement drifted from the reference Resampler"


def test_state_dict_keys_match_reference_manifest():
    with torch.device("meta"):
        m = modules.Resampler(**FULL)
    ours = {k: list(v.shape) for k, v in m.state_dict().items()}
    ref = json.loads((HERE / "golden" / "state_dict_manifest_resampler.json").read_text())
    assert ours == ref


def test_engine_program_on_emulator():
    import ops_emulator
    from tooncrafter_b200.cond_engine import ResamplerEngine
    m = _tiny_module()
    eng = ResamplerEngine(m, device="cpu", plan_only=True)
    x = tiny_input()
    y = eng.forward(x, executor=ops_emulator.executor)
    with torch.no_grad():
        ref = resampler_oracle.resampler_forward(m.state_dict(), x, heads=TINY["heads"])
    assert (y - ref).abs().max().item() < 3e-3 * ref.abs().max().item() + 4e-3     # fp16 storage between the launches


def test_engine_refuses_cpu():
    from tooncrafter_b200.cond_engine import ResamplerEngine
    with pytest.raises(RuntimeError):
        ResamplerEngine(_tiny_module())


@pytest.mark.gpu
def test_engine_on_gpu_matches_oracle():
    m = _tiny_module().cuda()
    x = tiny_input()
    with torch.no_grad():
        ref = resampler_oracle.resampler_forward({k: v.cpu() for k, v in m.state_dict().items()}, x, heads=TINY["heads"])
        y = m(x.cuda()).cpu()
        # yardstick: the same algorithm under fp16 autocast (what the reference runs, inference.py:186)
        with torch.autocast("cuda", dtype=torch.float16):
            ya = resampler_oracle.resampler_forward(m.state_dict(), x.cuda(), heads=TINY["heads"]).float().cpu()
    err, err_ac = (y - ref).abs().max().item(), (ya - ref).abs().max().item()
    assert err <= 3 * err_ac + 2e-3 * ref.abs().max().item(), (err, err_ac)


@pytest.mark.gpu
def test_full_size_resampler_runs_on_gpu():
    """Shapes of configs/inference_512_v1.0.yaml: 257 CLIP tokens x 1280 -> 256 context tokens x 1024."""
    torch.manual_seed(0)
    m = modules.Resampler(**FULL).eval()
    synthetic.fill_module_(m, seed=SEED, prefix="image_proj_model.")
    x = torch.randn(1, 257, 1280, generator=synthetic._gen("resampler.full.x", 5))
    with torch.no_grad():
        ref = resampler_oracle.resampler_forward(m.state_dict(), x, heads=FULL["heads"])
        y = m.cuda()(x.cuda()).cpu()
    assert y.shape == (1, 256, 1024)
    assert (y - ref).abs().max().item() < 2e-2 * ref.abs().max().item() + 1e-2

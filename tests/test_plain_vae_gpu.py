"""The plain AutoencoderKL first stage and `animate` on the H100: the plain decode program against the unmodified
reference (tiny golden) and against the fp32 / autocast oracle at full width (320 x 512 and 576 x 1024, T = 16), and the
pipeline with a plain first stage against the reference glue restated from the public classes.

Tolerances are those of the dual-reference decoder's tests: the engine is at most 3x as far from the fp32 result as the
reference algorithm under torch.autocast(fp16) is (+ 2e-3 of the output scale), and at full size the fraction of
elements outside rtol 1e-3 / atol 1e-4 is bounded by 1.5x the autocast fraction + 2 % (tests/test_fullsize_gpu.py)."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

pytestmark = pytest.mark.gpu

from make_golden_plain_vae import SEED  # noqa: E402
from test_engine_gpu import _report  # noqa: E402
from test_fullsize_gpu import _check  # noqa: E402
from test_pipeline import _scale_close, keyframes, model_config  # noqa: E402
from tiny_config import FULL_DDCONFIG, FULL_UNET, TINY_DDCONFIG, TINY_T  # noqa: E402

DEV = "cuda"
# full-width pipeline runs compared across batch shapes (UNet at 4 vs 2 rows, encoder at 1 vs 16 frames): the fp16
# roundings of different GEMM tilings, carried through two eta = 1 DDIM steps and the decoder, reach about 1 % of the
# output scale in the largest of 7.9 M elements (measured 0.95-1.02 % on the H100); a wrong seed, c_concat or splice
# is an O(1) difference
FULL_REL = 2e-2
GOLD = np.load(HERE / "golden" / "plain_decoder_tiny.npz")


def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _plain_ae(ddconfig):
    from tooncrafter_b200 import diffusion, synthetic
    with torch.device("meta"):
        sk = diffusion.AutoencoderKL(ddconfig=ddconfig, embed_dim=4)
    ae = sk.to_empty(device=DEV)
    with torch.no_grad():
        for k, p in ae.named_parameters():
            p.copy_(synthetic.synthetic_tensor("first_stage_model." + k, tuple(p.shape), SEED).to(DEV))
    return ae.eval()


def _oracle(sd, lay, z, chunk=4):
    """decode_plain frame chunk by frame chunk (every frame is independent): fp32 and under autocast."""
    from oracle import plain_vae_oracle
    y32, y16 = [], []
    for i in range(0, z.shape[0], chunk):
        y32.append(plain_vae_oracle.decode_plain(sd, lay, z[i:i + chunk]).cpu())
        with torch.autocast("cuda", dtype=torch.float16):
            y16.append(plain_vae_oracle.decode_plain(sd, lay, z[i:i + chunk]).float().cpu())
    return torch.cat(y32), torch.cat(y16)


def test_tiny_plain_decoder_matches_reference_golden():
    from oracle import plain_vae_oracle
    from tooncrafter_b200 import diffusion, layout, synthetic
    _no_tf32()
    ae = _plain_ae(TINY_DDCONFIG)
    sd = {"first_stage_model." + k: v for k, v in ae.state_dict().items()}
    lay = layout.plain_decoder_layout(TINY_DDCONFIG)
    z = torch.from_numpy(GOLD["z"]).to(DEV)
    y = ae.decode(z)
    assert y.dtype == torch.float16 and tuple(y.shape) == GOLD["decode"].shape
    y32 = plain_vae_oracle.decode_plain(sd, lay, z)
    with torch.autocast("cuda", dtype=torch.float16):
        y16 = plain_vae_oracle.decode_plain(sd, lay, z)
    gold = torch.from_numpy(GOLD["decode"])
    assert (y32.cpu() - gold).abs().max().item() < 2e-3, "fp32 oracle on the GPU disagrees with the reference golden"
    _report("plain decoder", y, gold, y16)
    assert torch.equal(ae.decode(z), y), "graph replay differs from the first run"
    # decode_first_stage on a 5-D latent (two perframe_ae chunks, post_quant_conv applied) vs the reference
    m = diffusion.instantiate_from_config(synthetic.with_first_stage(model_config(), "plain"))
    synthetic.fill_module_(m, seed=SEED)
    m = m.to(DEV).eval()
    m.perframe_ae, m.temporal_length = True, TINY_T
    z5 = torch.from_numpy(GOLD["z5"]).to(DEV)
    v = m.decode_first_stage(z5)
    v32 = plain_vae_oracle.decode_first_stage_plain(sd, lay, z5)
    assert (v32.cpu() - torch.from_numpy(GOLD["decode_first_stage"])).abs().max().item() < 2e-3
    with torch.autocast("cuda", dtype=torch.float16):
        v16 = plain_vae_oracle.decode_first_stage_plain(sd, lay, z5)
    _report("plain decode_first_stage", v, torch.from_numpy(GOLD["decode_first_stage"]), v16)


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("h,w", [(40, 64), (72, 128)])
def test_full_size_plain_decoder_program(h, w):
    """16 frames at 320 x 512 and at 576 x 1024 (configs/training_1024_v1.0) through the full-width plain decoder vs
    the fp32 oracle on the same seeded weights, with the autocast evaluation as yardstick."""
    from tooncrafter_b200 import layout
    _no_tf32()
    ae = _plain_ae(FULL_DDCONFIG)
    g = torch.Generator().manual_seed(17)
    z = (torch.randn(16, 4, h, w, generator=g) * 3.0).to(DEV)
    y = ae.decode(z).float().cpu()
    assert tuple(y.shape) == (16, 3, 8 * h, 8 * w)
    plan = ae.decoder_engine().plan_for(16, h, w)
    print(f"plain decoder 16 x {8 * h} x {8 * w}: arena {plan.arena.buf.numel() / 2 ** 30:.2f} GiB")
    sd = {"first_stage_model." + k: v for k, v in ae.state_dict().items()}
    y32, y16 = _oracle(sd, layout.plain_decoder_layout(FULL_DDCONFIG), z)
    _check(f"plain decoder 16 x {8 * h} x {8 * w} vs fp32 oracle", y, y32, y16)


# ------------------------------------------------------------------------------------------ pipeline at full width
@pytest.fixture(scope="module")
def full_plain_model():
    from tooncrafter_b200 import synthetic
    from tooncrafter_b200.interpolate import rewrite_targets
    _no_tf32()
    cfg = model_config(FULL_UNET, FULL_DDCONFIG)
    p = cfg["params"]
    p["cond_stage_config"] = {"target": "lvdm.modules.encoders.condition.FrozenOpenCLIPEmbedder",
                              "params": {"freeze": True, "layer": "penultimate"}}
    p["img_cond_stage_config"] = {"target": "lvdm.modules.encoders.condition.FrozenOpenCLIPImageEmbedderV2",
                                  "params": {"freeze": True}}
    p["image_proj_stage_config"] = {"target": "lvdm.modules.encoders.resampler.Resampler",
                                    "params": dict(dim=1024, depth=4, dim_head=64, heads=12, num_queries=16,
                                                   embedding_dim=1280, output_dim=1024, ff_mult=4, video_length=16)}
    m = synthetic.synthetic_model(rewrite_targets(cfg), torch.device(DEV), first_stage="plain")
    m.perframe_ae = True
    return m


@pytest.mark.timeout(1800)
def test_full_size_animate_matches_restated_image_guided_synthesis(full_plain_model):
    import test_plain_vae
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    m = full_plain_model
    image = keyframes(1, (320, 512), seed=3)[0]
    got = ToonCrafterPipeline(m).animate(image, steps=2, seed=55, output="float")
    u8 = ToonCrafterPipeline(m).animate(image, steps=2, seed=55)
    with torch.no_grad():
        ref = test_plain_vae.restated_animate(m, image, 55, 2)
    assert got.shape == (3, 16, 320, 512) and u8.shape == (16, 320, 512, 3) and u8.is_cuda
    assert torch.equal(u8.cpu(), test_plain_vae.save_path_u8(got.cpu()))
    _scale_close(got, ref, "full-size animate (plain first stage) vs restated image_guided_synthesis(interp=False)",
                 rel=FULL_REL)


@pytest.mark.timeout(1800)
def test_full_size_plain_interpolate_k3_matches_pair_runs(full_plain_model):
    """K = 3, DDIM-2, plain first stage: each segment against a K = 2 run on its pair with seed + k."""
    from test_pipeline import joined_from_segments
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    pipe = ToonCrafterPipeline(full_plain_model)
    kf = keyframes(3, (320, 512), seed=9)
    three = pipe.interpolate(kf, steps=2, seed=60, output="float")
    u8 = pipe.interpolate(kf, steps=2, seed=60)
    assert three.shape == (2, 3, 16, 320, 512) and u8.shape == (31, 320, 512, 3)
    assert torch.equal(u8.cpu(), joined_from_segments(three, loop=False))
    for k in range(2):
        pair = pipe.interpolate(kf[k:k + 2], steps=2, seed=60 + k, output="float")
        _scale_close(three[k], pair[0], f"plain first stage: segment {k} of K=3 vs K=2 on its pair", rel=FULL_REL)
    assert (three[0] - three[1]).abs().max().item() > 1e-2

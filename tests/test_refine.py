"""Refining a clip and regenerating chosen frames: DDIMSampler.stochastic_encode / decode / sample(mask, x0, t_start)
against the unmodified reference samplers (tests/golden/make_golden_refine.py) and a restatement of them on the
oracle, the fused path on the CPU program interpreter, ToonCrafterPipeline.refine's contract on the tiny model, and the
--init-video command line.  The same pipeline equalities run on the H100 in test_refine_gpu.py."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from make_golden import SEED  # noqa: E402
from make_golden_multicond import CFG_IMG  # noqa: E402
from make_golden_refine import S, T_START, refine_inputs  # noqa: E402
from test_n_samples import model  # noqa: E402
from test_pipeline import TINY_SIZE, keyframes  # noqa: E402
from tiny_config import TINY_T, TINY_UNET, model_config  # noqa: E402

from oracle import ddim_oracle, unet_oracle  # noqa: E402
from tooncrafter_b200 import diffusion, layout, runtime, synthetic  # noqa: E402
from tooncrafter_b200.pipeline import ToonCrafterPipeline, preprocess  # noqa: E402
from tooncrafter_b200.sampler import DDIMSampler, DDIMSamplerMultiCond  # noqa: E402

GOLD = np.load(HERE / "golden" / "refine_tiny.npz")
T = TINY_T
BOUND = 3e-2          # test_sampler_cpu.py: fp16 activations in the interpreted UNet, 4 steps


def _gold(name):
    return torch.from_numpy(GOLD[name])


# ----------------------------------------------------------------------------------------- oracle restatement
def oracle_stochastic_encode(sched, tab, x0, t, noise, use_original_steps=False):
    """ddim.py:303-318 (the sampler's own sqrt tables: fp32 square roots of the fp32 alphas_cumprod, ddim.py:38-39)."""
    if use_original_steps:
        ac = sched["alphas_cumprod"]
        sa, s1 = torch.sqrt(ac), torch.sqrt(1.0 - ac)
    else:
        sa, s1 = torch.sqrt(tab["alphas"]), torch.as_tensor(tab["sqrt_one_minus_alphas"])
    size = (t.shape[0],) + (1,) * (x0.dim() - 1)
    return sa.gather(-1, t).reshape(size) * x0 + s1.gather(-1, t).reshape(size) * noise


def oracle_sample(apply_model, sched, x, cond, uncond, S_, noises, t_start=None, phi=0.7, fs=None, mask=None,
                  x0=None, q_noises=None, cfg_img=None, uncond_img=None):
    """ddim.py:135-203 with the last t_start steps only (decode, ddim.py:282-300) and the masked blend (:172-180,
    ddpm3d.py:306-309); three-way guidance (ddim_multiplecond.py:229-234) with cfg_img."""
    tab = ddim_oracle.ddim_tables(sched, S_, 1.0)
    steps = tab["timesteps"] if t_start is None else tab["timesteps"][:t_start]
    n = len(steps)
    for i, step in enumerate(np.flip(steps)):
        index = n - i - 1
        ts = torch.full((x.shape[0],), int(step), dtype=torch.long)
        if mask is not None:
            g = lambda a: a.gather(-1, ts).reshape(-1, 1, 1, 1, 1)
            orig = x0 if q_noises is None else (g(sched["sqrt_alphas_cumprod"]) * x0 +
                                                g(sched["sqrt_one_minus_alphas_cumprod"]) * q_noises[i])
            x = orig * mask + (1.0 - mask) * x
        e_c, e_uc = apply_model(x, ts, cond, fs), apply_model(x, ts, uncond, fs)
        co = ddim_oracle.step_coefficients(sched, tab, index)
        if cfg_img is None:
            x, _ = ddim_oracle.ddim_update(x, e_c, e_uc, noises[i], co, 7.5, phi)
        else:
            e_img = apply_model(x, ts, uncond_img, fs)
            v = e_uc + cfg_img * (e_img - e_uc) + 7.5 * (e_c - e_img)
            x, _ = ddim_oracle.ddim_update(x, e_c, v, noises[i], co, 0.0, phi)       # v + 0 * (e_c - v) = v
    return x


@pytest.fixture(scope="module")
def tiny_sd():
    import json
    man = json.loads((HERE / "golden" / "state_dict_manifest_tiny.json").read_text())
    return {k: synthetic.synthetic_tensor(k, tuple(shape), SEED) for k, shape in man.items()
            if k.startswith(("model.", "first_stage_model."))}


def test_oracle_restatement_matches_reference_golden(tiny_sd):
    gi = refine_inputs()
    sched = ddim_oracle.model_schedule()
    tab = ddim_oracle.ddim_tables(sched, S, 1.0)
    for pre in ("", "mc_"):
        assert torch.equal(oracle_stochastic_encode(sched, tab, gi["x0_rows"], gi["t_ddim"], gi["enc_noise_rows"]),
                           _gold(pre + "enc_ddim"))
        assert torch.equal(oracle_stochastic_encode(sched, tab, gi["x0_rows"], gi["t_ddpm"], gi["enc_noise_rows"],
                                                    True), _gold(pre + "enc_ddpm"))
    ulay = layout.unet_layout(TINY_UNET)

    def apply_model(x, t, c, fs):
        fs = torch.tensor([ulay.default_fs]) if fs is None else fs
        return unet_oracle.unet_forward(tiny_sd, ulay, torch.cat([x] + c["c_concat"], 1), t,
                                        torch.cat(c["c_crossattn"], 1), fs, prefix="model.diffusion_model.")

    def close(a, name, tol=2e-4):
        b = _gold(name)
        assert (a - b).abs().max().item() <= tol * max(1.0, b.abs().max().item()), name

    z_enc = oracle_stochastic_encode(sched, tab, gi["x0"], torch.tensor([T_START - 1]), gi["enc_noise"])
    close(oracle_sample(apply_model, sched, z_enc, gi["cond"], gi["uncond"], S, gi["noises"], t_start=T_START, phi=0.0),
          "decode")
    common = dict(fs=gi["fs"], mask=gi["mask"], x0=gi["x0"])
    close(oracle_sample(apply_model, sched, gi["x_T"], gi["cond"], gi["uncond"], S, gi["noises"],
                        q_noises=gi["q_noises"], **common), "masked")
    close(oracle_sample(apply_model, sched, gi["x_T"], gi["cond"], gi["uncond"], S, gi["noises"], **common),
          "masked_clean")
    close(oracle_sample(apply_model, sched, gi["x_T"], gi["cond"], gi["uncond"], S, gi["noises"],
                        q_noises=gi["q_noises"], cfg_img=CFG_IMG, uncond_img=gi["uncond_img"], **common),
          "mc_masked")


# ----------------------------------------------------------------------------------------- sampler
@pytest.fixture(scope="module")
def tiny_model():
    from tooncrafter_b200.engine import UNetEngine
    m = diffusion.instantiate_from_config(model_config())
    synthetic.fill_module_(m, seed=SEED)
    m = m.eval()
    unet = m.model.diffusion_model
    unet._engine = UNetEngine(unet, device="cpu", plan_only=True)
    return m


class _Forced:
    """Teacher-forced RNG: torch.randn and torch.randn_like return the given tensors in order (the sampler's
    q_sample draw of a step comes before its DDIM draw on both paths, as in the reference)."""

    def __init__(self, draws):
        self.it = iter(draws)

    def __enter__(self):
        self.saved = torch.randn, torch.randn_like
        torch.randn = lambda *a, **k: next(self.it)
        torch.randn_like = lambda *a, **k: next(self.it)

    def __exit__(self, *exc):
        torch.randn, torch.randn_like = self.saved


def _run(m, cls, fused, fn):
    """fn(sampler) on the fused path (program interpreter) or the general path (apply_model through the same
    interpreted engine)."""
    import clip_emulator
    unet = m.model.diffusion_model
    s = cls(m)
    saved = unet.forward
    if fused:
        s._test_executor = clip_emulator.executor
    else:
        s._test_executor = None
        unet.forward = lambda x, t, context=None, fs=None, **kw: unet._engine.forward(
            x, t, context, fs, executor=clip_emulator.executor).clone()
    try:
        return fn(s)
    finally:
        unet.forward = saved


def test_stochastic_encode_is_the_reference_on_cpu(tiny_model):
    gi = refine_inputs()
    for cls, pre in ((DDIMSampler, ""), (DDIMSamplerMultiCond, "mc_")):
        s = cls(tiny_model)
        s.make_schedule(S, "uniform_trailing", 1.0, verbose=False)
        assert torch.equal(s.stochastic_encode(gi["x0_rows"], gi["t_ddim"], noise=gi["enc_noise_rows"]),
                           _gold(pre + "enc_ddim"))
        assert torch.equal(s.stochastic_encode(gi["x0_rows"], gi["t_ddpm"], use_original_steps=True,
                                               noise=gi["enc_noise_rows"]), _gold(pre + "enc_ddpm"))
        with _Forced([gi["enc_noise_rows"]]):
            assert torch.equal(s.stochastic_encode(gi["x0_rows"], gi["t_ddim"]), _gold(pre + "enc_ddim"))


def _masked(s, gi, clean, multicond):
    draws = ([q for pair in zip(gi["q_noises"], gi["noises"]) for q in pair] if not clean else list(gi["noises"]))
    extra = dict(cfg_img=CFG_IMG, unconditional_conditioning_img_nonetext=gi["uncond_img"]) if multicond else {}
    with _Forced(draws):
        out, _ = s.sample(S=S, batch_size=1, shape=list(gi["x_T"].shape[1:]), conditioning=gi["cond"],
                          unconditional_conditioning=gi["uncond"], eta=1.0, unconditional_guidance_scale=7.5,
                          x_T=gi["x_T"], fs=gi["fs"], timestep_spacing="uniform_trailing", guidance_rescale=0.7,
                          verbose=False, mask=gi["mask"], x0=gi["x0"], clean_cond=clean, **extra)
    return out


def _decode(s, gi):
    s.make_schedule(S, "uniform_trailing", 1.0, verbose=False)
    z_enc = s.stochastic_encode(gi["x0"], torch.tensor([T_START - 1]), noise=gi["enc_noise"])
    with _Forced(gi["noises"]):
        return s.decode(z_enc, gi["cond"], T_START, unconditional_guidance_scale=7.5,
                        unconditional_conditioning=gi["uncond"])


def _scale_err(a, name):
    b = _gold(name)
    return (a - b).abs().max().item() / b.abs().max().item()


@pytest.mark.parametrize("multicond", [False, True])
def test_fused_and_general_paths_match_reference_golden(tiny_model, multicond):
    """decode (two-way only: the reference's multi-condition decode raises KeyError) and masked sample with and without
    clean_cond, on the fused path and on the general path, against the reference and against each other."""
    gi = refine_inputs()
    cls, pre = (DDIMSamplerMultiCond, "mc_") if multicond else (DDIMSampler, "")
    runs = [("masked", lambda s: _masked(s, gi, False, multicond)),
            ("masked_clean", lambda s: _masked(s, gi, True, multicond))]
    if not multicond:
        runs.append(("decode", lambda s: _decode(s, gi)))
    for name, fn in runs:
        fused, general = _run(tiny_model, cls, True, fn), _run(tiny_model, cls, False, fn)
        assert _scale_err(fused, pre + name) < BOUND, (name, _scale_err(fused, pre + name))
        assert _scale_err(general, pre + name) < BOUND, (name, _scale_err(general, pre + name))
        assert (fused - general).abs().max().item() < BOUND * general.abs().max().item(), name


def test_multicond_decode_raises_key_error_as_the_reference(tiny_model):
    gi = refine_inputs()
    with pytest.raises(KeyError, match="unconditional_conditioning_img_nonetext"):
        _run(tiny_model, DDIMSamplerMultiCond, False, lambda s: _decode(s, gi))


def test_fused_blend_touches_only_masked_frames(tiny_model):
    """One step from a constant latent with a binary frame mask and clean_cond: after the fused path's tc_q_sample the
    latent holds x0 on the masked frames and is unchanged elsewhere."""
    import clip_emulator
    gi = refine_inputs()
    x_T = torch.full_like(gi["x_T"], 0.25)
    mask = torch.zeros(1, 1, T, 1, 1)
    mask[:, :, [1, 2]] = 1.0
    seen = []

    def spy(fn, args, kw):
        clip_emulator.executor(fn, args, kw)
        if fn.__name__ == "q_sample":
            seen.append(args[0].clone())

    s = DDIMSampler(tiny_model)
    s._test_executor = spy
    s.sample(S=S, batch_size=1, shape=list(x_T.shape[1:]), conditioning=gi["cond"],
             unconditional_conditioning=gi["uncond"], eta=1.0, unconditional_guidance_scale=7.5, x_T=x_T, fs=gi["fs"],
             timestep_spacing="uniform_trailing", verbose=False, mask=mask, x0=gi["x0"], clean_cond=True, t_start=1)
    assert len(seen) == 1
    assert torch.equal(seen[0][:, :, [1, 2]], gi["x0"][:, :, [1, 2]])
    assert torch.equal(seen[0][:, :, [0, 3]], x_T[:, :, [0, 3]])


def test_t_start_is_checked(tiny_model):
    gi = refine_inputs()
    s = DDIMSampler(tiny_model)
    kw = dict(S=S, batch_size=1, shape=list(gi["x_T"].shape[1:]), conditioning=gi["cond"], verbose=False)
    with pytest.raises(ValueError, match="x_T"):
        s.sample(t_start=2, **kw)
    for bad in (0, S + 1, 1.5, True, "2"):
        with pytest.raises(ValueError, match="t_start"):
            s.sample(t_start=bad, x_T=gi["x_T"], **kw)


# ----------------------------------------------------------------------------------------- pipeline
class Emulated:
    """A pipeline run on the CPU program interpreter (clip_emulator), or on the GPU when dev is cuda;
    results come back on the CPU."""

    def __init__(self, pipe, dev="cpu"):
        self.pipe, self.dev = pipe, dev

    def __getattr__(self, name):
        fn = getattr(self.pipe, name)

        def run(*a, **kw):
            if self.dev != "cpu":
                return fn(*a, **kw).cpu()
            import clip_emulator
            runtime.TEST_EXECUTOR = clip_emulator.executor
            try:
                return fn(*a, **kw)
            finally:
                runtime.TEST_EXECUTOR = None
        return run


def check_refine_is_interpolate(p, steps=2, T_=T, size=TINY_SIZE, **kw):
    """refine(clip, 1.0) equals interpolate([clip[0], clip[-1]], video_length=T) bit for bit (the model's schedule has
    zero terminal SNR, so the encoded latent is exactly the noise), uint8 and float."""
    clip = keyframes(T_, size=size, seed=71)
    for output in ("uint8", "float"):
        a = p.refine(clip, 1.0, steps=steps, seed=17, size=size, output=output, **kw)
        b = p.interpolate(clip[[0, T_ - 1]], steps=steps, seed=17, size=size, video_length=T_, output=output, **kw)
        assert a.shape == (b.shape if output == "uint8" else b.shape[1:]), output
        assert torch.equal(a, b if output == "uint8" else b[0]), output


def check_variants_and_keep(p, steps=2, T_=T, size=TINY_SIZE):
    """n_samples=2 variant 0 is the single-sample call, with and without keep; keep changes the result; the shape is
    that of a one-segment interpolate."""
    clip = keyframes(T_, size=size, seed=72)
    keep = [0, 1, T_ - 2, T_ - 1]
    kw = dict(steps=steps, seed=5, size=size, segments_per_batch=1)
    one = p.refine(clip, 0.5, **kw)
    two = p.refine(clip, 0.5, n_samples=2, **kw)
    assert one.shape == (T_, *size, 3) and two.shape == (2, T_, *size, 3)
    assert torch.equal(two[0], one) and not torch.equal(two[1], two[0])
    kept = p.refine(clip, 0.5, keep=keep, **kw)
    kept2 = p.refine(clip, 0.5, keep=keep, n_samples=2, **kw)
    assert kept.shape == (T_, *size, 3) and torch.equal(kept2[0], kept)
    assert not torch.equal(kept, one)
    return one, kept


@pytest.mark.parametrize("first_stage", ["dualref", "plain"])
def test_refine_at_full_strength_is_interpolate_on_emulator(first_stage):
    check_refine_is_interpolate(Emulated(ToonCrafterPipeline(model(first_stage, "cpu"))))


def test_refine_three_way_guidance_at_full_strength_is_interpolate_on_emulator():
    check_refine_is_interpolate(Emulated(ToonCrafterPipeline(model("dualref", "cpu"))), steps=1, cfg_img=3.0)


def test_refine_variants_and_keep_on_emulator():
    check_variants_and_keep(Emulated(ToonCrafterPipeline(model("dualref", "cpu"))))


def test_refine_encodes_interior_frames_in_decode_chunks():
    """The interior frames go through the encoder in chunks of en_and_decode_n_samples_a_time, and frame j's latent
    does not depend on the chunking."""
    m = model("dualref", "cpu")
    p = ToonCrafterPipeline(m)
    import clip_emulator
    clip = keyframes(8, seed=73)
    frames = preprocess(clip, TINY_SIZE)
    runtime.TEST_EXECUTOR = clip_emulator.executor
    seen = []
    enc = m.first_stage_model.encode
    try:
        m.first_stage_model.encode = lambda x, **kw: (seen.append(x.shape[0]), enc(x, **kw))[1]
        z_ends = torch.zeros(2, 4, TINY_SIZE[0] // 8, TINY_SIZE[1] // 8)
        saved = m.en_and_decode_n_samples_a_time
        m.en_and_decode_n_samples_a_time = 4
        a = p._clip_latents(z_ends, frames[1:7], list(range(100, 106)))
        m.en_and_decode_n_samples_a_time = 1
        b = p._clip_latents(z_ends, frames[1:7], list(range(100, 106)))
    finally:
        m.first_stage_model.encode = enc
        m.en_and_decode_n_samples_a_time = saved
        runtime.TEST_EXECUTOR = None
    assert seen == [4, 2] + [1] * 6
    assert a.shape == (1, 4, 8, *z_ends.shape[-2:])
    assert (a - b).abs().max().item() <= 1e-2 * b.abs().max().item()


@pytest.mark.parametrize("kw", [dict(strength=0.0), dict(strength=1.5), dict(strength=-0.5), dict(strength=True),
                                dict(strength="0.5"), dict(strength=None), dict(strength=0.01),
                                dict(keep=[0, T]), dict(keep=[-1]), dict(keep=[1, 1]), dict(keep=[1.0]),
                                dict(keep=[True]), dict(n_samples=0), dict(output="png")])
def test_refine_refuses_bad_arguments_before_any_work(kw):
    p = ToonCrafterPipeline(model("dualref", "cpu"))
    p._generate = p._render = lambda *a, **k: pytest.fail("work started")
    args = dict(strength=0.5, steps=10, size=TINY_SIZE)
    args.update(kw)
    with pytest.raises(ValueError):
        p.refine(keyframes(T, seed=1), **args)


@pytest.mark.parametrize("length", [3, 5, 66])
def test_refine_refuses_bad_clip_lengths(length):
    p = ToonCrafterPipeline(model("dualref", "cpu"))
    p._generate = lambda *a, **k: pytest.fail("work started")
    with pytest.raises(ValueError, match="video_length"):
        p.refine(torch.zeros(length, 8, 8, 3, dtype=torch.uint8), 0.5)


# ----------------------------------------------------------------------------------------- command line
def test_init_video_readers(tmp_path):
    from PIL import Image

    from tooncrafter_b200.interpolate import read_init_video, write_video
    v = keyframes(6, size=(16, 24), seed=3).numpy()
    write_video(v, str(tmp_path / "out"), 8)
    assert np.array_equal(read_init_video(str(tmp_path / "out")), v)              # frame_%04d.png
    assert np.array_equal(read_init_video(str(tmp_path / "out" / "video.npy")), v)
    d = tmp_path / "mixed"
    d.mkdir()
    for i, name in enumerate(["b.png", "a.jpg", "c.PNG"]):                       # get_filelist: by suffix, then sorted
        Image.fromarray(v[i]).save(d / name)
    got = read_init_video(str(d))
    assert got.shape == (3, 16, 24, 3)
    assert np.array_equal(got[1], v[0]) and np.array_equal(got[2], v[2])        # a.jpg (lossy), b.png, c.PNG
    cv2 = pytest.importorskip("cv2")
    path = str(tmp_path / "clip.avi")
    wr = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), 8, (24, 16))
    if not wr.isOpened():
        pytest.skip("no OpenCV video writer")
    for fr in v:
        wr.write(np.ascontiguousarray(fr[..., ::-1]))
    wr.release()
    got = read_init_video(path)
    assert got.shape == v.shape and got.dtype == np.uint8
    for bad, what in ((tmp_path / "none", "no such"), (tmp_path / "empty", "no images")):
        if what == "no images":
            bad.mkdir()
        with pytest.raises(ValueError, match=what):
            read_init_video(str(bad))
    np.save(tmp_path / "f.npy", v.astype(np.float32))
    with pytest.raises(ValueError, match="uint8"):
        read_init_video(str(tmp_path / "f.npy"))


def test_keep_frames_parsing():
    from tooncrafter_b200.interpolate import parse_frame_ranges
    assert parse_frame_ranges("0-3,12-15", 16) == [0, 1, 2, 3, 12, 13, 14, 15]
    assert parse_frame_ranges("5", 16) == [5]
    assert parse_frame_ranges(" 1 , 3-4", 8) == [1, 3, 4]
    for bad in ("0-16", "3-1", "a", "1,1", "0-2,2", "", "-1", "1-"):
        with pytest.raises(ValueError):
            parse_frame_ranges(bad, 16)


def test_cli_init_video_arguments(tmp_path, capsys):
    from tooncrafter_b200.interpolate import main
    v = keyframes(8, size=(16, 24), seed=3).numpy()
    np.save(tmp_path / "clip.npy", v)
    np.save(tmp_path / "odd.npy", v[:7])
    base = ["--config", "c.yaml", "--out", str(tmp_path / "o"), "--synthetic-weights"]
    clip = ["--init-video", str(tmp_path / "clip.npy")]
    bad = [clip,                                                                 # no --strength
           clip + ["--frames", "a.png", "--strength", "0.5"],                   # two sources
           ["--prompt-dir", str(tmp_path), "--init-video", str(tmp_path / "clip.npy"), "--strength", "0.5"],
           ["--frames", "a.png", "b.png", "--strength", "0.5"],                 # --strength without --init-video
           ["--frames", "a.png", "b.png", "--keep-frames", "0-1"],
           clip + ["--strength", "1.5"], clip + ["--strength", "0.01"],
           clip + ["--strength", "0.5", "--keep-frames", "0-8"],
           clip + ["--strength", "0.5", "--loop"],
           clip + ["--strength", "0.5", "--video-length", "16"],
           ["--init-video", str(tmp_path / "odd.npy"), "--strength", "0.5"],
           ["--init-video", str(tmp_path / "missing"), "--strength", "0.5"]]
    for extra in bad:
        with pytest.raises(SystemExit) as e:
            main(base + extra)
        assert e.value.code == 2, extra
    # a valid command line gets past parsing and reading to the model (the config file does not exist)
    with pytest.raises((FileNotFoundError, SystemExit)) as e:
        main(base + clip + ["--strength", "0.5", "--keep-frames", "0-1,6-7", "--n-samples", "2"])
    assert not (isinstance(e.value, SystemExit) and e.value.code == 2)

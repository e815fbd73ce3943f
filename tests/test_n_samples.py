"""Several samples per input (`n_samples`, the reference's --n_samples) and keyframe-pair directories
(`interpolate_pairs`, the reference's --prompt_dir with --interp): shapes, argument checks, the variant and pair RNG
contracts and the directory reader, on the CPU program interpreter; the same equalities, a full-width run and the
command line on the H100.

Variants are extra rows of the same sample() calls; with one row (or pair) per call a variant or a pair is the same
computation whatever else runs, so those comparisons are bit for bit.  Larger batches change the UNet program's rows and
are held to the batch-tiling bound of the RNG-contract tests (1 % of the output scale), or to 3 % where the encoder
and tower batches change as well."""
import os
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from test_pipeline import TINY_SIZE, _scale_close, joined_from_segments, keyframes  # noqa: E402
from tiny_config import TINY_T  # noqa: E402
from tooncrafter_b200 import runtime  # noqa: E402
from tooncrafter_b200.interpolate import get_parser, main, read_prompt_dir  # noqa: E402
from tooncrafter_b200.modules import clip_tokenize  # noqa: E402
from tooncrafter_b200.pipeline import (ToonCrafterPipeline, check_count, check_n_samples,  # noqa: E402
                                       default_pairs_per_batch)

T = TINY_T


def token_ids(P):
    """P distinct prompts as token ids (<start_of_text> word <end_of_text>), so no tokenizer is needed."""
    ids = clip_tokenize([""] * P)
    eot = ids[0, 1].item()
    for i in range(P):
        ids[i, 1], ids[i, 2] = 320 + 7 * i, eot
    return ids


def pair_list(P, seed=13):
    kf = keyframes(2 * P, seed=seed)
    return [(kf[2 * i], kf[2 * i + 1]) for i in range(P)]


class _Emulated:
    """Runs the pipeline on the CPU program interpreter (clip_emulator), or on the GPU when dev is cuda."""

    def __init__(self, pipe, dev):
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


_MODELS = {}


def model(first_stage, dev):
    """test_pipeline.py's tiny model with the given first stage on `dev` (cached)."""
    if (first_stage, dev) not in _MODELS:
        from test_pipeline import SEED, tiny_config
        from tooncrafter_b200 import diffusion, synthetic
        from tooncrafter_b200.interpolate import rewrite_targets
        m = diffusion.instantiate_from_config(rewrite_targets(synthetic.with_first_stage(tiny_config(), first_stage)))
        synthetic.fill_module_(m, seed=SEED)
        m.perframe_ae = True
        _MODELS[(first_stage, dev)] = m.to(dev).eval()
    return _MODELS[(first_stage, dev)]


def pipe_on(first_stage, dev):
    return _Emulated(ToonCrafterPipeline(model(first_stage, dev)), dev)


# the equalities, shared by the CPU (interpreter) and GPU tests; steps=1 keeps the interpreter runs short
def check_none_is_one(p, K, loop, output, steps=1):
    kw = dict(steps=steps, seed=31, size=TINY_SIZE, loop=loop, output=output)
    kf = keyframes(K, seed=3)
    none, one = p.interpolate(kf, **kw), p.interpolate(kf, n_samples=1, **kw)
    S = K if loop else K - 1
    F = (T - 1) * S + (0 if loop else 1)
    assert none.shape == ((F, *TINY_SIZE, 3) if output == "uint8" else (S, 3, T, *TINY_SIZE))
    assert one.shape == (1,) + tuple(none.shape) and torch.equal(one[0], none)


def check_animate_none_is_one(p, steps=1):
    """One variant per sample() call (the CPU interpreter's matmuls round differently at other batch sizes)."""
    kw = dict(steps=steps, seed=9, size=TINY_SIZE, segments_per_batch=1)
    image = keyframes(1, seed=5)[0]
    none, two = p.animate(image, **kw), p.animate(image, n_samples=2, **kw)
    assert none.shape == (T, *TINY_SIZE, 3) and two.shape == (2, T, *TINY_SIZE, 3)
    assert torch.equal(two[0], none)
    assert not torch.equal(two[1], two[0])
    vf = p.animate(image, n_samples=2, output="float", **kw)
    assert vf.shape == (2, 3, T, *TINY_SIZE)
    assert torch.equal(two[1], joined_from_segments(vf[1:2], False))


def check_variants(p, steps=1):
    """Variant v of an n = 3 call is variant v of an n = 2 call (one row per sample() call), variants differ, and the
    uint8 video of each variant is its float segments joined by the seam rule."""
    kf = keyframes(3, seed=4)
    kw = dict(steps=steps, seed=40, size=TINY_SIZE, segments_per_batch=1)
    three = p.interpolate(kf, n_samples=3, output="float", **kw)
    two = p.interpolate(kf, n_samples=2, output="float", **kw)
    assert three.shape == (3, 2, 3, T, *TINY_SIZE) and two.shape == (2, 2, 3, T, *TINY_SIZE)
    assert torch.equal(three[:2], two)
    scale = three.abs().max().item()
    assert (three[1] - three[0]).abs().max().item() > 1e-2 * scale, "variants 0 and 1 are the same video"
    assert (three[2] - three[1]).abs().max().item() > 1e-2 * scale, "variants 1 and 2 are the same video"
    u8 = p.interpolate(kf, n_samples=3, **kw)
    assert u8.shape == (3, 2 * (T - 1) + 1, *TINY_SIZE, 3) and u8.dtype == torch.uint8
    for v in range(3):
        assert torch.equal(u8[v].cpu(), joined_from_segments(three[v], False))
    return three


def check_pairs(p, steps=1):
    """interpolate_pairs with P = 3, n = 2, distinct prompts: with one pair per group bit for bit the per-pair
    interpolate calls of its contract; with the default groups within the batch-tiling bound."""
    P, n, seed = 3, 2, 50
    pairs, ids = pair_list(P), token_ids(P)
    kw = dict(steps=steps, size=TINY_SIZE, output="float")
    got = p.interpolate_pairs(pairs, prompts=ids, n_samples=n, seed=seed, pairs_per_batch=1, **kw)
    assert got.shape == (P, n, 3, T, *TINY_SIZE)
    for i, (a, b) in enumerate(pairs):
        ref = p.interpolate(torch.stack([a, b]), prompts=ids[i:i + 1], seed=seed + i, n_samples=n,
                            segments_per_batch=n, **kw)
        assert torch.equal(got[i], ref[:, 0]), f"pair {i} differs from its interpolate call"
    assert (got[0] - got[1]).abs().max().item() > 1e-2 * got.abs().max().item()
    # the default group holds all three pairs: the VAE encoder (6 images against 2), both towers and the UNet program
    # (12 rows against 4) all change batch size; 1.1 % of the output scale was measured on the H100 at DDIM-3, so this
    # is held to the 3 % bound test_video_length.py applies where three DDIM steps amplify a batch-size change
    batched = p.interpolate_pairs(pairs, prompts=ids, n_samples=n, seed=seed, **kw)
    _scale_close(batched, got, "interpolate_pairs default groups vs one pair per group", rel=3e-2)
    u8 = p.interpolate_pairs(pairs, prompts=ids, n_samples=n, seed=seed, pairs_per_batch=1, steps=steps,
                             size=TINY_SIZE)
    assert u8.shape == (P, n, T, *TINY_SIZE, 3) and u8.dtype == torch.uint8
    for i in range(P):
        assert torch.equal(u8[i].cpu(), torch.stack([joined_from_segments(got[i, v:v + 1], False) for v in range(n)]))


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("bad", [0, -1, 1.0, 2.5, True, False, "2", None])
def test_invalid_n_samples_are_refused_before_any_work(bad):
    """A model object with nothing but temporal_length is enough: the check comes before any work."""
    pipe = ToonCrafterPipeline(SimpleNamespace(temporal_length=16))
    for call in (lambda: pipe.interpolate_pairs([(None, None)], n_samples=bad),
                 lambda: check_n_samples(bad)):
        with pytest.raises(ValueError, match="n_samples"):
            call()
    if bad is not None:                       # None is the single-sample default of interpolate and animate
        with pytest.raises(ValueError, match="n_samples"):
            pipe.interpolate(None, n_samples=bad)
        with pytest.raises(ValueError, match="n_samples"):
            pipe.animate(None, n_samples=bad)
    assert [check_n_samples(n) for n in (1, 2, np.int64(8))] == [1, 2, 8]


@pytest.mark.parametrize("bad", [0, -1, True])
def test_invalid_rows_per_batch_are_refused_before_any_work(bad):
    """segments_per_batch of interpolate, animate and refine, and pairs_per_batch, with a model object that has
    nothing but temporal_length: the check comes before any work."""
    pipe = ToonCrafterPipeline(SimpleNamespace(temporal_length=16))
    for call in (lambda: pipe.interpolate(None, segments_per_batch=bad),
                 lambda: pipe.animate(None, segments_per_batch=bad),
                 lambda: pipe.refine([None] * 16, 0.5, segments_per_batch=bad)):
        with pytest.raises(ValueError, match="segments_per_batch must be an integer >= 1"):
            call()
    with pytest.raises(ValueError, match="pairs_per_batch must be an integer >= 1"):
        pipe.interpolate_pairs([(None, None)], pairs_per_batch=bad)
    assert [check_count(n, "pairs_per_batch") for n in (1, np.int64(3))] == [1, 3]


def test_interpolate_pairs_refuses_bad_arguments_before_any_work():
    pipe = ToonCrafterPipeline(SimpleNamespace(temporal_length=16))
    pairs = pair_list(2)
    with pytest.raises(ValueError, match="pairs"):
        pipe.interpolate_pairs([])
    with pytest.raises(ValueError, match="pairs"):
        pipe.interpolate_pairs([(pairs[0][0],)])
    with pytest.raises(ValueError, match="3 prompts for 2 pairs"):
        pipe.interpolate_pairs(pairs, prompts=["a", "b", "c"])
    with pytest.raises(ValueError, match="token ids"):
        pipe.interpolate_pairs(pairs, prompts=token_ids(3))
    with pytest.raises(ValueError, match="pairs_per_batch"):
        pipe.interpolate_pairs(pairs, pairs_per_batch=0)


def test_default_pairs_per_batch_keeps_the_rows_budget():
    assert [default_pairs_per_batch((320, 512), 16, n) for n in (1, 2, 3, 4, 8)] == [4, 2, 1, 1, 1]
    assert default_pairs_per_batch((320, 512), 8, 2) == 4 and default_pairs_per_batch((576, 1024), 16, 1) == 1


@pytest.mark.parametrize("first_stage,K,loop,output", [("dualref", 3, True, "uint8"), ("plain", 2, False, "float")])
def test_n_samples_none_and_one_are_the_same_bits_on_emulator(first_stage, K, loop, output):
    check_none_is_one(pipe_on(first_stage, "cpu"), K, loop, output)


@pytest.mark.parametrize("first_stage", ["dualref", "plain"])
def test_animate_variants_on_emulator(first_stage):
    check_animate_none_is_one(pipe_on(first_stage, "cpu"))


def test_variants_rng_contract_on_emulator():
    check_variants(pipe_on("dualref", "cpu"))


def test_interpolate_pairs_contract_on_emulator():
    check_pairs(pipe_on("dualref", "cpu"))


# ------------------------------------------------------------------------------ the directory reader (CPU, no GPU)
def _image(path, seed):
    from PIL import Image
    Image.fromarray(keyframes(1, (40, 56), seed=seed)[0].numpy()).save(path)


def make_prompt_dir(d, n_pairs=2, prompts=("a cat walks", "", "a dog runs"), extra_images=0):
    """prompts/512_interp's naming: <name>_frame1.png / <name>_frame3.png per pair and one prompts.txt (blank lines are
    skipped)."""
    d.mkdir(parents=True, exist_ok=True)
    names = [f"{chr(ord('a') + i)}{i}" for i in range(n_pairs + extra_images)]
    for i, name in enumerate(names[:n_pairs]):
        _image(d / f"{name}_frame1.png", 2 * i)
        _image(d / f"{name}_frame3.png", 2 * i + 1)
    for j, name in enumerate(names[n_pairs:]):
        _image(d / f"{name}_frame1.png", 100 + j)
    (d / "prompts.txt").write_text("\n".join(prompts) + "\n")
    return d


def test_prompt_dir_reader_follows_the_reference_layout(tmp_path):
    d = make_prompt_dir(tmp_path / "interp")
    (d / "zz_other.txt").write_text("never used\n")                  # only the first .txt by name is read
    pairs, prompts, names = read_prompt_dir(str(d))
    assert [(os.path.basename(a), os.path.basename(b)) for a, b in pairs] == [
        ("a0_frame1.png", "a0_frame3.png"), ("b1_frame1.png", "b1_frame3.png")]
    assert prompts == ["", ""] and names == ["a0_frame1", "b1_frame1"]
    assert read_prompt_dir(str(d), text_input=True)[1] == ["a cat walks", "a dog runs"]


def test_prompt_dir_reader_sorts_mixed_extensions_as_get_filelist(tmp_path):
    """Files of every suffix are collected and then sorted together: upper-case names and suffixes sort first (byte
    order), and a name with several dots is cut at the first one."""
    d = tmp_path / "mixed"
    d.mkdir()
    files = ["b.jpg", "B.PNG", "a.JPEG", "a.jpeg", "c.v2.png", "Z.png", "skip.gif", "skip.Jpg"]
    for i, f in enumerate(files):
        _image(d / f, i) if not f.endswith(("gif", "Jpg")) else (d / f).write_bytes(b"x")
    (d / "p.txt").write_text("one\ntwo\nthree\n")
    pairs, prompts, names = read_prompt_dir(str(d), text_input=True)
    order = sorted(files[:6])
    assert order == ["B.PNG", "Z.png", "a.JPEG", "a.jpeg", "b.jpg", "c.v2.png"]
    assert [tuple(os.path.basename(x) for x in p) for p in pairs] == [tuple(order[2 * i:2 * i + 2]) for i in range(3)]
    assert names == ["B", "a", "b"] and prompts == ["one", "two", "three"]


def test_prompt_dir_reader_rejects_bad_directories(tmp_path):
    d = make_prompt_dir(tmp_path / "short", n_pairs=1, prompts=("x", "y"))
    with pytest.raises(ValueError, match="2 images for 2 prompts"):
        read_prompt_dir(str(d))
    (d / "prompts.txt").unlink()
    with pytest.raises(ValueError, match="no prompt file"):
        read_prompt_dir(str(d))
    (d / "prompts.txt").write_text("\n  \n")
    with pytest.raises(ValueError, match="no prompts"):
        read_prompt_dir(str(d))
    with pytest.raises(ValueError, match="not a directory"):
        read_prompt_dir(str(tmp_path / "missing"))
    # an odd image left over is not used
    d2 = make_prompt_dir(tmp_path / "odd", n_pairs=2, prompts=("p", "q"), extra_images=1)
    assert len(read_prompt_dir(str(d2))[0]) == 2


def test_cli_arguments_of_n_samples_and_prompt_dir(tmp_path, capsys):
    base = ["--config", "c.yaml", "--out", "o", "--synthetic-weights"]
    args = get_parser().parse_args(base + ["--frames", "a.png", "b.png"])
    assert args.n_samples is None and args.prompt_dir is None and not args.text_input
    d = make_prompt_dir(tmp_path / "dir")
    args = get_parser().parse_args(base + ["--prompt-dir", str(d), "--n-samples", "3", "--text-input"])
    assert (args.prompt_dir, args.n_samples, args.text_input, args.frames) == (str(d), 3, True, None)
    refusals = [(["--frames", "a.png", "b.png", "--n-samples", "0"], "n_samples must be an integer >= 1"),
                (["--prompt-dir", str(d), "--loop"], "--loop does not apply to --prompt-dir"),
                (["--prompt-dir", str(d), "--prompt", "x"], "reads its prompts from the directory"),
                (["--frames", "a.png", "b.png", "--text-input"], "apply to --prompt-dir"),
                (["--frames", "a.png", "b.png", "--segments-per-batch", "0"], "segments_per_batch must be an integer"),
                (["--prompt-dir", str(d), "--pairs-per-batch", "0"], "pairs_per_batch must be an integer >= 1"),
                (["--prompt-dir", str(tmp_path / "none")], "not a directory"),
                (["--frames", "a.png", "--prompt-dir", str(d)], "not allowed with"),
                ([], "one of the arguments --frames --prompt-dir is required")]
    for extra, msg in refusals:
        with pytest.raises(SystemExit):
            main(base + extra)
        assert msg in capsys.readouterr().err, extra


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def cuda_tf32_off():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


@pytest.mark.gpu
@pytest.mark.parametrize("first_stage", ["dualref", "plain"])
def test_n_samples_equalities_on_gpu(cuda_tf32_off, first_stage):
    """The interpreter tests' equalities with the CUDA library, tiny config, both first stages, with and without
    loop, at DDIM-3."""
    p = pipe_on(first_stage, "cuda")
    for K, loop in ((3, False), (3, True)):
        for output in ("uint8", "float"):
            check_none_is_one(p, K, loop, output, steps=3)
    check_animate_none_is_one(p, steps=3)
    check_variants(p, steps=3)


@pytest.mark.gpu
def test_interpolate_pairs_contract_on_gpu(cuda_tf32_off):
    check_pairs(pipe_on("dualref", "cuda"), steps=3)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_full_width_batched_variants_match_one_variant_per_call(cuda_tf32_off):
    """Full-size synthetic weights at 320 x 512, K = 2, n = 4, DDIM-10: the four variants as the rows of one sample()
    call (the default, 4 rows) against one variant per call (segments_per_batch=1); the variants differ."""
    sys.path.insert(0, str(HERE.parent / "scripts"))
    from bench_pipeline import full_pipeline_config
    from tooncrafter_b200 import synthetic
    m = synthetic.synthetic_model(full_pipeline_config(), torch.device("cuda"))
    m.perframe_ae = True
    kf = [keyframes(1, (320, 512), seed=s)[0] for s in (7, 8)]
    pipe = ToonCrafterPipeline(m)
    kw = dict(steps=10, n_samples=4, output="float")
    batched = pipe.interpolate(kf, **kw).cpu()
    single = pipe.interpolate(kf, segments_per_batch=1, **kw).cpu()
    assert batched.shape == (4, 1, 3, 16, 320, 512) and torch.isfinite(batched).all()
    err = (batched - single).abs()
    print(f"full width n=4: batched vs one variant per call, max {err.max().item():.3e}, mean {err.mean().item():.3e}, "
          f"scale {single.abs().max().item():.3e}, bit-identical {torch.equal(batched, single)}")
    _scale_close(batched, single, "full width n=4 batched vs one variant per call")
    scale = single.abs().max().item()
    for v in range(1, 4):
        assert (batched[v] - batched[0]).abs().max().item() > 1e-2 * scale, f"variant {v} equals variant 0"


@pytest.mark.gpu
def test_cli_prompt_dir_writes_each_pair_and_sample(cuda_tf32_off, tmp_path):
    """--prompt-dir without --text-input on a generated directory, synthetic weights: one directory per (pair,
    sample), and every video.npy equal to its slice of interpolate_pairs on the same model, seed and groups."""
    import yaml
    from PIL import Image

    from test_pipeline import tiny_config
    from tooncrafter_b200 import synthetic
    from tooncrafter_b200.interpolate import rewrite_targets
    d = make_prompt_dir(tmp_path / "dir", n_pairs=3, prompts=("one", "two", "three"))
    cfg_path = tmp_path / "tiny.yaml"
    cfg_path.write_text(yaml.safe_dump({"model": tiny_config()}))
    out = tmp_path / "out"
    rc = main(["--config", str(cfg_path), "--synthetic-weights", "--prompt-dir", str(d), "--out", str(out),
               "--n-samples", "2", "--pairs-per-batch", "2", "--height", str(TINY_SIZE[0]), "--width",
               str(TINY_SIZE[1]), "--ddim-steps", "2", "--seed", "17"])
    assert rc == 0
    pairs, prompts, names = read_prompt_dir(str(d))
    assert sorted(p.name for p in out.iterdir()) == sorted(f"{nm}_sample{v}" for nm in names for v in range(2))
    m = synthetic.synthetic_model(rewrite_targets(tiny_config()), torch.device("cuda"), seed=0)
    m.perframe_ae = True
    images = [[np.asarray(Image.open(x).convert("RGB")) for x in p] for p in pairs]
    ref = ToonCrafterPipeline(m).interpolate_pairs(images, prompts=prompts, n_samples=2, steps=2, seed=17,
                                                   size=TINY_SIZE, pairs_per_batch=2).cpu().numpy()
    for i, nm in enumerate(names):
        for v in range(2):
            sub = out / f"{nm}_sample{v}"
            video = np.load(sub / "video.npy")
            assert video.shape == (T, *TINY_SIZE, 3) and video.dtype == np.uint8
            assert np.array_equal(video, ref[i, v]), (nm, v)
            assert sorted(x.name for x in sub.glob("frame_*.png")) == [f"frame_{f:04d}.png" for f in range(T)]

"""DPM-Solver++(2M) on the H100: tc_dpm_step / tc_dpm_step3 against an fp64 restatement, the order-1 identity with the
DDIM fused path bit for bit (tiny model and 320 x 512 with synthetic weights), convergence through tc_dpm_step against
the exact Gaussian solution, and the pipeline with sampler="dpmpp_2m", on one GPU and as two ranks sharing it."""
import sys
from pathlib import Path

import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from test_dpm_solver import (ORDER1_CASES, check_convergence, convergence_errors, run_update_loop,  # noqa: E402
                             sample_kwargs, sampler_pair, schedule_model, zero_weights)
from tiny_config import FULL_DDCONFIG, FULL_UNET, TINY_CONTEXT_DIM, TINY_LATENT_HW, TINY_T, model_config  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
RTOL, ATOL = 1e-3, 1e-4


@pytest.fixture(scope="module")
def ops():
    from tooncrafter_b200 import _lib, ops as ops_
    _lib.load()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return ops_


def _rand(*shape, seed, scale=1.0):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale).to(DEV)


def dpm_step_fp64(e_c, e_uc, e_img, x, noise, prev, coef):
    """tc_dpm_step* restated: the guidance combine and rescale in fp16 torch ops (one rounding per op, as the
    reference under autocast); the std ratio from fp64 sums of the fp16 values, rounded to fp16 like torch.std on fp16;
    then v -> (eps, x0), the DDIM update and + c * (x0 - prev) in fp64."""
    s, phi, sqrt_ac, sqrt_1mac, rescale, sqrt_aprev, dir_coef, sigma = [float(v) for v in coef[:8]]
    k = 8 if e_img is None else 9
    c = float(coef[k])
    v = e_uc + s * (e_c - e_uc) if e_img is None else e_uc + float(coef[8]) * (e_img - e_uc) + s * (e_c - e_img)
    if phi > 0:
        def std(t):
            d = t.double().flatten(1)
            n = d.shape[1]
            return ((d.pow(2).sum(1) - d.sum(1).pow(2) / n) / (n - 1)).clamp_min(0).sqrt().half()
        ratio = (std(e_c) / std(v)).view(-1, *([1] * (v.dim() - 1)))
        v = phi * (v * ratio) + (1 - phi) * v
    v, x, noise, prev = v.double(), x.double(), noise.double(), prev.double()
    eps = sqrt_ac * v + sqrt_1mac * x
    x0 = (sqrt_ac * x - sqrt_1mac * v) * rescale
    x_prev = sqrt_aprev * x0 + dir_coef * eps + sigma * noise
    return (x_prev + c * (x0 - prev) if c != 0.0 else x_prev), x0


def _violations(out, ref):
    return int(((out.double() - ref).abs() > ATOL + RTOL * ref.abs()).sum().item())


@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("three", [False, True], ids=["dpm_step", "dpm_step3"])
def test_dpm_step_matches_fp64_restatement(ops, three, B, phi):
    n = 4 * 16 * 40 * 64 + 77                                    # odd: a partial last block in every row
    e_c = _rand(B, n, seed=211).half()
    e_uc = (e_c.float() + 0.3 * _rand(B, n, seed=212)).half()
    e_img = (e_c.float() + 0.2 * _rand(B, n, seed=213)).half() if three else None
    x, noise, prev = _rand(B, n, seed=214), _rand(B, n, seed=215), _rand(B, n, seed=216, scale=0.8)
    coef_l = [7.5, phi, 0.6, 0.8, 0.98, 0.7, 0.3, 0.5] + ([2.5] if three else []) + [0.37]
    coef = torch.tensor(coef_l, device=DEV)
    x_prev, x0 = torch.full_like(x, float("nan")), torch.full_like(x, float("nan"))
    ws = torch.zeros(4 * B * ops.DDIM_PARTIALS, dtype=torch.float64, device=DEV)
    if three:
        ops.dpm_step3(e_c, e_uc, e_img, x, noise, prev, x_prev, x0, coef, ws, B=B, n=n)
    else:
        ops.dpm_step(e_c, e_uc, x, noise, prev, x_prev, x0, coef, ws, B=B, n=n)
    ref_prev, ref_x0 = dpm_step_fp64(e_c, e_uc, e_img, x, noise, prev, coef_l)
    for name, out, ref in (("pred_x0", x0, ref_x0), ("x_prev", x_prev, ref_prev)):
        err = (out.double() - ref).abs().max().item()
        print(f"{name} B={B} phi={phi} three={three}: max err {err:.3e}, violations {_violations(out, ref)}")
        assert _violations(out, ref) == 0, name


@pytest.mark.parametrize("three", [False, True], ids=["dpm_step", "dpm_step3"])
def test_zero_weight_dpm_step_is_the_ddim_step_and_leaves_prev_unread(ops, three):
    B, n = 2, 4 * 16 * 40 * 64 + 3
    e_c = _rand(B, n, seed=221).half()
    e_uc = (e_c.float() + 0.3 * _rand(B, n, seed=222)).half()
    e_img = (e_c.float() + 0.2 * _rand(B, n, seed=223)).half()
    x, noise = _rand(B, n, seed=224), _rand(B, n, seed=225)
    nan = torch.full_like(x, float("nan"))
    head = [7.5, 0.7, 0.6, 0.8, 0.98, 0.7, 0.3, 0.5] + ([2.5] if three else [])
    ws = torch.zeros(4 * B * ops.DDIM_PARTIALS, dtype=torch.float64, device=DEV)
    outs = [torch.empty_like(x) for _ in range(4)]
    if three:
        ops.ddim_step3(e_c, e_uc, e_img, x, noise, outs[0], outs[1], torch.tensor(head, device=DEV), ws, B=B, n=n)
        ops.dpm_step3(e_c, e_uc, e_img, x, noise, nan, outs[2], outs[3], torch.tensor(head + [0.0], device=DEV), ws,
                      B=B, n=n)
    else:
        ops.ddim_step(e_c, e_uc, x, noise, outs[0], outs[1], torch.tensor(head, device=DEV), ws, B=B, n=n)
        ops.dpm_step(e_c, e_uc, x, noise, nan, outs[2], outs[3], torch.tensor(head + [0.0], device=DEV), ws, B=B, n=n)
    assert torch.equal(outs[0], outs[2]) and torch.equal(outs[1], outs[3])


def test_dpm_step_refuses_aliased_pred_x0(ops):
    from tooncrafter_b200._lib import TcError
    x = torch.zeros(1, 64, device=DEV)
    e = x.half()
    ws = torch.zeros(4 * ops.DDIM_PARTIALS, dtype=torch.float64, device=DEV)
    n0 = ops.launch_count()
    with pytest.raises(TcError):
        ops.dpm_step(e, e, x, x, x, torch.empty_like(x), x, torch.zeros(9, device=DEV), ws, B=1, n=64)
    assert ops.launch_count() == n0


@pytest.mark.parametrize("s", [1.0, 2.0])
def test_convergence_through_tc_dpm_step(ops, s):
    m = schedule_model()
    m.use_dynamic_rescale = False
    run = lambda order2: lambda S: run_update_loop(ops.ddim_step, ops.dpm_step, m, s, order2, S, device=DEV)
    ddim, dpm = convergence_errors(run(False), m, s), convergence_errors(run(True), m, s)
    print(f"s={s}: DDIM {ddim}, DPM++(2M) {dpm}")
    check_convergence(ddim, dpm)


# ------------------------------------------------------------------------------------------------ order-1 identity
def _inputs(T, h, w, ctx_dim, seed=3):
    from tooncrafter_b200 import synthetic
    x_T, cond, uncond = synthetic.synthetic_inputs(1, T, h, w, ctx_dim, seed=seed)
    _, uimg, _ = synthetic.synthetic_inputs(1, T, h, w, ctx_dim, seed=seed + 1)
    return x_T, cond, uncond, {"c_crossattn": uimg["c_crossattn"], "c_concat": cond["c_concat"]}


def _order1_equal(m, inputs, three, mask, t_start, eta):
    ddim_cls, dpm_cls = sampler_pair(three)
    outs = []
    for cls in (ddim_cls, dpm_cls):
        s = zero_weights(cls(m)) if cls is dpm_cls else cls(m)
        kw = sample_kwargs(*inputs, three, eta, mask, t_start, device=DEV)
        outs.append(s.sample(**kw)[0])
        outs.append(torch.stack([torch.randn(2, generator=g, device=DEV) for g in kw["noise_generators"]]))
    return torch.equal(outs[0], outs[2]) and torch.equal(outs[1], outs[3])


@pytest.fixture(scope="module")
def tiny_gpu_model():
    from tooncrafter_b200 import diffusion, synthetic
    m = diffusion.instantiate_from_config(model_config())
    synthetic.fill_module_(m, seed=1234)
    m = m.to(DEV).eval()
    m.perframe_ae = True
    return m


@pytest.mark.parametrize("eta", [0.0, 1.0])
@pytest.mark.parametrize(**ORDER1_CASES)
def test_order1_identity_tiny(ops, tiny_gpu_model, three, mask, t_start, eta):
    inputs = _inputs(TINY_T, *TINY_LATENT_HW, TINY_CONTEXT_DIM)
    assert _order1_equal(tiny_gpu_model, inputs, three, mask, t_start, eta)


@pytest.fixture(scope="module")
def full_model():
    from tooncrafter_b200 import diffusion, synthetic
    with torch.device("meta"):
        sk = diffusion.instantiate_from_config(model_config(FULL_UNET, FULL_DDCONFIG))
    m = sk.to_empty(device=DEV)
    m.reset_schedule_buffers()
    with torch.no_grad():
        for k, p in m.named_parameters():
            p.copy_(synthetic.synthetic_tensor(k, tuple(p.shape), 1234).to(DEV))
    m.perframe_ae = True
    m.temporal_length = 16
    return m.eval()


@pytest.mark.parametrize("eta", [0.0, 1.0])
@pytest.mark.parametrize(**ORDER1_CASES)
def test_order1_identity_320x512(ops, full_model, three, mask, t_start, eta):
    inputs = _inputs(16, 40, 64, 1024)
    assert _order1_equal(full_model, inputs, three, mask, t_start, eta)


# ------------------------------------------------------------------------------------------------ pipeline
def test_pipeline_dpm_solver_on_the_gpu(ops):
    from test_pipeline import TINY_SIZE, keyframes, tiny_model
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    pipe = ToonCrafterPipeline(tiny_model(DEV))
    kf = keyframes(3, seed=51)
    kw = dict(steps=6, seed=60, size=TINY_SIZE, output="float", eta=0.0)
    dpm = pipe.interpolate(kf, sampler="dpmpp_2m", loop=True, **kw)
    ddim, default = pipe.interpolate(kf, sampler="ddim", loop=True, **kw), pipe.interpolate(kf, loop=True, **kw)
    assert torch.equal(ddim, default)
    assert dpm.shape == ddim.shape and torch.isfinite(dpm).all() and (dpm - ddim).abs().max().item() > 1e-4
    one = pipe.interpolate(kf, sampler="dpmpp_2m", loop=True, segments_per_batch=1, **kw)
    pair = pipe.interpolate(kf[1:3], sampler="dpmpp_2m", segments_per_batch=1, **dict(kw, seed=61))
    assert torch.equal(one[1], pair[0])
    u8 = pipe.refine(keyframes(TINY_T, seed=12), 0.75, keep=[0, TINY_T - 1], sampler="dpmpp_2m", n_samples=2,
                     steps=6, seed=8, size=TINY_SIZE, eta=1.0)
    assert u8.shape == (2, TINY_T, *TINY_SIZE, 3)


def _two_ranks_worker(rank, world):
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from test_pipeline import TINY_SIZE, keyframes, tiny_model
        from tooncrafter_b200.pipeline import ToonCrafterPipeline
        m = tiny_model(DEV)
        kw = dict(steps=5, seed=60, size=TINY_SIZE, segments_per_batch=1, output="float", sampler="dpmpp_2m", eta=0.0)
        got = ToonCrafterPipeline(m, dist.group.WORLD).interpolate(keyframes(3, seed=51), **kw)
        ref = ToonCrafterPipeline(m).interpolate(keyframes(3, seed=51), **kw)
        return bool(got.shape == ref.shape and torch.equal(got, ref))
    finally:
        dist.destroy_process_group()


def test_two_ranks_on_one_gpu_give_the_single_process_result(ops):
    from distributed_harness import spawn
    assert all(spawn(_two_ranks_worker, world=2).values())

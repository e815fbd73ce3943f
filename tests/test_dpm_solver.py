"""DPM-Solver++(2M) (tooncrafter_b200.sampler.DPMSolverSampler / DPMSolverSamplerMultiCond, pipeline sampler=
"dpmpp_2m") on the CPU: the correction-weight table against an independent float64 statement of the definition, the
order-1 identity with DDIM on the program interpreter, convergence against the exact probability-flow solution for
Gaussian data, both sampler paths against an fp64 restatement on the tiny model, and the pipeline and command line."""
import math
import os
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))

from tiny_config import TINY_CONTEXT_DIM, TINY_LATENT_HW, TINY_T, model_config  # noqa: E402

from oracle import ddim_oracle  # noqa: E402
from tooncrafter_b200 import diffusion, ops, runtime, synthetic  # noqa: E402
from tooncrafter_b200.sampler import (DDIMSampler, DDIMSamplerMultiCond, DPMSolverSampler,  # noqa: E402
                                      DPMSolverSamplerMultiCond)

SEED = 1234
CFG_IMG = 2.5


# ------------------------------------------------------------------------------------------------ shared helpers
def emulated_dpm_step(e_c, e_uc, x, noise, prev_pred_x0, x_prev, pred_x0, coef, ws, *, B, n, e_img=None):
    """ops.dpm_step on the CPU interpreter: ops_emulator's DDIM update, then the correction in fp32, one rounding per
    op, skipped where its weight is 0 (tc_dpm_step's contract)."""
    import ops_emulator
    k = 8 if e_img is None else 9
    ops_emulator.ddim_step(e_c, e_uc, x, noise, x_prev, pred_x0, coef[:k], ws, B=B, n=n, e_img=e_img)
    c = float(coef[k])
    if c != 0.0:
        xp = x_prev.reshape(B, n)
        xp.copy_(xp + c * (pred_x0.reshape(B, n) - prev_pred_x0.reshape(B, n)))


def emulated_dpm_step3(e_c, e_uc, e_img, x, noise, prev_pred_x0, x_prev, pred_x0, coef, ws, *, B, n):
    emulated_dpm_step(e_c, e_uc, x, noise, prev_pred_x0, x_prev, pred_x0, coef, ws, B=B, n=n, e_img=e_img)


@pytest.fixture
def dpm_emulator(monkeypatch):
    """The program interpreter with entries for ops.dpm_step / ops.dpm_step3."""
    import ops_emulator
    monkeypatch.setitem(ops_emulator._TABLE, "dpm_step", emulated_dpm_step)
    monkeypatch.setitem(ops_emulator._TABLE, "dpm_step3", emulated_dpm_step3)
    return ops_emulator.executor


def reference_weights(alphas, alphas_prev, eta):
    """c for every DDIM index from the definition, through logs: lambda = log(alpha) - log(sigma), h = lambda' - lambda,
    r = h(index + 1) / h(index); 0 where the predecessor (index + 1) has lambda = -inf, and for index S - 1."""
    a, ap = [float(v) for v in alphas], [float(v) for v in alphas_prev]
    lam = lambda v: (0.5 * math.log(v) - 0.5 * math.log1p(-v)) if v > 0 else -math.inf
    h = [lam(ap[k]) - lam(a[k]) for k in range(len(a))]
    out = []
    for k in range(len(a)):
        if k == len(a) - 1 or lam(a[k + 1]) == -math.inf:
            out.append(0.0)
            continue
        r = h[k + 1] / h[k]
        decay = math.exp(-h[k]) if eta == 0 else math.exp(-2.0 * h[k])
        out.append(math.sqrt(ap[k]) * (1.0 - decay) / (2.0 * r))
    return out


def schedule_model():
    """The tiny model's schedule (the 512 config's: linear betas, zero terminal SNR, dynamic rescale) on meta weights."""
    with torch.device("meta"):
        m = diffusion.instantiate_from_config(model_config())
    m = m.to_empty(device="cpu")
    m.reset_schedule_buffers()
    return m


def gaussian_v_model(m, s):
    """apply_model of the exact denoiser for data N(0, s^2): v = alpha*eps - sigma*x0 with E[x0|x] = alpha s^2 x / d,
    E[eps|x] = sigma x / d, d = alpha^2 s^2 + sigma^2 (alpha, sigma: the model's fp32 buffers, evaluated in fp64)."""
    def apply_model(x, t, c, **kw):
        al = m.sqrt_alphas_cumprod[t].double().view(-1, *([1] * (x.dim() - 1)))
        sg = m.sqrt_one_minus_alphas_cumprod[t].double().view_as(al)
        d = al * al * s * s + sg * sg
        return (al * sg * (1.0 - s * s) * x.double() / d).to(x.dtype)
    return apply_model


def exact_gain(m, s):
    """x_end / x_T along the probability-flow ODE from t = 999 to the last step's target alphas_cumprod[0]."""
    a_T, a_0 = float(m.alphas_cumprod[999].double()), float(m.alphas_cumprod[0].double())
    return math.sqrt(a_0 * s * s + 1.0 - a_0) / math.sqrt(a_T * s * s + 1.0 - a_T)


def convergence_errors(run, m, s, steps=(20, 40, 80)):
    """{steps: max |x_end - exact| / max |exact|} for run(S) -> (x_T, x_end)."""
    out = {}
    for S in steps:
        x_T, x_end = run(S)
        exact = exact_gain(m, s) * x_T.double()
        out[S] = ((x_end.double() - exact).abs().max() / exact.abs().max()).item()
    return out


def check_convergence(ddim, dpm):
    """DPM++(2M) falls by >= 2.5x per doubling, DDIM by <= 2.1x, and DPM++ is below DDIM at 40 and 80 steps."""
    for a, b in ((20, 40), (40, 80)):
        assert dpm[a] / dpm[b] >= 2.5, (dpm, ddim)
        assert ddim[a] / ddim[b] <= 2.1, (dpm, ddim)
    assert dpm[40] < ddim[40] and dpm[80] < ddim[80], (dpm, ddim)


def dpm_update_fp64(x, v, noise, prev, co, c):
    """One step in fp64 from the guided (and rescaled) v: DDIM's update (ddim_oracle.ddim_update's formula), then
    + c * (x0 - prev) (prev None: c must be 0).  Returns (x_prev, x0)."""
    eps = co["sqrt_ac"] * v + co["sqrt_1mac"] * x
    x0 = (co["sqrt_ac"] * x - co["sqrt_1mac"] * v) * co["rescale"]
    x_prev = co["sqrt_aprev"] * x0 + co["dir_coef"] * eps + co["sigma"] * noise
    return (x_prev if prev is None else x_prev + c * (x0 - prev)), x0


# ------------------------------------------------------------------------------------------------ coefficient table
@pytest.mark.parametrize("eta", [0, 1])
@pytest.mark.parametrize("S", [2, 3, 10, 25, 50])
@pytest.mark.parametrize("spacing", ["uniform_trailing", "uniform"])
def test_order2_weights_match_the_definition(spacing, S, eta):
    m = schedule_model()
    sched = ddim_oracle.model_schedule()
    assert torch.equal(m.alphas_cumprod.float(), sched["alphas_cumprod"])
    s = DPMSolverSampler(m)
    if spacing == "uniform" and len(range(0, 1000, 1000 // S)) != S:
        with pytest.raises(IndexError):        # the reference's "uniform" steps reach t = 1000 here (S = 3)
            s.make_schedule(S, spacing, eta, verbose=False)
        return
    s.make_schedule(S, spacing, eta, verbose=False)
    got = s.order2_weights()
    tab = ddim_oracle.ddim_tables(sched, S, eta, spacing)
    want = reference_weights(tab["alphas"], tab["alphas_prev"], eta)
    assert np.isfinite(got).all()
    for k in range(S):
        first_order = k == S - 1 or float(tab["alphas"][k + 1]) == 0.0
        if first_order:
            assert got[k] == 0.0, (k, got[k])
        else:
            assert got[k] != 0.0 and math.isclose(got[k], want[k], rel_tol=1e-9, abs_tol=0.0), (k, got[k], want[k])
    if spacing == "uniform_trailing":        # t = 999 runs first at alpha = 0, so its successor is first order too
        assert got[S - 2] == 0.0
    # the fused path's column: the first step that runs is first order, whatever its index (t_start)
    for start in range(S):
        col = s._order2_coefficients(list(range(start, -1, -1)))
        assert col[0] == 0.0 and col[1:] == [float(got[k]) for k in range(start - 1, -1, -1)]


def test_eta_other_than_0_or_1_is_refused():
    m = schedule_model()
    for eta in (0.5, -1.0, 2.0, True):
        with pytest.raises(ValueError, match="eta 0 or 1"):
            DPMSolverSampler(m).make_schedule(10, "uniform_trailing", eta, verbose=False)
        with pytest.raises(ValueError, match="eta 0 or 1"):
            DPMSolverSamplerMultiCond(m).sample(S=10, batch_size=1, shape=[4, TINY_T, 2, 2], eta=eta, verbose=False)
    DPMSolverSampler(m).make_schedule(10, "uniform_trailing", 1.0, verbose=False)
    DPMSolverSampler(m).make_schedule(10, "uniform_trailing", 0, verbose=False)


# ------------------------------------------------------------------------------------------------ convergence
def run_general(m, s, sampler_cls, S):
    m.apply_model = gaussian_v_model(m, s)
    x_T = torch.randn(1, 4, TINY_T, 2, 2, generator=torch.Generator().manual_seed(5))
    out, _ = sampler_cls(m).sample(S=S, batch_size=1, shape=list(x_T.shape[1:]), eta=0.0, x_T=x_T,
                                   timestep_spacing="uniform_trailing", verbose=False)
    return x_T, out


@pytest.mark.parametrize("s", [1.0, 2.0])
def test_convergence_to_the_exact_solution_on_the_general_path(s):
    """Gaussian data N(0, s^2): the exact denoiser makes the probability-flow ODE linear with a closed-form solution.
    Dynamic rescale off, eta 0, zero-SNR schedule, uniform_trailing; cfg 1 (no guidance) is the general path."""
    m = schedule_model()
    m.use_dynamic_rescale = False
    ddim = convergence_errors(lambda S: run_general(m, s, DDIMSampler, S), m, s)
    dpm = convergence_errors(lambda S: run_general(m, s, DPMSolverSampler, S), m, s)
    print(f"s={s}: DDIM {ddim}, DPM++(2M) {dpm}")
    check_convergence(ddim, dpm)


def run_update_loop(ddim_step, dpm_step, m, s, order2, S, device="cpu"):
    """The fused update alone, driven with the Gaussian denoiser of gaussian_v_model: e_c = e_uc = v in fp16 (so the
    guidance combine returns v), phi 0, eta 0, the fused path's coefficient table.  ddim_step / dpm_step: ops.* or
    their emulations.  Returns (x_T, x_end)."""
    smp = (DPMSolverSampler if order2 else DDIMSampler)(m)
    smp.make_schedule(S, "uniform_trailing", 0.0, verbose=False)
    steps = [(S - 1 - i, int(t)) for i, t in enumerate(np.flip(smp.ddim_timesteps))]
    c2 = smp._order2_coefficients([k for k, _ in steps]) if order2 else None
    table = torch.tensor([smp.step_coefficients(k, 7.5, 0.0) + ([c2[i]] if order2 else []) for i, (k, _) in
                          enumerate(steps)], dtype=torch.float32, device=device)
    x_T = torch.randn(1, 4, TINY_T, 8, 8, generator=torch.Generator().manual_seed(5))
    x = x_T.to(device, copy=True)
    n = x.numel()
    x_next, pred, prev = torch.empty_like(x), torch.empty_like(x), torch.zeros_like(x)
    noise = torch.zeros_like(x)
    ws = torch.empty(4 * ops.DDIM_PARTIALS, dtype=torch.float64, device=device)
    apply = gaussian_v_model(m, s)
    for i, (_, t) in enumerate(steps):
        v = apply(x.cpu(), torch.tensor([t]), None).half().to(device)
        if order2:
            pred, prev = prev, pred
            dpm_step(v, v, x, noise, prev, x_next, pred, table[i], ws, B=1, n=n)
        else:
            ddim_step(v, v, x, noise, x_next, pred, table[i], ws, B=1, n=n)
        x, x_next = x_next, x
    return x_T, x.cpu()


@pytest.mark.parametrize("s", [1.0, 2.0])
def test_convergence_through_the_fused_update_on_the_interpreter(s):
    """As above, through the fused update's arithmetic (fp16 v) on the CPU interpreter; the GPU test runs tc_dpm_step."""
    import ops_emulator
    m = schedule_model()
    m.use_dynamic_rescale = False
    run = lambda order2: lambda S: run_update_loop(ops_emulator.ddim_step, emulated_dpm_step, m, s, order2, S)
    ddim, dpm = convergence_errors(run(False), m, s), convergence_errors(run(True), m, s)
    print(f"s={s}: DDIM {ddim}, DPM++(2M) {dpm}")
    check_convergence(ddim, dpm)


# ------------------------------------------------------------------------------------------------ tiny model
_TINY = {}


def tiny_unet_model():
    """The tiny model with seeded synthetic weights and its UNet engine on the program interpreter (cached)."""
    if "m" not in _TINY:
        from tooncrafter_b200.engine import UNetEngine
        m = diffusion.instantiate_from_config(model_config())
        synthetic.fill_module_(m, seed=SEED)
        m = m.eval()
        unet = m.model.diffusion_model
        unet._engine = UNetEngine(unet, device="cpu", plan_only=True)
        _TINY["m"] = m
    return _TINY["m"]


def tiny_inputs(b=1, seed=3):
    h, w = TINY_LATENT_HW
    x_T, cond, uncond = synthetic.synthetic_inputs(b, TINY_T, h, w, TINY_CONTEXT_DIM, seed=seed)
    _, uimg, _ = synthetic.synthetic_inputs(b, TINY_T, h, w, TINY_CONTEXT_DIM, seed=seed + 1)
    uimg = {"c_crossattn": uimg["c_crossattn"], "c_concat": cond["c_concat"]}
    return x_T, cond, uncond, uimg


def sample_kwargs(x_T, cond, uncond, uimg, three, eta, mask=False, t_start=None, S=4, device="cpu"):
    """sample()'s keywords for one tiny-model case; three: three-way guidance; mask: frames 0 and T-1 held to x0."""
    b = x_T.shape[0]
    to = lambda c: {k: [t.to(device) for t in v] for k, v in c.items()}
    kw = dict(S=S, batch_size=b, shape=list(x_T.shape[1:]), conditioning=to(cond), unconditional_conditioning=to(uncond),
              eta=eta, unconditional_guidance_scale=7.5, x_T=x_T.to(device), fs=torch.tensor([10] * b, device=device),
              timestep_spacing="uniform_trailing", guidance_rescale=0.7, verbose=False,
              noise_generators=[torch.Generator(device=device).manual_seed(40 + r) for r in range(b)])
    if three:
        kw.update(cfg_img=CFG_IMG, unconditional_conditioning_img_nonetext=to(uimg))
    if mask:
        T = x_T.shape[2]
        mk = torch.zeros(1, 1, T, 1, 1, device=device)
        mk[:, :, [0, T - 1]] = 1.0
        x0 = torch.randn(x_T.shape, generator=torch.Generator().manual_seed(9)).to(device)
        kw.update(mask=mk, x0=x0)
    if t_start is not None:
        kw["t_start"] = t_start
    return kw


def sampler_pair(three):
    return (DDIMSamplerMultiCond, DPMSolverSamplerMultiCond) if three else (DDIMSampler, DPMSolverSampler)


ORDER1_CASES = dict(argnames="three,mask,t_start",
                    argvalues=[(False, False, None), (True, False, None), (False, True, None), (True, True, 3),
                               (False, False, 3)],
                    ids=["two_way", "three_way", "two_way_mask", "three_way_mask_t_start", "two_way_t_start"])


def zero_weights(s):
    s.order2_weights = lambda: np.zeros(len(s.ddim_timesteps))
    return s


@pytest.mark.parametrize("eta", [0.0, 1.0])
@pytest.mark.parametrize(**ORDER1_CASES)
def test_order1_fused_step_is_the_ddim_step_on_the_interpreter(dpm_emulator, three, mask, t_start, eta):
    """With every weight forced to 0 the fused DPM path (tc_dpm_step*, its table column, its buffer swap) gives the
    DDIM fused path's result bit for bit, noise streams included."""
    m = tiny_unet_model()
    inputs = tiny_inputs()
    ddim_cls, dpm_cls = sampler_pair(three)
    outs = []
    for cls in (ddim_cls, dpm_cls):
        s = zero_weights(cls(m)) if cls is dpm_cls else cls(m)
        s._test_executor = dpm_emulator
        kw = sample_kwargs(*inputs, three, eta, mask, t_start)
        outs.append(s.sample(**kw)[0])
        outs.append(torch.stack([torch.randn(2, generator=g) for g in kw["noise_generators"]]))   # stream position
    assert torch.equal(outs[0], outs[2]) and torch.equal(outs[1], outs[3])


def fp64_dpm_sample(m, x_T, cond, uncond, uimg, three, eta, S, gens_seed, phi=0.7):
    """The sampler restated in fp64 torch from the definition: the tiny oracle UNet (fp32, as the oracle computes it),
    then guidance, rescale, DDIM update and the correction with reference_weights in fp64; the step noise drawn as
    sample() draws it (one generator per row)."""
    from oracle import unet_oracle
    from tooncrafter_b200 import layout
    from tiny_config import TINY_UNET
    sched = ddim_oracle.model_schedule()
    tab = ddim_oracle.ddim_tables(sched, S, eta)
    w = reference_weights(tab["alphas"], tab["alphas_prev"], eta)
    sd = {k: v for k, v in m.state_dict().items() if k.startswith("model.diffusion_model.")}
    lay = layout.unet_layout(TINY_UNET)
    gens = [torch.Generator().manual_seed(gens_seed + r) for r in range(x_T.shape[0])]
    x, prev = x_T.double(), None
    fs = torch.tensor([10] * x.shape[0])
    for i, step in enumerate(np.flip(tab["timesteps"])):
        index = S - i - 1
        ts = torch.full((x.shape[0],), int(step), dtype=torch.long)
        es = [unet_oracle.unet_forward(sd, lay, torch.cat([x.float()] + c["c_concat"], 1), ts,
                                       torch.cat(c["c_crossattn"], 1), fs, "model.diffusion_model.").double()
              for c in ((cond, uncond, uimg) if three else (cond, uncond))]
        if three:
            v = es[1] + CFG_IMG * (es[2] - es[1]) + 7.5 * (es[0] - es[2])
        else:
            v = es[1] + 7.5 * (es[0] - es[1])
        v = ddim_oracle.rescale_noise_cfg(v, es[0], phi)
        noise = torch.stack([torch.randn(tuple(x.shape[1:]), generator=g) for g in gens]).double()
        co = ddim_oracle.step_coefficients(sched, tab, index)
        x, prev = dpm_update_fp64(x, v, noise, prev, co, w[index])
    return x


@pytest.mark.parametrize("eta", [0.0, 1.0])
@pytest.mark.parametrize("three", [False, True], ids=["two_way", "three_way"])
def test_fused_and_general_paths_match_fp64_restatement(dpm_emulator, three, eta):
    """6 steps (uniform_trailing: 4 second-order steps) on the tiny model: the fused path on the interpreter and the
    general path (three or two UNet passes through the same interpreted engine) within test_sampler_cpu.py's 3 %."""
    m = tiny_unet_model()
    unet = m.model.diffusion_model
    inputs = tiny_inputs()
    S = 6
    ref = fp64_dpm_sample(m, *inputs, three, eta, S, gens_seed=40)
    cls = sampler_pair(three)[1]
    s = cls(m)
    s._test_executor = dpm_emulator
    fused = s.sample(**sample_kwargs(*inputs, three, eta, S=S))[0]
    kw = sample_kwargs(*inputs, three, eta, S=S)
    real = unet.forward
    unet.forward = lambda x, t, context=None, fs=None, **k: unet._engine.forward(x, t, context, fs,
                                                                                 executor=dpm_emulator).clone()
    try:
        kw["precision"] = None
        general = cls(m)
        general._fast_path_ok = lambda *a, **k: False
        general = general.sample(**kw)[0]
    finally:
        unet.forward = real
    scale = ref.abs().max().item()
    for name, out in (("fused", fused), ("general", general)):
        err = (out.double() - ref).abs().max().item()
        print(f"{name}: max err {err:.3e} of scale {scale:.3e}")
        assert err < 3e-2 * scale, (name, err, scale)
    ddim = zero_weights(cls(m))
    ddim._test_executor = dpm_emulator
    first = ddim.sample(**sample_kwargs(*inputs, three, eta, S=S))[0]
    assert (first - fused).abs().max().item() > 1e-3 * scale, "the correction changed nothing"


# ------------------------------------------------------------------------------------------------ pipeline
_PIPE = {}


def _pipe_run(method, *args, **kw):
    """One pipeline call on the tiny model of test_pipeline.py through the CPU program interpreter (cached)."""
    import clip_emulator
    import ops_emulator
    from test_pipeline import TINY_SIZE, tiny_model
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    key = (method, repr(args), tuple(sorted((k, repr(v)) for k, v in kw.items())))
    if key not in _PIPE:
        if "model" not in _PIPE:
            _PIPE["model"] = tiny_model()
        saved = {k: ops_emulator._TABLE.get(k) for k in ("dpm_step", "dpm_step3")}
        ops_emulator._TABLE.update(dpm_step=emulated_dpm_step, dpm_step3=emulated_dpm_step3)
        runtime.TEST_EXECUTOR = clip_emulator.executor
        try:
            pipe = ToonCrafterPipeline(_PIPE["model"])
            _PIPE[key] = getattr(pipe, method)(*args, size=TINY_SIZE, **kw)
        finally:
            runtime.TEST_EXECUTOR = None
            for k, v in saved.items():
                if v is None:
                    ops_emulator._TABLE.pop(k, None)
                else:
                    ops_emulator._TABLE[k] = v
    return _PIPE[key]


def _kf(K, seed=11):
    from test_pipeline import keyframes
    return keyframes(K, seed=seed)


# name -> (call, eta); steps=3 under uniform_trailing: the last step is second order
PIPELINE_CASES = {
    "k3_loop": (lambda **kw: _pipe_run("interpolate", _kf(3), steps=3, loop=True, seed=5, segments_per_batch=1, **kw),
                0.0),
    "n_samples": (lambda **kw: _pipe_run("interpolate", _kf(2), steps=3, seed=6, n_samples=2, **kw), 1.0),
    "animate": (lambda **kw: _pipe_run("animate", _kf(1, seed=4)[0], steps=3, seed=7, **kw), 0.0),
    "refine_keep": (lambda **kw: _pipe_run("refine", _kf(TINY_T, seed=12), 1.0, keep=[0, TINY_T - 1], steps=3, seed=8,
                                           **kw), 1.0),
    "pairs": (lambda **kw: _pipe_run("interpolate_pairs", [(a, b) for a, b in _kf(4, seed=13).view(2, 2, *_kf(1).shape[1:])],
                                     n_samples=1, steps=3, seed=9, **kw), 0.0),
}


@pytest.mark.parametrize("case", sorted(PIPELINE_CASES))
def test_pipeline_runs_dpm_solver(case):
    """Every public method takes sampler="dpmpp_2m": DDIM's shape, finite, and different from DDIM's result."""
    call, eta = PIPELINE_CASES[case]
    dpm = call(sampler="dpmpp_2m", eta=eta, output="float")
    ddim = call(sampler="ddim", eta=eta, output="float")
    assert dpm.shape == ddim.shape and torch.isfinite(dpm).all()
    assert (dpm - ddim).abs().max().item() > 1e-4


def test_ddim_keyword_is_the_default():
    call, eta = PIPELINE_CASES["animate"]
    assert torch.equal(call(sampler="ddim", output="float", eta=eta), call(output="float", eta=eta))


def test_rng_contract_holds_for_dpm_solver():
    """Segment 1 of the K = 3 loop is the K = 2 run on keyframes (1, 2) with seed + 1 (per-row generators), up to the
    towers' and the encoder's other batches: 2 % of the output scale (DDIM on the same case at eta 0 differs by 0.8 %,
    DPM++(2M) by 1.1 %)."""
    from test_pipeline import _scale_close
    call, eta = PIPELINE_CASES["k3_loop"]
    three = call(sampler="dpmpp_2m", eta=eta, output="float")
    pair = _pipe_run("interpolate", _kf(3)[1:3], steps=3, seed=6, segments_per_batch=1, output="float",
                     sampler="dpmpp_2m", eta=eta)
    _scale_close(three[1], pair[0], "dpmpp_2m: segment 1 of K=3 vs K=2 on its pair", rel=2e-2)
    assert (three[0] - pair[0]).abs().max().item() > 1e-2, "different segments gave the same video"


@pytest.mark.parametrize("bad", [dict(sampler="unipc"), dict(sampler="dpmpp_2m", eta=0.5),
                                 dict(sampler="DDIM"), dict(sampler=None)])
def test_bad_sampler_arguments_raise_before_any_launch(bad):
    from test_pipeline import TINY_SIZE, tiny_model
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    if "model" not in _PIPE:
        _PIPE["model"] = tiny_model()
    pipe = ToonCrafterPipeline(_PIPE["model"])
    kw = dict(dict(eta=1.0), **bad)
    n0 = ops.launch_count()
    calls = [lambda: pipe.interpolate(_kf(2), steps=4, size=TINY_SIZE, **kw),
             lambda: pipe.animate(_kf(1)[0], steps=4, size=TINY_SIZE, **kw),
             lambda: pipe.refine(_kf(TINY_T), 0.5, steps=4, size=TINY_SIZE, **kw),
             lambda: pipe.interpolate_pairs([(_kf(2)[0], _kf(2)[1])], steps=4, size=TINY_SIZE, **kw)]
    for call in calls:
        with pytest.raises(ValueError):
            call()
    assert ops.launch_count() == n0


def test_command_line_refuses_bad_sampler_arguments(capsys):
    from tooncrafter_b200 import interpolate
    base = ["--config", "x.yaml", "--frames", "a.png", "b.png", "--out", "o", "--synthetic-weights"]
    for extra, msg in ((["--sampler", "euler"], "sampler must be one of"),
                       (["--sampler", "dpmpp_2m", "--ddim-eta", "0.3"], "eta 0 or 1")):
        with pytest.raises(SystemExit) as e:
            interpolate.main(base + extra)
        assert e.value.code == 2 and msg in capsys.readouterr().err
    assert interpolate.get_parser().parse_args(base).sampler == "ddim"


# ------------------------------------------------------------------------------------------------ two gloo ranks
def _sharded_worker(rank, world):
    import torch.distributed as dist

    import clip_emulator
    import ops_emulator
    from test_pipeline import TINY_SIZE, keyframes, tiny_model
    from tooncrafter_b200.pipeline import ToonCrafterPipeline
    torch.set_num_threads(max(1, (os.cpu_count() or 2) // world))
    ops_emulator._TABLE.update(dpm_step=emulated_dpm_step, dpm_step3=emulated_dpm_step3)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        runtime.TEST_EXECUTOR = clip_emulator.executor
        m = tiny_model()
        call = lambda pipe: pipe.interpolate(keyframes(3, seed=31), steps=3, seed=3, size=TINY_SIZE, eta=0.0,
                                             segments_per_batch=1, output="float", sampler="dpmpp_2m").numpy()
        res = {"sharded": call(ToonCrafterPipeline(m, dist.group.WORLD))}
        if rank == 0:
            res["single"] = call(ToonCrafterPipeline(m))
        return res
    finally:
        runtime.TEST_EXECUTOR = None
        dist.destroy_process_group()


def test_two_gloo_ranks_give_the_single_process_result():
    from distributed_harness import spawn
    got = spawn(_sharded_worker, world=2)
    single = got[0]["single"]
    for r in range(2):
        assert np.array_equal(got[r]["sharded"], single), r

"""DDIMSampler with the reference's public API (lvdm/models/samplers/ddim.py:10-279), H100-native inside.

Fast path (the configuration scripts/run.sh uses: v-parameterisation, classifier-free guidance with a conditioning
dict, no corrector / quantiser, with or without mask / x0): per step ONE batched UNet program replay (cond and uncond
rows as B = 2b, CUDA graph) + ONE fused DDIM-update launch pair (tc_ddim_step: CFG combine in fp16 like ddim.py:226,
per-sample std reductions, guidance rescale, v -> eps / x0, dynamic rescale, x_prev) with the step coefficients taken
from a device table — no per-step `.item()` synchronisation, no materialised torch.full tensors.  With a mask, one
tc_q_sample launch per step blends the noised x0 in before the replay (ddim.py:172-180).

Any other option combination falls back to the general path below, which follows the reference control flow with
torch elementwise plumbing around `model.apply_model` (still the CUDA UNet engine).
"""
from __future__ import annotations

import numpy as np
import torch

from . import ops


def make_ddim_timesteps(method, num_ddim, num_ddpm, verbose=False):
    """lvdm/models/utils_diffusion.py:56-76."""
    if method == "uniform":
        steps = np.asarray(list(range(0, num_ddpm, num_ddpm // num_ddim))) + 1
    elif method == "uniform_trailing":
        steps = np.flip(np.round(np.arange(num_ddpm, 0, -(num_ddpm / num_ddim)))).astype(np.int64) - 1
    elif method == "quad":
        steps = ((np.linspace(0, np.sqrt(num_ddpm * 0.8), num_ddim)) ** 2).astype(int) + 1
    else:
        raise NotImplementedError(f'There is no ddim discretization method called "{method}"')
    if verbose:
        print(f"Selected timesteps for ddim sampler: {steps}")
    return steps


def make_ddim_sampling_parameters(alphacums, ddim_timesteps, eta, verbose=False):
    """lvdm/models/utils_diffusion.py:79-91 (alphas fp32 tensor, alphas_prev float64 ndarray, sigmas float64)."""
    alphas = alphacums[ddim_timesteps]
    alphas_prev = np.asarray([alphacums[0]] + alphacums[ddim_timesteps[:-1]].tolist())
    sigmas = eta * np.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
    return sigmas, alphas, alphas_prev


def randn_rows(shape, device, generators=None):
    """torch.randn(shape) or, with one torch.Generator per batch row, each row drawn from its own generator (so a row's
    noise does not depend on which batch it runs in)."""
    if generators is None:
        return torch.randn(shape, device=device)
    if len(generators) != shape[0]:
        raise ValueError(f"noise_generators: {len(generators)} generators for {shape[0]} batch rows")
    return torch.stack([torch.randn(tuple(shape[1:]), generator=g, device=device) for g in generators])


def rescale_noise_cfg(noise_cfg, noise_pred_text, guidance_rescale=0.0):
    dims = list(range(1, noise_pred_text.ndim))
    factor = noise_pred_text.std(dim=dims, keepdim=True) / noise_cfg.std(dim=dims, keepdim=True)
    return guidance_rescale * (noise_cfg * factor) + (1 - guidance_rescale) * noise_cfg


class DDIMSampler(object):
    def __init__(self, model, schedule="linear", **kwargs):
        super().__init__()
        # optional: a 2-rank torch.distributed group (distributed.latency_pairs()); the fused path then evaluates one
        # guidance branch per rank and all-gathers the two predictions every step
        self.latency_group = None
        # tests only: interpret the engine's recorded programs and the fused update on the PyTorch emulator (no GPU)
        from . import runtime
        self._test_executor = runtime.TEST_EXECUTOR
        self.model = model
        self.ddpm_num_timesteps = model.num_timesteps
        self.schedule = schedule
        self.counter = 0

    def register_buffer(self, name, attr):
        if isinstance(attr, torch.Tensor) and attr.device != self.model.device:
            attr = attr.to(self.model.device)
        setattr(self, name, attr)

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0.0, verbose=True):
        m = self.model
        self.ddim_timesteps = make_ddim_timesteps(ddim_discretize, ddim_num_steps, self.ddpm_num_timesteps, verbose)
        ac = m.alphas_cumprod
        assert ac.shape[0] == self.ddpm_num_timesteps, "alphas have to be defined for each timestep"
        f32 = lambda x: x.clone().detach().to(torch.float32).to(m.device)
        if m.use_dynamic_rescale:
            self.ddim_scale_arr = m.scale_arr[self.ddim_timesteps]
            self.ddim_scale_arr_prev = torch.cat([self.ddim_scale_arr[0:1], self.ddim_scale_arr[:-1]])
        self.register_buffer("betas", f32(m.betas))
        self.register_buffer("alphas_cumprod", f32(ac))
        self.register_buffer("alphas_cumprod_prev", f32(m.alphas_cumprod_prev))
        acc = ac.cpu()
        self.register_buffer("sqrt_alphas_cumprod", f32(np.sqrt(acc)))
        self.register_buffer("sqrt_one_minus_alphas_cumprod", f32(np.sqrt(1.0 - acc)))
        with np.errstate(divide="ignore"):
            self.register_buffer("log_one_minus_alphas_cumprod", f32(np.log(1.0 - acc)))
            self.register_buffer("sqrt_recip_alphas_cumprod", f32(np.sqrt(1.0 / acc)))
            self.register_buffer("sqrt_recipm1_alphas_cumprod", f32(np.sqrt(1.0 / acc - 1)))
        sig, al, alp = make_ddim_sampling_parameters(acc, self.ddim_timesteps, ddim_eta, verbose)
        self.register_buffer("ddim_sigmas", sig)
        self.register_buffer("ddim_alphas", al)
        self.register_buffer("ddim_alphas_prev", alp)
        self.register_buffer("ddim_sqrt_one_minus_alphas", np.sqrt(1.0 - al))
        with np.errstate(divide="ignore", invalid="ignore"):
            s0 = ddim_eta * torch.sqrt((1 - self.alphas_cumprod_prev) / (1 - self.alphas_cumprod) *
                                       (1 - self.alphas_cumprod / self.alphas_cumprod_prev))
        self.register_buffer("ddim_sigmas_for_original_num_steps", s0)

    # -------------------------------------------------------------------------------------------- public API
    @torch.no_grad()
    def sample(self, S, batch_size, shape, conditioning=None, callback=None, normals_sequence=None,
               img_callback=None, quantize_x0=False, eta=0.0, mask=None, x0=None, temperature=1.0,
               noise_dropout=0.0, score_corrector=None, corrector_kwargs=None, verbose=True, schedule_verbose=False,
               x_T=None, log_every_t=100, unconditional_guidance_scale=1.0, unconditional_conditioning=None,
               precision=None, fs=None, timestep_spacing="uniform", guidance_rescale=0.0, **kwargs):
        """Reference signature, plus two keywords of this library:

        noise_generators: None (the global RNG, as the reference) or one torch.Generator per batch row on the model's
        device, from which that row's x_T (when not given) and every step's DDIM noise are drawn; with `mask` (and
        not clean_cond) also each step's q_sample noise of x0, drawn before that step's DDIM noise.

        t_start: None, or k in 1 .. S: run only the last k DDIM steps (indices k-1 .. 0) from `x_T`, which is then
        required (the SDEdit pair with stochastic_encode at DDIM index k-1; `decode` is this for the reference)."""
        noise_generators = kwargs.pop("noise_generators", None)
        t_start = kwargs.pop("t_start", None)
        if t_start is not None:
            if isinstance(t_start, bool) or not isinstance(t_start, (int, np.integer)) or not 1 <= t_start <= S:
                raise ValueError(f"t_start must be an integer from 1 to S={S}, got {t_start!r}")
            if x_T is None:
                raise ValueError("t_start needs x_T: the latent to continue from")
            kwargs["t_start"] = int(t_start)
        if conditioning is not None:
            first = conditioning[list(conditioning.keys())[0]] if isinstance(conditioning, dict) else conditioning
            cbs = (first[0] if isinstance(first, (list, tuple)) else first).shape[0]
            if cbs != batch_size:
                print(f"Warning: Got {cbs} conditionings but batch-size is {batch_size}")
        self.make_schedule(ddim_num_steps=S, ddim_discretize=timestep_spacing, ddim_eta=eta, verbose=schedule_verbose)
        size = (batch_size, *shape)
        return self.ddim_sampling(conditioning, size, callback=callback, img_callback=img_callback,
                                  quantize_denoised=quantize_x0, mask=mask, x0=x0, ddim_use_original_steps=False,
                                  noise_dropout=noise_dropout, temperature=temperature,
                                  score_corrector=score_corrector, corrector_kwargs=corrector_kwargs, x_T=x_T,
                                  log_every_t=log_every_t, unconditional_guidance_scale=unconditional_guidance_scale,
                                  unconditional_conditioning=unconditional_conditioning, verbose=verbose,
                                  precision=precision, fs=fs, guidance_rescale=guidance_rescale,
                                  noise_generators=noise_generators, **kwargs)

    @torch.no_grad()
    def stochastic_encode(self, x0, t, use_original_steps=False, noise=None):
        """ddim.py:303-318: x0 noised to the level of per-row index t, a long tensor [B] of DDIM indices (of the last
        make_schedule), or of DDPM timesteps with use_original_steps.  noise None: torch.randn_like(x0).  A CUDA fp32
        x0 goes through tc_q_sample (the same fp32 arithmetic, bit for bit)."""
        if use_original_steps:
            sqrt_ac, sqrt_1mac = self.sqrt_alphas_cumprod, self.sqrt_one_minus_alphas_cumprod
        else:
            sqrt_ac, sqrt_1mac = torch.sqrt(self.ddim_alphas), self.ddim_sqrt_one_minus_alphas
        if noise is None:
            noise = torch.randn_like(x0)
        t = torch.as_tensor(t, device=sqrt_ac.device)
        if not (x0.is_cuda and x0.dtype == torch.float32 and noise.dtype == torch.float32):
            size = (t.shape[0],) + (1,) * (x0.dim() - 1)
            return sqrt_ac.gather(-1, t).reshape(size) * x0 + sqrt_1mac.gather(-1, t).reshape(size) * noise
        B = x0.shape[0]
        if t.shape != (B,):
            raise ValueError(f"stochastic_encode: t must hold one index per row, [{B}], got {tuple(t.shape)}")
        coef = torch.stack([sqrt_ac.gather(-1, t), sqrt_1mac.gather(-1, t)], 1).to(x0.device, torch.float32)
        x0c = x0.contiguous()
        out = torch.empty_like(x0c)
        ops.q_sample(out, x0c, noise.expand(x0.shape).contiguous(), None, coef.reshape(-1), B=B, n=x0c[0].numel())
        return out

    @torch.no_grad()
    def decode(self, x_latent, cond, t_start, unconditional_guidance_scale=1.0, unconditional_conditioning=None,
               use_original_steps=False, callback=None):
        """ddim.py:282-300: the last t_start steps of the last make_schedule's DDIM schedule (of the DDPM schedule with
        use_original_steps) from x_latent, without fs (the model's default_fs) or guidance rescale.  Runs on the fused
        path under the same conditions as sample()."""
        img, _ = self.ddim_sampling(cond, tuple(x_latent.shape), x_T=x_latent,
                                    ddim_use_original_steps=use_original_steps, callback=callback,
                                    unconditional_guidance_scale=unconditional_guidance_scale,
                                    unconditional_conditioning=unconditional_conditioning, verbose=False,
                                    t_start=t_start)
        return img

    def _fast_path_ok(self, cond, uc, cfg_scale, mask, quantize, corrector, noise_dropout, precision, orig_steps,
                      shape, kwargs=None):
        m = self.model
        unet = getattr(getattr(m, "model", None), "diffusion_model", None)
        return (m.parameterization == "v" and uc is not None and cfg_scale != 1.0 and isinstance(cond, dict)
                and isinstance(uc, dict) and not quantize and corrector is None
                and noise_dropout == 0.0 and precision is None and not orig_steps and len(shape) == 5
                and getattr(m.model, "conditioning_key", None) == "hybrid" and hasattr(unet, "layout")
                and (m.device.type == "cuda" or getattr(self, "_test_executor", None) is not None))

    @torch.no_grad()
    def ddim_sampling(self, cond, shape, x_T=None, ddim_use_original_steps=False, callback=None, timesteps=None,
                      quantize_denoised=False, mask=None, x0=None, img_callback=None, log_every_t=100,
                      temperature=1.0, noise_dropout=0.0, score_corrector=None, corrector_kwargs=None,
                      unconditional_guidance_scale=1.0, unconditional_conditioning=None, verbose=True,
                      precision=None, fs=None, guidance_rescale=0.0, noise_generators=None, t_start=None, **kwargs):
        device = self.model.betas.device
        b = shape[0]
        img = randn_rows(shape, device, noise_generators) if x_T is None else x_T
        if precision == 16:
            img = img.to(dtype=torch.float16)
        if timesteps is None:
            timesteps = self.ddpm_num_timesteps if ddim_use_original_steps else self.ddim_timesteps
        elif not ddim_use_original_steps:
            subset_end = int(min(timesteps / self.ddim_timesteps.shape[0], 1) * self.ddim_timesteps.shape[0]) - 1
            timesteps = self.ddim_timesteps[:subset_end]
        if t_start is not None:                          # the last t_start steps only (ddim.py:284-287)
            timesteps = min(timesteps, t_start) if ddim_use_original_steps else timesteps[:t_start]
        intermediates = {"x_inter": [img], "pred_x0": [img]}
        time_range = reversed(range(0, timesteps)) if ddim_use_original_steps else np.flip(timesteps)
        total_steps = timesteps if ddim_use_original_steps else timesteps.shape[0]
        clean_cond = kwargs.pop("clean_cond", False)

        if self._fast_path_ok(cond, unconditional_conditioning, unconditional_guidance_scale, mask,
                              quantize_denoised, score_corrector, noise_dropout, precision,
                              ddim_use_original_steps, shape, kwargs):
            return self._sample_fused(self._guidance_branches(cond, unconditional_conditioning, kwargs), img,
                                      list(time_range), total_steps, unconditional_guidance_scale, guidance_rescale,
                                      temperature, fs, callback, img_callback, log_every_t, intermediates,
                                      cfg_img=self._cfg_img(unconditional_guidance_scale, kwargs),
                                      noise_generators=noise_generators, mask=mask, x0=x0, clean_cond=clean_cond)

        for i, step in enumerate(time_range):
            index = total_steps - i - 1
            ts = torch.full((b,), int(step), device=device, dtype=torch.long)
            if mask is not None:
                assert x0 is not None
                if clean_cond:
                    img_orig = x0
                else:
                    q_noise = None if noise_generators is None else randn_rows(x0.shape, device, noise_generators)
                    img_orig = self.model.q_sample(x0, ts, noise=q_noise)
                img = img_orig * mask + (1.0 - mask) * img
            img, pred_x0 = self.p_sample_ddim(img, cond, ts, index=index, use_original_steps=ddim_use_original_steps,
                                              quantize_denoised=quantize_denoised, temperature=temperature,
                                              noise_dropout=noise_dropout, score_corrector=score_corrector,
                                              corrector_kwargs=corrector_kwargs,
                                              unconditional_guidance_scale=unconditional_guidance_scale,
                                              unconditional_conditioning=unconditional_conditioning, mask=mask, x0=x0,
                                              fs=fs, guidance_rescale=guidance_rescale,
                                              noise_generators=noise_generators, **kwargs)
            if callback:
                callback(i)
            if img_callback:
                img_callback(pred_x0, i)
            if index % log_every_t == 0 or index == total_steps - 1:
                intermediates["x_inter"].append(img)
                intermediates["pred_x0"].append(pred_x0)
        return img, intermediates

    # -------------------------------------------------------------------------------------------- fused fast path
    def _guidance_branches(self, cond, uc, kwargs):
        """Conditioning dicts evaluated per step, in the row order of the batched UNet program: [cond, uncond]."""
        return [cond, uc]

    def _cfg_img(self, cfg_scale, kwargs):
        return None

    def step_coefficients(self, index, cfg_scale, phi, temperature=1.0):
        """The 8 scalars of tc_ddim_step for DDIM index `index`, evaluated in the reference's op order / precision
        (ddim.py:251-254,263-264,271; fp32 torch.full tensors)."""
        one = lambda v: torch.full((1,), float(v), dtype=torch.float32)
        t = int(self.ddim_timesteps[index])
        a_prev, sigma = one(self.ddim_alphas_prev[index]), one(self.ddim_sigmas[index])
        if self.model.use_dynamic_rescale:
            rescale = float(one(self.ddim_scale_arr_prev[index]) / one(self.ddim_scale_arr[index]))
        else:
            rescale = 1.0
        return [float(cfg_scale), float(phi), float(self.model.sqrt_alphas_cumprod[t]),
                float(self.model.sqrt_one_minus_alphas_cumprod[t]), rescale, float(a_prev.sqrt()),
                float((1.0 - a_prev - sigma ** 2).sqrt()), float(sigma) * float(temperature)]

    def _fused_setup(self, cond, uc, shape, steps, cfg_scale, phi, temperature, fs, extra_branches=(), cfg_img=None,
                     q_coefficients=False):
        """Everything of the fused path that is per-`sample()` call: engine / plan lookup, conditioning K/V program,
        concat channels, fps, and the device tables of per-step coefficients.  `steps` = [(ddim index, t), ...] in
        execution order.  `extra_branches`: further conditioning dicts batched after [cond, uncond] (the multi-condition
        sampler's image-without-text branch, with `cfg_img`).  q_coefficients: each table row also holds, from column
        st.q_off, tc_q_sample's per-row pair (sqrt_alphas_cumprod[t], sqrt_one_minus_alphas_cumprod[t]) for the b rows
        (the masked blend of ddpm3d.py:306-309).  Returns the state `_fused_step` consumes."""
        from .engine import _P
        m = self.model
        dev = m.device
        unet = m.model.diffusion_model
        from .engine import UNetEngine
        ex = getattr(self, "_test_executor", None)
        eng = UNetEngine.cached(unet, "_engine", ex)
        b, c, T, H, W = shape
        group = getattr(self, "latency_group", None)
        if group is not None:
            # latency mode: this rank evaluates ONE guidance branch (pair-rank 0: conditional, 1: unconditional)
            import torch.distributed as dist
            branch = dist.get_rank(group)
            mine = cond if branch == 0 else uc
            ctx = torch.cat(mine["c_crossattn"], 1)
            cc = torch.cat(mine["c_concat"], 1)
            nb = b
        else:
            branches = [cond, uc, *extra_branches]
            ctx = torch.cat([torch.cat(c_["c_crossattn"], 1) for c_ in branches], 0)
            cc = torch.cat([torch.cat(c_["c_concat"], 1) for c_ in branches], 0)
            nb = len(branches) * b
        plan = eng.plan_for(nb, T, H, W, ctx.shape[1])
        eng.set_context(plan, ctx, ex)                  # always re-run: a new prompt must never see old K/V
        plan.x_in[:, c:].copy_(cc)
        if eng.lay.fs_condition:
            if fs is None:
                plan.fs_in.fill_(float(eng.lay.default_fs))
            else:
                f = torch.as_tensor(fs, device=dev).to(torch.float32).reshape(-1)
                plan.fs_in.copy_(torch.cat([f.expand(b)] * (nb // b)))
        st = _P(eng=eng, plan=plan, ex=ex, group=group, b=b, c=c, nb=nb, n=c * T * H * W, dev=dev,
                three=len(extra_branches) == 1)
        if len(extra_branches) > 1 or (extra_branches and group is not None):
            raise NotImplementedError("fused path: at most one extra guidance branch, not in latency mode")
        tail = [float(cfg_img)] if st.three else []
        order2 = self._order2_coefficients([index for index, _ in steps])
        st.order2 = order2 is not None
        st.q_off = 8 + len(tail) + st.order2
        q = lambda t: ([float(m.sqrt_alphas_cumprod[t]), float(m.sqrt_one_minus_alphas_cumprod[t])] * b
                       if q_coefficients else [])
        c2 = lambda i: [order2[i]] if st.order2 else []
        st.coef_table = torch.tensor([self.step_coefficients(index, cfg_scale, phi, temperature) + tail + c2(i) +
                                      q(int(t)) for i, (index, t) in enumerate(steps)], dtype=torch.float32, device=dev)
        st.t_table = torch.tensor([float(t) for _, t in steps], dtype=torch.float32, device=dev)
        st.ws = torch.empty(4 * b * ops.DDIM_PARTIALS, dtype=torch.float64, device=dev)
        if group is not None:
            st.e_all = torch.empty((2 * b,) + tuple(plan.y_out.shape[1:]), dtype=plan.y_out.dtype, device=dev)
        return st

    def _order2_coefficients(self, indices):
        """None for DDIM; a second-order sampler returns the weight of its correction term for each step of `indices`
        (DDIM indices in execution order), which the fused update reads from the table column after cfg_img."""
        return None

    def _fused_step(self, st, i, x, noise, x_next, pred_x0, prev_pred_x0=None):
        """One DDIM step (row i of the tables): batched UNet program replay + the fused update.  Writes x_next and
        pred_x0; afterwards st.plan.y_out still holds the two UNet predictions of this step.  prev_pred_x0: the previous
        step's pred_x0, read by the second-order update (st.order2)."""
        plan, b, c = st.plan, st.b, st.c
        for r in range(st.nb // b):                                          # the same latent under every branch
            plan.x_in[r * b:(r + 1) * b, :c].copy_(x)
        plan.t_in.copy_(st.t_table[i].expand(st.nb))
        st.eng._execute(plan.main, st.ex, st.eng.use_graph)
        e_img = None
        if st.group is None:
            y = plan.y_out
            e_c, e_uc = y[:b], y[b:2 * b]
            if st.three:
                e_img = y[2 * b:3 * b]
        else:
            from .distributed import pair_all_gather
            pair_all_gather(st.e_all, plan.y_out, st.group)                      # the step's only exchange (2 x 327 KB)
            e_c, e_uc = st.e_all[:b], st.e_all[b:]
        if st.order2:
            fn, args = ((ops.dpm_step3, (e_c, e_uc, e_img, x, noise, prev_pred_x0, x_next, pred_x0, st.coef_table[i],
                                         st.ws)) if st.three
                        else (ops.dpm_step, (e_c, e_uc, x, noise, prev_pred_x0, x_next, pred_x0, st.coef_table[i],
                                             st.ws)))
        else:
            fn, args = ((ops.ddim_step3, (e_c, e_uc, e_img, x, noise, x_next, pred_x0, st.coef_table[i], st.ws))
                        if st.three else (ops.ddim_step, (e_c, e_uc, x, noise, x_next, pred_x0, st.coef_table[i], st.ws)))
        if st.ex is None:
            fn(*args, B=b, n=st.n)
        else:
            st.ex(fn, args, dict(B=b, n=st.n))

    def _sample_fused(self, branches, img, time_range, total_steps, cfg_scale, phi, temperature, fs, callback,
                      img_callback, log_every_t, intermediates, cfg_img=None, noise_generators=None, mask=None,
                      x0=None, clean_cond=False):
        steps = [(total_steps - i - 1, time_range[i]) for i in range(total_steps)]
        st = self._fused_setup(branches[0], branches[1], tuple(img.shape), steps, cfg_scale, phi, temperature, fs,
                               extra_branches=tuple(branches[2:]), cfg_img=cfg_img,
                               q_coefficients=mask is not None and not clean_cond)
        x = img.to(torch.float32).contiguous().clone()
        x_next = torch.empty_like(x)
        pred_x0 = torch.empty_like(x)
        # second order: the update reads the previous step's pred_x0 from one buffer and writes into the other
        prev_pred_x0 = torch.zeros_like(x) if st.order2 else None
        if mask is not None:
            assert x0 is not None
            # expanded once per call; the blend is then one tc_q_sample launch per step
            mask = mask.to(device=st.dev, dtype=torch.float32).expand(x.shape).contiguous()
            x0 = x0.to(device=st.dev, dtype=torch.float32).expand(x.shape).contiguous()
        if st.group is not None:
            from .distributed import sync_pair_state
            # same x_T on both ranks, and the same noise: from pair-rank 0's global RNG stream, or from the per-row
            # generators, which both ranks seed alike
            sync_pair_state(x, st.group, rng_state=noise_generators is None)
        for i, (index, _) in enumerate(steps):
            if mask is not None:                                            # ddim.py:172-180, before the UNet
                q_noise = None if clean_cond else randn_rows(x.shape, st.dev, noise_generators)
                args = (x, x0, q_noise, mask, None if clean_cond else st.coef_table[i, st.q_off:])
                kw = dict(B=st.b, n=st.n, clean=bool(clean_cond))
                if st.ex is None:
                    ops.q_sample(*args, **kw)
                else:
                    st.ex(ops.q_sample, args, kw)
            noise = randn_rows(x.shape, st.dev, noise_generators)          # one draw per step, as ddim.py:273
            if prev_pred_x0 is not None:
                pred_x0, prev_pred_x0 = prev_pred_x0, pred_x0
            self._fused_step(st, i, x, noise, x_next, pred_x0, prev_pred_x0)
            x, x_next = x_next, x
            if callback:
                callback(i)
            if img_callback:
                img_callback(pred_x0, i)
            if index % log_every_t == 0 or index == total_steps - 1:
                intermediates["x_inter"].append(x.clone())
                intermediates["pred_x0"].append(pred_x0.clone())
        return x, intermediates

    # -------------------------------------------------------------------------------------------- general path
    @torch.no_grad()
    def p_sample_ddim(self, x, c, t, index, repeat_noise=False, use_original_steps=False, quantize_denoised=False,
                      temperature=1.0, noise_dropout=0.0, score_corrector=None, corrector_kwargs=None,
                      unconditional_guidance_scale=1.0, unconditional_conditioning=None, uc_type=None,
                      conditional_guidance_scale_temporal=None, mask=None, x0=None, guidance_rescale=0.0,
                      noise_generators=None, **kwargs):
        m = self.model
        b, device = x.shape[0], x.device
        if unconditional_conditioning is None or unconditional_guidance_scale == 1.0:
            model_output = m.apply_model(x, t, c, **kwargs)
        else:
            if not isinstance(c, (torch.Tensor, dict)):
                raise NotImplementedError
            e_c = m.apply_model(x, t, c, **kwargs).clone()
            e_uc = m.apply_model(x, t, unconditional_conditioning, **kwargs)
            model_output = e_uc + unconditional_guidance_scale * (e_c - e_uc)
            if guidance_rescale > 0.0:
                model_output = rescale_noise_cfg(model_output, e_c, guidance_rescale=guidance_rescale)
        return self._ddim_update(x, t, index, model_output, c, repeat_noise, use_original_steps, quantize_denoised,
                                 temperature, noise_dropout, score_corrector, corrector_kwargs, noise_generators)

    def _ddim_update(self, x, t, index, model_output, c, repeat_noise, use_original_steps, quantize_denoised,
                     temperature, noise_dropout, score_corrector, corrector_kwargs, noise_generators=None):
        """ddim.py:231-277: v -> (eps, x0), dynamic rescale, x_{t-1}; noise_generators: see sample()."""
        m = self.model
        b, device = x.shape[0], x.device
        e_t = m.predict_eps_from_z_and_v(x, t, model_output) if m.parameterization == "v" else model_output
        if score_corrector is not None:
            assert m.parameterization == "eps", "not implemented"
            e_t = score_corrector.modify_score(m, e_t, x, t, c, **corrector_kwargs)
        alphas = m.alphas_cumprod if use_original_steps else self.ddim_alphas
        alphas_prev = m.alphas_cumprod_prev if use_original_steps else self.ddim_alphas_prev
        sqrt_1ma = m.sqrt_one_minus_alphas_cumprod if use_original_steps else self.ddim_sqrt_one_minus_alphas
        sigmas = self.ddim_sigmas_for_original_num_steps if use_original_steps else self.ddim_sigmas
        size = (b,) + (1,) * (x.dim() - 1)
        full = lambda v: torch.full(size, float(v), device=device)
        a_t, a_prev, sigma_t, s1ma = full(alphas[index]), full(alphas_prev[index]), full(sigmas[index]), full(sqrt_1ma[index])
        if m.parameterization != "v":
            pred_x0 = (x - s1ma * e_t) / a_t.sqrt()
        else:
            pred_x0 = m.predict_start_from_z_and_v(x, t, model_output)
        if m.use_dynamic_rescale:
            pred_x0 = pred_x0 * (full(self.ddim_scale_arr_prev[index]) / full(self.ddim_scale_arr[index]))
        if quantize_denoised:
            pred_x0, _, *_ = m.first_stage_model.quantize(pred_x0)
        dir_xt = (1.0 - a_prev - sigma_t ** 2).sqrt() * e_t
        if repeat_noise:
            gens = None if noise_generators is None else noise_generators[:1]
            nz = randn_rows((1, *x.shape[1:]), device, gens).repeat(b, *((1,) * (x.dim() - 1)))
        else:
            nz = randn_rows(x.shape, device, noise_generators)
        noise = sigma_t * nz * temperature
        if noise_dropout > 0.0:
            noise = torch.nn.functional.dropout(noise, p=noise_dropout)
        return a_prev.sqrt() * pred_x0 + dir_xt + noise, pred_x0


class DDIMSamplerMultiCond(DDIMSampler):
    """lvdm/models/samplers/ddim_multiplecond.py:10-320 — three-way guidance (text / image-without-text / uncond):
    v = e_uc + cfg_img * (e_img - e_uc) + s * (e_c - e_img)  (:229-234).

    Fused path (same option set as DDIMSampler's): the three branches run as ONE B = 3b UNet program per step and
    tc_ddim_step3 does the three-way combine, guidance rescale and update.  Other option combinations take the
    general path below: three passes through the CUDA UNet engine + torch elementwise plumbing."""

    def _fast_path_ok(self, cond, uc, cfg_scale, mask, quantize, corrector, noise_dropout, precision, orig_steps,
                      shape, kwargs=None):
        img_uc = (kwargs or {}).get("unconditional_conditioning_img_nonetext")
        return (isinstance(img_uc, dict) and self.latency_group is None and
                super()._fast_path_ok(cond, uc, cfg_scale, mask, quantize, corrector, noise_dropout, precision,
                                      orig_steps, shape, kwargs))

    def _guidance_branches(self, cond, uc, kwargs):
        return [cond, uc, kwargs["unconditional_conditioning_img_nonetext"]]

    def _cfg_img(self, cfg_scale, kwargs):
        v = kwargs.get("cfg_img")
        return float(cfg_scale if v is None else v)

    @torch.no_grad()
    def p_sample_ddim(self, x, c, t, index, repeat_noise=False, use_original_steps=False, quantize_denoised=False,
                      temperature=1.0, noise_dropout=0.0, score_corrector=None, corrector_kwargs=None,
                      unconditional_guidance_scale=1.0, unconditional_conditioning=None, uc_type=None, cfg_img=None,
                      mask=None, x0=None, guidance_rescale=0.0, noise_generators=None, **kwargs):
        m = self.model
        cfg_img = unconditional_guidance_scale if cfg_img is None else cfg_img
        uc_img = kwargs["unconditional_conditioning_img_nonetext"]
        if unconditional_conditioning is None or unconditional_guidance_scale == 1.0:
            model_output = m.apply_model(x, t, c, **kwargs)
        else:
            e_c = m.apply_model(x, t, c, **kwargs).clone()
            e_uc = m.apply_model(x, t, unconditional_conditioning, **kwargs).clone()
            e_img = m.apply_model(x, t, uc_img, **kwargs)
            model_output = e_uc + cfg_img * (e_img - e_uc) + unconditional_guidance_scale * (e_c - e_img)
            if guidance_rescale > 0.0:
                model_output = rescale_noise_cfg(model_output, e_c, guidance_rescale=guidance_rescale)
        return self._ddim_update(x, t, index, model_output, c, repeat_noise, use_original_steps, quantize_denoised,
                                 temperature, noise_dropout, score_corrector, corrector_kwargs, noise_generators)


def check_dpm_eta(eta) -> float:
    """DPM-Solver++(2M) is defined for eta 0 (the ODE solver) and eta 1 (its SDE form): its first-order step is the DDIM
    step with that eta, and no other eta has such a counterpart."""
    if isinstance(eta, bool) or eta not in (0, 1):
        raise ValueError(f"DPM-Solver++(2M) takes eta 0 or 1, got {eta!r}")
    return float(eta)


class _DPMSolverPP2M:
    """DPM-Solver++(2M) in data-prediction form, as the DDIM step plus one correction (INTEGRATION.md):

        x' = DDIM_eta(x, p_i) + c_i * (p_i - p_{i-1}),   p_i = pred_x0 of step i (after the dynamic rescale)

    With a = ddim_alphas[index], a' = ddim_alphas_prev[index], alpha = sqrt(a), sigma = sqrt(1 - a),
    lambda = log(alpha / sigma) and h_i = lambda' - lambda:  c_i = alpha' (1 - e^{-h_i}) / (2 r_i) for eta 0,
    alpha' (1 - e^{-2 h_i}) / (2 r_i) for eta 1, with r_i = h_{i-1} / h_i.  c_i = 0 (a DDIM step) on the first step that
    runs and on a step whose predecessor started at lambda = -inf (zero terminal SNR).  The noise draws are DDIM's, so
    either sampler consumes a generator's stream alike.  Works on the fused path (tc_dpm_step*) and the general path."""

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform", ddim_eta=0.0, verbose=True):
        self.dpm_eta = check_dpm_eta(ddim_eta)
        super().make_schedule(ddim_num_steps, ddim_discretize, ddim_eta, verbose)

    def order2_weights(self) -> np.ndarray:
        """float64 [S] of the last make_schedule: entry k is c of a step at DDIM index k whose predecessor ran at index
        k + 1; 0 for index S - 1 and wherever that predecessor has alpha = 0.  Always finite."""
        a = self.ddim_alphas.detach().double().cpu().numpy()
        ap = np.asarray(self.ddim_alphas_prev, dtype=np.float64)
        al, sg, alp, sgp = np.sqrt(a), np.sqrt(1.0 - a), np.sqrt(ap), np.sqrt(1.0 - ap)
        with np.errstate(divide="ignore"):
            h = np.log((alp * sg) / (sgp * al))                     # lambda' - lambda; inf where alpha = 0
        e_mh = (al * sgp) / (sg * alp)                               # e^{-h}, as the ratio
        w = 1.0 - (e_mh if self.dpm_eta == 0.0 else e_mh * e_mh)
        c = np.zeros(a.shape[0])
        for k in range(a.shape[0] - 1):
            if al[k + 1] > 0.0:
                c[k] = alp[k] * w[k] / (2.0 * (h[k + 1] / h[k]))
        return c

    def _order2_coefficients(self, indices):
        w = self.order2_weights()
        return [0.0] + [float(w[k]) for k in indices[1:]]

    @torch.no_grad()
    def ddim_sampling(self, cond, shape, x_T=None, ddim_use_original_steps=False, **kwargs):
        if ddim_use_original_steps:
            raise NotImplementedError("DPM-Solver++(2M) runs on the DDIM schedule, not the original DDPM steps")
        self._order2_w = self.order2_weights()
        self._prev_pred_x0 = None                        # the general path's p_{i-1}; None: the next step is first order
        return super().ddim_sampling(cond, shape, x_T=x_T, ddim_use_original_steps=False, **kwargs)

    def _ddim_update(self, x, t, index, *args, **kwargs):
        """The general path: DDIM's update in torch, then the correction in fp32, one rounding per op (as tc_dpm_step)."""
        x_prev, pred_x0 = super()._ddim_update(x, t, index, *args, **kwargs)
        prev, self._prev_pred_x0 = self._prev_pred_x0, pred_x0
        c = float(np.float32(self._order2_w[index])) if prev is not None else 0.0
        if c != 0.0:
            x_prev = x_prev + c * (pred_x0 - prev)
        return x_prev, pred_x0


class DPMSolverSampler(_DPMSolverPP2M, DDIMSampler):
    """DDIMSampler's interface (sample, stochastic_encode, decode, noise_generators, t_start, mask / x0, latency_group)
    with DPM-Solver++(2M) steps; eta must be 0 or 1."""


class DPMSolverSamplerMultiCond(_DPMSolverPP2M, DDIMSamplerMultiCond):
    """DDIMSamplerMultiCond's three-way guidance (cfg_img) with DPM-Solver++(2M) steps; eta must be 0 or 1."""


SAMPLERS = {"ddim": (DDIMSampler, DDIMSamplerMultiCond), "dpmpp_2m": (DPMSolverSampler, DPMSolverSamplerMultiCond)}


def check_sampler(name, eta) -> str:
    """A key of SAMPLERS, with an eta that sampler takes (dpmpp_2m: 0 or 1); ValueError otherwise."""
    if name not in SAMPLERS:
        raise ValueError(f"sampler must be one of {sorted(SAMPLERS)}, got {name!r}")
    if name == "dpmpp_2m":
        check_dpm_eta(eta)
    return name

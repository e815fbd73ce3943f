"""Inference-side mirror of the reference's model objects (the Python surface scripts/evaluation/inference.py,
scripts/evaluation/funcs.py and gradio_app.py touch), backed by the CUDA engines.

Mirrors (interface, attribute names, buffer names, semantics; paths relative to /root/reference):
  DDPM / LatentDiffusion / LatentVisualDiffusion   lvdm/models/ddpm3d.py:41-187, 465-560, 598-683, 735-750, 1041-1062
  DiffusionWrapper                                 lvdm/models/ddpm3d.py:1243-1264
  AutoencoderKL / AutoencoderKL_Dualref            lvdm/models/autoencoder.py:13-116, 238-258
  DiagonalGaussianDistribution                     lvdm/distributions.py:24-64
  instantiate_from_config                          utils/utils.py:27-42
Training/logging methods of the reference classes are out of scope.
"""
from __future__ import annotations

import importlib
import math

import numpy as np
import torch
import torch.nn as nn

from . import modules


def get_obj_from_str(string: str):
    module, cls = string.rsplit(".", 1)
    return getattr(importlib.import_module(module), cls)


def instantiate_from_config(config):
    if "target" not in config:
        if config in ("__is_first_stage__", "__is_unconditional__"):
            return None
        raise KeyError("Expected key `target` to instantiate.")
    params = config.get("params", dict())
    return get_obj_from_str(config["target"])(**(params if params is not None else {}))


def _cfg_get(cfg, key, default=None):
    try:
        return cfg[key]
    except (KeyError, TypeError):
        return getattr(cfg, key, default)


class DiagonalGaussianDistribution:
    def __init__(self, parameters, deterministic=False):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if deterministic:
            self.var = self.std = torch.zeros_like(self.mean)

    def sample(self, noise=None):
        if noise is None:
            noise = torch.randn(self.mean.shape)          # CPU generator, like the reference (distributions.py:35-40)
        return self.mean + self.std * noise.to(device=self.parameters.device)

    def mode(self):
        return self.mean


# ---------------------------------------------------------------------------------------------------- schedule
def linear_beta_schedule(n, linear_start, linear_end):
    return (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, n, dtype=torch.float64, device="cpu") ** 2).numpy()


def enforce_zero_terminal_snr(betas):
    """Algorithm 1 of arXiv 2305.08891 (reference: lvdm/models/utils_diffusion.py:112-144)."""
    root = np.sqrt(np.cumprod(1.0 - betas, axis=0))
    first, last = root[0].copy(), root[-1].copy()
    root = (root - last) * (first / (first - last))
    abar = root ** 2
    return 1.0 - np.concatenate([abar[0:1], abar[1:] / abar[:-1]])


class DiffusionWrapper(nn.Module):
    def __init__(self, diff_model_config, conditioning_key):
        super().__init__()
        self.diffusion_model = instantiate_from_config(diff_model_config)
        self.conditioning_key = conditioning_key

    def forward(self, x, t, c_concat: list = None, c_crossattn: list = None, **kwargs):
        key = self.conditioning_key
        if key is None:
            return self.diffusion_model(x, t)
        if key == "concat":
            return self.diffusion_model(torch.cat([x] + c_concat, dim=1), t, **kwargs)
        if key == "crossattn":
            return self.diffusion_model(x, t, context=torch.cat(c_crossattn, 1), **kwargs)
        if key == "hybrid":
            return self.diffusion_model(torch.cat([x] + c_concat, dim=1), t, context=torch.cat(c_crossattn, 1), **kwargs)
        raise NotImplementedError(f"conditioning_key {key!r} is outside the supported hot path")


class AutoencoderKL(nn.Module):
    def __init__(self, ddconfig, lossconfig=None, embed_dim=4, ckpt_path=None, ignore_keys=(), image_key="image",
                 colorize_nlabels=None, monitor=None, test=False, logdir=None, input_dim=4, test_args=None,
                 additional_decode_keys=None, use_checkpoint=False, diff_boost_factor=3.0):
        super().__init__()
        dd = dict(ddconfig)
        if not dd.get("double_z", True):
            raise NotImplementedError("double_z=False is outside the supported hot path")
        self.image_key = image_key
        self.embed_dim = embed_dim
        self.encoder = modules.Encoder(**dd)
        self.decoder = self._make_decoder(dd)
        self.quant_conv = nn.Conv2d(2 * dd["z_channels"], 2 * embed_dim, 1)
        self.post_quant_conv = nn.Conv2d(embed_dim, dd["z_channels"], 1)
        self._dec_engine = None
        self._enc_engine = None
        if ckpt_path is not None:
            sd = torch.load(ckpt_path, map_location="cpu")
            self.load_state_dict(sd.get("state_dict", sd), strict=False)

    def _make_decoder(self, dd):
        return modules.Decoder(**dd)

    @property
    def device(self):
        return next(self.parameters()).device

    def encode(self, x, return_hidden_states=False, **kwargs):
        from . import runtime
        from .vae_engine import EncoderEngine
        ex = runtime.TEST_EXECUTOR
        moments, hidden = EncoderEngine.cached(self, "_enc_engine", ex).encode(x, executor=ex)
        post = DiagonalGaussianDistribution(moments)
        return (post, hidden) if return_hidden_states else post

    def decode(self, z, **kwargs):
        """z [N, embed_dim, h, w] -> [N, 3, 8h, 8w] fp16.  Like the reference, post_quant_conv runs only when no kwargs
        are given; the plain Decoder takes none (ae_modules.py:538), so decode(z) is its one form."""
        if kwargs:
            raise NotImplementedError("the plain AutoencoderKL decoder takes no decode kwargs (ref_context / "
                                      "timesteps belong to AutoencoderKL_Dualref)")
        from . import runtime
        return self.decoder_engine().decode(z.float(), executor=runtime.TEST_EXECUTOR).clone()

    def decoder_engine(self):
        """The PlainDecoderEngine decode() runs on (built on first use).  Its decode() returns a view of the plan's
        static output buffer, valid until the next decode of the same geometry: for callers that consume it in place."""
        from . import runtime
        from .vae_engine import PlainDecoderEngine
        return PlainDecoderEngine.cached(self, "_dec_engine", runtime.TEST_EXECUTOR)


class AutoencoderKL_Dualref(AutoencoderKL):
    def _make_decoder(self, dd):
        return modules.VideoDecoder(**dd)

    def decode(self, z, **kwargs):
        """kwargs: ref_context (5 maps [b, C, 2, H, W]) and timesteps, as decode_core passes them."""
        if len(kwargs) == 0:
            raise NotImplementedError("decode() without ref_context/timesteps never happens on the VideoDecoder path")
        from . import runtime
        ex = runtime.TEST_EXECUTOR
        eng = self.decoder_engine()
        ref = kwargs.get("ref_context")
        T = kwargs.get("timesteps") or z.shape[0]
        if z.shape[0] != T:
            raise NotImplementedError("one clip per decode call (the reference mixes clips for B > 1)")
        return eng.decode(z.float(), ref, executor=ex).clone()

    def decoder_engine(self):
        """The DecoderEngine decode() runs on (built on first use).  Its decode() returns a view of the plan's static
        output buffer, valid until the next decode of the same T: for callers that consume it in place."""
        from . import runtime
        from .vae_engine import DecoderEngine
        return DecoderEngine.cached(self, "_dec_engine", runtime.TEST_EXECUTOR, module=self.decoder)


class LatentVisualDiffusion(nn.Module):
    """LatentVisualDiffusion ⊂ LatentDiffusion ⊂ DDPM of the reference, inference subset, same ctor kwargs."""

    def __init__(self, unet_config, first_stage_config, cond_stage_config, img_cond_stage_config,
                 image_proj_stage_config, timesteps=1000, beta_schedule="linear", linear_start=1e-4, linear_end=2e-2,
                 cosine_s=8e-3, given_betas=None, parameterization="eps", rescale_betas_zero_snr=False,
                 conditioning_key=None, num_timesteps_cond=None, cond_stage_key="caption", cond_stage_trainable=False,
                 cond_stage_forward=None, uncond_prob=0.2, uncond_type="empty_seq", scale_factor=1.0,
                 scale_by_std=False, encoder_type="2d", use_dynamic_rescale=False, base_scale=0.7, turning_step=400,
                 loop_video=False, fps_condition_type="fs", perframe_ae=False, en_and_decode_n_samples_a_time=None,
                 first_stage_key="image", image_size=256, channels=3, use_ema=True, v_posterior=0.0,
                 freeze_embedder=True, image_proj_model_trainable=True, **ignored):
        super().__init__()
        if parameterization not in ("eps", "x0", "v"):
            raise ValueError('currently only supporting "eps" and "x0" and "v"')
        if beta_schedule != "linear" or given_betas is not None:
            raise NotImplementedError("only the linear beta schedule is on the supported hot path")
        self.parameterization = parameterization
        self.cond_stage_model = None
        self.first_stage_key, self.cond_stage_key = first_stage_key, cond_stage_key
        self.channels = channels
        self.temporal_length = _cfg_get(_cfg_get(unet_config, "params"), "temporal_length")
        self.image_size = [image_size, image_size] if isinstance(image_size, int) else image_size
        self.model = DiffusionWrapper(unet_config, conditioning_key if conditioning_key is not None else "crossattn")
        self.use_ema = False
        self.rescale_betas_zero_snr = rescale_betas_zero_snr
        self.v_posterior = v_posterior
        self.num_timesteps_cond = num_timesteps_cond if num_timesteps_cond is not None else 1
        self.scale_by_std = scale_by_std
        self.cond_stage_trainable, self.cond_stage_forward = cond_stage_trainable, cond_stage_forward
        self.use_dynamic_rescale = use_dynamic_rescale
        self.loop_video, self.fps_condition_type = loop_video, fps_condition_type
        self.perframe_ae = perframe_ae
        self.en_and_decode_n_samples_a_time = en_and_decode_n_samples_a_time
        self.encoder_type = encoder_type
        self.uncond_prob, self.uncond_type = uncond_prob, uncond_type
        self.clip_denoised = False
        self._register_schedule(timesteps, linear_start, linear_end)
        if scale_by_std:
            self.register_buffer("scale_factor", torch.tensor(scale_factor))
        else:
            self.scale_factor = scale_factor
        if use_dynamic_rescale:
            self._scale_arr_np = np.concatenate((np.linspace(1.0, base_scale, turning_step),
                                                 np.full(self.num_timesteps, base_scale)))
            self.register_buffer("scale_arr", torch.tensor(self._scale_arr_np, dtype=torch.float32))
        self.first_stage_model = instantiate_from_config(first_stage_config).eval()
        self.cond_stage_model = instantiate_from_config(cond_stage_config)
        self.embedder = instantiate_from_config(img_cond_stage_config)
        self.image_proj_model = instantiate_from_config(image_proj_stage_config)
        for p in self.parameters():
            p.requires_grad_(False)
        self.eval()

    # ---- schedule buffers, names and dtypes as ddpm3d.py:124-187 registers them
    def _schedule_arrays(self):
        timesteps, linear_start, linear_end = self._sched_args
        betas = linear_beta_schedule(timesteps, linear_start, linear_end)
        if self.rescale_betas_zero_snr:
            betas = enforce_zero_terminal_snr(betas)
        alphas = 1.0 - betas
        ac = np.cumprod(alphas, axis=0)
        ac_prev = np.append(1.0, ac[:-1])
        n = int(betas.shape[0])
        out = dict(betas=betas, alphas_cumprod=ac, alphas_cumprod_prev=ac_prev, sqrt_alphas_cumprod=np.sqrt(ac),
                   sqrt_one_minus_alphas_cumprod=np.sqrt(1.0 - ac))
        with np.errstate(divide="ignore", invalid="ignore"):
            out["log_one_minus_alphas_cumprod"] = np.log(1.0 - ac)
            if self.parameterization != "v":
                out["sqrt_recip_alphas_cumprod"] = np.sqrt(1.0 / ac)
                out["sqrt_recipm1_alphas_cumprod"] = np.sqrt(1.0 / ac - 1)
            else:
                out["sqrt_recip_alphas_cumprod"] = np.zeros(n)
                out["sqrt_recipm1_alphas_cumprod"] = np.zeros(n)
            post_var = (1 - self.v_posterior) * betas * (1.0 - ac_prev) / (1.0 - ac) + self.v_posterior * betas
            out["posterior_variance"] = post_var
            out["posterior_log_variance_clipped"] = np.log(np.maximum(post_var, 1e-20))
            out["posterior_mean_coef1"] = betas * np.sqrt(ac_prev) / (1.0 - ac)
            out["posterior_mean_coef2"] = (1.0 - ac_prev) * np.sqrt(alphas) / (1.0 - ac)
        return out

    def _register_schedule(self, timesteps, linear_start, linear_end):
        self._sched_args = (timesteps, linear_start, linear_end)
        self.linear_start, self.linear_end = linear_start, linear_end
        arrays = self._schedule_arrays()
        self.num_timesteps = int(arrays["betas"].shape[0])
        for k, a in arrays.items():
            self.register_buffer(k, torch.tensor(a, dtype=torch.float32))

    def reset_schedule_buffers(self):
        """Recompute every schedule buffer in place (after `to_empty()` / meta-device construction)."""
        with torch.no_grad():
            for k, a in self._schedule_arrays().items():
                getattr(self, k).copy_(torch.tensor(a, dtype=torch.float32, device="cpu"))
            if self.use_dynamic_rescale:
                self.scale_arr.copy_(torch.tensor(self._scale_arr_np, dtype=torch.float32, device="cpu"))

    @property
    def device(self):
        return self.betas.device

    # ---- conditioning / first stage plumbing (ddpm3d.py:598-683)
    def get_learned_conditioning(self, c):
        m = self.cond_stage_model
        if self.cond_stage_forward is not None:
            return getattr(m, self.cond_stage_forward)(c)
        if hasattr(m, "encode") and callable(m.encode):
            c = m.encode(c)
            return c.mode() if isinstance(c, DiagonalGaussianDistribution) else c
        return m(c)

    def get_first_stage_encoding(self, encoder_posterior, noise=None):
        if isinstance(encoder_posterior, DiagonalGaussianDistribution):
            z = encoder_posterior.sample(noise=noise)
        elif isinstance(encoder_posterior, torch.Tensor):
            z = encoder_posterior
        else:
            raise NotImplementedError(type(encoder_posterior))
        return self.scale_factor * z

    @torch.no_grad()
    def encode_first_stage(self, x):
        five_d = self.encoder_type == "2d" and x.dim() == 5
        if five_d:
            b, _, t, _, _ = x.shape
            x = x.permute(0, 2, 1, 3, 4).reshape(b * t, *x.shape[1:2], *x.shape[3:])
        if not self.perframe_ae:
            z = self.get_first_stage_encoding(self.first_stage_model.encode(x))
        else:
            z = torch.cat([self.get_first_stage_encoding(self.first_stage_model.encode(x[i:i + 1]))
                           for i in range(x.shape[0])], dim=0)
        if five_d:
            z = z.reshape(b, t, *z.shape[1:]).permute(0, 2, 1, 3, 4)
        return z

    def decode_core(self, z, **kwargs):
        five_d = self.encoder_type == "2d" and z.dim() == 5
        if five_d:
            b, _, t, _, _ = z.shape
            z = z.permute(0, 2, 1, 3, 4).reshape(b * t, z.shape[1], *z.shape[3:])
        z = 1.0 / self.scale_factor * z
        video_decoder = isinstance(self.first_stage_model.decoder, modules.VideoDecoder)
        if not self.perframe_ae:
            if video_decoder:
                raise NotImplementedError("VideoDecoder needs the chunked (perframe_ae=True) path")
            out = self.first_stage_model.decode(z, **kwargs)
        else:
            n = self.en_and_decode_n_samples_a_time or self.temporal_length
            outs = []
            for i in range(0, z.shape[0], n):
                chunk = z[i:i + n]
                # ddpm3d.py:664-667: only a VideoDecoder gets the caller's kwargs plus timesteps; any other decoder none
                kw = dict(kwargs, timesteps=chunk.shape[0]) if video_decoder else {}
                outs.append(self.first_stage_model.decode(chunk, **kw))
            out = torch.cat(outs, dim=0)
        if five_d:
            out = out.reshape(b, t, *out.shape[1:]).permute(0, 2, 1, 3, 4)
        return out

    @torch.no_grad()
    def decode_first_stage(self, z, **kwargs):
        return self.decode_core(z, **kwargs)

    # ---- denoiser access used by the samplers (ddpm3d.py:240-252, 306-311, 735-750)
    def apply_model(self, x_noisy, t, cond, **kwargs):
        if not isinstance(cond, dict):
            cond = {("c_concat" if self.model.conditioning_key == "concat" else "c_crossattn"):
                    cond if isinstance(cond, list) else [cond]}
        out = self.model(x_noisy, t, **cond, **kwargs)
        return out[0] if isinstance(out, tuple) else out

    @staticmethod
    def _gather(a, t, x_shape):
        return a.gather(-1, t).reshape(t.shape[0], *((1,) * (len(x_shape) - 1)))

    def predict_start_from_z_and_v(self, x_t, t, v):
        return (self._gather(self.sqrt_alphas_cumprod, t, x_t.shape) * x_t -
                self._gather(self.sqrt_one_minus_alphas_cumprod, t, x_t.shape) * v)

    def predict_eps_from_z_and_v(self, x_t, t, v):
        return (self._gather(self.sqrt_alphas_cumprod, t, x_t.shape) * v +
                self._gather(self.sqrt_one_minus_alphas_cumprod, t, x_t.shape) * x_t)

    def q_sample(self, x_start, t, noise=None):
        noise = torch.randn_like(x_start) if noise is None else noise
        return (self._gather(self.sqrt_alphas_cumprod, t, x_start.shape) * x_start +
                self._gather(self.sqrt_one_minus_alphas_cumprod, t, x_start.shape) * noise)


LatentDiffusion = LatentVisualDiffusion

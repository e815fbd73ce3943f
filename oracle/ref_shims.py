"""TEST INFRASTRUCTURE ONLY — import the UNMODIFIED reference (/root/reference) with three harness shims.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may import anything
under oracle/.  The product path (tooncrafter_b200/) never does.

The reference cannot travel to the GPU box (it only exists in the authoring container), so this module is used
to (a) validate oracle/ against the real reference and (b) generate tests/golden/ fixtures.  Shims:
  1. stub `pytorch_lightning` (ddpm3d.py:21-22, autoencoder.py:7 only need LightningModule/rank_zero_only);
  2. fake `xformers.ops.memory_efficient_attention` backed by F.scaled_dot_product_attention
     (autoencoder_dualref.py:190,316,326 call it unconditionally); installed AFTER lvdm.modules.attention is
     imported so the UNet keeps the explicit einsum+softmax path (attention.py:81-144);
  3. device-agnostic DDIMSampler.register_buffer (ddim.py:18-22 hard-codes "cuda").
Nothing in the reference is edited.
"""
from __future__ import annotations

import sys
import types
from pathlib import Path

import torch
import torch.nn as nn
import torch.nn.functional as F

REFERENCE_ROOT = Path("/root/reference")


def reference_available() -> bool:
    return (REFERENCE_ROOT / "lvdm" / "models" / "ddpm3d.py").exists()


class AttrDict(dict):
    """dict with attribute access, recursive (stands in for OmegaConf: ddpm3d.py:82 reads cfg.params.x)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    @staticmethod
    def wrap(o):
        if isinstance(o, dict):
            return AttrDict({k: AttrDict.wrap(v) for k, v in o.items()})
        if isinstance(o, (list, tuple)):
            return type(o)(AttrDict.wrap(v) for v in o)
        return o


_installed = False


def install():
    """Make `import lvdm...` resolve to the reference, with the shims in place.  Idempotent."""
    global _installed
    if _installed:
        return
    if not reference_available():
        raise RuntimeError("/root/reference is not present (expected on the GPU box); use tests/golden fixtures")
    # our own repo also ships an `lvdm` alias package: make sure the reference wins in this process
    for name in [m for m in sys.modules if m == "lvdm" or m.startswith("lvdm.") or m == "utils" or m.startswith("utils.")]:
        del sys.modules[name]
    sys.path.insert(0, str(REFERENCE_ROOT))
    # the reference's `lvdm` / `utils` are namespace packages (no __init__.py) and would lose against this repo's
    # regular alias packages wherever they sit on sys.path: pin both names to the reference's directories
    for name in ("lvdm", "utils"):
        pkg = types.ModuleType(name)
        pkg.__path__ = [str(REFERENCE_ROOT / name)]
        sys.modules[name] = pkg

    pl = types.ModuleType("pytorch_lightning")

    class LightningModule(nn.Module):
        @property
        def device(self):
            return next(self.parameters()).device

    pl.LightningModule = LightningModule
    pl.utilities = types.ModuleType("pytorch_lightning.utilities")
    pl.utilities.rank_zero_only = lambda f: f
    sys.modules["pytorch_lightning"] = pl
    sys.modules["pytorch_lightning.utilities"] = pl.utilities

    # import the UNet attention first so XFORMERS_IS_AVAILBLE is False there (explicit einsum path)
    import lvdm.modules.attention  # noqa: F401

    xf = types.ModuleType("xformers")
    xf.__version__ = "0.0.0"
    xf.ops = types.ModuleType("xformers.ops")

    def mea(q, k, v, attn_bias=None, op=None):
        # 4-D lift keeps the CPU on the flash kernel (3-D inputs would materialise Lq x Lk scores)
        return F.scaled_dot_product_attention(q[None], k[None], v[None])[0]

    xf.ops.memory_efficient_attention = mea
    sys.modules["xformers"] = xf
    sys.modules["xformers.ops"] = xf.ops
    _installed = True


def make_sampler(model):
    install()
    from lvdm.models.samplers.ddim import DDIMSampler

    class OracleSampler(DDIMSampler):
        def register_buffer(self, name, attr):
            if isinstance(attr, torch.Tensor):
                attr = attr.to(self.model.device)
            setattr(self, name, attr)

    return OracleSampler(model)


def build_reference_unet(params: dict):
    install()
    from lvdm.modules.networks.openaimodel3d import UNetModel
    p = dict(params)
    p["use_checkpoint"] = False       # scripts/evaluation/inference.py:286
    return UNetModel(**p)


def build_reference_vae(ddconfig: dict, embed_dim: int = 4):
    install()
    from lvdm.models.autoencoder import AutoencoderKL_Dualref
    return AutoencoderKL_Dualref(ddconfig=dict(ddconfig), lossconfig={"target": "torch.nn.Identity"},
                                 embed_dim=embed_dim)


def build_reference_model(model_cfg: dict):
    """Full LatentVisualDiffusion from a YAML-style dict (conditioning stages should target torch.nn.Identity)."""
    install()
    from utils.utils import instantiate_from_config
    cfg = AttrDict.wrap(model_cfg)
    cfg["params"]["unet_config"]["params"]["use_checkpoint"] = False
    return instantiate_from_config(cfg)

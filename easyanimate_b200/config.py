"""diffusers-free stand-ins for the ``ConfigMixin`` / output-dataclass surface the reference pipelines read.

The reference modules derive from diffusers ``ModelMixin, ConfigMixin`` and decorate ``__init__`` with
``@register_to_config`` (easyanimate/models/transformer3d.py:1346-1350, autoencoder_magvit.py:59,93); the pipelines
then read ``module.config.<name>`` and ``module.config.get(name, default)``.  ``FrozenConfig`` gives
the same read surface without importing diffusers.
"""
from __future__ import annotations

import inspect
import json
import os
from dataclasses import dataclass
from typing import Any, Dict

import torch


class FrozenConfig(dict):
    """dict with attribute access, like diffusers' FrozenDict."""

    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError as e:
            raise AttributeError(name) from e

    def __setattr__(self, name, value):
        raise AttributeError("config is read-only")


def capture_init_config(obj, local_vars: Dict[str, Any]) -> FrozenConfig:
    """Collect the constructor arguments of ``obj.__init__`` from its locals() (the @register_to_config contract)."""
    sig = inspect.signature(type(obj).__init__)
    cfg = {}
    for name, param in sig.parameters.items():
        if name == "self" or param.kind in (param.VAR_KEYWORD, param.VAR_POSITIONAL):
            continue
        v = local_vars[name]
        cfg[name] = list(v) if isinstance(v, tuple) else v
    cfg["_class_name"] = type(obj).__name__
    return FrozenConfig(cfg)


class ConfigMixinLite:
    config: FrozenConfig

    @classmethod
    def load_config(cls, path: str, subfolder: str | None = None) -> Dict[str, Any]:
        if subfolder is not None:
            path = os.path.join(path, subfolder)
        with open(os.path.join(path, "config.json")) as f:
            return json.load(f)

    @classmethod
    def from_config(cls, config: Dict[str, Any], **kwargs):
        sig = inspect.signature(cls.__init__)
        accepted = {k for k in sig.parameters if k != "self"}
        merged = {k: v for k, v in dict(config).items() if k in accepted}
        merged.update({k: v for k, v in kwargs.items() if k in accepted})
        return cls(**merged)

    @property
    def dtype(self) -> torch.dtype:
        for p in self.parameters():
            return p.dtype
        return torch.float32

    @property
    def device(self) -> torch.device:
        for p in self.parameters():
            return p.device
        return torch.device("cpu")


@dataclass
class Transformer2DModelOutput:
    sample: torch.Tensor

    def __getitem__(self, i):
        return (self.sample,)[i]


@dataclass
class DecoderOutput:
    sample: torch.Tensor

    def __getitem__(self, i):
        return (self.sample,)[i]


class DiagonalGaussianDistribution:
    """The posterior object `vae.encode(x)[0]` returns in the reference (diffusers autoencoders/vae.py): `parameters` is the
    moments tensor [B, 2*C, T, h, w] = (mean | logvar); the pipelines call `.sample()` or `.mode()` on it
    (pipeline_easyanimate_inpaint.py:769-826).  Small host-side torch ops on the latent-sized tensor."""

    def __init__(self, parameters: torch.Tensor, deterministic: bool = False):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)

    def sample(self, generator=None) -> torch.Tensor:
        noise = torch.randn(self.mean.shape, generator=generator, device=self.parameters.device, dtype=self.parameters.dtype)
        return self.mean + self.std * noise

    def mode(self) -> torch.Tensor:
        return self.mean


@dataclass
class AutoencoderKLOutput:
    latent_dist: DiagonalGaussianDistribution

    def __getitem__(self, i):
        return (self.latent_dist,)[i]


def load_state_dict_from_dir(path: str) -> Dict[str, torch.Tensor]:
    """safetensors / .bin loader used by from_pretrained(_2d) (transformer3d.py:1692-1809, autoencoder_magvit.py:478-505)."""
    import glob

    st = os.path.join(path, "diffusion_pytorch_model.safetensors")
    if os.path.exists(st):
        from safetensors.torch import load_file

        return load_file(st)
    shards = sorted(glob.glob(os.path.join(path, "*.safetensors")))
    if shards:
        from safetensors.torch import load_file

        out: Dict[str, torch.Tensor] = {}
        for s in shards:
            out.update(load_file(s))
        return out
    b = os.path.join(path, "diffusion_pytorch_model.bin")
    if os.path.exists(b):
        return torch.load(b, map_location="cpu", weights_only=True)
    raise RuntimeError(f"no weights found under {path}")

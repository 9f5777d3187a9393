"""easyanimate_b200 — H100-native (sm_90a) implementation of the EasyAnimateV5.1 sampling hot path.

Drop-in replacements for the reference's ``easyanimate.models`` name maps (easyanimate/models/__init__.py:6-14):
importing this package requires the in-tree CUDA library ``libea_b200.so`` (there is no CPU/PyTorch fallback).
"""
from . import _lib  # noqa: F401  (fails loudly if the CUDA extension has not been built)
from .autoencoder_magvit import AutoencoderKLMagvit
from .long_video import generate_long_video
from .pipeline import EasyAnimateSampler, rope_table
from .pipelines import (EasyAnimateControlPipeline, EasyAnimateInpaintPipeline, EasyAnimatePipeline,
                        EasyAnimatePipelineOutput, load_pipeline)
from .scheduler import FlowMatchEulerDiscreteScheduler
from .transformer3d import EasyAnimateTransformer3DModel

name_to_transformer3d = {"EasyAnimateTransformer3DModel": EasyAnimateTransformer3DModel}
name_to_autoencoder_magvit = {"AutoencoderKLMagvit": AutoencoderKLMagvit}

__all__ = ["AutoencoderKLMagvit", "EasyAnimateControlPipeline", "EasyAnimateInpaintPipeline", "EasyAnimatePipeline",
           "EasyAnimatePipelineOutput", "EasyAnimateSampler", "EasyAnimateTransformer3DModel", "FlowMatchEulerDiscreteScheduler",
           "generate_long_video", "load_pipeline", "name_to_autoencoder_magvit", "name_to_transformer3d", "rope_table"]

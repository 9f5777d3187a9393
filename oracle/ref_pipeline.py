"""ORACLE helper (test infrastructure only): the reference's own `EasyAnimatePipeline`
(easyanimate/pipeline/pipeline_easyanimate.py:175-1148, executed unmodified from /root/reference) with the third-party
`diffusers` names it imports supplied by oracle/_refshim (DiffusionPipeline plumbing, FlowMatchEulerDiscreteScheduler,
get_3d_rotary_pos_embed, randn_tensor; everything else a placeholder).

Two uses:
  * tests/test_ref_pipeline_cpu.py drives `EasyAnimatePipeline.__call__` with the PRODUCT modules plugged in (the boundary of
    the duck-typed nn.Module surface) and with the reference's own modules, and compares the two;
  * tests/golden/make_golden.py mints `pipe_ref_t2v.safetensors` (latents in, text embeds in, frames out) from the reference's
    pipeline + the reference's transformer and VAE, which the GPU test of the sampler compares with.

Works only where /root/reference exists (the authoring container).  Never imported on the GPU box or by the product path."""
from __future__ import annotations

import importlib
import os
import sys
import types

from . import ref_dit, ref_vae

REFERENCE_ROOT = ref_dit.REFERENCE_ROOT


def available() -> bool:
    return ref_dit.available() and os.path.isfile(
        os.path.join(REFERENCE_ROOT, "easyanimate", "pipeline", "pipeline_easyanimate.py"))


def _reference_pipeline_module():
    if not available():
        raise RuntimeError("/root/reference is not present here")
    tmod = ref_dit._reference_models()            # easyanimate, easyanimate.models (synthetic parents) + transformer3d
    for name, rel in (("easyanimate.vae", "easyanimate/vae"), ("easyanimate.vae.ldm", "easyanimate/vae/ldm"),
                      ("easyanimate.vae.ldm.models", "easyanimate/vae/ldm/models"),
                      ("easyanimate.pipeline", "easyanimate/pipeline")):
        if name not in sys.modules:
            pkg = types.ModuleType(name)
            pkg.__path__ = [os.path.join(REFERENCE_ROOT, rel)]
            sys.modules[name] = pkg
    vmod = importlib.import_module("easyanimate.models.autoencoder_magvit")
    # `from ..models import AutoencoderKLMagvit, EasyAnimateTransformer3DModel` (pipeline_easyanimate.py:44): the synthetic
    # parent package exposes the two classes without executing easyanimate/models/__init__.py (text encoders, ...)
    models = sys.modules["easyanimate.models"]
    models.AutoencoderKLMagvit = vmod.AutoencoderKLMagvit
    models.EasyAnimateTransformer3DModel = tmod.EasyAnimateTransformer3DModel
    return importlib.import_module("easyanimate.pipeline.pipeline_easyanimate")


def _tokenizer():
    # encode_prompt reads tokenizer.model_max_length even when the embeddings are given (pipeline_easyanimate.py:361-363)
    return types.SimpleNamespace(model_max_length=256)


def _scheduler():
    from diffusers.schedulers import FlowMatchEulerDiscreteScheduler  # real install if present, else the shim

    return FlowMatchEulerDiscreteScheduler(num_train_timesteps=1000, shift=1.0)  # V5.1 scheduler config (shift 1)


def reference_inpaint_pipeline(transformer, vae, scheduler=None):
    """The reference's `EasyAnimateInpaintPipeline` (pipeline_easyanimate_inpaint.py:245-1604; predict_i2v.py builds it), no
    CLIP image encoder (V5.1: enable_clip_in_inpaint false), text encoders = None."""
    _reference_pipeline_module()
    mod = importlib.import_module("easyanimate.pipeline.pipeline_easyanimate_inpaint")
    return mod.EasyAnimateInpaintPipeline(vae=vae, text_encoder=None, tokenizer=_tokenizer(), text_encoder_2=None, tokenizer_2=None,
                                          transformer=transformer, scheduler=scheduler or _scheduler())


def reference_control_pipeline(transformer, vae, scheduler=None):
    """The reference's `EasyAnimateControlPipeline` (pipeline_easyanimate_control.py:200-1282; predict_v2v_control.py builds it)."""
    _reference_pipeline_module()
    mod = importlib.import_module("easyanimate.pipeline.pipeline_easyanimate_control")
    return mod.EasyAnimateControlPipeline(vae=vae, text_encoder=None, tokenizer=_tokenizer(), text_encoder_2=None, tokenizer_2=None,
                                          transformer=transformer, scheduler=scheduler or _scheduler())


def run_control(pipe, latents, control_video, ref_image, prompt_embeds, negative_prompt_embeds, *, height, width, video_length,
                num_inference_steps, guidance_scale=6.0):
    """One Control call the way predict_v2v_control.py makes it: control_video [B,3,F,H,W] in [0,1] (pose / depth / canny
    frames), ref_image [B,3,1,H,W] in [0,1] or None, precomputed embeddings, given start latents."""
    import torch

    ones = torch.ones(prompt_embeds.shape[:2], dtype=torch.long)
    with torch.no_grad():
        out = pipe(prompt=None, video_length=video_length, control_video=control_video, ref_image=ref_image, height=height,
                   width=width, num_inference_steps=num_inference_steps, guidance_scale=guidance_scale, latents=latents,
                   prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
                   prompt_attention_mask=ones, negative_prompt_attention_mask=ones.clone(),
                   prompt_embeds_2=prompt_embeds, prompt_attention_mask_2=ones.clone(), output_type="latent")
    return out.frames


def run_inpaint(pipe, video, mask_video, prompt_embeds, negative_prompt_embeds, *, height, width, num_inference_steps, seed,
                guidance_scale=6.0, noise_aug_strength=0.0563):
    """One I2V call the way predict_i2v.py:301-314 makes it (video [B,3,F,H,W] in [0,1], mask_video [B,1,F,H,W] in {0,255}),
    with precomputed embeddings.  The start noise (and the reference-video noise of add_noise_in_inpaint_model) is drawn from a
    seeded CPU generator: with a flow-matching scheduler the pipeline cannot take `latents=` (prepare_latents leaves `noise`
    unbound on that branch, pipeline_easyanimate_inpaint.py:893-905)."""
    import torch

    ones = torch.ones(prompt_embeds.shape[:2], dtype=torch.long)
    with torch.no_grad():
        out = pipe(prompt=None, video_length=video.shape[2], video=video, mask_video=mask_video, height=height, width=width,
                   num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                   generator=torch.Generator().manual_seed(seed), noise_aug_strength=noise_aug_strength,
                   prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
                   prompt_attention_mask=ones, negative_prompt_attention_mask=ones.clone(),
                   prompt_embeds_2=prompt_embeds, prompt_attention_mask_2=ones.clone(), output_type="latent")
    return out.frames


def reference_pipeline(transformer, vae, scheduler=None):
    """`EasyAnimatePipeline(vae=, transformer=, scheduler=, text encoders = None)` - the reference's class, with whatever
    modules the caller plugs in (the reference's own or the product's).  Prompts must be passed as embeddings."""
    mod = _reference_pipeline_module()
    return mod.EasyAnimatePipeline(vae=vae, text_encoder=None, tokenizer=_tokenizer(), text_encoder_2=None, tokenizer_2=None,
                                   transformer=transformer, scheduler=scheduler or _scheduler())


def run(pipe, latents, prompt_embeds, negative_prompt_embeds, *, height, width, video_length, num_inference_steps,
        guidance_scale=6.0):
    """One `pipe(...)` call the way predict_t2v.py:247-256 makes it, with precomputed embeddings; returns frames
    [B, 3, F, H, W] float32 in [0, 1] (`output_type='latent'` is the reference's name for 'torch tensor of frames')."""
    import torch

    ones = torch.ones(prompt_embeds.shape[:2], dtype=torch.long)
    with torch.no_grad():
        out = pipe(prompt=None, video_length=video_length, height=height, width=width,
                   num_inference_steps=num_inference_steps, guidance_scale=guidance_scale, latents=latents,
                   prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
                   prompt_attention_mask=ones, negative_prompt_attention_mask=ones.clone(),
                   # check_inputs (pipeline_easyanimate.py:635-638) insists on prompt_embeds_2 when no prompt string is given;
                   # with tokenizer_2 = None (V5.1) __call__ discards it again (:953-957)
                   prompt_embeds_2=prompt_embeds, prompt_attention_mask_2=ones.clone(), output_type="latent")
    return out.frames

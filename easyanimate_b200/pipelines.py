"""The reference's three pipeline entry points with their call signatures, on the H100 modules and WITHOUT diffusers:

    EasyAnimatePipeline          easyanimate/pipeline/pipeline_easyanimate.py:175-1148          (predict_t2v.py)
    EasyAnimateInpaintPipeline   easyanimate/pipeline/pipeline_easyanimate_inpaint.py:245-1604  (predict_i2v.py, predict_v2v.py)
    EasyAnimateControlPipeline   easyanimate/pipeline/pipeline_easyanimate_control.py:200-1282  (predict_v2v_control.py)

The reference's own pipeline classes accept the native transformer / VAE objects unchanged (INTEGRATION.md section 1, tested by
tests/test_ref_pipeline_cpu.py); these classes are for deployments that do not install diffusers, and they run the loop the
fused way: per step ONE transformer call on the CFG batch and ONE `ea_cfg_euler_step` (CFG combine + Euler update), frames
leave the GPU once through `ea_frames_out` (EasyAnimateSampler).  Same keyword arguments, same defaults, same output object
(`.frames`: [B, 3, F, H, W] float32 in [0, 1]; a torch tensor for output_type="latent" like the reference's
`torch.from_numpy(video)`, else a numpy array), same exceptions for malformed inputs.

Conditioning preparation (before the loop, once per call) is torch code like the reference's: mask / video normalisation,
`resize_mask` (trilinear), the reference-video noise, `vae.encode(...)[0].mode() * scaling_factor` - the encode itself runs on
the CUDA kernels.  What is NOT carried over (raises NotImplementedError, never a silent difference): `guidance_rescale > 0`,
the CLIP-image branch of the inpaint pipeline (V5.1: `enable_clip_in_inpaint: false`), blending-style inpainting with a
16-channel transformer, the Bert/T5 tokenizer branch of V5 (`text_embed_dim_t5`), non flow-matching schedulers, ComfyUI's bar."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple, Union

import numpy as np
import torch
import torch.nn.functional as F

from .pipeline import EasyAnimateSampler, rope_table
from .scheduler import FlowMatchEulerDiscreteScheduler

bf16 = torch.bfloat16


@dataclass
class EasyAnimatePipelineOutput:
    """pipeline_easyanimate_inpaint.py:231-241 (`frames`), indexable like diffusers' BaseOutput."""
    frames: Union[torch.Tensor, np.ndarray]

    def __getitem__(self, i):
        return (self.frames,)[i]


def _as_b200_scheduler(s) -> FlowMatchEulerDiscreteScheduler:
    """Our scheduler as is; a diffusers FlowMatchEulerDiscreteScheduler by its config (shift / dynamic shifting)."""
    if s is None:
        return FlowMatchEulerDiscreteScheduler()
    if isinstance(s, FlowMatchEulerDiscreteScheduler):
        return s
    cfg = getattr(s, "config", None)
    if cfg is None or "shift" not in cfg:
        raise NotImplementedError(f"easyanimate_b200 pipelines run the flow-matching Euler scheduler only, got {type(s).__name__}")
    return FlowMatchEulerDiscreteScheduler(num_train_timesteps=cfg.get("num_train_timesteps", 1000), shift=cfg["shift"],
                                           use_dynamic_shifting=cfg.get("use_dynamic_shifting", False))


def randn_like_reference(shape, generator, device, dtype):
    """diffusers.utils.torch_utils.randn_tensor: a CPU generator draws on the CPU and the result moves to `device`."""
    if isinstance(generator, (list, tuple)):
        if len(generator) != shape[0]:
            raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an effective batch"
                             f" size of {shape[0]}. Make sure the batch size matches the length of the generators.")
        return torch.cat([randn_like_reference((1,) + tuple(shape[1:]), g, device, dtype) for g in generator])
    where = generator.device if generator is not None else torch.device(device)
    return torch.randn(tuple(shape), generator=generator, device=where, dtype=dtype).to(device)


def resize_mask(mask: torch.Tensor, latent: torch.Tensor, process_first_frame_only: bool = True) -> torch.Tensor:
    """pipeline_easyanimate_inpaint.py:116-149: the pixel-space mask [B,1,F,H,W] brought to the latent grid by trilinear
    interpolation; with the MagViT chunking (1 + 4k frames -> 1 + k latent frames) frame 0 is resized on its own."""
    t, h, w = latent.shape[2:]
    if not process_first_frame_only:
        return F.interpolate(mask, size=(t, h, w), mode="trilinear", align_corners=False)
    parts = [F.interpolate(mask[:, :, :1], size=(1, h, w), mode="trilinear", align_corners=False)]
    if t > 1:
        parts.append(F.interpolate(mask[:, :, 1:], size=(t - 1, h, w), mode="trilinear", align_corners=False))
    return torch.cat(parts, dim=2)


def add_noise_to_reference_video(image: torch.Tensor, ratio: Optional[float] = None, generator=None) -> torch.Tensor:
    """pipeline_easyanimate_inpaint.py:153-168: Gaussian noise of std `ratio` (or exp(N(-3, 0.5)) per sample) on the
    conditioning video, except where it is exactly -1 (the masked-out pixels)."""
    if ratio is None:
        sigma = torch.exp(torch.normal(mean=-3.0, std=0.5, size=(image.shape[0],)).to(image.device)).to(image.dtype)
    else:
        sigma = torch.ones((image.shape[0],)).to(image.device, image.dtype) * ratio
    if generator is not None:
        noise = torch.randn(image.size(), generator=generator, dtype=image.dtype, device=image.device)
    else:
        noise = torch.randn_like(image)
    noise = noise * sigma[:, None, None, None, None]
    return image + torch.where(image == -1, torch.zeros_like(image), noise)


class _NativePipelineBase:
    """Constructor / properties / prompt handling / loop shared by the three pipelines."""
    _callback_tensor_inputs = ["latents", "prompt_embeds", "negative_prompt_embeds", "prompt_embeds_2", "negative_prompt_embeds_2"]

    def __init__(self, vae, text_encoder=None, tokenizer=None, text_encoder_2=None, tokenizer_2=None, transformer=None,
                 scheduler=None, clip_image_processor=None, clip_image_encoder=None, cfg_group=None):
        if transformer is None or vae is None:
            raise ValueError("`transformer` and `vae` are required")
        self.vae, self.transformer = vae, transformer
        self.text_encoder, self.tokenizer = text_encoder, tokenizer
        self.text_encoder_2, self.tokenizer_2 = text_encoder_2, tokenizer_2
        self.clip_image_processor, self.clip_image_encoder = clip_image_processor, clip_image_encoder
        self.scheduler = _as_b200_scheduler(scheduler)
        self.vae_scale_factor = 2 ** (len(self.vae.config.block_out_channels) - 1)
        self.cfg_group = cfg_group
        self._guidance_scale, self._guidance_rescale, self._num_timesteps, self._interrupt = 1.0, 0.0, 0, False

    # ---- the reference pipelines' read-only properties
    @property
    def guidance_scale(self):
        return self._guidance_scale

    @property
    def guidance_rescale(self):
        return self._guidance_rescale

    @property
    def do_classifier_free_guidance(self):
        return self._guidance_scale > 1

    @property
    def num_timesteps(self):
        return self._num_timesteps

    @property
    def interrupt(self):
        return self._interrupt

    @property
    def _execution_device(self):
        return next(self.transformer.parameters()).device

    @property
    def _dtype(self):
        """pipeline_easyanimate.py:906-911: the text encoder's dtype when there is one, else the transformer's."""
        for m in (self.text_encoder, self.text_encoder_2):
            if m is not None:
                return m.dtype
        d = self.transformer.dtype
        return bf16 if d == torch.float8_e4m3fn else d  # fp8 weight STORAGE computes in bf16 (transformer3d.py)

    def to(self, device):
        self.transformer.to(device)
        self.vae.to(device)
        for m in (self.text_encoder, self.text_encoder_2):
            if m is not None:
                m.to(device)
        return self

    # ---- prompts -------------------------------------------------------------------------------------------------
    def _encode_text(self, text_or_list, device, max_length):
        """The LLM branch of encode_prompt (pipeline_easyanimate.py:421-457): chat template -> fixed-length tokens -> the
        text encoder's second-to-last hidden state."""
        if self.tokenizer is None or self.text_encoder is None:
            raise ValueError("a prompt string needs `tokenizer` and `text_encoder`; otherwise pass `prompt_embeds`")
        if hasattr(self.tokenizer, "batch_decode") and not hasattr(self.tokenizer, "apply_chat_template"):
            raise NotImplementedError("the Bert / T5 tokenizer branch (EasyAnimate V5 multi text encoder) is not carried over")
        items = [text_or_list] if isinstance(text_or_list, str) else list(text_or_list)
        messages = [{"role": "user", "content": [{"type": "text", "text": p}]} for p in items]
        text = self.tokenizer.apply_chat_template(messages, tokenize=False, add_generation_prompt=True)
        tok = self.tokenizer(text=[text], padding="max_length", max_length=max_length, truncation=True,
                             return_attention_mask=True, padding_side="right", return_tensors="pt")
        tok = tok.to(self.text_encoder.device)
        if not self.transformer.config.enable_text_attention_mask:
            raise ValueError("LLM needs attention_mask")
        hidden = self.text_encoder(input_ids=tok.input_ids, attention_mask=tok.attention_mask,
                                   output_hidden_states=True).hidden_states[-2]
        return hidden, tok.attention_mask

    def encode_prompt(self, prompt, device, dtype, num_images_per_prompt=1, do_classifier_free_guidance=True, negative_prompt=None,
                      prompt_embeds=None, negative_prompt_embeds=None, prompt_attention_mask=None,
                      negative_prompt_attention_mask=None, max_sequence_length=None, text_encoder_index=0,
                      actual_max_sequence_length=256):
        """pipeline_easyanimate.py:306-598 for text_encoder_index 0: returns (embeds, negative embeds, mask, negative mask)."""
        if text_encoder_index != 0:
            raise NotImplementedError("the second text encoder (EasyAnimate V5 mT5) is not carried over")
        max_length = max_sequence_length
        if max_length is None and self.tokenizer is not None:
            max_length = min(self.tokenizer.model_max_length, actual_max_sequence_length)
        n = num_images_per_prompt
        if prompt_embeds is None:
            prompt_embeds, prompt_attention_mask = self._encode_text(prompt, device, max_length)
            prompt_attention_mask = prompt_attention_mask.repeat(n, 1)
        prompt_embeds = prompt_embeds.to(dtype=dtype, device=device)
        b, s, _ = prompt_embeds.shape
        prompt_embeds = prompt_embeds.repeat(1, n, 1).view(b * n, s, -1)
        prompt_attention_mask = prompt_attention_mask.to(device=device)
        if do_classifier_free_guidance:
            if negative_prompt_embeds is None:
                negative_prompt_embeds, negative_prompt_attention_mask = self._encode_text(
                    negative_prompt if negative_prompt is not None else "", device, max_length)
                negative_prompt_attention_mask = negative_prompt_attention_mask.repeat(n, 1)
            s = negative_prompt_embeds.shape[1]
            negative_prompt_embeds = negative_prompt_embeds.to(dtype=dtype, device=device).repeat(1, n, 1).view(b * n, s, -1)
            negative_prompt_attention_mask = negative_prompt_attention_mask.to(device=device)
        return prompt_embeds, negative_prompt_embeds, prompt_attention_mask, negative_prompt_attention_mask

    def check_inputs(self, prompt, height, width, negative_prompt=None, prompt_embeds=None, negative_prompt_embeds=None,
                     prompt_attention_mask=None, negative_prompt_attention_mask=None, prompt_embeds_2=None,
                     negative_prompt_embeds_2=None, prompt_attention_mask_2=None, negative_prompt_attention_mask_2=None,
                     callback_on_step_end_tensor_inputs=None):
        """The ValueErrors of pipeline_easyanimate.py:600-674, including its insistence on `prompt_embeds_2` when the prompt is
        given as embeddings."""
        if height % 16 != 0 or width % 16 != 0:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        bad = [k for k in (callback_on_step_end_tensor_inputs or []) if k not in self._callback_tensor_inputs]
        if bad:
            raise ValueError(f"`callback_on_step_end_tensor_inputs` has to be in {self._callback_tensor_inputs}, but found {bad}")
        if prompt is not None and prompt_embeds is not None:
            raise ValueError(f"Cannot forward both `prompt`: {prompt} and `prompt_embeds`: {prompt_embeds}. Please make sure to"
                             " only forward one of the two.")
        if prompt is None and prompt_embeds is None:
            raise ValueError("Provide either `prompt` or `prompt_embeds`. Cannot leave both `prompt` and `prompt_embeds` undefined.")
        if prompt is None and prompt_embeds_2 is None:
            raise ValueError("Provide either `prompt` or `prompt_embeds_2`. Cannot leave both `prompt` and `prompt_embeds_2` undefined.")
        if prompt is not None and not isinstance(prompt, (str, list)):
            raise ValueError(f"`prompt` has to be of type `str` or `list` but is {type(prompt)}")
        if prompt_embeds is not None and prompt_attention_mask is None:
            raise ValueError("Must provide `prompt_attention_mask` when specifying `prompt_embeds`.")
        if prompt_embeds_2 is not None and prompt_attention_mask_2 is None:
            raise ValueError("Must provide `prompt_attention_mask_2` when specifying `prompt_embeds_2`.")
        if negative_prompt is not None and negative_prompt_embeds is not None:
            raise ValueError(f"Cannot forward both `negative_prompt`: {negative_prompt} and `negative_prompt_embeds`:"
                             f" {negative_prompt_embeds}. Please make sure to only forward one of the two.")
        if negative_prompt_embeds is not None and negative_prompt_attention_mask is None:
            raise ValueError("Must provide `negative_prompt_attention_mask` when specifying `negative_prompt_embeds`.")
        if negative_prompt_embeds_2 is not None and negative_prompt_attention_mask_2 is None:
            raise ValueError("Must provide `negative_prompt_attention_mask_2` when specifying `negative_prompt_embeds_2`.")
        if prompt_embeds is not None and negative_prompt_embeds is not None and prompt_embeds.shape != negative_prompt_embeds.shape:
            raise ValueError("`prompt_embeds` and `negative_prompt_embeds` must have the same shape when passed directly, but"
                             f" got: `prompt_embeds` {prompt_embeds.shape} != `negative_prompt_embeds` {negative_prompt_embeds.shape}.")

    # ---- shapes, noise, schedule ---------------------------------------------------------------------------------
    def _latent_shape(self, batch, channels, video_length, height, width):
        """pipeline_easyanimate.py:677-689 for the MagViT VAE: 1 + 4k frames -> 1 + k latent frames (cache_mag_vae)."""
        me, md = self.vae.mini_batch_encoder, self.vae.mini_batch_decoder
        if video_length == 1:
            frames = 1
        elif self.vae.cache_mag_vae:
            frames = int((video_length - 1) // me * md + 1)
        else:
            frames = int(video_length // me * md)
        return (batch, channels, frames, height // self.vae_scale_factor, width // self.vae_scale_factor)

    def _set_timesteps(self, num_inference_steps, timesteps, strength=1.0):
        if timesteps is not None:  # retrieve_timesteps: FlowMatchEulerDiscreteScheduler.set_timesteps takes no `timesteps`
            raise ValueError(f"The current scheduler class {self.scheduler.__class__}'s `set_timesteps` does not support custom"
                             " timestep schedules. Please check whether you are using the correct scheduler.")
        self.scheduler.set_timesteps(num_inference_steps, device="cpu", mu=1)
        start = max(num_inference_steps - min(int(num_inference_steps * strength), num_inference_steps), 0)
        return start, num_inference_steps - start  # first schedule index of the loop, number of steps (get_timesteps, inpaint :760-767)

    def _encode_to_latents(self, pixels: torch.Tensor, device, dtype) -> torch.Tensor:
        """`vae.encode(x)[0].mode() * scaling_factor`, one sample at a time (pipeline_easyanimate_inpaint.py:800-812)."""
        pixels = pixels.to(device=device, dtype=dtype)
        out = [self.vae.encode(pixels[i:i + 1])[0].mode() for i in range(pixels.shape[0])]
        return torch.cat(out, dim=0) * self.vae.config.scaling_factor

    @staticmethod
    def _normalise_video(video: torch.Tensor, height: int, width: int) -> torch.Tensor:
        """What `VaeImageProcessor(do_normalize=True).preprocess` does to a [B,3,F,H,W] tensor: resize if needed, [0,1] -> [-1,1]
        unless the tensor already has negative values; float32."""
        b, c, f = video.shape[:3]
        x = video.permute(0, 2, 1, 3, 4).reshape(b * f, c, *video.shape[-2:])
        if tuple(x.shape[-2:]) != (height, width):
            x = F.interpolate(x, size=(height, width))
        if x.min() >= 0:
            x = 2.0 * x - 1.0
        return x.reshape(b, f, c, height, width).permute(0, 2, 1, 3, 4).to(torch.float32)

    @staticmethod
    def _binarise_mask(mask: torch.Tensor, height: int, width: int) -> torch.Tensor:
        """`VaeImageProcessor(do_normalize=False, do_binarize=True, do_convert_grayscale=True).preprocess` on [B,1,F,H,W]."""
        b, c, f = mask.shape[:3]
        x = mask.permute(0, 2, 1, 3, 4).reshape(b * f, c, *mask.shape[-2:])
        if tuple(x.shape[-2:]) != (height, width):
            x = F.interpolate(x, size=(height, width))
        x = (x >= 0.5).to(torch.float32)
        return x.reshape(b, f, c, height, width).permute(0, 2, 1, 3, 4)

    # ---- the loop + decode ---------------------------------------------------------------------------------------
    def _denoise(self, latents, prompt_embeds, negative_prompt_embeds, height, width, first_index, num_steps, guidance_scale,
                 inpaint_latents=None, control_latents=None, callback_on_step_end=None, callback_tensor_inputs=("latents",)):
        device = latents.device
        sampler = EasyAnimateSampler(self.transformer, vae=self.vae, scheduler=self.scheduler, guidance_scale=guidance_scale,
                                     cfg_group=self.cfg_group)
        cfgm = self.transformer.config
        rope = rope_table(height, width, latents.shape[2], cfgm.attention_head_dim, cfgm.patch_size, device=device)
        cfg_on = sampler.do_cfg
        embeds = (torch.cat([negative_prompt_embeds, prompt_embeds]) if cfg_on else prompt_embeds).to(device=device, dtype=bf16)
        latents = latents.to(bf16)
        self._num_timesteps = num_steps
        for k in range(num_steps):
            if self._interrupt:
                continue
            i = first_index + k
            latents = sampler.step(latents, i, embeds, rope, inpaint_latents, control_latents=control_latents)
            if callback_on_step_end is not None:
                have = {"latents": latents, "prompt_embeds": prompt_embeds, "negative_prompt_embeds": negative_prompt_embeds,
                        "prompt_embeds_2": None, "negative_prompt_embeds_2": None}
                got = callback_on_step_end(self, k, self.scheduler.timesteps[i], {n: have[n] for n in callback_tensor_inputs})
                latents = got.pop("latents", latents)
                if "prompt_embeds" in got or "negative_prompt_embeds" in got:
                    prompt_embeds = got.pop("prompt_embeds", prompt_embeds)
                    negative_prompt_embeds = got.pop("negative_prompt_embeds", negative_prompt_embeds)
                    embeds = (torch.cat([negative_prompt_embeds, prompt_embeds]) if cfg_on else prompt_embeds).to(device=device, dtype=bf16)
        self._sampler = sampler
        return latents

    def decode_latents(self, latents: torch.Tensor) -> np.ndarray:
        """pipeline_easyanimate.py:722-742: numpy float32 [B,3,F,H,W] in [0,1] (a view of the pinned host buffer the output
        kernel wrote)."""
        sampler = EasyAnimateSampler(self.transformer, vae=self.vae, scheduler=self.scheduler)
        return sampler.decode_latents(latents).numpy()

    def _finish(self, latents, output_type, return_dict):
        video = self.decode_latents(latents)
        if output_type == "latent":
            video = torch.from_numpy(video)
        return EasyAnimatePipelineOutput(frames=video) if return_dict else video

    def _prologue(self, prompt, height, width, guidance_scale, guidance_rescale, comfyui_progressbar, kw_check):
        if guidance_rescale and guidance_rescale > 0.0:
            raise NotImplementedError("guidance_rescale > 0 (rescale_noise_cfg) is not part of the fused CFG + Euler kernel")
        if comfyui_progressbar:
            raise NotImplementedError("comfyui_progressbar needs ComfyUI")
        height = int(height // 16 * 16)
        width = int(width // 16 * 16)
        self.check_inputs(prompt, height, width, **kw_check)
        self._guidance_scale, self._guidance_rescale, self._interrupt = guidance_scale, guidance_rescale, False
        return height, width

    def _embeds(self, prompt, negative_prompt, num_images_per_prompt, prompt_embeds, negative_prompt_embeds, prompt_attention_mask,
                negative_prompt_attention_mask):
        device, dtype = self._execution_device, self._dtype
        return self.encode_prompt(prompt=prompt, device=device, dtype=dtype, num_images_per_prompt=num_images_per_prompt,
                                  do_classifier_free_guidance=self.do_classifier_free_guidance, negative_prompt=negative_prompt,
                                  prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
                                  prompt_attention_mask=prompt_attention_mask,
                                  negative_prompt_attention_mask=negative_prompt_attention_mask, text_encoder_index=0)

    @staticmethod
    def _batch_size(prompt, prompt_embeds):
        if isinstance(prompt, str):
            return 1
        return len(prompt) if isinstance(prompt, list) else prompt_embeds.shape[0]


class EasyAnimatePipeline(_NativePipelineBase):
    """Text-to-video: pipeline_easyanimate.py:769-1148."""

    @torch.no_grad()
    def __call__(self, prompt: Union[str, List[str]] = None, video_length: Optional[int] = None, height: Optional[int] = None,
                 width: Optional[int] = None, num_inference_steps: Optional[int] = 50, guidance_scale: Optional[float] = 5.0,
                 negative_prompt: Optional[Union[str, List[str]]] = None, num_images_per_prompt: Optional[int] = 1,
                 eta: Optional[float] = 0.0, generator=None, latents: Optional[torch.Tensor] = None,
                 prompt_embeds: Optional[torch.Tensor] = None, prompt_embeds_2: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, negative_prompt_embeds_2: Optional[torch.Tensor] = None,
                 prompt_attention_mask: Optional[torch.Tensor] = None, prompt_attention_mask_2: Optional[torch.Tensor] = None,
                 negative_prompt_attention_mask: Optional[torch.Tensor] = None,
                 negative_prompt_attention_mask_2: Optional[torch.Tensor] = None, output_type: Optional[str] = "latent",
                 return_dict: bool = True, callback_on_step_end: Optional[Callable[..., Dict]] = None,
                 callback_on_step_end_tensor_inputs: List[str] = ["latents"], guidance_rescale: float = 0.0,
                 original_size: Optional[Tuple[int, int]] = (1024, 1024), target_size: Optional[Tuple[int, int]] = None,
                 crops_coords_top_left: Tuple[int, int] = (0, 0), comfyui_progressbar: bool = False,
                 timesteps: Optional[List[int]] = None):
        height, width = self._prologue(prompt, height, width, guidance_scale, guidance_rescale, comfyui_progressbar, dict(
            negative_prompt=negative_prompt, prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
            prompt_attention_mask=prompt_attention_mask, negative_prompt_attention_mask=negative_prompt_attention_mask,
            prompt_embeds_2=prompt_embeds_2, negative_prompt_embeds_2=negative_prompt_embeds_2,
            prompt_attention_mask_2=prompt_attention_mask_2, negative_prompt_attention_mask_2=negative_prompt_attention_mask_2,
            callback_on_step_end_tensor_inputs=callback_on_step_end_tensor_inputs))
        batch = self._batch_size(prompt, prompt_embeds)
        device, dtype = self._execution_device, self._dtype
        pe, ne, _, _ = self._embeds(prompt, negative_prompt, num_images_per_prompt, prompt_embeds, negative_prompt_embeds,
                                    prompt_attention_mask, negative_prompt_attention_mask)
        first, steps = self._set_timesteps(num_inference_steps, timesteps)
        shape = self._latent_shape(batch * num_images_per_prompt, self.transformer.config.in_channels, video_length, height, width)
        latents = randn_like_reference(shape, generator, device, dtype) if latents is None else latents.to(device)
        latents = self._denoise(latents, pe, ne, height, width, first, steps, guidance_scale,
                                callback_on_step_end=callback_on_step_end, callback_tensor_inputs=callback_on_step_end_tensor_inputs)
        return self._finish(latents, output_type, return_dict)


class EasyAnimateInpaintPipeline(_NativePipelineBase):
    """Image-to-video / video-to-video with the InP transformer (33 input channels = 16 latent + 1 mask + 16 masked-video
    latents): pipeline_easyanimate_inpaint.py:978-1604."""

    def _inpaint_latents(self, latents, init_video, mask_video, masked_video_latents, height, width, generator,
                         noise_aug_strength, device, dtype):
        """pipeline_easyanimate_inpaint.py:1320-1411 for the InP transformer -> [B, 1 + 16, F', h, w] (mask first)."""
        cfgm = self.transformer.config
        directly = self.transformer.resize_inpaint_mask_directly
        if mask_video is None or (cfgm.get("enable_zero_in_inpaint", True) and bool((mask_video == 255).all())):
            # nothing is given (pure text-to-video through the InP model): all-zero conditioning
            mask_latents = torch.zeros_like(latents)[:, :1] if directly else torch.zeros_like(latents)
            return torch.cat([mask_latents, torch.zeros_like(latents)], dim=1).to(device, dtype)
        mask = self._binarise_mask(mask_video, height, width)                      # 1 = to be generated
        if masked_video_latents is None:
            tile = torch.tile(mask, [1, 3, 1, 1, 1])
            masked = init_video * (tile < 0.5) + torch.ones_like(init_video) * (tile > 0.5) * -1
        else:
            masked = masked_video_latents
        masked = masked.to(device=device, dtype=dtype)
        if cfgm.add_noise_in_inpaint_model:
            masked = add_noise_to_reference_video(masked, ratio=noise_aug_strength, generator=generator)
        video_latents = self._encode_to_latents(masked, device, dtype).to(device=device, dtype=dtype)
        if directly:
            mask_latents = resize_mask(1 - mask, video_latents, self.vae.cache_mag_vae).to(device, dtype) * self.vae.config.scaling_factor
        else:
            mask_latents = self._encode_to_latents(torch.tile(mask, [1, 3, 1, 1, 1]), device, dtype)
        return torch.cat([mask_latents, video_latents], dim=1).to(dtype)

    @torch.no_grad()
    def __call__(self, prompt: Union[str, List[str]] = None, video_length: Optional[int] = None,
                 video: Optional[torch.Tensor] = None, mask_video: Optional[torch.Tensor] = None,
                 masked_video_latents: Optional[torch.Tensor] = None, height: Optional[int] = None, width: Optional[int] = None,
                 num_inference_steps: Optional[int] = 50, guidance_scale: Optional[float] = 5.0,
                 negative_prompt: Optional[Union[str, List[str]]] = None, num_images_per_prompt: Optional[int] = 1,
                 eta: Optional[float] = 0.0, generator=None, latents: Optional[torch.Tensor] = None,
                 prompt_embeds: Optional[torch.Tensor] = None, prompt_embeds_2: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, negative_prompt_embeds_2: Optional[torch.Tensor] = None,
                 prompt_attention_mask: Optional[torch.Tensor] = None, prompt_attention_mask_2: Optional[torch.Tensor] = None,
                 negative_prompt_attention_mask: Optional[torch.Tensor] = None,
                 negative_prompt_attention_mask_2: Optional[torch.Tensor] = None, output_type: Optional[str] = "latent",
                 return_dict: bool = True, callback_on_step_end: Optional[Callable[..., Dict]] = None,
                 callback_on_step_end_tensor_inputs: List[str] = ["latents"], guidance_rescale: float = 0.0,
                 original_size: Optional[Tuple[int, int]] = (1024, 1024), target_size: Optional[Tuple[int, int]] = None,
                 crops_coords_top_left: Tuple[int, int] = (0, 0), clip_image=None, clip_apply_ratio: float = 0.40,
                 strength: float = 1.0, noise_aug_strength: float = 0.0563, comfyui_progressbar: bool = False,
                 timesteps: Optional[List[int]] = None):
        height, width = self._prologue(prompt, height, width, guidance_scale, guidance_rescale, comfyui_progressbar, dict(
            negative_prompt=negative_prompt, prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
            prompt_attention_mask=prompt_attention_mask, negative_prompt_attention_mask=negative_prompt_attention_mask,
            prompt_embeds_2=prompt_embeds_2, negative_prompt_embeds_2=negative_prompt_embeds_2,
            prompt_attention_mask_2=prompt_attention_mask_2, negative_prompt_attention_mask_2=negative_prompt_attention_mask_2,
            callback_on_step_end_tensor_inputs=callback_on_step_end_tensor_inputs))
        n_lat, n_tr = self.vae.config.latent_channels, self.transformer.config.in_channels
        if n_tr == n_lat:
            raise NotImplementedError("blending-style inpainting with a 16-channel transformer is not carried over: use the InP model")
        if clip_image is not None and getattr(self.transformer, "enable_clip_in_inpaint", False):
            raise NotImplementedError("the CLIP-image branch (enable_clip_in_inpaint) is not carried over (V5.1 does not use it)")
        batch = self._batch_size(prompt, prompt_embeds) * num_images_per_prompt
        device, dtype = self._execution_device, self._dtype
        pe, ne, _, _ = self._embeds(prompt, negative_prompt, num_images_per_prompt, prompt_embeds, negative_prompt_embeds,
                                    prompt_attention_mask, negative_prompt_attention_mask)
        first, steps = self._set_timesteps(num_inference_steps, timesteps, strength)
        init_video = None
        if video is not None:
            video_length = video.shape[2]
            init_video = self._normalise_video(video, height, width)
        shape = self._latent_shape(batch, n_lat, video_length, height, width)
        if latents is None:
            noise = randn_like_reference(shape, generator, device, dtype)
            if strength == 1.0:
                latents = noise
            else:  # start from the encoded video noised to the first timestep (scale_noise), inpaint :876-899
                video_latents = self._encode_to_latents(init_video, device, dtype)
                video_latents = video_latents.repeat(batch // video_latents.shape[0], 1, 1, 1, 1)
                latents = self.scheduler.scale_noise(video_latents.to(dtype), None, noise, index=first)
        else:
            latents = latents.to(device)
        if init_video is None and mask_video is not None:
            raise ValueError("`mask_video` needs `video`")
        inpaint = self._inpaint_latents(latents, init_video, mask_video, masked_video_latents, height, width, generator,
                                        noise_aug_strength, device, dtype)
        if n_lat + inpaint.shape[1] != n_tr:
            raise ValueError(f"Incorrect configuration settings! The config of `pipeline.transformer`: {self.transformer.config} "
                             f"expects {n_tr} but received `num_channels_latents`: {n_lat} + `num_channels_mask`: "
                             f"{inpaint.shape[1] - n_lat} + `num_channels_masked_image`: {n_lat} = {n_lat + inpaint.shape[1]}. "
                             "Please verify the config of `pipeline.transformer` or your `mask_image` or `image` input.")
        latents = self._denoise(latents, pe, ne, height, width, first, steps, guidance_scale, inpaint_latents=inpaint,
                                callback_on_step_end=callback_on_step_end, callback_tensor_inputs=callback_on_step_end_tensor_inputs)
        return self._finish(latents, output_type, return_dict)


class EasyAnimateControlPipeline(_NativePipelineBase):
    """Control (pose / depth / canny video, camera trajectories, reference image): pipeline_easyanimate_control.py:833-1282."""

    @torch.no_grad()
    def __call__(self, prompt: Union[str, List[str]] = None, video_length: Optional[int] = None, height: Optional[int] = None,
                 width: Optional[int] = None, control_video: Optional[torch.Tensor] = None,
                 control_camera_video: Optional[torch.Tensor] = None, ref_image: Optional[torch.Tensor] = None,
                 num_inference_steps: Optional[int] = 50, guidance_scale: Optional[float] = 5.0,
                 negative_prompt: Optional[Union[str, List[str]]] = None, num_images_per_prompt: Optional[int] = 1,
                 eta: Optional[float] = 0.0, generator=None, latents: Optional[torch.Tensor] = None,
                 prompt_embeds: Optional[torch.Tensor] = None, prompt_embeds_2: Optional[torch.Tensor] = None,
                 negative_prompt_embeds: Optional[torch.Tensor] = None, negative_prompt_embeds_2: Optional[torch.Tensor] = None,
                 prompt_attention_mask: Optional[torch.Tensor] = None, prompt_attention_mask_2: Optional[torch.Tensor] = None,
                 negative_prompt_attention_mask: Optional[torch.Tensor] = None,
                 negative_prompt_attention_mask_2: Optional[torch.Tensor] = None, output_type: Optional[str] = "latent",
                 return_dict: bool = True, callback_on_step_end: Optional[Callable[..., Dict]] = None,
                 callback_on_step_end_tensor_inputs: List[str] = ["latents"], guidance_rescale: float = 0.0,
                 original_size: Optional[Tuple[int, int]] = (1024, 1024), target_size: Optional[Tuple[int, int]] = None,
                 crops_coords_top_left: Tuple[int, int] = (0, 0), comfyui_progressbar: bool = False,
                 timesteps: Optional[List[int]] = None):
        height, width = self._prologue(prompt, height, width, guidance_scale, guidance_rescale, comfyui_progressbar, dict(
            negative_prompt=negative_prompt, prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds,
            prompt_attention_mask=prompt_attention_mask, negative_prompt_attention_mask=negative_prompt_attention_mask,
            prompt_embeds_2=prompt_embeds_2, negative_prompt_embeds_2=negative_prompt_embeds_2,
            prompt_attention_mask_2=prompt_attention_mask_2, negative_prompt_attention_mask_2=negative_prompt_attention_mask_2,
            callback_on_step_end_tensor_inputs=callback_on_step_end_tensor_inputs))
        batch = self._batch_size(prompt, prompt_embeds) * num_images_per_prompt
        device, dtype = self._execution_device, self._dtype
        pe, ne, _, _ = self._embeds(prompt, negative_prompt, num_images_per_prompt, prompt_embeds, negative_prompt_embeds,
                                    prompt_attention_mask, negative_prompt_attention_mask)
        first, steps = self._set_timesteps(num_inference_steps, timesteps)
        n_lat = self.vae.config.latent_channels
        shape = self._latent_shape(batch, n_lat, video_length, height, width)
        latents = randn_like_reference(shape, generator, device, dtype) if latents is None else latents.to(device)
        # control_latents (pipeline_easyanimate_control.py:1063-1125): camera trajectories resized like a mask and scaled by 6,
        # or the encoded control video, or zeros; then the reference image's latent in frame 0 of 16 further channels
        if control_camera_video is not None:
            control = (resize_mask(control_camera_video, latents, process_first_frame_only=True) * 6).to(device, dtype)
        elif control_video is not None:
            control = self._encode_to_latents(self._normalise_video(control_video, height, width), device, dtype)
        else:
            control = torch.zeros_like(latents).to(device, dtype)
        if ref_image is not None:
            ref_lat = self._encode_to_latents(self._normalise_video(ref_image, height, width), device, dtype)
            slot = torch.zeros_like(latents)
            if latents.shape[2] != 1:
                slot[:, :, :1] = ref_lat
            control = torch.cat([control, slot.to(device, dtype)], dim=1)
        elif self.transformer.config.get("add_ref_latent_in_control_model", False):
            control = torch.cat([control, torch.zeros_like(latents).to(device, dtype)], dim=1)
        latents = self._denoise(latents, pe, ne, height, width, first, steps, guidance_scale, control_latents=control,
                                callback_on_step_end=callback_on_step_end, callback_tensor_inputs=callback_on_step_end_tensor_inputs)
        return self._finish(latents, output_type, return_dict)


def load_pipeline(model_name: str, config: Union[str, dict, None] = None, weight_dtype=bf16, device="cuda",
                  transformer_path: Optional[str] = None, vae_path: Optional[str] = None, load_text_encoder: bool = True,
                  cfg_group=None):
    """The loading sequence of predict_t2v.py:94-255 / predict_i2v.py for a released EasyAnimateV5.1 directory
    (`transformer/`, `vae/`, `scheduler/`, `tokenizer/`, `text_encoder/`), ending in the pipeline object those scripts build:
    `EasyAnimateInpaintPipeline` when the transformer has more input channels than the VAE has latent channels (the InP /
    I2V checkpoints), else `EasyAnimatePipeline`.

    config: the model YAML the scripts read (config/easyanimate_video_v5.1_magvit_qwen.yaml) as a path or a dict with
    `transformer_additional_kwargs` / `vae_kwargs` / `text_encoder_kwargs`; None = the V5.1 values.
    transformer_path / vae_path: optional fine-tuned weights loaded over the released ones (non-strict, like the scripts).
    load_text_encoder: the Qwen2-VL tokenizer and text encoder through `transformers` when their folders exist; without them
    the pipeline takes `prompt_embeds` (+ masks) instead of prompt strings."""
    import os

    from .autoencoder_magvit import AutoencoderKLMagvit
    from .transformer3d import EasyAnimateTransformer3DModel

    if config is None:
        config = {"transformer_additional_kwargs": {"transformer_type": "EasyAnimateTransformer3DModel", "after_norm": False,
                                                    "time_position_encoding_type": "3d_rope", "resize_inpaint_mask_directly": True,
                                                    "enable_text_attention_mask": True, "enable_clip_in_inpaint": False,
                                                    "add_ref_latent_in_control_model": True},
                  "vae_kwargs": {"vae_type": "AutoencoderKLMagvit", "mini_batch_encoder": 4, "mini_batch_decoder": 1,
                                 "slice_mag_vae": False, "slice_compression_vae": False, "cache_compression_vae": False,
                                 "cache_mag_vae": True},
                  "text_encoder_kwargs": {"enable_multi_text_encoder": False, "replace_t5_to_llm": True}}
    elif isinstance(config, str):
        import yaml
        with open(config) as f:
            config = yaml.safe_load(f)
    tkw = dict(config.get("transformer_additional_kwargs", {}))
    if tkw.get("transformer_type", "EasyAnimateTransformer3DModel") != "EasyAnimateTransformer3DModel":
        raise NotImplementedError(f"transformer_type {tkw.get('transformer_type')}: only the V5 / V5.1 EasyAnimateTransformer3DModel")
    if config.get("vae_kwargs", {}).get("vae_type", "AutoencoderKLMagvit") != "AutoencoderKLMagvit":
        raise NotImplementedError("only the MagViT VAE (vae_type AutoencoderKLMagvit)")
    if config.get("text_encoder_kwargs", {}).get("enable_multi_text_encoder", False):
        raise NotImplementedError("enable_multi_text_encoder (EasyAnimate V5 Bert + T5) is not carried over")

    def overlay(module, path):
        if path.endswith("safetensors"):
            from safetensors.torch import load_file
            state = load_file(path)
        else:
            state = torch.load(path, map_location="cpu")
        state = state["state_dict"] if "state_dict" in state else state
        return module.load_state_dict(state, strict=False)

    transformer = EasyAnimateTransformer3DModel.from_pretrained_2d(model_name, subfolder="transformer",
                                                                   transformer_additional_kwargs=tkw, torch_dtype=weight_dtype,
                                                                   low_cpu_mem_usage=True)
    if transformer_path is not None:
        overlay(transformer, transformer_path)
    vae = AutoencoderKLMagvit.from_pretrained(model_name, subfolder="vae",
                                              vae_additional_kwargs=dict(config.get("vae_kwargs", {}))).to(weight_dtype)
    if vae_path is not None:
        overlay(vae, vae_path)
    tokenizer = text_encoder = None
    if load_text_encoder and os.path.isdir(os.path.join(model_name, "tokenizer")) and os.path.isdir(os.path.join(model_name, "text_encoder")):
        from transformers import Qwen2Tokenizer, Qwen2VLForConditionalGeneration
        tokenizer = Qwen2Tokenizer.from_pretrained(os.path.join(model_name, "tokenizer"))
        text_encoder = Qwen2VLForConditionalGeneration.from_pretrained(os.path.join(model_name, "text_encoder"),
                                                                       torch_dtype=weight_dtype).to(device)
    scheduler = (FlowMatchEulerDiscreteScheduler.from_pretrained(model_name, subfolder="scheduler")
                 if os.path.isfile(os.path.join(model_name, "scheduler", "scheduler_config.json")) else FlowMatchEulerDiscreteScheduler())
    kind = EasyAnimateInpaintPipeline if transformer.config.in_channels != vae.config.latent_channels else EasyAnimatePipeline
    return kind(vae=vae.to(device), transformer=transformer.to(device), scheduler=scheduler, tokenizer=tokenizer,
                text_encoder=text_encoder, cfg_group=cfg_group)

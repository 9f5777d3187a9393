"""Public sampling API of easyanimate_b200: the denoise loop of ``EasyAnimatePipeline.__call__`` + ``decode_latents``
(/root/reference/easyanimate/pipeline/pipeline_easyanimate.py:998-1011,1052-1137,722-742) on the H100 modules, for
callers that do not go through diffusers' ``DiffusionPipeline`` (bench.py, smoke tests, services that feed
pre-computed text embeddings).  The reference pipelines themselves can be handed
``easyanimate_b200.EasyAnimateTransformer3DModel`` / ``AutoencoderKLMagvit`` / ``FlowMatchEulerDiscreteScheduler``
objects directly (INTEGRATION.md).

Multi-GPU: with ``cfg_group`` (a 2-rank torch.distributed group) the two classifier-free-guidance branches, which
the reference evaluates as one batch of 2 on one GPU (pipeline_easyanimate.py:1074,1103), run on two GPUs and exchange
the 6 MB noise prediction with one all_gather per step.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch

from . import ops
from .scheduler import FlowMatchEulerDiscreteScheduler

bf16 = torch.bfloat16


# ---------------------------------------------------------------------------------------------------------------
# 3-D RoPE table (host, once per call) — pipeline_easyanimate.py:82-97,998-1011 + diffusers get_3d_rotary_pos_embed
# ---------------------------------------------------------------------------------------------------------------
def get_resize_crop_region_for_grid(src, tgt_width, tgt_height):
    tw, th = tgt_width, tgt_height
    h, w = src
    r = h / w
    if r > (th / tw):
        resize_height, resize_width = th, int(round(th / h * w))
    else:
        resize_width, resize_height = tw, int(round(tw / w * h))
    crop_top = int(round((th - resize_height) / 2.0))
    crop_left = int(round((tw - resize_width) / 2.0))
    return (crop_top, crop_left), (crop_top + resize_height, crop_left + resize_width)


def _axis_freqs(dim: int, pos: np.ndarray, theta: float = 10000.0):
    inv = 1.0 / (theta ** (torch.arange(0, dim, 2)[: dim // 2].float() / dim))
    f = torch.outer(torch.from_numpy(pos).float(), inv)
    return f.cos().repeat_interleave(2, dim=1).float(), f.sin().repeat_interleave(2, dim=1).float()


def rope_table(height: int, width: int, latent_frames: int, head_dim: int = 64, patch_size: int = 2,
               device=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(cos, sin), each [F*H/16*W/16, head_dim] fp32, for a video of `height` x `width` pixels."""
    gh, gw = height // 8 // patch_size, width // 8 // patch_size
    base_w, base_h = 720 // 8 // patch_size, 480 // 8 // patch_size
    (top, left), (bottom, right) = get_resize_crop_region_for_grid((gh, gw), base_w, base_h)
    grid_h = np.linspace(top, bottom, gh, endpoint=False, dtype=np.float32)
    grid_w = np.linspace(left, right, gw, endpoint=False, dtype=np.float32)
    grid_t = np.linspace(0, latent_frames, latent_frames, endpoint=False, dtype=np.float32)
    dt, dh, dw = head_dim // 4, head_dim // 8 * 3, head_dim // 8 * 3
    (tc, ts), (hc, hs), (wc, ws) = _axis_freqs(dt, grid_t), _axis_freqs(dh, grid_h), _axis_freqs(dw, grid_w)

    def combine(t, h, w):
        t = t[:, None, None, :].expand(-1, gh, gw, -1)
        h = h[None, :, None, :].expand(latent_frames, -1, gw, -1)
        w = w[None, None, :, :].expand(latent_frames, gh, -1, -1)
        return torch.cat([t, h, w], dim=-1).reshape(latent_frames * gh * gw, -1).contiguous()

    cos, sin = combine(tc, hc, wc), combine(ts, hs, ws)
    if device is not None:
        cos, sin = cos.to(device), sin.to(device)
    return cos, sin


# ---------------------------------------------------------------------------------------------------------------
class EasyAnimateSampler:
    """Denoise loop + VAE decode on device-resident tensors, with an optional host-buffer entry point."""

    def __init__(self, transformer, vae=None, scheduler: Optional[FlowMatchEulerDiscreteScheduler] = None,
                 guidance_scale: float = 6.0, cfg_group=None, euler_fn=None):
        self.transformer = transformer
        # CFG combine + Euler update kernel; injectable so the multi-rank host logic can be unit-tested on CPU (gloo)
        self._euler = euler_fn or ops.cfg_euler_step
        self.vae = vae
        self.scheduler = scheduler or FlowMatchEulerDiscreteScheduler()
        self.guidance_scale = guidance_scale
        self.do_cfg = guidance_scale > 1.0
        self.cfg_group = cfg_group
        self._cfg_rank = None
        if cfg_group is not None:
            import torch.distributed as dist
            assert dist.get_world_size(cfg_group) == 2, "CFG-parallel needs a group of exactly 2 ranks"
            self._cfg_rank = dist.get_rank(cfg_group)
            if hasattr(transformer, "set_cfg_parallel_group"):
                transformer.set_cfg_parallel_group(cfg_group)  # TeaCache decisions from the joint batch of 2

    def set_timesteps(self, num_inference_steps: int, device=None):
        self.scheduler.set_timesteps(num_inference_steps, device=device, mu=1.0)  # pipeline_easyanimate.py:972
        return self.scheduler.timesteps

    # -- one scheduler step ------------------------------------------------------------------------------------
    def step(self, latents: torch.Tensor, i: int, embeds: torch.Tensor, rope, inpaint_latents=None, control_latents=None) -> torch.Tensor:
        """latents [B,C,F,h,w]; embeds [2B,S_t,E] = cat(negative, positive) when CFG is on (pipeline_easyanimate.py:1052-1056).
        inpaint_latents / control_latents: [B,...] (the same conditioning for both branches, what
        pipeline_easyanimate_inpaint.py:1496-1511 and pipeline_easyanimate_control.py:1066-1125 build with cat([x] * 2)) or
        [2B,...] = cat(unconditional-branch, text-branch) conditioning."""
        t = self.scheduler.timesteps[i]
        sigma, sigma_next = self.scheduler.sigma_pair(i)
        B = latents.shape[0]
        extra = {}  # keyword only when given: the plain text-to-video call stays exactly the call the GPU suite validated
        if not self.do_cfg:
            if control_latents is not None:
                extra["control_latents"] = control_latents
            t_expand = t.reshape(1).expand(B).to(device=latents.device, dtype=bf16)
            pred = self.transformer(latents, t_expand, encoder_hidden_states=embeds, image_rotary_emb=rope,
                                    inpaint_latents=inpaint_latents, return_dict=False, **extra)[0]
            return self._euler(pred, latents, 1.0, sigma, sigma_next, use_cfg=False)
        if self.cfg_group is None:
            latent_in = torch.cat([latents] * 2)
            inp = inpaint_latents
            if inp is not None and inp.shape[0] == B:
                inp = torch.cat([inp] * 2)
            if control_latents is not None:
                extra["control_latents"] = torch.cat([control_latents] * 2) if control_latents.shape[0] == B else control_latents
            t_expand = t.reshape(1).expand(2 * B).to(device=latents.device, dtype=bf16)
            pred = self.transformer(latent_in, t_expand, encoder_hidden_states=embeds, image_rotary_emb=rope,
                                    inpaint_latents=inp, return_dict=False, **extra)[0]
        else:
            import torch.distributed as dist
            r = self._cfg_rank  # rank 0: unconditional branch, rank 1: text-conditioned branch
            t_expand = t.reshape(1).expand(B).to(device=latents.device, dtype=bf16)
            inp = inpaint_latents
            if inp is not None and inp.shape[0] == 2 * B:
                inp = inp[r * B:(r + 1) * B].contiguous()
            if control_latents is not None:
                extra["control_latents"] = (control_latents[r * B:(r + 1) * B].contiguous() if control_latents.shape[0] == 2 * B
                                            else control_latents)
            mine = self.transformer(latents, t_expand, encoder_hidden_states=embeds[r * B:(r + 1) * B].contiguous(),
                                    image_rotary_emb=rope, inpaint_latents=inp, return_dict=False, **extra)[0]
            pred = torch.empty((2 * B,) + tuple(mine.shape[1:]), device=mine.device, dtype=mine.dtype)
            dist.all_gather_into_tensor(pred, mine.contiguous(), group=self.cfg_group)
        return self._euler(pred, latents, self.guidance_scale, sigma, sigma_next, use_cfg=True)

    def step_from_host(self, latents_host: torch.Tensor, i: int, embeds_host: torch.Tensor, rope,
                       out_host: Optional[torch.Tensor] = None, device="cuda", inpaint_latents=None) -> torch.Tensor:
        """Same step with HOST (pinned) inputs and output: H2D of the step's inputs and D2H of its result included."""
        lat = latents_host.to(device, non_blocking=True)
        emb = embeds_host.to(device, non_blocking=True)
        new = self.step(lat, i, emb, rope, inpaint_latents)
        if out_host is None:
            out_host = torch.empty(new.shape, dtype=new.dtype, pin_memory=True)
        out_host.copy_(new, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return out_host

    # -- full loop ---------------------------------------------------------------------------------------------
    @torch.no_grad()
    def sample(self, latents: torch.Tensor, prompt_embeds: torch.Tensor, negative_prompt_embeds: Optional[torch.Tensor],
               height: int, width: int, num_inference_steps: int, inpaint_latents=None, decode: bool = False):
        dev = latents.device
        self.set_timesteps(num_inference_steps, device="cpu")
        rope = rope_table(height, width, latents.shape[2], self.transformer.config.attention_head_dim,
                          self.transformer.config.patch_size, device=dev)
        embeds = torch.cat([negative_prompt_embeds, prompt_embeds]) if self.do_cfg else prompt_embeds
        embeds = embeds.to(device=dev, dtype=bf16)
        latents = latents.to(bf16)
        for i in range(num_inference_steps):
            latents = self.step(latents, i, embeds, rope, inpaint_latents)
        if decode:
            return self.decode_latents(latents)
        return latents

    @torch.no_grad()
    def decode_latents(self, latents: torch.Tensor, out: Optional[torch.Tensor] = None, dtype=torch.float32,
                       to_host: bool = True) -> torch.Tensor:
        """pipeline_easyanimate.py:722-742: /scaling_factor -> vae.decode -> clamp(-1,1) -> /2+.5 -> clamp(0,1) ->
        `.cpu().float()`: returns the [B,3,T,H,W] float32 frames in (pinned) HOST memory by default - `torch.from_numpy` /
        `.numpy()` views of it are what the reference pipeline hands back as `.frames` (:1136-1148).  No torch arithmetic:
        the scale rides in the latent-preparation kernel, the tail is `ea_frames_out` (AutoencoderKLMagvit.decode_scaled)."""
        return self.vae.decode_scaled(latents.to(bf16), out=out, dtype=dtype, to_host=to_host)

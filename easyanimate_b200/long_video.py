"""Long-video generation: the reference's "Long Video Generation" mode (easyanimate/ui/ui.py:485-552, also behind
api/api.py:107) on the native inpaint pipeline.

EasyAnimateV5.1 makes at most 49 frames per call.  Longer videos are made window after window: each window after the first
is an image-to-video call conditioned on the last `overlap_video_length` frames of the video so far, its first
`overlap_video_length` frames are cross-faded into that tail and the rest is appended.  Every window's frames stay on the
GPU until `ea_frames_out_blend` writes them, cross-faded, into the pinned host buffer of the whole video; the frames that
condition the next window are made on the device by `ea_frames_out` (uint8 = trunc(255 * v), what ui.py:540-544 gets from
`(x * 255).numpy().astype(np.uint8)` and PIL).  The PIL round trip of ui.py is an exact copy: `Image.fromarray` then
`resize` to the size the image already has returns the same pixels, so the uint8 frames condition the next window as they are."""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np
import torch

from . import vae_ops
from .pipelines import EasyAnimateInpaintPipeline, EasyAnimatePipelineOutput

# uint8 -> float32 as the reference's `uint8_tensor / 255` computes it on the CPU (a true division; torch on CUDA multiplies
# by float32(1/255) instead, which differs in the last bit for some values)
_UNIT = torch.arange(256, dtype=torch.float32) / 255


def long_video_windows(video_length: int, partial_video_length: int, overlap_video_length: int, mini_batch_encoder: int = 4,
                       cache_mag_vae: bool = True) -> List[Tuple[int, int]]:
    """(first frame, frame count) of each window, in the order ui.py:488-549 runs them: `partial_video_length` frames per
    window; the window that reaches `video_length` gets the rest, rounded down to 1 + 4m frames (m * 4 without cache_mag_vae),
    and a rest that rounds to <= 0 frames ends the loop; the next window starts `overlap_video_length` frames before the
    previous one ends."""
    windows = []
    init_frames, last_frames = 0, partial_video_length
    while init_frames < video_length:
        if last_frames >= video_length:
            n = video_length - init_frames
            n = (n - 1) // mini_batch_encoder * mini_batch_encoder + 1 if cache_mag_vae else n // mini_batch_encoder * mini_batch_encoder
            if n <= 0:
                break
        else:
            n = partial_video_length
        windows.append((init_frames, n))
        if last_frames >= video_length:
            break
        init_frames += n - overlap_video_length
        last_frames = init_frames + n
    return windows


def _frames_u8(images, height: int, width: int, device) -> torch.Tensor:
    """PIL image(s) resized like get_image_to_video_latent (utils.py:75-120) does, or uint8 [3,H,W] / [n,3,H,W] tensors ->
    uint8 [3, n, H, W] on `device`."""
    if isinstance(images, torch.Tensor):
        t = images[None] if images.dim() == 3 else images
        if t.dtype != torch.uint8 or t.dim() != 4 or tuple(t.shape[1:]) != (3, height, width):
            raise ValueError(f"image tensors must be uint8 [3, {height}, {width}] or [n, 3, {height}, {width}], got "
                             f"{t.dtype} {list(images.shape)}")
        return t.to(device).permute(1, 0, 2, 3)
    arrays = [np.array(im.resize([width, height])) for im in (images if isinstance(images, list) else [images])]
    if not arrays or any(a.shape != (height, width, 3) for a in arrays):
        raise ValueError("start_image / end_image must be RGB images")
    return torch.from_numpy(np.stack(arrays)).to(device).permute(3, 0, 1, 2)


def _conditioning(start: Optional[torch.Tensor], end: Optional[torch.Tensor], n: int, height: int, width: int, device):
    """get_image_to_video_latent (utils.py:75-160) for uint8 start / end frames [3, k, H, W]: video [1,3,n,H,W] in [0, 1] (the
    first start frame everywhere, the start frames first and the end frames last) and mask_video [1,1,n,H,W], 0 on the given
    frames and 255 on the frames to generate.  No start frame: zeros and 255 everywhere."""
    if start is None:
        return (torch.zeros((1, 3, n, height, width), device=device),
                torch.full((1, 1, n, height, width), 255.0, device=device))
    video = start[:, :1].repeat(1, n, 1, 1)
    video[:, :start.shape[1]] = start
    mask = torch.zeros((1, 1, n, height, width), device=device)
    mask[:, :, start.shape[1]:] = 255
    if end is not None:
        video[:, n - end.shape[1]:] = end
        mask[:, :, n - end.shape[1]:] = 0
    return _UNIT.to(device)[video.long()][None], mask


@torch.no_grad()
def generate_long_video(pipe, prompt=None, *, video_length: int, partial_video_length: int, overlap_video_length: int = 4,
                        start_image=None, end_image=None, height: int, width: int, num_inference_steps: int,
                        guidance_scale: float, generator=None, negative_prompt=None, **pipe_kwargs) -> EasyAnimatePipelineOutput:
    """A video of up to `video_length` frames from overlapping image-to-video windows of `partial_video_length` frames, as
    the reference's "Long Video Generation" mode makes it (ui.py:485-552).

    pipe: an `EasyAnimateInpaintPipeline` (what `load_pipeline` builds for an InP checkpoint).
    start_image / end_image: a PIL image or a list of them (resized to width x height like the reference), or uint8 tensors
    [3,H,W] / [n,3,H,W].  The start image conditions the first window, `end_image` the last one.
    generator: one generator for all windows, so the noise of each window continues the random stream of the one before.
    pipe_kwargs: further keyword arguments of the pipeline call (prompt embeddings and masks, noise_aug_strength, ...).

    Returns `EasyAnimatePipelineOutput(frames=[1, 3, L, H, W] float32)` in pinned host memory, L = the end of the last
    window.  With a `cfg_group` or a strip-parallel VAE every rank returns the whole video.  Raises ValueError for what the
    reference refuses (a pipeline that is not image-to-video, `video=`, an end image without a start image) and for windows
    it would not run to completion: an overlap outside [1, partial_video_length), windows the VAE cannot decode to their
    length, a last window shorter than the overlap, or a window whose chained frames would include cross-faded ones
    (partial_video_length < 2 * overlap_video_length with three or more windows)."""
    if not isinstance(pipe, EasyAnimateInpaintPipeline) or \
            pipe.transformer.config.in_channels == pipe.vae.config.latent_channels:
        raise ValueError("Please select an image to video pretrained model while using long video generation.")
    if pipe_kwargs.get("video") is not None:
        raise ValueError("Video to Video is not Support Long Video Generation now.")
    own = sorted(k for k in ("video", "mask_video", "masked_video_latents", "latents", "strength", "video_length",
                             "output_type", "return_dict") if k in pipe_kwargs)
    if own:
        raise ValueError(f"generate_long_video sets {own} for each window itself")
    if start_image is None and end_image is not None:
        raise ValueError("If specifying the ending image of the video, please specify a starting image of the video.")
    if height % 16 or width % 16:
        raise ValueError(f"height and width must be multiples of 16, got {height} x {width}")
    pe = pipe_kwargs.get("prompt_embeds")
    if (isinstance(prompt, list) and len(prompt) != 1) or (pe is not None and pe.shape[0] != 1) or \
            pipe_kwargs.get("num_images_per_prompt", 1) != 1:
        raise ValueError("generate_long_video makes one video: one prompt, num_images_per_prompt = 1")
    ov = overlap_video_length
    if not 1 <= ov < partial_video_length:
        raise ValueError(f"overlap_video_length must be in [1, partial_video_length), got {ov} and {partial_video_length}")
    vae = pipe.vae
    mbe = vae.mini_batch_encoder
    if (partial_video_length - 1 if vae.cache_mag_vae else partial_video_length) % mbe:
        raise ValueError(f"partial_video_length must be {'1 + ' if vae.cache_mag_vae else ''}a multiple of {mbe}, "
                         f"got {partial_video_length}")
    windows = long_video_windows(video_length, partial_video_length, ov, mbe, vae.cache_mag_vae)
    if not windows:
        raise ValueError(f"video_length {video_length} gives no window")
    if len(windows) > 1 and windows[-1][1] < ov:
        raise ValueError(f"the last window has {windows[-1][1]} frames, fewer than overlap_video_length = {ov}")
    if len(windows) > 2 and partial_video_length < 2 * ov:
        raise ValueError(f"partial_video_length = {partial_video_length} < 2 * overlap_video_length: a window would be"
                         " conditioned on cross-faded frames")

    device = pipe._execution_device
    length = windows[-1][0] + windows[-1][1]
    out = torch.empty((1, 3, length, height, width), dtype=torch.float32, pin_memory=device.type == "cuda")
    start = None if start_image is None else _frames_u8(start_image, height, width, device)
    end = None if end_image is None else _frames_u8(end_image, height, width, device)
    for k, (t0, n) in enumerate(windows):
        last = k == len(windows) - 1
        video, mask = _conditioning(start, end if last else None, n, height, width, device)
        latents = pipe.denoise_to_latents(prompt, video_length=n, video=video, mask_video=mask, height=height, width=width,
                                          num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                                          generator=generator, negative_prompt=negative_prompt, strength=1, **pipe_kwargs)
        with pipe._on_device("vae"):  # model CPU offload: the VAE visits the GPU for the decode only
            frames = vae.decode_scaled_video(latents).contiguous()
        if tuple(frames.shape) != (1, 3, n, height, width):
            raise ValueError(f"window {k} decoded to {list(frames.shape)}, expected [1, 3, {n}, {height}, {width}]")
        vae_ops.frames_out_blend(frames, out[:, :, t0:t0 + n], ov if k else 0)
        if not last:  # the next window's start frames: the last `ov` frames, as uint8
            tail = torch.empty((3, ov, height, width), dtype=torch.uint8, device=device)
            start = vae_ops.frames_out(frames[0, :, n - ov:].contiguous(), tail)
    if out.is_pinned():
        torch.cuda.current_stream(device).synchronize()
    return EasyAnimatePipelineOutput(frames=out)

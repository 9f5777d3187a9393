"""ORACLE (test infrastructure only): the reference's "Long Video Generation" loop (easyanimate/ui/ui.py:485-552) restated
over any pipeline with the reference's call signature - in tests/test_long_video_cpu.py the reference's own
`EasyAnimateInpaintPipeline` (oracle/ref_pipeline.py) - with PIL for the chained frames, and `get_image_to_video_latent`
(easyanimate/utils/utils.py:75-160) restated for PIL images and lists of them."""
import numpy as np
import torch
from PIL import Image


def _stack(images):
    return torch.cat([torch.from_numpy(np.array(im)).permute(2, 0, 1).unsqueeze(1).unsqueeze(0) for im in images], dim=2)


def get_image_to_video_latent(image_start, image_end, video_length, sample_size):
    """utils.py:75-160 for PIL inputs: (input_video [1,3,F,H,W] in [0,1], input_video_mask [1,1,F,H,W] in {0,255})."""
    if image_start is None:
        return (torch.zeros([1, 3, video_length, sample_size[0], sample_size[1]]),
                torch.ones([1, 1, video_length, sample_size[0], sample_size[1]]) * 255)
    size = [sample_size[1], sample_size[0]]
    if isinstance(image_start, list):
        image_start = [im.resize(size) for im in image_start]
        start_video = _stack(image_start)
        input_video = torch.tile(start_video[:, :, :1], [1, 1, video_length, 1, 1])
        input_video[:, :, :len(image_start)] = start_video
        first = len(image_start)
    else:
        image_start = image_start.resize(size)
        input_video = torch.tile(_stack([image_start]), [1, 1, video_length, 1, 1])
        first = 1
    input_video_mask = torch.zeros_like(input_video[:, :1])
    input_video_mask[:, :, first:] = 255
    if image_end is not None:
        ends = [im.resize(size) for im in (image_end if isinstance(image_end, list) else [image_end])]
        input_video[:, :, -len(ends):] = _stack(ends)
        input_video_mask[:, :, -len(ends):] = 0
    return input_video / 255, input_video_mask


def long_video(pipe, *, length_slider, partial_video_length, overlap_video_length, start_image, end_image, height, width,
               mini_batch_encoder=4, cache_mag_vae=True, **call_kw):
    """ui.py:485-552: returns (frames [1,3,L,H,W] float32, [(window length, start frame), ...]).  `call_kw` are the further
    keyword arguments of the pipeline call (prompt embeddings, steps, guidance, generator...)."""
    windows = []
    init_frames = 0
    last_frames = init_frames + partial_video_length
    new_sample = None
    while init_frames < length_slider:
        if last_frames >= length_slider:
            _partial_video_length = length_slider - init_frames
            if cache_mag_vae:
                _partial_video_length = int((_partial_video_length - 1) // mini_batch_encoder * mini_batch_encoder) + 1
            else:
                _partial_video_length = int(_partial_video_length // mini_batch_encoder * mini_batch_encoder)
            if _partial_video_length <= 0:
                break
        else:
            _partial_video_length = partial_video_length
        windows.append((init_frames, _partial_video_length))
        input_video, input_video_mask = get_image_to_video_latent(
            start_image, end_image if last_frames >= length_slider else None, _partial_video_length, (height, width))
        with torch.no_grad():
            sample = pipe(height=height, width=width, video_length=_partial_video_length, video=input_video,
                          mask_video=input_video_mask, strength=1, **call_kw).frames
        if init_frames != 0:
            mix_ratio = torch.from_numpy(np.array([float(i) / float(overlap_video_length) for i in range(overlap_video_length)],
                                                  np.float32)).unsqueeze(0).unsqueeze(0).unsqueeze(-1).unsqueeze(-1)
            new_sample[:, :, -overlap_video_length:] = new_sample[:, :, -overlap_video_length:] * (1 - mix_ratio) + \
                sample[:, :, :overlap_video_length] * mix_ratio
            new_sample = torch.cat([new_sample, sample[:, :, overlap_video_length:]], dim=2)
            sample = new_sample
        else:
            new_sample = sample
        if last_frames >= length_slider:
            break
        start_image = [Image.fromarray((sample[0, :, i].transpose(0, 1).transpose(1, 2) * 255).numpy().astype(np.uint8))
                       for i in range(-overlap_video_length, 0)]
        init_frames = init_frames + _partial_video_length - overlap_video_length
        last_frames = init_frames + _partial_video_length
    return new_sample, windows

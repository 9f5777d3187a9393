"""On the GPU: `ea_frames_out_blend` (the long-video cross-fade fused with the output tail) against torch's float32 op sequence,
and `generate_long_video` against the same windows run as separate `EasyAnimateInpaintPipeline` calls with the chaining and
cross-fading done on the host by the restated reference loop (tests/long_video_oracle.py).  The GPU-free prelude also runs in
the CPU suite (tests/test_long_video_cpu.py)."""
import numpy as np
import pytest
import torch
from PIL import Image

bf16 = torch.bfloat16
gpu = pytest.mark.gpu
H, W = 64, 96
CFG = dict(num_attention_heads=4, attention_head_dim=64, in_channels=33, out_channels=16, patch_size=2, num_layers=2,
           time_embed_dim=128, add_norm_text_encoder=True, text_embed_dim=256, text_embed_dim_t5=None)
BOC = [64, 64, 128, 128]
EA_ERR_INVALID = -1  # include/ea_b200.h


def prelude_long_video(device="cuda"):
    """Seeded tiny InP transformer + MagViT VAE (with encoder) on `device`, prompt embeddings and a start image."""
    from oracle import dit, vae
    from easyanimate_b200 import EasyAnimateInpaintPipeline
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel
    flags = dict(resize_inpaint_mask_directly=True, enable_clip_in_inpaint=False, add_noise_in_inpaint_model=True)
    ob = dit.init_weights_(dit.OracleTransformer3D(**CFG), 81).to(bf16)
    t = EasyAnimateTransformer3DModel(**CFG, **flags).to(bf16)
    t.load_state_dict(ob.state_dict(), strict=True)
    ov = vae.init_weights_(vae.OracleAutoencoderKLMagvit(block_out_channels=BOC, with_encoder=True), 82).to(bf16)
    v = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True, mid_block_attention_type="spatial",
                            block_out_channels=BOC, scaling_factor=0.7125, mini_batch_encoder=4, mini_batch_decoder=1).to(bf16)
    v.load_state_dict(ov.state_dict(), strict=True)
    g = torch.Generator().manual_seed(83)
    pe, ne = (torch.randn(1, 24, 256, generator=g) * 3).to(bf16), (torch.randn(1, 24, 256, generator=g) * 3).to(bf16)
    ones = torch.ones(1, 24, dtype=torch.long)
    kw = dict(prompt_embeds=pe.to(device), negative_prompt_embeds=ne.to(device), prompt_attention_mask=ones.to(device),
              negative_prompt_attention_mask=ones.to(device), prompt_embeds_2=pe.to(device), prompt_attention_mask_2=ones.to(device),
              height=H, width=W, num_inference_steps=3, guidance_scale=6.0)
    start = Image.fromarray(torch.randint(0, 256, (H, W, 3), generator=g, dtype=torch.uint8).numpy())
    return EasyAnimateInpaintPipeline(vae=v.to(device), transformer=t.to(device)), kw, start


def _blend_reference(x, dst, ov):
    """The reference's ops: the output tail on the bf16 tensor (pipeline_easyanimate.py:738-741), then the float32 cross-fade
    of ui.py:524-531 on the host."""
    f = (x.clamp(-1, 1) / 2 + 0.5).clamp(0, 1).float().cpu()
    want = dst.clone().cpu()
    if ov:
        r = torch.from_numpy(np.array([float(i) / float(ov) for i in range(ov)], np.float32)).view(1, 1, -1, 1, 1)
        want[:, :, :ov] = want[:, :, :ov] * (1 - r) + f[:, :, :ov] * r
    want[:, :, ov:] = f[:, :, ov:]
    return want


@gpu
@pytest.mark.parametrize("ov", [0, 1, 4])
@pytest.mark.parametrize("where", ["device", "pinned_host"])
def test_frames_out_blend_kernel_bit_exact(ov, where):
    """Bit for bit the torch ops, for a window written into the middle of a longer video, with a ragged frame size (not a
    multiple of 8 elements) and NaN inputs; exactly one launch; the frames of the video outside the window are untouched."""
    from easyanimate_b200 import _lib as L
    from easyanimate_b200 import vae_ops
    g = torch.Generator(device="cuda").manual_seed(ov)
    for h, w in ((16, 24), (17, 33)):
        x = (torch.randn(1, 3, 5, h, w, device="cuda", generator=g) * 1.5).to(bf16)
        x[0, 1, 0, 0, 0] = float("nan")
        x[0, 2, 4, 1, 2] = float("nan")
        full = torch.rand(1, 3, 12, h, w, device="cuda", generator=g)
        full[0, 0, 3, 2, 2] = float("nan")  # a NaN already in the video's overlap
        if where == "pinned_host":
            full = full.cpu().pin_memory()
        before = full.clone().cpu()
        want = _blend_reference(x, before[:, :, 3:8], ov)
        n0 = L.ea_launch_count()
        vae_ops.frames_out_blend(x, full[:, :, 3:8], ov)
        assert L.ea_launch_count() - n0 == 1
        torch.cuda.synchronize()
        got = full.cpu()
        assert torch.equal(torch.nan_to_num(got[:, :, 3:8], nan=-7.0), torch.nan_to_num(want, nan=-7.0))
        assert torch.equal(got[:, :, 3:8].isnan(), want.isnan())
        assert torch.equal(got[:, :, :3], before[:, :, :3]) and torch.equal(got[:, :, 8:], before[:, :, 8:])


@gpu
def test_frames_out_blend_argument_errors():
    from easyanimate_b200 import _lib as L
    from easyanimate_b200 import vae_ops
    x = torch.zeros(1, 3, 5, 8, 8, device="cuda", dtype=bf16)
    d = torch.zeros(1, 3, 5, 8, 8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    bad = [(0, d.data_ptr(), 3, 5, 64, 320, 0), (x.data_ptr(), 0, 3, 5, 64, 320, 0), (x.data_ptr(), d.data_ptr(), 3, 5, 64, 320, 6),
           (x.data_ptr(), d.data_ptr(), 3, 5, 64, 320, -1), (x.data_ptr(), d.data_ptr(), 3, 5, 0, 320, 0),
           (x.data_ptr(), d.data_ptr(), 3, 5, 64, 100, 0), (x.data_ptr(), d.data_ptr(), 70000, 1, 64, 320, 0)]
    for args in bad:
        assert L.ea_frames_out_blend(*args, s) == EA_ERR_INVALID, args
    with pytest.raises(Exception, match="pinned"):
        vae_ops.frames_out_blend(x, torch.zeros(1, 3, 5, 8, 8), 0)
    with pytest.raises(Exception, match="frame range"):
        vae_ops.frames_out_blend(x, torch.zeros(1, 5, 3, 8, 8, device="cuda").transpose(1, 2), 0)


@gpu
def test_long_video_equals_separate_pipeline_calls_chained_on_the_host():
    """Three windows (9 + 9 + 5 frames, overlap 4) on the H100: the device-resident path (conditioning frames by ea_frames_out,
    cross-fade by ea_frames_out_blend into pinned host memory) gives bit for bit the frames of the reference's loop run over the
    same pipeline with its frames, PIL images and cross-fade on the host."""
    from easyanimate_b200 import generate_long_video
    from tests import long_video_oracle
    pipe, kw, start = prelude_long_video()
    got = generate_long_video(pipe, video_length=17, partial_video_length=9, overlap_video_length=4, start_image=start,
                              generator=torch.Generator(device="cuda").manual_seed(84), **kw).frames
    want, windows = long_video_oracle.long_video(pipe, length_slider=17, partial_video_length=9, overlap_video_length=4,
                                                 start_image=start, end_image=None,
                                                 generator=torch.Generator(device="cuda").manual_seed(84), **kw)
    assert windows == [(0, 9), (5, 9), (10, 5)]
    assert got.is_pinned() and got.shape == want.shape == (1, 3, 15, H, W)
    assert 0.0 < float(got.std())
    assert torch.equal(got, want), float((got - want).abs().max())

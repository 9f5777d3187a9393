"""On the GPU: the multi-step CFG sampler (pipeline_easyanimate.py:1065-1111) against
the oracle's denoise loop, `decode_latents` (pipeline_easyanimate.py:722-742) including the fused scale / clamp / float32-to-host
tail, and the checkpoint loaders (`from_pretrained_2d` with its `proj.weight` channel-resize shim, transformer3d.py:1775-1787;
`AutoencoderKLMagvit.from_pretrained`, autoencoder_magvit.py:478-505).  Each test's GPU-free prelude also runs in the CPU
suite (tests/test_gpu_preludes_cpu.py)."""
import json
import os

import pytest
import torch

from tests.parity import three_way

bf16 = torch.bfloat16
gpu = pytest.mark.gpu

CFG = dict(num_attention_heads=4, attention_head_dim=64, in_channels=16, out_channels=16, patch_size=2, num_layers=2,
           time_embed_dim=128, add_norm_text_encoder=True, text_embed_dim=256, text_embed_dim_t5=None)
BOC = [64, 64, 128, 128]


# ---------------------------------------------------------------------------------------------------------------
# a1: the denoise loop
# ---------------------------------------------------------------------------------------------------------------
def prelude_sampler(device="cuda", cfg=CFG, seed=1234):
    from oracle import dit
    from easyanimate_b200.pipeline import EasyAnimateSampler
    from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel
    o32 = dit.init_weights_(dit.OracleTransformer3D(**cfg), seed)
    ob = dit.OracleTransformer3D(**cfg).to(bf16)
    ob.load_state_dict({k: v.to(bf16) for k, v in o32.state_dict().items()})
    o32.load_state_dict({k: v.float() for k, v in ob.state_dict().items()})
    ours = EasyAnimateTransformer3DModel(**cfg).to(bf16)
    ours.load_state_dict(ob.state_dict(), strict=True)
    sampler = EasyAnimateSampler(ours.to(device), guidance_scale=6.0)
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(1, 16, 3, 8, 12, generator=g).to(bf16)
    pe = (torch.randn(1, 24, cfg["text_embed_dim"], generator=g) * 3).to(bf16)
    ne = (torch.randn(1, 24, cfg["text_embed_dim"], generator=g) * 3).to(bf16)
    return o32, ob, sampler, lat, pe, ne


@gpu
@pytest.mark.parametrize("steps,shift", [(3, 1.0), (5, 3.0)])
def test_sampler_multi_step_cfg_matches_oracle_loop(steps, shift):
    """N flow-matching Euler steps with classifier-free guidance through EasyAnimateSampler.sample == the oracle's
    restatement of the reference loop (same schedule, same bf16 rounding points of CFG combine and Euler update)."""
    from oracle import dit
    from easyanimate_b200.scheduler import FlowMatchEulerDiscreteScheduler
    o32, ob, sampler, lat, pe, ne = prelude_sampler()
    sampler.scheduler = FlowMatchEulerDiscreteScheduler(shift=shift)
    rope = dit.rope_for_video(64, 96, 3)
    truth = dit.denoise_loop(o32, lat.float(), pe.float(), ne.float(), rope, num_steps=steps, guidance_scale=6.0, shift=shift)
    ref = dit.denoise_loop(ob, lat, pe, ne, rope, num_steps=steps, guidance_scale=6.0, shift=shift)
    got = sampler.sample(lat.cuda(), pe.cuda(), ne.cuda(), height=64, width=96, num_inference_steps=steps)
    assert got.shape == lat.shape and got.dtype == bf16
    # errors compound over the steps (each step feeds the next): same criterion, the bf16 oracle sets the scale
    three_way(got, ref, truth, slack=2.0, name=f"sampler_{steps}steps_shift{shift}")


@gpu
def test_sampler_step_from_host_equals_device_step():
    _, _, sampler, lat, pe, ne = prelude_sampler()
    from easyanimate_b200.pipeline import rope_table
    sampler.set_timesteps(4, device="cpu")
    rope = rope_table(64, 96, 3, device="cuda")
    emb = torch.cat([ne, pe])
    a = sampler.step(lat.cuda(), 1, emb.cuda(), rope)
    out = sampler.step_from_host(lat.pin_memory(), 1, emb.pin_memory(), rope)
    assert not out.is_cuda and torch.equal(out, a.cpu())


# ---------------------------------------------------------------------------------------------------------------
# a10: decode_latents
# ---------------------------------------------------------------------------------------------------------------
def prelude_decode_latents(device="cuda", **kw):
    from oracle import vae
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    from easyanimate_b200.pipeline import EasyAnimateSampler
    o32 = vae.init_weights_(vae.OracleAutoencoderKLMagvit(block_out_channels=BOC, **kw), 7)
    ob = vae.OracleAutoencoderKLMagvit(block_out_channels=BOC, **kw).to(bf16)
    ob.load_state_dict({k: v.to(bf16) for k, v in o32.state_dict().items()})
    o32.load_state_dict({k: v.float() for k, v in ob.state_dict().items()})
    ours = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True, mid_block_attention_type="spatial",
                               block_out_channels=BOC, scaling_factor=0.7125, **kw).to(bf16)
    missing, unexpected = ours.load_state_dict(ob.state_dict(), strict=False)
    assert not unexpected and all(k.startswith(("quant_conv", "encoder.")) for k in missing)
    sampler = EasyAnimateSampler(None, vae=ours.to(device))
    g = torch.Generator().manual_seed(5)
    lat = (torch.randn(1, 16, 2, 8, 12, generator=g) * 0.7125 * 1.3).to(bf16)  # scaled latents, some decoded values beyond [-1,1]
    return o32, ob, sampler, lat


def _reference_tail(video):
    """pipeline_easyanimate.py:729,738-741 with torch ops on whatever dtype `video` has."""
    video = video.clamp(-1, 1)
    video = (video / 2 + 0.5).clamp(0, 1)
    return video.cpu().float()


@gpu
@pytest.mark.parametrize("tiled", [False, True])
def test_decode_latents_matches_reference_op_sequence(tiled):
    kw = dict(use_tiling=True, tile_sample_min_size=64) if tiled else {}
    o32, ob, sampler, lat = prelude_decode_latents(**kw)
    vae_mod = sampler.vae
    sf = vae_mod.config.scaling_factor
    with torch.no_grad():
        truth = _reference_tail(o32.decode(1 / sf * lat.float())[0])
        ref = _reference_tail(ob.decode(1 / sf * lat)[0])
    frames = sampler.decode_latents(lat.cuda())
    assert frames.dtype == torch.float32 and not frames.is_cuda and frames.is_pinned()
    assert frames.shape == (1, 3, 5, 64, 96) and float(frames.min()) >= 0.0 and float(frames.max()) <= 1.0
    assert float((frames == 0).float().mean()) > 0 or float((frames == 1).float().mean()) > 0, "the clamp must be exercised"
    three_way(frames, ref, truth, name="decode_latents" + ("_tiled" if tiled else ""))
    # the fused pieces are exact restatements of the reference's separate tensor ops: (1) scale folded into the latent
    # preparation == decode of the torch-scaled latents, bit for bit; (2) the tail kernel == the torch op sequence on the
    # same decoded tensor, bit for bit; (3) uint8 output == trunc(255 * float frames) (utils.py:57)
    dec = vae_mod.decode((1 / sf * lat.cuda()).to(bf16))[0]
    assert torch.equal(frames, _reference_tail(dec))
    u8 = sampler.decode_latents(lat.cuda(), dtype=torch.uint8)
    assert u8.dtype == torch.uint8 and torch.equal(u8, (frames * 255).to(torch.uint8))
    dev = sampler.decode_latents(lat.cuda(), to_host=False)
    assert dev.is_cuda and torch.equal(dev.cpu(), frames)


@gpu
def test_frames_out_kernel_bit_exact_including_ragged_tail_and_nan():
    from easyanimate_b200 import vae_ops
    g = torch.Generator(device="cuda").manual_seed(3)
    for n in (8, 4096 + 3, 3 * 5 * 33 * 17):
        x = (torch.randn(n, device="cuda", generator=g) * 1.5).to(bf16)
        x[0] = float("nan")
        want = (x.clamp(-1, 1) / 2 + 0.5).clamp(0, 1).float()
        got = vae_ops.frames_out(x, torch.empty(n, device="cuda", dtype=torch.float32))
        assert torch.equal(torch.nan_to_num(got, nan=-7.0), torch.nan_to_num(want, nan=-7.0))
        host = vae_ops.frames_out(x, torch.empty(n, dtype=torch.uint8, pin_memory=True))  # straight into pinned host memory
        torch.cuda.synchronize()
        w8 = (torch.nan_to_num(want, nan=0.0) * 255).to(torch.uint8).cpu()
        assert torch.equal(host[1:], w8[1:])
    with pytest.raises(Exception, match="pinned"):
        vae_ops.frames_out(x, torch.empty(x.numel(), dtype=torch.float32))


# ---------------------------------------------------------------------------------------------------------------
# a1 + a10 against the REFERENCE's own pipeline call (fixture minted by EasyAnimatePipeline.__call__ itself)
# ---------------------------------------------------------------------------------------------------------------
def prelude_reference_pipeline_golden(device="cuda"):
    """tests/golden/pipe_ref_t2v.safetensors (make_golden.make_pipeline_reference): inputs, final latents and frames of the
    reference's EasyAnimatePipeline.__call__ over the reference's transformer + VAE, in bf16 and in fp32.  The product modules
    load the same seeded, bf16-rounded weights."""
    from safetensors import safe_open
    from safetensors.torch import load_file
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    from easyanimate_b200.pipeline import EasyAnimateSampler
    from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel
    from tests.golden import make_golden as G
    path = os.path.join(os.path.dirname(__file__), "golden", "pipe_ref_t2v.safetensors")
    with safe_open(path, "pt") as f:
        t = {k: f.get_tensor(k) for k in f.keys()}
        meta = f.metadata()
    t.update(load_file(path.replace(".safetensors", "_2.safetensors")))  # frames_fp32 (files are kept under 1 MB)
    ot, ov = G.pipeline_case_modules(bf16)
    lat, pe, ne = G.pipeline_case_inputs()
    assert torch.equal(lat, t["latents"]) and torch.equal(pe, t["prompt_embeds"]) and torch.equal(ne, t["negative_prompt_embeds"])
    ours_t = EasyAnimateTransformer3DModel(**G.PIPE_CFG).to(bf16)
    ours_t.load_state_dict(ot.state_dict(), strict=True)
    ours_v = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True, mid_block_attention_type="spatial",
                                 block_out_channels=list(G.PIPE_BOC), scaling_factor=0.7125).to(bf16)
    missing, unexpected = ours_v.load_state_dict(ov.state_dict(), strict=False)
    assert not unexpected and all(k.startswith(("quant_conv", "encoder.")) for k in missing)
    sampler = EasyAnimateSampler(ours_t.to(device), vae=ours_v.to(device), guidance_scale=float(meta["guidance_scale"]))
    return t, meta, sampler


@gpu
def test_sampler_and_decode_match_the_reference_pipeline_call():
    """The whole hot path - 4 CFG flow-matching steps, decode_latents, float32 frames on the host - against what the reference's
    own `EasyAnimatePipeline.__call__` produced from the same latents / embeddings / weights (bf16 run = reference execution,
    fp32 run = truth)."""
    t, meta, sampler = prelude_reference_pipeline_golden()
    h, w, steps = int(meta["height"]), int(meta["width"]), int(meta["steps"])
    z = sampler.sample(t["latents"].cuda(), t["prompt_embeds"].cuda(), t["negative_prompt_embeds"].cuda(), height=h, width=w,
                       num_inference_steps=steps)
    three_way(z, t["z_bf16"], t["z_fp32"], slack=2.0, name="reference_pipeline_latents")
    frames = sampler.decode_latents(z)
    assert frames.shape == t["frames_fp32"].shape == (1, 3, int(meta["video_length"]), h, w) and frames.dtype == torch.float32
    three_way(frames, t["frames_bf16"], t["frames_fp32"], slack=2.0, name="reference_pipeline_frames")
    # the decode on its own, from the reference's latents: isolates the VAE from the loop's compounding
    frames_ref_z = sampler.decode_latents(t["z_bf16"].cuda())
    three_way(frames_ref_z, t["frames_bf16"], t["frames_fp32"], name="reference_pipeline_decode_of_reference_latents")


@gpu
def test_native_pipeline_call_matches_the_reference_pipeline_call():
    """easyanimate_b200.EasyAnimatePipeline.__call__ (the reference's signature, no diffusers) on the GPU: same keyword arguments
    the reference's call was minted with -> the same frames as sampler.sample + decode_latents, bit for bit, and within the
    three-way criterion of the reference's own frames."""
    from easyanimate_b200 import EasyAnimatePipeline
    t, meta, sampler = prelude_reference_pipeline_golden()
    h, w, steps, frames_n = int(meta["height"]), int(meta["width"]), int(meta["steps"]), int(meta["video_length"])
    pe, ne = t["prompt_embeds"], t["negative_prompt_embeds"]
    ones = torch.ones(pe.shape[:2], dtype=torch.long)
    pipe = EasyAnimatePipeline(vae=sampler.vae, transformer=sampler.transformer)
    out = pipe(video_length=frames_n, height=h, width=w, num_inference_steps=steps, guidance_scale=float(meta["guidance_scale"]),
               latents=t["latents"], prompt_embeds=pe, negative_prompt_embeds=ne, prompt_attention_mask=ones,
               negative_prompt_attention_mask=ones.clone(), prompt_embeds_2=pe, prompt_attention_mask_2=ones.clone())
    frames = out.frames
    assert isinstance(frames, torch.Tensor) and frames.dtype == torch.float32 and not frames.is_cuda
    three_way(frames, t["frames_bf16"], t["frames_fp32"], slack=2.0, name="native_pipeline_frames")
    z = sampler.sample(t["latents"].cuda(), pe.cuda(), ne.cuda(), height=h, width=w, num_inference_steps=steps)
    assert torch.equal(frames, sampler.decode_latents(z))


# ---------------------------------------------------------------------------------------------------------------
# a17 / boundary: checkpoint loaders
# ---------------------------------------------------------------------------------------------------------------
def _write_transformer_dir(path, cfg, state):
    from safetensors.torch import save_file
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(dict(cfg, _class_name="EasyAnimateTransformer3DModel"), f)
    save_file({k: v.contiguous() for k, v in state.items()}, os.path.join(path, "diffusion_pytorch_model.safetensors"))


def prelude_from_pretrained_2d(device="cuda", tmp=None):
    """A T2V checkpoint (16 input channels) loaded into an InP model (33 channels) and the reverse: the reference pads the
    patch-embed weight with zeros / truncates it (transformer3d.py:1775-1787) and skips nothing else."""
    import tempfile
    from oracle import dit
    from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel
    tmp = tmp or tempfile.mkdtemp(prefix="ea_ckpt_")
    src16 = dit.init_weights_(dit.OracleTransformer3D(**CFG), 99).state_dict()
    src33 = dit.init_weights_(dit.OracleTransformer3D(**dict(CFG, in_channels=33)), 98).state_dict()
    d16, d33 = os.path.join(tmp, "t2v", "transformer"), os.path.join(tmp, "inp", "transformer")
    _write_transformer_dir(d16, CFG, src16)
    _write_transformer_dir(d33, dict(CFG, in_channels=33), src33)
    # 16-channel weights, 33-channel model (transformer_additional_kwargs overrides the config like the reference's call sites)
    grown = EasyAnimateTransformer3DModel.from_pretrained_2d(os.path.join(tmp, "t2v"), subfolder="transformer",
                                                             transformer_additional_kwargs={"in_channels": 33})
    assert grown.dtype == bf16 and grown.proj.weight.shape == (256, 33, 2, 2)
    assert torch.equal(grown.proj.weight[:, :16], src16["proj.weight"].to(bf16))
    assert torch.count_nonzero(grown.proj.weight[:, 16:]) == 0
    shrunk = EasyAnimateTransformer3DModel.from_pretrained_2d(os.path.join(tmp, "inp"), subfolder="transformer",
                                                              transformer_additional_kwargs={"in_channels": 16})
    assert torch.equal(shrunk.proj.weight, src33["proj.weight"][:, :16].to(bf16))
    for k, v in src16.items():
        if k != "proj.weight":
            assert torch.equal(grown.state_dict()[k], v.to(bf16)), k
    return src16, grown.to(device), shrunk.to(device)


@gpu
def test_from_pretrained_2d_proj_weight_resize_shim_and_forward():
    from oracle import dit
    src16, grown, _ = prelude_from_pretrained_2d()
    # zero-padded input channels: the 33-channel model with ANY inpaint latents must reproduce the 16-channel model
    ob = dit.OracleTransformer3D(**CFG).to(bf16)
    ob.load_state_dict({k: v.to(bf16) for k, v in src16.items()})
    g = torch.Generator().manual_seed(1)
    lat = torch.randn(2, 16, 2, 8, 8, generator=g).to(bf16)
    inp = torch.randn(2, 17, 2, 8, 8, generator=g).to(bf16)
    enc = (torch.randn(2, 16, CFG["text_embed_dim"], generator=g) * 3).to(bf16)
    t = torch.tensor([900.0, 900.0]).to(bf16)
    rope = dit.rope_for_video(64, 64, 2)
    with torch.no_grad():
        ref = ob(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope)[0]
    got = grown(lat.cuda(), t.cuda(), encoder_hidden_states=enc.cuda(), image_rotary_emb=(rope[0].cuda(), rope[1].cuda()),
                inpaint_latents=inp.cuda(), return_dict=False)[0]
    torch.testing.assert_close(got.float().cpu(), ref.float(), rtol=0.05, atol=0.05)


@gpu
def test_vae_from_pretrained_round_trip(tmp_path):
    from safetensors.torch import save_file
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    _, ob, sampler, lat = prelude_decode_latents()
    ours = sampler.vae
    d = tmp_path / "vae"
    d.mkdir()
    (d / "config.json").write_text(json.dumps({k: v for k, v in ours.config.items()}))
    save_file({k: v.detach().cpu().contiguous() for k, v in ours.state_dict().items()}, str(d / "diffusion_pytorch_model.safetensors"))
    loaded = AutoencoderKLMagvit.from_pretrained(str(tmp_path), subfolder="vae").to(bf16).cuda()
    assert set(loaded.state_dict()) == set(ours.state_dict())
    a, b = ours.decode(lat.cuda())[0], loaded.decode(lat.cuda())[0]
    assert torch.equal(a, b)

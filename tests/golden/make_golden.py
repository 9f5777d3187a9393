"""Mint golden vectors from the REFERENCE ITSELF (run in the authoring container, where /root/reference exists).

VAE: the reference's own `Decoder` (easyanimate/vae/ldm/models/omnigen_enc_dec.py) is imported through
oracle/ref_vae.py and run in its v5.1 execution mode (cache_mag_vae=True, one latent frame per chunk,
padding_flag 3/4) in fp32 on CPU.  Weights come from oracle.vae.init_weights_(seed) so the fixtures stay small:
only inputs and outputs are stored.

DiT: the reference's own `EasyAnimateTransformer3DModel` (easyanimate/models/transformer3d.py with attention.py,
processor.py, norm.py, executed unmodified) is imported through oracle/ref_dit.py - diffusers itself is not installable
here, so the third-party primitives it uses come from oracle/_refshim (restated from diffusers 0.30/0.31) - and run in
fp32 on CPU: `dit_ref_*.safetensors` hold inputs and the reference's outputs (T2V forward, I2V forward with
inpaint_latents, a 6-call TeaCache sequence with its skip decisions).  `dit_tiny` (3-step CFG denoise loop, scheduler
and RoPE tables) is produced by the oracle and is a regression fixture, not a reference vector.

Usage:  python tests/golden/make_golden.py
"""
import os
import sys

import torch
from safetensors.torch import save_file

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HERE = os.path.dirname(os.path.abspath(__file__))

from oracle import dit, ref_dit, ref_vae, vae  # noqa: E402

VAE_CASES = {
    # name: (block_out_channels, mid_attention, z shape, seed)
    "vae_small_attn": ((64, 64, 128, 128), True, (1, 16, 3, 8, 8), 11),
    "vae_small_noattn_ragged": ((64, 64, 128, 128), False, (1, 16, 2, 6, 10), 12),
    "vae_full_arch": ((128, 256, 512, 512), True, (1, 16, 2, 8, 8), 13),
}

DIT_CFG = dict(num_attention_heads=2, attention_head_dim=64, in_channels=16, out_channels=16, patch_size=2, num_layers=2,
               time_embed_dim=64, add_norm_text_encoder=True, text_embed_dim=128, text_embed_dim_t5=None)


def make_vae():
    for name, (boc, attn, zshape, seed) in VAE_CASES.items():
        ref = ref_vae.reference_decoder(cache_mag_vae=True, mid_block_use_attention=attn, block_out_channels=boc)
        mine = vae.init_weights_(vae.OracleDecoder(block_out_channels=boc, mid_block_use_attention=attn), seed)
        ref.load_state_dict(mine.state_dict(), strict=True)
        z = torch.randn(zshape, generator=torch.Generator().manual_seed(seed + 100))
        with torch.no_grad():
            out = ref(z)
        save_file({"z": z, "out": out.contiguous()}, os.path.join(HERE, f"{name}.safetensors"),
                  metadata={"source": "reference Decoder (cache_mag_vae=True, fp32, CPU)", "seed": str(seed),
                            "block_out_channels": str(boc), "mid_attention": str(attn)})
        print(name, tuple(out.shape), float(out.abs().max()))


def make_dit():
    m = dit.init_weights_(dit.OracleTransformer3D(**DIT_CFG), 1234)
    g = torch.Generator().manual_seed(7)
    lat = torch.randn(1, 16, 3, 8, 12, generator=g)
    pe, ne = torch.randn(1, 9, 128, generator=g), torch.randn(1, 9, 128, generator=g)
    rope = dit.rope_for_video(64, 96, 3)
    out = dit.denoise_loop(m, lat, pe, ne, rope, num_steps=3, guidance_scale=6.0)
    sched = dit.FlowMatchEulerScheduler(shift=3.0)
    sched.set_timesteps(25, mu=1.0)
    cos720, sin720 = dit.rope_for_video(720, 1280, 2)
    save_file({"latents": lat, "prompt_embeds": pe, "negative_prompt_embeds": ne, "out_3steps_cfg6": out,
               "rope_cos": rope[0], "rope_sin": rope[1], "sigmas_shift3_25": sched.sigmas,
               "timesteps_shift3_25": sched.timesteps, "rope720_cos_head": cos720[:200].contiguous(),
               "rope720_sin_tail": sin720[-200:].contiguous()},
              os.path.join(HERE, "dit_tiny.safetensors"), metadata={"source": "oracle restatement (parity unpinned)"})
    print("dit_tiny", tuple(out.shape), float(out.std()))


def make_vae_tiled():
    """The reference's AutoencoderKLMagvit.tiled_decode (autoencoder_magvit.py:381-448) on a latent that needs 3 x 3
    tiles plus the lower-right corner pass; also its untiled decode of the same latent."""
    boc, seed = (64, 64, 128, 128), 31
    ref = ref_vae.reference_autoencoder(block_out_channels=boc, use_tiling=True, tile_sample_min_size=64)
    mine = vae.init_weights_(vae.OracleAutoencoderKLMagvit(block_out_channels=boc, use_tiling=True, tile_sample_min_size=64), seed)
    ref.load_state_dict(mine.state_dict(), strict=False)
    z = torch.randn(1, 16, 2, 14, 13, generator=torch.Generator().manual_seed(seed + 100))
    with torch.no_grad():
        tiled = ref.decode(z).sample
        ref.use_tiling = False
        full = ref.decode(z).sample
    meta = {"source": "reference AutoencoderKLMagvit.decode (tiled_decode and untiled, fp32, CPU)", "seed": str(seed),
            "block_out_channels": str(boc), "tile_sample_min_size": "64"}
    # two files, each under 1 MB
    save_file({"z": z, "out_tiled": tiled.contiguous()}, os.path.join(HERE, "vae_ref_tiled.safetensors"), metadata=meta)
    save_file({"out_untiled": full.contiguous()}, os.path.join(HERE, "vae_ref_tiled_2.safetensors"), metadata=meta)
    print("vae_ref_tiled", tuple(tiled.shape), float((tiled - full).abs().max()))


def make_vae_encode():
    """The reference's AutoencoderKLMagvit.encode (autoencoder_magvit.py:230-269: chunked Encoder, first frame alone and
    then 4 frames at a time, + quant_conv) and tiled_encode (:339-379): the moments tensor of the returned posterior."""
    boc, seed = (64, 64, 128, 128), 41
    ref = ref_vae.reference_autoencoder(block_out_channels=boc, use_tiling=False)
    mine = vae.init_weights_(vae.OracleAutoencoderKLMagvit(block_out_channels=boc, with_encoder=True), seed)
    ref.load_state_dict(mine.state_dict(), strict=True)
    x = torch.randn(1, 3, 9, 40, 56, generator=torch.Generator().manual_seed(seed + 100))
    with torch.no_grad():
        moments = ref.encode(x).latent_dist.parameters
        ref.use_tiling, ref.tile_sample_min_size, ref.tile_latent_min_size = True, 32, 4
        moments_tiled = ref.encode(x).latent_dist.parameters
    save_file({"x": x, "moments": moments.contiguous(), "moments_tiled32": moments_tiled.contiguous()},
              os.path.join(HERE, "vae_ref_encode.safetensors"),
              metadata={"source": "reference AutoencoderKLMagvit.encode / tiled_encode (fp32, CPU)", "seed": str(seed),
                        "block_out_channels": str(boc)})
    print("vae_ref_encode", tuple(moments.shape), float(moments.abs().max()))


DIT_REF_CASES = {
    # name: (config overrides, (B, F, H, W, S_text), weight seed, inpaint channels)
    "dit_ref_t2v": (dict(), (2, 3, 8, 12, 40), 21, 0),
    "dit_ref_i2v_inpaint": (dict(in_channels=33), (1, 2, 6, 10, 7), 22, 17),
    "dit_ref_3heads_3layers": (dict(num_attention_heads=3, num_layers=3, time_embed_dim=96, text_embed_dim=192), (1, 1, 4, 6, 9), 23, 0),
}


CONTROL_REF_OVER = dict(ref_channels=16, clip_channels=96, sample_width=20, sample_height=12)


def _dit_inputs(cfg, shape, seed, inpaint_c):
    B, F, H, W, St = shape
    g = torch.Generator().manual_seed(seed + 100)
    t = {"latents": torch.randn(B, 16, F, H, W, generator=g), "encoder_hidden_states": torch.randn(B, St, cfg["text_embed_dim"], generator=g) * 3.0,
         "timestep": torch.tensor([937.0, 421.0][:B])}
    if inpaint_c:
        t["inpaint_latents"] = torch.randn(B, inpaint_c, F, H, W, generator=g)
    return t


def make_dit_reference():
    """Golden vectors from the REFERENCE's transformer code (oracle/ref_dit.py)."""
    for name, (over, shape, seed, inpaint_c) in DIT_REF_CASES.items():
        cfg = {**DIT_CFG, **over}
        ref = ref_dit.reference_transformer(**cfg).eval()
        ref.load_state_dict(dit.init_weights_(dit.OracleTransformer3D(**cfg), seed).state_dict(), strict=True)
        t = _dit_inputs(cfg, shape, seed, inpaint_c)
        rope = dit.rope_for_video(shape[2] * 8, shape[3] * 8, shape[1])
        with torch.no_grad():
            out = ref(t["latents"], t["timestep"], encoder_hidden_states=t["encoder_hidden_states"], image_rotary_emb=rope,
                      inpaint_latents=t.get("inpaint_latents"), return_dict=False)[0]
        t["out"] = out.contiguous()
        save_file(t, os.path.join(HERE, f"{name}.safetensors"),
                  metadata={"source": "reference EasyAnimateTransformer3DModel (fp32, CPU, diffusers primitives from oracle/_refshim)",
                            "seed": str(seed), "config": repr(cfg), "shape": repr(shape)})
        print(name, tuple(out.shape), float(out.std()))
    # v5.1 Control with a reference image and CLIP tokens (transformer3d.py:1420-1429,1538-1561); fp32 modules (the float64
    # position-table buffer follows .to(float32) like it follows .to(bfloat16) in the pipelines)
    cfg, seed = {**DIT_CFG, **CONTROL_REF_OVER}, 25
    ref = ref_dit.reference_transformer(**cfg).eval().to(torch.float32)
    ref.load_state_dict(dit.init_weights_(dit.OracleTransformer3D(**cfg), seed).state_dict(), strict=True)
    t = _dit_inputs(cfg, (2, 2, 8, 12, 9), seed, 0)
    g = torch.Generator().manual_seed(seed + 200)
    t["ref_latents"] = torch.randn(2, cfg["ref_channels"], 1, 8, 12, generator=g)
    t["clip_encoder_hidden_states"] = torch.randn(2, 5, cfg["clip_channels"], generator=g)
    rope = dit.rope_for_video(64, 96, 2)
    with torch.no_grad():
        out = ref(t["latents"], t["timestep"], encoder_hidden_states=t["encoder_hidden_states"], image_rotary_emb=rope,
                  ref_latents=t["ref_latents"], clip_encoder_hidden_states=t["clip_encoder_hidden_states"], return_dict=False)[0]
        out_ref_only = ref(t["latents"], t["timestep"], encoder_hidden_states=t["encoder_hidden_states"], image_rotary_emb=rope,
                           ref_latents=t["ref_latents"], return_dict=False)[0]
    t["out"], t["out_ref_only"] = out.contiguous(), out_ref_only.contiguous()
    save_file(t, os.path.join(HERE, "dit_ref_control_ref_clip.safetensors"),
              metadata={"source": "reference EasyAnimateTransformer3DModel with ref_channels / clip_channels (fp32, CPU, diffusers "
                                  "primitives incl. get_2d_sincos_pos_embed from oracle/_refshim)", "seed": str(seed),
                        "config": repr(cfg), "shape": repr((2, 2, 8, 12, 9))})
    print("dit_ref_control_ref_clip", tuple(out.shape), float(out.std()))
    # TeaCache: 6 calls with slowly drifting inputs; record every output and which calls were skipped
    cfg, seed = DIT_CFG, 24
    ref = ref_dit.reference_transformer(**cfg).eval()
    ref.load_state_dict(dit.init_weights_(dit.OracleTransformer3D(**cfg), seed).state_dict(), strict=True)
    ref.enable_teacache(6, 0.08, coefficients=TEACACHE_COEFFS)
    base = _dit_inputs(cfg, (2, 3, 8, 12, 40), seed, 0)
    rope = dit.rope_for_video(64, 96, 3)
    outs, skipped = [], []
    with torch.no_grad():
        for i in range(6):
            lat = base["latents"] * (1.0 - 0.01 * i)
            tt = base["timestep"] - 30.0 * i
            before = ref.teacache.previous_residual
            out = ref(lat, tt, encoder_hidden_states=base["encoder_hidden_states"], image_rotary_emb=rope, return_dict=False)[0]
            skipped.append(1.0 if (ref.teacache.previous_residual is before and i > 0) else 0.0)
            outs.append(out)
    base["outs"] = torch.stack(outs).contiguous()
    base["skipped"] = torch.tensor(skipped)
    save_file(base, os.path.join(HERE, "dit_ref_teacache.safetensors"),
              metadata={"source": "reference EasyAnimateTransformer3DModel + TeaCache (fp32, CPU)", "seed": str(seed),
                        "config": repr(cfg), "num_steps": "6", "rel_l1_thresh": "0.08", "coefficients": repr(TEACACHE_COEFFS)})
    print("dit_ref_teacache skipped:", skipped)


PIPE_CFG = dict(num_attention_heads=4, attention_head_dim=64, in_channels=16, out_channels=16, patch_size=2, num_layers=2,
                time_embed_dim=128, add_norm_text_encoder=True, text_embed_dim=256, text_embed_dim_t5=None)
PIPE_BOC = (64, 64, 128, 128)


def pipeline_case_modules(dtype, transformer_seed=41, vae_seed=42):
    """bf16-rounded weights in `dtype` for the reference-pipeline fixture: (oracle transformer, oracle VAE) state dicts are
    what both the reference modules here and the product modules in tests/test_pipeline_gpu.py load."""
    ot = dit.init_weights_(dit.OracleTransformer3D(**PIPE_CFG), transformer_seed)
    ov = vae.init_weights_(vae.OracleAutoencoderKLMagvit(block_out_channels=list(PIPE_BOC)), vae_seed)
    for m in (ot, ov):
        m.load_state_dict({k: v.to(torch.bfloat16).to(dtype) for k, v in m.state_dict().items()})
    return ot.to(dtype), ov.to(dtype)


def pipeline_case_inputs(seed=43):
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(1, 16, 3, 8, 12, generator=g).to(torch.bfloat16)
    pe = (torch.randn(1, 24, PIPE_CFG["text_embed_dim"], generator=g) * 3).to(torch.bfloat16)
    ne = (torch.randn(1, 24, PIPE_CFG["text_embed_dim"], generator=g) * 3).to(torch.bfloat16)
    return lat, pe, ne


def make_pipeline_reference():
    """`pipe_ref_t2v.safetensors`: the REFERENCE's own EasyAnimatePipeline.__call__ (pipeline_easyanimate.py:769-1148, through
    oracle/ref_pipeline.py) over the reference's own transformer and VAE: 4 CFG flow-matching steps + decode_latents, once in
    bf16 (the execution the product reproduces) and once in fp32 with the same bf16-rounded weights (the truth of the
    three-way criterion).  Stored: the inputs, the final latents of both runs, the frames of both runs."""
    from oracle import ref_pipeline
    lat, pe, ne = pipeline_case_inputs()
    t = {"latents": lat, "prompt_embeds": pe, "negative_prompt_embeds": ne}
    for tag, dtype in (("bf16", torch.bfloat16), ("fp32", torch.float32)):
        ot, ov = pipeline_case_modules(dtype)
        rt = ref_dit.reference_transformer(**PIPE_CFG, time_position_encoding_type="3d_rope").eval().to(dtype)
        rt.load_state_dict(ot.state_dict(), strict=True)
        rv = ref_vae.reference_autoencoder(block_out_channels=PIPE_BOC).eval().to(dtype)
        missing, unexpected = rv.load_state_dict(ov.state_dict(), strict=False)
        assert not unexpected and all(k.startswith(("encoder.", "quant_conv")) for k in missing)
        pipe = ref_pipeline.reference_pipeline(rt, rv)
        seen, orig = {}, pipe.decode_latents
        pipe.decode_latents = lambda z, seen=seen, orig=orig: (seen.setdefault("z", z.clone()), orig(z))[1]
        frames = ref_pipeline.run(pipe, lat.to(dtype), pe.to(dtype), ne.to(dtype), height=64, width=96, video_length=9,
                                  num_inference_steps=4, guidance_scale=6.0)
        t[f"z_{tag}"], t[f"frames_{tag}"] = seen["z"].contiguous(), frames.contiguous()
        print("pipe_ref_t2v", tag, tuple(frames.shape), float(frames.mean()), float(seen["z"].float().std()))
    meta = {"source": "reference EasyAnimatePipeline.__call__ + reference transformer + reference AutoencoderKLMagvit "
                                  "(CPU; diffusers names from oracle/_refshim: FlowMatchEulerDiscreteScheduler shift=1, "
                                  "get_3d_rotary_pos_embed)", "config": repr(PIPE_CFG), "block_out_channels": repr(PIPE_BOC),
                        "steps": "4", "guidance_scale": "6.0", "height": "64", "width": "96", "video_length": "9",
                        "seeds": "transformer 41, vae 42, inputs 43"}
    # two files, each under 1 MB
    save_file({k: v for k, v in t.items() if k != "frames_fp32"}, os.path.join(HERE, "pipe_ref_t2v.safetensors"), metadata=meta)
    save_file({"frames_fp32": t["frames_fp32"]}, os.path.join(HERE, "pipe_ref_t2v_2.safetensors"), metadata=meta)


TEACACHE_COEFFS = [1.07862322, -4.19362456, 3.06725828, 0.33161686, 0.02374758]  # transformer3d.py:131 (v5.1-7b)


if __name__ == "__main__":
    if not ref_vae.available():
        raise SystemExit("/root/reference not present: golden VAE vectors can only be minted in the authoring container")
    make_vae()
    make_vae_tiled()
    make_vae_encode()
    make_dit()
    make_dit_reference()
    make_pipeline_reference()

"""The product module's HOST LOGIC on CPU: EasyAnimateTransformer3DModel.forward (buffer plumbing, text/video stream split,
in-place gated residuals, I2V channel concat, TeaCache bookkeeping) run end to end with torch stand-ins for the CUDA entry
points (tests/cpu_ops.py) and compared with the oracle - no kernel is exercised here, the GPU suite does that."""
import pytest
import torch

from oracle import dit
from tests import cpu_ops

bf16 = torch.bfloat16
CFG = dict(num_attention_heads=2, attention_head_dim=64, in_channels=16, out_channels=16, patch_size=2, num_layers=2,
           time_embed_dim=64, add_norm_text_encoder=True, text_embed_dim=128, text_embed_dim_t5=None)


def _models(cfg, seed=11):
    from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel
    ob = dit.init_weights_(dit.OracleTransformer3D(**cfg), seed).to(bf16)
    ours = EasyAnimateTransformer3DModel(**cfg).to(bf16)
    ours.load_state_dict(ob.state_dict(), strict=True)
    return ob, ours


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


@pytest.mark.parametrize("inpaint", [False, True])
def test_forward_host_logic_matches_oracle(monkeypatch, inpaint):
    cpu_ops.use_stand_ins(monkeypatch)
    cfg = dict(CFG, in_channels=33) if inpaint else CFG
    ob, ours = _models(cfg)
    g = torch.Generator().manual_seed(2)
    lat = torch.randn(2, 16, 3, 8, 12, generator=g).to(bf16)
    enc = (torch.randn(2, 9, 128, generator=g) * 3).to(bf16)
    inp = torch.randn(2, 17, 3, 8, 12, generator=g).to(bf16) if inpaint else None
    t = torch.tensor([937.0, 421.0]).to(bf16)
    rope = dit.rope_for_video(64, 96, 3)
    with torch.no_grad():
        ref = ob(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, inpaint_latents=inp)[0]
        got = ours(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, inpaint_latents=inp, return_dict=False)[0]
    assert got.shape == ref.shape == (2, 16, 3, 8, 12)
    assert _rel(got, ref) < 2e-2  # bf16 round-off of two different op orders; a plumbing error is O(1)


def test_teacache_host_logic_matches_oracle(monkeypatch):
    cpu_ops.use_stand_ins(monkeypatch)
    ob, ours = _models(CFG)
    coeffs = [1.07862322, -4.19362456, 3.06725828, 0.33161686, 0.02374758]
    ob.teacache = dit.OracleTeaCache(coeffs, 6, 0.08)
    ours.enable_teacache(6, 0.08, coefficients=coeffs)
    g = torch.Generator().manual_seed(4)
    lat = torch.randn(2, 16, 3, 8, 12, generator=g).to(bf16)
    enc = (torch.randn(2, 9, 128, generator=g) * 3).to(bf16)
    rope = dit.rope_for_video(64, 96, 3)
    with torch.no_grad():
        for i in range(6):
            x, t = (lat.float() * (1.0 - 0.01 * i)).to(bf16), torch.tensor([900.0 - 30 * i] * 2).to(bf16)
            ref = ob(x, t, encoder_hidden_states=enc, image_rotary_emb=rope)[0]
            got = ours(x, t, encoder_hidden_states=enc, image_rotary_emb=rope, return_dict=False)[0]
            assert _rel(got, ref) < 3e-2, i
    assert ours.teacache.cnt == 0 and ob.teacache.cnt == 0  # both wrapped around after num_steps calls
    assert ob.teacache.skipped >= 1 and ours.teacache.skipped == ob.teacache.skipped  # the cached path is exercised, same decisions


# ---- VAE: decode / tiled decode host logic (layer order, channels-last plumbing, fused residual / frame duplication flags,
# tile cropping, blend order, corner pass) with torch stand-ins for the kernels, against the oracle ----
def _vae_pair(**kw):
    from oracle import vae
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    boc = [64, 64, 128, 128]
    ob = vae.init_weights_(vae.OracleAutoencoderKLMagvit(block_out_channels=boc, **kw), 21).to(bf16)
    ours = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True,
                               mid_block_attention_type="spatial", block_out_channels=boc, **kw).to(bf16)
    ours.load_state_dict(ob.state_dict(), strict=False)
    return ob, ours


def test_vae_decode_host_logic_matches_oracle(monkeypatch):
    cpu_ops.use_stand_ins(monkeypatch)
    ob, ours = _vae_pair()
    z = torch.randn(1, 16, 3, 6, 8, generator=torch.Generator().manual_seed(5)).to(bf16)
    with torch.no_grad():
        ref = ob.decode(z)[0]
        got = ours.decode(z).sample
    assert got.shape == ref.shape == (1, 3, 9, 48, 64)
    assert _rel(got, ref) < 3e-2


def test_vae_tiled_decode_host_logic_matches_oracle(monkeypatch):
    cpu_ops.use_stand_ins(monkeypatch)
    ob, ours = _vae_pair(use_tiling=True, tile_sample_min_size=64)
    z = torch.randn(1, 16, 2, 14, 13, generator=torch.Generator().manual_seed(6)).to(bf16)
    with torch.no_grad():
        ref = ob.decode(z)[0]
        got = ours.decode(z).sample
    assert got.shape == ref.shape == (1, 3, 5, 112, 104)
    assert _rel(got, ref) < 3e-2


def test_sampler_loop_host_logic_matches_oracle_denoise_loop(monkeypatch):
    """EasyAnimateSampler.sample (timesteps, CFG batching [negative, positive], bf16 timestep expansion, Euler update) over
    the product transformer, all with CPU stand-ins for the kernels, against oracle.dit.denoise_loop."""
    from easyanimate_b200.pipeline import EasyAnimateSampler
    cpu_ops.use_stand_ins(monkeypatch)
    ob, ours = _models(CFG)
    g = torch.Generator().manual_seed(8)
    lat = torch.randn(1, 16, 3, 8, 12, generator=g).to(bf16)
    pe, ne = (torch.randn(1, 9, 128, generator=g) * 3).to(bf16), (torch.randn(1, 9, 128, generator=g) * 3).to(bf16)
    with torch.no_grad():
        ref = dit.denoise_loop(ob, lat, pe, ne, dit.rope_for_video(64, 96, 3), 3, 6.0)
        sampler = EasyAnimateSampler(ours, guidance_scale=6.0)
        got = sampler.sample(lat, pe, ne, height=64, width=96, num_inference_steps=3)
    got = got[0] if isinstance(got, (tuple, list)) else got
    assert got.shape == ref.shape and _rel(got, ref) < 3e-2


def _vae_pair_enc(**kw):
    from oracle import vae
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    boc = [64, 64, 128, 128]
    ob = vae.init_weights_(vae.OracleAutoencoderKLMagvit(block_out_channels=boc, with_encoder=True, **kw), 31).to(bf16)
    ours = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True,
                               mid_block_attention_type="spatial", block_out_channels=boc, **kw).to(bf16)
    ours.load_state_dict(ob.state_dict(), strict=True)
    return ob, ours


def test_vae_encode_host_logic_matches_oracle(monkeypatch):
    """encode: planar->channels-last, stride-2 convolutions as stride-1 + strided pick, mid block, conv_out, quant_conv."""
    cpu_ops.use_stand_ins(monkeypatch)
    ob, ours = _vae_pair_enc()
    x = torch.randn(1, 3, 9, 40, 56, generator=torch.Generator().manual_seed(7)).to(bf16)
    with torch.no_grad():
        ref = ob.encode_moments(x)
        got = ours.encode(x).latent_dist.parameters
    assert got.shape == ref.shape == (1, 32, 3, 5, 7)
    assert _rel(got, ref) < 3e-2


def test_vae_tiled_encode_host_logic_matches_oracle(monkeypatch):
    cpu_ops.use_stand_ins(monkeypatch)
    ob, ours = _vae_pair_enc(use_tiling=True, tile_sample_min_size=32)
    ob.tile_latent_min_size = ours.tile_latent_min_size  # 32 / 8
    x = torch.randn(1, 3, 5, 40, 56, generator=torch.Generator().manual_seed(9)).to(bf16)
    with torch.no_grad():
        ref = ob.encode_moments(x)
        got = ours.encode(x).latent_dist.parameters
    assert got.shape == ref.shape == (1, 32, 2, 5, 7)
    assert _rel(got, ref) < 3e-2


def test_posterior_object_surface():
    from easyanimate_b200.config import AutoencoderKLOutput, DiagonalGaussianDistribution
    m = torch.randn(2, 32, 3, 4, 5)
    d = DiagonalGaussianDistribution(m)
    assert torch.equal(d.mode(), m[:, :16]) and d.sample(generator=torch.Generator().manual_seed(0)).shape == (2, 16, 3, 4, 5)
    out = AutoencoderKLOutput(latent_dist=d)
    assert out[0] is d and out.latent_dist.parameters is m


# ---- row f4: fp8 weight storage (predict_t2v.py:37,106 + utils/fp8_optimization.py:6-35) and control_latents ----
def test_fp8_weight_storage_host_logic_matches_reference_mode(monkeypatch):
    """from_pretrained_2d(torch_dtype=float8_e4m3fn) semantics: every parameter is stored as e4m3 and expanded to bf16 around the
    module that uses it.  The oracle run with weights = bf16(e4m3(w)) is the reference's arithmetic; our staging path (head
    parameters once, one block at a time, q/k/v straight into the fused projection operand) must reproduce it."""
    cpu_ops.use_stand_ins(monkeypatch)
    cfg = dict(CFG, num_layers=3, mmdit_layers=2) if False else dict(CFG, num_layers=3)
    ob, ours = _models(cfg)
    q8 = {k: v.to(torch.float8_e4m3fn) for k, v in ob.state_dict().items()}
    ob.load_state_dict({k: v.to(bf16) for k, v in q8.items()})           # bf16(e4m3(w)): what each reference module computes with
    ours = ours.to(torch.float8_e4m3fn)
    assert ours.dtype == torch.float8_e4m3fn and all(p.dtype == torch.float8_e4m3fn for p in ours.parameters())
    g = torch.Generator().manual_seed(2)
    lat = torch.randn(2, 16, 3, 8, 12, generator=g).to(bf16)
    enc = (torch.randn(2, 9, 128, generator=g) * 3).to(bf16)
    t = torch.tensor([937.0, 421.0]).to(bf16)
    rope = dit.rope_for_video(64, 96, 3)
    with torch.no_grad():
        ref = ob(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope)[0]
        got = ours(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, return_dict=False)[0]
        again = ours(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, return_dict=False)[0]
    assert _rel(got, ref) < 2e-2 and torch.equal(got, again)
    # the staging block really is refilled per block: a model whose blocks differ must not reuse block 0's weights
    with torch.no_grad():
        ours.transformer_blocks[2].ff.net[2].weight.zero_()
        ob.transformer_blocks[2].ff.net[2].weight.zero_()
        ref2 = ob(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope)[0]
        got2 = ours(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, return_dict=False)[0]
    assert _rel(got2, ref2) < 2e-2 and not torch.equal(got2, got)


def test_control_latents_channel_concat_host_logic(monkeypatch):
    """v5.1 Control models: the pipeline concatenates control (and reference-image) latents on channels and hands them over as
    `control_latents` (pipeline_easyanimate_control.py:1066-1125,1229; transformer3d.py:1525-1526); with inpaint_latents too
    the order is hidden | inpaint | control."""
    cpu_ops.use_stand_ins(monkeypatch)
    cfg = dict(CFG, in_channels=16 + 17 + 16)
    ob, ours = _models(cfg)
    g = torch.Generator().manual_seed(3)
    lat = torch.randn(2, 16, 2, 8, 8, generator=g).to(bf16)
    inp = torch.randn(2, 17, 2, 8, 8, generator=g).to(bf16)
    ctl = torch.randn(2, 16, 2, 8, 8, generator=g).to(bf16)
    enc = (torch.randn(2, 9, 128, generator=g) * 3).to(bf16)
    t = torch.tensor([500.0, 500.0]).to(bf16)
    rope = dit.rope_for_video(64, 64, 2)
    with torch.no_grad():
        ref = ob(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, inpaint_latents=torch.cat([inp, ctl], 1))[0]
        got = ours(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, inpaint_latents=inp, control_latents=ctl,
                   return_dict=False)[0]
    assert _rel(got, ref) < 2e-2


@pytest.mark.parametrize("with_clip", [False, True])
def test_control_ref_and_clip_tokens_host_logic(monkeypatch, with_clip):
    """v5.1 Control with a reference image (transformer3d.py:1420-1429,1538-1561): ref_proj patch tokens + the resized 2-D
    sin-cos table REPLACE the text tokens; CLIP tokens (clip_proj) are concatenated in front of them."""
    cpu_ops.use_stand_ins(monkeypatch)
    cfg = dict(CFG, ref_channels=16, clip_channels=96, sample_width=20, sample_height=12)
    ob, ours = _models(cfg)
    assert ours.ref_pos_embedding.dtype == bf16 and torch.equal(ours.ref_pos_embedding, ob.ref_pos_embedding)
    g = torch.Generator().manual_seed(4)
    lat = torch.randn(2, 16, 2, 8, 12, generator=g).to(bf16)
    enc = (torch.randn(2, 9, 128, generator=g) * 3).to(bf16)
    refl = torch.randn(2, 16, 1, 8, 12, generator=g).to(bf16)
    clip = torch.randn(2, 5, 96, generator=g).to(bf16) if with_clip else None
    t = torch.tensor([500.0, 300.0]).to(bf16)
    rope = dit.rope_for_video(64, 96, 2)
    with torch.no_grad():
        ref = ob(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, ref_latents=refl, clip_encoder_hidden_states=clip)[0]
        got = ours(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, ref_latents=refl, clip_encoder_hidden_states=clip,
                   return_dict=False)[0]
        plain = ours(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, return_dict=False)[0]
    assert _rel(got, ref) < 2e-2 and _rel(got, plain) > 2 * _rel(got, ref)  # (the reference-image tokens do change the result)
    with pytest.raises(ValueError):
        ours(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, clip_encoder_hidden_states=torch.zeros(2, 5, 96).to(bf16))


def test_weight_data_edits_need_invalidate_weight_caches(monkeypatch):
    """The reference's LoRA merge writes `layer.weight.data += delta` (utils/lora_utils.py:425-429): no new storage, no version
    bump, so the fused q/k/v copy of an attention module cannot notice it.  `invalidate_weight_caches()` is the documented
    hand-shake; parameter updates that go through the version counter (load_state_dict, in-place ops) are picked up by themselves."""
    cpu_ops.use_stand_ins(monkeypatch)
    ob, ours = _models(CFG)
    g = torch.Generator().manual_seed(8)
    lat = torch.randn(1, 16, 2, 8, 12, generator=g).to(bf16)
    enc = (torch.randn(1, 9, 128, generator=g) * 3).to(bf16)
    t = torch.tensor([500.0]).to(bf16)
    rope = dit.rope_for_video(64, 96, 2)

    def run(m):
        with torch.no_grad():
            out = m(lat, t, encoder_hidden_states=enc, image_rotary_emb=rope, return_dict=False)
        return out[0]

    base = run(ours)
    w = ours.transformer_blocks[0].attn1.to_q.weight
    delta = torch.randn(w.shape, generator=g).to(bf16) * 0.05
    original = w.detach().clone()
    w.data += delta                                   # what merge_lora does
    ob.transformer_blocks[0].attn1.to_q.weight.data += delta
    assert torch.equal(run(ours), base)               # stale fused copy: the edit is invisible ...
    ours.invalidate_weight_caches()
    merged = run(ours)
    assert not torch.equal(merged, base) and _rel(merged, run(ob)) < 2e-2  # ... until the caches are dropped
    with torch.no_grad():
        w.copy_(original)                             # an in-place op on the parameter itself bumps its version: noticed
    assert torch.equal(run(ours), base)

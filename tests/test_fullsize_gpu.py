"""Parity at BASELINE.json's FULL sizes (49 frames @720x1280: 47 056 tokens, latent 13x90x160) through size-independent
properties - the oracle cannot run these sizes in seconds, so each check is either exact by construction or compared
with an fp32 PyTorch evaluation of a SAMPLE of the outputs (GPU only)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

S_FULL, S_TEXT = 47056, 256


def _rand(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(bf16)


def test_attention_full_sequence_sampled_rows_and_convexity():
    """softmax(QK^T/8)V over all 47 056 keys: (1) 192 sampled query rows against an fp32 evaluation of exactly those
    rows; (2) V = const => every output equals the constant (the weights of a row sum to one whatever the reference
    value subtracted inside the kernel); (3) outputs stay inside the per-channel [min, max] hull of V."""
    from easyanimate_b200 import ops
    B, H = 1, 3
    q, k, v = _rand((B, H, S_FULL, 64), 1, 1.5), _rand((B, H, S_FULL, 64), 2), _rand((B, H, S_FULL, 64), 3)
    ot, ov = ops.attention(q, k, v, S_TEXT)
    out = torch.cat([ot, ov], 1).view(B, S_FULL, H, 64)
    rows = torch.cat([torch.arange(0, 64), torch.arange(S_TEXT - 32, S_TEXT + 32), torch.arange(S_FULL - 64, S_FULL)]).cuda()
    ref = torch.softmax(q[:, :, rows].float() @ k.float().transpose(-1, -2) * 0.125, dim=-1) @ v.float()  # [B,H,192,64]
    torch.testing.assert_close(out[:, rows].permute(0, 2, 1, 3).float(), ref, rtol=2e-2, atol=2e-3)
    lo, hi = v.float().amin(dim=2), v.float().amax(dim=2)  # [B,H,64]
    o = out.permute(0, 2, 1, 3).float()
    assert (o >= lo[:, :, None] - 1e-2).all() and (o <= hi[:, :, None] + 1e-2).all()
    vc = torch.full_like(v, 0.7421875)
    ot, ov = ops.attention(q, k, vc, S_TEXT)
    assert torch.equal(ot, torch.full_like(ot, 0.7421875)) or (ot.float() - 0.7421875).abs().max() <= 2 ** -8
    assert (ov.float() - 0.7421875).abs().max() <= 2 ** -8


def test_gemm_full_token_count_sampled_rows():
    """[47 056, 3072] x [12 288, 3072]^T + bias with GELU(tanh) epilogue (the feed-forward up-projection of the 7B
    shape): 256 sampled rows against fp32."""
    from easyanimate_b200 import _lib as L
    from easyanimate_b200 import ops
    a, w, b = _rand((S_FULL, 3072), 4), _rand((12288, 3072), 5, 0.02), _rand((12288,), 6)
    out = ops.gemm(a, w, b, epilogue=L.EPI_BIAS_GELU)
    rows = torch.randint(0, S_FULL, (256,), generator=torch.Generator().manual_seed(0)).cuda()
    ref = torch.nn.functional.gelu(a[rows].float() @ w.float().t() + b.float(), approximate="tanh")
    torch.testing.assert_close(out[rows].float(), ref, rtol=2 ** -7, atol=2e-2)
    assert torch.isfinite(out).all()


def test_dit_block_full_token_count_is_identity_when_gates_are_zero():
    """AdaLN-zero: with the modulation linears zeroed, every gate is 0 and EasyAnimateDiTBlock must return its inputs
    bit for bit (attention.py:1137-1163) whatever attention and feed-forward computed - at the full 46 800 + 256 tokens."""
    from easyanimate_b200.transformer3d import EasyAnimateTransformer3DModel
    cfg = dict(num_attention_heads=8, attention_head_dim=64, in_channels=16, out_channels=16, patch_size=2, num_layers=1,
               time_embed_dim=128, add_norm_text_encoder=True, text_embed_dim=256, text_embed_dim_t5=None)
    with torch.device("cuda"):
        m = EasyAnimateTransformer3DModel(**cfg).to(bf16)
    with torch.no_grad():
        for n, p in m.named_parameters():
            p.normal_(0.0, 0.05)
        blk = m.transformer_blocks[0]
        for norm in (blk.norm1, blk.norm2):
            norm.linear.weight.zero_()
            norm.linear.bias.zero_()
    from easyanimate_b200.pipeline import rope_table
    from easyanimate_b200.transformer3d import _Workspace
    d, S_v = 8 * 64, S_FULL - S_TEXT
    x_v, x_t = _rand((S_v, d), 7), _rand((S_TEXT, d), 8)
    temb = _rand((1, 128), 9)
    rope = rope_table(720, 1280, 13, device="cuda")
    ws = _Workspace(1, S_v, S_TEXT, d, 8, 4 * d, torch.device("cuda"))
    with torch.no_grad():
        y_v, y_t = blk(x_v.clone(), x_t.clone(), temb, rope, ws)
    assert torch.equal(y_v, x_v) and torch.equal(y_t, x_t)
    # and with the gates open the block does change its inputs (the identity above is not a no-op kernel path)
    with torch.no_grad():
        blk.norm1.linear.bias.normal_(0.0, 0.5)
        z_v, _ = blk(x_v.clone(), x_t.clone(), temb, rope, ws)
    assert not torch.equal(z_v, x_v) and torch.isfinite(z_v).all()


def test_vae_decode_720p_is_causal_in_time():
    """CausalConv3d / per-frame GroupNorm / per-frame attention: decoding the first k latent frames gives exactly the
    first 4(k-1)+1 video frames of decoding all 13 (omnigen_enc_dec.py:586-677 processes latent frames in order with a
    causal cache) - at the full 90x160 latent, untiled."""
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    with torch.device("cuda"):
        vae = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True,
                                  mid_block_attention_type="spatial", mini_batch_decoder=1, scaling_factor=0.7125).to(bf16)
    with torch.no_grad():
        for n, p in vae.named_parameters():
            if p.dim() >= 2:
                p.normal_(0, (1.0 / p[0].numel()) ** 0.5)
            elif "norm" in n and n.endswith("weight"):
                p.normal_(1.0, 0.05)
            else:
                p.normal_(0, 0.05)
    vae.use_tiling = False
    z = _rand((1, 16, 13, 90, 160), 10)
    from easyanimate_b200 import vae_ops
    saved = vae_ops.CONV_VARIANT
    try:
        # (1) the 3-frame and the 13-frame decode take the same tile shapes for every layer (variant bit 2 of the ABI is
        # accepted and selects the same kernel)
        vae_ops.CONV_VARIANT = saved | 2
        with torch.no_grad():
            full = vae.decode(z).sample
            assert full.shape == (1, 3, 49, 720, 1280) and torch.isfinite(full).all()
            head = vae.decode(z[:, :, :3].contiguous()).sample
        assert head.shape == (1, 3, 9, 720, 1280)
        assert torch.equal(head, full[:, :, :9])
        # (2) the default configuration (CTA-pair convolutions on the large layers): same frames up to bf16 round-off
        vae_ops.CONV_VARIANT = saved
        with torch.no_grad():
            full_p = vae.decode(z).sample
            head_p = vae.decode(z[:, :, :3].contiguous()).sample
        assert torch.isfinite(full_p).all()
        d = (head_p.float() - full_p[:, :, :9].float()).abs()
        assert d.max() <= 0.5 and d.mean() <= 1e-2
        d2 = (full_p.float() - full.float()).abs()
        assert d2.max() <= 0.5 and d2.mean() <= 1e-2
    finally:
        vae_ops.CONV_VARIANT = saved

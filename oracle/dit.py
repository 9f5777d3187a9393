"""ORACLE (test infrastructure only) — CPU restatement of the EasyAnimateV5.1 MMDiT denoising step.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference`` legs may import
this module; it is the checker, never the product path.

PARITY PINNED for everything the reference repository itself defines: the reference's own
``easyanimate/models/{transformer3d,attention,processor,norm}.py`` are imported UNMODIFIED from /root/reference in the
authoring container (oracle/ref_dit.py) and this restatement reproduces ``EasyAnimateTransformer3DModel.forward`` bit
for bit in fp32 AND in bf16 with the same weights (tests/test_oracle_cpu.py::
test_dit_oracle_matches_live_reference_bit_for_bit), including the I2V ``inpaint_latents`` branch and a six-call
TeaCache sequence (skip decisions and outputs); ``tests/golden/dit_ref_*.safetensors`` hold inputs and outputs produced
BY THE REFERENCE (tests/golden/make_golden.py), so the pin travels to the GPU box.
What stays unpinned is third-party: ``diffusers`` (pinned ``>=0.30.1,<=0.31.0`` in /root/reference/requirements.txt:25)
is neither installed nor vendored and there is no network, so the diffusers building blocks the reference calls
(Attention container, FeedForward/GELU, AdaLayerNorm, Timesteps, TimestepEmbedding, apply_rotary_emb,
get_3d_rotary_pos_embed, FlowMatchEulerDiscreteScheduler) are restated from their published 0.30/0.31 algorithms - here
and, for running the reference's files, in oracle/_refshim/diffusers.  The scheduler and the RoPE table are therefore
checked by properties and regression fixtures only (tests/test_oracle_cpu.py), not against diffusers itself.

Reference lines followed (paths relative to /root/reference):
  easyanimate/models/transformer3d.py:1351-1483  (EasyAnimateTransformer3DModel.__init__)
  easyanimate/models/transformer3d.py:1496-1689  (forward)
  easyanimate/models/attention.py:1028-1163      (EasyAnimateDiTBlock)
  easyanimate/models/processor.py:218-312        (EasyAnimateAttnProcessor2_0)
  easyanimate/models/norm.py:16-42,135-166       (FP32LayerNorm, EasyAnimateRMSNorm, EasyAnimateLayerNormZero)
  easyanimate/pipeline/pipeline_easyanimate.py:82-97,998-1011,1065-1111 (RoPE grid, denoise loop)

Every op is executed as a separate torch op in the module dtype, exactly like the reference does, so a bf16 run of
this oracle reproduces the reference's op-by-op bf16 rounding; an fp32/fp64 run is the "true value" yardstick.
State-dict keys equal the reference's so the same weights load into the oracle and into easyanimate_b200.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


# ---------------------------------------------------------------------------------------------------------------
# diffusers pieces (restated)
# ---------------------------------------------------------------------------------------------------------------
def get_timestep_embedding(timesteps: torch.Tensor, embedding_dim: int, flip_sin_to_cos: bool = False,
                           downscale_freq_shift: float = 1, scale: float = 1, max_period: int = 10000) -> torch.Tensor:
    """diffusers.models.embeddings.get_timestep_embedding (fp32 sinusoid)."""
    half_dim = embedding_dim // 2
    exponent = -math.log(max_period) * torch.arange(start=0, end=half_dim, dtype=torch.float32, device=timesteps.device)
    exponent = exponent / (half_dim - downscale_freq_shift)
    emb = torch.exp(exponent)
    emb = timesteps[:, None].float() * emb[None, :]
    emb = scale * emb
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
    if flip_sin_to_cos:
        emb = torch.cat([emb[:, half_dim:], emb[:, :half_dim]], dim=-1)
    if embedding_dim % 2 == 1:
        emb = F.pad(emb, (0, 1, 0, 0))
    return emb


class TimestepEmbedding(nn.Module):
    """diffusers TimestepEmbedding(in, time_embed_dim, act_fn='silu'): linear_1 -> SiLU -> linear_2."""

    def __init__(self, in_channels: int, time_embed_dim: int):
        super().__init__()
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.linear_2 = nn.Linear(time_embed_dim, time_embed_dim)

    def forward(self, sample):
        return self.linear_2(F.silu(self.linear_1(sample)))


class GELUProj(nn.Module):
    """diffusers.models.activations.GELU(dim_in, dim_out, approximate='tanh')."""

    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out)

    def forward(self, x):
        return F.gelu(self.proj(x), approximate="tanh")


class FeedForward(nn.Module):
    """diffusers FeedForward(dim, activation_fn='gelu-approximate', final_dropout=True): net = [GELU, Dropout, Linear, Dropout]."""

    def __init__(self, dim: int, mult: int = 4):
        super().__init__()
        self.net = nn.ModuleList([GELUProj(dim, dim * mult), nn.Dropout(0.0), nn.Linear(dim * mult, dim), nn.Dropout(0.0)])

    def forward(self, x):
        for m in self.net:
            x = m(x)
        return x


class Attention(nn.Module):
    """Parameter container matching diffusers Attention(query_dim, heads, dim_head, qk_norm='layer_norm', eps=1e-6, bias=True)."""

    def __init__(self, dim: int, heads: int, dim_head: int, eps: float = 1e-6):
        super().__init__()
        inner = heads * dim_head
        self.heads = heads
        self.to_q = nn.Linear(dim, inner, bias=True)
        self.to_k = nn.Linear(dim, inner, bias=True)
        self.to_v = nn.Linear(dim, inner, bias=True)
        self.norm_q = nn.LayerNorm(dim_head, eps=eps)
        self.norm_k = nn.LayerNorm(dim_head, eps=eps)
        self.to_out = nn.ModuleList([nn.Linear(inner, dim, bias=True), nn.Dropout(0.0)])


def apply_rotary_emb(x: torch.Tensor, freqs_cis: Tuple[torch.Tensor, torch.Tensor]) -> torch.Tensor:
    """diffusers apply_rotary_emb(use_real=True, use_real_unbind_dim=-1); x [B,H,S,D], cos/sin [S,D]."""
    cos, sin = freqs_cis
    cos, sin = cos[None, None].to(x.device), sin[None, None].to(x.device)
    x_real, x_imag = x.reshape(*x.shape[:-1], -1, 2).unbind(-1)
    x_rotated = torch.stack([-x_imag, x_real], dim=-1).flatten(3)
    return (x.float() * cos + x_rotated.float() * sin).to(x.dtype)


def get_1d_rotary_pos_embed(dim: int, pos, theta: float = 10000.0):
    if isinstance(pos, np.ndarray):
        pos = torch.from_numpy(pos)
    freqs = 1.0 / (theta ** (torch.arange(0, dim, 2)[: (dim // 2)].float() / dim))
    freqs = torch.outer(pos.float(), freqs)
    return freqs.cos().repeat_interleave(2, dim=1).float(), freqs.sin().repeat_interleave(2, dim=1).float()


def get_3d_rotary_pos_embed(embed_dim, crops_coords, grid_size, temporal_size, theta: int = 10000):
    """diffusers 0.30/0.31 get_3d_rotary_pos_embed(use_real=True) -> (cos, sin) each [T*H*W, embed_dim] fp32."""
    start, stop = crops_coords
    gh, gw = grid_size
    grid_h = np.linspace(start[0], stop[0], gh, endpoint=False, dtype=np.float32)
    grid_w = np.linspace(start[1], stop[1], gw, endpoint=False, dtype=np.float32)
    grid_t = np.linspace(0, temporal_size, temporal_size, endpoint=False, dtype=np.float32)
    dim_t, dim_h, dim_w = embed_dim // 4, embed_dim // 8 * 3, embed_dim // 8 * 3
    ft, fh, fw = (get_1d_rotary_pos_embed(dim_t, grid_t, theta), get_1d_rotary_pos_embed(dim_h, grid_h, theta),
                  get_1d_rotary_pos_embed(dim_w, grid_w, theta))

    def combine(t, h, w):
        t = t[:, None, None, :].expand(-1, gh, gw, -1)
        h = h[None, :, None, :].expand(temporal_size, -1, gw, -1)
        w = w[None, None, :, :].expand(temporal_size, gh, -1, -1)
        return torch.cat([t, h, w], dim=-1).reshape(temporal_size * gh * gw, -1)

    return combine(ft[0], fh[0], fw[0]).contiguous(), combine(ft[1], fh[1], fw[1]).contiguous()


def get_resize_crop_region_for_grid(src, tgt_width, tgt_height):
    """pipeline_easyanimate.py:82-97."""
    tw, th = tgt_width, tgt_height
    h, w = src
    r = h / w
    if r > (th / tw):
        resize_height = th
        resize_width = int(round(th / h * w))
    else:
        resize_width = tw
        resize_height = int(round(tw / w * h))
    crop_top = int(round((th - resize_height) / 2.0))
    crop_left = int(round((tw - resize_width) / 2.0))
    return (crop_top, crop_left), (crop_top + resize_height, crop_left + resize_width)


def rope_for_video(height: int, width: int, latent_frames: int, head_dim: int = 64, patch_size: int = 2):
    """pipeline_easyanimate.py:998-1011 for time_position_encoding_type == '3d_rope'. height/width in pixels."""
    grid_h, grid_w = height // 8 // patch_size, width // 8 // patch_size
    base_w, base_h = 720 // 8 // patch_size, 480 // 8 // patch_size
    crops = get_resize_crop_region_for_grid((grid_h, grid_w), base_w, base_h)
    return get_3d_rotary_pos_embed(head_dim, crops, grid_size=(grid_h, grid_w), temporal_size=latent_frames)


# ---------------------------------------------------------------------------------------------------------------
# EasyAnimate-owned modules
# ---------------------------------------------------------------------------------------------------------------
class FP32LayerNorm(nn.LayerNorm):
    """norm.py:16-26."""

    def forward(self, inputs):
        dt = inputs.dtype
        return F.layer_norm(inputs.float(), self.normalized_shape, self.weight.float(), self.bias.float(), self.eps).to(dt)


class EasyAnimateRMSNorm(nn.Module):
    """norm.py:28-39."""

    def __init__(self, hidden_size, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps

    def forward(self, hidden_states):
        input_dtype = hidden_states.dtype
        hidden_states = hidden_states.to(torch.float32)
        variance = hidden_states.pow(2).mean(-1, keepdim=True)
        hidden_states = hidden_states * torch.rsqrt(variance + self.variance_epsilon)
        return self.weight * hidden_states.to(input_dtype)


class EasyAnimateLayerNormZero(nn.Module):
    """norm.py:135-166."""

    def __init__(self, conditioning_dim, embedding_dim, eps=1e-5):
        super().__init__()
        self.linear = nn.Linear(conditioning_dim, 6 * embedding_dim, bias=True)
        self.norm = FP32LayerNorm(embedding_dim, eps=eps, elementwise_affine=True)

    def forward(self, hidden_states, encoder_hidden_states, temb):
        shift, scale, gate, enc_shift, enc_scale, enc_gate = self.linear(F.silu(temb)).chunk(6, dim=1)
        hidden_states = self.norm(hidden_states) * (1 + scale)[:, None, :] + shift[:, None, :]
        encoder_hidden_states = self.norm(encoder_hidden_states) * (1 + enc_scale)[:, None, :] + enc_shift[:, None, :]
        return hidden_states, encoder_hidden_states, gate[:, None, :], enc_gate[:, None, :]


class AdaLayerNorm(nn.Module):
    """diffusers AdaLayerNorm(embedding_dim=time_embed_dim, output_dim=2*dim, chunk_dim=1): shift first, then scale."""

    def __init__(self, embedding_dim, output_dim, eps):
        super().__init__()
        self.linear = nn.Linear(embedding_dim, output_dim)
        self.norm = nn.LayerNorm(output_dim // 2, eps, True)

    def forward(self, x, temb):
        temb = self.linear(F.silu(temb))
        shift, scale = temb.chunk(2, dim=1)
        return self.norm(x) * (1 + scale[:, None, :]) + shift[:, None, :]


def joint_attention(attn1: Attention, attn2: Optional[Attention], hidden_states, encoder_hidden_states, image_rotary_emb):
    """processor.py:218-312 (EasyAnimateAttnProcessor2_0.__call__), attention_mask=None."""
    text_seq_length = encoder_hidden_states.size(1)
    batch_size = encoder_hidden_states.shape[0]
    heads = attn1.heads
    if attn2 is None:
        hidden_states = torch.cat([encoder_hidden_states, hidden_states], dim=1)

    def proj(a: Attention, x):
        q, k, v = a.to_q(x), a.to_k(x), a.to_v(x)
        hd = k.shape[-1] // heads
        q = q.view(batch_size, -1, heads, hd).transpose(1, 2)
        k = k.view(batch_size, -1, heads, hd).transpose(1, 2)
        v = v.view(batch_size, -1, heads, hd).transpose(1, 2)
        return a.norm_q(q), a.norm_k(k), v

    query, key, value = proj(attn1, hidden_states)
    if attn2 is not None:
        qt, kt, vt = proj(attn2, encoder_hidden_states)
        query = torch.cat([qt, query], dim=2)
        key = torch.cat([kt, key], dim=2)
        value = torch.cat([vt, value], dim=2)
    if image_rotary_emb is not None:
        query[:, :, text_seq_length:] = apply_rotary_emb(query[:, :, text_seq_length:], image_rotary_emb)
        key[:, :, text_seq_length:] = apply_rotary_emb(key[:, :, text_seq_length:], image_rotary_emb)
    hidden_states = F.scaled_dot_product_attention(query, key, value, attn_mask=None, dropout_p=0.0, is_causal=False)
    hidden_states = hidden_states.transpose(1, 2).reshape(batch_size, -1, heads * query.shape[-1])
    if attn2 is None:
        hidden_states = attn1.to_out[0](hidden_states)
        encoder_hidden_states, hidden_states = hidden_states.split(
            [text_seq_length, hidden_states.size(1) - text_seq_length], dim=1)
    else:
        encoder_hidden_states, hidden_states = hidden_states.split(
            [text_seq_length, hidden_states.size(1) - text_seq_length], dim=1)
        hidden_states = attn1.to_out[0](hidden_states)
        encoder_hidden_states = attn2.to_out[0](encoder_hidden_states)
    return hidden_states, encoder_hidden_states


class EasyAnimateDiTBlock(nn.Module):
    """attention.py:1028-1163 (after_norm=False, is_swa=False)."""

    def __init__(self, dim, num_attention_heads, attention_head_dim, time_embed_dim, norm_eps=1e-5, is_mmdit_block=True):
        super().__init__()
        self.norm1 = EasyAnimateLayerNormZero(time_embed_dim, dim, norm_eps)
        self.attn1 = Attention(dim, num_attention_heads, attention_head_dim, eps=1e-6)
        self.attn2 = Attention(dim, num_attention_heads, attention_head_dim, eps=1e-6) if is_mmdit_block else None
        self.norm2 = EasyAnimateLayerNormZero(time_embed_dim, dim, norm_eps)
        self.ff = FeedForward(dim)
        self.txt_ff = FeedForward(dim) if is_mmdit_block else None

    def forward(self, hidden_states, encoder_hidden_states, temb, image_rotary_emb=None):
        n_h, n_e, gate_msa, enc_gate_msa = self.norm1(hidden_states, encoder_hidden_states, temb)
        a_h, a_e = joint_attention(self.attn1, self.attn2, n_h, n_e, image_rotary_emb)
        hidden_states = hidden_states + gate_msa * a_h
        encoder_hidden_states = encoder_hidden_states + enc_gate_msa * a_e
        n_h, n_e, gate_ff, enc_gate_ff = self.norm2(hidden_states, encoder_hidden_states, temb)
        n_h = self.ff(n_h)
        n_e = self.txt_ff(n_e) if self.txt_ff is not None else self.ff(n_e)
        hidden_states = hidden_states + gate_ff * n_h
        encoder_hidden_states = encoder_hidden_states + enc_gate_ff * n_e
        return hidden_states, encoder_hidden_states


class OracleTeaCache:
    """transformer3d.py:90-121 state holder (the decision logic is restated inside OracleTransformer3D.forward)."""

    def __init__(self, coefficients, num_steps, rel_l1_thresh=0.0):
        self.coefficients, self.num_steps, self.rel_l1_thresh = list(coefficients), num_steps, rel_l1_thresh
        self.cnt, self.accumulated_rel_l1_distance, self.skipped = 0, 0, 0
        self.previous_modulated_input = None
        self.previous_residual = None


def sincos_pos_embed_2d(embed_dim, grid_size, base_size=16):
    """diffusers 0.30/0.31 `get_2d_sincos_pos_embed(embed_dim, (H, W))` restated from its published algorithm (third-party,
    unpinned): numpy float64 [H*W, embed_dim]."""
    def one_d(dim, pos):
        omega = 1.0 / 10000 ** (np.arange(dim // 2, dtype=np.float64) / (dim / 2.0))
        out = np.einsum("m,d->md", pos.reshape(-1), omega)
        return np.concatenate([np.sin(out), np.cos(out)], axis=1)
    grid_h = np.arange(grid_size[0], dtype=np.float32) / (grid_size[0] / base_size)
    grid_w = np.arange(grid_size[1], dtype=np.float32) / (grid_size[1] / base_size)
    grid = np.stack(np.meshgrid(grid_w, grid_h), axis=0).reshape([2, 1, grid_size[1], grid_size[0]])
    return np.concatenate([one_d(embed_dim // 2, grid[0]), one_d(embed_dim // 2, grid[1])], axis=1)


class OracleTransformer3D(nn.Module):
    """transformer3d.py:1346-1689, v5.1 configuration space incl. the control model's ref / clip token branches
    (transformer3d.py:1420-1429,1538-1561); TeaCache via `teacache`."""

    def __init__(self, num_attention_heads=30, attention_head_dim=64, in_channels=16, out_channels=16, patch_size=2,
                 num_layers=30, mmdit_layers=10000, time_embed_dim=512, add_norm_text_encoder=True, text_embed_dim=3584,
                 text_embed_dim_t5=None, norm_eps=1e-5, flip_sin_to_cos=True, freq_shift=0, sample_width=90, sample_height=60,
                 ref_channels=None, clip_channels=None, **unused):
        super().__init__()
        self.cfg = dict(num_attention_heads=num_attention_heads, attention_head_dim=attention_head_dim,
                        in_channels=in_channels, out_channels=out_channels, patch_size=patch_size, num_layers=num_layers,
                        mmdit_layers=mmdit_layers, time_embed_dim=time_embed_dim,
                        add_norm_text_encoder=add_norm_text_encoder, text_embed_dim=text_embed_dim,
                        text_embed_dim_t5=text_embed_dim_t5, norm_eps=norm_eps, flip_sin_to_cos=flip_sin_to_cos,
                        freq_shift=freq_shift)
        d = num_attention_heads * attention_head_dim
        self.inner_dim, self.patch_size = d, patch_size
        self.flip_sin_to_cos, self.freq_shift = flip_sin_to_cos, freq_shift
        self.time_embedding = TimestepEmbedding(d, time_embed_dim)
        self.proj = nn.Conv2d(in_channels, d, kernel_size=(patch_size, patch_size), stride=patch_size, bias=True)
        if not add_norm_text_encoder:
            self.text_proj = nn.Linear(text_embed_dim, d)
            if text_embed_dim_t5 is not None:
                self.text_proj_t5 = nn.Linear(text_embed_dim_t5, d)
        else:
            self.text_proj = nn.Sequential(EasyAnimateRMSNorm(text_embed_dim), nn.Linear(text_embed_dim, d))
            if text_embed_dim_t5 is not None:
                self.text_proj_t5 = nn.Sequential(EasyAnimateRMSNorm(text_embed_dim), nn.Linear(text_embed_dim_t5, d))
        self.transformer_blocks = nn.ModuleList([
            EasyAnimateDiTBlock(d, num_attention_heads, attention_head_dim, time_embed_dim, norm_eps,
                                is_mmdit_block=i < mmdit_layers) for i in range(num_layers)])
        self.post_patch_height, self.post_patch_width = sample_height // patch_size, sample_width // patch_size
        if ref_channels is not None:  # transformer3d.py:1420-1426
            self.ref_proj = nn.Conv2d(ref_channels, d, kernel_size=(patch_size, patch_size), stride=patch_size, bias=True)
            self.register_buffer("ref_pos_embedding", torch.from_numpy(
                sincos_pos_embed_2d(d, (self.post_patch_height, self.post_patch_width))), persistent=False)
        if clip_channels is not None:  # transformer3d.py:1428-1429
            self.clip_proj = nn.Linear(clip_channels, d)
        self.norm_final = nn.LayerNorm(d, norm_eps, True)
        self.norm_out = AdaLayerNorm(time_embed_dim, 2 * d, norm_eps)
        self.proj_out = nn.Linear(d, patch_size * patch_size * out_channels)

    def forward(self, hidden_states, timestep, encoder_hidden_states=None, encoder_hidden_states_t5=None,
                image_rotary_emb=None, inpaint_latents=None, control_latents=None, ref_latents=None,
                clip_encoder_hidden_states=None, **ignored):
        batch_size, channels, video_length, height, width = hidden_states.size()
        p = self.patch_size
        temb = get_timestep_embedding(timestep, self.inner_dim, self.flip_sin_to_cos, self.freq_shift)
        temb = self.time_embedding(temb.to(dtype=hidden_states.dtype))
        if inpaint_latents is not None:
            hidden_states = torch.concat([hidden_states, inpaint_latents], 1)
        if control_latents is not None:
            hidden_states = torch.concat([hidden_states, control_latents], 1)
        x = hidden_states.permute(0, 2, 1, 3, 4).flatten(0, 1)  # (b f) c h w
        x = self.proj(x)
        x = x.unflatten(0, (batch_size, video_length)).permute(0, 2, 1, 3, 4)  # b c f h w
        hidden_states = x.flatten(2).transpose(1, 2)
        encoder_hidden_states = self.text_proj(encoder_hidden_states)
        if encoder_hidden_states_t5 is not None:
            encoder_hidden_states_t5 = self.text_proj_t5(encoder_hidden_states_t5)
            encoder_hidden_states = torch.cat([encoder_hidden_states, encoder_hidden_states_t5], dim=1).contiguous()
        if ref_latents is not None:  # transformer3d.py:1538-1556: the reference-image tokens REPLACE the text tokens
            rb, rc, rf, rh, rw = ref_latents.shape
            r = self.ref_proj(ref_latents.permute(0, 2, 1, 3, 4).flatten(0, 1))
            r = r.unflatten(0, (rb, rf)).permute(0, 2, 1, 3, 4).flatten(2).transpose(1, 2)  # [b, f*h*w, d]
            emb = hidden_states.size()[-1]
            pe = self.ref_pos_embedding.view(1, 1, self.post_patch_height, self.post_patch_width, emb).permute([0, 4, 1, 2, 3])
            pe = F.interpolate(pe, size=[1, height // p, width // p], mode="trilinear", align_corners=False)
            pe = pe.permute([0, 2, 3, 4, 1]).view(1, -1, emb)
            ref_latents = r + pe
            encoder_hidden_states = ref_latents
        if clip_encoder_hidden_states is not None:  # transformer3d.py:1558-1561
            clip_encoder_hidden_states = self.clip_proj(clip_encoder_hidden_states)
            encoder_hidden_states = torch.concat([clip_encoder_hidden_states, ref_latents], dim=1)
        # TeaCache (transformer3d.py:1563-1636)
        tc = getattr(self, "teacache", None)
        should_calc = True
        if tc is not None:
            modulated_inp, _, _, _ = self.transformer_blocks[0].norm1(hidden_states.clone(), encoder_hidden_states.clone(),
                                                                      temb.clone())
            if tc.cnt == 0 or tc.cnt == tc.num_steps - 1:
                tc.accumulated_rel_l1_distance = 0
            else:
                prev = tc.previous_modulated_input
                rel = ((torch.abs(modulated_inp - prev).mean()) / torch.abs(prev).mean()).item()
                tc.accumulated_rel_l1_distance += float(np.poly1d(tc.coefficients)(rel))
                if tc.accumulated_rel_l1_distance < tc.rel_l1_thresh:
                    should_calc = False
                else:
                    tc.accumulated_rel_l1_distance = 0
            tc.previous_modulated_input = modulated_inp
            tc.cnt += 1
            if tc.cnt == tc.num_steps:
                tc.cnt, tc.previous_modulated_input, tc.previous_residual = 0, None, None
        if not should_calc:
            tc.skipped += 1
            hidden_states = hidden_states + tc.previous_residual
        else:
            ori_hidden_states = hidden_states.clone()
            for block in self.transformer_blocks:
                hidden_states, encoder_hidden_states = block(hidden_states, encoder_hidden_states, temb, image_rotary_emb)
            hidden_states = torch.cat([encoder_hidden_states, hidden_states], dim=1)
            hidden_states = self.norm_final(hidden_states)
            hidden_states = hidden_states[:, encoder_hidden_states.size()[1]:]
            hidden_states = self.norm_out(hidden_states, temb=temb)
            if tc is not None:
                tc.previous_residual = hidden_states - ori_hidden_states
        hidden_states = self.proj_out(hidden_states)
        output = hidden_states.reshape(batch_size, video_length, height // p, width // p, channels, p, p)
        output = output.permute(0, 4, 1, 2, 5, 3, 6).flatten(5, 6).flatten(3, 4)
        return (output,)


# ---------------------------------------------------------------------------------------------------------------
# scheduler + denoise loop
# ---------------------------------------------------------------------------------------------------------------
class FlowMatchEulerScheduler:
    """diffusers FlowMatchEulerDiscreteScheduler (0.30/0.31) restated: set_timesteps + step."""

    def __init__(self, num_train_timesteps=1000, shift=1.0, use_dynamic_shifting=False):
        self.num_train_timesteps, self.shift, self.use_dynamic_shifting = num_train_timesteps, shift, use_dynamic_shifting
        timesteps = np.linspace(1, num_train_timesteps, num_train_timesteps, dtype=np.float32)[::-1].copy()
        sigmas = torch.from_numpy(timesteps).to(dtype=torch.float32) / num_train_timesteps
        if not use_dynamic_shifting:
            sigmas = shift * sigmas / (1 + (shift - 1) * sigmas)
        self.sigma_min, self.sigma_max = sigmas[-1].item(), sigmas[0].item()
        self.order = 1

    def _sigma_to_t(self, sigma):
        return sigma * self.num_train_timesteps

    def set_timesteps(self, num_inference_steps, mu: Optional[float] = None):
        timesteps = np.linspace(self._sigma_to_t(self.sigma_max), self._sigma_to_t(self.sigma_min), num_inference_steps)
        sigmas = timesteps / self.num_train_timesteps
        if self.use_dynamic_shifting:
            sigmas = math.exp(mu) / (math.exp(mu) + (1 / sigmas - 1) ** 1.0)
        else:
            sigmas = self.shift * sigmas / (1 + (self.shift - 1) * sigmas)
        sigmas = torch.from_numpy(sigmas).to(dtype=torch.float32)
        self.timesteps = sigmas * self.num_train_timesteps
        self.sigmas = torch.cat([sigmas, torch.zeros(1)])
        self.step_index = 0

    def step(self, model_output, sample):
        sample = sample.to(torch.float32)
        sigma, sigma_next = self.sigmas[self.step_index], self.sigmas[self.step_index + 1]
        prev_sample = sample + (sigma_next - sigma) * model_output
        self.step_index += 1
        return prev_sample.to(model_output.dtype)


@torch.no_grad()
def denoise_loop(model: OracleTransformer3D, latents, prompt_embeds, negative_prompt_embeds, rope, num_steps: int,
                 guidance_scale: float = 6.0, shift: float = 1.0, inpaint_latents=None):
    """pipeline_easyanimate.py:1052-1111 with synthetic embeds: CFG batch = [negative, positive]."""
    sched = FlowMatchEulerScheduler(shift=shift)
    sched.set_timesteps(num_steps, mu=1.0)
    do_cfg = guidance_scale > 1.0
    embeds = torch.cat([negative_prompt_embeds, prompt_embeds]) if do_cfg else prompt_embeds
    for t in sched.timesteps:
        latent_model_input = torch.cat([latents] * 2) if do_cfg else latents
        t_expand = torch.tensor([t] * latent_model_input.shape[0]).to(dtype=latent_model_input.dtype)
        inp = torch.cat([inpaint_latents] * 2) if (inpaint_latents is not None and do_cfg) else inpaint_latents
        noise_pred = model(latent_model_input, t_expand, encoder_hidden_states=embeds, image_rotary_emb=rope,
                           inpaint_latents=inp)[0]
        if do_cfg:
            u, c = noise_pred.chunk(2)
            noise_pred = u + guidance_scale * (c - u)
        latents = sched.step(noise_pred, latents)
    return latents


def init_weights_(module: nn.Module, seed: int = 1234, std: float = 0.02):
    """Synthetic init: weights ~N(0,std), norm weights 1+N(0,std), biases N(0,std); AdaLN linears
    larger (std 0.1) so gates/scales exercise every branch."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            is_norm_w = p.dim() == 1 and name.endswith("weight") and (
                "norm" in name or name.endswith("text_proj.0.weight") or name.endswith("text_proj_t5.0.weight"))
            s = 0.1 if (".norm1.linear." in name or ".norm2.linear." in name or name.startswith("norm_out.linear.")) else std
            v = torch.randn(p.shape, generator=g, dtype=torch.float32) * s
            if is_norm_w:
                v = 1.0 + v
            p.copy_(v.to(p.dtype))
    return module

"""ORACLE (test infrastructure only) — CPU restatement of AutoencoderKLMagvit.decode (and, as preparation for the I2V
conditioning, .encode) for EasyAnimateV5.1.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference`` legs may import
this module; it is the checker, never the product path.

PARITY PINNED: this restatement is checked (tests/test_oracle_vae.py, and the generator tests/golden/make_golden.py)
against the reference's own ``easyanimate.vae.ldm.models.omnigen_enc_dec.Decoder`` imported from /root/reference in
the authoring container (through a one-symbol ``diffusers.utils.is_torch_version`` stub, oracle/_refshim), in BOTH of
the reference's execution modes: chunked/cached (``cache_mag_vae=True``, the v5.1 default: padding_flag 3/4) and
whole-sequence; the committed fixtures under tests/golden/ come from the reference Decoder itself.

Reference lines followed (paths relative to /root/reference):
  easyanimate/models/autoencoder_magvit.py:94-200,271-317,319-337,381-448  (ctor, _decode/decode, blend, tiled_decode)
  easyanimate/vae/ldm/models/omnigen_enc_dec.py:368-465,555-677            (Decoder)
  easyanimate/vae/ldm/modules/vaemodules/common.py:31-179,254-323          (CausalConv3d, ResidualBlock3D)
  easyanimate/vae/ldm/modules/vaemodules/mid_blocks.py:38-196              (MidBlock3D)
  easyanimate/vae/ldm/modules/vaemodules/up_blocks.py:96-147,344-395       (Spatial/SpatialTemporal up blocks)
  easyanimate/vae/ldm/modules/vaemodules/upsamplers.py:21-37,123-153       (upsamplers)
  easyanimate/vae/ldm/modules/vaemodules/attention.py:391-423, attention_processors.py:68-139 (SpatialAttention)

The reference decodes one latent frame at a time and carries the last two input frames of every CausalConv3d in a
cache (padding_flag 3 for the first chunk, 4 afterwards).  That is arithmetically one causal convolution over the
whole sequence with the first frame replicated twice on the left; the first latent frame is not temporally
up-sampled, every other one is doubled by each SpatialTemporalUpsampler3D (nearest, because spatial_group_norm
switches the upsamplers to "nearest").  This module implements that whole-sequence form.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F


class CausalConv3d(nn.Conv3d):
    """common.py:31-96 with padding_flag == 0: left replicate-pad (k_t-1) frames, zero-pad 1 px spatially."""

    def __init__(self, in_channels, out_channels, kernel_size=3):
        super().__init__(in_channels, out_channels, kernel_size=kernel_size, padding=(0, 1, 1))
        self.temporal_padding = kernel_size - 1

    def forward(self, x):
        x = F.pad(x, pad=(0, 0, 0, 0, self.temporal_padding, 0), mode="replicate")
        return super().forward(x)


def frame_group_norm(norm: nn.GroupNorm, x):
    """common.py:301-305: 'b c t h w -> (b t) c h w' so statistics are per frame."""
    b, c, t, h, w = x.shape
    y = norm(x.permute(0, 2, 1, 3, 4).reshape(b * t, c, h, w))
    return y.reshape(b, t, c, h, w).permute(0, 2, 1, 3, 4)


class ResidualBlock3D(nn.Module):
    def __init__(self, in_channels, out_channels, groups=32, eps=1e-6):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps, affine=True)
        self.conv1 = CausalConv3d(in_channels, out_channels)
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps, affine=True)
        self.conv2 = CausalConv3d(out_channels, out_channels)
        self.shortcut = nn.Conv3d(in_channels, out_channels, kernel_size=1) if in_channels != out_channels else nn.Identity()

    def forward(self, x):
        shortcut = self.shortcut(x)
        x = F.silu(frame_group_norm(self.norm1, x))
        x = self.conv1(x)
        x = F.silu(frame_group_norm(self.norm2, x))
        x = self.conv2(x)
        return (x + shortcut) / 1.0


class SpatialAttention(nn.Module):
    """attention.py:391-423 + AttnProcessor2_0 (attention_processors.py:68-139): per-frame, 1 head of C channels."""

    def __init__(self, channels, heads=1, groups=32, eps=1e-6):
        super().__init__()
        self.nheads = heads
        self.scale = (channels // heads) ** -0.5
        self.group_norm = nn.GroupNorm(groups, channels, eps=eps, affine=True)
        self.to_q = nn.Linear(channels, channels, bias=True)
        self.to_k = nn.Linear(channels, channels, bias=True)
        self.to_v = nn.Linear(channels, channels, bias=True)
        self.to_out = nn.Linear(channels, channels, bias=True)

    def forward(self, x):
        b, c, t, h, w = x.shape
        hs = x.permute(0, 2, 3, 4, 1).reshape(b * t, h * w, c)
        residual = hs
        hs = self.group_norm(hs.transpose(1, 2)).transpose(1, 2)
        q, k, v = self.to_q(hs), self.to_k(hs), self.to_v(hs)
        hd = c // self.nheads
        q = q.view(b * t, -1, self.nheads, hd).transpose(1, 2)
        k = k.view(b * t, -1, self.nheads, hd).transpose(1, 2)
        v = v.view(b * t, -1, self.nheads, hd).transpose(1, 2)
        o = F.scaled_dot_product_attention(q, k, v, dropout_p=0.0, is_causal=False, scale=self.scale)
        o = o.transpose(1, 2).reshape(b * t, -1, c).to(q.dtype)
        o = self.to_out(o) + residual
        o = o / 1.0
        return o.reshape(b, t, h, w, c).permute(0, 4, 1, 2, 3)


class MidBlock3D(nn.Module):
    def __init__(self, channels, num_layers=2, add_attention=True):
        super().__init__()
        self.convs = nn.ModuleList([ResidualBlock3D(channels, channels)])
        self.attentions = nn.ModuleList([])
        for _ in range(num_layers - 1):
            self.attentions.append(SpatialAttention(channels) if add_attention else None)
            self.convs.append(ResidualBlock3D(channels, channels))

    def forward(self, x):
        x = self.convs[0](x)
        for attn, resnet in zip(self.attentions, self.convs[1:]):
            if attn is not None:
                x = attn(x)
            x = resnet(x)
        return x


class Upsampler(nn.Module):
    """upsamplers.py:21-37 (spatial) / :123-153 (spatial+temporal, nearest, first frame not doubled)."""

    def __init__(self, channels, temporal: bool):
        super().__init__()
        self.conv = CausalConv3d(channels, channels)
        self.temporal = temporal

    def forward(self, x):
        x = F.interpolate(x, scale_factor=(1, 2, 2), mode="nearest")
        x = self.conv(x)
        if self.temporal and x.shape[2] > 1:
            first, rest = x[:, :, :1], x[:, :, 1:]
            rest = F.interpolate(rest, scale_factor=(2, 1, 1), mode="nearest")
            x = torch.cat([first, rest], dim=2)
        return x


class UpBlock(nn.Module):
    def __init__(self, in_channels, out_channels, num_layers, add_upsample, temporal, upsampler_on_input_channels):
        super().__init__()
        self.convs = nn.ModuleList([ResidualBlock3D(in_channels if i == 0 else out_channels, out_channels)
                                    for i in range(num_layers)])
        # SpatialUpBlock3D builds its upsampler on in_channels (up_blocks.py:111-112), SpatialTemporalUpBlock3D on
        # out_channels (:379-380); they coincide for the released architecture.
        ch = in_channels if upsampler_on_input_channels else out_channels
        self.upsampler = Upsampler(ch, temporal) if add_upsample else None

    def forward(self, x):
        for conv in self.convs:
            x = conv(x)
        if self.upsampler is not None:
            x = self.upsampler(x)
        return x


class OracleDecoder(nn.Module):
    """omnigen_enc_dec.py:368-465 + single_forward :555-615 with spatial_group_norm=True, whole-sequence."""

    def __init__(self, in_channels=16, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 up_block_types=("SpatialUpBlock3D", "SpatialTemporalUpBlock3D", "SpatialTemporalUpBlock3D",
                                 "SpatialTemporalUpBlock3D"), mid_block_use_attention=True, norm_num_groups=32):
        super().__init__()
        self.conv_in = CausalConv3d(in_channels, block_out_channels[-1])
        self.mid_block = MidBlock3D(block_out_channels[-1], num_layers=layers_per_block, add_attention=mid_block_use_attention)
        self.up_blocks = nn.ModuleList([])
        rev = list(reversed(block_out_channels))
        out_ch = rev[0]
        for i, typ in enumerate(up_block_types):
            in_ch, out_ch = out_ch, rev[i]
            final = i == len(block_out_channels) - 1
            self.up_blocks.append(UpBlock(in_ch, out_ch, layers_per_block + 1, add_upsample=not final,
                                          temporal=typ == "SpatialTemporalUpBlock3D",
                                          upsampler_on_input_channels=typ == "SpatialUpBlock3D"))
        self.conv_norm_out = nn.GroupNorm(norm_num_groups, block_out_channels[0], eps=1e-6)
        self.conv_out = CausalConv3d(block_out_channels[0], out_channels)

    def forward(self, x):
        x = self.conv_in(x)
        x = self.mid_block(x)
        for up in self.up_blocks:
            x = up(x)
        x = F.silu(frame_group_norm(self.conv_norm_out, x))
        return self.conv_out(x)


class DownsampleConv3d(nn.Conv3d):
    """The convolution of SpatialDownsampler3D / SpatialTemporalDownsampler3D (downsamplers.py:24-46,74-96): kernel 3,
    stride (t_stride, 2, 2), no conv padding - the downsampler zero-pads one pixel on the right and bottom - and the causal
    left replicate pad of CausalConv3d.  Whole-sequence form of the chunked padding_flag 3/4 path (common.py:97-141): output
    frame k reads input frames (s k - 2, s k - 1, s k) with negative indices clamped to 0."""

    def __init__(self, channels, t_stride):
        super().__init__(channels, channels, kernel_size=3, stride=(t_stride, 2, 2), padding=0)

    def forward(self, x):
        x = F.pad(x, (0, 1, 0, 1))
        x = F.pad(x, pad=(0, 0, 0, 0, 2, 0), mode="replicate")
        return super().forward(x)


class Downsampler(nn.Module):
    def __init__(self, channels, temporal: bool):
        super().__init__()
        self.conv = DownsampleConv3d(channels, 2 if temporal else 1)

    def forward(self, x):
        return self.conv(x)


class DownBlock(nn.Module):
    """down_blocks.py:156-212 (SpatialDownBlock3D) / :272-328 (SpatialTemporalDownBlock3D), no gc_block."""

    def __init__(self, in_channels, out_channels, num_layers, add_downsample, temporal):
        super().__init__()
        self.convs = nn.ModuleList([ResidualBlock3D(in_channels if i == 0 else out_channels, out_channels)
                                    for i in range(num_layers)])
        self.downsampler = Downsampler(out_channels, temporal) if add_downsample else None

    def forward(self, x):
        for conv in self.convs:
            x = conv(x)
        if self.downsampler is not None:
            x = self.downsampler(x)
        return x


class OracleEncoder(nn.Module):
    """omnigen_enc_dec.py:24-155 + single_forward :225-272 with spatial_group_norm=True, whole-sequence: the reference
    encodes frame 0 alone and then mini_batch_encoder (4) frames at a time with the last two input frames of every
    CausalConv3d cached (padding_flag 3/4), which is one causal pass over 1 + 4m frames."""

    def __init__(self, in_channels=3, out_channels=16, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 down_block_types=("SpatialDownBlock3D", "SpatialTemporalDownBlock3D", "SpatialTemporalDownBlock3D",
                                   "SpatialTemporalDownBlock3D"), mid_block_use_attention=True, norm_num_groups=32,
                 double_z=True):
        super().__init__()
        self.conv_in = CausalConv3d(in_channels, block_out_channels[0])
        self.down_blocks = nn.ModuleList([])
        out_ch = block_out_channels[0]
        for i, typ in enumerate(down_block_types):
            in_ch, out_ch = out_ch, block_out_channels[i]
            final = i == len(block_out_channels) - 1
            self.down_blocks.append(DownBlock(in_ch, out_ch, layers_per_block, add_downsample=not final,
                                              temporal=typ == "SpatialTemporalDownBlock3D"))
        self.mid_block = MidBlock3D(block_out_channels[-1], num_layers=layers_per_block, add_attention=mid_block_use_attention)
        self.conv_norm_out = nn.GroupNorm(norm_num_groups, block_out_channels[-1], eps=1e-6)
        self.conv_out = CausalConv3d(block_out_channels[-1], 2 * out_channels if double_z else out_channels)

    def forward(self, x):
        assert (x.shape[2] - 1) % 4 == 0, "the reference's chunking needs 1 + 4m frames"
        # (contiguous: PyTorch's CPU bf16 conv3d intermittently returns NaN for a strided tile view with a degenerate
        #  width - 2 of 150 runs on an [1,3,5,32,8] slice; it changes nothing arithmetically)
        x = self.conv_in(x.contiguous())
        for down in self.down_blocks:
            x = down(x)
        x = self.mid_block(x)
        x = F.silu(frame_group_norm(self.conv_norm_out, x))
        return self.conv_out(x)


class OracleAutoencoderKLMagvit(nn.Module):
    """Decode side of autoencoder_magvit.py:59-505 (post_quant_conv + Decoder + tiling/blending)."""

    def __init__(self, latent_channels=16, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 mid_block_use_attention=True, use_tiling=False, use_tiling_decoder=False, tile_sample_min_size=384,
                 tile_overlap_factor=0.25, scaling_factor=0.7125, with_encoder=False, in_channels=3, **unused):
        super().__init__()
        self.decoder = OracleDecoder(latent_channels, out_channels, block_out_channels, layers_per_block,
                                     mid_block_use_attention=mid_block_use_attention)
        self.post_quant_conv = nn.Conv3d(latent_channels, latent_channels, kernel_size=1)
        self.use_tiling, self.use_tiling_decoder = use_tiling, use_tiling_decoder
        self.tile_sample_min_size, self.tile_overlap_factor = tile_sample_min_size, tile_overlap_factor
        self.tile_latent_min_size = int(tile_sample_min_size / (2 ** (len(block_out_channels) - 1)))
        self.scaling_factor = scaling_factor
        if with_encoder:  # registered AFTER the decode side so that init_weights_(seed) gives the decoder the same weights
            self.encoder = OracleEncoder(in_channels, latent_channels, block_out_channels, layers_per_block,
                                         mid_block_use_attention=mid_block_use_attention)
            self.quant_conv = nn.Conv3d(2 * latent_channels, 2 * latent_channels, kernel_size=1)

    @staticmethod
    def blend_v(a, b, blend_extent):
        blend_extent = min(a.shape[3], b.shape[3], blend_extent)
        for y in range(blend_extent):
            b[:, :, :, y, :] = a[:, :, :, -blend_extent + y, :] * (1 - y / blend_extent) + b[:, :, :, y, :] * (y / blend_extent)
        return b

    @staticmethod
    def blend_h(a, b, blend_extent):
        blend_extent = min(a.shape[4], b.shape[4], blend_extent)
        for x in range(blend_extent):
            b[:, :, :, :, x] = a[:, :, :, :, -blend_extent + x] * (1 - x / blend_extent) + b[:, :, :, :, x] * (x / blend_extent)
        return b

    def tiled_decode(self, z):
        tl = self.tile_latent_min_size
        overlap_size = int(tl * (1 - self.tile_overlap_factor))
        blend_extent = int(self.tile_sample_min_size * self.tile_overlap_factor)
        row_limit = self.tile_sample_min_size - blend_extent
        rows = []
        for i in range(0, z.shape[3], overlap_size):
            row = []
            for j in range(0, z.shape[4], overlap_size):
                tile = z[:, :, :, i:i + tl, j:j + tl].contiguous()  # (see OracleEncoder.forward)
                row.append(self.decoder(self.post_quant_conv(tile)))
            rows.append(row)
        result_rows = []
        for i, row in enumerate(rows):
            result_row = []
            for j, tile in enumerate(row):
                if i > 0:
                    tile = self.blend_v(rows[i - 1][j], tile, blend_extent)
                if j > 0:
                    tile = self.blend_h(row[j - 1], tile, blend_extent)
                result_row.append(tile[:, :, :, :row_limit, :row_limit])
            result_rows.append(torch.cat(result_row, dim=4))
        dec = torch.cat(result_rows, dim=3)
        lower_right = self.decoder(self.post_quant_conv(z[:, :, :, -tl:, -tl:]))
        H, W = lower_right.size(-2), lower_right.size(-1)
        x_weights = torch.linspace(0, 1, W).unsqueeze(0).repeat(H, 1)
        y_weights = torch.linspace(0, 1, H).unsqueeze(1).repeat(1, W)
        weights = torch.min(x_weights, y_weights)[None, None, None].to(dec.device)
        area = dec[:, :, :, -H:, -W:]
        dec[:, :, :, -H:, -W:] = weights * lower_right + (1 - weights) * area
        return dec

    def tiled_encode(self, x):
        """autoencoder_magvit.py:339-379: moments of overlapping 384-pixel tiles, blended in latent space."""
        ts, tl = self.tile_sample_min_size, self.tile_latent_min_size
        overlap_size = int(ts * (1 - self.tile_overlap_factor))
        blend_extent = int(tl * self.tile_overlap_factor)
        row_limit = tl - blend_extent
        rows = []
        for i in range(0, x.shape[3], overlap_size):
            row = []
            for j in range(0, x.shape[4], overlap_size):
                row.append(self.quant_conv(self.encoder(x[:, :, :, i:i + ts, j:j + ts])))
            rows.append(row)
        result_rows = []
        for i, row in enumerate(rows):
            result_row = []
            for j, tile in enumerate(row):
                if i > 0:
                    tile = self.blend_v(rows[i - 1][j], tile, blend_extent)
                if j > 0:
                    tile = self.blend_h(row[j - 1], tile, blend_extent)
                result_row.append(tile[:, :, :, :row_limit, :row_limit])
            result_rows.append(torch.cat(result_row, dim=4))
        return torch.cat(result_rows, dim=3)

    def encode_moments(self, x):
        """autoencoder_magvit.py:230-269: the moments tensor [B, 2*latent, T', h, w] (mean | logvar) the reference wraps in
        DiagonalGaussianDistribution; `.mode()` is its first half."""
        ts = self.tile_sample_min_size
        if self.use_tiling and (x.shape[-1] > ts or x.shape[-2] > ts):
            return self.tiled_encode(x)
        return self.quant_conv(self.encoder(x))

    def decode(self, z):
        tl = self.tile_latent_min_size
        if (self.use_tiling or self.use_tiling_decoder) and (z.shape[-1] > tl or z.shape[-2] > tl):
            return (self.tiled_decode(z),)
        return (self.decoder(self.post_quant_conv(z)),)


def init_weights_(module: nn.Module, seed: int = 4321):
    """Synthetic init that keeps activations O(1) through 35 conv layers: conv weights ~N(0, 1/fan_in) scaled."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if p.dim() >= 2:
                fan_in = p[0].numel()
                v = torch.randn(p.shape, generator=g) * (1.0 / fan_in) ** 0.5
            elif "norm" in name and name.endswith("weight"):
                v = 1.0 + 0.05 * torch.randn(p.shape, generator=g)
            else:
                v = 0.05 * torch.randn(p.shape, generator=g)
            p.copy_(v.to(p.dtype))
    return module

"""H100-native drop-in for the decode side of ``easyanimate.models.autoencoder_magvit.AutoencoderKLMagvit``.

Same constructor arguments, ``.config`` surface, ``decode`` signature and decoder ``state_dict`` keys as the reference
(/root/reference/easyanimate/models/autoencoder_magvit.py:59-505 with the Decoder of
easyanimate/vae/ldm/models/omnigen_enc_dec.py:339-677).  The nn.Conv3d / nn.GroupNorm / nn.Linear objects only own
parameters under the reference's key names; decode() runs exclusively on libea_b200.so kernels: channels-last
activations, wgmma implicit-GEMM causal convolutions executed over the WHOLE frame sequence in one launch per
layer (the reference's per-latent-frame loop with conv caches, omnigen_enc_dec.py:621-629 / common.py:97-141, is
arithmetically the same convolution), per-frame GroupNorm+SiLU kernels, wgmma GEMMs for the 1x1x1 shortcuts and
the mid-block spatial attention.

``encode`` (I2V / inpaint conditioning prep) runs on the same kernels: the encoder's
stride-2 convolutions (downsamplers.py:24-96) are the implicit-GEMM kernel with TMA element strides (no wasted FLOPs); the
stride-1 kernel + strided pick (output (t, i, j) of the strided conv == output (2t, 2i+1, 2j+1) of the stride-1 one) stays
as an A/B path (EA_ENC_STRIDED=0).  Host logic is checked on CPU against the oracle, which is pinned to the reference's
Encoder (tests/test_host_logic_cpu.py); GPU parity against the reference-minted fixture in tests/test_zz_vae_encode_gpu.py.
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn as nn

from . import _lib as L
from . import ops, vae_ops
from .config import (AutoencoderKLOutput, ConfigMixinLite, DecoderOutput, DiagonalGaussianDistribution, capture_init_config,
                     load_state_dict_from_dir)

bf16 = torch.bfloat16

DEFAULT_UP_BLOCKS = ("SpatialUpBlock3D", "SpatialTemporalUpBlock3D", "SpatialTemporalUpBlock3D", "SpatialTemporalUpBlock3D")
DEFAULT_DOWN_BLOCKS = ("SpatialDownBlock3D", "SpatialTemporalDownBlock3D", "SpatialTemporalDownBlock3D",
                       "SpatialTemporalDownBlock3D")


def str_eval(item):
    return eval(item) if isinstance(item, str) else item  # autoencoder_magvit.py:38-42


class _PackedConv(nn.Conv3d):
    """Owns a CausalConv3d's weight/bias (reference keys) and caches the tap-major packed copy the kernel consumes."""

    def __init__(self, cin, cout, cin_pad=0, cout_pad=0):
        super().__init__(cin, cout, kernel_size=3, padding=(0, 1, 1))
        self._cin_pad, self._cout_pad = cin_pad, cout_pad
        self._packed: Optional[tuple] = None

    def packed(self):
        w = self.weight
        key = ops.param_key(w)
        if self._packed is None or self._packed[0] != key:
            self._packed = (key, vae_ops.pack_conv_weight(w, self._cin_pad, self._cout_pad))
        return self._packed[1]

    def run(self, x, **kw):
        return vae_ops.conv3d_causal(x, self.packed(), self.bias, self.out_channels, **kw)


class _WholeFrame:
    """The four primitives the layer sequence below is written against, for whole frames on one GPU.  vae_strips.StripDecoder
    supplies the same four for one horizontal strip of the frame; every `run(x, ex)` takes either."""

    def conv(self, c: _PackedConv, x, **kw):
        return c.run(x, **kw)

    def gn(self, norm: nn.GroupNorm, x, silu):
        return vae_ops.groupnorm(x, norm.weight, norm.bias, norm.num_groups, norm.eps, silu)

    def attn(self, a: "_SpatialAttention", n, x):
        return a.attend(n, x)

    def upsample(self, x):
        return vae_ops.upsample2x(x)


_WHOLE_FRAME = _WholeFrame()


class _ResBlock(nn.Module):  # common.py:254-323
    def __init__(self, cin, cout, groups, eps=1e-6):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=eps, affine=True)
        self.conv1 = _PackedConv(cin, cout)
        self.norm2 = nn.GroupNorm(groups, cout, eps=eps, affine=True)
        self.conv2 = _PackedConv(cout, cout)
        self.shortcut = nn.Conv3d(cin, cout, kernel_size=1) if cin != cout else nn.Identity()

    def run(self, x, ex):
        T, H, W, Cin = x.shape
        if isinstance(self.shortcut, nn.Identity):
            sc = x
        else:
            co = self.shortcut.out_channels
            sc = ops.gemm(x.view(T * H * W, Cin), self.shortcut.weight.view(co, Cin), self.shortcut.bias).view(T, H, W, co)
        h = ex.gn(self.norm1, x, True)
        h = ex.conv(self.conv1, h)
        h = ex.gn(self.norm2, h, True)
        return ex.conv(self.conv2, h, residual=sc)


class _SpatialAttention(nn.Module):  # vaemodules/attention.py:63-160,391-423
    def __init__(self, channels, groups, eps=1e-6):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, channels, eps=eps, affine=True)
        self.to_q = nn.Linear(channels, channels, bias=True)
        self.to_k = nn.Linear(channels, channels, bias=True)
        self.to_v = nn.Linear(channels, channels, bias=True)
        self.to_out = nn.Linear(channels, channels, bias=True)
        self.scale = channels ** -0.5  # one head of `channels` dims
        self._fused: Optional[tuple] = None

    def _qkv(self):
        ps = (self.to_q.weight, self.to_k.weight, self.to_v.weight, self.to_q.bias, self.to_k.bias, self.to_v.bias)
        key = ops.param_key(*ps)
        if self._fused is None or self._fused[0] != key:
            self._fused = (key, torch.cat([p.detach() for p in ps[:3]], 0).contiguous(),
                           torch.cat([p.detach() for p in ps[3:]], 0).contiguous())
        return self._fused[1], self._fused[2]

    def run(self, x, ex):
        return ex.attn(self, ex.gn(self.group_norm, x, False), x)

    def attend(self, n, x, **kw):
        """n [T,H,W,C]: the normalised whole frames (keys / values); x [T,Hq,W,C]: the residual, one row per query (all of
        the frame, or with q_rows=(first, last) the pixels of n that a strip owns)."""
        T, H, W, Cc = n.shape
        Hq = x.shape[1]
        w, b = self._qkv()
        out = vae_ops.spatial_attention(n.view(T * H * W, Cc), w, b, self.to_out.weight, self.to_out.bias,
                                        x.view(T * Hq * W, Cc), T, self.scale, **kw)
        return out.view(T, Hq, W, Cc)


class _MidBlock(nn.Module):  # mid_blocks.py:38-196
    def __init__(self, channels, num_layers, add_attention, groups):
        super().__init__()
        self.convs = nn.ModuleList([_ResBlock(channels, channels, groups)])
        self.attentions = nn.ModuleList([])
        for _ in range(num_layers - 1):
            self.attentions.append(_SpatialAttention(channels, groups) if add_attention else None)
            self.convs.append(_ResBlock(channels, channels, groups))

    def run(self, x, ex):
        x = self.convs[0].run(x, ex)
        for attn, res in zip(self.attentions, self.convs[1:]):
            if attn is not None:
                x = attn.run(x, ex)
            x = res.run(x, ex)
        return x


class _Upsampler(nn.Module):  # upsamplers.py:21-37,123-153
    def __init__(self, channels, temporal):
        super().__init__()
        self.conv = _PackedConv(channels, channels)
        self.temporal = temporal

    def run(self, x, ex):
        x = ex.upsample(x)
        # nearest temporal x2 of every frame but the first is fused into the conv's store
        return ex.conv(self.conv, x, dup_frames=self.temporal and x.shape[0] > 1)


class _UpBlock(nn.Module):  # up_blocks.py:96-147,344-395
    def __init__(self, cin, cout, num_layers, add_upsample, temporal, upsampler_on_input, groups):
        super().__init__()
        self.convs = nn.ModuleList([_ResBlock(cin if i == 0 else cout, cout, groups) for i in range(num_layers)])
        self.upsampler = _Upsampler(cin if upsampler_on_input else cout, temporal) if add_upsample else None

    def run(self, x, ex):
        for c in self.convs:
            x = c.run(x, ex)
        if self.upsampler is not None:
            x = self.upsampler.run(x, ex)
        return x


class _Decoder(nn.Module):  # omnigen_enc_dec.py:339-677
    def __init__(self, in_channels, out_channels, up_block_types, block_out_channels, layers_per_block, norm_num_groups,
                 mid_block_use_attention, mid_block_attention_type):
        super().__init__()
        if mid_block_use_attention and mid_block_attention_type != "spatial":
            raise NotImplementedError("only mid_block_attention_type='spatial' (the v5/v5.1 VAE, "
                                      "vae/configs/autoencoder/autoencoder_kl_32x32x4_mag_v2.yaml:6) is implemented")
        self.conv_in = _PackedConv(in_channels, block_out_channels[-1], cin_pad=64)
        self.mid_block = _MidBlock(block_out_channels[-1], layers_per_block, mid_block_use_attention, norm_num_groups)
        self.up_blocks = nn.ModuleList([])
        rev = list(reversed(block_out_channels))
        out_ch = rev[0]
        for i, typ in enumerate(up_block_types):
            if typ not in ("SpatialUpBlock3D", "SpatialTemporalUpBlock3D"):
                raise NotImplementedError(f"up block type {typ} is not used by the v5/v5.1 VAE")
            in_ch, out_ch = out_ch, rev[i]
            final = i == len(block_out_channels) - 1
            self.up_blocks.append(_UpBlock(in_ch, out_ch, layers_per_block + 1, not final,
                                           typ == "SpatialTemporalUpBlock3D", typ == "SpatialUpBlock3D", norm_num_groups))
        self.conv_norm_out = nn.GroupNorm(norm_num_groups, block_out_channels[0], eps=1e-6)
        self.conv_out = _PackedConv(block_out_channels[0], out_channels, cout_pad=32)

    def run(self, x, ex):
        """x [T,h,w,64] channels-last (post_quant_conv already applied) -> planar [3,T',8h,8w]; with a strip executor, the
        strip's rows of both."""
        x = ex.conv(self.conv_in, x)
        x = self.mid_block.run(x, ex)
        for up in self.up_blocks:
            x = up.run(x, ex)
        x = ex.gn(self.conv_norm_out, x, True)
        return ex.conv(self.conv_out, x, out_planar=True)


class _Downsampler(nn.Module):  # downsamplers.py:24-46 (spatial), :74-96 (spatial + temporal)
    def __init__(self, channels, temporal):
        super().__init__()
        self.conv = _PackedConv(channels, channels)
        self.temporal = temporal

    strided_kernel = os.environ.get("EA_ENC_STRIDED", "1") != "0"  # 0: stride-1 kernel + strided pick (A/B, 4-8x the FLOPs)

    def run(self, x, ex):
        # CausalConv3d(kernel 3, stride (s_t, 2, 2), no spatial padding) after F.pad(x, (0,1,0,1)): output (t,i,j) reads
        # frames 2t-2..2t (clamped at 0) and pixels 2i..2i+2 / 2j..2j+2 with zeros past the right/bottom edge.  The
        # implicit-GEMM kernel does that directly (TMA element strides, ea_conv3d_args.stride_*); it is also output
        # (s_t*t, 2i+1, 2j+1) of the stride-1 causal convolution with 1-pixel zero padding, which the A/B path picks from.
        if self.strided_kernel:
            return ex.conv(self.conv, x, stride_t=2 if self.temporal else 1, stride_hw=2)
        y = ex.conv(self.conv, x)
        if self.temporal:
            y = y[::2]
        return y[:, 1::2, 1::2].contiguous()


class _DownBlock(nn.Module):  # down_blocks.py:156-212, 272-328
    def __init__(self, cin, cout, num_layers, add_downsample, temporal, groups):
        super().__init__()
        self.convs = nn.ModuleList([_ResBlock(cin if i == 0 else cout, cout, groups) for i in range(num_layers)])
        self.downsampler = _Downsampler(cout, temporal) if add_downsample else None

    def run(self, x, ex):
        for c in self.convs:
            x = c.run(x, ex)
        if self.downsampler is not None:
            x = self.downsampler.run(x, ex)
        return x


class _Encoder(nn.Module):  # omnigen_enc_dec.py:24-337
    def __init__(self, in_channels, latent_channels, down_block_types, block_out_channels, layers_per_block, norm_num_groups,
                 mid_block_use_attention):
        super().__init__()
        self.conv_in = _PackedConv(in_channels, block_out_channels[0], cin_pad=64)
        self.down_blocks = nn.ModuleList([])
        out_ch = block_out_channels[0]
        for i, typ in enumerate(down_block_types):
            if typ not in ("SpatialDownBlock3D", "SpatialTemporalDownBlock3D"):
                raise NotImplementedError(f"down block type {typ} is not used by the v5/v5.1 VAE")
            in_ch, out_ch = out_ch, block_out_channels[i]
            final = i == len(block_out_channels) - 1
            self.down_blocks.append(_DownBlock(in_ch, out_ch, layers_per_block, not final,
                                               typ == "SpatialTemporalDownBlock3D", norm_num_groups))
        self.mid_block = _MidBlock(block_out_channels[-1], layers_per_block, mid_block_use_attention, norm_num_groups)
        self.conv_norm_out = nn.GroupNorm(norm_num_groups, block_out_channels[-1], eps=1e-6)
        self.conv_out = _PackedConv(block_out_channels[-1], 2 * latent_channels, cout_pad=32)

    def run(self, x, ex):
        """x [T,H,W,64] channels-last (RGB in the first 3 channels) -> planar [2*latent, T', H/8, W/8]."""
        x = ex.conv(self.conv_in, x)
        for down in self.down_blocks:
            x = down.run(x, ex)
        x = self.mid_block.run(x, ex)
        x = ex.gn(self.conv_norm_out, x, True)
        return ex.conv(self.conv_out, x, out_planar=True)


def _require_cuda(t: torch.Tensor, what: str) -> None:
    """There is no CPU path: decode / encode refuse host tensors.  (One function so that the CPU host-logic tests, which swap
    the kernels for torch stand-ins, can lift exactly this guard and nothing else.)"""
    if not t.is_cuda:
        raise L.EaError(f"easyanimate_b200 has no CPU path: {what} must be on a CUDA device")


def _stitch_tiles(rows, blend_extent: int, row_limit: int) -> torch.Tensor:
    """rows[i][j] [1,C,T,h,w]: overlapping tiles in row-major order.  Every tile is blended (in place) over `blend_extent`
    rows / columns with the tile above it and the tile to its left, and its first `row_limit` rows and columns are copied
    to their place in the result (autoencoder_magvit.py:360-373 in tiled_encode, :403-416 in tiled_decode)."""
    first = rows[0][0]
    widths = [min(t.shape[4], row_limit) for t in rows[0]]
    heights = [min(r[0].shape[3], row_limit) for r in rows]
    out = torch.empty((1, first.shape[1], first.shape[2], sum(heights), sum(widths)), device=first.device, dtype=bf16)
    r0 = 0
    for i, row in enumerate(rows):
        c0 = 0
        for j, tile in enumerate(row):
            if i > 0:
                vae_ops.tile_blend(rows[i - 1][j], tile, blend_extent, 0)
            if j > 0:
                vae_ops.tile_blend(row[j - 1], tile, blend_extent, 1)
            vae_ops.copy2d(tile, out, heights[i], widths[j], r0, c0)
            c0 += widths[j]
        r0 += heights[i]
    return out


class AutoencoderKLMagvit(nn.Module, ConfigMixinLite):
    _supports_gradient_checkpointing = False

    def __init__(
        self,
        in_channels: int = 3,
        out_channels: int = 3,
        ch=128,
        ch_mult=[1, 2, 4, 4],
        block_out_channels=[128, 256, 512, 512],
        use_gc_blocks=None,
        down_block_types: tuple = None,
        up_block_types: tuple = None,
        mid_block_type: str = "MidBlock3D",
        mid_block_use_attention: bool = True,
        mid_block_attention_type: str = "3d",
        mid_block_num_attention_heads: int = 1,
        layers_per_block: int = 2,
        act_fn: str = "silu",
        num_attention_heads: int = 1,
        latent_channels: int = 4,
        norm_num_groups: int = 32,
        scaling_factor: float = 0.1825,
        force_upcast: float = True,
        slice_mag_vae=True,
        slice_compression_vae=False,
        cache_compression_vae=False,
        cache_mag_vae=False,
        use_tiling=False,
        use_tiling_encoder=False,
        use_tiling_decoder=False,
        mini_batch_encoder=9,
        mini_batch_decoder=3,
        upcast_vae=False,
        spatial_group_norm=False,
        tile_sample_min_size=384,
        tile_overlap_factor=0.25,
    ):
        super().__init__()
        object.__setattr__(self, "config", capture_init_config(self, locals()))
        up_block_types = str_eval(up_block_types) or DEFAULT_UP_BLOCKS
        if block_out_channels is None:
            block_out_channels = [ch * m for m in ch_mult]
        if not (cache_mag_vae and spatial_group_norm):
            raise NotImplementedError(
                "easyanimate_b200 implements the v5/v5.1 VAE execution mode only: cache_mag_vae=True with "
                "spatial_group_norm=True (config/easyanimate_video_v5.1_magvit_qwen.yaml:9-19). The slice_* modes of the "
                "v2-v4 VAEs compute different (chunk-local) results and are out of scope.")
        if use_gc_blocks is not None and any(use_gc_blocks):
            raise NotImplementedError("global-context blocks are not used by the v5/v5.1 VAE")
        if mid_block_num_attention_heads != 1 or act_fn != "silu" or mid_block_type != "MidBlock3D":
            raise NotImplementedError("only MidBlock3D / silu / 1 mid-block attention head is implemented")
        if latent_channels > 32:
            raise NotImplementedError("latent_channels > 32")
        self.decoder = _Decoder(latent_channels, out_channels, up_block_types, list(block_out_channels), layers_per_block,
                                norm_num_groups, mid_block_use_attention, mid_block_attention_type)
        self.quant_conv = nn.Conv3d(2 * latent_channels, 2 * latent_channels, kernel_size=1)
        self.post_quant_conv = nn.Conv3d(latent_channels, latent_channels, kernel_size=1)
        down_block_types = str_eval(down_block_types) or DEFAULT_DOWN_BLOCKS
        if 2 * latent_channels > 32 or in_channels > 32:
            raise NotImplementedError("encode needs 2*latent_channels <= 32 and in_channels <= 32")
        # registered after the decode side: module order (and with it any seeded init loop over named_parameters) of the
        # decoder is what it was before the encoder existed
        self.encoder = _Encoder(in_channels, latent_channels, down_block_types, list(block_out_channels), layers_per_block,
                                norm_num_groups, mid_block_use_attention)
        self.slice_mag_vae = slice_mag_vae
        self.slice_compression_vae = slice_compression_vae
        self.cache_compression_vae = cache_compression_vae
        self.cache_mag_vae = cache_mag_vae
        self.mini_batch_encoder = mini_batch_encoder
        self.mini_batch_decoder = mini_batch_decoder
        self.use_slicing = False
        self.use_tiling = use_tiling
        self.use_tiling_encoder = use_tiling_encoder
        self.use_tiling_decoder = use_tiling_decoder
        self.upcast_vae = upcast_vae
        self.tile_sample_min_size = tile_sample_min_size
        self.tile_overlap_factor = tile_overlap_factor
        self.tile_latent_min_size = int(self.tile_sample_min_size / (2 ** (len(ch_mult) - 1)))
        self.scaling_factor = scaling_factor
        self.tile_parallel_group = None  # torch.distributed group for tile-parallel tiled_decode (one all-gather)
        self.strip_parallel_group = None  # torch.distributed group for the strip-parallel UNTILED decode (vae_strips.py)
        self._latent_in_scale = 1.0      # decode_scaled() folds decode_latents' 1/scaling_factor into the first kernel

    def set_strip_parallel_group(self, group):
        """Shard the UNTILED decode of one video over the ranks of `group` by horizontal strips (vae_strips.py: halo rows for
        the convolutions, all-gathered GroupNorm sums, one all-gather of the frames); every rank must call decode with the
        same latents and gets the whole video.  None restores single-GPU decoding."""
        self.strip_parallel_group = group

    def set_tile_parallel_group(self, group):
        """Shard the reference's tiled_decode tiles over the ranks of `group` (every rank must call decode with the
        same latents); None restores single-GPU decoding."""
        self.tile_parallel_group = group

    # ----------------------------------------------------------------------------------------------------------
    def _decode_one(self, z: torch.Tensor) -> torch.Tensor:
        """z [C,T,h,w] planar -> [1,3,T',8h,8w]: post_quant_conv + Decoder (autoencoder_magvit.py:281-282)."""
        pq = self.post_quant_conv
        x = vae_ops.prepare_latents(z, pq.weight, pq.bias, 64, in_scale=self._latent_in_scale)
        return self.decoder.run(x, _WHOLE_FRAME).unsqueeze(0)

    def _tiled_decode_one(self, z: torch.Tensor) -> torch.Tensor:
        """autoencoder_magvit.py:381-448 for one batch element (z [C,T,h,w])."""
        tl = self.tile_latent_min_size
        overlap_size = int(tl * (1 - self.tile_overlap_factor))
        blend_extent = int(self.tile_sample_min_size * self.tile_overlap_factor)
        row_limit = self.tile_sample_min_size - blend_extent
        coords = [[(i, j) for j in range(0, z.shape[3], overlap_size)] for i in range(0, z.shape[2], overlap_size)]
        group = self.tile_parallel_group
        if group is None:
            rows = [[self._decode_one(z[:, :, i:i + tl, j:j + tl].contiguous()) for (i, j) in row] for row in coords]
            lower_right = None
        else:
            rows, lower_right = self._decode_tiles_parallel(z, coords, tl, group)
        dec = _stitch_tiles(rows, blend_extent, row_limit)
        if lower_right is None:
            lower_right = self._decode_one(z[:, :, -tl:, -tl:].contiguous())
        vae_ops.corner_blend(lower_right, dec)
        return dec

    def _decode_tiles_parallel(self, z, coords, tl, group):
        """Tile-parallel decode: the reference's tiles are independent decoder passes
        (autoencoder_magvit.py:389-402,418-426), so rank r decodes tiles r, r+N, ... of the row-major tile list
        (+ the lower-right corner pass as the last entry) and ONE all-gather of the padded tiles makes every rank
        hold all of them; blending then runs identically on every rank."""
        import torch.distributed as dist

        rank, world = dist.get_rank(group), dist.get_world_size(group)
        flat = [c for row in coords for c in row]
        specs = [z[:, :, i:i + tl, j:j + tl] for (i, j) in flat] + [z[:, :, -tl:, -tl:]]
        per_rank = (len(specs) + world - 1) // world
        Tp = 4 * (z.shape[1] - 1) + 1
        buf = torch.zeros((per_rank, self.config.out_channels, Tp, 8 * tl, 8 * tl), device=z.device, dtype=bf16)
        for slot, k in enumerate(k for k in range(len(specs)) if k % world == rank):
            out = self._decode_one(specs[k].contiguous())  # [1,3,T',8h,8w]
            vae_ops.copy2d(out, buf[slot:slot + 1], out.shape[3], out.shape[4], 0, 0)
        gathered = torch.empty((world * per_rank,) + tuple(buf.shape[1:]), device=z.device, dtype=bf16)
        dist.all_gather_into_tensor(gathered, buf, group=group)  # rank r's slots land at [r*per_rank, (r+1)*per_rank)

        def tile(k):
            hk, wk = 8 * specs[k].shape[2], 8 * specs[k].shape[3]
            return gathered[(k % world) * per_rank + k // world][None, :, :, :hk, :wk]

        rows, k = [], 0
        for row in coords:
            rows.append([tile(k + n) for n in range(len(row))])
            k += len(row)
        return rows, tile(len(specs) - 1).contiguous()

    def _bf16_input(self, t: torch.Tensor, verb: str, what: str) -> torch.Tensor:
        """The guards decode and encode share; `verb` / `what` word the errors."""
        if self.upcast_vae:
            raise NotImplementedError(f"upcast_vae (fp32 {verb}) is not implemented: easyanimate_b200 computes in bf16")
        if self.dtype != bf16:
            raise L.EaError("easyanimate_b200 computes in bf16: call .to(torch.bfloat16) on the module first")
        _require_cuda(t, what)
        return t.to(bf16)

    def _decode(self, z: torch.Tensor) -> torch.Tensor:
        z = self._bf16_input(z, "decode", "latents")
        tl = self.tile_latent_min_size
        tiled = (self.use_tiling or self.use_tiling_decoder) and (z.shape[-1] > tl or z.shape[-2] > tl)
        if not tiled and self.strip_parallel_group is not None:
            from .vae_strips import decode_strips
            outs = [decode_strips(self, zb, self.strip_parallel_group, self._latent_in_scale) for zb in z]
        else:
            outs = [(self._tiled_decode_one(zb) if tiled else self._decode_one(zb)) for zb in z]
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=0)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True, generator=None):
        """autoencoder_magvit.py:289-317."""
        decoded = self._decode(z)
        if not return_dict:
            return (decoded,)
        return DecoderOutput(sample=decoded)

    @torch.no_grad()
    def decode_scaled(self, latents: torch.Tensor, out: Optional[torch.Tensor] = None, dtype=torch.float32,
                      to_host: bool = False) -> torch.Tensor:
        """`EasyAnimatePipeline.decode_latents` (pipeline_easyanimate.py:722-742) as ONE call: `1 / scaling_factor *
        latents` is folded into the latent-preparation kernel (one bf16 rounding, like the reference's tensor op), the decode
        runs as in decode(), and the tail clamp(-1,1) -> /2+0.5 -> clamp(0,1) -> float32 (or uint8 = trunc(255*v), what
        utils.py:57 makes of the frames) is ONE kernel whose destination is `out`: a CUDA tensor, or with to_host=True a
        pinned host tensor the kernel writes over PCIe directly (no bf16 staging copy, no host-side .float()).  The call
        returns after the stream has been synchronised when the destination is on the host."""
        video = self.decode_scaled_video(latents)
        if out is None:
            out = (torch.empty(video.shape, dtype=dtype, pin_memory=True) if to_host
                   else torch.empty(video.shape, dtype=dtype, device=video.device))
        vae_ops.frames_out(video.contiguous(), out)
        if not out.is_cuda:
            torch.cuda.current_stream(video.device).synchronize()
        return out

    @torch.no_grad()
    def decode_scaled_video(self, latents: torch.Tensor) -> torch.Tensor:
        """decode_scaled before its output tail: the decoded bf16 video [B,3,F,H,W] on the device, for callers that apply
        a tail of their own (the long-video cross-fade, `vae_ops.frames_out_blend`)."""
        self._latent_in_scale = 1.0 / float(self.config.scaling_factor)
        try:
            return self._decode(latents)
        finally:
            self._latent_in_scale = 1.0

    # ---- encode (I2V / inpaint conditioning prep) ---------------------------------------------------------------
    def _encode_one(self, x: torch.Tensor) -> torch.Tensor:
        """x [C_in,T,H,W] planar bf16 -> moments planar [1, 2*latent, T', H/8, W/8]: Encoder + quant_conv
        (autoencoder_magvit.py:262-265).  T must be 1 + 4m (the reference's chunking, omnigen_enc_dec.py:283-290)."""
        cin = x.shape[0]
        if (x.shape[1] - 1) % 4:
            raise ValueError(f"encode needs 1 + 4m frames (the reference encodes frame 0 and then 4 frames at a time), got {x.shape[1]}")
        eye = torch.eye(cin, device=x.device, dtype=bf16)
        xin = vae_ops.prepare_latents(x, eye, torch.zeros(cin, device=x.device, dtype=bf16), 64)  # planar -> [T,H,W,64]
        h = self.encoder.run(xin, _WHOLE_FRAME)                     # planar [2L, T', h, w]
        qc = self.quant_conv
        m = vae_ops.prepare_latents(h, qc.weight, qc.bias, h.shape[0])  # 1x1x1 conv -> channels-last [T', h, w, 2L]
        return m.permute(3, 0, 1, 2).unsqueeze(0).contiguous()

    def _tiled_encode_one(self, x: torch.Tensor) -> torch.Tensor:
        """autoencoder_magvit.py:339-379 for one batch element: overlapping tiles encoded separately, moments blended."""
        ts, tl = self.tile_sample_min_size, self.tile_latent_min_size
        overlap_size = int(ts * (1 - self.tile_overlap_factor))
        blend_extent = int(tl * self.tile_overlap_factor)
        row_limit = tl - blend_extent
        rows = [[self._encode_one(x[:, :, i:i + ts, j:j + ts].contiguous()) for j in range(0, x.shape[3], overlap_size)]
                for i in range(0, x.shape[2], overlap_size)]
        return _stitch_tiles(rows, blend_extent, row_limit)

    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """autoencoder_magvit.py:229-269: x [B,3,T,H,W] in [-1,1] -> posterior over [B,latent,T',H/8,W/8] (T = 1 + 4m)."""
        x = self._bf16_input(x, "encode", "the video")
        ts = self.tile_sample_min_size
        tiled = (self.use_tiling or self.use_tiling_encoder) and (x.shape[-1] > ts or x.shape[-2] > ts)
        outs = [(self._tiled_encode_one(xb) if tiled else self._encode_one(xb.contiguous())) for xb in x]
        moments = outs[0] if len(outs) == 1 else torch.cat(outs, dim=0)
        posterior = DiagonalGaussianDistribution(moments)
        if not return_dict:
            return (posterior,)
        return AutoencoderKLOutput(latent_dist=posterior)

    def _clear_conv_cache(self):  # the whole-sequence kernels keep no cache; kept for API compatibility
        return None

    def invalidate_weight_caches(self) -> None:
        """Drop the packed convolution weights and fused q/k/v copies (rebuilt on the next call); needed only after edits of
        `weight.data` that bypass the parameters' version counters (see EasyAnimateTransformer3DModel.invalidate_weight_caches)."""
        for m in self.modules():
            if isinstance(m, _PackedConv):
                m._packed = None
            elif isinstance(m, _SpatialAttention):
                m._fused = None

    # ----------------------------------------------------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, pretrained_model_path, subfolder=None, **vae_additional_kwargs):
        """autoencoder_magvit.py:478-505: every key of the released checkpoint has a home (encoder, quant_conv, post_quant_conv,
        decoder); tensors whose shape does not match are skipped like the reference does."""
        if subfolder is not None:
            pretrained_model_path = os.path.join(pretrained_model_path, subfolder)
        config = cls.load_config(pretrained_model_path)
        model = cls.from_config(config, **vae_additional_kwargs)
        state_dict = load_state_dict_from_dir(pretrained_model_path)
        own = model.state_dict()
        filtered = {k: v for k, v in state_dict.items() if k in own and own[k].shape == v.shape}
        model.load_state_dict(filtered, strict=False)
        return model

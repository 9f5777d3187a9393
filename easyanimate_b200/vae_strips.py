"""Exact UNTILED decode of one latent video on several GPUs by horizontal strips.

The reference offers two decodes: untiled (autoencoder_magvit.py:271-287; the whole frame through the Decoder, per-frame
GroupNorm statistics and mid-block attention over the WHOLE frame) and `tiled_decode` (:381-448; 16 independent decoder passes
at 720p with tile-local statistics, 1.81x the FLOPs, a different result).  Tile-parallel decoding (`set_tile_parallel_group`)
shards the second; this module shards the FIRST: rank r owns rows [r h / N, (r+1) h / N) of the latent and the corresponding
rows of every activation.  Per layer:
  * 3x3x3 causal convolution (common.py:84-141): one halo row from each neighbour (zeros at the frame edge - the
    convolution's own zero padding) is attached above and below the strip and the kernel computes the strip's rows only
    (`ea_conv3d_args.out_row0 / out_rows`); the temporal taps stay inside the strip.  Output pixels see exactly the operands
    they see on one GPU, in the same k order: bit-identical.
  * per-frame GroupNorm (common.py:301-305): every rank reduces its rows to fp64 (sum, sum of squares) per (frame, group), ONE
    all-gather of [T, 32, 2] doubles, the pairs are added in rank order on every rank (`ea_groupnorm_sums / _finalize`).  Same
    statistics up to the association of the fp64 additions.
  * mid-block spatial attention (attention_processors.py:105-137): keys / values of the whole 90x160 frame are needed by every
    query - the normalised input (small: 13 x 14 400 x 512) is all-gathered and each rank evaluates its own query rows.
  * nearest x2 up-sampling, 1x1x1 shortcuts, SiLU: row-local.
  * ONE all-gather of the decoded RGB strips at the end (north_star: "a single NCCL all-gather over NVLink at the end of
    decode").
Collectives go through torch.distributed (NCCL on GPUs, gloo in the CPU tests); halo rows are point-to-point.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn as nn

from . import ops, vae_ops

bf16 = torch.bfloat16


def strip_bounds(h: int, world: int) -> List[int]:
    """Row r of the partition is [b[r], b[r+1]); every strip is non-empty for h >= world."""
    return [(h * r) // world for r in range(world + 1)]


class StripDecoder:
    def __init__(self, vae, group):
        import torch.distributed as dist

        self.dist = dist
        self.vae = vae
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.ranks = dist.get_process_group_ranks(group)  # global ranks, for point-to-point
        self.stats = {"halo_bytes": 0, "gathers": 0}

    # ---- communication --------------------------------------------------------------------------------------------
    def _halo_rows(self, x: torch.Tensor):
        """x [T,Hs,W,C] -> (row above, row below), each [T,1,W,C]; zeros at the top / bottom edge of the frame."""
        dist = self.dist
        T, Hs, W, Cc = x.shape
        top = torch.zeros((T, 1, W, Cc), device=x.device, dtype=x.dtype)
        bot = torch.zeros((T, 1, W, Cc), device=x.device, dtype=x.dtype)
        opsl = []
        keep = []
        if self.rank > 0:
            first = x[:, :1].contiguous()
            keep.append(first)
            opsl.append(dist.P2POp(dist.isend, first, self.ranks[self.rank - 1], self.group))
            opsl.append(dist.P2POp(dist.irecv, top, self.ranks[self.rank - 1], self.group))
        if self.rank < self.world - 1:
            last = x[:, -1:].contiguous()
            keep.append(last)
            opsl.append(dist.P2POp(dist.isend, last, self.ranks[self.rank + 1], self.group))
            opsl.append(dist.P2POp(dist.irecv, bot, self.ranks[self.rank + 1], self.group))
        if opsl:
            for w in dist.batch_isend_irecv(opsl):
                w.wait()
            self.stats["halo_bytes"] += top.numel() * 2 * (len(opsl) // 2)
        return top, bot

    def _gather_rows(self, x: torch.Tensor, dim: int, bounds: List[int]) -> torch.Tensor:
        """All-gather strips that differ in extent along `dim` (bounds in units of that dimension): padded to the tallest
        strip, ONE all_gather_into_tensor, then cut back and concatenated."""
        hmax = max(bounds[r + 1] - bounds[r] for r in range(self.world))
        pad_shape = list(x.shape)
        pad_shape[dim] = hmax
        buf = torch.zeros(pad_shape, device=x.device, dtype=x.dtype)
        buf.narrow(dim, 0, x.shape[dim]).copy_(x)
        out = torch.empty([self.world * pad_shape[0]] + pad_shape[1:], device=x.device, dtype=x.dtype)  # concatenated along dim 0
        self.dist.all_gather_into_tensor(out, buf, group=self.group)
        out = out.view([self.world] + pad_shape)
        self.stats["gathers"] += 1
        return torch.cat([out[r].narrow(dim, 0, bounds[r + 1] - bounds[r]) for r in range(self.world)], dim=dim)

    # ---- layers ---------------------------------------------------------------------------------------------------
    def conv(self, c, x: torch.Tensor, **kw) -> torch.Tensor:
        top, bot = self._halo_rows(x)
        xe = torch.cat([top, x, bot], dim=1)  # data movement only: [T, Hs+2, W, C]
        return vae_ops.conv3d_causal(xe, c.packed(), c.bias, c.out_channels, out_row0=1, out_rows=x.shape[1], **kw)

    def gn(self, norm: nn.GroupNorm, x: torch.Tensor, H_full: int, silu: bool) -> torch.Tensor:
        T, Hs, W, Cc = x.shape
        G = norm.num_groups
        sums = vae_ops.groupnorm_sums(x, G)
        all_sums = torch.empty((self.world * T, G, 2), device=x.device, dtype=torch.float64)
        self.dist.all_gather_into_tensor(all_sums, sums, group=self.group)
        all_sums = all_sums.view(self.world, T, G, 2)
        count = float(H_full) * W * (Cc // G)
        return vae_ops.groupnorm_from_sums(x, all_sums, count, norm.weight, norm.bias, G, norm.eps, silu)

    def res(self, r, x: torch.Tensor, H_full: int) -> torch.Tensor:
        T, Hs, W, Cin = x.shape
        if isinstance(r.shortcut, nn.Identity):
            sc = x
        else:
            co = r.shortcut.out_channels
            sc = ops.gemm(x.view(T * Hs * W, Cin), r.shortcut.weight.view(co, Cin), r.shortcut.bias).view(T, Hs, W, co)
        h = self.gn(r.norm1, x, H_full, True)
        h = self.conv(r.conv1, h)
        h = self.gn(r.norm2, h, H_full, True)
        return self.conv(r.conv2, h, residual=sc)

    def attn(self, a, x: torch.Tensor, bounds: List[int]) -> torch.Tensor:
        T, Hs, W, Cc = x.shape
        H_full = bounds[-1]
        n = self.gn(a.group_norm, x, H_full, False)
        n_full = self._gather_rows(n, 1, bounds).contiguous()  # [T, H, W, C]
        w, b = a._qkv()
        r0, r1 = bounds[self.rank], bounds[self.rank + 1]
        out = vae_ops.spatial_attention(n_full.view(T * H_full * W, Cc), w, b, a.to_out.weight, a.to_out.bias,
                                        x.view(T * Hs * W, Cc), T, a.scale, q_rows=(r0 * W, r1 * W))
        return out.view(T, Hs, W, Cc)

    # ---- the decoder ----------------------------------------------------------------------------------------------
    def decode(self, z: torch.Tensor, in_scale: float = 1.0) -> torch.Tensor:
        """z [C,T,h,w] planar (the SAME latent on every rank) -> [1,3,T',8h,8w] on every rank."""
        vae, dec = self.vae, self.vae.decoder
        h = z.shape[2]
        if h < self.world:
            raise ValueError(f"strip-parallel decode needs at least one latent row per rank ({h} rows, {self.world} ranks)")
        lat = strip_bounds(h, self.world)
        r0, r1 = lat[self.rank], lat[self.rank + 1]
        pq = vae.post_quant_conv
        x = vae_ops.prepare_latents(z[:, :, r0:r1].contiguous(), pq.weight, pq.bias, 64, in_scale=in_scale)
        scale = 1
        H = h
        x = self.conv(dec.conv_in, x)
        mid = dec.mid_block
        x = self.res(mid.convs[0], x, H)
        for a, r in zip(mid.attentions, mid.convs[1:]):
            if a is not None:
                x = self.attn(a, x, [b * scale for b in lat])
            x = self.res(r, x, H)
        for up in dec.up_blocks:
            for r in up.convs:
                x = self.res(r, x, H)
            if up.upsampler is not None:
                x = vae_ops.upsample2x(x)
                scale *= 2
                H *= 2
                x = self.conv(up.upsampler.conv, x, dup_frames=up.upsampler.temporal and x.shape[0] > 1)
        x = self.gn(dec.conv_norm_out, x, H, True)
        y = self.conv(dec.conv_out, x, out_planar=True)  # [3, T', 8 hs, 8 w]
        full = self._gather_rows(y, 2, [b * scale for b in lat])
        return full.unsqueeze(0)


def decode_strips(vae, z: torch.Tensor, group, in_scale: float = 1.0) -> torch.Tensor:
    return StripDecoder(vae, group).decode(z, in_scale)

"""world_size-2 gloo check of the VAE tile-parallel plumbing (partition of the reference's tiled_decode tiles over
ranks, padding, all-gather layout, reassembly order) with CPU stand-ins for the decoder pass and the copy kernel."""
import pytest
import torch
import torch.distributed as dist

from tests import cpu_ops
from tests.gloo import run_ranks

bf16 = torch.bfloat16


def _fake_decode(self, zt):  # [C,T,h,w] -> [1,3,T',8h,8w]: deterministic function of the tile content
    C, T, h, w = zt.shape
    base = zt.float().mean(dim=0)[:1].repeat_interleave(8, dim=1).repeat_interleave(8, dim=2)  # [1,8h,8w]
    return (base[None, None].expand(1, 3, 4 * (T - 1) + 1, 8 * h, 8 * w) + 1.0).to(bf16).contiguous()


def _tile_layout(rank):
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    m = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True, mid_block_attention_type="spatial",
                            block_out_channels=[64, 64, 128, 128], use_tiling=True, tile_sample_min_size=64)
    z = torch.randn(16, 2, 14, 20, generator=torch.Generator().manual_seed(3)).to(bf16)
    tl, ov = m.tile_latent_min_size, int(m.tile_latent_min_size * 0.75)
    coords = [[(i, j) for j in range(0, 20, ov)] for i in range(0, 14, ov)]
    with pytest.MonkeyPatch.context() as mp:
        cpu_ops.use_stand_ins(mp)
        mp.setattr(AutoencoderKLMagvit, "_decode_one", _fake_decode)
        rows, corner = m._decode_tiles_parallel(z, coords, tl, dist.new_group([0, 1]))
    ok = True
    for row_c, row_t in zip(coords, rows):
        for (i, j), t in zip(row_c, row_t):
            ok &= torch.equal(t, _fake_decode(m, z[:, :, i:i + tl, j:j + tl]))
    ok &= torch.equal(corner, _fake_decode(m, z[:, :, -tl:, -tl:]))
    return bool(ok), len(rows), len(rows[0])


def test_vae_tile_parallel_gather_reassembles_every_tile():
    res = run_ranks(_tile_layout, 2, timeout=120)
    assert all(r[0] for r in res) and res[0][1:] == (3, 4), res


# ---- the real module (all decoder layers, blending, corner pass) with torch stand-ins for the kernels (tests/cpu_ops.py) ----
def _real_decode(group):
    from oracle import vae
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    boc = [64, 64, 128, 128]
    ob = vae.init_weights_(vae.OracleAutoencoderKLMagvit(block_out_channels=boc, use_tiling=True, tile_sample_min_size=64), 21)
    m = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True, mid_block_attention_type="spatial",
                            block_out_channels=boc, use_tiling=True, tile_sample_min_size=64).to(bf16)
    m.load_state_dict({k: v.to(bf16) for k, v in ob.state_dict().items()}, strict=False)
    m.set_tile_parallel_group(group)
    z = torch.randn(1, 16, 2, 14, 13, generator=torch.Generator().manual_seed(6)).to(bf16)
    with pytest.MonkeyPatch.context() as mp:
        cpu_ops.use_stand_ins(mp)
        return m.decode(z).sample.float()


def _tile_parallel_decode(rank):
    return _real_decode(dist.new_group([0, 1]))


def test_vae_tile_parallel_decode_equals_single_process_tiled_decode():
    res = run_ranks(_tile_parallel_decode, 2, timeout=300)
    single = _real_decode(None)
    assert single.shape == (1, 3, 5, 112, 104)
    assert torch.equal(res[0], res[1]) and torch.equal(res[0], single)


# ---- strip-parallel UNTILED decode (easyanimate_b200/vae_strips.py): halo rows, gathered GroupNorm sums, gathered frames ----
def groupnorm_one_part(x, gamma, beta, groups, eps, silu):
    # the single-process decode through the SAME stand-in arithmetic as the strips (on the GPU both forms end in the same
    # apply kernel; F.group_norm rounds differently from the explicit (x - mean) * rstd form)
    T, H, W, C = x.shape
    return cpu_ops.groupnorm_from_sums(x, cpu_ops.groupnorm_sums(x, groups)[None], float(H * W * (C // groups)), gamma, beta,
                                       groups, eps, silu)


def _strip_decode(group, h=11, w=6):
    from oracle import vae
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    boc = [64, 64, 128, 128]
    ob = vae.init_weights_(vae.OracleAutoencoderKLMagvit(block_out_channels=boc), 33)
    m = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True, mid_block_attention_type="spatial",
                            block_out_channels=boc).to(bf16)
    m.load_state_dict({k: v.to(bf16) for k, v in ob.state_dict().items()}, strict=False)
    m.set_strip_parallel_group(group)
    z = torch.randn(1, 16, 2, h, w, generator=torch.Generator().manual_seed(8)).to(bf16)
    with pytest.MonkeyPatch.context() as mp:
        cpu_ops.use_stand_ins(mp, groupnorm=groupnorm_one_part)
        return m.decode(z).sample.float()


def _strip_parallel_decode(rank, world):
    return _strip_decode(dist.new_group(list(range(world))))


def test_vae_strip_parallel_decode_equals_single_process_untiled_decode():
    """11 latent rows over 2 and over 3 ranks (uneven strips, a middle rank with two neighbours): every rank ends with the whole
    video, identical across ranks, and equal to the single-process untiled decode up to bf16 round-off.  With the torch
    stand-ins every layer at latent resolution (conv_in, mid block with attention, first up block) is bit-identical; from the
    first up-sampled convolution on, PyTorch's CPU conv3d blocks a strip-shaped input differently from the full frame (fp32
    summation order), which flips a few bf16 roundings that a random-init network then spreads - hence a tolerance here.  On
    the GPU the convolution's k order does not depend on the strip (tools/test_multigpu.py checks that decode)."""
    single = _strip_decode(None)
    assert single.shape == (1, 3, 5, 88, 48)
    for world in (2, 3):
        outs = run_ranks(_strip_parallel_decode, world, world, timeout=300)
        for o in outs[1:]:
            assert torch.equal(o, outs[0])
        diff = (outs[0] - single).abs()
        scale = single.abs().max().item()
        assert diff.max().item() <= 0.05 * scale, (world, diff.max().item(), scale)
        assert diff.mean().item() <= 0.004 * scale, (world, diff.mean().item(), scale)

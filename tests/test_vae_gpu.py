"""VAE decode kernels and the AutoencoderKLMagvit drop-in: unit checks against PyTorch references of the same op,
module checks against the oracle (itself pinned to the reference Decoder by tests/golden)."""
import ast
import os

import pytest
import torch
import torch.nn.functional as F
from safetensors import safe_open
from safetensors.torch import load_file

from tests.parity import three_way

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _rand(shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(bf16)


def _ref_causal_conv(x_cl, w, b):
    """x_cl [T,H,W,C] bf16 -> fp32 reference of CausalConv3d (common.py:89-96) -> [T,H,W,Cout]"""
    x = x_cl.permute(3, 0, 1, 2)[None].float()
    x = F.pad(x, (0, 0, 0, 0, 2, 0), mode="replicate")
    y = F.conv3d(x, w.float(), b.float(), padding=(0, 1, 1))
    return y[0].permute(1, 2, 3, 0)


@pytest.mark.parametrize("T,H,W,Cin,Cout", [(1, 8, 16, 64, 64), (3, 10, 20, 64, 128), (2, 9, 7, 128, 256), (4, 16, 32, 256, 128),
                                            (2, 24, 40, 512, 512),
                                            # frames of many 128-pixel tiles, exact and ragged
                                            (5, 128, 160, 64, 128), (5, 122, 150, 64, 128), (3, 90, 160, 128, 256),
                                            # 256- and 128-wide weight tiles over more tiles than SMs (persistent tile loop)
                                            (3, 208, 256, 128, 256), (3, 400, 250, 64, 128)])
def test_conv3d_causal(T, H, W, Cin, Cout):
    from easyanimate_b200 import vae_ops
    x = _rand((T, H, W, Cin), 1.0, 1)
    w = _rand((Cout, Cin, 3, 3, 3), (27 * Cin) ** -0.5, 2)
    b = _rand((Cout,), 0.1, 3)
    out = vae_ops.conv3d_causal(x, vae_ops.pack_conv_weight(w), b, Cout)
    ref = _ref_causal_conv(x, w, b)
    torch.testing.assert_close(out.float(), ref, rtol=2 ** -7, atol=2e-2)
    # fused residual add and temporal duplication
    res = _rand((T, H, W, Cout), 1.0, 4)
    out2 = vae_ops.conv3d_causal(x, vae_ops.pack_conv_weight(w), b, Cout, residual=res)
    torch.testing.assert_close(out2.float(), (ref.to(bf16) + res).float(), rtol=2 ** -6, atol=3e-2)
    if T > 1:
        out3 = vae_ops.conv3d_causal(x, vae_ops.pack_conv_weight(w), b, Cout, dup_frames=True)
        idx = [0] + [i for t in range(1, T) for i in (t, t)]
        assert out3.shape[0] == 2 * T - 1 and torch.equal(out3, out[idx])


@pytest.mark.parametrize("T,H,W,Cin,Cout", [(2, 21, 24, 64, 128), (3, 70, 160, 128, 256), (3, 300, 250, 64, 128)])
@pytest.mark.parametrize("variant", [0, 4])
def test_conv3d_output_row_window_is_the_same_convolution(T, H, W, Cin, Cout, variant, monkeypatch):
    """ea_conv3d_args.out_row0 / out_rows (strip-parallel decode): the rows of a window are bit-identical to the same rows of the
    whole-frame convolution, with residual, frame duplication and the planar store - for both accepted values of the ABI's
    `variant` field (0 and the former tap-per-box bit 4, which now select the same kernel)."""
    from easyanimate_b200 import vae_ops
    monkeypatch.setattr(vae_ops, "CONV_VARIANT", variant)
    x = _rand((T, H, W, Cin), 1.0, 1)
    w = vae_ops.pack_conv_weight(_rand((Cout, Cin, 3, 3, 3), (27 * Cin) ** -0.5, 2))
    b = _rand((Cout,), 0.1, 3)
    res = _rand((T, H, W, Cout), 1.0, 4)
    full = vae_ops.conv3d_causal(x, w, b, Cout, residual=res, dup_frames=T > 1)
    for (r0, r1) in ((0, 7), (5, H - 3), (H - 9, H)):
        lo, hi = max(r0 - 1, 0), min(r1 + 1, H)  # the window plus one halo row where the frame continues
        win = vae_ops.conv3d_causal(x[:, lo:hi].contiguous(), w, b, Cout, residual=res[:, r0:r1].contiguous(), dup_frames=T > 1,
                                    out_row0=r0 - lo, out_rows=r1 - r0)
        if lo == r0 or hi == r1:  # the frame edge: zero padding is what both see
            pass
        assert torch.equal(win, full[:, r0:r1]), (r0, r1)
    w3 = vae_ops.pack_conv_weight(_rand((3, Cin, 3, 3, 3), (27 * Cin) ** -0.5, 5), cout_pad=32)
    b3 = _rand((3,), 0.1, 6)
    fullp = vae_ops.conv3d_causal(x, w3, b3, 3, out_planar=True)
    winp = vae_ops.conv3d_causal(x[:, 4:15].contiguous(), w3, b3, 3, out_planar=True, out_row0=1, out_rows=9)
    assert torch.equal(winp, fullp[:, :, 5:14])


def test_groupnorm_from_gathered_sums_and_attention_query_rows():
    """The strip-parallel forms of GroupNorm and of the mid-block attention: one part == ea_groupnorm_stats bit for bit, and so
    are two parts (rows split 9 + 12): the statistics are accumulated per image row and the rows added in fp64 (exact
    additions), so the split does not matter; query rows [p0, p1) of the attention are the same rows of the full evaluation."""
    from easyanimate_b200 import vae_ops
    T, H, W, Cc, G = 3, 21, 16, 128, 32
    x = _rand((T, H, W, Cc), 2.0, 1) + 0.5
    gamma, beta = _rand((Cc,), 0.1, 2) + 1.0, _rand((Cc,), 0.1, 3)
    ref = vae_ops.groupnorm(x, gamma, beta, G, 1e-6, True)
    count = float(H * W * (Cc // G))
    one = vae_ops.groupnorm_from_sums(x, vae_ops.groupnorm_sums(x, G)[None].contiguous(), count, gamma, beta, G, 1e-6, True)
    assert torch.equal(one, ref)
    a, b = x[:, :9].contiguous(), x[:, 9:].contiguous()
    sums = torch.stack([vae_ops.groupnorm_sums(a, G), vae_ops.groupnorm_sums(b, G)]).contiguous()
    two = torch.cat([vae_ops.groupnorm_from_sums(a, sums, count, gamma, beta, G, 1e-6, True),
                     vae_ops.groupnorm_from_sums(b, sums, count, gamma, beta, G, 1e-6, True)], dim=1)
    assert torch.equal(two, ref)
    # attention query rows
    C2 = 128
    n, res = _rand((T * H * W, C2), 1.0, 4), _rand((T * H * W, C2), 1.0, 5)
    wq, bq = _rand((3 * C2, C2), C2 ** -0.5, 6), _rand((3 * C2,), 0.1, 7)
    wo, bo = _rand((C2, C2), C2 ** -0.5, 8), _rand((C2,), 0.1, 9)
    full = vae_ops.spatial_attention(n, wq, bq, wo, bo, res, T, C2 ** -0.5).view(T, H * W, C2)
    p0, p1 = 5 * W, 17 * W
    part = vae_ops.spatial_attention(n, wq, bq, wo, bo, res.view(T, H * W, C2)[:, p0:p1].reshape(-1, C2).contiguous(), T, C2 ** -0.5,
                                     q_rows=(p0, p1)).view(T, p1 - p0, C2)
    assert torch.equal(part, full[:, p0:p1])


def test_conv3d_planar_rgb_and_padded_input_channels():
    from easyanimate_b200 import vae_ops
    T, H, W = 3, 16, 24
    x = _rand((T, H, W, 128), 1.0, 1)
    w, b = _rand((3, 128, 3, 3, 3), (27 * 128) ** -0.5, 2), _rand((3,), 0.1, 3)
    out = vae_ops.conv3d_causal(x, vae_ops.pack_conv_weight(w, cout_pad=32), b, 3, out_planar=True)
    ref = _ref_causal_conv(x, w, b).permute(3, 0, 1, 2)
    torch.testing.assert_close(out.float(), ref, rtol=2 ** -7, atol=2e-2)
    # conv_in: 16 latent channels zero-padded to 64
    z = _rand((16, T, 6, 10), 1.0, 4)
    pw, pb = _rand((16, 16, 1, 1, 1), 0.25, 5), _rand((16,), 0.1, 6)
    x64 = vae_ops.prepare_latents(z, pw, pb, 64)
    ref_pq = (torch.einsum("oc,cthw->thwo", pw.view(16, 16).float(), z.float()) + pb.float()).to(bf16)
    torch.testing.assert_close(x64[..., :16].float(), ref_pq.float(), rtol=2 ** -7, atol=1e-2)
    assert torch.count_nonzero(x64[..., 16:]) == 0
    w2, b2 = _rand((64, 16, 3, 3, 3), (27 * 16) ** -0.5, 7), _rand((64,), 0.1, 8)
    out2 = vae_ops.conv3d_causal(x64, vae_ops.pack_conv_weight(w2, cin_pad=64), b2, 64)
    torch.testing.assert_close(out2.float(), _ref_causal_conv(x64[..., :16], w2, b2), rtol=2 ** -7, atol=2e-2)


@pytest.mark.parametrize("C,silu", [(128, True), (256, True), (512, False), (64, True)])
def test_groupnorm_per_frame(C, silu):
    from easyanimate_b200 import vae_ops
    T, H, W = 3, 12, 20
    x = _rand((T, H, W, C), 2.0, 1) + 0.5
    g, b = 1 + _rand((C,), 0.1, 2), _rand((C,), 0.1, 3)
    out = vae_ops.groupnorm(x, g, b, 32, 1e-6, silu)
    xr = x.permute(0, 3, 1, 2)  # (t) c h w : one statistic set per frame
    ref = F.group_norm(xr, 32, g, b, 1e-6)
    if silu:
        ref = F.silu(ref)
    torch.testing.assert_close(out.permute(0, 3, 1, 2).float(), ref.float(), rtol=2 ** -7, atol=2e-2)


def test_upsample_softmax_transpose():
    from easyanimate_b200 import vae_ops
    x = _rand((2, 5, 7, 64), 1.0, 1)
    up = vae_ops.upsample2x(x)
    ref = F.interpolate(x.permute(0, 3, 1, 2).float(), scale_factor=2, mode="nearest").permute(0, 2, 3, 1).to(bf16)
    assert torch.equal(up, ref)
    s = torch.randn(50, 60, device="cuda") * 3
    p = vae_ops.softmax_rows(s, 64)
    torch.testing.assert_close(p[:, :60].float(), torch.softmax(s, -1), rtol=2 ** -7, atol=1e-3)
    m = _rand((60, 128), 1.0, 2)
    assert torch.equal(vae_ops.transpose2d(m, 64)[:, :60], m.t())


def _load_case(name):
    path = os.path.join(GOLD, f"{name}.safetensors")
    with safe_open(path, framework="pt") as f:
        meta = f.metadata()
    return load_file(path), meta


GOLDEN_DECODE_CASES = ["vae_small_attn", "vae_small_noattn_ragged", "vae_full_arch"]


def prelude_decode_golden(name):
    """Everything of test_vae_decode_matches_reference_golden that needs no GPU (fixture, oracle pair, product module,
    state-dict load and its key assertions); tests/test_gpu_preludes_cpu.py runs it on the authoring box."""
    from oracle import vae
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    t, meta = _load_case(name)
    boc = list(ast.literal_eval(meta["block_out_channels"]))
    attn = meta["mid_attention"] == "True"
    o32 = vae.init_weights_(vae.OracleAutoencoderKLMagvit(block_out_channels=boc, mid_block_use_attention=attn), 77)
    # decoder weights exactly as in the golden file; post_quant_conv = identity so that golden(z) is comparable
    o32.decoder.load_state_dict(vae.init_weights_(vae.OracleDecoder(block_out_channels=boc, mid_block_use_attention=attn),
                                                  int(meta["seed"])).state_dict())
    with torch.no_grad():
        o32.post_quant_conv.weight.copy_(torch.eye(16).view(16, 16, 1, 1, 1))
        o32.post_quant_conv.bias.zero_()
    ob = vae.OracleAutoencoderKLMagvit(block_out_channels=boc, mid_block_use_attention=attn).to(bf16)
    ob.load_state_dict({k: v.to(bf16) for k, v in o32.state_dict().items()})
    o32.load_state_dict({k: v.float() for k, v in ob.state_dict().items()})
    ours = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True,
                               mid_block_attention_type="spatial", mid_block_use_attention=attn, mini_batch_decoder=1,
                               block_out_channels=boc, scaling_factor=0.7125).to(bf16)
    missing, unexpected = ours.load_state_dict(ob.state_dict(), strict=False)
    # the decode-only oracle has no encoder / quant_conv: those (and only those) keys stay at their init values
    assert not unexpected and all(k.startswith(("quant_conv", "encoder.")) for k in missing), (missing, unexpected)
    return t, o32, ob, ours


@pytest.mark.parametrize("name", GOLDEN_DECODE_CASES)
def test_vae_decode_matches_reference_golden(name):
    """decode() vs the output of the reference's own chunked Decoder (fp32 golden) and vs the oracle run in bf16."""
    t, o32, ob, ours = prelude_decode_golden(name)
    ours = ours.cuda()
    z = t["z"].to(bf16)
    with torch.no_grad():
        truth = o32.decode(z.float())[0]
        ref = ob.decode(z)[0]
        got = ours.decode(z.cuda()).sample
    assert got.shape == t["out"].shape and got.dtype == bf16
    # the golden came from fp32 weights; bf16-rounded weights move it a little, so compare loosely here ...
    assert (truth - t["out"]).abs().max() < 0.15
    # ... and exactly (three-way) against the oracle with identical bf16 weights
    three_way(got, ref, truth, name=name)


def prelude_tiled_oracle():
    from oracle import vae
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    boc = [64, 64, 128, 128]
    kw = dict(block_out_channels=boc, mid_block_use_attention=True, use_tiling=True, tile_sample_min_size=64)
    o32 = vae.init_weights_(vae.OracleAutoencoderKLMagvit(**kw), 21)
    ob = vae.OracleAutoencoderKLMagvit(**kw).to(bf16)
    ob.load_state_dict({k: v.to(bf16) for k, v in o32.state_dict().items()})
    o32.load_state_dict({k: v.float() for k, v in ob.state_dict().items()})
    ours = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True,
                               mid_block_attention_type="spatial", block_out_channels=boc, use_tiling=True,
                               tile_sample_min_size=64).to(bf16)
    missing, unexpected = ours.load_state_dict(ob.state_dict(), strict=False)
    assert not unexpected and all(k.startswith(("quant_conv", "encoder.")) for k in missing), (missing, unexpected)
    return o32, ob, ours


def test_vae_tiled_decode_matches_oracle():
    o32, ob, ours = prelude_tiled_oracle()
    ours = ours.cuda()
    z = torch.randn(1, 16, 2, 12, 20, generator=torch.Generator().manual_seed(3)).to(bf16)
    with torch.no_grad():
        truth = o32.decode(z.float())[0]
        ref = ob.decode(z)[0]
        got = ours.decode(z.cuda(), return_dict=False)[0]
        again = ours.decode(z.cuda(), return_dict=False)[0]
    assert got.shape == (1, 3, 5, 96, 160)
    three_way(got, ref, truth, name="vae_tiled")
    # no atomics anywhere in the decode: a second run must reproduce the first bit for bit (the tile-parallel path,
    # tools/test_multigpu.py, compares ranks' tiles against a single-GPU decode with torch.equal)
    assert torch.equal(got, again)


def prelude_tiled_reference_golden():
    from oracle import vae
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    path = os.path.join(GOLD, "vae_ref_tiled.safetensors")
    t = {**load_file(path), **load_file(os.path.join(GOLD, "vae_ref_tiled_2.safetensors"))}  # files are kept under 1 MB
    with safe_open(path, framework="pt") as f:
        meta = f.metadata()
    boc = list(ast.literal_eval(meta["block_out_channels"]))
    kw = dict(block_out_channels=boc, use_tiling=True, tile_sample_min_size=int(meta["tile_sample_min_size"]))
    o32 = vae.init_weights_(vae.OracleAutoencoderKLMagvit(**kw), int(meta["seed"]))
    ob = vae.OracleAutoencoderKLMagvit(**kw).to(bf16)
    ob.load_state_dict({k: v.to(bf16) for k, v in o32.state_dict().items()})
    ours = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True, mid_block_attention_type="spatial",
                               **kw).to(bf16)
    missing, unexpected = ours.load_state_dict(ob.state_dict(), strict=False)
    assert not unexpected and all(k.startswith(("quant_conv", "encoder.")) for k in missing), (missing, unexpected)
    return t, ob, ours


def test_vae_tiled_decode_matches_reference_golden():
    """Against the output of the REFERENCE's own AutoencoderKLMagvit.tiled_decode (fp32; tests/golden/make_golden.py::
    make_vae_tiled): 3 x 3 ragged tiles + the lower-right corner pass."""
    t, ob, ours = prelude_tiled_reference_golden()
    ours = ours.cuda()
    with torch.no_grad():
        ref = ob.decode(t["z"].to(bf16))[0]
        got = ours.decode(t["z"].to(bf16).cuda(), return_dict=False)[0]
    assert got.shape == t["out_tiled"].shape
    three_way(got, ref, t["out_tiled"], name="vae_tiled_vs_reference_fixture")

"""AutoencoderKLMagvit.encode on the GPU (I2V / inpaint conditioning prep).

encode() runs the encoder's stride-2 convolutions as the strided implicit-GEMM kernel (ea_conv3d_causal with stride fields)
or, for A/B, as the stride-1 kernel plus a strided pick; both are compared here with fp32 PyTorch references and with the
moments the REFERENCE's own AutoencoderKLMagvit.encode / tiled_encode produced (tests/golden/vae_ref_encode.safetensors)."""
import ast
import os

import pytest
import torch

from tests.parity import three_way

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


def test_strided_convolution_as_stride1_plus_pick():
    """The encoder's downsampling convolutions: stride (2,2,2) / (1,2,2), right/bottom zero pad, causal replicate pad."""
    import torch.nn.functional as F
    from easyanimate_b200 import vae_ops
    g = torch.Generator(device="cuda").manual_seed(1)
    T, H, W, C = 5, 18, 22, 64
    x = torch.randn((T, H, W, C), device="cuda", generator=g).to(bf16)
    w = (torch.randn((C, C, 3, 3, 3), device="cuda", generator=g) * (27 * C) ** -0.5).to(bf16)
    b = (torch.randn((C,), device="cuda", generator=g) * 0.1).to(bf16)
    y = vae_ops.conv3d_causal(x, vae_ops.pack_conv_weight(w), b, C)
    xin = x.float().permute(3, 0, 1, 2)[None]
    xin = F.pad(F.pad(xin, (0, 1, 0, 1)), (0, 0, 0, 0, 2, 0), mode="replicate")
    for st in (1, 2):
        ref = F.conv3d(xin, w.float(), b.float(), stride=(st, 2, 2))[0].permute(1, 2, 3, 0)
        got = (y[::2] if st == 2 else y)[:, 1::2, 1::2]
        assert got.shape == ref.shape
        torch.testing.assert_close(got.float(), ref, rtol=2 ** -7, atol=2e-2)


@pytest.mark.parametrize("T,H,W,Cin,Cout,st", [(5, 18, 22, 64, 64, 2), (5, 18, 22, 64, 64, 1), (9, 33, 47, 128, 128, 2), (1, 16, 16, 64, 128, 1),
                                              # frames of many 128-pixel tiles
                                              (5, 256, 320, 128, 128, 2), (3, 416, 512, 128, 256, 1)])
def test_strided_convolution_kernel(T, H, W, Cin, Cout, st, monkeypatch):
    """ea_conv3d_causal with stride (st, 2, 2) (TMA element strides) against F.conv3d on the reference's padding recipe
    (downsamplers.py:24-96), and bit for bit against the stride-1 form of the same kernel + strided pick (with the ABI's
    former tap-per-box variant bit set, which selects the same kernel)."""
    import torch.nn.functional as F
    from easyanimate_b200 import vae_ops
    g = torch.Generator(device="cuda").manual_seed(T * H + W)
    x = torch.randn((T, H, W, Cin), device="cuda", generator=g).to(bf16)
    w = (torch.randn((Cout, Cin, 3, 3, 3), device="cuda", generator=g) * (27 * Cin) ** -0.5).to(bf16)
    b = (torch.randn((Cout,), device="cuda", generator=g) * 0.1).to(bf16)
    wp = vae_ops.pack_conv_weight(w)
    got = vae_ops.conv3d_causal(x, wp, b, Cout, stride_t=st, stride_hw=2)
    xin = x.float().permute(3, 0, 1, 2)[None]
    xin = F.pad(F.pad(xin, (0, 1, 0, 1)), (0, 0, 0, 0, 2, 0), mode="replicate")
    ref = F.conv3d(xin, w.float(), b.float(), stride=(st, 2, 2))[0].permute(1, 2, 3, 0)
    assert got.shape == ref.shape == ((T + 1) // 2 if st == 2 else T, H // 2, W // 2, Cout)
    torch.testing.assert_close(got.float(), ref, rtol=2 ** -7, atol=2e-2)
    monkeypatch.setattr(vae_ops, "CONV_VARIANT", vae_ops.CONV_VARIANT | 4)
    full = vae_ops.conv3d_causal(x, wp, b, Cout)
    pick = (full[::2] if st == 2 else full)[:, 1::2, 1::2]
    assert torch.equal(got, pick[:, :H // 2, :W // 2])  # same taps, same k order, same accumulator: identical


def prelude_encode_golden():
    """The part of test_vae_encode_matches_reference_golden that needs no GPU (run on CPU by tests/test_gpu_preludes_cpu.py)."""
    from safetensors import safe_open
    from safetensors.torch import load_file
    from oracle import vae
    from easyanimate_b200.autoencoder_magvit import AutoencoderKLMagvit
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vae_ref_encode.safetensors")
    t = load_file(path)
    with safe_open(path, framework="pt") as f:
        meta = f.metadata()
    boc = list(ast.literal_eval(meta["block_out_channels"]))
    o32 = vae.init_weights_(vae.OracleAutoencoderKLMagvit(block_out_channels=boc, with_encoder=True), int(meta["seed"]))
    ob = vae.OracleAutoencoderKLMagvit(block_out_channels=boc, with_encoder=True).to(bf16)
    ob.load_state_dict({k: v.to(bf16) for k, v in o32.state_dict().items()})
    ours = AutoencoderKLMagvit(latent_channels=16, cache_mag_vae=True, spatial_group_norm=True, mid_block_attention_type="spatial",
                               block_out_channels=boc).to(bf16)
    ours.load_state_dict(ob.state_dict(), strict=True)
    return t, ob, ours


def test_vae_encode_matches_reference_golden():
    """Against the moments produced by the REFERENCE's AutoencoderKLMagvit.encode / tiled_encode (fp32, CPU)."""
    t, ob, ours = prelude_encode_golden()
    ours = ours.cuda()
    x = t["x"].to(bf16)
    with torch.no_grad():
        ref = ob.encode_moments(x)
        post = ours.encode(x.cuda()).latent_dist
    assert post.parameters.shape == t["moments"].shape and post.mode().shape[1] == 16
    three_way(post.parameters, ref, t["moments"], name="vae_encode_vs_reference_fixture")
    # tiled_encode with 32-pixel tiles
    for m in (ob, ours):
        m.use_tiling, m.tile_sample_min_size, m.tile_latent_min_size = True, 32, 4
    with torch.no_grad():
        ref_t = ob.encode_moments(x)
        got_t = ours.encode(x.cuda(), return_dict=False)[0].parameters
    three_way(got_t, ref_t, t["moments_tiled32"], name="vae_tiled_encode_vs_reference_fixture")
    # run-to-run reproducible
    with torch.no_grad():
        assert torch.equal(ours.encode(x.cuda())[0].parameters, got_t)

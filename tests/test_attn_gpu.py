"""wgmma attention kernel against an fp32 PyTorch reference of softmax(QK^T/sqrt(64))V (GPU only)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

# The variant codes of include/ea_b200.h `ea_attn_args.variant`: every sixth-generation code (0x1?c, 0x2?c, 0x9?c) runs the one
# sm_90a kernel and must give the same softmax; codes of generations that are not built in are skipped
def _variants(all_of):
    from easyanimate_b200 import _lib
    gens = _lib.ea_attn_generations()

    def built(v):
        if (v & 0x1100) == 0x100:
            return True
        return bool(gens & ((1 << 9) if v & 0x1000 else (1 << 4) if (v & 12) == 12 else (1 << 1)))
    return [v for v in all_of if built(v)]


VARIANTS = _variants([0x10C, 0x11C, 0x12C, 0x15C, 0x16C, 0x90C, 0x210C, 0x211C, 0x214C, 0x217C, 0x290C, 0x294C, 0x100C, 0x101C, 0x102C, 0x104C, 0x1C, 0x0C, 0x3C, 0x1, 0x0, 0x3])
SHAPES = [(1, 2, 128, 0), (1, 2, 256, 64), (2, 3, 1000, 77), (1, 4, 4176, 256), (1, 1, 8, 3), (2, 2, 300, 300)]


def _ref(q, k, v):
    B, H, S, _ = q.shape
    return torch.nn.functional.scaled_dot_product_attention(q.float(), k.float(), v.float()).transpose(1, 2).reshape(B, S, H * 64)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("B,H,S,St", SHAPES)
def test_attention_matches_fp32_reference(variant, B, H, S, St):
    from easyanimate_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(S + variant)
    q, k, v = [torch.randn(B, H, S, 64, device="cuda", generator=g).to(bf16) for _ in range(3)]
    ot, ov = ops.attention(q, k, v, St, variant=variant)
    assert ot.shape == (B, St, H * 64) and ov.shape == (B, S - St, H * 64)
    got = torch.cat([ot, ov], 1).float()
    ref = _ref(q, k, v)
    # bf16 P and bf16 output: a few 1e-3 absolute on outputs of O(0.1-1)
    torch.testing.assert_close(got, ref, rtol=2e-2, atol=4e-3)


def test_attention_large_logits_and_running_max_rescale():
    """Scores that keep growing along the key axis force the lazy running-max rescale path of every kernel."""
    from easyanimate_b200 import ops
    B, H, S = 1, 2, 1024
    g = torch.Generator(device="cuda").manual_seed(7)
    q = torch.randn(B, H, S, 64, device="cuda", generator=g)
    k = torch.randn(B, H, S, 64, device="cuda", generator=g)
    ramp = torch.linspace(0, 6, S, device="cuda").view(1, 1, S, 1)
    k = k + ramp * q.mean(dim=2, keepdim=True).sign()  # later keys align more and more with the queries
    q, k = (q * 3).to(bf16), k.to(bf16)
    v = torch.randn(B, H, S, 64, device="cuda", generator=g).to(bf16)
    ref = _ref(q, k, v)
    for variant in VARIANTS:
        ot, ov = ops.attention(q, k, v, 0, variant=variant)
        assert torch.isfinite(ov).all()
        torch.testing.assert_close(ov.float(), ref, rtol=3e-2, atol=2e-2)


@pytest.mark.parametrize("variant", _variants([0x10C, 0x11C, 0x13C, 0x15C, 0x90C, 0x210C, 0x211C, 0x214C, 0x217C, 0x100C, 0x101C, 0x102C, 0x1C]))
@pytest.mark.parametrize("col,mag", [(640, 150.0), (643, 150.0), (640, 1500.0), (643, 1500.0), (130, 40.0), (1023, 800.0), (740, 1500.0), (700, 150.0)])
def test_attention_outlier_key_beyond_the_kept_reference(variant, col, mag):
    """One key whose score exceeds everything before it by far more than 2^30, at several columns of a 128-key block and in
    a ragged last block: the online softmax must rescale O and the row sum by the new running maximum; rows anti-aligned with
    the key see a hugely negative score instead."""
    from easyanimate_b200 import ops
    B, H, S = 1, 2, 1100
    g = torch.Generator(device="cuda").manual_seed(11)
    u = torch.nn.functional.normalize(torch.randn(64, device="cuda", generator=g), dim=0)
    q = torch.randn(B, H, S, 64, device="cuda", generator=g) + 3.0 * u
    k = torch.randn(B, H, S, 64, device="cuda", generator=g)
    k[:, :, col] = mag * u
    v = torch.randn(B, H, S, 64, device="cuda", generator=g)
    q, k, v = q.to(bf16), k.to(bf16), v.to(bf16)
    ref = _ref(q, k, v)
    ot, ov = ops.attention(q, k, v, 0, variant=variant)
    assert torch.isfinite(ov).all()
    torch.testing.assert_close(ov.float(), ref, rtol=3e-2, atol=2e-2)

"""The joint attention kernel (attn_tc6.cu) against an emulation of its own block-wise softmax (tests/attn_emulation.py),
element by element: every output within ulp_bf16 + 2^-8 sum p|v| of the emulation and at least 99 % of them bit-equal
(attn_emulation.accept).  The shapes put S and S_text on either side of the 64-row warpgroup split and of the 128-key block
and query tile, wrap the 3-stage K/V ring several times and reach the production lengths and head count (GPU only).

The bit-equal fraction falls where more P roundings can flip: the kernel's fp32 scores (wgmma's summation order) and
ex2.approx differ from the emulation's in the last bits, so an exponential next to a bf16 midpoint may round the other way.
Rows of more keys hold more such P, and large scores carry larger absolute score errors.  Where that pulls the fraction
under 99 %, the floor is the fraction measured on an H100 SXM (700 W), less a margin; see each case."""
import ctypes as C

import pytest
import torch

from tests.attn_emulation import accept, anti_aligned_inputs, attention_inputs, emulate_attention, ulp_bf16

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
FLAT, PEAKED = 1.0, 3.0  # std of the scaled scores q.k / 8
SENTINEL = -1024.0


def _check(q, k, v, S_text, scale=None, min_equal=0.99):
    from easyanimate_b200 import ops
    B, H, S, _ = q.shape
    got = ops.attention(q, k, v, S_text, scale=scale)
    assert got[0].shape == (B, S_text, H * 64) and got[1].shape == (B, S - S_text, H * 64)
    r = accept(got, emulate_attention(q, k, v, S_text, scale=scale), q, k, v, scale=scale, min_equal=min_equal)
    print(f"attention B={B} H={H} S={S} S_text={S_text}: bit-equal {r.equal_fraction:.5f}, bound ratio {r.bound_ratio:.3f}")
    assert r.ok, r


@pytest.mark.parametrize("std", [FLAT, PEAKED])
@pytest.mark.parametrize("S", [1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 383, 384, 385, 640, 1000])
def test_sequence_length_sweep(S, std):
    """S around multiples of 64 (the two consumer warpgroups' rows) and 128 (key block, query tile); S = 640 and 1000
    run 5 and 8 key blocks through the 3-stage ring."""
    _check(*attention_inputs(1, 2, S, std, seed=S, device="cuda"), 0)


@pytest.mark.parametrize("std", [FLAT, PEAKED])
@pytest.mark.parametrize("S_text", [0, 1, 63, 64, 65, 127, 128, 129, 256, 999, 1000])
def test_text_length_sweep(S_text, std):
    """The text / video split of the stored rows, at and around the tile boundaries, and all-text / all-video."""
    _check(*attention_inputs(2, 2, 1000, std, seed=S_text, device="cuda"), S_text)


# (B, H, S, S_text, min bit-equal fraction).  1280: one block of bench.py's CPU sample with CFG (1024 video + 256 text
# tokens, 48 heads); 13 568: 512p, 49 frames; 47 056: 720p, 49 frames, a last key block of 80 keys.  Measured on an H100
# (flat / peaked): 0.9973 / 0.9986 at 1280, 0.9858 / 0.9919 at 13 568, 0.9703 / 0.9781 at 47 056.  The floor at 47 056 is
# 0.97, the least this test accepts at any length, and is only 0.0003 under the flat measurement.
PRODUCTION = [(2, 48, 1280, 256, 0.99), (1, 2, 13568, 256, 0.98), (1, 2, 47056, 256, 0.97)]


@pytest.mark.parametrize("std", [FLAT, PEAKED])
@pytest.mark.parametrize("B,H,S,S_text,min_equal", PRODUCTION, ids=[f"S{s[2]}" for s in PRODUCTION])
def test_production_shapes(B, H, S, S_text, min_equal, std):
    _check(*attention_inputs(B, H, S, std, seed=S, device="cuda"), S_text, min_equal=min_equal)


@pytest.mark.parametrize("S,S_text,min_equal", [(129, 0, 0.99), (1000, 0, 0.97), (47056, 256, 0.93)])
def test_ragged_last_block_mask_on_anti_aligned_scores(S, S_text, min_equal):
    """Every valid scaled score is about -24: a zero-filled key of the ragged last block that escaped the mask would
    score 0 and take almost all of each row's weight, so no element stays bit-equal (tests/test_attn_emulation_cpu.py);
    at S = 47 056 this, not the floor of test_production_shapes, is what guards the mask.  Raw scores near -192 carry
    fp32 errors of 2^-16 and more, so more P roundings flip than on random inputs: measured on an H100, 0.9927, 0.9808
    and 0.9448 of the elements are bit-equal."""
    _check(*anti_aligned_inputs(1, 2, S, seed=S, device="cuda"), S_text, min_equal=min_equal)


def test_zero_queries_give_the_mean_of_v():
    """q = 0: every score is 0 and every P exactly 1, so each output is the column mean of V up to one bf16 ulp."""
    from easyanimate_b200 import ops
    B, H, S, S_text = 2, 3, 1000, 77
    _, k, v = attention_inputs(B, H, S, seed=5, device="cuda")
    q = torch.zeros_like(k)
    got = torch.cat(ops.attention(q, k, v, S_text), 1).view(B, S, H, 64).double()
    mean = v.double().mean(2)[:, None]  # [B, 1, H, 64]
    assert ((got - mean).abs() <= ulp_bf16(mean)).all()


def test_non_default_scale():
    _check(*attention_inputs(2, 3, 1000, FLAT, seed=9, device="cuda"), 77, scale=0.2)


def test_no_stores_outside_the_outputs():
    """The last query tile covers rows 128..255 of S = 200; rows from S on exist only as TMA's zero fill and must not be
    stored: not into the guard rows around the outputs, and not into batch 1's rows (batch 0's padding rows would land
    there).  The outputs are carved out of sentinel-filled buffers with 128 guard rows on either side."""
    from easyanimate_b200 import _lib as L
    from easyanimate_b200 import ops
    B, H, S, S_text, G = 2, 3, 200, 77, 128
    q, k, v = attention_inputs(B, H, S, FLAT, seed=11, device="cuda")
    bufs = [torch.full((2 * G + B * n, H * 64), SENTINEL, device="cuda", dtype=bf16) for n in (S_text, S - S_text)]
    out_text, out_video = (b[G:-G].view(B, -1, H * 64) for b in bufs)
    args = L.AttnArgs(q=q.data_ptr(), k=k.data_ptr(), v=v.data_ptr(), out_text=out_text.data_ptr(),
                      out_video=out_video.data_ptr(), B=B, H=H, S=S, S_text=S_text, S_pad=0, head_dim=64, scale=0.125,
                      variant=ops.ATTN_VARIANT, peers=None)
    L.check(L.ea_attn_fwd(C.byref(args), torch.cuda.current_stream().cuda_stream), "ea_attn_fwd")
    torch.cuda.synchronize()
    for b in bufs:
        assert (b[:G] == SENTINEL).all() and (b[-G:] == SENTINEL).all()
    ref_text, ref_video = ops.attention(q, k, v, S_text)
    assert torch.equal(out_text, ref_text) and torch.equal(out_video, ref_video)
    # a padding row of batch 0 has q = 0: the column mean of batch 0's V, per head
    pad_row = v[0].double().mean(1)  # [H, 64]
    near = (out_video[1].view(-1, H, 64).double() - pad_row).abs() <= ulp_bf16(pad_row)
    assert not near.all(-1).any()
    r = accept((out_text, out_video), emulate_attention(q, k, v, S_text), q, k, v)
    assert r.ok, r


def test_deterministic():
    from easyanimate_b200 import ops
    q, k, v = attention_inputs(2, 48, 1280, FLAT, seed=13, device="cuda")
    a, b = ops.attention(q, k, v, 256), ops.attention(q, k, v, 256)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])

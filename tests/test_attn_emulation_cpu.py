"""The emulation of the joint attention kernel (tests/attn_emulation.py) and its acceptance rule, checked without a GPU:
the emulation is the fp64 softmax up to its roundings, a kernel that differs only by ex2.approx and the order of its sums
is accepted, and each of the known ways to get the kernel wrong is rejected."""
import pytest
import torch

from tests.attn_emulation import (accept, anti_aligned_inputs, attention_inputs, emulate_attention, round_bf16, scale_log2,
                                  sdpa_fp64, ulp_bf16, weighted_abs_v)

MUTANTS = ["unmask_pad", "mask_off_by_one", "truncate_p", "no_rescale_l"]
NOISE = 2.0 ** -21  # relative error of ex2.approx and of the wgmma / shuffle summation order


def _emu(q, k, v, S_text=0, **kw):
    return torch.cat(emulate_attention(q, k, v, S_text, **kw), 1)


def test_helpers():
    assert scale_log2(0.125) == float(torch.tensor(0.125 * 1.4426950408889634, dtype=torch.float32))
    x = torch.tensor([1.0 + 2.0 ** -8 + 2.0 ** -30, 1.0 + 2.0 ** -8 - 2.0 ** -30, 1.0 + 2.0 ** -8, -3.0], dtype=torch.float64)
    # the first two lie 2^-30 off a bf16 midpoint: fp32 rounds them onto it, bf16 must still round away from it
    assert round_bf16(x).tolist() == [1.0 + 2.0 ** -7, 1.0, 1.0, -3.0]
    assert x.to(torch.bfloat16).tolist()[0] == 1.0  # what rounding twice gives
    assert ulp_bf16(torch.tensor([1.0, 1.99, -0.5, 0.0])).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -8, 2.0 ** -133]


@pytest.mark.parametrize("kt", [64, 128])
@pytest.mark.parametrize("S", [1, 129, 300, 1000])
@pytest.mark.parametrize("std", [1.0, 3.0])
def test_emulation_without_rounding_is_the_fp64_softmax(S, std, kt):
    """The block-wise algorithm itself (running maximum, rescale, mask of the ragged last block) is exact."""
    q, k, v = attention_inputs(2, 2, S, std, seed=S)
    got = _emu(q, k, v, min(S, 77), kt=kt, rounding=False)
    assert got.dtype == torch.float64
    assert (got - sdpa_fp64(q, k, v)).abs().max() <= 1e-12


@pytest.mark.parametrize("kt", [64, 128])
@pytest.mark.parametrize("S", [129, 300, 1000])
@pytest.mark.parametrize("std", [1.0, 3.0])
def test_emulation_with_rounding_stays_within_one_p_rounding_of_the_fp64_softmax(S, std, kt):
    """|emu - sdpa| <= ulp/2 + c sum p|v|, whatever the block size: the output rounding, and the P roundings, each off
    by at most 2^-8 relative (bf16 keeps 8 significant bits) while the row sum takes the unrounded exponentials, so
    c = 2^-8 holds always.  On a flat softmax the roundings of many keys average out and c = 2^-9 holds; on a peaked one
    a few keys carry the row and it does not (ratios to the 2^-9 bound reach 1.1)."""
    q, k, v = attention_inputs(2, 2, S, std, seed=S + 7)
    emu = _emu(q, k, v, 77, kt=kt)
    assert emu.dtype == torch.bfloat16
    err = (emu.double() - sdpa_fp64(q, k, v)).abs()
    half_ulp, wv = ulp_bf16(emu) / 2, weighted_abs_v(q, k, v)
    assert (err <= half_ulp + 2.0 ** -8 * wv).all()
    if std == 1.0:
        assert (err <= half_ulp + 2.0 ** -9 * wv).all()


def test_emulation_honours_scale():
    q, k, v = attention_inputs(1, 2, 300, 1.0, seed=3)
    assert (_emu(q, k, v, scale=0.2, rounding=False) - sdpa_fp64(q, k, v, scale=0.2)).abs().max() <= 1e-12
    assert accept(_emu(q, k, v, scale=0.2), _emu(q, k, v, scale=0.2), q, k, v, scale=0.2).ok
    assert not accept(_emu(q, k, v), _emu(q, k, v, scale=0.2), q, k, v, scale=0.2).ok


@pytest.mark.parametrize("S", [129, 300, 1000, 1100])
@pytest.mark.parametrize("std", [1.0, 3.0])
def test_accept_passes_the_emulation_with_noise(S, std):
    q, k, v = attention_inputs(1, 2, S, std, seed=S)
    emu = _emu(q, k, v)
    noisy = _emu(q, k, v, noise=NOISE, generator=torch.Generator().manual_seed(S))
    r = accept(noisy, emu, q, k, v)
    assert r.ok and r.equal_fraction < 1.0, r  # the noise does flip roundings, and the rule allows for it


def test_accept_passes_the_emulation_with_noise_on_anti_aligned_scores():
    q, k, v = anti_aligned_inputs(1, 2, 1000, seed=1)
    noisy = _emu(q, k, v, noise=NOISE, generator=torch.Generator().manual_seed(1))
    r = accept(noisy, _emu(q, k, v), q, k, v)
    assert r.ok, r


@pytest.mark.parametrize("mutant", MUTANTS)
@pytest.mark.parametrize("S", [300, 1000, 1100])
def test_accept_rejects_each_mutant_on_flat_scores(S, mutant):
    q, k, v = attention_inputs(1, 2, S, 1.0, seed=S)
    r = accept(_emu(q, k, v, **{mutant: True}), _emu(q, k, v), q, k, v)
    assert not r.ok, r


@pytest.mark.parametrize("mutant", MUTANTS)
def test_accept_rejects_each_mutant_on_anti_aligned_scores(mutant):
    q, k, v = anti_aligned_inputs(1, 2, 1000, seed=1)
    r = accept(_emu(q, k, v, **{mutant: True}), _emu(q, k, v), q, k, v)
    assert not r.ok, r


@pytest.mark.parametrize("mutant", ["unmask_pad", "mask_off_by_one"])
@pytest.mark.parametrize("S", [129, 1000])
def test_one_escaped_key_breaks_bound_a_on_anti_aligned_scores(S, mutant):
    """A zero-filled key that escapes the mask scores 0 against valid scores of about -24: it takes almost all of every
    row's weight, so not one element is bit-equal and the per-element bound alone rejects it by far."""
    q, k, v = anti_aligned_inputs(1, 2, S, seed=1)
    r = accept(_emu(q, k, v, **{mutant: True}), _emu(q, k, v), q, k, v)
    assert r.equal_fraction < 0.01 and r.bound_ratio > 10, r

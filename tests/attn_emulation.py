"""The joint attention kernel's algorithm in torch, and the rule that decides whether a kernel output matches it.

`emulate_attention` follows attn6_kernel (easyanimate_b200/csrc/attn_tc6.cu:83-237) step by step: keys in blocks of
kt = kKT = 128 (attn_tc6.cu:18), the last block's missing keys zero-filled by TMA and masked to -inf (attn_tc6.cu:168-175),
a running maximum per query row (attn_tc6.cu:176-197), P = bf16(2^(s * scale_log2 - m)) (attn_tc6.cu:198-208) and
out = bf16(O / l) (attn_tc6.cu:222-236).  The fp32 and bf16 roundings of the kernel are reproduced; every sum is taken in
fp64 and rounded once.  What the emulation cannot know (the order in which wgmma accumulates, the error of ex2.approx) is
what `accept` allows for.

Switches model the known ways to get the kernel wrong, so the tests can show that `accept` sees each of them."""
from __future__ import annotations

from typing import NamedTuple, Optional

import torch

f32, f64, bf16 = torch.float32, torch.float64, torch.bfloat16
LOG2E = 1.4426950408889634  # attn_tc6.cu launch(): scale_log2 = scale * 1.4426950408889634f, an fp32 product
KT = 128  # attn_tc6.cu:18 kKT: keys per block (and query rows per CTA tile)
_BUDGET = 1 << 24  # elements of one [B, H, rows, keys] fp64 temporary (128 MB): S = 47 056 fits on one GPU


def scale_log2(scale: float) -> float:
    """fp32(fp32(scale) * fp32(log2 e)), as launch() computes it."""
    return float(torch.tensor(scale, dtype=f32) * torch.tensor(LOG2E, dtype=f32))


def round_bf16(x: torch.Tensor) -> torch.Tensor:
    """fp64 -> bf16, rounded once to nearest even.  x.to(bf16) goes through fp32 and can round twice: an fp32 value that
    lands on a bf16 midpoint without being exact is stepped one fp32 ulp towards x first, so the tie breaks as x says."""
    f = x.float()
    tie = ((f.view(torch.int32) & 0xFFFF) == 0x8000) & (f.double() != x)
    toward = torch.where(x > f.double(), torch.full_like(f, float("inf")), torch.full_like(f, -float("inf")))
    return torch.where(tie, torch.nextafter(f, toward), f).to(bf16)


def emulate_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, S_text: int, scale: Optional[float] = None,
                      kt: int = KT, *, rounding: bool = True, unmask_pad: bool = False, mask_off_by_one: bool = False,
                      truncate_p: bool = False, no_rescale_l: bool = False, noise: float = 0.0,
                      generator: Optional[torch.Generator] = None):
    """softmax(q k^T * scale) v as attn6_kernel computes it, for q, k, v [B, H, S, 64] on any device.  Returns
    (out_text [B, S_text, H*64], out_video [B, S - S_text, H*64]) in bf16, the layout of ops.attention.

    rounding=False keeps every intermediate in fp64 and returns fp64: the block-wise algorithm alone.
    noise: relative noise, uniform in [-noise, noise], on every exponential and on every row sum (ex2.approx, and the
    order of the wgmma and shuffle sums).
    Mutants: unmask_pad - the zero-filled keys of the last block take part with score 0; mask_off_by_one - `> valid`
    for `>= valid`, so the first zero-filled key takes part; truncate_p - P rounded toward zero; no_rescale_l - the row
    sum is never multiplied by the rescale factor `f` when the running maximum grows."""
    B, H, S, D = q.shape
    dev = q.device
    scale = D ** -0.5 if scale is None else scale
    sl2 = scale_log2(scale) if rounding else scale * LOG2E
    nblk = -(-S // kt)
    Sp = nblk * kt
    kd = k.double().transpose(-1, -2)
    vd = torch.zeros(B, H, Sp, D, dtype=f64, device=dev)
    vd[:, :, :S] = v.double()  # TMA zero-fills V past S as well
    pad = torch.full((Sp - S,), -float("inf"), dtype=f64, device=dev)
    if unmask_pad:
        pad[:] = 0.0  # a zero-filled key scores q . 0 = 0
    elif mask_off_by_one and Sp > S:
        pad[0] = 0.0

    def jitter(x):
        return x * (1 + noise * (2 * torch.rand(x.shape, dtype=f64, device=dev, generator=generator) - 1)) if noise else x

    out = torch.empty(B, H, S, D, dtype=f64, device=dev)
    rows = max(1, _BUDGET // (B * H * Sp))
    for r0 in range(0, S, rows):
        s = q[:, :, r0:r0 + rows].double() @ kd
        if rounding:
            s = s.float().double()  # the fp32 score of wgmma, here the fp64 dot product rounded once
        c = s.shape[2]
        blk = torch.cat([s, pad.expand(B, H, c, -1)], -1).view(B, H, c, nblk, kt)
        mx = blk.amax(-1) * sl2  # exact in fp64: 24-bit x 24-bit significands
        if rounding:
            mx = mx.float().double()
        m = torch.cummax(mx, -1).values  # the running maximum after each block
        x = blk * sl2 - m[..., None]  # fmaf(s, sl2, -m): one rounding to fp32
        if rounding:
            x = x.float().double()
        e = jitter(torch.exp2(x))
        if rounding:
            e32 = e.float()
            e32 = torch.where(e32 < 2.0 ** -126, torch.zeros_like(e32), e32)  # ex2.approx.ftz flushes denormal results
            if truncate_p:
                p = (e32.view(torch.int32) & ~0xFFFF).view(f32).double()
            else:
                p = e32.to(bf16).double()
            e = e32.double()
        else:
            p = e
        f = torch.exp2(m - m[..., -1:])  # block j's share rescaled into the final maximum
        lb = e.sum(-1)
        l = jitter(lb.sum(-1) if no_rescale_l else (lb * f).sum(-1))
        o = (p * f[..., None]).reshape(B, H, c, Sp) @ vd
        out[:, :, r0:r0 + c] = o / l[..., None]
    out = out.transpose(1, 2).reshape(B, S, H * D)
    if rounding:
        out = round_bf16(out)
    return out[:, :S_text], out[:, S_text:]


def sdpa_fp64(q, k, v, scale=None):
    """softmax(q k^T * scale) v in fp64, [B, S, H*64]."""
    B, H, S, D = q.shape
    scale = D ** -0.5 if scale is None else scale
    p = torch.softmax((q.double() @ k.double().transpose(-1, -2)) * scale, -1)
    return (p @ v.double()).transpose(1, 2).reshape(B, S, H * D)


def weighted_abs_v(q, k, v, scale=None):
    """sum_j p_j |v_j| with p the fp64 softmax, [B, S, H*64]: the scale of what one rounding of every P can move."""
    B, H, S, D = q.shape
    scale = D ** -0.5 if scale is None else scale
    kd, va = k.double().transpose(-1, -2), v.double().abs()
    out = torch.empty(B, H, S, D, dtype=f64, device=q.device)
    rows = max(1, _BUDGET // (B * H * S))
    for r0 in range(0, S, rows):
        p = torch.softmax((q[:, :, r0:r0 + rows].double() @ kd) * scale, -1)
        out[:, :, r0:r0 + rows] = p @ va
    return out.transpose(1, 2).reshape(B, S, H * D)


def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """The spacing of bf16 at |x| (at 0: the smallest normal's), in fp64."""
    a = x.double().abs().clamp_min(2.0 ** -126)
    return torch.ldexp(torch.ones_like(a), torch.frexp(a).exponent - 8)


class Acceptance(NamedTuple):
    equal_fraction: float  # elements bit-equal to the emulation
    bound_ratio: float  # max |got - emu| / (ulp_bf16(emu) + 2^-8 sum_j p_j |v_j|)
    min_equal: float

    @property
    def ok(self) -> bool:
        return self.bound_ratio <= 1.0 and self.equal_fraction >= self.min_equal


def _joined(x):
    return torch.cat(x, 1) if isinstance(x, tuple) else x


def accept(got, emu, q, k, v, scale=None, min_equal: float = 0.99) -> Acceptance:
    """Does a kernel output `got` match the emulation `emu`?  Both are [B, S, H*64] or (out_text, out_video) pairs.
    (a) every element: |got - emu| <= ulp_bf16(|emu|) + 2^-8 sum_j p_j |v_j|, however the softmax is split into blocks.
        The kernel's fp32 scores (summed by wgmma in its own order) and ex2.approx differ from the emulation's in the
        last bits, so an exponential that lies on a bf16 midpoint can round the other way; that moves the output by one
        whole bf16 step of P, 2^-8 to 2^-7 of p_j |v_j|.  Half that (2^-9) is not enough: on an H100 one such P
        (e = 0.3037, p = 0.14, carrying 36 % of sum p|v|) took an element to 1.16 times a 2^-9 bound.
    (b) at least `min_equal` of the elements are bit-equal to the emulation.
    (a) caps the error of every element; (b) sees a small systematic change (P truncated, one unmasked key under a
    peaked softmax) that stays inside (a)."""
    got, emu = _joined(got), _joined(emu)
    assert got.shape == emu.shape and got.dtype == emu.dtype == bf16, (got.shape, emu.shape, got.dtype, emu.dtype)
    bound = ulp_bf16(emu) + 2.0 ** -8 * weighted_abs_v(q, k, v, scale)
    ratio = ((got.double() - emu.double()).abs() / bound).max()
    return Acceptance(float((got == emu).double().mean()), float(ratio), min_equal)


# ---- seeded inputs (drawn on the CPU, so the same seed gives the same tensors on every device)

def attention_inputs(B, H, S, score_std=1.0, seed=0, device="cpu"):
    """q, k, v ~ randn in bf16 with q scaled so that the scaled scores q.k / 8 have about `score_std`: 1 gives a flat
    softmax, 3 a peaked one."""
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, H, S, 64, generator=g) for _ in range(3))
    return tuple(t.to(bf16).to(device) for t in (q * score_std, k, v))


def anti_aligned_inputs(B, H, S, seed=0, device="cpu"):
    """k anti-aligned with q: q = 12 u + 0.3 randn, k = -16 u + 0.3 randn for one unit vector u, so every scaled score
    is about -24.  A zero-filled key that escapes the mask scores 0 and takes almost all of a row's weight."""
    g = torch.Generator().manual_seed(seed)
    u = torch.nn.functional.normalize(torch.randn(64, generator=g), dim=0)
    q = 12.0 * u + 0.3 * torch.randn(B, H, S, 64, generator=g)
    k = -16.0 * u + 0.3 * torch.randn(B, H, S, 64, generator=g)
    v = torch.randn(B, H, S, 64, generator=g)
    return tuple(t.to(bf16).to(device) for t in (q, k, v))

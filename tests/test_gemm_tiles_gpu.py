"""Every fused GEMM epilogue at every N-tile width the dispatcher launches (64, 128, 256), on the strided layouts the model
passes, against a step-by-step torch emulation of the epilogue's rounding sequence (include/ea_b200.h, EA_EPI_*).

gemm_tc.cu:dispatch_bn picks the width from the tile count relative to the SM count, so a shape that selects the 256-wide
tile on one GPU may select a narrower one on another: the shapes are built from the device's SM count by rows_for_width()
below, and test_gemm_kernel_instantiations confirms with torch.profiler which gemm_tc_kernel<BN, EPI> actually ran.
tests/test_gemm_tiles_cpu.py checks the shape helpers without a GPU; nothing here touches CUDA at import time."""
import re

import pytest
import torch
import torch.nn.functional as F

from tests.test_gemm_gpu import _rand, _ulp_close, qkv_inputs, qkv_reference

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

BM = 128  # gemm_tc.cu kBM: rows of one output tile
WIDTHS = (64, 128, 256)
EPI_BIAS, EPI_BIAS_GELU, EPI_BIAS_GATE_RES, EPI_SCALE_F32, EPI_BIAS_RES = 0, 1, 2, 3, 4  # include/ea_b200.h
EPI_QKV = 100  # gemm_tc.cu: the template argument of the fused q/k/v projection
EPILOGUES = {"bias": EPI_BIAS, "gelu": EPI_BIAS_GELU, "gate_res": EPI_BIAS_GATE_RES, "scale_f32": EPI_SCALE_F32,
             "bias_res": EPI_BIAS_RES}
BATCHES = 3  # GATE_RES gate rows: batch = row / rows_per_batch
# Lowest fraction of bf16 outputs that must equal the emulated epilogue bit for bit.  The only admissible difference is the
# fp32 accumulation order of the GEMM (~1e-6 relative at K = 3072) moving a value across a bf16 rounding boundary (half an
# ulp = 2e-3 relative); a missing or extra bf16 rounding point changes a large share of the elements.  Observed on H100
# 80GB HBM3 (SXM, 132 SMs; the same values at 400 W and 700 W power limits), the lowest fraction over widths and N: at
# K = 328 0.9998 for every epilogue; at K = 3072 BIAS 0.9981, GELU 0.9983, GATE_RES 0.9996, BIAS_RES 0.9996; the
# ragged-edge columns alone 0.9982; the QKV epilogue's v 0.9997.
MIN_BIT_EXACT = 0.99


def _tiles(M, N, bn):
    return -(-M // BM) * -(-N // bn)


def tile_width(M, N, sms):
    """Python mirror of gemm_tc.cu:dispatch_bn (keep the two in sync): the widest N tile that still gives every SM a tile
    (256) or at least half of them (128), else 64."""
    if N >= 256 and _tiles(M, N, 256) >= sms:
        return 256
    if N >= 128 and _tiles(M, N, 128) >= sms // 2:
        return 128
    return 64


def rows_for_width(width, N, sms, batches=BATCHES):
    """A row count M for which dispatch_bn launches the `width`-wide tile for N columns on `sms` SMs.  M is a multiple of
    `batches` whose per-batch row count is not a multiple of 64 (batch boundaries fall inside a tile) and the last row tile
    is partial.  For widths 128 and 256 there are more tiles than SMs, so CTAs of the persistent kernel run several."""
    nt256, nt128 = -(-N // 256), -(-N // 128)
    if width == 256:
        m_tiles = -(-sms // nt256) + 1
    elif width == 128:
        m_tiles = -(-sms // nt128) + 4
    elif width == 64:
        m_tiles = max(1, (sms // 2 - 1) // nt128)
    else:
        raise ValueError(width)
    M = batches * ((BM * m_tiles - 20) // batches)
    assert -(-M // BM) == m_tiles and (M // batches) % 64 != 0, (width, N, sms, M)
    assert tile_width(M, N, sms) == width, (width, N, sms, M)
    assert width == 64 or _tiles(M, N, width) > sms, (width, N, sms, M)
    return M


def qkv_width(d):
    """gemm_tc.cu:ea_qkv_gemm_ln_rope: the widest tile that divides d, so that no tile straddles the q|k|v boundaries."""
    return 256 if d % 256 == 0 else (128 if d % 128 == 0 else 64)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def emulate_epilogue(epi, acc, bias, residual, gate, rows_per_batch, scale):
    """include/ea_b200.h EA_EPI_* one rounding point at a time, from the fp64 GEMM acc [M, N]: the kernel accumulates in fp32
    and adds the bias in fp32, every later step computes in fp32 and rounds where the header says."""
    acc = acc.float()
    if epi == EPI_SCALE_F32:
        return acc * scale
    lin = (acc + bias.float()).to(bf16)  # bf16(acc + bias)
    if epi == EPI_BIAS:
        return lin
    if epi == EPI_BIAS_GELU:  # bf16(gelu_tanh(bf16(acc + bias)))
        return F.gelu(lin.float(), approximate="tanh").to(bf16)
    if epi == EPI_BIAS_GATE_RES:  # bf16(res + bf16(gate[b] * lin))
        g = gate.float().repeat_interleave(rows_per_batch, dim=0)
        return (residual.float() + (g * lin.float()).to(bf16).float()).to(bf16)
    if epi == EPI_BIAS_RES:  # bf16(lin + res)
        return (lin.float() + residual.float()).to(bf16)
    raise ValueError(epi)


def _operands(M, N, K, seed=0):
    """Operands in the strided layouts production passes: A a column slice of a wider activation (lda > K), W the middle
    third of a [N, 3K] matrix (ldw = 3K: the k / v slices of spatial_attention's fused qkv), the residual a column slice
    (ldr > N), the gate one [B, N] slice of a [B, 6N] modulation tensor."""
    a = _rand((M, K + 72), 1.0, seed + 1)[:, 40:40 + K]
    w = _rand((N, 3 * K), K ** -0.5, seed + 2)[:, K:2 * K]
    bias = _rand((N,), 0.5, seed + 3)
    residual = _rand((M, N + 40), 1.0, seed + 4)[:, :N]
    gate = _rand((BATCHES, 6 * N), 1.0, seed + 5)[:, 2 * N:3 * N]
    assert a.stride(0) > K and w.stride(0) == 3 * K and residual.stride(0) > N and gate.stride(0) == 6 * N
    return a, w, bias, residual, gate


def bit_exact_fraction(out, ref):
    return (out == ref).float().mean().item()


def _bf16_ulp(x):
    """One bf16 ulp at |x| (8 significant bits)."""
    return torch.exp2((torch.frexp(x.float()).exponent - 8).float())


def _gate_res_close(out, ref, acc, bias, gate, rows_per_batch):
    """_ulp_close's bound plus what the one admissible upstream difference does downstream: lin = bf16(acc + bias) one ulp
    off (accumulation order at a rounding boundary) moves gate * lin by |gate| ulp(lin), and the two later roundings
    (y = bf16(gate * lin), bf16(res + y)) can each add one ulp.  On an H100 1-2 outputs in a million at K = 3072 need it."""
    lin = (acc.float() + bias.float()).to(bf16).float()
    g = gate.float().repeat_interleave(rows_per_batch, dim=0)
    y = (g * lin).to(bf16).float()
    ref = ref.float()
    limit = 2e-2 + 2 ** -7 * ref.abs() + g.abs() * _bf16_ulp(lin) + _bf16_ulp(y) + _bf16_ulp(ref)
    err = (out.float() - ref).abs()
    bad = err > limit
    assert not bad.any(), f"{int(bad.sum())} outputs beyond the bound, worst {float((err - limit).max()):.4g} over it"


def _run_epilogue(epi, M, N, K, out_pad=24):
    """One ea_gemm call into a padded output (ldo > N); returns (out, reference, operands) after checking that the pad
    columns were not written."""
    from easyanimate_b200 import ops
    a, w, bias, residual, gate = _operands(M, N, K)
    rpb = M // BATCHES
    scale = N ** -0.5
    dt = torch.float32 if epi == EPI_SCALE_F32 else bf16
    buf = torch.full((M, N + out_pad), -777.0, device="cuda", dtype=dt)
    out = buf[:, :N]
    ops.gemm(a, w, None if epi == EPI_SCALE_F32 else bias, epilogue=epi, out=out,
             residual=residual if epi in (EPI_BIAS_GATE_RES, EPI_BIAS_RES) else None,
             gate=gate if epi == EPI_BIAS_GATE_RES else None, rows_per_batch=rpb, scale=scale)
    assert (buf[:, N:] == -777.0).all(), "store beyond column N (ldo > N)"
    acc = a.double() @ w.double().t()
    ref = emulate_epilogue(epi, acc, bias, residual, gate, rpb, scale)
    return out, ref, (a, w, bias, residual, gate, rpb, scale, acc)


@pytest.mark.parametrize("K", [328, 3072])
@pytest.mark.parametrize("N", [1024, 1000], ids=["N1024", "N1000_ragged"])
@pytest.mark.parametrize("width", WIDTHS)
@pytest.mark.parametrize("epi_name", list(EPILOGUES))
def test_epilogue_at_tile_width(epi_name, width, N, K):
    epi = EPILOGUES[epi_name]
    M = rows_for_width(width, N, _sms())
    out, ref, (a, w, bias, residual, gate, rpb, scale, acc) = _run_epilogue(epi, M, N, K)
    assert torch.isfinite(out).all()
    if epi == EPI_BIAS_GATE_RES:
        _gate_res_close(out, ref, acc, bias, gate, rpb)
    else:
        _ulp_close(out, ref)
    if epi == EPI_SCALE_F32:
        # fp32 output, no rounding point to hit: bound the difference to the fp64 product by the fp32 accumulation error,
        # |err| <= 2^-16 * sum_k |a_k w_k| (~100x tighter than a bf16 ulp)
        bound = (a.double().abs() @ w.double().abs().t()) * scale * 2.0 ** -16
        excess = ((out.double() - acc * scale).abs() - bound).max().item()
        assert excess <= 0, f"scale_f32 off by more than the fp32 accumulation bound ({excess:.3g})"
        return
    frac = bit_exact_fraction(out, ref)
    # the ragged right edge (N % 32 columns) runs its own scalar path, gemm_tc.cu:epilogue_tail: counted on its own too
    tail = slice(N - N % 32, N)
    frac_tail = bit_exact_fraction(out[:, tail], ref[:, tail]) if N % 32 else 1.0
    print(f"BIT_EXACT {epi_name} BN={width} M={M} N={N} K={K}: {frac:.5f} (ragged-edge columns {frac_tail:.5f})")
    assert frac >= MIN_BIT_EXACT, f"only {frac:.4%} of the outputs equal the emulated epilogue bit for bit"
    assert frac_tail >= MIN_BIT_EXACT, f"only {frac_tail:.4%} of the ragged-edge outputs equal the emulated epilogue"


@pytest.mark.parametrize("N", [1024, 1000], ids=["N1024", "N1000_ragged"])
@pytest.mark.parametrize("width", WIDTHS)
def test_gate_residual_in_place_equals_out_of_place(width, N):
    """The residual stream is updated in place (out is residual, ldo = ldr > N): the result must equal the out-of-place
    call bit for bit, including the second staging pass (columns 128..255) of the 256-wide tile."""
    from easyanimate_b200 import ops
    M, K = rows_for_width(width, N, _sms()), 328
    a, w, bias, _, gate = _operands(M, N, K)
    rpb = M // BATCHES
    stream = _rand((M, N + 40), 1.0, 9)  # the residual stream: ldr = ldo = N + 40
    before = stream.clone()
    out = ops.gemm(a, w, bias, epilogue=EPI_BIAS_GATE_RES, residual=before[:, :N], gate=gate, rows_per_batch=rpb)
    x = stream[:, :N]
    ops.gemm(a, w, bias, epilogue=EPI_BIAS_GATE_RES, residual=x, gate=gate, rows_per_batch=rpb, out=x)
    assert torch.equal(x, out)
    assert torch.equal(stream[:, N:], before[:, N:])


@pytest.mark.parametrize("d,B,S_part,S_text,rope", [(384, 2, 333, 77, True), (384, 2, 333, 77, False),
                                                    (192, 3, 205, 40, True), (192, 3, 205, 40, False)])
def test_qkv_at_narrow_tile_widths(d, B, S_part, S_text, rope):
    """ea_qkv_gemm_ln_rope at d = 384 (128-wide tiles) and d = 192 (64-wide tiles): ragged rows_per_batch, a part that
    starts at seq_offset > 0 and rows after it that must stay untouched."""
    from easyanimate_b200 import ops
    assert qkv_width(d) in (128, 64)
    H, S = d // 64, S_text + S_part + 19
    a, w, b, lnq, lnk, rope_cs = qkv_inputs(B, S_part, d, rope, seed=11)
    q = torch.zeros((B, H, S, 64), device="cuda", dtype=bf16)
    k, v = torch.zeros_like(q), torch.zeros_like(q)
    ops.qkv_gemm_ln_rope(a, w, b, lnq, lnk, rope_cs, q, k, v, rows_per_batch=S_part, seq_offset=S_text, eps=1e-6)
    rq, rk, rv = qkv_reference(a, w, b, lnq, lnk, rope_cs, B, S_part)
    rows = slice(S_text, S_text + S_part)
    for got, ref in ((q, rq), (k, rk), (v, rv)):
        _ulp_close(got[:, :, rows], ref, rtol=2 ** -6, atol=3e-2)
        assert torch.count_nonzero(got[:, :, :S_text]) == 0 and torch.count_nonzero(got[:, :, S_text + S_part:]) == 0
    frac = bit_exact_fraction(v[:, :, rows], rv)  # v is bf16(acc + bias): no LayerNorm in between
    print(f"BIT_EXACT qkv.v d={d} BN={qkv_width(d)}: {frac:.5f}")
    assert frac >= MIN_BIT_EXACT


_KERNEL_RE = (re.compile(r"gemm_tc_kernel<(\d+), (\d+)>"), re.compile(r"gemm_tc_kernelILi(\d+)ELi(\d+)E"))


def gemm_kernels_launched(calls):
    """Runs every fn of `calls` in one CUDA-only torch.profiler session and returns the (BN, EPI) of each gemm_tc_kernel
    instantiation they launched, in launch order (one stream)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn in calls:
            fn()
        torch.cuda.synchronize()
    found = []
    for e in sorted(prof.events(), key=lambda e: e.time_range.start):
        for rx in _KERNEL_RE:
            m = rx.search(e.name)
            if m:
                found.append((int(m.group(1)), int(m.group(2))))
                break
    return found


def _qkv_call(d):
    from easyanimate_b200 import ops
    a, w, b, lnq, lnk, rope_cs = qkv_inputs(2, 100, d, True, seed=11)
    q = torch.zeros((2, d // 64, 100, 64), device="cuda", dtype=bf16)
    k, v = torch.zeros_like(q), torch.zeros_like(q)
    return lambda: ops.qkv_gemm_ln_rope(a, w, b, lnq, lnk, rope_cs, q, k, v, rows_per_batch=100, seq_offset=0, eps=1e-6)


def test_gemm_kernel_instantiations():
    """The shapes of the tests above run the kernels they claim to: every epilogue at widths 64, 128 and 256, and the q/k/v
    epilogue at 128 and 64 (d = 384, 192) and 256 (d = 512)."""
    sms, N, K = _sms(), 1000, 328
    labels, expected, calls = [], [], []
    for width in WIDTHS:
        M = rows_for_width(width, N, sms)
        for name, epi in EPILOGUES.items():
            labels.append(f"{name} M={M}")
            expected.append((width, epi))
            calls.append(lambda epi=epi, M=M: _run_epilogue(epi, M, N, K))
    for d in (512, 384, 192):
        labels.append(f"qkv d={d}")
        expected.append((qkv_width(d), EPI_QKV))
        calls.append(_qkv_call(d))
    got = gemm_kernels_launched(calls)
    assert got == expected, list(zip(labels, expected, got + [None] * (len(expected) - len(got))))
    print("GEMM_INSTANTIATIONS", sorted(set(got)))
    assert len(set(got)) == len(WIDTHS) * (len(EPILOGUES) + 1)

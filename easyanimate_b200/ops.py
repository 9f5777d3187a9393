"""Torch-tensor front end of the C ABI: each function checks shapes/dtypes, hands raw device pointers and the
current CUDA stream to ``libea_b200.so`` and returns torch tensors it allocated.  PyTorch is only the allocator and
the stream owner here; none of these functions computes anything with torch ops.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Tuple

import torch

from . import _lib as L

bf16 = torch.bfloat16
ATTN_TIMING = None  # set to a list by bench.py to collect (start, end) CUDA events around every attention launch
# attention kernel selector (include/ea_b200.h `ea_attn_args.variant`); every sixth-generation value runs the one sm_90a
# attention kernel
ATTN_VARIANT = int(os.environ.get("EA_ATTN_VARIANT", "0x217c"), 0)
ATTN_GENERATIONS = L.ea_attn_generations()  # bit 6


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def param_key(*params) -> tuple:
    """Cache key for derived copies of parameters (fused / packed weights): storage address, dtype, device and the in-place
    version counter - which inference-mode tensors do not have (reading it raises), so it is optional."""
    key = []
    for p in params:
        try:
            ver = p._version
        except Exception:
            ver = -1
        key.append((p.data_ptr(), ver, p.dtype, p.device))
    return tuple(key)


def _req(t: torch.Tensor, dtype=bf16, name="tensor"):
    if not t.is_cuda:
        raise L.EaError(f"{name} must be a CUDA tensor (easyanimate_b200 has no CPU path)")
    if t.dtype != dtype:
        raise L.EaError(f"{name} must be {dtype}, got {t.dtype}")


def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, epilogue: int = L.EPI_BIAS,
         out: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
         gate: Optional[torch.Tensor] = None, rows_per_batch: int = 0, scale: float = 1.0) -> torch.Tensor:
    """out[M,N] = epilogue(a[M,K] @ w[N,K]^T + bias). a/w may be row-strided views (last dim contiguous)."""
    _req(a, name="a"); _req(w, name="w")
    assert a.dim() == 2 and w.dim() == 2 and a.shape[1] == w.shape[1], (a.shape, w.shape)
    assert a.stride(1) == 1 and w.stride(1) == 1
    M, K = a.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((M, N), device=a.device, dtype=torch.float32 if epilogue == L.EPI_SCALE_F32 else bf16)
    assert out.shape == (M, N) and out.stride(1) == 1
    args = L.GemmArgs(
        a=_p(a), w=_p(w), bias=_p(bias), out=_p(out), M=M, N=N, K=K,
        lda=a.stride(0), ldw=w.stride(0), ldo=out.stride(0), epilogue=epilogue, scale=scale,
        residual=_p(residual), ldr=residual.stride(0) if residual is not None else 0,
        gate=_p(gate), gate_stride=gate.stride(0) if gate is not None else 0, rows_per_batch=rows_per_batch)
    L.check(L.ea_gemm(C.byref(args), _stream()), "ea_gemm")
    return out


def qkv_gemm_ln_rope(a: torch.Tensor, w_qkv: torch.Tensor, b_qkv: torch.Tensor, ln_q: Tuple[torch.Tensor, torch.Tensor],
                     ln_k: Tuple[torch.Tensor, torch.Tensor], rope: Optional[Tuple[torch.Tensor, torch.Tensor]],
                     q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, *, rows_per_batch: int, seq_offset: int,
                     eps: float = 1e-6, peers=None) -> None:
    """Fused q/k/v projection + per-head LayerNorm + RoPE, written into q/k/v[B,H,S,64] at seq_offset.
    peers (an _lib.QkvPeers): sequence parallelism - q/k/v are this rank's [B,H/P,S,64] buffers and head h of every row is
    stored into the buffer of the rank that owns it (include/ea_b200.h ea_qkv_peers)."""
    _req(a, name="a"); _req(w_qkv, name="w_qkv")
    M, d = a.shape
    assert w_qkv.shape == (3 * d, d) and w_qkv.is_contiguous() and b_qkv.shape == (3 * d,)
    B, H, S, hd = q.shape
    assert hd == 64 and H * 64 == (d if peers is None else peers.heads_per_peer * 64) and k.shape == q.shape and v.shape == q.shape
    assert q.is_contiguous() and k.is_contiguous() and v.is_contiguous()
    cos = sin = None
    if rope is not None:
        cos, sin = rope
        _req(cos, torch.float32, "rope cos"); _req(sin, torch.float32, "rope sin")
        assert cos.shape == (rows_per_batch, 64) and sin.shape == cos.shape and cos.is_contiguous() and sin.is_contiguous()
    args = L.QkvArgs(
        a=_p(a), w=_p(w_qkv), bias=_p(b_qkv), ln_q_w=_p(ln_q[0]), ln_q_b=_p(ln_q[1]), ln_k_w=_p(ln_k[0]),
        ln_k_b=_p(ln_k[1]), rope_cos=_p(cos), rope_sin=_p(sin), q=_p(q), k=_p(k), v=_p(v), M=M, d=d, lda=a.stride(0),
        rows_per_batch=rows_per_batch, S=S, seq_offset=seq_offset, ln_eps=eps,
        peers=None if peers is None else C.pointer(peers))
    L.check(L.ea_qkv_gemm_ln_rope(C.byref(args), _stream()), "ea_qkv_gemm_ln_rope")


def skinny_linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], *, act_in: int = 0,
                  act_out: int = 0) -> torch.Tensor:
    _req(x, name="x"); _req(w, name="w")
    M, K = x.shape
    N = w.shape[0]
    assert w.shape[1] == K and x.is_contiguous() and w.is_contiguous()
    out = torch.empty((M, N), device=x.device, dtype=bf16)
    for m0 in range(0, M, 8):  # the kernel keeps up to 8 input rows in shared memory; larger batches go in row chunks
        m = min(8, M - m0)
        args = L.SkinnyArgs(x=x.data_ptr() + m0 * K * 2, w=_p(w), bias=_p(bias), out=out.data_ptr() + m0 * N * 2, M=m, N=N,
                            K=K, act_in=act_in, act_out=act_out)
        L.check(L.ea_skinny_linear(C.byref(args), _stream()), "ea_skinny_linear")
    return out


def layernorm_modulate(x: torch.Tensor, w: Optional[torch.Tensor], b: Optional[torch.Tensor], eps: float, *,
                       shift: Optional[torch.Tensor] = None, scale: Optional[torch.Tensor] = None,
                       rows_per_batch: int = 0, pre: Optional[Tuple[torch.Tensor, torch.Tensor, float]] = None,
                       out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x: [rows, d] (row stride free). shift/scale: [B, d] views (row stride free, last dim contiguous)."""
    _req(x, name="x")
    rows, d = x.shape
    assert x.stride(1) == 1
    if out is None:
        out = torch.empty((rows, d), device=x.device, dtype=bf16)
    mod_stride = 0
    if shift is not None:
        assert scale is not None and shift.stride(0) == scale.stride(0) and shift.stride(1) == 1
        mod_stride = shift.stride(0)
    args = L.LnArgs(
        x=_p(x), y=_p(out), rows=rows, d=d, ldx=x.stride(0), ldy=out.stride(0), rows_per_batch=rows_per_batch,
        pre_w=_p(pre[0]) if pre else None, pre_b=_p(pre[1]) if pre else None, pre_eps=pre[2] if pre else 0.0,
        w=_p(w), b=_p(b), eps=eps, shift=_p(shift), scale=_p(scale), mod_stride=mod_stride)
    L.check(L.ea_layernorm_modulate(C.byref(args), _stream()), "ea_layernorm_modulate")
    return out


def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    _req(x, name="x")
    rows, d = x.shape
    assert x.is_contiguous()
    out = torch.empty_like(x)
    args = L.RmsArgs(x=_p(x), y=_p(out), w=_p(w), rows=rows, d=d, eps=eps)
    L.check(L.ea_rmsnorm(C.byref(args), _stream()), "ea_rmsnorm")
    return out


def timestep_embedding(t: torch.Tensor, dim: int, flip_sin_to_cos: bool = True, freq_shift: float = 0.0) -> torch.Tensor:
    _req(t, name="timestep")
    out = torch.empty((t.shape[0], dim), device=t.device, dtype=bf16)
    L.check(L.ea_timestep_embedding(_p(t), _p(out), t.shape[0], dim, freq_shift, int(flip_sin_to_cos), _stream()),
            "ea_timestep_embedding")
    return out


def patchify(x: torch.Tensor, x2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[B,C,F,H,W] (+ optional channel-concat source) -> A[B*F*(H/2)*(W/2), ld] with ld = 4C rounded up to 8."""
    _req(x, name="latents")
    B, C1, F, H, W = x.shape
    C2 = 0
    if x2 is not None:
        _req(x2, name="inpaint latents")
        assert x2.shape[0] == B and x2.shape[2:] == x.shape[2:]
        C2 = x2.shape[1]
        x2 = x2.contiguous()
    x = x.contiguous()
    kvalid = 4 * (C1 + C2)
    ldk = (kvalid + 7) // 8 * 8
    a = torch.empty((B * F * (H // 2) * (W // 2), ldk), device=x.device, dtype=bf16)
    L.check(L.ea_patchify(_p(x), _p(x2), _p(a), B, C1, C2, F, H, W, ldk, _stream()), "ea_patchify")
    return a


def unpatchify(y: torch.Tensor, B: int, C: int, F: int, H: int, W: int) -> torch.Tensor:
    _req(y, name="proj_out output")
    out = torch.empty((B, C, F, H, W), device=y.device, dtype=bf16)
    L.check(L.ea_unpatchify(_p(y), _p(out), B, C, F, H, W, y.stride(0), _stream()), "ea_unpatchify")
    return out


def cfg_euler_step(noise_pred: torch.Tensor, latents: torch.Tensor, guidance_scale: float, sigma: float,
                   sigma_next: float, use_cfg: bool = True) -> torch.Tensor:
    """noise_pred: [2B,...] (uncond first, then text) when use_cfg else [B,...]; latents [B,...]."""
    _req(noise_pred, name="noise_pred"); _req(latents, name="latents")
    noise_pred = noise_pred.contiguous(); latents = latents.contiguous()
    n = latents.numel()
    out = torch.empty_like(latents)
    if use_cfg:
        assert noise_pred.numel() == 2 * n
        pu, pt = noise_pred.data_ptr(), noise_pred.data_ptr() + n * 2
    else:
        assert noise_pred.numel() == n
        pu, pt = noise_pred.data_ptr(), None
    L.check(L.ea_cfg_euler_step(pu, pt, _p(latents), _p(out), n, guidance_scale, int(use_cfg), sigma, sigma_next,
                                _stream()), "ea_cfg_euler_step")
    return out


def l1_sums(cur: torch.Tensor, prev: torch.Tensor) -> Tuple[float, float]:
    """(sum |bf16(cur - prev)|, sum |prev|) as the two doubles ea_l1_sums produces: the additive pieces of TeaCache's
    rel-L1 distance, which callers may sum over ranks before rel_l1_from_sums.  Synchronises the stream (the reference's
    .cpu().item() does too)."""
    _req(cur, name="cur"); _req(prev, name="prev")
    assert cur.shape == prev.shape and cur.is_contiguous() and prev.is_contiguous()
    sums = torch.empty((2,), device=cur.device, dtype=torch.float64)
    L.check(L.ea_l1_sums(_p(cur), _p(prev), _p(sums), cur.numel(), _stream()), "ea_l1_sums")
    num, den = (float(x) for x in sums.cpu())
    return num, den


def rel_l1_from_sums(num: float, den: float, n: int) -> float:
    """TeaCache.compute_rel_l1_distance (transformer3d.py:113-117), (|cur-prev|.mean() / |prev|.mean()).item(), from the
    sums of l1_sums over n elements, with the reference's bf16 rounding of each mean and of their ratio."""
    mean_diff = torch.tensor(num / n, dtype=torch.float32).to(bf16)  # .mean() of a bf16 tensor is a bf16 scalar
    mean_prev = torch.tensor(den / n, dtype=torch.float32).to(bf16)
    return float((mean_diff / mean_prev).item())


def dequant_e4m3(w8: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """float8_e4m3fn tensor -> the same values in bf16 (exact), written into `out` (same number of elements)."""
    if not w8.is_cuda or w8.dtype != torch.float8_e4m3fn:
        raise L.EaError(f"dequant_e4m3 takes a CUDA float8_e4m3fn tensor, got {w8.dtype} on {w8.device}")
    _req(out, name="out")
    assert w8.is_contiguous() and out.is_contiguous() and out.numel() == w8.numel()
    L.check(L.ea_dequant_e4m3(_p(w8), _p(out), w8.numel(), _stream()), "ea_dequant_e4m3")
    return out


def e4m3_segment_table(segments) -> tuple:
    """[(byte offset in the packed source, bf16 CUDA destination tensor)] -> the ctypes table expand_e4m3_segments takes.
    Build it once per (slot, staging block) pair: the destinations' addresses are baked in."""
    if not 0 < len(segments) <= L.MAX_E4M3_SEGMENTS:
        raise L.EaError(f"expand_e4m3_segments takes 1 to {L.MAX_E4M3_SEGMENTS} segments, got {len(segments)}")
    n = len(segments)
    offs, dsts, counts = (L.i64 * n)(), (L.vp * n)(), (L.i64 * n)()
    for i, (off, dst) in enumerate(segments):
        _req(dst, name="segment destination")
        assert dst.is_contiguous()
        offs[i], dsts[i], counts[i] = off, dst.data_ptr(), dst.numel()
    return offs, dsts, counts, n


def expand_e4m3_segments(src: torch.Tensor, table) -> None:
    """Expand a packed e4m3 block (a uint8 / float8_e4m3fn CUDA buffer) into bf16 destinations in one launch; `table` from
    e4m3_segment_table.  Bit-identical to one dequant_e4m3 per segment."""
    if not src.is_cuda or src.dtype not in (torch.uint8, torch.float8_e4m3fn):
        raise L.EaError(f"expand_e4m3_segments takes a CUDA uint8 / float8_e4m3fn buffer, got {src.dtype} on {src.device}")
    offs, dsts, counts, n = table
    L.check(L.ea_expand_e4m3_segments(_p(src), offs, dsts, counts, n, _stream()), "ea_expand_e4m3_segments")


def h2d_block(dst: torch.Tensor, src: torch.Tensor, wait_event: Optional[torch.cuda.Event], done_event: torch.cuda.Event,
              copy_stream: torch.cuda.Stream) -> None:
    """Enqueue on copy_stream: wait for wait_event, copy the pinned host buffer src into the device slot dst (its first
    src.nbytes bytes), record done_event."""
    if not dst.is_cuda or src.is_cuda or not src.is_pinned():
        raise L.EaError("h2d_block copies a pinned host buffer into a CUDA buffer")
    assert src.is_contiguous() and dst.is_contiguous() and src.nbytes <= dst.nbytes
    L.check(L.ea_h2d_block(_p(dst), _p(src), src.nbytes, None if wait_event is None else wait_event.cuda_event,
                           done_event.cuda_event, copy_stream.cuda_stream), "ea_h2d_block")


def ew_add(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None, subtract: bool = False) -> torch.Tensor:
    _req(a, name="a"); _req(b, name="b")
    assert a.shape == b.shape and a.is_contiguous() and b.is_contiguous()
    if out is None:
        out = torch.empty_like(a)
    L.check(L.ea_ew_addsub(_p(a), _p(b), _p(out), a.numel(), int(subtract), _stream()), "ea_ew_addsub")
    return out


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, S_text: int, *, scale: Optional[float] = None,
              variant: int = ATTN_VARIANT, peers=None) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """softmax(q k^T * scale) v for q,k,v [B,H,S,64]; returns (out_text [B,S_text,H*64], out_video [B,S-S_text,H*64]).
    peers (an _lib.AttnPeers): sequence parallelism - the rows are stored into the owning ranks' buffers instead
    (include/ea_b200.h ea_attn_peers) and (None, None) is returned."""
    _req(q, name="q"); _req(k, name="k"); _req(v, name="v")
    B, H, S, hd = q.shape
    assert hd == 64 and k.shape == q.shape and q.is_contiguous() and k.is_contiguous()
    if scale is None:
        scale = hd ** -0.5
    S_pad = 0
    if (variant & 0x1102) == 2:  # A/B build only: first-generation kernel with a pre-transposed V
        S_pad = (S + 7) // 8 * 8
        vt = torch.empty((B, H, 64, S_pad), device=q.device, dtype=bf16)
        fn = L.lib.ea_transpose_v
        fn.argtypes, fn.restype = [L.vp, L.vp, L.i64, L.i64, L.i64, L.vp], C.c_int
        L.check(fn(_p(v.contiguous()), _p(vt), B * H, S, S_pad, _stream()), "ea_transpose_v")
        v = vt
    else:
        assert v.shape == q.shape and v.is_contiguous()
    out_text = out_video = None
    if peers is None:
        out_text = torch.empty((B, S_text, H * 64), device=q.device, dtype=bf16)
        out_video = torch.empty((B, S - S_text, H * 64), device=q.device, dtype=bf16)
    args = L.AttnArgs(q=_p(q), k=_p(k), v=_p(v), out_text=_p(out_text) if (S_text and peers is None) else None,
                      out_video=_p(out_video) if (S - S_text and peers is None) else None, B=B, H=H, S=S, S_text=S_text,
                      S_pad=S_pad, head_dim=64, scale=scale, variant=variant, peers=None if peers is None else C.pointer(peers))
    timing = ATTN_TIMING
    if timing is not None:  # bench.py: per-launch CUDA events on the launching stream for the roofline line
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    L.check(L.ea_attn_fwd(C.byref(args), _stream()), "ea_attn_fwd")
    if timing is not None:
        e1.record()
        timing.append((e0, e1))
    return out_text, out_video

"""Torch-tensor front end of the VAE entry points of the C ABI (see include/ea_b200.h).  Activations are
channels-last ``[T,H,W,C]`` bf16 tensors for one batch element; torch only allocates."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

from . import _lib as L
from .ops import _p, _req, _stream, bf16, gemm

CONV_VARIANT = int(os.environ.get("EA_CONV_VARIANT", "0"), 0)  # include/ea_b200.h ea_conv3d_args.variant (accepted, one kernel)


def conv3d_causal(x: torch.Tensor, w_packed: torch.Tensor, bias: torch.Tensor, cout: int, *,
                  residual: Optional[torch.Tensor] = None, dup_frames: bool = False, out_planar: bool = False,
                  stride_t: int = 1, stride_hw: int = 1, out_row0: int = 0, out_rows: int = 0) -> torch.Tensor:
    """x [T,H,W,Cin] -> [T',H',W',cout] (or planar [cout,T',H,W]); w_packed [Cout_pad, 27*Cin] from pack_conv_weight.
    stride_hw / stride_t = 2: the encoder's down-sampling convolutions (include/ea_b200.h ea_conv3d_args.stride_*).
    out_rows > 0: only output rows [out_row0, out_row0 + out_rows) are computed (x carries halo rows around the window;
    strip-parallel decode) and the result / residual have out_rows rows."""
    _req(x, name="x"); _req(w_packed, name="w")
    T, H, W, Cin = x.shape
    assert x.is_contiguous() and w_packed.is_contiguous() and w_packed.shape[1] == 27 * Cin, (x.shape, w_packed.shape)
    T_out = 2 * T - 1 if dup_frames else ((T + 1) // 2 if stride_t == 2 else T)
    if stride_hw == 2:
        H, W = H // 2, W // 2
    if out_rows > 0:
        assert stride_hw == 1 and stride_t == 1 and 0 <= out_row0 and out_row0 + out_rows <= H
        H = out_rows
    shape = (cout, T_out, H, W) if out_planar else (T_out, H, W, cout)
    out = torch.empty(shape, device=x.device, dtype=bf16)
    if residual is not None:
        assert residual.shape == (T, H, W, cout) and residual.is_contiguous()
    args = L.ConvArgs(x=_p(x), w=_p(w_packed), bias=_p(bias), residual=_p(residual), out=_p(out), T=T, H=x.shape[1], W=x.shape[2],
                      Cin=Cin, Cout=cout, Cout_pad=w_packed.shape[0], dup_frames=int(dup_frames),
                      out_planar=int(out_planar), variant=CONV_VARIANT, stride_t=stride_t, stride_hw=stride_hw,
                      out_row0=out_row0, out_rows=out_rows)
    L.check(L.ea_conv3d_causal(C.byref(args), _stream()), "ea_conv3d_causal")
    return out


def pack_conv_weight(w: torch.Tensor, cin_pad: int = 0, cout_pad: int = 0) -> torch.Tensor:
    """[Cout,Cin,3,3,3] -> [Cout_pad, 27*Cin_pad], k = ((kt*3+kh)*3+kw)*Cin_pad + ci (one-time weight preparation)."""
    Cout, Cin = w.shape[:2]
    cin_pad = max(cin_pad, Cin)
    cout_pad = max(cout_pad, Cout)
    wp = torch.zeros((cout_pad, 27, cin_pad), device=w.device, dtype=w.dtype)
    wp[:Cout, :, :Cin] = w.detach().permute(0, 2, 3, 4, 1).reshape(Cout, 27, Cin)
    return wp.reshape(cout_pad, 27 * cin_pad).contiguous()


def prepare_latents(z: torch.Tensor, w: torch.Tensor, b: torch.Tensor, cpad: int = 64, in_scale: float = 1.0) -> torch.Tensor:
    """z [C,T,H,W] planar -> bf16(in_scale * z) -> post_quant_conv -> [T,H,W,cpad] channels-last."""
    _req(z, name="z")
    Cc, T, H, W = z.shape
    z = z.contiguous()
    y = torch.empty((T, H, W, cpad), device=z.device, dtype=bf16)
    L.check(L.ea_vae_prepare_latents(_p(z), _p(w.reshape(Cc, Cc).contiguous()), _p(b), _p(y), Cc, cpad, T, H, W,
                                     float(in_scale), _stream()), "ea_vae_prepare_latents")
    return y


def frames_out(video: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """decode_latents' tail (pipeline_easyanimate.py:729,738-741) in one pass: video bf16 (any shape, contiguous) ->
    out = clamp(clamp(video,-1,1)/2+0.5, 0, 1) as float32 or uint8 (trunc(255*v)).  `out` is a CUDA tensor or a PINNED host
    tensor (the kernel then stores straight into host memory over PCIe; the caller synchronises the stream before reading)."""
    _req(video, name="video")
    assert video.is_contiguous() and out.is_contiguous() and out.numel() == video.numel()
    if out.dtype not in (torch.float32, torch.uint8):
        raise L.EaError(f"frames_out writes float32 or uint8, got {out.dtype}")
    if not out.is_cuda and not out.is_pinned():
        raise L.EaError("frames_out: a host destination must be pinned memory (torch.empty(..., pin_memory=True))")
    kind = L.FRAMES_F32 if out.dtype == torch.float32 else L.FRAMES_U8
    L.check(L.ea_frames_out(_p(video), out.data_ptr(), video.numel(), kind, _stream()), "ea_frames_out")
    return out


def groupnorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int, eps: float, silu: bool) -> torch.Tensor:
    """Per-frame GroupNorm (+SiLU) of x [T,H,W,C]."""
    _req(x, name="x")
    T, H, W, Cc = x.shape
    assert x.is_contiguous()
    stats = torch.empty((T, groups, 2), device=x.device, dtype=torch.float32)
    ws_bytes = L.ea_groupnorm_workspace(T, H, groups)
    ws = torch.empty((ws_bytes,), device=x.device, dtype=torch.uint8)
    L.check(L.ea_groupnorm_stats(_p(x), _p(stats), _p(ws), ws_bytes, T, H, W, Cc, groups, eps, _stream()),
            "ea_groupnorm_stats")
    y = torch.empty_like(x)
    L.check(L.ea_groupnorm_apply(_p(x), _p(y), _p(gamma), _p(beta), _p(stats), T, H * W, Cc, groups, int(silu),
                                 _stream()), "ea_groupnorm_apply")
    return y


def groupnorm_sums(x: torch.Tensor, groups: int) -> torch.Tensor:
    """(sum, sum of squares) per (frame, group) of THIS rank's rows x [T,Hs,W,C] -> float64 [T, groups, 2] (strip-parallel decode)."""
    _req(x, name="x")
    T, H, W, Cc = x.shape
    assert x.is_contiguous()
    sums = torch.empty((T, groups, 2), device=x.device, dtype=torch.float64)
    ws_bytes = L.ea_groupnorm_workspace(T, H, groups)
    ws = torch.empty((ws_bytes,), device=x.device, dtype=torch.uint8)
    L.check(L.ea_groupnorm_sums(_p(x), _p(sums), _p(ws), ws_bytes, T, H, W, Cc, groups, _stream()), "ea_groupnorm_sums")
    return sums


def groupnorm_from_sums(x: torch.Tensor, sums_all: torch.Tensor, count: float, gamma: torch.Tensor, beta: torch.Tensor,
                        groups: int, eps: float, silu: bool) -> torch.Tensor:
    """Per-frame GroupNorm (+SiLU) of this rank's rows with statistics from the gathered sums of ALL ranks
    (sums_all float64 [parts, T, groups, 2], added in rank order; count = pixels of the whole frame x channels per group)."""
    _req(x, name="x")
    T, H, W, Cc = x.shape
    assert sums_all.dtype == torch.float64 and sums_all.is_contiguous() and sums_all.shape[1:] == (T, groups, 2)
    stats = torch.empty((T, groups, 2), device=x.device, dtype=torch.float32)
    L.check(L.ea_groupnorm_finalize(_p(sums_all), _p(stats), sums_all.shape[0], T, groups, float(count), eps, _stream()),
            "ea_groupnorm_finalize")
    y = torch.empty_like(x)
    L.check(L.ea_groupnorm_apply(_p(x), _p(y), _p(gamma), _p(beta), _p(stats), T, H * W, Cc, groups, int(silu), _stream()),
            "ea_groupnorm_apply")
    return y


def upsample2x(x: torch.Tensor) -> torch.Tensor:
    _req(x, name="x")
    T, H, W, Cc = x.shape
    y = torch.empty((T, 2 * H, 2 * W, Cc), device=x.device, dtype=bf16)
    L.check(L.ea_upsample2x(_p(x), _p(y), T, H, W, Cc, _stream()), "ea_upsample2x")
    return y


def softmax_rows(s: torch.Tensor, ldp: int) -> torch.Tensor:
    _req(s, torch.float32, "scores")
    M, N = s.shape
    p = torch.empty((M, ldp), device=s.device, dtype=bf16)
    L.check(L.ea_softmax_rows(_p(s), _p(p), M, N, s.stride(0), ldp, _stream()), "ea_softmax_rows")
    return p


def transpose2d(x: torch.Tensor, ldo: int) -> torch.Tensor:
    """x [R,C] (row stride free) -> [C, ldo] with the first R columns valid."""
    _req(x, name="x")
    R, Cc = x.shape
    out = torch.empty((Cc, ldo), device=x.device, dtype=bf16)
    L.check(L.ea_transpose2d(_p(x), _p(out), R, Cc, x.stride(0), ldo, _stream()), "ea_transpose2d")
    return out


def spatial_attention(n: torch.Tensor, w_qkv: torch.Tensor, b_qkv: torch.Tensor, w_out: torch.Tensor, b_out: torch.Tensor,
                      residual: torch.Tensor, frames: int, scale: float, q_rows: Optional[tuple] = None) -> torch.Tensor:
    """AttnProcessor2_0 (attention_processors.py:105-137) per frame with one head: n [frames*HW, C].
    q_rows = (p0, p1): strip-parallel decode - n holds ALL pixels of every frame (gathered), only the queries of pixels
    [p0, p1) of each frame are evaluated (against all keys) and residual / the result are [frames*(p1-p0), C]."""
    M, Cc = n.shape
    HW = M // frames
    p0, p1 = q_rows if q_rows is not None else (0, HW)
    nq = p1 - p0
    qkv = gemm(n, w_qkv, b_qkv)  # [M, 3C]
    ld = (HW + 7) // 8 * 8
    o = torch.empty((frames * nq, Cc), device=n.device, dtype=bf16)
    for f in range(frames):
        rows = slice(f * HW, (f + 1) * HW)
        qr = slice(f * HW + p0, f * HW + p1)
        q, k, v = qkv[qr, 0:Cc], qkv[rows, Cc:2 * Cc], qkv[rows, 2 * Cc:3 * Cc]
        s = torch.empty((nq, ld), device=n.device, dtype=torch.float32)[:, :HW]
        gemm(q, k, None, epilogue=L.EPI_SCALE_F32, scale=scale, out=s)  # [nq, HW] fp32 scores
        p = softmax_rows(s, ld)
        vt = transpose2d(v, ld)  # [C, ld]
        gemm(p[:, :HW], vt[:, :HW], None, out=o[f * nq:(f + 1) * nq])
    return gemm(o, w_out, b_out, epilogue=L.EPI_BIAS_RES, residual=residual)


def tile_blend(a: torch.Tensor, b: torch.Tensor, extent: int, axis: int) -> None:
    """blend_v (axis 0) / blend_h (axis 1) of autoencoder_magvit.py:319-337 on [..., H, W] views, in place on b."""
    planes = a.shape[0] * a.shape[1] * a.shape[2]
    Ha, Wa, Hb, Wb = a.shape[3], a.shape[4], b.shape[3], b.shape[4]
    if axis == 0:
        extent = min(Ha, Hb, extent)
        rows, cols, off_r, off_c = extent, min(Wa, Wb), Ha - extent, 0
    else:
        extent = min(Wa, Wb, extent)
        rows, cols, off_r, off_c = min(Ha, Hb), extent, 0, Wa - extent
    (pa, la), (pb, lb) = _planar(a), _planar(b)
    L.check(L.ea_tile_blend(_p(a), pa, la, off_r, off_c, _p(b), pb, lb, planes, rows, cols, extent, axis,
                            _stream()), "ea_tile_blend")


def _planar(t: torch.Tensor):
    """(plane stride, row stride) of a [1,C,T,H,W] tensor or crop view whose C*T planes are uniformly strided."""
    assert t.dim() == 5 and t.shape[0] == 1 and t.stride(4) == 1 and t.stride(1) == t.shape[2] * t.stride(2), t.stride()
    return t.stride(2), t.stride(3)


def copy2d(src: torch.Tensor, dst: torch.Tensor, rows: int, cols: int, dst_r0: int, dst_c0: int) -> None:
    """dst[..., dst_r0:dst_r0+rows, dst_c0:dst_c0+cols] = src[..., :rows, :cols] for contiguous [..,H,W] tensors."""
    planes = src.shape[0] * src.shape[1] * src.shape[2]
    (ps, ls), (pd, ld) = _planar(src), _planar(dst)
    dptr = dst.data_ptr() + (dst_r0 * ld + dst_c0) * 2
    L.check(L.ea_copy2d(_p(src), ps, ls, dptr, pd, ld, planes, rows, cols, _stream()), "ea_copy2d")


def corner_blend(src: torch.Tensor, dst: torch.Tensor) -> None:
    """dst[..., -H:, -W:] = w*src + (1-w)*dst[..., -H:, -W:] (autoencoder_magvit.py:429-443)."""
    planes = src.shape[0] * src.shape[1] * src.shape[2]
    Hc, Wc, Hd, Wd = src.shape[3], src.shape[4], dst.shape[3], dst.shape[4]
    assert src.is_contiguous()
    pd, ld = _planar(dst)
    dptr = dst.data_ptr() + ((Hd - Hc) * ld + (Wd - Wc)) * 2
    L.check(L.ea_corner_blend(_p(src), dptr, pd, ld, planes, Hc, Wc, _stream()), "ea_corner_blend")

"""Torch (CPU) stand-ins for the entry points of easyanimate_b200.ops that EasyAnimateTransformer3DModel.forward calls, with
the argument conventions of the real wrappers (shapes, in-place outputs, row-per-batch gates, head-major q/k/v, patchify
column order) and the rounding points documented in include/ea_b200.h, and for those of easyanimate_b200.vae_ops.
TEST INFRASTRUCTURE: `use_stand_ins` installs them all, so that the CPU suite runs the product modules' HOST LOGIC (buffer
plumbing, stream split, sequence-parallel sharding, decode dispatch) end to end without a GPU; they are never used by the
product path."""
import math

import torch

bf16 = torch.bfloat16
EPI_BIAS, EPI_BIAS_GELU, EPI_BIAS_GATE_RES, EPI_SCALE_F32, EPI_BIAS_RES = 0, 1, 2, 3, 4


def _r(x):  # one bf16 rounding point
    return x.to(bf16).float()


def gemm(a, w, bias=None, *, epilogue=EPI_BIAS, out=None, residual=None, gate=None, rows_per_batch=0, scale=1.0):
    acc = a.float() @ w.float().t()
    if epilogue == EPI_SCALE_F32:
        y = acc * scale
        if out is not None:
            out.copy_(y)
            return out
        return y
    y = _r(acc + (bias.float() if bias is not None else 0.0))
    if epilogue == EPI_BIAS_GELU:
        y = _r(torch.nn.functional.gelu(y, approximate="tanh"))
    elif epilogue == EPI_BIAS_GATE_RES:
        batch = torch.arange(a.shape[0]) // rows_per_batch
        y = _r(residual.float() + _r(gate.float()[batch] * y))
    elif epilogue == EPI_BIAS_RES:
        y = _r(y + residual.float())
    y = y.to(bf16)
    if out is not None:
        out.copy_(y)
        return out
    return y


def skinny_linear(x, w, bias, *, act_in=0, act_out=0):
    xf = x.float()
    if act_in:
        xf = _r(torch.nn.functional.silu(xf))
    y = _r(xf @ w.float().t() + (bias.float() if bias is not None else 0.0))
    if act_out:
        y = _r(torch.nn.functional.silu(y))
    return y.to(bf16)


def layernorm_modulate(x, w, b, eps, *, shift=None, scale=None, rows_per_batch=0, pre=None, out=None):
    d = x.shape[1]
    y = x.float()
    if pre is not None:
        y = _r(torch.nn.functional.layer_norm(y, (d,), pre[0].float(), pre[1].float(), pre[2]))
    y = torch.nn.functional.layer_norm(y, (d,), None if w is None else w.float(), None if b is None else b.float(), eps)
    y = _r(y)
    if shift is not None:
        batch = torch.arange(x.shape[0]) // rows_per_batch
        y = _r(_r(y * (1 + scale.float()[batch])) + shift.float()[batch])
    y = y.to(bf16)
    if out is not None:
        out.copy_(y)
        return out
    return y


def rmsnorm(x, w, eps):
    xf = x.float()
    y = _r(xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps))
    return (w.float() * y).to(bf16)


def timestep_embedding(t, dim, flip_sin_to_cos=True, freq_shift=0.0):
    half = dim // 2
    exponent = -math.log(10000) * torch.arange(half, dtype=torch.float32) / (half - freq_shift)
    emb = t.float()[:, None] * torch.exp(exponent)[None, :]
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
    if flip_sin_to_cos:
        emb = torch.cat([emb[:, half:], emb[:, :half]], dim=-1)
    return emb.to(bf16)


def patchify(x, x2=None):
    if x2 is not None:
        x = torch.cat([x, x2], dim=1)
    B, C, F, H, W = x.shape
    a = x.view(B, C, F, H // 2, 2, W // 2, 2).permute(0, 2, 3, 5, 1, 4, 6).reshape(B * F * (H // 2) * (W // 2), C * 4)
    ldk = (4 * C + 7) // 8 * 8
    out = torch.zeros((a.shape[0], ldk), dtype=bf16)
    out[:, :4 * C] = a
    return out


def unpatchify(y, B, C, F, H, W):
    t = y[:, :4 * C].reshape(B, F, H // 2, W // 2, C, 2, 2)
    return t.permute(0, 4, 1, 2, 5, 3, 6).reshape(B, C, F, H, W).contiguous().to(bf16)


def qkv_gemm_ln_rope(a, w_qkv, b_qkv, ln_q, ln_k, rope, q, k, v, *, rows_per_batch, seq_offset, eps=1e-6):
    M, d = a.shape
    B, H = q.shape[0], q.shape[1]
    y = _r(a.float() @ w_qkv.float().t() + b_qkv.float()).view(B, rows_per_batch, 3, H, 64)
    qq, kk, vv = y[:, :, 0], y[:, :, 1], y[:, :, 2]  # [B, rows, H, 64]
    qq = _r(torch.nn.functional.layer_norm(qq, (64,), ln_q[0].float(), ln_q[1].float(), eps))
    kk = _r(torch.nn.functional.layer_norm(kk, (64,), ln_k[0].float(), ln_k[1].float(), eps))
    if rope is not None:
        cos, sin = rope[0][None, :, None, :], rope[1][None, :, None, :]

        def rot(t):
            tr = t.reshape(*t.shape[:-1], 32, 2)
            rotated = torch.stack([-tr[..., 1], tr[..., 0]], dim=-1).flatten(-2)
            return _r(t * cos + rotated * sin)

        qq, kk = rot(qq), rot(kk)
    sl = slice(seq_offset, seq_offset + rows_per_batch)
    q[:, :, sl] = qq.permute(0, 2, 1, 3).to(bf16)
    k[:, :, sl] = kk.permute(0, 2, 1, 3).to(bf16)
    v[:, :, sl] = vv.permute(0, 2, 1, 3).to(bf16)


def attention(q, k, v, S_text, *, scale=None, variant=0):
    B, H, S, hd = q.shape
    o = torch.nn.functional.scaled_dot_product_attention(q.float(), k.float(), v.float(), scale=scale)
    o = o.transpose(1, 2).reshape(B, S, H * hd).to(bf16)
    return o[:, :S_text].contiguous(), o[:, S_text:].contiguous()


def ew_add(a, b, out=None, subtract=False):
    y = (a.float() - b.float() if subtract else a.float() + b.float()).to(bf16)
    if out is not None:
        out.copy_(y)
        return out
    return y


def l1_sums(cur, prev):
    num = (cur.float() - prev.float()).to(bf16).double().abs().sum().item()
    return num, prev.double().abs().sum().item()


# -----------------------------------------------------------------------------------------------------------------------
# VAE entry points (easyanimate_b200.vae_ops): channels-last [T,H,W,C] activations for one batch element
# -----------------------------------------------------------------------------------------------------------------------
def conv3d_causal(x, w_packed, bias, cout, *, residual=None, dup_frames=False, out_planar=False, stride_t=1, stride_hw=1,
                  out_row0=0, out_rows=0):
    T, H, W, Cin = x.shape
    w = w_packed.float().view(w_packed.shape[0], 3, 3, 3, Cin).permute(0, 4, 1, 2, 3)[:cout]  # [cout,Cin,kt,kh,kw]
    xin = x.float().permute(3, 0, 1, 2)[None]  # [1,Cin,T,H,W]
    xin = torch.nn.functional.pad(xin, (0, 0, 0, 0, 2, 0), mode="replicate")
    if stride_hw == 2:  # downsamplers.py:24-96: zero pad right / bottom by one, no padding inside the convolution
        xin = torch.nn.functional.pad(xin, (0, 1, 0, 1))
        y = torch.nn.functional.conv3d(xin, w, bias.float()[:cout], stride=(stride_t, 2, 2))[0]
    else:
        y = torch.nn.functional.conv3d(xin, w, bias.float()[:cout], padding=(0, 1, 1), stride=(stride_t, 1, 1))[0]  # [cout,T,H,W]
    if out_rows > 0:  # ea_conv3d_args.out_row0 / out_rows: only the window's rows exist in the output
        y = y[:, :, out_row0:out_row0 + out_rows]
    y = _r(y)
    if residual is not None:
        y = _r(y + residual.float().permute(3, 0, 1, 2))
    if dup_frames and T > 1:
        idx = [0] + [i for t in range(1, T) for i in (t, t)]
        y = y[:, idx]
    y = y.to(bf16)
    return y.contiguous() if out_planar else y.permute(1, 2, 3, 0).contiguous()


def prepare_latents(z, w, b, cpad=64, in_scale=1.0):
    Cc, T, H, W = z.shape
    zs = _r(z.float() * torch.tensor(in_scale, dtype=torch.float32))
    y = _r(torch.einsum("oc,cthw->othw", w.float().reshape(Cc, Cc), zs) + b.float()[:, None, None, None])
    out = torch.zeros((T, H, W, cpad), dtype=bf16)
    out[..., :Cc] = y.permute(1, 2, 3, 0)
    return out


def groupnorm(x, gamma, beta, groups, eps, silu):
    T, H, W, C = x.shape
    y = torch.nn.functional.group_norm(x.float().permute(0, 3, 1, 2), groups, gamma.float(), beta.float(), eps)  # per frame
    y = _r(y)
    if silu:
        y = _r(torch.nn.functional.silu(y))
    return y.permute(0, 2, 3, 1).contiguous().to(bf16)


def groupnorm_sums(x, groups):
    T, H, W, C = x.shape
    xg = x.double().view(T, H * W, groups, C // groups)
    return torch.stack([xg.sum(dim=(1, 3)), (xg * xg).sum(dim=(1, 3))], dim=-1).contiguous()  # [T, G, 2] fp64


def groupnorm_from_sums(x, sums_all, count, gamma, beta, groups, eps, silu):
    T, H, W, C = x.shape
    tot = torch.zeros_like(sums_all[0])
    for r in range(sums_all.shape[0]):  # rank order, like ea_groupnorm_finalize
        tot = tot + sums_all[r]
    mean = tot[..., 0] / count
    var = (tot[..., 1] / count - mean * mean).clamp_min(0)
    mean, rstd = mean.float(), (1.0 / torch.sqrt(var + eps)).float()  # [T, G]
    cpg = C // groups
    m = mean.repeat_interleave(cpg, dim=1)[:, None, None, :]
    r_ = rstd.repeat_interleave(cpg, dim=1)[:, None, None, :]
    a = r_ * gamma.float()  # the affine form of PyTorch's GroupNorm kernels and of gn_apply2_kernel: y = a x + b
    y = _r(x.float() * a + (beta.float() - a * m))
    if silu:
        y = _r(torch.nn.functional.silu(y))
    return y.contiguous().to(bf16)


def upsample2x(x):
    return x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).contiguous()


def spatial_attention(n, w_qkv, b_qkv, w_out, b_out, residual, frames, scale, q_rows=None):
    M, C = n.shape
    HW = M // frames
    qkv = _r(n.float() @ w_qkv.float().t() + b_qkv.float()).view(frames, HW, 3, C)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    if q_rows is not None:
        q = q[:, q_rows[0]:q_rows[1]]
    p = _r(torch.softmax(q @ k.transpose(1, 2) * scale, dim=-1))
    o = _r(p @ v).reshape(-1, C)
    return _r(_r(o @ w_out.float().t() + b_out.float()) + residual.float()).to(bf16)


def tile_blend(a, b, extent, axis):
    if axis == 0:
        extent = min(a.shape[3], b.shape[3], extent)
        for y in range(extent):
            b[:, :, :, y, :] = (_r(a[:, :, :, -extent + y, :].float() * (1 - y / extent)) +
                                _r(b[:, :, :, y, :].float() * (y / extent))).to(bf16)
    else:
        extent = min(a.shape[4], b.shape[4], extent)
        for x in range(extent):
            b[:, :, :, :, x] = (_r(a[:, :, :, :, -extent + x].float() * (1 - x / extent)) +
                                _r(b[:, :, :, :, x].float() * (x / extent))).to(bf16)


def copy2d(src, dst, rows, cols, dst_r0, dst_c0):
    dst[..., dst_r0:dst_r0 + rows, dst_c0:dst_c0 + cols] = src[..., :rows, :cols]


def corner_blend(src, dst):
    Hc, Wc = src.shape[3], src.shape[4]
    wx = torch.linspace(0, 1, Wc).unsqueeze(0).repeat(Hc, 1)
    wy = torch.linspace(0, 1, Hc).unsqueeze(1).repeat(1, Wc)
    wgt = torch.min(wx, wy)[None, None, None]
    area = dst[..., -Hc:, -Wc:].float()
    dst[..., -Hc:, -Wc:] = (wgt * src.float() + (1 - wgt) * area).to(bf16)


def dequant_e4m3(w8, out):
    out.copy_(w8.to(bf16).reshape(out.shape))
    return out


def frames_out(video, out):
    """include/ea_b200.h ea_frames_out: the reference's op sequence on a bf16 tensor (pipeline_easyanimate.py:729,738-741)."""
    v = (video.clamp(-1, 1) / 2 + 0.5).clamp(0, 1).float()
    out.copy_(v if out.dtype == torch.float32 else (v * 255).to(torch.uint8))
    return out


def frames_out_blend(video, out, overlap):
    """ea_frames_out_blend as the reference's tensor ops (pipeline_easyanimate.py:738-741, then ui.py:524-531)."""
    f = (video.clamp(-1, 1) / 2 + 0.5).clamp(0, 1).float()
    if overlap:
        r = torch.tensor([float(i) / float(overlap) for i in range(overlap)], dtype=torch.float32).view(1, 1, -1, 1, 1)
        out[:, :, :overlap] = out[:, :, :overlap] * (1 - r) + f[:, :, :overlap] * r
    out[:, :, overlap:] = f[:, :, overlap:]
    return out


def cfg_euler_step(noise_pred, latents, guidance_scale, sigma, sigma_next, use_cfg=True):
    """include/ea_b200.h ea_cfg_euler_step: v = u + g*(c-u) in bf16 ops; x_out = bf16(float(x) + bf16(bf16(dt) * v))."""
    if use_cfg:
        u, c = noise_pred.chunk(2)
        v = u + guidance_scale * (c - u)  # bf16 tensor ops, like the reference
    else:
        v = noise_pred
    dt = torch.tensor(sigma_next - sigma, dtype=torch.float32).to(bf16)
    return (latents.float() + (dt * v).float()).to(bf16)


OPS = ("gemm", "skinny_linear", "layernorm_modulate", "rmsnorm", "timestep_embedding", "patchify", "unpatchify", "qkv_gemm_ln_rope",
       "attention", "ew_add", "l1_sums", "cfg_euler_step", "dequant_e4m3")
VAE_OPS = ("conv3d_causal", "prepare_latents", "groupnorm", "groupnorm_sums", "groupnorm_from_sums", "upsample2x",
           "spatial_attention", "tile_blend", "copy2d", "corner_blend", "frames_out", "frames_out_blend")


def _decode_scaled(self, latents, out=None, dtype=torch.float32, to_host=False):
    """AutoencoderKLMagvit.decode_scaled with its tail in host memory (pinned buffers and stream synchronisation need a GPU)."""
    video = self.decode_scaled_video(latents)
    return frames_out(video.contiguous(), torch.empty(video.shape, dtype=dtype) if out is None else out)


def use_stand_ins(mp, **fakes):
    """Run the product's host logic on the CPU: every entry point of easyanimate_b200.ops / vae_ops that has a stand-in above
    is routed to it (or to `fakes[name]`, a test's own variant), the VAE's no-CPU guard `_require_cuda` is lifted (nothing
    else of it), and decode_scaled writes its frames to host memory.  `mp` is a pytest.MonkeyPatch, which undoes all of it.
    Its setattr raises AttributeError for a name the target module does not have, so renaming an entry point in the product
    fails here rather than leaving the renamed one unreplaced."""
    import easyanimate_b200.autoencoder_magvit as A
    from easyanimate_b200 import ops, vae_ops
    assert set(fakes) <= set(OPS + VAE_OPS), sorted(set(fakes) - set(OPS + VAE_OPS))
    for module, names in ((ops, OPS), (vae_ops, VAE_OPS)):
        for name in names:
            mp.setattr(module, name, fakes.get(name, globals()[name]))
    mp.setattr(A, "_require_cuda", lambda t, what: None)
    mp.setattr(A.AutoencoderKLMagvit, "decode_scaled", _decode_scaled)

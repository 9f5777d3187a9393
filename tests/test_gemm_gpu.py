"""wgmma GEMM and its fused epilogues against a plain PyTorch fp32 reference of the same op (GPU only)."""
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


def _rand(shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(bf16)


def _ulp_close(out, ref, rtol=2 ** -7, atol=2e-2):
    # within ~2 bf16 ulps of an fp32-accumulated reference rounded once
    torch.testing.assert_close(out.float(), ref.float(), rtol=rtol, atol=atol)


@pytest.mark.parametrize("M,N,K", [
    (128, 256, 64), (128, 256, 512), (256, 512, 1024), (300, 256, 192), (1000, 3072, 3072),
    (128, 64, 64), (77, 64, 136), (512, 128, 3584), (4096, 12288, 3072), (2000, 3072, 12288), (37, 96, 72),
    (4700, 4352, 320),  # cluster-of-two / multicast-W path with an odd number of row tiles (the last pair is half empty)
])
def test_gemm_bias(M, N, K):
    from easyanimate_b200 import ops
    a, w, b = _rand((M, K), 1.0, 1), _rand((N, K), 0.05, 2), _rand((N,), 1.0, 3)
    out = ops.gemm(a, w, b)
    ref = (a.float() @ w.float().t() + b.float()).to(bf16)
    _ulp_close(out, ref)


def test_gemm_no_bias_strided():
    from easyanimate_b200 import ops
    big = _rand((512, 1024), 1.0, 4)
    a = big[:, 256:768]  # row-strided view
    w = _rand((256, 512), 0.05, 5)
    out = ops.gemm(a, w, None)
    ref = (a.float() @ w.float().t()).to(bf16)
    _ulp_close(out, ref)


def test_gemm_gelu():
    from easyanimate_b200 import ops, _lib as L
    a, w, b = _rand((640, 512), 1.0, 1), _rand((1024, 512), 0.05, 2), _rand((1024,), 0.5, 3)
    out = ops.gemm(a, w, b, epilogue=L.EPI_BIAS_GELU)
    lin = (a.float() @ w.float().t() + b.float()).to(bf16)
    ref = torch.nn.functional.gelu(lin, approximate="tanh")
    _ulp_close(out, ref)


def test_gemm_gate_residual():
    from easyanimate_b200 import ops, _lib as L
    B, S, d = 2, 300, 512
    a, w, b = _rand((B * S, d), 1.0, 1), _rand((d, d), 0.05, 2), _rand((d,), 0.5, 3)
    res = _rand((B * S, d), 1.0, 4)
    mod = _rand((B, 6 * d), 1.0, 5)
    gate = mod[:, 2 * d:3 * d]
    out = ops.gemm(a, w, b, epilogue=L.EPI_BIAS_GATE_RES, residual=res, gate=gate, rows_per_batch=S)
    lin = (a.float() @ w.float().t() + b.float()).to(bf16)
    ref = res.view(B, S, d) + gate[:, None, :] * lin.view(B, S, d)
    _ulp_close(out.view(B, S, d), ref)
    # in-place on the residual stream
    res2 = res.clone()
    ops.gemm(a, w, b, epilogue=L.EPI_BIAS_GATE_RES, residual=res2, gate=gate, rows_per_batch=S, out=res2)
    assert torch.equal(res2, out)


def test_gemm_scale_f32_and_bias_res():
    from easyanimate_b200 import ops, _lib as L
    a, w = _rand((200, 512), 1.0, 1), _rand((320, 512), 1.0, 2)
    out = ops.gemm(a, w, None, epilogue=L.EPI_SCALE_F32, scale=0.125)
    ref = (a.float() @ w.float().t()) * 0.125
    torch.testing.assert_close(out, ref, rtol=1e-4, atol=1e-3)
    b, res = _rand((320,), 1.0, 3), _rand((200, 320), 1.0, 4)
    out2 = ops.gemm(a, w * 0.05, b, epilogue=L.EPI_BIAS_RES, residual=res)
    ref2 = ((a.float() @ (w * 0.05).float().t() + b.float()).to(bf16) + res)
    _ulp_close(out2, ref2)


@pytest.mark.parametrize("B,S_part,S,off,d,rope", [(2, 200, 264, 64, 256, True), (2, 64, 264, 0, 256, False),
                                                   (1, 1000, 1256, 256, 3072, True)])
def test_qkv_gemm_ln_rope(B, S_part, S, off, d, rope):
    from easyanimate_b200 import ops
    H = d // 64
    a = _rand((B * S_part, d), 1.0, 1)
    w, b = _rand((3 * d, d), 0.05, 2), _rand((3 * d,), 0.5, 3)
    lnq = (1 + _rand((64,), 0.1, 4), _rand((64,), 0.1, 5))
    lnk = (1 + _rand((64,), 0.1, 6), _rand((64,), 0.1, 7))
    cos = sin = None
    if rope:
        ang = torch.rand((S_part, 32), device="cuda") * 6.28
        cos = torch.cos(ang).repeat_interleave(2, dim=1).contiguous()
        sin = torch.sin(ang).repeat_interleave(2, dim=1).contiguous()
    q = torch.zeros((B, H, S, 64), device="cuda", dtype=bf16)
    k, v = torch.zeros_like(q), torch.zeros_like(q)
    ops.qkv_gemm_ln_rope(a, w, b, lnq, lnk, (cos, sin) if rope else None, q, k, v, rows_per_batch=S_part,
                         seq_offset=off, eps=1e-6)
    lin = (a.float() @ w.float().t() + b.float()).to(bf16).view(B, S_part, 3, H, 64)
    rq, rk, rv = [lin[:, :, i].transpose(1, 2) for i in range(3)]  # [B,H,S_part,64]
    rq = torch.nn.functional.layer_norm(rq, (64,), lnq[0], lnq[1], 1e-6)
    rk = torch.nn.functional.layer_norm(rk, (64,), lnk[0], lnk[1], 1e-6)

    def rot(x):
        xr, xi = x.reshape(*x.shape[:-1], -1, 2).unbind(-1)
        xrot = torch.stack([-xi, xr], dim=-1).flatten(3)
        return (x.float() * cos + xrot.float() * sin).to(x.dtype)

    if rope:
        rq, rk = rot(rq), rot(rk)
    for got, ref in ((q, rq), (k, rk), (v, rv)):
        _ulp_close(got[:, :, off:off + S_part], ref, rtol=2 ** -6, atol=3e-2)
        assert torch.count_nonzero(got[:, :, :off]) == 0 and torch.count_nonzero(got[:, :, off + S_part:]) == 0

"""The VAE mid-block attention (vae_ops.spatial_attention) against fp32 scaled_dot_product_attention, as the reference's
AttnProcessor2_0 computes it (vaemodules/attention_processors.py:105-137): to_q / to_k / to_v, one head of C channels,
SDPA, to_out, + residual."""
import pytest
import torch
import torch.nn.functional as F

from tests import cpu_ops
from tests.parity import three_way
from tests.test_gemm_gpu import _rand

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


def _sdpa_reference(n, w_qkv, b_qkv, w_out, b_out, residual, frames, scale):
    """fp32 throughout, one frame at a time as one batch element with one head: [frames * HW, C]."""
    M, C = n.shape
    qkv = (n.float() @ w_qkv.float().t() + b_qkv.float()).view(frames, 1, M // frames, 3, C)
    q, k, v = qkv.unbind(3)
    o = F.scaled_dot_product_attention(q, k, v, scale=scale).reshape(M, C)
    return o @ w_out.float().t() + b_out.float() + residual.float()


def test_spatial_attention_matches_sdpa_on_a_ragged_frame():
    """C = 512, T = 2, a 21 x 37 frame: HW = 777 is not a multiple of 32 or 8, so the fp32 score GEMM takes the ragged-N
    tail of the epilogue and writes into a row-padded buffer (ldo = 784 > N), and P.V runs with K = 777.  Also the
    strip-parallel form, query rows [p0, p1) of each frame."""
    from easyanimate_b200 import vae_ops
    C, T, H, W = 512, 2, 21, 37
    HW = H * W
    n = _rand((T * HW, C), 1.5, 1)
    residual = _rand((T * HW, C), 0.5, 2)
    # logits with a spread of several units, so that the softmax is far from uniform and P matters
    w_qkv, b_qkv = _rand((3 * C, C), 1.5 * C ** -0.5, 3), _rand((3 * C,), 0.1, 4)
    w_out, b_out = _rand((C, C), C ** -0.5, 5), _rand((C,), 0.1, 6)
    scale = C ** -0.5
    args = (n, w_qkv, b_qkv, w_out, b_out)
    got = vae_ops.spatial_attention(*args, residual, T, scale)
    truth = _sdpa_reference(*args, residual, T, scale)
    ref_bf16 = cpu_ops.spatial_attention(*args, residual, T, scale)  # the same op-by-op in bf16 (its rounding points)
    assert got.shape == (T * HW, C)
    three_way(got, ref_bf16, truth, name="vae_spatial_attention_21x37")

    p0, p1 = 5 * W + 3, 17 * W + 1
    rows = torch.cat([torch.arange(f * HW + p0, f * HW + p1) for f in range(T)]).cuda()
    part = vae_ops.spatial_attention(*args, residual[rows].contiguous(), T, scale, q_rows=(p0, p1))
    three_way(part, ref_bf16[rows], truth[rows], name="vae_spatial_attention_21x37_rows")

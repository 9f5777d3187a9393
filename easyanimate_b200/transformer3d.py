"""H100-native drop-in for ``easyanimate.models.transformer3d.EasyAnimateTransformer3DModel`` (v5 / v5.1 MMDiT).

Same constructor arguments, ``.config`` surface, ``forward`` signature and ``state_dict`` keys as the reference
(/root/reference/easyanimate/models/transformer3d.py:1346-1689), so ``EasyAnimatePipeline`` /
``EasyAnimateInpaintPipeline`` can be handed this module unchanged.  The nn.Linear / nn.LayerNorm / nn.Conv2d
objects below only OWN the parameters under the reference's key names; the forward pass never calls them — every
arithmetic step is a kernel of libea_b200.so (wgmma GEMMs with fused epilogues, wgmma attention, fused
LayerNorm/AdaLN kernels).  There is no PyTorch/CPU fallback.
"""
from __future__ import annotations

import os
from typing import Any, Dict, Optional

import torch
import torch.nn as nn

from . import _lib as L
from . import ops
from .config import ConfigMixinLite, Transformer2DModelOutput, capture_init_config, load_state_dict_from_dir

bf16 = torch.bfloat16


# ---------------------------------------------------------------------------------------------------------------
# parameter containers (reference key layout)
# ---------------------------------------------------------------------------------------------------------------
class _RMSNormParams(nn.Module):
    def __init__(self, dim: int, eps: float = 1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim))
        self.variance_epsilon = eps


class _LayerNormZero(nn.Module):  # norm.py:135-158
    def __init__(self, cond_dim: int, dim: int, eps: float, affine: bool):
        super().__init__()
        self.linear = nn.Linear(cond_dim, 6 * dim, bias=True)
        self.norm = nn.LayerNorm(dim, eps=eps, elementwise_affine=affine)


class _Attention(nn.Module):  # diffusers Attention(qk_norm="layer_norm", bias=True) as built at attention.py:1056-1074
    def __init__(self, dim: int, heads: int, dim_head: int, eps: float = 1e-6):
        super().__init__()
        inner = heads * dim_head
        self.heads = heads
        self.to_q = nn.Linear(dim, inner, bias=True)
        self.to_k = nn.Linear(dim, inner, bias=True)
        self.to_v = nn.Linear(dim, inner, bias=True)
        self.norm_q = nn.LayerNorm(dim_head, eps=eps)
        self.norm_k = nn.LayerNorm(dim_head, eps=eps)
        self.to_out = nn.ModuleList([nn.Linear(inner, dim, bias=True), nn.Dropout(0.0)])
        self._fused: Optional[tuple] = None
        self._fused_static: Optional[tuple] = None

    def fused_qkv(self):
        """[3d,d] weight / [3d] bias for the fused projection kernel; rebuilt when the parameters change."""
        if self._fused_static is not None:  # fp8 staging block: the buffers are filled by _Fp8Staging.block()
            return self._fused_static
        ps = (self.to_q.weight, self.to_k.weight, self.to_v.weight, self.to_q.bias, self.to_k.bias, self.to_v.bias)
        key = ops.param_key(*ps)
        if self._fused is None or self._fused[0] != key:
            w = torch.cat([p.detach() for p in ps[:3]], dim=0).contiguous()
            b = torch.cat([p.detach() for p in ps[3:]], dim=0).contiguous()
            self._fused = (key, w, b)
        return self._fused[1], self._fused[2]


class _GELUProj(nn.Module):
    def __init__(self, dim_in: int, dim_out: int):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out)


class _FeedForward(nn.Module):  # diffusers FeedForward(activation_fn="gelu-approximate"), attention.py:1082-1100
    def __init__(self, dim: int, inner_dim: Optional[int] = None):
        super().__init__()
        inner = inner_dim or dim * 4
        self.net = nn.ModuleList([_GELUProj(dim, inner), nn.Dropout(0.0), nn.Linear(inner, dim), nn.Dropout(0.0)])


class _AdaLayerNorm(nn.Module):  # diffusers AdaLayerNorm(chunk_dim=1), transformer3d.py:1472-1478
    def __init__(self, cond_dim: int, out_dim: int, eps: float, affine: bool):
        super().__init__()
        self.linear = nn.Linear(cond_dim, out_dim)
        self.norm = nn.LayerNorm(out_dim // 2, eps, affine)


class _TimestepEmbedding(nn.Module):
    def __init__(self, in_dim: int, time_embed_dim: int):
        super().__init__()
        self.linear_1 = nn.Linear(in_dim, time_embed_dim)
        self.linear_2 = nn.Linear(time_embed_dim, time_embed_dim)


class EasyAnimateDiTBlock(nn.Module):
    """attention.py:1028-1163 on the H100 kernels."""

    def __init__(self, dim, num_attention_heads, attention_head_dim, time_embed_dim, norm_elementwise_affine=True,
                 norm_eps=1e-5, is_mmdit_block=True, ff_inner_dim=None):
        super().__init__()
        self.norm1 = _LayerNormZero(time_embed_dim, dim, norm_eps, norm_elementwise_affine)
        self.attn1 = _Attention(dim, num_attention_heads, attention_head_dim)
        self.attn2 = _Attention(dim, num_attention_heads, attention_head_dim) if is_mmdit_block else None
        self.norm2 = _LayerNormZero(time_embed_dim, dim, norm_eps, norm_elementwise_affine)
        self.ff = _FeedForward(dim, ff_inner_dim)
        self.txt_ff = _FeedForward(dim, ff_inner_dim) if is_mmdit_block else None
        self.norm3 = None
        self.dim = dim

    @staticmethod
    def _ln_mod(x, zero: _LayerNormZero, mod, lo, rows_per_batch, out=None):
        d = x.shape[1]
        return ops.layernorm_modulate(x, zero.norm.weight, zero.norm.bias, zero.norm.eps, shift=mod[:, lo * d:(lo + 1) * d],
                                      scale=mod[:, (lo + 1) * d:(lo + 2) * d], rows_per_batch=rows_per_batch, out=out)

    def forward(self, x_v, x_t, silu_in_temb, rope, ws: "_Workspace"):
        """x_v [B*S_v,d], x_t [B*S_t,d] are updated in place and returned."""
        d = self.dim
        B, S_v, S_t = ws.B, ws.S_v, ws.S_t
        # --- attention half (attention.py:1117-1141)
        mod = ops.skinny_linear(silu_in_temb, self.norm1.linear.weight, self.norm1.linear.bias, act_in=1)  # [B,6d]
        n_v = self._ln_mod(x_v, self.norm1, mod, 0, S_v, out=ws.n_v)
        n_t = self._ln_mod(x_t, self.norm1, mod, 3, S_t, out=ws.n_t)
        a_t = self.attn2 if self.attn2 is not None else self.attn1
        w1, b1 = self.attn1.fused_qkv()
        w2, b2 = a_t.fused_qkv()
        ln1 = ((self.attn1.norm_q.weight, self.attn1.norm_q.bias), (self.attn1.norm_k.weight, self.attn1.norm_k.bias))
        ln2 = ((a_t.norm_q.weight, a_t.norm_q.bias), (a_t.norm_k.weight, a_t.norm_k.bias))
        if ws.px is not None:
            # sequence parallelism, fused exchange (sequence_parallel.PeerExchange): the projections store each head's rows
            # into the q/k/v buffer of the rank that owns the head, attention stores each token's row into the buffer of the
            # rank that owns the token; two 4-byte all-reduces order the kernels across GPUs
            px = ws.px
            ops.qkv_gemm_ln_rope(n_v, w1, b1, ln1[0], ln1[1], rope, px.q, px.k, px.v, rows_per_batch=S_v,
                                 seq_offset=S_t + px.rank * S_v, eps=self.attn1.norm_q.eps, peers=px.qkv_video)
            ops.qkv_gemm_ln_rope(n_t, w2, b2, ln2[0], ln2[1], None, px.q, px.k, px.v, rows_per_batch=S_t, seq_offset=0,
                                 eps=a_t.norm_q.eps, peers=px.qkv_text)
            px.barrier()
            ops.attention(px.q, px.k, px.v, S_t, peers=px.attn)
            px.barrier()
            o_t, o_v = px.out_text, px.out_video
        else:
            ops.qkv_gemm_ln_rope(n_v, w1, b1, ln1[0], ln1[1], rope, ws.q, ws.k, ws.v, rows_per_batch=S_v, seq_offset=S_t,
                                 eps=self.attn1.norm_q.eps)
            ops.qkv_gemm_ln_rope(n_t, w2, b2, ln2[0], ln2[1], None, ws.q, ws.k, ws.v, rows_per_batch=S_t, seq_offset=0,
                                 eps=a_t.norm_q.eps)
            o_t, o_v = ops.attention(ws.q, ws.k, ws.v, S_t) if ws.sp is None else ws.sp.attention(ws.q, ws.k, ws.v, S_t)
        ops.gemm(o_v.view(B * S_v, d), self.attn1.to_out[0].weight, self.attn1.to_out[0].bias,
                 epilogue=L.EPI_BIAS_GATE_RES, residual=x_v, gate=mod[:, 2 * d:3 * d], rows_per_batch=S_v, out=x_v)
        ops.gemm(o_t.view(B * S_t, d), a_t.to_out[0].weight, a_t.to_out[0].bias,
                 epilogue=L.EPI_BIAS_GATE_RES, residual=x_t, gate=mod[:, 5 * d:6 * d], rows_per_batch=S_t, out=x_t)
        # --- feed-forward half (attention.py:1144-1162)
        mod = ops.skinny_linear(silu_in_temb, self.norm2.linear.weight, self.norm2.linear.bias, act_in=1)
        n_v = self._ln_mod(x_v, self.norm2, mod, 0, S_v, out=ws.n_v)
        n_t = self._ln_mod(x_t, self.norm2, mod, 3, S_t, out=ws.n_t)
        ff_t = self.txt_ff if self.txt_ff is not None else self.ff
        h_v = ops.gemm(n_v, self.ff.net[0].proj.weight, self.ff.net[0].proj.bias, epilogue=L.EPI_BIAS_GELU, out=ws.h_v)
        ops.gemm(h_v, self.ff.net[2].weight, self.ff.net[2].bias, epilogue=L.EPI_BIAS_GATE_RES, residual=x_v,
                 gate=mod[:, 2 * d:3 * d], rows_per_batch=S_v, out=x_v)
        h_t = ops.gemm(n_t, ff_t.net[0].proj.weight, ff_t.net[0].proj.bias, epilogue=L.EPI_BIAS_GELU, out=ws.h_t)
        ops.gemm(h_t, ff_t.net[2].weight, ff_t.net[2].bias, epilogue=L.EPI_BIAS_GATE_RES, residual=x_t,
                 gate=mod[:, 5 * d:6 * d], rows_per_batch=S_t, out=x_t)
        return x_v, x_t


def get_teacache_coefficients(model_name: str):
    """transformer3d.py:124-137: polynomial that rescales the relative-L1 change, per released checkpoint family."""
    name = model_name.lower()
    if "v5.1-7b" in name:
        return [1.07862322, -4.19362456, 3.06725828, 0.33161686, 0.02374758]
    if "v5.1-12b" in name:
        return [-10.47857366, 8.33844143, -0.78477557, 0.68798618, 0.0136149]
    print(f"The model {model_name} is not supported by TeaCache.")
    return None


class TeaCache:
    """Timestep-embedding-aware step skipping, transformer3d.py:90-121: same counters, thresholds and polynomial
    rescale as the reference; `previous_modulated_input` / `previous_residual` are device tensors here."""

    def __init__(self, coefficients, num_steps: int, rel_l1_thresh: float = 0.0):
        if num_steps < 1:
            raise ValueError(f"`num_steps` must be greater than 0 but is {num_steps}.")
        if rel_l1_thresh < 0:
            raise ValueError(f"`rel_l1_thresh` must be greater than or equal to 0 but is {rel_l1_thresh}.")
        self.coefficients = list(coefficients)
        self.cnt = 0
        self.num_steps = num_steps
        self.rel_l1_thresh = rel_l1_thresh
        self.accumulated_rel_l1_distance = 0
        self.previous_modulated_input = None
        self.previous_residual = None
        self.skipped = 0

    def rescale_func(self, x: float) -> float:  # np.poly1d(coefficients)(x), highest degree first
        y = 0.0
        for c in self.coefficients:
            y = y * x + c
        return y

    def reset(self):
        self.cnt = 0
        self.previous_modulated_input = None
        self.previous_residual = None


def sincos_pos_embed_2d(embed_dim: int, grid_size, base_size: int = 16):
    """diffusers 0.30/0.31 `get_2d_sincos_pos_embed(embed_dim, (H, W))`, which the reference calls for the Control model's
    `ref_pos_embedding` buffer (transformer3d.py:1424), restated from its published (MAE) algorithm: numpy float64
    [H*W, embed_dim], rows in (h, w) order, columns (sin | cos) of the h axis then of the w axis."""
    import numpy as np

    def one_d(dim, pos):
        omega = 1.0 / 10000 ** (np.arange(dim // 2, dtype=np.float64) / (dim / 2.0))
        out = np.einsum("m,d->md", pos.reshape(-1), omega)
        return np.concatenate([np.sin(out), np.cos(out)], axis=1)
    grid_h = np.arange(grid_size[0], dtype=np.float32) / (grid_size[0] / base_size)
    grid_w = np.arange(grid_size[1], dtype=np.float32) / (grid_size[1] / base_size)
    grid = np.stack(np.meshgrid(grid_w, grid_h), axis=0).reshape([2, 1, grid_size[1], grid_size[0]])
    return np.concatenate([one_d(embed_dim // 2, grid[0]), one_d(embed_dim // 2, grid[1])], axis=1)


class _Fp8Staging:
    """bf16 staging for a model whose parameters are STORED as float8_e4m3fn - the reference's `model_cpu_offload_and_qfloat8`
    mode (predict_t2v.py:37,106: from_pretrained_2d(torch_dtype=float8_e4m3fn); utils/fp8_optimization.py:6-35 casts every
    module to bf16 around its own forward and back).  Same arithmetic here: every kernel consumes bf16(e4m3(w)); what stays
    resident is the e4m3 copy (half the bytes: 11.8 GB instead of 23.6 GB for the 12B model) plus ONE block's worth of bf16
    weights that `block()` refills with `ea_dequant_e4m3` right before the block runs, and the small non-block parameters."""

    def __init__(self, model: "EasyAnimateTransformer3DModel"):
        dev = next(model.parameters()).device
        cfg = {k: v for k, v in model.config.items() if not k.startswith("_")}
        cfg["num_layers"] = 0
        with torch.device(dev):
            self.head = EasyAnimateTransformer3DModel(**cfg).to(bf16)
        own = dict(self.head.named_parameters())
        for name, p8 in model.named_parameters():
            if not name.startswith("transformer_blocks."):
                ops.dequant_e4m3(p8.detach().contiguous(), own[name].detach())
        self._blocks: Dict[bool, EasyAnimateDiTBlock] = {}
        self._model_cfg = model.config
        self._dev = dev

    def _staging_block(self, mmdit: bool) -> "EasyAnimateDiTBlock":
        if mmdit not in self._blocks:
            c = self._model_cfg
            d = c.num_attention_heads * c.attention_head_dim
            with torch.device(self._dev):
                blk = EasyAnimateDiTBlock(d, c.num_attention_heads, c.attention_head_dim, c.time_embed_dim,
                                          c.norm_elementwise_affine, c.norm_eps, is_mmdit_block=mmdit).to(bf16)
                for a in (blk.attn1, blk.attn2):
                    if a is not None:
                        a._fused_static = (torch.empty((3 * d, d), dtype=bf16), torch.empty((3 * d,), dtype=bf16))
            self._blocks[mmdit] = blk
        return self._blocks[mmdit]

    def block(self, blk8: "EasyAnimateDiTBlock") -> "EasyAnimateDiTBlock":
        """Expand blk8's e4m3 parameters into the staging block (stream-ordered: the previous block's kernels that read the
        staging buffers are ahead of these writes on the same stream) and return it."""
        st = self._staging_block(blk8.attn2 is not None)
        for name, p8 in blk8.named_parameters():
            ops.dequant_e4m3(p8.detach().contiguous(), self.destination(st, name))
        return st

    @staticmethod
    def destination(st: "EasyAnimateDiTBlock", name: str) -> torch.Tensor:
        """Where the staging block `st` holds parameter `name` in bf16: q/k/v go straight into the fused projection operand."""
        parts = name.split(".")
        if parts[0] in ("attn1", "attn2") and parts[1] in ("to_q", "to_k", "to_v"):
            w, b = getattr(st, parts[0])._fused_static
            d = st.dim
            i = ("to_q", "to_k", "to_v").index(parts[1])
            return w[i * d:(i + 1) * d] if parts[2] == "weight" else b[i * d:(i + 1) * d]
        return st.get_parameter(name).detach()


class _Workspace:
    """Per-forward activation buffers shared by all blocks (allocated once per call through torch's caching allocator)."""

    def __init__(self, B, S_v, S_t, d, heads, ff_inner, device, sp=None):
        self.B, self.S_v, self.S_t = B, S_v, S_t
        self.sp = sp  # UlyssesAttention (sequence parallelism: S_v is then this rank's token count) or None
        S = S_v + S_t
        e = lambda *shape: torch.empty(shape, device=device, dtype=bf16)  # noqa: E731
        self.n_v, self.n_t = e(B * S_v, d), e(B * S_t, d)
        self.px = sp.exchange(B, heads, S_t, S_v, device) if (sp is not None and sp.p2p) else None
        if self.px is None:
            self.q, self.k, self.v = e(B, heads, S, 64), e(B, heads, S, 64), e(B, heads, S, 64)
        self.h_v, self.h_t = e(B * S_v, ff_inner), e(B * S_t, ff_inner)


class EasyAnimateTransformer3DModel(nn.Module, ConfigMixinLite):
    _supports_gradient_checkpointing = False

    def __init__(
        self,
        num_attention_heads: int = 30,
        attention_head_dim: int = 64,
        in_channels: Optional[int] = None,
        out_channels: Optional[int] = None,
        patch_size: Optional[int] = None,
        sample_width: int = 90,
        sample_height: int = 60,
        ref_channels: int = None,
        clip_channels: int = None,
        activation_fn: str = "gelu-approximate",
        timestep_activation_fn: str = "silu",
        freq_shift: int = 0,
        num_layers: int = 30,
        mmdit_layers: int = 10000,
        swa_layers: list = None,
        dropout: float = 0.0,
        time_embed_dim: int = 512,
        add_norm_text_encoder: bool = False,
        text_embed_dim: int = 4096,
        text_embed_dim_t5: int = 4096,
        norm_eps: float = 1e-5,
        norm_elementwise_affine: bool = True,
        flip_sin_to_cos: bool = True,
        time_position_encoding_type: str = "3d_rope",
        after_norm=False,
        resize_inpaint_mask_directly: bool = False,
        enable_clip_in_inpaint: bool = True,
        position_of_clip_embedding: str = "full",
        enable_text_attention_mask: bool = True,
        add_noise_in_inpaint_model: bool = False,
        add_ref_latent_in_control_model: bool = False,
    ):
        super().__init__()
        object.__setattr__(self, "config", capture_init_config(self, locals()))
        if attention_head_dim != 64:
            raise ValueError("easyanimate_b200 attention kernels are built for attention_head_dim=64 (all v5/v5.1 releases)")
        if patch_size != 2:
            raise ValueError("easyanimate_b200 patch-embed kernels are built for patch_size=2 (all v5/v5.1 releases)")
        if activation_fn != "gelu-approximate" or timestep_activation_fn != "silu":
            raise ValueError("only activation_fn='gelu-approximate' / timestep_activation_fn='silu' are implemented")
        if swa_layers is not None or after_norm:
            raise NotImplementedError("swa_layers / after_norm are not used by the v5.1 T2V / I2V / Control models")
        if not norm_elementwise_affine:
            raise NotImplementedError("norm_elementwise_affine=False is not used by any released config")
        self.num_heads = num_attention_heads
        self.inner_dim = num_attention_heads * attention_head_dim
        self.resize_inpaint_mask_directly = resize_inpaint_mask_directly
        self.enable_clip_in_inpaint = enable_clip_in_inpaint
        self.patch_size = patch_size
        self.post_patch_height = sample_height // patch_size
        self.post_patch_width = sample_width // patch_size
        d = self.inner_dim

        self.time_embedding = _TimestepEmbedding(d, time_embed_dim)
        self.proj = nn.Conv2d(in_channels, d, kernel_size=(patch_size, patch_size), stride=patch_size, bias=True)
        if not add_norm_text_encoder:
            self.text_proj = nn.Linear(text_embed_dim, d)
            if text_embed_dim_t5 is not None:
                self.text_proj_t5 = nn.Linear(text_embed_dim_t5, d)
        else:
            self.text_proj = nn.Sequential(_RMSNormParams(text_embed_dim), nn.Linear(text_embed_dim, d))
            if text_embed_dim_t5 is not None:
                # (the reference sizes this RMSNorm with text_embed_dim, transformer3d.py:1415-1418)
                self.text_proj_t5 = nn.Sequential(_RMSNormParams(text_embed_dim), nn.Linear(text_embed_dim_t5, d))
        if ref_channels is not None:  # v5.1 Control: reference-image tokens (transformer3d.py:1420-1426)
            self.ref_proj = nn.Conv2d(ref_channels, d, kernel_size=(patch_size, patch_size), stride=patch_size, bias=True)
            self.register_buffer("ref_pos_embedding", torch.from_numpy(
                sincos_pos_embed_2d(d, (self.post_patch_height, self.post_patch_width))), persistent=False)
        if clip_channels is not None:  # transformer3d.py:1428-1429
            self.clip_proj = nn.Linear(clip_channels, d)
        self.transformer_blocks = nn.ModuleList([
            EasyAnimateDiTBlock(d, num_attention_heads, attention_head_dim, time_embed_dim, norm_elementwise_affine,
                                norm_eps, is_mmdit_block=i < mmdit_layers) for i in range(num_layers)])
        self.norm_final = nn.LayerNorm(d, norm_eps, norm_elementwise_affine)
        self.norm_out = _AdaLayerNorm(time_embed_dim, 2 * d, norm_eps, norm_elementwise_affine)
        self.proj_out = nn.Linear(d, patch_size * patch_size * out_channels)
        self.teacache = None
        self.sequence_parallel = None  # UlyssesAttention, see set_sequence_parallel_group
        self.cfg_parallel_group = None  # 2-rank group holding the other CFG branch, see set_cfg_parallel_group
        self.gradient_checkpointing = False
        self._proj_w_cache: Dict[str, tuple] = {}
        self._ref_pos_cache: Optional[tuple] = None
        self._fp8: Optional[tuple] = None  # (parameter key, _Fp8Staging) when the parameters are stored as float8_e4m3fn
        self._offload = None  # offload.SequentialOffload, see enable_sequential_cpu_offload

    # ----------------------------------------------------------------------------------------------------------
    def enable_teacache(self, num_steps: int, rel_l1_thresh: float,
                        coefficients=(-10.47857366, 8.33844143, -0.78477557, 0.68798618, 0.0136149)):
        """transformer3d.py:1485-1491. The cache tensors stay on the device (the reference keeps them on the CPU)."""
        self.teacache = TeaCache(list(coefficients), num_steps, rel_l1_thresh=rel_l1_thresh)

    def set_sequence_parallel_group(self, group):
        """Ulysses sequence parallelism over the ranks of `group` for ONE video.  The reference has NO multi-GPU inference
        path at this commit; this is this framework's own answer to the per-block exchange joint
        attention needs (processor.py:287-289).  Every rank calls forward with the same inputs and
        gets the full output; video tokens and attention heads must divide by the group size.  None restores
        single-GPU execution."""
        from .sequence_parallel import UlyssesAttention
        old = getattr(self, "sequence_parallel", None)
        if old is not None:
            old.release()  # collective: every rank of the old group unmaps its peers' buffers
        self.sequence_parallel = None if group is None else UlyssesAttention(group)

    def set_cfg_parallel_group(self, group):
        """CFG-parallel execution (EasyAnimateSampler(cfg_group=...)): this module sees ONE branch of the reference's
        batch of 2 (pipeline_easyanimate.py:1074).  The only place where the branches interact inside the transformer is
        TeaCache, whose skip decision comes from the rel-L1 MEAN over the joint batch (transformer3d.py:1563-1586): the
        additive pieces are summed over `group` so that both ranks take the reference's decision."""
        self.cfg_parallel_group = group

    def enable_sequential_cpu_offload(self, device="cuda", streamer=None):
        """The reference's `sequential_cpu_offload` for this module: the non-block parameters move to `device`, each block's
        parameters into one pinned host buffer (in the dtype they are stored in: bf16, or float8_e4m3fn), and every forward
        streams the blocks through two device slots, copying block i+1 on a side stream while block i runs (offload.py).
        Results are bit-identical to resident execution.  Device memory for parameters: the non-block ones, two slots of one
        block each, and for e4m3 storage one bf16 staging block.  `.to(...)`, `load_state_dict` and invalidate_weight_caches()
        are followed: the blocks are repacked on the next forward when their parameters were replaced.  `streamer` replaces
        the CUDA copy stream and events (tests).  A forward of an offloaded module cannot be captured in a CUDA graph."""
        from .offload import SequentialOffload
        self._offload = None
        self.invalidate_weight_caches()  # device copies a resident forward derived from the blocks (fused q/k/v, ...)
        self._offload = SequentialOffload(self, device, streamer)
        return self

    def _set_gradient_checkpointing(self, module, value=False):
        self.gradient_checkpointing = value

    def invalidate_weight_caches(self) -> None:
        """Drop every derived copy of the parameters (fused q/k/v weights, the patch-embed GEMM operands, the fp8 staging block).
        They are rebuilt on the next forward.  Needed only after edits that bypass the parameters' version counters - the
        reference's LoRA merge / unmerge writes `layer.weight.data += ...` (utils/lora_utils.py:425-429,487-491), which neither
        moves the storage nor bumps `_version`; `load_state_dict`, `.to(...)` and in-place ops on the parameters themselves are
        detected without this call."""
        for m in self.modules():
            if isinstance(m, _Attention):
                m._fused = None
        self._proj_w_cache.clear()
        self._ref_pos_cache = None
        self._fp8 = None
        if self._offload is not None:
            self._offload.invalidate()

    def _fp8_staging(self) -> _Fp8Staging:
        key = ops.param_key(self.proj.weight, self.proj_out.weight)
        if self._fp8 is None or self._fp8[0] != key:
            self._fp8 = (key, _Fp8Staging(self))
        return self._fp8[1]

    def _patch_weight(self, ldk: int, which: str = "proj") -> torch.Tensor:
        """The 2x2 patch-embed Conv2d weight of `proj` / `ref_proj` as the [d, ldk] GEMM operand of ea_patchify's rows."""
        w = getattr(self, which).weight
        key = ops.param_key(w) + (ldk,)
        ent = self._proj_w_cache.get(which)
        if ent is None or ent[0] != key:
            w2 = w.detach().reshape(w.shape[0], -1)  # [d, C*4], K index = c*4 + ph*2 + pw
            if w2.shape[1] != ldk:
                w2 = torch.nn.functional.pad(w2, (0, ldk - w2.shape[1]))
            ent = self._proj_w_cache[which] = (key, w2.contiguous())
        return ent[1]

    def _ref_pos_table(self, gh: int, gw: int) -> torch.Tensor:
        """transformer3d.py:1546-1553: the 2-D sin-cos table of the (post_patch_height x post_patch_width) training grid resized
        to this call's patch grid with F.interpolate(trilinear) -> [gh*gw, d] in the buffer's dtype.  A table like the RoPE
        one: depends on the grid size only, built once per size with the reference's own torch call and cached."""
        buf = self.ref_pos_embedding
        key = (gh, gw, buf.data_ptr(), buf.dtype)
        if self._ref_pos_cache is None or self._ref_pos_cache[0] != key:
            emb = buf.shape[-1]
            pe = buf.view(1, 1, self.post_patch_height, self.post_patch_width, emb).permute([0, 4, 1, 2, 3])
            pe = torch.nn.functional.interpolate(pe, size=[1, gh, gw], mode="trilinear", align_corners=False)
            self._ref_pos_cache = (key, pe.permute([0, 2, 3, 4, 1]).reshape(gh * gw, emb).contiguous())
        return self._ref_pos_cache[1]

    def _text_tokens(self, seq, enc: torch.Tensor) -> torch.Tensor:
        B, S_t, E = enc.shape
        x = enc.reshape(B * S_t, E).contiguous()
        if isinstance(seq, nn.Sequential):
            x = ops.rmsnorm(x, seq[0].weight, seq[0].variance_epsilon)
            lin = seq[1]
        else:
            lin = seq
        return ops.gemm(x, lin.weight, lin.bias)

    @torch.no_grad()
    def forward(
        self,
        hidden_states,
        timestep,
        timestep_cond=None,
        encoder_hidden_states: Optional[torch.Tensor] = None,
        text_embedding_mask: Optional[torch.Tensor] = None,
        encoder_hidden_states_t5: Optional[torch.Tensor] = None,
        text_embedding_mask_t5: Optional[torch.Tensor] = None,
        image_meta_size=None,
        style=None,
        image_rotary_emb: Optional[torch.Tensor] = None,
        inpaint_latents: Optional[torch.Tensor] = None,
        control_latents: Optional[torch.Tensor] = None,
        ref_latents: Optional[torch.Tensor] = None,
        clip_encoder_hidden_states: Optional[torch.Tensor] = None,
        clip_attention_mask: Optional[torch.Tensor] = None,
        added_cond_kwargs: Dict[str, torch.Tensor] = None,
        return_dict=True,
    ):
        fp8 = self.dtype == torch.float8_e4m3fn
        if self.dtype != bf16 and not fp8:
            raise L.EaError("easyanimate_b200 computes in bf16: call .to(torch.bfloat16) on the module first (or store the "
                            "weights as torch.float8_e4m3fn: they are expanded to bf16 block by block)")
        off = self._offload
        if off is not None:
            off.start()  # before the staging: it puts the non-block parameters back on the device if they were moved
        staging = self._fp8_staging() if fp8 else None
        P = staging.head if fp8 else self  # owner of the non-block parameters the kernels read
        if timestep_cond is not None:
            raise NotImplementedError("timestep_cond is not used by any v5.1 pipeline (TimestepEmbedding is built without cond_proj)")
        if clip_encoder_hidden_states is not None and ref_latents is None:
            raise ValueError("clip_encoder_hidden_states needs ref_latents (the reference concatenates the two, transformer3d.py:1561)")
        B, C, F, H, W = hidden_states.shape
        d, p = self.inner_dim, self.patch_size
        dev = hidden_states.device

        # 1. time embedding (transformer3d.py:1519-1520)
        t = timestep.to(device=dev, dtype=bf16).reshape(-1)
        if t.numel() == 1 and B > 1:
            t = t.expand(B).contiguous()
        temb_in = ops.timestep_embedding(t.contiguous(), d, self.config.flip_sin_to_cos, float(self.config.freq_shift))
        te = P.time_embedding
        temb = ops.skinny_linear(temb_in, te.linear_1.weight, te.linear_1.bias)
        temb = ops.skinny_linear(temb, te.linear_2.weight, te.linear_2.bias, act_in=1)  # [B, time_embed_dim]

        # 2. patch embedding (transformer3d.py:1523-1531): channel concat + 2x2 patchify + GEMM
        extra = inpaint_latents
        if control_latents is not None:
            extra = control_latents if extra is None else torch.cat([extra, control_latents], 1)
        a = ops.patchify(hidden_states.to(bf16), None if extra is None else extra.to(bf16))
        x_v = ops.gemm(a, P._patch_weight(a.shape[1]), P.proj.bias)  # [B*S_v, d]
        S_v = F * (H // p) * (W // p)

        # 3. text tokens (transformer3d.py:1533-1536)
        x_t = self._text_tokens(P.text_proj, encoder_hidden_states.to(bf16))
        S_t = encoder_hidden_states.shape[1]
        if encoder_hidden_states_t5 is not None:
            x_t5 = self._text_tokens(P.text_proj_t5, encoder_hidden_states_t5.to(bf16))
            S_t5 = encoder_hidden_states_t5.shape[1]
            x_t = torch.cat([x_t.view(B, S_t, d), x_t5.view(B, S_t5, d)], dim=1).reshape(B * (S_t + S_t5), d).contiguous()
            S_t += S_t5

        # 3b. v5.1 Control: reference-image tokens REPLACE the text tokens, CLIP tokens go in front (transformer3d.py:1538-1561)
        if ref_latents is not None:
            if ref_latents.shape[2] != 1 or tuple(ref_latents.shape[3:]) != (H, W):
                raise ValueError("ref_latents must be one latent frame of the video's size (the reference adds a [1, h*w, d] "
                                 "position table to them, transformer3d.py:1554)")
            ar = ops.patchify(ref_latents.to(bf16))
            r = ops.gemm(ar, P._patch_weight(ar.shape[1], "ref_proj"), P.ref_proj.bias)  # [B*hw, d]
            pe = P._ref_pos_table(H // p, W // p).to(bf16)
            x_t = ops.ew_add(r, pe.unsqueeze(0).expand(B, -1, -1).reshape(r.shape).contiguous())
            S_t = (H // p) * (W // p)
            if clip_encoder_hidden_states is not None:
                S_c = clip_encoder_hidden_states.shape[1]
                c = ops.gemm(clip_encoder_hidden_states.to(bf16).reshape(B * S_c, -1).contiguous(), P.clip_proj.weight, P.clip_proj.bias)
                x_t = torch.cat([c.view(B, S_c, d), x_t.view(B, S_t, d)], dim=1).reshape(B * (S_c + S_t), d).contiguous()
                S_t += S_c

        rope = None
        if image_rotary_emb is not None:
            cos, sin = image_rotary_emb
            rope = (cos.to(device=dev, dtype=torch.float32).contiguous(), sin.to(device=dev, dtype=torch.float32).contiguous())

        # sequence parallelism: from here to the output projection every rank works on its slice of the video tokens
        sp = self.sequence_parallel
        S_v_full = S_v
        if sp is not None:
            s0, s1 = sp.local_range(S_v)
            x_v = sp.shard_tokens(x_v, B, S_v)
            if rope is not None:
                rope = (rope[0][s0:s1].contiguous(), rope[1][s0:s1].contiguous())
            S_v = s1 - s0

        # 4. transformer blocks (transformer3d.py:1639-1671)
        ff_inner = self.transformer_blocks[0].ff.net[2].weight.shape[1] if len(self.transformer_blocks) else 4 * d
        # TeaCache decision (transformer3d.py:1563-1586): relative-L1 change of block 0's modulated video input
        tc = self.teacache
        should_calc = True
        if tc is not None:
            if off is not None:
                blk0 = off.block(0, staging)
            else:
                blk0 = staging.block(self.transformer_blocks[0]) if fp8 else self.transformer_blocks[0]
            mod0 = ops.skinny_linear(temb, blk0.norm1.linear.weight, blk0.norm1.linear.bias, act_in=1)
            modulated = EasyAnimateDiTBlock._ln_mod(x_v, blk0.norm1, mod0, 0, S_v)
            if tc.cnt == 0 or tc.cnt == tc.num_steps - 1:
                tc.accumulated_rel_l1_distance = 0
            else:
                # the decision must be the reference's (one per step, from the means over ALL tokens of BOTH CFG branches)
                # and the same on every rank: the additive pieces are summed over the ranks of this video (none on one GPU)
                from .sequence_parallel import all_reduce_floats, group_size
                groups = [g for g in ((sp.group if sp is not None else None), self.cfg_parallel_group) if g is not None]
                num, den = ops.l1_sums(modulated, tc.previous_modulated_input)
                n = modulated.numel()
                for g in groups:
                    num, den = all_reduce_floats((num, den), g)
                    n *= group_size(g)
                dist = ops.rel_l1_from_sums(num, den, n)
                tc.accumulated_rel_l1_distance += tc.rescale_func(dist)
                if tc.accumulated_rel_l1_distance < tc.rel_l1_thresh:
                    should_calc = False
                else:
                    tc.accumulated_rel_l1_distance = 0
            tc.previous_modulated_input = modulated
            tc.cnt += 1
            if tc.cnt == tc.num_steps:
                tc.reset()

        if not should_calc:
            # transformer3d.py:1589-1590: reuse the cached residual; the reference skips the final norms on this path
            tc.skipped += 1
            y = ops.ew_add(x_v, tc.previous_residual)
        else:
            ori = x_v.clone() if tc is not None else None  # (device copy; the blocks update x_v in place)
            ws = _Workspace(B, S_v, S_t, d, self.num_heads, ff_inner, dev, sp=sp)
            for i, block in enumerate(self.transformer_blocks):
                if off is not None:
                    x_v, x_t = off.block(i, staging)(x_v, x_t, temb, rope, ws)
                    off.release(i)
                else:
                    x_v, x_t = (staging.block(block) if fp8 else block)(x_v, x_t, temb, rope, ws)

            # 5. final norms + projection (transformer3d.py:1673-1680): norm_final is row-wise, so the text rows that
            #    the reference concatenates and then drops never need to be computed.
            mod = ops.skinny_linear(temb, P.norm_out.linear.weight, P.norm_out.linear.bias, act_in=1)  # shift|scale
            y = ops.layernorm_modulate(x_v, P.norm_out.norm.weight, P.norm_out.norm.bias, P.norm_out.norm.eps,
                                       shift=mod[:, :d], scale=mod[:, d:], rows_per_batch=S_v,
                                       pre=(P.norm_final.weight, P.norm_final.bias, P.norm_final.eps), out=ws.n_v)
            if tc is not None:
                tc.previous_residual = ops.ew_add(y, ori, subtract=True)  # transformer3d.py:1634
        z = ops.gemm(y, P.proj_out.weight, P.proj_out.bias)  # [B*S_v, p*p*C_out]
        if sp is not None:
            z = sp.gather_tokens(z, B, S_v)  # every rank gets all S_v_full tokens back
            assert z.shape[0] == B * S_v_full

        # 6. unpatchify (transformer3d.py:1683-1685); like the reference, the output channel count is taken from the
        #    input latent (`channels`), which equals out_channels for every released model.
        output = ops.unpatchify(z, B, C, F, H, W)
        if not return_dict:
            return (output,)
        return Transformer2DModelOutput(sample=output)

    # ----------------------------------------------------------------------------------------------------------
    @classmethod
    def from_pretrained_2d(cls, pretrained_model_path, subfolder=None, transformer_additional_kwargs={},
                           low_cpu_mem_usage=False, torch_dtype=torch.bfloat16):
        """transformer3d.py:1692-1809: config.json + safetensors/bin, `proj.weight` channel-resize shim, skip of
        shape-mismatched tensors, strict=False load."""
        if subfolder is not None:
            pretrained_model_path = os.path.join(pretrained_model_path, subfolder)
        config = cls.load_config(pretrained_model_path)
        model = cls.from_config(config, **dict(transformer_additional_kwargs))
        state_dict = load_state_dict_from_dir(pretrained_model_path)
        own = model.state_dict()
        if "proj.weight" in state_dict and state_dict["proj.weight"].shape != own["proj.weight"].shape:
            new = own["proj.weight"].clone()
            src = state_dict["proj.weight"]
            if own["proj.weight"].shape[1] > src.shape[1]:
                new[:, :src.shape[1]] = src
                new[:, src.shape[1]:] = 0
            else:
                new = src[:, :own["proj.weight"].shape[1]].clone()
            state_dict["proj.weight"] = new
        filtered = {k: v for k, v in state_dict.items() if k in own and own[k].shape == v.shape}
        model.load_state_dict(filtered, strict=False)
        return model.to(torch_dtype)

"""ctypes binding of libea_b200.so (the C ABI declared in include/ea_b200.h).

The library is built in-tree by ``easyanimate_b200/csrc/build.sh`` (``__graft_entry__.build()``).  There is no
CPU or PyTorch fallback: if the shared object is missing the import of any product module fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libea_b200.so")


class EaError(RuntimeError):
    pass


def _load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()'"
            " or easyanimate_b200/csrc/build.sh). easyanimate_b200 has no CPU/PyTorch fallback."
        )
    return C.CDLL(LIB_PATH)


lib = _load()

i64, i32, f32, vp = C.c_int64, C.c_int32, C.c_float, C.c_void_p

# epilogues (keep in sync with include/ea_b200.h)
EPI_BIAS, EPI_BIAS_GELU, EPI_BIAS_GATE_RES, EPI_SCALE_F32, EPI_BIAS_RES = 0, 1, 2, 3, 4
FRAMES_F32, FRAMES_U8 = 0, 1
ABI_VERSION = 4


class GemmArgs(C.Structure):
    _fields_ = [
        ("a", vp), ("w", vp), ("bias", vp), ("out", vp),
        ("M", i64), ("N", i64), ("K", i64),
        ("lda", i64), ("ldw", i64), ("ldo", i64),
        ("epilogue", i32), ("scale", f32),
        ("residual", vp), ("ldr", i64),
        ("gate", vp), ("gate_stride", i64), ("rows_per_batch", i64),
    ]


MAX_PEERS = 8


class QkvPeers(C.Structure):
    _fields_ = [("q", vp * MAX_PEERS), ("k", vp * MAX_PEERS), ("v", vp * MAX_PEERS), ("heads_per_peer", i64)]


class AttnPeers(C.Structure):
    _fields_ = [("out_video", vp * MAX_PEERS), ("out_text", vp * MAX_PEERS), ("n_peers", i64), ("tokens_per_peer", i64),
                ("out_heads", i64), ("head0", i64)]


class QkvArgs(C.Structure):
    _fields_ = [
        ("a", vp), ("w", vp), ("bias", vp),
        ("ln_q_w", vp), ("ln_q_b", vp), ("ln_k_w", vp), ("ln_k_b", vp),
        ("rope_cos", vp), ("rope_sin", vp),
        ("q", vp), ("k", vp), ("v", vp),
        ("M", i64), ("d", i64), ("lda", i64),
        ("rows_per_batch", i64), ("S", i64), ("seq_offset", i64),
        ("ln_eps", f32), ("peers", C.POINTER(QkvPeers)),
    ]


class SkinnyArgs(C.Structure):
    _fields_ = [
        ("x", vp), ("w", vp), ("bias", vp), ("out", vp),
        ("M", i64), ("N", i64), ("K", i64),
        ("act_in", i32), ("act_out", i32),
    ]


class LnArgs(C.Structure):
    _fields_ = [
        ("x", vp), ("y", vp),
        ("rows", i64), ("d", i64), ("ldx", i64), ("ldy", i64), ("rows_per_batch", i64),
        ("pre_w", vp), ("pre_b", vp), ("pre_eps", f32),
        ("w", vp), ("b", vp), ("eps", f32),
        ("shift", vp), ("scale", vp), ("mod_stride", i64),
    ]


class RmsArgs(C.Structure):
    _fields_ = [("x", vp), ("y", vp), ("w", vp), ("rows", i64), ("d", i64), ("eps", f32)]


class AttnArgs(C.Structure):
    _fields_ = [
        ("q", vp), ("k", vp), ("v", vp),
        ("out_text", vp), ("out_video", vp),
        ("B", i64), ("H", i64), ("S", i64), ("S_text", i64), ("S_pad", i64), ("head_dim", i64),
        ("scale", f32), ("variant", i32), ("peers", C.POINTER(AttnPeers)),
    ]


MAX_E4M3_SEGMENTS = 64
LORA_W_BF16, LORA_W_E4M3 = 0, 1
LORA_C_BF16, LORA_C_F32 = 0, 1


class ConvArgs(C.Structure):
    _fields_ = [
        ("x", vp), ("w", vp), ("bias", vp), ("residual", vp), ("out", vp),
        ("T", i64), ("H", i64), ("W", i64), ("Cin", i64), ("Cout", i64), ("Cout_pad", i64),
        ("dup_frames", i32), ("out_planar", i32), ("variant", i32), ("stride_t", i32), ("stride_hw", i32),
        ("out_row0", i32), ("out_rows", i32),
    ]


def _sig(name, argtypes, restype=C.c_int):
    fn = getattr(lib, name)
    fn.argtypes = argtypes
    fn.restype = restype
    return fn


ea_last_error = _sig("ea_last_error", [], C.c_char_p)
ea_abi_version = _sig("ea_abi_version", [])
ea_launch_count = _sig("ea_launch_count", [], C.c_uint64)
ea_gemm = _sig("ea_gemm", [C.POINTER(GemmArgs), vp])
ea_qkv_gemm_ln_rope = _sig("ea_qkv_gemm_ln_rope", [C.POINTER(QkvArgs), vp])
ea_skinny_linear = _sig("ea_skinny_linear", [C.POINTER(SkinnyArgs), vp])
ea_layernorm_modulate = _sig("ea_layernorm_modulate", [C.POINTER(LnArgs), vp])
ea_rmsnorm = _sig("ea_rmsnorm", [C.POINTER(RmsArgs), vp])
ea_timestep_embedding = _sig("ea_timestep_embedding", [vp, vp, i64, i64, f32, i32, vp])
ea_patchify = _sig("ea_patchify", [vp, vp, vp, i64, i64, i64, i64, i64, i64, i64, vp])
ea_unpatchify = _sig("ea_unpatchify", [vp, vp, i64, i64, i64, i64, i64, i64, vp])
ea_attn_fwd = _sig("ea_attn_fwd", [C.POINTER(AttnArgs), vp])
ea_attn_generations = _sig("ea_attn_generations", [])
ea_enable_peer_access = _sig("ea_enable_peer_access", [i32])
ea_cfg_euler_step = _sig("ea_cfg_euler_step", [vp, vp, vp, vp, i64, f32, i32, f32, f32, vp])
ea_l1_sums = _sig("ea_l1_sums", [vp, vp, vp, i64, vp])
ea_ew_addsub = _sig("ea_ew_addsub", [vp, vp, vp, i64, i32, vp])
ea_dequant_e4m3 = _sig("ea_dequant_e4m3", [vp, vp, i64, vp])
ea_h2d_block = _sig("ea_h2d_block", [vp, vp, i64, vp, vp, vp])
ea_expand_e4m3_segments = _sig("ea_expand_e4m3_segments", [vp, C.POINTER(i64), C.POINTER(vp), C.POINTER(i64), i32, vp])
ea_lora_merge = _sig("ea_lora_merge", [vp, vp, vp, i64, i64, i64, i64, i64, i64, f32, i32, i32, vp])
ea_ipc_export = _sig("ea_ipc_export", [vp, vp, C.POINTER(i64)])
ea_ipc_open = _sig("ea_ipc_open", [vp, C.POINTER(vp)])
ea_ipc_close = _sig("ea_ipc_close", [vp])
ea_conv3d_causal = _sig("ea_conv3d_causal", [C.POINTER(ConvArgs), vp])
ea_vae_prepare_latents = _sig("ea_vae_prepare_latents", [vp, vp, vp, vp, i64, i64, i64, i64, i64, f32, vp])
ea_frames_out = _sig("ea_frames_out", [vp, vp, i64, i32, vp])
ea_frames_out_blend = _sig("ea_frames_out_blend", [vp, vp, i64, i64, i64, i64, i32, vp])
ea_groupnorm_workspace = _sig("ea_groupnorm_workspace", [i64, i64, i64], C.c_size_t)
ea_groupnorm_stats = _sig("ea_groupnorm_stats", [vp, vp, vp, C.c_size_t, i64, i64, i64, i64, i64, f32, vp])
ea_groupnorm_sums = _sig("ea_groupnorm_sums", [vp, vp, vp, C.c_size_t, i64, i64, i64, i64, i64, vp])
ea_groupnorm_finalize = _sig("ea_groupnorm_finalize", [vp, vp, i64, i64, i64, C.c_double, f32, vp])
ea_groupnorm_apply = _sig("ea_groupnorm_apply", [vp, vp, vp, vp, vp, i64, i64, i64, i64, i32, vp])
ea_upsample2x = _sig("ea_upsample2x", [vp, vp, i64, i64, i64, i64, vp])
ea_softmax_rows = _sig("ea_softmax_rows", [vp, vp, i64, i64, i64, i64, vp])
ea_transpose2d = _sig("ea_transpose2d", [vp, vp, i64, i64, i64, i64, vp])
ea_tile_blend = _sig("ea_tile_blend", [vp, i64, i64, i64, i64, vp, i64, i64, i64, i64, i64, i64, i32, vp])
ea_copy2d = _sig("ea_copy2d", [vp, i64, i64, vp, i64, i64, i64, i64, i64, vp])
ea_corner_blend = _sig("ea_corner_blend", [vp, vp, i64, i64, i64, i64, i64, vp])


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = ea_last_error()
        raise EaError(f"{what} failed ({rc}): {msg.decode() if msg else '?'}")

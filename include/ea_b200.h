/*
 * libea_b200.so — C ABI of the H100-native (sm_90a) kernels behind EasyAnimateV5.1's sampling hot path.
 *
 * The reference (aigc-apps/EasyAnimate @ c2a70d1) is 100 % Python: its "operator interface" for this path is the
 * list of torch library calls made by EasyAnimateTransformer3DModel.forward (easyanimate/models/transformer3d.py:1496-1689),
 * EasyAnimateDiTBlock.forward (easyanimate/models/attention.py:1107-1163), EasyAnimateAttnProcessor2_0.__call__
 * (easyanimate/models/processor.py:218-312), EasyAnimateLayerNormZero.forward (easyanimate/models/norm.py:160-166)
 * and AutoencoderKLMagvit.decode (easyanimate/models/autoencoder_magvit.py:271-317, 381-448) /
 * Decoder.forward (easyanimate/vae/ldm/models/omnigen_enc_dec.py:555-677).  Each entry point below names the
 * reference call sites it replaces.
 *
 * Conventions
 *  - every function only ENQUEUES work on `stream` (a cudaStream_t passed as void*): no allocation, no
 *    synchronisation, no global state; safe to capture in a CUDA graph.
 *  - all pointers are device pointers unless stated otherwise; activations/weights are bf16 unless stated.
 *  - return value 0 = ok, negative = error; `ea_last_error()` returns a thread-local message.
 *  - no torch types cross this boundary.
 */
#ifndef EA_B200_H_
#define EA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EA_OK 0
#define EA_ERR_INVALID (-1)
#define EA_ERR_CUDA (-2)
#define EA_ERR_WORKSPACE (-3)

const char* ea_last_error(void);
int ea_abi_version(void);
/* number of kernels launched through this library since load (bench.py's gpu_launches counter) */
uint64_t ea_launch_count(void);

/* ------------------------------------------------------------------------------------------------------------
 * Dense contraction on wgmma tensor cores:  out[M,N] = epilogue(A[M,K] · W[N,K]^T + bias[N])
 * Replaces every nn.Linear on the path (F.linear -> cuBLAS in the reference): processor.py:244-246,261-263,303-311
 * (q/k/v/out projections), diffusers FeedForward built at attention.py:1082-1100 (net.0.proj, net.2),
 * transformer3d.py:1402-1404 (patch-embed Conv2d == GEMM over 2x2 patches), :1410-1413 (text_proj Linear),
 * :1680 (proj_out); VAE 1x1x1 convs (autoencoder_magvit.py:182,281; common.py:291-294) and the VAE
 * mid-block attention projections (attention_processors.py:105-131).
 * A, W are K-major bf16 (row strides lda/ldw in elements, multiples of 8). fp32 accumulation in registers (wgmma).
 * ------------------------------------------------------------------------------------------------------------ */
enum {
  EA_EPI_BIAS = 0,          /* out = bf16(acc + bias)                                                       */
  EA_EPI_BIAS_GELU = 1,     /* out = bf16(gelu_tanh(bf16(acc + bias)))            (FeedForward net.0)       */
  EA_EPI_BIAS_GATE_RES = 2, /* out = bf16(res + bf16(gate[b] * bf16(acc + bias))) (attention.py:1140-41,1161-62) */
  EA_EPI_SCALE_F32 = 3,     /* out(fp32) = scale * acc                            (VAE attention scores)    */
  EA_EPI_BIAS_RES = 4,      /* out = bf16(bf16(acc + bias) + res)                 (VAE shortcut / attn residual) */
};

typedef struct {
  const void* a;        /* [M,K] bf16 */
  const void* w;        /* [N,K] bf16 */
  const void* bias;     /* [N] bf16 or NULL */
  void* out;            /* [M,N] bf16 (fp32 for EA_EPI_SCALE_F32) */
  int64_t M, N, K;
  int64_t lda, ldw, ldo;
  int32_t epilogue;
  float scale;            /* EA_EPI_SCALE_F32 */
  const void* residual;   /* [M,N] bf16, row stride ldr (GATE_RES, BIAS_RES) */
  int64_t ldr;
  const void* gate;       /* [batch, N] bf16, row stride gate_stride; batch = row / rows_per_batch (GATE_RES) */
  int64_t gate_stride;
  int64_t rows_per_batch;
} ea_gemm_args;

int ea_gemm(const ea_gemm_args* args, void* stream);

/* Fused Q/K/V projection: A[M,d] · Wqkv[3d,d]^T + bias, then per-head LayerNorm(64) on q,k (affine, eps),
 * 3-D RoPE on q,k for video rows, written head-major into q/k/v[B,H,S,64] at sequence offset seq_offset.
 * Replaces processor.py:244-285 (to_q/to_k/to_v, view/transpose, norm_q/norm_k, cat, apply_rotary_emb).
 * M = B * rows_per_batch (rows_per_batch = S_text or S_video). d = H*64. */
/* Sequence parallelism for ONE video over up to EA_MAX_PEERS GPUs of a node (no counterpart in the reference, which has
 * no multi-GPU inference path: the two exchanges joint attention needs per block (processor.py:287-289
 * sees every token of every head) are FUSED into the kernels on either side of it.  Each GPU projects q/k/v for its slice
 * of the video tokens and all heads; head h of those rows is stored by the projection's epilogue directly into the q/k/v
 * buffer [B, heads_per_peer, S, 64] of the GPU that owns head h (entry h / heads_per_peer: this GPU's own buffer or a
 * peer's buffer mapped through CUDA IPC - the store then travels over NVLink).  NULL entries are skipped (the replicated
 * text rows are projected on every GPU for its own heads only). */
#define EA_MAX_PEERS 8
typedef struct {
  void* q[EA_MAX_PEERS];
  void* k[EA_MAX_PEERS];
  void* v[EA_MAX_PEERS];
  int64_t heads_per_peer;
} ea_qkv_peers;

typedef struct {
  const void* a;          /* [M,d] bf16, row stride lda */
  const void* w;          /* [3d,d] bf16: rows [0,d)=to_q, [d,2d)=to_k, [2d,3d)=to_v */
  const void* bias;       /* [3d] bf16 */
  const void* ln_q_w;     /* [64] bf16 (norm_q.weight) */
  const void* ln_q_b;
  const void* ln_k_w;
  const void* ln_k_b;
  const float* rope_cos;  /* [rows_per_batch,64] fp32 or NULL (text rows: no RoPE) */
  const float* rope_sin;
  void* q;                /* [B,H,S,64] bf16 */
  void* k;
  void* v;
  int64_t M, d, lda;
  int64_t rows_per_batch; /* S_part */
  int64_t S;              /* total sequence length of q/k/v */
  int64_t seq_offset;     /* where this part's rows start inside S */
  float ln_eps;
  const ea_qkv_peers* peers; /* NULL: q/k/v above hold all d/64 heads; else see ea_qkv_peers (q/k/v are then ignored) */
} ea_qkv_args;

int ea_qkv_gemm_ln_rope(const ea_qkv_args* args, void* stream);

/* Small-M linear (M <= 8), one warp per output feature: out[M,N] = act(x)[M,K] · W[N,K]^T + bias.
 * Replaces norm.py:163 (Linear(512->6d) on SiLU(temb)), diffusers AdaLayerNorm linear (transformer3d.py:1472-1478),
 * TimestepEmbedding linear_1/linear_2 (transformer3d.py:1399-1400,1519-1520).
 * act_in: 0 none, 1 SiLU on the input; act_out: 0 none, 1 SiLU on the output (both with bf16 rounding points
 * matching the reference's op-by-op bf16 execution). */
typedef struct {
  const void* x;    /* [M,K] bf16 */
  const void* w;    /* [N,K] bf16 */
  const void* bias; /* [N] bf16 or NULL */
  void* out;        /* [M,N] bf16 */
  int64_t M, N, K;
  int32_t act_in, act_out;
} ea_skinny_linear_args;

int ea_skinny_linear(const ea_skinny_linear_args* args, void* stream);

/* y = [modulate]( LN( [LN_pre](x) ) ): row-wise LayerNorm over d with fp32 statistics, bf16 output, optionally
 * preceded by a first affine LayerNorm and followed by AdaLN modulation y*(1+scale[b])+shift[b].
 * Replaces EasyAnimateLayerNormZero.forward (norm.py:160-166, FP32LayerNorm norm.py:16-26) for both streams, and the
 * tail transformer3d.py:1673-1678 (norm_final -> norm_out AdaLayerNorm) with pre_* = norm_final. */
typedef struct {
  const void* x;
  void* y;
  int64_t rows, d, ldx, ldy;
  int64_t rows_per_batch; /* batch index of a row = row / rows_per_batch (selects the shift/scale row) */
  const void* pre_w;      /* optional first LayerNorm affine [d] (NULL = skip) */
  const void* pre_b;
  float pre_eps;
  const void* w;          /* LayerNorm affine [d] or NULL */
  const void* b;
  float eps;
  const void* shift;      /* [B, mod_stride] bf16 or NULL */
  const void* scale;
  int64_t mod_stride;
} ea_ln_args;

int ea_layernorm_modulate(const ea_ln_args* args, void* stream);

/* EasyAnimateRMSNorm (norm.py:28-39): y = w * bf16(x * rsqrt(mean(x^2) + eps)) */
typedef struct {
  const void* x;
  void* y;
  const void* w;
  int64_t rows, d;
  float eps;
} ea_rmsnorm_args;

int ea_rmsnorm(const ea_rmsnorm_args* args, void* stream);

/* diffusers Timesteps(dim, flip_sin_to_cos, freq_shift) on a bf16 timestep vector t[B] -> out[B,dim] bf16
 * (transformer3d.py:1399,1519; the pipeline rounds t to bf16 first, pipeline_easyanimate.py:1079-1081). */
int ea_timestep_embedding(const void* t, void* out, int64_t B, int64_t dim, float freq_shift,
                          int32_t flip_sin_to_cos, void* stream);

/* Patch-embed im2col for kernel=stride=2 (transformer3d.py:1523-1531): A[(b,f,hh,ww), c*4+ph*2+pw] =
 * cat(x[B,C1,F,H,W], x2[B,C2,F,H,W])[b,c,f,2hh+ph,2ww+pw]; row stride ldk (columns >= 4(C1+C2) zero-filled). */
int ea_patchify(const void* x, const void* x2, void* a, int64_t B, int64_t C1, int64_t C2, int64_t F, int64_t H,
                int64_t W, int64_t ldk, void* stream);

/* Unpatchify (transformer3d.py:1683-1685): out[B,C,F,H,W] from y[(b,f,hh,ww), c*4+ph*2+pw], row stride ldy. */
int ea_unpatchify(const void* y, void* out, int64_t B, int64_t C, int64_t F, int64_t H, int64_t W, int64_t ldy,
                  void* stream);

/* Classifier-free-guidance combine + FlowMatchEuler step (pipeline_easyanimate.py:1102-1111; diffusers
 * FlowMatchEulerDiscreteScheduler.step): v = u + g*(c-u); x_out = bf16(float(x) + bf16(bf16(sigma_next-sigma)*v)).
 * n elements (even). use_cfg=0: v = pred_uncond. */
int ea_cfg_euler_step(const void* pred_uncond, const void* pred_text, const void* x, void* x_out, int64_t n,
                      float guidance_scale, int32_t use_cfg, float sigma, float sigma_next, void* stream);

/* TeaCache support (transformer3d.py:90-121 `compute_rel_l1_distance`, :1563-1636): sums[0] = sum |bf16(cur-prev)|,
 * sums[1] = sum |prev| (two doubles on the device, zeroed by the call); and out = a +/- b elementwise in bf16
 * (cached-residual add at :1590, residual capture at :1634). n even. */
int ea_l1_sums(const void* cur, const void* prev, void* sums, int64_t n, void* stream);
int ea_ew_addsub(const void* a, const void* b, void* out, int64_t n, int32_t subtract, void* stream);

/* fp8 weight storage (the reference's "model_cpu_offload_and_qfloat8" mode: predict_t2v.py:37,106 loads the transformer with
 * torch_dtype=float8_e4m3fn and utils/fp8_optimization.py:6-35 casts each module to bf16 around its forward): parameters stay
 * e4m3 in HBM (half the bytes) and are expanded to bf16 - exactly, every e4m3 value is a bf16 value - into a scratch buffer
 * right before the kernels that consume them.  n elements; both pointers 16-byte aligned. */
int ea_dequant_e4m3(const void* w8, void* w16, int64_t n, void* stream);

/* Sequential CPU offload (the reference's `sequential_cpu_offload` GPU_memory_mode, predict_t2v.py:256-265): the MMDiT's
 * blocks live packed in pinned host memory and are streamed through a ring of device slots while the previous block computes.
 *
 * ea_h2d_block enqueues on `copy_stream`: wait for `wait_event` (recorded by the caller on the compute stream after the
 * slot's previous reader; NULL = none), copy `bytes` from the PINNED host buffer `src_host` into the device slot `dst`, record
 * `done_event` (the compute stream waits on it before reading the slot).  Events are cudaEvent_t created by the caller. */
int ea_h2d_block(void* dst, const void* src_host, int64_t bytes, void* wait_event, void* done_event, void* copy_stream);

/* One launch expands a packed e4m3 block slot into its bf16 staging parameters: segment s turns counts[s] weights at
 * src + src_offsets[s] (bytes) into bf16 at dsts[s], bit-identical to ea_dequant_e4m3.  The three segment arrays are HOST
 * arrays of n_segs <= EA_MAX_E4M3_SEGMENTS entries, read during the call; src, every offset and every dst 16-byte aligned. */
#define EA_MAX_E4M3_SEGMENTS 64
int ea_expand_e4m3_segments(const void* src, const int64_t* src_offsets, void* const* dsts, const int64_t* counts,
                            int32_t n_segs, void* stream);

/* LoRA merge (the reference's merge_lora / unmerge_lora, utils/lora_utils.py:424-430,486-492: the layer cast to the merge
 * dtype c, W += multiplier * alpha * mm(up, down), cast back): W[rows, cols] += scale * up[rows, rank] · down[rank, cols] in
 * place, in W's own storage.  up and down are in c (EA_LORA_C_*).  Per element, with rnd_c the rounding to c (none for fp32):
 *   acc = fp32 FMA chain over k = 0 .. rank-1 in ascending order, starting from +0.0 (CUDA cores, no tensor cores)
 *   d = rnd_c(acc);  d2 = rnd_c(fp32(scale * d));  w = rnd_c(fp32(W + d2));  W = storage(w)
 * storage: bf16 round to nearest even, or float8_e4m3fn exactly as torch's .to(float8_e4m3fn) (nearest even, a magnitude
 * rounding past 448 becomes NaN, no saturation).  Unmerge is the same call with -scale.  Strides in elements. */
enum { EA_LORA_W_BF16 = 0, EA_LORA_W_E4M3 = 1 };
enum { EA_LORA_C_BF16 = 0, EA_LORA_C_F32 = 1 };
/* w [rows, cols] row stride ldw, updated in place; up [rows, rank] row stride ldu; down [rank, cols] row stride ldd.
 * scale: multiplier * alpha / rank rounded to fp32, negative for unmerge.  w_kind: EA_LORA_W_BF16 | EA_LORA_W_E4M3.
 * compute: EA_LORA_C_BF16 | EA_LORA_C_F32, the dtype of up / down and of the rounding points. */
int ea_lora_merge(void* w, const void* up, const void* down, int64_t rows, int64_t cols, int64_t rank, int64_t ldw,
                  int64_t ldu, int64_t ldd, float scale, int32_t w_kind, int32_t compute, void* stream);

/* Joint text+video self-attention, non-causal, no mask, head_dim 64:  O = softmax(Q K^T * scale) V.
 * Replaces F.scaled_dot_product_attention + transpose/reshape/split at processor.py:287-303.
 * q,k,v: [B,H,S,64] bf16 contiguous.  Output is token-major and split at S_text:
 * out_text[B,S_text,H*64], out_video[B,S-S_text,H*64].
 * variant: kept for ABI compatibility.  Any value with (variant & 0x1100) == 0x100 (the sixth-generation codes 0x1?c, 0x2?c,
 * 0x9?c, ...; the Python layer passes 0x217c) runs the one kernel: a 128-row query tile per CTA, 128-key blocks, wgmma for
 * Q K^T and P V, online softmax in registers, P rounded to bf16.  The remaining bits no longer select anything.  Other values
 * are EA_ERR_INVALID; ea_attn_generations() returns 1 << 6. */
/* The return half of the exchange, fused into the attention epilogue: this GPU ran attention for heads
 * [head0, head0 + H) of out_heads over ALL S tokens; the row of video token v goes into out_video[v / tokens_per_peer]
 * (the token-major [B, tokens_per_peer, out_heads*64] buffer of the GPU that owns the token), text rows into the
 * [B, S_text, out_heads*64] buffer of EVERY GPU (the text stream is replicated). */
typedef struct {
  void* out_video[EA_MAX_PEERS];
  void* out_text[EA_MAX_PEERS];
  int64_t n_peers, tokens_per_peer, out_heads, head0;
} ea_attn_peers;

typedef struct {
  const void* q;
  const void* k;
  const void* v;
  void* out_text;
  void* out_video;
  int64_t B, H, S, S_text, S_pad, head_dim;
  float scale;
  int32_t variant;
  const ea_attn_peers* peers; /* NULL: out_text / out_video above; else see ea_attn_peers (they are then ignored) */
} ea_attn_args;

int ea_attn_fwd(const ea_attn_args* args, void* stream);
int ea_attn_generations(void);

/* cudaDeviceEnablePeerAccess(peer_device) from the current device (idempotent): kernels of this library on the current
 * device may then dereference pointers into `peer_device`'s memory (ea_qkv_peers / ea_attn_peers buffers). */
int ea_enable_peer_access(int32_t peer_device);

/* Export a device buffer to the other processes of the node (the 64-byte cudaIpcMemHandle_t of the allocation that holds
 * `ptr`, and ptr's byte offset in it), and import one: */
/* Import a peer process's device allocation (a 64-byte cudaIpcMemHandle_t of its base) into the CURRENT device's context so
 * that kernels launched on the current device may store into it (cudaIpcOpenMemHandle with lazy peer access); base_out is
 * the mapped base address.  One open per handle and process; ea_ipc_close unmaps. */
int ea_ipc_export(const void* ptr, void* handle64_out, int64_t* offset_out); /* handle of the allocation holding ptr + ptr's offset */
int ea_ipc_open(const void* handle64, void** base_out);
int ea_ipc_close(void* base);

/* ------------------------------------------------------------------------------------------------------------
 * MagViT VAE decode (AutoencoderKLMagvit.decode, autoencoder_magvit.py:271-317,381-448; Decoder,
 * omnigen_enc_dec.py:555-677).  Activations are channels-last [T,H,W,C] bf16 for one batch element.
 * ------------------------------------------------------------------------------------------------------------ */

/* Whole-sequence causal 3x3x3 convolution (CausalConv3d.forward, vaemodules/common.py:84-141; temporal left
 * replicate padding 2, spatial zero padding 1) as an implicit GEMM on wgmma.
 *   x   [T,H,W,Cin]  bf16, Cin % 64 == 0
 *   w   [Cout_pad, 27*Cin] bf16, k = ((kt*3+kh)*3+kw)*Cin + ci  (rows >= Cout are zero)
 *   out [T',H,W,Cout] channels-last, or planar [Cout,T',H,W] when out_planar (conv_out);
 *       T' = 2T-1 when dup_frames (nearest temporal x2 of every frame but the first, upsamplers.py:146-152), else T
 *   residual (optional) [T,H,W,Cout]: out = bf16(bf16(conv + bias) + residual)   (ResidualBlock3D, common.py:323) */
typedef struct {
  const void* x;
  const void* w;
  const void* bias;     /* [Cout] bf16 */
  const void* residual; /* or NULL */
  void* out;
  int64_t T, H, W, Cin, Cout, Cout_pad;
  int32_t dup_frames;
  int32_t out_planar;
  int32_t variant;      /* historical tiling codes, accepted and ignored: every call runs the one sm_90a kernel (a TMA
                         * box of 128 pixels per tap and 64-channel slice, wgmma into 64 x Cout_tile register tiles) */
  /* Encoder down-sampling convolutions (downsamplers.py:24-96: F.pad(x, (0,1,0,1)) then CausalConv3d(stride=(s_t,2,2),
   * padding 0)): stride_hw = 2 -> out[t,i,j] reads input rows 2i..2i+2 / columns 2j..2j+2 (zeros past the bottom / right
   * edge), out is [T', H/2, W/2, Cout]; stride_t = 2 -> out frame t reads input frames 2t-2..2t (clamped at 0), T' = (T+1)/2.
   * 0 or 1 = unit stride.  Strided calls take no residual / dup_frames / out_planar. */
  int32_t stride_t, stride_hw;
  /* Output row window (strip-parallel decode): out_rows > 0 -> only output rows
   * [out_row0, out_row0 + out_rows) of the H input rows are computed and `out` / `residual` are [T', out_rows, W, Cout]
   * (planar: [Cout, T', out_rows, W]); the input then carries its neighbours' halo rows (or zeros at the frame edge) above
   * and below the window.  0 = all rows.  Unit stride only. */
  int32_t out_row0, out_rows;
} ea_conv3d_args;

int ea_conv3d_causal(const ea_conv3d_args* args, void* stream);

/* post_quant_conv (1x1x1, autoencoder_magvit.py:182,281) fused with NCTHW->THWC and with decode_latents'
 * `1 / scaling_factor * latents` (pipeline_easyanimate.py:724; in_scale = 1 leaves z untouched): z [C,T,H,W] planar ->
 * y [T,H,W,Cpad] = bf16(W * bf16(in_scale * z) + bias) (channels >= C zero). C <= 32. */
int ea_vae_prepare_latents(const void* z, const void* w, const void* bias, void* y, int64_t C, int64_t Cpad, int64_t T,
                           int64_t H, int64_t W, float in_scale, void* stream);

/* decode_latents' tail (pipeline_easyanimate.py:729,738-741): out = clamp(bf16(bf16(clamp(x,-1,1) / 2) + 0.5), 0, 1) over
 * n bf16 elements, written as float32 (what `.cpu().float().numpy()` returns) or as uint8 = trunc(255 * v)
 * (utils.py:57).  `out` is a device pointer OR a device-mapped pinned HOST pointer (cudaHostAlloc / torch pin_memory under
 * UVA): the frames then go straight to host memory without a device staging copy.  Both pointers 16-byte aligned. */
enum { EA_FRAMES_F32 = 0, EA_FRAMES_U8 = 1 };
int ea_frames_out(const void* x, void* out, int64_t n, int32_t out_kind, void* stream);

/* ea_frames_out (float32) fused with the long-video cross-fade (ui.py:524-531): x [planes, frames, frame_elems] bf16 is one
 * decoded window, and its frame t of plane p goes to dst + p * dst_plane + t * frame_elems (float32; the window's slice of
 * the whole video, a device pointer or a device-mapped pinned host pointer).  For t < ov, dst = dst * (1 - r) + f * r with
 * r = float32(t / ov), each product and sum rounded on its own like torch's float32 tensor ops; the other frames are
 * overwritten with f.  ov = 0 is a plain strided ea_frames_out.  planes * frames <= 65535, 0 <= ov <= frames. */
int ea_frames_out_blend(const void* x, void* dst, int64_t planes, int64_t frames, int64_t frame_elems, int64_t dst_plane,
                        int32_t ov, void* stream);

/* Per-frame GroupNorm (common.py:301-319 with set_3dgroupnorm; omnigen_enc_dec.py:603-609) of x [frames, rows, W, C]:
 * stats[frames,groups,2] = (mean, rstd) fp32; workspace = ea_groupnorm_workspace() bytes of scratch.  The statistics are
 * accumulated per image row and the rows added in fp64, so they do not depend on how a frame's rows are split over GPUs. */
size_t ea_groupnorm_workspace(int64_t frames, int64_t rows, int64_t groups);
int ea_groupnorm_stats(const void* x, void* stats, void* workspace, size_t workspace_bytes, int64_t frames, int64_t rows,
                       int64_t W, int64_t C, int64_t groups, float eps, void* stream);
/* y = [SiLU](bf16((x-mean)*rstd*gamma+beta)) */
/* Strip-parallel decode (one frame sequence split into row strips over several GPUs): the per-frame
 * GroupNorm statistics are global, so each GPU reduces ITS rows to (sum, sum of squares) per (frame, group) in fp64
 * [frames, groups, 2] (ea_groupnorm_sums; workspace as ea_groupnorm_stats), the pairs of all GPUs are gathered
 * [parts, frames, groups, 2] and added in rank order into the same mean / rstd on every GPU (ea_groupnorm_finalize; count =
 * pixels of the WHOLE frame x channels per group).  With parts = 1 the result equals ea_groupnorm_stats; with more parts
 * too: the per-row partial sums are the same and the fp64 association differences (~1e-16) vanish in the fp32 result. */
int ea_groupnorm_sums(const void* x, void* sums, void* workspace, size_t workspace_bytes, int64_t frames, int64_t rows, int64_t W,
                      int64_t C, int64_t groups, void* stream);
int ea_groupnorm_finalize(const void* sums, void* stats, int64_t parts, int64_t frames, int64_t groups, double count, float eps,
                          void* stream);
int ea_groupnorm_apply(const void* x, void* y, const void* gamma, const void* beta, const void* stats, int64_t frames,
                       int64_t HW, int64_t C, int64_t groups, int32_t silu, void* stream);

/* F.interpolate(scale_factor=(1,2,2), mode="nearest") (upsamplers.py:35,143): [T,H,W,C] -> [T,2H,2W,C] */
int ea_upsample2x(const void* x, void* y, int64_t T, int64_t H, int64_t W, int64_t C, void* stream);

/* mid-block SpatialAttention helpers (attention_processors.py:118-131): row softmax of fp32 scores -> bf16, and a
 * 2-D bf16 transpose (V^T as the K-major operand of P·V). */
int ea_softmax_rows(const void* s, void* p, int64_t M, int64_t N, int64_t lds, int64_t ldp, void* stream);
int ea_transpose2d(const void* in, void* out, int64_t R, int64_t C, int64_t ldi, int64_t ldo, void* stream);

/* tiled_decode blending (autoencoder_magvit.py:319-337,403-443) on planar [planes][H][W] images:
 * ea_tile_blend: b[r][c] = a[a_off_r+r][a_off_c+c]*(1-k/extent) + b[r][c]*(k/extent), k = r (axis 0) or c (axis 1)
 * ea_copy2d: strided crop/concat copy;
 * ea_corner_blend: dst[r][c] = w*src[r][c] + (1-w)*dst[r][c] with w = min(wx[c], wy[r]), every product and sum an fp32
 *   op of its own, bf16 on store.  wx [Wc] / wy [Hc] are fp32 device vectors holding torch.linspace(0, 1, N) as torch
 *   computes it on the CPU (autoencoder_magvit.py:430-431). */
int ea_tile_blend(const void* a, int64_t a_plane, int64_t a_ld, int64_t a_off_r, int64_t a_off_c, void* b,
                  int64_t b_plane, int64_t b_ld, int64_t planes, int64_t rows, int64_t cols, int64_t extent,
                  int32_t axis, void* stream);
int ea_copy2d(const void* src, int64_t s_plane, int64_t s_ld, void* dst, int64_t d_plane, int64_t d_ld, int64_t planes,
              int64_t rows, int64_t cols, void* stream);
int ea_corner_blend(const void* src, void* dst, int64_t d_plane, int64_t d_ld, int64_t planes, int64_t Hc, int64_t Wc,
                    const float* wx, const float* wy, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* EA_B200_H_ */

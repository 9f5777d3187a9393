// Persistent, warp-specialised wgmma GEMM for sm_90a:  D[M,N] = epi(A[M,K] · W[N,K]^T).
//
// The TMA / wgmma pipeline is tc_pipeline.cuh: 128 x BN output tiles, one TMA box of A (128x64) and one of W (BNx64) per
// k-block.  In the epilogue each thread owns one row of 32 (or, for QKV, 64) consecutive staged columns: fused bias /
// GELU / gate+residual / per-head LayerNorm + RoPE, bf16 stores.
//
// Replaces the cuBLAS calls behind every nn.Linear of the reference path (see include/ea_b200.h for call sites).
#include "host.h"
#include "tc_pipeline.cuh"
#include "../../include/ea_b200.h"

namespace ea {

enum { EPI_QKV = 100 };

struct GemmDevArgs {
  int M, N, K;
  const bf16* bias;
  void* out;
  int64_t ldo;
  float scale;
  const bf16* residual;
  int64_t ldr;
  const bf16* gate;
  int64_t gate_stride;
  int rows_per_batch;
  // qkv epilogue
  const bf16* ln_q_w;
  const bf16* ln_q_b;
  const bf16* ln_k_w;
  const bf16* ln_k_b;
  const float* rope_cos;
  const float* rope_sin;
  bf16* q;
  bf16* k;
  bf16* v;
  int d;
  int heads;
  int S;
  int seq_offset;
  float ln_eps;
  // sequence parallelism (ea_qkv_peers): head h is stored on the GPU that owns it, q_peers[h / heads_per_peer] (this GPU's
  // own buffer or a peer's, mapped over NVLink); 0 = everything goes to q/k/v above
  int heads_per_peer;
  bf16* q_peers[EA_MAX_PEERS];
  bf16* k_peers[EA_MAX_PEERS];
  bf16* v_peers[EA_MAX_PEERS];
};

// ------------------------------------------------------------------------------------------------
// epilogue helpers: one thread owns one accumulator row, `x` holds 32 consecutive columns
// ------------------------------------------------------------------------------------------------
// Ragged right edge (N % 32 != 0): same arithmetic as the vector path, one column at a time.
template <int EPI>
EA_DEVICE void epilogue_tail(const GemmDevArgs& p, int row, int col0, int nvalid, const float (&x)[32]) {
#pragma unroll 1
  for (int j = 0; j < nvalid; ++j) {
    const int col = col0 + j;
    float v = x[j];
    if constexpr (EPI == EA_EPI_SCALE_F32) {
      reinterpret_cast<float*>(p.out)[(int64_t)row * p.ldo + col] = v * p.scale;
    } else {
      if (p.bias != nullptr) v += __bfloat162float(p.bias[col]);
      v = bf16_round(v);
      if constexpr (EPI == EA_EPI_BIAS_GELU) v = gelu_tanh(v);
      if constexpr (EPI == EA_EPI_BIAS_GATE_RES) {
        const int b = row / p.rows_per_batch;
        const float g = __bfloat162float(p.gate[(int64_t)b * p.gate_stride + col]);
        v = __bfloat162float(p.residual[(int64_t)row * p.ldr + col]) + bf16_round(g * v);
      }
      if constexpr (EPI == EA_EPI_BIAS_RES) v += __bfloat162float(p.residual[(int64_t)row * p.ldr + col]);
      reinterpret_cast<bf16*>(p.out)[(int64_t)row * p.ldo + col] = __float2bfloat16_rn(v);
    }
  }
}

template <int EPI>
EA_DEVICE void epilogue_chunk32(const GemmDevArgs& p, int row, int col0, const float (&acc)[32]) {
  // row < M guaranteed by caller
  if (col0 + 32 > p.N) {
    epilogue_tail<EPI>(p, row, col0, p.N - col0, acc);
    return;
  }
  if constexpr (EPI == EA_EPI_SCALE_F32) {
    float* o = reinterpret_cast<float*>(p.out) + (int64_t)row * p.ldo + col0;
#pragma unroll
    for (int j = 0; j < 32; j += 4)
      *reinterpret_cast<float4*>(o + j) =
          make_float4(acc[j] * p.scale, acc[j + 1] * p.scale, acc[j + 2] * p.scale, acc[j + 3] * p.scale);
  } else {
    float x[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) x[j] = acc[j];
    if (p.bias != nullptr) add_bf16<32>(x, p.bias + col0);
    // the reference materialises the Linear output in bf16 before the next op
#pragma unroll
    for (int j = 0; j < 32; ++j) x[j] = bf16_round(x[j]);

    if constexpr (EPI == EA_EPI_BIAS_GELU) {
#pragma unroll
      for (int j = 0; j < 32; ++j) x[j] = gelu_tanh(x[j]);
    }
    if constexpr (EPI == EA_EPI_BIAS_GATE_RES) {
      int b = row / p.rows_per_batch;
      const uint4* gp = reinterpret_cast<const uint4*>(p.gate + (int64_t)b * p.gate_stride + col0);
      const uint4* rp = reinterpret_cast<const uint4*>(p.residual + (int64_t)row * p.ldr + col0);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint4 g = __ldg(gp + j);
        uint4 r = __ldg(rp + j);
        uint32_t gw[4] = {g.x, g.y, g.z, g.w};
        uint32_t rw[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          float2 gf = unpack_bf16x2(gw[t]);
          float2 rf = unpack_bf16x2(rw[t]);
          float y0 = bf16_round(gf.x * x[j * 8 + 2 * t]);
          float y1 = bf16_round(gf.y * x[j * 8 + 2 * t + 1]);
          x[j * 8 + 2 * t] = rf.x + y0;
          x[j * 8 + 2 * t + 1] = rf.y + y1;
        }
      }
    }
    if constexpr (EPI == EA_EPI_BIAS_RES) add_bf16<32>(x, p.residual + (int64_t)row * p.ldr + col0);
    store_bf16<32>(reinterpret_cast<bf16*>(p.out) + (int64_t)row * p.ldo + col0, x);
  }
}

// QKV epilogue for one head (64 columns) of one row.
EA_DEVICE void epilogue_qkv_head(const GemmDevArgs& p, int row, int col0, const float* src) {
  float x[64];
#pragma unroll
  for (int j = 0; j < 64; j += 4) *reinterpret_cast<float4*>(x + j) = *reinterpret_cast<const float4*>(src + j);
  add_bf16<64>(x, p.bias + col0);
#pragma unroll
  for (int j = 0; j < 64; ++j) x[j] = bf16_round(x[j]);

  const int which = col0 / p.d;  // 0 q, 1 k, 2 v
  const int head = (col0 - which * p.d) >> 6;
  const int b = row / p.rows_per_batch;
  const int s = row - b * p.rows_per_batch;

  if (which < 2) {
    // LayerNorm(64), fp32 statistics, affine, output rounded to bf16 (nn.LayerNorm on a bf16 tensor)
    float mean = 0.f;
#pragma unroll
    for (int j = 0; j < 64; ++j) mean += x[j];
    mean *= (1.0f / 64.0f);
    float var = 0.f;
#pragma unroll
    for (int j = 0; j < 64; ++j) {
      float dlt = x[j] - mean;
      var += dlt * dlt;
    }
    var *= (1.0f / 64.0f);
    const float rstd = rsqrtf(var + p.ln_eps);
    const bf16* lw = which == 0 ? p.ln_q_w : p.ln_k_w;
    const bf16* lb = which == 0 ? p.ln_q_b : p.ln_k_b;
    const uint4* wp = reinterpret_cast<const uint4*>(lw);
    const uint4* bp = reinterpret_cast<const uint4*>(lb);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint4 w4 = __ldg(wp + j);
      uint4 b4 = __ldg(bp + j);
      uint32_t ww[4] = {w4.x, w4.y, w4.z, w4.w};
      uint32_t bw[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        float2 wf = unpack_bf16x2(ww[t]);
        float2 bf = unpack_bf16x2(bw[t]);
        x[j * 8 + 2 * t] = bf16_round((x[j * 8 + 2 * t] - mean) * rstd * wf.x + bf.x);
        x[j * 8 + 2 * t + 1] = bf16_round((x[j * 8 + 2 * t + 1] - mean) * rstd * wf.y + bf.y);
      }
    }
    if (p.rope_cos != nullptr) {
      // diffusers apply_rotary_emb(use_real=True, unbind_dim=-1): out = x*cos + rot(x)*sin in fp32,
      // rot(x)[2i] = -x[2i+1], rot(x)[2i+1] = x[2i]
      const float4* cp = reinterpret_cast<const float4*>(p.rope_cos + (int64_t)s * 64);
      const float4* sp = reinterpret_cast<const float4*>(p.rope_sin + (int64_t)s * 64);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float4 c = __ldg(cp + j);
        float4 sn = __ldg(sp + j);
        float e0 = x[4 * j], o0 = x[4 * j + 1], e1 = x[4 * j + 2], o1 = x[4 * j + 3];
        x[4 * j] = e0 * c.x + (-o0) * sn.x;
        x[4 * j + 1] = o0 * c.y + e0 * sn.y;
        x[4 * j + 2] = e1 * c.z + (-o1) * sn.z;
        x[4 * j + 3] = o1 * c.w + e1 * sn.w;
      }
    }
  }
  bf16* base = which == 0 ? p.q : (which == 1 ? p.k : p.v);
  int head_l = head, heads_l = p.heads;
  if (p.heads_per_peer > 0) {
    // Ulysses exchange fused into the projection: the row goes straight into the q/k/v buffer [B, heads_per_peer, S, 64] of
    // the GPU that runs attention for this head - a 128-byte store over NVLink when that is a peer (a NULL entry = a head
    // this call does not have to deliver: the replicated text rows are projected on every GPU for its own heads only)
    const int owner = head / p.heads_per_peer;
    base = (which == 0 ? p.q_peers : (which == 1 ? p.k_peers : p.v_peers))[owner];
    if (base == nullptr) return;
    head_l = head - owner * p.heads_per_peer;
    heads_l = p.heads_per_peer;
  }
  store_bf16<64>(base + (((int64_t)b * heads_l + head_l) * p.S + p.seq_offset + s) * 64, x);
}

// ------------------------------------------------------------------------------------------------
// kernel
// ------------------------------------------------------------------------------------------------
template <int BN, int EPI>
__global__ void __launch_bounds__(kTcThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const GemmDevArgs p) {
  const int num_n_tiles = (p.N + BN - 1) / BN;
  const int num_tiles = ((p.M + kTcBM - 1) / kTcBM) * num_n_tiles;
  // tile -> (m0, n0): its first row of A and of W
  auto decode = [&](int tile) { return make_int2((tile / num_n_tiles) * kTcBM, (tile % num_n_tiles) * BN); };
  auto load = [](int2 mn, int kb, const CUtensorMap* ta, const CUtensorMap* tb, void* a, void* b, uint64_t* bar) {
    tma_load_2d(a, ta, bar, kb * kTcBK, mn.x);
    tma_load_2d(b, tb, bar, kb * kTcBK, mn.y);
  };
  // one row of 32 columns, or for QKV of one head (64 columns), per item
  auto epilogue = [&](int2 mn, int r, int c, const float* src) {
    const int row = mn.x + r, col = mn.y + c;
    if (row >= p.M || col >= p.N) return;
    if constexpr (EPI == EPI_QKV) {
      epilogue_qkv_head(p, row, col, src);
    } else {
      float x[32];
#pragma unroll
      for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(x + j) = *reinterpret_cast<const float4*>(src + j);
      epilogue_chunk32<EPI>(p, row, col, x);
    }
  };
  tc_pipeline<BN, EPI == EPI_QKV ? 64 : 32>(&tmap_a, &tmap_b, num_tiles, (p.K + kTcBK - 1) / kTcBK, decode, load, epilogue);
}

// ------------------------------------------------------------------------------------------------
// host launch
// ------------------------------------------------------------------------------------------------
template <int BN, int EPI>
static int launch_gemm(const void* a, int64_t lda, const void* w, int64_t ldw, const GemmDevArgs& p, void* stream) {
  CUtensorMap ta, tb;
  {
    uint64_t dims[2] = {(uint64_t)p.K, (uint64_t)p.M};
    uint64_t strides[1] = {(uint64_t)lda * 2};
    uint32_t box[2] = {kTcBK, kTcBM};
    int rc = make_tmap_bf16(&ta, a, 2, dims, strides, box, true);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {(uint64_t)p.K, (uint64_t)p.N};
    uint64_t strides[1] = {(uint64_t)ldw * 2};
    uint32_t box[2] = {kTcBK, (uint32_t)BN};
    int rc = make_tmap_bf16(&tb, w, 2, dims, strides, box, true);
    if (rc) return rc;
  }
  static PerDeviceFlag smem_done;
  const int num_tiles = ((p.M + kTcBM - 1) / kTcBM) * ((p.N + BN - 1) / BN);
  return launch_persistent(gemm_tc_kernel<BN, EPI>, num_tiles, kTcThreads, TcCfg<BN>::kSmemBytes, smem_done, stream,
                           "gemm_tc_kernel", ta, tb, p);
}

template <int EPI>
static int dispatch_bn(const void* a, int64_t lda, const void* w, int64_t ldw, const GemmDevArgs& p, void* stream) {
  // Wide tiles unless they would leave most SMs idle.
  const int sms = sm_count();
  auto tiles = [&](int bn) { return (int64_t)((p.M + kTcBM - 1) / kTcBM) * ((p.N + bn - 1) / bn); };
  // (ragged N is fine for every width: TMA zero-fills the missing weight rows, the epilogue masks the columns)
  if (p.N >= 256 && tiles(256) >= sms) return launch_gemm<256, EPI>(a, lda, w, ldw, p, stream);
  if (p.N >= 128 && tiles(128) >= sms / 2) return launch_gemm<128, EPI>(a, lda, w, ldw, p, stream);
  return launch_gemm<64, EPI>(a, lda, w, ldw, p, stream);
}

}  // namespace ea

using namespace ea;

extern "C" int ea_gemm(const ea_gemm_args* g, void* stream) {
  EA_REQUIRE(g != nullptr, "ea_gemm: null args");
  EA_REQUIRE(g->a && g->w && g->out, "ea_gemm: null pointer");
  EA_REQUIRE(g->M > 0 && g->N > 0 && g->K > 0, "ea_gemm: empty problem");
  EA_REQUIRE(g->M < (1ll << 31) && g->N < (1ll << 31) && g->K < (1ll << 31), "ea_gemm: dims exceed int32");
  EA_REQUIRE(g->lda % 8 == 0 && g->ldw % 8 == 0, "ea_gemm: lda/ldw must be multiples of 8 (16-byte TMA strides)");
  EA_REQUIRE(g->lda >= g->K && g->ldw >= g->K && g->ldo >= g->N, "ea_gemm: leading dimension too small");
  EA_REQUIRE((reinterpret_cast<uintptr_t>(g->a) & 15) == 0 && (reinterpret_cast<uintptr_t>(g->w) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(g->out) & 15) == 0,
             "ea_gemm: pointers must be 16-byte aligned");
  EA_REQUIRE(g->ldo % 8 == 0, "ea_gemm: ldo must be a multiple of 8");
  GemmDevArgs p{};
  p.M = (int)g->M; p.N = (int)g->N; p.K = (int)g->K;
  p.bias = reinterpret_cast<const bf16*>(g->bias);
  p.out = g->out; p.ldo = g->ldo; p.scale = g->scale;
  p.residual = reinterpret_cast<const bf16*>(g->residual); p.ldr = g->ldr;
  p.gate = reinterpret_cast<const bf16*>(g->gate); p.gate_stride = g->gate_stride;
  p.rows_per_batch = (int)(g->rows_per_batch > 0 ? g->rows_per_batch : g->M);
  switch (g->epilogue) {
    case EA_EPI_BIAS: return dispatch_bn<EA_EPI_BIAS>(g->a, g->lda, g->w, g->ldw, p, stream);
    case EA_EPI_BIAS_GELU: return dispatch_bn<EA_EPI_BIAS_GELU>(g->a, g->lda, g->w, g->ldw, p, stream);
    case EA_EPI_BIAS_GATE_RES:
      EA_REQUIRE(g->residual && g->gate, "ea_gemm: GATE_RES needs residual and gate");
      EA_REQUIRE(g->ldr % 8 == 0 && g->gate_stride % 8 == 0, "ea_gemm: ldr/gate_stride must be multiples of 8");
      return dispatch_bn<EA_EPI_BIAS_GATE_RES>(g->a, g->lda, g->w, g->ldw, p, stream);
    case EA_EPI_SCALE_F32: return dispatch_bn<EA_EPI_SCALE_F32>(g->a, g->lda, g->w, g->ldw, p, stream);
    case EA_EPI_BIAS_RES:
      EA_REQUIRE(g->residual, "ea_gemm: BIAS_RES needs residual");
      EA_REQUIRE(g->ldr % 8 == 0, "ea_gemm: ldr must be a multiple of 8");
      return dispatch_bn<EA_EPI_BIAS_RES>(g->a, g->lda, g->w, g->ldw, p, stream);
    default: return fail(EA_ERR_INVALID, "ea_gemm: unknown epilogue");
  }
}

extern "C" int ea_qkv_gemm_ln_rope(const ea_qkv_args* g, void* stream) {
  EA_REQUIRE(g != nullptr, "ea_qkv: null args");
  EA_REQUIRE(g->a && g->w && g->bias && ((g->q && g->k && g->v) || g->peers), "ea_qkv: null pointer");
  EA_REQUIRE(g->ln_q_w && g->ln_q_b && g->ln_k_w && g->ln_k_b, "ea_qkv: null LayerNorm parameter");
  EA_REQUIRE(g->d > 0 && g->d % 64 == 0, "ea_qkv: d must be a multiple of the head size 64");
  EA_REQUIRE(g->M > 0 && g->rows_per_batch > 0 && g->M % g->rows_per_batch == 0, "ea_qkv: M must be B*rows_per_batch");
  EA_REQUIRE(g->lda % 8 == 0 && g->lda >= g->d, "ea_qkv: bad lda");
  EA_REQUIRE(g->seq_offset >= 0 && g->seq_offset + g->rows_per_batch <= g->S, "ea_qkv: part does not fit in S");
  EA_REQUIRE((g->rope_cos == nullptr) == (g->rope_sin == nullptr), "ea_qkv: cos/sin must both be given or both NULL");
  GemmDevArgs p{};
  p.M = (int)g->M; p.N = (int)(3 * g->d); p.K = (int)g->d;
  p.bias = reinterpret_cast<const bf16*>(g->bias);
  p.ln_q_w = reinterpret_cast<const bf16*>(g->ln_q_w); p.ln_q_b = reinterpret_cast<const bf16*>(g->ln_q_b);
  p.ln_k_w = reinterpret_cast<const bf16*>(g->ln_k_w); p.ln_k_b = reinterpret_cast<const bf16*>(g->ln_k_b);
  p.rope_cos = g->rope_cos; p.rope_sin = g->rope_sin;
  p.q = reinterpret_cast<bf16*>(g->q); p.k = reinterpret_cast<bf16*>(g->k); p.v = reinterpret_cast<bf16*>(g->v);
  p.d = (int)g->d; p.heads = (int)(g->d / 64); p.S = (int)g->S; p.seq_offset = (int)g->seq_offset;
  p.rows_per_batch = (int)g->rows_per_batch; p.ln_eps = g->ln_eps;
  if (g->peers != nullptr) {
    const ea_qkv_peers* pe = g->peers;
    EA_REQUIRE(pe->heads_per_peer > 0 && (g->d / 64) % pe->heads_per_peer == 0 && (g->d / 64) / pe->heads_per_peer <= EA_MAX_PEERS,
               "ea_qkv: heads_per_peer must divide the head count into at most EA_MAX_PEERS groups");
    p.heads_per_peer = (int)pe->heads_per_peer;
    for (int i = 0; i < EA_MAX_PEERS; ++i) {
      p.q_peers[i] = reinterpret_cast<bf16*>(pe->q[i]);
      p.k_peers[i] = reinterpret_cast<bf16*>(pe->k[i]);
      p.v_peers[i] = reinterpret_cast<bf16*>(pe->v[i]);
    }
  }
  // an N tile must not straddle the q|k|v boundaries: the widest tile that divides d
  if (g->d % 256 == 0) return launch_gemm<256, EPI_QKV>(g->a, g->lda, g->w, g->d, p, stream);
  if (g->d % 128 == 0) return launch_gemm<128, EPI_QKV>(g->a, g->lda, g->w, g->d, p, stream);
  return launch_gemm<64, EPI_QKV>(g->a, g->lda, g->w, g->d, p, stream);
}

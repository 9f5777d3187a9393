// Persistent, warp-specialised wgmma GEMM for sm_90a:  D[M,N] = epi(A[M,K] · W[N,K]^T).
//
//   warpgroup 0 (1 thread) : TMA producer — cp.async.bulk.tensor tiles of A (128x64) and W (BNx64) into a SWIZZLE_128B
//                            shared-memory ring, completion on `full` mbarriers.
//   warpgroups 1, 2        : consumers — rows [0,64) / [64,128) of the 128 x BN tile: wgmma.m64nBNk16 (bf16 -> fp32 in
//                            registers) from both operands in shared memory, then the epilogue: the accumulators go through
//                            a shared-memory staging buffer so that each thread owns one row of 32 (or 64) consecutive
//                            columns, fused bias / GELU / gate+residual / per-head LayerNorm + RoPE, bf16 stores.
// The producer keeps fetching the next tile's k-blocks while the consumers run the epilogue.
//
// Replaces the cuBLAS calls behind every nn.Linear of the reference path (see include/ea_b200.h for call sites).
#include "common.cuh"
#include "host.h"
#include "../../include/ea_b200.h"

namespace ea {

extern void count_launch();

constexpr int kBM = 128;
constexpr int kBK = 64;
constexpr int kGemmThreads = 384;
constexpr int kStagePitch = 132;  // fp32 staging row pitch: conflict-free 16-byte row reads

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

template <int BN>
struct GemmCfg {
  static constexpr int kStages = BN == 256 ? 3 : (BN == 128 ? 4 : 6);
  static constexpr int kABytes = kBM * kBK * 2;
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kCW = BN < 128 ? BN : 128;  // columns staged per epilogue pass
  static constexpr int kStagingBytes = 2 * 64 * kStagePitch * 4;
  static constexpr int kSmemBytes = kStages * kStageBytes + kStagingBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kSmemBytes <= 227 * 1024, "shared memory");
};

// ------------------------------------------------------------------------------------------------
// epilogue helpers: one thread owns one accumulator row, `v` holds 32 consecutive columns
// ------------------------------------------------------------------------------------------------
// Ragged right edge (N % 32 != 0): same arithmetic as the vector path, one column at a time.
template <int EPI>
EA_DEVICE void epilogue_tail(const GemmDevArgs& p, int row, int col0, int nvalid, uint32_t (&acc)[32]) {
#pragma unroll 1
  for (int j = 0; j < nvalid; ++j) {
    const int col = col0 + j;
    float v = __uint_as_float(acc[j]);
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
EA_DEVICE void epilogue_chunk32(const GemmDevArgs& p, int row, int col0, uint32_t (&acc)[32]) {
  // row < M guaranteed by caller
  if (col0 + 32 > p.N) {
    epilogue_tail<EPI>(p, row, col0, p.N - col0, acc);
    return;
  }
  if constexpr (EPI == EA_EPI_SCALE_F32) {
    float* o = reinterpret_cast<float*>(p.out) + (int64_t)row * p.ldo + col0;
#pragma unroll
    for (int j = 0; j < 32; j += 4) {
      float4 f;
      f.x = __uint_as_float(acc[j]) * p.scale;
      f.y = __uint_as_float(acc[j + 1]) * p.scale;
      f.z = __uint_as_float(acc[j + 2]) * p.scale;
      f.w = __uint_as_float(acc[j + 3]) * p.scale;
      *reinterpret_cast<float4*>(o + j) = f;
    }
    return;
  } else {
    float x[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) x[j] = __uint_as_float(acc[j]);
    if (p.bias != nullptr) {
      const uint4* bp = reinterpret_cast<const uint4*>(p.bias + col0);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint4 b = __ldg(bp + j);
        float2 f0 = unpack_bf16x2(b.x), f1 = unpack_bf16x2(b.y), f2 = unpack_bf16x2(b.z), f3 = unpack_bf16x2(b.w);
        x[j * 8 + 0] += f0.x; x[j * 8 + 1] += f0.y; x[j * 8 + 2] += f1.x; x[j * 8 + 3] += f1.y;
        x[j * 8 + 4] += f2.x; x[j * 8 + 5] += f2.y; x[j * 8 + 6] += f3.x; x[j * 8 + 7] += f3.y;
      }
    }
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
    if constexpr (EPI == EA_EPI_BIAS_RES) {
      const uint4* rp = reinterpret_cast<const uint4*>(p.residual + (int64_t)row * p.ldr + col0);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint4 r = __ldg(rp + j);
        uint32_t rw[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          float2 rf = unpack_bf16x2(rw[t]);
          x[j * 8 + 2 * t] += rf.x;
          x[j * 8 + 2 * t + 1] += rf.y;
        }
      }
    }
    bf16* o = reinterpret_cast<bf16*>(p.out) + (int64_t)row * p.ldo + col0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint4 w;
      w.x = pack_bf16x2(x[j * 8 + 0], x[j * 8 + 1]);
      w.y = pack_bf16x2(x[j * 8 + 2], x[j * 8 + 3]);
      w.z = pack_bf16x2(x[j * 8 + 4], x[j * 8 + 5]);
      w.w = pack_bf16x2(x[j * 8 + 6], x[j * 8 + 7]);
      *reinterpret_cast<uint4*>(o + j * 8) = w;
    }
  }
}

// QKV epilogue for one head (64 columns) of one row.
EA_DEVICE void epilogue_qkv_head(const GemmDevArgs& p, int row, int col0, const float* src) {
  float x[64];
#pragma unroll
  for (int j = 0; j < 64; j += 4) *reinterpret_cast<float4*>(x + j) = *reinterpret_cast<const float4*>(src + j);
  {
    const uint4* bp = reinterpret_cast<const uint4*>(p.bias + col0);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint4 b = __ldg(bp + j);
      float2 f0 = unpack_bf16x2(b.x), f1 = unpack_bf16x2(b.y), f2 = unpack_bf16x2(b.z), f3 = unpack_bf16x2(b.w);
      x[j * 8 + 0] += f0.x; x[j * 8 + 1] += f0.y; x[j * 8 + 2] += f1.x; x[j * 8 + 3] += f1.y;
      x[j * 8 + 4] += f2.x; x[j * 8 + 5] += f2.y; x[j * 8 + 6] += f3.x; x[j * 8 + 7] += f3.y;
    }
  }
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
  bf16* o = base + (((int64_t)b * heads_l + head_l) * p.S + p.seq_offset + s) * 64;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    uint4 w;
    w.x = pack_bf16x2(x[j * 8 + 0], x[j * 8 + 1]);
    w.y = pack_bf16x2(x[j * 8 + 2], x[j * 8 + 3]);
    w.z = pack_bf16x2(x[j * 8 + 4], x[j * 8 + 5]);
    w.w = pack_bf16x2(x[j * 8 + 6], x[j * 8 + 7]);
    *reinterpret_cast<uint4*>(o + j * 8) = w;
  }
}

// ------------------------------------------------------------------------------------------------
// kernel
// ------------------------------------------------------------------------------------------------
template <int BN, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const GemmDevArgs p) {
  using Cfg = GemmCfg<BN>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kCW = Cfg::kCW;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * Cfg::kABytes;
  float* staging = reinterpret_cast<float*>(smem + kStages * Cfg::kStageBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes + Cfg::kStagingBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;

  const int num_m_tiles = (p.M + kBM - 1) / kBM;
  const int num_n_tiles = (p.N + BN - 1) / BN;
  const int num_tiles = num_m_tiles * num_n_tiles;
  const int num_k_blocks = (p.K + kBK - 1) / kBK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // lane 0 of each consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      // ===== TMA producer =====
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile / num_n_tiles) * kBM;
        const int n0 = (tile % num_n_tiles) * BN;
        for (int kb = 0; kb < num_k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_2d(smem_a + stage * Cfg::kABytes, &tmap_a, &full_bar[stage], kb * kBK, m0);
          tma_load_2d(smem_b + stage * Cfg::kBBytes, &tmap_b, &full_bar[stage], kb * kBK, n0);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ===== consumers: rows [64 (wg-1), 64 wg) of the tile =====
    const int cw = wg - 1;
    const int tid = threadIdx.x & 127;
    float* stage_buf = staging + cw * 64 * kStagePitch;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m0 = (tile / num_n_tiles) * kBM;
      const int n0 = (tile % num_n_tiles) * BN;
      float acc[BN / 2];
      int prev = -1;
      for (int kb = 0; kb < num_k_blocks; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t adesc = gmma_desc_sw128(smem_u32(smem_a + stage * Cfg::kABytes + cw * 64 * 128));
        const uint64_t bdesc = gmma_desc_sw128(smem_u32(smem_b + stage * Cfg::kBBytes));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k) {
          // advance 16 bf16 = 32 B inside the 128 B swizzle row: +2 in the (addr >> 4) field
          wgmma_ss<BN>(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the k-block before this one has been read: release its stage
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence<BN / 2>(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);

      // ===== epilogue: kCW columns at a time through the staging buffer, one row per thread and column chunk =====
#pragma unroll
      for (int cb = 0; cb < BN / kCW; ++cb) {
        named_bar_sync(1 + cw, 128);  // the previous pass has finished reading the staging buffer
        stage_acc<kCW>(acc + cb * (kCW / 2), stage_buf, kStagePitch);
        named_bar_sync(1 + cw, 128);
        const int c0 = n0 + cb * kCW;
        if constexpr (EPI == EPI_QKV) {
#pragma unroll 1
          for (int i = tid; i < 64 * (kCW / 64); i += 128) {
            const int r = i & 63, h = i >> 6;
            const int row = m0 + cw * 64 + r;
            if (row < p.M && c0 + h * 64 < p.N) epilogue_qkv_head(p, row, c0 + h * 64, stage_buf + r * kStagePitch + h * 64);
          }
        } else {
#pragma unroll 1
          for (int i = tid; i < 64 * (kCW / 32); i += 128) {
            const int r = i & 63, c = i >> 6;
            const int row = m0 + cw * 64 + r;
            if (row < p.M && c0 + c * 32 < p.N) {
              uint32_t a32[32];
              const float* src = stage_buf + r * kStagePitch + c * 32;
#pragma unroll
              for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(a32 + j) = *reinterpret_cast<const float4*>(src + j);
              epilogue_chunk32<EPI>(p, row, c0 + c * 32, a32);
            }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host launch
// ------------------------------------------------------------------------------------------------
template <int BN, int EPI>
static int launch_gemm(const void* a, int64_t lda, const void* w, int64_t ldw, const GemmDevArgs& p,
                       cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  CUtensorMap ta, tb;
  {
    uint64_t dims[2] = {(uint64_t)p.K, (uint64_t)p.M};
    uint64_t strides[1] = {(uint64_t)lda * 2};
    uint32_t box[2] = {kBK, kBM};
    int rc = make_tmap_bf16(&ta, a, 2, dims, strides, box, true);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {(uint64_t)p.K, (uint64_t)p.N};
    uint64_t strides[1] = {(uint64_t)ldw * 2};
    uint32_t box[2] = {kBK, (uint32_t)BN};
    int rc = make_tmap_bf16(&tb, w, 2, dims, strides, box, true);
    if (rc) return rc;
  }
  auto kern = gemm_tc_kernel<BN, EPI>;
  static ::ea::PerDeviceFlag attr_flag;
  const int attr_dev = ::ea::current_device();
  if (!attr_flag.get(attr_dev)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) return fail(EA_ERR_CUDA, std::string("cudaFuncSetAttribute(gemm): ") + cudaGetErrorString(e));
    attr_flag.set(attr_dev);
  }
  const int num_tiles = ((p.M + kBM - 1) / kBM) * ((p.N + BN - 1) / BN);
  int grid = num_tiles < sm_count() ? num_tiles : sm_count();
  kern<<<grid, kGemmThreads, Cfg::kSmemBytes, stream>>>(ta, tb, p);
  count_launch();
  return check_launch("gemm_tc_kernel");
}

template <int EPI>
static int dispatch_bn(const void* a, int64_t lda, const void* w, int64_t ldw, const GemmDevArgs& p,
                       cudaStream_t stream) {
  // Wide tiles unless they would leave most SMs idle.
  const int sms = sm_count();
  auto tiles = [&](int bn) { return (int64_t)((p.M + kBM - 1) / kBM) * ((p.N + bn - 1) / bn); };
  // (ragged N is fine for every width: TMA zero-fills the missing weight rows, the epilogue masks the columns)
  if (p.N >= 256 && tiles(256) >= sms) return launch_gemm<256, EPI>(a, lda, w, ldw, p, stream);
  if (p.N >= 128 && tiles(128) >= sms / 2) return launch_gemm<128, EPI>(a, lda, w, ldw, p, stream);
  return launch_gemm<64, EPI>(a, lda, w, ldw, p, stream);
}

}  // namespace ea

using namespace ea;

extern "C" int ea_gemm(const ea_gemm_args* g, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
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

extern "C" int ea_qkv_gemm_ln_rope(const ea_qkv_args* g, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
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

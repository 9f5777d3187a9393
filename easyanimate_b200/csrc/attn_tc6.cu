// Joint text+video attention forward on sm_90a: softmax(Q K^T * scale) V for head_dim 64, one (batch, head) per grid row.
//
//   warpgroup 0 (1 thread) : TMA producer — Q once (128 rows), K_j / V_j 128-key tiles through 3-stage rings.
//   warpgroups 1, 2        : query rows [0,64) / [64,128) of the CTA's tile.  Per key block:
//                              S = Q K_j^T      wgmma.m64n128k16, both operands in shared memory (SWIZZLE_128B, K-major)
//                              online softmax   in registers (row max / sum across the 4 threads of a quad), exp2 on MUFU
//                              O += P V_j       wgmma.m64n64k16, P as bf16 register fragments, V MN-major in shared memory
// P is rounded to bf16 (as the reference's bf16 attention does), O, the running maximum and the row sums stay fp32.  The
// two consumer warpgroups run independently, so one's softmax overlaps the other's MMAs.
#include "common.cuh"
#include "host.h"
#include "../../include/ea_b200.h"

namespace ea {

extern void count_launch();

namespace a6 {

constexpr int kQT = 128;
constexpr int kKT = 128;
constexpr int kHD = 64;
constexpr int kStages = 3;
constexpr int kThreads = 384;
constexpr int kQBytes = kQT * kHD * 2;
constexpr int kKVBytes = kKT * kHD * 2;
constexpr int kOffK = kQBytes;
constexpr int kOffV = kOffK + kStages * kKVBytes;
constexpr int kOffBar = kOffV + kStages * kKVBytes;
constexpr int kTotal = kOffBar + 256 + 1024;

struct Args {
  bf16* out_text;
  bf16* out_video;
  int B, H, S, S_text;
  float scale_log2;
  // sequence parallelism (ea_attn_peers): this GPU computed heads [head0, head0 + H) of out_heads for ALL tokens; a video
  // token's row goes to the GPU that owns the token (tokens_per_peer each), the text rows to every GPU.  n_peers = 0: local.
  int n_peers, tokens_per_peer, out_heads, head0;
  bf16* out_video_peers[EA_MAX_PEERS];
  bf16* out_text_peers[EA_MAX_PEERS];
};

EA_DEVICE float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Stores one 64-wide output row fragment: `v` holds columns 8 jb + c, 8 jb + c + 1 for jb = 0..7 (already normalised).
EA_DEVICE void store_row(const Args& p, int bh, int srow, int c, const float* v) {
  if (srow >= p.S) return;
  const int bb = bh / p.H, h = bh % p.H;
  bf16* dst;
  int ndst = 1;  // text rows under sequence parallelism are delivered to every GPU of the group
  int64_t text_off = 0;
  if (p.n_peers == 0) {
    const int64_t d = (int64_t)p.H * kHD;
    if (srow < p.S_text)
      dst = p.out_text + ((int64_t)bb * p.S_text + srow) * d + h * kHD;
    else
      dst = p.out_video + ((int64_t)bb * (p.S - p.S_text) + (srow - p.S_text)) * d + h * kHD;
  } else {
    // Ulysses return exchange fused into the epilogue: [token, head] rows stored straight into the token-major
    // [B, tokens, out_heads * 64] buffer of the GPU that owns the token (NVLink when it is a peer)
    const int64_t d = (int64_t)p.out_heads * kHD;
    if (srow < p.S_text) {
      text_off = ((int64_t)bb * p.S_text + srow) * d + (int64_t)(p.head0 + h) * kHD;
      dst = p.out_text_peers[0] + text_off;
      ndst = p.n_peers;
    } else {
      const int v = srow - p.S_text;
      const int owner = v / p.tokens_per_peer;
      dst = p.out_video_peers[owner] + ((int64_t)bb * p.tokens_per_peer + (v - owner * p.tokens_per_peer)) * d +
            (int64_t)(p.head0 + h) * kHD;
    }
  }
#pragma unroll
  for (int jb = 0; jb < 8; ++jb) {
    const uint32_t w = pack_bf16x2(v[2 * jb], v[2 * jb + 1]);
    *reinterpret_cast<uint32_t*>(dst + 8 * jb + c) = w;
    for (int pr = 1; pr < ndst; ++pr) *reinterpret_cast<uint32_t*>(p.out_text_peers[pr] + text_off + 8 * jb + c) = w;
  }
}

__global__ void __launch_bounds__(kThreads, 1)
attn6_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
             const __grid_constant__ CUtensorMap tmap_v, const Args p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = smem + kOffK;
  uint8_t* sV = smem + kOffV;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;
  uint64_t* k_empty = k_full + kStages;
  uint64_t* v_full = k_empty + kStages;
  uint64_t* v_empty = v_full + kStages;

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kQT;
  const int bh = blockIdx.y;
  const int nblk = (p.S + kKT - 1) / kKT;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    mbar_init(q_full, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 8);  // lane 0 of each consumer warp
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      // ===== TMA producer =====
      mbar_arrive_expect_tx(q_full, kQBytes);
      tma_load_3d(sQ, &tmap_q, q_full, 0, q0, bh);
      int st = 0;
      uint32_t ph = 0;
      for (int j = 0; j < nblk; ++j) {
        mbar_wait(&k_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&k_full[st], kKVBytes);
        tma_load_3d(sK + st * kKVBytes, &tmap_k, &k_full[st], 0, j * kKT, bh);
        mbar_wait(&v_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&v_full[st], kKVBytes);
        tma_load_3d(sV + st * kKVBytes, &tmap_v, &v_full[st], 0, j * kKT, bh);
        if (++st == kStages) { st = 0; ph ^= 1; }
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  // ===== consumers: 64 query rows each; this thread holds rows r and r + 8 of them, columns 8 jb + c, + 1 =====
  const int cw = wg - 1;
  const int r = 16 * ((threadIdx.x & 127) >> 5) + (lane >> 2);
  const int c = 2 * (lane & 3);
  const float sl2 = p.scale_log2;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY};  // running maximum of the scaled scores (log2 domain)
  float l[2] = {0.f, 0.f};              // this thread's share of the row sums

  mbar_wait(q_full, 0);
  const uint64_t qdesc = gmma_desc_sw128(smem_u32(sQ + cw * 64 * 128));
  int st = 0;
  uint32_t ph = 0;
  for (int j = 0; j < nblk; ++j) {
    float s[64];
    mbar_wait(&k_full[st], ph);
    const uint64_t kdesc = gmma_desc_sw128(smem_u32(sK + st * kKVBytes));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kHD / 16; ++k) wgmma_ss<128>(s, qdesc + 2 * k, kdesc + 2 * k, k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<64>(s);
    if (lane == 0) mbar_arrive(&k_empty[st]);

    const int valid = p.S - j * kKT;  // < kKT only in the last block (TMA zero-filled the missing keys)
    if (valid < kKT) {
#pragma unroll
      for (int jb = 0; jb < 16; ++jb)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (8 * jb + c + (e & 1) >= valid) s[4 * jb + e] = -INFINITY;
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int jb = 0; jb < 16; ++jb) {
      mx[0] = fmaxf(mx[0], fmaxf(s[4 * jb], s[4 * jb + 1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[4 * jb + 2], s[4 * jb + 3]));
    }
    float nm[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float m_new = fmaxf(m[h], mx[h] * sl2);
      const float f = ex2(m[h] - m_new);  // 0 for the first block (m = -inf)
      l[h] *= f;
#pragma unroll
      for (int jb = 0; jb < 8; ++jb) {
        o[4 * jb + 2 * h] *= f;
        o[4 * jb + 2 * h + 1] *= f;
      }
      m[h] = m_new;
      nm[h] = -m_new;
    }
    // P = 2^(s * scale_log2 - m) as bf16 A fragments of m64n64k16: k-step kk takes key columns [16 kk, 16 kk + 16)
    uint32_t pa[8][4];
#pragma unroll
    for (int jb = 0; jb < 16; ++jb) {
      const float e0 = ex2(fmaf(s[4 * jb], sl2, nm[0])), e1 = ex2(fmaf(s[4 * jb + 1], sl2, nm[0]));
      const float e2 = ex2(fmaf(s[4 * jb + 2], sl2, nm[1])), e3 = ex2(fmaf(s[4 * jb + 3], sl2, nm[1]));
      l[0] += e0 + e1;
      l[1] += e2 + e3;
      pa[jb >> 1][2 * (jb & 1)] = pack_bf16x2(e0, e1);
      pa[jb >> 1][2 * (jb & 1) + 1] = pack_bf16x2(e2, e3);
    }

    mbar_wait(&v_full[st], ph);
    const uint32_t vaddr = smem_u32(sV + st * kKVBytes);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kKT / 16; ++kk) wgmma_rs_tb<64>(o, pa[kk], gmma_desc_sw128(vaddr + kk * 2048, 1024, kKVBytes));
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<32>(o);
    if (lane == 0) mbar_arrive(&v_empty[st]);
    if (++st == kStages) { st = 0; ph ^= 1; }
  }

  // ===== epilogue: O / l, bf16 rows to the text / video outputs (or the peers') =====
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float lt = l[h];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const float inv_l = 1.0f / lt;
    float v[16];
#pragma unroll
    for (int jb = 0; jb < 8; ++jb) {
      v[2 * jb] = o[4 * jb + 2 * h] * inv_l;
      v[2 * jb + 1] = o[4 * jb + 2 * h + 1] * inv_l;
    }
    store_row(p, bh, q0 + cw * 64 + r + 8 * h, c, v);
  }
}

static int launch(const ea_attn_args* g, cudaStream_t stream) {
  const int64_t BH = g->B * g->H;
  CUtensorMap tq, tk, tv;
  uint64_t dims[3] = {(uint64_t)kHD, (uint64_t)g->S, (uint64_t)BH};
  uint64_t strides[2] = {(uint64_t)kHD * 2, (uint64_t)g->S * kHD * 2};
  uint32_t box_q[3] = {kHD, kQT, 1};
  uint32_t box_kv[3] = {kHD, kKT, 1};
  int rc = make_tmap_bf16(&tq, g->q, 3, dims, strides, box_q, true);
  if (rc) return rc;
  rc = make_tmap_bf16(&tk, g->k, 3, dims, strides, box_kv, true);
  if (rc) return rc;
  rc = make_tmap_bf16(&tv, g->v, 3, dims, strides, box_kv, true);
  if (rc) return rc;
  Args p{};
  p.out_text = reinterpret_cast<bf16*>(g->out_text);
  p.out_video = reinterpret_cast<bf16*>(g->out_video);
  p.B = (int)g->B; p.H = (int)g->H; p.S = (int)g->S; p.S_text = (int)g->S_text;
  p.scale_log2 = g->scale * 1.4426950408889634f;
  if (g->peers != nullptr) {
    const ea_attn_peers* pe = g->peers;
    if (pe->n_peers < 1 || pe->n_peers > EA_MAX_PEERS || pe->tokens_per_peer <= 0 || pe->out_heads < pe->head0 + g->H ||
        pe->tokens_per_peer * pe->n_peers != g->S - g->S_text)
      return fail(EA_ERR_INVALID, "ea_attn_fwd: bad ea_attn_peers (n_peers, tokens_per_peer x n_peers == video tokens, head range)");
    p.n_peers = (int)pe->n_peers; p.tokens_per_peer = (int)pe->tokens_per_peer; p.out_heads = (int)pe->out_heads; p.head0 = (int)pe->head0;
    for (int i = 0; i < p.n_peers; ++i) {
      if (!pe->out_video[i] || (g->S_text > 0 && !pe->out_text[i])) return fail(EA_ERR_INVALID, "ea_attn_fwd: NULL peer output buffer");
      p.out_video_peers[i] = reinterpret_cast<bf16*>(pe->out_video[i]);
      p.out_text_peers[i] = reinterpret_cast<bf16*>(pe->out_text[i]);
    }
  }
  auto kern = attn6_kernel;
  static ::ea::PerDeviceFlag attr_flag;
  const int attr_dev = ::ea::current_device();
  if (!attr_flag.get(attr_dev)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kTotal);
    if (e != cudaSuccess) return fail(EA_ERR_CUDA, std::string("cudaFuncSetAttribute(attn6): ") + cudaGetErrorString(e));
    attr_flag.set(attr_dev);
  }
  dim3 grid((unsigned)((g->S + kQT - 1) / kQT), (unsigned)BH);
  kern<<<grid, kThreads, kTotal, stream>>>(tq, tk, tv, p);
  count_launch();
  return check_launch("attn6_kernel");
}

}  // namespace a6

// One kernel on sm_90a: the exponential-split (bits 4-6), truncated-P (0x800) and three-tile layout (0x2000) selections of
// ea_attn_args.variant are accepted and all run it.
int launch_attn6(const ea_attn_args* g, cudaStream_t stream) {
  return a6::launch(g, stream);
}

}  // namespace ea

// HBM-bound kernels of the MMDiT step: LayerNorm(+AdaLN modulate), RMSNorm, timestep sinusoid, small-M linear,
// patchify / unpatchify, CFG combine + Euler step.  One warp per token row, 16-byte vector loads/stores, values
// held in registers so every tensor is read once and written once.  bf16 rounding points follow the reference's
// op-by-op bf16 execution (each torch op materialises a bf16 tensor).
#include <algorithm>

#include "common.cuh"
#include "host.h"
#include "../../include/ea_b200.h"

namespace ea {

struct LnArgs {
  const bf16* x;
  bf16* y;
  int64_t rows;
  int d;
  int64_t ldx, ldy;
  int rows_per_batch;
  const bf16* pre_w;  // optional first LayerNorm (norm_final) applied before the main one
  const bf16* pre_b;
  float pre_eps;
  const bf16* w;  // main LayerNorm affine (may be NULL)
  const bf16* b;
  float eps;
  const bf16* shift;  // [B, mod_stride] or NULL
  const bf16* scale;
  int64_t mod_stride;
};

// NI = ceil(d / 256): number of 8-element vectors each lane owns.
template <int NI>
__global__ void __launch_bounds__(256) ln_modulate_kernel(const LnArgs a) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= a.rows) return;
  const int64_t row = warp;
  const int nvec = a.d >> 3;
  const uint4* xp = reinterpret_cast<const uint4*>(a.x + row * a.ldx);
  float v[NI][8];
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    const int vi = lane + 32 * i;
    if (vi < nvec) {
      unpack_bf16x8(xp[vi], v[i]);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[i][j] = 0.f;
    }
  }
  const float inv_d = 1.0f / (float)a.d;

  auto layer_norm = [&](const bf16* w, const bf16* b, float eps) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NI; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j];
    const float mean = warp_sum(s) * inv_d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const int vi = lane + 32 * i;
      if (vi < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float dlt = v[i][j] - mean;
          q += dlt * dlt;
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(q) * inv_d + eps);
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const int vi = lane + 32 * i;
      if (vi < nvec) {
        float wv[8], bv[8];
        if (w != nullptr) {
          unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(w) + vi), wv);
          unpack_bf16x8(__ldg(reinterpret_cast<const uint4*>(b) + vi), bv);
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) { wv[j] = 1.f; bv[j] = 0.f; }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) v[i][j] = bf16_round((v[i][j] - mean) * rstd * wv[j] + bv[j]);
      }
    }
  };

  if (a.pre_w != nullptr) layer_norm(a.pre_w, a.pre_b, a.pre_eps);
  layer_norm(a.w, a.b, a.eps);

  uint4* yp = reinterpret_cast<uint4*>(a.y + row * a.ldy);
  const int bidx = (int)(row / a.rows_per_batch);
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    const int vi = lane + 32 * i;
    if (vi < nvec) {
      if (a.scale != nullptr) {
        uint4 su = __ldg(reinterpret_cast<const uint4*>(a.scale + (int64_t)bidx * a.mod_stride) + vi);
        uint4 hu = __ldg(reinterpret_cast<const uint4*>(a.shift + (int64_t)bidx * a.mod_stride) + vi);
        uint32_t sw[4] = {su.x, su.y, su.z, su.w};
        uint32_t hw[4] = {hu.x, hu.y, hu.z, hu.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          float2 sf = unpack_bf16x2(sw[t]);
          float2 hf = unpack_bf16x2(hw[t]);
          // norm(x) * (1 + scale) + shift, each op rounded to bf16 (norm.py:164-165)
          float s0 = bf16_round(1.0f + sf.x), s1 = bf16_round(1.0f + sf.y);
          float m0 = bf16_round(v[i][2 * t] * s0), m1 = bf16_round(v[i][2 * t + 1] * s1);
          v[i][2 * t] = m0 + hf.x;
          v[i][2 * t + 1] = m1 + hf.y;
        }
      }
      yp[vi] = pack_bf16x8(v[i]);
    }
  }
}

struct RmsArgs {
  const bf16* x;
  bf16* y;
  const bf16* w;
  int64_t rows;
  int d;
  float eps;
};

template <int NI>
__global__ void __launch_bounds__(256) rmsnorm_kernel(const RmsArgs a) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= a.rows) return;
  const int nvec = a.d >> 3;
  const uint4* xp = reinterpret_cast<const uint4*>(a.x + (int64_t)warp * a.d);
  float v[NI][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    const int vi = lane + 32 * i;
    if (vi < nvec) {
      unpack_bf16x8(xp[vi], v[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j] * v[i][j];
    }
  }
  const float rstd = rsqrtf(warp_sum(s) / (float)a.d + a.eps);
  uint4* yp = reinterpret_cast<uint4*>(a.y + (int64_t)warp * a.d);
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    const int vi = lane + 32 * i;
    if (vi < nvec) {
      uint4 wu = __ldg(reinterpret_cast<const uint4*>(a.w) + vi);
      uint32_t ww[4] = {wu.x, wu.y, wu.z, wu.w};
      uint32_t o[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        float2 wf = unpack_bf16x2(ww[t]);
        // weight * (x * rsqrt(var + eps)).to(bf16)   (norm.py:35-39)
        float n0 = bf16_round(v[i][2 * t] * rstd), n1 = bf16_round(v[i][2 * t + 1] * rstd);
        o[t] = pack_bf16x2(wf.x * n0, wf.y * n1);
      }
      yp[vi] = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

// diffusers Timesteps(num_channels=dim, flip_sin_to_cos=True, downscale_freq_shift): fp32 sinusoid -> bf16
__global__ void timestep_embedding_kernel(const bf16* t, bf16* out, int B, int dim, float freq_shift, int flip) {
  const int half = dim / 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * half) return;
  const int b = idx / half, i = idx % half;
  const float tv = __bfloat162float(t[b]);
  const float exponent = -logf(10000.0f) * (float)i / ((float)half - freq_shift);
  const float arg = tv * expf(exponent);
  const float sv = sinf(arg), cv = cosf(arg);
  bf16* o = out + (int64_t)b * dim;
  if (flip) {
    o[i] = __float2bfloat16_rn(cv);
    o[half + i] = __float2bfloat16_rn(sv);
  } else {
    o[i] = __float2bfloat16_rn(sv);
    o[half + i] = __float2bfloat16_rn(cv);
  }
}

// out[m, n] = sum_k act(x[m,k]) * w[n,k] + bias[n];  M <= 8; one warp per n.
template <int MAXM>
__global__ void __launch_bounds__(256) skinny_linear_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w,
                                                            const bf16* __restrict__ bias, bf16* __restrict__ out,
                                                            int M, int N, int K, int act_in, int act_out) {
  extern __shared__ float xs[];  // [M][K]
  for (int i = threadIdx.x; i < M * K; i += blockDim.x) {
    float v = __bfloat162float(x[i]);
    if (act_in == 1) v = bf16_round(silu(v));
    xs[i] = v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + warp;
  if (n >= N) return;
  float acc[MAXM];
#pragma unroll
  for (int m = 0; m < MAXM; ++m) acc[m] = 0.f;
  const uint4* wp = reinterpret_cast<const uint4*>(w + (int64_t)n * K);
  const int nvec = K >> 3;
  for (int vi = lane; vi < nvec; vi += 32) {
    float wv[8];
    unpack_bf16x8(__ldg(wp + vi), wv);
#pragma unroll
    for (int m = 0; m < MAXM; ++m) {
      if (m < M) {
        const float* xr = xs + m * K + vi * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[m] += wv[j] * xr[j];
      }
    }
  }
#pragma unroll
  for (int m = 0; m < MAXM; ++m) acc[m] = warp_sum(acc[m]);
  if (lane == 0) {
    const float bv = bias ? __bfloat162float(bias[n]) : 0.f;
    for (int m = 0; m < M; ++m) {
      float r = bf16_round(acc[m] + bv);
      if (act_out == 1) r = silu(r);
      out[(int64_t)m * N + n] = __float2bfloat16_rn(r);
    }
  }
}

// idx -> (b, c, f, hh, ww) of a [B][C][F][Hp][Wp] index space, ww fastest
struct PatchPos {
  int b, c, f, hh, ww;
};
EA_DEVICE PatchPos patch_pos(int64_t idx, int C, int F, int Hp, int Wp) {
  const int ww = idx % Wp;
  int64_t r = idx / Wp;
  const int hh = r % Hp; r /= Hp;
  const int f = r % F; r /= F;
  const int c = r % C; r /= C;
  return {(int)r, c, f, hh, ww};
}

// A[(b,f,hh,ww), c*4 + ph*2 + pw] = cat(x, x2)[b, c, f, 2hh+ph, 2ww+pw];  columns >= 4*C are zero (K padding)
__global__ void patchify_kernel(const bf16* __restrict__ x, const bf16* __restrict__ x2, bf16* __restrict__ a, int B,
                                int C1, int C2, int F, int H, int W, int ldk) {
  const int Hp = H / 2, Wp = W / 2;
  const int C = C1 + C2;
  const int64_t total = (int64_t)B * F * Hp * Wp * C;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  // thread -> (row, c): ww fastest so reads of x rows are (2-element) coalesced
  const auto [b, c, f, hh, ww] = patch_pos(idx, C, F, Hp, Wp);
  const bf16* src;
  int cc, CC;
  if (c < C1) { src = x; cc = c; CC = C1; } else { src = x2; cc = c - C1; CC = C2; }
  const int64_t base = ((((int64_t)b * CC + cc) * F + f) * H + 2 * hh) * W + 2 * ww;
  const uint32_t top = *reinterpret_cast<const uint32_t*>(src + base);
  const uint32_t bot = *reinterpret_cast<const uint32_t*>(src + base + W);
  const int64_t row = (((int64_t)b * F + f) * Hp + hh) * Wp + ww;
  uint2 o = make_uint2(top, bot);
  *reinterpret_cast<uint2*>(a + row * ldk + c * 4) = o;
}
__global__ void patchify_pad_kernel(bf16* __restrict__ a, int64_t rows, int kvalid, int ldk) {
  const int padw = ldk - kvalid;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * padw) return;
  a[(idx / padw) * ldk + kvalid + idx % padw] = __float2bfloat16_rn(0.f);
}

// out[b, c, f, 2hh+ph, 2ww+pw] = y[(b,f,hh,ww), c*4 + ph*2 + pw]     (transformer3d.py:1683-1685)
__global__ void unpatchify_kernel(const bf16* __restrict__ y, bf16* __restrict__ out, int B, int C, int F, int H, int W,
                                  int ldy) {
  const int Hp = H / 2, Wp = W / 2;
  const int64_t total = (int64_t)B * C * F * Hp * Wp;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const auto [b, c, f, hh, ww] = patch_pos(idx, C, F, Hp, Wp);
  const int64_t row = (((int64_t)b * F + f) * Hp + hh) * Wp + ww;
  const uint2 v = *reinterpret_cast<const uint2*>(y + row * ldy + c * 4);
  const int64_t base = ((((int64_t)b * C + c) * F + f) * H + 2 * hh) * W + 2 * ww;
  *reinterpret_cast<uint32_t*>(out + base) = v.x;
  *reinterpret_cast<uint32_t*>(out + base + W) = v.y;
}

// pipeline_easyanimate.py:1102-1111: v = u + g*(c-u) (bf16 ops), x <- bf16(float(x) + bf16(bf16(dt) * v))
__global__ void cfg_euler_kernel(const bf16* __restrict__ pred_uncond, const bf16* __restrict__ pred_text,
                                 const bf16* __restrict__ x, bf16* __restrict__ x_out, int64_t n, float guidance,
                                 int use_cfg, float dt) {
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 2;
  if (i >= n) return;
  const float dtb = bf16_round(dt);
  float2 u = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(pred_uncond + i));
  float2 v = u;
  if (use_cfg) {
    float2 c = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(pred_text + i));
    v.x = bf16_round(u.x + bf16_round(guidance * bf16_round(c.x - u.x)));
    v.y = bf16_round(u.y + bf16_round(guidance * bf16_round(c.y - u.y)));
  }
  float2 xs = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(x + i));
  const float o0 = xs.x + bf16_round(dtb * v.x);
  const float o1 = xs.y + bf16_round(dtb * v.y);
  *reinterpret_cast<uint32_t*>(x_out + i) = pack_bf16x2(o0, o1);
}

// ---- TeaCache support (transformer3d.py:90-121,1563-1636): relative-L1 change of the block-0 modulated input and
//      the cached-residual add/sub, kept on the device (the reference round-trips both tensors through the CPU).
__global__ void __launch_bounds__(256) l1_sums_kernel(const bf16* __restrict__ cur, const bf16* __restrict__ prev,
                                                      double* __restrict__ sums, int64_t n) {
  float s_diff = 0.f, s_prev = 0.f;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 2; i < n; i += (int64_t)gridDim.x * blockDim.x * 2) {
    const float2 c = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(cur + i));
    const float2 p = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(prev + i));
    s_diff += fabsf(bf16_round(c.x - p.x)) + fabsf(bf16_round(c.y - p.y));  // torch.abs(cur - prev) on bf16 tensors
    s_prev += fabsf(p.x) + fabsf(p.y);
  }
  s_diff = warp_sum(s_diff);
  s_prev = warp_sum(s_prev);
  __shared__ float sh[2][8];
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { sh[0][w] = s_diff; sh[1][w] = s_prev; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int i = 0; i < 8; ++i) { a += sh[0][i]; b += sh[1][i]; }
    atomicAdd(&sums[0], (double)a);
    atomicAdd(&sums[1], (double)b);
  }
}
__global__ void ew_addsub_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, bf16* __restrict__ out,
                                 int64_t n, int sub) {
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 2;
  if (i >= n) return;
  const float2 x = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(a + i));
  const float2 y = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(b + i));
  *reinterpret_cast<uint32_t*>(out + i) = sub ? pack_bf16x2(x.x - y.x, x.y - y.y) : pack_bf16x2(x.x + y.x, x.y + y.y);
}
// e4m3fn (1-4-3, bias 7, no infinities, S.1111.111 = NaN) -> bf16, exact: every e4m3 value is a bf16 value.  The 256-entry
// table is rebuilt per block in shared memory (blockDim.x == 256: one entry per thread).
__device__ __forceinline__ void build_e4m3_lut(uint16_t* lut) {
  const int v = threadIdx.x;
  const int sgn = v >> 7, e = (v >> 3) & 15, m = v & 7;
  float f;
  if (e == 15 && m == 7) f = __int_as_float(0x7fc00000);
  else if (e == 0) f = ldexpf((float)m, -9);              // subnormal: m/8 * 2^-6
  else f = ldexpf(1.0f + (float)m * 0.125f, e - 7);
  f = sgn ? -f : f;
  lut[v] = __bfloat16_as_ushort(__float2bfloat16_rn(f));
}

// 16 weights: one 16-byte load, two 16-byte stores.
__device__ __forceinline__ void expand_e4m3x16(const uint16_t* lut, const uint8_t* src, bf16* dst) {
  const uint4 u = *reinterpret_cast<const uint4*>(src);
  const uint32_t uw[4] = {u.x, u.y, u.z, u.w};
  uint32_t o[8];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    o[2 * k] = lut[uw[k] & 0xff] | ((uint32_t)lut[(uw[k] >> 8) & 0xff] << 16);
    o[2 * k + 1] = lut[(uw[k] >> 16) & 0xff] | ((uint32_t)lut[uw[k] >> 24] << 16);
  }
  uint4* d = reinterpret_cast<uint4*>(dst);
  d[0] = make_uint4(o[0], o[1], o[2], o[3]);
  d[1] = make_uint4(o[4], o[5], o[6], o[7]);
}

__global__ void dequant_e4m3_kernel(const uint8_t* __restrict__ w8, bf16* __restrict__ w16, int64_t n) {
  __shared__ uint16_t lut[256];
  build_e4m3_lut(lut);
  __syncthreads();
  const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 16;
  if (i0 >= n) return;
  if (i0 + 16 <= n) {
    expand_e4m3x16(lut, w8 + i0, w16 + i0);
  } else {
    for (int64_t i = i0; i < n; ++i) w16[i] = __ushort_as_bfloat16(lut[w8[i]]);
  }
}

// A whole packed block in one launch: segment s expands n[s] weights from src + src_off[s] into dst[s].  first_vec[s] is the
// index of the segment's first 16-weight vector in the launch (prefix sums, first_vec[count] = total); a grid-stride loop
// walks the vectors and finds each one's segment by binary search in the parameter table.
struct E4m3Segments {
  const uint8_t* src;
  int64_t src_off[EA_MAX_E4M3_SEGMENTS];
  bf16* dst[EA_MAX_E4M3_SEGMENTS];
  int64_t n[EA_MAX_E4M3_SEGMENTS];
  int64_t first_vec[EA_MAX_E4M3_SEGMENTS + 1];
  int count;
};

__global__ void __launch_bounds__(256) expand_e4m3_segments_kernel(const __grid_constant__ E4m3Segments t) {
  __shared__ uint16_t lut[256];
  build_e4m3_lut(lut);
  __syncthreads();
  const int64_t total = t.first_vec[t.count];
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < total; v += (int64_t)gridDim.x * blockDim.x) {
    int lo = 0, hi = t.count - 1;  // last segment with first_vec <= v
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (t.first_vec[mid] <= v) lo = mid;
      else hi = mid - 1;
    }
    const int64_t i0 = (v - t.first_vec[lo]) * 16;
    const uint8_t* src = t.src + t.src_off[lo] + i0;
    bf16* dst = t.dst[lo] + i0;
    const int64_t left = t.n[lo] - i0;
    if (left >= 16) {
      expand_e4m3x16(lut, src, dst);
    } else {
      for (int64_t i = 0; i < left; ++i) dst[i] = __ushort_as_bfloat16(lut[src[i]]);
    }
  }
}

}  // namespace ea

using namespace ea;

#define EA_DISPATCH_NI(ni, CALL)                                                         \
  switch (ni) {                                                                          \
    case 1: CALL(1); break;   case 2: CALL(2); break;   case 3: CALL(3); break;          \
    case 4: CALL(4); break;   case 5: CALL(5); break;   case 6: CALL(6); break;          \
    case 7: CALL(7); break;   case 8: CALL(8); break;   case 9: CALL(9); break;          \
    case 10: CALL(10); break; case 11: CALL(11); break; case 12: CALL(12); break;        \
    case 13: CALL(13); break; case 14: CALL(14); break; case 15: CALL(15); break;        \
    case 16: CALL(16); break;                                                            \
    default: return fail(EA_ERR_INVALID, "feature dimension larger than 4096 is not supported"); \
  }

// The LayerNorm and RMSNorm kernels take one warp per row: 8 rows per block of 256 threads.
extern "C" int ea_layernorm_modulate(const ea_ln_args* g, void* stream) {
  EA_REQUIRE(g && g->x && g->y, "ea_layernorm_modulate: null pointer");
  EA_REQUIRE(g->rows > 0 && g->d > 0 && g->d % 8 == 0, "ea_layernorm_modulate: d must be a positive multiple of 8");
  EA_REQUIRE(g->ldx % 8 == 0 && g->ldy % 8 == 0, "ea_layernorm_modulate: row strides must be multiples of 8");
  EA_REQUIRE((g->w == nullptr) == (g->b == nullptr), "ea_layernorm_modulate: weight and bias must come together");
  EA_REQUIRE((g->pre_w == nullptr) == (g->pre_b == nullptr), "ea_layernorm_modulate: pre weight/bias must come together");
  EA_REQUIRE((g->shift == nullptr) == (g->scale == nullptr), "ea_layernorm_modulate: shift and scale must come together");
  LnArgs a{};
  a.x = (const bf16*)g->x; a.y = (bf16*)g->y; a.rows = g->rows; a.d = (int)g->d;
  a.ldx = g->ldx; a.ldy = g->ldy;
  a.rows_per_batch = (int)(g->rows_per_batch > 0 ? g->rows_per_batch : g->rows);
  a.pre_w = (const bf16*)g->pre_w; a.pre_b = (const bf16*)g->pre_b; a.pre_eps = g->pre_eps;
  a.w = (const bf16*)g->w; a.b = (const bf16*)g->b; a.eps = g->eps;
  a.shift = (const bf16*)g->shift; a.scale = (const bf16*)g->scale; a.mod_stride = g->mod_stride;
  const int ni = (int)((g->d + 255) / 256);
#define CALL(n) return launch(ln_modulate_kernel<n>, grid_1d(a.rows, 8), 256, 0, stream, "ln_modulate_kernel", a)
  EA_DISPATCH_NI(ni, CALL)
#undef CALL
}

extern "C" int ea_rmsnorm(const ea_rmsnorm_args* g, void* stream) {
  EA_REQUIRE(g && g->x && g->y && g->w, "ea_rmsnorm: null pointer");
  EA_REQUIRE(g->rows > 0 && g->d > 0 && g->d % 8 == 0, "ea_rmsnorm: d must be a positive multiple of 8");
  RmsArgs a{(const bf16*)g->x, (bf16*)g->y, (const bf16*)g->w, g->rows, (int)g->d, g->eps};
  const int ni = (int)((g->d + 255) / 256);
#define CALL(n) return launch(rmsnorm_kernel<n>, grid_1d(a.rows, 8), 256, 0, stream, "rmsnorm_kernel", a)
  EA_DISPATCH_NI(ni, CALL)
#undef CALL
}

extern "C" int ea_timestep_embedding(const void* t, void* out, int64_t B, int64_t dim, float freq_shift,
                                     int32_t flip_sin_to_cos, void* stream) {
  EA_REQUIRE(t && out && B > 0 && dim > 0 && dim % 2 == 0, "ea_timestep_embedding: bad arguments");
  const int n = (int)(B * dim / 2);
  return launch(timestep_embedding_kernel, grid_1d(n, 256), 256, 0, stream, "timestep_embedding_kernel", (const bf16*)t,
                (bf16*)out, (int)B, (int)dim, freq_shift, flip_sin_to_cos);
}

extern "C" int ea_skinny_linear(const ea_skinny_linear_args* g, void* stream) {
  EA_REQUIRE(g && g->x && g->w && g->out, "ea_skinny_linear: null pointer");
  EA_REQUIRE(g->M >= 1 && g->M <= 8, "ea_skinny_linear: M must be in [1,8]");
  EA_REQUIRE(g->K > 0 && g->K % 8 == 0 && g->N > 0, "ea_skinny_linear: K must be a positive multiple of 8");
  const size_t smem = (size_t)g->M * g->K * sizeof(float);
  EA_REQUIRE(smem <= 96 * 1024, "ea_skinny_linear: M*K too large for the shared-memory input stage");
  static PerDeviceFlag smem_done;
  const int rc = set_max_dynamic_smem(reinterpret_cast<const void*>(skinny_linear_kernel<8>), 96 * 1024, smem_done,
                                      "skinny_linear_kernel");
  if (rc) return rc;
  // one warp per output column, 8 per block
  return launch(skinny_linear_kernel<8>, grid_1d(g->N, 8), 256, smem, stream, "skinny_linear_kernel", (const bf16*)g->x,
                (const bf16*)g->w, (const bf16*)g->bias, (bf16*)g->out, (int)g->M, (int)g->N, (int)g->K, g->act_in,
                g->act_out);
}

extern "C" int ea_patchify(const void* x, const void* x2, void* a, int64_t B, int64_t C1, int64_t C2, int64_t F,
                           int64_t H, int64_t W, int64_t ldk, void* stream) {
  EA_REQUIRE(x && a, "ea_patchify: null pointer");
  EA_REQUIRE(C2 == 0 || x2 != nullptr, "ea_patchify: second source missing");
  EA_REQUIRE(H % 2 == 0 && W % 2 == 0, "ea_patchify: H and W must be even (patch size 2)");
  EA_REQUIRE(ldk >= 4 * (C1 + C2) && ldk % 8 == 0, "ea_patchify: ldk must be a multiple of 8 and >= 4*C");
  const int64_t rows = B * F * (H / 2) * (W / 2);
  int rc = launch(patchify_kernel, grid_1d(rows * (C1 + C2), 256), 256, 0, stream, "patchify_kernel", (const bf16*)x,
                  (const bf16*)x2, (bf16*)a, (int)B, (int)C1, (int)C2, (int)F, (int)H, (int)W, (int)ldk);
  const int kvalid = (int)(4 * (C1 + C2));
  if (rc == EA_OK && ldk > kvalid)
    rc = launch(patchify_pad_kernel, grid_1d(rows * (ldk - kvalid), 256), 256, 0, stream, "patchify_pad_kernel", (bf16*)a,
                rows, kvalid, (int)ldk);
  return rc;
}

extern "C" int ea_unpatchify(const void* y, void* out, int64_t B, int64_t C, int64_t F, int64_t H, int64_t W,
                             int64_t ldy, void* stream) {
  EA_REQUIRE(y && out, "ea_unpatchify: null pointer");
  EA_REQUIRE(H % 2 == 0 && W % 2 == 0 && ldy >= 4 * C && ldy % 4 == 0, "ea_unpatchify: bad shape");
  return launch(unpatchify_kernel, grid_1d(B * C * F * (H / 2) * (W / 2), 256), 256, 0, stream, "unpatchify_kernel",
                (const bf16*)y, (bf16*)out, (int)B, (int)C, (int)F, (int)H, (int)W, (int)ldy);
}

extern "C" int ea_cfg_euler_step(const void* pred_uncond, const void* pred_text, const void* x, void* x_out, int64_t n,
                                 float guidance_scale, int32_t use_cfg, float sigma, float sigma_next, void* stream) {
  EA_REQUIRE(pred_uncond && x && x_out, "ea_cfg_euler_step: null pointer");
  EA_REQUIRE(!use_cfg || pred_text, "ea_cfg_euler_step: CFG needs the text-conditioned prediction");
  EA_REQUIRE(n > 0 && n % 2 == 0, "ea_cfg_euler_step: element count must be even");
  const float dt = sigma_next - sigma;  // fp32 subtraction of fp32 sigmas, as the scheduler does
  return launch(cfg_euler_kernel, grid_1d(n / 2, 256), 256, 0, stream, "cfg_euler_kernel", (const bf16*)pred_uncond,
                (const bf16*)pred_text, (const bf16*)x, (bf16*)x_out, n, guidance_scale, use_cfg, dt);
}

extern "C" int ea_dequant_e4m3(const void* w8, void* w16, int64_t n, void* stream) {
  EA_REQUIRE(w8 && w16 && n > 0, "ea_dequant_e4m3: bad arguments");
  EA_REQUIRE((reinterpret_cast<uintptr_t>(w8) & 15) == 0 && (reinterpret_cast<uintptr_t>(w16) & 15) == 0,
             "ea_dequant_e4m3: pointers must be 16-byte aligned");
  return launch(dequant_e4m3_kernel, grid_1d((n + 15) / 16, 256), 256, 0, stream, "dequant_e4m3_kernel",
                (const uint8_t*)w8, (bf16*)w16, n);
}

extern "C" int ea_expand_e4m3_segments(const void* src, const int64_t* src_offsets, void* const* dsts, const int64_t* counts,
                                       int32_t n_segs, void* stream) {
  EA_REQUIRE(src && src_offsets && dsts && counts, "ea_expand_e4m3_segments: null pointer");
  EA_REQUIRE(n_segs > 0 && n_segs <= EA_MAX_E4M3_SEGMENTS, "ea_expand_e4m3_segments: 1 to EA_MAX_E4M3_SEGMENTS segments");
  EA_REQUIRE((reinterpret_cast<uintptr_t>(src) & 15) == 0, "ea_expand_e4m3_segments: src must be 16-byte aligned");
  E4m3Segments t{};
  t.src = (const uint8_t*)src;
  t.count = n_segs;
  int64_t vecs = 0;
  for (int s = 0; s < n_segs; ++s) {
    EA_REQUIRE(dsts[s] && counts[s] > 0 && src_offsets[s] >= 0, "ea_expand_e4m3_segments: bad segment");
    EA_REQUIRE(src_offsets[s] % 16 == 0 && (reinterpret_cast<uintptr_t>(dsts[s]) & 15) == 0,
               "ea_expand_e4m3_segments: segment offsets and destinations must be 16-byte aligned");
    t.src_off[s] = src_offsets[s];
    t.dst[s] = (bf16*)dsts[s];
    t.n[s] = counts[s];
    t.first_vec[s] = vecs;
    vecs += (counts[s] + 15) / 16;
  }
  t.first_vec[n_segs] = vecs;
  const unsigned blocks = std::min(grid_1d(vecs, 256), 8u * sm_count());
  return launch(expand_e4m3_segments_kernel, blocks, 256, 0, stream, "expand_e4m3_segments_kernel", t);
}

extern "C" int ea_l1_sums(const void* cur, const void* prev, void* sums, int64_t n, void* stream) {
  EA_REQUIRE(cur && prev && sums && n > 0 && n % 2 == 0, "ea_l1_sums: bad arguments");
  const cudaError_t e = cudaMemsetAsync(sums, 0, 2 * sizeof(double), static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail(EA_ERR_CUDA, std::string("cudaMemsetAsync(l1_sums_kernel): ") + cudaGetErrorString(e));
  const unsigned blocks = std::min(grid_1d(n / 2, 256), 4u * sm_count());
  return launch(l1_sums_kernel, blocks, 256, 0, stream, "l1_sums_kernel", (const bf16*)cur, (const bf16*)prev,
                (double*)sums, n);
}

extern "C" int ea_ew_addsub(const void* a, const void* b, void* out, int64_t n, int32_t subtract, void* stream) {
  EA_REQUIRE(a && b && out && n > 0 && n % 2 == 0, "ea_ew_addsub: bad arguments");
  return launch(ew_addsub_kernel, grid_1d(n / 2, 256), 256, 0, stream, "ew_addsub_kernel", (const bf16*)a, (const bf16*)b,
                (bf16*)out, n, subtract);
}

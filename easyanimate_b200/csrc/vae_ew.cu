// HBM-bound kernels of the MagViT VAE decode: latent preparation (post_quant_conv + layout change), per-frame
// GroupNorm statistics / apply(+SiLU), nearest spatial up-sampling, row softmax and transpose for the mid-block
// attention, tile blending and the final clamp.  Channels-last [T,H,W,C] bf16 activations, 16-byte vector accesses.
#include <stdlib.h>

#include "common.cuh"
#include "host.h"
#include "../../include/ea_b200.h"

namespace ea {

// z[b][c][t][h][w] (planar, C channels) -> y[t][h][w][Cpad] = bf16(W z + bias) for c < C, 0 above.
// autoencoder_magvit.py:281 post_quant_conv (1x1x1 Conv3d) fused with the NCTHW -> THWC transposition.
__global__ void vae_prepare_latents_kernel(const bf16* __restrict__ z, const bf16* __restrict__ w,
                                           const bf16* __restrict__ bias, bf16* __restrict__ y, int C, int Cpad,
                                           int64_t thw, int64_t z_c_stride, float in_scale) {
  extern __shared__ float sw[];  // [C*C] weights + [C] bias
  for (int i = threadIdx.x; i < C * C; i += blockDim.x) sw[i] = __bfloat162float(w[i]);
  for (int i = threadIdx.x; i < C; i += blockDim.x) sw[C * C + i] = __bfloat162float(bias[i]);
  __syncthreads();
  const int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= thw) return;
  float in[32];
  // in_scale: decode_latents' `1 / scaling_factor * latents` (pipeline_easyanimate.py:724), a bf16 tensor op of its own in
  // the reference, hence one bf16 rounding before the 1x1x1 convolution (exact when in_scale == 1)
  for (int c = 0; c < C; ++c) in[c] = bf16_round(__bfloat162float(z[c * z_c_stride + pix]) * in_scale);
  bf16* o = y + pix * Cpad;
  for (int co = 0; co < Cpad; co += 2) {
    float a0 = 0.f, a1 = 0.f;
    if (co < C) {
      a0 = sw[C * C + co];
      for (int c = 0; c < C; ++c) a0 += sw[co * C + c] * in[c];
    }
    if (co + 1 < C) {
      a1 = sw[C * C + co + 1];
      for (int c = 0; c < C; ++c) a1 += sw[(co + 1) * C + c] * in[c];
    }
    *reinterpret_cast<uint32_t*>(o + co) = pack_bf16x2(a0, a1);
  }
}

// ---- GroupNorm: per-frame statistics (common.py:301-305 rearranges '(b t) c h w' so every frame has its own) ----
// Deterministic (no atomics: a decode must be reproducible bit for bit, tests/test_vae_gpu.py) AND independent of how the rows
// of a frame are split over GPUs (strip-parallel decode, vae_strips.py): the unit of work is ONE IMAGE ROW.  A block reduces
// one row of one frame - every thread sums a fixed pixel subset of one 8-channel vector in fp32, the block adds the threads
// in a fixed order in fp64 - to a (sum, sum of squares) pair per group, which depends on the row's content and (W, C) only.
// Rows are then added in fp64: a different association (rows of a strip first, then the strips) moves the sums by ~1e-16
// relative, which disappears in the conversion of mean / rstd to fp32 except when a sum sits within that distance of an fp32
// rounding boundary (~1e-9 per statistic) - the statistics of a strip-parallel decode are the single-GPU ones.
__global__ void __launch_bounds__(256) gn_row_partial_kernel(const bf16* __restrict__ x, double* __restrict__ part, int rows,
                                                             int W, int C, int G) {
  extern __shared__ float red[];  // [2][pstride][C]
  const int t = blockIdx.y, r = blockIdx.x;
  const int nvec = C >> 3;
  const int cv = threadIdx.x % nvec;
  const int prow = threadIdx.x / nvec;
  const int pstride = blockDim.x / nvec;
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  const bf16* base = x + ((int64_t)t * rows + r) * W * C + cv * 8;
  auto accumulate = [&](const uint4& u) {
    const uint32_t uw[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16x2(uw[k]);
      s[2 * k] += f.x; q[2 * k] += f.x * f.x;
      s[2 * k + 1] += f.y; q[2 * k + 1] += f.y * f.y;
    }
  };
  // four 16-byte loads in flight per thread (the first version of this pass ran at 1.7 TB/s with one)
  int p = prow;
  for (; p + 3 * pstride < W; p += 4 * pstride) {
    uint4 u[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) u[i] = __ldg(reinterpret_cast<const uint4*>(base + (int64_t)(p + i * pstride) * C));
#pragma unroll
    for (int i = 0; i < 4; ++i) accumulate(u[i]);
  }
  for (; p < W; p += pstride) accumulate(__ldg(reinterpret_cast<const uint4*>(base + (int64_t)p * C)));
  float* rs = red + (size_t)prow * C + cv * 8;
  float* rq = red + (size_t)(pstride + prow) * C + cv * 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    rs[j] = s[j];
    rq[j] = q[j];
  }
  __syncthreads();
  const int cpg = C / G;
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    double a = 0.0, b = 0.0;
    for (int c = 0; c < cpg; ++c)
      for (int pr = 0; pr < pstride; ++pr) {
        a += (double)red[(size_t)pr * C + g * cpg + c];
        b += (double)red[(size_t)(pstride + pr) * C + g * cpg + c];
      }
    double* dst = part + (((int64_t)t * rows + r) * G + g) * 2;
    dst[0] = a;
    dst[1] = b;
  }
}
// One warp per (frame, group): lane l adds rows l, l + 32, ... in order, the lanes are combined by a fixed shuffle tree.
EA_DEVICE void gn_rows_sum(const double* __restrict__ part, int i, int G, int rows, double& a, double& b) {
  const int t = i / G, g = i % G, lane = threadIdx.x & 31;
  a = 0.0;
  b = 0.0;
  for (int r = lane; r < rows; r += 32) {
    const double* src = part + (((int64_t)t * rows + r) * G + g) * 2;
    a += src[0];
    b += src[1];
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, off);
    b += __shfl_xor_sync(0xffffffffu, b, off);
  }
}
// (mean, rstd) of group i from its fp64 (sum, sum of squares) over `count` elements
EA_DEVICE void gn_store_stats(float* __restrict__ stats, int i, double a, double b, double count, float eps) {
  const double mean = a / count;
  double var = b / count - mean * mean;
  var = var < 0 ? 0 : var;
  stats[2 * i] = (float)mean;
  stats[2 * i + 1] = (float)(1.0 / sqrt(var + (double)eps));
}
__global__ void gn_finalize_kernel(const double* __restrict__ part, float* __restrict__ stats, int n, int G, int rows,
                                   double count, float eps) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // (frame, group)
  if (i >= n) return;
  double a, b;
  gn_rows_sum(part, i, G, rows, a, b);
  if ((threadIdx.x & 31) == 0) gn_store_stats(stats, i, a, b, count, eps);
}
// Strip-parallel decode: the rows of ONE rank reduced to a (sum, sum of squares) pair per (frame, group) ...
__global__ void gn_sums_kernel(const double* __restrict__ part, double* __restrict__ sums, int n, int G, int rows) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n) return;
  double a, b;
  gn_rows_sum(part, i, G, rows, a, b);
  if ((threadIdx.x & 31) != 0) return;
  sums[2 * i] = a;
  sums[2 * i + 1] = b;
}
// ... and the statistics from the gathered pairs of all `parts` ranks, added in rank order (identical on every rank)
__global__ void gn_finalize_parts_kernel(const double* __restrict__ sums, float* __restrict__ stats, int n, int parts,
                                         double count, float eps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double a = 0.0, b = 0.0;
  for (int r = 0; r < parts; ++r) {
    a += sums[((int64_t)r * n + i) * 2];
    b += sums[((int64_t)r * n + i) * 2 + 1];
  }
  gn_store_stats(stats, i, a, b, count, eps);
}
// y = [silu](bf16((x - mean) * rstd * gamma + beta)); one 8-channel vector per thread
__global__ void gn_apply_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, const bf16* __restrict__ gamma,
                                const bf16* __restrict__ beta, const float* __restrict__ stats, int64_t HW, int C, int G,
                                int64_t total_vec, int do_silu) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total_vec) return;
  const int nvec = C >> 3;
  const int cv = (int)(idx % nvec);
  const int64_t pix = idx / nvec;
  const int t = (int)(pix / HW);
  const int cpg = C / G;
  const uint4 u = *reinterpret_cast<const uint4*>(x + idx * 8);
  const uint4 gw = __ldg(reinterpret_cast<const uint4*>(gamma) + cv);
  const uint4 bw = __ldg(reinterpret_cast<const uint4*>(beta) + cv);
  const uint32_t uw[4] = {u.x, u.y, u.z, u.w}, gg[4] = {gw.x, gw.y, gw.z, gw.w}, bb[4] = {bw.x, bw.y, bw.z, bw.w};
  uint32_t o[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = cv * 8 + 2 * k;
    const int g0 = c / cpg, g1 = (c + 1) / cpg;
    const float2 st0 = *reinterpret_cast<const float2*>(stats + ((int64_t)t * G + g0) * 2);
    const float2 st1 = *reinterpret_cast<const float2*>(stats + ((int64_t)t * G + g1) * 2);
    const float2 xf = unpack_bf16x2(uw[k]), gf = unpack_bf16x2(gg[k]), bf = unpack_bf16x2(bb[k]);
    float v0 = bf16_round((xf.x - st0.x) * st0.y * gf.x + bf.x);
    float v1 = bf16_round((xf.y - st1.x) * st1.y * gf.y + bf.y);
    if (do_silu) {
      v0 = v0 / (1.0f + expf(-v0));
      v1 = v1 / (1.0f + expf(-v1));
    }
    o[k] = pack_bf16x2(v0, v1);
  }
  *reinterpret_cast<uint4*>(y + idx * 8) = make_uint4(o[0], o[1], o[2], o[3]);
}

// Restructured for bandwidth: a block walks a pixel range of ONE frame, a thread keeps one 8-channel vector position, so the
// per-channel affine form of the normalisation sits in registers for the whole range - a = rstd * gamma, b = beta - a * mean,
// y = a * x + b in fp32, which is how PyTorch's own GroupNorm kernels (CPU and CUDA) evaluate it, one FFMA per element instead
// of three operations; four 16-byte loads in flight per thread; SiLU through ex2.approx / rcp.approx (relative error 2^-21,
// far below the bf16 rounding that follows).  The pass is instruction-bound, not HBM-bound: ~10 instructions per element.
__global__ void __launch_bounds__(256) gn_apply2_kernel(const bf16* __restrict__ x, bf16* __restrict__ y,
                                                        const bf16* __restrict__ gamma, const bf16* __restrict__ beta,
                                                        const float* __restrict__ stats, int64_t HW, int C, int G,
                                                        int pix_per_block, int do_silu) {
  const int t = blockIdx.y;
  const int nvec = C >> 3;
  const int cv = threadIdx.x % nvec;
  const int prow = threadIdx.x / nvec;
  const int pstride = blockDim.x / nvec;
  const int cpg = C / G;
  float ga[8], gb[8];
  {
    const uint4 gw = __ldg(reinterpret_cast<const uint4*>(gamma) + cv);
    const uint4 bw = __ldg(reinterpret_cast<const uint4*>(beta) + cv);
    const uint32_t gg[4] = {gw.x, gw.y, gw.z, gw.w}, bb[4] = {bw.x, bw.y, bw.z, bw.w};
    float gm[8], bt[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 gf = unpack_bf16x2(gg[k]), bf = unpack_bf16x2(bb[k]);
      gm[2 * k] = gf.x; gm[2 * k + 1] = gf.y;
      bt[2 * k] = bf.x; bt[2 * k + 1] = bf.y;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 st = __ldg(reinterpret_cast<const float2*>(stats + ((int64_t)t * G + (cv * 8 + j) / cpg) * 2));
      ga[j] = st.y * gm[j];
      gb[j] = fmaf(-ga[j], st.x, bt[j]);
    }
  }
  const int64_t p0 = (int64_t)blockIdx.x * pix_per_block;
  const int64_t p1 = p0 + pix_per_block < HW ? p0 + pix_per_block : HW;
  const bf16* xb = x + (int64_t)t * HW * C + cv * 8;
  bf16* yb = y + (int64_t)t * HW * C + cv * 8;
  auto apply = [&](const uint4& u) {
    const uint32_t uw[4] = {u.x, u.y, u.z, u.w};
    uint32_t o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 xf = unpack_bf16x2(uw[k]);
      float v0 = bf16_round(fmaf(ga[2 * k], xf.x, gb[2 * k]));
      float v1 = bf16_round(fmaf(ga[2 * k + 1], xf.y, gb[2 * k + 1]));
      if (do_silu) {
        v0 = __fdividef(v0, 1.0f + __expf(-v0));
        v1 = __fdividef(v1, 1.0f + __expf(-v1));
      }
      o[k] = pack_bf16x2(v0, v1);
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
  };
  int64_t p = p0 + prow;
  for (; p + 3 * (int64_t)pstride < p1; p += 4 * (int64_t)pstride) {
    uint4 u[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) u[i] = __ldg(reinterpret_cast<const uint4*>(xb + (p + (int64_t)i * pstride) * C));
#pragma unroll
    for (int i = 0; i < 4; ++i) *reinterpret_cast<uint4*>(yb + (p + (int64_t)i * pstride) * C) = apply(u[i]);
  }
  for (; p < p1; p += pstride) *reinterpret_cast<uint4*>(yb + p * C) = apply(__ldg(reinterpret_cast<const uint4*>(xb + p * C)));
}

// nearest x2 in H and W (upsamplers.py:35,143): y[t][2h+a][2w+b][c] = x[t][h][w][c]
__global__ void upsample2x_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int64_t T, int H, int W, int C) {
  const int nvec = C >> 3;
  const int64_t total = T * (int64_t)(2 * H) * (2 * W) * nvec;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cv = (int)(idx % nvec);
  int64_t r = idx / nvec;
  const int wo = (int)(r % (2 * W)); r /= (2 * W);
  const int ho = (int)(r % (2 * H));
  const int64_t t = r / (2 * H);
  const uint4 v = *reinterpret_cast<const uint4*>(x + (((t * H + (ho >> 1)) * W + (wo >> 1)) * C) + cv * 8);
  *reinterpret_cast<uint4*>(y + idx * 8) = v;
}

// P[r][:] = bf16(softmax(S[r][:])) for fp32 scores (already scaled); one CTA per row
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ s, bf16* __restrict__ p, int N,
                                                           int64_t lds, int64_t ldp) {
  __shared__ float red[32];
  const float* row = s + (int64_t)blockIdx.x * lds;
  bf16* out = p + (int64_t)blockIdx.x * ldp;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < N; i += blockDim.x) mx = fmaxf(mx, row[i]);
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x; i < N; i += blockDim.x) sum += expf(row[i] - mx);
  sum = warp_sum(sum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) sum += red[i];
  const float inv = 1.0f / sum;
  for (int i = threadIdx.x; i < N; i += blockDim.x) out[i] = __float2bfloat16_rn(expf(row[i] - mx) * inv);
}

// out[c][r] = in[r][c]
__global__ void transpose2d_kernel(const bf16* __restrict__ in, bf16* __restrict__ out, int R, int Cc, int64_t ldi,
                                   int64_t ldo) {
  __shared__ bf16 tile[32][34];
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < R && c < Cc) ? in[(int64_t)r * ldi + c] : __float2bfloat16_rn(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (c < Cc && r < R) out[(int64_t)c * ldo + r] = tile[threadIdx.x][i];
  }
}

// idx -> (plane, row, col) of a planes x rows x cols index space, col fastest
struct PlanarPos {
  int pl, r, c;
};
EA_DEVICE PlanarPos planar_pos(int64_t idx, int rows, int cols) {
  const int c = (int)(idx % cols);
  const int r = (int)((idx / cols) % rows);
  return {(int)(idx / ((int64_t)cols * rows)), r, c};
}

// dst[..., y0+i, x0+j] blended in place with src tile: dst = src*(1-wgt) + dst*wgt  (blend_v / blend_h,
// autoencoder_magvit.py:319-337), planar [C*T][H][W] images. axis 0: ramp along rows, 1: along columns.
__global__ void blend_kernel(const bf16* __restrict__ a, int64_t a_plane, int a_ld, int a_off_r, int a_off_c,
                             bf16* __restrict__ b, int64_t b_plane, int b_ld, int planes, int rows, int cols, int extent,
                             int axis) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)planes * rows * cols) return;
  const auto [pl, r, c] = planar_pos(idx, rows, cols);
  const int k = axis == 0 ? r : c;
  // python: b = a * (1 - k/extent) + b * (k/extent): python-float weights enter the bf16 ops at fp32 precision
  const float wb = (float)((double)k / (double)extent);
  const float wa = (float)(1.0 - (double)k / (double)extent);
  const float av = __bfloat162float(a[pl * a_plane + (int64_t)(a_off_r + r) * a_ld + a_off_c + c]);
  bf16* bp = b + pl * b_plane + (int64_t)r * b_ld + c;
  const float bv = __bfloat162float(*bp);
  const float t0 = bf16_round(av * wa), t1 = bf16_round(bv * wb);
  *bp = __float2bfloat16_rn(t0 + t1);
}

// strided 2-D copy of planar images (crop + concatenate of decoded tiles)
__global__ void copy2d_kernel(const bf16* __restrict__ src, int64_t s_plane, int s_ld, bf16* __restrict__ dst,
                              int64_t d_plane, int d_ld, int planes, int rows, int cols) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)planes * rows * cols) return;
  const auto [pl, r, c] = planar_pos(idx, rows, cols);
  dst[pl * d_plane + (int64_t)r * d_ld + c] = src[pl * s_plane + (int64_t)r * s_ld + c];
}

// lower-right corner re-blend (autoencoder_magvit.py:429-443): dst = w*src + (1-w)*dst, w = min(wx[c], wy[r]).
// wx / wy are the reference's torch.linspace(0, 1, N) fp32 weights, built by the caller (no closed form here reproduces
// torch's linspace for every N).  The reference combines fp32 tensors op by op, each product and sum rounded on its own:
// the _rn intrinsics keep nvcc from contracting them into an FMA.  bf16 on store (the assignment into the bf16 video).
__global__ void corner_blend_kernel(const bf16* __restrict__ src, bf16* __restrict__ dst, int64_t d_plane, int d_ld,
                                    int planes, int Hc, int Wc, const float* __restrict__ wx, const float* __restrict__ wy) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)planes * Hc * Wc) return;
  const auto [pl, r, c] = planar_pos(idx, Hc, Wc);
  const float wgt = fminf(__ldg(wx + c), __ldg(wy + r));
  const float s = __bfloat162float(src[(int64_t)pl * Hc * Wc + (int64_t)r * Wc + c]);
  bf16* dp = dst + pl * d_plane + (int64_t)r * d_ld + c;
  const float d = __bfloat162float(*dp);
  *dp = __float2bfloat16_rn(__fadd_rn(__fmul_rn(wgt, s), __fmul_rn(__fsub_rn(1.0f, wgt), d)));
}

// decode_latents' tail (pipeline_easyanimate.py:729,738-740) on one decoded value: clamp(-1,1) -> /2 + 0.5 (two bf16 ops)
// -> clamp(0,1), as float32 (what `.cpu().float().numpy()` yields).
__device__ __forceinline__ float frame_value(float v) {
  float a = fminf(fmaxf(v, -1.0f), 1.0f);     // video.clamp(-1, 1)      (NaN propagates like torch.clamp)
  a = v != v ? v : a;
  a = bf16_round(bf16_round(a * 0.5f) + 0.5f);  // video / 2 + 0.5        (bf16 tensor ops)
  const float c = fminf(fmaxf(a, 0.0f), 1.0f);  // .clamp(0, 1)
  return a != a ? a : c;
}

// frame_value as float32 or uint8 = trunc(255 * v) (utils.py:57 `(x * 255).numpy().astype(np.uint8)`).
// `out` may be device memory or device-mapped pinned host memory: 8 elements per thread, 32 B (16 B) contiguous stores.
template <typename OutT>
__global__ void frames_out_kernel(const bf16* __restrict__ x, OutT* __restrict__ out, int64_t n) {
  const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (i0 >= n) return;
  float v[8];
  if (i0 + 8 <= n) {
    unpack_bf16x8(*reinterpret_cast<const uint4*>(x + i0), v);
  } else {
    for (int k = 0; k < 8; ++k) v[k] = i0 + k < n ? __bfloat162float(x[i0 + k]) : 0.f;
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] = frame_value(v[k]);
  if constexpr (sizeof(OutT) == 4) {
    if (i0 + 8 <= n) {
      *reinterpret_cast<float4*>(out + i0) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(out + i0 + 4) = make_float4(v[4], v[5], v[6], v[7]);
    } else {
      for (int k = 0; k < 8 && i0 + k < n; ++k) out[i0 + k] = (OutT)v[k];
    }
  } else {
    uint8_t b[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) b[k] = (uint8_t)(int)(v[k] * 255.0f);
    if (i0 + 8 <= n) {
      uint2 w;
      w.x = b[0] | (b[1] << 8) | (b[2] << 16) | ((uint32_t)b[3] << 24);
      w.y = b[4] | (b[5] << 8) | (b[6] << 16) | ((uint32_t)b[7] << 24);
      *reinterpret_cast<uint2*>(out + i0) = w;
    } else {
      for (int k = 0; k < 8 && i0 + k < n; ++k) out[i0 + k] = (OutT)b[k];
    }
  }
}

// The long-video cross-fade (ui.py:524-531) fused with frames_out: x [planes, frames, frame_elems] bf16 is one decoded
// window; frame t of plane p goes to dst + p * dst_plane + t * frame_elems.  The first `ov` frames are blended into what dst
// holds, dst = dst * (1 - r_t) + f * r_t with r_t = float32(t / ov), every product and sum rounded on its own like torch's
// float32 tensor ops (the _rn intrinsics keep nvcc from contracting them into an FMA); the other frames are stored as they are.
// One row (plane, frame) per blockIdx.y.
__global__ void frames_out_blend_kernel(const bf16* __restrict__ x, float* dst, int64_t frames, int64_t frame_elems,
                                        int64_t dst_plane, int ov) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= frame_elems) return;
  const int64_t row = blockIdx.y, p = row / frames, t = row % frames;
  const float f = frame_value(__bfloat162float(x[row * frame_elems + e]));
  float* d = dst + p * dst_plane + t * frame_elems + e;
  if (t < ov) {
    const float r = (float)((double)t / (double)ov);  // np.float32(float(t) / float(ov))
    *d = __fadd_rn(__fmul_rn(*d, __fsub_rn(1.0f, r)), __fmul_rn(f, r));
  } else {
    *d = f;
  }
}

}  // namespace ea

using namespace ea;

extern "C" int ea_frames_out(const void* x, void* out, int64_t n, int32_t out_kind, void* stream) {
  EA_REQUIRE(x && out && n > 0, "ea_frames_out: bad arguments");
  EA_REQUIRE(out_kind == EA_FRAMES_F32 || out_kind == EA_FRAMES_U8, "ea_frames_out: out_kind must be EA_FRAMES_F32 or EA_FRAMES_U8");
  EA_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
             "ea_frames_out: pointers must be 16-byte aligned");
  const unsigned blocks = grid_1d((n + 7) / 8, 256);
  if (out_kind == EA_FRAMES_F32)
    return launch(frames_out_kernel<float>, blocks, 256, 0, stream, "frames_out_kernel", (const bf16*)x, (float*)out, n);
  return launch(frames_out_kernel<uint8_t>, blocks, 256, 0, stream, "frames_out_kernel", (const bf16*)x, (uint8_t*)out, n);
}

extern "C" int ea_frames_out_blend(const void* x, void* dst, int64_t planes, int64_t frames, int64_t frame_elems,
                                   int64_t dst_plane, int32_t ov, void* stream) {
  EA_REQUIRE(x && dst && planes > 0 && frames > 0 && frame_elems > 0, "ea_frames_out_blend: bad arguments");
  EA_REQUIRE(planes * frames <= 65535, "ea_frames_out_blend: planes * frames must be <= 65535");
  EA_REQUIRE(ov >= 0 && ov <= frames, "ea_frames_out_blend: need 0 <= ov <= frames");
  EA_REQUIRE(dst_plane >= frames * frame_elems, "ea_frames_out_blend: dst_plane must hold the window's frames");
  const dim3 grid(grid_1d(frame_elems, 256), (unsigned)(planes * frames));
  return launch(frames_out_blend_kernel, grid, 256, 0, stream, "frames_out_blend_kernel", (const bf16*)x, (float*)dst, frames,
                frame_elems, dst_plane, (int)ov);
}

extern "C" int ea_vae_prepare_latents(const void* z, const void* w, const void* bias, void* y, int64_t C, int64_t Cpad,
                                      int64_t T, int64_t H, int64_t W, float in_scale, void* stream) {
  EA_REQUIRE(z && w && bias && y, "ea_vae_prepare_latents: null pointer");
  EA_REQUIRE(C > 0 && C <= 32 && Cpad >= C && Cpad % 8 == 0, "ea_vae_prepare_latents: need C <= 32, Cpad % 8 == 0");
  const int64_t thw = T * H * W;
  const size_t smem = (size_t)(C * C + C) * sizeof(float);
  return launch(vae_prepare_latents_kernel, grid_1d(thw, 128), 128, smem, stream, "vae_prepare_latents_kernel",
                (const bf16*)z, (const bf16*)w, (const bf16*)bias, (bf16*)y, (int)C, (int)Cpad, thw, thw, in_scale);
}

extern "C" size_t ea_groupnorm_workspace(int64_t frames, int64_t rows, int64_t groups) {
  return (size_t)frames * rows * groups * 2 * sizeof(double);
}

static int gn_row_partials(const char* who, const void* x, void* workspace, size_t workspace_bytes, int64_t frames, int64_t rows,
                           int64_t W, int64_t C, int64_t groups, void* stream) {
  if (!(C % 8 == 0 && C % groups == 0 && C <= 2048 && 256 % (C / 8) == 0))
    return fail(EA_ERR_INVALID, std::string(who) + ": C must be a multiple of 8 dividing into 256 threads, and of groups");
  if (workspace_bytes < ea_groupnorm_workspace(frames, rows, groups)) return fail(EA_ERR_WORKSPACE, std::string(who) + ": workspace too small");
  if (!(frames > 0 && rows > 0 && W > 0 && frames <= 65535 && rows < (1ll << 31) && W < (1ll << 24)))
    return fail(EA_ERR_INVALID, std::string(who) + ": bad frame / row / width count");
  const size_t smem = 2 * (size_t)(256 / (C / 8)) * C * sizeof(float);  // 16 KB
  return launch(gn_row_partial_kernel, dim3((unsigned)rows, (unsigned)frames), 256, smem, stream, "gn_row_partial_kernel",
                (const bf16*)x, (double*)workspace, (int)rows, (int)W, (int)C, (int)groups);
}

// The reductions over the row partials take one warp per (frame, group), four per block.
extern "C" int ea_groupnorm_stats(const void* x, void* stats, void* workspace, size_t workspace_bytes, int64_t frames,
                                  int64_t rows, int64_t W, int64_t C, int64_t groups, float eps, void* stream) {
  EA_REQUIRE(x && stats && workspace, "ea_groupnorm_stats: null pointer");
  const int rc = gn_row_partials("ea_groupnorm_stats", x, workspace, workspace_bytes, frames, rows, W, C, groups, stream);
  if (rc) return rc;
  const int n = (int)(frames * groups);
  return launch(gn_finalize_kernel, grid_1d(n * 32, 128), 128, 0, stream, "gn_finalize_kernel", (const double*)workspace,
                (float*)stats, n, (int)groups, (int)rows, (double)rows * (double)W * (double)(C / groups), eps);
}

extern "C" int ea_groupnorm_sums(const void* x, void* sums, void* workspace, size_t workspace_bytes, int64_t frames,
                                 int64_t rows, int64_t W, int64_t C, int64_t groups, void* stream) {
  EA_REQUIRE(x && sums && workspace, "ea_groupnorm_sums: null pointer");
  const int rc = gn_row_partials("ea_groupnorm_sums", x, workspace, workspace_bytes, frames, rows, W, C, groups, stream);
  if (rc) return rc;
  const int n = (int)(frames * groups);
  return launch(gn_sums_kernel, grid_1d(n * 32, 128), 128, 0, stream, "gn_sums_kernel", (const double*)workspace,
                (double*)sums, n, (int)groups, (int)rows);
}

extern "C" int ea_groupnorm_finalize(const void* sums, void* stats, int64_t parts, int64_t frames, int64_t groups, double count,
                                     float eps, void* stream) {
  EA_REQUIRE(sums && stats && parts > 0 && frames > 0 && groups > 0 && count > 0, "ea_groupnorm_finalize: bad arguments");
  const int n = (int)(frames * groups);
  return launch(gn_finalize_parts_kernel, grid_1d(n, 128), 128, 0, stream, "gn_finalize_parts_kernel",
                (const double*)sums, (float*)stats, n, (int)parts, count, eps);
}

extern "C" int ea_groupnorm_apply(const void* x, void* y, const void* gamma, const void* beta, const void* stats,
                                  int64_t frames, int64_t HW, int64_t C, int64_t groups, int32_t silu, void* stream) {
  EA_REQUIRE(x && y && gamma && beta && stats, "ea_groupnorm_apply: null pointer");
  EA_REQUIRE(C % 8 == 0 && C % groups == 0, "ea_groupnorm_apply: bad channel count");
  static const bool legacy = getenv("EA_GN_LEGACY_APPLY") != nullptr;  // A/B: the first (one vector per thread) kernel
  if (!legacy && C <= 2048 && 256 % (C / 8) == 0 && frames <= 65535) {
    // ~8 blocks per SM and frame-sized work items: 1 024 pixels per block, never fewer than one wave of blocks per call
    int pix_per_block = 1024;
    while (pix_per_block > 64 && frames * ((HW + pix_per_block - 1) / pix_per_block) < 4 * (int64_t)sm_count()) pix_per_block >>= 1;
    return launch(gn_apply2_kernel, dim3(grid_1d(HW, pix_per_block), (unsigned)frames), 256, 0, stream, "gn_apply2_kernel",
                  (const bf16*)x, (bf16*)y, (const bf16*)gamma, (const bf16*)beta, (const float*)stats, HW, (int)C,
                  (int)groups, pix_per_block, silu);
  }
  const int64_t total_vec = frames * HW * (C / 8);
  return launch(gn_apply_kernel, grid_1d(total_vec, 256), 256, 0, stream, "gn_apply_kernel", (const bf16*)x, (bf16*)y,
                (const bf16*)gamma, (const bf16*)beta, (const float*)stats, HW, (int)C, (int)groups, total_vec, silu);
}

extern "C" int ea_upsample2x(const void* x, void* y, int64_t T, int64_t H, int64_t W, int64_t C, void* stream) {
  EA_REQUIRE(x && y && C % 8 == 0, "ea_upsample2x: bad arguments");
  return launch(upsample2x_kernel, grid_1d(T * 2 * H * 2 * W * (C / 8), 256), 256, 0, stream, "upsample2x_kernel",
                (const bf16*)x, (bf16*)y, T, (int)H, (int)W, (int)C);
}

extern "C" int ea_softmax_rows(const void* s, void* p, int64_t M, int64_t N, int64_t lds, int64_t ldp, void* stream) {
  EA_REQUIRE(s && p && M > 0 && N > 0 && lds >= N && ldp >= N, "ea_softmax_rows: bad arguments");
  return launch(softmax_rows_kernel, (unsigned)M, 256, 0, stream, "softmax_rows_kernel", (const float*)s, (bf16*)p, (int)N,
                lds, ldp);
}

extern "C" int ea_transpose2d(const void* in, void* out, int64_t R, int64_t Cc, int64_t ldi, int64_t ldo, void* stream) {
  EA_REQUIRE(in && out && R > 0 && Cc > 0 && ldi >= Cc && ldo >= R, "ea_transpose2d: bad arguments");
  return launch(transpose2d_kernel, dim3(grid_1d(Cc, 32), grid_1d(R, 32)), dim3(32, 8), 0, stream, "transpose2d_kernel",
                (const bf16*)in, (bf16*)out, (int)R, (int)Cc, ldi, ldo);
}

extern "C" int ea_tile_blend(const void* a, int64_t a_plane, int64_t a_ld, int64_t a_off_r, int64_t a_off_c, void* b,
                             int64_t b_plane, int64_t b_ld, int64_t planes, int64_t rows, int64_t cols, int64_t extent,
                             int32_t axis, void* stream) {
  EA_REQUIRE(a && b && planes > 0 && rows > 0 && cols > 0 && extent > 0, "ea_tile_blend: bad arguments");
  return launch(blend_kernel, grid_1d(planes * rows * cols, 256), 256, 0, stream, "blend_kernel", (const bf16*)a, a_plane,
                (int)a_ld, (int)a_off_r, (int)a_off_c, (bf16*)b, b_plane, (int)b_ld, (int)planes, (int)rows, (int)cols,
                (int)extent, axis);
}

extern "C" int ea_copy2d(const void* src, int64_t s_plane, int64_t s_ld, void* dst, int64_t d_plane, int64_t d_ld,
                         int64_t planes, int64_t rows, int64_t cols, void* stream) {
  EA_REQUIRE(src && dst && planes > 0 && rows > 0 && cols > 0, "ea_copy2d: bad arguments");
  return launch(copy2d_kernel, grid_1d(planes * rows * cols, 256), 256, 0, stream, "copy2d_kernel", (const bf16*)src,
                s_plane, (int)s_ld, (bf16*)dst, d_plane, (int)d_ld, (int)planes, (int)rows, (int)cols);
}

extern "C" int ea_corner_blend(const void* src, void* dst, int64_t d_plane, int64_t d_ld, int64_t planes, int64_t Hc,
                               int64_t Wc, const float* wx, const float* wy, void* stream) {
  EA_REQUIRE(src && dst && wx && wy && planes > 0 && Hc > 0 && Wc > 0, "ea_corner_blend: bad arguments");
  return launch(corner_blend_kernel, grid_1d(planes * Hc * Wc, 256), 256, 0, stream, "corner_blend_kernel",
                (const bf16*)src, (bf16*)dst, d_plane, (int)d_ld, (int)planes, (int)Hc, (int)Wc, wx, wy);
}

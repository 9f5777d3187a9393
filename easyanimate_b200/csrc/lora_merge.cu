// LoRA merge: W[rows, cols] += scale * up[rows, rank] · down[rank, cols], in place, in the weight's own storage (bf16 or e4m3).
// The reference merges with torch ops on the module cast to the merge dtype (utils/lora_utils.py:424-430,486-492); this kernel
// does the same sequence with a fixed product order so that it can be emulated bit for bit on the host (include/ea_b200.h).
// CUDA cores, fp32 FMAs in ascending k: a tensor-core MMA would sum in an unspecified order.
#include <algorithm>

#include "common.cuh"
#include "host.h"
#include "../../include/ea_b200.h"

namespace ea {
namespace {

constexpr int LM_TILE = 128;   // W tile per block: 128 x 128
constexpr int LM_BK = 16;      // rank chunk staged in shared memory
constexpr int LM_PAD = 4;      // row padding of the up chunk (keeps float4 alignment, halves store conflicts)

struct LoraArgs {
  void* w;
  const void* up;
  const void* down;
  int64_t rows, cols, rank, ldw, ldu, ldd;
  float scale;
};

template <class T>
EA_DEVICE float load_f32(const T* p) {
  if constexpr (sizeof(T) == 4) return __ldg(reinterpret_cast<const float*>(p));
  else return __bfloat162float(__ldg(reinterpret_cast<const bf16*>(p)));
}

// The compute dtype's rounding point (torch materialising a tensor of that dtype); fp32 values are already rounded.
template <class T>
EA_DEVICE float round_c(float x) {
  if constexpr (sizeof(T) == 4) return x;
  else return bf16_round(x);
}

EA_DEVICE float e4m3_to_f32(uint32_t b) {
  const uint32_t e = (b >> 3) & 15, m = b & 7;
  float v;
  if ((b & 0x7f) == 0x7f) v = __uint_as_float(0x7fc00000u);
  else if (e == 0) v = (float)m * 0.001953125f;  // subnormal: m * 2^-9
  else v = __uint_as_float(((e + 120) << 23) | (m << 20));
  return (b & 0x80) ? -v : v;
}

// fp32 -> float8_e4m3fn as torch's `.to(torch.float8_e4m3fn)`: round to nearest even; a magnitude that rounds past 448 (above
// 464), inf and NaN give the NaN code 0x7f with the input's sign.  No saturation, unlike PTX's cvt.satfinite.
EA_DEVICE uint32_t f32_to_e4m3(float f) {
  const uint32_t bits = __float_as_uint(f);
  const uint32_t sign = (bits >> 24) & 0x80, a = bits & 0x7fffffffu;
  if (a >= 0x43f00000u) return sign | 0x7f;  // >= 480, inf, NaN
  const uint32_t e = a >> 23;
  if (e >= 121) {  // normal in e4m3 (>= 2^-6): keep 3 mantissa bits, round the 20 dropped ones to nearest even
    uint32_t r = a - (120u << 23);
    r += 0x7ffffu + ((r >> 20) & 1);
    return sign | (r >> 20);  // rounding up from 464 < |f| < 480 lands on 0x7f
  }
  if (e < 117) return sign;  // below 2^-10: rounds to zero
  // subnormal grid of 2^-9: q = |f| / 2^-9 = mant >> shift, rounded to nearest even (q = 8 is the smallest normal, 0x08)
  const uint32_t mant = (a & 0x7fffffu) | 0x800000u, shift = 141 - e;  // 21..24
  uint32_t q = mant >> shift;
  const uint32_t rem = mant & ((1u << shift) - 1), half = 1u << (shift - 1);
  if (rem > half || (rem == half && (q & 1))) ++q;
  return sign | q;
}

// One W element: d = rnd_c(acc), d2 = rnd_c(scale * d), w = rnd_c(W + d2), stored rounded to the storage type.
template <class T>
EA_DEVICE float merged(float w_old, float acc, float scale) {
  const float d = round_c<T>(acc);
  const float d2 = round_c<T>(__fmul_rn(scale, d));
  return round_c<T>(__fadd_rn(w_old, d2));
}

template <bool E4M3>
EA_DEVICE float load_w(const void* w, int64_t i) {
  if constexpr (E4M3) return e4m3_to_f32(reinterpret_cast<const uint8_t*>(w)[i]);
  else return __bfloat162float(reinterpret_cast<const bf16*>(w)[i]);
}

template <bool E4M3>
EA_DEVICE void store_w(void* w, int64_t i, float v) {
  if constexpr (E4M3) reinterpret_cast<uint8_t*>(w)[i] = (uint8_t)f32_to_e4m3(v);
  else reinterpret_cast<bf16*>(w)[i] = __float2bfloat16_rn(v);
}

// four consecutive W elements (4- or 8-byte aligned)
template <bool E4M3>
EA_DEVICE void load_w4(const void* w, int64_t i, float* f) {
  if constexpr (E4M3) {
    const uint32_t u = reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(w) + i)[0];
#pragma unroll
    for (int q = 0; q < 4; ++q) f[q] = e4m3_to_f32((u >> (8 * q)) & 0xff);
  } else {
    const uint2 u = reinterpret_cast<const uint2*>(reinterpret_cast<const bf16*>(w) + i)[0];
    const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
  }
}

template <bool E4M3>
EA_DEVICE void store_w4(void* w, int64_t i, const float* f) {
  if constexpr (E4M3) {
    const uint32_t u = f32_to_e4m3(f[0]) | (f32_to_e4m3(f[1]) << 8) | (f32_to_e4m3(f[2]) << 16) | (f32_to_e4m3(f[3]) << 24);
    reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(w) + i)[0] = u;
  } else {
    reinterpret_cast<uint2*>(reinterpret_cast<bf16*>(w) + i)[0] = make_uint2(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]));
  }
}

// One block per 128 x 128 W tile, 256 threads as 16 x 16; thread (ty, tx) owns rows {ty*4 .. +3} and {64 + ty*4 .. +3} and the
// same split of columns (8 x 8 accumulators; the split keeps the float4 shared-memory reads of a warp conflict-free).  The
// rank is walked in chunks of 16 through shared memory, each accumulator gets one fp32 FMA per k in ascending order, starting
// from +0, and every W element is read and written once.  `vec`: W rows allow 4-element vector access.
template <class T, bool E4M3>
__global__ void __launch_bounds__(256) lora_merge_kernel(const LoraArgs a, const int vec) {
  __shared__ __align__(16) float su[LM_BK][LM_TILE + LM_PAD];  // su[k][r] = up[r0 + r][k0 + k]
  __shared__ __align__(16) float sd[LM_BK][LM_TILE];           // sd[k][c] = down[k0 + k][c0 + c]
  const T* up = reinterpret_cast<const T*>(a.up);
  const T* down = reinterpret_cast<const T*>(a.down);
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t r0 = (int64_t)blockIdx.y * LM_TILE, c0 = (int64_t)blockIdx.x * LM_TILE;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  for (int64_t k0 = 0; k0 < a.rank; k0 += LM_BK) {
    const int kn = a.rank - k0 < LM_BK ? (int)(a.rank - k0) : LM_BK;
#pragma unroll
    for (int q = 0; q < LM_BK * LM_TILE / 256; ++q) {
      const int e = tid + 256 * q;
      {  // up: consecutive threads walk k within a row
        const int k = e & (LM_BK - 1), r = e / LM_BK;
        const int64_t gr = r0 + r;
        su[k][r] = (k < kn && gr < a.rows) ? load_f32(up + gr * a.ldu + k0 + k) : 0.f;
      }
      {  // down: consecutive threads walk columns within a row
        const int c = e & (LM_TILE - 1), k = e / LM_TILE;
        const int64_t gc = c0 + c;
        sd[k][c] = (k < kn && gc < a.cols) ? load_f32(down + (k0 + k) * a.ldd + gc) : 0.f;
      }
    }
    __syncthreads();
    // Only the chunk's real k: an FMA with a zero pad would turn an accumulator of -0 into +0.
    auto step = [&](int k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&su[k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&su[k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&sd[k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&sd[k][64 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = __fmaf_rn(av[i], bv[j], acc[i][j]);
    };
    if (kn == LM_BK) {
#pragma unroll
      for (int k = 0; k < LM_BK; ++k) step(k);
    } else {
      for (int k = 0; k < kn; ++k) step(k);
    }
    __syncthreads();
  }

  const float s = a.scale;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t row = r0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (row >= a.rows) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t col = c0 + h * 64 + tx * 4;
      const int64_t base = row * a.ldw + col;
      if (vec && col + 4 <= a.cols) {
        float f[4];
        load_w4<E4M3>(a.w, base, f);
#pragma unroll
        for (int q = 0; q < 4; ++q) f[q] = merged<T>(f[q], acc[i][h * 4 + q], s);
        store_w4<E4M3>(a.w, base, f);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (col + q < a.cols) store_w<E4M3>(a.w, base + q, merged<T>(load_w<E4M3>(a.w, base + q), acc[i][h * 4 + q], s));
      }
    }
  }
}

}  // namespace
}  // namespace ea

using namespace ea;

extern "C" int ea_lora_merge(void* w, const void* up, const void* down, int64_t rows, int64_t cols, int64_t rank, int64_t ldw,
                             int64_t ldu, int64_t ldd, float scale, int32_t w_kind, int32_t compute, void* stream) {
  EA_REQUIRE(w && up && down, "ea_lora_merge: null pointer");
  EA_REQUIRE(rows > 0 && cols > 0 && rank > 0, "ea_lora_merge: rows, cols and rank must be positive");
  EA_REQUIRE(ldw >= cols && ldu >= rank && ldd >= cols, "ea_lora_merge: a row stride is shorter than its row");
  EA_REQUIRE(w_kind == EA_LORA_W_BF16 || w_kind == EA_LORA_W_E4M3, "ea_lora_merge: w_kind must be EA_LORA_W_BF16 or _E4M3");
  EA_REQUIRE(compute == EA_LORA_C_BF16 || compute == EA_LORA_C_F32, "ea_lora_merge: compute must be EA_LORA_C_BF16 or _F32");
  EA_REQUIRE((rows + LM_TILE - 1) / LM_TILE <= 65535, "ea_lora_merge: more than 65535 * 128 rows");
  const size_t wsize = w_kind == EA_LORA_W_E4M3 ? 1 : 2, csize = compute == EA_LORA_C_F32 ? 4 : 2;
  EA_REQUIRE(reinterpret_cast<uintptr_t>(w) % wsize == 0 && reinterpret_cast<uintptr_t>(up) % csize == 0 &&
                 reinterpret_cast<uintptr_t>(down) % csize == 0,
             "ea_lora_merge: pointers must be aligned to their element size");
  const LoraArgs a{w, up, down, rows, cols, rank, ldw, ldu, ldd, scale};
  const int vec = ldw % 4 == 0 && reinterpret_cast<uintptr_t>(w) % (4 * wsize) == 0;
  const dim3 grid((unsigned)((cols + LM_TILE - 1) / LM_TILE), (unsigned)((rows + LM_TILE - 1) / LM_TILE));
  const bool e4m3 = w_kind == EA_LORA_W_E4M3;
  if (compute == EA_LORA_C_F32)
    return e4m3 ? launch(lora_merge_kernel<float, true>, grid, 256, 0, stream, "lora_merge_kernel<f32,e4m3>", a, vec)
                : launch(lora_merge_kernel<float, false>, grid, 256, 0, stream, "lora_merge_kernel<f32,bf16>", a, vec);
  return e4m3 ? launch(lora_merge_kernel<bf16, true>, grid, 256, 0, stream, "lora_merge_kernel<bf16,e4m3>", a, vec)
              : launch(lora_merge_kernel<bf16, false>, grid, 256, 0, stream, "lora_merge_kernel<bf16,bf16>", a, vec);
}

// The persistent, warp-specialised TMA -> wgmma pipeline shared by the GEMM (gemm_tc.cu) and the causal conv3d
// (conv3d_tc.cu) kernels.  One CTA of 384 threads walks the output tiles blockIdx.x, blockIdx.x + gridDim.x, ...:
//
//   warpgroup 0 (1 thread) : TMA producer - per k-block one 128x64 A box and one BNx64 B box into a SWIZZLE_128B
//                            shared-memory ring, completion on `full` mbarriers.
//   warpgroups 1, 2        : consumers - rows [0,64) / [64,128) of the 128 x BN tile: wgmma.m64nBNk16 (bf16 -> fp32 in
//                            registers) from both operands in shared memory, then the epilogue: the accumulators go through
//                            a shared-memory staging buffer, kCW columns per pass, so that each thread can own whole rows.
// The producer keeps fetching the next tile's k-blocks while the consumers run the epilogue.
//
// A kernel supplies three hooks:
//   decode(tile)                                   -> its tile coordinates (any copyable type)
//   load(coords, kb, tmap_a, tmap_b, a, b, bar)    producer thread: issue the two TMA loads of k-block kb into the ring
//                                                  slots a, b, completing on bar
//   epilogue(coords, row, col, src)                one consumer thread: tile row `row`, tile columns [col, col + kItem),
//                                                  staged in fp32 at src
// The staging buffer of a consumer warpgroup holds its 64 rows x kCW columns of one pass; its 128 threads take the rows'
// kItem-column pieces in turn.
#pragma once
#include "common.cuh"

namespace ea {

constexpr int kTcBM = 128;
constexpr int kTcBK = 64;
constexpr int kTcThreads = 384;
constexpr int kTcPitch = 132;  // fp32 staging row pitch: conflict-free 16-byte row reads

template <int BN>
struct TcCfg {
  static constexpr int kABytes = kTcBM * kTcBK * 2;
  static constexpr int kBBytes = BN * kTcBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (150 * 1024) / kStageBytes > 8 ? 8 : (150 * 1024) / kStageBytes;
  static constexpr int kCW = BN < 128 ? BN : 128;  // columns staged per epilogue pass
  static constexpr int kStagingBytes = 2 * 64 * kTcPitch * 4;
  static constexpr int kSmemBytes = kStages * kStageBytes + kStagingBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kSmemBytes <= 227 * 1024, "shared memory");
};

// The whole kernel body; tmap_a / tmap_b are the kernel's __grid_constant__ parameters (TMA reads the descriptor from
// param space, so they are passed on by address and never copied).
template <int BN, int kItem, class Decode, class Load, class Epilogue>
EA_DEVICE void tc_pipeline(const CUtensorMap* tmap_a, const CUtensorMap* tmap_b, int num_tiles, int num_k_blocks,
                           Decode decode, Load load, Epilogue epilogue) {
  using Cfg = TcCfg<BN>;
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

  if (threadIdx.x == 0) {
    tma_prefetch_desc(tmap_a);
    tma_prefetch_desc(tmap_b);
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
        const auto coords = decode(tile);
        for (int kb = 0; kb < num_k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          load(coords, kb, tmap_a, tmap_b, smem_a + stage * Cfg::kABytes, smem_b + stage * Cfg::kBBytes, &full_bar[stage]);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ===== consumers: rows [64 (wg-1), 64 wg) of the tile =====
    const int cw = wg - 1;
    const int tid = threadIdx.x & 127;
    float* stage_buf = staging + cw * 64 * kTcPitch;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const auto coords = decode(tile);
      float acc[BN / 2];
      int prev = -1;
      // the previous tile's epilogue diverged: reconverge the warp before the warpgroup-wide wgmma k-loop (without
      // this ptxas cannot prove convergence there and keeps the loop's stage / phase bookkeeping out of uniform registers)
      __syncwarp();
      for (int kb = 0; kb < num_k_blocks; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t adesc = gmma_desc_sw128(smem_u32(smem_a + stage * Cfg::kABytes + cw * 64 * 128));
        const uint64_t bdesc = gmma_desc_sw128(smem_u32(smem_b + stage * Cfg::kBBytes));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kTcBK / 16; ++k) {
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

      // ===== epilogue: kCW columns at a time through the staging buffer =====
#pragma unroll
      for (int cb = 0; cb < BN / kCW; ++cb) {
        named_bar_sync(1 + cw, 128);  // the previous pass has finished reading the staging buffer
        stage_acc<kCW>(acc + cb * (kCW / 2), stage_buf, kTcPitch);
        named_bar_sync(1 + cw, 128);
#pragma unroll 1
        for (int i = tid; i < 64 * (kCW / kItem); i += 128) {
          const int r = i & 63, c = i >> 6;
          epilogue(coords, cw * 64 + r, cb * kCW + c * kItem, static_cast<const float*>(stage_buf + r * kTcPitch + c * kItem));
        }
      }
    }
  }
}

}  // namespace ea

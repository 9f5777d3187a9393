// Causal 3x3x3 convolution of the MagViT VAE as an im2col-free implicit GEMM on sm_90a wgmma.
//
// Replaces CausalConv3d.forward (easyanimate/vae/ldm/modules/vaemodules/common.py:84-141, called from
// ResidualBlock3D common.py:298-323, the upsamplers upsamplers.py:34-37,142-153, the down-samplers downsamplers.py:24-96
// and Decoder.conv_in/conv_out omnigen_enc_dec.py:555-615).  The reference runs it one latent frame at a time with a
// 2-frame cache (padding_flag 3/4); that is one causal convolution over the whole sequence with the first frame replicated
// on the left, which is what this kernel computes in a single launch per layer.
//
// Layout: activations are channels-last [T,H,W,C] bf16.  For an output tile of TH x TW pixels (= 128 GEMM rows) of
// frame t and every tap (kt,kh,kw) x 64-channel slice, ONE TMA box {64ch, TW, TH, 1} of the input at
// (w0+kw-1, h0+kh-1, max(t+kt-2,0)) lands in shared memory as a SWIZZLE_128B K-major [128 x 64] A tile - spatial
// zero padding is TMA out-of-bounds fill, causal replicate padding is the coordinate clamp; nothing is gathered or
// materialised.  Weights are pre-arranged [Cout, 27*Cin] (tap-major K).  Warpgroup / barrier / epilogue-staging structure
// as gemm_tc.cu: one TMA producer thread, two consumer warpgroups of 64 pixels x BN output channels each.
// Fused in the epilogue: bias, residual add, nearest temporal x2 duplication (frames >= 1), planar NCTHW store.
#include "common.cuh"
#include "host.h"
#include "../../include/ea_b200.h"

namespace ea {

extern void count_launch();

constexpr int kConvThreads = 384;
constexpr int kConvPitch = 132;  // fp32 staging row pitch
constexpr int kCM = 128;
constexpr int kCK = 64;

struct ConvDevArgs {
  int T, H, W, Cin, Cout;
  int TH, TW;  // TH*TW == 128
  int tiles_h, tiles_w, tiles_n;
  int kt_taps;  // 3 (causal 3x3x3) — kept as a parameter so 1x3x3 could reuse the kernel
  const bf16* bias;
  const bf16* residual;
  bf16* out;
  int dup_frames;
  int out_planar;
  int T_out;
  int row0, Hout;  // output row window [row0, row0 + Hout) (strip-parallel decode: the input carries halo rows), stored at row h - row0
  int st, shw;  // temporal / spatial stride (1 or 2): T, H, W above are the OUTPUT extents (see ea_conv3d_args.stride_*)
};

template <int BN>
struct ConvCfg {
  static constexpr int kABytes = kCM * kCK * 2;
  static constexpr int kBBytes = BN * kCK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (150 * 1024) / kStageBytes > 8 ? 8 : (150 * 1024) / kStageBytes;
  static constexpr int kCW = BN < 128 ? BN : 128;  // columns staged per epilogue pass
  static constexpr int kStagingBytes = 2 * 64 * kConvPitch * 4;
  static constexpr int kSmemBytes = kStages * kStageBytes + kStagingBytes + 1024 + 256;
  static_assert(kSmemBytes <= 227 * 1024, "shared memory");
};

// bias, residual, frame duplication and the channels-last or planar store of 32 output channels of one pixel
EA_DEVICE void conv_epilogue_chunk(const ConvDevArgs& p, int t, int ho, int w, int col0, float (&x)[32]) {
  const int t_out = p.dup_frames ? (t == 0 ? 0 : 2 * t - 1) : t;
  const int ncopies = (p.dup_frames && t > 0) ? 2 : 1;
  if (p.out_planar) {
    // conv_out: few real channels, planar [Cout, T_out, H, W] store
    for (int j = 0; j < 32 && col0 + j < p.Cout; ++j) {
      const float v = x[j] + __bfloat162float(p.bias[col0 + j]);
      for (int cpy = 0; cpy < ncopies; ++cpy)
        p.out[(((int64_t)(col0 + j) * p.T_out + t_out + cpy) * p.Hout + ho) * p.W + w] = __float2bfloat16_rn(v);
    }
    return;
  }
  {
    const uint4* bp = reinterpret_cast<const uint4*>(p.bias + col0);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint4 b = __ldg(bp + j);
      float2 f0 = unpack_bf16x2(b.x), f1 = unpack_bf16x2(b.y), f2 = unpack_bf16x2(b.z), f3 = unpack_bf16x2(b.w);
      x[j * 8 + 0] += f0.x; x[j * 8 + 1] += f0.y; x[j * 8 + 2] += f1.x; x[j * 8 + 3] += f1.y;
      x[j * 8 + 4] += f2.x; x[j * 8 + 5] += f2.y; x[j * 8 + 6] += f3.x; x[j * 8 + 7] += f3.y;
    }
  }
  if (p.residual != nullptr) {
    // (conv2(x) + shortcut): the conv output is a bf16 tensor in the reference before the add (common.py:323)
    const uint4* rp = reinterpret_cast<const uint4*>(p.residual + (((int64_t)t * p.Hout + ho) * p.W + w) * p.Cout + col0);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint4 rr = __ldg(rp + j);
      uint32_t rw[4] = {rr.x, rr.y, rr.z, rr.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float2 rf = unpack_bf16x2(rw[q]);
        x[j * 8 + 2 * q] = bf16_round(x[j * 8 + 2 * q]) + rf.x;
        x[j * 8 + 2 * q + 1] = bf16_round(x[j * 8 + 2 * q + 1]) + rf.y;
      }
    }
  }
  uint4 o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    o[j].x = pack_bf16x2(x[j * 8 + 0], x[j * 8 + 1]);
    o[j].y = pack_bf16x2(x[j * 8 + 2], x[j * 8 + 3]);
    o[j].z = pack_bf16x2(x[j * 8 + 4], x[j * 8 + 5]);
    o[j].w = pack_bf16x2(x[j * 8 + 6], x[j * 8 + 7]);
  }
  for (int cpy = 0; cpy < ncopies; ++cpy) {
    uint4* op = reinterpret_cast<uint4*>(p.out + ((((int64_t)(t_out + cpy)) * p.Hout + ho) * p.W + w) * p.Cout + col0);
#pragma unroll
    for (int j = 0; j < 4; ++j) op[j] = o[j];
  }
}

template <int BN>
__global__ void __launch_bounds__(kConvThreads, 1)
conv3d_tc_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                 const ConvDevArgs p) {
  using Cfg = ConvCfg<BN>;
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
  const int num_tiles = p.T * p.tiles_h * p.tiles_w * p.tiles_n;
  const int cchunks = p.Cin / kCK;
  const int num_k_blocks = p.kt_taps * 9 * cchunks;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_w);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // lane 0 of each consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  auto decode_tile = [&](int tile, int& t, int& h0, int& w0, int& n0) {
    n0 = (tile % p.tiles_n) * BN;
    int r = tile / p.tiles_n;
    w0 = (r % p.tiles_w) * p.TW;
    r /= p.tiles_w;
    h0 = p.row0 + (r % p.tiles_h) * p.TH;
    t = r / p.tiles_h;
  };

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      // ===== TMA producer =====
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int t, h0, w0, n0;
        decode_tile(tile, t, h0, w0, n0);
        for (int kb = 0; kb < num_k_blocks; ++kb) {
          const int tap = kb / cchunks;
          const int c0 = (kb - tap * cchunks) * kCK;
          const int kt = tap / 9, kh = (tap % 9) / 3, kw = tap % 3;
          int tin = t * p.st + kt - (p.kt_taps - 1);  // causal: taps reach back in time; left edge replicates frame 0
          tin = tin < 0 ? 0 : tin;
          // stride 1: 1-pixel zero border on every side (x = w0 + kw - 1).  stride 2 (downsamplers.py:24-96: F.pad right /
          // bottom by one, no padding in the convolution): output (i, j) reads input rows 2i..2i+2, columns 2j..2j+2, and the
          // tensor map walks the box with element stride 2, so one box still lands as TH x TW consecutive GEMM rows.
          const int xw = p.shw == 1 ? w0 + kw - 1 : 2 * w0 + kw;
          const int xh = p.shw == 1 ? h0 + kh - 1 : 2 * h0 + kh;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_4d(smem_a + stage * Cfg::kABytes, &tmap_x, &full_bar[stage], c0, xw, xh, tin);
          tma_load_2d(smem_b + stage * Cfg::kBBytes, &tmap_w, &full_bar[stage], tap * p.Cin + c0, n0);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ===== consumers: GEMM rows (pixels) [64 (wg-1), 64 wg) of the tile =====
    const int cw = wg - 1;
    const int tid = threadIdx.x & 127;
    float* stage_buf = staging + cw * 64 * kConvPitch;
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int t, h0, w0, n0;
      decode_tile(tile, t, h0, w0, n0);
      float acc[BN / 2];
      int prev = -1;
      for (int kb = 0; kb < num_k_blocks; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t adesc = gmma_desc_sw128(smem_u32(smem_a + stage * Cfg::kABytes + cw * 64 * 128));
        const uint64_t bdesc = gmma_desc_sw128(smem_u32(smem_b + stage * Cfg::kBBytes));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kCK / 16; ++k) wgmma_ss<BN>(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();  // the k-block before this one has been read: release its stage
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      reg_fence<BN / 2>(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);

      // ===== epilogue: one output pixel and 32 channels per thread and item =====
#pragma unroll
      for (int cb = 0; cb < BN / kCW; ++cb) {
        named_bar_sync(1 + cw, 128);  // the previous pass has finished reading the staging buffer
        stage_acc<kCW>(acc + cb * (kCW / 2), stage_buf, kConvPitch);
        named_bar_sync(1 + cw, 128);
#pragma unroll 1
        for (int i = tid; i < 64 * (kCW / 32); i += 128) {
          const int r = i & 63, c = i >> 6;
          const int row = cw * 64 + r;
          const int h = h0 + row / p.TW, w = w0 + row % p.TW;
          const int col0 = n0 + cb * kCW + c * 32;
          if (h >= p.row0 + p.Hout || w >= p.W || col0 >= p.Cout) continue;
          float x[32];
          const float* src = stage_buf + r * kConvPitch + c * 32;
#pragma unroll
          for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(x + j) = *reinterpret_cast<const float4*>(src + j);
          conv_epilogue_chunk(p, t, h - p.row0, w, col0, x);
        }
      }
    }
  }
}

template <int BN>
static int launch_conv(const ea_conv3d_args* g, cudaStream_t stream) {
  using Cfg = ConvCfg<BN>;
  ConvDevArgs p{};
  p.st = g->stride_t == 2 ? 2 : 1;
  p.shw = g->stride_hw == 2 ? 2 : 1;
  // output extents: every second frame from frame 0 (T = 1 + 2m -> m + 1), floor(H / 2) x floor(W / 2) pixels
  p.T = p.st == 2 ? (int)((g->T + 1) / 2) : (int)g->T;
  p.H = p.shw == 2 ? (int)(g->H / 2) : (int)g->H;
  p.W = p.shw == 2 ? (int)(g->W / 2) : (int)g->W;
  p.Cin = (int)g->Cin; p.Cout = (int)g->Cout;
  p.row0 = g->out_rows > 0 ? (int)g->out_row0 : 0;
  p.Hout = g->out_rows > 0 ? (int)g->out_rows : p.H;
  // tile shape: 8x16 or 4x32 pixels, whichever wastes fewer out-of-range pixels
  auto waste = [&](int th, int tw) {
    return (int64_t)((p.Hout + th - 1) / th) * th * ((p.W + tw - 1) / tw) * tw;
  };
  if (waste(4, 32) < waste(8, 16)) { p.TH = 4; p.TW = 32; } else { p.TH = 8; p.TW = 16; }
  p.tiles_h = (p.Hout + p.TH - 1) / p.TH;
  p.tiles_w = (p.W + p.TW - 1) / p.TW;
  p.tiles_n = (int)((g->Cout_pad + BN - 1) / BN);
  p.kt_taps = 3;
  p.bias = reinterpret_cast<const bf16*>(g->bias);
  p.residual = reinterpret_cast<const bf16*>(g->residual);
  p.out = reinterpret_cast<bf16*>(g->out);
  p.dup_frames = g->dup_frames;
  p.out_planar = g->out_planar;
  p.T_out = g->dup_frames ? (int)(2 * g->T - 1) : p.T;

  CUtensorMap tx, tw;
  {
    uint64_t dims[4] = {(uint64_t)g->Cin, (uint64_t)g->W, (uint64_t)g->H, (uint64_t)g->T};
    uint64_t strides[3] = {(uint64_t)g->Cin * 2, (uint64_t)g->W * g->Cin * 2, (uint64_t)g->H * g->W * g->Cin * 2};
    // with a spatial stride the box spans shw x as many input elements, walked with element stride shw
    // (cuTensorMapEncodeTiled elementStrides): the number of elements that land is still TW x TH
    uint32_t box[4] = {kCK, (uint32_t)(p.TW * p.shw), (uint32_t)(p.TH * p.shw), 1};
    uint32_t estr[4] = {1, (uint32_t)p.shw, (uint32_t)p.shw, 1};
    int rc = make_tmap_bf16(&tx, g->x, 4, dims, strides, box, true, estr);
    if (rc) return rc;
  }
  {
    const uint64_t K = (uint64_t)27 * g->Cin;
    uint64_t dims[2] = {K, (uint64_t)g->Cout_pad};
    uint64_t strides[1] = {K * 2};
    uint32_t box[2] = {kCK, (uint32_t)BN};
    int rc = make_tmap_bf16(&tw, g->w, 2, dims, strides, box, true);
    if (rc) return rc;
  }
  auto kern = conv3d_tc_kernel<BN>;
  static ::ea::PerDeviceFlag attr_flag;
  const int attr_dev = ::ea::current_device();
  if (!attr_flag.get(attr_dev)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) return fail(EA_ERR_CUDA, std::string("cudaFuncSetAttribute(conv): ") + cudaGetErrorString(e));
    attr_flag.set(attr_dev);
  }
  const int64_t num_tiles = (int64_t)p.T * p.tiles_h * p.tiles_w * p.tiles_n;
  if (num_tiles >= (1ll << 31)) return fail(EA_ERR_INVALID, "ea_conv3d: too many tiles");
  const int grid = (int)(num_tiles < sm_count() ? num_tiles : sm_count());
  kern<<<grid, kConvThreads, Cfg::kSmemBytes, stream>>>(tx, tw, p);
  count_launch();
  return check_launch("conv3d_tc_kernel");
}

}  // namespace ea

using namespace ea;

extern "C" int ea_conv3d_causal(const ea_conv3d_args* g, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  EA_REQUIRE(g && g->x && g->w && g->bias && g->out, "ea_conv3d_causal: null pointer");
  EA_REQUIRE(g->T > 0 && g->H > 0 && g->W > 0, "ea_conv3d_causal: empty input");
  EA_REQUIRE(g->Cin > 0 && g->Cin % 64 == 0, "ea_conv3d_causal: Cin must be a multiple of 64 (pad the channels)");
  EA_REQUIRE(g->Cout > 0 && g->Cout_pad >= g->Cout && g->Cout_pad % 32 == 0,
             "ea_conv3d_causal: Cout_pad must be a multiple of 32 and >= Cout");
  EA_REQUIRE(g->out_planar || g->Cout % 32 == 0, "ea_conv3d_causal: channels-last output needs Cout % 32 == 0");
  EA_REQUIRE(!(g->out_planar && g->residual), "ea_conv3d_causal: planar output cannot take a residual");
  EA_REQUIRE(g->W < 32768 && g->H < 32768, "ea_conv3d_causal: frame too large");
  EA_REQUIRE((g->stride_t == 0 || g->stride_t == 1 || g->stride_t == 2) && (g->stride_hw == 0 || g->stride_hw == 1 || g->stride_hw == 2),
             "ea_conv3d_causal: strides are 1 or 2");
  EA_REQUIRE(g->out_rows >= 0 && g->out_row0 >= 0 && (g->out_rows == 0 || g->out_row0 + g->out_rows <= g->H),
             "ea_conv3d_causal: output row window outside the input");
  if (g->stride_t == 2 || g->stride_hw == 2) {
    EA_REQUIRE(g->out_rows == 0, "ea_conv3d_causal: a strided convolution takes no output row window");
    EA_REQUIRE(!g->residual && !g->dup_frames && !g->out_planar, "ea_conv3d_causal: a strided convolution takes no residual / frame "
               "duplication / planar output");
    EA_REQUIRE(g->stride_hw != 2 || (g->H >= 2 && g->W >= 2), "ea_conv3d_causal: frame too small for stride 2");
  }
  // (ea_conv3d_args.variant selected B200 tile layouts; every value runs the one kernel below)
  if (g->Cout_pad % 256 == 0) return launch_conv<256>(g, stream);
  if (g->Cout_pad % 128 == 0) return launch_conv<128>(g, stream);
  if (g->Cout_pad % 64 == 0) return launch_conv<64>(g, stream);
  return launch_conv<32>(g, stream);
}

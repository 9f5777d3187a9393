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
// materialised.  Weights are pre-arranged [Cout, 27*Cin] (tap-major K).  The TMA / wgmma pipeline is tc_pipeline.cuh,
// shared with the GEMM: two consumer warpgroups of 64 pixels x BN output channels each.
// Fused in the epilogue: bias, residual add, nearest temporal x2 duplication (frames >= 1), planar NCTHW store.
#include "host.h"
#include "tc_pipeline.cuh"
#include "../../include/ea_b200.h"

namespace ea {

constexpr int kTaps = 3;  // temporal taps of the causal 3x3x3 kernel: output frame t reads input frames t-2 .. t

struct ConvDevArgs {
  int T, H, W, Cin, Cout;
  int TH, TW;  // TH*TW == 128
  int tiles_h, tiles_w, tiles_n;
  const bf16* bias;
  const bf16* residual;
  bf16* out;
  int dup_frames;
  int out_planar;
  int T_out;
  int row0, Hout;  // output row window [row0, row0 + Hout) (strip-parallel decode: the input carries halo rows), stored at row h - row0
  int st, shw;  // temporal / spatial stride (1 or 2): T, H, W above are the OUTPUT extents (see ea_conv3d_args.stride_*)
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
  add_bf16<32>(x, p.bias + col0);
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
  for (int cpy = 0; cpy < ncopies; ++cpy)
    store_bf16<32>(p.out + ((((int64_t)(t_out + cpy)) * p.Hout + ho) * p.W + w) * p.Cout + col0, x);
}

template <int BN>
__global__ void __launch_bounds__(kTcThreads, 1)
conv3d_tc_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                 const ConvDevArgs p) {
  const int cchunks = p.Cin / kTcBK;
  struct Tile { int t, h0, w0, n0; };
  auto decode = [&](int tile) {
    Tile c;
    c.n0 = (tile % p.tiles_n) * BN;
    int r = tile / p.tiles_n;
    c.w0 = (r % p.tiles_w) * p.TW;
    r /= p.tiles_w;
    c.h0 = p.row0 + (r % p.tiles_h) * p.TH;
    c.t = r / p.tiles_h;
    return c;
  };
  auto load = [&](const Tile& c, int kb, const CUtensorMap* tx, const CUtensorMap* tw, void* a, void* b, uint64_t* bar) {
    const int tap = kb / cchunks;
    const int c0 = (kb - tap * cchunks) * kTcBK;
    const int kt = tap / 9, kh = (tap % 9) / 3, kw = tap % 3;
    int tin = c.t * p.st + kt - (kTaps - 1);  // causal: taps reach back in time; left edge replicates frame 0
    tin = tin < 0 ? 0 : tin;
    // stride 1: 1-pixel zero border on every side (x = w0 + kw - 1).  stride 2 (downsamplers.py:24-96: F.pad right /
    // bottom by one, no padding in the convolution): output (i, j) reads input rows 2i..2i+2, columns 2j..2j+2, and the
    // tensor map walks the box with element stride 2, so one box still lands as TH x TW consecutive GEMM rows.
    const int xw = p.shw == 1 ? c.w0 + kw - 1 : 2 * c.w0 + kw;
    const int xh = p.shw == 1 ? c.h0 + kh - 1 : 2 * c.h0 + kh;
    tma_load_4d(a, tx, bar, c0, xw, xh, tin);
    tma_load_2d(b, tw, bar, tap * p.Cin + c0, c.n0);
  };
  // one output pixel and 32 channels per item
  auto epilogue = [&](const Tile& c, int r, int col, const float* src) {
    const int h = c.h0 + r / p.TW, w = c.w0 + r % p.TW;
    const int col0 = c.n0 + col;
    if (h >= p.row0 + p.Hout || w >= p.W || col0 >= p.Cout) return;
    float x[32];
#pragma unroll
    for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(x + j) = *reinterpret_cast<const float4*>(src + j);
    conv_epilogue_chunk(p, c.t, h - p.row0, w, col0, x);
  };
  tc_pipeline<BN, 32>(&tmap_x, &tmap_w, p.T * p.tiles_h * p.tiles_w * p.tiles_n, kTaps * 9 * cchunks, decode, load, epilogue);
}

template <int BN>
static int launch_conv(const ea_conv3d_args* g, void* stream) {
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
    uint32_t box[4] = {kTcBK, (uint32_t)(p.TW * p.shw), (uint32_t)(p.TH * p.shw), 1};
    uint32_t estr[4] = {1, (uint32_t)p.shw, (uint32_t)p.shw, 1};
    int rc = make_tmap_bf16(&tx, g->x, 4, dims, strides, box, true, estr);
    if (rc) return rc;
  }
  {
    const uint64_t K = (uint64_t)kTaps * 9 * g->Cin;
    uint64_t dims[2] = {K, (uint64_t)g->Cout_pad};
    uint64_t strides[1] = {K * 2};
    uint32_t box[2] = {kTcBK, (uint32_t)BN};
    int rc = make_tmap_bf16(&tw, g->w, 2, dims, strides, box, true);
    if (rc) return rc;
  }
  const int64_t num_tiles = (int64_t)p.T * p.tiles_h * p.tiles_w * p.tiles_n;
  if (num_tiles >= (1ll << 31)) return fail(EA_ERR_INVALID, "ea_conv3d: too many tiles");
  static PerDeviceFlag smem_done;
  return launch_persistent(conv3d_tc_kernel<BN>, num_tiles, kTcThreads, TcCfg<BN>::kSmemBytes, smem_done, stream,
                           "conv3d_tc_kernel", tx, tw, p);
}

}  // namespace ea

using namespace ea;

extern "C" int ea_conv3d_causal(const ea_conv3d_args* g, void* stream) {
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

// conv_split.cuh - geometry / layout of the fp16 plane pairs shared by the tensor-core conv kernels (conv_split.cu).
// See conv_split.cu for the layout description.
#pragma once
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace nisqa {

enum { SP_POOL_NONE = 0, SP_POOL_ADAPT = 1, SP_POOL_2X2 = 2 };


// byte offset of chunk c (8 halves) of plane row g, rows of ROWB bytes: Swizzle<log2(ROWB/16), 4, 3>
template <int ROWB>
__device__ __forceinline__ size_t split_off(int g, int c) {
  const size_t o = (size_t)g * ROWB + (size_t)c * 16;
  return o ^ ((o >> 3) & (size_t)(ROWB - 16));
}

// Geometry of conv layer 2..6 on an H x W input map (the next layer's input, or the fp32 features, is HO x WO).  A
// compile-time layer type (SpCfg) holds its members as constants, a run-time geometry type (SpRt) takes it as the
// kernel argument.  GEMM rows: only the tile's interior output positions, KW per row from plane column X0 (conv6 of the
// AdaptCNN: one), in (segment, h, w) order, packed into NBLK m64 blocks.  GEMM row m reads its taps around tile row
// HALO + gemm_row(g, m).
struct SpGeom {
  int H, W, P, BLK, G, HALO, KW, SEG_ROWS, KEPT, NBLK;
  int HO, WO, OP, OBLK;      // the output map (the next layer's input): pooled, H x W, or H x 1 (conv6 of the AdaptCNN)
  int OUT_COLS, OUT_LD;      // the last layer: HO WO COUT features in rows of OUT_LD floats (a multiple of 64, zero-padded)
  int X0;                    // plane column of a row's first output position: 1, or 2 for the centre column of a 3-wide
                             // map (conv6 of the shipped AdaptCNN: its padded 3 x 3 conv evaluated at column 1 only)
};
constexpr SpGeom sp_geom(int H, int W, int KW, int X0, int HO, int WO, int cout) {
  SpGeom g{};
  g.H = H; g.W = W; g.P = W + 1;                  // row pitch: W interior columns + 1 shared zero column
  g.BLK = (H + 1) * g.P;                          // rows per segment: H interior rows + 1 shared zero row
  g.G = 256 / g.BLK;                              // segments per tile (256 GEMM rows)
  g.HALO = g.P + 1;                               // |row offset| of the farthest 3 x 3 tap
  g.KW = KW; g.X0 = X0;
  g.SEG_ROWS = H * KW; g.KEPT = g.G * g.SEG_ROWS; g.NBLK = (g.KEPT + 63) / 64;
  g.HO = HO; g.WO = WO; g.OP = WO + 1; g.OBLK = (HO + 1) * g.OP;
  g.OUT_COLS = HO * WO * cout; g.OUT_LD = (g.OUT_COLS + 63) / 64 * 64;    // 6 x 16 -> 128
  return g;
}

// Plane row of GEMM row m of geometry g (an SpGeom, or a compile-time layer type), counted from the zero row of the
// tile's first segment.  Rows m >= KEPT read that zero row; the rows of segments past the end of a short last tile read
// the copied range as it lies.  Neither is staged.
template <class Geo>
__host__ __device__ constexpr int gemm_row(const Geo& g, int m) {
  if (m >= g.KEPT) return 0;
  const int s = m / g.SEG_ROWS, q = m - s * g.SEG_ROWS, h = q / g.KW, w = q - h * g.KW;
  // One value, grouped two ways: the grouping decides how nvcc folds the column into the staging-store offsets, and
  // each kind keeps the instructions its kernels were measured with.
  if constexpr (std::is_same<Geo, SpGeom>::value) return s * g.BLK + (h + 1) * g.P + w + g.X0;
  else return s * g.BLK + (h + 1) * g.P + (w + g.X0);
}

// Shared memory of conv_split_kernel: NTAP weight taps, resident for the CTA's life, activation tiles of AROWS rows of
// CIN halves and an fp32 staging tile of 256 rows of COUT.  Three ways to fit, the first that fits: the activation tile
// double-buffered (the next tile's copy lands during this tile's GEMM and epilogue), one activation buffer beside the
// staging tile (the next tile's copy lands during this tile's epilogue), or one buffer that the staging tile reuses
// (ALIAS: the copy waits for the epilogue).  Buffer b: hi plane at b * A_BUF, lo plane at b * A_BUF + A_BYTES.
template <int NTAP_, int AROWS_, int CIN_, int COUT_>
struct SpLayout {
  static constexpr int NT = 4 * 128;             // four warpgroups; warpgroup b < NBLK runs m64 block b
  static constexpr int NTAP = NTAP_, AROWS = AROWS_, CIN = CIN_, COUT = COUT_;
  static constexpr int ROWB = CIN * 2;            // bytes per row
  static constexpr int OROWB = COUT * 2;          // bytes per row of the output planes
  static constexpr int A_BYTES = ((AROWS + 7) * ROWB + 1023) & ~1023;     // + placement shift (g0 & 7 rows)
  static constexpr int B_STAGE = 2 * (CIN / 8) * COUT * 16;   // one tap: [CIN/8][hi co | lo co][8 halves]
  // epilogue staging: one fp32 row per GEMM row (bias + ReLU applied)
  static constexpr int STG_STRIDE = COUT + 4;
  static constexpr int STG_BYTES = 256 * STG_STRIDE * 4;
  static constexpr int SMEM_BUDGET = 227 * 1024 - 2048;
  static constexpr int A_BUF = 2 * A_BYTES;
  static constexpr int ONE_BUF = A_BUF + STG_BYTES + NTAP * B_STAGE;  // one unaliased activation buffer
  static constexpr bool ALIAS = ONE_BUF > SMEM_BUDGET;
  static constexpr int A_BUFS = (ALIAS || ONE_BUF + A_BUF > SMEM_BUDGET) ? 1 : 2;
  static constexpr int OFF_A_HI = 0;
  static constexpr int OFF_A_LO = A_BYTES;
  static constexpr int OFF_STG = ALIAS ? 0 : A_BUFS * A_BUF;
  static constexpr int OFF_B = ((ALIAS ? (A_BUF > STG_BYTES ? A_BUF : STG_BYTES) : A_BUFS * A_BUF + STG_BYTES) + 1023) & ~1023;
  // NTAP weight-tap barriers, then a full barrier per activation buffer, then (double-buffered) an empty barrier per buffer
  static constexpr int OFF_BAR = OFF_B + NTAP * B_STAGE;
  static constexpr int NBAR = NTAP + 2 * A_BUFS;
  static constexpr int SMEM_BYTES = OFF_BAR + 8 * NBAR + 1024;    // + slack: the tile is aligned to 1024 B
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
  static_assert(ALIAS || A_BUFS * A_BUF + STG_BYTES + NTAP * B_STAGE <= SMEM_BUDGET,
                "the activation buffers fit beside the staging tile and the weights");
  static_assert(CIN % 16 == 0 && (COUT == 16 || COUT == 32 || COUT == 64), "shape");
  static_assert(ROWB == 32 || ROWB == 64 || ROWB == 128, "rows are 32 / 64 / 128 bytes (one swizzle atom)");
};

// A layer whose map sizes are compile-time constants: 3 x 3 taps, padding 1; conv2 / conv4 pool (POOL) to H / 2 x POW.
// The last layer (F32OUT) writes the CNN features as fp32 channels-last; CENTER: conv6 of the AdaptCNN, kernel (3, 3),
// padding (1, 0) on a 3-wide map == the padded conv evaluated at column 1 only.
template <int H_, int W_, int CIN_, int COUT_, int POOL_, int POW, bool F32OUT = false, bool CENTER = false>
struct SpCfg : SpLayout<9, 256 + 2 * (W_ + 2), CIN_, COUT_> {
  static constexpr int POOL = POOL_, KX = 3, PADX = 1;
  static constexpr bool RT = false;
  static constexpr bool ONE_STEP_UNITS = H_ == 24 && COUT_ == 64;  // conv2 at 64 output channels (TapUnits)
  static constexpr bool OUT_SPLIT = !F32OUT;
  static constexpr SpGeom GEO = sp_geom(H_, W_, CENTER ? 1 : W_, CENTER ? 2 : 1, POOL == SP_POOL_NONE ? H_ : H_ / 2,
                                        POOL == SP_POOL_NONE ? (CENTER ? 1 : W_) : POW, COUT_);
  // GEO's members as constants: the kernels read the geometry through them (geom), so it folds into their code
  static constexpr int H = GEO.H, W = GEO.W, P = GEO.P, BLK = GEO.BLK, G = GEO.G, HALO = GEO.HALO, KW = GEO.KW,
                       SEG_ROWS = GEO.SEG_ROWS, KEPT = GEO.KEPT, NBLK = GEO.NBLK, HO = GEO.HO, WO = GEO.WO, OP = GEO.OP,
                       OBLK = GEO.OBLK, OUT_COLS = GEO.OUT_COLS, OUT_LD = GEO.OUT_LD, X0 = GEO.X0;
  __host__ __device__ static constexpr SpCfg geom(const SpGeom&) { return {}; }
  static_assert(HALO <= kSplitLead, "kSplitLead");
  static_assert(!CENTER || F32OUT, "the centre-column variant only exists as the last layer");
  static_assert(OUT_SPLIT || POOL == SP_POOL_NONE, "fp32 output is not pooled");
  static_assert(G >= 1, "tile");
  static_assert(NBLK <= 4 && (!CENTER || W == 3), "GEMM rows");
};

// Layers 2..6.  AdaptCNN: one instance per (layer, CIN, COUT) that cnn_c_out_1/2/3 in {16, 32, 64} reach - conv2
// c1 -> c2, conv3 c2 -> c3, conv4..conv6 c3 -> c3 (NISQA_SP_ADAPT_LAYERS lists them, conv_split.cu instantiates them).
// StandardCNN: the shipped 16 / 32 / 64 channels, std_mode selects its geometry (W 8/4/2, MaxPool2d(2)).
template <int L, int CIN, int COUT> struct SpAdaptLayer;
//                                                                H   W  CIN COUT POOL           POW F32OUT CENTER
template <int CIN, int COUT> struct SpAdaptLayer<2, CIN, COUT> { using T = SpCfg<24, 7, CIN, COUT, SP_POOL_ADAPT, 5>; };
template <int CIN, int COUT> struct SpAdaptLayer<3, CIN, COUT> { using T = SpCfg<12, 5, CIN, COUT, SP_POOL_NONE, 0>; };
template <int CIN, int COUT> struct SpAdaptLayer<4, CIN, COUT> { using T = SpCfg<12, 5, CIN, COUT, SP_POOL_ADAPT, 3>; };
template <int CIN, int COUT> struct SpAdaptLayer<5, CIN, COUT> { using T = SpCfg<6, 3, CIN, COUT, SP_POOL_NONE, 0>; };
template <int CIN, int COUT> struct SpAdaptLayer<6, CIN, COUT> { using T = SpCfg<6, 3, CIN, COUT, SP_POOL_NONE, 0, true, true>; };
template <int L, int CIN, int COUT> using SpAdapt = typename SpAdaptLayer<L, CIN, COUT>::T;
// X(layer, CIN, COUT) for every AdaptCNN instance
#define NISQA_SP_ANY_TO(X, L, CO) X(L, 16, CO) X(L, 32, CO) X(L, 64, CO)
#define NISQA_SP_ADAPT_LAYERS(X)                                                                   \
  NISQA_SP_ANY_TO(X, 2, 16) NISQA_SP_ANY_TO(X, 2, 32) NISQA_SP_ANY_TO(X, 2, 64)                   \
  NISQA_SP_ANY_TO(X, 3, 16) NISQA_SP_ANY_TO(X, 3, 32) NISQA_SP_ANY_TO(X, 3, 64)                   \
  X(4, 16, 16) X(4, 32, 32) X(4, 64, 64) X(5, 16, 16) X(5, 32, 32) X(5, 64, 64) X(6, 16, 16) X(6, 32, 32) X(6, 64, 64)
// the shipped 16 / 32 / 64 AdaptCNN (the same types as SpAdapt's)
using SpConv2A = SpCfg<24, 7, 16, 32, SP_POOL_ADAPT, 5>;
using SpConv3A = SpCfg<12, 5, 32, 64, SP_POOL_NONE, 0>;
using SpConv4A = SpCfg<12, 5, 64, 64, SP_POOL_ADAPT, 3>;
using SpConv5A = SpCfg<6, 3, 64, 64, SP_POOL_NONE, 0>;
using SpConv6A = SpCfg<6, 3, 64, 64, SP_POOL_NONE, 0, true, true>;
static_assert(std::is_same<SpConv2A, SpAdapt<2, 16, 32>>::value && std::is_same<SpConv3A, SpAdapt<3, 32, 64>>::value &&
              std::is_same<SpConv4A, SpAdapt<4, 64, 64>>::value && std::is_same<SpConv5A, SpAdapt<5, 64, 64>>::value &&
              std::is_same<SpConv6A, SpAdapt<6, 64, 64>>::value, "shipped AdaptCNN layers");
using SpConv2S = SpCfg<24, 8, 16, 32, SP_POOL_2X2, 4>;
using SpConv3S = SpCfg<12, 4, 32, 64, SP_POOL_NONE, 0>;
using SpConv4S = SpCfg<12, 4, 64, 64, SP_POOL_2X2, 2>;
using SpConv5S = SpCfg<6, 2, 64, 64, SP_POOL_NONE, 0>;
using SpConv6S = SpCfg<6, 2, 64, 64, SP_POOL_NONE, 0, true>;

// A run-time geometry layer: AdaptCNN conv layer L (2..6) whose map sizes come from the checkpoint's pools
// (cnn_pool_1/2/3) and reach the kernel as its SpGeom argument.
//   conv2..conv5: 3 x 3 taps, padding 1, output H x W, then (conv2, conv4) F.adaptive_max_pool2d to HO x WO.
//   conv6: NTAP = 3 x KX taps (KX = its input width 1..3), padding (1, 0): output H x 1, the fp32 CNN features.
// Shared memory is sized for the largest accepted map: a 256-row tile whose halo is kSplitLead rows.
template <int L, int CIN_, int COUT_, int NTAP_ = 9>
struct SpRt : SpLayout<NTAP_, 256 + 2 * kSplitLead, CIN_, COUT_> {
  static constexpr int KX = NTAP_ / 3, PADX = L == 6 ? 0 : 1;
  static constexpr int POOL = (L == 2 || L == 4) ? SP_POOL_ADAPT : SP_POOL_NONE;
  static constexpr bool RT = true;
  static constexpr bool ONE_STEP_UNITS = L == 2 && COUT_ == 64, OUT_SPLIT = L != 6;
  // the argument, whose first column (X0 = 1 for every run-time geometry layer) stays a constant
  __host__ __device__ static constexpr SpGeom geom(SpGeom g) {
    g.X0 = 1;
    return g;
  }
  static_assert(NTAP_ % 3 == 0 && (L == 6 || NTAP_ == 9), "taps");
};
// X(layer, CIN, COUT, NTAP) for every run-time geometry instance: the (layer, CIN, COUT) of NISQA_SP_ADAPT_LAYERS for
// conv2..conv5, conv6 per width and tap count 3, 6, 9 (pool_3 widths 1, 2, 3)
#define NISQA_SP_RT_TO(X, L, CO) X(L, 16, CO, 9) X(L, 32, CO, 9) X(L, 64, CO, 9)
#define NISQA_SP_RT_C6(X, C) X(6, C, C, 3) X(6, C, C, 6) X(6, C, C, 9)
#define NISQA_SP_RT_LAYERS(X)                                                                          \
  NISQA_SP_RT_TO(X, 2, 16) NISQA_SP_RT_TO(X, 2, 32) NISQA_SP_RT_TO(X, 2, 64)                           \
  NISQA_SP_RT_TO(X, 3, 16) NISQA_SP_RT_TO(X, 3, 32) NISQA_SP_RT_TO(X, 3, 64)                           \
  X(4, 16, 16, 9) X(4, 32, 32, 9) X(4, 64, 64, 9) X(5, 16, 16, 9) X(5, 32, 32, 9) X(5, 64, 64, 9)     \
  NISQA_SP_RT_C6(X, 16) NISQA_SP_RT_C6(X, 32) NISQA_SP_RT_C6(X, 64)

// Shared memory of the fused conv1 + conv2 kernel (conv12_kernel) on the conv2 geometry C: three activation buffers
// (conv1 fills one while the two MMA warpgroups read the other two), one staging tile per MMA warpgroup and a ring of
// MEL_R mel blocks (one segment's kSegLen frames x kMels, copied whole by one cp.async.bulk; 16-byte aligned like its
// source) with the segment's clamp threshold beside each.
template <class C>
struct SpFused {
  static constexpr int A_BUFS = 3;
  static constexpr int OFF_A = 0;                         // buffer b at b * C::A_BUF (1024-aligned: A_BYTES is)
  static constexpr int OFF_STG = A_BUFS * C::A_BUF;       // MMA warpgroup w's staging tile at OFF_STG + w * C::STG_BYTES
  static constexpr int OFF_B = (OFF_STG + 2 * C::STG_BYTES + 1023) & ~1023;
  static constexpr int OFF_W1 = OFF_B + 9 * C::B_STAGE;   // conv1 weights [9][16] + biases [16]
  static constexpr int MEL_R = 4;                         // ring slots: tile j + 2's copy lands during conv1 of tile j
  static constexpr int MEL_BYTES = kSegLen * kMels * 4;   // 2880
  static constexpr int OFF_MEL = OFF_W1 + 1024;           // slot s at OFF_MEL + s * MEL_BYTES
  static constexpr int OFF_THR = OFF_MEL + MEL_R * MEL_BYTES;   // float [MEL_R]
  // 9 weight-tap barriers, then A full[A_BUFS], A empty[A_BUFS], mel full[MEL_R], mel empty[MEL_R]
  static constexpr int OFF_BAR = OFF_THR + 4 * MEL_R;
  static constexpr int SMEM_BYTES = OFF_BAR + 8 * (9 + 2 * A_BUFS + 2 * MEL_R) + 1024;
  static_assert(!C::ALIAS && C::G == 1 && C::CIN == 16, "conv2 geometry");
  static_assert(C::NBLK == 3, "an MMA warpgroup runs m64 blocks 0, 1 and 2 of its tile");
  static_assert(MEL_BYTES % 16 == 0 && OFF_MEL % 16 == 0 && OFF_BAR % 8 == 0, "bulk copy / mbarrier alignment");
  static_assert(SMEM_BYTES <= C::SMEM_BUDGET, "shared memory budget");
};

}  // namespace nisqa

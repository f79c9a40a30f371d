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

template <int H_, int W_, int CIN_, int COUT_, int POOL_, int POW_, bool F32OUT_ = false, bool CENTER_ = false>
struct SpCfg {
  static constexpr int NT = 4 * 128;             // four warpgroups; warpgroup b < NBLK runs m64 block b
  static constexpr int H = H_, W = W_, CIN = CIN_, COUT = COUT_, POOL = POOL_, POW = POW_;
  static constexpr int NTAP = 9;                  // weight taps (3 x 3)
  static constexpr bool ONE_STEP_UNITS = H == 24 && COUT == 64;   // conv2 at 64 output channels (TapUnits)
  static constexpr bool CENTER = CENTER_;         // conv6 of the AdaptCNN: kernel (3,3), padding (1,0) on a
                                                  // 3-wide map == the padded conv evaluated at column 1 only
  static constexpr bool OUT_SPLIT = !F32OUT_;     // the last layer writes the CNN features as fp32 channels-last
  static constexpr int P = W + 1;                 // row pitch: W interior columns + 1 shared zero column
  static constexpr int BLK = (H + 1) * P;         // rows per segment: H interior rows + 1 shared zero row
  static constexpr int G = 256 / BLK;             // segments per tile (256 GEMM rows)
  static constexpr int HALO = P + 1;              // |row offset| of the farthest tap
  static constexpr int AROWS = 256 + 2 * HALO;    // rows of the tile (copied)
  // GEMM rows: only the tile's interior output positions, in (segment, h, w) order (conv6A: the centre column only),
  // packed into NBLK m64 blocks.  GEMM row m reads its taps around tile row HALO + gemm_row(m).
  static constexpr int KW = CENTER ? 1 : W;       // output columns per row
  static constexpr int SEG_ROWS = H * KW;         // GEMM rows per segment
  static constexpr int KEPT = G * SEG_ROWS;
  static constexpr int NBLK = (KEPT + 63) / 64;
  // plane row of GEMM row m, counted from the zero row of the tile's first segment.  Rows m >= KEPT read that zero row;
  // the rows of segments past the end of a short last tile read the copied range as it lies.  Neither is staged.
  __host__ __device__ static constexpr int gemm_row(int m) {
    if (m >= KEPT) return 0;
    const int s = m / SEG_ROWS, q = m - s * SEG_ROWS, h = q / KW, w = q - h * KW;
    return s * BLK + (h + 1) * P + (CENTER ? 2 : w + 1);
  }
  static constexpr int ROWB = CIN * 2;            // bytes per row
  static constexpr int A_BYTES = ((AROWS + 7) * ROWB + 1023) & ~1023;     // + placement shift (g0 & 7 rows)
  static constexpr int NCH = CIN / 8;             // 16-byte K chunks (8 halves)
  static constexpr int B_HALF = NCH * COUT * 16;  // per hi / lo
  static constexpr int B_STAGE = 2 * B_HALF;      // one tap: [CIN/8][hi co | lo co][8 halves]
  // output geometry (= the next layer's input geometry)
  static constexpr int HO = (POOL == SP_POOL_NONE) ? H : H / 2;
  static constexpr int WO = (POOL == SP_POOL_NONE) ? (CENTER ? 1 : W) : POW;
  static constexpr int OP = WO + 1, OBLK = (HO + 1) * OP, OROWB = COUT * 2;
  // fp32 output (the CNN features): one row per segment, zero-padded to a multiple of 64 columns (6 x 16 -> 128)
  static constexpr int OUT_COLS = HO * WO * COUT, OUT_LD = (OUT_COLS + 63) / 64 * 64;
  // epilogue staging: one fp32 row per GEMM row (bias + ReLU applied)
  static constexpr int STG_STRIDE = COUT + 4;
  static constexpr int STG_BYTES = 256 * STG_STRIDE * 4;
  // Three ways to fit beside the nine resident weight taps, the first that fits: the activation tile double-buffered
  // (the next tile's copy lands during this tile's GEMM and epilogue), one activation buffer beside the staging tile (the
  // next tile's copy lands during this tile's epilogue), or one buffer that the staging tile reuses (ALIAS: the copy
  // waits for the epilogue).  Buffer b: hi plane at b * A_BUF, lo plane at b * A_BUF + A_BYTES.
  static constexpr int SMEM_BUDGET = 227 * 1024 - 2048;
  static constexpr int A_BUF = 2 * A_BYTES;
  static constexpr int ONE_BUF = A_BUF + STG_BYTES + 9 * B_STAGE;     // one unaliased activation buffer
  static constexpr bool ALIAS = ONE_BUF > SMEM_BUDGET;
  static constexpr int A_BUFS = (ALIAS || ONE_BUF + A_BUF > SMEM_BUDGET) ? 1 : 2;
  static constexpr int OFF_A_HI = 0;
  static constexpr int OFF_A_LO = A_BYTES;
  static constexpr int OFF_STG = ALIAS ? 0 : A_BUFS * A_BUF;
  static constexpr int OFF_B = ((ALIAS ? (A_BUF > STG_BYTES ? A_BUF : STG_BYTES) : A_BUFS * A_BUF + STG_BYTES) + 1023) & ~1023;
  static constexpr int OFF_W1 = OFF_B + 9 * B_STAGE;      // conv1 weights [9][16] + biases [16] (fused conv1 + conv2 only)
  // 9 weight-tap barriers, then a full barrier per activation buffer, then (double-buffered) an empty barrier per buffer
  static constexpr int OFF_BAR = OFF_W1 + 1024;
  static constexpr int NBAR = 9 + 2 * A_BUFS;
  static constexpr int SMEM_BYTES = OFF_BAR + 8 * NBAR + 1024;    // + slack: the tile is aligned to 1024 B
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
  static_assert(ALIAS || A_BUFS * A_BUF + STG_BYTES + 9 * B_STAGE <= SMEM_BUDGET,
                "the activation buffers fit beside the staging tile and the weights");
  static_assert(B_STAGE % 16 == 0 && CIN % 16 == 0 && (COUT == 16 || COUT == 32 || COUT == 64), "shape");
  static_assert(ROWB == 32 || ROWB == 64 || ROWB == 128, "rows are 32 / 64 / 128 bytes (one swizzle atom)");
  static_assert(HALO <= kSplitLead, "kSplitLead");
  static_assert(!CENTER || F32OUT_, "the centre-column variant only exists as the last layer");
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

// ---- AdaptCNN layers whose map sizes come from the checkpoint's pools (cnn_pool_1/2/3) ----
// Run-time geometry of one such layer (conv_split_rt_kernel): the members of SpCfg that depend on H and W.
//   conv2..conv5: 3 x 3 taps, padding 1, output H x W, then (conv2, conv4) adaptive max-pool to HO x WO.
//   conv6: kernel (3, W), padding (1, 0): output H x 1, written as the fp32 CNN features [seg][H][COUT].
// GEMM row m reads its taps around plane row HALO + gemm_row(m), at column w + 1 (conv6: column 1).
struct SpGeom {
  int H, W, P, BLK, G, HALO, KW, SEG_ROWS, KEPT, NBLK;
  int HO, WO, OP, OBLK;      // the output map (the next layer's input): pooled, H x W, or H x 1 (conv6)
  int OUT_COLS, OUT_LD;      // conv6: H COUT features in rows of OUT_LD floats (a multiple of 64, zero-padded)
  __host__ __device__ int gemm_row(int m) const {
    if (m >= KEPT) return 0;
    const int s = m / SEG_ROWS, q = m - s * SEG_ROWS, h = q / KW, w = q - h * KW;
    return s * BLK + (h + 1) * P + w + 1;
  }
};
// (H, W) input -> (HO, WO) output of conv layer `layer` (2..6) with COUT output channels
inline SpGeom sp_geom(int layer, int H, int W, int HO, int WO, int cout) {
  SpGeom g;
  g.H = H; g.W = W; g.P = W + 1; g.BLK = (H + 1) * g.P; g.G = 256 / g.BLK; g.HALO = g.P + 1;
  g.KW = layer == 6 ? 1 : W;
  g.SEG_ROWS = H * g.KW; g.KEPT = g.G * g.SEG_ROWS; g.NBLK = (g.KEPT + 63) / 64;
  g.HO = layer == 6 ? H : HO; g.WO = layer == 6 ? 1 : WO;
  g.OP = g.WO + 1; g.OBLK = (g.HO + 1) * g.OP;
  g.OUT_COLS = g.HO * g.WO * cout; g.OUT_LD = (g.OUT_COLS + 63) / 64 * 64;
  return g;
}

// Compile-time part of a run-time geometry layer L (2..6) with CIN -> COUT channels and NTAP = 3 x KX weight taps (conv6:
// KX = its input width 1..3; the others 3 x 3 with padding 1).  Shared memory is sized for the largest accepted map, a
// 256-row tile whose halo is kSplitLead rows; otherwise the layout rules are SpCfg's.
template <int L, int CIN_, int COUT_, int NTAP_ = 9>
struct SpRt {
  static constexpr int NT = 4 * 128;
  static constexpr int CIN = CIN_, COUT = COUT_, NTAP = NTAP_, KX = NTAP / 3, PADX = L == 6 ? 0 : 1;
  static constexpr bool ONE_STEP_UNITS = L == 2 && COUT == 64;
  static constexpr bool POOLED = L == 2 || L == 4, OUT_SPLIT = L != 6;
  static constexpr int AROWS = 256 + 2 * kSplitLead;
  static constexpr int ROWB = CIN * 2;
  static constexpr int A_BYTES = ((AROWS + 7) * ROWB + 1023) & ~1023;
  static constexpr int NCH = CIN / 8;
  static constexpr int B_HALF = NCH * COUT * 16;
  static constexpr int B_STAGE = 2 * B_HALF;
  static constexpr int STG_STRIDE = COUT + 4;
  static constexpr int STG_BYTES = 256 * STG_STRIDE * 4;
  static constexpr int SMEM_BUDGET = 227 * 1024 - 2048;
  static constexpr int A_BUF = 2 * A_BYTES;
  static constexpr int ONE_BUF = A_BUF + STG_BYTES + NTAP * B_STAGE;
  static constexpr bool ALIAS = ONE_BUF > SMEM_BUDGET;
  static constexpr int A_BUFS = (ALIAS || ONE_BUF + A_BUF > SMEM_BUDGET) ? 1 : 2;
  static constexpr int OFF_A_HI = 0;
  static constexpr int OFF_A_LO = A_BYTES;
  static constexpr int OFF_STG = ALIAS ? 0 : A_BUFS * A_BUF;
  static constexpr int OFF_B = ((ALIAS ? (A_BUF > STG_BYTES ? A_BUF : STG_BYTES) : A_BUFS * A_BUF + STG_BYTES) + 1023) & ~1023;
  static constexpr int OFF_BAR = OFF_B + NTAP * B_STAGE;
  static constexpr int NBAR = NTAP + 2 * A_BUFS;
  static constexpr int SMEM_BYTES = OFF_BAR + 8 * NBAR + 1024;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
  static_assert(ALIAS || A_BUFS * A_BUF + STG_BYTES + NTAP * B_STAGE <= SMEM_BUDGET, "buffers");
  static_assert(CIN % 16 == 0 && (COUT == 16 || COUT == 32 || COUT == 64), "shape");
  static_assert(NTAP % 3 == 0 && (L == 6 || NTAP == 9), "taps");
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

// Shared memory of the fused conv1 + conv2 kernel (conv12_kernel) on the conv2 geometry C: two activation buffers
// (conv1 fills one while the GEMM reads the other), two staging tiles (tile i's is written while stragglers of the
// MMA warpgroups may still read tile i - 1's) and a ring of MEL_R mel blocks (one segment's kSegLen frames x kMels,
// copied whole by one cp.async.bulk; 16-byte aligned like its source) with the segment's clamp threshold beside each.
template <class C>
struct SpFused {
  static constexpr int OFF_A = 0;                         // buffer b at b * C::A_BUF (1024-aligned: A_BYTES is)
  static constexpr int OFF_STG = 2 * C::A_BUF;            // staging tile b at OFF_STG + b * C::STG_BYTES
  static constexpr int OFF_B = (OFF_STG + 2 * C::STG_BYTES + 1023) & ~1023;
  static constexpr int OFF_W1 = OFF_B + 9 * C::B_STAGE;   // conv1 weights [9][16] + biases [16]
  static constexpr int MEL_R = 4;                         // ring slots: tile j + 2's copy lands while tile j computes
  static constexpr int MEL_BYTES = kSegLen * kMels * 4;   // 2880
  static constexpr int OFF_MEL = OFF_W1 + 1024;           // slot s at OFF_MEL + s * MEL_BYTES
  static constexpr int OFF_THR = OFF_MEL + MEL_R * MEL_BYTES;   // float [MEL_R]
  // 9 weight-tap barriers, then A full[2], A empty[2], mel full[MEL_R], mel empty[MEL_R]
  static constexpr int OFF_BAR = OFF_THR + 4 * MEL_R;
  static constexpr int SMEM_BYTES = OFF_BAR + 8 * (13 + 2 * MEL_R) + 1024;
  static_assert(!C::ALIAS && C::G == 1 && C::CIN == 16, "conv2 geometry");
  static_assert(C::NBLK == 3, "the MMA warpgroups run m64 blocks {0, 1} and {2}");
  static_assert(MEL_BYTES % 16 == 0 && OFF_MEL % 16 == 0 && OFF_BAR % 8 == 0, "bulk copy / mbarrier alignment");
  static_assert(SMEM_BYTES <= C::SMEM_BUDGET, "shared memory budget");
};

}  // namespace nisqa

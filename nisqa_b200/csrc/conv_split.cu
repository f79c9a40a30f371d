// conv_split.cu - conv2..conv6 of the AdaptCNN / StandardCNN (reference nisqa/NISQA_lib.py:692-706,
// 816-830) as implicit GEMMs on the Hopper tensor cores (wgmma), with an error-compensated two-term FP16 split so
// that the result stays within fp32 rounding noise of the reference (plain TF32 / BF16 operands move MOS by
// 2e-3 / 1.7e-2, SURVEY.md 0.8):
//      a = a_hi + a_lo,  b = b_hi + b_lo      (fp16 parts: 11 + 11 significant bits)
//      a*b ~= a_hi*b_hi + a_hi*b_lo + a_lo*b_hi          (dropped a_lo*b_lo ~ 2^-22 |a b|)
// The main accumulator only ever sees the hi*hi products; hi*lo and lo*hi go to a second, small accumulator, and the
// epilogue adds the two.  The weights are pre-scaled by 2^S on the host (S chosen per layer so that max|w| 2^S <= 1024)
// to keep b_lo out of the fp16 subnormal range; the epilogue multiplies by 2^-S (exact).  Activations are stored
// multiplied by 2^-e (e per layer, from its folded BatchNorm) for the same reason; the consuming layer's epilogue
// multiplies by 2^(e_in - S).  Every stored fp16 value is therefore unchanged when a checkpoint is rescaled by
// powers of two (BatchNorm i times 2^k, conv i+1 times 2^-k), and so is every score.
//
// The activations travel BETWEEN the layers already in the form the GEMM consumes: two fp16 planes (hi, lo), laid out
// in HBM as the exact shared-memory image of the A tile:
//
//   plane row g(seg, hh, ww) = kSplitLead + seg * BLK + hh * P + ww,   P = W + 1, BLK = (H + 1) * P
//     hh = 0 / ww = 0 are the shared zero row / zero column (never written: the planes are zeroed
//     when they are allocated), interior positions are hh = h + 1, ww = w + 1
//   row = CIN halves (32 / 64 / 128 bytes); the 16-byte chunk c of row g sits at chunk position
//     c ^ f(g), f = the 32B / 64B / 128B swizzle of a row whose index is == g (mod 8)
//
// so that a tile's activations (256 + 2 * HALO consecutive rows, two planes) arrive with TWO cp.async.bulk copies
// issued by one thread (placed at row offset g0 & 7 inside a 1024-byte aligned buffer, so that the swizzle phase of
// every row is its plane row's), and the producing layer's epilogue does the split once, right where the fp32 value
// exists.  The 9 taps are the same tile read at row-shifted addresses: im2col is never materialised.
//
// GEMM view:  D[pos, co] = sum_{tap, ci} X[pos + off(tap), ci] * W[tap][co][ci]
//   M = the interior output positions of G segments (SpCfg::gemm_row: GEMM row -> plane row; the zero row / column
//   positions are not computed), N = C_out, K = 9 * C_in.  Warpgroup b < NBLK owns GEMM rows 64 b .. 64 b + 63: A
//   fragments come from the swizzled tile with ldmatrix, one gathered row address per lane (8 rows of distinct
//   plane row mod 8 hit 8 distinct 16-byte bank groups; a group that crosses a zero column may repeat one), B
//   (all nine weight taps, resident for the CTA's life) through shared-memory descriptors, accumulators in
//   registers.  CTAs are persistent: the weights are loaded once per CTA, the tiles are walked with a grid stride.
//   Epilogue: registers -> bias / ReLU -> fp32 staging tile -> (max-pool) -> split -> planes of the next layer.
//   One tap (CIN <= 32) or half a tap (CIN 64) is kept in flight: its A fragments load while the previous unit's
//   wgmmas run.  Where the staging tile does not alias the A tile, the A tile is double-buffered (conv_split_kernel).
//
// The fused kernel (conv12_kernel) also computes conv1 + BN + ReLU + pool1 of the tile's segment straight into the A
// tile, so pool1 never reaches HBM; two warpgroups run the GEMM while the other two compute conv1 of the next tile
// and the epilogue of the previous one.
#include <cuda_fp16.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "conv1_cell.cuh"
#include "conv_split.cuh"
#include "launch.cuh"
#include "tc_ptx.cuh"

namespace nisqa {

// ---- pieces shared by the two kernels ----

// The K steps of one tap go to the tensor cores in units of UK k16 steps: a whole tap for CIN <= 32, half a tap for
// CIN 64 (two fragment sets of a whole 64-channel tap do not fit beside the accumulators in 128 registers).  conv2 at
// 64 output channels (24 x 7 maps) takes one k16 step per unit: with two, ptxas spills (CIN 32: 16 bytes, CIN 64: 72).
template <class C>
struct TapUnits {
  static constexpr int KS = C::CIN / 16, UK = (KS < 2 || C::ONE_STEP_UNITS) ? 1 : 2, PER_TAP = KS / UK,
                       N = C::NTAP * PER_TAP;
};

// A fragments of K steps k0 .. k0 + UK - 1 of one tap (row offset tapoff) for this warpgroup's NB m64 blocks: block b
// reads tile row row[b] + tapoff
template <class C, int NB>
__device__ __forceinline__ void load_unit(uint32_t a_hi, uint32_t a_lo, const int (&row)[NB], int tapoff, int k0, int lchunk,
                                          uint32_t (&ah)[NB][TapUnits<C>::UK][4], uint32_t (&al)[NB][TapUnits<C>::UK][4]) {
#pragma unroll
  for (int b = 0; b < NB; ++b)
#pragma unroll
    for (int ks = 0; ks < TapUnits<C>::UK; ++ks) {
      const uint32_t ao = (uint32_t)split_off<C::ROWB>(row[b] + tapoff, 2 * (k0 + ks) + lchunk);
      ldsm_x4(a_hi + ao, ah[b][ks]);
      ldsm_x4(a_lo + ao, al[b][ks]);
    }
}

// the wgmmas of K steps k0 .. k0 + UK - 1 of one tap (weights at bst) for NB m64 blocks; no fence / commit
template <class C, int NB>
__device__ __forceinline__ void mma_unit(float (&acc_m)[NB][C::COUT / 2], float (&acc_s)[NB][C::COUT / 2],
                                         const uint32_t (&ah)[NB][TapUnits<C>::UK][4],
                                         const uint32_t (&al)[NB][TapUnits<C>::UK][4], uint32_t bst, int k0) {
  constexpr int COUT = C::COUT;
#pragma unroll
  for (int b = 0; b < NB; ++b)
#pragma unroll
    for (int ks = 0; ks < TapUnits<C>::UK; ++ks) {
      const uint32_t bk = bst + (uint32_t)(2 * (k0 + ks)) * (2 * COUT * 16);
      const uint64_t dbh = make_desc_b(bk, 2 * COUT * 16), dbl = make_desc_b(bk + COUT * 16, 2 * COUT * 16);
      wgmma_rs<COUT>(acc_m[b], ah[b][ks], dbh);
      wgmma_rs<COUT>(acc_s[b], ah[b][ks], dbl);
      wgmma_rs<COUT>(acc_s[b], al[b][ks], dbh);
    }
}

// All nine weight taps have landed.  Called before tile_gemm, never between its in-flight wgmmas: a wait loop there
// makes ptxas serialize them.
__device__ __forceinline__ void wait_weights(uint32_t bar_w) {
  for (int t = 0; t < 9; ++t) mbar_wait(bar_w + 8 * t, 0);
}

// The GEMM of one tile for this warpgroup's NB m64 blocks: acc_m[b] = hi*hi, acc_s[b] = hi*lo + lo*hi over the nine
// taps, in tap order.  row[b] is this lane's ldmatrix row of block b at tap offset 0.  The weights must have landed
// (wait_weights).
template <class C, int NB>
__device__ __forceinline__ void tile_gemm(float (&acc_m)[NB][C::COUT / 2], float (&acc_s)[NB][C::COUT / 2], uint32_t a_hi,
                                          uint32_t a_lo, uint32_t b_base, const int (&row)[NB], int lchunk) {
  using U = TapUnits<C>;
  constexpr int P = C::P, UK = U::UK, PT = U::PER_TAP;
  static_assert(C::CIN <= 32 || NB == 1, "CIN 64: one m64 block per warpgroup");
#pragma unroll
  for (int b = 0; b < NB; ++b)
#pragma unroll
    for (int i = 0; i < C::COUT / 2; ++i) { acc_m[b][i] = 0.f; acc_s[b][i] = 0.f; }
  // one unit in flight: unit u + 1's fragments load into the other register set while unit u's wgmmas run
  uint32_t ah[2][NB][UK][4], al[2][NB][UK][4];
  load_unit<C, NB>(a_hi, a_lo, row, -P - 1, 0, lchunk, ah[0], al[0]);
#pragma unroll
  for (int u = 0; u < U::N; ++u) {
    wgmma_fence();
    mma_unit<C, NB>(acc_m, acc_s, ah[u & 1], al[u & 1], b_base + (u / PT) * C::B_STAGE, (u % PT) * UK);
    wgmma_commit();
    if (u + 1 < U::N) {
      wgmma_wait<1>();                           // unit u - 1 is done with the set that unit u + 1 loads into
      const int v = u + 1, t = v / PT;
      load_unit<C, NB>(a_hi, a_lo, row, (t / 3 - 1) * P + (t % 3 - 1), (v % PT) * UK, lchunk, ah[v & 1], al[v & 1]);
    }
  }
  wgmma_wait<0>();
}

// this lane's accumulator columns of the bias: bb[j] = bias[8 j + acol], bias[8 j + acol + 1]
template <class C>
__device__ __forceinline__ void load_bias(const float* __restrict__ bias, int acol, float2 (&bb)[C::COUT / 8]) {
#pragma unroll
  for (int j = 0; j < C::COUT / 8; ++j) bb[j] = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + acol));
}

// epilogue part 1 for one m64 block: accumulators of GEMM rows m0 and m0 + 8 -> bias (load_bias) + ReLU -> the staging
// rows of their plane positions (every interior position of the tile's live segments is written: store_tile reads them
// all)
template <class C>
__device__ __forceinline__ void stage_rows(const float (&acc_m)[C::COUT / 2], const float (&acc_s)[C::COUT / 2], int m0,
                                           int acol, int seg0, int n_seg, const float2 (&bb)[C::COUT / 8], float out_scale,
                                           float* stg) {
  constexpr int SS = C::STG_STRIDE;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int m = m0 + 8 * half;
    if (m < C::KEPT && seg0 + m / C::SEG_ROWS < n_seg) {
      const int r = C::gemm_row(m);
#pragma unroll
      for (int j = 0; j < C::COUT / 8; ++j) {
        const int col = 8 * j + acol;
        const float v0 = fmaxf(fmaf(acc_m[4 * j + 2 * half] + acc_s[4 * j + 2 * half], out_scale, bb[j].x), 0.f);
        const float v1 = fmaxf(fmaf(acc_m[4 * j + 2 * half + 1] + acc_s[4 * j + 2 * half + 1], out_scale, bb[j].y), 0.f);
        *reinterpret_cast<float2*>(stg + r * SS + col) = make_float2(v0, v1);
      }
    }
  }
}

// epilogue part 2 (threads t0, t0 + nthr, ...): staging tile -> max-pool / split / store of the tile's nvalid segments
template <class C>
__device__ __forceinline__ void store_tile(const float* stg, int seg0, int nvalid, int t0, int nthr, float store_scale,
                                           unsigned char* __restrict__ out_hi, unsigned char* __restrict__ out_lo,
                                           float* __restrict__ out_f32) {
  constexpr int H = C::H, W = C::W, COUT = C::COUT, P = C::P, BLK = C::BLK, SS = C::STG_STRIDE;
  if constexpr (C::POOL != SP_POOL_NONE) {
    constexpr int POW = C::POW, HO = H / 2, C8 = COUT / 8;
    for (int i = t0; i < nvalid * HO * POW * C8; i += nthr) {
      const int c8 = i % C8;
      int rest = i / C8;
      const int pw = rest % POW; rest /= POW;
      const int ph = rest % HO;
      const int s = rest / HO;
      int x0, x1;
      if (C::POOL == SP_POOL_ADAPT) { x0 = (pw * W) / POW; x1 = ((pw + 1) * W + POW - 1) / POW; }
      else { x0 = 2 * pw; x1 = 2 * pw + 2; }
      float4 ma = make_float4(0.f, 0.f, 0.f, 0.f), mb = ma;       // post-ReLU values are >= 0
      for (int hy = 2 * ph; hy < 2 * ph + 2; ++hy)
        for (int x = x0; x < x1; ++x) {
          const float4* tp = reinterpret_cast<const float4*>(stg + (s * BLK + (hy + 1) * P + (x + 1)) * SS + c8 * 8);
          const float4 ta = tp[0], tb = tp[1];
          ma.x = fmaxf(ma.x, ta.x); ma.y = fmaxf(ma.y, ta.y); ma.z = fmaxf(ma.z, ta.z); ma.w = fmaxf(ma.w, ta.w);
          mb.x = fmaxf(mb.x, tb.x); mb.y = fmaxf(mb.y, tb.y); mb.z = fmaxf(mb.z, tb.z); mb.w = fmaxf(mb.w, tb.w);
        }
      uint4 hi, lo;
      split8(ma, mb, store_scale, hi, lo);
      const int g = kSplitLead + (seg0 + s) * C::OBLK + (ph + 1) * C::OP + (pw + 1);
      const size_t o = split_off<C::OROWB>(g, c8);
      *reinterpret_cast<uint4*>(out_hi + o) = hi;
      *reinterpret_cast<uint4*>(out_lo + o) = lo;
    }
  } else if constexpr (C::OUT_SPLIT) {
    // the whole image of the tile's segments, zero row / column positions included (as zeros)
    constexpr int C8 = COUT / 8;
    for (int i = t0; i < nvalid * BLK * C8; i += nthr) {
      const int c8 = i % C8, r = i / C8;
      const int q = r % BLK, hh = q / P, ww = q - hh * P;
      uint4 hi = make_uint4(0u, 0u, 0u, 0u), lo = hi;
      if (hh >= 1 && ww >= 1) {
        const float4* tp = reinterpret_cast<const float4*>(stg + r * SS + c8 * 8);
        split8(tp[0], tp[1], store_scale, hi, lo);
      }
      const size_t o = split_off<C::OROWB>(kSplitLead + seg0 * BLK + r, c8);
      *reinterpret_cast<uint4*>(out_hi + o) = hi;
      *reinterpret_cast<uint4*>(out_lo + o) = lo;
    }
  } else {
    // fp32 CNN features, channels-last [seg][HO][WO][COUT] in rows of OUT_LD floats
    constexpr int HO = C::HO, WO = C::WO, C4 = COUT / 4;
    for (int i = t0; i < nvalid * HO * WO * C4; i += nthr) {
      const int c4 = i % C4;
      int rest = i / C4;
      const int w = rest % WO; rest /= WO;
      const int h = rest % HO;
      const int s = rest / HO;
      const int r = s * BLK + (h + 1) * P + (C::CENTER ? 2 : w + 1);
      float* dst = C::OUT_LD == C::OUT_COLS ? out_f32 + ((size_t)(seg0 + s) * (HO * WO) + h * WO + w) * COUT + c4 * 4
                                            : out_f32 + (size_t)(seg0 + s) * C::OUT_LD + (h * WO + w) * COUT + c4 * 4;
      *reinterpret_cast<float4*>(dst) = *reinterpret_cast<const float4*>(stg + r * SS + c4 * 4);
    }
    if constexpr (C::OUT_LD > C::OUT_COLS) {
      // the padding columns are written as zeros: the Linear behind reads them (against zero weights)
      constexpr int PAD4 = (C::OUT_LD - C::OUT_COLS) / 4;
      for (int i = t0; i < nvalid * PAD4; i += nthr)
        *reinterpret_cast<float4*>(out_f32 + (size_t)(seg0 + i / PAD4) * C::OUT_LD + C::OUT_COLS + (i % PAD4) * 4) =
            make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// ---- conv2..conv6 on planes ----
// Warpgroup b < NBLK owns m64 block b (3 blocks, 1 for conv6A) and runs GEMM and epilogue part 1; all four run part 2.
// One warpgroup's wgmmas already use the tensor cores of all four SM sub-partitions.  With two activation buffers (the
// shipped conv2, conv3) one thread issues the next tile's copy into the other buffer as soon as that buffer's readers
// (the previous tile's GEMM) have arrived on its empty barrier; with one unaliased buffer (CIN 64 -> COUT 32) it issues
// the copy once this tile's GEMM is done, so that it lands during the epilogue.
template <class C>
__global__ void __launch_bounds__(C::NT, 1)
conv_split_kernel(const unsigned char* __restrict__ in_hi, const unsigned char* __restrict__ in_lo,
                  const __half* __restrict__ wtc /*[9][CIN/8][hi co | lo co][8] fp16, scaled by 2^S*/,
                  const float* __restrict__ bias, float out_scale /*2^(e_in - S)*/, float store_scale /*2^-e_out*/,
                  unsigned char* __restrict__ out_hi, unsigned char* __restrict__ out_lo,
                  float* __restrict__ out_f32 /*last layer only*/, int n_seg) {
  constexpr int G = C::G, BLK = C::BLK, HALO = C::HALO, ROWB = C::ROWB, NT = C::NT;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // swizzle atoms repeat every 1024 B
  const uint32_t sbase = smem_u32(smem);
  const uint32_t b_base = sbase + C::OFF_B;
  const uint32_t bar_w = sbase + C::OFF_BAR, bar_full = bar_w + 8 * 9, bar_empty = bar_full + 8 * C::A_BUFS;
  float* stg = reinterpret_cast<float*>(smem + C::OFF_STG);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int n_tiles = (n_seg + G - 1) / G;

  // one thread: both planes of tile `tile` into activation buffer b, placed at row g0 & 7 (tile row == plane row mod 8)
  auto issue_tile = [&](int tile, int b) {
    constexpr uint32_t A_COPY = (uint32_t)C::AROWS * ROWB;
    const int g0 = kSplitLead + tile * G * BLK - HALO;
    const uint32_t dst = sbase + C::OFF_A_HI + b * C::A_BUF + (uint32_t)(g0 & 7) * ROWB;
    mbar_expect_tx(bar_full + 8 * b, 2 * A_COPY);
    bulk_g2s(dst, in_hi + (size_t)g0 * ROWB, A_COPY, bar_full + 8 * b);
    bulk_g2s(dst + C::A_BYTES, in_lo + (size_t)g0 * ROWB, A_COPY, bar_full + 8 * b);
  };

  if (tid == 0) {
    for (int t = 0; t < 9; ++t) mbar_init(bar_w + 8 * t, 1);
    for (int b = 0; b < C::A_BUFS; ++b) mbar_init(bar_full + 8 * b, 1);
    if constexpr (C::A_BUFS == 2)
      for (int b = 0; b < 2; ++b) mbar_init(bar_empty + 8 * b, NT);
    fence_barrier_init();
    for (int t = 0; t < 9; ++t) {                // all nine taps stay resident; tap t's MMAs start once it has landed
      mbar_expect_tx(bar_w + 8 * t, C::B_STAGE);
      bulk_g2s(b_base + t * C::B_STAGE, wtc + (size_t)t * (C::B_STAGE / 2), C::B_STAGE, bar_w + 8 * t);
    }
    if constexpr (!C::ALIAS) issue_tile(blockIdx.x, 0);
  }
  __syncthreads();

  // this lane's ldmatrix row (the tile row of GEMM row m within its warp's 16 rows) and K chunk; its accumulator rows
  const int lrow = HALO + C::gemm_row(wg * 64 + (warp & 3) * 16 + (lane & 7) + ((lane >> 3) & 1) * 8);
  const int lchunk = lane >> 4;
  const int arow0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int acol = 2 * (lane & 3);

  int it = 0;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
    const int seg0 = tile * G;
    const int g0 = kSplitLead + seg0 * BLK - HALO;         // first plane row of this tile
    const int ab = C::A_BUFS == 1 ? 0 : (it & 1);
    if constexpr (C::ALIAS) {
      if (tid == 0) issue_tile(tile, 0);
      mbar_wait(bar_full, it & 1);
    } else if constexpr (C::A_BUFS == 1) {
      mbar_wait(bar_full, it & 1);               // issued by the prologue or the previous tile
    } else {
      const int next = tile + gridDim.x;
      if (tid == 0 && next < n_tiles) {
        const int nb = (it + 1) & 1;
        mbar_wait(bar_empty + 8 * nb, (((it + 1) >> 1) & 1) ^ 1);   // tile it - 1's GEMM is done with buffer nb
        issue_tile(next, nb);
      }
      mbar_wait(bar_full + 8 * ab, (it >> 1) & 1);
    }

    // ===== GEMM: warpgroup wg < NBLK, GEMM rows 64 wg .. 64 wg + 63; the others have no rows and wait =====
    const uint32_t a_hi = sbase + C::OFF_A_HI + ab * C::A_BUF, a_lo = a_hi + C::A_BYTES;
    // The accumulators are defined on both sides of the branch and its condition is broadcast from lane 0: without
    // either, ptxas spills (CIN 64) or serializes the wgmmas (CIN <= 32).
    float acc_m[1][C::COUT / 2], acc_s[1][C::COUT / 2];      // hi*hi ; hi*lo + lo*hi
#pragma unroll
    for (int i = 0; i < C::COUT / 2; ++i) { acc_m[0][i] = 0.f; acc_s[0][i] = 0.f; }
    if (__shfl_sync(0xffffffffu, wg < C::NBLK, 0)) {
      const int row[1] = {(g0 & 7) + lrow};
      wait_weights(bar_w);
      tile_gemm<C, 1>(acc_m, acc_s, a_hi, a_lo, b_base, row, lchunk);
    }
    if constexpr (C::A_BUFS == 2) mbar_arrive(bar_empty + 8 * ab);
    __syncthreads();                             // ALIAS: every warpgroup is done with the A tile the staging tile
                                                 // overwrites; otherwise the previous tile's part 2 is done with it
    if constexpr (!C::ALIAS && C::A_BUFS == 1) {
      if (tid == 0 && tile + (int)gridDim.x < n_tiles) issue_tile(tile + gridDim.x, 0);   // the GEMM is done with it
    }

    // ===== epilogue part 1: accumulators -> bias + ReLU -> staging row of each GEMM row's plane position =====
    float2 bb[C::COUT / 8];
    load_bias<C>(bias, acol, bb);
    stage_rows<C>(acc_m[0], acc_s[0], arow0, acol, seg0, n_seg, bb, out_scale, stg);   // (no rows past block NBLK - 1)
    __syncthreads();

    // ===== epilogue part 2 (all threads): max-pool / split / store =====
    store_tile<C>(stg, seg0, min(G, n_seg - seg0), tid, NT, store_scale, out_hi, out_lo, out_f32);
    if constexpr (C::ALIAS) {
      fence_proxy_async();                       // staging stores (generic proxy) before the next tile's bulk copy
      __syncthreads();
    }
  }
}

// ---- conv2..conv6 of an AdaptCNN with other pools: the same kernel on a run-time geometry ----
// The pieces below are tile_gemm / stage_rows / store_tile with SpGeom's sizes in place of SpCfg's: the same tap order, the
// same split and the same scales, so at equal sizes the values are those of conv_split_kernel.

// tile_gemm over C::NTAP taps: tap t = 3 x KX position (t / KX, t % KX) reads tile row offset (t / KX - 1) P + t % KX - PADX
template <class C>
__device__ __forceinline__ void tile_gemm_rt(float (&acc_m)[1][C::COUT / 2], float (&acc_s)[1][C::COUT / 2], uint32_t a_hi,
                                             uint32_t a_lo, uint32_t b_base, const int (&row)[1], int lchunk, int P) {
  using U = TapUnits<C>;
  constexpr int UK = U::UK, PT = U::PER_TAP;
#pragma unroll
  for (int i = 0; i < C::COUT / 2; ++i) { acc_m[0][i] = 0.f; acc_s[0][i] = 0.f; }
  uint32_t ah[2][1][UK][4], al[2][1][UK][4];
  load_unit<C, 1>(a_hi, a_lo, row, -P - C::PADX, 0, lchunk, ah[0], al[0]);
#pragma unroll
  for (int u = 0; u < U::N; ++u) {
    wgmma_fence();
    mma_unit<C, 1>(acc_m, acc_s, ah[u & 1], al[u & 1], b_base + (u / PT) * C::B_STAGE, (u % PT) * UK);
    wgmma_commit();
    if (u + 1 < U::N) {
      wgmma_wait<1>();
      const int v = u + 1, t = v / PT;
      load_unit<C, 1>(a_hi, a_lo, row, (t / C::KX - 1) * P + (t % C::KX - C::PADX), (v % PT) * UK, lchunk, ah[v & 1], al[v & 1]);
    }
  }
  wgmma_wait<0>();
}

template <class C>
__device__ __forceinline__ void stage_rows_rt(const SpGeom& g, const float (&acc_m)[C::COUT / 2], const float (&acc_s)[C::COUT / 2],
                                              int m0, int acol, int seg0, int n_seg, const float2 (&bb)[C::COUT / 8],
                                              float out_scale, float* stg) {
  constexpr int SS = C::STG_STRIDE;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int m = m0 + 8 * half;
    if (m < g.KEPT && seg0 + m / g.SEG_ROWS < n_seg) {
      const int r = g.gemm_row(m);
#pragma unroll
      for (int j = 0; j < C::COUT / 8; ++j) {
        const int col = 8 * j + acol;
        const float v0 = fmaxf(fmaf(acc_m[4 * j + 2 * half] + acc_s[4 * j + 2 * half], out_scale, bb[j].x), 0.f);
        const float v1 = fmaxf(fmaf(acc_m[4 * j + 2 * half + 1] + acc_s[4 * j + 2 * half + 1], out_scale, bb[j].y), 0.f);
        *reinterpret_cast<float2*>(stg + r * SS + col) = make_float2(v0, v1);
      }
    }
  }
}

// store_tile on a run-time geometry.  The pooling layers run F.adaptive_max_pool2d in both dimensions: cell (ph, pw) is the
// maximum over rows [floor(ph H / HO), ceil((ph + 1) H / HO)) x columns [floor(pw W / WO), ceil((pw + 1) W / WO)) - windows
// that may overlap, or repeat a row / column when the output is larger than the input.
template <class C>
__device__ __forceinline__ void store_tile_rt(const SpGeom& g, const float* stg, int seg0, int nvalid, int t0, int nthr,
                                              float store_scale, unsigned char* __restrict__ out_hi,
                                              unsigned char* __restrict__ out_lo, float* __restrict__ out_f32) {
  constexpr int COUT = C::COUT, SS = C::STG_STRIDE;
  const int H = g.H, W = g.W, P = g.P, BLK = g.BLK;
  if constexpr (C::POOLED) {
    constexpr int C8 = COUT / 8;
    const int HO = g.HO, WO = g.WO;
    for (int i = t0; i < nvalid * HO * WO * C8; i += nthr) {
      const int c8 = i % C8;
      int rest = i / C8;
      const int pw = rest % WO; rest /= WO;
      const int ph = rest % HO;
      const int s = rest / HO;
      const int y0 = (ph * H) / HO, y1 = ((ph + 1) * H + HO - 1) / HO;
      const int x0 = (pw * W) / WO, x1 = ((pw + 1) * W + WO - 1) / WO;
      float4 ma = make_float4(0.f, 0.f, 0.f, 0.f), mb = ma;       // post-ReLU values are >= 0
      for (int hy = y0; hy < y1; ++hy)
        for (int x = x0; x < x1; ++x) {
          const float4* tp = reinterpret_cast<const float4*>(stg + (s * BLK + (hy + 1) * P + (x + 1)) * SS + c8 * 8);
          const float4 ta = tp[0], tb = tp[1];
          ma.x = fmaxf(ma.x, ta.x); ma.y = fmaxf(ma.y, ta.y); ma.z = fmaxf(ma.z, ta.z); ma.w = fmaxf(ma.w, ta.w);
          mb.x = fmaxf(mb.x, tb.x); mb.y = fmaxf(mb.y, tb.y); mb.z = fmaxf(mb.z, tb.z); mb.w = fmaxf(mb.w, tb.w);
        }
      uint4 hi, lo;
      split8(ma, mb, store_scale, hi, lo);
      const int gr = kSplitLead + (seg0 + s) * g.OBLK + (ph + 1) * g.OP + (pw + 1);
      const size_t o = split_off<COUT * 2>(gr, c8);
      *reinterpret_cast<uint4*>(out_hi + o) = hi;
      *reinterpret_cast<uint4*>(out_lo + o) = lo;
    }
  } else if constexpr (C::OUT_SPLIT) {
    constexpr int C8 = COUT / 8;
    for (int i = t0; i < nvalid * BLK * C8; i += nthr) {
      const int c8 = i % C8, r = i / C8;
      const int q = r % BLK, hh = q / P, ww = q - hh * P;
      uint4 hi = make_uint4(0u, 0u, 0u, 0u), lo = hi;
      if (hh >= 1 && ww >= 1) {
        const float4* tp = reinterpret_cast<const float4*>(stg + r * SS + c8 * 8);
        split8(tp[0], tp[1], store_scale, hi, lo);
      }
      const size_t o = split_off<COUT * 2>(kSplitLead + seg0 * BLK + r, c8);
      *reinterpret_cast<uint4*>(out_hi + o) = hi;
      *reinterpret_cast<uint4*>(out_lo + o) = lo;
    }
  } else {
    // conv6: fp32 CNN features [seg][H][COUT] in rows of OUT_LD floats, zero padding columns
    constexpr int C4 = COUT / 4;
    for (int i = t0; i < nvalid * H * C4; i += nthr) {
      const int c4 = i % C4, rest = i / C4, h = rest % H, s = rest / H;
      *reinterpret_cast<float4*>(out_f32 + (size_t)(seg0 + s) * g.OUT_LD + h * COUT + c4 * 4) =
          *reinterpret_cast<const float4*>(stg + (s * BLK + (h + 1) * P + 1) * SS + c4 * 4);
    }
    const int pad4 = (g.OUT_LD - g.OUT_COLS) / 4;
    for (int i = t0; i < nvalid * pad4; i += nthr)
      *reinterpret_cast<float4*>(out_f32 + (size_t)(seg0 + i / pad4) * g.OUT_LD + g.OUT_COLS + (i % pad4) * 4) =
          make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// conv_split_kernel with SpGeom's sizes: the same persistent CTA, tile copies, barriers and roles
template <class C>
__global__ void __launch_bounds__(C::NT, 1)
conv_split_rt_kernel(const unsigned char* __restrict__ in_hi, const unsigned char* __restrict__ in_lo,
                     const __half* __restrict__ wtc, const float* __restrict__ bias, float out_scale, float store_scale,
                     unsigned char* __restrict__ out_hi, unsigned char* __restrict__ out_lo, float* __restrict__ out_f32,
                     int n_seg, const SpGeom g) {
  constexpr int ROWB = C::ROWB, NT = C::NT, NTAP = C::NTAP;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t b_base = sbase + C::OFF_B;
  const uint32_t bar_w = sbase + C::OFF_BAR, bar_full = bar_w + 8 * NTAP, bar_empty = bar_full + 8 * C::A_BUFS;
  float* stg = reinterpret_cast<float*>(smem + C::OFF_STG);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int G = g.G, BLK = g.BLK, HALO = g.HALO;
  const int n_tiles = (n_seg + G - 1) / G;

  auto issue_tile = [&](int tile, int b) {
    const uint32_t a_copy = (uint32_t)(256 + 2 * HALO) * ROWB;
    const int g0 = kSplitLead + tile * G * BLK - HALO;
    const uint32_t dst = sbase + C::OFF_A_HI + b * C::A_BUF + (uint32_t)(g0 & 7) * ROWB;
    mbar_expect_tx(bar_full + 8 * b, 2 * a_copy);
    bulk_g2s(dst, in_hi + (size_t)g0 * ROWB, a_copy, bar_full + 8 * b);
    bulk_g2s(dst + C::A_BYTES, in_lo + (size_t)g0 * ROWB, a_copy, bar_full + 8 * b);
  };

  if (tid == 0) {
    for (int t = 0; t < NTAP; ++t) mbar_init(bar_w + 8 * t, 1);
    for (int b = 0; b < C::A_BUFS; ++b) mbar_init(bar_full + 8 * b, 1);
    if constexpr (C::A_BUFS == 2)
      for (int b = 0; b < 2; ++b) mbar_init(bar_empty + 8 * b, NT);
    fence_barrier_init();
    for (int t = 0; t < NTAP; ++t) {
      mbar_expect_tx(bar_w + 8 * t, C::B_STAGE);
      bulk_g2s(b_base + t * C::B_STAGE, wtc + (size_t)t * (C::B_STAGE / 2), C::B_STAGE, bar_w + 8 * t);
    }
    if constexpr (!C::ALIAS) issue_tile(blockIdx.x, 0);
  }
  __syncthreads();

  const int lrow = HALO + g.gemm_row(wg * 64 + (warp & 3) * 16 + (lane & 7) + ((lane >> 3) & 1) * 8);
  const int lchunk = lane >> 4;
  const int arow0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int acol = 2 * (lane & 3);

  int it = 0;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
    const int seg0 = tile * G;
    const int g0 = kSplitLead + seg0 * BLK - HALO;
    const int ab = C::A_BUFS == 1 ? 0 : (it & 1);
    if constexpr (C::ALIAS) {
      if (tid == 0) issue_tile(tile, 0);
      mbar_wait(bar_full, it & 1);
    } else if constexpr (C::A_BUFS == 1) {
      mbar_wait(bar_full, it & 1);
    } else {
      const int next = tile + gridDim.x;
      if (tid == 0 && next < n_tiles) {
        const int nb = (it + 1) & 1;
        mbar_wait(bar_empty + 8 * nb, (((it + 1) >> 1) & 1) ^ 1);
        issue_tile(next, nb);
      }
      mbar_wait(bar_full + 8 * ab, (it >> 1) & 1);
    }

    const uint32_t a_hi = sbase + C::OFF_A_HI + ab * C::A_BUF, a_lo = a_hi + C::A_BYTES;
    float acc_m[1][C::COUT / 2], acc_s[1][C::COUT / 2];
#pragma unroll
    for (int i = 0; i < C::COUT / 2; ++i) { acc_m[0][i] = 0.f; acc_s[0][i] = 0.f; }
    if (__shfl_sync(0xffffffffu, wg < g.NBLK, 0)) {
      const int row[1] = {(g0 & 7) + lrow};
      for (int t = 0; t < NTAP; ++t) mbar_wait(bar_w + 8 * t, 0);
      tile_gemm_rt<C>(acc_m, acc_s, a_hi, a_lo, b_base, row, lchunk, g.P);
    }
    if constexpr (C::A_BUFS == 2) mbar_arrive(bar_empty + 8 * ab);
    __syncthreads();
    if constexpr (!C::ALIAS && C::A_BUFS == 1) {
      if (tid == 0 && tile + (int)gridDim.x < n_tiles) issue_tile(tile + gridDim.x, 0);
    }

    float2 bb[C::COUT / 8];
    load_bias<C>(bias, acol, bb);
    stage_rows_rt<C>(g, acc_m[0], acc_s[0], arow0, acol, seg0, n_seg, bb, out_scale, stg);
    __syncthreads();

    store_tile_rt<C>(g, stg, seg0, min(G, n_seg - seg0), tid, NT, store_scale, out_hi, out_lo, out_f32);
    if constexpr (C::ALIAS) {
      fence_proxy_async();
      __syncthreads();
    }
  }
}

// ---- conv1 + pool1 + conv2 + pool2 ----
// conv1 + BN + ReLU + pool1 (conv1_cell.cuh, the same fp32 arithmetic as conv1_pool1_kernel) of one segment per tile
// goes straight into the A tile; the conv2 GEMM and epilogue are the same code on the same values as conv_split_kernel,
// so results are bit-identical to the separate kernels.  The persistent CTA splits into two roles:
//   warpgroups 0, 1 (MMA):   wait A full[i & 1]; GEMM of m64 blocks 0, 1 (warpgroup 0) or block 2 (warpgroup 1);
//                            arrive A empty[i & 1]; bias + ReLU into staging tile i & 1; named barrier of the 256 MMA
//                            threads; max-pool / split / store of tile i
//   warpgroups 2, 3 (conv1): one thread copies the mel block of tile i + 3 into the mel ring; wait mel full[(i + 1) % 4]
//                            and A empty[(i + 1) & 1]; conv1 of tile i + 1 from the ring into A buffer (i + 1) & 1;
//                            arrive mel empty and A full
// so conv1 of the next tile runs while the tensor cores work on this one, and its mel reads never wait for global
// memory.  The A and mel empty barriers count the 256 threads of the role that arrives on them (mel full: the copying
// thread, plus the copy's bytes); a barrier's k-th use waits on parity k & 1 (full) or (k & 1) ^ 1 (empty: a fresh
// barrier's "previous phase" counts as complete).  Staging tile i & 1 is next written at tile i + 2, after the named
// barrier of tile i + 1, which every MMA thread reaches only after its part of tile i's store.
template <class C, int MODE>
__global__ void __launch_bounds__(C::NT, 1)
conv12_kernel(const __half* __restrict__ wtc, const float* __restrict__ bias, float out_scale, float store_scale,
              unsigned char* __restrict__ out_hi, unsigned char* __restrict__ out_lo, int n_seg,
              const float* __restrict__ mel, const int* __restrict__ seg_frame0, const float* __restrict__ seg_thr,
              const float* __restrict__ w1 /*[9][16]*/, const float* __restrict__ b1 /*[16]*/,
              float c1_scale /*2^-e1: conv1's activation scale*/) {
  using L = SpFused<C>;
  constexpr int W = C::W, P = C::P, HALO = C::HALO, ROWB = C::ROWB, NT = C::NT, NR = NT / 2;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t b_base = sbase + L::OFF_B;
  const uint32_t bar_w = sbase + L::OFF_BAR, a_full = bar_w + 8 * 9, a_empty = a_full + 16;
  const uint32_t mel_full = a_empty + 16, mel_empty = mel_full + 8 * L::MEL_R;
  float* ws = reinterpret_cast<float*>(smem + L::OFF_W1);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);   // warp-uniform as far as ptxas can tell: the role branch
                                                           // below must not count as divergent around the wgmmas
  const int n_tiles = n_seg;                     // G == 1

  // the zero row / zero column / halo rows of both A buffers are never written again
  for (int i = tid; i < 2 * C::A_BUF / 16; i += NT) reinterpret_cast<uint4*>(smem + L::OFF_A)[i] = make_uint4(0u, 0u, 0u, 0u);
  for (int i = tid; i < 9 * 16 + 16; i += NT) ws[i] = (i < 144) ? __ldg(w1 + i) : __ldg(b1 + i - 144);
  if (tid == 0) {
    for (int t = 0; t < 9; ++t) mbar_init(bar_w + 8 * t, 1);
    for (int b = 0; b < 4; ++b) mbar_init(a_full + 8 * b, NR);
    for (int s = 0; s < L::MEL_R; ++s) {
      mbar_init(mel_full + 8 * s, 1);
      mbar_init(mel_empty + 8 * s, NR);
    }
    fence_barrier_init();
    for (int t = 0; t < 9; ++t) {
      mbar_expect_tx(bar_w + 8 * t, C::B_STAGE);
      bulk_g2s(b_base + t * C::B_STAGE, wtc + (size_t)t * (C::B_STAGE / 2), C::B_STAGE, bar_w + 8 * t);
    }
  }
  __syncthreads();

  // registers: 64 accumulators and two fragment sets per MMA thread; 2 x 128 x (160 + 96) = the whole register file
  if (wg < 2) {
    // ===== MMA warpgroups: warpgroup 0 runs m64 blocks 0 and 1 (GEMM rows 0 .. 127), warpgroup 1 block 2 (rows
    // 128 .. 191); block 3 would hold only rows m >= KEPT, which are never staged =====
    setmaxnreg_inc<160>();
    const int lm = (warp & 3) * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;   // ldmatrix row within an m64 block
    const int am = (warp & 3) * 16 + (lane >> 2);                          // accumulator row within an m64 block
    const int lchunk = lane >> 4;
    const int acol = 2 * (lane & 3);
    // the whole tile loop of a warpgroup that owns NB blocks from block b0 on: the branch between the two instances is
    // taken once, outside the loop, on the warp-uniform wg
    float2 bb[C::COUT / 8];
    load_bias<C>(bias, acol, bb);
    wait_weights(bar_w);
    auto mma_role = [&](auto nb, int b0) {
      constexpr int NB = decltype(nb)::value;
      int lrow[NB];
#pragma unroll
      for (int b = 0; b < NB; ++b) lrow[b] = HALO + C::gemm_row(lm + 64 * (b0 + b));
      int it = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
        const int ab = it & 1;
        const uint32_t par = (uint32_t)(it >> 1) & 1u;
        mbar_wait(a_full + 8 * ab, par);
        const uint32_t a_hi = sbase + L::OFF_A + ab * C::A_BUF, a_lo = a_hi + C::A_BYTES;
        float acc_m[NB][C::COUT / 2], acc_s[NB][C::COUT / 2];
        tile_gemm<C, NB>(acc_m, acc_s, a_hi, a_lo, b_base, lrow, lchunk);
        mbar_arrive(a_empty + 8 * ab);
        float* stg = reinterpret_cast<float*>(smem + L::OFF_STG + ab * C::STG_BYTES);
#pragma unroll
        for (int b = 0; b < NB; ++b)
          stage_rows<C>(acc_m[b], acc_s[b], am + 64 * (b0 + b), acol, tile, n_seg, bb, out_scale, stg);
        named_bar_sync<1, NR>();
        store_tile<C>(stg, tile, 1, tid, NR, store_scale, out_hi, out_lo, nullptr);
      }
    };
    if (wg == 0) mma_role(std::integral_constant<int, 2>(), 0);
    else mma_role(std::integral_constant<int, 1>(), 2);
  } else {
    // ===== worker warpgroups =====
    setmaxnreg_dec<96>();
    const int wt = tid - NR;
    constexpr int R = L::MEL_R, MEL_FLOATS = L::MEL_BYTES / 4;
    const float* ring = reinterpret_cast<const float*>(smem + L::OFF_MEL);
    float* ring_thr = reinterpret_cast<float*>(smem + L::OFF_THR);
    // Mel ring, thread wt == 0 only: the CTA's k-th segment goes to slot k % R once every worker has arrived on the
    // slot's empty barrier for segment k - R.  The segment's 15 frames are one contiguous block of 2880 bytes at
    // mel + kMels f0: the mel workspace comes from cudaMalloc (256-byte aligned) and kMels * 4 = 192 bytes per frame,
    // so the source is 16-byte aligned for any f0.  seg_frame0 / seg_thr of the next segment to copy are loaded one
    // copy ahead, so the thread that issues never waits for them.
    int nf0 = 0;
    float nthr = 0.f;
    auto prefetch_seg = [&](int k) {
      const int seg = blockIdx.x + k * gridDim.x;
      if (seg < n_tiles) { nf0 = __ldg(seg_frame0 + seg); nthr = __ldg(seg_thr + seg); }
    };
    auto issue_mel = [&](int k) {
      if (blockIdx.x + k * gridDim.x >= n_tiles) return;
      const int s = k % R;
      mbar_wait(mel_empty + 8 * s, ((uint32_t)(k / R) & 1u) ^ 1u);
      ring_thr[s] = nthr;                        // published by the arrive below (release) to the full barrier's waiters
      mbar_expect_tx(mel_full + 8 * s, L::MEL_BYTES);
      bulk_g2s(sbase + L::OFF_MEL + s * L::MEL_BYTES, mel + (size_t)nf0 * kMels, L::MEL_BYTES, mel_full + 8 * s);
      prefetch_seg(k + 1);
    };
    if (wt == 0) {
      prefetch_seg(0);
      for (int k = 0; k < R - 2; ++k) issue_mel(k);
    }
    // conv1 + BN + ReLU + pool1 of the CTA's j-th segment (mel ring slot j % R) into A buffer j & 1.  Thread wt < 192
    // owns one strip for the kernel's life: pooled row ph, channel quad cq, and the left (pw < W / 2) or right half of
    // the pooled cells (warp-uniform: 96 strips = 3 warps per half); conv1_strip computes each conv1 output position
    // of the strip once.  The quad's weights and biases stay in registers.  A warp's lanes run over cq, then ph: its 8
    // distinct mel addresses are rows 2 apart, on distinct banks.  Each cell -> one 8-byte half of a 16-byte chunk.
    constexpr int NSTRIP = 2 * 4 * 24;
    const int cq = wt & 3, ph = (wt >> 2) % 24;
    const bool right = __shfl_sync(0xffffffffu, wt >= NSTRIP / 2, 0);
    float wq[9][4], bq[4];
#pragma unroll
    for (int t = 0; t < 9; ++t)
#pragma unroll
      for (int c = 0; c < 4; ++c) wq[t][c] = ws[t * 16 + cq * 4 + c];
#pragma unroll
    for (int c = 0; c < 4; ++c) bq[c] = ws[144 + cq * 4 + c];
    auto fill = [&](int j) {
      const int b = j & 1, s = j % R;
      if (wt == 0) issue_mel(j + R - 2);         // its slot held segment j - 2
      mbar_wait(a_empty + 8 * b, ((uint32_t)(j >> 1) & 1u) ^ 1u);
      mbar_wait(mel_full + 8 * s, (uint32_t)(j / R) & 1u);
      unsigned char* a = smem + L::OFF_A + b * C::A_BUF;
      const float* slot = ring + s * MEL_FLOATS;
      const float thr = ring_thr[s];
      auto emit = [&](int pw, const float (&res)[4]) {
        uint2 hi, lo;
        split4(make_float4(res[0], res[1], res[2], res[3]), c1_scale, hi, lo);
        const uint32_t o = (uint32_t)split_off<ROWB>(HALO + (ph + 1) * P + (pw + 1), cq >> 1) + 8 * (cq & 1);
        *reinterpret_cast<uint2*>(a + o) = hi;
        *reinterpret_cast<uint2*>(a + C::A_BYTES + o) = lo;
      };
      if (wt < NSTRIP) {
        if (right) conv1_strip<MODE, W / 2, W, kMels>(slot, thr, wq, bq, ph, emit);
        else conv1_strip<MODE, 0, W / 2, kMels>(slot, thr, wq, bq, ph, emit);
      }
      mbar_arrive(mel_empty + 8 * s);
      mbar_arrive(a_full + 8 * b);
    };
    int it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) fill(it);
  }
}

// planes -> fp32 channels-last [seg][H][W][C] (stage dumps for the parity tests; x_hi + x_lo == x 2^-e to 2^-22,
// unit = 2^e undoes the activation scale exactly)
template <int ROWB>
__global__ void unsplit_kernel(const unsigned char* __restrict__ hi, const unsigned char* __restrict__ lo,
                               float* __restrict__ out, long long n_items, int H, int W, float unit) {
  constexpr int C8 = ROWB / 16;
  const int P = W + 1, BLK = (H + 1) * P;
  for (long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x; it < n_items; it += (long long)gridDim.x * blockDim.x) {
    const int c8 = (int)(it % C8);
    long long rest = it / C8;
    const int w = (int)(rest % W); rest /= W;
    const int h = (int)(rest % H);
    const int seg = (int)(rest / H);
    const int g = kSplitLead + seg * BLK + (h + 1) * P + (w + 1);
    const size_t o = split_off<ROWB>(g, c8);
    const uint4 a = *reinterpret_cast<const uint4*>(hi + o), b = *reinterpret_cast<const uint4*>(lo + o);
    const __half2* ah = reinterpret_cast<const __half2*>(&a);
    const __half2* bh = reinterpret_cast<const __half2*>(&b);
    float r[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 x = __half22float2(ah[i]), y = __half22float2(bh[i]);
      r[2 * i] = (x.x + y.x) * unit; r[2 * i + 1] = (x.y + y.y) * unit;
    }
    float4* dst = reinterpret_cast<float4*>(out + it * 8);
    dst[0] = make_float4(r[0], r[1], r[2], r[3]);
    dst[1] = make_float4(r[4], r[5], r[6], r[7]);
  }
}

static int device_sms() {
  int dev = 0, n = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 1;
}

template <class C>
static void launch_sp(cudaStream_t st, const unsigned char* in_hi, const unsigned char* in_lo, const __half* wtc,
                      const float* b, float scale, float store_scale, unsigned char* out_hi, unsigned char* out_lo,
                      float* out_f32, int n_seg) {
  static unsigned long long configured = 0;
  static int n_sm = 0;
  if (first_launch_on_device(configured)) {
    cudaFuncSetAttribute(conv_split_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    n_sm = device_sms();
  }
  const int n_tiles = (n_seg + C::G - 1) / C::G;
  const int grid = std::min(n_tiles, n_sm);              // one persistent CTA per SM
  conv_split_kernel<C><<<grid, C::NT, C::SMEM_BYTES, st>>>(in_hi, in_lo, wtc, b, scale, store_scale, out_hi, out_lo,
                                                           out_f32, n_seg);
}

template <class C, int MODE>
static void launch_c12(cudaStream_t st, const __half* wtc, const float* b, float scale, float store_scale,
                       unsigned char* out_hi, unsigned char* out_lo, int n_seg, const float* mel, const int* seg_frame0,
                       const float* seg_thr, const float* w1, const float* b1, float c1_scale) {
  static unsigned long long configured = 0;
  static int n_sm = 0;
  if (first_launch_on_device(configured)) {
    cudaFuncSetAttribute(conv12_kernel<C, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SpFused<C>::SMEM_BYTES);
    n_sm = device_sms();
  }
  const int grid = std::min(n_seg, n_sm);                // one persistent CTA per SM, one segment per tile
  conv12_kernel<C, MODE><<<grid, C::NT, SpFused<C>::SMEM_BYTES, st>>>(wtc, b, scale, store_scale, out_hi, out_lo, n_seg,
                                                                      mel, seg_frame0, seg_thr, w1, b1, c1_scale);
}

template <class C>
static void launch_sp_rt(cudaStream_t st, const unsigned char* in_hi, const unsigned char* in_lo, const __half* wtc,
                         const float* b, float scale, float store_scale, unsigned char* out_hi, unsigned char* out_lo,
                         float* out_f32, int n_seg, const SpGeom& g) {
  static unsigned long long configured = 0;
  static int n_sm = 0;
  if (first_launch_on_device(configured)) {
    cudaFuncSetAttribute(conv_split_rt_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    n_sm = device_sms();
  }
  const int n_tiles = (n_seg + g.G - 1) / g.G;
  const int grid = std::min(n_tiles, n_sm);
  conv_split_rt_kernel<C><<<grid, C::NT, C::SMEM_BYTES, st>>>(in_hi, in_lo, wtc, b, scale, store_scale, out_hi, out_lo,
                                                              out_f32, n_seg, g);
}

#define NISQA_SP_GEOM(L, CI, CO) static_assert(input_is<SpAdapt<L, CI, CO>>(0, L), "SpCfg geometry differs from split_geometry");
NISQA_SP_ADAPT_LAYERS(NISQA_SP_GEOM)
#undef NISQA_SP_GEOM
static_assert(input_is<SpConv2S>(1, 2) && input_is<SpConv3S>(1, 3) && input_is<SpConv4S>(1, 4) && input_is<SpConv5S>(1, 5) &&
              input_is<SpConv6S>(1, 6), "SpCfg geometry differs from split_geometry");
static_assert(kMaxPoolW + 2 <= kSplitLead && kMaxPoolCells <= 256,
              "the run-time geometry kernels: a halo of at most kSplitLead rows, one segment per 256-row tile at least");

// Bytes of one plane of the pair that feeds conv layer `layer` (2..6) with C channels for n_seg segments: per segment
// (H + 1) rows of W + 1 pixels (shared zero row / column), the zero lead rows and the tile over-read.
size_t split_plane_bytes(int std_mode, int layer, int C, int n_seg, const CnnPools& pools) {
  const ConvGeom g = split_geometry(std_mode, layer, C, pools);
  const size_t rows = (size_t)kSplitLead + (size_t)n_seg * (g.H + 1) * (g.W + 1) + 256 + 32;
  return (rows * (size_t)g.C * 2 + 1023) & ~(size_t)1023;
}

bool conv_split_supported(int cin, int cout) {
  return (cin == 16 || cin == 32 || cin == 64) && (cout == 16 || cout == 32 || cout == 64);
}

// conv layer 2..6 (cin -> cout channels) on planes; the last layer (6) writes the fp32 CNN features (adapt:
// [seg][pool_3 h][c3] in rows padded to a multiple of 64 floats; standard: [seg][6][2][64]).  AdaptCNN layers whose input
// map and output pooling are the shipped ones run the compile-time instances, every other one the run-time geometry
// kernel.  false: no instance for the shape.
bool launch_conv_split(cudaStream_t st, int std_mode, int layer, int cin, int cout, const void* in_hi, const void* in_lo,
                       const void* wtc, const float* b, float out_scale, float store_scale, void* out_hi,
                       void* out_lo, float* out_f32, int n_seg, const CnnPools& pools) {
  const __half* w = reinterpret_cast<const __half*>(wtc);
  const unsigned char* ih = static_cast<const unsigned char*>(in_hi);
  const unsigned char* il = static_cast<const unsigned char*>(in_lo);
  unsigned char* oh = static_cast<unsigned char*>(out_hi);
  unsigned char* ol = static_cast<unsigned char*>(out_lo);
  if (!std_mode && !shipped_layer_geometry(layer, pools)) {
    const ConvGeom in = split_geometry(0, layer, cin, pools);
    const ConvGeom out = layer < 6 ? split_geometry(0, layer + 1, cout, pools) : ConvGeom{in.H, 1, cout};
    const SpGeom g = sp_geom(layer, in.H, in.W, out.H, out.W, cout);
    const int ntap = layer == 6 ? 3 * in.W : 9;
#define NISQA_SP_RT_LAUNCH(L, CI, CO, NT)                                                                    \
    if (layer == L && cin == CI && cout == CO && ntap == NT) {                                                \
      launch_sp_rt<SpRt<L, CI, CO, NT>>(st, ih, il, w, b, out_scale, store_scale, oh, ol, out_f32, n_seg, g);  \
      return true;                                                                                            \
    }
    NISQA_SP_RT_LAYERS(NISQA_SP_RT_LAUNCH)
#undef NISQA_SP_RT_LAUNCH
    return false;
  }
  if (!std_mode) {
#define NISQA_SP_LAUNCH(L, CI, CO)                                                                           \
    if (layer == L && cin == CI && cout == CO) {                                                              \
      launch_sp<SpAdapt<L, CI, CO>>(st, ih, il, w, b, out_scale, store_scale, oh, ol, out_f32, n_seg);        \
      return true;                                                                                            \
    }
    NISQA_SP_ADAPT_LAYERS(NISQA_SP_LAUNCH)
#undef NISQA_SP_LAUNCH
    return false;
  }
  if (cin != split_geometry(1, layer, 0).C || cout != (layer == 2 ? 32 : 64)) return false;
  switch (layer) {
    case 2: launch_sp<SpConv2S>(st, ih, il, w, b, out_scale, store_scale, oh, ol, out_f32, n_seg); break;
    case 3: launch_sp<SpConv3S>(st, ih, il, w, b, out_scale, store_scale, oh, ol, out_f32, n_seg); break;
    case 4: launch_sp<SpConv4S>(st, ih, il, w, b, out_scale, store_scale, oh, ol, out_f32, n_seg); break;
    case 5: launch_sp<SpConv5S>(st, ih, il, w, b, out_scale, store_scale, oh, ol, out_f32, n_seg); break;
    default: launch_sp<SpConv6S>(st, ih, il, w, b, out_scale, store_scale, oh, ol, out_f32, n_seg); break;
  }
  return true;
}

bool conv12_supported(int std_mode, int c1, int c2) { return c1 == 16 && (c2 == 32 || (!std_mode && c2 == 16)); }

// conv1 + pool1 + conv2 + pool2 in one kernel: mel segments -> the plane pair feeding conv3 (conv12_supported shapes)
void launch_conv12(cudaStream_t st, int std_mode, int c2, const float* mel, const int* seg_frame0, const float* seg_thr,
                   const float* w1, const float* b1, float c1_scale, const void* wtc2, const float* bias2,
                   float scale2, float store_scale, void* out_hi, void* out_lo, int n_seg) {
  const __half* w = reinterpret_cast<const __half*>(wtc2);
  unsigned char* oh = static_cast<unsigned char*>(out_hi);
  unsigned char* ol = static_cast<unsigned char*>(out_lo);
  if (std_mode)
    launch_c12<SpConv2S, 1>(st, w, bias2, scale2, store_scale, oh, ol, n_seg, mel, seg_frame0, seg_thr, w1, b1, c1_scale);
  else if (c2 == 16)
    launch_c12<SpAdapt<2, 16, 16>, 0>(st, w, bias2, scale2, store_scale, oh, ol, n_seg, mel, seg_frame0, seg_thr, w1, b1, c1_scale);
  else
    launch_c12<SpConv2A, 0>(st, w, bias2, scale2, store_scale, oh, ol, n_seg, mel, seg_frame0, seg_thr, w1, b1, c1_scale);
}

void launch_unsplit(cudaStream_t st, int std_mode, int layer, int C, const void* hi, const void* lo, float unit, float* out,
                    int n_seg, const CnnPools& pools) {
  const ConvGeom g = split_geometry(std_mode, layer, C, pools);
  const long long items = (long long)n_seg * g.H * g.W * (g.C / 8);
  const unsigned char* h = static_cast<const unsigned char*>(hi);
  const unsigned char* l = static_cast<const unsigned char*>(lo);
  const int grid = (int)std::min<long long>((items + 255) / 256, (long long)device_sms() * 16);
  if (g.C == 16) unsplit_kernel<32><<<grid, 256, 0, st>>>(h, l, out, items, g.H, g.W, unit);
  else if (g.C == 32) unsplit_kernel<64><<<grid, 256, 0, st>>>(h, l, out, items, g.H, g.W, unit);
  else unsplit_kernel<128><<<grid, 256, 0, st>>>(h, l, out, items, g.H, g.W, unit);
}

}  // namespace nisqa

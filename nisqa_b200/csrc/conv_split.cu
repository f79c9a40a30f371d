// conv_split.cu - conv2..conv6 of the AdaptCNN / StandardCNN (reference nisqa/NISQA_lib.py:692-706,
// 816-830) as implicit GEMMs on the Hopper tensor cores (wgmma), with an error-compensated two-term FP16 split so
// that the result stays within fp32 rounding noise of the reference (plain TF32 / BF16 operands move MOS by
// 2e-3 / 1.7e-2, SURVEY.md 0.8):
//      a = a_hi + a_lo,  b = b_hi + b_lo      (fp16 parts: 11 + 11 significant bits)
//      a*b ~= a_hi*b_hi + a_hi*b_lo + a_lo*b_hi          (dropped a_lo*b_lo ~ 2^-22 |a b|)
// The main accumulator only ever sees the hi*hi products; hi*lo and lo*hi go to a second, small accumulator, and the
// epilogue adds the two.  The weights are pre-scaled by 2^S on the host (S chosen per layer so that max|w| 2^S <= 1024)
// to keep b_lo out of the fp16 subnormal range; the epilogue multiplies by 2^-S (exact).
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
//   M = 256 tile rows (G segments), N = C_out, K = 9 * C_in.  Four warpgroups own 64 rows each: A fragments come
//   from the swizzled tile with ldmatrix (conflict free: 8 consecutive rows hit 8 distinct 16-byte bank groups), B
//   (all nine weight taps, resident for the CTA's life) through shared-memory descriptors, accumulators in
//   registers.  CTAs are persistent: the weights are loaded once per CTA, the tiles are walked with a grid stride.
//   Epilogue: registers -> bias / ReLU -> fp32 staging tile -> (max-pool) -> split -> planes of the next layer.
//
// The fused variant (FUSE = 1 + MODE) also computes conv1 + BN + ReLU + pool1 (conv1_cell.cuh, the same fp32
// arithmetic as conv1_pool1_kernel) of the tile's segment straight into the A tile, so pool1 never reaches HBM; its
// conv2 GEMM is the same code on the same values: results are bit-identical to the separate kernels.
#include <cuda_fp16.h>

#include <algorithm>

#include "common.cuh"
#include "conv1_cell.cuh"
#include "conv_split.cuh"
#include "tc_ptx.cuh"

namespace nisqa {

template <class C, int FUSE>
__global__ void __launch_bounds__(C::NT, 1)
conv_split_kernel(const unsigned char* __restrict__ in_hi, const unsigned char* __restrict__ in_lo,
                  const __half* __restrict__ wtc /*[9][CIN/8][hi co | lo co][8] fp16, scaled by 2^S*/,
                  const float* __restrict__ bias, float out_scale /*2^-S*/,
                  unsigned char* __restrict__ out_hi, unsigned char* __restrict__ out_lo,
                  float* __restrict__ out_f32 /*last layer only*/, int n_seg,
                  const float* __restrict__ mel, const int* __restrict__ seg_frame0, const float* __restrict__ seg_thr,
                  const float* __restrict__ w1 /*[9][16]*/, const float* __restrict__ b1 /*[16]*/) {
  constexpr int H = C::H, W = C::W, CIN = C::CIN, COUT = C::COUT, P = C::P, BLK = C::BLK, G = C::G;
  constexpr int HALO = C::HALO, ROWB = C::ROWB, NT = C::NT, SS = C::STG_STRIDE;
  static_assert(FUSE == 0 || (G == 1 && CIN == 16 && !C::ALIAS), "fused conv1: one segment per tile, conv2 geometry");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // swizzle atoms repeat every 1024 B
  const uint32_t sbase = smem_u32(smem);
  const uint32_t a_hi = sbase + C::OFF_A_HI, a_lo = sbase + C::OFF_A_LO, b_base = sbase + C::OFF_B;
  const uint32_t bar_w = sbase + C::OFF_BAR, bar_a = bar_w + 8 * 9;
  float* stg = reinterpret_cast<float*>(smem + C::OFF_STG);
  float* ws = reinterpret_cast<float*>(smem + C::OFF_W1);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int n_tiles = (n_seg + G - 1) / G;

  if constexpr (FUSE != 0) {
    // the zero row / zero column / halo rows of the A tile are never written again
    for (int i = tid; i < 2 * C::A_BYTES / 16; i += NT) reinterpret_cast<uint4*>(smem + C::OFF_A_HI)[i] = make_uint4(0u, 0u, 0u, 0u);
    for (int i = tid; i < 9 * 16 + 16; i += NT) ws[i] = (i < 144) ? __ldg(w1 + i) : __ldg(b1 + i - 144);
  }
  if (tid == 0) {
    for (int t = 0; t < 9; ++t) mbar_init(bar_w + 8 * t, 1);
    mbar_init(bar_a, 1);
    fence_barrier_init();
    for (int t = 0; t < 9; ++t) {                // all nine taps stay resident; tap t's MMAs start once it has landed
      mbar_expect_tx(bar_w + 8 * t, C::B_STAGE);
      bulk_g2s(b_base + t * C::B_STAGE, wtc + (size_t)t * (C::B_STAGE / 2), C::B_STAGE, bar_w + 8 * t);
    }
  }
  __syncthreads();

  // this lane's ldmatrix row (within its warp's 16 rows) and K chunk; its accumulator rows
  const int lrow = wg * 64 + (warp & 3) * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
  const int lchunk = lane >> 4;
  const int arow0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int acol = 2 * (lane & 3);

  int it = 0;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
    const int seg0 = tile * G;
    const int g0 = kSplitLead + seg0 * BLK - HALO;         // first plane row of this tile
    const uint32_t sh = FUSE ? 0u : (uint32_t)(g0 & 7);    // tile row == plane row (mod 8)
    if constexpr (FUSE == 0) {
      if (tid == 0) {
        constexpr uint32_t A_COPY = (uint32_t)C::AROWS * ROWB;
        mbar_expect_tx(bar_a, 2 * A_COPY);
        bulk_g2s(a_hi + sh * ROWB, in_hi + (size_t)g0 * ROWB, A_COPY, bar_a);
        bulk_g2s(a_lo + sh * ROWB, in_lo + (size_t)g0 * ROWB, A_COPY, bar_a);
      }
      mbar_wait(bar_a, it & 1);
    } else {
      // conv1 + BN + ReLU + pool1 of segment `tile`: one thread per pooled cell, all 16 channels
      constexpr int PW = W, NCELL = 24 * PW;
      if (tid < NCELL) {
        const int ph = tid / PW, pw = tid - ph * PW;
        float res[16];
        conv1_cell<FUSE - 1>(mel, __ldg(seg_frame0 + tile), __ldg(seg_thr + tile), ws, ph, pw, res);
        const int row = HALO + (ph + 1) * P + (pw + 1);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          uint4 hi, lo;
          split8(make_float4(res[8 * c], res[8 * c + 1], res[8 * c + 2], res[8 * c + 3]),
                 make_float4(res[8 * c + 4], res[8 * c + 5], res[8 * c + 6], res[8 * c + 7]), hi, lo);
          const uint32_t o = (uint32_t)split_off<ROWB>(row, c);
          *reinterpret_cast<uint4*>(smem + C::OFF_A_HI + o) = hi;
          *reinterpret_cast<uint4*>(smem + C::OFF_A_LO + o) = lo;
        }
      }
      __syncthreads();
    }

    // ===== GEMM: warpgroup wg, rows 64 wg .. 64 wg + 63 =====
    float acc_m[COUT / 2], acc_s[COUT / 2];      // hi*hi ; hi*lo + lo*hi
#pragma unroll
    for (int i = 0; i < COUT / 2; ++i) { acc_m[i] = 0.f; acc_s[i] = 0.f; }
#pragma unroll 1
    for (int t = 0; t < 9; ++t) {
      mbar_wait(bar_w + 8 * t, 0);
      const int tapoff = (t / 3 - 1) * P + (t % 3 - 1);
      const int row = (int)sh + HALO + tapoff + lrow;
      const uint32_t bst = b_base + t * C::B_STAGE;
      uint32_t ah[CIN / 16][4], al[CIN / 16][4];
#pragma unroll
      for (int ks = 0; ks < CIN / 16; ++ks) {
        const uint32_t ao = (uint32_t)split_off<ROWB>(row, 2 * ks + lchunk);
        ldsm_x4(a_hi + ao, ah[ks]);
        ldsm_x4(a_lo + ao, al[ks]);
      }
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < CIN / 16; ++ks) {
        const uint32_t bk = bst + (uint32_t)(2 * ks) * (2 * COUT * 16);
        const uint64_t dbh = make_desc_b(bk, 2 * COUT * 16), dbl = make_desc_b(bk + COUT * 16, 2 * COUT * 16);
        wgmma_rs<COUT>(acc_m, ah[ks], dbh);
        wgmma_rs<COUT>(acc_s, ah[ks], dbl);
        wgmma_rs<COUT>(acc_s, al[ks], dbh);
      }
      wgmma_commit();
      wgmma_wait0();                             // the A fragments are overwritten by the next tap's loads
    }
    __syncthreads();                             // every warpgroup is done with the A tile (the staging tile may alias it)

    // ===== epilogue part 1: accumulators -> bias + ReLU -> staging row r =====
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int r = arow0 + 8 * half;
      const int s = r / BLK, q = r - s * BLK;
      const int hh = q / P, ww = q - hh * P;
      bool valid = (s < G) && (seg0 + s < n_seg) && hh >= 1 && ww >= 1;
      if (C::CENTER) valid = valid && (ww == 2);
      if (valid) {
#pragma unroll
        for (int j = 0; j < COUT / 8; ++j) {
          const int col = 8 * j + acol;
          const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + col));
          const float v0 = fmaxf(fmaf(acc_m[4 * j + 2 * half] + acc_s[4 * j + 2 * half], out_scale, bb.x), 0.f);
          const float v1 = fmaxf(fmaf(acc_m[4 * j + 2 * half + 1] + acc_s[4 * j + 2 * half + 1], out_scale, bb.y), 0.f);
          *reinterpret_cast<float2*>(stg + r * SS + col) = make_float2(v0, v1);
        }
      }
    }
    __syncthreads();

    // ===== epilogue part 2 (all threads): max-pool / split / store =====
    const int nvalid = min(G, n_seg - seg0);
    if constexpr (C::POOL != SP_POOL_NONE) {
      constexpr int POW = C::POW, HO = H / 2, C8 = COUT / 8;
      for (int i = tid; i < nvalid * HO * POW * C8; i += NT) {
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
        split8(ma, mb, hi, lo);
        const int g = kSplitLead + (seg0 + s) * C::OBLK + (ph + 1) * C::OP + (pw + 1);
        const size_t o = split_off<C::OROWB>(g, c8);
        *reinterpret_cast<uint4*>(out_hi + o) = hi;
        *reinterpret_cast<uint4*>(out_lo + o) = lo;
      }
    } else if constexpr (C::OUT_SPLIT) {
      // the whole image of the tile's segments, zero row / column positions included (as zeros)
      constexpr int C8 = COUT / 8;
      for (int i = tid; i < nvalid * BLK * C8; i += NT) {
        const int c8 = i % C8, r = i / C8;
        const int q = r % BLK, hh = q / P, ww = q - hh * P;
        uint4 hi = make_uint4(0u, 0u, 0u, 0u), lo = hi;
        if (hh >= 1 && ww >= 1) {
          const float4* tp = reinterpret_cast<const float4*>(stg + r * SS + c8 * 8);
          split8(tp[0], tp[1], hi, lo);
        }
        const size_t o = split_off<C::OROWB>(kSplitLead + seg0 * BLK + r, c8);
        *reinterpret_cast<uint4*>(out_hi + o) = hi;
        *reinterpret_cast<uint4*>(out_lo + o) = lo;
      }
    } else {
      // fp32 CNN features, channels-last [seg][HO][WO][COUT]
      constexpr int HO = C::HO, WO = C::WO, C4 = COUT / 4;
      for (int i = tid; i < nvalid * HO * WO * C4; i += NT) {
        const int c4 = i % C4;
        int rest = i / C4;
        const int w = rest % WO; rest /= WO;
        const int h = rest % HO;
        const int s = rest / HO;
        const int r = s * BLK + (h + 1) * P + (C::CENTER ? 2 : w + 1);
        *reinterpret_cast<float4*>(out_f32 + ((size_t)(seg0 + s) * (HO * WO) + h * WO + w) * COUT + c4 * 4) =
            *reinterpret_cast<const float4*>(stg + r * SS + c4 * 4);
      }
    }
    fence_proxy_async();                         // staging stores (generic proxy) before the next tile's bulk copy
    __syncthreads();
  }
}

// planes -> fp32 channels-last [seg][H][W][C] (stage dumps for the parity tests; x_hi + x_lo == x to 2^-22)
template <int ROWB>
__global__ void unsplit_kernel(const unsigned char* __restrict__ hi, const unsigned char* __restrict__ lo,
                               float* __restrict__ out, long long n_items, int H, int W) {
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
      r[2 * i] = x.x + y.x; r[2 * i + 1] = x.y + y.y;
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

template <class C, int FUSE>
static void launch_sp(cudaStream_t st, const unsigned char* in_hi, const unsigned char* in_lo, const __half* wtc,
                      const float* b, float scale, unsigned char* out_hi, unsigned char* out_lo, float* out_f32,
                      int n_seg, const float* mel = nullptr, const int* seg_frame0 = nullptr,
                      const float* seg_thr = nullptr, const float* w1 = nullptr, const float* b1 = nullptr) {
  static unsigned long long configured = 0;
  static int n_sm = 0;
  if (first_launch_on_device(configured)) {
    cudaFuncSetAttribute(conv_split_kernel<C, FUSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    n_sm = device_sms();
  }
  const int n_tiles = (n_seg + C::G - 1) / C::G;
  const int grid = std::min(n_tiles, n_sm);              // one persistent CTA per SM
  conv_split_kernel<C, FUSE><<<grid, C::NT, C::SMEM_BYTES, st>>>(in_hi, in_lo, wtc, b, scale, out_hi, out_lo, out_f32,
                                                                 n_seg, mel, seg_frame0, seg_thr, w1, b1);
}

// Geometry of the plane pair that feeds conv layer `layer` (2..6): rows of the padded image per segment,
// bytes per row, and the bytes of one plane for n_seg segments (tile over-read included).
void split_geometry(int std_mode, int layer, int* H, int* W, int* C) {
  static const int ha[7] = {0, 0, 24, 12, 12, 6, 6}, ca[7] = {0, 0, 16, 32, 64, 64, 64};
  static const int wa[7] = {0, 0, 7, 5, 5, 3, 3}, ws[7] = {0, 0, 8, 4, 4, 2, 2};
  *H = ha[layer]; *C = ca[layer]; *W = std_mode ? ws[layer] : wa[layer];
}
size_t split_plane_bytes(int std_mode, int layer, int n_seg) {
  int H, W, C;
  split_geometry(std_mode, layer, &H, &W, &C);
  const size_t rows = (size_t)kSplitLead + (size_t)n_seg * (H + 1) * (W + 1) + 256 + 32;
  return (rows * (size_t)C * 2 + 1023) & ~(size_t)1023;
}

// conv layer 2..6 on planes; the last layer (6) writes the fp32 CNN features (adapt: [seg][6][64];
// standard: [seg][6][2][64])
void launch_conv_split(cudaStream_t st, int std_mode, int layer, const void* in_hi, const void* in_lo,
                       const void* wtc, const float* b, float out_scale, void* out_hi, void* out_lo,
                       float* out_f32, int n_seg) {
  const __half* w = reinterpret_cast<const __half*>(wtc);
  const unsigned char* ih = static_cast<const unsigned char*>(in_hi);
  const unsigned char* il = static_cast<const unsigned char*>(in_lo);
  unsigned char* oh = static_cast<unsigned char*>(out_hi);
  unsigned char* ol = static_cast<unsigned char*>(out_lo);
  if (!std_mode) {
    switch (layer) {
      case 2: launch_sp<SpConv2A, 0>(st, ih, il, w, b, out_scale, oh, ol, out_f32, n_seg); break;
      case 3: launch_sp<SpConv3A, 0>(st, ih, il, w, b, out_scale, oh, ol, out_f32, n_seg); break;
      case 4: launch_sp<SpConv4A, 0>(st, ih, il, w, b, out_scale, oh, ol, out_f32, n_seg); break;
      case 5: launch_sp<SpConv5A, 0>(st, ih, il, w, b, out_scale, oh, ol, out_f32, n_seg); break;
      default: launch_sp<SpConv6A, 0>(st, ih, il, w, b, out_scale, oh, ol, out_f32, n_seg); break;
    }
  } else {
    switch (layer) {
      case 2: launch_sp<SpConv2S, 0>(st, ih, il, w, b, out_scale, oh, ol, out_f32, n_seg); break;
      case 3: launch_sp<SpConv3S, 0>(st, ih, il, w, b, out_scale, oh, ol, out_f32, n_seg); break;
      case 4: launch_sp<SpConv4S, 0>(st, ih, il, w, b, out_scale, oh, ol, out_f32, n_seg); break;
      case 5: launch_sp<SpConv5S, 0>(st, ih, il, w, b, out_scale, oh, ol, out_f32, n_seg); break;
      default: launch_sp<SpConv6S, 0>(st, ih, il, w, b, out_scale, oh, ol, out_f32, n_seg); break;
    }
  }
}

// conv1 + pool1 + conv2 + pool2 in one kernel: mel segments -> the plane pair feeding conv3
void launch_conv12(cudaStream_t st, int std_mode, const float* mel, const int* seg_frame0, const float* seg_thr,
                   const float* w1, const float* b1, const void* wtc2, const float* bias2, float scale2,
                   void* out_hi, void* out_lo, int n_seg) {
  const __half* w = reinterpret_cast<const __half*>(wtc2);
  unsigned char* oh = static_cast<unsigned char*>(out_hi);
  unsigned char* ol = static_cast<unsigned char*>(out_lo);
  if (std_mode) launch_sp<SpConv2S, 2>(st, nullptr, nullptr, w, bias2, scale2, oh, ol, nullptr, n_seg, mel, seg_frame0, seg_thr, w1, b1);
  else launch_sp<SpConv2A, 1>(st, nullptr, nullptr, w, bias2, scale2, oh, ol, nullptr, n_seg, mel, seg_frame0, seg_thr, w1, b1);
}

void launch_unsplit(cudaStream_t st, int std_mode, int layer, const void* hi, const void* lo, float* out, int n_seg) {
  int H, W, C;
  split_geometry(std_mode, layer, &H, &W, &C);
  const long long items = (long long)n_seg * H * W * (C / 8);
  const unsigned char* h = static_cast<const unsigned char*>(hi);
  const unsigned char* l = static_cast<const unsigned char*>(lo);
  const int grid = (int)std::min<long long>((items + 255) / 256, (long long)device_sms() * 16);
  if (C == 16) unsplit_kernel<32><<<grid, 256, 0, st>>>(h, l, out, items, H, W);
  else if (C == 32) unsplit_kernel<64><<<grid, 256, 0, st>>>(h, l, out, items, H, W);
  else unsplit_kernel<128><<<grid, 256, 0, st>>>(h, l, out, items, H, W);
}

}  // namespace nisqa

// cnn.cu - framewise CNN over mel segments (reference nisqa/NISQA_lib.py:688-710 AdaptCNN,
// lib:811-836 StandardCNN; eval-mode BatchNorm folded into the conv weights on the host).
//
// Segments are never materialised: segment s is the view mel[frame0(s) .. frame0(s)+seg_len][n_mels]
// (x[i,0,m,t] = spec[m, i*seg_hop + t], lib:2266-2273).  Activations between layers live in
// HBM/L2 as channels-last [segment][h][w][c] fp32.
//
//   conv1_pool1_kernel : conv1(1->16)+BN+ReLU fused with the first max-pool, direct.
//   conv3x3_kernel<C>  : conv{2..6} as an fp32 implicit GEMM on the FFMA pipe.  Lanes of a
//                        warp own output channels (weights read as one contiguous, conflict-
//                        free shared-memory row per tap), a warp owns TH output rows x all
//                        columns of SPW segments (activations read as warp-broadcast
//                        LDS.128), max-pool + bias + ReLU fused into the epilogue.
// fp32 FFMA is a parity decision: TF32 operands alone move MOS by 2e-3 (SURVEY.md 0.8).
#include "common.cuh"
#include "tc_ptx.cuh"
#include "conv1_cell.cuh"
#include "conv_split.cuh"
#include "launch.cuh"

namespace nisqa {

// ----------------------------------------------------------------------------------------
// conv1 + BN + ReLU + pool1 of segments of n_mels x seg_len cells (mel rows n_mels floats apart)
//   MODE 0 (adapt, lib:690-691): adaptive_max_pool2d n_mels x seg_len -> PH x PW = cnn_pool_1 (conv1_adapt_cell; 48x15 ->
//          24 x 7: rows {2i,2i+1}, cols [2j,2j+3))
//   MODE 1 (standard, lib:813-814): MaxPool2d(2, stride 2, padding (0,1)) -> 24x8 : cols {2j-1,2j} (48 x 15 only)
// thread = one pooled cell of one segment, all C1 channels (16, 32 or 64 for AdaptCNN, in groups of 16).
// SPLIT: the output goes out as the two fp16 planes conv2's tensor-core kernel consumes (conv_split.cu:
// padded rows of C1 halves = 2 C1 bytes, swizzled) instead of fp32 channels-last (C1 = 16 only).
// (__launch_bounds__ minimum of 2 CTAs: without it ptxas holds the AdaptCNN cell at 80 registers and spills)
template <int MODE, bool SPLIT, int C1 = 16>
__global__ void __launch_bounds__(256, 2)
conv1_pool1_kernel(const float* __restrict__ mel, int n_mels, int seg_len, const int* __restrict__ seg_frame0,
                   const float* __restrict__ seg_thr, const float* __restrict__ w1 /*[9][C1]*/,
                   const float* __restrict__ b1 /*[C1]*/, float* __restrict__ out,
                   unsigned char* __restrict__ out_hi, unsigned char* __restrict__ out_lo, int n_seg, int PH, int PW) {
  static_assert(C1 == 16 || (MODE == 0 && SPLIT), "StandardCNN and the fp32 output: 16 channels");
  __shared__ __align__(16) float ws[9 * C1 + C1];
  for (int i = threadIdx.x; i < 9 * C1 + C1; i += blockDim.x)
    ws[i] = (i < 9 * C1) ? __ldg(w1 + i) : __ldg(b1 + i - 9 * C1);
  __syncthreads();

  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int seg = (int)(gid / (PH * PW));
  if (seg >= n_seg) return;
  const int cell = (int)(gid - (long long)seg * (PH * PW));
  const int ph = cell % PH, pw = cell / PH;      // lanes run along mel rows: coalesced reads
  const int f0 = __ldg(seg_frame0 + seg);
  const float thr = __ldg(seg_thr + seg);

  // channels 16 cg .. 16 cg + 15 -> the two 16-byte chunks 2 cg, 2 cg + 1 of the cell's plane row
  auto store_split = [&](const float (&res)[16], int cg) {
    const int g = kSplitLead + seg * ((PH + 1) * (PW + 1)) + (ph + 1) * (PW + 1) + (pw + 1);
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      uint4 hi, lo;
      split8(make_float4(res[8 * c], res[8 * c + 1], res[8 * c + 2], res[8 * c + 3]),
             make_float4(res[8 * c + 4], res[8 * c + 5], res[8 * c + 6], res[8 * c + 7]), hi, lo);
      const size_t o = split_off<2 * C1>(g, 2 * cg + c);
      *reinterpret_cast<uint4*>(out_hi + o) = hi;
      *reinterpret_cast<uint4*>(out_lo + o) = lo;
    }
  };
  float res[16];
  if constexpr (MODE == 0) {
    for (int cg = 0; cg < C1 / 16; ++cg) {     // one group of 16 channels at a time (the registers of one cell)
      conv1_adapt_cell<C1>(mel + (size_t)f0 * n_mels, n_mels, seg_len, PH, PW, thr, ws, ph, pw, 16 * cg, res);
      if constexpr (SPLIT) store_split(res, cg);
    }
  } else {
    conv1_cell<MODE>(mel, f0, thr, ws, ph, pw, res);
    if constexpr (SPLIT) store_split(res, 0);
  }
  if constexpr (!SPLIT) {
    float4* o = reinterpret_cast<float4*>(out + ((size_t)seg * PH * PW + ph * PW + pw) * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q)
      o[q] = make_float4(res[q * 4], res[q * 4 + 1], res[q * 4 + 2], res[q * 4 + 3]);
  }
}

// ----------------------------------------------------------------------------------------
// generic 3x3 conv (+bias+ReLU, + optional max-pool) on channels-last activations
enum { POOL_NONE = 0, POOL_ADAPT = 1, POOL_2X2 = 2 };

template <int H_, int W_, int CIN_, int COUT_, int PADW_, int POOL_, int POW_, int TH_, int SPW_,
          int NWARPS_, int MINB_>
struct ConvCfg {
  static constexpr int H = H_, W = W_, CIN = CIN_, COUT = COUT_, PADW = PADW_, POOL = POOL_;
  static constexpr int POW = POW_;                 // pooled output width (POOL != NONE)
  static constexpr int TH = TH_, SPW = SPW_, NWARPS = NWARPS_, MINB = MINB_;
  static constexpr int NT = NWARPS * 32;
  static constexpr int NC = COUT / 32;             // output channels per lane
  static constexpr int WO = W + 2 * PADW - 2;      // conv output width
  static constexpr int WP4 = ((W + 2 * PADW) + 3) / 4 * 4;   // padded smem row
  static constexpr int PLANE = (H + 2) * WP4 + 4;  // +4: spreads the channel planes over banks
  static constexpr int RB = H / TH;                // row blocks per segment
  static constexpr int G = (NWARPS / RB) * SPW;    // segments per CTA
  static constexpr int CK = 16;                    // input channels per staged chunk
  static constexpr int W_ELEMS = CK * 9 * COUT;
  static constexpr int A_ELEMS = G * CK * PLANE;
  static constexpr int SMEM_BYTES = (W_ELEMS + A_ELEMS) * 4;
  static constexpr int HO = (POOL == POOL_NONE) ? H : H / 2;
  static constexpr int WOUT = (POOL == POOL_NONE) ? WO : POW;
  static_assert(H % TH == 0 && NWARPS % RB == 0, "tile shape");
  static_assert(COUT % 32 == 0 && CIN % CK == 0, "channel shape");
  static_assert(POOL == POOL_NONE || TH % 2 == 0, "pooling needs row pairs");
};

template <class C>
__global__ void __launch_bounds__(C::NT, C::MINB)
conv3x3_kernel(const float* __restrict__ in, const float* __restrict__ wpack /*[CIN][9][COUT]*/,
               const float* __restrict__ bias, float* __restrict__ out, int n_seg) {
  constexpr int H = C::H, W = C::W, CIN = C::CIN, COUT = C::COUT, PADW = C::PADW;
  constexpr int TH = C::TH, SPW = C::SPW, NC = C::NC, WO = C::WO, WP4 = C::WP4;
  constexpr int PLANE = C::PLANE, CK = C::CK, NT = C::NT, G = C::G;
  extern __shared__ __align__(16) float smem[];
  float* wS = smem;
  float* aS = smem + C::W_ELEMS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int seg0 = blockIdx.x * G;
  const int sl0 = (warp / C::RB) * SPW;           // first CTA-local segment of this warp
  const int rb = warp % C::RB;                    // row block

  for (int i = tid; i < C::A_ELEMS / 4; i += NT)
    reinterpret_cast<float4*>(aS)[i] = make_float4(0.f, 0.f, 0.f, 0.f);   // zero halo (stays zero)

  float acc[SPW][TH][WO][NC];
#pragma unroll
  for (int s = 0; s < SPW; ++s)
#pragma unroll
    for (int r = 0; r < TH; ++r)
#pragma unroll
      for (int x = 0; x < WO; ++x)
#pragma unroll
        for (int c = 0; c < NC; ++c) acc[s][r][x][c] = 0.f;

  for (int ci0 = 0; ci0 < CIN; ci0 += CK) {
    __syncthreads();
    {  // weights chunk: contiguous [CK][9][COUT]
      const float4* src = reinterpret_cast<const float4*>(wpack + (size_t)ci0 * 9 * COUT);
      for (int i = tid; i < C::W_ELEMS / 4; i += NT) reinterpret_cast<float4*>(wS)[i] = __ldg(src + i);
    }
    // activation chunk: channels-last global -> per-channel planes with a zero halo
    for (int e = tid; e < G * H * W * (CK / 4); e += NT) {
      const int c4 = e % (CK / 4);
      const int pos = e / (CK / 4);
      const int w = pos % W, h = (pos / W) % H, sl = pos / (W * H);
      const int seg = seg0 + sl;
      if (seg < n_seg) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(
            in + ((size_t)seg * (H * W) + h * W + w) * CIN + ci0 + c4 * 4));
        float* dst = aS + (sl * CK + c4 * 4) * PLANE + (h + 1) * WP4 + w + PADW;
        dst[0] = v.x; dst[PLANE] = v.y; dst[2 * PLANE] = v.z; dst[3 * PLANE] = v.w;
      }
    }
    __syncthreads();

#pragma unroll 1
    for (int ci = 0; ci < CK; ++ci) {
      float wreg[9][NC];
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const float* wp = wS + (ci * 9 + tap) * COUT + lane * NC;
        if (NC == 2) {
          const float2 t = *reinterpret_cast<const float2*>(wp);
          wreg[tap][0] = t.x; wreg[tap][NC - 1] = t.y;
        } else {
#pragma unroll
          for (int c = 0; c < NC; ++c) wreg[tap][c] = wp[c];
        }
      }
#pragma unroll
      for (int s = 0; s < SPW; ++s) {
        const float* plane = aS + ((sl0 + s) * CK + ci) * PLANE + (rb * TH) * WP4;
#pragma unroll
        for (int ri = 0; ri < TH + 2; ++ri) {
          float a[WP4];
#pragma unroll
          for (int q = 0; q < WP4 / 4; ++q) {
            const float4 t = *reinterpret_cast<const float4*>(plane + ri * WP4 + q * 4);
            a[q * 4] = t.x; a[q * 4 + 1] = t.y; a[q * 4 + 2] = t.z; a[q * 4 + 3] = t.w;
          }
#pragma unroll
          for (int ky = 0; ky < 3; ++ky) {
            const int ro = ri - ky;
            if (ro >= 0 && ro < TH) {
#pragma unroll
              for (int x = 0; x < WO; ++x)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx)
#pragma unroll
                  for (int c = 0; c < NC; ++c)
                    acc[s][ro][x][c] = fmaf(a[x + kx], wreg[ky * 3 + kx][c], acc[s][ro][x][c]);
            }
          }
        }
      }
    }
  }

  // ---- epilogue: bias + ReLU (+ max-pool), channels-last store
  float bv[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) bv[c] = __ldg(bias + lane * NC + c);
#pragma unroll
  for (int s = 0; s < SPW; ++s) {
    const int seg = seg0 + sl0 + s;
    if (seg >= n_seg) continue;
    if (C::POOL == POOL_NONE) {
#pragma unroll
      for (int r = 0; r < TH; ++r)
#pragma unroll
        for (int x = 0; x < WO; ++x) {
          float* o = out + ((size_t)seg * (H * WO) + (rb * TH + r) * WO + x) * COUT + lane * NC;
#pragma unroll
          for (int c = 0; c < NC; ++c) o[c] = fmaxf(acc[s][r][x][c] + bv[c], 0.f);
        }
    } else {
      constexpr int POW = C::POW;
#pragma unroll
      for (int pr = 0; pr < TH / 2; ++pr)
#pragma unroll
        for (int pc = 0; pc < POW; ++pc) {
          // adaptive_max_pool2d window [floor(pc*WO/POW), ceil((pc+1)*WO/POW)); 2x2: [2pc, 2pc+2)
          const int x0 = (C::POOL == POOL_ADAPT) ? (pc * WO) / POW : 2 * pc;
          const int x1 = (C::POOL == POOL_ADAPT) ? ((pc + 1) * WO + POW - 1) / POW : 2 * pc + 2;
          float* o = out + ((size_t)seg * (C::HO * POW) + (rb * (TH / 2) + pr) * POW + pc) * COUT + lane * NC;
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            float m = -INFINITY;
#pragma unroll
            for (int x = 0; x < WO; ++x)
              if (x >= x0 && x < x1) m = fmaxf(m, fmaxf(acc[s][2 * pr][x][c], acc[s][2 * pr + 1][x][c]));
            o[c] = fmaxf(m + bv[c], 0.f);
          }
        }
    }
  }
}

// NHWC [n][HW][C] (rows of ld floats) -> NCHW [n][C][HW] (stage dumps only; matches the reference tensor layout)
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ in, int ld, float* __restrict__ out,
                                    long long n, int hw, int ch) {
  const long long total = n * hw * ch;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(i % hw);
    const int c = (int)((i / hw) % ch);
    const long long s = i / ((long long)hw * ch);
    out[i] = in[s * ld + p * ch + c];
  }
}

// ------------------------------------------------------------------------ layer configs
//                       H   W  CIN COUT PADW POOL        POW TH SPW NWARPS MINB
using Conv2A = ConvCfg<24, 7, 16, 32, 1, POOL_ADAPT, 5, 8, 1, 6, 3>;   // -> [12][5][32]
using Conv3A = ConvCfg<12, 5, 32, 64, 1, POOL_NONE, 0, 4, 1, 6, 3>;   // -> [12][5][64]
using Conv4A = ConvCfg<12, 5, 64, 64, 1, POOL_ADAPT, 3, 4, 1, 6, 3>;   // -> [6][3][64]
using Conv5A = ConvCfg<6, 3, 64, 64, 1, POOL_NONE, 0, 6, 1, 8, 2>;    // -> [6][3][64]
using Conv6A = ConvCfg<6, 3, 64, 64, 0, POOL_NONE, 0, 6, 4, 8, 2>;    // -> [6][1][64]
using Conv2S = ConvCfg<24, 8, 16, 32, 1, POOL_2X2, 4, 8, 1, 6, 3>;     // -> [12][4][32]
using Conv3S = ConvCfg<12, 4, 32, 64, 1, POOL_NONE, 0, 4, 1, 6, 3>;   // -> [12][4][64]
using Conv4S = ConvCfg<12, 4, 64, 64, 1, POOL_2X2, 2, 4, 1, 6, 3>;     // -> [6][2][64]
using Conv5S = ConvCfg<6, 2, 64, 64, 1, POOL_NONE, 0, 6, 2, 8, 2>;    // -> [6][2][64]
using Conv6S = Conv5S;

static_assert(input_is<Conv2A>(0, 2) && input_is<Conv3A>(0, 3) && input_is<Conv4A>(0, 4) && input_is<Conv5A>(0, 5) &&
              input_is<Conv6A>(0, 6) && input_is<Conv2S>(1, 2) && input_is<Conv3S>(1, 3) && input_is<Conv4S>(1, 4) &&
              input_is<Conv5S>(1, 5) && input_is<Conv6S>(1, 6), "ConvCfg geometry differs from split_geometry");

template <class C>
static void launch_conv(cudaStream_t st, const float* in, const float* w, const float* b,
                        float* out, int n_seg) {
  static unsigned long long configured = 0;
  if (first_launch_on_device(configured)) {
    cudaFuncSetAttribute(conv3x3_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         C::SMEM_BYTES);
  }
  const int grid = (n_seg + C::G - 1) / C::G;
  conv3x3_kernel<C><<<grid, C::NT, C::SMEM_BYTES, st>>>(in, w, b, out, n_seg);
}

bool launch_conv1(cudaStream_t st, int std_mode, int c1, const float* mel, int n_mels, int seg_len, const int* seg_frame0,
                  const float* seg_thr, const float* w1, const float* b1, float* out, int n_seg, void* out_hi, void* out_lo,
                  int ph, int pw) {
  if (c1 != 16 && (std_mode || !out_hi || (c1 != 32 && c1 != 64))) return false;
  if (std_mode) { ph = 24; pw = 8; }
  const long long total = (long long)n_seg * ph * pw;
  const int grid = (int)((total + 255) / 256);
  unsigned char* oh = static_cast<unsigned char*>(out_hi);
  unsigned char* ol = static_cast<unsigned char*>(out_lo);
  const int H = n_mels, W = seg_len;
  if (out_hi) {
    if (std_mode) conv1_pool1_kernel<1, true><<<grid, 256, 0, st>>>(mel, H, W, seg_frame0, seg_thr, w1, b1, out, oh, ol, n_seg, ph, pw);
    else if (c1 == 32) conv1_pool1_kernel<0, true, 32><<<grid, 256, 0, st>>>(mel, H, W, seg_frame0, seg_thr, w1, b1, out, oh, ol, n_seg, ph, pw);
    else if (c1 == 64) conv1_pool1_kernel<0, true, 64><<<grid, 256, 0, st>>>(mel, H, W, seg_frame0, seg_thr, w1, b1, out, oh, ol, n_seg, ph, pw);
    else conv1_pool1_kernel<0, true><<<grid, 256, 0, st>>>(mel, H, W, seg_frame0, seg_thr, w1, b1, out, oh, ol, n_seg, ph, pw);
  } else {
    if (std_mode) conv1_pool1_kernel<1, false><<<grid, 256, 0, st>>>(mel, H, W, seg_frame0, seg_thr, w1, b1, out, oh, ol, n_seg, ph, pw);
    else conv1_pool1_kernel<0, false><<<grid, 256, 0, st>>>(mel, H, W, seg_frame0, seg_thr, w1, b1, out, oh, ol, n_seg, ph, pw);
  }
  return true;
}

// layer = 2..6
void launch_conv_layer(cudaStream_t st, int std_mode, int layer, const float* in, const float* w,
                       const float* b, float* out, int n_seg) {
  if (!std_mode) {
    switch (layer) {
      case 2: launch_conv<Conv2A>(st, in, w, b, out, n_seg); break;
      case 3: launch_conv<Conv3A>(st, in, w, b, out, n_seg); break;
      case 4: launch_conv<Conv4A>(st, in, w, b, out, n_seg); break;
      case 5: launch_conv<Conv5A>(st, in, w, b, out, n_seg); break;
      default: launch_conv<Conv6A>(st, in, w, b, out, n_seg); break;
    }
  } else {
    switch (layer) {
      case 2: launch_conv<Conv2S>(st, in, w, b, out, n_seg); break;
      case 3: launch_conv<Conv3S>(st, in, w, b, out, n_seg); break;
      case 4: launch_conv<Conv4S>(st, in, w, b, out, n_seg); break;
      case 5: launch_conv<Conv5S>(st, in, w, b, out, n_seg); break;
      default: launch_conv<Conv6S>(st, in, w, b, out, n_seg); break;
    }
  }
}

void launch_nhwc_to_nchw(cudaStream_t st, const float* in, int ld, float* out, long long n, int hw, int ch) {
  nhwc_to_nchw_kernel<<<1024, 256, 0, st>>>(in, ld, out, n, hw, ch);
}

}  // namespace nisqa

// conv1_cell.cuh - conv1(1->16) + BN + ReLU fused with the first max-pool for ONE pooled cell of one segment (all 16
// channels), for conv1_pool1_kernel (cnn.cu), and the strip form of the fused conv1 + conv2 kernel (conv_split.cu).
// conv1_adapt_cell takes 16 of the C1 = 16 / 32 / 64 channels of an AdaptCNN conv1 (cnn_c_out_1) at a time.
//   MODE 0 (adapt, reference lib:690-691): adaptive_max_pool2d 48x15 -> 24x7 : rows {2i,2i+1}, cols [2j,2j+3)
//   MODE 1 (standard, lib:813-814): MaxPool2d(2, stride 2, padding (0,1)) -> 24x8 : cols {2j-1,2j}
//   conv1_adapt_cell: AdaptCNN at any n_mels x seg_len (adaptive windows from the runtime shape)
#pragma once
#include "common.cuh"
#include "f32x2.cuh"

namespace nisqa {

// ws: [9][16] folded conv1 weights followed by the 16 biases (shared memory).  LDG: `mel` is global memory read through
// the read-only path; false: a shared-memory copy of the segment's 15 mel rows (f0 = 0), rows PITCH floats apart.
// NCQ channel quads starting at quad cq0 (NCQ = 4, cq0 = 0: all 16 channels; the fused kernel splits them over two warp groups).
template <int MODE, bool LDG = true, int PITCH = kMels, int NCQ = 4>
__device__ __forceinline__ void conv1_cell(const float* __restrict__ mel, int f0, float thr, const float* ws,
                                           int ph, int pw, float (&res)[4 * NCQ], int cq0 = 0) {
  constexpr int NWC = (MODE == 0) ? 3 : 2;       // window columns
  constexpr int PC = NWC + 2;                    // patch columns
  const int r0 = 2 * ph - 1;                     // first patch row (mel index)
  const int c0 = (MODE == 0) ? 2 * pw - 1 : 2 * pw - 2;   // first patch col (frame in segment)
  float patch[4][PC];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < PC; ++j) {
      const int r = r0 + i, t = c0 + j;
      float v = 0.f;                             // zero padding of the segment's own border
      if (r >= 0 && r < kMels && t >= 0 && t < kSegLen)
        v = fmaxf(LDG ? __ldg(mel + (size_t)(f0 + t) * PITCH + r) : mel[(f0 + t) * PITCH + r], thr);
      patch[i][j] = v;
    }

  // 16 channels as 8 pairs (f32x2.cuh: the same fp32 FMA per element and tap order as one fmaf per channel)
#pragma unroll
  for (int cq_ = 0; cq_ < NCQ; ++cq_) {
    const int cq = cq0 + cq_;
    f2 acc[2][NWC][2];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < NWC; ++j) { acc[i][j][0] = 0ull; acc[i][j][1] = 0ull; }
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const float4 w = *reinterpret_cast<const float4*>(ws + tap * 16 + cq * 4);
      const f2 w01 = pk(w.x, w.y), w23 = pk(w.z, w.w);
      const int ky = tap / 3, kx = tap % 3;
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < NWC; ++j) {
          const f2 a = bc(patch[i + ky][j + kx]);
          acc[i][j][0] = fma2(a, w01, acc[i][j][0]);
          acc[i][j][1] = fma2(a, w23, acc[i][j][1]);
        }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < NWC; ++j) {
          const int col = c0 + 1 + j;            // conv output column of this window slot
          if (MODE == 0 || (col >= 0 && col < kSegLen)) {
            const float2 v = upk(acc[i][j][h]);
            m0 = fmaxf(m0, v.x); m1 = fmaxf(m1, v.y);
          }
        }
      res[cq_ * 4 + 2 * h] = fmaxf(m0 + ws[144 + cq * 4 + 2 * h], 0.f);           // bias + ReLU commute with max
      res[cq_ * 4 + 2 * h + 1] = fmaxf(m1 + ws[144 + cq * 4 + 2 * h + 1], 0.f);
    }
  }
}

// AdaptCNN conv1 + BN + ReLU + adaptive_max_pool2d to PH x PW (cnn_pool_1, shipped 24 x 7) for one pooled cell (ph, pw),
// channels c0 .. c0 + 15 of C1, of a segment of H mel rows x W frames (seg: its frame 0, rows H floats apart; ws: [9][C1]
// weights, then C1 biases).  The cell's window (F.adaptive_max_pool2d) is conv rows [floor(ph H / PH), ceil((ph + 1) H / PH))
// x columns [floor(pw W / PW), ceil((pw + 1) W / PW)).  Each conv position is the fmaf chain of conv1_cell (zero start, taps
// 0..8, inputs clamped at thr, zero outside the segment), each cell the max, + bias, ReLU: at 48 x 15 -> 24 x 7 the windows
// are conv1_cell<0>'s and the results bit-identical to it and to conv1_strip.
template <int C1>
__device__ __forceinline__ void conv1_adapt_cell(const float* __restrict__ seg, int H, int W, int PH, int PW, float thr,
                                                 const float* ws, int ph, int pw, int c0, float (&res)[16]) {
  const int y0 = (ph * H) / PH, y1 = ((ph + 1) * H + PH - 1) / PH;
  const int x0 = (pw * W) / PW, x1 = ((pw + 1) * W + PW - 1) / PW;
  float mx[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) mx[c] = -INFINITY;
  for (int y = y0; y < y1; ++y)
    for (int x = x0; x < x1; ++x) {
      float a[9];
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const int r = y - 1 + tap / 3, t = x - 1 + tap % 3;
        a[tap] = (r >= 0 && r < H && t >= 0 && t < W) ? fmaxf(__ldg(seg + (size_t)t * H + r), thr) : 0.f;
      }
      float acc[16];
#pragma unroll
      for (int c = 0; c < 16; ++c) acc[c] = 0.f;
#pragma unroll
      for (int tap = 0; tap < 9; ++tap)
#pragma unroll
        for (int c = 0; c < 16; ++c) acc[c] = fmaf(a[tap], ws[tap * C1 + c0 + c], acc[c]);
#pragma unroll
      for (int c = 0; c < 16; ++c) mx[c] = fmaxf(mx[c], acc[c]);
    }
#pragma unroll
  for (int c = 0; c < 16; ++c) res[c] = fmaxf(mx[c] + ws[9 * C1 + c0 + c], 0.f);   // bias + ReLU commute with max
}

// Pooled cells PW0 .. PW1 - 1 of pooled row ph for the 4 channels of one quad, with every conv1 output position computed
// once (AdaptCNN: a column shared by two overlapping windows feeds both maxima instead of being computed twice).  Each
// position is the same fmaf chain as in conv1_cell (zero start, taps 0..8), each cell the same max, + bias, ReLU, so the
// results are bit-identical to conv1_cell's.  mel: the segment's frames (f0 = 0), PITCH floats apart; wq / bq: the
// quad's folded weights and biases.  emit(pw, res) receives each cell as soon as its last column is done.
template <int MODE, int PW0, int PW1, int PITCH, class Emit>
__device__ __forceinline__ void conv1_strip(const float* mel, float thr, const float (&wq)[9][4], const float (&bq)[4],
                                            int ph, Emit&& emit) {
  constexpr int NC = PW1 - PW0;
  // conv columns of cell pw: [lo(pw), hi(pw)] (MODE 1: the padding column -1 and column 15 do not exist)
  auto lo = [](int pw) { return MODE == 0 ? 2 * pw : (2 * pw - 1 < 0 ? 0 : 2 * pw - 1); };
  auto hi = [](int pw) { return MODE == 0 ? 2 * pw + 2 : (2 * pw < kSegLen - 1 ? 2 * pw : kSegLen - 1); };
  constexpr int X0 = MODE == 0 ? 2 * PW0 : (2 * PW0 - 1 < 0 ? 0 : 2 * PW0 - 1);
  constexpr int X1 = MODE == 0 ? 2 * (PW1 - 1) + 2 : (2 * (PW1 - 1) < kSegLen - 1 ? 2 * (PW1 - 1) : kSegLen - 1);
  const int r0 = 2 * ph - 1;                     // first mel row of the 3x3 windows of conv rows 2 ph, 2 ph + 1
  // mel frame t, rows r0 .. r0 + 3 (clamped at thr; zero outside the segment)
  auto load_frame = [&](int t, float (&v)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = r0 + i;
      v[i] = 0.f;
      if (t >= 0 && t < kSegLen && r >= 0 && r < kMels) v[i] = fmaxf(mel[t * PITCH + r], thr);
    }
  };
  float fr[3][4];                                // frames x - 1, x, x + 1 at fr[(t - X0 + 1) % 3]
  load_frame(X0 - 1, fr[0]);
  load_frame(X0, fr[1]);
  float mx[NC][4];
#pragma unroll
  for (int p = 0; p < NC; ++p)
#pragma unroll
    for (int c = 0; c < 4; ++c) mx[p][c] = -INFINITY;
#pragma unroll
  for (int x = X0; x <= X1; ++x) {
    load_frame(x + 1, fr[(x - X0 + 2) % 3]);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const int ky = tap / 3, kx = tap % 3;
        const float a = fr[(x - 1 + kx - X0 + 1) % 3][i + ky];
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[c] = fmaf(a, wq[tap][c], acc[c]);
      }
#pragma unroll
      for (int p = 0; p < NC; ++p)
        if (x >= lo(PW0 + p) && x <= hi(PW0 + p))
#pragma unroll
          for (int c = 0; c < 4; ++c) mx[p][c] = fmaxf(mx[p][c], acc[c]);
    }
#pragma unroll
    for (int p = 0; p < NC; ++p)
      if (x == hi(PW0 + p)) {
        float res[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) res[c] = fmaxf(mx[p][c] + bq[c], 0.f);   // bias + ReLU commute with max
        emit(PW0 + p, res);
      }
  }
}

}  // namespace nisqa

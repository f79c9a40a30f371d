// td.cu - the time-dependency and pooling kernels that are not register-tiled GEMMs (the self-attention stacks live in
// td_tiled.cu):
//   standard arch : fc_out 768->20 (reference nisqa/NISQA_lib.py:832-834, linear_rows_kernel), BiLSTM (lib:925-943, one
//                   CTA per sequence or NB sequences per CTA in lock step), PoolLastStepBi (lib:1107-1115)
//   both archs    : the pooling modules - PoolAttFF (lib:1156-1183) behind self-attention, whose logits td_sa_kernel
//                   computes, and PoolAtt / PoolAvg / PoolMax / PoolLastStep behind either time-dependency block
// Clips are ragged: every kernel works on the clip's valid rows only, so no key-padding mask exists.
#include <algorithm>

#include "common.cuh"
#include "launch.cuh"

namespace nisqa {

constexpr int kRows = 128;       // rows (threads) per CTA in the row-thread kernels
constexpr int kXS = 65;          // padded row stride of the per-thread smem row

// acc[j] += sum_{k<kc} xrow[k] * ws[k*NCOL + j]
template <int NCOL>
__device__ __forceinline__ void rowgemm(float (&acc)[NCOL], const float* xrow, const float* ws, int kc) {
  static_assert(NCOL % 4 == 0, "NCOL");
#pragma unroll 4
  for (int k = 0; k < kc; ++k) {
    const float xv = xrow[k];
    const float4* w4 = reinterpret_cast<const float4*>(ws + k * NCOL);
#pragma unroll
    for (int q = 0; q < NCOL / 4; ++q) {
      const float4 w = w4[q];
      acc[q * 4 + 0] = fmaf(xv, w.x, acc[q * 4 + 0]);
      acc[q * 4 + 1] = fmaf(xv, w.y, acc[q * 4 + 1]);
      acc[q * 4 + 2] = fmaf(xv, w.z, acc[q * 4 + 2]);
      acc[q * 4 + 3] = fmaf(xv, w.w, acc[q * 4 + 3]);
    }
  }
}

__device__ __forceinline__ void stage_f4(float* dst, const float* __restrict__ src, int n_floats) {
  const float4* s = reinterpret_cast<const float4*>(src);
  for (int i = threadIdx.x; i < n_floats / 4; i += blockDim.x) reinterpret_cast<float4*>(dst)[i] = __ldg(s + i);
}

// ---------------------------------------------------------------------------------------
// out[row][0..NOUT) = in[row][0..K) @ WT[K][NOUT] + bias   K % 64 == 0; one thread per row
template <int NOUT>
__global__ void __launch_bounds__(kRows)
linear_rows_kernel(const float* __restrict__ in, int K, const float* __restrict__ WT,
                   const float* __restrict__ bias, float* __restrict__ out, int n_rows) {
  extern __shared__ __align__(16) float sm[];
  float* xs = sm;                       // [kRows][kXS]
  float* ws = sm + kRows * kXS;         // [64][NOUT]
  const int row0 = blockIdx.x * kRows, tid = threadIdx.x;
  float acc[NOUT];
#pragma unroll
  for (int j = 0; j < NOUT; ++j) acc[j] = __ldg(bias + j);
  for (int k0 = 0; k0 < K; k0 += 64) {
    __syncthreads();
    for (int i = tid; i < kRows * 64; i += kRows) {
      const int r = i >> 6, k = i & 63;
      xs[r * kXS + k] = (row0 + r < n_rows) ? __ldg(in + (size_t)(row0 + r) * K + k0 + k) : 0.f;
    }
    stage_f4(ws, WT + (size_t)k0 * NOUT, 64 * NOUT);
    __syncthreads();
    rowgemm<NOUT>(acc, xs + tid * kXS, ws, 64);
  }
  if (row0 + tid >= n_rows) return;
  float* o = out + (size_t)(row0 + tid) * NOUT;
#pragma unroll
  for (int q = 0; q < NOUT / 4; ++q)
    reinterpret_cast<float4*>(o)[q] = make_float4(acc[q * 4], acc[q * 4 + 1], acc[q * 4 + 2], acc[q * 4 + 3]);
}

// ---------------------------------------------------------------------------------------
// PoolAttFF: softmax over the clip's time steps, weighted sum of x, Linear D->1   (lib:1177-1181)
// grid = n_clips, block = 64 * n_heads; thread (h, d) owns features d, d + 64, .. < D (rows ldx floats apart).  The softmax numerators are formed once per (head, step) into shared
// memory; the weighted sum keeps ONE accumulator per thread in step order (the result does not depend on the unrolling) with
// eight independent loads in flight.
__global__ void pool_final_kernel(const float* __restrict__ x, const float* __restrict__ logits,
                                  const ClipDesc* __restrict__ clips, PoolHeadParams P, int n_heads, int max_seg, int D, int ldx,
                                  float* __restrict__ scores) {
  __shared__ float red[5 * 64];
  extern __shared__ float pnum[];                       // [n_heads][max_seg] softmax numerators
  const ClipDesc cd = clips[blockIdx.x];
  const int S = cd.n_seg;
  const int h = threadIdx.x >> 6, d = threadIdx.x & 63;
  if (S <= 0) { if (d == 0) scores[blockIdx.x * n_heads + h] = __int_as_float(0x7fc00000); return; }
  const float* lg = logits + (size_t)cd.seg_off * n_heads + h;
  float* pn = pnum + (size_t)h * max_seg;
  float mx = -INFINITY;
  for (int t = d; t < S; t += 64) mx = fmaxf(mx, __ldg(lg + (size_t)t * n_heads));
  red[threadIdx.x] = mx;
  __syncthreads();
  for (int o = 32; o > 0; o >>= 1) { if (d < o) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + o]); __syncthreads(); }
  mx = red[h * 64];
  __syncthreads();
  float sum = 0.f;
  for (int t = d; t < S; t += 64) { const float e = expf(__ldg(lg + (size_t)t * n_heads) - mx); pn[t] = e; sum += e; }
  red[threadIdx.x] = sum;
  __syncthreads();
  for (int o = 32; o > 0; o >>= 1) { if (d < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
  sum = red[h * 64];
  __syncthreads();
  float tot = 0.f;
  for (int c = 0; c < D; c += 64) {
    float acc = 0.f;
    if (c + d < D) {                  // (D = 32 / 96 behind an LSTM: the last chunk is partial)
      const float* xb = x + (size_t)cd.seg_off * ldx + c + d;
      int t = 0;
      for (; t + 8 <= S; t += 8) {
        float xv[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) xv[u] = __ldg(xb + (size_t)(t + u) * ldx);
#pragma unroll
        for (int u = 0; u < 8; ++u) acc = fmaf(pn[t + u], xv[u], acc);
      }
      for (; t < S; ++t) acc = fmaf(pn[t], __ldg(xb + (size_t)t * ldx), acc);
      acc = (acc / sum) * __ldg(P.w3 + h * D + c + d);
    }
    tot = c ? tot + acc : acc;
  }
  red[threadIdx.x] = tot;
  __syncthreads();
  for (int o = 32; o > 0; o >>= 1) { if (d < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
  if (d == 0) scores[blockIdx.x * n_heads + h] = red[h * 64] + __ldg(P.b3 + h);
}

// ---------------------------------------------------------------------------------------
// The other pooling modules of the reference (user-trained checkpoints, SURVEY.md 8f.4), one CTA per clip, D threads
// (thread d owns feature d; D = 64..256 after self-attention, dirs H = 32..512 after an LSTM; rows ldx floats apart):
//   mode 1 PoolAtt       (lib:1131-1154): att_t = a1 . x_t + a1b, softmax over the clip's steps, sum_t att_t x_t, Linear
//   mode 2 PoolAvg       (lib:1185-1204): mean over the clip's steps, Linear
//   mode 3 PoolMax       (lib:1206-1225): max over the clip's steps, Linear
//   mode 4 PoolLastStep  (lib:1117-1129): x at the last valid step, Linear
//   mode 5 PoolLastStepBi (lib:1107-1115): the forward half at the last valid step, the backward half at step 0, Linear
// One Linear(D -> 1) per head (NISQA_DIM: five heads with their own weights, lib:260-268).

template <int D>
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < D / 32; ++w) t += red[w];
  return t;
}
template <int D>
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = -INFINITY;
#pragma unroll
  for (int w = 0; w < D / 32; ++w) t = fmaxf(t, red[w]);
  return t;
}

template <int D>
__global__ void __launch_bounds__(D, 1)
pool_simple_kernel(const float* __restrict__ x /*[n_seg][ldx]*/, int ldx, const ClipDesc* __restrict__ clips, int mode,
                   PoolSimpleParams P, int n_heads, float* __restrict__ scores) {
  extern __shared__ __align__(16) float slog[];          // mode 1: softmax numerators of the clip's steps
  __shared__ float red[D / 32];
  const ClipDesc cd = clips[blockIdx.x];
  const int S = cd.n_seg, d = threadIdx.x, lane = d & 31, warp = d >> 5;
  if (S <= 0) { if (d < n_heads) scores[blockIdx.x * n_heads + d] = __int_as_float(0x7fc00000); return; }
  const float* xb = x + (size_t)cd.seg_off * ldx;
  float pooled = 0.f;
  if (mode == 2) {
    for (int t = 0; t < S; ++t) pooled += __ldg(xb + (size_t)t * ldx + d);
    pooled = pooled / (float)S;
  } else if (mode == 3) {
    pooled = -INFINITY;
    for (int t = 0; t < S; ++t) pooled = fmaxf(pooled, __ldg(xb + (size_t)t * ldx + d));
  } else if (mode == 4) {
    pooled = __ldg(xb + (size_t)(S - 1) * ldx + d);
  } else if (mode == 5) {
    pooled = __ldg(xb + (size_t)(d < D / 2 ? S - 1 : 0) * ldx + d);
  }
  for (int h = 0; h < n_heads; ++h) {
    if (mode == 1) {
      __syncthreads();                                    // slog of the previous head consumed
      for (int t = warp; t < S; t += D / 32) {
        float a = 0.f;
        for (int k = lane; k < D; k += 32) a = fmaf(__ldg(xb + (size_t)t * ldx + k), __ldg(P.a1 + h * D + k), a);
        a = warp_sum(a);
        if (lane == 0) slog[t] = a + __ldg(P.a1b + h);
      }
      __syncthreads();
      float mx = -INFINITY;
      for (int t = d; t < S; t += D) mx = fmaxf(mx, slog[t]);
      mx = block_max<D>(mx, red);
      float sum = 0.f;
      for (int t = d; t < S; t += D) { const float e = expf(slog[t] - mx); slog[t] = e; sum += e; }
      sum = block_sum<D>(sum, red);                       // (its barriers also publish the numerators)
      float acc = 0.f;
      for (int t = 0; t < S; ++t) acc = fmaf(slog[t], __ldg(xb + (size_t)t * ldx + d), acc);
      pooled = acc / sum;
    }
    const float tot = block_sum<D>(pooled * __ldg(P.w3 + h * D + d), red);
    if (d == 0) scores[blockIdx.x * n_heads + h] = tot + __ldg(P.b3 + h);
  }
}

// ---------------------------------------------------------------------------------------
// BiLSTM(20 -> 128), one CTA per (clip, direction), 512 threads = 512 gate rows.  The four gates
// of hidden unit j live in one lane quad (thread t: unit t>>2, gate t&3 in PyTorch order i,f,g,o),
// so the gate exchange is four shuffles, the cell update is replicated in the quad, and a step
// needs ONE barrier (h and x are double buffered).  W_hh row: first 64 taps in registers, last 64
// in shared memory [k][512].
constexpr int kLstmSmemFloats = 64 * 512 + 2 * 128 + 2 * 32 + 128;

__global__ void __launch_bounds__(512, 1)
lstm_kernel(const float* __restrict__ feats /*[n_seg][20]*/, const ClipDesc* __restrict__ clips,
            LstmParams P, float* __restrict__ td_out /*[n_seg][256]*/, float* __restrict__ partial /*[n_clips][2]*/) {
  extern __shared__ __align__(16) float sm[];
  float* whs = sm;                   // [64][512]  taps 64..127, indexed by thread
  float* hbuf = sm + 64 * 512;       // [2][128]
  float* xbuf = hbuf + 256;          // [2][32] input of the current / next step (20 used)
  float* red = xbuf + 64;            // [128]
  const int clip = blockIdx.x >> 1, dir = blockIdx.x & 1;
  const ClipDesc cd = clips[clip];
  const int S = cd.n_seg;
  const int t = threadIdx.x, lane = t & 31;
  const int unit = t >> 2, gate = t & 3;
  const int grow = gate * 128 + unit;          // row of the PyTorch gate matrices
  if (S <= 0) { if (t == 0) partial[clip * 2 + dir] = 0.f; return; }

  float wr[64], wi[20];
  {
    const float* wrow = P.w_hh + ((size_t)dir * 512 + grow) * 128;
#pragma unroll
    for (int k = 0; k < 64; ++k) wr[k] = __ldg(wrow + k);
    for (int k = 0; k < 64; ++k) whs[k * 512 + t] = __ldg(wrow + 64 + k);
    const float* irow = P.w_ih + ((size_t)dir * 512 + grow) * 20;
#pragma unroll
    for (int k = 0; k < 20; ++k) wi[k] = __ldg(irow + k);
  }
  const float bias = __ldg(P.b + dir * 512 + grow);
  if (t < 256) hbuf[t] = 0.f;
  if (t < 64) xbuf[t] = 0.f;
  float cstate = 0.f, hlast = 0.f;
  const float* fb = feats + (size_t)cd.seg_off * 20;
  __syncthreads();
  if (t < 20) xbuf[t] = __ldg(fb + (size_t)(dir ? S - 1 : 0) * 20 + t);
  __syncthreads();

  for (int step = 0; step < S; ++step) {
    const int tt = dir ? S - 1 - step : step;
    const float* h = hbuf + (step & 1) * 128;
    const float* xt = xbuf + (step & 1) * 32;
    // prefetch the next input row while this step computes
    float xnext = 0.f;
    if (t < 20 && step + 1 < S) xnext = __ldg(fb + (size_t)(dir ? S - 2 - step : step + 1) * 20 + t);
    float a0 = bias, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
    for (int k = 0; k < 20; k += 4) {
      const float4 xv = *reinterpret_cast<const float4*>(xt + k);
      a0 = fmaf(wi[k], xv.x, a0); a1 = fmaf(wi[k+1], xv.y, a1); a2 = fmaf(wi[k+2], xv.z, a2); a3 = fmaf(wi[k+3], xv.w, a3);
    }
#pragma unroll
    for (int k = 0; k < 64; k += 4) {
      const float4 hv = *reinterpret_cast<const float4*>(h + k);
      a0 = fmaf(wr[k], hv.x, a0); a1 = fmaf(wr[k+1], hv.y, a1); a2 = fmaf(wr[k+2], hv.z, a2); a3 = fmaf(wr[k+3], hv.w, a3);
    }
#pragma unroll 8
    for (int k = 0; k < 64; k += 4) {
      const float4 hv = *reinterpret_cast<const float4*>(h + 64 + k);
      a0 = fmaf(whs[(k) * 512 + t], hv.x, a0); a1 = fmaf(whs[(k+1) * 512 + t], hv.y, a1);
      a2 = fmaf(whs[(k+2) * 512 + t], hv.z, a2); a3 = fmaf(whs[(k+3) * 512 + t], hv.w, a3);
    }
    const float pre = (a0 + a1) + (a2 + a3);
    // gate nonlinearity: gate 2 is the cell candidate (tanh), the others sigmoid
    const float act = (gate == 2) ? tanhf(pre) : 1.0f / (1.0f + expf(-pre));
    const int q0 = lane & ~3;
    const float ig = __shfl_sync(0xffffffffu, act, q0);
    const float fg = __shfl_sync(0xffffffffu, act, q0 + 1);
    const float gg = __shfl_sync(0xffffffffu, act, q0 + 2);
    const float og = __shfl_sync(0xffffffffu, act, q0 + 3);
    cstate = fmaf(fg, cstate, ig * gg);
    hlast = og * tanhf(cstate);
    if (gate == 0) {
      hbuf[((step + 1) & 1) * 128 + unit] = hlast;
      td_out[((size_t)cd.seg_off + tt) * 256 + dir * 128 + unit] = hlast;
    }
    if (t < 20) xbuf[((step + 1) & 1) * 32 + t] = xnext;
    __syncthreads();
  }
  // PoolLastStepBi: this direction's final hidden state . w_pool half
  if (gate == 0) red[unit] = hlast * __ldg(P.w_pool + dir * 128 + unit);
  __syncthreads();
  if (t < 32) {
    float v = red[t] + red[t + 32] + red[t + 64] + red[t + 96];
    v = warp_sum(v);
    if (t == 0) partial[clip * 2 + dir] = v;
  }
}

// ---------------------------------------------------------------------------------------
// Batched BiLSTM (round 2): one CTA advances NB clips of one direction in lock step, so that the recurrent weights
// (512 x 128 fp32 = 256 KB: half in registers, half in shared memory) are fetched once per step for NB sequences
// instead of once per sequence - the step is FMA bound (2 x 148 x NB FMAs per thread) instead of LDS / barrier bound,
// and 256 clips x 2 directions fit on the chip in ONE wave (the one-sequence kernel above needed 3.5 waves of
// 987 serial steps).  256 threads: thread t owns hidden unit u = t >> 1 and the gate pair gp = t & 1 ((i, f) or
// (g, o), PyTorch row order i, f, g, o), i.e. two rows of W_hh / W_ih; the pair of lanes of a unit exchanges its four
// gate values with two shuffles per sequence and both update the (replicated) cell state.  Sequences of a group may
// have different lengths (clips are sorted by length on the host): a finished sequence keeps its state.
// `order` lists the clips of the pass by decreasing n_seg; group g = clips order[NB g .. NB g + NB).
template <int NB>
__global__ void __launch_bounds__(256, 1)
lstm_batched_kernel(const float* __restrict__ feats /*[n_seg][20]*/, const ClipDesc* __restrict__ clips,
                    const int* __restrict__ order, int n_clips, LstmParams P,
                    float* __restrict__ td_out /*[n_seg][256] or nullptr*/, float* __restrict__ partial /*[n_clips][2]*/) {
  extern __shared__ __align__(16) float sm[];
  float2* whs = reinterpret_cast<float2*>(sm);       // [64 k][256 t]: taps 64..127 of this thread's two rows
  float* hbuf = sm + 2 * 64 * 256;                   // [2][NB][128]
  float* xbuf = hbuf + 2 * NB * 128;                 // [2][NB][32]   (20 used)
  float* red = xbuf + 2 * NB * 32;                   // [NB][128]
  const int t = threadIdx.x, u = t >> 1, gp = t & 1;
  const int dir = blockIdx.x & 1, g0 = (blockIdx.x >> 1) * NB;
  int S[NB], clip[NB];
  const float* fb[NB];
  size_t seg_off[NB];
  int maxS = 0;
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    clip[b] = (g0 + b < n_clips) ? __ldg(order + g0 + b) : -1;
    S[b] = 0; fb[b] = feats; seg_off[b] = 0;
    if (clip[b] >= 0) {
      const ClipDesc cd = clips[clip[b]];
      S[b] = cd.n_seg; seg_off[b] = (size_t)cd.seg_off; fb[b] = feats + (size_t)cd.seg_off * 20;
    }
    maxS = max(maxS, S[b]);
  }
  const int rowA = (2 * gp) * 128 + u, rowB = rowA + 128;
  float wrA[64], wrB[64], wiA[20], wiB[20];
  {
    const float* ra = P.w_hh + ((size_t)dir * 512 + rowA) * 128;
    const float* rb = P.w_hh + ((size_t)dir * 512 + rowB) * 128;
#pragma unroll
    for (int k = 0; k < 64; ++k) { wrA[k] = __ldg(ra + k); wrB[k] = __ldg(rb + k); }
    for (int k = 0; k < 64; ++k) whs[k * 256 + t] = make_float2(__ldg(ra + 64 + k), __ldg(rb + 64 + k));
    const float* ia = P.w_ih + ((size_t)dir * 512 + rowA) * 20;
    const float* ib = P.w_ih + ((size_t)dir * 512 + rowB) * 20;
#pragma unroll
    for (int k = 0; k < 20; ++k) { wiA[k] = __ldg(ia + k); wiB[k] = __ldg(ib + k); }
  }
  const float biasA = __ldg(P.b + dir * 512 + rowA), biasB = __ldg(P.b + dir * 512 + rowB);
  for (int i = t; i < 2 * NB * 128; i += 256) hbuf[i] = 0.f;
  for (int i = t; i < 2 * NB * 32; i += 256) xbuf[i] = 0.f;
  float cst[NB], hl[NB];
#pragma unroll
  for (int b = 0; b < NB; ++b) { cst[b] = 0.f; hl[b] = 0.f; }
  __syncthreads();
  // x of step 0: thread t < NB * 32 loads element (b = t >> 5, k = t & 31)
  const int xb_ = t >> 5, xk_ = t & 31;
  if (t < NB * 32 && xk_ < 20) {
    int Sb = 0; const float* f = feats;
#pragma unroll
    for (int b = 0; b < NB; ++b) if (b == xb_) { Sb = S[b]; f = fb[b]; }
    if (Sb > 0) xbuf[xb_ * 32 + xk_] = __ldg(f + (size_t)(dir ? Sb - 1 : 0) * 20 + xk_);
  }
  __syncthreads();

  for (int step = 0; step < maxS; ++step) {
    const float* h = hbuf + (step & 1) * NB * 128;
    const float* xt = xbuf + (step & 1) * NB * 32;
    float xnext = 0.f;
    bool xload = false;
    if (t < NB * 32 && xk_ < 20) {
      int Sb = 0; const float* f = feats;
#pragma unroll
      for (int b = 0; b < NB; ++b) if (b == xb_) { Sb = S[b]; f = fb[b]; }
      if (step + 1 < Sb) { xnext = __ldg(f + (size_t)(dir ? Sb - 2 - step : step + 1) * 20 + xk_); xload = true; }
    }
    // every row keeps two partial sums (even / odd taps), whatever NB is: a clip's result must not depend on how many
    // clips share its CTA (alone == in a batch, bit for bit), and one 148-long dependent FMA chain per row would
    // leave the NB = 1 variant latency bound
    constexpr int PART = 2;
    float pA[NB][PART], pB[NB][PART];
#pragma unroll
    for (int b = 0; b < NB; ++b)
#pragma unroll
      for (int q = 0; q < PART; ++q) { pA[b][q] = q ? 0.f : biasA; pB[b][q] = q ? 0.f : biasB; }
#pragma unroll
    for (int k = 0; k < 20; k += 4) {
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float4 xv = *reinterpret_cast<const float4*>(xt + b * 32 + k);
        pA[b][0] = fmaf(wiA[k], xv.x, pA[b][0]); pA[b][1 % PART] = fmaf(wiA[k + 1], xv.y, pA[b][1 % PART]);
        pA[b][2 % PART] = fmaf(wiA[k + 2], xv.z, pA[b][2 % PART]); pA[b][3 % PART] = fmaf(wiA[k + 3], xv.w, pA[b][3 % PART]);
        pB[b][0] = fmaf(wiB[k], xv.x, pB[b][0]); pB[b][1 % PART] = fmaf(wiB[k + 1], xv.y, pB[b][1 % PART]);
        pB[b][2 % PART] = fmaf(wiB[k + 2], xv.z, pB[b][2 % PART]); pB[b][3 % PART] = fmaf(wiB[k + 3], xv.w, pB[b][3 % PART]);
      }
    }
#pragma unroll
    for (int k = 0; k < 64; k += 4) {
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float4 hv = *reinterpret_cast<const float4*>(h + b * 128 + k);
        pA[b][0] = fmaf(wrA[k], hv.x, pA[b][0]); pA[b][1 % PART] = fmaf(wrA[k + 1], hv.y, pA[b][1 % PART]);
        pA[b][2 % PART] = fmaf(wrA[k + 2], hv.z, pA[b][2 % PART]); pA[b][3 % PART] = fmaf(wrA[k + 3], hv.w, pA[b][3 % PART]);
        pB[b][0] = fmaf(wrB[k], hv.x, pB[b][0]); pB[b][1 % PART] = fmaf(wrB[k + 1], hv.y, pB[b][1 % PART]);
        pB[b][2 % PART] = fmaf(wrB[k + 2], hv.z, pB[b][2 % PART]); pB[b][3 % PART] = fmaf(wrB[k + 3], hv.w, pB[b][3 % PART]);
      }
    }
#pragma unroll 4
    for (int k = 0; k < 64; k += 4) {
      const float2 w0 = whs[(k) * 256 + t], w1 = whs[(k + 1) * 256 + t], w2 = whs[(k + 2) * 256 + t], w3 = whs[(k + 3) * 256 + t];
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float4 hv = *reinterpret_cast<const float4*>(h + b * 128 + 64 + k);
        pA[b][0] = fmaf(w0.x, hv.x, pA[b][0]); pA[b][1 % PART] = fmaf(w1.x, hv.y, pA[b][1 % PART]);
        pA[b][2 % PART] = fmaf(w2.x, hv.z, pA[b][2 % PART]); pA[b][3 % PART] = fmaf(w3.x, hv.w, pA[b][3 % PART]);
        pB[b][0] = fmaf(w0.y, hv.x, pB[b][0]); pB[b][1 % PART] = fmaf(w1.y, hv.y, pB[b][1 % PART]);
        pB[b][2 % PART] = fmaf(w2.y, hv.z, pB[b][2 % PART]); pB[b][3 % PART] = fmaf(w3.y, hv.w, pB[b][3 % PART]);
      }
    }
    float aA[NB], aB[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      if (PART == 4) { aA[b] = (pA[b][0] + pA[b][1 % PART]) + (pA[b][2 % PART] + pA[b][3 % PART]); aB[b] = (pB[b][0] + pB[b][1 % PART]) + (pB[b][2 % PART] + pB[b][3 % PART]); }
      else if (PART == 2) { aA[b] = pA[b][0] + pA[b][1 % PART]; aB[b] = pB[b][0] + pB[b][1 % PART]; }
      else { aA[b] = pA[b][0]; aB[b] = pB[b][0]; }
    }
    float* hn = hbuf + ((step + 1) & 1) * NB * 128;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      // gp == 0: (aA, aB) = pre-activations of (i, f); gp == 1: of (g, o)
      const float actA = gp ? tanhf(aA[b]) : 1.0f / (1.0f + expf(-aA[b]));
      const float actB = 1.0f / (1.0f + expf(-aB[b]));
      const float pA = __shfl_xor_sync(0xffffffffu, actA, 1), pB = __shfl_xor_sync(0xffffffffu, actB, 1);
      const float ig = gp ? pA : actA, fg = gp ? pB : actB, gg = gp ? actA : pA, og = gp ? actB : pB;
      if (step < S[b]) {                       // warp-uniform: S[b] is the same for every thread
        cst[b] = fmaf(fg, cst[b], ig * gg);
        hl[b] = og * tanhf(cst[b]);
        if (gp == 0) {
          hn[b * 128 + u] = hl[b];
          if (td_out) td_out[(seg_off[b] + (size_t)(dir ? S[b] - 1 - step : step)) * 256 + dir * 128 + u] = hl[b];
        }
      } else if (gp == 0) {
        hn[b * 128 + u] = hl[b];               // finished sequence: state carried along unchanged
      }
    }
    if (xload) xbuf[((step + 1) & 1) * NB * 32 + xb_ * 32 + xk_] = xnext;
    __syncthreads();
  }
  // PoolLastStepBi: this direction's final hidden state . w_pool half (lib:1107-1115)
  if (gp == 0) {
    const float w = P.w_pool ? __ldg(P.w_pool + dir * 128 + u) : 0.f;      // (other pooling modes read td_out instead)
#pragma unroll
    for (int b = 0; b < NB; ++b) red[b * 128 + u] = hl[b] * w;
  }
  __syncthreads();
  if (t < 32 * NB) {
    const int b = t >> 5, lane = t & 31;
    float v = red[b * 128 + lane] + red[b * 128 + lane + 32] + red[b * 128 + lane + 64] + red[b * 128 + lane + 96];
    v = warp_sum(v);
    int cb = -1;
#pragma unroll
    for (int bb = 0; bb < NB; ++bb) if (bb == b) cb = clip[bb];
    if (lane == 0 && cb >= 0) partial[cb * 2 + dir] = v;      // clips without segments: 0 (lastbi_final writes NaN for them)
  }
}

__global__ void lastbi_final_kernel(const float* __restrict__ partial, const ClipDesc* __restrict__ clips,
                                    float bias, float* __restrict__ scores, int n_clips) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_clips) return;
  scores[c] = (clips[c].n_seg > 0) ? (partial[2 * c] + partial[2 * c + 1]) + bias
                                   : __int_as_float(0x7fc00000);
}

// ---------------------------------------------------------------------------------------
// One layer of a stacked LSTM of any accepted shape (checkpoints trained with other td_lstm_h / td_lstm_num_layers /
// td_lstm_bidirectional / cnn_fc_out_h, reference lib:925-943).  The input projection gx = x W_ih^T + b of every step and
// direction is one tile GEMM before this launch, so a step is the recurrence alone: pre = gx[t] + W_hh h.
// A direction's 4H gate rows are split over C = H / 64 CTAs of a thread-block cluster for H = 192 / 256 (W_hh is 576 KB /
// 1 MB in fp32) and held by one CTA (C = 1) for H <= 128.  Each CTA owns U = H / C hidden units with 2U threads:
// thread t owns unit u = t >> 1 and the gate pair gp = t & 1 ((i, f) or (g, o)), i.e. two rows of W_hh, of which the
// first min(H, 64) taps live in registers and the rest in shared memory, like lstm_batched_kernel.  NB sequences of one
// direction advance in lock step (group g = clips order[NB g .. NB g + NB)); a finished sequence keeps its state.
// Each CTA holds the whole h of the step (double buffered): with C > 1 every CTA stores its U new values into every CTA's
// next buffer through distributed shared memory, and one cluster barrier (release / acquire) ends the step.
// gx of the next step is loaded while the current step computes.  Every row keeps two partial sums (even / odd taps)
// whatever NB is, so a clip's result does not depend on NB or on the clips that share its CTA.
__device__ __forceinline__ unsigned cluster_ctarank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_barrier() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// store v into the shared-memory word `local` (a shared-window address of this CTA's layout) of cluster CTA `rank`
__device__ __forceinline__ void st_cluster(unsigned local, unsigned rank, float v) {
  unsigned remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(rank));
  asm volatile("st.shared::cluster.f32 [%0], %1;" :: "r"(remote), "f"(v) : "memory");
}

template <int H, int NB, int C>
struct LstmLayerShape {
  static constexpr int U = H / C;                    // hidden units per CTA
  static constexpr int T = 2 * U;                    // threads
  static constexpr int KR = H < 64 ? H : 64;         // taps per row in registers
  static constexpr int KS = H - KR;                  // taps per row in shared memory
  static constexpr int kSmemBytes = (KS * T * 2 + 2 * NB * H) * 4;
  static_assert(H % (4 * C) == 0 && KR % 4 == 0 && KS % 4 == 0, "shape");
};

template <int H, int NB, int C>
__global__ void __launch_bounds__(LstmLayerShape<H, NB, C>::T, 1)
lstm_layer_kernel(const ClipDesc* __restrict__ clips, const int* __restrict__ order, int n_clips, LstmLayerParams P) {
  using L = LstmLayerShape<H, NB, C>;
  extern __shared__ __align__(16) float sm[];
  float2* whs = reinterpret_cast<float2*>(sm);       // [KS k][T t]: taps KR.. of this thread's two rows
  float* hbuf = sm + L::KS * L::T * 2;               // [2][NB][H]
  const int t = threadIdx.x, u = t >> 1, gp = t & 1;
  const unsigned rank = C > 1 ? cluster_ctarank() : 0;
  const int gu = (int)rank * L::U + u;               // this thread's hidden unit
  const int dir = blockIdx.y, g0 = blockIdx.z * NB;
  int S[NB];
  size_t seg_off[NB];
  int maxS = 0;
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    const int clip = (g0 + b < n_clips) ? __ldg(order + g0 + b) : -1;
    S[b] = 0; seg_off[b] = 0;
    if (clip >= 0) { const ClipDesc cd = clips[clip]; S[b] = cd.n_seg; seg_off[b] = (size_t)cd.seg_off; }
    maxS = max(maxS, S[b]);
  }
  const int rowA = (2 * gp) * H + gu, rowB = rowA + H;
  float wrA[L::KR], wrB[L::KR];
  {
    const float* ra = P.w_hh + ((size_t)dir * 4 * H + rowA) * H;
    const float* rb = P.w_hh + ((size_t)dir * 4 * H + rowB) * H;
#pragma unroll
    for (int k = 0; k < L::KR; ++k) { wrA[k] = __ldg(ra + k); wrB[k] = __ldg(rb + k); }
    for (int k = 0; k < L::KS; ++k) whs[k * L::T + t] = make_float2(__ldg(ra + L::KR + k), __ldg(rb + L::KR + k));
  }
  for (int i = t; i < 2 * NB * H; i += L::T) hbuf[i] = 0.f;
  const float* gxd = P.gx + (size_t)dir * 4 * H;
  // gx of (sequence b, step) for this thread's two rows
  auto gx_row = [&](int b, int step) { return gxd + (seg_off[b] + (size_t)(dir ? S[b] - 1 - step : step)) * P.ldg; };
  float gA[NB], gB[NB], cst[NB], hl[NB];
#pragma unroll
  for (int b = 0; b < NB; ++b) {
    cst[b] = 0.f; hl[b] = 0.f; gA[b] = 0.f; gB[b] = 0.f;
    if (S[b] > 0) { gA[b] = __ldg(gx_row(b, 0) + rowA); gB[b] = __ldg(gx_row(b, 0) + rowB); }
  }
  if (C > 1) cluster_barrier(); else __syncthreads();        // every CTA's h buffers are cleared before anyone stores

  for (int step = 0; step < maxS; ++step) {
    const float* h = hbuf + (step & 1) * NB * H;
    float nA[NB], nB[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      nA[b] = 0.f; nB[b] = 0.f;
      if (step + 1 < S[b]) { nA[b] = __ldg(gx_row(b, step + 1) + rowA); nB[b] = __ldg(gx_row(b, step + 1) + rowB); }
    }
    float pA[NB][2], pB[NB][2];
#pragma unroll
    for (int b = 0; b < NB; ++b) { pA[b][0] = gA[b]; pA[b][1] = 0.f; pB[b][0] = gB[b]; pB[b][1] = 0.f; }
#pragma unroll
    for (int k = 0; k < L::KR; k += 4) {
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float4 hv = *reinterpret_cast<const float4*>(h + b * H + k);
        pA[b][0] = fmaf(wrA[k], hv.x, pA[b][0]); pA[b][1] = fmaf(wrA[k + 1], hv.y, pA[b][1]);
        pA[b][0] = fmaf(wrA[k + 2], hv.z, pA[b][0]); pA[b][1] = fmaf(wrA[k + 3], hv.w, pA[b][1]);
        pB[b][0] = fmaf(wrB[k], hv.x, pB[b][0]); pB[b][1] = fmaf(wrB[k + 1], hv.y, pB[b][1]);
        pB[b][0] = fmaf(wrB[k + 2], hv.z, pB[b][0]); pB[b][1] = fmaf(wrB[k + 3], hv.w, pB[b][1]);
      }
    }
#pragma unroll 4
    for (int k = 0; k < L::KS; k += 4) {
      const float2 w0 = whs[k * L::T + t], w1 = whs[(k + 1) * L::T + t], w2 = whs[(k + 2) * L::T + t],
                   w3 = whs[(k + 3) * L::T + t];
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float4 hv = *reinterpret_cast<const float4*>(h + b * H + L::KR + k);
        pA[b][0] = fmaf(w0.x, hv.x, pA[b][0]); pA[b][1] = fmaf(w1.x, hv.y, pA[b][1]);
        pA[b][0] = fmaf(w2.x, hv.z, pA[b][0]); pA[b][1] = fmaf(w3.x, hv.w, pA[b][1]);
        pB[b][0] = fmaf(w0.y, hv.x, pB[b][0]); pB[b][1] = fmaf(w1.y, hv.y, pB[b][1]);
        pB[b][0] = fmaf(w2.y, hv.z, pB[b][0]); pB[b][1] = fmaf(w3.y, hv.w, pB[b][1]);
      }
    }
    float* hn = hbuf + ((step + 1) & 1) * NB * H;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const float aA = pA[b][0] + pA[b][1], aB = pB[b][0] + pB[b][1];
      // gp == 0: (aA, aB) = pre-activations of (i, f); gp == 1: of (g, o)
      const float actA = gp ? tanhf(aA) : 1.0f / (1.0f + expf(-aA));
      const float actB = 1.0f / (1.0f + expf(-aB));
      const float qA = __shfl_xor_sync(0xffffffffu, actA, 1), qB = __shfl_xor_sync(0xffffffffu, actB, 1);
      const float ig = gp ? qA : actA, fg = gp ? qB : actB, gg = gp ? actA : qA, og = gp ? actB : qB;
      if (step < S[b]) {                       // uniform over the CTA: S[b] is the same for every thread
        cst[b] = fmaf(fg, cst[b], ig * gg);
        hl[b] = og * tanhf(cst[b]);
        if (gp == 0) P.out[(seg_off[b] + (size_t)(dir ? S[b] - 1 - step : step)) * P.ldo + dir * H + gu] = hl[b];
      }
      if (gp == 0) {                           // (a finished sequence: its state carried along unchanged)
        if (C == 1) {
          hn[b * H + gu] = hl[b];
        } else {
          const unsigned a = (unsigned)__cvta_generic_to_shared(hn + b * H + gu);
#pragma unroll
          for (int r = 0; r < C; ++r) st_cluster(a, r, hl[b]);
        }
      }
      gA[b] = nA[b]; gB[b] = nB[b];
    }
    if (C > 1) cluster_barrier(); else __syncthreads();
  }
}

// PoolAttFF logits behind an LSTM: one warp per (row, head), logit = w2_h . hid[row][h 128 ..] + b2_h
__global__ void att_logits_kernel(const float* __restrict__ hid, const float* __restrict__ w2, const float* __restrict__ b2,
                                  int n_heads, int n_rows, float* __restrict__ logits) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (wid >= n_rows * n_heads) return;
  const int row = wid / n_heads, h = wid - row * n_heads;
  const float4 x = __ldg(reinterpret_cast<const float4*>(hid + ((size_t)row * n_heads + h) * 128) + lane);
  const float4 w = __ldg(reinterpret_cast<const float4*>(w2 + h * 128) + lane);
  float a = fmaf(x.x, w.x, fmaf(x.y, w.y, fmaf(x.z, w.z, x.w * w.w)));
  a = warp_sum(a);
  if (lane == 0) logits[wid] = a + __ldg(b2 + h);
}

// ---------------------------------------------------------------------------------------
// Pooling over wide rows: the framewise rows of a checkpoint without a time-dependency model (td = 'skip'), D real
// columns (up to 4096) at a row stride of ldx floats, every pooling module but PoolLastStepBi, 1 or 5 heads.
// grid = (column slab of kPoolWideSlab, clip), kPoolWarps warps: lane l of warp g owns the slab's columns 4l..4l+3 over
// the clip's steps t = g, g + kPoolWarps, .., one accumulator per head and column updated in step order, so x is read
// from HBM once for every head.  PoolAtt / PoolAttFF: the softmax numerators exp(logit - max) of the precomputed logits
// [n_seg][NH] are staged kPoolChunk steps at a time; every slab CTA forms the clip's max and sum in the same fixed order.
// The warps' sums are added in warp order, dotted with each head's Linear over the slab's columns and written to
// partial[clip][slab][head]; pool_wide_finish_kernel adds the slabs in slab order plus the bias.  Every sum's order
// depends only on D and the clip's own steps (not on the batch or the pass split); columns >= D are never read.
constexpr int kPoolWarps = 4, kPoolChunk = 256;
enum { PW_ATT = 0, PW_AVG = 1, PW_MAX = 2, PW_LAST = 3 };
static_assert(kPoolWideSlab == 128, "one float4 of columns per lane");

__device__ __forceinline__ float4 ld_cols(const float* __restrict__ p, int nv) {      // the first nv (<= 4) of 4 columns
  if (nv >= 4) return __ldg(reinterpret_cast<const float4*>(p));
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (nv > 0) v.x = __ldg(p);
  if (nv > 1) v.y = __ldg(p + 1);
  if (nv > 2) v.z = __ldg(p + 2);
  return v;
}

template <int NH, int MODE>
__global__ void __launch_bounds__(kPoolWarps * 32)
pool_wide_kernel(const float* __restrict__ x, int D, int ldx, const float* __restrict__ logits,
                 const ClipDesc* __restrict__ clips, const float* __restrict__ w3, float* __restrict__ partial) {
  constexpr int NA = MODE == PW_ATT ? NH : 1;           // accumulators per column
  __shared__ float pn[MODE == PW_ATT ? NH * kPoolChunk : 1];
  __shared__ float red[kPoolWarps][NA][kPoolWideSlab];
  __shared__ float wred[kPoolWarps][NH];
  __shared__ float mx[NH], sum[NH];
  const ClipDesc cd = clips[blockIdx.y];
  const int S = cd.n_seg;
  if (S <= 0) return;                                   // (pool_wide_finish_kernel writes NaN)
  const int tid = threadIdx.x, lane = tid & 31, g = tid >> 5, c0 = blockIdx.x * kPoolWideSlab;
  const float* lg = logits + (size_t)cd.seg_off * NH;
  if constexpr (MODE == PW_ATT) {
    for (int h = 0; h < NH; ++h) {
      float m = -INFINITY;
      for (int t = tid; t < S; t += kPoolWarps * 32) m = fmaxf(m, __ldg(lg + (size_t)t * NH + h));
      m = warp_max(m);
      if (lane == 0) wred[g][h] = m;
    }
    __syncthreads();
    if (tid < NH) {
      float m = wred[0][tid];
      for (int w = 1; w < kPoolWarps; ++w) m = fmaxf(m, wred[w][tid]);
      mx[tid] = m;
    }
    __syncthreads();
    for (int h = 0; h < NH; ++h) {
      float s = 0.f;
      for (int t = tid; t < S; t += kPoolWarps * 32) s += expf(__ldg(lg + (size_t)t * NH + h) - mx[h]);
      s = warp_sum(s);
      if (lane == 0) wred[g][h] = s;
    }
    __syncthreads();
    if (tid < NH) {
      float s = wred[0][tid];
      for (int w = 1; w < kPoolWarps; ++w) s += wred[w][tid];
      sum[tid] = s;
    }
  }
  if constexpr (MODE != PW_LAST) {
    const int nv = D - (c0 + 4 * lane);
    const float* xb = x + (size_t)cd.seg_off * ldx + c0 + 4 * lane;
    float acc[NA][4];
#pragma unroll
    for (int a = 0; a < NA; ++a)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[a][i] = MODE == PW_MAX ? -INFINITY : 0.f;
    auto step = [&](const float4 v, int tc) {           // tc: the step's index in the chunk
      const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int a = 0; a < NA; ++a) {
        const float p = MODE == PW_ATT ? pn[a * kPoolChunk + tc] : 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i)
          acc[a][i] = MODE == PW_ATT ? fmaf(p, e[i], acc[a][i]) : MODE == PW_MAX ? fmaxf(acc[a][i], e[i]) : acc[a][i] + e[i];
      }
    };
    for (int t0 = 0; t0 < S; t0 += kPoolChunk) {
      const int n = min(kPoolChunk, S - t0);
      if constexpr (MODE == PW_ATT) {
        __syncthreads();                                // (the previous chunk's numerators consumed; mx published)
        for (int i = tid; i < n * NH; i += kPoolWarps * 32) {
          const int t = i / NH, h = i - t * NH;
          pn[h * kPoolChunk + t] = expf(__ldg(lg + (size_t)(t0 + t) * NH + h) - mx[h]);
        }
        __syncthreads();
      }
      if (nv > 0) {
        int t = g;
        for (; t + 7 * kPoolWarps < n; t += 8 * kPoolWarps) {      // eight steps in flight
          float4 v[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) v[u] = ld_cols(xb + (size_t)(t0 + t + u * kPoolWarps) * ldx, nv);
#pragma unroll
          for (int u = 0; u < 8; ++u) step(v[u], t + u * kPoolWarps);
        }
        for (; t < n; t += kPoolWarps) step(ld_cols(xb + (size_t)(t0 + t) * ldx, nv), t);
      }
    }
#pragma unroll
    for (int a = 0; a < NA; ++a)
#pragma unroll
      for (int i = 0; i < 4; ++i) red[g][a][4 * lane + i] = acc[a][i];
  }
  __syncthreads();
  // thread tid: column c0 + tid of the slab, the warps' sums in warp order, then each head's Linear
  const int c = c0 + tid;
  float last = 0.f;
  if constexpr (MODE == PW_LAST) last = c < D ? __ldg(x + ((size_t)cd.seg_off + S - 1) * ldx + c) : 0.f;
#pragma unroll
  for (int h = 0; h < NH; ++h) {
    float pooled;
    if constexpr (MODE == PW_LAST) {
      pooled = last;
    } else {
      const int a = MODE == PW_ATT ? h : 0;
      pooled = red[0][a][tid];
      for (int w = 1; w < kPoolWarps; ++w) pooled = MODE == PW_MAX ? fmaxf(pooled, red[w][a][tid]) : pooled + red[w][a][tid];
      if (MODE == PW_ATT) pooled = pooled / sum[h];
      if (MODE == PW_AVG) pooled = pooled / (float)S;
    }
    const float v = warp_sum(c < D ? pooled * __ldg(w3 + (size_t)h * D + c) : 0.f);
    if (lane == 0) wred[g][h] = v;
  }
  __syncthreads();
  if (tid < NH) {
    float s = wred[0][tid];
    for (int w = 1; w < kPoolWarps; ++w) s += wred[w][tid];
    partial[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * NH + tid] = s;
  }
}

// scores[clip][h] = sum over the slabs in slab order + b3[h]; NaN for a clip without segments
__global__ void pool_wide_finish_kernel(const float* __restrict__ partial, int n_slabs, const ClipDesc* __restrict__ clips,
                                        int n_clips, int n_heads, const float* __restrict__ b3, float* __restrict__ scores) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_clips * n_heads) return;
  const int clip = i / n_heads, h = i - clip * n_heads;
  if (clips[clip].n_seg <= 0) { scores[i] = __int_as_float(0x7fc00000); return; }
  float s = 0.f;
  for (int k = 0; k < n_slabs; ++k) s += partial[((size_t)clip * n_slabs + k) * n_heads + h];
  scores[i] = s + __ldg(b3 + h);
}

// PoolAtt's logits over wide rows, one warp per row: logits[row][h] = a1_h . x[row][0..D) + a1b_h (lanes over the columns)
template <int NH>
__global__ void pool_att_logits_kernel(const float* __restrict__ x, int D, int ldx, const float* __restrict__ a1,
                                       const float* __restrict__ a1b, int n_rows, float* __restrict__ logits) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n_rows) return;
  const float* xr = x + (size_t)row * ldx;
  float a[NH];
#pragma unroll
  for (int h = 0; h < NH; ++h) a[h] = 0.f;
  for (int k = lane; k < D; k += 32) {
    const float v = __ldg(xr + k);
#pragma unroll
    for (int h = 0; h < NH; ++h) a[h] = fmaf(v, __ldg(a1 + (size_t)h * D + k), a[h]);
  }
#pragma unroll
  for (int h = 0; h < NH; ++h) {
    const float s = warp_sum(a[h]);
    if (lane == 0) logits[row * NH + h] = s + __ldg(a1b + h);
  }
}

// ---------------------------------------------------------------------------------------
// Per-segment scores and pooling weights (nisqa_predict_device_batch_segments).  Segment t's score under head h is the
// pooling module applied to the one-step sequence x[t:t+1]: its last Linear, w3_h . x_t + b3_h, for every module.  Its
// weight is the module's softmax weight of step t (PoolAtt, PoolAttFF), 1 / S (PoolAvg), [t == S - 1] (PoolLastStep)
// or NaN (PoolMax, PoolLastStepBi: no weight per step reproduces the clip's score).  One CTA per clip, its warps over
// the clip's segments, lanes over the columns.  Sweep 1 writes the scores and parks the attention logits in the
// weight rows while it keeps each warp's running max and rescaled sum; sweep 2 turns the logits into weights.  Clips
// with row_off < 0 (skipped, or NISQA_DE reference clips) get no rows.  About n_seg n_heads D FMAs and one read of the
// rows: far too little work for the tensor cores.
constexpr int kSegWarps = 8;

// The attention softmax of a clip's steps as a running max m and a sum s rescaled to it: warp g folds the logits of
// steps g, g + kSegWarps, ... in order (softmax_fold), then softmax_merge combines the warps' (m, s) [kSegWarps][NH] in
// warp order into the clip's max and sum.  The segments and the embeddings kernels both use this arithmetic, so they
// agree on every weight.  softmax_fold returns the max before the fold: s was rescaled by exp(that - m).
__device__ __forceinline__ float softmax_fold(float& m, float& s, float l) {
  const float m0 = m, nm = fmaxf(m, l);
  s = s * expf(m - nm) + expf(l - nm);
  m = nm;
  return m0;
}
// thread h < NH: mx[h], sum[h] from the warps' wm / ws (a warp without steps has ws == 0 and adds nothing)
template <int NH>
__device__ __forceinline__ void softmax_merge(const float (*wm)[NH], const float (*ws)[NH], float* mx, float* sum) {
  if (threadIdx.x < NH) {
    const int h = threadIdx.x;
    float M = wm[0][h];
    for (int w = 1; w < kSegWarps; ++w) M = fmaxf(M, wm[w][h]);
    float tot = 0.f;
    for (int w = 0; w < kSegWarps; ++w) tot += ws[w][h] == 0.f ? 0.f : ws[w][h] * expf(wm[w][h] - M);
    mx[h] = M;
    sum[h] = tot;
  }
}

template <int NH>
__global__ void __launch_bounds__(kSegWarps * 32)
segment_scores_kernel(const float* __restrict__ x, int D, int ldx, const float* __restrict__ logits, PoolSimpleParams P,
                      int mode, const ClipDesc* __restrict__ clips, const long long* __restrict__ row_off,
                      float* __restrict__ seg_scores, float* seg_weights) {
  __shared__ float wm[kSegWarps][NH], ws[kSegWarps][NH];
  __shared__ float mx[NH], sum[NH];
  const ClipDesc cd = clips[blockIdx.x];
  const long long r0 = row_off[blockIdx.x];
  const int S = cd.n_seg;
  if (S <= 0 || r0 < 0) return;
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  const bool att = mode == 0 || mode == 1, own_logits = mode == 1 && logits == nullptr;
  float m[NH], s[NH];
#pragma unroll
  for (int h = 0; h < NH; ++h) { m[h] = -INFINITY; s[h] = 0.f; }
  for (int t = g; t < S; t += kSegWarps) {
    const float* xr = x + (size_t)(cd.seg_off + t) * ldx;
    float acc[NH], la[NH];
#pragma unroll
    for (int h = 0; h < NH; ++h) { acc[h] = 0.f; la[h] = 0.f; }
    for (int k = lane; k < D; k += 32) {
      const float v = __ldg(xr + k);
#pragma unroll
      for (int h = 0; h < NH; ++h) {
        acc[h] = fmaf(v, __ldg(P.w3 + (size_t)h * D + k), acc[h]);
        if (own_logits) la[h] = fmaf(v, __ldg(P.a1 + (size_t)h * D + k), la[h]);
      }
    }
    const long long row = r0 + t;
#pragma unroll
    for (int h = 0; h < NH; ++h) {
      const float sc = warp_sum(acc[h]) + __ldg(P.b3 + h);
      float l = 0.f;
      if (own_logits) l = warp_sum(la[h]) + __ldg(P.a1b + h);
      else if (att) l = __ldg(logits + (size_t)(cd.seg_off + t) * NH + h);
      if (lane == 0) {
        seg_scores[row * NH + h] = sc;
        if (att) seg_weights[row * NH + h] = l;
      }
      if (att) softmax_fold(m[h], s[h], l);
    }
  }
  if (att) {
    if (lane == 0)
#pragma unroll
      for (int h = 0; h < NH; ++h) { wm[g][h] = m[h]; ws[g][h] = s[h]; }
    __syncthreads();
    softmax_merge<NH>(wm, ws, mx, sum);
  }
  __syncthreads();                       // (also makes sweep 1's parked logits visible to the whole CTA)
  const float nan = __int_as_float(0x7fc00000);
  for (int i = threadIdx.x; i < S * NH; i += kSegWarps * 32) {
    const int t = i / NH, h = i - t * NH;
    float* wp = seg_weights + (r0 + t) * NH + h;
    *wp = att ? expf(*wp - mx[h]) / sum[h] : mode == 2 ? 1.f / (float)S : mode == 4 ? (t == S - 1 ? 1.f : 0.f) : nan;
  }
}

// ---------------------------------------------------------------------------------------
// Quality embeddings (nisqa_predict_device_batch_embeddings): each pooling head's pooled vector - the input of its last
// Linear - and optionally the rows the module read, both in the reference's column order (src_col[j]: the column of
// x that holds reference column j; nullptr: the same order).  PoolAtt / PoolAttFF: sum_t a_t[h] x_t with the softmax
// weights of segment_scores_kernel, formed on the fly: each warp folds its steps into a running max and rescaled sum
// (softmax_fold) and rescales its accumulators with the sum, then the warps merge (softmax_merge).  The logits are the
// ones the pooling path wrote, or a1 . x_t + a1b, formed here as the segments kernel forms them (PoolAtt over rows of
// at most 512 columns, which one CTA row covers).  PoolAvg: (sum_t x_t) / S; PoolMax: the column-wise max; PoolLastStep:
// x_{S-1}; PoolLastStepBi: the forward half of x_{S-1} and the backward half of x_0 (copies of the rows).  The modules
// without parameters write the same vector for every head.  One CTA per (clip, block of kEmbCols columns), its warps
// over the clip's steps, lanes over the columns; rows with row_off >= 0 are written as they are read.  Clips that did
// not run and NISQA_DE's reference clips (odd clips when de) get NaN vectors.  About S n_heads W FMAs and one read of
// the rows: memory-bound, plain fp32.
constexpr int kEmbCols = 128;
constexpr int kEmbPer = kEmbCols / 32;

template <int NH>
__global__ void __launch_bounds__(kSegWarps * 32)
pool_embed_kernel(const float* __restrict__ x, int W, int ldx, const int* __restrict__ src_col,
                  const float* __restrict__ logits, PoolSimpleParams P, int mode, int de, const ClipDesc* __restrict__ clips,
                  const long long* __restrict__ row_off, float* __restrict__ pooled, float* __restrict__ rows) {
  __shared__ float wm[kSegWarps][NH], ws[kSegWarps][NH];
  __shared__ float mx[NH], sum[NH];
  __shared__ float part[kSegWarps][NH][kEmbCols];
  const int clip = blockIdx.x, j0 = blockIdx.y * kEmbCols;
  const ClipDesc cd = clips[clip];
  const int S = cd.n_seg;
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5;
  float* out = pooled + (size_t)clip * NH * W;
  if (S <= 0 || (de && (clip & 1))) {
    for (int i = threadIdx.x; i < NH * kEmbCols; i += kSegWarps * 32) {
      const int h = i / kEmbCols, j = j0 + i % kEmbCols;
      if (j < W) out[(size_t)h * W + j] = __int_as_float(0x7fc00000);
    }
    return;
  }
  const long long r0 = rows ? row_off[clip] : -1;
  const bool att = mode == 0 || mode == 1, own_logits = mode == 1 && logits == nullptr, last = mode >= 4;
  int col[kEmbPer];
#pragma unroll
  for (int i = 0; i < kEmbPer; ++i) {
    const int j = j0 + lane + 32 * i;
    col[i] = j >= W ? -1 : src_col ? __ldg(src_col + j) : j;
  }
  float m[NH], s[NH], acc[NH][kEmbPer];
#pragma unroll
  for (int h = 0; h < NH; ++h) {
    m[h] = -INFINITY; s[h] = 0.f;
#pragma unroll
    for (int i = 0; i < kEmbPer; ++i) acc[h][i] = mode == 3 ? -INFINITY : 0.f;
  }
  for (int t = g; t < S; t += kSegWarps) {
    if (last && r0 < 0 && t != S - 1 && t != 0) continue;     // (the last-step modules read one or two rows)
    const float* xr = x + (size_t)(cd.seg_off + t) * ldx;
    float v[kEmbPer];
#pragma unroll
    for (int i = 0; i < kEmbPer; ++i) v[i] = col[i] >= 0 ? __ldg(xr + col[i]) : 0.f;
    if (r0 >= 0) {
      float* rr = rows + (size_t)(r0 + t) * W;
#pragma unroll
      for (int i = 0; i < kEmbPer; ++i)
        if (col[i] >= 0) rr[j0 + lane + 32 * i] = v[i];
    }
    if (att) {
      float la[NH];
#pragma unroll
      for (int h = 0; h < NH; ++h) la[h] = 0.f;
      if (own_logits)
        for (int k = lane; k < W; k += 32) {
          const float xv = __ldg(xr + k);
#pragma unroll
          for (int h = 0; h < NH; ++h) la[h] = fmaf(xv, __ldg(P.a1 + (size_t)h * W + k), la[h]);
        }
#pragma unroll
      for (int h = 0; h < NH; ++h) {
        const float l = own_logits ? warp_sum(la[h]) + __ldg(P.a1b + h) : __ldg(logits + (size_t)(cd.seg_off + t) * NH + h);
        const float m0 = softmax_fold(m[h], s[h], l);
        const float r = expf(m0 - m[h]), e = expf(l - m[h]);
#pragma unroll
        for (int i = 0; i < kEmbPer; ++i) acc[h][i] = fmaf(e, v[i], acc[h][i] * r);
      }
    } else if (mode == 2) {
#pragma unroll
      for (int i = 0; i < kEmbPer; ++i) acc[0][i] += v[i];
    } else if (mode == 3) {
#pragma unroll
      for (int i = 0; i < kEmbPer; ++i) acc[0][i] = fmaxf(acc[0][i], v[i]);
    } else {
#pragma unroll
      for (int i = 0; i < kEmbPer; ++i) {
        const int j = j0 + lane + 32 * i;
        const bool fwd = mode == 4 || j < W / 2;
        if (col[i] >= 0 && ((fwd && t == S - 1) || (!fwd && t == 0)))
#pragma unroll
          for (int h = 0; h < NH; ++h) out[(size_t)h * W + j] = v[i];
      }
    }
  }
  if (last) return;
#pragma unroll
  for (int h = 0; h < NH; ++h)
    if (att || h == 0)
#pragma unroll
      for (int i = 0; i < kEmbPer; ++i) part[g][h][lane + 32 * i] = acc[h][i];
  if (att && lane == 0)
#pragma unroll
    for (int h = 0; h < NH; ++h) { wm[g][h] = m[h]; ws[g][h] = s[h]; }
  __syncthreads();
  if (att) {
    softmax_merge<NH>(wm, ws, mx, sum);
    __syncthreads();
  }
  for (int i = threadIdx.x; i < NH * kEmbCols; i += kSegWarps * 32) {
    const int h = i / kEmbCols, c = i % kEmbCols, j = j0 + c;
    if (j >= W) continue;
    float o;
    if (att) {
      o = 0.f;
      for (int w = 0; w < kSegWarps; ++w)
        if (ws[w][h] != 0.f) o = fmaf(part[w][h][c], expf(wm[w][h] - mx[h]), o);
      o /= sum[h];
    } else if (mode == 2) {
      o = 0.f;
      for (int w = 0; w < kSegWarps; ++w) o += part[w][0][c];
      o /= (float)S;
    } else {
      o = part[0][0][c];
      for (int w = 1; w < kSegWarps; ++w) o = fmaxf(o, part[w][0][c]);
    }
    out[(size_t)h * W + j] = o;
  }
}

// ------------------------------------------------------------------ host launchers
constexpr int kRowSmem20 = (kRows * kXS + 64 * 20) * 4;

void launch_fc20(cudaStream_t st, const float* feats, const float* WT, const float* b, float* out, int n_rows) {
  linear_rows_kernel<20><<<(n_rows + kRows - 1) / kRows, kRows, kRowSmem20, st>>>(feats, 768, WT, b, out, n_rows);
}
void launch_pool_final(cudaStream_t st, const float* x, int D, int ldx, const float* logits, const ClipDesc* clips, int n_clips,
                       const PoolHeadParams& P, int n_heads, int max_seg, float* scores) {
  const int smem = n_heads * std::max(max_seg, 1) * 4;          // <= 5 x 1300 x 4 bytes at ms_max_segments = 1300
  if (smem > 40 * 1024) cudaFuncSetAttribute(pool_final_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  pool_final_kernel<<<n_clips, 64 * n_heads, smem, st>>>(x, logits, clips, P, n_heads, std::max(max_seg, 1), D, ldx, scores);
}
void launch_lstm(cudaStream_t st, const float* feats20, const ClipDesc* clips, int n_clips,
                 const LstmParams& P, float* td_out, float* partial, float pool_bias, float* scores) {
  static unsigned long long cfg = 0;
  const int smem = kLstmSmemFloats * 4;
  if (first_launch_on_device(cfg)) { cudaFuncSetAttribute(lstm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); }
  lstm_kernel<<<2 * n_clips, 512, smem, st>>>(feats20, clips, P, td_out, partial);
  if (scores) lastbi_final_kernel<<<(n_clips + 127) / 128, 128, 0, st>>>(partial, clips, pool_bias, scores, n_clips);
}

template <int D>
void pool_simple_instance(cudaStream_t st, const float* x, int ldx, const ClipDesc* clips, int n_clips, int mode,
                          const PoolSimpleParams& P, int n_heads, int smem, float* scores) {
  if (smem > 48 * 1024) cudaFuncSetAttribute(pool_simple_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  pool_simple_kernel<D><<<n_clips, D, smem, st>>>(x, ldx, clips, mode, P, n_heads, scores);
}
void launch_pool_simple(cudaStream_t st, const float* x, int D, int ldx, const ClipDesc* clips, int n_clips, int mode,
                        const PoolSimpleParams& P, int n_heads, int max_seg, float* scores) {
  const int smem = (mode == 1 ? max_seg : 0) * 4 + 16;
  switch (D) {
    case 32: pool_simple_instance<32>(st, x, ldx, clips, n_clips, mode, P, n_heads, smem, scores); break;
    case 64: pool_simple_instance<64>(st, x, ldx, clips, n_clips, mode, P, n_heads, smem, scores); break;
    case 96: pool_simple_instance<96>(st, x, ldx, clips, n_clips, mode, P, n_heads, smem, scores); break;
    case 128: pool_simple_instance<128>(st, x, ldx, clips, n_clips, mode, P, n_heads, smem, scores); break;
    case 192: pool_simple_instance<192>(st, x, ldx, clips, n_clips, mode, P, n_heads, smem, scores); break;
    case 256: pool_simple_instance<256>(st, x, ldx, clips, n_clips, mode, P, n_heads, smem, scores); break;
    case 384: pool_simple_instance<384>(st, x, ldx, clips, n_clips, mode, P, n_heads, smem, scores); break;
    case 512: pool_simple_instance<512>(st, x, ldx, clips, n_clips, mode, P, n_heads, smem, scores); break;
  }
}

template <int NB> constexpr int lstm_batched_smem() { return (2 * 64 * 256 + 2 * NB * 128 + 2 * NB * 32 + NB * 128) * 4; }

// `order`: device array of the pass's clip indices sorted by decreasing n_seg (host-built, run_pass); the batch
// width follows the number of sequences per SM: n_SM x NB sequences per direction pair of CTAs in one wave
void launch_lstm_batched(cudaStream_t st, const float* feats20, const ClipDesc* clips, const int* order, int n_clips,
                         const LstmParams& P, float* td_out, float* partial, float pool_bias, float* scores) {
  static unsigned long long cfg = 0;
  static int n_sm = 132;
  if (first_launch_on_device(cfg)) {
    cudaFuncSetAttribute(lstm_batched_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, lstm_batched_smem<1>());
    cudaFuncSetAttribute(lstm_batched_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, lstm_batched_smem<2>());
    cudaFuncSetAttribute(lstm_batched_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, lstm_batched_smem<4>());
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  }
  const int seqs = 2 * n_clips;
  if (seqs <= n_sm)
    lstm_batched_kernel<1><<<2 * n_clips, 256, lstm_batched_smem<1>(), st>>>(feats20, clips, order, n_clips, P, td_out, partial);
  else if (seqs <= 2 * n_sm)
    lstm_batched_kernel<2><<<2 * ((n_clips + 1) / 2), 256, lstm_batched_smem<2>(), st>>>(feats20, clips, order, n_clips, P, td_out, partial);
  else
    lstm_batched_kernel<4><<<2 * ((n_clips + 3) / 4), 256, lstm_batched_smem<4>(), st>>>(feats20, clips, order, n_clips, P, td_out, partial);
  if (scores) lastbi_final_kernel<<<(n_clips + 127) / 128, 128, 0, st>>>(partial, clips, pool_bias, scores, n_clips);
}

template <int H, int C>
void lstm_layer_instance(cudaStream_t st, int dirs, const ClipDesc* clips, const int* order, int n_clips, const LstmLayerParams& P) {
  static unsigned long long cfg = 0;
  static int n_sm = 132;
  if (first_launch_on_device(cfg)) {
    cudaFuncSetAttribute(lstm_layer_kernel<H, 1, C>, cudaFuncAttributeMaxDynamicSharedMemorySize, LstmLayerShape<H, 1, C>::kSmemBytes);
    cudaFuncSetAttribute(lstm_layer_kernel<H, 2, C>, cudaFuncAttributeMaxDynamicSharedMemorySize, LstmLayerShape<H, 2, C>::kSmemBytes);
    cudaFuncSetAttribute(lstm_layer_kernel<H, 4, C>, cudaFuncAttributeMaxDynamicSharedMemorySize, LstmLayerShape<H, 4, C>::kSmemBytes);
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  }
  // the fewest sequences per CTA that still put every CTA of the launch on the chip at once
  const int ctas = dirs * n_clips * C;
  const int nb = ctas <= n_sm ? 1 : ctas <= 2 * n_sm ? 2 : 4;
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3(C, dirs, (n_clips + nb - 1) / nb);
  lc.blockDim = dim3(LstmLayerShape<H, 1, C>::T);
  lc.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = C; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  lc.attrs = attr;
  lc.numAttrs = C > 1 ? 1 : 0;
  if (nb == 1) { lc.dynamicSmemBytes = LstmLayerShape<H, 1, C>::kSmemBytes; cudaLaunchKernelEx(&lc, lstm_layer_kernel<H, 1, C>, clips, order, n_clips, P); }
  else if (nb == 2) { lc.dynamicSmemBytes = LstmLayerShape<H, 2, C>::kSmemBytes; cudaLaunchKernelEx(&lc, lstm_layer_kernel<H, 2, C>, clips, order, n_clips, P); }
  else { lc.dynamicSmemBytes = LstmLayerShape<H, 4, C>::kSmemBytes; cudaLaunchKernelEx(&lc, lstm_layer_kernel<H, 4, C>, clips, order, n_clips, P); }
}
bool lstm_layer_supported(int H) { return H == 32 || H == 64 || H == 96 || H == 128 || H == 192 || H == 256; }
void launch_lstm_layer(cudaStream_t st, int H, int dirs, const ClipDesc* clips, const int* order, int n_clips,
                       const LstmLayerParams& P) {
  switch (H) {
    case 32: lstm_layer_instance<32, 1>(st, dirs, clips, order, n_clips, P); break;
    case 64: lstm_layer_instance<64, 1>(st, dirs, clips, order, n_clips, P); break;
    case 96: lstm_layer_instance<96, 1>(st, dirs, clips, order, n_clips, P); break;
    case 128: lstm_layer_instance<128, 1>(st, dirs, clips, order, n_clips, P); break;
    case 192: lstm_layer_instance<192, 3>(st, dirs, clips, order, n_clips, P); break;
    case 256: lstm_layer_instance<256, 4>(st, dirs, clips, order, n_clips, P); break;
  }
}
void launch_att_logits(cudaStream_t st, const float* hid, const float* w2, const float* b2, int n_heads, int n_rows,
                       float* logits) {
  const long long warps = (long long)n_rows * n_heads;
  if (warps > 0) att_logits_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(hid, w2, b2, n_heads, n_rows, logits);
}

template <int NH>
void pool_wide_instance(cudaStream_t st, const float* x, int D, int ldx, int mode, const PoolSimpleParams& P, float* logits,
                        int n_seg, const ClipDesc* clips, int n_clips, float* partial, float* scores) {
  const int slabs = pool_wide_slabs(D);
  if (mode == 1 && n_seg > 0)
    pool_att_logits_kernel<NH><<<(unsigned)(((long long)n_seg + 7) / 8), 256, 0, st>>>(x, D, ldx, P.a1, P.a1b, n_seg, logits);
  const dim3 grid(slabs, n_clips), block(kPoolWarps * 32);
  if (mode <= 1) pool_wide_kernel<NH, PW_ATT><<<grid, block, 0, st>>>(x, D, ldx, logits, clips, P.w3, partial);
  else if (mode == 2) pool_wide_kernel<NH, PW_AVG><<<grid, block, 0, st>>>(x, D, ldx, logits, clips, P.w3, partial);
  else if (mode == 3) pool_wide_kernel<NH, PW_MAX><<<grid, block, 0, st>>>(x, D, ldx, logits, clips, P.w3, partial);
  else pool_wide_kernel<NH, PW_LAST><<<grid, block, 0, st>>>(x, D, ldx, logits, clips, P.w3, partial);
  pool_wide_finish_kernel<<<(n_clips * NH + 127) / 128, 128, 0, st>>>(partial, slabs, clips, n_clips, NH, P.b3, scores);
}
void launch_pool_wide(cudaStream_t st, const float* x, int D, int ldx, int mode, const PoolSimpleParams& P, int n_heads,
                      float* logits, int n_seg, const ClipDesc* clips, int n_clips, float* partial, float* scores) {
  if (n_clips <= 0) return;
  if (n_heads == 5) pool_wide_instance<5>(st, x, D, ldx, mode, P, logits, n_seg, clips, n_clips, partial, scores);
  else pool_wide_instance<1>(st, x, D, ldx, mode, P, logits, n_seg, clips, n_clips, partial, scores);
}

void launch_segment_scores(cudaStream_t st, const float* x, int D, int ldx, const float* logits, const PoolSimpleParams& P,
                           int n_heads, int mode, const ClipDesc* clips, int n_clips, const long long* row_off,
                           float* seg_scores, float* seg_weights) {
  if (n_clips <= 0) return;
  if (n_heads == 5)
    segment_scores_kernel<5><<<n_clips, kSegWarps * 32, 0, st>>>(x, D, ldx, logits, P, mode, clips, row_off, seg_scores, seg_weights);
  else
    segment_scores_kernel<1><<<n_clips, kSegWarps * 32, 0, st>>>(x, D, ldx, logits, P, mode, clips, row_off, seg_scores, seg_weights);
}

void launch_pool_embed(cudaStream_t st, const float* x, int W, int ldx, const int* src_col, const float* logits,
                       const PoolSimpleParams& P, int n_heads, int mode, int de, const ClipDesc* clips, int n_clips,
                       const long long* row_off, float* pooled, float* rows) {
  if (n_clips <= 0) return;
  const dim3 grid(n_clips, (W + kEmbCols - 1) / kEmbCols);
  if (n_heads == 5)
    pool_embed_kernel<5><<<grid, kSegWarps * 32, 0, st>>>(x, W, ldx, src_col, logits, P, mode, de, clips, row_off, pooled, rows);
  else
    pool_embed_kernel<1><<<grid, kSegWarps * 32, 0, st>>>(x, W, ldx, src_col, logits, P, mode, de, clips, row_off, pooled, rows);
}

}  // namespace nisqa

// td_tiled.cu - time-dependency block + attention-pool logits of the adapt architecture as register-tiled fp32
// GEMMs (round 2; replaces the one-thread-per-row kernels of td.cu, which ran at 6 % occupancy), for self-attention
// widths D = 64 NC, NC = 1..4 (one template instance each) and any feed-forward width F (a multiple of 64):
//
//   td_in_kernel   : Linear in->D + LayerNorm (reference nisqa/NISQA_lib.py:989-991) and, fused behind it, the
//                    QKV projection of encoder layer 0 (in_proj of nn.MultiheadAttention, lib:1032)
//   td_sa_kernel   : one encoder layer for 64 queries of one clip (lib:1025-1040): softmax(q k^T) v over the clip's
//                    own keys (flash-style, keys in blocks of 64, online max / sum), out_proj, +x, LN1, FFN(ReLU)
//                    streamed over F in chunks of 64, +, LN2 - and, fused behind it, either the NEXT layer's QKV
//                    projection or (last layer) the PoolAttFF logits of all heads  w2_h . relu(W1_h x + b1_h) + b2_h
//                    (lib:1173)
//
// Every matrix product is a 64 x 64 x 64 tile product on the FFMA pipe: 256 threads = 16 (ty) x 16 (tx), a thread
// owns rows 4ty..4ty+3 and four columns, operands sit in shared memory, the A operand always row-major
// [row][k] with a padded leading dimension of 68 floats and read as float4 along k:
//   gemm_nn : B k-major [k][n]  (weights as packed by the engine, V), columns 4tx..4tx+3, LDS.128 along n
//   gemm_nt : B row-major [n][k] (K of q k^T), columns tx, tx+16, tx+32, tx+48 - consecutive lanes read consecutive
//             rows of pitch 68 floats = 4 banks apart: conflict-free LDS.128 along k
// A row's D columns live in the 16 lanes of one half-warp (4 NC per lane), so softmax / LayerNorm reductions are four
// xor-shuffles, and P (the softmax numerators) is written and re-read by the same half-warp: no block barrier inside a
// key block.  Operand tiles (16 KB, L2 resident) stream through a ring of shared-memory slots with cp.async, the next
// ones in flight while the current one is multiplied.  fp32 throughout (parity: +-1e-4 on the scores).
#include "../../include/nisqa_b200.h"
#include "common.cuh"
#include "launch.cuh"

namespace nisqa {

namespace {

constexpr int kT = 64;            // tile edge (rows, columns, k chunk)
constexpr int kLd = 68;           // leading dimension of row-major tiles (floats): 16-byte aligned rows, 4 banks apart
constexpr int kTileF = kT * kLd;  // floats of a padded tile
constexpr int kNT = 256;

__device__ __forceinline__ void cp16(float* dst_smem, const float* src, bool valid) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst_smem);
  const int bytes = valid ? 16 : 0;                       // src-size 0: the 16 bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// 64 rows x 64 floats, global (row pitch src_ld floats) -> shared (row pitch dst_ld floats); rows >= rows_valid are
// zero-filled.  All 256 threads, 4 x 16 bytes each.
__device__ __forceinline__ void tile_load_async(float* dst, int dst_ld, const float* src, long long src_ld, int rows_valid, int tid) {
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int idx = tid + it * kNT;
    const int r = idx >> 4, c4 = idx & 15;
    const bool ok = r < rows_valid;
    cp16(dst + r * dst_ld + c4 * 4, src + (ok ? (long long)r * src_ld + c4 * 4 : 0), ok);
  }
}

__device__ __forceinline__ void zero_acc(float (&acc)[4][4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
}

// acc[i][j] += sum_k A[4ty+i][k] * B[k][4tx+j]
__device__ __forceinline__ void gemm_nn(float (&acc)[4][4], const float* __restrict__ A, const float* __restrict__ B,
                                        int ldb, int ty, int tx) {
  const float* a0 = A + (4 * ty) * kLd;
  const float* b0 = B + 4 * tx;
#pragma unroll 2
  for (int k = 0; k < kT; k += 4) {
    float4 a[4], b[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const float4*>(a0 + i * kLd + k);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) b[kk] = *reinterpret_cast<const float4*>(b0 + (k + kk) * ldb);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float av[4] = {a[i].x, a[i].y, a[i].z, a[i].w};
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        acc[i][0] = fmaf(av[kk], b[kk].x, acc[i][0]);
        acc[i][1] = fmaf(av[kk], b[kk].y, acc[i][1]);
        acc[i][2] = fmaf(av[kk], b[kk].z, acc[i][2]);
        acc[i][3] = fmaf(av[kk], b[kk].w, acc[i][3]);
      }
    }
  }
}

// acc[i][j] += sum_k A[4ty+i][k] * B[tx+16j][k]
__device__ __forceinline__ void gemm_nt(float (&acc)[4][4], const float* __restrict__ A, const float* __restrict__ B,
                                        int ty, int tx) {
  const float* a0 = A + (4 * ty) * kLd;
  const float* b0 = B + tx * kLd;
#pragma unroll 2
  for (int k = 0; k < kT; k += 4) {
    float4 a[4], b[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const float4*>(a0 + i * kLd + k);
#pragma unroll
    for (int j = 0; j < 4; ++j) b[j] = *reinterpret_cast<const float4*>(b0 + (16 * j) * kLd + k);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float s = acc[i][j];
        s = fmaf(a[i].x, b[j].x, s); s = fmaf(a[i].y, b[j].y, s);
        s = fmaf(a[i].z, b[j].z, s); s = fmaf(a[i].w, b[j].w, s);
        acc[i][j] = s;
      }
  }
}

// reductions over the 16 lanes (tx) that share a row
__device__ __forceinline__ float row_sum(float v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float row_max(float v) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ void store_rows_smem(float* X, const float (&v)[4][4], int ty, int tx) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
    *reinterpret_cast<float4*>(X + (4 * ty + i) * kLd + 4 * tx) = make_float4(v[i][0], v[i][1], v[i][2], v[i][3]);
}

// Tiles stream through a ring of RS shared-memory slots of SLOT floats.  src(t, slot) issues the cp.async copies of the
// stream's tile t (nothing past its end); acquire() returns the slot of the next tile once it has landed for every
// thread.  One block barrier per tile: tile t + RS - 1 goes into the slot of tile t - 1 right after the barrier of tile
// t, when every thread is done with tile t - 1.  The barrier also publishes every shared-memory store made before it.
template <int RS, int SLOT, class Src>
struct TileStream {
  float* ring;
  const Src& src;
  int t = 0;
  __device__ __forceinline__ TileStream(float* r, const Src& s) : ring(r), src(s) {
#pragma unroll
    for (int i = 0; i < RS - 1; ++i) { src(i, ring + i * SLOT); cp_commit(); }
  }
  __device__ __forceinline__ float* acquire() {
    cp_wait<RS - 2>();
    __syncthreads();
    src(t + RS - 1, ring + ((t + RS - 1) % RS) * SLOT);
    cp_commit();
    return ring + (t++ % RS) * SLOT;
  }
};

__device__ __forceinline__ void bias_rows(float (&acc)[4][4], const float* __restrict__ b, int tx) {
  const float4 bb = __ldg(reinterpret_cast<const float4*>(b) + tx);
#pragma unroll
  for (int i = 0; i < 4; ++i) { acc[i][0] = bb.x; acc[i][1] = bb.y; acc[i][2] = bb.z; acc[i][3] = bb.w; }
}

// nn.LayerNorm(64 NC) (biased variance, eps 1e-5) of the rows held as v[n][i][0..3] = columns 64 n + 4tx .. 64 n + 4tx + 3:
// the chunks are summed in order before the xor-shuffles
template <int NC>
__device__ __forceinline__ void layernorm_rows(float (&v)[NC][4][4], const float* __restrict__ gamma,
                                               const float* __restrict__ beta, int tx) {
  constexpr float inv_d = 1.0f / (64.0f * NC);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float s = (v[0][i][0] + v[0][i][1]) + (v[0][i][2] + v[0][i][3]);
#pragma unroll
    for (int n = 1; n < NC; ++n) s += (v[n][i][0] + v[n][i][1]) + (v[n][i][2] + v[n][i][3]);
    const float mean = row_sum(s) * inv_d;
    float q = 0.f;
#pragma unroll
    for (int n = 0; n < NC; ++n) {
      const float d0 = v[n][i][0] - mean, d1 = v[n][i][1] - mean, d2 = v[n][i][2] - mean, d3 = v[n][i][3] - mean;
      const float qn = fmaf(d0, d0, d1 * d1) + fmaf(d2, d2, d3 * d3);
      q = n ? q + qn : qn;
      v[n][i][0] = d0; v[n][i][1] = d1; v[n][i][2] = d2; v[n][i][3] = d3;
    }
    const float var = row_sum(q) * inv_d;
    const float rstd = 1.0f / sqrtf(var + 1e-5f);
#pragma unroll
    for (int n = 0; n < NC; ++n) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + 64 * n) + tx);
      const float4 be = __ldg(reinterpret_cast<const float4*>(beta + 64 * n) + tx);
      v[n][i][0] = v[n][i][0] * rstd * g.x + be.x; v[n][i][1] = v[n][i][1] * rstd * g.y + be.y;
      v[n][i][2] = v[n][i][2] * rstd * g.z + be.z; v[n][i][3] = v[n][i][3] * rstd * g.w + be.w;
    }
  }
}

// rows 4ty..4ty+3 of a [64][ld] row block, columns 4tx..4tx+3, rows >= rows_valid not written
__device__ __forceinline__ void store_rows_global(float* __restrict__ dst, long long ld, const float (&v)[4][4], int rows_valid,
                                                  int ty, int tx) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (4 * ty + i < rows_valid)
      *reinterpret_cast<float4*>(dst + (4 * ty + i) * ld + 4 * tx) = make_float4(v[i][0], v[i][1], v[i][2], v[i][3]);
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// The time-dependency kernels are templates on NC = d_model / 64 (1..4).  A thread holds 4 rows x 4 NC columns: chunk n
// is columns 64 n + 4tx .. 64 n + 4tx + 3.  A transposed weight W^T [K][N] is packed in 64-column chunks: chunk n is the
// k-major [K][64] block at n K 64, so tile (k chunk c, column chunk n) is the contiguous [64][64] block (n K / 64 + c) 4096.
// Activations are row-major: x [n][D], qkv [n][3D] = q | k | v.  q is scaled by D^-1/2 after the projection (qscale) or,
// where that is a power of two, by the packed weights (qscale = 1).
template <int NC> struct TdShape {
  static constexpr int kMinBlocks = NC == 1 ? 2 : 1;     // CTAs per SM the register budget is sized for (NC 2 spills at 128)
  static constexpr int kRing = 4;                        // td_sa ring slots: 102 KB (NC 1), 119 KB (2), 136 KB (3), 153 KB (4)
  static constexpr int kSaFloats = NC * kTileF + kTileF + kRing * kTileF;
  static constexpr int kInSlot = kTileF + 4096;          // td_in ring slot: input tile | weight tile
  static constexpr int kInFloats = NC * kTileF + 2 * kInSlot;
};

// Linear(64 nk -> D) + LayerNorm (reference nisqa/NISQA_lib.py:989-991), the positional encoding, and the QKV projection
// of encoder layer 0 (in_proj of nn.MultiheadAttention, lib:1032) for 64 rows.  Per column chunk n: acc[n] = b + sum_c
// A_c W(c, n), A_c re-read for every n (one ring slot carries A_c and W(c, n)).
template <int NC>
__global__ void __launch_bounds__(kNT, TdShape<NC>::kMinBlocks)
td_in_kernel(const float* __restrict__ feats /*[n][64 nk]*/, const float* __restrict__ WT /*[NC][64 nk][64]*/, int nk,
             const float* __restrict__ bias, const float* __restrict__ gamma, const float* __restrict__ beta,
             const float* __restrict__ qkvT /*[3 NC][D][64]*/, const float* __restrict__ qkvb /*[3D]*/, float qscale,
             const float* __restrict__ pe /*[max_len][D] positional encoding or nullptr*/,
             const int* __restrict__ seg_clip, const ClipDesc* __restrict__ clips,
             float* __restrict__ x0 /*[n][D]*/, float* __restrict__ qkv /*[n][3D]*/, int n_rows) {
  constexpr int D = 64 * NC, SLOT = TdShape<NC>::kInSlot;
  extern __shared__ __align__(16) float sm[];
  float* Xs = sm;                               // [NC][64][68] LayerNorm output, input of the QKV projection
  float* ring = sm + NC * kTileF;               // 2 x (A tile [64][68] | weight tile [64][64])
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const long long row0 = (long long)blockIdx.x * kT;
  const int rows_valid = (int)min((long long)kT, (long long)n_rows - row0);
  const int ld = 64 * nk;                       // 384 CNN features, cnn_fc_out_h, the fused features, or the first stack's D
  const float* rows = feats + row0 * ld;
  const int t_lin = NC * nk;
  auto src = [&](int t, float* dst) {
    if (t < t_lin) {
      const int n = t / nk, c = t - n * nk;
      tile_load_async(dst, kLd, rows + c * 64, ld, rows_valid, tid);
      tile_load_async(dst + kTileF, 64, WT + (size_t)t * 4096, 64, 64, tid);        // tile (c, n) = (n nk + c) 4096
    } else if (t < t_lin + 3 * NC * NC) {
      tile_load_async(dst + kTileF, 64, qkvT + (size_t)(t - t_lin) * 4096, 64, 64, tid);
    }
  };
  TileStream<2, SLOT, decltype(src)> st(ring, src);
  float acc[NC][4][4];
#pragma unroll
  for (int n = 0; n < NC; ++n) {
    bias_rows(acc[n], bias + 64 * n, tx);
#pragma unroll 1
    for (int c = 0; c < nk; ++c) {
      const float* s = st.acquire();
      gemm_nn(acc[n], s, s + kTileF, 64, ty, tx);
    }
  }
  layernorm_rows<NC>(acc, gamma, beta, tx);
  if (pe != nullptr) {
    // PositionalEncoding (lib:1042-1062): x[t] += pe[t], t = position of the segment inside its clip
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const long long row = row0 + min(4 * ty + i, rows_valid - 1);
      const int t = (int)(row - clips[__ldg(seg_clip + row)].seg_off);
#pragma unroll
      for (int n = 0; n < NC; ++n) {
        const float4 pv = __ldg(reinterpret_cast<const float4*>(pe + (size_t)t * D + 64 * n) + tx);
        acc[n][i][0] += pv.x; acc[n][i][1] += pv.y; acc[n][i][2] += pv.z; acc[n][i][3] += pv.w;
      }
    }
  }
#pragma unroll
  for (int n = 0; n < NC; ++n) {
    store_rows_smem(Xs + n * kTileF, acc[n], ty, tx);
    store_rows_global(x0 + row0 * D + 64 * n, D, acc[n], rows_valid, ty, tx);
  }
  // QKV of layer 0: output chunk p = b + sum_c X_c W(c, p); the stream's next acquire publishes Xs
#pragma unroll 1
  for (int p = 0; p < 3 * NC; ++p) {
    float q[4][4];
    bias_rows(q, qkvb + 64 * p, tx);
#pragma unroll 1
    for (int c = 0; c < NC; ++c) {
      const float* s = st.acquire();
      gemm_nn(q, Xs + c * kTileF, s + kTileF, 64, ty, tx);
    }
    if (p < NC && qscale != 1.f) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) q[i][j] *= qscale;
    }
    store_rows_global(qkv + row0 * (3 * D) + 64 * p, 3 * D, q, rows_valid, ty, tx);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// One encoder layer for 64 queries of one clip (lib:1025-1040): softmax(q k^T) v over the clip's own keys (flash-style,
// keys in blocks of 64, online max / sum), out_proj, +x, LN1, FFN(ReLU) streamed over the hidden width F in chunks of 64
// (out += relu(X W1[:, f] + b1_f) W2[f, :]: the hidden layer is never held whole), +, LN2 - and, fused behind it, either
// the NEXT layer's QKV projection or (last layer) the PoolAttFF logits of all heads  w2_h . relu(W1_h x + b1_h) + b2_h
// (lib:1173).  Every operand tile after Q - K and V chunks of each key block, then the weight tiles - comes through
// one TileStream, so the loads of the next phase are in flight while the current one computes.
// shared memory: Qs [NC][64][68] | Ps [64][68] | ring [kRing][64][68]
template <int NC>
__global__ void __launch_bounds__(kNT, TdShape<NC>::kMinBlocks)
td_sa_kernel(const float* __restrict__ x_in, const float* __restrict__ qkv, const ClipDesc* __restrict__ clips,
             int n_clips, const int* __restrict__ qtile_prefix /*64-row tiles*/, SaLayerParams P, int F,
             float* __restrict__ x_out,
             const float* __restrict__ next_qkvT, const float* __restrict__ next_qkvb, float qscale, float* __restrict__ qkv_next,
             PoolHeadParams H, int n_heads, float* __restrict__ logits) {
  constexpr int D = 64 * NC;
  extern __shared__ __align__(16) float sm[];
  float* Qs = sm;                          // queries -> attention output -> LN1 output (FFN input) -> layer output
  float* Ps = sm + NC * kTileF;            // softmax numerators -> FFN hidden chunk
  float* ring = Ps + kTileF;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int c = upper_slot(qtile_prefix, n_clips, blockIdx.x);
  const ClipDesc cd = clips[c];
  const int S = cd.n_seg;
  const int q0 = (blockIdx.x - __ldg(qtile_prefix + c)) * kT;
  const int rows_valid = min(kT, S - q0);
  const long long row0 = (long long)cd.seg_off + q0;
  const float* kv_base = qkv + (long long)cd.seg_off * (3 * D);
  const int n_kb = (S + kT - 1) / kT, FC = F / 64;
  const bool last = next_qkvT == nullptr;
  // the layer's tile stream: per key block K chunks 0..NC-1 (row-major [key][d], pitch 68) then V chunks 0..NC-1
  // (k-major, pitch 64); out_proj tiles (c, n); per hidden chunk f the W1 tiles (c, f), then the W2 tiles (f, n); then
  // the next layer's QKV tiles (c, p) or the PoolAttFF W1 tiles (c) of every (head, half) of W1T [head][D][128]
  const int t_att = 2 * NC * n_kb, t_out = t_att + NC * NC, t_ffn = t_out + 2 * NC * FC;
  auto src = [&](int t, float* dst) {
    if (t < t_att) {
      const int kb = t / (2 * NC), r = t - kb * 2 * NC;
      const float* kv = kv_base + (long long)kb * kT * (3 * D) + D;
      const int nv = min(kT, S - kb * kT);
      if (r < NC) tile_load_async(dst, kLd, kv + 64 * r, 3 * D, nv, tid);
      else tile_load_async(dst, 64, kv + D + 64 * (r - NC), 3 * D, nv, tid);
    } else if (t < t_out) {
      tile_load_async(dst, 64, P.WoT + (size_t)(t - t_att) * 4096, 64, 64, tid);                   // WoT [NC][D][64]
    } else if (t < t_ffn) {
      const int u = t - t_out, f = u / (2 * NC), r = u - f * 2 * NC;
      if (r < NC) tile_load_async(dst, 64, P.W1T + ((size_t)f * NC + r) * 4096, 64, 64, tid);      // W1T [F/64][D][64]
      else tile_load_async(dst, 64, P.W2T + ((size_t)(r - NC) * FC + f) * 4096, 64, 64, tid);     // W2T [NC][F][64]
    } else if (!last) {
      const int u = t - t_ffn;
      if (u < 3 * NC * NC) tile_load_async(dst, 64, next_qkvT + (size_t)u * 4096, 64, 64, tid);   // [3 NC][D][64]
    } else {
      const int u = t - t_ffn, q = u / NC, k = u - q * NC;                                         // q = 2 head + half
      if (q < 2 * n_heads) tile_load_async(dst, 64, H.W1T + ((size_t)(q >> 1) * D + 64 * k) * 128 + (q & 1) * 64, 128, 64, tid);
    }
  };

  // ---- attention
#pragma unroll
  for (int n = 0; n < NC; ++n) tile_load_async(Qs + n * kTileF, kLd, qkv + row0 * (3 * D) + 64 * n, 3 * D, rows_valid, tid);
  TileStream<TdShape<NC>::kRing, kTileF, decltype(src)> st(ring, src);      // (its first group carries Q)
  float o[NC][4][4];
#pragma unroll
  for (int n = 0; n < NC; ++n) zero_acc(o[n]);
  float m[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { m[i] = -INFINITY; l[i] = 0.f; }
#pragma unroll 1
  for (int kb = 0; kb < n_kb; ++kb) {
    float s[4][4];
    zero_acc(s);
#pragma unroll 1
    for (int k = 0; k < NC; ++k) gemm_nt(s, Qs + k * kTileF, st.acquire(), ty, tx);   // s[i][j]: query 4ty+i, key 64 kb + tx + 16j
    const int nk = S - kb * kT;                                                      // keys >= nk of this block do not exist
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float bm = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) { if (tx + 16 * j >= nk) s[i][j] = -INFINITY; bm = fmaxf(bm, s[i][j]); }
      bm = row_max(bm);                                        // every block holds >= 1 real key: bm is finite
      const float mn = fmaxf(m[i], bm);
      const float sc = expf(m[i] - mn);                        // first block: expf(-inf) = 0
      float ps = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float p = expf(s[i][j] - mn);                    // masked keys: expf(-inf) = 0
        ps += p;
        Ps[(4 * ty + i) * kLd + tx + 16 * j] = p;
      }
      l[i] = l[i] * sc + row_sum(ps);
      m[i] = mn;
#pragma unroll
      for (int n = 0; n < NC; ++n) { o[n][i][0] *= sc; o[n][i][1] *= sc; o[n][i][2] *= sc; o[n][i][3] *= sc; }
    }
    __syncwarp();                                  // P rows 4ty..4ty+3 are written and read by this half-warp only
#pragma unroll
    for (int n = 0; n < NC; ++n) gemm_nn(o[n], Ps, st.acquire(), 64, ty, tx);   // o[n][i][j]: query 4ty+i, d = 64 n + 4tx + j
  }
  // the attention output replaces Q: every thread has read Q for the last time before the barrier of the last V chunk
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float inv = 1.0f / l[i];
#pragma unroll
    for (int n = 0; n < NC; ++n) { o[n][i][0] *= inv; o[n][i][1] *= inv; o[n][i][2] *= inv; o[n][i][3] *= inv; }
  }
#pragma unroll
  for (int n = 0; n < NC; ++n) store_rows_smem(Qs + n * kTileF, o[n], ty, tx);

  // ---- out_proj + residual + LN1
  float v[NC][4][4];
#pragma unroll
  for (int n = 0; n < NC; ++n) {
    bias_rows(v[n], P.bo + 64 * n, tx);
#pragma unroll 1
    for (int k = 0; k < NC; ++k) gemm_nn(v[n], Qs + k * kTileF, st.acquire(), 64, ty, tx);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = min(4 * ty + i, rows_valid - 1);                             // rows beyond the clip: any valid row
#pragma unroll
    for (int n = 0; n < NC; ++n) {
      const float4 xr = __ldg(reinterpret_cast<const float4*>(x_in + (row0 + r) * D + 64 * n) + tx);
      v[n][i][0] += xr.x; v[n][i][1] += xr.y; v[n][i][2] += xr.z; v[n][i][3] += xr.w;
    }
  }
  layernorm_rows<NC>(v, P.ln1_g, P.ln1_b, tx);
  __syncthreads();                                 // every thread is done with the attention output
#pragma unroll
  for (int n = 0; n < NC; ++n) store_rows_smem(Qs + n * kTileF, v[n], ty, tx);   // FFN input and residual

  // ---- FFN over hidden chunks of 64
#pragma unroll
  for (int n = 0; n < NC; ++n) bias_rows(v[n], P.b2 + 64 * n, tx);           // v now accumulates the FFN output
#pragma unroll 1
  for (int f = 0; f < FC; ++f) {
    float h[4][4];
    bias_rows(h, P.b1 + 64 * f, tx);
#pragma unroll 1
    for (int k = 0; k < NC; ++k) gemm_nn(h, Qs + k * kTileF, st.acquire(), 64, ty, tx);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) h[i][j] = fmaxf(h[i][j], 0.f);
    store_rows_smem(Ps, h, ty, tx);                // (every thread is done with the previous chunk: barrier of W1 tile k = 0)
#pragma unroll
    for (int n = 0; n < NC; ++n) gemm_nn(v[n], Ps, st.acquire(), 64, ty, tx);
  }
#pragma unroll
  for (int n = 0; n < NC; ++n)
#pragma unroll
    for (int i = 0; i < 4; ++i) {                  // + residual: this thread's own elements of the FFN input
      const float4 xr = *reinterpret_cast<const float4*>(Qs + n * kTileF + (4 * ty + i) * kLd + 4 * tx);
      v[n][i][0] = xr.x + v[n][i][0]; v[n][i][1] = xr.y + v[n][i][1];
      v[n][i][2] = xr.z + v[n][i][2]; v[n][i][3] = xr.w + v[n][i][3];
    }
  layernorm_rows<NC>(v, P.ln2_g, P.ln2_b, tx);
#pragma unroll
  for (int n = 0; n < NC; ++n) {
    store_rows_global(x_out + row0 * D + 64 * n, D, v[n], rows_valid, ty, tx);
    store_rows_smem(Qs + n * kTileF, v[n], ty, tx);   // input of the fused tail (the FFN input was last read before the W2 barriers)
  }

  if (!last) {
    // ---- next layer's QKV projection
#pragma unroll 1
    for (int p = 0; p < 3 * NC; ++p) {
      float acc[4][4];
      bias_rows(acc, next_qkvb + 64 * p, tx);
#pragma unroll 1
      for (int k = 0; k < NC; ++k) gemm_nn(acc, Qs + k * kTileF, st.acquire(), 64, ty, tx);
      if (p < NC && qscale != 1.f) {
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] *= qscale;
      }
      store_rows_global(qkv_next + row0 * (3 * D) + 64 * p, 3 * D, acc, rows_valid, ty, tx);
    }
  } else {
    // ---- PoolAttFF logits of every head (n_heads == 0: another pooling module follows)
    float part_logit[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
    for (int q = 0; q < 2 * n_heads; ++q) {
      const int hd = q >> 1, half = q & 1;
      float acc[4][4];
      bias_rows(acc, H.b1 + hd * 128 + half * 64, tx);
      const float4 w2 = __ldg(reinterpret_cast<const float4*>(H.w2 + hd * 128 + half * 64) + tx);
#pragma unroll 1
      for (int k = 0; k < NC; ++k) gemm_nn(acc, Qs + k * kTileF, st.acquire(), 64, ty, tx);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float t = part_logit[i];
        t = fmaf(w2.x, fmaxf(acc[i][0], 0.f), t); t = fmaf(w2.y, fmaxf(acc[i][1], 0.f), t);
        t = fmaf(w2.z, fmaxf(acc[i][2], 0.f), t); t = fmaf(w2.w, fmaxf(acc[i][3], 0.f), t);
        part_logit[i] = t;
      }
      if (half == 1) {
        const float b2 = __ldg(H.b2 + hd);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float tot = row_sum(part_logit[i]);
          if (tx == 0 && 4 * ty + i < rows_valid) logits[(row0 + 4 * ty + i) * n_heads + hd] = tot + b2;
          part_logit[i] = 0.f;
        }
      }
    }
  }
  cp_wait<0>();                                    // (only empty groups can be pending here)
}

// ---------------------------------------------------------------------------------------------------------------
// Double-ended model (NISQA_DE, reference lib:272-424): time alignment of the reference clip's features to the degraded
// clip's (Alignment, lib:1228-1285) and feature fusion (Fusion, lib:1380-1417), for 64 degraded steps of one pair.
//   x = time_dependency output of the degraded clip (clip 2p), y = of the reference clip (clip 2p + 1): rows of W real
//   columns (td's fan_out) at a pitch of ld = 64 NC (NC = 1..8), the pad columns zero - so they add nothing to a dot
//   product, a distance or a norm
//   score[i][j] : dot  x_i . y_j (AttDot, lib:1287-1296) | cosine similarity x_i . y_j rx_i ry_j, r = 1 / max(|row|, 1e-8)
//                 (AttCosine, lib:1298-1308) | -(1/W) sum_d |x_id - y_jd| (AttDistance with its default norms,
//                 lib:1310-1323) | x_i . yp_j, yp = W y + b (AttLuong, lib:1344-1357) | v . tanh(xq_i + yk_j), xq = Wq x + bq,
//                 yk = Wy y + by (AttBahdanau, att_dim 128, lib:1325-1342; its output bias shifts every score of a row
//                 alike and drops out of softmax / argmax); keys j >= n_wins_y masked.  The projections yp, xq | yk and
//                 the reciprocal norms r come from launch_de_align's tile GEMM / row_rnorm_kernel over all rows of the pass.
//   hard        : y_al[i] = y[argmax_j softmax(score[i])] = y[first maximal score] (ApplyHardAttention, lib:1359-1368)
//   soft        : y_al[i] = softmax_j(score[i]) . y (ApplySoftAttention, lib:1370-1378), online max / sum over key blocks
//   fuse        : [x, y_al, x - y_al] | [x + y_al, x - y_al] | [x, y_al]  ->  fused[row][nf ld], part p at column p ld
// Same 64 x 64 register tiling as td_sa_kernel.  The query operand (x, or xq for AttBahdanau) of the CTA's 64 steps stays
// resident; per key block the n_sc score chunks of the keys (row-major, pitch 68) and - soft - the value chunks of y the
// CTA outputs (k-major, pitch 64) stream through one TileStream.  A soft CTA outputs a group of at most G column chunks
// (blockIdx.y: the group) and recomputes the scores for it, so at most 4 output chunks sit in registers.
// AL (alignment calls): also the online softmax sum l and position sum c = sum_j exp(s_ij - m) j of every row, rescaled
// per key block like the soft path's (hard application: besides its running first maximum), and - the blockIdx.y == 0
// CTA only, the others recompute the same scores - ref_seg = the first maximal key, weight = 1 / l, centroid = c / l,
// peak = m + pbias (AttBahdanau's v bias, which the softmax drops) at al.row_off[c] + row.

// s[i][j] -= sum_k |A[4ty+i][k] - B[tx+16j][k]|
__device__ __forceinline__ void absdiff_nt(float (&s)[4][4], const float* __restrict__ A, const float* __restrict__ B, int ty, int tx) {
  const float* a0 = A + (4 * ty) * kLd;
  const float* b0 = B + tx * kLd;
#pragma unroll 2
  for (int k = 0; k < kT; k += 4) {
    float4 a[4], b[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const float4*>(a0 + i * kLd + k);
#pragma unroll
    for (int j = 0; j < 4; ++j) b[j] = *reinterpret_cast<const float4*>(b0 + (16 * j) * kLd + k);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        s[i][j] -= (fabsf(a[i].x - b[j].x) + fabsf(a[i].y - b[j].y)) + (fabsf(a[i].z - b[j].z) + fabsf(a[i].w - b[j].w));
  }
}

// s[i][j] += sum_k v[k] tanh(A[4ty+i][k] + B[tx+16j][k])
__device__ __forceinline__ void tanh_nt(float (&s)[4][4], const float* __restrict__ A, const float* __restrict__ B,
                                        const float* __restrict__ v, int ty, int tx) {
  const float* a0 = A + (4 * ty) * kLd;
  const float* b0 = B + tx * kLd;
#pragma unroll 1
  for (int k = 0; k < kT; k += 4) {
    const float4 vv = __ldg(reinterpret_cast<const float4*>(v + k));
    float4 a[4], b[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const float4*>(a0 + i * kLd + k);
#pragma unroll
    for (int j = 0; j < 4; ++j) b[j] = *reinterpret_cast<const float4*>(b0 + (16 * j) * kLd + k);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float t = s[i][j];
        t = fmaf(vv.x, tanhf(a[i].x + b[j].x), t); t = fmaf(vv.y, tanhf(a[i].y + b[j].y), t);
        t = fmaf(vv.z, tanhf(a[i].z + b[j].z), t); t = fmaf(vv.w, tanhf(a[i].w + b[j].w), t);
        s[i][j] = t;
      }
  }
}

// Fusion (lib:1402-1417) of four columns at `col` of one row; part p of the row starts at column p ld
__device__ __forceinline__ void fuse_store(float* __restrict__ dst, int ld, int col, float4 xv, float4 yv, int fuse) {
  const float4 df = make_float4(xv.x - yv.x, xv.y - yv.y, xv.z - yv.z, xv.w - yv.w);
  if (fuse == NISQA_DE_FUSE_XY_MINUS) {
    *reinterpret_cast<float4*>(dst + col) = xv; *reinterpret_cast<float4*>(dst + ld + col) = yv;
    *reinterpret_cast<float4*>(dst + 2 * ld + col) = df;
  } else if (fuse == NISQA_DE_FUSE_PLUS_MINUS) {
    *reinterpret_cast<float4*>(dst + col) = make_float4(xv.x + yv.x, xv.y + yv.y, xv.z + yv.z, xv.w + yv.w);
    *reinterpret_cast<float4*>(dst + ld + col) = df;
  } else {
    *reinterpret_cast<float4*>(dst + col) = xv; *reinterpret_cast<float4*>(dst + ld + col) = yv;
  }
}

constexpr int kDeRing = 3;              // de_align_kernel ring slots
// shared memory of de_align_kernel: Qs [n_sc][64][68] | Ps [64][68] | ring [kDeRing][64][68]; n_sc <= 8: 204 KB
constexpr int de_smem_bytes(int n_sc) { return (n_sc + 1 + kDeRing) * kTileF * 4; }

// G: output chunks per soft CTA (hard application runs G = 1 and writes every chunk of y[best]).  Al: empty (the plain
// instances, whose parameter list stays that of the kernel without alignment outputs) or one DeAlignOut (AL).
template <typename T> __device__ __forceinline__ const T& first_arg(const T& t) { return t; }
template <int G, typename... Al>
__global__ void __launch_bounds__(kNT, G <= 2 ? 2 : 1)
de_align_kernel(const float* __restrict__ x_td /*[n_seg][ld]*/, int ld, int W, const ClipDesc* __restrict__ clips, int n_clips,
                const int* __restrict__ qtile_prefix /*64-row tiles*/, int align, int soft, int fuse,
                const float* __restrict__ qsrc, const float* __restrict__ ksrc, int pld, int n_sc,
                const float* __restrict__ rnorm, const float* __restrict__ v, float* __restrict__ fused /*[n_seg][nf ld]*/,
                Al... al_arg) {
  constexpr bool AL = sizeof...(Al) > 0;
  extern __shared__ __align__(16) float sm[];
  float* Qs = sm;                          // [n_sc][64][68] query operand of the CTA's degraded steps
  float* Ps = sm + n_sc * kTileF;          // [64][68] softmax numerators (soft attention)
  float* ring = Ps + kTileF;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int c = upper_slot(qtile_prefix, n_clips, blockIdx.x);
  if (c & 1) return;                       // reference clips are keys only
  const ClipDesc cd = clips[c], cr = clips[cd.ref_clip];
  const int Sx = cd.n_seg, Sy = cr.n_seg;
  if (Sx <= 0 || Sy <= 0) return;
  const int q0 = (blockIdx.x - __ldg(qtile_prefix + c)) * kT;
  const int rows_valid = min(kT, Sx - q0);
  const long long row0 = (long long)cd.seg_off + q0, yrow0 = cr.seg_off;
  const int NC = ld / 64, nf = fuse == NISQA_DE_FUSE_XY_MINUS ? 3 : 2;
  const int c0 = blockIdx.y * G, ng = soft ? min(G, NC - c0) : 0;       // the CTA's output chunks c0 .. c0 + ng - 1
  const int n_kb = (Sy + kT - 1) / kT, per_kb = n_sc + ng;
  // the tile stream: per key block its n_sc score chunks, then (soft) its value chunks c0 .. c0 + ng - 1
  auto src = [&](int t, float* dst) {
    if (t >= n_kb * per_kb) return;
    const int kb = t / per_kb, r = t - kb * per_kb;
    const int nv = min(kT, Sy - kb * kT);
    const long long j0 = yrow0 + (long long)kb * kT;
    if (r < n_sc) tile_load_async(dst, kLd, ksrc + j0 * pld + 64 * r, pld, nv, tid);
    else tile_load_async(dst, 64, x_td + j0 * ld + 64 * (c0 + r - n_sc), ld, nv, tid);
  };
#pragma unroll 1
  for (int k = 0; k < n_sc; ++k) tile_load_async(Qs + k * kTileF, kLd, qsrc + row0 * pld + 64 * k, pld, rows_valid, tid);
  TileStream<kDeRing, kTileF, decltype(src)> st(ring, src);      // (its first group carries the query operand)
  const float wf = (float)W;
  float o[G][4][4];
#pragma unroll
  for (int n = 0; n < G; ++n) zero_acc(o[n]);
  float m[4], l[4], cpos[4];
  int best[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { m[i] = -INFINITY; l[i] = 0.f; best[i] = 0; }
  if constexpr (AL) {
#pragma unroll
    for (int i = 0; i < 4; ++i) cpos[i] = 0.f;
  }
#pragma unroll 1
  for (int kb = 0; kb < n_kb; ++kb) {
    const int j0 = kb * kT, nkeys = Sy - j0;            // keys >= nkeys of this block do not exist
    float s[4][4];
    zero_acc(s);
#pragma unroll 1
    for (int k = 0; k < n_sc; ++k) {                    // s[i][j]: query 4ty+i, key j0 + tx + 16j
      const float* K = st.acquire();
      if (align == NISQA_DE_ALIGN_BAHDANAU) tanh_nt(s, Qs + k * kTileF, K, v + 64 * k, ty, tx);
      else if (align == NISQA_DE_ALIGN_DISTANCE) absdiff_nt(s, Qs + k * kTileF, K, ty, tx);
      else gemm_nt(s, Qs + k * kTileF, K, ty, tx);
    }
    if (align == NISQA_DE_ALIGN_DISTANCE) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] /= wf;
    } else if (align == NISQA_DE_ALIGN_COSINE) {
      float rq[4], ry[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) rq[i] = __ldg(rnorm + row0 + min(4 * ty + i, rows_valid - 1));
#pragma unroll
      for (int j = 0; j < 4; ++j) ry[j] = __ldg(rnorm + yrow0 + j0 + min(tx + 16 * j, nkeys - 1));
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = s[i][j] * rq[i] * ry[j];
    }
    if (!soft) {
      // first maximal score of the row: columns of a thread ascend with j and with the block; ties between threads
      // are resolved towards the smaller key index
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float bv = -INFINITY; int bi = 0x7fffffff;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (tx + 16 * j < nkeys && s[i][j] > bv) { bv = s[i][j]; bi = j0 + tx + 16 * j; }
#pragma unroll
        for (int of = 8; of > 0; of >>= 1) {
          const float ov = __shfl_xor_sync(0xffffffffu, bv, of);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, of);
          if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if constexpr (AL) {                              // (bv: the block's maximum, on all 16 lanes of the row)
          const float mn = fmaxf(m[i], bv);
          const float sc = expf(m[i] - mn);
          float ps = 0.f, pc = 0.f;
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (tx + 16 * j < nkeys) {
              const float p = expf(s[i][j] - mn);
              ps += p;
              pc = fmaf(p, (float)(j0 + tx + 16 * j), pc);
            }
          l[i] = l[i] * sc + row_sum(ps);
          cpos[i] = cpos[i] * sc + row_sum(pc);
        }
        if (bv > m[i]) { m[i] = bv; best[i] = bi; }       // (strictly greater: an earlier block keeps a tie)
      }
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if constexpr (AL) {                              // the first maximal key, as the hard path finds it
          float bv = -INFINITY; int bi = 0x7fffffff;
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (tx + 16 * j < nkeys && s[i][j] > bv) { bv = s[i][j]; bi = j0 + tx + 16 * j; }
#pragma unroll
          for (int of = 8; of > 0; of >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, of);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, of);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
          }
          if (bv > m[i]) best[i] = bi;
        }
        float bm = -INFINITY;
#pragma unroll
        for (int j = 0; j < 4; ++j) { if (tx + 16 * j >= nkeys) s[i][j] = -INFINITY; bm = fmaxf(bm, s[i][j]); }
        bm = row_max(bm);
        const float mn = fmaxf(m[i], bm);
        const float sc = expf(m[i] - mn);
        float ps = 0.f, pc = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float p = expf(s[i][j] - mn);
          ps += p;
          if constexpr (AL) pc = fmaf(p, (float)(j0 + tx + 16 * j), pc);
          Ps[(4 * ty + i) * kLd + tx + 16 * j] = p;
        }
        l[i] = l[i] * sc + row_sum(ps);
        if constexpr (AL) cpos[i] = cpos[i] * sc + row_sum(pc);
        m[i] = mn;
#pragma unroll
        for (int n = 0; n < G; ++n) { o[n][i][0] *= sc; o[n][i][1] *= sc; o[n][i][2] *= sc; o[n][i][3] *= sc; }
      }
      __syncwarp();                                  // P rows 4ty..4ty+3 are written and read by this half-warp only
#pragma unroll
      for (int n = 0; n < G; ++n)
        if (n < ng) gemm_nn(o[n], Ps, st.acquire(), 64, ty, tx);   // o[n][i][d] += sum_j p[i][j] y[j][64 (c0 + n) + d]
    }
  }
  if constexpr (AL) {
    const DeAlignOut al = first_arg(al_arg...);
    if (blockIdx.y == 0 && tx == 0) {
      const long long r0 = al.row_off[c] + q0 + 4 * ty;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (4 * ty + i >= rows_valid) continue;
        const float inv = 1.0f / l[i];
        al.ref_seg[r0 + i] = best[i];
        al.weight[r0 + i] = inv;
        al.centroid[r0 + i] = cpos[i] * inv;
        al.peak[r0 + i] = m[i] + al.pbias;
      }
    }
  }
  // ---- fusion (lib:1402-1417): x from the td rows, y_al from y[best] (hard) or the accumulators (soft)
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (4 * ty + i >= rows_valid) continue;
    const float* xr = x_td + (row0 + 4 * ty + i) * ld;
    float* dst = fused + (row0 + 4 * ty + i) * (long long)(nf * ld);
    if (!soft) {
      const float* yr = x_td + (yrow0 + best[i]) * ld;
#pragma unroll 1
      for (int n = 0; n < NC; ++n) {
        const int col = 64 * n + 4 * tx;
        fuse_store(dst, ld, col, __ldg(reinterpret_cast<const float4*>(xr + col)), __ldg(reinterpret_cast<const float4*>(yr + col)), fuse);
      }
    } else {
      const float inv = 1.0f / l[i];
#pragma unroll
      for (int n = 0; n < G; ++n) {
        if (n >= ng) continue;
        const int col = 64 * (c0 + n) + 4 * tx;
        fuse_store(dst, ld, col, __ldg(reinterpret_cast<const float4*>(xr + col)),
                   make_float4(o[n][i][0] * inv, o[n][i][1] * inv, o[n][i][2] * inv, o[n][i][3] * inv), fuse);
      }
    }
  }
  cp_wait<0>();                                    // (only empty groups can be pending here)
}

// 1 / max(|x_r|, 1e-8) over the W real columns of every row (AttCosine's norms), one warp per row
__global__ void row_rnorm_kernel(const float* __restrict__ x, int ld, int W, int n_rows, float* __restrict__ out) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= n_rows) return;
  float ss = 0.f;
  for (int k = lane; k < W; k += 32) { const float v = __ldg(x + (size_t)row * ld + k); ss = fmaf(v, v, ss); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if (lane == 0) out[row] = 1.0f / fmaxf(sqrtf(ss), 1e-8f);
}

// scores of a double-ended pass: row 2p = the pair's score (NaN when either clip was skipped), row 2p + 1 = NaN
__global__ void de_finalize_kernel(const ClipDesc* __restrict__ clips, int n_clips, int n_out, float* __restrict__ scores) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_clips) return;
  const bool bad = (c & 1) || clips[c].n_seg <= 0 || clips[clips[c].ref_clip].n_seg <= 0;
  if (bad) for (int h = 0; h < n_out; ++h) scores[c * n_out + h] = __int_as_float(0x7fc00000);
}


// ---------------------------------------------------------------------------------------------------------------
// Framewise models without convolutions (reference lib:504-583, user checkpoints): SkipCNN = BatchNorm2d(1) + flatten
// (+ Linear), DFF = BatchNorm2d(1) + flatten + 4 x (Linear + BatchNorm1d + ReLU).
//   seg_feats_kernel  : segment s -> row [ld]: a * max(mel[frame0 + t][m], thr) + c at index m * seg_len + t
//                       (x.view(-1, fan_in), fan_in = n_mels * seg_len, lib:531 / 572), columns fan_in .. ld - 1 zero
//                       (ld: fan_in rounded up to 64, the rows feed 64-wide k chunks)
//   linear_tile_kernel: Y[n][N] = act(X[n][K] W^T + b), 64 x 64 output tiles, K in chunks of 64 (K, N multiples of 64),
//                       the same register-tiled fp32 product as the time-dependency block
__global__ void seg_feats_kernel(const float* __restrict__ mel, int n_mels, int seg_len, int ld,
                                 const int* __restrict__ seg_frame0, const float* __restrict__ seg_thr,
                                 const float* __restrict__ bn /*a, c*/, int n_seg, float* __restrict__ out /*[n_seg][ld]*/) {
  const int s = blockIdx.x;
  if (s >= n_seg) return;
  const float* src = mel + (size_t)__ldg(seg_frame0 + s) * n_mels;
  const float thr = __ldg(seg_thr + s), a = __ldg(bn), c = __ldg(bn + 1);
  for (int j = threadIdx.x; j < ld; j += blockDim.x) {
    float v = 0.f;
    if (j < n_mels * seg_len) {
      const int m = j / seg_len, t = j - m * seg_len;
      v = fmaf(a, fmaxf(__ldg(src + t * n_mels + m), thr), c);
    }
    out[(size_t)s * ld + j] = v;
  }
}

constexpr int kLinSmemFloats = 2 * kTileF + 2 * 4096;

__global__ void __launch_bounds__(kNT, 2)
linear_tile_kernel(const float* __restrict__ X, int ldx, const float* __restrict__ WT /*[K][N]*/, const float* __restrict__ bias,
                   int relu, float* __restrict__ Y, int ldy, int n_rows, int K, int N) {
  extern __shared__ __align__(16) float sm[];
  float* As = sm;                       // [2][64][68]
  float* Ws = sm + 2 * kTileF;          // [2][64][64]
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const long long row0 = (long long)blockIdx.x * kT;
  const int n0 = blockIdx.y * kT;
  const int rows_valid = (int)min((long long)kT, (long long)n_rows - row0);
  const float* src = X + row0 * ldx;
  const int nk = K / kT;
  tile_load_async(As, kLd, src, ldx, rows_valid, tid);
  tile_load_async(Ws, 64, WT + n0, N, 64, tid);
  cp_commit();
  float acc[4][4];
  {
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + n0) + tx);
#pragma unroll
    for (int i = 0; i < 4; ++i) { acc[i][0] = bb.x; acc[i][1] = bb.y; acc[i][2] = bb.z; acc[i][3] = bb.w; }
  }
#pragma unroll 1
  for (int c = 0; c < nk; ++c) {
    if (c + 1 < nk) {
      tile_load_async(As + ((c + 1) & 1) * kTileF, kLd, src + (c + 1) * 64, ldx, rows_valid, tid);
      tile_load_async(Ws + ((c + 1) & 1) * 4096, 64, WT + (size_t)(c + 1) * 64 * N + n0, N, 64, tid);
    }
    cp_commit();
    cp_wait<1>();
    __syncthreads();
    gemm_nn(acc, As + (c & 1) * kTileF, Ws + (c & 1) * 4096, 64, ty, tx);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (4 * ty + i < rows_valid) {
      float4 v = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
      *reinterpret_cast<float4*>(Y + (row0 + 4 * ty + i) * ldy + n0 + 4 * tx) = v;
    }
}

// ------------------------------------------------------------------ host launchers
// d_model = 64 nc, nc in 1..4
template <int NC>
void td_in_instance(cudaStream_t st, const float* feats, const float* WT, int nk, const float* b, const float* g, const float* be,
                    const float* qkvT, const float* qkvb, float qscale, const float* pe, const int* seg_clip, const ClipDesc* clips,
                    float* x0, float* qkv, int n_rows) {
  static unsigned long long cfg = 0;
  const int smem = TdShape<NC>::kInFloats * 4;
  if (first_launch_on_device(cfg)) cudaFuncSetAttribute(td_in_kernel<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  td_in_kernel<NC><<<(n_rows + kT - 1) / kT, kNT, smem, st>>>(feats, WT, nk, b, g, be, qkvT, qkvb, qscale, pe, seg_clip, clips,
                                                              x0, qkv, n_rows);
}
void launch_td_in(cudaStream_t st, int nc, const float* feats, const float* WT, int nk, const float* b, const float* g,
                  const float* be, const float* qkvT, const float* qkvb, float qscale, const float* pe, const int* seg_clip,
                  const ClipDesc* clips, float* x0, float* qkv, int n_rows) {
  switch (nc) {
    case 1: td_in_instance<1>(st, feats, WT, nk, b, g, be, qkvT, qkvb, qscale, pe, seg_clip, clips, x0, qkv, n_rows); break;
    case 2: td_in_instance<2>(st, feats, WT, nk, b, g, be, qkvT, qkvb, qscale, pe, seg_clip, clips, x0, qkv, n_rows); break;
    case 3: td_in_instance<3>(st, feats, WT, nk, b, g, be, qkvT, qkvb, qscale, pe, seg_clip, clips, x0, qkv, n_rows); break;
    case 4: td_in_instance<4>(st, feats, WT, nk, b, g, be, qkvT, qkvb, qscale, pe, seg_clip, clips, x0, qkv, n_rows); break;
  }
}

template <int G, typename... Al>
void de_align_instance(cudaStream_t st, dim3 grid, int smem, const float* x_td, int ld, int W, const ClipDesc* clips,
                       int n_clips, const int* qtile64_prefix, int align, int soft, int fuse, const float* q, const float* k,
                       int pld, int n_sc, const float* rnorm, const float* v, float* fused, Al... al) {
  static unsigned long long cfg = 0;
  if (first_launch_on_device(cfg))
    cudaFuncSetAttribute(de_align_kernel<G, Al...>, cudaFuncAttributeMaxDynamicSharedMemorySize, de_smem_bytes(8));
  de_align_kernel<G, Al...><<<grid, kNT, smem, st>>>(x_td, ld, W, clips, n_clips, qtile64_prefix, align, soft, fuse, q, k,
                                                     pld, n_sc, rnorm, v, fused, al...);
}
template <int G>
void de_align_select(const DeAlignOut* al, cudaStream_t st, dim3 grid, int smem, const float* x_td, int ld, int W,
                     const ClipDesc* clips, int n_clips, const int* qtile64_prefix, int align, int soft, int fuse,
                     const float* q, const float* k, int pld, int n_sc, const float* rnorm, const float* v, float vb,
                     float* fused) {
  if (!al) {
    de_align_instance<G>(st, grid, smem, x_td, ld, W, clips, n_clips, qtile64_prefix, align, soft, fuse, q, k, pld, n_sc, rnorm,
                         v, fused);
    return;
  }
  DeAlignOut o = *al;
  o.pbias = align == NISQA_DE_ALIGN_BAHDANAU ? vb : 0.f;
  de_align_instance<G>(st, grid, smem, x_td, ld, W, clips, n_clips, qtile64_prefix, align, soft, fuse, q, k, pld, n_sc, rnorm,
                       v, fused, o);
}

size_t de_align_work_floats(int W, int align, int n_rows) {
  const int ld = (W + 63) / 64 * 64;
  return (size_t)n_rows * (align == NISQA_DE_ALIGN_LUONG ? ld : align == NISQA_DE_ALIGN_BAHDANAU ? 256 : align == NISQA_DE_ALIGN_COSINE ? 1 : 0);
}

int de_align_launches(int align) {
  return align == NISQA_DE_ALIGN_LUONG || align == NISQA_DE_ALIGN_BAHDANAU || align == NISQA_DE_ALIGN_COSINE ? 2 : 1;
}

void launch_de_align(cudaStream_t st, const float* x_td, int W, int n_rows, const ClipDesc* clips, int n_clips,
                     const int* qtile64_prefix, int n_qtiles, int align, int soft, int fuse, const DeAlignParams& A,
                     float* work, float* fused, const DeAlignOut* al) {
  const int NC = (W + 63) / 64, ld = 64 * NC;
  const float *q = x_td, *k = x_td;
  int pld = ld, n_sc = NC;
  if (align == NISQA_DE_ALIGN_LUONG) {               // yp = W y + b for every row
    launch_linear_tile(st, x_td, ld, A.wT, A.b, 0, work, ld, n_rows, ld, ld);
    k = work;
  } else if (align == NISQA_DE_ALIGN_BAHDANAU) {     // xq | yk = Wq x + bq | Wy y + by for every row
    launch_linear_tile(st, x_td, ld, A.wqyT, A.bqy, 0, work, 256, n_rows, ld, 256);
    q = work; k = work + 128; pld = 256; n_sc = 2;
  } else if (align == NISQA_DE_ALIGN_COSINE) {
    row_rnorm_kernel<<<(n_rows + 7) / 8, 256, 0, st>>>(x_td, ld, W, n_rows, work);
  }
  // output chunks per soft CTA: NC up to 4 in one group, 5..8 in two
  const int G = !soft ? 1 : NC <= 4 ? NC : (NC + 1) / 2;
  const dim3 grid(n_qtiles, soft ? (NC + G - 1) / G : 1);
  const int smem = de_smem_bytes(n_sc);
  switch (G) {
    case 1: de_align_select<1>(al, st, grid, smem, x_td, ld, W, clips, n_clips, qtile64_prefix, align, soft, fuse, q, k, pld, n_sc, work, A.v, A.vb, fused); break;
    case 2: de_align_select<2>(al, st, grid, smem, x_td, ld, W, clips, n_clips, qtile64_prefix, align, soft, fuse, q, k, pld, n_sc, work, A.v, A.vb, fused); break;
    case 3: de_align_select<3>(al, st, grid, smem, x_td, ld, W, clips, n_clips, qtile64_prefix, align, soft, fuse, q, k, pld, n_sc, work, A.v, A.vb, fused); break;
    default: de_align_select<4>(al, st, grid, smem, x_td, ld, W, clips, n_clips, qtile64_prefix, align, soft, fuse, q, k, pld, n_sc, work, A.v, A.vb, fused); break;
  }
}

void launch_seg_feats(cudaStream_t st, const float* mel, int n_mels, int seg_len, int ld, const int* seg_frame0,
                      const float* seg_thr, const float* bn, int n_seg, float* out) {
  if (n_seg > 0) seg_feats_kernel<<<n_seg, 256, 0, st>>>(mel, n_mels, seg_len, ld, seg_frame0, seg_thr, bn, n_seg, out);
}

void launch_linear_tile(cudaStream_t st, const float* X, int ldx, const float* WT, const float* bias, int relu, float* Y, int ldy,
                        int n_rows, int K, int N) {
  static unsigned long long cfg = 0;
  const int smem = kLinSmemFloats * 4;
  if (first_launch_on_device(cfg)) cudaFuncSetAttribute(linear_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  const dim3 grid((n_rows + kT - 1) / kT, N / kT);
  linear_tile_kernel<<<grid, kNT, smem, st>>>(X, ldx, WT, bias, relu, Y, ldy, n_rows, K, N);
}

void launch_de_finalize(cudaStream_t st, const ClipDesc* clips, int n_clips, int n_out, float* scores) {
  de_finalize_kernel<<<(n_clips + 127) / 128, 128, 0, st>>>(clips, n_clips, n_out, scores);
}

template <int NC>
void td_sa_instance(cudaStream_t st, const float* x_in, const float* qkv, const ClipDesc* clips, int n_clips,
                    const int* qtile64_prefix, int n_qtiles, const SaLayerParams& P, int F, float* x_out,
                    const float* next_qkvT, const float* next_qkvb, float qscale, float* qkv_next,
                    const PoolHeadParams& H, int n_heads, float* logits) {
  static unsigned long long cfg = 0;
  const int smem = TdShape<NC>::kSaFloats * 4;
  if (first_launch_on_device(cfg)) cudaFuncSetAttribute(td_sa_kernel<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  td_sa_kernel<NC><<<n_qtiles, kNT, smem, st>>>(x_in, qkv, clips, n_clips, qtile64_prefix, P, F, x_out,
                                                next_qkvT, next_qkvb, qscale, qkv_next, H, n_heads, logits);
}
void launch_td_sa(cudaStream_t st, int nc, const float* x_in, const float* qkv, const ClipDesc* clips, int n_clips,
                  const int* qtile64_prefix, int n_qtiles, const SaLayerParams& P, int F, float* x_out,
                  const float* next_qkvT, const float* next_qkvb, float qscale, float* qkv_next,
                  const PoolHeadParams& H, int n_heads, float* logits) {
  switch (nc) {
    case 1: td_sa_instance<1>(st, x_in, qkv, clips, n_clips, qtile64_prefix, n_qtiles, P, F, x_out, next_qkvT, next_qkvb, qscale, qkv_next, H, n_heads, logits); break;
    case 2: td_sa_instance<2>(st, x_in, qkv, clips, n_clips, qtile64_prefix, n_qtiles, P, F, x_out, next_qkvT, next_qkvb, qscale, qkv_next, H, n_heads, logits); break;
    case 3: td_sa_instance<3>(st, x_in, qkv, clips, n_clips, qtile64_prefix, n_qtiles, P, F, x_out, next_qkvT, next_qkvb, qscale, qkv_next, H, n_heads, logits); break;
    case 4: td_sa_instance<4>(st, x_in, qkv, clips, n_clips, qtile64_prefix, n_qtiles, P, F, x_out, next_qkvT, next_qkvb, qscale, qkv_next, H, n_heads, logits); break;
  }
}

}  // namespace nisqa

// frontend.cu - PCM -> mel dB  (reference nisqa/NISQA_lib.py:2308-2330 via librosa 0.8.1
// stft / filters.mel / amplitude_to_db; restated in oracle/librosa_compat.py).
//
// One CTA (4 warps) per PAIR of STFT frames of one clip.  The two real frames are packed as
// z = a + i*b into one complex transform.  Only win <= 1024*Q of the 4096 inputs are non-zero
// (Hann window zero-padded to n_fft), and a circular shift does not change |X|, so the
// 4096-point DFT is computed as a radix-4 decimation-in-frequency step whose butterflies
// collapse to a twiddle multiply, followed by four independent 1024-point FFTs (one per warp,
// residue r = k mod 4).  Each 1024-point FFT is two in-register radix-32 passes with one
// shared-memory transpose.  Then, fused per mel band: unpack the two real spectra, |.|, sparse
// mel (band-major CSR), 10*log10(max(1e-8, M^2)), and a per-clip atomic max for the top_db
// clamp, which is applied by the consumers (conv1 / stage dump) as max(dB, clipmax - 80).
// Grid: x = frame pair, y = clip.
#include "common.cuh"
#include "f32x2.cuh"

// experiment switches (-DNAME=value when building a variant library); the defaults are the variants the kernel is tuned with
#ifndef NISQA_FE_PK_FFT
#define NISQA_FE_PK_FFT 0      // butterflies / twiddle products as packed FADD2 / FMUL2 / FFMA2
#endif
#ifndef NISQA_FE_PK_MAG
#define NISQA_FE_PK_MAG 0      // magnitude stage with packed adds
#endif
#ifndef NISQA_FE_DIT
#define NISQA_FE_DIT 1         // 32-point transforms as decimation in time with fused twiddle butterflies (6 FMAs instead of 8 FP instructions)
#endif
#ifndef NISQA_FE_MEL
#define NISQA_FE_MEL 2         // 0: scalar band loop unrolled by 4, 1: rolled packed loop, 2: packed loop unrolled by 4
#endif

namespace nisqa {

// e^{-2 pi i k / 32}, k = 0..15
__device__ __forceinline__ float2 w32(int k) {
  switch (k) {
    case 0:  return make_float2(1.0f, 0.0f);
    case 1:  return make_float2(0.98078528040323043f, -0.19509032201612825f);
    case 2:  return make_float2(0.92387953251128674f, -0.38268343236508978f);
    case 3:  return make_float2(0.83146961230254524f, -0.55557023301960218f);
    case 4:  return make_float2(0.70710678118654757f, -0.70710678118654757f);
    case 5:  return make_float2(0.55557023301960229f, -0.83146961230254524f);
    case 6:  return make_float2(0.38268343236508984f, -0.92387953251128674f);
    case 7:  return make_float2(0.19509032201612833f, -0.98078528040323043f);
    case 8:  return make_float2(0.0f, -1.0f);
    case 9:  return make_float2(-0.19509032201612819f, -0.98078528040323043f);
    case 10: return make_float2(-0.38268343236508973f, -0.92387953251128674f);
    case 11: return make_float2(-0.55557023301960196f, -0.83146961230254535f);
    case 12: return make_float2(-0.70710678118654746f, -0.70710678118654757f);
    case 13: return make_float2(-0.83146961230254535f, -0.55557023301960218f);
    case 14: return make_float2(-0.92387953251128674f, -0.38268343236508989f);
    default: return make_float2(-0.98078528040323043f, -0.19509032201612861f);
  }
}

__host__ __device__ constexpr int rev5(int i) {
  return ((i & 1) << 4) | ((i & 2) << 2) | (i & 4) | ((i & 8) >> 2) | ((i & 16) >> 4);
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// In-register 32-point forward DFT, decimation in frequency: X[rev5(i)] ends up in x[i].  Complex values are packed
// (re, im) register pairs (f32x2.cuh): a butterfly's sum / difference is one FADD2 each, a twiddle product FMUL2 + FFMA2;
// the -i products are formed from the scalar halves (two FADDs, no multiply).
__device__ __forceinline__ void fft32(f2 (&x)[32]) {
#pragma unroll
  for (int half = 16; half >= 1; half >>= 1) {
#pragma unroll
    for (int base = 0; base < 32; base += 2 * half) {
#pragma unroll
      for (int j = 0; j < half; ++j) {
        const int k = j * (16 / half);
#if NISQA_FE_PK_FFT
        const f2 a = x[base + j], b = x[base + j + half];
        x[base + j] = add2(a, b);
        if (k == 0) {
          x[base + j + half] = sub2(a, b);
        } else if (k == 8) {                       // (a - b) * (-i) = (d.y, -d.x)
          const float2 af = upk(a), bf = upk(b);
          x[base + j + half] = pk(af.y - bf.y, bf.x - af.x);
        } else {
          const float2 w = w32(k);
          x[base + j + half] = cmul2(sub2(a, b), pk(w.x, w.y), pk(-w.y, w.x));
        }
#else
        const float2 a = upk(x[base + j]), b = upk(x[base + j + half]);
        x[base + j] = pk(a.x + b.x, a.y + b.y);
        const float2 d = make_float2(a.x - b.x, a.y - b.y);
        if (k == 0) x[base + j + half] = pk(d);
        else if (k == 8) x[base + j + half] = pk(d.y, -d.x);
        else x[base + j + half] = pk(cmul(d, w32(k)));
#endif
      }
    }
  }
}

// The same transform as decimation in TIME: input n sits at x[rev5(n)], X[k] ends up in x[k].  A butterfly with a
// non-trivial twiddle is out1 = a + w b (4 FMAs), out2 = 2 a - out1 (2 FMAs) instead of add, subtract and a 4-instruction
// complex product; 34 of the 80 butterflies of a 32-point transform have one.
// One stage per template instance: every loop has a compile-time trip count, so the array indices are constants and
// `x` stays in registers (a stage loop over `half` is not fully unrolled by the sm_90 compiler, which puts x in local memory).
template <int HALF>
__device__ __forceinline__ void fft32_dit_stage(f2 (&x)[32]) {
  constexpr int half = HALF;
#pragma unroll
    for (int base = 0; base < 32; base += 2 * half) {
#pragma unroll
      for (int j = 0; j < half; ++j) {
        const int k = j * (16 / half);                 // twiddle W_32^k = e^{-2 pi i j / (2 half)}
        const float2 a = upk(x[base + j]), b = upk(x[base + j + half]);
        if (k == 0) {
          x[base + j] = pk(a.x + b.x, a.y + b.y);
          x[base + j + half] = pk(a.x - b.x, a.y - b.y);
        } else if (k == 8) {                            // w = -i: w b = (b.y, -b.x)
          x[base + j] = pk(a.x + b.y, a.y - b.x);
          x[base + j + half] = pk(a.x - b.y, a.y + b.x);
        } else {
          const float2 w = w32(k);
          const float ox = fmaf(w.x, b.x, fmaf(-w.y, b.y, a.x));
          const float oy = fmaf(w.x, b.y, fmaf(w.y, b.x, a.y));
          x[base + j] = pk(ox, oy);
          x[base + j + half] = pk(fmaf(2.0f, a.x, -ox), fmaf(2.0f, a.y, -oy));
        }
      }
    }
}
__device__ __forceinline__ void fft32_dit(f2 (&x)[32]) {
  fft32_dit_stage<1>(x);
  fft32_dit_stage<2>(x);
  fft32_dit_stage<4>(x);
  fft32_dit_stage<8>(x);
  fft32_dit_stage<16>(x);
}

// slot of input / output index i in the register array handed to the 32-point transform
__host__ __device__ constexpr int fe_in(int i) { return NISQA_FE_DIT ? rev5(i) : i; }
__host__ __device__ constexpr int fe_out(int i) { return NISQA_FE_DIT ? i : rev5(i); }
__device__ __forceinline__ void fe_fft32(f2 (&x)[32]) {
#if NISQA_FE_DIT
  fft32_dit(x);
#else
  fft32(x);
#endif
}

__device__ __forceinline__ int reflect_index(int i, int n) {
  // numpy.pad(mode='reflect') index map, valid for any i (repeated reflection when the pad
  // is longer than the signal)
  if ((unsigned)i < (unsigned)n) return i;      // interior frames: no reflection
  if (n <= 1) return 0;
  const int period = 2 * n - 2;
  int m = i % period;
  if (m < 0) m += period;
  return (m < n) ? m : period - m;
}

// One step of a multi-value butterfly reduction across the lanes: lane L keeps slot i or i + O (bit O of L / S) and sends
// the other to its partner at lane distance O * S.  A template per step keeps the trip counts constant, so that `v`
// stays in registers (a loop over O is not fully unrolled by the sm_90 compiler, which puts v in local memory).
template <int O, int S = 1, int N>
__device__ __forceinline__ void fold_step(float (&v)[N], int lane) {
  const bool up = (lane & (O * S)) != 0;
#pragma unroll
  for (int i = 0; i < O; ++i) {
    const float lo = v[i], hi = v[i + O];
    v[i] = sel(up, hi, lo) + __shfl_xor_sync(0xffffffffu, sel(up, lo, hi), O * S);
  }
}
template <int O, int S = 1, int N>
__device__ __forceinline__ void fold_step(f2 (&v)[N], int lane) {
  const bool up = (lane & (O * S)) != 0;
#pragma unroll
  for (int i = 0; i < O; ++i) {
    const f2 lo = v[i], hi = v[i + O];
    v[i] = add2(sel(up, hi, lo), __shfl_xor_sync(0xffffffffu, sel(up, lo, hi), O * S));
  }
}

template <typename T> __device__ __forceinline__ float sample_to_float(T v);
template <> __device__ __forceinline__ float sample_to_float<short>(short v) {
  return (float)v * (1.0f / 32768.0f);   // libsndfile PCM16 -> float
}
template <> __device__ __forceinline__ float sample_to_float<float>(float v) { return v; }

constexpr int kFeThreads = 128;
constexpr int kScratchPerWarp = 32 * 33 + 4;      // float2 elements: padded transpose tile (+4: the
                                                  // four residue planes start 8 banks apart)

__host__ __device__ constexpr int fe_region0_bytes(int Q) { return 1024 * Q * 8; }
int frontend_smem_bytes(int Q) { return fe_region0_bytes(Q) + 4 * kScratchPerWarp * 8; }

// ---- shared pieces of the two front-end kernels ---------------------------------------------
// 1024-point FFT of one residue plane: x[j] = input n = lane + 32 j (already twiddled by
// W_4096^(r n)); result Z_r[m] is left in tile[m] (m = 0..1023).  tw2x[q][lane] = (t.x, t.y, -t.y, t.x), t = W_1024^(lane q):
// both operand forms of the packed complex product in one 16-byte load.
__device__ __forceinline__ void fft1024_plane(f2 (&x)[32], float2* tile_, int lane,
                                              const float4* __restrict__ tw2x) {
  // x[fe_in(j)] = input n = lane + 32 j on entry
  f2* tile = reinterpret_cast<f2*>(tile_);
  fe_fft32(x);                                   // A_l[q] at x[fe_out(q)]
#pragma unroll
  for (int q = 0; q < 32; ++q) {
    f2 v = x[fe_out(q)];
    if (q != 0) {
#if NISQA_FE_PK_FFT
      const float4 t = __ldg(tw2x + q * 32 + lane);                        // W_1024^(l q), coalesced
      v = cmul2(v, pk(t.x, t.y), pk(t.z, t.w));
#else
      const float2 t = __ldg(reinterpret_cast<const float2*>(tw2x) - 1024 + q * 32 + lane);   // the float2 table sits in front
      v = pk(cmul(upk(v), t));
#endif
    }
    tile[lane * 33 + q] = v;
  }
  __syncwarp();
#pragma unroll
  for (int l = 0; l < 32; ++l) x[fe_in(l)] = tile[l * 33 + lane];
  __syncwarp();
  fe_fft32(x);                                   // Z_r[lane + 32 p] at x[fe_out(p)]
#pragma unroll
  for (int p = 0; p < 32; ++p) tile[lane + 32 * p] = x[fe_out(p)];
}

// Fused unpack of the two real spectra, |.|, sparse mel, dB for the 12 bands of this warp
// (b = warp + 4*slot).  Lanes stride over a band's bins and keep one partial sum per (slot, frame);
// the 24 partials are reduced across the warp with ONE multi-value butterfly (31 shuffles instead of
// 24 x 5): at the step with offset o the 2*o live values are paired (i, i+o), a lane whose bit o is set
// keeps the upper one and sends the lower one, so lane L ends up with the total of value index L =
// (slot L>>1, frame L&1) and one log10f serves the whole warp.  A bin belongs to two adjacent
// triangles, so its magnitudes are formed twice - cheaper than a shared-memory round trip.
// Returns this lane's dB value (or -inf) for the clip maximum.
__device__ __forceinline__ float mel_bands(const float2* scratch, const int* band_meta,
                                           const float* __restrict__ weights, int warp, int lane,
                                           bool validB, float* __restrict__ mel_row0 /*frame A row*/) {
  float v[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = 0.f;
#pragma unroll
  for (int slot = 0; slot < kMels / 4; ++slot) {
    const int b = warp + slot * 4;
    // band rows are zero-padded to a multiple of 32 weights (engine build_fb): warp-uniform trip
    // count, no divergence, every lane loads unconditionally (the padded bins stay inside the planes)
    const int beg = band_meta[b], iters = (band_meta[b + 1] - beg) >> 5;
    const int k = band_meta[kMels + 1 + b] + lane;
    const int kk = (kNfft - k) & (kNfft - 1);
    // Z planes: bin k lives at plane (k & 3), slot (k >> 2); k advances by 32 per iteration,
    // so both indices move by +-8 and the plane never changes.
    const float2* pk = scratch + (k & 3) * kScratchPerWarp + (k >> 2);
    const float2* pn = scratch + (kk & 3) * kScratchPerWarp + (kk >> 2);
    const float* wt = weights + beg + lane;
    float s0 = 0.f, s1 = 0.f;
#pragma unroll 2
    for (int it = 0; it < iters; ++it) {
      const float w = __ldg(wt);
      const float2 zk = *pk, zn = *pn;
      wt += 32; pk += 8; pn -= 8;
      const float ar = zk.x + zn.x, ai = zk.y - zn.y;      // 2 * X_a[k]
      const float br = zk.y + zn.y, bi = zk.x - zn.x;      // 2 * X_b[k] (up to a unit factor)
      float ma, mb;
      asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(ma) : "f"(fmaf(ar, ar, ai * ai)));
      asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(mb) : "f"(fmaf(br, br, bi * bi)));
      s0 = fmaf(w, ma, s0);
      s1 = fmaf(w, mb, s1);
    }
    v[2 * slot] = s0;
    v[2 * slot + 1] = s1;
  }
  fold_step<16>(v, lane); fold_step<8>(v, lane); fold_step<4>(v, lane); fold_step<2>(v, lane); fold_step<1>(v, lane);
  float out = -INFINITY;
  const int my_slot = lane >> 1, f = lane & 1;
  if (lane < 2 * (kMels / 4) && (f == 0 || validB)) {
    const float sv = 0.5f * v[0];                          // the 1/2 of the real-pair unpacking
    const float p = sv * sv;
    out = 10.0f * log10f(fmaxf(p, 1e-8f));
    mel_row0[(size_t)f * kMels + warp + my_slot * 4] = out;
  }
  return out;
}

// ---- two-stage variant used by the pipelined kernel (round 2) ---------------------------------------------------
// Stage A (whole CTA): |X_a[k]|, |X_b[k]| of the two packed real frames for the bins that carry a filterbank weight
// (k < n_mag), each formed ONCE and written over Z[k] in its plane (Z[k] is read by the owner of bin k and, as a mirror,
// by the owner of bin 4096 - k >= 2048 > n_mag - 1 only: in place is race free; k = 2048 mirrors itself).
__device__ __forceinline__ void mag_stage(float2* scratch, int n_mag, int tid) {
  // k = tid + 128 it: plane (k & 3) = tid & 3 and slot (k >> 2) = (tid >> 2) + 32 it
  f2* pk_ = reinterpret_cast<f2*>(scratch + (tid & 3) * kScratchPerWarp + (tid >> 2));
  const int kk0 = (kNfft - tid) & (kNfft - 1);
  const f2* pn = reinterpret_cast<const f2*>(scratch + (kk0 & 3) * kScratchPerWarp + (kk0 >> 2));
  for (int k = tid; k < n_mag; k += kFeThreads) {
    const f2 zk = *pk_, zn = *pn;
    float ma, mb;
#if NISQA_FE_PK_MAG
    const f2 sm = add2(zk, zn);                            // (2 Re X_a[k], 2 Re X_b[k])
    const float2 df = upk(sub2(zk, zn));                   // (-+2 Im X_b[k], 2 Im X_a[k])
    const float2 pw = upk(mul2(sm, sm));
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(ma) : "f"(fmaf(df.y, df.y, pw.x)));
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(mb) : "f"(fmaf(df.x, df.x, pw.y)));
#else
    {
      const float2 k_ = upk(zk), n_ = upk(zn);
      const float ar = k_.x + n_.x, ai = k_.y - n_.y;      // 2 * X_a[k]
      const float br = k_.y + n_.y, bi = k_.x - n_.x;      // 2 * X_b[k] (up to a unit factor)
      asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(ma) : "f"(fmaf(ar, ar, ai * ai)));
      asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(mb) : "f"(fmaf(br, br, bi * bi)));
    }
#endif
    *pk_ = pk(ma, mb);
    pk_ += 32; pn -= 32;                                    // (tid = 0, it = 0: k = kk = 0 reads the same slot twice)
    if (k == 0) pn += 1024;                                 // 4096 - 0 wraps to bin 0; from k = 128 on the mirror is 3968 - ...
  }
}

// Stage B: the 12 bands of this warp as weighted sums of the staged magnitudes, then the same multi-value butterfly
// reduction and dB as mel_bands.  `pscale` = 2^-30 for PCM16 input fed as raw integers (|X| scales by 2^15 exactly).
__device__ __forceinline__ float mel_bands_staged(const float2* scratch, const int* band_meta,
                                                  const float* __restrict__ weights, int warp, int lane,
                                                  bool validB, float pscale, float* __restrict__ mel_row0) {
  // v[i]: packed (frame A, frame B) partial sums of slot i in this lane.  The band loop is kept rolled: one weight load,
  // one magnitude pair, one FFMA2 per 32 bins and lane; trip counts (1 .. ~10 rows per band) are warp uniform.
  f2 v[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = 0ull;
#pragma unroll
  for (int slot = 0; slot < kMels / 4; ++slot) {
    const int b = warp + slot * 4;
    const int beg = band_meta[b], end = band_meta[b + 1];
    const int k = band_meta[kMels + 1 + b] + lane;
    const f2* pm = reinterpret_cast<const f2*>(scratch + (k & 3) * kScratchPerWarp + (k >> 2));
    const float* wt = weights + beg + lane;
    // padded bins (weight 0) may hold raw spectrum values: finite, times 0
#if NISQA_FE_MEL == 0
    float s0 = 0.f, s1 = 0.f;
#pragma unroll 4
    for (int it = (end - beg) >> 5; it > 0; --it, wt += 32, pm += 8) {
      const float w = __ldg(wt);
      const float2 m = upk(*pm);
      s0 = fmaf(w, m.x, s0);
      s1 = fmaf(w, m.y, s1);
    }
    v[slot] = pk(s0, s1);
#elif NISQA_FE_MEL == 1
    f2 acc = 0ull;
#pragma unroll 1
    for (int it = (end - beg) >> 5; it > 0; --it, wt += 32, pm += 8) acc = fma2(bc(__ldg(wt)), *pm, acc);
    v[slot] = acc;
#else
    f2 acc = 0ull;
#pragma unroll 4
    for (int it = (end - beg) >> 5; it > 0; --it, wt += 32, pm += 8) acc = fma2(bc(__ldg(wt)), *pm, acc);
    v[slot] = acc;
#endif
  }
  // multi-value butterfly over the 12 (padded to 16) packed values: after the steps with lane offsets 16, 8, 4, 2 lane L
  // holds the value of slot (L >> 1) & ... summed over 16 lanes; the last step adds the partner lane (L ^ 1)
  fold_step<8, 2>(v, lane); fold_step<4, 2>(v, lane); fold_step<2, 2>(v, lane); fold_step<1, 2>(v, lane);
  const float2 tot = upk(add2(v[0], __shfl_xor_sync(0xffffffffu, v[0], 1)));
  // lane L now holds slot s(L) = bit-reversal free index: bits 4..1 of L select the slot (offset 16 -> +8, 8 -> +4, ...)
  float out = -INFINITY;
  const int my_slot = lane >> 1, f = lane & 1;
  if (my_slot < kMels / 4 && (f == 0 || validB)) {
    const float sv = 0.5f * (f == 0 ? tot.x : tot.y);
    const float p = (sv * sv) * pscale;
    out = 10.0f * log10f(fmaxf(p, 1e-8f));
    mel_row0[(size_t)f * kMels + warp + my_slot * 4] = out;
  }
  return out;
}

// ---- generic kernel: one CTA per frame pair, any window length (win <= 1024*Q <= n_fft) ------
template <typename T>
__global__ void __launch_bounds__(kFeThreads, 5)
frontend_kernel(const T* __restrict__ pcm, const ClipDesc* __restrict__ clips, int n_clips,
                const FbTables* __restrict__ fbs,
                const float2* __restrict__ tw1 /*[3][32][32]: W4096^(r*(lane+32j))*/,
                const float4* __restrict__ tw2 /*[32][32]: W1024^(lane*q) as (x, y, -y, x)*/, float* __restrict__ mel,
                unsigned* __restrict__ clipmax, int Q) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2* zin = reinterpret_cast<float2*>(smem_raw);                     // [1024*Q] packed input
  float2* scratch = reinterpret_cast<float2*>(smem_raw + fe_region0_bytes(Q));
  __shared__ int band_meta[2 * kMels + 1];        // [0..48] CSR offsets, [49..96] first bin per band

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // grid: x = frame pair within the clip, y = clip (no search, no dependent loads)
  const int c = blockIdx.y;
  const ClipDesc cd = clips[c];
  const int tA = 2 * blockIdx.x;
  if (tA >= cd.n_frames) return;
  const FbTables fb = fbs[cd.fb_id];
  const int tB = tA + 1;
  const bool validB = tB < cd.n_frames;
  const T* y = pcm + cd.pcm_off;
  if (tid <= kMels) band_meta[tid] = __ldg(fb.band_start + tid);
  else if (tid < 2 * kMels + 1) band_meta[tid] = __ldg(fb.band_k0 + tid - kMels - 1);

  // ---- a. windowed, reflect-padded frame pair -> zin  (8 elements per thread per 1024 chunk,
  //         all loads of a chunk issued before they are consumed)
  for (int q0 = 0; q0 < Q; ++q0) {
    float wv[8], sa[8], sb[8];
    const int ia0 = cd.s0 + tA * cd.hop + q0 * 1024 + tid;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int n = q0 * 1024 + tid + i * kFeThreads;
      wv[i] = 0.f; sa[i] = 0.f; sb[i] = 0.f;
      if (n < cd.win) {
        wv[i] = __ldg(fb.window + n);
        const int ia = ia0 + i * kFeThreads;
        sa[i] = sample_to_float<T>(y[reflect_index(ia, cd.n_samples)]);
        if (validB) sb[i] = sample_to_float<T>(y[reflect_index(ia + cd.hop, cd.n_samples)]);
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i)
      zin[q0 * 1024 + tid + i * kFeThreads] = make_float2(wv[i] * sa[i], wv[i] * sb[i]);
  }
  __syncthreads();

  // ---- b. warp r: 1024-point FFT of the residue-r subsequence
  {
    const int r = warp;
    f2 x[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int n = lane + 32 * j;
      float2 v = zin[n];
      for (int q = 1; q < Q; ++q) {               // general radix-4 DIF butterfly (Q==1: none)
        const float2 u = zin[n + 1024 * q];
        switch ((r * q) & 3) {                    // u * (-i)^(r q)
          case 0: v.x += u.x; v.y += u.y; break;
          case 1: v.x += u.y; v.y -= u.x; break;
          case 2: v.x -= u.x; v.y -= u.y; break;
          default: v.x -= u.y; v.y += u.x; break;
        }
      }
      if (r != 0) v = cmul(v, __ldg(tw1 + ((r - 1) * 32 + j) * 32 + lane));   // coalesced per-lane table
      x[fe_in(j)] = pk(v);
    }
    fft1024_plane(x, scratch + r * kScratchPerWarp, lane, tw2);
  }
  __syncthreads();

  // ---- c. mel + dB + clip max
  float wmax = mel_bands(scratch, band_meta, fb.weights, warp, lane, validB,
                         mel + (size_t)(cd.frame_off + tA) * kMels);
  wmax = warp_max(wmax);
  if (lane == 0 && wmax > -INFINITY) atomicMax(clipmax + c, f2key(wmax));
}

// ---- pipelined kernel for win <= 1024 and hop + win <= 1536 (every standard rate up to 51.2 kHz)
// One CTA walks kPairsPerCta consecutive frame pairs of one clip, so the dependent prologue loads
// (ClipDesc -> filterbank tables) are paid once per 8 pairs, and the hop + win raw samples of pair
// p+1 are fetched with cp.async (16-byte chunks, no registers) into a two-slot shared-memory ring
// while pair p is transformed: the global-load latency that opens every pair in the generic kernel
// (46 % of its stall samples) is off the critical path.  Pairs that touch the reflect padding
// (the first / last one or two of a clip) fill their slot with plain indexed loads instead.
// The FFT input stage reads samples straight from the ring (window via the read-only path).
constexpr int kPairsPerCta = 2;
constexpr int kSpanMax = 1536;                    // hop + win limit of this kernel
template <typename T> __host__ __device__ constexpr int pp_slot_bytes() {
  return ((kSpanMax + 16 / (int)sizeof(T)) * (int)sizeof(T) + 15) / 16 * 16;
}
#ifndef NISQA_FE_CTAS
#define NISQA_FE_CTAS 6        // PCM16 input: resident CTAs per SM the kernel is built for (6 = one sample slot, <= 80 registers)
#endif
// PCM16 with six CTAs per SM: ONE sample slot (the slot is only live during the input stage: the next pair's copy is issued
// behind the barrier that follows the FFT, still a whole mel stage ahead of its use) - 37.4 KB of shared memory per CTA
template <typename T> __host__ __device__ constexpr int pp_slots() { return (sizeof(T) == 2 && NISQA_FE_CTAS >= 6) ? 1 : 2; }
template <typename T> constexpr int pp_smem_bytes() { return pp_slots<T>() * pp_slot_bytes<T>() + 4 * kScratchPerWarp * 8; }

template <typename T>
__device__ __forceinline__ void pp_issue_pair(const T* __restrict__ y, int a, int span, int n_samples,
                                              T* slot, int tid) {
  if (a >= 0 && a + span <= n_samples) {
    const char* src = reinterpret_cast<const char*>(y + a);
    const int mis = (int)(reinterpret_cast<uintptr_t>(src) & 15);
    src -= mis;
    const int chunks = (mis + span * (int)sizeof(T) + 15) >> 4;
    const unsigned dst = (unsigned)__cvta_generic_to_shared(slot);
    for (int i = tid; i < chunks; i += kFeThreads)
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 16 * i), "l"(src + 16 * i) : "memory");
  } else {
    for (int i = tid; i < span; i += kFeThreads) slot[i] = y[reflect_index(a + i, n_samples)];
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

template <typename T>
__global__ void __launch_bounds__(kFeThreads, (sizeof(T) == 2 && NISQA_FE_CTAS >= 6) ? 6 : 5)
frontend_pp_kernel(const T* __restrict__ pcm, const ClipDesc* __restrict__ clips,
                   const FbTables* __restrict__ fbs, const float2* __restrict__ tw1,
                   const float4* __restrict__ tw2, float* __restrict__ mel, unsigned* __restrict__ clipmax,
                   int ppc /*frame pairs per CTA*/) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int NSLOT = pp_slots<T>();
  float2* scratch = reinterpret_cast<float2*>(smem_raw + NSLOT * pp_slot_bytes<T>());
  __shared__ int band_meta[2 * kMels + 1];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int c = blockIdx.y;
  const ClipDesc cd = clips[c];
  const int n_pairs = (cd.n_frames + 1) >> 1;
  const int p0 = blockIdx.x * ppc;
  if (p0 >= n_pairs) return;
  const int p1 = min(p0 + ppc, n_pairs);
  const T* y = pcm + cd.pcm_off;
  const int span = cd.hop + cd.win;
  pp_issue_pair<T>(y, cd.s0 + 2 * p0 * cd.hop, span, cd.n_samples, reinterpret_cast<T*>(smem_raw), tid);
  const FbTables fb = fbs[cd.fb_id];
  if (tid <= kMels) band_meta[tid] = __ldg(fb.band_start + tid);
  else if (tid < 2 * kMels + 1) band_meta[tid] = __ldg(fb.band_k0 + tid - kMels - 1);

  const int r = warp;
  float wmax = -INFINITY;
  for (int p = p0; p < p1; ++p) {
    const int s = NSLOT == 2 ? (p - p0) & 1 : 0;
    const int a = cd.s0 + 2 * p * cd.hop;
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();                    // slot s complete and visible; planes of pair p-1 consumed
    if (NSLOT == 2 && p + 1 < p1)
      pp_issue_pair<T>(y, a + 2 * cd.hop, span, cd.n_samples,
                       reinterpret_cast<T*>(smem_raw + (s ^ 1) * pp_slot_bytes<T>()), tid);
    const bool validB = 2 * p + 1 < cd.n_frames;
    const bool interior = a >= 0 && a + span <= cd.n_samples;
    const int shift = interior ? (int)((reinterpret_cast<uintptr_t>(y + a) & 15) / sizeof(T)) : 0;
    const T* src = reinterpret_cast<const T*>(smem_raw + s * pp_slot_bytes<T>()) + shift;
    // input stage: ONE table load per element (window x residue twiddle, zero beyond the window), samples as raw
    // integers (PCM16: the 2^-15 of libsndfile's conversion is exact and is applied to the band power at the end),
    // loads of 4 elements in flight together; the sample index is clamped into the slot for n >= win
    // (an odd clip's last pair has no frame B: hopB = 0 transforms frame A twice, the copy is neither stored nor counted)
    f2 x[32];
    const int hopB = validB ? cd.hop : 0;
    const float2* wtab = fb.wtab + r * 1024 + lane;
    // PCM16: 1023 + hop + shift < the slot's 1544 elements (hop <= 512 whenever win <= 1024), unfilled elements are
    // finite integers under a zero window weight; float input could hold non-finite garbage there: clamped
    const int nmax = sizeof(T) == 2 ? 4096 : cd.win - 1;
    constexpr int CH = 4;
#pragma unroll
    for (int j0 = 0; j0 < 32; j0 += CH) {
      float2 wt[CH];
      float sa[CH], sb[CH];
#pragma unroll
      for (int u = 0; u < CH; ++u) {
        const int n = lane + 32 * (j0 + u);
        const int ni = sizeof(T) == 2 ? n : min(n, nmax);
        wt[u] = __ldg(wtab + 32 * (j0 + u));
        sa[u] = (float)src[ni];
        sb[u] = (float)src[ni + hopB];
      }
#pragma unroll
      for (int u = 0; u < CH; ++u)
        x[fe_in(j0 + u)] = pk(fmaf(sa[u], wt[u].x, -(sb[u] * wt[u].y)), fmaf(sa[u], wt[u].y, sb[u] * wt[u].x));
    }
    fft1024_plane(x, scratch + r * kScratchPerWarp, lane, tw2);
    __syncthreads();                    // all four planes written (and every warp is past the input stage: the slot is free)
    if (NSLOT == 1 && p + 1 < p1)
      pp_issue_pair<T>(y, a + 2 * cd.hop, span, cd.n_samples, reinterpret_cast<T*>(smem_raw), tid);
    mag_stage(scratch, fb.n_mag, tid);
    __syncthreads();                    // magnitudes staged
    wmax = fmaxf(wmax, mel_bands_staged(scratch, band_meta, fb.weights, warp, lane, validB,
                                        sizeof(T) == 2 ? 9.313225746154785e-10f : 1.0f,
                                        mel + (size_t)(cd.frame_off + 2 * p) * kMels));
  }
  wmax = warp_max(wmax);
  if (lane == 0 && wmax > -INFINITY) atomicMax(clipmax + c, f2key(wmax));
}

// Per-segment lookup rows, built once per pass after the front-end:
//   seg_frame0[s] = first mel row of segment s,  seg_thr[s] = clipmax(clip) - 80  (top_db)
__global__ void seg_table_kernel(const ClipDesc* __restrict__ clips, int n_clips,
                                 const int* __restrict__ seg_prefix,
                                 const unsigned* __restrict__ clipmax, int seg_hop, int n_seg,
                                 int* __restrict__ seg_frame0, float* __restrict__ seg_thr,
                                 int* __restrict__ seg_clip) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_seg) return;
  const int c = upper_slot(seg_prefix, n_clips, s);
  const ClipDesc cd = clips[c];
  seg_frame0[s] = cd.frame_off + (s - cd.seg_off) * seg_hop;
  seg_thr[s] = key2f(clipmax[c]) - 80.0f;
  seg_clip[s] = c;
}

// stage dump helper: mel[frame][48] -> per clip [48][n_frames] with the top_db clamp applied
__global__ void mel_dump_kernel(const float* __restrict__ mel, const ClipDesc* __restrict__ clips,
                                int n_clips, const unsigned* __restrict__ clipmax,
                                float* __restrict__ out) {
  const int c = blockIdx.y;
  const ClipDesc cd = clips[c];
  const float thr = key2f(clipmax[c]) - 80.0f;
  const int n = cd.n_frames * kMels;
  float* o = out + (size_t)cd.frame_off * kMels;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int b = i / cd.n_frames, t = i - b * cd.n_frames;
    o[i] = fmaxf(mel[(size_t)(cd.frame_off + t) * kMels + b], thr);
  }
}

// ------------------------------------------------------------------ host launchers
void launch_frontend(cudaStream_t st, const void* pcm, int fmt_f32, const ClipDesc* clips,
                     int n_clips, int max_pairs, const FbTables* fbs,
                     const float2* tw, float* mel, unsigned* clipmax, int Q, int max_span, int ppc) {
  const float2* tw1 = tw;               // [3][32][32]
  const float4* tw2 = reinterpret_cast<const float4*>(tw + 4 * 1024);    // [32][32] (x, y, -y, x)
  if (Q == 1 && max_span <= kSpanMax) { // the pipelined multi-pair kernel
    static unsigned long long configured = 0;
    if (first_launch_on_device(configured)) {
      cudaFuncSetAttribute(frontend_pp_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, pp_smem_bytes<float>());
      cudaFuncSetAttribute(frontend_pp_kernel<short>, cudaFuncAttributeMaxDynamicSharedMemorySize, pp_smem_bytes<short>());
    }
    if (ppc < 1) ppc = kPairsPerCta;
    const dim3 grid((max_pairs + ppc - 1) / ppc, n_clips);
    if (fmt_f32)
      frontend_pp_kernel<float><<<grid, kFeThreads, pp_smem_bytes<float>(), st>>>((const float*)pcm, clips, fbs, tw1, tw2, mel, clipmax, ppc);
    else
      frontend_pp_kernel<short><<<grid, kFeThreads, pp_smem_bytes<short>(), st>>>((const short*)pcm, clips, fbs, tw1, tw2, mel, clipmax, ppc);
    return;
  }
  const int smem = frontend_smem_bytes(Q);
  // the opt-in is per device (several engines - one per GPU - may live in one process): ask once per device
  // for the largest window this kernel supports (Q = 4: win up to n_fft)
  static unsigned long long configured = 0;
  if (first_launch_on_device(configured)) {
    cudaFuncSetAttribute(frontend_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, frontend_smem_bytes(4));
    cudaFuncSetAttribute(frontend_kernel<short>, cudaFuncAttributeMaxDynamicSharedMemorySize, frontend_smem_bytes(4));
  }
  const dim3 grid(max_pairs, n_clips);
  if (fmt_f32) {
    frontend_kernel<float><<<grid, kFeThreads, smem, st>>>(
        (const float*)pcm, clips, n_clips, fbs, tw1, tw2, mel, clipmax, Q);
  } else {
    frontend_kernel<short><<<grid, kFeThreads, smem, st>>>(
        (const short*)pcm, clips, n_clips, fbs, tw1, tw2, mel, clipmax, Q);
  }
}

void launch_seg_table(cudaStream_t st, const ClipDesc* clips, int n_clips, const int* seg_prefix,
                      const unsigned* clipmax, int seg_hop, int n_seg, int* seg_frame0,
                      float* seg_thr, int* seg_clip) {
  seg_table_kernel<<<(n_seg + 255) / 256, 256, 0, st>>>(clips, n_clips, seg_prefix, clipmax,
                                                        seg_hop, n_seg, seg_frame0, seg_thr,
                                                        seg_clip);
}

void launch_mel_dump(cudaStream_t st, const float* mel, const ClipDesc* clips, int n_clips,
                     const unsigned* clipmax, float* out) {
  dim3 grid(8, n_clips);
  mel_dump_kernel<<<grid, 256, 0, st>>>(mel, clips, n_clips, clipmax, out);
}

}  // namespace nisqa

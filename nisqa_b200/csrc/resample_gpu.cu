// resample_gpu.cu - sample-rate conversion of the ingest ON THE DEVICE (SURVEY.md 8f.2): what lb.load(path, sr=ms_sr)
// does at reference nisqa/NISQA_lib.py:2300-2304 for checkpoints with ms_sr != None - librosa 0.8.1 resample
// ('kaiser_best', fix=True, scale=False) = resampy's band-limited sinc interpolation with linear interpolation between
// the entries of a Kaiser-windowed sinc table.  Same arithmetic, in the same order, as the host routine
// (csrc/resample.cpp, bit-identical to the oracle's restatement): float64 weights, the float32 output element
// rounded after every addition, products and sums un-fused (__dmul_rn / __dadd_rn: the host code has no FMA).
//
// resampy advances its float64 time register by repeated addition (t_{k+1} = t_k + 1 / ratio); to stay bit-identical
// the registers are produced by one sequential chain per clip (resample_times_kernel: every 256th value goes to HBM),
// and every CTA of the interpolation kernel re-runs the 255 additions of its own chunk.  One thread per output sample
// then walks the two filter wings (~64 taps each when up-sampling, 64 / ratio when down-sampling): FP64-latency bound,
// 2 table loads per tap out of a 262 KB L2-resident table.  A 10 s clip takes ~2 ms of one SM's time instead of
// 0.28 s of a host core.
#include "common.cuh"
#include "launch.cuh"

namespace nisqa {

constexpr int kRsChunk = 256;

// one thread per clip: the sequential float64 chain of time registers, every kRsChunk-th value stored
__global__ void resample_times_kernel(const ResampleClip* __restrict__ clips, int n_clips, double* __restrict__ t_start) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_clips) return;
  const ResampleClip cl = clips[c];
  if (cl.copy) return;
  const double inc = 1.0 / cl.ratio;
  double t = 0.0;
  double* dst = t_start + cl.time_off;
  for (int k = 0; k < cl.n_out; ++k) {
    if ((k & (kRsChunk - 1)) == 0) dst[k / kRsChunk] = t;
    t = __dadd_rn(t, inc);
  }
}

template <typename T> __device__ __forceinline__ double rs_sample(const T* x, long long i);
template <> __device__ __forceinline__ double rs_sample<float>(const float* x, long long i) { return (double)x[i]; }
template <> __device__ __forceinline__ double rs_sample<short>(const short* x, long long i) {
  return (double)((float)x[i] * (1.0f / 32768.0f));       // libsndfile's PCM16 -> float32, as the host ingest does
}

// grid (chunks of 256 outputs, clips)
template <typename T>
__global__ void __launch_bounds__(kRsChunk)
resample_kernel(const T* __restrict__ raw, const ResampleClip* __restrict__ clips, const double* __restrict__ t_start,
                const double* __restrict__ win /*[nwin] right half of the windowed sinc*/, int nwin, int num_table,
                float* __restrict__ out) {
  __shared__ double t_reg[kRsChunk];
  const ResampleClip cl = clips[blockIdx.y];
  const int t0 = blockIdx.x * kRsChunk;
  if (t0 >= cl.n_fix) return;
  const int t = t0 + threadIdx.x;
  const T* x = raw + cl.in_off;
  float* y = out + cl.out_off;
  if (cl.copy) {
    if (t < cl.n_fix) y[t] = (float)rs_sample<T>(x, t);
    return;
  }
  if (threadIdx.x == 0) {
    const double inc = 1.0 / cl.ratio;
    double tr = t0 < cl.n_out ? t_start[cl.time_off + blockIdx.x] : 0.0;
    for (int k = 0; k < kRsChunk; ++k) { t_reg[k] = tr; tr = __dadd_rn(tr, inc); }
  }
  __syncthreads();
  if (t >= cl.n_fix) return;
  if (t >= cl.n_out) { y[t] = 0.f; return; }                     // fix_length: zero padding
  const double rs = cl.ratio < 1.0 ? cl.ratio : 1.0;             // the filter is scaled when down-sampling
  const double scale = rs;
  const long long index_step = (long long)(scale * num_table);
  const double time_register = t_reg[threadIdx.x];
  const long long nn = (long long)time_register;
  float acc = 0.f;
  double frac = __dmul_rn(scale, __dsub_rn(time_register, (double)nn));
  double index_frac = __dmul_rn(frac, (double)num_table);
  long long offset = (long long)index_frac;
  double eta = __dsub_rn(index_frac, (double)offset);
  {
    long long i_max = (nwin - offset) / index_step;
    if (nn + 1 < i_max) i_max = nn + 1;
    long long e = offset;
    for (long long i = 0; i < i_max; ++i, e += index_step) {
      const double w0 = __dmul_rn(win[e], rs);
      const double w1 = e + 1 < nwin ? __dmul_rn(win[e + 1], rs) : 0.0;
      const double d = e + 1 < nwin ? __dsub_rn(w1, w0) : 0.0;
      const double weight = __dadd_rn(w0, __dmul_rn(eta, d));
      acc = (float)__dadd_rn((double)acc, __dmul_rn(weight, rs_sample<T>(x, nn - i)));
    }
  }
  frac = __dsub_rn(scale, frac);
  index_frac = __dmul_rn(frac, (double)num_table);
  offset = (long long)index_frac;
  eta = __dsub_rn(index_frac, (double)offset);
  {
    long long k_max = (nwin - offset) / index_step;
    if ((long long)cl.n_in - nn - 1 < k_max) k_max = (long long)cl.n_in - nn - 1;
    long long e = offset;
    for (long long k = 0; k < k_max; ++k, e += index_step) {
      const double w0 = __dmul_rn(win[e], rs);
      const double w1 = e + 1 < nwin ? __dmul_rn(win[e + 1], rs) : 0.0;
      const double d = e + 1 < nwin ? __dsub_rn(w1, w0) : 0.0;
      const double weight = __dadd_rn(w0, __dmul_rn(eta, d));
      acc = (float)__dadd_rn((double)acc, __dmul_rn(weight, rs_sample<T>(x, nn + k + 1)));
    }
  }
  y[t] = acc;
}

void launch_resample(cudaStream_t st, const void* raw, int fmt_f32, const ResampleClip* clips, int n_clips, int max_fix,
                     double* t_start, const double* win, int nwin, int num_table, float* out) {
  resample_times_kernel<<<(n_clips + 31) / 32, 32, 0, st>>>(clips, n_clips, t_start);
  const dim3 grid((max_fix + kRsChunk - 1) / kRsChunk, n_clips);
  if (fmt_f32) resample_kernel<float><<<grid, kRsChunk, 0, st>>>((const float*)raw, clips, t_start, win, nwin, num_table, out);
  else resample_kernel<short><<<grid, kRsChunk, 0, st>>>((const short*)raw, clips, t_start, win, nwin, num_table, out);
}

}  // namespace nisqa

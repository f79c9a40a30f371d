// ingest.cu - device ingest of nisqa_predict_device_batch: the caller's strided [clips][channels][length] int16 / float32
// memory -> the packed mono PCM (16-sample aligned clips) the front end or the resampler reads.  It does on the device
// what the file ingest does on the host (csrc/wavio.cpp): a channel pick copies that channel, the mono mix is
// numpy.mean over float32 channels - int16 scaled by 1/32768 first, a sequential float32 sum in channel order, then a
// division by the channel count - with every operation rounded on its own (no FMA contraction), so the packed clips are
// bit for bit what the host path uploads.  Memory bound: one read and one write of every sample.
#include <algorithm>

#include "common.cuh"
#include "launch.cuh"
#include "windows.cuh"

namespace nisqa {

constexpr int kIngestThreads = 256;
constexpr int kIngestPerThread = 4;      // samples per thread and grid-stride step (grid.x capped below)

__device__ __forceinline__ float ingest_f32(const short* x, long long i) { return __fmul_rn((float)x[i], 1.0f / 32768.0f); }
__device__ __forceinline__ float ingest_f32(const float* x, long long i) { return x[i]; }

__device__ __forceinline__ bool ingest_row(const ClipDesc& c, long long* off, int* n, int* g) {
  *off = c.pcm_off; *n = c.n_samples; *g = c.src_clip;
  return c.n_frames > 0;                 // a skipped clip (too short / too long, or its pair's) is never read
}
__device__ __forceinline__ bool ingest_row(const ResampleClip& c, long long* off, int* n, int* g) {
  *off = c.in_off; *n = c.n_in; *g = c.src_clip;
  return c.n_in > 0;
}

template <class Tin, class Tout>
__device__ __forceinline__ void ingest_clip(const IngestSrc& s, long long b, int n, Tout* __restrict__ y) {
  const Tin* x = static_cast<const Tin*>(s.data) + b * s.clip_stride;
  const bool mix = s.n_channels > 1 && s.channel < 0;
  if (!mix && s.n_channels > 1) x += (long long)s.channel * s.channel_stride;
  const int step = gridDim.x * blockDim.x;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += step) {
    if constexpr (sizeof(Tout) == 2) {
      y[t] = x[t];                       // int16 out: an int16 source read from one channel
    } else if (!mix) {
      y[t] = ingest_f32(x, t);
    } else {
      float acc = 0.f;
      for (int c = 0; c < s.n_channels; ++c) acc = __fadd_rn(acc, ingest_f32(x, (long long)c * s.channel_stride + t));
      y[t] = __fdiv_rn(acc, (float)s.n_channels);
    }
  }
}

// grid (sample blocks, clips); each row names the clip of the sources it packs (src_clip, IngestSources order)
template <class Row>
__global__ void __launch_bounds__(kIngestThreads)
ingest_kernel(IngestSources src, const Row* __restrict__ rows, int out_f32, void* __restrict__ out) {
  long long off;
  int n, g;
  if (!ingest_row(rows[blockIdx.y], &off, &n, &g)) return;
  const IngestSrc s = g % src.n_src ? src.s[1] : src.s[0];     // (no dynamic index into the parameter struct: no stack)
  const long long b = g / src.n_src;
  if (out_f32) {
    float* y = static_cast<float*>(out) + off;
    if (s.f32) ingest_clip<float, float>(s, b, n, y);
    else ingest_clip<short, float>(s, b, n, y);
  } else {
    ingest_clip<short, short>(s, b, n, static_cast<short*>(out) + off);
  }
}

template <class Row>
static void launch_ingest_rows(cudaStream_t st, const IngestSources& src, const Row* rows, int n_clips,
                               long long max_n, int out_f32, void* out) {
  if (n_clips <= 0 || max_n <= 0) return;
  const long long per_block = (long long)kIngestThreads * kIngestPerThread;
  const dim3 grid((unsigned)std::min<long long>((max_n + per_block - 1) / per_block, 4096), n_clips);
  ingest_kernel<Row><<<grid, kIngestThreads, 0, st>>>(src, rows, out_f32, out);
}

// nisqa_predict_device_windows: each recording span of a pass packed once, however many windows read it; grid (sample
// blocks, spans)
__global__ void __launch_bounds__(kIngestThreads)
ingest_span_kernel(IngestSrc s, const WinSpan* __restrict__ spans, int out_f32, void* __restrict__ out) {
  const WinSpan sp = spans[blockIdx.y];
  if (sp.n_win <= 0) return;             // (no window of the span runs)
  s.data = static_cast<const char*>(s.data) + sp.src_off * (s.f32 ? 4 : 2);
  if (out_f32) {
    float* y = static_cast<float*>(out) + sp.pcm_off;
    if (s.f32) ingest_clip<float, float>(s, sp.src, sp.n_samples, y);
    else ingest_clip<short, float>(s, sp.src, sp.n_samples, y);
  } else {
    ingest_clip<short, short>(s, sp.src, sp.n_samples, static_cast<short*>(out) + sp.pcm_off);
  }
}

void launch_ingest_spans(cudaStream_t st, const IngestSrc& src, const WinSpan* spans, int n_spans, long long max_n,
                         int out_f32, void* out) {
  if (n_spans <= 0 || max_n <= 0) return;
  const long long per_block = (long long)kIngestThreads * kIngestPerThread;
  const dim3 grid((unsigned)std::min<long long>((max_n + per_block - 1) / per_block, 4096), n_spans);
  ingest_span_kernel<<<grid, kIngestThreads, 0, st>>>(src, spans, out_f32, out);
}

// Live feeds: feed b's chunk (clip b of the push) appended to its sample ring, samples t0 .. t0 + n_in - 1 at ring
// positions t mod R, and again at R + (t mod R) where that is below W (the mirror); grid (sample blocks, feeds).  Up to
// four contiguous runs, each converted by ingest_clip, so a ring sample is the sample the span ingest would pack.
template <class Tin, class Tout>
__device__ __forceinline__ void ingest_feed_runs(const IngestSrc& s, int b, const FeedPush& fp, const FeedGeom& g,
                                                 Tout* __restrict__ y) {
  const long long n = fp.n_in, u = fp.t0 % g.R, nA = min(n, (long long)g.R - u);
  auto run = [&](long long i0, long long len, long long at) {
    if (len <= 0) return;
    IngestSrc r = s;
    r.data = static_cast<const Tin*>(s.data) + i0;
    ingest_clip<Tin, Tout>(r, b, (int)len, y + at);
  };
  run(0, nA, u);                                       // up to the end of the ring
  run(nA, n - nA, 0);                                  // wrapped to its start
  run(0, min(nA, (long long)g.W - u), g.R + u);        // the mirror of positions below W
  run(nA, min(n - nA, (long long)g.W), g.R);
}

__global__ void __launch_bounds__(kIngestThreads)
ingest_feed_kernel(IngestSrc s, const FeedPush* __restrict__ push, FeedGeom g, int out_f32, void* __restrict__ ring) {
  const int b = blockIdx.y;
  const FeedPush fp = push[b];
  if (fp.n_in <= 0) return;
  const long long at = (long long)b * g.stride;
  if (out_f32) {
    float* y = static_cast<float*>(ring) + at;
    if (s.f32) ingest_feed_runs<float, float>(s, b, fp, g, y);
    else ingest_feed_runs<short, float>(s, b, fp, g, y);
  } else {
    ingest_feed_runs<short, short>(s, b, fp, g, static_cast<short*>(ring) + at);
  }
}

void launch_ingest_feed(cudaStream_t st, const IngestSrc& src, const FeedPush* push, int n_feeds, long long max_n,
                        const FeedGeom& g, int out_f32, void* ring) {
  if (n_feeds <= 0 || max_n <= 0) return;
  const long long per_block = (long long)kIngestThreads * kIngestPerThread;
  const dim3 grid((unsigned)std::min<long long>((max_n + per_block - 1) / per_block, 4096), n_feeds);
  ingest_feed_kernel<<<grid, kIngestThreads, 0, st>>>(src, push, g, out_f32, ring);
}

void launch_ingest(cudaStream_t st, const IngestSources& src, const ClipDesc* clips, int n_clips, long long max_n,
                   int out_f32, void* out) {
  launch_ingest_rows(st, src, clips, n_clips, max_n, out_f32, out);
}
void launch_ingest(cudaStream_t st, const IngestSources& src, const ResampleClip* clips, int n_clips, long long max_n,
                   int out_f32, void* out) {
  launch_ingest_rows(st, src, clips, n_clips, max_n, out_f32, out);
}

}  // namespace nisqa

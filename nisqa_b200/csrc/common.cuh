// common.cuh - shared device structs / helpers for the sm_90a NISQA kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nisqa {

// The shipped Mel-spectrogram shape: the only one the fused conv1 + conv2 kernel (conv_split.cu) and StandardCNN take.
// Every other kernel takes n_mels / seg_len from the engine (frontend.cu: one instance per band count).
constexpr int kMels = 48;        // ms_n_mels
constexpr int kSegLen = 15;      // ms_seg_length
constexpr int kNfft = 4096;      // ms_n_fft
constexpr int kBins = kNfft / 2 + 1;
constexpr int kSplitLead = 16;  // zero rows in front of segment 0 of an fp16 plane pair (conv_split.cu) >= the largest tap halo

// One row per clip of the current pass (device copy lives in HBM).
struct ClipDesc {
  long long pcm_off;   // element offset of the clip's first sample in the packed PCM buffer
  int n_samples;
  int fb_id;           // index of the per-sample-rate tables (window, filterbank)
  int hop, win;        // (int)(sr*hop_s), (int)(sr*win_s)  - reference lib:2308-2309
  int s0;              // sample index of window tap 0 of frame 0: lpad - n_fft/2
  int n_frames;        // 1 + n_samples / hop    (0 when the clip is skipped)
  int frame_off;       // first row of this clip in the mel buffer [total_frames][n_mels]
  int pair_off;        // first frame-pair work item of this clip
  int n_seg;           // segments ("n_wins" after seg_hop, lib:2271-2273)
  int seg_off;         // first segment row of this clip in the segment-major buffers
  int ref_clip;        // NISQA_DE, degraded clip c: the pass slot whose rows are its pair's reference (c + 1, or in a
                       // shared-reference call the slot of that reference's first pair in the pass)
  int src_clip;        // device ingest: the clip's position in IngestSources order (clip src_clip / n_src of source
                       // src_clip % n_src); in the struct's tail padding
};
static_assert(sizeof(ClipDesc) == 56, "ClipDesc: ref_clip and src_clip fill the layout of the former padding");

// Per-sample-rate front-end tables (device pointers).
struct FbTables {
  const float* window;     // [win] periodic Hann (float32 of scipy's float64 values)
  const int*   band_start; // [n_mels + 1] prefix offsets into weights
  const int*   band_k0;    // [n_mels] first FFT bin of each band
  const float* weights;    // concatenated non-zero runs, band-major
  const float2* wtab;      // [4][1024] window[n] * W_4096^(r n) (0 for n >= win): window and residue twiddle in one load
  int n_mag;               // bins 0 .. n_mag-1 carry a non-zero filterbank weight (magnitudes are formed for these only)
  int pad_;
};

// Kernel attributes (the dynamic shared-memory opt-in) are per device and several engines - one per GPU - may live
// in one process: true the first time it is called with `mask` while the calling thread's current device is active.
inline bool first_launch_on_device(unsigned long long& mask) {
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (mask & bit) return false;
  mask |= bit;
  return true;
}

// order-preserving float <-> uint key (for atomicMax over signed floats)
__device__ __forceinline__ unsigned f2key(float f) {
  unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key2f(unsigned k) {
  unsigned b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(b);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// largest i in [0, n) with prefix[i] <= x   (prefix is non-decreasing, prefix[0] == 0)
__device__ __forceinline__ int upper_slot(const int* __restrict__ prefix, int n, int x) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (__ldg(prefix + mid) <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

}  // namespace nisqa

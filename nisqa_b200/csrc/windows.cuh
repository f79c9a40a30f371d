// windows.cuh - the recording spans of nisqa_predict_device_windows, shared by the host runtime (engine.cu), the windows
// front end (frontend.cu) and the span ingest (ingest.cu).
#pragma once
#include <cuda_runtime.h>

namespace nisqa {

// Windows of a recording (nisqa_predict_device_windows): one row per run of consecutive windows of one recording in a
// pass.  Every window is also a ClipDesc row of the pass (its own bounds, mel rows and clip max); the span is the PCM
// those windows read, packed once.
struct WinSpan {
  long long pcm_off;   // element offset of the span's first sample (its first window's start) in the pass's PCM
  long long src_off;   // first sample of the span in its recording (model rate; the ingest reads from there)
  int src;             // the recording's index in the caller's batch (ingest)
  int n_samples;       // first window's start .. last window's end
  int clip0;           // the span's windows are ClipDesc rows clip0 .. ; window i starts at sample i * H of the span
  int n_win;           // leading windows the pass runs (only a recording's last window can be too short)
  int H, hf;           // window hop in samples and in mel frames (H = hf * hop)
  int W;               // window length in samples
  int pad_;
};

// Frame pairs p = 0 .. (n_frames + 1) / 2 - 1 of a clip whose taps (s0 + 2 p hop .. + hop + win - 1) all lie inside
// [0, n_samples) - no reflect padding - are the interior ones: p in [*lead, *tail).  The others are its edge pairs.
__host__ __device__ inline void interior_pairs(int n_frames, int n_samples, int s0, int hop, int win, int* lead, int* tail) {
  const int n_pairs = (n_frames + 1) / 2;
  int l = s0 < 0 ? (-s0 + 2 * hop - 1) / (2 * hop) : 0;
  l = l < n_pairs ? l : n_pairs;
  const long long num = (long long)n_samples - hop - win - s0;
  int t = num < 0 ? 0 : (int)(num / (2 * hop)) + 1;
  t = t < l ? l : t > n_pairs ? n_pairs : t;
  *lead = l; *tail = t;
}

}  // namespace nisqa

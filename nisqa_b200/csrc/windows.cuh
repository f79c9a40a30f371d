// windows.cuh - the recording spans of nisqa_predict_device_windows and the rings of the live feeds (nisqa_feed_*), shared
// by the host runtime (engine.cu), the windows front end (frontend.cu) and the span and feed ingest (ingest.cu).
#pragma once
#include <cuda_runtime.h>

namespace nisqa {

// Windows of a recording (nisqa_predict_device_windows, nisqa_predict_device_window_pairs): one row per run of
// consecutive windows of one recording in a pass that all run, window i starting at sample i * H of the span and
// covering W samples or up to the span's end.  Every window is also a ClipDesc row of the pass (its own bounds, mel rows
// and clip max); the span is the PCM those windows read, packed once.
struct WinSpan {
  long long pcm_off;   // element offset of the span's first sample (its first window's start) in the pass's PCM
  long long src_off;   // first sample of the span in its recording (model rate; the ingest reads from there)
  int src;             // the recording's index in the caller's batch (ingest)
  int n_samples;       // first window's start .. last window's end
  int clip0;           // window i of the span is ClipDesc row clip0 + i * cstride
  int n_win;           // windows of the span
  int H, hf;           // window hop in samples and in mel frames (H = hf * hop)
  int W;               // window length in samples
  int cstride;         // 1; window pairs: 2 (the clips of a pass alternate degraded and reference windows)
};

// Live feeds (nisqa_feed_*): n_feeds recordings that grow push by push, from one source (nisqa_feed_create) or two
// (nisqa_feed_pair_create: degraded, reference), each source with its own FeedGeom and its own region of the object's
// sample ring and frame ring.  Window k of a source covers [k H - off, k H - off + W) (clipped to the recording); feed
// b's samples live in a ring of R samples at element b * stride of the source's region, sample t at t mod R; the first W
// ring positions are mirrored at R .. R + W - 1 (stride = R + W), so that any W consecutive samples of the recording are
// contiguous.  Its interior frame pairs (taps inside every window k >= ceil(off / H) that holds them) are computed once,
// as soon as their last tap arrives, into a ring of P pair slots of 2 n_mels floats at (b P + slot) 2 n_mels of the
// source's frame region: the pair of global first frame j at slot (j / (3 - ncls)) mod P (ncls 1: window k pairs the
// frames from k hf - off / hop, all of parity par; 2: the window hop is an odd number of frames, both pairings are kept).
// The windows k < ceil(off / H) start at sample 0 (front-clipped reference windows) and are computed per window.
struct FeedGeom {
  long long stride;    // elements per feed in the sample ring (R + W)
  int R, W, H, hf;     // ring length; window length (reference: window + 2 margin) and hop (samples, mel frames)
  int hop, win, s0;    // the model rate's mel frame hop, window and first tap of frame 0 (ClipDesc)
  int P, ncls, fb_id;  // pair slots per feed, pairing classes, front-end tables
  int off, par;        // window k starts at k H - off (the reference margin M; 0 for degraded and single-ended
                       // feeds); the parity of the frames its pairs start at when ncls is 1 ((off / hop) & 1)
};
// One feed in one push (uploaded per push)
struct FeedPush {
  long long t0;        // samples of the feed's recording before this push (the ring position of the chunk's first sample)
  long long j0;        // global first frame of the first pair computed in this push (then j0 + (3 - ncls) x)
  int n_in;            // samples appended
  int n_pairs;         // pairs computed
};
// One window of a feed in a pass (one per ClipDesc row of the pass)
struct FeedWin {
  long long j0;        // global frame of the window's frame 0 (k hf - off / hop); -1: a front-clipped reference window,
                       // whose rows come from the pass's spans rather than the frame ring
  int feed;
  int src;             // 0: degraded (or single-ended), 1: reference - the FeedGeom and frame ring it reads
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

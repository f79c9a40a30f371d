// engine.cu - C-ABI of libnisqa_b200.so (include/nisqa_b200.h) and the host runtime around the
// kernels: checkpoint tensor repacking (BatchNorm folding, k-major linears), per-sample-rate
// front-end tables (periodic Hann, Slaney mel filterbank as band-major CSR - restating
// librosa.filters.mel in double precision), pass planning (exact frame / segment counts,
// reference nisqa/NISQA_lib.py:2308-2309, 2257-2277), device workspaces and launches.
//
// There is no CPU fallback: without a usable CUDA device nisqa_create fails.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/nisqa_b200.h"
#include "common.cuh"
#include "launch.cuh"
#include "windows.cuh"

using namespace nisqa;

namespace {

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  // reserve; a (re)allocated buffer is zero-filled on `st` (fp16 plane pairs rely on never-written
  // padding rows / columns being zero)
  cudaError_t reserve_zeroed(size_t bytes, cudaStream_t st) {
    if (bytes <= cap) return cudaSuccess;
    cudaError_t e = reserve(bytes);
    if (e != cudaSuccess) return e;
    return cudaMemsetAsync(p, 0, cap, st);
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct HostBuf {  // pinned
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    size_t want = bytes + bytes / 4 + 256;
    cudaError_t e = cudaHostAlloc(&p, want, cudaHostAllocDefault);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct FbEntry {
  int sr = 0, hop = 0, win = 0;
  std::vector<float> dense;      // [n_mels][n_bins] host copy (nisqa_mel_filterbank)
  DevBuf window, band_start, band_k0, weights, wtab;
  int n_mag = 0;
};

struct ClipPlan {
  int hop, win, n_frames, n_seg, status, fb_id;
  int run;     // processed by the pass: status OK and, in a double-ended engine, its partner's status OK too
};

struct Ticket {          // one asynchronous nisqa_submit_pcm call
  bool active = false;
  int64_t id = 0;
  size_t bytes = 0;
  float* user_scores = nullptr;
  HostBuf pinned;
  DevBuf scores;         // device scores of this submission (calls in flight do not share one)
  cudaEvent_t done = nullptr;
};

// A compute lane: everything one in-flight pass needs - its own stream, host->device staging and
// activation workspaces.  Passes rotate over the lanes, so the kernels of consecutive passes /
// submissions run on different streams: wave tails and the small low-occupancy kernels of one
// pass are filled with CTAs of another (+8..12 % throughput measured, tools/two_engines.py), and
// the upload of the next pass (copy stream) overlaps compute.
constexpr int kLanes = 3;
constexpr int kStages = 6;     // staging slots / submissions in flight (uploads run ahead of the lanes)
struct Lane {
  cudaStream_t stream = nullptr;
  // td's stage works in tdout (self-attention: its TD_IN rows; LSTM: its output) and xa / xb, td_2's in td2in (its TD_IN
  // rows), td2out (an LSTM's output) and ya / yb, so that td's output is still there after td_2 (NISQA_STAGE_TD1_OUT)
  DevBuf mel, segtab, feats, xa, xb, ya, yb, qkv, qkv2, logits, feats20, tdout, td2out, partial, fused, td2in, ffa, ffb, gx, atth;
  DevBuf dework;           // NISQA_DE: the alignment's projections / norms (de_align_work_floats)
  DevBuf act[7];           // act[l]: fp32 channels-last map feeding conv layer l (2..6) on the FFMA path (and stage dumps)
  DevBuf planes[7];        // planes[l]: fp16 hi | lo plane pair feeding conv layer l (2..6), conv_split.cu
  size_t plane_bytes[7] = {0, 0, 0, 0, 0, 0, 0};   // offset of the lo plane inside planes[l] (half of the allocation)
  ConvGeom plane_g[7] = {};                        // the map planes[l] was zeroed for (its zero rows / columns)
  void release() {
    for (auto& b : act) b.release();
    for (auto& b : planes) b.release();
    DevBuf* all[] = {&mel, &segtab, &feats, &xa, &xb, &ya, &yb, &qkv, &qkv2, &logits, &feats20, &tdout, &td2out, &partial,
                     &fused, &td2in, &ffa, &ffb, &gx, &atth, &dework};
    for (auto* b : all) b->release();
    if (stream) cudaStreamDestroy(stream);
  }
};
// Host->device staging of one pass: pinned tables, device tables, packed PCM, and the two events that
// order it (copied: upload finished on the copy stream; done: the pass's kernels finished on its lane).
struct Stage {
  cudaEvent_t ev_copied = nullptr, ev_done = nullptr;
  bool busy = false;
  int lane = 0;
  HostBuf h_tables;
  DevBuf pcm, clips, prefixes, clipmax;
  DevBuf seg_row;        // segments call: each clip's first output row (int64, < 0: none)
  DevBuf spans;          // windows call: the pass's recording spans (WinSpan)
  DevBuf fwins;          // feed push: the pass's windows (FeedWin)
  DevBuf pair_scores;    // window-pairs call: the pass's (degraded, reference) score rows, before the compact copy
  DevBuf pair_pooled;    // shared-reference embeddings call: the pass's pooled vectors, before the compact copy
  void release() {
    DevBuf* all[] = {&pcm, &clips, &prefixes, &clipmax, &seg_row, &spans, &fwins, &pair_scores, &pair_pooled};
    for (auto* b : all) b->release();
    h_tables.release();
    if (ev_copied) cudaEventDestroy(ev_copied);
    if (ev_done) cudaEventDestroy(ev_done);
  }
};

// Conversion buffers of the device resampler (ms_sr, resample_gpu.cu): the raw packed input, the converted PCM, the
// clip and time-register tables.  A device-batch call leaves its slot in use until its last pass is done (done, busy);
// the calls rotate over kRsSlots of them, so the host can enqueue the next ms_sr call while the previous one runs.
constexpr int kRsSlots = 2;
struct RsSlot {
  DevBuf raw, out, clips, times;
  HostBuf host;                  // pinned copy of the clip table
  cudaEvent_t ready = nullptr;   // the converted PCM is in `out` (recorded on the converting stream)
  cudaEvent_t done = nullptr;    // the call that used the slot last is done with it
  bool busy = false;
  void release() {
    DevBuf* all[] = {&raw, &out, &clips, &times};
    for (auto* b : all) b->release();
    host.release();
    if (ready) cudaEventDestroy(ready);
    if (done) cudaEventDestroy(done);
  }
};

struct TimerSlot {
  std::string name;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev;
  double ms = 0.0;
  int launches = 0;
};

// The packed weights: device pointers into the weights arena, set by pack_weights on every load.  A weight that the
// checkpoint's architecture does not use stays nullptr.
struct Linear { const float* wT = nullptr; const float* b = nullptr; };    // k-major weight, bias
struct ConvWeights {
  const float* w = nullptr;      // [ci][tap][co] fp32, BatchNorm folded in (conv1, and conv2..6 on the FFMA path)
  const float* b = nullptr;      // [co]
  // The tensor-core path stores output channel c as v 2^-e_c (pack_conv): its weights and bias carry that factor
  const float* w_split = nullptr;  // conv1: w, channel c times 2^-e_c
  const float* b_split = nullptr;  // [co] b 2^-e_c
  const float* wtc = nullptr;      // conv2..6: fp16 hi / lo split (pack_conv_tc)
  const float* unit = nullptr;     // [co] 2^e_c: channel c's value from what the path stores (stage dumps, conv6 features)
};
constexpr int kMaxSaLayers = 8;  // nisqa_create's limit on sa_layers / td2_layers
struct SaStackWeights {
  Linear in;                     // Linear(in -> D), 64-column chunks
  const float* ln_g = nullptr;   // the LayerNorm behind it
  const float* ln_b = nullptr;
  const float* pe = nullptr;     // positional encoding [max_len][D], when the stack has one
  SaLayerParams layer[kMaxSaLayers] = {};
  Linear qkv[kMaxSaLayers];      // in_proj of each layer (q pre-scaled by q_fold)
};
struct Weights {
  ConvWeights conv[7];           // conv1..conv6
  // output channels of conv1..conv6 (cnn_c[0]: the one input channel), read from the checkpoint's tensors: AdaptCNN
  // c1 / c2 / c3 / c3 / c3 / c3 with each in {16, 32, 64}, StandardCNN 16 / 32 / 64 / 64 / 64 / 64
  int cnn_c[7] = {1, 16, 32, 64, 64, 64, 64};
  bool shipped_channels() const { return cnn_c[1] == 16 && cnn_c[2] == 32 && cnn_c[3] == 64; }
  CnnPools pools = kShippedPools;  // AdaptCNN's cnn_pool_1/2/3 (nisqa_set_cnn_pools before the load)
  int feat_cols() const { return pools.p[4] * cnn_c[6]; }         // AdaptCNN's framewise fan-out c3 h3 (lib:706)
  int feat_ld() const { return (feat_cols() + 63) / 64 * 64; }    // its row stride: zero columns up to a multiple of 64
  const float* ff_bn = nullptr;  // SkipCNN / DFF: BatchNorm2d(1) as (scale, shift)
  Linear ff[4];                  // SkipCNN's Linear, or DFF's four, BatchNorm1d folded in
  Linear ffc;                    // AdaptCNN's Linear behind conv6 (cnn_fc_out_h)
  SaStackWeights sa[2];          // time_dependency, time_dependency_2
  Linear defuse;                 // NISQA_DE Fusion.lin_fusion
  DeAlignParams de = {};
  PoolHeadParams pool_head = {};       // PoolAttFF
  PoolSimpleParams pool_simple = {};   // the other pooling modules
  Linear fc;                     // StandardCNN fc_out 768 -> 20 (any other path: any width, 64-column padded)
  int std_fc = 0;                // StandardCNN's fc_out width, read from cnn.model.fc_out.weight (0: none, 768 features)
  // The shipped StandardCNN + LSTM shape (fc_out 20, one bidirectional layer of 128, one output, no attention pooling, no
  // td_2) keeps lstm_batched_kernel and its LstmParams; every other LSTM runs as a stack of lstm_layer_kernel layers.
  bool lstm_shipped = false;
  LstmParams lstm = {};
  // A stacked LSTM (td or td_2), its shape read from the checkpoint's tensors: W_ih^T of each layer k-major
  // [K pad 64][dirs 4H], bias b_ih + b_hh, and W_hh [dirs][4H][H]
  struct LstmShape { int H = 0, layers = 0, dirs = 0; };
  struct LstmStack { LstmShape s; Linear ih[4]; const float* hh[4] = {}; };
  LstmStack lstm_st[2];          // time_dependency, time_dependency_2
  Linear lstm_att;               // PoolAttFF behind an LSTM: linear1 of every head, k-major [D pad 64][n_heads 128]
  // the rows the pooling module reads: their width, and the engine column of each reference column (td = 'skip' conv6
  // features; empty: the reference's order)
  int pool_width = 0;
  std::vector<int> pool_src;
};

}  // namespace

struct nisqa_engine {
  nisqa_config cfg;
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  int64_t launches = 0;
  bool weights_loaded = false;
  bool profiling = false;
  int fe_ppc = 0;          // frame pairs per front-end CTA (0: kernel default)
  int conv12 = 1;          // conv1 + pool1 + conv2 + pool2 in one kernel (conv_split.cu): pool1 never reaches HBM
  bool last_conv12 = false;
  bool last_split = false; // the last pass ran the plane pipeline (stage dumps convert back to fp32)
  int lstm_batched = 1;    // BiLSTM: NB clips per CTA in lock step (td.cu lstm_batched_kernel); 0: one CTA per (clip, direction)
  int keep_td_out = 0;     // standard arch: also write the per-step LSTM outputs [n_seg][256] (only the stage dump reads them)
  int conv_tc = 1;         // 1: conv2..6 on the tensor cores (fp16 two-term split, fp16 plane pairs between the layers); 0: fp32 FFMA
  CnnPools pools_next = kShippedPools;   // AdaptCNN pools of the next nisqa_load_weights (nisqa_set_cnn_pools)
  std::vector<TimerSlot> timers;

  // weights arena (device) and the pointers into it
  DevBuf warena;
  Weights w;
  DevBuf rs_win;                 // device resampler of the ingest (resample_gpu.cu): its interpolation table ...
  int rs_nwin = 0, rs_num_table = 0;
  RsSlot rs[kRsSlots];           // ... and its conversion buffers, used in turn
  int64_t rs_next = 0;
  // nisqa_predict_device_batch: ev_in is recorded on the caller's stream (the lanes wait for it), ev_out behind the
  // call's last pass (the caller's stream waits for it)
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;
  float pool_bias_std = 0.f;
  // nisqa_predict_device_batch_embeddings: Weights.pool_src on the device (unset when the rows are in the reference's
  // order)
  DevBuf emb_src;
  float tc_scale[8] = {1, 1, 1, 1, 1, 1, 1, 1};   // 2^-S_i: undoes the weight pre-scale of conv i on the tensor cores
  // widths of the self-attention stacks (0 in the config = 64) and of the rows the pooling module reads
  int sa_d() const { return cfg.sa_d_model ? cfg.sa_d_model : 64; }
  int sa_f() const { return cfg.sa_ff ? cfg.sa_ff : 64; }
  int td2_d() const { return cfg.td2_d_model ? cfg.td2_d_model : 64; }
  int td2_f() const { return cfg.td2_ff ? cfg.td2_ff : 64; }
  // which time-dependency model each stage runs, and the CNN geometry (StandardCNN: W 8/4/2, 768 features)
  bool td_lstm() const { return cfg.arch == NISQA_ARCH_STD_LSTM_LASTBI || cfg.arch == NISQA_ARCH_LSTM_LSTM; }
  bool td_skip() const { return cfg.arch == NISQA_ARCH_SKIP || cfg.arch == NISQA_ARCH_SKIP_LSTM; }     // no td stage
  bool td_sa() const { return !td_lstm() && !td_skip(); }
  bool td2_lstm() const {
    return cfg.arch == NISQA_ARCH_SA_LSTM || cfg.arch == NISQA_ARCH_LSTM_LSTM || cfg.arch == NISQA_ARCH_SKIP_LSTM;
  }
  bool td2_runs() const { return cfg.td2_layers > 0 || td2_lstm(); }
  bool std_cnn() const { return td_lstm() || cfg.cnn_kind == NISQA_CNN_STANDARD; }
  bool conv_net() const { return cfg.cnn_kind == NISQA_CNN_CONV || cfg.cnn_kind == NISQA_CNN_STANDARD; }
  // SkipCNN / DFF rows: n_mels * seg_len features (x.view(-1, fan_in), lib:520 / 556), zero-padded to a multiple of 64
  int ff_fan_in() const { return cfg.n_mels * cfg.seg_len; }
  int ff_fan_in_pad() const { return (ff_fan_in() + 63) / 64 * 64; }
  // conv1 + conv2 in one kernel (conv_split.cu): tensor-core path, the shipped 48 x 15 segments, pool_1 and pool_2, conv1
  // 16 channels wide
  bool fused12() const {
    return conv_tc != 0 && conv12 != 0 && cfg.n_mels == kMels && cfg.seg_len == kSegLen &&
           (std_cnn() || shipped_layer_geometry(2, w.pools)) && conv12_supported(std_cnn(), w.cnn_c[1], w.cnn_c[2]);
  }
  int pool_d() const { return cfg.td2_layers > 0 ? td2_d() : sa_d(); }

  // front-end tables
  std::vector<FbEntry*> fbs;
  DevBuf fb_table;       // FbTables[]
  DevBuf tw4096;         // float2[4096] (twiddle tables of the front-end)

  // per-pass state lives in the lanes; `stream` aliases lane 0's stream (nisqa_stream)
  Lane lanes[kLanes];
  Stage stages[kStages];
  int last_stage = 0;
  cudaStream_t copy_stream = nullptr;
  cudaStream_t cur_stream = nullptr;     // stream of the pass being enqueued (kernel timers)
  HostBuf h_scores;
  int last_lane = 0;
  int64_t pass_counter = 0;
  Ticket tickets[kStages];
  int64_t next_ticket = 1;
  DevBuf scores, dump;

  // description of the last pass (stage dumps)
  std::vector<ClipDesc> last_clips;
  int last_n_seg = 0, last_n_frames = 0, last_passes = 0;
  const float* last_td_in = nullptr;
  const float* last_td_out = nullptr;
  int last_td_out_d = 64;       // row width of last_td_out
  int last_td_out_ld = 0;       // its row stride (0: the width)
  int last_td_out_hw = 0;       // td = 'skip': conv6 features in the engine's order [hw][c3] (pool_3 h / 12); 0: the reference's
  const float* last_td1_out = nullptr;    // td's output when a td_2 stage ran (NISQA_STAGE_TD1_OUT)
  int last_td1_out_d = 0, last_td1_out_ld = 0;
  const float* last_de_fused = nullptr;   // de_align_kernel's output (NISQA_STAGE_DE_FUSED)
  int last_de_fused_d = 0;

  // engine-owned NCCL communicator (multi-GPU gather, SURVEY.md 8e)
  void* nccl_comm = nullptr;
  int nccl_world = 1, nccl_rank = 0;
  float* gather_dst = nullptr;      // when set: every asynchronous / device-path call ends with an
  int gather_rows = 0;              // ncclAllGather of its [gather_rows, n_out] scores on its own lane

  ~nisqa_engine() {
    for (auto* f : fbs) { f->window.release(); f->band_start.release(); f->band_k0.release(); f->weights.release(); f->wtab.release(); delete f; }
    DevBuf* all[] = {&warena, &fb_table, &tw4096, &scores, &dump, &rs_win, &emb_src};
    for (auto& r : rs) r.release();
    for (auto* b : all) b->release();
    h_scores.release();
    for (auto& tk : tickets) { tk.pinned.release(); tk.scores.release(); if (tk.done) cudaEventDestroy(tk.done); }
    if (copy_stream) cudaStreamDestroy(copy_stream);
    for (auto& l : lanes) l.release();
    for (auto& g : stages) g.release();
    stream = nullptr;
    for (auto& t : timers) for (auto& e : t.ev) { cudaEventDestroy(e.first); cudaEventDestroy(e.second); }
    for (cudaEvent_t ev : {ev_in, ev_out}) if (ev) cudaEventDestroy(ev);
  }
};

// A feed object (nisqa_feed_create, nisqa_feed_pair_create): n_feeds live recordings at one rate from n_src sources (1;
// pair feeds: 2, degraded and reference), their rings (windows.cuh: one sample allocation and one frame allocation, each
// source's region at ring_at[s] elements / frames_at[s] floats) and the host state of each feed and source.  Its pushes
// run in push order: a push's ingest waits for the last push's passes (done), so one ring holds what any push reads
// (feed_create derives the ring lengths).
constexpr int kFeedSlots = 4;      // push tables in flight (pinned -> device)
struct nisqa_feed {
  nisqa_engine* e = nullptr;
  int n_feeds = 0, rate = 0, n_src = 1;
  int64_t max_push = 0, max_skew = 0;
  FeedGeom g[2] = {};                      // per source
  int fmt = -1;                            // the rings' sample format (NISQA_FMT_*) while a feed holds samples
  std::vector<int64_t> held[2];            // samples of each feed's current recording, per source
  std::vector<int64_t> j_next[2];          // each feed's first frame whose pair is not computed yet, per source
  long long ring_at[2] = {0, 0};           // each source's first element in the sample ring
  size_t frames_at[2] = {0, 0};            // each source's first float in the frame ring
  void* ring = nullptr;                    // [n_src][n_feeds][stride] samples (4 bytes each reserved)
  float* frames = nullptr;                 // [n_src][n_feeds][P][2 n_mels]
  size_t ring_bytes = 0, frame_bytes = 0;
  struct Slot { HostBuf h; DevBuf d; cudaEvent_t copied = nullptr; bool busy = false; } slots[kFeedSlots];
  int64_t n_push = 0;
  cudaEvent_t ready = nullptr;             // this push's samples and pairs are in the rings
  cudaEvent_t done = nullptr;              // the last push's passes are done
  bool pending = false;
  ~nisqa_feed() {         // (nisqa_feed_destroy first waits for the work in flight)
    for (auto& sl : slots) {
      sl.h.release(); sl.d.release();
      if (sl.copied) cudaEventDestroy(sl.copied);
    }
    if (ring) cudaFree(ring);
    if (frames) cudaFree(frames);
    for (cudaEvent_t ev : {ready, done}) if (ev) cudaEventDestroy(ev);
  }
};

namespace {

int fail(nisqa_engine* e, int code, const std::string& msg) {
  if (e) e->err = msg;
  return code;
}
#define CK(call)                                                                          \
  do {                                                                                    \
    cudaError_t _e = (call);                                                              \
    if (_e != cudaSuccess)                                                                \
      return fail(e, NISQA_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e)); \
  } while (0)

// ---------------------------------------------------------------- timing of kernel groups
struct Scope {
  nisqa_engine* e; TimerSlot* slot = nullptr; cudaEvent_t stop = nullptr;
  Scope(nisqa_engine* e_, const char* name, int n_launch = 1) : e(e_) {
    e->launches += n_launch;
    if (!e->profiling) return;
    for (auto& t : e->timers) if (t.name == name) slot = &t;
    if (!slot) { e->timers.push_back(TimerSlot()); slot = &e->timers.back(); slot->name = name; }
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    cudaEventRecord(a, e->cur_stream);
    slot->ev.push_back({a, b});
    slot->launches += n_launch;
    stop = b;
  }
  ~Scope() { if (stop) cudaEventRecord(stop, e->cur_stream); }
};

void collect_timers(nisqa_engine* e) {
  for (auto& t : e->timers) {
    for (auto& ev : t.ev) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, ev.first, ev.second) == cudaSuccess) t.ms += ms;
      cudaEventDestroy(ev.first); cudaEventDestroy(ev.second);
    }
    t.ev.clear();
  }
}

// ---------------------------------------------------------------- host arithmetic (a2, a6)
void plan_clip(const nisqa_config& c, int64_t n_samples, int sr, ClipPlan* p) {
  // reference lib:2308-2309: int(sr * seconds) in double precision, truncation
  p->hop = (int)((double)sr * c.hop_s);
  p->win = (int)((double)sr * c.win_s);
  p->n_frames = 0; p->n_seg = 0; p->status = NISQA_CLIP_TOO_SHORT; p->fb_id = -1;
  if (p->hop < 1 || p->win < 1 || p->win > c.n_fft || n_samples < 1) return;
  // librosa.stft(center=True): frames = 1 + (n + 2*(n_fft/2) - n_fft) / hop = 1 + n / hop
  const int64_t frames = 1 + n_samples / p->hop;
  const int64_t n_wins = frames - (c.seg_len - 1);          // lib:2257
  p->n_frames = (int)std::min<int64_t>(frames, INT32_MAX);
  if (n_wins < 1) return;                                    // lib:2258-2263
  const int64_t n_seg = (c.seg_hop > 1) ? (n_wins + c.seg_hop - 1) / c.seg_hop : n_wins;  // lib:2271-2273
  p->n_seg = (int)std::min<int64_t>(n_seg, INT32_MAX);
  if (c.max_segments > 0 && n_seg > c.max_segments) { p->status = NISQA_CLIP_TOO_LONG; return; }  // lib:2276-2277
  p->status = NISQA_CLIP_OK;
}

// Windows of a recording (nisqa_predict_device_windows) at the model rate sr: window `window` samples, hop `hop_frames` mel
// frames = *H samples, so that every window starts on a mel frame of the recording.  false (the reason in *why) for a
// geometry the checkpoint cannot score: a hop longer than the window, or a window of more than max_segments segments or
// of none.
bool window_geometry(const nisqa_config& c, int sr, int64_t window, int32_t hop_frames, int* H, std::string* why) {
  if (window < 1 || window > INT32_MAX) { *why = "window = " + std::to_string(window) + ": not within 1 .. 2^31 - 1 samples"; return false; }
  ClipPlan pl;
  plan_clip(c, window, sr, &pl);
  if (pl.hop < 1) { *why = "sample rate " + std::to_string(sr) + ": no mel frame hop"; return false; }
  if (hop_frames < 1) { *why = "hop_frames = " + std::to_string(hop_frames) + ": at least one mel frame"; return false; }
  const int64_t h = (int64_t)hop_frames * pl.hop;
  if (h > window) {
    *why = "hop_frames = " + std::to_string(hop_frames) + ": a window hop of " + std::to_string(h) +
           " samples is longer than the window (" + std::to_string(window) + " samples)";
    return false;
  }
  if (pl.status == NISQA_CLIP_TOO_LONG) {
    *why = "window = " + std::to_string(window) + " samples: " + std::to_string(pl.n_seg) + " segments > max_segments " +
           std::to_string(c.max_segments);
    return false;
  }
  if (pl.status != NISQA_CLIP_OK) { *why = "window = " + std::to_string(window) + " samples: too short for one segment"; return false; }
  *H = (int)h;
  return true;
}
int64_t window_count(int64_t T, int64_t W, int64_t H) { return T <= W ? 1 : 1 + (T - W + H - 1) / H; }
// Window pairs (nisqa_predict_device_window_pairs): the degraded windows of window_geometry and a reference margin of
// margin_frames mel frames = *M samples on either side.  false (the reason in *why) for what window_geometry refuses, a
// negative margin, or a reference window of W + 2M samples with more than max_segments segments.
bool window_pair_geometry(const nisqa_config& c, int sr, int64_t window, int32_t hop_frames, int32_t margin_frames, int* H,
                          int64_t* M, std::string* why) {
  if (!window_geometry(c, sr, window, hop_frames, H, why)) return false;
  if (margin_frames < 0) { *why = "margin_frames = " + std::to_string(margin_frames) + ": a margin cannot be negative"; return false; }
  *M = (int64_t)margin_frames * (*H / hop_frames);
  ClipPlan pl;
  plan_clip(c, window + 2 * *M, sr, &pl);
  if (window + 2 * *M > INT32_MAX || pl.status == NISQA_CLIP_TOO_LONG) {
    *why = "margin_frames = " + std::to_string(margin_frames) + ": a reference window of " + std::to_string(window + 2 * *M) +
           " samples has " + std::to_string(pl.n_seg) + " segments > max_segments " + std::to_string(c.max_segments);
    return false;
  }
  return true;
}
// Pair k of a degraded recording of T samples and its reference of T_ref: the reference window [max(0, kH - M),
// min(T_ref, kH + W + M)), empty (length 0) once kH - M >= T_ref
void ref_window(int64_t k, int64_t T_ref, int64_t W, int64_t H, int64_t M, int64_t* start, int64_t* n) {
  *start = std::max<int64_t>(0, k * H - M);
  *n = std::max<int64_t>(0, std::min(T_ref, k * H + W + M) - *start);
}
// The windows a push of n[b] samples to feeds that held held[b] completes, as emit(feed, k, T, T_ref) in feed then
// window order (T, T_ref: the feed's lengths after the push): window k once the feed holds k H + W samples; with end[b],
// every remaining window of the final length T (window_count: the last may be short; a feed that ended with no sample has
// none).  Pair feeds (ref_held / ref_n not null; margin M): pair k once the feed also holds k H + W + M reference
// samples; with end[b], every remaining pair of the final degraded length.  Both conditions are monotone in k, so a push
// emits a contiguous range of pairs per feed, a function of the held counts alone.
template <class Emit>
void feed_windows(int n_feeds, int64_t W, int64_t H, int64_t M, const int64_t* held, const int64_t* n,
                  const int64_t* ref_held, const int64_t* ref_n, const uint8_t* end, Emit emit) {
  auto complete = [&](int64_t T, int64_t w) { return T >= w ? (T - w) / H + 1 : 0; };
  auto both = [&](int64_t T, int64_t T_ref) { return ref_held ? std::min(complete(T, W), complete(T_ref, W + M)) : complete(T, W); };
  for (int b = 0; b < n_feeds; ++b) {
    const int64_t T = held[b] + n[b], T_ref = ref_held ? ref_held[b] + ref_n[b] : 0;
    const int64_t k1 = end && end[b] && T > 0 ? window_count(T, W, H) : both(T, T_ref);
    for (int64_t k = both(held[b], ref_held ? ref_held[b] : 0); k < k1; ++k) emit(b, k, T, T_ref);
  }
}

// ---------------------------------------------------------------- librosa.filters.mel in double
double hz_to_mel(double f) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = (min_log_hz - 0.0) / f_sp;
  const double logstep = log(6.4) / 27.0;
  if (f >= min_log_hz) return min_log_mel + log(f / min_log_hz) / logstep;
  return (f - 0.0) / f_sp;
}
double mel_to_hz(double m) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = (min_log_hz - 0.0) / f_sp;
  const double logstep = log(6.4) / 27.0;
  if (m >= min_log_mel) return min_log_hz * exp(logstep * (m - min_log_mel));
  return 0.0 + f_sp * m;
}
void np_linspace(double start, double stop, int num, std::vector<double>& y) {
  y.resize(num);
  const double step = (stop - start) / (double)(num - 1);
  for (int i = 0; i < num; ++i) { volatile double t = (double)i * step; y[i] = t + start; }
  y[num - 1] = stop;
}

int build_fb(nisqa_engine* e, int sr, int hop, int win, int* id_out) {
  for (size_t i = 0; i < e->fbs.size(); ++i)
    if (e->fbs[i]->sr == sr) { *id_out = (int)i; return 0; }
  const nisqa_config& c = e->cfg;
  const int n_bins = c.n_fft / 2 + 1, n_mels = c.n_mels;
  FbEntry* fb = new FbEntry();
  fb->sr = sr; fb->hop = hop; fb->win = win;
  std::vector<double> fftfreqs, mels, mel_f(n_mels + 2);
  np_linspace(0.0, (double)sr / 2, n_bins, fftfreqs);
  np_linspace(hz_to_mel(0.0), hz_to_mel(c.fmax), n_mels + 2, mels);
  for (int i = 0; i < n_mels + 2; ++i) mel_f[i] = mel_to_hz(mels[i]);
  fb->dense.assign((size_t)n_mels * n_bins, 0.f);
  std::vector<int> band_start(n_mels + 1, 0), band_k0(n_mels, 0);
  std::vector<float> wts;
  for (int i = 0; i < n_mels; ++i) {
    const double fd0 = mel_f[i + 1] - mel_f[i], fd1 = mel_f[i + 2] - mel_f[i + 1];
    const double enorm = 2.0 / (mel_f[i + 2] - mel_f[i]);
    int k0 = -1, k1 = -1;
    for (int k = 0; k < n_bins; ++k) {
      const double lower = -(mel_f[i] - fftfreqs[k]) / fd0;
      const double upper = (mel_f[i + 2] - fftfreqs[k]) / fd1;
      const float tri = (float)std::max(0.0, std::min(lower, upper));   // float32 triangle ...
      const float w = (float)((double)tri * enorm);                      // ... then `weights *= enorm`
      fb->dense[(size_t)i * n_bins + k] = w;
      if (w != 0.f) { if (k0 < 0) k0 = k; k1 = k; }
    }
    band_start[i] = (int)wts.size();
    band_k0[i] = k0 < 0 ? 0 : k0;
    if (k0 >= 0) for (int k = k0; k <= k1; ++k) wts.push_back(fb->dense[(size_t)i * n_bins + k]);
    while (wts.size() % 32) wts.push_back(0.f);     // rows padded to the warp width (frontend mel_bands)
  }
  band_start[n_mels] = (int)wts.size();
  if (wts.empty()) wts.push_back(0.f);
  // scipy.signal.get_window('hann', win, fftbins=True): periodic Hann in float64 -> float32
  std::vector<float> window((size_t)(win + 1023) / 1024 * 1024, 0.f);   // zero-padded to the FFT sub-length
  for (int n = 0; n < win; ++n) window[n] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * (double)n / (double)win));
  if (win == 1) window[0] = 1.f;
  // fused window x residue twiddle table of the pipelined front-end: wt[r][n] = hann[n] * e^{-2 pi i r n / 4096}
  std::vector<float2> wtab(4 * 1024, make_float2(0.f, 0.f));
  for (int r = 0; r < 4; ++r)
    for (int nn = 0; nn < win && nn < 1024; ++nn) {
      const double wv = (win == 1) ? 1.0 : 0.5 - 0.5 * cos(2.0 * M_PI * (double)nn / (double)win);
      const float wf = (float)wv;                                   // the float32 window the reference multiplies with
      const double a = -2.0 * M_PI * (double)(((long)r * nn) & 4095) / 4096.0;
      wtab[r * 1024 + nn] = make_float2((float)((double)wf * cos(a)), (float)((double)wf * sin(a)));
    }
  int n_mag = 0;
  for (int i = 0; i < n_mels; ++i)
    for (int k = 0; k < n_bins; ++k)
      if (fb->dense[(size_t)i * n_bins + k] != 0.f) n_mag = std::max(n_mag, k + 1);
  fb->n_mag = n_mag;
  CK(fb->wtab.reserve(wtab.size() * sizeof(float2)));
  CK(cudaMemcpy(fb->wtab.p, wtab.data(), wtab.size() * sizeof(float2), cudaMemcpyHostToDevice));
  CK(fb->window.reserve(window.size() * 4));
  CK(fb->band_start.reserve(band_start.size() * 4));
  CK(fb->band_k0.reserve(band_k0.size() * 4));
  CK(fb->weights.reserve(wts.size() * 4));
  CK(cudaMemcpy(fb->window.p, window.data(), window.size() * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(fb->band_start.p, band_start.data(), band_start.size() * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(fb->band_k0.p, band_k0.data(), band_k0.size() * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(fb->weights.p, wts.data(), wts.size() * 4, cudaMemcpyHostToDevice));
  e->fbs.push_back(fb);
  // refresh the device table of FbTables
  std::vector<FbTables> tab(e->fbs.size());
  for (size_t i = 0; i < e->fbs.size(); ++i) {
    tab[i].window = e->fbs[i]->window.as<float>();
    tab[i].band_start = e->fbs[i]->band_start.as<int>();
    tab[i].band_k0 = e->fbs[i]->band_k0.as<int>();
    tab[i].weights = e->fbs[i]->weights.as<float>();
    tab[i].wtab = e->fbs[i]->wtab.as<float2>();
    tab[i].n_mag = e->fbs[i]->n_mag;
    tab[i].pad_ = 0;
  }
  CK(cudaDeviceSynchronize());      // the table may be in use by passes in flight on any lane
  CK(e->fb_table.reserve(tab.size() * sizeof(FbTables) + 64 * sizeof(FbTables)));
  CK(cudaMemcpy(e->fb_table.p, tab.data(), tab.size() * sizeof(FbTables), cudaMemcpyHostToDevice));
  *id_out = (int)e->fbs.size() - 1;
  return 0;
}

// ---------------------------------------------------------------- weight repacking
struct TensorView { const float* d; int nd; int64_t dims[4]; int64_t numel; };

struct Packer {
  std::map<std::string, TensorView> t;
  std::vector<float> arena;
  Weights w;                                               // its pointers are set by pack_weights once `arena` is uploaded
  std::vector<std::pair<const float**, size_t>> slots;     // (member of w, float offset of its block in arena)
  std::string err;
  bool fail(const std::string& msg) { if (err.empty()) err = msg; return false; }
  const TensorView* get(const std::string& name, std::initializer_list<int64_t> shape) {
    auto it = t.find(name);
    if (it == t.end()) { fail("missing tensor " + name); return nullptr; }
    const TensorView& v = it->second;
    bool ok = v.nd == (int)shape.size();
    int i = 0;
    for (int64_t s : shape) { if (ok && v.dims[i] != s) ok = false; ++i; }
    if (!ok) { fail("bad shape for tensor " + name); return nullptr; }
    return &v;
  }
  // a zero-filled block of n floats for `dst`, 256-byte aligned (the conv kernels read their weights with 16-byte cp.async
  // and bulk copies); returns its offset in arena
  size_t alloc(const float*& dst, size_t n) {
    const size_t off = (arena.size() + 63) / 64 * 64;
    arena.resize(off + n, 0.f);
    slots.push_back({&dst, off});
    return off;
  }
  void copy(const float*& dst, const float* src, size_t n) { memcpy(&arena[alloc(dst, n)], src, n * 4); }
};

// Activation exponents of conv<idx>'s output channels (BatchNorm tensors g, be): e_c = ilogb(E_c sqrt(2) / 4) of the
// channel's BN output estimate E_c = |beta_c| + 3 |gamma_c| (three standard deviations), so that the stored v 2^-e_c
// lies in [2.8, 5.7) at E_c.  e_c moves by exactly k when channel c's BatchNorm weight and bias are multiplied by 2^k.
// It is kept at most kExpWindow binades below the layer's largest: a dead channel (E_c zero or denormal) must not push a
// folded weight out of fp32 range.
constexpr int kExpWindow = 64;
std::vector<int> act_exponents(const TensorView* g, const TensorView* be, int cout) {
  std::vector<double> E(cout);
  double emax = 0.0;
  for (int co = 0; co < cout; ++co) {
    E[co] = fabs((double)be->d[co]) + 3.0 * fabs((double)g->d[co]);
    if (std::isfinite(E[co])) emax = std::max(emax, E[co]);
  }
  const int top = emax > 0.0 ? ilogb(emax * sqrt(2.0) / 4.0) : 0, floor = top - kExpWindow;
  std::vector<int> e(cout, floor);
  for (int co = 0; co < cout; ++co)
    if (E[co] > 0.0 && std::isfinite(E[co])) e[co] = std::max(floor, ilogb(E[co] * sqrt(2.0) / 4.0));
  return e;
}

// conv<idx> (kernel 3 x kw: AdaptCNN's conv6 is 3 x pool_3[1]) with bn<idx> folded in, as [ci][tap][co] (conv1: [tap][16]),
// for the FFMA path; the tensor-core path's bias (and conv1's weights) with 2^-e_c folded into output channel c, and 2^e_c.
// *e: the activation exponents of the output channels; *w_off: the offset of the fp32 weights in the arena
bool pack_conv(Packer& P, int idx, int cin, int cout, std::vector<int>* e, size_t* w_off, int kw = 3) {
  const std::string cv = "cnn.model.conv" + std::to_string(idx) + ".", bn = "cnn.model.bn" + std::to_string(idx) + ".";
  const int ntap = 3 * kw;
  const TensorView* w = P.get(cv + "weight", {cout, cin, 3, kw});
  const TensorView* b = P.get(cv + "bias", {cout});
  const TensorView* g = P.get(bn + "weight", {cout});
  const TensorView* be = P.get(bn + "bias", {cout});
  const TensorView* mu = P.get(bn + "running_mean", {cout});
  const TensorView* var = P.get(bn + "running_var", {cout});
  if (!w || !b || !g || !be || !mu || !var) return false;
  *e = act_exponents(g, be, cout);
  ConvWeights& cw = P.w.conv[idx];
  const size_t wo = P.alloc(cw.w, (size_t)cin * ntap * cout);
  const size_t bo = P.alloc(cw.b, cout), bso = P.alloc(cw.b_split, cout), uo = P.alloc(cw.unit, cout);
  const size_t wso = idx == 1 ? P.alloc(cw.w_split, (size_t)ntap * cout) : 0;
  for (int co = 0; co < cout; ++co) {
    // eval-mode BatchNorm2d (eps 1e-5) folded into the convolution (SURVEY.md Appendix A)
    const double s = (double)g->d[co] / sqrt((double)var->d[co] + 1e-5);
    P.arena[bo + co] = (float)(((double)b->d[co] - (double)mu->d[co]) * s + (double)be->d[co]);
    for (int ci = 0; ci < cin; ++ci)
      for (int tap = 0; tap < ntap; ++tap)
        P.arena[wo + ((size_t)ci * ntap + tap) * cout + co] =
            (float)((double)w->d[((size_t)co * cin + ci) * ntap + tap] * s);
    // powers of two of the fp32 values: exact
    P.arena[bso + co] = (float)ldexp((double)P.arena[bo + co], -(*e)[co]);
    P.arena[uo + co] = (float)ldexp(1.0, (*e)[co]);
    if (idx == 1)
      for (int tap = 0; tap < ntap; ++tap)
        P.arena[wso + (size_t)tap * cout + co] = (float)ldexp((double)P.arena[wo + (size_t)tap * cout + co], -(*e)[co]);
  }
  *w_off = wo;
  return true;
}

// conv2..conv6 for the tensor-core path, from the folded fp32 weights at `src` (ntap taps): [tap][ci/8][hi co | lo co][8]
// fp16 two-term split of w 2^(e_in[ci] - e_out[co] + S): input channel ci stored at 2^-e_in[ci], output channel co to be
// stored at 2^-e_out[co] (pack_conv), and S chosen so that the largest of these lies in (512, 1024] whatever the weights'
// range (b_lo stays out of the fp16 subnormals)
void pack_conv_tc(Packer& P, int idx, int ci_n, int co_n, size_t src, const std::vector<int>& e_in,
                  const std::vector<int>& e_out, float* tc_scale, int ntap = 9) {
  std::vector<float> ws((size_t)ci_n * ntap * co_n);
  float wmax = 0.f;
  for (int ci = 0; ci < ci_n; ++ci)
    for (int tap = 0; tap < ntap; ++tap)
      for (int co = 0; co < co_n; ++co) {
        const size_t j = ((size_t)ci * ntap + tap) * co_n + co;
        ws[j] = (float)ldexp((double)P.arena[src + j], e_in[ci] - e_out[co]);
        wmax = std::max(wmax, fabsf(ws[j]));
      }
  int S = 0;
  if (wmax > 0.f && std::isfinite(wmax)) {
    S = 9 - ilogbf(wmax);                                         // max|w| 2^S in [512, 1024)
    if (ldexpf(wmax, S) == 512.f) ++S;                            // a power of two: 1024 itself
  }
  *tc_scale = ldexpf(1.f, -S);
  const size_t n_half = (size_t)ntap * 2 * ci_n * co_n;
  const size_t dst = P.alloc(P.w.conv[idx].wtc, (n_half + 1) / 2);   // fp16 payload inside the float arena
  for (int tap = 0; tap < ntap; ++tap)
    for (int ci = 0; ci < ci_n; ++ci)
      for (int co = 0; co < co_n; ++co) {
        const float w = ldexpf(ws[((size_t)ci * ntap + tap) * co_n + co], S);
        const __half hi = __float2half_rn(w);
        const __half lo = __float2half_rn(w - __half2float(hi));
        __half* base = reinterpret_cast<__half*>(&P.arena[dst]) + (size_t)tap * 2 * ci_n * co_n;
        // per 16-byte K chunk: rows [0,co_n) = hi, rows [co_n, 2 co_n) = lo  (one N = 2*C_out operand)
        const size_t off = ((size_t)(ci / 8) * (2 * co_n) + co) * 8 + (ci & 7);
        base[off] = hi;
        base[off + (size_t)co_n * 8] = lo;
      }
}

// dst[k][j] = src[j][perm(k)] for a [n_out][n_in] PyTorch Linear weight
void pack_linear_T(Packer& P, size_t off, const TensorView* w, int n_out, int n_in, float scale = 1.f) {
  for (int k = 0; k < n_in; ++k)
    for (int j = 0; j < n_out; ++j) P.arena[off + (size_t)k * n_out + j] = w->d[(size_t)j * n_in + k] * scale;
}

// W^T of an nn.Linear(n_in -> n_out) in 64-column chunks (the layout of the td_tiled.cu kernels): chunk n is the k-major
// [k_pad][64] block at n k_pad 64; engine input row k < k_rows (default n_in) reads checkpoint input column col(k); rows
// with col(k) < 0 and rows >= k_rows stay zero
template <class Col>
void pack_linear_chunked(Packer& P, size_t off, const TensorView* w, int n_out, int n_in, int k_pad, Col col, int k_rows = -1) {
  if (k_rows < 0) k_rows = n_in;
  for (int n = 0; n < n_out / 64; ++n)
    for (int k = 0; k < k_rows; ++k) {
      const int kc = col(k);
      if (kc < 0) continue;
      for (int j = 0; j < 64; ++j) P.arena[off + ((size_t)n * k_pad + k) * 64 + j] = w->d[(size_t)(n * 64 + j) * n_in + kc];
    }
}

// nn.MultiheadAttention scales q by D^-1/2 after the in-projection: folded into the packed q weights where that is a power
// of two (exact), otherwise applied by the kernels to the projected q (qscale)
float q_fold(int D) { return D == 64 ? 0.125f : D == 256 ? 0.0625f : 1.f; }
float q_scale(int D) { return q_fold(D) == 1.f ? (float)(1.0 / std::sqrt((double)D)) : 1.f; }

// SkipCNN / DFF Linear `name` (n_in -> n_out) k-major with n_in_pad rows, the eval-mode BatchNorm1d `bn` behind it
// (eps 1e-5; none when empty) folded in
bool pack_ff_linear(Packer& P, Linear& dst, const std::string& name, const std::string& bn, int n_in, int n_in_pad, int n_out) {
  const std::string p = "cnn.model.";
  const TensorView* w = P.get(p + name + ".weight", {n_out, n_in});
  const TensorView* b = P.get(p + name + ".bias", {n_out});
  if (!w || !b) return false;
  std::vector<double> sc(n_out, 1.0), sh(n_out, 0.0);
  if (!bn.empty()) {
    const TensorView* g2 = P.get(p + bn + ".weight", {n_out});
    const TensorView* b2 = P.get(p + bn + ".bias", {n_out});
    const TensorView* m2 = P.get(p + bn + ".running_mean", {n_out});
    const TensorView* v2 = P.get(p + bn + ".running_var", {n_out});
    if (!g2 || !b2 || !m2 || !v2) return false;
    for (int j = 0; j < n_out; ++j) {
      sc[j] = (double)g2->d[j] / sqrt((double)v2->d[j] + 1e-5);
      sh[j] = (double)b2->d[j] - (double)m2->d[j] * sc[j];
    }
  }
  const size_t ow = P.alloc(dst.wT, (size_t)n_in_pad * n_out), ob = P.alloc(dst.b, n_out);
  for (int k = 0; k < n_in; ++k)
    for (int j = 0; j < n_out; ++j) P.arena[ow + (size_t)k * n_out + j] = (float)((double)w->d[(size_t)j * n_in + k] * sc[j]);
  for (int j = 0; j < n_out; ++j) P.arena[ob + j] = (float)((double)b->d[j] * sc[j] + sh[j]);
  return true;
}

// SkipCNN / DFF (lib:504-583): the BatchNorm2d(1) in front as a scalar affine map (applied by seg_feats_kernel, so
// that the Linear layers see what the reference's see), Linear layers k-major, DFF's BatchNorm1d folded into them
bool pack_ffnet(Packer& P, const nisqa_config& c) {
  const int fan_in = c.n_mels * c.seg_len, fan_pad = (fan_in + 63) / 64 * 64;
  const bool dff = c.cnn_kind == NISQA_CNN_DFF;
  const std::string bn = dff ? "cnn.model.bn1." : "cnn.model.bn.";
  const TensorView* g = P.get(bn + "weight", {1});
  const TensorView* be = P.get(bn + "bias", {1});
  const TensorView* mu = P.get(bn + "running_mean", {1});
  const TensorView* var = P.get(bn + "running_var", {1});
  if (!g || !be || !mu || !var) return false;
  const double a = (double)g->d[0] / sqrt((double)var->d[0] + 1e-5);
  const size_t o = P.alloc(P.w.ff_bn, 2);
  P.arena[o] = (float)a; P.arena[o + 1] = (float)((double)be->d[0] - (double)mu->d[0] * a);
  const int H = c.cnn_fc;
  if (dff)
    return pack_ff_linear(P, P.w.ff[0], "lin1", "bn2", fan_in, fan_pad, H) && pack_ff_linear(P, P.w.ff[1], "lin2", "bn3", H, H, H) &&
           pack_ff_linear(P, P.w.ff[2], "lin3", "bn4", H, H, H) && pack_ff_linear(P, P.w.ff[3], "lin4", "bn5", H, H, H);
  return H == 0 || pack_ff_linear(P, P.w.ff[0], "linear", "", fan_in, fan_pad, H);
}

// AdaptCNN's channel counts from its tensors: conv1..conv3's output channels c1, c2, c3 (cnn_c_out_1/2/3), each 16, 32
// or 64 (one fp16 row of a plane pair is one 32 / 64 / 128-byte swizzle atom and a whole number of k16 steps);
// conv4..conv6 stay at c3 (pack_conv checks their shapes)
bool read_cnn_channels(Packer& P, int* cc) {
  for (int i = 1; i <= 3; ++i) {
    const std::string name = "cnn.model.conv" + std::to_string(i) + ".weight";
    auto it = P.t.find(name);
    if (it == P.t.end()) return P.fail("missing tensor " + name);
    const int co = it->second.nd == 4 ? (int)it->second.dims[0] : 0;
    if (co != 16 && co != 32 && co != 64)
      return P.fail("tensor " + name + ": " + std::to_string(co) + " output channels (cnn_c_out_" + std::to_string(i) +
                    "): the engine runs AdaptCNN channel counts 16, 32 or 64");
    cc[i] = co;
  }
  cc[4] = cc[5] = cc[6] = cc[3];
  return true;
}

// The framewise model: AdaptCNN / StandardCNN (fp32 and tensor-core weights, activation scales) with AdaptCNN's optional
// Linear, or SkipCNN / DFF
bool pack_framewise(Packer& P, nisqa_engine* e) {
  const nisqa_config& c = e->cfg;
  if (!e->conv_net()) return pack_ffnet(P, c);
  int* cc = P.w.cnn_c;
  if (!e->std_cnn() && !read_cnn_channels(P, cc)) return false;
  if (!e->std_cnn()) P.w.pools = e->pools_next;
  const int h3 = P.w.pools.p[4], w3 = e->std_cnn() ? 3 : P.w.pools.p[5];
  if (!e->std_cnn() && h3 * cc[6] > kMaxCnnFeatures)
    return P.fail("tensor cnn.model.conv6.weight: " + std::to_string(cc[6]) + " channels x pool_3 height " + std::to_string(h3) +
                  " = " + std::to_string(h3 * cc[6]) + " features (cnn_c_out_3 x cnn_pool_3[0]): the engine runs up to " +
                  std::to_string(kMaxCnnFeatures));
  std::vector<int> ex[7];                  // ex[i][c]: the activation exponent of conv i's output channel c
  for (int i = 1; i <= 6; ++i) {
    size_t w_off = 0;
    const int kw = i == 6 ? w3 : 3;        // conv6: kernel (3, pool_3[1]), padding (1, 0) (lib:674-678)
    if (!pack_conv(P, i, cc[i - 1], cc[i], &ex[i], &w_off, kw)) return false;
    if (i >= 2) pack_conv_tc(P, i, cc[i - 1], cc[i], w_off, ex[i - 1], ex[i], &e->tc_scale[i], 3 * kw);
  }
  if (c.cnn_fc > 0) {
    // AdaptCNN's optional Linear (lib:682-684, 708-709): k-major, rows in the engine's feature order h*c3 + c, zero rows
    // up to the padded feature width
    const int H = c.cnn_fc, C3 = cc[6], K = P.w.feat_cols();
    const TensorView* w = P.get("cnn.model.fc.weight", {H, K});
    const TensorView* b = P.get("cnn.model.fc.bias", {H});
    if (!w || !b) return false;
    const size_t ow = P.alloc(P.w.ffc.wT, (size_t)P.w.feat_ld() * H);
    for (int h = 0; h < h3; ++h)
      for (int ch = 0; ch < C3; ++ch)
        for (int j = 0; j < H; ++j) P.arena[ow + ((size_t)h * C3 + ch) * H + j] = w->d[(size_t)j * K + ch * h3 + h];
    P.copy(P.w.ffc.b, b->d, H);
  }
  return true;
}

// The rows that feed a time-dependency stage: `dim` features, padded with zero columns to a multiple of 64, in the order
// of the checkpoint's Linear (PLAIN) or - conv6's `ch` channels over `h` rows - in the engine's order: AdaptCNN k' = h*ch + c
// <-> reference view(-1, ch*h3) order c*h3 + h (lib:706), StandardCNN k' = (h*2 + w)*64 + c <-> c*12 + h*2 + w (lib:830).
// NISQA_DE's fused rows (IN_DE_FUSED): `dim` = nf W reference columns, part p of W columns at engine row p h (h = W padded
// to a multiple of 64, ch = W); in_col is -1 on the pad rows.
enum InOrder { IN_PLAIN, IN_ADAPT_CONV, IN_STD_CONV, IN_DE_FUSED };
struct InRows { int dim; InOrder order; int ch = 64; int h = 6; };
int in_col(const InRows& in, int k) {
  if (in.order == IN_DE_FUSED) return k % in.h < in.ch ? (k / in.h) * in.ch + k % in.h : -1;
  return in.order == IN_ADAPT_CONV ? (k % in.ch) * in.h + k / in.ch : in.order == IN_STD_CONV ? (k & 63) * 12 + (k >> 6) : k;
}
// engine rows of `in`: the padded fused layout, or dim rounded up to a multiple of 64
int in_rows(const InRows& in) { return in.order == IN_DE_FUSED ? in.dim / in.ch * in.h : (in.dim + 63) / 64 * 64; }

// One SelfAttention stack (lib:945-1040) of width D and feed-forward width F, checkpoint prefix `ck`: Linear(in -> D) +
// LayerNorm + `layers` encoder layers.  The Linear's rows beyond in.dim (the padding of the input rows) stay zero.
bool pack_sa_stack(Packer& P, SaStackWeights& S, const std::string& ck, InRows in, int layers, int D, int F) {
  const int in_dim = in.dim;
  const TensorView* lw = P.get(ck + "linear.weight", {D, in_dim});
  const TensorView* lb = P.get(ck + "linear.bias", {D});
  const TensorView* ng = P.get(ck + "norm1.weight", {D});
  const TensorView* nb = P.get(ck + "norm1.bias", {D});
  if (!lw || !lb || !ng || !nb) return false;
  const int k_pad = in_rows(in);
  const size_t o = P.alloc(S.in.wT, (size_t)k_pad * D);
  pack_linear_chunked(P, o, lw, D, in_dim, k_pad, [&](int k) { return in_col(in, k); }, in.order == IN_DE_FUSED ? k_pad : in_dim);
  P.copy(S.in.b, lb->d, D);
  P.copy(S.ln_g, ng->d, D);
  P.copy(S.ln_b, nb->d, D);
  const auto id = [](int k) { return k; };
  for (int l = 0; l < layers; ++l) {
    const std::string p = ck + "layers." + std::to_string(l) + ".";
    const TensorView* iw = P.get(p + "self_attn.in_proj_weight", {3 * D, D});
    const TensorView* ib = P.get(p + "self_attn.in_proj_bias", {3 * D});
    const TensorView* ow = P.get(p + "self_attn.out_proj.weight", {D, D});
    const TensorView* ob = P.get(p + "self_attn.out_proj.bias", {D});
    const TensorView* w1 = P.get(p + "linear1.weight", {F, D});
    const TensorView* b1 = P.get(p + "linear1.bias", {F});
    const TensorView* w2 = P.get(p + "linear2.weight", {D, F});
    const TensorView* b2 = P.get(p + "linear2.bias", {D});
    const TensorView* g1 = P.get(p + "norm1.weight", {D});
    const TensorView* e1 = P.get(p + "norm1.bias", {D});
    const TensorView* g2 = P.get(p + "norm2.weight", {D});
    const TensorView* e2 = P.get(p + "norm2.bias", {D});
    if (!iw || !ib || !ow || !ob || !w1 || !b1 || !w2 || !b2 || !g1 || !e1 || !g2 || !e2) return false;
    const float qf = q_fold(D);
    const size_t oq = P.alloc(S.qkv[l].wT, (size_t)3 * D * D);
    pack_linear_chunked(P, oq, iw, 3 * D, D, D, id);
    for (size_t i = 0; i < (size_t)D * D; ++i) P.arena[oq + i] *= qf;          // the q chunks come first
    const size_t oqb = P.alloc(S.qkv[l].b, 3 * D);
    for (int j = 0; j < 3 * D; ++j) P.arena[oqb + j] = ib->d[j] * (j < D ? qf : 1.f);
    SaLayerParams& L = S.layer[l];
    pack_linear_chunked(P, P.alloc(L.WoT, (size_t)D * D), ow, D, D, D, id);
    P.copy(L.bo, ob->d, D);
    pack_linear_chunked(P, P.alloc(L.W1T, (size_t)F * D), w1, F, D, D, id);
    P.copy(L.b1, b1->d, F);
    pack_linear_chunked(P, P.alloc(L.W2T, (size_t)D * F), w2, D, F, F, id);
    P.copy(L.b2, b2->d, D);
    P.copy(L.ln1_g, g1->d, D);
    P.copy(L.ln1_b, e1->d, D);
    P.copy(L.ln2_g, g2->d, D);
    P.copy(L.ln2_b, e2->d, D);
  }
  return true;
}

// the positional encoding of the stack under `ck`: registered buffer [max_len, 1, D] (lib:1051-1058)
bool pack_pos_enc(Packer& P, const nisqa_config& c, const std::string& ck, SaStackWeights& S, int D) {
  auto it = P.t.find(ck + "pos_encoder.pe");
  if (it == P.t.end() || it->second.nd != 3 || it->second.dims[1] != 1 || it->second.dims[2] != D)
    return P.fail("missing tensor " + ck + "pos_encoder.pe");
  if (c.max_segments > 0 && it->second.dims[0] < c.max_segments)
    return P.fail("positional encoding shorter than ms_max_segments");
  P.copy(S.pe, it->second.d, (size_t)it->second.numel);
  return true;
}

int round64(int n) { return (n + 63) / 64 * 64; }

// NISQA_DE's learned alignment at td's fan_out W (q_dim = y_dim = W, lib:404-410): AttLuong W = Linear(y_dim -> q_dim)
// (lib:1348-1351), AttBahdanau Wq, Wy (-> att_dim 128) and v (lib:1329-1337); k-major with W padded to a multiple of 64
// by zero rows (and, for AttLuong, zero columns and bias), so that the projections of the padded td rows are exact and
// their pad columns zero
bool pack_de_align(Packer& P, const nisqa_config& c, int W) {
  DeAlignParams& A = P.w.de;
  const int ld = round64(W);
  if (c.de_align == NISQA_DE_ALIGN_LUONG) {
    const TensorView* w = P.get("align.att.W.weight", {W, W});
    const TensorView* b = P.get("align.att.W.bias", {W});
    if (!w || !b) return false;
    const size_t o = P.alloc(A.wT, (size_t)ld * ld);
    for (int k = 0; k < W; ++k)
      for (int j = 0; j < W; ++j) P.arena[o + (size_t)k * ld + j] = w->d[(size_t)j * W + k];
    memcpy(&P.arena[P.alloc(A.b, ld)], b->d, (size_t)W * 4);
  }
  if (c.de_align == NISQA_DE_ALIGN_BAHDANAU) {
    const TensorView* wq = P.get("align.att.Wq.weight", {128, W});
    const TensorView* bq = P.get("align.att.Wq.bias", {128});
    const TensorView* wy = P.get("align.att.Wy.weight", {128, W});
    const TensorView* by = P.get("align.att.Wy.bias", {128});
    const TensorView* v = P.get("align.att.v.weight", {1, 128});
    if (!wq || !bq || !wy || !by || !v) return false;
    const size_t o = P.alloc(A.wqyT, (size_t)ld * 256), ob = P.alloc(A.bqy, 256);
    for (int k = 0; k < W; ++k)
      for (int j = 0; j < 128; ++j) {
        P.arena[o + (size_t)k * 256 + j] = wq->d[(size_t)j * W + k];
        P.arena[o + (size_t)k * 256 + 128 + j] = wy->d[(size_t)j * W + k];
      }
    memcpy(&P.arena[ob], bq->d, 512);
    memcpy(&P.arena[ob + 128], by->d, 512);
    P.copy(A.v, v->d, 128);
    auto vb = P.t.find("align.att.v.bias");     // (only the peak an alignment call reports reads it: softmax drops it)
    A.vb = vb != P.t.end() && vb->second.numel == 1 ? vb->second.d[0] : 0.f;
  }
  return true;
}

// The pooling module behind the time-dependency block, one head per output (order mos, noi, dis, col, loud:
// lib:1461-1465), reading rows of in.dim features: PoolAttFF, or PoolAtt / PoolAvg / PoolMax / PoolLastStep /
// PoolLastStepBi.  Every vector over the features is laid out in the rows' column order (in_col: the framewise rows of
// td = 'skip' hold conv6 features in the engine's order); a plain description packs the checkpoint's order unchanged.
// PoolAttFF's linear1: [head][Dp][128] for td_sa_kernel's fused tail (self-attention), or - behind an LSTM or the
// framewise model - k-major [Dp padded to 64][head 128] for the tile GEMM (lstm_att), zero in the padding rows
bool pack_pool_heads(Packer& P, const nisqa_config& c, InRows in, bool gemm = false) {
  const int nh = c.n_out, Dp = in.dim;
  P.w.pool_width = Dp;
  P.w.pool_src.clear();
  if (in.order != IN_PLAIN) {
    P.w.pool_src.assign(Dp, 0);
    for (int k = 0; k < Dp; ++k) P.w.pool_src[in_col(in, k)] = k;
  }
  auto prefix = [&](int h) { return nh == 1 ? std::string("pool.model.") : "pool_layers." + std::to_string(h) + ".model."; };
  auto put_row = [&](size_t o, const TensorView* v) {          // one [1, Dp] weight in the rows' column order
    for (int k = 0; k < Dp; ++k) P.arena[o + k] = v->d[in_col(in, k)];
  };
  if (c.pool == NISQA_POOL_ATT_FF) {
    PoolHeadParams& H = P.w.pool_head;
    const size_t oW1 = gemm ? P.alloc(P.w.lstm_att.wT, (size_t)round64(Dp) * nh * 128) : P.alloc(H.W1T, (size_t)nh * Dp * 128),
                 ob1 = gemm ? P.alloc(P.w.lstm_att.b, nh * 128) : P.alloc(H.b1, nh * 128),
                 ow2 = P.alloc(H.w2, nh * 128), ob2 = P.alloc(H.b2, nh),
                 ow3 = P.alloc(H.w3, nh * Dp), ob3 = P.alloc(H.b3, nh);
    for (int h = 0; h < nh; ++h) {
      const std::string p = prefix(h);
      const TensorView* w1 = P.get(p + "linear1.weight", {128, Dp});
      const TensorView* b1 = P.get(p + "linear1.bias", {128});
      const TensorView* w2 = P.get(p + "linear2.weight", {1, 128});
      const TensorView* b2 = P.get(p + "linear2.bias", {1});
      const TensorView* w3 = P.get(p + "linear3.weight", {1, Dp});
      const TensorView* b3 = P.get(p + "linear3.bias", {1});
      if (!w1 || !b1 || !w2 || !b2 || !w3 || !b3) return false;
      if (gemm) {
        for (int k = 0; k < Dp; ++k) {
          const int kc = in_col(in, k);
          for (int j = 0; j < 128; ++j) P.arena[oW1 + (size_t)k * nh * 128 + h * 128 + j] = w1->d[(size_t)j * Dp + kc];
        }
      } else {
        pack_linear_T(P, oW1 + (size_t)h * Dp * 128, w1, 128, Dp);        // [head][D][128] (self-attention rows: plain)
      }
      memcpy(&P.arena[ob1 + h * 128], b1->d, 512);
      memcpy(&P.arena[ow2 + h * 128], w2->d, 512);
      P.arena[ob2 + h] = b2->d[0];
      put_row(ow3 + (size_t)h * Dp, w3);
      P.arena[ob3 + h] = b3->d[0];
    }
    return true;
  }
  // PoolAtt: linear1 (D -> 1 attention logit) + linear2 (D -> 1); PoolAvg / PoolMax / PoolLastStep: linear (D -> 1)
  PoolSimpleParams& Q = P.w.pool_simple;
  const bool att = c.pool == NISQA_POOL_ATT;
  const size_t oa1 = att ? P.alloc(Q.a1, nh * Dp) : 0, oa1b = att ? P.alloc(Q.a1b, nh) : 0;
  const size_t ow3 = P.alloc(Q.w3, nh * Dp), ob3 = P.alloc(Q.b3, nh);
  for (int h = 0; h < nh; ++h) {
    const std::string p = prefix(h);
    const TensorView* a1 = att ? P.get(p + "linear1.weight", {1, Dp}) : nullptr;
    const TensorView* a1b = att ? P.get(p + "linear1.bias", {1}) : nullptr;
    const TensorView* w3 = P.get(p + (att ? "linear2.weight" : "linear.weight"), {1, Dp});
    const TensorView* b3 = P.get(p + (att ? "linear2.bias" : "linear.bias"), {1});
    if ((att && (!a1 || !a1b)) || !w3 || !b3) return false;
    if (att) { put_row(oa1 + (size_t)h * Dp, a1); P.arena[oa1b + h] = a1b->d[0]; }
    put_row(ow3 + (size_t)h * Dp, w3);
    P.arena[ob3 + h] = b3->d[0];
  }
  return true;
}

// The shipped StandardCNN + LSTM shape (nisqa_tts.tar): fc_out 768 -> 20, the BiLSTM(20 -> 128) and its pooling module
bool pack_bilstm128(Packer& P, nisqa_engine* e) {
  const TensorView* fw = P.get("cnn.model.fc_out.weight", {20, 768});
  const TensorView* fb = P.get("cnn.model.fc_out.bias", {20});
  if (!fw || !fb) return false;
  P.w.pool_width = 256;                   // (fwd || bwd)
  const size_t o = P.alloc(P.w.fc.wT, 768 * 20);
  // engine order k' = (h*2 + w)*64 + c  <->  reference view order c*12 + h*2 + w (lib:830)
  for (int hw = 0; hw < 12; ++hw)
    for (int c = 0; c < 64; ++c)
      for (int j = 0; j < 20; ++j) P.arena[o + ((size_t)hw * 64 + c) * 20 + j] = fw->d[(size_t)j * 768 + c * 12 + hw];
  memcpy(&P.arena[P.alloc(P.w.fc.b, 32)], fb->d, 80);
  const std::string p = "time_dependency.model.lstm.";
  LstmParams& L = P.w.lstm;
  const size_t owi = P.alloc(L.w_ih, 2 * 512 * 20), owh = P.alloc(L.w_hh, 2 * 512 * 128), obb = P.alloc(L.b, 2 * 512);
  for (int d = 0; d < 2; ++d) {
    const std::string sfx = d ? "_reverse" : "";
    const TensorView* wi = P.get(p + "weight_ih_l0" + sfx, {512, 20});
    const TensorView* wh = P.get(p + "weight_hh_l0" + sfx, {512, 128});
    const TensorView* bi = P.get(p + "bias_ih_l0" + sfx, {512});
    const TensorView* bh = P.get(p + "bias_hh_l0" + sfx, {512});
    if (!wi || !wh || !bi || !bh) return false;
    memcpy(&P.arena[owi + (size_t)d * 512 * 20], wi->d, 512 * 20 * 4);
    memcpy(&P.arena[owh + (size_t)d * 512 * 128], wh->d, 512 * 128 * 4);
    for (int g = 0; g < 512; ++g) P.arena[obb + d * 512 + g] = bi->d[g] + bh->d[g];
  }
  const TensorView* pw = P.get("pool.model.linear.weight", {1, 256});      // every pooling module of this arch: Linear(256 -> 1)
  const TensorView* pb = P.get("pool.model.linear.bias", {1});
  if (!pw || !pb) return false;
  P.copy(L.w_pool, pw->d, 256);
  e->pool_bias_std = pb->d[0];
  P.copy(P.w.pool_simple.w3, pw->d, 256);
  P.copy(P.w.pool_simple.b3, pb->d, 1);
  return true;
}

// StandardCNN's fc_out (lib:811-836): its width from cnn.model.fc_out.weight (absent: none, 0)
bool read_std_fc(Packer& P, int* fc) {
  *fc = 0;
  auto it = P.t.find("cnn.model.fc_out.weight");
  if (it == P.t.end()) return true;
  *fc = it->second.nd == 2 ? (int)it->second.dims[0] : 0;
  if (*fc < 1 || *fc > 1024) return P.fail("tensor cnn.model.fc_out.weight: width " + std::to_string(*fc) + " outside 1..1024");
  return true;
}

// fc_out 768 -> F k-major with F padded to a multiple of 64 (zero columns), rows in the engine's conv6 order
bool pack_std_fc(Packer& P, int F) {
  const TensorView* fw = P.get("cnn.model.fc_out.weight", {F, 768});
  const TensorView* fb = P.get("cnn.model.fc_out.bias", {F});
  if (!fw || !fb) return false;
  const int Fp = round64(F);
  const size_t o = P.alloc(P.w.fc.wT, (size_t)768 * Fp);
  for (int k = 0; k < 768; ++k)
    for (int j = 0; j < F; ++j) P.arena[o + (size_t)k * Fp + j] = fw->d[(size_t)j * 768 + in_col({768, IN_STD_CONV}, k)];
  memcpy(&P.arena[P.alloc(P.w.fc.b, Fp)], fb->d, (size_t)F * 4);
  return true;
}

// The shape of the LSTM under prefix `p` from its tensors: the weight_hh_l{k}[_reverse] shapes give H, the layer count and
// the directions.  `arg` names the checkpoint argument in the refusal (td_lstm_h / td_2_lstm_h).
bool read_lstm_shape(Packer& P, const std::string& p, const char* arg, Weights::LstmShape* L) {
  auto it = P.t.find(p + "weight_hh_l0");
  if (it == P.t.end()) return P.fail("missing tensor " + p + "weight_hh_l0");
  L->H = it->second.nd == 2 ? (int)it->second.dims[1] : 0;
  if (!lstm_layer_supported(L->H) || it->second.dims[0] != 4 * L->H)
    return P.fail("tensor " + p + "weight_hh_l0: hidden size " + std::to_string(L->H) + " is not implemented by the engine (" +
                  arg + " 32, 64, 96, 128, 192 or 256)");
  L->layers = 0;
  while (P.t.count(p + "weight_hh_l" + std::to_string(L->layers))) ++L->layers;
  if (L->layers > 4) return P.fail("tensor " + p + "weight_hh_l4: the engine runs 1 to 4 LSTM layers");
  L->dirs = P.t.count(p + "weight_hh_l0_reverse") ? 2 : 1;
  return true;
}

// A stacked LSTM of any accepted shape under prefix `p`: W_ih and W_hh of each layer.  Layer 0 reads `in` (its padding
// rows of W_ih stay zero); layer l > 0 reads layer l - 1's dirs H outputs, padded the same way.  Zero weights in the
// padding keep every product exact.
bool pack_lstm_stack(Packer& P, Weights::LstmStack& S, const std::string& p, InRows in0) {
  const Weights::LstmShape& L = S.s;
  const int H = L.H, N = L.dirs * 4 * H, D = L.dirs * H;
  for (int l = 0; l < L.layers; ++l) {
    const int in = l ? D : in0.dim, K = round64(in);
    const size_t owi = P.alloc(S.ih[l].wT, (size_t)K * N), ob = P.alloc(S.ih[l].b, N);
    const size_t owh = P.alloc(S.hh[l], (size_t)L.dirs * 4 * H * H);
    for (int d = 0; d < L.dirs; ++d) {
      const std::string sfx = "_l" + std::to_string(l) + (d ? "_reverse" : "");
      const TensorView* wi = P.get(p + "weight_ih" + sfx, {4 * H, in});
      const TensorView* wh = P.get(p + "weight_hh" + sfx, {4 * H, H});
      const TensorView* bi = P.get(p + "bias_ih" + sfx, {4 * H});
      const TensorView* bh = P.get(p + "bias_hh" + sfx, {4 * H});
      if (!wi || !wh || !bi || !bh) return false;
      for (int k = 0; k < in; ++k) {
        const int kc = l == 0 ? in_col(in0, k) : k;
        for (int g = 0; g < 4 * H; ++g) P.arena[owi + (size_t)k * N + d * 4 * H + g] = wi->d[(size_t)g * in + kc];
      }
      for (int g = 0; g < 4 * H; ++g) P.arena[ob + d * 4 * H + g] = bi->d[g] + bh->d[g];
      memcpy(&P.arena[owh + (size_t)d * 4 * H * H], wh->d, (size_t)4 * H * H * 4);
    }
  }
  return true;
}

// The time-dependency model behind the framewise model - td (self-attention or LSTM), then td_2 (NISQA_DE's fusion,
// alignment and stack, or NISQA / NISQA_DIM's self-attention or LSTM stage, lib:114-141, 236-268) - and the pooling
// module over the last stage's rows
bool pack_td_model(Packer& P, nisqa_engine* e) {
  const nisqa_config& c = e->cfg;
  Weights& W = P.w;
  const std::string td = "time_dependency.model.", td2 = "time_dependency_2.model.";
  // the rows feeding td: AdaptCNN's h3 c3 (engine order; 96 padded to 128 at 6 x 16), SkipCNN's n_mels * seg_len (padded
  // to a multiple of 64 with zero rows: 720 -> 768 at 48 x 15), cnn_fc_out_h, or
  // StandardCNN's fc_out / 768 conv6 features (engine order)
  InRows in;
  if (e->std_cnn()) {
    if (!read_std_fc(P, &W.std_fc)) return false;
    in = W.std_fc ? InRows{W.std_fc, IN_PLAIN} : InRows{768, IN_STD_CONV};
  } else {
    const bool conv_net = c.cnn_kind == NISQA_CNN_CONV;
    in = {c.cnn_fc > 0 ? c.cnn_fc : (conv_net ? W.feat_cols() : e->ff_fan_in()), conv_net && c.cnn_fc == 0 ? IN_ADAPT_CONV : IN_PLAIN,
          W.cnn_c[6], W.pools.p[4]};
  }
  const Weights::LstmShape* last_lstm = nullptr;      // the last stage, when it is an LSTM
  int d1;                                             // td's fan_out
  if (e->td_skip()) {
    // no td (TimeDependency._skip, lib:839-895): td_2 or the pooling module reads the framewise rows themselves
    if (W.std_fc > 0 && !pack_std_fc(P, W.std_fc)) return false;
    if (c.td2_layers > 0) {
      if (!pack_sa_stack(P, W.sa[1], td2, in, c.td2_layers, e->td2_d(), e->td2_f())) return false;
      if (c.td2_pos_enc && !pack_pos_enc(P, c, td2, W.sa[1], e->td2_d())) return false;
      return pack_pool_heads(P, c, {e->td2_d(), IN_PLAIN});
    }
    if (e->td2_lstm()) {
      Weights::LstmShape& L2 = W.lstm_st[1].s;
      if (!read_lstm_shape(P, td2 + "lstm.", "td_2_lstm_h", &L2)) return false;
      if (!pack_lstm_stack(P, W.lstm_st[1], td2 + "lstm.", in)) return false;
      if (c.pool == NISQA_POOL_LAST_STEP_BI && L2.dirs != 2)
        return P.fail("missing tensor " + td2 + "lstm.weight_hh_l0_reverse: PoolLastStepBi needs a bidirectional LSTM");
      return pack_pool_heads(P, c, {L2.dirs * L2.H, IN_PLAIN}, true);
    }
    return pack_pool_heads(P, c, in, true);
  }
  if (e->td_lstm()) {
    Weights::LstmShape& L = W.lstm_st[0].s;
    if (!read_lstm_shape(P, td + "lstm.", "td_lstm_h", &L)) return false;
    W.lstm_shipped = W.std_fc == 20 && L.H == 128 && L.layers == 1 && L.dirs == 2 && c.n_out == 1 && c.pool != NISQA_POOL_ATT &&
                     c.pool != NISQA_POOL_ATT_FF && !e->td2_runs() && !c.double_ended;
    if (W.lstm_shipped) return pack_bilstm128(P, e);
    if (W.std_fc > 0 && !pack_std_fc(P, W.std_fc)) return false;
    if (!pack_lstm_stack(P, W.lstm_st[0], td + "lstm.", in)) return false;
    d1 = L.dirs * L.H;
    last_lstm = &L;
  } else {
    if (W.std_fc > 0 && !pack_std_fc(P, W.std_fc)) return false;
    if (!pack_sa_stack(P, W.sa[0], td, in, c.sa_layers, e->sa_d(), e->sa_f())) return false;
    d1 = e->sa_d();
  }
  int dp = d1;                                        // width of the rows the pooling module reads
  if (c.double_ended || c.td2_layers > 0) {
    // time_dependency_2: behind the fusion of the double-ended model (input nf d1, in the padded fused layout: part p
    // at engine row p round64(d1)), or a second stack behind td in NISQA / NISQA_DIM (input: td's fan_out)
    const int nf = c.de_fuse == NISQA_DE_FUSE_XY_MINUS ? 3 : 2;
    InRows fin = !c.double_ended ? InRows{d1, IN_PLAIN} : InRows{nf * d1, IN_DE_FUSED, d1, round64(d1)};
    if (c.double_ended && c.de_fuse_dim > 0) {        // Fusion.lin_fusion (lib:1399-1401)
      const int D = c.de_fuse_dim, K = fin.dim, rows = in_rows(fin);
      const TensorView* w = P.get("fuse.lin_fusion.weight", {D, K});
      const TensorView* b = P.get("fuse.lin_fusion.bias", {D});
      if (!w || !b) return false;
      const size_t o = P.alloc(W.defuse.wT, (size_t)rows * D);
      for (int k = 0; k < rows; ++k) {
        const int kc = in_col(fin, k);
        if (kc >= 0) for (int j = 0; j < D; ++j) P.arena[o + (size_t)k * D + j] = w->d[(size_t)j * K + kc];
      }
      P.copy(W.defuse.b, b->d, D);
      fin = {D, IN_PLAIN};
    }
    if (!pack_sa_stack(P, W.sa[1], td2, fin, c.td2_layers, e->td2_d(), e->td2_f())) return false;
    if (c.td2_pos_enc && !pack_pos_enc(P, c, td2, W.sa[1], e->td2_d())) return false;
    if (c.double_ended && !pack_de_align(P, c, d1)) return false;
    dp = e->td2_d();
    last_lstm = nullptr;
  } else if (e->td2_lstm()) {
    Weights::LstmShape& L2 = W.lstm_st[1].s;
    if (!read_lstm_shape(P, td2 + "lstm.", "td_2_lstm_h", &L2)) return false;
    if (!pack_lstm_stack(P, W.lstm_st[1], td2 + "lstm.", {d1, IN_PLAIN})) return false;
    dp = L2.dirs * L2.H;
    last_lstm = &L2;
  }
  if (!e->td_lstm() && c.pos_enc && !pack_pos_enc(P, c, td, W.sa[0], e->sa_d())) return false;
  if (c.pool == NISQA_POOL_LAST_STEP_BI && (!last_lstm || last_lstm->dirs != 2))
    return P.fail("missing tensor " + (e->td2_lstm() ? td2 : td) + "lstm.weight_hh_l0_reverse: PoolLastStepBi needs a bidirectional LSTM");
  return pack_pool_heads(P, c, {dp, IN_PLAIN}, last_lstm != nullptr);
}

int pack_weights(nisqa_engine* e, const nisqa_tensor* tensors, int n) {
  Packer P;
  for (int i = 0; i < n; ++i) {
    if (!tensors[i].name || !tensors[i].data) continue;
    TensorView v; v.d = tensors[i].data; v.nd = tensors[i].ndim; v.numel = 1;
    for (int d = 0; d < 4; ++d) { v.dims[d] = d < v.nd ? tensors[i].dims[d] : 1; v.numel *= v.dims[d]; }
    P.t[tensors[i].name] = v;
  }
  const bool ok = pack_framewise(P, e) && pack_td_model(P, e);
  if (!ok) return fail(e, NISQA_ERR_WEIGHTS, P.err);
  CK(e->warena.reserve(P.arena.size() * 4));
  CK(cudaMemcpy(e->warena.p, P.arena.data(), P.arena.size() * 4, cudaMemcpyHostToDevice));
  for (auto& s : P.slots) *s.first = e->warena.as<float>() + s.second;
  if (!P.w.pool_src.empty()) {
    CK(e->emb_src.reserve(P.w.pool_src.size() * 4));
    CK(cudaMemcpy(e->emb_src.p, P.w.pool_src.data(), P.w.pool_src.size() * 4, cudaMemcpyHostToDevice));
  }
  e->w = P.w;
  return 0;
}

// ---------------------------------------------------------------- one pass over a run of clips
// The rings of a feed object (nisqa_feed_push, nisqa_feed_pair_push), as its passes read them: per source (clip i of a
// pass reads source i % n_src) its geometry, its first element in the sample rings and its frame-pair rings
struct FeedRings {
  FeedGeom g[2];
  long long ring_at[2];
  const float* frames[2];
};
// A windows call (nisqa_predict_device_windows): its windows are the clips of the call, in recording order.  A
// window-pairs call (nisqa_predict_device_window_pairs, n_src 2): clip 2p is pair p's degraded window, clip 2p + 1 its
// reference window, and the scores are compact, one row per pair.
struct WinLayout {
  const int* rec;              // [clips] recording of each window
  const int64_t* start;        // [clips] first sample of each window in its recording (model rate)
  const int64_t* rec_off;      // [recordings * n_src] element offset of each converted recording (clip order: recording
                               // b's source s at b * n_src + s) in dev_pcm (ms_sr), or nullptr: the ingest packs each
                               // pass's spans from the caller's batch
  int H, hf, W;                // window hop (samples, mel frames) and length
  const FeedRings* feed = nullptr;    // a feed push: the windows read the feeds' rings (rec: the feed)
  int n_src = 1;               // clips alternate over n_src sources (IngestSources order)
};
// The recording spans of one pass of a windows call and the launch shape of its front end
struct WinPass {
  std::vector<WinSpan> spans;      // source 0's spans, then source 1's
  int n_spans[2] = {0, 0};         // spans per source
  std::vector<int64_t> pcm_off;    // each window's first sample in the pass's PCM (ClipDesc.pcm_off)
  long long pcm_elems = 0;         // ingest: the packed spans
  long long max_span = 0;          // the longest span
  int edge = 0, pairs = 0, ncls = 1;
  const FeedRings* feed = nullptr;   // a feed push: each window's FeedWin row and the most interior pairs of one
  std::vector<FeedWin> fwins;
  int interior = 0;
};

// One scoring call, as its entry point describes it: the clips, exactly one input, the outputs and how the call
// completes.  plan_call fills `plan` and `seg_row`.
struct Call {
  int n_clips;
  const int64_t* n_samples;           // [n_clips] at the rate the clips are scored at
  const int32_t* sample_rate;         // [n_clips]
  int fmt;                            // NISQA_FMT_* of the input
  // the input, exactly one of: per-clip host pointers; a packed device buffer and each clip's element offset (a windows
  // call or feed push: dev_off nullptr, `win` places the windows); the caller's strided device batch
  const void* const* host_pcm = nullptr;
  const void* dev_pcm = nullptr;
  const int64_t* dev_off = nullptr;
  const IngestSources* ingest = nullptr;
  // target_sr > 0 (ms_sr): the caller's batch holds n_rec recordings of rec_n samples at rec_sr (IngestSources order),
  // converted whole to target_sr before the passes, as a span converted alone differs at its edges
  int32_t target_sr = 0;
  int n_rec = 0;
  const int64_t* rec_n = nullptr;
  const int32_t* rec_sr = nullptr;
  // outputs: host or device scores [n_clips][n_out] (a window-pairs call: one row per pair), each clip's segment count
  // and status, and a segments or embeddings call's outputs
  float* scores_host = nullptr;
  float* scores_dev = nullptr;
  int32_t* n_segments;
  int32_t* status;
  const nisqa_segment_out* seg = nullptr;
  const nisqa_embedding_out* emb = nullptr;
  const nisqa_alignment_out* al = nullptr;
  // completion: synchronous, a ticket, or in stream order (the lanes wait for `ready` before they read the input or
  // write outputs)
  bool sync = false;
  int64_t* ticket = nullptr;
  cudaEvent_t ready = nullptr;
  WinLayout* win = nullptr;           // a windows call or feed push
  // a shared-reference call (NISQA_DE): clip 2p + 1 is a slot of pair p's reference ref_index[p] (of n_refs).  Each pass
  // computes a reference once, in the slot of its first running pair there; the pass's other pairs of that reference get
  // alias slots (nothing computed, ClipDesc.ref_clip names the real slot).  The scores are compact, one row per pair.
  const int32_t* ref_index = nullptr;
  int n_refs = 0;
  const int* src_clip = nullptr;      // the caller's batch: [n_clips] each clip's position in IngestSources order (nullptr: g)
  const int* rec_src = nullptr;       // ms_sr: [n_rec] each recording's position in IngestSources order (nullptr: its index)
  const int* clip_rec = nullptr;      // ms_sr: [n_clips] the converted recording each clip reads (nullptr: recording g)
  std::vector<ClipPlan> plan;         // [n_clips]
  std::vector<long long> seg_row;     // segments / embeddings / alignment call: each clip's first output row (-1: none)
  Call(int n, const int64_t* ns, const int32_t* sr, int fmt_, int32_t* n_seg, int32_t* st)
      : n_clips(n), n_samples(ns), sample_rate(sr), fmt(fmt_), n_segments(n_seg), status(st) {}
};

// What one pass reads of its call: clips first_clip .. first_clip + n_clips - 1
struct PassInput {
  int n_clips;
  const ClipPlan* plan;               // [n_clips]
  const int64_t* n_samples;           // [n_clips]
  // exactly one of the three sources:
  const void* const* host_pcm;        // per-clip host pointers, or
  const void* dev_pcm; const int64_t* dev_off;   // packed device buffer + element offsets, or
  const IngestSources* ingest; int first_clip;   // the caller's strided device batch (clips first_clip.. of the call)
  const int* src_clip = nullptr;      // [n_clips] the clips' positions in IngestSources order (nullptr: first_clip + i)
  const int* ref_clip = nullptr;      // NISQA_DE: [n_clips] ClipDesc.ref_clip (nullptr: i + 1); an odd slot that its pair
                                      // does not name is an alias slot (a shared-reference call)
  cudaEvent_t ready;                  // when set, the lane waits for it before it reads the input or writes scores
  int fmt;
  float* scores_dev_out;              // device destination [n_clips][n_out]
  int slot;                           // compute lane
  int stage;                          // staging slot
  const WinPass* win;                 // windows call: the pass's spans (else nullptr)
  bool pair_rows = false;             // window-pairs or shared-reference call: scores_dev_out (and an embeddings call's
                                      // pooled vectors) compact, [n_clips / 2][n_out]
  const nisqa_segment_out* seg;       // segments call: its outputs (else nullptr)
  const nisqa_embedding_out* emb;     // embeddings call: its outputs (else nullptr)
  const nisqa_alignment_out* al;      // alignment call: its outputs (else nullptr)
  const long long* seg_row;           // any of them: the first output row of each clip (-1: none)
};

int lane_allgather(nisqa_engine* e, const float* src, float* dst, size_t count, cudaStream_t st);

// A pass while it is enqueued: where it runs, its device tables and its sizes
struct Pass {
  nisqa_engine* e;
  const nisqa_config& c;
  const Weights& w;
  Lane& LN;                    // compute lane: stream and activation workspaces
  Stage& SG;                   // staging slot: tables and PCM
  cudaStream_t st;
  bool std_mode;
  float* scores;               // [n][n_out]
  int n;
  int n_frames = 0, n_seg = 0, n_qt64 = 0, max_n_seg = 0;
  int max_pairs = 0, Q = 1, max_span = 0;     // launch shape of the front end
  const void* pcm = nullptr;                  // packed PCM on the device
  const ClipDesc* clips = nullptr;            // device tables (staging slot)
  unsigned* clipmax = nullptr;
  const int* seg_prefix = nullptr;
  const int* qt64_prefix = nullptr;
  const int* by_len = nullptr;
  int* seg_frame0 = nullptr;                  // segment table (lane, seg_table_kernel)
  float* seg_thr = nullptr;
  int* seg_clip = nullptr;
  const long long* seg_row = nullptr;         // segments / embeddings / alignment call: the clips' first output rows (staging slot)
  const nisqa_alignment_out* al = nullptr;    // alignment call: its outputs
  const WinSpan* spans = nullptr;             // windows call: the recording spans (staging slot)
  const FeedWin* fwins = nullptr;             // feed push: the windows' rows (staging slot)
  // the rows the pooling module read (segment_rows): D real columns at a stride of ld, the attention logits the pooling
  // path wrote (or nullptr), and each head's last Linear (PoolSimpleParams.w3 / b3; a1 / a1b for PoolAtt)
  const float* pool_x = nullptr;
  int pool_D = 0, pool_ld = 0;
  const float* pool_logits = nullptr;
  PoolSimpleParams pool_P = {};
  Pass(nisqa_engine* e_, const PassInput& in)
      : e(e_), c(e_->cfg), w(e_->w), LN(e_->lanes[in.slot]), SG(e_->stages[in.stage]), st(LN.stream),
        std_mode(e_->std_cnn()), scores(in.scores_dev_out), n(in.n_clips), al(in.al) {}
};

// [n_seg][64 nk] rows that feed a time-dependency block
struct Rows { const float* x; int nk; };

// The pass's host tables - ClipDesc rows, prefix sums of frame pairs, segments, 128- and 64-row query tiles, the clips by
// decreasing length (batched BiLSTM groups) - and, when it has segments, its PCM: uploaded on the copy stream, which the
// lane's stream then waits for
int upload_inputs(Pass& p, const PassInput& in) {
  nisqa_engine* e = p.e;
  const nisqa_config& c = p.c;
  const int n = p.n;
  std::vector<ClipDesc>& cl = e->last_clips;
  cl.assign(n, ClipDesc());
  const size_t np = (size_t)n + 1;
  std::vector<int> pre(5 * np, 0);             // pair | seg | qt | qt64 prefixes | by_len, [n + 1] each
  int* pair_prefix = &pre[0]; int* seg_prefix = &pre[np]; int* qt_prefix = &pre[2 * np]; int* qt64_prefix = &pre[3 * np];
  int* by_len = &pre[4 * np];
  long long pcm_elems = 0, max_run_samples = 0;
  int n_pairs = 0, n_qt = 0;
  for (int i = 0; i < n; ++i) {
    const ClipPlan& pl = in.plan[i];
    ClipDesc& d = cl[i];
    const bool ok = pl.run != 0;
    d.n_samples = (int)in.n_samples[i];
    d.fb_id = ok ? pl.fb_id : 0;
    d.hop = pl.hop; d.win = pl.win;
    d.s0 = (c.n_fft - pl.win) / 2 - c.n_fft / 2;      // pad_center lpad minus the reflect pad
    d.n_frames = ok ? pl.n_frames : 0;
    d.n_seg = ok ? pl.n_seg : 0;
    d.frame_off = p.n_frames; d.seg_off = p.n_seg; d.pair_off = n_pairs;
    d.ref_clip = in.ref_clip ? in.ref_clip[i] : i + 1;
    d.src_clip = in.src_clip ? in.src_clip[i] : in.first_clip + i;
    const bool alias = in.ref_clip && (i & 1) && in.ref_clip[i - 1] != i;       // (no PCM: it is never read)
    if (in.win) d.pcm_off = in.win->pcm_off[i];
    else if (in.host_pcm || in.ingest) { d.pcm_off = pcm_elems; if (!alias) pcm_elems += ((long long)in.n_samples[i] + 15) / 16 * 16; }
    else d.pcm_off = in.dev_off[i];
    if (ok) max_run_samples = std::max<long long>(max_run_samples, in.n_samples[i]);
    pair_prefix[i] = n_pairs; seg_prefix[i] = p.n_seg; qt_prefix[i] = n_qt; qt64_prefix[i] = p.n_qt64;
    p.n_frames += d.n_frames; p.n_seg += d.n_seg;
    n_pairs += (d.n_frames + 1) / 2;
    p.max_pairs = std::max(p.max_pairs, (d.n_frames + 1) / 2);
    n_qt += (d.n_seg + 127) / 128;
    p.n_qt64 += (d.n_seg + 63) / 64;
    p.max_n_seg = std::max(p.max_n_seg, d.n_seg);
    if (ok) { p.Q = std::max(p.Q, (pl.win + 1023) / 1024); p.max_span = std::max(p.max_span, pl.hop + pl.win); }
  }
  pair_prefix[n] = n_pairs; seg_prefix[n] = p.n_seg; qt_prefix[n] = n_qt; qt64_prefix[n] = p.n_qt64;
  if (in.win) { pcm_elems = in.win->pcm_elems; max_run_samples = in.win->max_span; }
  for (int i = 0; i < n; ++i) by_len[i] = i;
  std::stable_sort(by_len, by_len + n, [&](int a, int b) { return cl[a].n_seg > cl[b].n_seg; });
  e->last_n_seg = p.n_seg; e->last_n_frames = p.n_frames;

  // the staging slot (pinned tables, device tables, PCM buffer) is reused every kStages-th pass; the
  // lane's activation workspaces are protected by stream order alone
  Stage& SG = p.SG;
  cudaStream_t cs = e->copy_stream;
  if (SG.busy) { CK(cudaEventSynchronize(SG.ev_done)); SG.busy = false; }
  SG.lane = in.slot;
  // one pinned block: ClipDesc[n] | the prefix arrays
  const size_t tb_clips = (size_t)n * sizeof(ClipDesc), tb_pref = pre.size() * 4;
  const size_t tb_rows_at = (tb_clips + tb_pref + 7) / 8 * 8, tb_rows = in.seg || in.emb || in.al ? (size_t)n * 8 : 0;
  const size_t tb_spans_at = tb_rows_at + tb_rows, tb_spans = in.win ? in.win->spans.size() * sizeof(WinSpan) : 0;
  const size_t tb_fwins_at = (tb_spans_at + tb_spans + 15) / 16 * 16, tb_fwins = in.win ? in.win->fwins.size() * sizeof(FeedWin) : 0;
  CK(SG.h_tables.reserve(tb_fwins_at + tb_fwins));
  char* ht = SG.h_tables.as<char>();
  memcpy(ht, cl.data(), tb_clips);
  memcpy(ht + tb_clips, pre.data(), tb_pref);
  if (tb_rows) {      // (a segments, embeddings or alignment call: the rows of the pass's clips)
    memcpy(ht + tb_rows_at, in.seg_row, tb_rows);
    CK(SG.seg_row.reserve(tb_rows));
    CK(cudaMemcpyAsync(SG.seg_row.p, ht + tb_rows_at, tb_rows, cudaMemcpyHostToDevice, cs));
    p.seg_row = SG.seg_row.as<long long>();
  }
  if (tb_spans) {     // (a windows call: the pass's recording spans)
    memcpy(ht + tb_spans_at, in.win->spans.data(), tb_spans);
    CK(SG.spans.reserve(tb_spans));
    CK(cudaMemcpyAsync(SG.spans.p, ht + tb_spans_at, tb_spans, cudaMemcpyHostToDevice, cs));
    p.spans = SG.spans.as<WinSpan>();
  }
  if (tb_fwins) {     // (a feed push: the pass's windows in the feeds' rings)
    memcpy(ht + tb_fwins_at, in.win->fwins.data(), tb_fwins);
    CK(SG.fwins.reserve(tb_fwins));
    CK(cudaMemcpyAsync(SG.fwins.p, ht + tb_fwins_at, tb_fwins, cudaMemcpyHostToDevice, cs));
    p.fwins = SG.fwins.as<FeedWin>();
  }
  CK(SG.clips.reserve(tb_clips));
  CK(SG.prefixes.reserve(tb_pref));
  CK(SG.clipmax.reserve((size_t)n * 4));
  CK(cudaMemcpyAsync(SG.clips.p, ht, tb_clips, cudaMemcpyHostToDevice, cs));
  CK(cudaMemcpyAsync(SG.prefixes.p, ht + tb_clips, tb_pref, cudaMemcpyHostToDevice, cs));
  CK(cudaMemsetAsync(SG.clipmax.p, 0, (size_t)n * 4, cs));
  p.clips = SG.clips.as<ClipDesc>();
  p.clipmax = SG.clipmax.as<unsigned>();
  p.seg_prefix = SG.prefixes.as<int>() + np;
  p.qt64_prefix = SG.prefixes.as<int>() + 3 * np;
  p.by_len = SG.prefixes.as<int>() + 4 * np;
  e->last_lane = in.slot;
  e->last_stage = in.stage;

  p.pcm = in.dev_pcm;
  if (p.n_seg > 0 && in.host_pcm) {
    const size_t esz = in.fmt == NISQA_FMT_F32 ? 4 : 2;
    CK(SG.pcm.reserve((size_t)pcm_elems * esz));
    // clips that are back to back in host memory with the same 16-element alignment as the
    // device packing travel as ONE copy (a pinned batch buffer becomes a single large DMA)
    for (int i = 0; i < n;) {
      if (cl[i].n_frames <= 0) { ++i; continue; }
      const char* h0 = static_cast<const char*>(in.host_pcm[i]);
      const long long o0 = cl[i].pcm_off;
      size_t bytes = (size_t)in.n_samples[i] * esz;
      int j = i + 1;
      while (j < n && cl[j].n_frames > 0 &&
             static_cast<const char*>(in.host_pcm[j]) == h0 + (size_t)(cl[j].pcm_off - o0) * esz) {
        bytes = (size_t)(cl[j].pcm_off - o0) * esz + (size_t)in.n_samples[j] * esz;
        ++j;
      }
      CK(cudaMemcpyAsync(SG.pcm.as<char>() + (size_t)o0 * esz, h0, bytes, cudaMemcpyHostToDevice, cs));
      i = j;
    }
    p.pcm = SG.pcm.p;
  }
  CK(cudaEventRecord(SG.ev_copied, cs));
  CK(cudaStreamWaitEvent(p.st, SG.ev_copied, 0));
  if (in.ready) CK(cudaStreamWaitEvent(p.st, in.ready, 0));
  if (p.n_seg > 0 && in.ingest) {
    // the caller's batch -> packed mono PCM in the staging slot, on the lane (behind `ready`: the caller's stream order)
    CK(SG.pcm.reserve((size_t)pcm_elems * (in.fmt == NISQA_FMT_F32 ? 4 : 2)));
    Scope sc(e, "ingest");
    if (in.win) {       // each recording span once, however many windows read it (window pairs: the reference mixed)
      for (int k = 0, s0 = 0; k < in.ingest->n_src; s0 += in.win->n_spans[k++])
        launch_ingest_spans(p.st, in.ingest->s[k], p.spans + s0, in.win->n_spans[k], max_run_samples,
                            in.fmt == NISQA_FMT_F32, SG.pcm.p);
    } else
      launch_ingest(p.st, *in.ingest, p.clips, n, max_run_samples, in.fmt == NISQA_FMT_F32, SG.pcm.p);
    p.pcm = SG.pcm.p;
  }
  return 0;
}

// AdaptCNN / StandardCNN: conv1 (fused with conv2 on the tensor-core path), then conv2..conv6 on fp16 plane pairs
// (conv_split.cu) or as fp32 FFMA convolutions (cnn.cu); conv6 writes the features to LN.feats
int conv_layers(Pass& p) {
  nisqa_engine* e = p.e;
  Lane& LN = p.LN;
  const Weights& w = p.w;
  const int* cc = w.cnn_c;
  const bool split = e->conv_tc != 0, fused12 = e->fused12();
  auto plane_hi = [&](int l) { return LN.planes[l].as<char>(); };
  auto plane_lo = [&](int l) { return LN.planes[l].as<char>() + LN.plane_bytes[l]; };
  auto no_kernel = [&](int l) {
    return fail(e, NISQA_ERR_STATE, "no conv" + std::to_string(l) + " kernel for " + std::to_string(cc[l - 1]) + " -> " +
                                        std::to_string(cc[l]) + " channels");
  };
  if (fused12) {
    Scope s(e, "conv12");
    launch_conv12(p.st, p.std_mode, cc[2], LN.mel.as<float>(), p.seg_frame0, p.seg_thr, w.conv[1].w_split,
                  w.conv[1].b_split, w.conv[2].wtc, w.conv[2].b_split, e->tc_scale[2], plane_hi(3), plane_lo(3), p.n_seg);
  } else {
    Scope s(e, "conv1");
    if (!launch_conv1(p.st, p.std_mode, cc[1], LN.mel.as<float>(), p.c.n_mels, p.c.seg_len, p.seg_frame0, p.seg_thr,
                      split ? w.conv[1].w_split : w.conv[1].w, split ? w.conv[1].b_split : w.conv[1].b,
                      split ? nullptr : LN.act[2].as<float>(), p.n_seg, split ? plane_hi(2) : nullptr,
                      split ? plane_lo(2) : nullptr, w.pools.p[0], w.pools.p[1]))
      return no_kernel(1);
  }
  static const char* const names[7] = {"", "", "conv2", "conv3", "conv4", "conv5", "conv6"};
  for (int l = fused12 ? 3 : 2; l <= 6; ++l) {
    Scope s(e, names[l]);
    if (split) {
      if (!launch_conv_split(p.st, p.std_mode, l, cc[l - 1], cc[l], plane_hi(l), plane_lo(l), w.conv[l].wtc, w.conv[l].b_split,
                             e->tc_scale[l], w.conv[l].unit, l < 6 ? plane_hi(l + 1) : nullptr,
                             l < 6 ? plane_lo(l + 1) : nullptr, l == 6 ? LN.feats.as<float>() : nullptr, p.n_seg, w.pools))
        return no_kernel(l);
    } else {
      launch_conv_layer(p.st, p.std_mode, l, LN.act[l].as<float>(), w.conv[l].w, w.conv[l].b,
                        l < 6 ? LN.act[l + 1].as<float>() : LN.feats.as<float>(), p.n_seg);
    }
  }
  return 0;
}

// SkipCNN / DFF (lib:504-583): BN + flatten (+ Linear layers), no convolution
int ff_layers(Pass& p, Rows* out) {
  nisqa_engine* e = p.e;
  Lane& LN = p.LN;
  const Weights& w = p.w;
  Scope s(e, "framewise", 5);
  const int H = p.c.cnn_fc, n_seg = p.n_seg, K = e->ff_fan_in_pad();
  CK(LN.ffa.reserve((size_t)n_seg * std::max(K, H) * 4));
  float* ffa = LN.ffa.as<float>();
  launch_seg_feats(p.st, LN.mel.as<float>(), p.c.n_mels, p.c.seg_len, K, p.seg_frame0, p.seg_thr, w.ff_bn, n_seg, ffa);
  *out = {ffa, K / 64};
  if (H == 0) return 0;
  CK(LN.ffb.reserve((size_t)n_seg * H * 4));
  float* ffb = LN.ffb.as<float>();
  const bool dff = p.c.cnn_kind == NISQA_CNN_DFF;
  launch_linear_tile(p.st, ffa, K, w.ff[0].wT, w.ff[0].b, dff, ffb, H, n_seg, K, H);
  *out = {ffb, H / 64};
  if (!dff) return 0;
  float* pp[2] = {ffa, ffb};
  for (int l = 1; l <= 3; ++l)       // ffb -> ffa -> ffb -> ffa
    launch_linear_tile(p.st, pp[l & 1], H, w.ff[l].wT, w.ff[l].b, 1, pp[(l + 1) & 1], H, n_seg, H, H);
  *out = {ffa, H / 64};
  return 0;
}

// The framewise model: workspaces, front end, segment table, then the CNN (+ AdaptCNN's Linear or StandardCNN's fc_out)
// or SkipCNN / DFF.  `out`: the rows that feed the time-dependency block (the shipped LSTM shape reads LN.feats itself).
int framewise(Pass& p, int fmt, Rows* out, const WinPass* win) {
  nisqa_engine* e = p.e;
  const nisqa_config& c = p.c;
  Lane& LN = p.LN;
  const int n_seg = p.n_seg;
  const bool conv_net = e->conv_net(), split = e->conv_tc != 0;
  CK(LN.mel.reserve((size_t)p.n_frames * c.n_mels * 4));
  CK(LN.segtab.reserve((size_t)n_seg * 12));
  e->last_split = split;
  for (int l = e->fused12() ? 3 : 2; conv_net && l <= 6; ++l) {
    if (split) {
      // the lo plane sits at a fixed offset of the ALLOCATION (not of this pass's n_seg): the zero rows /
      // columns of both planes must stay where they were when the buffer was cleared.  No kernel writes them, so a
      // buffer cleared for another row width or map size (weights of other channel counts or pools loaded since) is
      // cleared again.
      const ConvGeom g = split_geometry(p.std_mode, l, p.w.cnn_c[l - 1], p.w.pools);
      if (LN.plane_g[l].C != g.C || LN.plane_g[l].H != g.H || LN.plane_g[l].W != g.W) {
        LN.planes[l].release();
        LN.plane_g[l] = g;
      }
      CK(LN.planes[l].reserve_zeroed(2 * split_plane_bytes(p.std_mode, l, g.C, n_seg, p.w.pools), p.st));
      LN.plane_bytes[l] = (LN.planes[l].cap / 2) & ~(size_t)1023;
    } else {
      const ConvGeom g = split_geometry(p.std_mode, l, p.w.cnn_c[l - 1]);
      CK(LN.act[l].reserve((size_t)n_seg * g.H * g.W * g.C * 4));
    }
  }
  CK(LN.feats.reserve((size_t)n_seg * (p.std_mode ? 768 : p.w.feat_ld()) * 4));
  p.seg_frame0 = LN.segtab.as<int>();
  p.seg_thr = reinterpret_cast<float*>(p.seg_frame0 + n_seg);
  p.seg_clip = p.seg_frame0 + 2 * (size_t)n_seg;

  { Scope s(e, "frontend");
    if (win) {          // windows: each interior frame pair of a recording span once, the edge pairs per window
      launch_frontend_windows(p.st, c.n_mels, p.pcm, fmt == NISQA_FMT_F32, p.clips, p.n, win->edge, p.spans,
                              (int)win->spans.size(), win->pairs, win->ncls, e->fb_table.as<FbTables>(),
                              e->tw4096.as<float2>(), LN.mel.as<float>(), p.clipmax, p.Q, p.max_span);
      if (win->feed)    // a feed push: the interior rows, computed as their samples arrived, from the rings
        launch_feed_rows(p.st, c.n_mels, p.clips, p.fwins, p.n, win->interior, win->feed->g[0], win->feed->g[1],
                         win->feed->frames[0], win->feed->frames[1], LN.mel.as<float>(), p.clipmax);
    } else {
      launch_frontend(p.st, c.n_mels, p.pcm, fmt == NISQA_FMT_F32, p.clips, p.n, p.max_pairs, e->fb_table.as<FbTables>(),
                      e->tw4096.as<float2>(), LN.mel.as<float>(), p.clipmax, p.Q, p.max_span, e->fe_ppc);
    } }
  { Scope s(e, "seg_table");
    launch_seg_table(p.st, p.clips, p.n, p.seg_prefix, p.clipmax, c.seg_hop, n_seg, p.seg_frame0, p.seg_thr, p.seg_clip); }
  e->last_conv12 = e->fused12();
  if (!conv_net) return ff_layers(p, out);
  const int rc = conv_layers(p);
  if (rc) return rc;
  *out = {LN.feats.as<float>(), p.std_mode ? 12 : p.w.feat_ld() / 64};
  if (p.std_mode && p.w.std_fc > 0 && !p.w.lstm_shipped) {      // StandardCNN's fc_out (lib:830-835), 64-column padded
    Scope s(e, "fc_out");
    const int Fp = round64(p.w.std_fc);
    CK(LN.feats20.reserve((size_t)n_seg * Fp * 4));
    launch_linear_tile(p.st, LN.feats.as<float>(), 768, p.w.fc.wT, p.w.fc.b, 0, LN.feats20.as<float>(), Fp, n_seg, 768, Fp);
    *out = {LN.feats20.as<float>(), Fp / 64};
  }
  if (c.cnn_fc > 0) {      // AdaptCNN's Linear behind conv6 (lib:708-709)
    Scope s(e, "framewise");
    CK(LN.ffb.reserve((size_t)n_seg * c.cnn_fc * 4));
    const int K = p.w.feat_ld();
    launch_linear_tile(p.st, LN.feats.as<float>(), K, p.w.ffc.wT, p.w.ffc.b, 0, LN.ffb.as<float>(), c.cnn_fc, n_seg, K,
                       c.cnn_fc);
    *out = {LN.ffb.as<float>(), c.cnn_fc / 64};
  }
  return 0;
}

// One SelfAttention stack (k = 0: time_dependency, 1: time_dependency_2) over `in`, written to x0 first: Linear + LayerNorm
// (+ positional encoding, + QKV of layer 0) | per layer: attention + out_proj + FFN + LNs (+ next QKV, or - in the stack
// that feeds the pooling module - the PoolAttFF logits behind the last layer).  qkv ping-pongs between two buffers: a
// layer's CTAs read keys / values of rows whose next-layer projection other CTAs are already writing.  Returns the output.
const float* sa_stack(Pass& p, int k, Rows in, bool feeds_pool, float* x0) {
  nisqa_engine* e = p.e;
  const nisqa_config& c = p.c;
  Lane& LN = p.LN;
  const SaStackWeights& S = p.w.sa[k];
  const int D = k ? e->td2_d() : e->sa_d(), F = k ? e->td2_f() : e->sa_f(), layers = k ? c.td2_layers : c.sa_layers;
  const int nc = D / 64;
  const float qs = q_scale(D);
  const int n_heads = (feeds_pool && c.pool == NISQA_POOL_ATT_FF) ? c.n_out : 0;
  float* pp[2] = {(k ? LN.ya : LN.xa).as<float>(), (k ? LN.yb : LN.xb).as<float>()};
  float* qk[2] = {LN.qkv.as<float>(), LN.qkv2.as<float>()};
  { Scope s(e, "lin_ln");
    launch_td_in(p.st, nc, in.x, S.in.wT, in.nk, S.in.b, S.ln_g, S.ln_b, S.qkv[0].wT, S.qkv[0].b, qs, S.pe, p.seg_clip,
                 p.clips, x0, qk[0], p.n_seg); }
  const float* cur = x0;
  for (int l = 0; l < layers; ++l) {
    const bool last = l + 1 == layers;
    Scope s(e, "sa_layer");
    launch_td_sa(p.st, nc, cur, qk[l & 1], p.clips, p.n, p.qt64_prefix, p.n_qt64, S.layer[l], F, pp[l & 1],
                 last ? nullptr : S.qkv[l + 1].wT, last ? nullptr : S.qkv[l + 1].b, qs, qk[(l + 1) & 1], p.w.pool_head,
                 n_heads, LN.logits.as<float>());
    cur = pp[l & 1];
  }
  return cur;
}

// NISQA_DE (lib:404-424): align the reference clip's rows to the degraded clip's and fuse them (+ Fusion.lin_fusion,
// lib:1414-1415).  td_rows: td's output, W real columns at a pitch of round64(W) with zero pad columns.  The fused rows
// are [x, y_al, x - y_al] / [x + y_al, x - y_al] / [x, y_al] with part p at column p round64(W), pad columns zero.
// `out`: the rows that feed time_dependency_2.
int de_fuse(Pass& p, const float* td_rows, int W, Rows* out) {
  nisqa_engine* e = p.e;
  const nisqa_config& c = p.c;
  Lane& LN = p.LN;
  const int n_seg = p.n_seg, nf = c.de_fuse == NISQA_DE_FUSE_XY_MINUS ? 3 : 2, fd = nf * round64(W);
  const size_t work = de_align_work_floats(W, c.de_align, n_seg);
  CK(LN.fused.reserve((size_t)n_seg * fd * 4));
  if (work) CK(LN.dework.reserve(work * 4));
  CK(cudaMemsetAsync(LN.fused.p, 0, (size_t)n_seg * fd * 4, p.st));      // rows of the reference clips stay zero
  { Scope s(e, "de_align", de_align_launches(c.de_align));
    DeAlignOut al = {};
    if (p.al) al = {p.seg_row, p.al->ref_seg, p.al->weight, p.al->centroid, p.al->peak, 0.f};
    launch_de_align(p.st, td_rows, W, n_seg, p.clips, p.n, p.qt64_prefix, p.n_qt64, c.de_align,
                    c.de_align_apply == NISQA_DE_APPLY_SOFT, c.de_fuse, p.w.de, LN.dework.as<float>(), LN.fused.as<float>(),
                    p.al ? &al : nullptr); }
  *out = {LN.fused.as<float>(), fd / 64};
  e->last_de_fused = LN.fused.as<float>();      // (nothing behind the alignment writes fused: lin_fusion writes ffa, td_2 its own buffers)
  e->last_de_fused_d = fd;
  if (c.de_fuse_dim > 0) {
    Scope s(e, "de_align");
    CK(LN.ffa.reserve((size_t)n_seg * c.de_fuse_dim * 4));
    launch_linear_tile(p.st, LN.fused.as<float>(), fd, p.w.defuse.wT, p.w.defuse.b, 0, LN.ffa.as<float>(), c.de_fuse_dim,
                       n_seg, fd, c.de_fuse_dim);
    *out = {LN.ffa.as<float>(), c.de_fuse_dim / 64};
  }
  return 0;
}

// One LSTM stage (k = 0: time_dependency, 1: time_dependency_2) of any accepted shape over `in`: per layer the input
// projection of every step and direction (tile GEMM into gx) and the recurrence (lstm_layer_kernel).  Intermediate layers
// alternate between two workspaces, the last one writes `dst`.  Rows are padded to a multiple of 64 floats with zero
// columns (the next GEMM's K).  `out`: the last layer's rows.
int lstm_stage(Pass& p, int k, Rows in, float* dst, Rows* out) {
  nisqa_engine* e = p.e;
  Lane& LN = p.LN;
  const Weights::LstmStack& S = p.w.lstm_st[k];
  const Weights::LstmShape& L = S.s;
  const int n_seg = p.n_seg, H = L.H, N = L.dirs * 4 * H, D = L.dirs * H, Dp = round64(D);
  float* inter[2] = {(k ? LN.ya : LN.xa).as<float>(), (k ? LN.yb : LN.xb).as<float>()};
  const float* x = in.x;
  int ldx = 64 * in.nk;
  for (int l = 0; l < L.layers; ++l) {
    float* o = l + 1 == L.layers ? dst : inter[l & 1];
    if (Dp != D) CK(cudaMemsetAsync(o, 0, (size_t)n_seg * Dp * 4, p.st));     // the padding columns the next GEMM reads
    Scope s(e, "lstm", 2);
    launch_linear_tile(p.st, x, ldx, S.ih[l].wT, S.ih[l].b, 0, LN.gx.as<float>(), N, n_seg, ldx, N);
    const LstmLayerParams P = {LN.gx.as<float>(), N, S.hh[l], o, Dp};
    launch_lstm_layer(p.st, H, L.dirs, p.clips, p.by_len, p.n, P);
    x = o; ldx = Dp;
  }
  *out = {x, Dp / 64};
  return 0;
}

// The pooling module over the last stage's rows x (D features at a stride of ld).  Behind a self-attention stack the
// PoolAttFF logits come out of its last td_sa layer; behind an LSTM they are a tile GEMM + att_logits.
int pool_rows(Pass& p, const float* x, int D, int ld, bool after_lstm) {
  nisqa_engine* e = p.e;
  const nisqa_config& c = p.c;
  Lane& LN = p.LN;
  const Weights& w = p.w;
  const int n_seg = p.n_seg, nh = c.n_out;
  p.pool_x = x; p.pool_D = D; p.pool_ld = ld;
  p.pool_P = w.pool_simple;
  if (c.pool == NISQA_POOL_ATT_FF) p.pool_P = {nullptr, nullptr, w.pool_head.w3, w.pool_head.b3};
  if (!after_lstm) {
    Scope s(e, "pool");
    if (c.pool == NISQA_POOL_ATT_FF)
      launch_pool_final(p.st, x, D, ld, LN.logits.as<float>(), p.clips, p.n, w.pool_head, nh, p.max_n_seg, p.scores);
    else
      launch_pool_simple(p.st, x, D, ld, p.clips, p.n, c.pool, w.pool_simple, nh, p.max_n_seg, p.scores);
    if (c.double_ended) launch_de_finalize(p.st, p.clips, p.n, nh, p.scores);
    if (c.pool == NISQA_POOL_ATT_FF) p.pool_logits = LN.logits.as<float>();     // (written by the last td_sa layer)
    return 0;
  }
  Scope s(e, "pool", c.pool == NISQA_POOL_ATT_FF ? 3 : 1);
  if (c.pool == NISQA_POOL_ATT_FF) {
    CK(LN.atth.reserve((size_t)n_seg * nh * 128 * 4));
    CK(LN.logits.reserve((size_t)n_seg * nh * 4));
    launch_linear_tile(p.st, x, ld, w.lstm_att.wT, w.lstm_att.b, 1, LN.atth.as<float>(), nh * 128, n_seg, ld, nh * 128);
    launch_att_logits(p.st, LN.atth.as<float>(), w.pool_head.w2, w.pool_head.b2, nh, n_seg, LN.logits.as<float>());
    launch_pool_final(p.st, x, D, ld, LN.logits.as<float>(), p.clips, p.n, w.pool_head, nh, p.max_n_seg, p.scores);
    p.pool_logits = LN.logits.as<float>();      // (taken after the reserve above, which may move the buffer)
  } else {
    launch_pool_simple(p.st, x, D, ld, p.clips, p.n, c.pool, w.pool_simple, nh, p.max_n_seg, p.scores);
  }
  return 0;
}

// The pooling module over the framewise rows of a checkpoint without td and td_2 (x: D real features at a stride of ld):
// launch_pool_wide, the PoolAttFF logits from the tile GEMM + att_logits as behind an LSTM
int pool_framewise(Pass& p, const float* x, int D, int ld) {
  nisqa_engine* e = p.e;
  const nisqa_config& c = p.c;
  Lane& LN = p.LN;
  const Weights& w = p.w;
  const int n_seg = p.n_seg, nh = c.n_out;
  const bool attff = c.pool == NISQA_POOL_ATT_FF, att = c.pool == NISQA_POOL_ATT;
  Scope s(e, "pool", attff ? 4 : att ? 3 : 2);
  if (attff || att) CK(LN.logits.reserve((size_t)n_seg * nh * 4));
  CK(LN.partial.reserve((size_t)p.n * pool_wide_slabs(D) * nh * 4));
  PoolSimpleParams P = w.pool_simple;
  if (attff) {
    CK(LN.atth.reserve((size_t)n_seg * nh * 128 * 4));
    launch_linear_tile(p.st, x, ld, w.lstm_att.wT, w.lstm_att.b, 1, LN.atth.as<float>(), nh * 128, n_seg, ld, nh * 128);
    launch_att_logits(p.st, LN.atth.as<float>(), w.pool_head.w2, w.pool_head.b2, nh, n_seg, LN.logits.as<float>());
    P.w3 = w.pool_head.w3;
    P.b3 = w.pool_head.b3;
  }
  launch_pool_wide(p.st, x, D, ld, c.pool, P, nh, LN.logits.as<float>(), n_seg, p.clips, p.n, LN.partial.as<float>(), p.scores);
  p.pool_x = x; p.pool_D = D; p.pool_ld = ld; p.pool_P = P;
  if (attff || att) p.pool_logits = LN.logits.as<float>();      // (PoolAtt's too: launch_pool_wide wrote them)
  return 0;
}

// The time-dependency model - td (none for td = 'skip'), then td_2 when it runs (NISQA_DE: alignment, fusion and a
// stack) - and the pooling module over the last stage's rows, or over the framewise rows when neither runs.  A
// self-attention stage is sa_stack (the PoolAttFF logits fused into its last layer when it feeds the pooling module),
// an LSTM stage is lstm_stage.  td works in tdout / xa / xb, td_2 in td2in / td2out / ya / yb:
// td's output stays readable after td_2 (NISQA_STAGE_TD1_OUT).
int td_stages(Pass& p, Rows rows) {
  nisqa_engine* e = p.e;
  const nisqa_config& c = p.c;
  Lane& LN = p.LN;
  const Weights& w = p.w;
  const int n_seg = p.n_seg;
  const bool de = c.double_ended != 0, skip = e->td_skip(), sa1 = e->td_sa(), sa2 = c.td2_layers > 0, lstm2 = e->td2_lstm();
  const Weights::LstmShape &L1 = w.lstm_st[0].s, &L2 = w.lstm_st[1].s;      // (L1: all zero without an LSTM td)
  auto res = [&](DevBuf& b, size_t floats) { return b.reserve(floats * 4); };
  // workspaces of the stages that run, reserved before the first launch
  const size_t D1 = skip ? 0 : sa1 ? e->sa_d() : round64(L1.dirs * L1.H), D2 = sa2 ? e->td2_d() : lstm2 ? round64(L2.dirs * L2.H) : 0;
  size_t qkv = 0, gx = 0;
  if (sa1) qkv = 3 * D1; else gx = (size_t)L1.dirs * 4 * L1.H;
  if (sa2) qkv = std::max(qkv, 3 * D2);
  if (lstm2) gx = std::max(gx, (size_t)L2.dirs * 4 * L2.H);
  if (sa1 || L1.layers > 1) { CK(res(LN.xa, n_seg * D1)); CK(res(LN.xb, n_seg * D1)); }
  if (sa2 || (lstm2 && L2.layers > 1)) { CK(res(LN.ya, n_seg * D2)); CK(res(LN.yb, n_seg * D2)); }
  if (qkv) {
    CK(res(LN.qkv, n_seg * qkv));
    CK(res(LN.qkv2, n_seg * qkv));
    CK(res(LN.logits, (size_t)n_seg * c.n_out));
  }
  if (gx) CK(res(LN.gx, n_seg * gx));
  if (D1) CK(res(LN.tdout, n_seg * D1));
  if (sa2) CK(res(LN.td2in, n_seg * D2));
  if (lstm2) CK(res(LN.td2out, n_seg * D2));

  Rows cur;
  int D;                                              // width of cur's rows
  e->last_td_in = nullptr;
  if (skip) {
    cur = rows;
    D = p.std_mode ? (w.std_fc ? w.std_fc : 768) : c.cnn_fc ? c.cnn_fc : c.cnn_kind == NISQA_CNN_CONV ? w.feat_cols() : e->ff_fan_in();
  } else if (sa1) {
    e->last_td_in = LN.tdout.as<float>();
    cur = {sa_stack(p, 0, rows, !e->td2_runs(), LN.tdout.as<float>()), e->sa_d() / 64};
    D = e->sa_d();
  } else {
    const int rc = lstm_stage(p, 0, rows, LN.tdout.as<float>(), &cur);
    if (rc) return rc;
    D = L1.dirs * L1.H;
  }
  e->last_td1_out = nullptr;
  e->last_de_fused = nullptr;
  if (e->td2_runs() && !skip) { e->last_td1_out = cur.x; e->last_td1_out_d = D; e->last_td1_out_ld = 64 * cur.nk; }
  if (de) {
    Rows fused;
    const int rc = de_fuse(p, cur.x, D, &fused);
    if (rc) return rc;
    cur = {sa_stack(p, 1, fused, true, LN.td2in.as<float>()), e->td2_d() / 64};
    D = e->td2_d();
  } else if (sa2) {
    if (!e->last_td_in) e->last_td_in = LN.td2in.as<float>();
    cur = {sa_stack(p, 1, cur, true, LN.td2in.as<float>()), e->td2_d() / 64};
    D = e->td2_d();
  } else if (lstm2) {
    const int rc = lstm_stage(p, 1, cur, LN.td2out.as<float>(), &cur);
    if (rc) return rc;
    D = L2.dirs * L2.H;
  }
  e->last_td_out = cur.x;
  e->last_td_out_d = D;
  e->last_td_out_ld = 64 * cur.nk;
  e->last_td_out_hw = 0;
  if (skip && !e->td2_runs()) {
    if (cur.x == LN.feats.as<float>()) e->last_td_out_hw = p.std_mode ? 12 : w.pools.p[4];   // conv6 features, engine order
    return pool_framewise(p, cur.x, D, 64 * cur.nk);
  }
  return pool_rows(p, cur.x, D, 64 * cur.nk, lstm2 || (!sa1 && !sa2));
}

// The shipped shape's fc_out 768 -> 20, BiLSTM and pooling (PoolLastStepBi fused into the BiLSTM launch)
int lstm_head(Pass& p, const PassInput& in) {
  nisqa_engine* e = p.e;
  const nisqa_config& c = p.c;
  Lane& LN = p.LN;
  const Weights& w = p.w;
  const int n_seg = p.n_seg;
  CK(LN.feats20.reserve((size_t)n_seg * 20 * 4));
  CK(LN.tdout.reserve((size_t)n_seg * 256 * 4));
  CK(LN.partial.reserve((size_t)p.n * 2 * 4));
  { Scope s(e, "fc_out"); launch_fc20(p.st, LN.feats.as<float>(), w.fc.wT, w.fc.b, LN.feats20.as<float>(), n_seg); }
  const bool lastbi = c.pool == NISQA_POOL_LAST_STEP_BI;
  // the other pooling modules read every step's output, and so do segments and embeddings calls
  const bool keep = e->keep_td_out || !lastbi || in.seg || in.emb;
  { Scope s(e, "lstm", 2);
    if (e->lstm_batched)
      launch_lstm_batched(p.st, LN.feats20.as<float>(), p.clips, p.by_len, p.n, w.lstm, keep ? LN.tdout.as<float>() : nullptr,
                          LN.partial.as<float>(), e->pool_bias_std, lastbi ? p.scores : nullptr);
    else
      launch_lstm(p.st, LN.feats20.as<float>(), p.clips, p.n, w.lstm, LN.tdout.as<float>(), LN.partial.as<float>(),
                  e->pool_bias_std, lastbi ? p.scores : nullptr); }
  if (!lastbi) {
    Scope s(e, "pool");
    launch_pool_simple(p.st, LN.tdout.as<float>(), 256, 256, p.clips, p.n, c.pool, w.pool_simple, 1, p.max_n_seg, p.scores);
  }
  e->last_td_in = nullptr;
  e->last_td1_out = nullptr;
  e->last_de_fused = nullptr;
  e->last_td_out = (e->lstm_batched && !keep) ? nullptr : LN.tdout.as<float>();
  e->last_td_out_d = 256;
  e->last_td_out_ld = 256;
  p.pool_x = LN.tdout.as<float>(); p.pool_D = 256; p.pool_ld = 256; p.pool_P = w.pool_simple;
  return 0;
}

// A segments call: every segment's score and pooling weight under each head; an embeddings call: each head's pooled
// vector and optionally the segments' rows - from the rows the pooling module read, to the call's outputs.  A clip the
// call counts rows for but the pass did not run (NISQA_DE: its reference is too short or too long) gets NaN rows, like
// its score; in an alignment call (whose rows de_fuse wrote) ref_seg -1 and NaN values.
int segment_rows(Pass& p, const PassInput& in) {
  nisqa_engine* e = p.e;
  const int nh = p.c.n_out, W = p.w.pool_width;
  const nisqa_segment_out* so = in.seg;
  const nisqa_embedding_out* eo = in.emb;
  for (int i = 0; i < p.n; ++i) {
    const long long r = in.seg_row[i];
    if (r < 0 || in.plan[i].run) continue;
    const size_t n = in.plan[i].n_seg;
    if (so) {
      CK(cudaMemsetAsync(so->scores + (size_t)r * nh, 0xFF, n * nh * 4, p.st));
      CK(cudaMemsetAsync(so->weights + (size_t)r * nh, 0xFF, n * nh * 4, p.st));
    }
    if (eo && eo->rows) CK(cudaMemsetAsync(eo->rows + (size_t)r * W, 0xFF, n * W * 4, p.st));
    if (const nisqa_alignment_out* ao = in.al) {        // (0xFFFFFFFF: int32 -1, a float NaN)
      CK(cudaMemsetAsync(ao->ref_seg + r, 0xFF, n * 4, p.st));
      CK(cudaMemsetAsync(ao->weight + r, 0xFF, n * 4, p.st));
      CK(cudaMemsetAsync(ao->centroid + r, 0xFF, n * 4, p.st));
      CK(cudaMemsetAsync(ao->peak + r, 0xFF, n * 4, p.st));
    }
  }
  const int n_pooled = in.pair_rows ? p.n / 2 : p.n;          // (compact: one vector per pair)
  float* pooled = eo ? eo->pooled + (size_t)(in.pair_rows ? in.first_clip / 2 : in.first_clip) * nh * W : nullptr;
  if (p.n_seg == 0) {     // (nothing ran: NaN vectors, like the scores)
    if (eo) CK(cudaMemsetAsync(pooled, 0xFF, (size_t)n_pooled * nh * W * 4, p.st));
    return 0;
  }
  if (so) {
    Scope s(e, "segments");
    launch_segment_scores(p.st, p.pool_x, p.pool_D, p.pool_ld, p.pool_logits, p.pool_P, nh, p.c.pool, p.clips, p.n, p.seg_row,
                          so->scores, so->weights);
  }
  if (eo) {
    Scope s(e, "embed");
    float* dst = pooled;
    if (in.pair_rows) {   // the pass's interleaved vectors in its staging slot, then row 2p to row p
      CK(p.SG.pair_pooled.reserve((size_t)p.n * nh * W * 4));
      dst = p.SG.pair_pooled.as<float>();
    }
    launch_pool_embed(p.st, p.pool_x, W, p.pool_ld, p.w.pool_src.empty() ? nullptr : e->emb_src.as<int>(), p.pool_logits,
                      p.pool_P, nh, p.c.pool, p.c.double_ended, p.clips, p.n, p.seg_row, dst, eo->rows);
    if (in.pair_rows) {
      const size_t row = (size_t)nh * W * 4;
      CK(cudaMemcpy2DAsync(pooled, row, dst, 2 * row, row, n_pooled, cudaMemcpyDeviceToDevice, p.st));
    }
  }
  return 0;
}

int run_pass(nisqa_engine* e, const PassInput& in) {
  Pass p(e, in);
  e->cur_stream = p.st;
  int rc = upload_inputs(p, in);
  if (rc) return rc;
  if (in.pair_rows) {   // the pass's interleaved pair rows in its staging slot (free once upload_inputs returns)
    CK(p.SG.pair_scores.reserve((size_t)p.n * p.c.n_out * 4));
    p.scores = p.SG.pair_scores.as<float>();
  }
  if (p.n_seg == 0) {   // nothing valid in this pass: NaN scores
    CK(cudaMemsetAsync(p.scores, 0xFF, (size_t)p.n * p.c.n_out * 4, p.st));
  } else {
    Rows rows;
    rc = framewise(p, in.fmt, &rows, in.win);
    if (!rc) rc = p.w.lstm_shipped ? lstm_head(p, in) : td_stages(p, rows);
    if (rc) return rc;
  }
  if (in.seg || in.emb || in.al) {
    rc = segment_rows(p, in);
    if (rc) return rc;
  }
  if (in.pair_rows) {   // row 2p (pair p's score) of each pair to row p of the caller's compact output
    const size_t row = (size_t)p.c.n_out * 4;
    CK(cudaMemcpy2DAsync(in.scores_dev_out, row, p.scores, 2 * row, row, p.n / 2, cudaMemcpyDeviceToDevice, p.st));
  }
  CK(cudaGetLastError());
  CK(cudaEventRecord(p.SG.ev_done, p.st));
  p.SG.busy = true;
  return 0;
}

// The spans of windows i0 .. i1 - 1 of a windows call, each window's offset in the pass's PCM and the launch shape of the
// windows front end (launch_frontend_windows).  A span is a run of windows of one source and recording, every L.n_src-th
// clip, that all run and share one geometry: window m starts m H after the first and covers the first's length or ends
// where the span ends (a recording's short last window; the reference windows that the end of the reference clips).  A
// window that does not run is in no span: no sample of it is packed and no row of it computed.
void win_pass(const nisqa_config& c, const WinLayout& L, const ClipPlan* plan, const int64_t* len, int i0, int i1,
              WinPass* w) {
  *w = WinPass();
  w->pcm_off.assign(i1 - i0, 0);
  const int u = L.n_src;
  for (int src = 0; src < u; ++src) {
    for (int i = i0 + src; i < i1;) {
      if (!plan[i].run) { i += u; continue; }
      const int b = L.rec[i];
      int j = i + u;
      for (; j < i1 && L.rec[j] == b && plan[j].run; j += u) {
        const int64_t pe = L.start[j - u] + len[j - u], e = L.start[j] + len[j];
        const bool full = len[j - u] == len[i];
        if (L.start[j] != L.start[j - u] + L.H || len[j] > len[i] || (full ? e < pe : e != pe)) break;
      }
      WinSpan s = {};
      s.src = b; s.src_off = L.start[i];
      s.n_samples = (int)(L.start[j - u] + len[j - u] - L.start[i]);
      if (L.rec_off) s.pcm_off = L.rec_off[(int64_t)b * u + src] + L.start[i];
      else { s.pcm_off = w->pcm_elems; w->pcm_elems += ((long long)s.n_samples + 15) / 16 * 16; }
      s.clip0 = i - i0; s.cstride = u;
      s.n_win = (j - i) / u;
      s.H = L.H; s.hf = L.hf; s.W = (int)len[i];
      const ClipPlan& pl = plan[i];
      const int s0 = (c.n_fft - pl.win) / 2 - c.n_fft / 2;
      const long long last = ((long long)s.n_samples - pl.hop - pl.win - s0) / pl.hop;    // last first frame of a pair
      if (last >= 0) w->pairs = std::max(w->pairs, (int)(last / 2 + 1));
      if (s.n_win > 1 && (s.hf & 1)) w->ncls = 2;
      for (int k = i; k < j; k += u) {
        w->pcm_off[k - i0] = s.pcm_off + (L.start[k] - L.start[i]);
        int lead, tail;
        interior_pairs(plan[k].n_frames, (int)len[k], s0, pl.hop, pl.win, &lead, &tail);
        w->edge = std::max(w->edge, lead + (plan[k].n_frames + 1) / 2 - tail);
      }
      w->max_span = std::max<long long>(w->max_span, s.n_samples);
      w->spans.push_back(s);
      ++w->n_spans[src];
      i = j;
    }
  }
}

// The windows i0 .. i1 - 1 of a feed push: each window's offset in the sample rings and FeedWin row, and the launch shape
// of its edge pairs and interior rows (nothing to ingest: the push appended its samples to the rings).  A front-clipped
// reference window (pair k with k H < M: it starts at sample 0, off the uniform windows' frame grid) is a one-window
// span, as in win_pass: the span launch computes its interior pairs from the ring, and feed_rows_kernel skips it.
void feed_pass(const WinLayout& L, const ClipPlan* plan, const int64_t* len, int i0, int i1, WinPass* w) {
  *w = WinPass();
  w->feed = L.feed;
  w->pcm_off.resize(i1 - i0);
  w->fwins.resize(i1 - i0);
  for (int i = i0; i < i1; ++i) {
    const int b = L.rec[i], src = i % L.n_src;
    const FeedGeom& g = L.feed->g[src];
    const bool clipped = src == 1 && L.start[i - 1] < g.off;      // (clip i - 1: the pair's degraded window, at k H)
    w->pcm_off[i - i0] = L.feed->ring_at[src] + b * g.stride + L.start[i] % g.R;
    w->fwins[i - i0] = {clipped ? -1 : (L.start[i] / g.hop), b, src};
    if (!plan[i].run) continue;
    int lead, tail;
    interior_pairs(plan[i].n_frames, (int)len[i], g.s0, g.hop, g.win, &lead, &tail);
    w->edge = std::max(w->edge, lead + (plan[i].n_frames + 1) / 2 - tail);
    if (!clipped) { w->interior = std::max(w->interior, tail - lead); continue; }
    WinSpan s = {};
    s.pcm_off = w->pcm_off[i - i0]; s.src = b;
    s.n_samples = (int)len[i];
    s.clip0 = i - i0; s.cstride = L.n_src; s.n_win = 1;
    s.H = L.H; s.hf = L.hf; s.W = (int)len[i];
    const long long last = ((long long)s.n_samples - g.hop - g.win - g.s0) / g.hop;    // last first frame of a pair
    if (last >= 0) w->pairs = std::max(w->pairs, (int)(last / 2 + 1));
    w->max_span = std::max<long long>(w->max_span, s.n_samples);
    w->spans.push_back(s);
    ++w->n_spans[src];
  }
}

// The lane of the next pass
int next_lane(const nisqa_engine* e) { return e->profiling ? 0 : (int)(e->pass_counter % kLanes); }

// The checks and the plan of a call, all before anything is enqueued: each clip's ClipPlan (its front-end tables built),
// segment count and status, and for a segments, embeddings or alignment call each OK clip's first output row, in clip
// order (NISQA_DE: the degraded clips only)
int plan_call(nisqa_engine* e, Call& c) {
  if (!e) return NISQA_ERR_INVALID;
  if (!e->weights_loaded) return fail(e, NISQA_ERR_STATE, "nisqa_load_weights has not been called");
  if (!e->conv_tc && e->conv_net() && !e->w.shipped_channels())
    return fail(e, NISQA_ERR_STATE, "conv_tc=0: the fp32 FFMA convolutions run AdaptCNN channel counts 16 / 32 / 64 only, this "
                                    "checkpoint has " + std::to_string(e->w.cnn_c[1]) + " / " + std::to_string(e->w.cnn_c[2]) +
                                    " / " + std::to_string(e->w.cnn_c[3]) + " (nisqa_set_option(\"conv_tc\", 1))");
  if (!e->conv_tc && e->conv_net() && e->w.pools != kShippedPools) {
    const int* q = e->w.pools.p;
    char buf[160];
    snprintf(buf, sizeof buf, "[%d, %d] [%d, %d] [%d, %d]", q[0], q[1], q[2], q[3], q[4], q[5]);
    return fail(e, NISQA_ERR_STATE, std::string("conv_tc=0: the fp32 FFMA convolutions run the AdaptCNN pools [24, 7] [12, 5] [6, 3] "
                                                "only, this checkpoint has ") + buf + " (nisqa_set_option(\"conv_tc\", 1))");
  }
  const int n_clips = c.n_clips;
  if (n_clips < 0 || (n_clips > 0 && (!c.n_samples || !c.sample_rate)))
    return fail(e, NISQA_ERR_INVALID, "null argument");
  if (c.fmt != NISQA_FMT_S16 && c.fmt != NISQA_FMT_F32) return fail(e, NISQA_ERR_INVALID, "sample_fmt");
  CK(cudaSetDevice(e->device));
  for (auto& t : e->timers) { t.ms = 0.0; t.launches = 0; }
  std::vector<ClipPlan>& plan = c.plan;
  plan.assign(n_clips, ClipPlan());
  for (int i = 0; i < n_clips; ++i) {
    if (c.n_samples[i] > (int64_t)INT32_MAX) return fail(e, NISQA_ERR_INVALID, "clip longer than 2^31 samples");
    plan_clip(e->cfg, c.n_samples[i], c.sample_rate[i], &plan[i]);
    if (plan[i].status == NISQA_CLIP_OK) {
      int rc = build_fb(e, c.sample_rate[i], plan[i].hop, plan[i].win, &plan[i].fb_id);
      if (rc) return rc;
    }
    plan[i].run = plan[i].status == NISQA_CLIP_OK;
    if (c.n_segments) c.n_segments[i] = plan[i].n_seg;
    if (c.status) c.status[i] = plan[i].status;
  }
  if (e->cfg.double_ended) {
    if (n_clips & 1) return fail(e, NISQA_ERR_INVALID, "a double-ended engine takes clips in (degraded, reference) pairs: n_clips must be even");
    for (int i = 0; i < n_clips; i += 2)
      if (!plan[i].run || !plan[i + 1].run) plan[i].run = plan[i + 1].run = 0;      // the pair scores NaN
  }
  if (c.seg || c.emb || c.al) {
    c.seg_row.assign(n_clips, -1);
    long long rows = 0;
    for (int g = 0; g < n_clips; ++g) {
      if (plan[g].status != NISQA_CLIP_OK || (e->cfg.double_ended && (g & 1))) continue;
      c.seg_row[g] = rows;
      rows += plan[g].n_seg;
    }
    if (c.seg && c.seg->n_rows < rows)
      return fail(e, NISQA_ERR_INVALID, "seg->n_rows = " + std::to_string(c.seg->n_rows) + ": the call has " +
                                            std::to_string(rows) + " segment rows");
    if (c.emb && c.emb->rows && c.emb->n_rows < rows)
      return fail(e, NISQA_ERR_INVALID, "emb->n_rows = " + std::to_string(c.emb->n_rows) + ": the call has " +
                                            std::to_string(rows) + " segment rows");
    if (c.al && c.al->n_rows < rows)
      return fail(e, NISQA_ERR_INVALID, "al->n_rows = " + std::to_string(c.al->n_rows) + ": the call has " +
                                            std::to_string(rows) + " degraded segment rows");
  }
  return 0;
}

// The passes of a planned call - runs of whole clips (NISQA_DE: pairs) over the lanes and staging slots in turn - and
// its completion.  *fin_out: the stream the call ends on, the last pass's lane once it has waited for the call's other
// lanes (no pass: the lane the first pass would have run on).
int run_call(nisqa_engine* e, const Call& c, cudaStream_t* fin_out) {
  const int n_clips = c.n_clips;
  const std::vector<ClipPlan>& plan = c.plan;
  const int unit = e->cfg.double_ended ? 2 : 1;      // clips travel in (degraded, reference) pairs through a double-ended engine
  // segments per internal pass: 131072 segments keep ~8 GB of activation planes per compute lane (three lanes stay
  // well inside the 80 GB of an H100) and give the BiLSTM >= 128 clips per launch at configs[3]; one 64-clip batch is 15 808
  // (scaled down for self-attention stacks wider than 64: their activation rows grow with d_model)
  const int d_max = std::max(e->sa_d(), e->cfg.td2_layers > 0 ? e->td2_d() : 64);
  const int max_seg = e->cfg.max_chunk_segments > 0 ? e->cfg.max_chunk_segments : 131072 / (d_max / 64);
  const bool shared = c.ref_index != nullptr;
  const bool pair_rows = shared || (c.win && c.win->n_src == 2);     // compact scores, one row per pair
  const int n_rows = pair_rows ? n_clips / 2 : n_clips;
  float* scores_all = c.scores_dev;
  if (!scores_all) {
    DevBuf& sb = c.ticket ? e->tickets[e->next_ticket % kStages].scores : e->scores;
    CK(sb.reserve((size_t)std::max(n_clips, 1) * e->cfg.n_out * 4));
    scores_all = sb.as<float>();
  }
  const int64_t first_pass = e->pass_counter;
  int i0 = 0;
  e->last_passes = 0;
  WinPass wp;
  // a shared-reference call: each reference's slot in the current pass (-1: none yet), the pass's ClipDesc.ref_clip and
  // its plans with alias slots not run
  std::vector<int> ref_slot(shared ? c.n_refs : 0, -1), ref_clip, named;
  std::vector<ClipPlan> pass_plan;
  while (i0 < n_clips) {
    int i1 = i0; long long segs = 0;
    while (i1 < n_clips) {
      long long s = 0;
      for (int u = 0; u < unit; ++u) s += plan[i1 + u].run ? plan[i1 + u].n_seg : 0;
      const int ru = shared && plan[i1].run ? c.ref_index[i1 / 2] : -1;     // (a pair that runs: its reference runs too)
      if (ru >= 0 && ref_slot[ru] >= 0) s -= plan[i1 + 1].n_seg;            // (its reference is in the pass already)
      if (i1 > i0 && (segs + s > max_seg || i1 - i0 >= 32768)) break;      // (clips ride in grid.y of the front-end: < 65536)
      if (ru >= 0 && ref_slot[ru] < 0) { ref_slot[ru] = i1 + 1 - i0; named.push_back(ru); }
      segs += s; i1 += unit;
    }
    PassInput in;
    in.n_clips = i1 - i0; in.plan = plan.data() + i0; in.n_samples = c.n_samples + i0;
    if (shared) {
      pass_plan.assign(plan.begin() + i0, plan.begin() + i1);
      ref_clip.resize(i1 - i0);
      for (int i = 0; i < i1 - i0; i += 2) {
        ref_clip[i] = ref_clip[i + 1] = i + 1;
        if (!pass_plan[i].run) continue;
        ref_clip[i] = ref_slot[c.ref_index[(i0 + i) / 2]];
        if (ref_clip[i] != i + 1) pass_plan[i + 1].run = 0;        // an alias slot: the front end, CNN and td skip it
      }
      for (int u : named) ref_slot[u] = -1;
      named.clear();
      in.plan = pass_plan.data();
      in.ref_clip = ref_clip.data();
    }
    in.host_pcm = c.host_pcm ? c.host_pcm + i0 : nullptr;
    in.dev_pcm = c.dev_pcm; in.dev_off = c.dev_off ? c.dev_off + i0 : nullptr;
    in.ingest = c.ingest; in.first_clip = i0;
    in.src_clip = c.src_clip ? c.src_clip + i0 : nullptr;
    in.ready = c.ready;
    in.fmt = c.fmt;
    in.pair_rows = pair_rows;
    in.scores_dev_out = scores_all + (size_t)(in.pair_rows ? i0 / 2 : i0) * e->cfg.n_out;
    in.seg = c.seg; in.emb = c.emb; in.al = c.al;
    in.seg_row = c.seg_row.empty() ? nullptr : c.seg_row.data() + i0;
    in.win = nullptr;
    if (c.win) {
      if (c.win->feed) feed_pass(*c.win, plan.data(), c.n_samples, i0, i1, &wp);
      else win_pass(e->cfg, *c.win, plan.data(), c.n_samples, i0, i1, &wp);
      in.win = &wp;
    }
    in.slot = next_lane(e);
    in.stage = (int)(e->pass_counter % kStages);
    ++e->pass_counter;
    int rc = run_pass(e, in);
    if (rc) return rc;
    ++e->last_passes;
    i0 = i1;
  }
  // the lane of the last pass collects: it waits for the other lanes this call used
  const int n_pass = (int)(e->pass_counter - first_pass);
  const cudaStream_t fin = e->lanes[n_pass ? e->last_lane : next_lane(e)].stream;
  for (int k = 0; k < kStages && n_pass > 1; ++k)      // passes of this call that ran on other lanes
    if (e->stages[k].busy && e->stages[k].lane != e->last_lane) CK(cudaStreamWaitEvent(fin, e->stages[k].ev_done, 0));
  if (e->gather_dst && e->nccl_comm && n_clips == e->gather_rows && (c.ticket || c.scores_dev) && !c.win && !shared) {
    // the path's single exchange step, enqueued behind this call's kernels on its own lane
    int rc = lane_allgather(e, scores_all, e->gather_dst, (size_t)n_clips * e->cfg.n_out, fin);
    if (rc) return rc;
    CK(cudaEventRecord(e->stages[e->last_stage].ev_done, fin));
  }
  if (fin_out) *fin_out = fin;
  if (c.ticket) {
    // asynchronous completion: scores land in the ticket's pinned block; nisqa_wait hands them over
    Ticket& tk = e->tickets[e->next_ticket % kStages];
    tk.bytes = (size_t)n_rows * e->cfg.n_out * 4;
    tk.user_scores = c.scores_host;
    CK(tk.pinned.reserve(std::max<size_t>(tk.bytes, 16)));
    if (tk.bytes) CK(cudaMemcpyAsync(tk.pinned.p, scores_all, tk.bytes, cudaMemcpyDeviceToHost, fin));
    if (!tk.done) CK(cudaEventCreateWithFlags(&tk.done, cudaEventDisableTiming));
    CK(cudaEventRecord(tk.done, fin));
    tk.active = true;
    tk.id = e->next_ticket++;
    *c.ticket = tk.id;
    return 0;
  }
  if (c.scores_host && n_rows > 0) {
    const size_t bytes = (size_t)n_rows * e->cfg.n_out * 4;
    CK(e->h_scores.reserve(bytes));
    CK(cudaMemcpyAsync(e->h_scores.p, scores_all, bytes, cudaMemcpyDeviceToHost, fin));
    CK(cudaStreamSynchronize(fin));
    memcpy(c.scores_host, e->h_scores.p, bytes);
  }
  if (c.sync || c.scores_host || e->profiling) CK(cudaStreamSynchronize(fin));
  if (e->profiling) collect_timers(e);
  return 0;
}

// A call of the host entry points: planned, then run
int score(nisqa_engine* e, Call& c) {
  const int rc = plan_call(e, c);
  return rc ? rc : run_call(e, c, nullptr);
}

int finish_ticket(nisqa_engine* e, Ticket& tk) {
  if (!tk.active) return 0;
  CK(cudaEventSynchronize(tk.done));
  if (tk.bytes && tk.user_scores) memcpy(tk.user_scores, tk.pinned.p, tk.bytes);
  tk.active = false;
  return 0;
}

}  // namespace

// ======================================================================== C ABI
extern "C" {

int nisqa_create(nisqa_engine** out, int device, const nisqa_config* cfg) {
  if (!out || !cfg) return NISQA_ERR_INVALID;
  *out = nullptr;
  nisqa_engine* e = new nisqa_engine();
  e->device = device;
  *out = e;     // returned even on failure so that nisqa_last_error() can be read
  // ABI 3 callers pass the smaller struct without the self-attention widths: never read past it (their widths are 64)
  if (cfg->abi_version != 3 && cfg->abi_version != NISQA_B200_ABI_VERSION) return fail(e, NISQA_ERR_INVALID, "abi_version mismatch");
  memset(&e->cfg, 0, sizeof e->cfg);
  memcpy(&e->cfg, cfg, cfg->abi_version == 3 ? offsetof(nisqa_config, sa_d_model) : sizeof(nisqa_config));
  cfg = &e->cfg;
  if (cfg->arch < NISQA_ARCH_ADAPT_SA_ATTFF || cfg->arch > NISQA_ARCH_SKIP_LSTM)
    return fail(e, NISQA_ERR_INVALID, "unsupported architecture");
  const bool sa_td = e->td_sa();             // a self-attention td: arch 0 and 2
  // the pooling module reads the rows of an LSTM (PoolLastStepBi needs it)
  const bool last_lstm = e->td2_lstm() || (e->td_lstm() && cfg->td2_layers == 0);
  const bool any_cnn = sa_td || cfg->arch == NISQA_ARCH_SKIP;       // every framewise model (cnn_kind, cnn_fc) may feed td
  if (e->td_skip() && (cfg->sa_layers != 0 || cfg->sa_d_model != 0 || cfg->sa_ff != 0 || cfg->pos_enc != 0))
    return fail(e, NISQA_ERR_INVALID, "sa_layers / sa_d_model / sa_ff / pos_enc: arch 4 and 5 have no td (keep them 0)");
  if (cfg->arch == NISQA_ARCH_SKIP_LSTM && cfg->cnn_kind != NISQA_CNN_STANDARD)
    return fail(e, NISQA_ERR_INVALID, "cnn_kind: arch 5 (an LSTM td_2 behind no td) needs StandardCNN");
  if (cfg->n_fft != kNfft)
    return fail(e, NISQA_ERR_INVALID, "n_fft = " + std::to_string(cfg->n_fft) + ": the front end runs n_fft 4096");
  if (!frontend_supports_mels(cfg->n_mels))
    return fail(e, NISQA_ERR_INVALID, "n_mels = " + std::to_string(cfg->n_mels) + ": the front end runs 32, 40, 48, 64, 80, 96 or 128 bands");
  if (cfg->seg_len < 3 || cfg->seg_len > 31 || cfg->seg_len % 2 == 0)
    return fail(e, NISQA_ERR_INVALID, "seg_len = " + std::to_string(cfg->seg_len) + ": the engine runs odd segment lengths of 3 to 31 frames");
  if (e->std_cnn() && (cfg->n_mels != kMels || cfg->seg_len != kSegLen))
    return fail(e, NISQA_ERR_INVALID, "n_mels = " + std::to_string(cfg->n_mels) + ", seg_len = " + std::to_string(cfg->seg_len) +
                                          ": StandardCNN is built for 48 x 15 segments");
  if (cfg->n_out != 1 && cfg->n_out != 5) return fail(e, NISQA_ERR_INVALID, "n_out must be 1 or 5");
  if (cfg->seg_hop < 1 || cfg->hop_s <= 0 || cfg->win_s <= 0 || cfg->fmax <= 0)
    return fail(e, NISQA_ERR_INVALID, "bad front-end parameters");
  if (sa_td && (cfg->sa_layers < 1 || cfg->sa_layers > 8))
    return fail(e, NISQA_ERR_INVALID, "sa_layers");
  if (cfg->pool < NISQA_POOL_ATT_FF || cfg->pool > NISQA_POOL_LAST_STEP_BI || (!last_lstm && cfg->pool == NISQA_POOL_LAST_STEP_BI))
    return fail(e, NISQA_ERR_INVALID, "pooling module not available for this architecture (PoolLastStepBi needs an LSTM as the last stage)");
  if (cfg->pos_enc && !sa_td) return fail(e, NISQA_ERR_INVALID, "pos_enc needs a self-attention td");
  if (cfg->cnn_kind < NISQA_CNN_CONV || cfg->cnn_kind > NISQA_CNN_STANDARD || cfg->cnn_fc < 0 || cfg->cnn_fc % 64 != 0 || cfg->cnn_fc > 8192 ||
      (cfg->cnn_kind == NISQA_CNN_DFF && cfg->cnn_fc == 0) || (cfg->cnn_fc != 0 && (!any_cnn || cfg->cnn_kind == NISQA_CNN_STANDARD)) ||
      (cfg->cnn_kind != NISQA_CNN_CONV && !any_cnn && cfg->arch != NISQA_ARCH_SKIP_LSTM) ||
      cfg->de_fuse_dim < 0 || cfg->de_fuse_dim % 64 != 0 || cfg->de_fuse_dim > 8192 || (cfg->de_fuse_dim != 0 && !cfg->double_ended))
    return fail(e, NISQA_ERR_INVALID, "cnn_kind / cnn_fc: SkipCNN, DFF and StandardCNN (cnn_kind) feed a self-attention td or no td; cnn_fc_out_h a "
                                      "multiple of 64 (StandardCNN's fc_out comes from the weights)");
  if (cfg->td2_layers < 0 || cfg->td2_layers > 8 || (cfg->td2_layers > 0 && e->td2_lstm()))
    return fail(e, NISQA_ERR_INVALID, "td_2 = 'self_att' needs arch 0, 1 or 4 (td2_layers 0..8)");
  {
    const int32_t w[4] = {cfg->sa_d_model, cfg->sa_ff, cfg->td2_d_model, cfg->td2_ff};
    const char* nm[4] = {"sa_d_model", "sa_ff", "td2_d_model", "td2_ff"};
    for (int i = 0; i < 4; ++i) {
      const int lim = (i & 1) ? 4096 : 256;        // d_model 64..256, feed-forward width 64..4096, multiples of 64 (0 = 64)
      if (w[i] < 0 || w[i] % 64 != 0 || w[i] > lim || (w[i] != 0 && (i < 2 ? !sa_td : cfg->td2_layers == 0)))
        return fail(e, NISQA_ERR_INVALID, std::string(nm[i]) + " = " + std::to_string(w[i]) +
                                              ": the self-attention kernels take d_model 64..256 and h 64..4096, multiples of 64");
    }
    if (cfg->double_ended && (e->sa_d() != 64 || e->td2_d() != 64))
      return fail(e, NISQA_ERR_INVALID, "NISQA_DE: the engine runs its self-attention stacks at d_model 64 (sa_d_model = td2_d_model = 64)");
  }
  if (cfg->double_ended) {
    // td: self-attention behind any framewise model, or an LSTM behind StandardCNN (arch 1); td_2: self-attention
    if ((cfg->arch != NISQA_ARCH_ADAPT_SA_ATTFF && cfg->arch != NISQA_ARCH_STD_LSTM_LASTBI) || cfg->n_out != 1)
      return fail(e, NISQA_ERR_INVALID, "NISQA_DE: a self-attention td behind any framewise model or an LSTM td behind "
                                        "StandardCNN (arch 0 or 1), one output");
    if (cfg->de_align < NISQA_DE_ALIGN_DOT || cfg->de_align > NISQA_DE_ALIGN_BAHDANAU)
      return fail(e, NISQA_ERR_INVALID, "de_align: dot, cosine, distance, luong or bahd");
    if (cfg->de_align_apply != NISQA_DE_APPLY_HARD && cfg->de_align_apply != NISQA_DE_APPLY_SOFT)
      return fail(e, NISQA_ERR_INVALID, "de_align_apply");
    if (cfg->de_fuse < NISQA_DE_FUSE_XY_MINUS || cfg->de_fuse > NISQA_DE_FUSE_XY) return fail(e, NISQA_ERR_INVALID, "de_fuse");
    if (cfg->td2_layers < 1 || cfg->td2_layers > 8) return fail(e, NISQA_ERR_INVALID, "td_2 must be a self-attention stack (td2_layers 1..8)");
  }
  int count = 0;
  CK(cudaGetDeviceCount(&count));
  if (device < 0 || device >= count) return fail(e, NISQA_ERR_CUDA, "no such CUDA device (there is no CPU fallback)");
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) return fail(e, NISQA_ERR_CUDA, "libnisqa_b200 is compiled for sm_90a (H100) only");
  CK(cudaStreamCreateWithFlags(&e->copy_stream, cudaStreamNonBlocking));
  for (auto& l : e->lanes) CK(cudaStreamCreateWithFlags(&l.stream, cudaStreamNonBlocking));
  for (auto& g : e->stages) {
    CK(cudaEventCreateWithFlags(&g.ev_copied, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&g.ev_done, cudaEventDisableTiming));
  }
  for (cudaEvent_t* ev : {&e->ev_in, &e->ev_out}) CK(cudaEventCreateWithFlags(ev, cudaEventDisableTiming));
  for (auto& r : e->rs) {
    CK(cudaEventCreateWithFlags(&r.ready, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&r.done, cudaEventDisableTiming));
  }
  e->stream = e->lanes[0].stream;
  e->cur_stream = e->stream;
  // twiddles laid out per lane so that every warp load is coalesced:
  //   tw1[r-1][j][lane] = W_4096^(r*(lane+32j)),  tw2[q][lane] = W_1024^(lane*q)
  std::vector<float2> tw(4 * 1024);     // tw1 [3][32][32], tw2 [32][32]
  auto w4096 = [](long k) {
    const double a = -2.0 * M_PI * (double)(k & 4095) / 4096.0;
    return make_float2((float)cos(a), (float)sin(a));
  };
  for (int r = 1; r <= 3; ++r)
    for (int j = 0; j < 32; ++j)
      for (int l = 0; l < 32; ++l) tw[((r - 1) * 32 + j) * 32 + l] = w4096((long)r * (l + 32 * j));
  for (int q = 0; q < 32; ++q)
    for (int l = 0; l < 32; ++l) tw[3 * 1024 + q * 32 + l] = w4096(4L * l * q);
  CK(e->tw4096.reserve(tw.size() * sizeof(float2)));
  CK(cudaMemcpy(e->tw4096.p, tw.data(), tw.size() * sizeof(float2), cudaMemcpyHostToDevice));
  return 0;
}

void nisqa_destroy(nisqa_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  delete e;
}

const char* nisqa_last_error(const nisqa_engine* e) { return e ? e->err.c_str() : "null engine"; }

int nisqa_load_weights(nisqa_engine* e, const nisqa_tensor* tensors, int n) {
  if (!e || !tensors || n <= 0) return NISQA_ERR_INVALID;
  if (!e->stream) return fail(e, NISQA_ERR_STATE, "engine was not created successfully");
  CK(cudaSetDevice(e->device));
  CK(cudaDeviceSynchronize());
  e->weights_loaded = false;      // a failed load may have freed the previous arena
  int prev_c[7];
  memcpy(prev_c, e->w.cnn_c, sizeof prev_c);
  const CnnPools prev_pools = e->w.pools;
  int rc = pack_weights(e, tensors, n);
  if (rc) return rc;
  // the last pass's maps were laid out for the previous channel counts and pools: its stage dumps are gone with them
  if (memcmp(prev_c, e->w.cnn_c, sizeof prev_c) != 0 || prev_pools != e->w.pools) e->last_passes = 0;
  e->weights_loaded = true;
  return 0;
}

int nisqa_predict_pcm(nisqa_engine* e, int n_clips, const void* const* pcm, const int64_t* n_samples,
                      const int32_t* sample_rate, int sample_fmt, float* scores_out,
                      int32_t* n_segments_out, int32_t* status_out) {
  if (!e) return NISQA_ERR_INVALID;
  if (n_clips > 0 && (!pcm || !scores_out)) return fail(e, NISQA_ERR_INVALID, "null argument");
  for (auto& tk : e->tickets) { int rc = finish_ticket(e, tk); if (rc) return rc; }
  Call c(n_clips, n_samples, sample_rate, sample_fmt, n_segments_out, status_out);
  c.host_pcm = pcm; c.scores_host = scores_out; c.sync = true;
  return score(e, c);
}

int nisqa_submit_pcm(nisqa_engine* e, int n_clips, const void* const* pcm, const int64_t* n_samples,
                     const int32_t* sample_rate, int sample_fmt, float* scores_out,
                     int32_t* n_segments_out, int32_t* status_out, int64_t* ticket) {
  if (!e || !ticket) return NISQA_ERR_INVALID;
  if (n_clips > 0 && (!pcm || !scores_out)) return fail(e, NISQA_ERR_INVALID, "null argument");
  if (e->profiling) return fail(e, NISQA_ERR_STATE, "profiling needs the synchronous entry points");
  int rc = finish_ticket(e, e->tickets[e->next_ticket % kStages]);      // at most kStages submissions in flight
  if (rc) return rc;
  Call c(n_clips, n_samples, sample_rate, sample_fmt, n_segments_out, status_out);
  c.host_pcm = pcm; c.scores_host = scores_out; c.ticket = ticket;
  return score(e, c);
}

int nisqa_wait(nisqa_engine* e, int64_t ticket) {
  if (!e) return NISQA_ERR_INVALID;
  CK(cudaSetDevice(e->device));
  // tickets complete in submission order: finish everything up to and including `ticket`
  for (int64_t id = ticket - kStages; id <= ticket; ++id)
    for (auto& tk : e->tickets)
      if (tk.active && tk.id == id) { int rc = finish_ticket(e, tk); if (rc) return rc; }
  return 0;
}

int nisqa_drain(nisqa_engine* e) {
  if (!e || !e->stream) return NISQA_ERR_INVALID;
  cudaSetDevice(e->device);
  // abandon every submission in flight: wait for the device, deliver nothing (the caller's score / PCM buffers
  // may already be gone - that is what this call is for)
  cudaError_t err = cudaDeviceSynchronize();
  for (auto& tk : e->tickets) { tk.active = false; tk.user_scores = nullptr; }
  for (auto& g : e->stages) g.busy = false;
  for (auto& r : e->rs) r.busy = false;
  if (err != cudaSuccess) return fail(e, NISQA_ERR_CUDA, std::string("cudaDeviceSynchronize: ") + cudaGetErrorString(err));
  return 0;
}

int nisqa_predict_pcm_device(nisqa_engine* e, int n_clips, const void* pcm_dev, const int64_t* pcm_offsets,
                             const int64_t* n_samples, const int32_t* sample_rate, int sample_fmt,
                             float* scores_dev, int32_t* n_segments_out, int32_t* status_out, int sync) {
  if (!e) return NISQA_ERR_INVALID;
  if (n_clips > 0 && (!pcm_dev || !pcm_offsets || !scores_dev)) return fail(e, NISQA_ERR_INVALID, "null argument");
  Call c(n_clips, n_samples, sample_rate, sample_fmt, n_segments_out, status_out);
  c.dev_pcm = pcm_dev; c.dev_off = pcm_offsets; c.scores_dev = scores_dev; c.sync = sync != 0;
  return score(e, c);
}


// ---- device resampler of the ingest (SURVEY.md 8f.2): clips at their own rates -> packed float32 PCM at `target` Hz
// in the `out` buffer of the next conversion slot, *slot_out (clip i at element offset offs[i], n_fix[i] samples), on
// stream st.  The clips come from host memory (pcm: copied in, st synchronised before the return) or from the caller's
// device batch (ingest: packed by the ingest kernel, nothing synchronised: the call that enqueued it records the slot's
// `done` behind its last use of the slot and marks it busy).  A busy slot is waited for before it is reused.
static int resample_to_device(nisqa_engine* e, cudaStream_t st, int n_clips, const void* const* pcm,
                              const IngestSources* ingest, const int64_t* n_samples, const int32_t* sample_rate, int fmt,
                              int32_t target, std::vector<int64_t>* offs, std::vector<int64_t>* n_fix, RsSlot** slot_out,
                              const int* src_clip = nullptr) {
  if (fmt != NISQA_FMT_S16 && fmt != NISQA_FMT_F32) return fail(e, NISQA_ERR_INVALID, "sample_fmt");
  if (target <= 0) return fail(e, NISQA_ERR_INVALID, "target sample rate");
  CK(cudaSetDevice(e->device));
  if (!e->rs_nwin) {
    std::vector<double> win;
    int num_table = 0;
    if (!resample_table(&win, &num_table))
      return fail(e, NISQA_ERR_STATE, "nisqa_resample_set_filter has not been called (the interpolation table)");
    CK(e->rs_win.reserve(win.size() * 8));
    CK(cudaMemcpy(e->rs_win.p, win.data(), win.size() * 8, cudaMemcpyHostToDevice));
    e->rs_nwin = (int)win.size(); e->rs_num_table = num_table;
  }
  const size_t esz = fmt == NISQA_FMT_F32 ? 4 : 2;
  std::vector<ResampleClip> rc(n_clips);
  offs->assign(n_clips, 0); n_fix->assign(n_clips, 0);
  long long in_elems = 0, out_elems = 0, t_entries = 0;
  int max_fix = 0;
  for (int i = 0; i < n_clips; ++i) {
    if (n_samples[i] < 0 || n_samples[i] > (int64_t)INT32_MAX / 4 || sample_rate[i] <= 0)
      return fail(e, NISQA_ERR_INVALID, "resample: clip length / sample rate");
    ResampleClip& c = rc[i];
    c.n_in = (int)n_samples[i];
    c.src_clip = src_clip ? src_clip[i] : i;
    c.copy = sample_rate[i] == target;
    c.ratio = (double)target / (double)sample_rate[i];
    c.n_out = c.copy ? c.n_in : (int)((double)c.n_in * c.ratio);                      // resampy: int(shape * ratio)
    c.n_fix = c.copy ? c.n_in : (int)ceil((double)c.n_in * c.ratio);                  // librosa fix_length
    if (!c.copy && c.n_out < 1) return fail(e, NISQA_ERR_INVALID, "resample: signal too short for the target rate");
    c.in_off = in_elems; in_elems += ((long long)c.n_in + 15) / 16 * 16;
    c.out_off = out_elems; out_elems += ((long long)c.n_fix + 15) / 16 * 16;
    c.time_off = t_entries; t_entries += (c.n_fix + 255) / 256 + 1;
    (*offs)[i] = c.out_off; (*n_fix)[i] = c.n_fix;
    max_fix = std::max(max_fix, c.n_fix);
  }
  RsSlot& S = e->rs[e->rs_next++ % kRsSlots];
  *slot_out = &S;
  if (n_clips == 0) return 0;
  if (S.busy) { CK(cudaEventSynchronize(S.done)); S.busy = false; }     // the device-batch call kRsSlots conversions back
  CK(S.raw.reserve((size_t)std::max<long long>(in_elems, 16) * esz));
  CK(S.out.reserve((size_t)std::max<long long>(out_elems, 16) * 4));
  CK(S.times.reserve((size_t)t_entries * 8));
  CK(S.clips.reserve(rc.size() * sizeof(ResampleClip)));
  CK(S.host.reserve(rc.size() * sizeof(ResampleClip)));
  memcpy(S.host.p, rc.data(), rc.size() * sizeof(ResampleClip));
  CK(cudaMemcpyAsync(S.clips.p, S.host.p, rc.size() * sizeof(ResampleClip), cudaMemcpyHostToDevice, st));
  if (ingest) {
    long long max_in = 0;
    for (const ResampleClip& c : rc) max_in = std::max<long long>(max_in, c.n_in);
    e->launches += 1;
    launch_ingest(st, *ingest, S.clips.as<ResampleClip>(), n_clips, max_in, fmt == NISQA_FMT_F32, S.raw.p);
  } else {
    for (int i = 0; i < n_clips; ++i)
      if (rc[i].n_in > 0)
        CK(cudaMemcpyAsync(S.raw.as<char>() + (size_t)rc[i].in_off * esz, pcm[i], (size_t)rc[i].n_in * esz, cudaMemcpyHostToDevice, st));
  }
  e->launches += 2;
  launch_resample(st, S.raw.p, fmt == NISQA_FMT_F32, S.clips.as<ResampleClip>(), n_clips, max_fix, S.times.as<double>(),
                  e->rs_win.as<double>(), e->rs_nwin, e->rs_num_table, S.out.as<float>());
  CK(cudaGetLastError());
  if (!ingest) CK(cudaStreamSynchronize(st));
  return 0;
}

int nisqa_resample_device(nisqa_engine* e, const void* x, int64_t n, int sample_fmt, int32_t sr_orig, int32_t sr_new,
                          float* y, int64_t cap) {
  if (!e || !x || !y) return NISQA_ERR_INVALID;
  std::vector<int64_t> offs, n_fix;
  const void* ptrs[1] = {x};
  RsSlot* S = nullptr;
  int rc = resample_to_device(e, e->lanes[0].stream, 1, ptrs, nullptr, &n, &sr_orig, sample_fmt, sr_new, &offs, &n_fix, &S);
  if (rc) return rc;
  if (n_fix[0] > cap) return fail(e, NISQA_ERR_INVALID, "resample: output buffer too small");
  CK(cudaMemcpy(y, S->out.as<float>() + offs[0], (size_t)n_fix[0] * 4, cudaMemcpyDeviceToHost));
  return (int)n_fix[0];
}

int nisqa_predict_pcm_resampled(nisqa_engine* e, int n_clips, const void* const* pcm, const int64_t* n_samples,
                                const int32_t* sample_rate, int sample_fmt, int32_t target_sr,
                                float* scores_out, int32_t* n_segments_out, int32_t* status_out) {
  if (!e) return NISQA_ERR_INVALID;
  if (n_clips > 0 && (!pcm || !n_samples || !sample_rate || !scores_out)) return fail(e, NISQA_ERR_INVALID, "null argument");
  std::vector<int64_t> offs, n_fix;
  RsSlot* S = nullptr;
  int rc = resample_to_device(e, e->lanes[0].stream, n_clips, pcm, nullptr, n_samples, sample_rate, sample_fmt, target_sr, &offs,
                              &n_fix, &S);
  if (rc) return rc;
  std::vector<int32_t> srs(n_clips, target_sr);
  // the converted clips are ordinary float32 PCM resident in HBM: the device entry of the predict path takes over
  Call c(n_clips, n_fix.data(), srs.data(), NISQA_FMT_F32, n_segments_out, status_out);
  c.dev_pcm = S->out.p; c.dev_off = offs.data(); c.scores_host = scores_out; c.sync = true;
  return score(e, c);
}

// The stream contract of the device calls (device batch, windows, feed pushes), for a planned call: ev_in is recorded on
// the caller's stream.  A call that prepares its input first does so on the lane of its first pass, behind ev_in - an
// ms_sr call converts the whole recordings of the caller's batch (a span converted alone differs at its edges), a feed
// push (f) runs feed_ingest, which appends its samples to the rings - and its passes wait for that; the others' passes
// wait for ev_in.  The caller's stream continues behind the last pass's lane, which has joined the call's other lanes
// (ev_out); the conversion slot and the feed stay in use until then.  On a failure, whatever was enqueued may still read
// the caller's input, the slot or the rings: the caller's stream waits for every lane, and the slot and the feed stay in
// use until then (best effort: the error is already reported).
static int enqueue_call(nisqa_engine* e, void* cuda_stream, Call& c, nisqa_feed* f = nullptr,
                        const std::function<int(cudaStream_t)>& feed_ingest = nullptr) {
  cudaStream_t caller = static_cast<cudaStream_t>(cuda_stream);
  RsSlot* S = nullptr;
  std::vector<int64_t> offs, n_fix, clip_off;
  const int err = [&]() -> int {
    CK(cudaEventRecord(e->ev_in, caller));
    c.ready = e->ev_in;
    if (c.target_sr > 0 || f) {
      cudaStream_t st = e->lanes[next_lane(e)].stream;
      CK(cudaStreamWaitEvent(st, e->ev_in, 0));
      const int rc = f ? feed_ingest(st) : resample_to_device(e, st, c.n_rec, nullptr, c.ingest, c.rec_n, c.rec_sr, c.fmt,
                                                              c.target_sr, &offs, &n_fix, &S, c.rec_src);
      if (rc) return rc;
      if (S) {
        CK(cudaEventRecord(S->ready, st));
        c.dev_pcm = S->out.p; c.ingest = nullptr; c.fmt = NISQA_FMT_F32; c.ready = S->ready;
        if (c.win) c.win->rec_off = offs.data();
        else if (!c.clip_rec) c.dev_off = offs.data();
        else {            // (a shared-reference call: each reference was converted once, its slots read that recording)
          clip_off.resize(c.n_clips);
          for (int g = 0; g < c.n_clips; ++g) clip_off[g] = offs[c.clip_rec[g]];
          c.dev_off = clip_off.data();
        }
      }
    }
    cudaStream_t fin = nullptr;
    const int rc = run_call(e, c, &fin);
    if (rc) return rc;
    if (S) {
      CK(cudaEventRecord(S->done, fin));
      S->busy = c.n_clips > 0;
    }
    if (f) {
      CK(cudaEventRecord(f->done, fin));
      f->pending = true;
    }
    CK(cudaEventRecord(e->ev_out, fin));
    CK(cudaStreamWaitEvent(caller, e->ev_out, 0));
    return 0;
  }();
  if (err) {
    for (auto& l : e->lanes)
      if (cudaEventRecord(e->ev_out, l.stream) == cudaSuccess) cudaStreamWaitEvent(caller, e->ev_out, 0);
    if (S && cudaEventRecord(S->done, caller) == cudaSuccess) S->busy = true;
    if (f && cudaEventRecord(f->done, caller) == cudaSuccess) f->pending = true;
  }
  return err;
}

// The sources of a device call: deg, read with its channel (or mixed to mono), and ref when given, always the mono mix.
// Each must be a batch of n_clips clips (ref: ref_n_clips when >= 0, a shared-reference call) of min_n .. length samples
// (0 for a feed push); messages name deg by deg_nm and ref by "ref.".  -> their ingest sources and the call's format:
// float32 if either is float32 or mixed, else int16.
static int check_sources(nisqa_engine* e, const std::string& deg_nm, const nisqa_device_batch& deg, const nisqa_device_batch* ref,
                         int n_clips, int min_n, IngestSources* ing, int* fmt, int ref_n_clips = -1) {
  const nisqa_device_batch* src[2] = {&deg, ref};
  *ing = {};
  ing->n_src = ref ? 2 : 1;
  bool f32 = false;
  for (int k = 0; k < ing->n_src; ++k) {
    const nisqa_device_batch& b = *src[k];
    const std::string nm = k ? "ref." : deg_nm;
    const int ch = k ? -1 : b.channel;
    if (b.sample_fmt != NISQA_FMT_S16 && b.sample_fmt != NISQA_FMT_F32) return fail(e, NISQA_ERR_INVALID, nm + "sample_fmt");
    if (b.n_clips < 0 || b.n_clips != (k && ref_n_clips >= 0 ? ref_n_clips : n_clips)) return fail(e, NISQA_ERR_INVALID, nm + "n_clips");
    if (b.n_channels < 1) return fail(e, NISQA_ERR_INVALID, nm + "n_channels");
    if (b.n_channels > 1 && (ch < -1 || ch >= b.n_channels)) return fail(e, NISQA_ERR_INVALID, nm + "channel out of range");
    if (b.length < 1 || b.clip_stride < 0 || b.channel_stride < 0) return fail(e, NISQA_ERR_INVALID, nm + "length / strides");
    if (b.sample_rate <= 0) return fail(e, NISQA_ERR_INVALID, nm + "sample_rate");
    if (b.n_clips > 0 && (!b.data || !b.n_samples)) return fail(e, NISQA_ERR_INVALID, nm + "data / n_samples: null argument");
    for (int i = 0; i < b.n_clips; ++i)
      if (b.n_samples[i] < min_n || b.n_samples[i] > b.length)
        return fail(e, NISQA_ERR_INVALID, nm + "n_samples[" + std::to_string(i) + "] = " + std::to_string(b.n_samples[i]) +
                                              ": not within " + std::to_string(min_n) + " .. length (" +
                                              std::to_string(b.length) + ")");
    const bool mix = b.n_channels > 1 && ch < 0;
    ing->s[k] = {b.data, b.clip_stride, b.channel_stride, b.n_channels, ch, b.sample_fmt == NISQA_FMT_F32 ? 1 : 0};
    f32 = f32 || b.sample_fmt == NISQA_FMT_F32 || mix;
  }
  *fmt = f32 ? NISQA_FMT_F32 : NISQA_FMT_S16;
  return 0;
}

// nisqa_predict_device_batch (seg == emb == al == nullptr), nisqa_predict_device_batch_segments,
// nisqa_predict_device_batch_embeddings and nisqa_predict_device_batch_alignment
static int device_batch_call(nisqa_engine* e, void* cuda_stream, const nisqa_device_batch* deg, const nisqa_device_batch* ref,
                             int32_t target_sr, float* scores_dev, const nisqa_segment_out* seg,
                             const nisqa_embedding_out* emb, int32_t* n_segments_out, int32_t* status_out,
                             const nisqa_alignment_out* al = nullptr) {
  if (!e) return NISQA_ERR_INVALID;
  if (!e->stream) return fail(e, NISQA_ERR_STATE, "engine was not created successfully");
  if (!deg) return fail(e, NISQA_ERR_INVALID, "deg: null argument");
  if (e->cfg.double_ended && !ref) return fail(e, NISQA_ERR_INVALID, "ref: a double-ended engine needs the reference batch");
  if (!e->cfg.double_ended && ref) return fail(e, NISQA_ERR_INVALID, "ref: only a double-ended engine takes a reference batch");
  if (target_sr < 0) return fail(e, NISQA_ERR_INVALID, "target_sr");
  IngestSources ing;
  int fmt;
  int rc = check_sources(e, "deg.", *deg, ref, deg->n_clips, 1, &ing, &fmt);
  if (rc) return rc;
  const int n_src = ing.n_src;
  const int n_clips = deg->n_clips * n_src;
  if (n_clips > 0 && !scores_dev) return fail(e, NISQA_ERR_INVALID, "scores_dev: null argument");
  if (seg && n_clips > 0 && (!seg->scores || !seg->weights)) return fail(e, NISQA_ERR_INVALID, "seg: null scores / weights");
  // the engine's clip order: clip g is clip g / n_src of source g % n_src (NISQA_DE: degraded, reference pairs), at its
  // own rate and, with ms_sr, at target_sr
  const nisqa_device_batch* src[2] = {deg, ref};
  std::vector<int64_t> ns(n_clips), n_model(n_clips);
  std::vector<int32_t> sr(n_clips), sr_model(n_clips, target_sr);
  for (int g = 0; g < n_clips; ++g) {
    ns[g] = src[g % n_src]->n_samples[g / n_src]; sr[g] = src[g % n_src]->sample_rate;
    n_model[g] = target_sr > 0 ? nisqa_resample_out_len(ns[g], sr[g], target_sr) : ns[g];
  }
  Call c(n_clips, n_model.data(), target_sr > 0 ? sr_model.data() : sr.data(), fmt, n_segments_out, status_out);
  c.ingest = &ing; c.scores_dev = scores_dev; c.seg = seg; c.emb = emb; c.al = al;
  c.target_sr = target_sr; c.n_rec = n_clips; c.rec_n = ns.data(); c.rec_sr = sr.data();
  rc = plan_call(e, c);
  return rc ? rc : enqueue_call(e, cuda_stream, c);
}

int nisqa_predict_device_batch(nisqa_engine* e, void* cuda_stream, const nisqa_device_batch* deg,
                               const nisqa_device_batch* ref, int32_t target_sr, float* scores_dev,
                               int32_t* n_segments_out, int32_t* status_out) {
  return device_batch_call(e, cuda_stream, deg, ref, target_sr, scores_dev, nullptr, nullptr, n_segments_out, status_out);
}

int nisqa_predict_device_batch_segments(nisqa_engine* e, void* cuda_stream, const nisqa_device_batch* deg,
                                        const nisqa_device_batch* ref, int32_t target_sr, float* scores_dev,
                                        const nisqa_segment_out* seg, int32_t* n_segments_out, int32_t* status_out) {
  if (e && !seg) return fail(e, NISQA_ERR_INVALID, "seg: null argument");
  return device_batch_call(e, cuda_stream, deg, ref, target_sr, scores_dev, seg, nullptr, n_segments_out, status_out);
}

// The refusals of an alignment call that precede its argument checks: a single-ended engine, a null struct or array
static int check_alignment_out(nisqa_engine* e, const nisqa_alignment_out* al) {
  if (!e) return NISQA_ERR_INVALID;
  if (!e->cfg.double_ended)
    return fail(e, NISQA_ERR_INVALID, "al: only a double-ended (NISQA_DE) engine aligns a reference to the degraded clip");
  if (!al) return fail(e, NISQA_ERR_INVALID, "al: null argument");
  if (!al->ref_seg || !al->weight || !al->centroid || !al->peak)
    return fail(e, NISQA_ERR_INVALID, "al: null ref_seg / weight / centroid / peak");
  return 0;
}

int nisqa_predict_device_batch_alignment(nisqa_engine* e, void* cuda_stream, const nisqa_device_batch* deg,
                                         const nisqa_device_batch* ref, int32_t target_sr, float* scores_dev,
                                         const nisqa_alignment_out* al, int32_t* n_segments_out, int32_t* status_out) {
  if (e && !e->stream) return fail(e, NISQA_ERR_STATE, "engine was not created successfully");
  const int rc = check_alignment_out(e, al);
  return rc ? rc : device_batch_call(e, cuda_stream, deg, ref, target_sr, scores_dev, nullptr, nullptr, n_segments_out,
                                     status_out, al);
}

int nisqa_embedding_width(const nisqa_engine* e, int32_t* width) {
  if (!e || !width) return NISQA_ERR_INVALID;
  if (!e->weights_loaded) return NISQA_ERR_STATE;
  *width = e->w.pool_width;
  return 0;
}

int nisqa_predict_device_batch_embeddings(nisqa_engine* e, void* cuda_stream, const nisqa_device_batch* deg,
                                          const nisqa_device_batch* ref, int32_t target_sr, float* scores_dev,
                                          const nisqa_embedding_out* emb, int32_t* n_segments_out, int32_t* status_out) {
  if (e && !emb) return fail(e, NISQA_ERR_INVALID, "emb: null argument");
  if (e && !emb->pooled) return fail(e, NISQA_ERR_INVALID, "emb->pooled: null argument");
  return device_batch_call(e, cuda_stream, deg, ref, target_sr, scores_dev, nullptr, emb, n_segments_out, status_out);
}

// The refusals of a shared-reference call that concern its pairing: a single-ended engine, no reference, a null or out
// of range ref_index
static int check_ref_index(nisqa_engine* e, int n_pairs, int n_refs, const int32_t* ref_index) {
  if (!e->cfg.double_ended)
    return fail(e, NISQA_ERR_INVALID, "ref_index: only a double-ended (NISQA_DE) engine pairs degraded clips with references");
  if (n_refs < 1) return fail(e, NISQA_ERR_INVALID, "ref: no reference clip (a shared-reference call needs at least one)");
  if (!ref_index) return fail(e, NISQA_ERR_INVALID, "ref_index: null argument");
  for (int p = 0; p < n_pairs; ++p)
    if (ref_index[p] < 0 || ref_index[p] >= n_refs)
      return fail(e, NISQA_ERR_INVALID, "ref_index[" + std::to_string(p) + "] = " + std::to_string(ref_index[p]) +
                                            ": not within 0 .. " + std::to_string(n_refs - 1));
  return 0;
}

// A planned shared-reference call's statuses split into its pairs' (the degraded clips') and its references' (each
// planned alone at the model rate: host arithmetic, reported for references no pair names too)
static void shared_ref_rows(const nisqa_engine* e, const Call& c, int n_refs, const int64_t* ref_n, int32_t ref_sr,
                            int32_t target_sr, int32_t* n_segments_out, int32_t* status_out, int32_t* ref_n_segments_out,
                            int32_t* ref_status_out) {
  for (int p = 0; p < c.n_clips / 2; ++p) {
    if (n_segments_out) n_segments_out[p] = c.plan[2 * p].n_seg;
    if (status_out) status_out[p] = c.plan[2 * p].status;
  }
  for (int u = 0; u < n_refs; ++u) {
    ClipPlan pl;
    plan_clip(e->cfg, target_sr > 0 ? nisqa_resample_out_len(ref_n[u], ref_sr, target_sr) : ref_n[u],
              target_sr > 0 ? target_sr : ref_sr, &pl);
    if (ref_n_segments_out) ref_n_segments_out[u] = pl.n_seg;
    if (ref_status_out) ref_status_out[u] = pl.status;
  }
}

int nisqa_predict_device_batch_shared_ref(nisqa_engine* e, void* cuda_stream, const nisqa_device_batch* deg,
                                          const nisqa_device_batch* ref, const int32_t* ref_index, int32_t target_sr,
                                          float* scores_dev, const nisqa_segment_out* seg, const nisqa_embedding_out* emb,
                                          const nisqa_alignment_out* al, int32_t* n_segments_out, int32_t* status_out,
                                          int32_t* ref_n_segments_out, int32_t* ref_status_out) {
  if (!e) return NISQA_ERR_INVALID;
  if (!e->stream) return fail(e, NISQA_ERR_STATE, "engine was not created successfully");
  if (!deg) return fail(e, NISQA_ERR_INVALID, "deg: null argument");
  if (!ref) return fail(e, NISQA_ERR_INVALID, "ref: null argument");
  int rc = check_ref_index(e, std::max(deg->n_clips, 0), ref->n_clips, ref_index);
  if (rc) return rc;
  if (target_sr < 0) return fail(e, NISQA_ERR_INVALID, "target_sr");
  if (al && (rc = check_alignment_out(e, al))) return rc;
  IngestSources ing;
  int fmt;
  if ((rc = check_sources(e, "deg.", *deg, ref, deg->n_clips, 1, &ing, &fmt, ref->n_clips))) return rc;
  const int B = deg->n_clips, n_clips = 2 * B;
  if (B > 0 && !scores_dev) return fail(e, NISQA_ERR_INVALID, "scores_dev: null argument");
  if (seg && B > 0 && (!seg->scores || !seg->weights)) return fail(e, NISQA_ERR_INVALID, "seg: null scores / weights");
  if (emb && !emb->pooled) return fail(e, NISQA_ERR_INVALID, "emb->pooled: null argument");
  // the engine's clips: pair p's degraded clip, then a slot of its reference (IngestSources position 2 u + 1); with ms_sr
  // the degraded clips and each named reference once are converted, in that order
  std::vector<int64_t> ns(n_clips), n_model(n_clips), rec_n;
  std::vector<int32_t> sr(n_clips), sr_model(n_clips, target_sr), rec_sr, nseg(n_clips), status(n_clips);
  std::vector<int> src(n_clips), rec_src, clip_rec(n_clips), rec_of(ref->n_clips, -1);
  for (int g = 0; g < n_clips; ++g) {
    const int u = ref_index[g / 2];
    const nisqa_device_batch& b = (g & 1) ? *ref : *deg;
    const int k = (g & 1) ? u : g / 2;
    ns[g] = b.n_samples[k]; sr[g] = b.sample_rate; src[g] = (g & 1) ? 2 * u + 1 : g;
    n_model[g] = target_sr > 0 ? nisqa_resample_out_len(ns[g], sr[g], target_sr) : ns[g];
    if (!(g & 1)) { clip_rec[g] = g / 2; rec_src.push_back(g); rec_n.push_back(ns[g]); rec_sr.push_back(sr[g]); }
  }
  for (int p = 0; p < B; ++p) {
    int& r = rec_of[ref_index[p]];
    if (r < 0) { r = (int)rec_src.size(); rec_src.push_back(src[2 * p + 1]); rec_n.push_back(ns[2 * p + 1]); rec_sr.push_back(ref->sample_rate); }
    clip_rec[2 * p + 1] = r;
  }
  Call c(n_clips, n_model.data(), target_sr > 0 ? sr_model.data() : sr.data(), fmt, nseg.data(), status.data());
  c.ingest = &ing; c.src_clip = src.data(); c.scores_dev = scores_dev; c.seg = seg; c.emb = emb; c.al = al;
  c.ref_index = ref_index; c.n_refs = ref->n_clips;
  c.target_sr = target_sr; c.n_rec = (int)rec_src.size(); c.rec_n = rec_n.data(); c.rec_sr = rec_sr.data();
  c.rec_src = rec_src.data(); c.clip_rec = clip_rec.data();
  if ((rc = plan_call(e, c))) return rc;
  shared_ref_rows(e, c, ref->n_clips, ref->n_samples, ref->sample_rate, target_sr, n_segments_out, status_out,
                  ref_n_segments_out, ref_status_out);
  return enqueue_call(e, cuda_stream, c);
}

int nisqa_submit_pcm_pairs(nisqa_engine* e, int n_pairs, const void* const* pcm, const int64_t* n_samples,
                           const int32_t* sample_rate, int n_refs, const void* const* ref_pcm, const int64_t* ref_n_samples,
                           const int32_t* ref_sample_rate, const int32_t* ref_index, int sample_fmt, float* scores_out,
                           int32_t* n_segments_out, int32_t* status_out, int32_t* ref_n_segments_out,
                           int32_t* ref_status_out, int64_t* ticket) {
  if (!e || !ticket) return NISQA_ERR_INVALID;
  if (n_pairs < 0) return fail(e, NISQA_ERR_INVALID, "n_pairs");
  int rc = check_ref_index(e, n_pairs, n_refs, ref_index);
  if (rc) return rc;
  if (n_pairs > 0 && (!pcm || !n_samples || !sample_rate || !scores_out)) return fail(e, NISQA_ERR_INVALID, "null argument");
  if (!ref_pcm || !ref_n_samples || !ref_sample_rate)
    return fail(e, NISQA_ERR_INVALID, "ref_pcm / ref_n_samples / ref_sample_rate: null argument");
  if (e->profiling) return fail(e, NISQA_ERR_STATE, "profiling needs the synchronous entry points");
  if ((rc = finish_ticket(e, e->tickets[e->next_ticket % kStages]))) return rc;      // at most kStages submissions in flight
  const int n_clips = 2 * n_pairs;
  std::vector<const void*> ptr(n_clips);
  std::vector<int64_t> ns(n_clips);
  std::vector<int32_t> sr(n_clips), nseg(n_clips), status(n_clips);
  for (int p = 0; p < n_pairs; ++p) {
    const int u = ref_index[p];
    ptr[2 * p] = pcm[p]; ns[2 * p] = n_samples[p]; sr[2 * p] = sample_rate[p];
    ptr[2 * p + 1] = ref_pcm[u]; ns[2 * p + 1] = ref_n_samples[u]; sr[2 * p + 1] = ref_sample_rate[u];
  }
  Call c(n_clips, ns.data(), sr.data(), sample_fmt, nseg.data(), status.data());
  c.host_pcm = ptr.data(); c.scores_host = scores_out; c.ticket = ticket;
  c.ref_index = ref_index; c.n_refs = n_refs;
  if ((rc = plan_call(e, c))) return rc;
  for (int p = 0; p < n_pairs; ++p) {
    if (n_segments_out) n_segments_out[p] = c.plan[2 * p].n_seg;
    if (status_out) status_out[p] = c.plan[2 * p].status;
  }
  for (int u = 0; u < n_refs; ++u) {
    ClipPlan pl;
    plan_clip(e->cfg, ref_n_samples[u], ref_sample_rate[u], &pl);
    if (ref_n_segments_out) ref_n_segments_out[u] = pl.n_seg;
    if (ref_status_out) ref_status_out[u] = pl.status;
  }
  return run_call(e, c, nullptr);
}

// The window list of a windows call or feed push, in recording order
struct WinList {
  std::vector<int> rec;
  std::vector<int64_t> start, len;
};
// Window k of recording b (T samples at the model rate) appended to the list, followed, when the call has a reference
// (n_src 2: T_ref samples, margin M), by its reference window
void add_window(WinList* w, int n_src, int b, int64_t k, int64_t T, int64_t T_ref, int64_t W, int64_t H, int64_t M) {
  w->rec.push_back(b); w->start.push_back(k * H); w->len.push_back(std::min(W, T - k * H));
  if (n_src == 2) {
    int64_t r0, rn;
    ref_window(k, T_ref, W, H, M, &r0, &rn);
    w->rec.push_back(b); w->start.push_back(r0); w->len.push_back(rn);
  }
}
// The per-clip segment counts and statuses of a window list as per-row outputs (each may be nullptr): row r is clip r,
// or with a reference (n_src 2) clips 2r (the degraded window) and 2r + 1 (the reference window)
void split_rows(int n_src, int64_t rows, const int32_t* nseg, const int32_t* status, int32_t* n_seg_out, int32_t* status_out,
                int32_t* ref_n_seg_out, int32_t* ref_status_out) {
  for (int64_t r = 0; r < rows; ++r) {
    if (n_seg_out) n_seg_out[r] = nseg[n_src * r];
    if (status_out) status_out[r] = status[n_src * r];
    if (n_src == 2 && ref_n_seg_out) ref_n_seg_out[r] = nseg[2 * r + 1];
    if (n_src == 2 && ref_status_out) ref_status_out[r] = status[2 * r + 1];
  }
}
// The rows of a window list planned at `rate` (host arithmetic: the counts a call reports)
void plan_rows(const nisqa_config& c, int rate, int n_src, const WinList& w, int32_t* n_seg_out, int32_t* status_out,
               int32_t* ref_n_seg_out, int32_t* ref_status_out) {
  const size_t n = w.len.size();
  std::vector<int32_t> nseg(n), status(n);
  for (size_t i = 0; i < n; ++i) {
    ClipPlan p;
    plan_clip(c, w.len[i], rate, &p);
    nseg[i] = p.n_seg; status[i] = p.status;
  }
  split_rows(n_src, n / n_src, nseg.data(), status.data(), n_seg_out, status_out, ref_n_seg_out, ref_status_out);
}

// nisqa_predict_device_windows (ref == nullptr, margin_frames 0; the recordings deg named `nm` "rec") and
// nisqa_predict_device_window_pairs (nm "deg")
static int windows_call(nisqa_engine* e, void* cuda_stream, const char* nm, const nisqa_device_batch* deg,
                        const nisqa_device_batch* ref, int32_t target_sr, int64_t window, int32_t hop_frames,
                        int32_t margin_frames, float* scores_dev, int64_t n_rows, int32_t* n_segments_out,
                        int32_t* status_out, int32_t* ref_n_segments_out, int32_t* ref_status_out,
                        const nisqa_alignment_out* al = nullptr) {
  if (target_sr < 0) return fail(e, NISQA_ERR_INVALID, "target_sr");
  IngestSources ing;
  int fmt;
  int rc = check_sources(e, std::string(nm) + ".", *deg, ref, deg->n_clips, 1, &ing, &fmt);
  if (rc) return rc;
  const int S = ing.n_src;
  if (ref && target_sr == 0 && ref->sample_rate != deg->sample_rate)
    return fail(e, NISQA_ERR_INVALID, "ref.sample_rate = " + std::to_string(ref->sample_rate) + ": the windows of both recordings "
                                      "run at one rate, deg.sample_rate = " + std::to_string(deg->sample_rate));
  const int rate = target_sr > 0 ? target_sr : deg->sample_rate;
  std::string why;
  int H = 0;
  int64_t M = 0;
  if (!window_pair_geometry(e->cfg, rate, window, hop_frames, margin_frames, &H, &M, &why))
    return fail(e, NISQA_ERR_INVALID, why);
  const int W = (int)window;
  // the windows (pairs) of every recording, in recording order (host arithmetic: nisqa_window_counts,
  // nisqa_window_pair_counts), and the recordings in IngestSources order for an ms_sr conversion
  const int n_rec = deg->n_clips;
  WinList wl;
  std::vector<int64_t> rs_n(S * (size_t)n_rec);
  std::vector<int32_t> rs_sr(S * (size_t)n_rec);
  for (int b = 0; b < n_rec; ++b) {
    int64_t T[2] = {0, 0};
    for (int k = 0; k < S; ++k) {
      const nisqa_device_batch* x = k ? ref : deg;
      rs_n[S * b + k] = x->n_samples[b]; rs_sr[S * b + k] = x->sample_rate;
      T[k] = target_sr > 0 ? nisqa_resample_out_len(x->n_samples[b], x->sample_rate, target_sr) : x->n_samples[b];
      if (T[k] > (int64_t)INT32_MAX)
        return fail(e, NISQA_ERR_INVALID, std::string(k ? "ref" : nm) + ".n_samples[" + std::to_string(b) + "]: " +
                                              std::to_string(T[k]) + " samples at the model rate, more than 2^31 - 1");
    }
    const int64_t K = window_count(T[0], W, H);
    if ((int64_t)wl.rec.size() + S * K > INT32_MAX)
      return fail(e, NISQA_ERR_INVALID, S == 2 ? "deg: more than 2^30 - 1 window pairs" : "rec: more than 2^31 - 1 windows");
    for (int64_t k = 0; k < K; ++k) add_window(&wl, S, b, k, T[0], T[1], W, H, M);
  }
  const int N = (int)wl.rec.size(), rows = N / S;
  if (n_rows < rows)
    return fail(e, NISQA_ERR_INVALID, "n_rows = " + std::to_string(n_rows) + ": the call has " + std::to_string(rows) +
                                          (S == 2 ? " window pairs" : " windows"));
  if (N > 0 && !scores_dev) return fail(e, NISQA_ERR_INVALID, "scores_dev: null argument");
  const int hop = (int)((double)rate * e->cfg.hop_s);
  WinLayout L = {wl.rec.data(), wl.start.data(), nullptr, H, H / hop, W};
  L.n_src = S;
  std::vector<int32_t> srs(N, rate), nseg(N), status(N);
  Call c(N, wl.len.data(), srs.data(), fmt, nseg.data(), status.data());
  c.ingest = &ing; c.scores_dev = scores_dev; c.win = &L; c.al = al;
  c.target_sr = target_sr; c.n_rec = S * n_rec; c.rec_n = rs_n.data(); c.rec_sr = rs_sr.data();
  rc = plan_call(e, c);
  if (!rc) rc = enqueue_call(e, cuda_stream, c);
  split_rows(S, rows, nseg.data(), status.data(), n_segments_out, status_out, ref_n_segments_out, ref_status_out);
  return rc;
}

int nisqa_predict_device_windows(nisqa_engine* e, void* cuda_stream, const nisqa_device_batch* rec, int32_t target_sr,
                                 int64_t window, int32_t hop_frames, float* scores_dev, int64_t n_rows,
                                 int32_t* n_segments_out, int32_t* status_out) {
  if (!e) return NISQA_ERR_INVALID;
  if (!e->stream) return fail(e, NISQA_ERR_STATE, "engine was not created successfully");
  if (e->cfg.double_ended)
    return fail(e, NISQA_ERR_INVALID, "a double-ended (NISQA_DE) engine scores (degraded, reference) pairs, not windows of a recording");
  if (!rec) return fail(e, NISQA_ERR_INVALID, "rec: null argument");
  return windows_call(e, cuda_stream, "rec", rec, nullptr, target_sr, window, hop_frames, 0, scores_dev, n_rows, n_segments_out,
                      status_out, nullptr, nullptr);
}

int nisqa_predict_device_window_pairs(nisqa_engine* e, void* cuda_stream, const nisqa_device_batch* deg,
                                      const nisqa_device_batch* ref, int32_t target_sr, int64_t window, int32_t hop_frames,
                                      int32_t margin_frames, float* scores_dev, int64_t n_rows, int32_t* n_segments_out,
                                      int32_t* status_out, int32_t* ref_n_segments_out, int32_t* ref_status_out) {
  if (!e) return NISQA_ERR_INVALID;
  if (!e->stream) return fail(e, NISQA_ERR_STATE, "engine was not created successfully");
  if (!e->cfg.double_ended)
    return fail(e, NISQA_ERR_INVALID, "ref: only a double-ended (NISQA_DE) engine scores window pairs");
  if (!deg) return fail(e, NISQA_ERR_INVALID, "deg: null argument");
  if (!ref) return fail(e, NISQA_ERR_INVALID, "ref: null argument");
  return windows_call(e, cuda_stream, "deg", deg, ref, target_sr, window, hop_frames, margin_frames, scores_dev, n_rows,
                      n_segments_out, status_out, ref_n_segments_out, ref_status_out);
}

int nisqa_predict_device_window_pairs_alignment(nisqa_engine* e, void* cuda_stream, const nisqa_device_batch* deg,
                                                const nisqa_device_batch* ref, int32_t target_sr, int64_t window,
                                                int32_t hop_frames, int32_t margin_frames, float* scores_dev, int64_t n_rows,
                                                const nisqa_alignment_out* al, int32_t* n_segments_out, int32_t* status_out,
                                                int32_t* ref_n_segments_out, int32_t* ref_status_out) {
  if (e && !e->stream) return fail(e, NISQA_ERR_STATE, "engine was not created successfully");
  const int rc = check_alignment_out(e, al);
  if (rc) return rc;
  if (!deg) return fail(e, NISQA_ERR_INVALID, "deg: null argument");
  if (!ref) return fail(e, NISQA_ERR_INVALID, "ref: null argument");
  return windows_call(e, cuda_stream, "deg", deg, ref, target_sr, window, hop_frames, margin_frames, scores_dev, n_rows,
                      n_segments_out, status_out, ref_n_segments_out, ref_status_out, al);
}

// nisqa_window_counts (n_src 1, margin_frames 0) and nisqa_window_pair_counts (n_src 2)
static int window_counts(const nisqa_config* cfg, int n_src, int64_t n_samples, int64_t ref_n_samples, int32_t sample_rate,
                         int64_t window, int32_t hop_frames, int32_t margin_frames, int64_t* n_windows, int32_t* n_segments,
                         int32_t* status, int32_t* ref_n_segments, int32_t* ref_status, int64_t cap) {
  if (!cfg || n_samples < 1 || (n_src == 2 && ref_n_samples < 1)) return NISQA_ERR_INVALID;
  std::string why;
  int H = 0;
  int64_t M = 0;
  if (!window_pair_geometry(*cfg, sample_rate, window, hop_frames, margin_frames, &H, &M, &why)) return NISQA_ERR_INVALID;
  const int64_t K = window_count(n_samples, window, H);
  if (n_windows) *n_windows = K;
  WinList w;
  for (int64_t k = 0; k < std::min(K, cap); ++k) add_window(&w, n_src, 0, k, n_samples, ref_n_samples, window, H, M);
  plan_rows(*cfg, sample_rate, n_src, w, n_segments, status, ref_n_segments, ref_status);
  return 0;
}

int nisqa_window_counts(const nisqa_config* cfg, int64_t n_samples, int32_t sample_rate, int64_t window, int32_t hop_frames,
                        int64_t* n_windows, int32_t* n_segments, int32_t* status, int64_t cap) {
  return window_counts(cfg, 1, n_samples, 0, sample_rate, window, hop_frames, 0, n_windows, n_segments, status, nullptr,
                       nullptr, cap);
}

int nisqa_window_pair_counts(const nisqa_config* cfg, int64_t n_samples, int64_t ref_n_samples, int32_t sample_rate,
                             int64_t window, int32_t hop_frames, int32_t margin_frames, int64_t* n_windows,
                             int32_t* n_segments, int32_t* status, int32_t* ref_n_segments, int32_t* ref_status, int64_t cap) {
  return window_counts(cfg, 2, n_samples, ref_n_samples, sample_rate, window, hop_frames, margin_frames, n_windows, n_segments,
                       status, ref_n_segments, ref_status, cap);
}

// ---- live feeds
// nisqa_feed_rows (n_src 1, margin_frames 0) and nisqa_feed_pair_rows (n_src 2)
static int feed_rows(const nisqa_config* cfg, int n_src, int32_t sample_rate, int64_t window, int32_t hop_frames,
                     int32_t margin_frames, int32_t n_feeds, const int64_t* held, const int64_t* ref_held,
                     const int64_t* n_samples, const int64_t* ref_n_samples, const uint8_t* end, int64_t* n_rows,
                     int32_t* feed, int64_t* index, int32_t* n_segments, int32_t* status, int32_t* ref_n_segments,
                     int32_t* ref_status, int64_t cap) {
  const bool pair = n_src == 2;
  if (!cfg || n_feeds < 0 || (n_feeds > 0 && (!held || !n_samples || (pair && (!ref_held || !ref_n_samples)))) || !n_rows)
    return NISQA_ERR_INVALID;
  std::string why;
  int H = 0;
  int64_t M = 0;
  if (!window_pair_geometry(*cfg, sample_rate, window, hop_frames, margin_frames, &H, &M, &why)) return NISQA_ERR_INVALID;
  for (int b = 0; b < n_feeds; ++b)
    if (held[b] < 0 || n_samples[b] < 0 || (pair && (ref_held[b] < 0 || ref_n_samples[b] < 0))) return NISQA_ERR_INVALID;
  int64_t r = 0;
  WinList w;
  feed_windows(n_feeds, window, H, M, held, n_samples, pair ? ref_held : nullptr, pair ? ref_n_samples : nullptr, end,
               [&](int b, int64_t k, int64_t T, int64_t T_ref) {
    if (r < cap) {
      if (feed) feed[r] = b;
      if (index) index[r] = k;
      add_window(&w, n_src, b, k, T, T_ref, window, H, M);
    }
    ++r;
  });
  *n_rows = r;
  plan_rows(*cfg, sample_rate, n_src, w, n_segments, status, ref_n_segments, ref_status);
  return 0;
}

int nisqa_feed_rows(const nisqa_config* cfg, int32_t sample_rate, int64_t window, int32_t hop_frames, int32_t n_feeds,
                    const int64_t* held, const int64_t* n_samples, const uint8_t* end, int64_t* n_rows, int32_t* feed,
                    int64_t* index, int32_t* n_segments, int32_t* status, int64_t cap) {
  return feed_rows(cfg, 1, sample_rate, window, hop_frames, 0, n_feeds, held, nullptr, n_samples, nullptr, end, n_rows, feed,
                   index, n_segments, status, nullptr, nullptr, cap);
}

int nisqa_feed_pair_rows(const nisqa_config* cfg, int32_t sample_rate, int64_t window, int32_t hop_frames,
                         int32_t margin_frames, int32_t n_feeds, const int64_t* held, const int64_t* ref_held,
                         const int64_t* n_samples, const int64_t* ref_n_samples, const uint8_t* end, int64_t* n_rows,
                         int32_t* feed, int64_t* index, int32_t* n_segments, int32_t* status, int32_t* ref_n_segments,
                         int32_t* ref_status, int64_t cap) {
  return feed_rows(cfg, 2, sample_rate, window, hop_frames, margin_frames, n_feeds, held, ref_held, n_samples, ref_n_samples,
                   end, n_rows, feed, index, n_segments, status, ref_n_segments, ref_status, cap);
}

// nisqa_feed_create (n_src 1: margin_frames = max_skew = 0) and nisqa_feed_pair_create (n_src 2)
static int feed_create(nisqa_engine* e, nisqa_feed** out, int32_t n_feeds, int32_t sample_rate, int64_t window,
                       int32_t hop_frames, int32_t margin_frames, int64_t max_push, int64_t max_skew, int n_src) {
  if (!e) return NISQA_ERR_INVALID;
  if (!out) return fail(e, NISQA_ERR_INVALID, "out: null argument");
  *out = nullptr;
  if (!e->stream) return fail(e, NISQA_ERR_STATE, "engine was not created successfully");
  if (n_src == 1 && e->cfg.double_ended)
    return fail(e, NISQA_ERR_INVALID, "a double-ended (NISQA_DE) engine scores (degraded, reference) pairs, not live feeds: "
                                      "nisqa_feed_pair_create scores live pairs");
  if (n_src == 2 && !e->cfg.double_ended)
    return fail(e, NISQA_ERR_INVALID, "nisqa_feed_pair_create: only a double-ended (NISQA_DE) engine scores live pairs; "
                                      "nisqa_feed_create scores live feeds");
  if (n_feeds < 1 || n_feeds > 65535)
    return fail(e, NISQA_ERR_INVALID, "n_feeds = " + std::to_string(n_feeds) + ": not within 1 .. 65535");
  if (sample_rate <= 0) return fail(e, NISQA_ERR_INVALID, "sample_rate = " + std::to_string(sample_rate));
  std::string why;
  int H = 0;
  int64_t M = 0;
  if (!window_pair_geometry(e->cfg, sample_rate, window, hop_frames, margin_frames, &H, &M, &why))
    return fail(e, NISQA_ERR_INVALID, why);
  if (max_push < 1 || max_push > (int64_t)INT32_MAX - 2 * window)
    return fail(e, NISQA_ERR_INVALID, "max_push = " + std::to_string(max_push) + ": not within 1 .. 2^31 - 1 - 2 window samples");
  // The ring of each source must keep every sample that a pair emitted by a push reads while that push appends its
  // samples: no position may alias modulo R.  With E_old = min(cd(Td_old), cr(Tr_old)) the first pair a push emits
  // (cd(T) = T >= W ? (T - W) / H + 1 : 0, cr(T) = T >= W + M ? (T - W - M) / H + 1 : 0, so cd(T) H >= T - W + 1 and
  // cr(T) H >= T - W - M + 1), the push reads degraded samples from E_old H and reference samples from max(0, E_old H -
  // M), and writes up to Td_old + max_push - 1 and Tr_old + max_push - 1, where |Td_old - Tr_old| <= max_skew (the bound
  // held after the last push):
  //   degraded:  Td_new - E_old H <= W + max_push - 1 (E_old = cd) or W + M + max_push + max_skew - 1 (E_old = cr)
  //              -> R_d = W + max_push + M + max_skew
  //   reference: Tr_new - E_old H + M <= W + 2M + max_push - 1 (E_old = cr) or W + M + max_push + max_skew - 1 (E_old = cd)
  //              -> R_r = W + max_push + M + max(M, max_skew)
  // (a single-ended feed: M = max_skew = 0, R = W + max_push).  The mirror of a source is its window length (reference:
  // W + 2M), so that any of its windows is contiguous.  The frame-pair ring of a source covers the frames of R samples,
  // which bound those a push writes and the pairs its emitted windows read alike.
  if (max_skew < 0 || window + max_push + M + std::max(M, max_skew) > (int64_t)INT32_MAX)
    return fail(e, NISQA_ERR_INVALID, "max_skew = " + std::to_string(max_skew) + ": not within 0 .. 2^31 - 1 - window - "
                                          "max_push - margin samples (with a margin, the reference ring must fit 2^31 - 1)");
  CK(cudaSetDevice(e->device));
  ClipPlan pl;
  plan_clip(e->cfg, window, sample_rate, &pl);
  int fb_id = -1;
  int rc = build_fb(e, sample_rate, pl.hop, pl.win, &fb_id);
  if (rc) return rc;
  std::unique_ptr<nisqa_feed> f(new nisqa_feed());
  f->e = e;
  f->n_feeds = n_feeds; f->rate = sample_rate; f->n_src = n_src;
  f->max_push = max_push; f->max_skew = max_skew;
  long long ring_elems = 0;
  size_t frame_floats = 0;
  for (int s = 0; s < n_src; ++s) {
    const int64_t m = s ? M : 0;
    FeedGeom& g = f->g[s];
    g = {};
    g.W = (int)(window + 2 * m); g.H = H; g.hf = hop_frames;
    g.R = (int)(window + max_push + M + (s ? std::max(M, max_skew) : max_skew));
    g.stride = ((long long)g.R + g.W + 15) / 16 * 16;
    g.hop = pl.hop; g.win = pl.win; g.s0 = (e->cfg.n_fft - pl.win) / 2 - e->cfg.n_fft / 2;
    g.ncls = (hop_frames & 1) ? 2 : 1;
    const int frames_live = g.R / pl.hop + 2;             // frames whose pairs one push may touch
    g.P = g.ncls == 2 ? frames_live : frames_live / 2 + 2;
    g.fb_id = fb_id;
    g.off = (int)m; g.par = (int)((m / pl.hop) & 1);
    f->held[s].assign(n_feeds, 0);
    f->j_next[s].assign(n_feeds, 0);
    f->ring_at[s] = ring_elems;
    ring_elems += (long long)n_feeds * g.stride;
    f->frames_at[s] = frame_floats;
    frame_floats += (size_t)n_feeds * g.P * 2 * e->cfg.n_mels;
  }
  const size_t ring_bytes = (size_t)ring_elems * 4;                     // (int16 rings use half)
  const size_t frame_bytes = frame_floats * 4;
  CK(cudaMalloc(&f->ring, ring_bytes));
  f->ring_bytes = ring_bytes;
  CK(cudaMalloc(&f->frames, frame_bytes));
  f->frame_bytes = frame_bytes;
  CK(cudaMemset(f->ring, 0, ring_bytes));
  CK(cudaMemset(f->frames, 0, frame_bytes));
  CK(cudaEventCreateWithFlags(&f->ready, cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&f->done, cudaEventDisableTiming));
  for (auto& sl : f->slots) CK(cudaEventCreateWithFlags(&sl.copied, cudaEventDisableTiming));
  *out = f.release();
  return 0;
}

int nisqa_feed_create(nisqa_engine* e, nisqa_feed** out, int32_t n_feeds, int32_t sample_rate, int64_t window,
                      int32_t hop_frames, int64_t max_push) {
  return feed_create(e, out, n_feeds, sample_rate, window, hop_frames, 0, max_push, 0, 1);
}

int nisqa_feed_pair_create(nisqa_engine* e, nisqa_feed** out, int32_t n_feeds, int32_t sample_rate, int64_t window,
                           int32_t hop_frames, int32_t margin_frames, int64_t max_push, int64_t max_skew) {
  return feed_create(e, out, n_feeds, sample_rate, window, hop_frames, margin_frames, max_push, max_skew, 2);
}

int64_t nisqa_feed_device_bytes(const nisqa_feed* f) {
  if (!f) return NISQA_ERR_INVALID;
  int64_t n = (int64_t)(f->ring_bytes + f->frame_bytes);
  for (const auto& sl : f->slots) n += (int64_t)sl.d.cap;
  return n;
}

// nisqa_feed_push (ref == nullptr) and nisqa_feed_pair_push: the chunk of each source appended to its rings, the
// interior pairs whose last tap it brings computed into its frame rings, then the windows (pairs) the push completes
// scored as the clips of a call that reads the rings
static int feed_push(nisqa_feed* f, void* cuda_stream, const nisqa_device_batch* deg, const nisqa_device_batch* ref,
                     const uint8_t* end, float* scores_dev, int64_t n_rows, int32_t* feed_out, int64_t* index_out,
                     int32_t* n_segments_out, int32_t* status_out, int32_t* ref_n_segments_out, int32_t* ref_status_out) {
  nisqa_engine* e = f->e;
  if (!e->weights_loaded) return fail(e, NISQA_ERR_STATE, "nisqa_load_weights has not been called");
  const int S = f->n_src, B = f->n_feeds;
  const nisqa_device_batch* src[2] = {deg, ref};
  const std::string nm[2] = {S == 2 ? "deg" : "chunk", "ref"};
  for (int s = 0; s < S; ++s) {
    const nisqa_device_batch* c = src[s];
    if (!c) return fail(e, NISQA_ERR_INVALID, nm[s] + ": null argument");
    if (c->n_clips != B)
      return fail(e, NISQA_ERR_INVALID, nm[s] + ".n_clips = " + std::to_string(c->n_clips) + ": the feed object has " +
                                            std::to_string(B) + " feeds");
    if (c->sample_rate != f->rate)
      return fail(e, NISQA_ERR_INVALID, nm[s] + ".sample_rate = " + std::to_string(c->sample_rate) + ": the feeds run at " +
                                            std::to_string(f->rate) + " Hz");
  }
  IngestSources ing;
  int fmt;
  int rc = check_sources(e, nm[0] + ".", *deg, ref, B, 0, &ing, &fmt);
  if (rc) return rc;
  long long max_in[2] = {0, 0};
  bool holds = false;
  for (int s = 0; s < S; ++s)
    for (int b = 0; b < B; ++b) {
      const int64_t n = src[s]->n_samples[b];
      if (n > f->max_push)
        return fail(e, NISQA_ERR_INVALID, nm[s] + ".n_samples[" + std::to_string(b) + "] = " + std::to_string(n) +
                                              ": more than max_push (" + std::to_string(f->max_push) + " samples)");
      max_in[s] = std::max<long long>(max_in[s], n);
      holds = holds || f->held[s][b] > 0;
    }
  if (S == 2)       // (the rings hold the faster side's backlog: measured before an end resets the feed)
    for (int b = 0; b < B; ++b) {
      const int64_t Td = f->held[0][b] + deg->n_samples[b], Tr = f->held[1][b] + ref->n_samples[b];
      if ((Td > Tr ? Td - Tr : Tr - Td) > f->max_skew)
        return fail(e, NISQA_ERR_INVALID, "deg.n_samples[" + std::to_string(b) + "] / ref.n_samples[" + std::to_string(b) +
                                              "]: feed " + std::to_string(b) + " would hold " + std::to_string(Td) +
                                              " degraded and " + std::to_string(Tr) + " reference samples, more than "
                                              "max_skew (" + std::to_string(f->max_skew) + " samples) apart");
    }
  // one format for both sources (as nisqa_predict_device_window_pairs)
  if (std::max(max_in[0], max_in[1]) > 0 && holds && f->fmt != fmt)
    return fail(e, NISQA_ERR_INVALID, (S == 2 ? std::string("deg.sample_fmt / ref.sample_fmt") : std::string("chunk.sample_fmt")) +
                                          ": the feeds hold " + (f->fmt == NISQA_FMT_F32 ? "float32" : "int16") +
                                          " samples and this push " +
                                          (fmt == NISQA_FMT_F32 ? "float32 (or mixed) ones" : "mono int16 ones") +
                                          "; a format holds until every feed has ended");
  // the windows (pairs: clips 2p and 2p + 1) the push completes (host arithmetic: nisqa_feed_rows, nisqa_feed_pair_rows)
  const FeedGeom& g = f->g[0];
  const int64_t M = S == 2 ? f->g[1].off : 0;
  WinList wl;
  std::vector<int64_t> widx;
  feed_windows(B, g.W, g.H, M, f->held[0].data(), deg->n_samples, S == 2 ? f->held[1].data() : nullptr,
               S == 2 ? ref->n_samples : nullptr, end, [&](int b, int64_t k, int64_t T, int64_t T_ref) {
    widx.push_back(k);
    add_window(&wl, S, b, k, T, T_ref, g.W, g.H, M);
  });
  const int N = (int)wl.rec.size(), rows = N / S;
  if (n_rows < rows)
    return fail(e, NISQA_ERR_INVALID, "n_rows = " + std::to_string(n_rows) + ": the push completes " + std::to_string(rows) +
                                          (S == 2 ? " window pairs" : " windows"));
  if (N > 0 && !scores_dev) return fail(e, NISQA_ERR_INVALID, "scores_dev: null argument");
  // the completed windows, each a clip of a pass that reads the rings
  FeedRings rings = {};
  for (int s = 0; s < 2; ++s) {
    const int u = s < S ? s : 0;        // (single-ended: both entries are the one source)
    rings.g[s] = f->g[u]; rings.ring_at[s] = f->ring_at[u]; rings.frames[s] = f->frames + f->frames_at[u];
  }
  WinLayout L = {wl.rec.data(), wl.start.data(), nullptr, g.H, g.hf, g.W, &rings};
  L.n_src = S;
  std::vector<int32_t> srs(N, f->rate), nseg(N), status(N);
  Call c(N, wl.len.data(), srs.data(), fmt, nseg.data(), status.data());
  c.dev_pcm = f->ring; c.scores_dev = scores_dev; c.win = &L;
  rc = plan_call(e, c);
  if (rc) return rc;

  // each source's new samples and the interior pairs whose last tap they bring
  auto& sl = f->slots[f->n_push % kFeedSlots];
  if (sl.busy) { CK(cudaEventSynchronize(sl.copied)); sl.busy = false; }
  CK(sl.h.reserve((size_t)S * B * sizeof(FeedPush)));
  FeedPush* tab = sl.h.as<FeedPush>();
  int max_pairs[2] = {0, 0};
  for (int s = 0; s < S; ++s) {
    const FeedGeom& gs = f->g[s];
    const int step = 3 - gs.ncls, ext = gs.hop + gs.win;
    const long long j_min = (-gs.s0 + gs.hop - 1) / gs.hop;     // the first frame whose taps start at or after sample 0
    for (int b = 0; b < B; ++b) {
      const long long t1 = f->held[s][b] + src[s]->n_samples[b], num = t1 - ext - gs.s0;
      const long long j_end = num < 0 ? 0 : num / gs.hop + 1;     // frames whose pair's taps have all arrived
      long long j0 = std::max<long long>(f->j_next[s][b], j_min);
      if ((j0 - gs.par) % step) ++j0;                              // (ncls 1: the windows' pairing parity)
      const long long np = j_end > j0 ? (j_end - j0 + step - 1) / step : 0;
      tab[s * B + b] = {f->held[s][b], j0, (int)src[s]->n_samples[b], (int)np};
      max_pairs[s] = std::max(max_pairs[s], (int)np);
      f->j_next[s][b] = std::max<long long>(f->j_next[s][b], j_end);
    }
  }
  rc = enqueue_call(e, cuda_stream, c, f, [&](cudaStream_t st) -> int {
    if (f->pending) CK(cudaStreamWaitEvent(st, f->done, 0));  // push order: the last push's passes are done with the rings
    if (std::max(max_in[0], max_in[1]) > 0) {
      CK(sl.d.reserve((size_t)S * B * sizeof(FeedPush)));
      CK(cudaMemcpyAsync(sl.d.p, tab, (size_t)S * B * sizeof(FeedPush), cudaMemcpyHostToDevice, st));
      CK(cudaEventRecord(sl.copied, st));
      sl.busy = true;
      ++f->n_push;
      e->cur_stream = st;
      const size_t esz = fmt == NISQA_FMT_F32 ? 4 : 2;
      for (int s = 0; s < S; ++s) {
        void* ring = static_cast<char*>(f->ring) + f->ring_at[s] * esz;
        const FeedPush* push = sl.d.as<FeedPush>() + s * B;
        if (max_in[s] > 0) {
          Scope sc(e, "ingest");
          launch_ingest_feed(st, ing.s[s], push, B, max_in[s], f->g[s], fmt == NISQA_FMT_F32, ring);
        }
        if (max_pairs[s] > 0) {
          Scope sc(e, "frontend");
          launch_frontend_feed_pairs(st, e->cfg.n_mels, ring, fmt == NISQA_FMT_F32, push, B, max_pairs[s], f->g[s],
                                     e->fb_table.as<FbTables>(), e->tw4096.as<float2>(), f->frames + f->frames_at[s]);
        }
      }
      CK(cudaGetLastError());
      f->fmt = fmt;
    }
    for (int b = 0; b < B; ++b) {
      for (int s = 0; s < S; ++s) f->held[s][b] += src[s]->n_samples[b];
      if (end && end[b])
        for (int s = 0; s < S; ++s) { f->held[s][b] = 0; f->j_next[s][b] = 0; }
    }
    CK(cudaEventRecord(f->ready, st));
    c.fmt = f->fmt;                     // (the passes read the rings, in the format they hold)
    c.ready = f->ready;
    return 0;
  });
  if (rc) return rc;
  for (int r = 0; r < rows; ++r) {
    if (feed_out) feed_out[r] = wl.rec[S * r];
    if (index_out) index_out[r] = widx[r];
  }
  split_rows(S, rows, nseg.data(), status.data(), n_segments_out, status_out, ref_n_segments_out, ref_status_out);
  return 0;
}

int nisqa_feed_push(nisqa_feed* f, void* cuda_stream, const nisqa_device_batch* chunk, const uint8_t* end, float* scores_dev,
                    int64_t n_rows, int32_t* feed_out, int64_t* index_out, int32_t* n_segments_out, int32_t* status_out) {
  if (!f) return NISQA_ERR_INVALID;
  if (f->n_src == 2)
    return fail(f->e, NISQA_ERR_INVALID, "nisqa_feed_push: a pair feed object (nisqa_feed_pair_create) takes its pushes "
                                         "through nisqa_feed_pair_push");
  return feed_push(f, cuda_stream, chunk, nullptr, end, scores_dev, n_rows, feed_out, index_out, n_segments_out, status_out,
                   nullptr, nullptr);
}

int nisqa_feed_pair_push(nisqa_feed* f, void* cuda_stream, const nisqa_device_batch* deg, const nisqa_device_batch* ref,
                         const uint8_t* end, float* scores_dev, int64_t n_rows, int32_t* feed_out, int64_t* index_out,
                         int32_t* n_segments_out, int32_t* status_out, int32_t* ref_n_segments_out,
                         int32_t* ref_status_out) {
  if (!f) return NISQA_ERR_INVALID;
  if (f->n_src != 2)
    return fail(f->e, NISQA_ERR_INVALID, "nisqa_feed_pair_push: a single-ended feed object (nisqa_feed_create) takes its "
                                         "pushes through nisqa_feed_push");
  return feed_push(f, cuda_stream, deg, ref, end, scores_dev, n_rows, feed_out, index_out, n_segments_out, status_out,
                   ref_n_segments_out, ref_status_out);
}

void nisqa_feed_destroy(nisqa_feed* f) {
  if (!f) return;
  cudaSetDevice(f->e->device);
  if (f->pending) cudaEventSynchronize(f->done);
  for (auto& sl : f->slots)
    if (sl.busy) cudaEventSynchronize(sl.copied);
  delete f;
}

int64_t nisqa_stage_dump(nisqa_engine* e, int stage, float* out, int64_t cap) {
  if (!e) return NISQA_ERR_INVALID;
  if (e->last_passes != 1) return fail(e, NISQA_ERR_STATE, "stage dump needs a predict call that ran in one pass");
  cudaSetDevice(e->device);
  Lane& LN = e->lanes[e->last_lane];
  Stage& SG = e->stages[e->last_stage];
  const int std_mode = e->std_cnn();
  const int64_t ns = e->last_n_seg;
  if (!e->conv_net() && stage >= NISQA_STAGE_POOL1 && stage <= NISQA_STAGE_CNN_FEAT)
    return fail(e, NISQA_ERR_INVALID, "stage not available: this checkpoint has no convolutional framewise model");
  const bool conv_map = stage >= NISQA_STAGE_POOL1 && stage <= NISQA_STAGE_CONV5;
  const int layer = stage - NISQA_STAGE_POOL1 + 2;      // POOL1 .. CONV5: the map that feeds conv layer 2 .. 6
  int64_t count = 0;
  const float* src = nullptr;
  int hw = 0, ch = 0;    // NHWC -> NCHW conversion when ch > 0 (rows of hw_ld floats; 0: hw * ch)
  int hw_ld = 0;
  int width = 0, ld = 0; // rows of `width` floats at a stride of `ld` (a padded row layout)
  const int* cc = e->w.cnn_c;
  if (conv_map) {
    const ConvGeom g = split_geometry(std_mode, layer, cc[layer - 1], e->w.pools);
    src = LN.act[layer].as<float>(); hw = g.H * g.W; ch = g.C;
  }
  switch (stage) {
    case NISQA_STAGE_MEL_DB: count = (int64_t)e->last_n_frames * e->cfg.n_mels; break;
    case NISQA_STAGE_POOL1: case NISQA_STAGE_POOL2: case NISQA_STAGE_CONV3: case NISQA_STAGE_POOL3: case NISQA_STAGE_CONV5: break;
    case NISQA_STAGE_CNN_FEAT:
      if (std_mode && e->w.lstm_shipped) {
        src = LN.feats20.as<float>(); count = ns * 20;
      } else if (std_mode && e->w.std_fc > 0) {
        src = LN.feats20.as<float>(); width = e->w.std_fc; ld = round64(width); count = ns * width;
      } else if (std_mode) {
        src = LN.feats.as<float>(); hw = 12; ch = 64;           // [h*2+w][c] -> c*12+h*2+w
      } else {
        src = LN.feats.as<float>(); hw = e->w.pools.p[4]; ch = cc[6]; hw_ld = e->w.feat_ld();    // [h][c] -> c*h3+h
      }
      break;
    case NISQA_STAGE_TD_IN:
      if (!e->last_td_in) return fail(e, NISQA_ERR_INVALID, "stage not available for this architecture");
      src = e->last_td_in; count = ns * (e->td_sa() ? e->sa_d() : e->td2_d()); break;
    case NISQA_STAGE_TD1_OUT:
      if (!e->last_td1_out) return fail(e, NISQA_ERR_INVALID, "stage not available: no td_2 stage ran");
      src = e->last_td1_out; count = ns * e->last_td1_out_d; width = e->last_td1_out_d; ld = e->last_td1_out_ld; break;
    case NISQA_STAGE_DE_FUSED:
      if (!e->last_de_fused) return fail(e, NISQA_ERR_INVALID, "stage not available: only a double-ended model aligns and fuses");
      src = e->last_de_fused; count = ns * e->last_de_fused_d; break;
    case NISQA_STAGE_TD_OUT:
      if (!e->last_td_out) return fail(e, NISQA_ERR_STATE, "the per-step BiLSTM outputs were not kept: nisqa_set_option(\"keep_td_out\", 1) before the predict call");
      src = e->last_td_out; count = ns * e->last_td_out_d; width = e->last_td_out_d; ld = e->last_td_out_ld;
      if (e->last_td_out_hw) { hw = e->last_td_out_hw; ch = cc[6]; hw_ld = ld; }   // conv6 features: [hw][c] -> c*hw + hw index
      break;
    default: return fail(e, NISQA_ERR_INVALID, "unknown stage");
  }
  if (ch > 0) count = ns * hw * ch;
  if (!out) return count;
  const bool from_planes = conv_map && e->last_split;     // the map lives in the plane pair planes[layer]
  if (from_planes && stage == NISQA_STAGE_POOL1 && e->last_conv12)
    return fail(e, NISQA_ERR_STATE, "pool1 lives only in shared memory on the fused conv1+conv2 path: nisqa_set_option(\"conv12\", 0) before the predict call");
  if (cap < count) return fail(e, NISQA_ERR_INVALID, "stage dump buffer too small");
  if (count == 0) return 0;
  cudaStream_t st = LN.stream;
  if (stage == NISQA_STAGE_MEL_DB) {
    CK(e->dump.reserve((size_t)count * 4));
    launch_mel_dump(st, LN.mel.as<float>(), SG.clips.as<ClipDesc>(), (int)e->last_clips.size(),
                    SG.clipmax.as<unsigned>(), e->cfg.n_mels, e->dump.as<float>());
    src = e->dump.as<float>();
  } else if (ch > 0) {
    if (from_planes) {
      CK(LN.act[layer].reserve((size_t)count * 4));
      launch_unsplit(st, std_mode, layer, ch, LN.planes[layer].as<char>(), LN.planes[layer].as<char>() + LN.plane_bytes[layer],
                     e->w.conv[layer - 1].unit, LN.act[layer].as<float>(), (int)ns, e->w.pools);
      src = LN.act[layer].as<float>();
    }
    CK(e->dump.reserve((size_t)count * 4));
    launch_nhwc_to_nchw(st, src, hw_ld ? hw_ld : hw * ch, e->dump.as<float>(), ns, hw, ch);
    src = e->dump.as<float>();
    ld = 0;                                               // (the converted rows are contiguous)
  }
  if (!src) return fail(e, NISQA_ERR_STATE, "stage was not produced");
  if (ld > width)
    CK(cudaMemcpy2DAsync(out, (size_t)width * 4, src, (size_t)ld * 4, (size_t)width * 4, (size_t)ns, cudaMemcpyDeviceToHost, st));
  else
    CK(cudaMemcpyAsync(out, src, (size_t)count * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return count;
}

int nisqa_segment_counts(const nisqa_config* cfg, int64_t n_samples, int32_t sample_rate,
                         int32_t* n_frames, int32_t* n_segments, int32_t* status) {
  if (!cfg) return NISQA_ERR_INVALID;
  ClipPlan p;
  plan_clip(*cfg, n_samples, sample_rate, &p);
  if (n_frames) *n_frames = p.n_frames;
  if (n_segments) *n_segments = p.n_seg;
  if (status) *status = p.status;
  return 0;
}

int nisqa_mel_filterbank(nisqa_engine* e, int32_t sample_rate, float* out, int64_t cap) {
  if (!e || !out) return NISQA_ERR_INVALID;
  if (!e->stream) return fail(e, NISQA_ERR_STATE, "engine was not created successfully");
  CK(cudaSetDevice(e->device));
  const int hop = (int)((double)sample_rate * e->cfg.hop_s), win = (int)((double)sample_rate * e->cfg.win_s);
  if (hop < 1 || win < 1 || win > e->cfg.n_fft) return fail(e, NISQA_ERR_INVALID, "unsupported sample rate");
  int id = -1;
  int rc = build_fb(e, sample_rate, hop, win, &id);
  if (rc) return rc;
  const std::vector<float>& d = e->fbs[id]->dense;
  if (cap < (int64_t)d.size()) return fail(e, NISQA_ERR_INVALID, "buffer too small");
  memcpy(out, d.data(), d.size() * 4);
  return 0;
}

int64_t nisqa_kernel_launches(const nisqa_engine* e) { return e ? e->launches : 0; }
void* nisqa_stream(const nisqa_engine* e) { return e ? (void*)e->stream : nullptr; }

int nisqa_join(nisqa_engine* e) {
  if (!e || !e->stream) return NISQA_ERR_INVALID;
  CK(cudaSetDevice(e->device));
  for (auto& g : e->stages)
    if (g.busy && g.lane != 0) CK(cudaStreamWaitEvent(e->stream, g.ev_done, 0));
  return 0;
}

int nisqa_set_option(nisqa_engine* e, const char* name, int value) {
  if (!e || !name) return NISQA_ERR_INVALID;
  if (strcmp(name, "conv_tc") == 0) { e->conv_tc = value != 0; return 0; }
  if (strcmp(name, "fe_ppc") == 0) { e->fe_ppc = value; return 0; }
  if (strcmp(name, "lstm_batched") == 0) { e->lstm_batched = value != 0; return 0; }
  if (strcmp(name, "keep_td_out") == 0) { e->keep_td_out = value != 0; return 0; }
  if (strcmp(name, "conv12") == 0) { e->conv12 = value != 0; return 0; }
  return fail(e, NISQA_ERR_INVALID, std::string("unknown option ") + name);
}

int nisqa_set_cnn_pools(nisqa_engine* e, const int32_t pools[6]) {
  if (!e || !pools) return NISQA_ERR_INVALID;
  static const char* const names[3] = {"cnn_pool_1", "cnn_pool_2", "cnn_pool_3"};
  CnnPools q;
  for (int i = 0; i < 3; ++i) {
    const int h = pools[2 * i], w = pools[2 * i + 1];
    const std::string v = std::string(names[i]) + "=[" + std::to_string(h) + ", " + std::to_string(w) + "]: ";
    if (h < 1 || w < 1 || w > kMaxPoolW || (h + 1) * (w + 1) > kMaxPoolCells)
      return fail(e, NISQA_ERR_INVALID, v + "the engine runs AdaptCNN pool sizes [h, w] with w <= " + std::to_string(kMaxPoolW) +
                                            " and (h + 1) * (w + 1) <= " + std::to_string(kMaxPoolCells));
    if (i == 2 && w > kMaxPool3W)
      return fail(e, NISQA_ERR_INVALID, v + "the engine runs pool_3 widths 1 to 3 (conv6's kernel is 3 x pool_3[1])");
    q.p[2 * i] = h; q.p[2 * i + 1] = w;
  }
  if (q != kShippedPools && !(e->conv_net() && !e->std_cnn()))
    return fail(e, NISQA_ERR_INVALID, "cnn_pool_1/2/3: only AdaptCNN takes other pool sizes");
  e->pools_next = q;
  return 0;
}

int nisqa_set_profiling(nisqa_engine* e, int on) {
  if (!e) return NISQA_ERR_INVALID;
  e->profiling = on != 0;
  return 0;
}

double nisqa_group_ms(const nisqa_engine* e, const char* group) {
  if (!e || !group) return -1.0;
  const std::string g(group);
  double total = 0.0; bool found = false;
  for (const auto& t : e->timers) {
    const bool cnn = t.name.compare(0, 4, "conv") == 0;
    const bool td = t.name == "lin_ln" || t.name == "qkv" || t.name == "sa_layer" || t.name == "fc_out" || t.name == "lstm";
    const bool match = t.name == g || (g == "cnn" && cnn) || (g == "td" && td) ||
                       (g == "frontend" && t.name == "seg_table");
    if (match) { total += t.ms; found = true; }
  }
  return found ? total : -1.0;
}

}  // extern "C"

// ------------------------------------------------------------------ NCCL (resolved at run time)
// The single exchange step of the multi-GPU path.  libnccl is bound with dlopen/dlsym so that
// the library has no link-time NCCL dependency (the torch-bundled libnccl.so.2 that is already
// in the process is reused when present).
struct NcclId { char internal[128]; };   // ncclUniqueId (passed by value to ncclCommInitRank)
namespace {
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, NcclId, int) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
NcclApi* nccl_api(std::string* why) {
  static NcclApi api;
  static bool tried = false;
  if (!tried) {
    tried = true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) { api.lib = dlopen(nm, RTLD_NOW | RTLD_NOLOAD); if (api.lib) break; }
    if (!api.lib) for (const char* nm : names) { api.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL); if (api.lib) break; }
    if (api.lib) {
      api.GetUniqueId = (int (*)(void*))dlsym(api.lib, "ncclGetUniqueId");
      api.CommInitRank = (int (*)(void**, int, NcclId, int))dlsym(api.lib, "ncclCommInitRank");
      api.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(api.lib, "ncclAllGather");
      api.CommDestroy = (int (*)(void*))dlsym(api.lib, "ncclCommDestroy");
      api.GetErrorString = (const char* (*)(int))dlsym(api.lib, "ncclGetErrorString");
    }
  }
  if (!api.lib || !api.GetUniqueId || !api.CommInitRank || !api.AllGather) {
    if (why) *why = "libnccl.so.2 could not be loaded (dlopen/dlsym)";
    return nullptr;
  }
  return &api;
}
}  // namespace

namespace {
int lane_allgather(nisqa_engine* e, const float* src, float* dst, size_t count, cudaStream_t st) {
  std::string why;
  NcclApi* a = nccl_api(&why);
  if (!a) return fail(e, NISQA_ERR_NCCL, why);
  int rc = a->AllGather(src, dst, count, /*ncclFloat32*/ 7, e->nccl_comm, st);
  if (rc) return fail(e, NISQA_ERR_NCCL, std::string("ncclAllGather: ") + (a->GetErrorString ? a->GetErrorString(rc) : "error"));
  e->launches += 1;
  return 0;
}
}  // namespace

extern "C" {

int nisqa_set_gather_target(nisqa_engine* e, float* global_dev, int rows) {
  if (!e || rows < 0) return NISQA_ERR_INVALID;
  e->gather_dst = global_dev; e->gather_rows = global_dev ? rows : 0;
  return 0;
}

int nisqa_nccl_unique_id(nisqa_engine* e, void* id128) {
  if (!e || !id128) return NISQA_ERR_INVALID;
  std::string why;
  NcclApi* a = nccl_api(&why);
  if (!a) return fail(e, NISQA_ERR_NCCL, why);
  int rc = a->GetUniqueId(id128);
  if (rc) return fail(e, NISQA_ERR_NCCL, std::string("ncclGetUniqueId: ") + (a->GetErrorString ? a->GetErrorString(rc) : "error"));
  return 0;
}

int nisqa_nccl_init(nisqa_engine* e, int world, int rank, const void* id128) {
  if (!e || !id128 || world < 1 || rank < 0 || rank >= world) return NISQA_ERR_INVALID;
  std::string why;
  NcclApi* a = nccl_api(&why);
  if (!a) return fail(e, NISQA_ERR_NCCL, why);
  CK(cudaSetDevice(e->device));
  NcclId id; memcpy(&id, id128, sizeof id);
  void* comm = nullptr;
  int rc = a->CommInitRank(&comm, world, id, rank);
  if (rc) return fail(e, NISQA_ERR_NCCL, std::string("ncclCommInitRank: ") + (a->GetErrorString ? a->GetErrorString(rc) : "error"));
  e->nccl_comm = comm; e->nccl_world = world; e->nccl_rank = rank;
  return 0;
}

int nisqa_gather_nccl(nisqa_engine* e, void* nccl_comm, const float* local_dev, int max_rows, float* global_dev) {
  if (!e || !local_dev || !global_dev || max_rows < 0) return NISQA_ERR_INVALID;
  std::string why;
  NcclApi* a = nccl_api(&why);
  if (!a) return fail(e, NISQA_ERR_NCCL, why);
  void* comm = nccl_comm ? nccl_comm : e->nccl_comm;
  if (!comm) return fail(e, NISQA_ERR_STATE, "no NCCL communicator: call nisqa_nccl_init or pass one");
  CK(cudaSetDevice(e->device));
  for (auto& g : e->stages)                 // the rows may have been produced on any lane
    if (g.busy && g.lane != 0) CK(cudaStreamWaitEvent(e->stream, g.ev_done, 0));
  const size_t count = (size_t)max_rows * e->cfg.n_out;
  int rc = a->AllGather(local_dev, global_dev, count, /*ncclFloat32*/ 7, comm, e->stream);
  if (rc) return fail(e, NISQA_ERR_NCCL, std::string("ncclAllGather: ") + (a->GetErrorString ? a->GetErrorString(rc) : "error"));
  e->launches += 1;
  CK(cudaStreamSynchronize(e->stream));
  return 0;
}

}  // extern "C"

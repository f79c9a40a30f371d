// launch.cuh - the boundary between the host runtime (engine.cu) and the kernel files: the parameter structs the
// kernels take by value and the host launchers each kernel file defines.  Every file that defines one of them
// includes this header, so a definition that drifts from its declaration is a compile or link error.
// Plain host C++ (resample.cpp includes it too): the device structs of common.cuh are only named here.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <vector>

namespace nisqa {

struct ClipDesc;
struct FbTables;
struct WinSpan;
struct FeedGeom;
struct FeedPush;
struct FeedWin;

// AdaptCNN's adaptive max-pool output sizes cnn_pool_1 / 2 / 3 as h1 w1 h2 w2 h3 w3 (lib:586-710), shipped 24 x 7, 12 x 5,
// 6 x 3.  The tensor-core kernels take any [h, w] with w <= kMaxPoolW and (h + 1) (w + 1) <= kMaxPoolCells (one
// segment's padded map in one 256-row GEMM tile, the tap halo w + 2 within kSplitLead), pool_3 widths 1..3 (conv6's
// 3 x w3 weight taps stay resident), and c3 h3 <= kMaxCnnFeatures framewise features.
struct CnnPools { int p[6]; };
constexpr CnnPools kShippedPools = {{24, 7, 12, 5, 6, 3}};
constexpr int kMaxPoolW = 14, kMaxPoolCells = 256, kMaxPool3W = 3, kMaxCnnFeatures = 4096;
inline bool operator==(const CnnPools& a, const CnnPools& b) {
  for (int i = 0; i < 6; ++i) if (a.p[i] != b.p[i]) return false;
  return true;
}
inline bool operator!=(const CnnPools& a, const CnnPools& b) { return !(a == b); }

// Geometry of one segment's activation map that feeds conv layer `layer` (2..6), i.e. the output of layer - 1:
// H rows, W columns, C channels.  AdaptCNN pools to cnn_pool_1 / 2 / 3 (adaptive max-pool; shipped widths 7 / 5 / 3),
// StandardCNN to 24 x 8, 12 x 4, 6 x 2 (MaxPool2d(2)).  C is the checkpoint's (conv layer - 1's output channels, read
// from its weights; StandardCNN: 16 / 32 / 64); C = 0 asks for StandardCNN's.  The fp16 plane pairs (conv_split.cu),
// the fp32 FFMA activations and the stage dumps all use it.
struct ConvGeom { int H, W, C; };
constexpr ConvGeom split_geometry(int std_mode, int layer, int C, const CnnPools& pools = kShippedPools) {
  return {std_mode ? (layer == 2 ? 24 : layer <= 4 ? 12 : 6) : pools.p[layer == 2 ? 0 : layer <= 4 ? 2 : 4],
          std_mode ? (layer == 2 ? 8 : layer <= 4 ? 4 : 2) : pools.p[layer == 2 ? 1 : layer <= 4 ? 3 : 5],
          C ? C : layer == 2 ? 16 : layer == 3 ? 32 : 64};
}
// true when AdaptCNN conv layer `layer` (2..6) reads the shipped input map and writes the shipped output map under `pools`:
// it runs the compile-time SpCfg instance (conv2: pool_1 and pool_2, conv3: pool_2, conv4: pool_2 and pool_3, conv5 and
// conv6: pool_3)
inline bool shipped_layer_geometry(int layer, const CnnPools& pools) {
  const int k0 = layer == 2 ? 0 : layer <= 4 ? 2 : 4, k1 = (layer == 2 || layer == 4) ? k0 + 2 : k0;
  for (int k = k0; k <= k1 + 1; ++k)
    if (pools.p[k] != kShippedPools.p[k]) return false;
  return true;
}
// true when the layer configuration C (cnn.cu ConvCfg, conv_split.cuh SpCfg) reads that geometry (StandardCNN: with its
// shipped input channels too; AdaptCNN's come from the weights)
template <class C>
constexpr bool input_is(int std_mode, int layer) {
  return split_geometry(std_mode, layer, C::CIN).H == C::H && split_geometry(std_mode, layer, C::CIN).W == C::W &&
         (!std_mode || split_geometry(std_mode, layer, 0).C == C::CIN);
}

// ---------------------------------------------------------------- parameter structs (device pointers)
// One post-norm encoder layer of a self-attention stack, weights k-major in 64-column chunks (td_tiled.cu)
struct SaLayerParams {
  const float* WoT; const float* bo; const float* W1T; const float* b1; const float* W2T;
  const float* b2; const float* ln1_g; const float* ln1_b; const float* ln2_g; const float* ln2_b;
};
// PoolAttFF (lib:1156-1183): the logits w2_h . relu(W1_h x + b1_h) + b2_h come out of td_sa_kernel's fused tail; x is D wide
struct PoolHeadParams {      // heads concatenated
  const float* W1T;   // [n_heads][D k][128 j]
  const float* b1;    // [n_heads][128]
  const float* w2;    // [n_heads][128]
  const float* b2;    // [n_heads]
  const float* w3;    // [n_heads][D]
  const float* b3;    // [n_heads]
};
// PoolAtt (a1, a1b: the attention logit) / PoolAvg / PoolMax / PoolLastStep: one Linear(D -> 1) per head (td.cu)
struct PoolSimpleParams { const float* a1; const float* a1b; const float* w3; const float* b3; };
struct LstmParams {
  const float* w_ih;   // [2][512][20]
  const float* w_hh;   // [2][512][128]
  const float* b;      // [2][512]   (bias_ih + bias_hh)
  const float* w_pool; // [256]
};
// One layer of a stacked LSTM of any accepted shape (td.cu lstm_layer_kernel): the input projection
// gx = x W_ih^T + b_ih + b_hh of every step and direction comes precomputed from the tile GEMM
struct LstmLayerParams {
  const float* gx;     // [n_seg][ldg]: direction d's gate rows at columns d 4H .. d 4H + 4H (PyTorch order i, f, g, o)
  int ldg;             // dirs 4H
  const float* w_hh;   // [dirs][4H][H]
  float* out;          // [n_seg][ldo]: direction d's hidden state at columns d H .. d H + H
  int ldo;
};
// learned weights of the alignment at td's fan_out W, rows padded to ld = 64 NC with zero rows / columns: AttLuong
// (wT [ld][ld] k-major, b [ld]) / AttBahdanau (wqyT [ld][256] k-major = Wq^T | Wy^T, bqy [256] = bq | by, v [128])
struct DeAlignParams { const float* wT; const float* b; const float* wqyT; const float* bqy; const float* v; float vb; };
// An alignment call's outputs (nisqa_alignment_out): degraded row i of clip c at row_off[c] + i; pbias is added to peak
// (launch_de_align sets it)
struct DeAlignOut { const long long* row_off; int* ref_seg; float* weight; float* centroid; float* peak; float pbias; };
struct ResampleClip {
  long long in_off;      // element offset of the clip in the raw input buffer (float32, or int16 scaled by 1/32768)
  long long out_off;     // element offset in the packed float32 output buffer
  long long time_off;    // first entry of the clip in the chunk-start time register table
  int n_in;              // input samples
  int n_out;             // resampy's int(n_in * ratio)
  int n_fix;             // librosa fix_length: ceil(n_in * ratio) (zero padded / trimmed)
  int copy;              // 1: sr_orig == sr_new, plain conversion / copy
  double ratio;          // sr_new / sr_orig
  int src_clip;          // device ingest: the clip's position in IngestSources order
};

// ---------------------------------------------------------------- frontend.cu
// mel: [frames][n_mels]; one kernel instance per band count, n_mels in {32, 40, 48, 64, 80, 96, 128} (frontend_supports_mels)
bool frontend_supports_mels(int n_mels);
void launch_frontend(cudaStream_t st, int n_mels, const void* pcm, int fmt_f32, const ClipDesc* clips, int n_clips, int max_pairs,
                     const FbTables* fbs, const float2* tw, float* mel, unsigned* clipmax, int Q, int max_span, int ppc);
// Windows of recordings (WinSpan rows; every window is also a ClipDesc row): the edge pairs of every window (grid
// edge_pairs x n_clips) and the interior pairs of every span once (grid span_pairs x n_spans * ncls; ncls 2 when the
// window hop is an odd number of frames), each stored into every window that holds it.  Rows bit-identical to
// launch_frontend over the windows as clips.
void launch_frontend_windows(cudaStream_t st, int n_mels, const void* pcm, int fmt_f32, const ClipDesc* clips, int n_clips,
                             int edge_pairs, const WinSpan* spans, int n_spans, int span_pairs, int ncls,
                             const FbTables* fbs, const float2* tw, float* mel, unsigned* clipmax, int Q, int max_span);
// Live feeds (FeedGeom): the interior frame pairs of a push of one source into its frame ring, once (grid max n_pairs x
// n_feeds), with the arithmetic the clip path picks for the feed's rate; then, in each pass, the interior rows of the
// pass's windows from their source's frame ring (g0 / frames0: degraded or single-ended, g1 / frames1: reference) into
// their mel rows, with each window's clip-max key (grid pair blocks x n_clips; the edge pairs, and every pair of a
// front-clipped reference window as a one-window span, come from launch_frontend_windows).  Rows bit-identical to
// launch_frontend over the windows as clips.
void launch_frontend_feed_pairs(cudaStream_t st, int n_mels, const void* ring, int fmt_f32, const FeedPush* push, int n_feeds,
                                int max_pairs, const FeedGeom& g, const FbTables* fbs, const float2* tw, float* frames);
constexpr int kFeedRowPairs = 32;    // interior pairs per CTA of the row copy
void launch_feed_rows(cudaStream_t st, int n_mels, const ClipDesc* clips, const FeedWin* wins, int n_clips, int max_interior,
                      const FeedGeom& g0, const FeedGeom& g1, const float* frames0, const float* frames1, float* mel,
                      unsigned* clipmax);
void launch_seg_table(cudaStream_t st, const ClipDesc* clips, int n_clips, const int* seg_prefix, const unsigned* clipmax,
                      int seg_hop, int n_seg, int* seg_frame0, float* seg_thr, int* seg_clip);
void launch_mel_dump(cudaStream_t st, const float* mel, const ClipDesc* clips, int n_clips, const unsigned* clipmax, int n_mels,
                     float* out);

// ---------------------------------------------------------------- cnn.cu (fp32 FFMA convolutions)
// conv1 + pool1 of segments of n_mels x seg_len mel cells (rows n_mels floats apart): AdaptCNN any accepted shape ->
// ph x pw (cnn_pool_1), StandardCNN 48 x 15 only -> 24 x 8.  c1 output channels: 16, 32 or 64 into the planes (out_hi),
// 16 into fp32 `out`.  The planes hold what w1, b1 give (the tensor-core path passes them with 2^-e_c folded into
// channel c).  false: no instance for the shape.
bool launch_conv1(cudaStream_t st, int std_mode, int c1, const float* mel, int n_mels, int seg_len, const int* seg_frame0,
                  const float* seg_thr, const float* w1, const float* b1, float* out, int n_seg, void* out_hi, void* out_lo,
                  int ph, int pw);
void launch_conv_layer(cudaStream_t st, int std_mode, int layer, const float* in, const float* w, const float* b, float* out,
                       int n_seg);
// rows of `ld` floats (>= hw * ch)
void launch_nhwc_to_nchw(cudaStream_t st, const float* in, int ld, float* out, long long n, int hw, int ch);

// ---------------------------------------------------------------- conv_split.cu (tensor-core convolutions on fp16 planes)
size_t split_plane_bytes(int std_mode, int layer, int C, int n_seg, const CnnPools& pools);
// AdaptCNN conv2..conv6 take cin, cout in {16, 32, 64} (the pairs cnn_c_out_1/2/3 reach) and any accepted pools;
// StandardCNN its shipped ones.  The fp32 features of conv6 go out in rows of (h3 cout + 63) / 64 * 64 floats (AdaptCNN),
// zero-padded, channel c times out_unit[c] (2^e_c: the activation scale folded into conv6's weights and bias).
bool conv_split_supported(int cin, int cout);
bool launch_conv_split(cudaStream_t st, int std_mode, int layer, int cin, int cout, const void* in_hi, const void* in_lo,
                       const void* wtc, const float* b, float out_scale, const float* out_unit, void* out_hi, void* out_lo,
                       float* out_f32, int n_seg, const CnnPools& pools);
// the fused conv1 + conv2 kernel: 48 x 15 segments, c1 = 16, c2 = 32 (AdaptCNN also 16)
bool conv12_supported(int std_mode, int c1, int c2);
void launch_conv12(cudaStream_t st, int std_mode, int c2, const float* mel, const int* seg_frame0, const float* seg_thr,
                   const float* w1, const float* b1, const void* wtc2, const float* bias2, float scale2, void* out_hi,
                   void* out_lo, int n_seg);
// planes -> fp32 channels-last, channel c times unit[c] (2^e_c)
void launch_unsplit(cudaStream_t st, int std_mode, int layer, int C, const void* hi, const void* lo, const float* unit,
                    float* out, int n_seg, const CnnPools& pools);

// ---------------------------------------------------------------- td.cu (fc_out, BiLSTM, pooling)
void launch_fc20(cudaStream_t st, const float* feats, const float* WT, const float* b, float* out, int n_rows);
void launch_lstm(cudaStream_t st, const float* feats20, const ClipDesc* clips, int n_clips, const LstmParams& P,
                 float* td_out, float* partial, float pool_bias, float* scores);
void launch_lstm_batched(cudaStream_t st, const float* feats20, const ClipDesc* clips, const int* order, int n_clips,
                         const LstmParams& P, float* td_out, float* partial, float pool_bias, float* scores);
// one layer of a stacked LSTM, H in {32, 64, 96, 128, 192, 256}, dirs 1 or 2 (H 192 / 256: clusters of H / 64 CTAs)
bool lstm_layer_supported(int H);
void launch_lstm_layer(cudaStream_t st, int H, int dirs, const ClipDesc* clips, const int* order, int n_clips,
                       const LstmLayerParams& P);
// PoolAttFF logits of rows whose hidden layer relu(W1 x + b1) is already computed: [n_rows][n_heads 128] -> [n_rows][n_heads]
void launch_att_logits(cudaStream_t st, const float* hid, const float* w2, const float* b2, int n_heads, int n_rows,
                       float* logits);
// x: rows of D features at a row stride of ldx floats
void launch_pool_final(cudaStream_t st, const float* x, int D, int ldx, const float* logits, const ClipDesc* clips, int n_clips,
                       const PoolHeadParams& P, int n_heads, int max_seg, float* scores);
void launch_pool_simple(cudaStream_t st, const float* x, int D, int ldx, const ClipDesc* clips, int n_clips, int mode,
                        const PoolSimpleParams& P, int n_heads, int max_seg, float* scores);
// Pooling over wide rows (td = 'skip': the framewise rows, D real columns at a stride of ldx, a multiple of 64), one CTA
// per (clip, column slab of kPoolWideSlab).  mode: enum nisqa_pool except PoolLastStepBi; P.w3 / P.b3: each head's score
// Linear [n_heads][D] (columns in the rows' order); logits [n_seg][n_heads]: PoolAttFF's, computed by the caller, or -
// PoolAtt - written here from P.a1 [n_heads][D] / P.a1b.  partial: [n_clips][pool_wide_slabs(D)][n_heads] floats.
constexpr int kPoolWideSlab = 128;
constexpr int pool_wide_slabs(int D) { return (D + kPoolWideSlab - 1) / kPoolWideSlab; }
void launch_pool_wide(cudaStream_t st, const float* x, int D, int ldx, int mode, const PoolSimpleParams& P, int n_heads,
                      float* logits, int n_seg, const ClipDesc* clips, int n_clips, float* partial, float* scores);
// Per-segment scores and weights [rows][n_heads] of the rows the pooling module read (x: D real columns at a stride of
// ldx, D <= 4096).  mode: enum nisqa_pool.  P.w3 / P.b3: each head's last Linear [n_heads][D] (columns in the rows'
// order).  logits [n_seg][n_heads]: the attention logits the pooling path wrote (PoolAttFF; PoolAtt over wide rows), or
// nullptr for PoolAtt, whose logits a1 . x + a1b (P.a1 [n_heads][D], P.a1b) are then formed here.  row_off [n_clips]:
// the clip's first output row, < 0 for a clip that gets none.
void launch_segment_scores(cudaStream_t st, const float* x, int D, int ldx, const float* logits, const PoolSimpleParams& P,
                           int n_heads, int mode, const ClipDesc* clips, int n_clips, const long long* row_off,
                           float* seg_scores, float* seg_weights);
// Each head's pooled vector [n_clips][n_heads][W] (the input of its last Linear) and, when rows != nullptr, the rows
// themselves [.][W] at row_off (< 0: none), both in the reference's column order: reference column j is x's column
// src_col[j] (nullptr: the same order; W <= 4096).  x, ldx, logits, P.a1 / P.a1b, mode as launch_segment_scores.  de:
// odd clips are NISQA_DE reference clips.  Clips with n_seg == 0 and reference clips get NaN vectors.
void launch_pool_embed(cudaStream_t st, const float* x, int W, int ldx, const int* src_col, const float* logits,
                       const PoolSimpleParams& P, int n_heads, int mode, int de, const ClipDesc* clips, int n_clips,
                       const long long* row_off, float* pooled, float* rows);

// ---------------------------------------------------------------- td_tiled.cu (self-attention, NISQA_DE, SkipCNN / DFF)
void launch_td_in(cudaStream_t st, int nc, const float* feats, const float* WT, int nk, const float* b, const float* g,
                  const float* be, const float* qkvT, const float* qkvb, float qscale, const float* pe, const int* seg_clip,
                  const ClipDesc* clips, float* x0, float* qkv, int n_rows);
void launch_td_sa(cudaStream_t st, int nc, const float* x_in, const float* qkv, const ClipDesc* clips, int n_clips,
                  const int* qtile64_prefix, int n_qtiles, const SaLayerParams& P, int F, float* x_out,
                  const float* next_qkvT, const float* next_qkvb, float qscale, float* qkv_next,
                  const PoolHeadParams& H, int n_heads, float* logits);
// NISQA_DE alignment + fusion over td's rows x_td (W real columns, W <= 512, at a pitch of ld = 64 NC, pad columns zero)
// into fused [n_rows][nf ld] (part p at column p ld; rows of reference clips untouched).  work: de_align_work_floats(W,
// align, n_rows) floats (AttLuong / AttBahdanau projections, AttCosine norms); de_align_launches(align) kernels.
// al (an alignment call, else nullptr): each degraded row's first maximal score, its softmax weight, the softmax-weighted
// key position and the score (+ AttBahdanau's v bias) to al's arrays
size_t de_align_work_floats(int W, int align, int n_rows);
int de_align_launches(int align);
void launch_de_align(cudaStream_t st, const float* x_td, int W, int n_rows, const ClipDesc* clips, int n_clips,
                     const int* qtile64_prefix, int n_qtiles, int align, int soft, int fuse, const DeAlignParams& A,
                     float* work, float* fused, const DeAlignOut* al = nullptr);
void launch_de_finalize(cudaStream_t st, const ClipDesc* clips, int n_clips, int n_out, float* scores);
// SkipCNN / DFF rows: n_mels * seg_len features at index m * seg_len + t, zero up to the row stride ld (a multiple of 64)
void launch_seg_feats(cudaStream_t st, const float* mel, int n_mels, int seg_len, int ld, const int* seg_frame0,
                      const float* seg_thr, const float* bn, int n_seg, float* out);
void launch_linear_tile(cudaStream_t st, const float* X, int ldx, const float* WT, const float* bias, int relu, float* Y, int ldy,
                        int n_rows, int K, int N);

// ---------------------------------------------------------------- resample_gpu.cu
void launch_resample(cudaStream_t st, const void* raw, int fmt_f32, const ResampleClip* clips, int n_clips, int max_fix,
                     double* t_start, const double* win, int nwin, int num_table, float* out);

// ---------------------------------------------------------------- ingest.cu (nisqa_predict_device_batch)
// One caller-owned strided [clips][channels][length] device array (nisqa_device_batch)
struct IngestSrc {
  const void* data;
  long long clip_stride, channel_stride;   // elements
  int n_channels;
  int channel;                             // -1: mono mix; else that channel (ignored for one channel)
  int f32;                                 // 1: float32 samples, 0: int16
};
// The clips of a call in the engine's order: clip g (of the whole call) is clip g / n_src of source g % n_src (NISQA_DE:
// source 0 the degraded batch, source 1 the reference batch)
struct IngestSources { IngestSrc s[2]; int n_src; };
// Packed mono PCM of the clips a table names (src_clip of each row), written where the table says: the pass's ClipDesc
// rows (pcm_off, n_samples; skipped clips are not read) or the resampler's ResampleClip rows (in_off, n_in).
// out_f32 0: int16 out (every source int16 and mono or picked); 1: float32 out (int16 scaled by 1/32768).
void launch_ingest(cudaStream_t st, const IngestSources& src, const ClipDesc* clips, int n_clips, long long max_n,
                   int out_f32, void* out);
void launch_ingest(cudaStream_t st, const IngestSources& src, const ResampleClip* clips, int n_clips, long long max_n,
                   int out_f32, void* out);
// nisqa_predict_device_windows: samples src_off .. src_off + n_samples - 1 of recording `src` of the batch to pcm_off, once
// per span (max_n: the longest span)
void launch_ingest_spans(cudaStream_t st, const IngestSrc& src, const WinSpan* spans, int n_spans, long long max_n,
                         int out_f32, void* out);
// Live feeds: the n_in samples of feed b's chunk (clip b of src) appended to its sample ring at t0 (and its mirror)
void launch_ingest_feed(cudaStream_t st, const IngestSrc& src, const FeedPush* push, int n_feeds, long long max_n,
                        const FeedGeom& g, int out_f32, void* ring);

// ---------------------------------------------------------------- resample.cpp
// the interpolation table of the resampler (set by nisqa_resample_set_filter); false before that call
bool resample_table(std::vector<double>* win, int* num_table);

}  // namespace nisqa

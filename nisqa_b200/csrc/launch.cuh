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
// learned weights of AttLuong (wT [64][64] k-major, b [64]) / AttBahdanau (wqT, wyT [64][128] k-major, bq, by, v [128])
struct DeAlignParams { const float* wT; const float* b; const float* wqT; const float* bq; const float* wyT; const float* by; const float* v; };
struct ResampleClip {
  long long in_off;      // element offset of the clip in the raw input buffer (float32, or int16 scaled by 1/32768)
  long long out_off;     // element offset in the packed float32 output buffer
  long long time_off;    // first entry of the clip in the chunk-start time register table
  int n_in;              // input samples
  int n_out;             // resampy's int(n_in * ratio)
  int n_fix;             // librosa fix_length: ceil(n_in * ratio) (zero padded / trimmed)
  int copy;              // 1: sr_orig == sr_new, plain conversion / copy
  double ratio;          // sr_new / sr_orig
};

// ---------------------------------------------------------------- frontend.cu
// mel: [frames][n_mels]; one kernel instance per band count, n_mels in {32, 40, 48, 64, 80, 96, 128} (frontend_supports_mels)
bool frontend_supports_mels(int n_mels);
void launch_frontend(cudaStream_t st, int n_mels, const void* pcm, int fmt_f32, const ClipDesc* clips, int n_clips, int max_pairs,
                     const FbTables* fbs, const float2* tw, float* mel, unsigned* clipmax, int Q, int max_span, int ppc);
void launch_seg_table(cudaStream_t st, const ClipDesc* clips, int n_clips, const int* seg_prefix, const unsigned* clipmax,
                      int seg_hop, int n_seg, int* seg_frame0, float* seg_thr, int* seg_clip);
void launch_mel_dump(cudaStream_t st, const float* mel, const ClipDesc* clips, int n_clips, const unsigned* clipmax, int n_mels,
                     float* out);

// ---------------------------------------------------------------- cnn.cu (fp32 FFMA convolutions)
// conv1 + pool1 of segments of n_mels x seg_len mel cells (rows n_mels floats apart): AdaptCNN any accepted shape ->
// ph x pw (cnn_pool_1), StandardCNN 48 x 15 only -> 24 x 8.  c1 output channels: 16, 32 or 64 into the planes (out_hi),
// 16 into fp32 `out`.  false: no instance for the shape.
bool launch_conv1(cudaStream_t st, int std_mode, int c1, const float* mel, int n_mels, int seg_len, const int* seg_frame0,
                  const float* seg_thr, const float* w1, const float* b1, float* out, int n_seg, void* out_hi, void* out_lo,
                  float store_scale, int ph, int pw);
void launch_conv_layer(cudaStream_t st, int std_mode, int layer, const float* in, const float* w, const float* b, float* out,
                       int n_seg);
// rows of `ld` floats (>= hw * ch)
void launch_nhwc_to_nchw(cudaStream_t st, const float* in, int ld, float* out, long long n, int hw, int ch);

// ---------------------------------------------------------------- conv_split.cu (tensor-core convolutions on fp16 planes)
size_t split_plane_bytes(int std_mode, int layer, int C, int n_seg, const CnnPools& pools);
// AdaptCNN conv2..conv6 take cin, cout in {16, 32, 64} (the pairs cnn_c_out_1/2/3 reach) and any accepted pools;
// StandardCNN its shipped ones.  The fp32 features of conv6 go out in rows of (h3 cout + 63) / 64 * 64 floats (AdaptCNN),
// zero-padded.
bool conv_split_supported(int cin, int cout);
bool launch_conv_split(cudaStream_t st, int std_mode, int layer, int cin, int cout, const void* in_hi, const void* in_lo,
                       const void* wtc, const float* b, float out_scale, float store_scale, void* out_hi, void* out_lo,
                       float* out_f32, int n_seg, const CnnPools& pools);
// the fused conv1 + conv2 kernel: 48 x 15 segments, c1 = 16, c2 = 32 (AdaptCNN also 16)
bool conv12_supported(int std_mode, int c1, int c2);
void launch_conv12(cudaStream_t st, int std_mode, int c2, const float* mel, const int* seg_frame0, const float* seg_thr,
                   const float* w1, const float* b1, float c1_scale, const void* wtc2, const float* bias2, float scale2,
                   float store_scale, void* out_hi, void* out_lo, int n_seg);
void launch_unsplit(cudaStream_t st, int std_mode, int layer, int C, const void* hi, const void* lo, float unit, float* out,
                    int n_seg, const CnnPools& pools);

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

// ---------------------------------------------------------------- td_tiled.cu (self-attention, NISQA_DE, SkipCNN / DFF)
void launch_td_in(cudaStream_t st, int nc, const float* feats, const float* WT, int nk, const float* b, const float* g,
                  const float* be, const float* qkvT, const float* qkvb, float qscale, const float* pe, const int* seg_clip,
                  const ClipDesc* clips, float* x0, float* qkv, int n_rows);
void launch_td_sa(cudaStream_t st, int nc, const float* x_in, const float* qkv, const ClipDesc* clips, int n_clips,
                  const int* qtile64_prefix, int n_qtiles, const SaLayerParams& P, int F, float* x_out,
                  const float* next_qkvT, const float* next_qkvb, float qscale, float* qkv_next,
                  const PoolHeadParams& H, int n_heads, float* logits);
void launch_de_align(cudaStream_t st, const float* x_td, const ClipDesc* clips, int n_clips, const int* qtile64_prefix,
                     int n_qtiles, int align, int soft, int fuse, const DeAlignParams& A, float* fused);
void launch_de_finalize(cudaStream_t st, const ClipDesc* clips, int n_clips, int n_out, float* scores);
// SkipCNN / DFF rows: n_mels * seg_len features at index m * seg_len + t, zero up to the row stride ld (a multiple of 64)
void launch_seg_feats(cudaStream_t st, const float* mel, int n_mels, int seg_len, int ld, const int* seg_frame0,
                      const float* seg_thr, const float* bn, int n_seg, float* out);
void launch_linear_tile(cudaStream_t st, const float* X, int ldx, const float* WT, const float* bias, int relu, float* Y, int ldy,
                        int n_rows, int K, int N);

// ---------------------------------------------------------------- resample_gpu.cu
void launch_resample(cudaStream_t st, const void* raw, int fmt_f32, const ResampleClip* clips, int n_clips, int max_fix,
                     double* t_start, const double* win, int nwin, int num_table, float* out);

// ---------------------------------------------------------------- resample.cpp
// the interpolation table of the resampler (set by nisqa_resample_set_filter); false before that call
bool resample_table(std::vector<double>* win, int* num_table);

}  // namespace nisqa

"""ctypes binding of libnisqa_b200.so (include/nisqa_b200.h) - the only way Python reaches the
CUDA hot path.  PyTorch / NumPy arrays are used as containers only: the library receives raw
pointers and sizes.

There is no CPU fallback: if the shared library is missing or no CUDA device is usable,
constructing an :class:`Engine` raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libnisqa_b200.so")

ABI_VERSION = 4
MAX_IN_FLIGHT = 6          # staging slots of the engine (nisqa_submit_pcm)
# enum nisqa_arch: td self-attention (0) or LSTM (1) with td_2 skip or self-attention; td_2 LSTM behind either (2, 3);
# no td (td='skip') with td_2 skip or self-attention (4), or StandardCNN with an LSTM td_2 (5)
ARCH_ADAPT_SA_ATTFF, ARCH_STD_LSTM_LASTBI, ARCH_SA_LSTM, ARCH_LSTM_LSTM, ARCH_SKIP, ARCH_SKIP_LSTM = 0, 1, 2, 3, 4, 5
FMT_S16, FMT_F32 = 0, 1
CLIP_OK, CLIP_TOO_SHORT, CLIP_TOO_LONG = 0, 1, 2
POOL_ATT_FF, POOL_ATT, POOL_AVG, POOL_MAX, POOL_LAST_STEP, POOL_LAST_STEP_BI = range(6)
# NISQA_DE options (enum nisqa_de_align / nisqa_de_apply / nisqa_de_fuse)
CNN_CONV, CNN_SKIP, CNN_DFF, CNN_STANDARD = 0, 1, 2, 3
DE_ALIGN = {"dot": 1, "cosine": 2, "distance": 3, "luong": 4, "bahd": 5}
DE_APPLY = {"hard": 0, "soft": 1}
DE_FUSE = {"x/y/-": 0, "+/-": 1, "x/y": 2}
(STAGE_MEL_DB, STAGE_POOL1, STAGE_POOL2, STAGE_CONV3, STAGE_POOL3, STAGE_CONV5, STAGE_CNN_FEAT,
 STAGE_TD_IN, STAGE_TD_OUT, STAGE_TD1_OUT, STAGE_DE_FUSED) = range(11)

# every symbol include/nisqa_b200.h declares (checked by tests/test_abi.py)
EXPORTS = [
    "nisqa_create", "nisqa_destroy", "nisqa_last_error", "nisqa_load_weights",
    "nisqa_predict_pcm", "nisqa_predict_pcm_device", "nisqa_stage_dump", "nisqa_segment_counts",
    "nisqa_mel_filterbank", "nisqa_gather_nccl", "nisqa_nccl_unique_id", "nisqa_nccl_init",
    "nisqa_kernel_launches", "nisqa_stream", "nisqa_set_profiling", "nisqa_group_ms", "nisqa_set_option",
    "nisqa_submit_pcm", "nisqa_wait", "nisqa_drain", "nisqa_join", "nisqa_set_gather_target",
    "nisqa_wav_probe", "nisqa_wav_decode", "nisqa_wav_probe_batch", "nisqa_wav_decode_batch",
    "nisqa_resample_set_filter", "nisqa_resample_out_len", "nisqa_resample_f32",
    "nisqa_resample_device", "nisqa_predict_pcm_resampled", "nisqa_set_cnn_pools", "nisqa_predict_device_batch",
    "nisqa_predict_device_batch_segments", "nisqa_window_counts", "nisqa_predict_device_windows",
    "nisqa_feed_create", "nisqa_feed_rows", "nisqa_feed_push", "nisqa_feed_device_bytes", "nisqa_feed_destroy",
    "nisqa_embedding_width", "nisqa_predict_device_batch_embeddings", "nisqa_window_pair_counts",
    "nisqa_predict_device_window_pairs", "nisqa_feed_pair_create", "nisqa_feed_pair_rows", "nisqa_feed_pair_push",
    "nisqa_predict_device_batch_alignment", "nisqa_predict_device_window_pairs_alignment",
    "nisqa_predict_device_batch_shared_ref", "nisqa_submit_pcm_pairs",
]


class NisqaConfig(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("arch", C.c_int32), ("n_out", C.c_int32),
                ("n_fft", C.c_int32), ("n_mels", C.c_int32), ("seg_len", C.c_int32),
                ("seg_hop", C.c_int32), ("max_segments", C.c_int32), ("hop_s", C.c_double),
                ("win_s", C.c_double), ("fmax", C.c_double), ("sa_layers", C.c_int32),
                ("max_chunk_segments", C.c_int32), ("pool", C.c_int32), ("pos_enc", C.c_int32),
                ("double_ended", C.c_int32), ("de_align", C.c_int32), ("de_align_apply", C.c_int32),
                ("de_fuse", C.c_int32), ("td2_layers", C.c_int32), ("td2_pos_enc", C.c_int32),
                ("cnn_kind", C.c_int32), ("cnn_fc", C.c_int32), ("de_fuse_dim", C.c_int32),
                ("sa_d_model", C.c_int32), ("sa_ff", C.c_int32), ("td2_d_model", C.c_int32), ("td2_ff", C.c_int32)]

SA_D_MODELS = (64, 128, 192, 256)     # self-attention widths the kernels are instantiated for (one head)
SA_FF_MAX = 4096                      # feed-forward width: a multiple of 64 up to this
LSTM_H = (32, 64, 96, 128, 192, 256)  # LSTM hidden sizes the kernels are instantiated for
LSTM_LAYERS_MAX = 4
CNN_FC_OUT_MAX = 1024                 # StandardCNN's fc_out width (None: the LSTM reads the 768 conv6 features)
N_MELS = (32, 40, 48, 64, 80, 96, 128)   # ms_n_mels: one front-end kernel instance per band count
SEG_LEN_MIN, SEG_LEN_MAX = 3, 31      # ms_seg_length, odd (128 x 31 bounds SkipCNN's / DFF's fan_in at 3968 < 4096)
CNN_CHANNELS = (16, 32, 64)           # AdaptCNN cnn_c_out_1/2/3: one fp16 plane row is one 32 / 64 / 128-byte swizzle atom
# AdaptCNN cnn_pool_1/2/3 [h, w]: one segment's padded (h + 1) x (w + 1) map fits a 256-row GEMM tile and the tap halo
# w + 2 stays within the 16 lead rows of a plane; conv6's 3 x pool_3[1] weight taps stay resident (w3 <= 3); the
# framewise fan-out c3 * h3 is at most 4096
SHIPPED_POOLS = ((24, 7), (12, 5), (6, 3))
POOL_W_MAX, POOL_CELLS_MAX, POOL3_W_MAX, CNN_FEATURES_MAX = 14, 256, 3, 4096


def _sa_widths(args, prefix, de=False):
    """(d_model, feed-forward width) of a self-attention stack's args ('td_sa' / 'td_2_sa'); refuses what the kernels do
    not implement, naming the value."""
    d, h, nhead = args.get(prefix + "_d_model"), args.get(prefix + "_h"), args.get(prefix + "_nhead")
    if nhead != 1:
        raise NotImplementedError("%s_nhead=%r: the engine runs one-head self-attention" % (prefix, nhead))
    if d not in SA_D_MODELS or (de and d != 64):
        raise NotImplementedError("%s_d_model=%r: the engine runs d_model %s%s" % (
            prefix, d, "64" if de else "64, 128, 192 or 256", " in NISQA_DE" if de else ""))
    if h is None or int(h) != h or h <= 0 or h % 64 != 0 or h > SA_FF_MAX:
        raise NotImplementedError("%s_h=%r: the engine needs a positive multiple of 64 up to %d" % (prefix, h, SA_FF_MAX))
    return int(d), int(h)


def _check_lstm(args, key):
    """Refuses the LSTM hyper-parameters ('td_lstm' / 'td_2_lstm') the kernels do not implement, naming the value; returns
    the LSTM's fan_out.  The engine reads the LSTM's shape from the checkpoint's tensors (nisqa_load_weights); nothing of
    it goes into nisqa_config."""
    where = "td_2='lstm' with " if key == "td_2_lstm" else ""
    h, nl = args.get(key + "_h"), args.get(key + "_num_layers")
    if h not in LSTM_H:
        raise NotImplementedError("%s%s_h=%r: the engine runs LSTM hidden sizes %s" % (where, key, h, ", ".join(map(str, LSTM_H))))
    if nl is None or int(nl) != nl or not 1 <= nl <= LSTM_LAYERS_MAX:
        raise NotImplementedError("%s%s_num_layers=%r: the engine runs 1 to %d LSTM layers" % (where, key, nl, LSTM_LAYERS_MAX))
    return (2 if args.get(key + "_bidirectional") else 1) * h


def _check_standard_cnn(args):
    """Refuses the StandardCNN hyper-parameters the kernels do not implement, naming the value.  Its fc_out width comes
    from the checkpoint's tensors."""
    fc = args.get("cnn_fc_out_h")
    if fc and (int(fc) != fc or not 1 <= fc <= CNN_FC_OUT_MAX):
        raise NotImplementedError("cnn_fc_out_h=%r: the engine runs fc_out widths 1 to %d (or None)" % (fc, CNN_FC_OUT_MAX))
    ch = (args.get("cnn_c_out_1"), args.get("cnn_c_out_2"), args.get("cnn_c_out_3"))
    if ch != (16, 32, 64):
        raise NotImplementedError("cnn_c_out_1/2/3=%r: the engine runs StandardCNN with 16, 32, 64 channels" % (ch,))
    _check_kernel_size(args)


def _check_kernel_size(args):
    ks = args.get("cnn_kernel_size")
    if not (ks == 3 or (isinstance(ks, (list, tuple)) and tuple(ks) == (3, 3))):
        raise NotImplementedError("cnn_kernel_size=%r: the engine runs 3x3 convolutions" % (ks,))


def _check_adapt_pools(args):
    """AdaptCNN's (cnn_pool_1, cnn_pool_2, cnn_pool_3) as ((h, w), ...); refuses what the kernels do not implement, naming
    the field and value."""
    pools = []
    for i in (1, 2, 3):
        key = "cnn_pool_%d" % i
        p = args.get(key)
        ok = isinstance(p, (list, tuple)) and len(p) == 2 and all(isinstance(v, int) and v >= 1 for v in p)
        if not ok or p[1] > POOL_W_MAX or (p[0] + 1) * (p[1] + 1) > POOL_CELLS_MAX:
            raise NotImplementedError("%s=%r: the engine runs AdaptCNN pool sizes [h, w] with w <= %d and (h + 1) * (w + 1) "
                                      "<= %d" % (key, p, POOL_W_MAX, POOL_CELLS_MAX))
        if i == 3 and p[1] > POOL3_W_MAX:
            raise NotImplementedError("%s=%r: the engine runs pool_3 widths 1 to %d (conv6's kernel is 3 x pool_3[1])"
                                      % (key, p, POOL3_W_MAX))
        pools.append((int(p[0]), int(p[1])))
    c3 = int(args["cnn_c_out_3"])
    if c3 * pools[2][0] > CNN_FEATURES_MAX:
        raise NotImplementedError("cnn_c_out_3=%d, cnn_pool_3=%r: the engine runs up to %d framewise features "
                                  "(cnn_c_out_3 * cnn_pool_3[0] = %d)" % (c3, args["cnn_pool_3"], CNN_FEATURES_MAX, c3 * pools[2][0]))
    return tuple(pools)


def _framewise(args):
    """(cnn_kind, cnn_fc, pools) of the framewise model in front of a self-attention td or of no td; refuses the
    hyper-parameters the kernels do not implement, naming the value (pools: AdaptCNN's cnn_pool_1/2/3, else None)."""
    cnn = args.get("cnn_model")
    if cnn == "standard":
        _check_standard_cnn(args)
        return CNN_STANDARD, 0, None
    cnn_kind = CNN_CONV if cnn == "adapt" else CNN_DFF if cnn == "dff" else CNN_SKIP
    pools = None
    if cnn == "adapt":
        # (the engine reads the channel counts from the conv / bn tensors in nisqa_load_weights)
        for i in (1, 2, 3):
            c = args.get("cnn_c_out_%d" % i)
            if c not in CNN_CHANNELS or int(c) != c:
                raise NotImplementedError("cnn_c_out_%d=%r: the engine runs AdaptCNN channel counts 16, 32 or 64" % (i, c))
        _check_kernel_size(args)
        pools = _check_adapt_pools(args)
    cnn_fc = int(args.get("cnn_fc_out_h") or 0)         # AdaptCNN's optional Linear behind conv6 (lib:682-684), SkipCNN's
    if cnn_kind == CNN_DFF and cnn_fc == 0:
        cnn_fc = 4096                                   # DFF's default hidden width (lib:544)
    if cnn_fc % 64 != 0:
        raise NotImplementedError("cnn_fc_out_h=%d: the engine needs a multiple of 64" % cnn_fc)
    return cnn_kind, cnn_fc, pools


class NisqaDeviceBatch(C.Structure):
    """nisqa_device_batch: clips in device memory as a strided [n_clips][n_channels][length] array"""
    _fields_ = [("data", C.c_void_p), ("sample_fmt", C.c_int32), ("n_clips", C.c_int32), ("n_channels", C.c_int32),
                ("channel", C.c_int32), ("length", C.c_int64), ("clip_stride", C.c_int64), ("channel_stride", C.c_int64),
                ("n_samples", C.POINTER(C.c_int64)), ("sample_rate", C.c_int32)]


class NisqaEmbeddingOut(C.Structure):
    """nisqa_embedding_out: device [rows][n_out][width] pooled vectors and optional [n_rows][width] segment rows"""
    _fields_ = [("pooled", C.c_void_p), ("rows", C.c_void_p), ("n_rows", C.c_int64)]


class NisqaSegmentOut(C.Structure):
    """nisqa_segment_out: device [n_rows][n_out] per-segment scores and pooling weights"""
    _fields_ = [("scores", C.c_void_p), ("weights", C.c_void_p), ("n_rows", C.c_int64)]


class NisqaAlignmentOut(C.Structure):
    """nisqa_alignment_out: device [n_rows] ref_seg (int32), weight, centroid and peak (fp32) of NISQA_DE's alignment"""
    _fields_ = [("ref_seg", C.c_void_p), ("weight", C.c_void_p), ("centroid", C.c_void_p), ("peak", C.c_void_p),
                ("n_rows", C.c_int64)]


class NisqaTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.POINTER(C.c_float)), ("ndim", C.c_int32),
                ("dims", C.c_int64 * 4)]


class EngineError(RuntimeError):
    pass


_lib = None


def load_library(path=None):
    """dlopen the engine.  Raises if it has not been built (python -m nisqa_b200.build)."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or os.environ.get("NISQA_LIB") or LIB_PATH          # NISQA_LIB: a variant build for A/B measurements
    if not os.path.exists(p):
        raise EngineError(
            "libnisqa_b200.so is missing (%s): build it with `python -m nisqa_b200.build`; "
            "there is no CPU fallback" % p)
    lib = C.CDLL(p)
    vp, i32p, i64p, f32p = C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_float)
    lib.nisqa_create.argtypes = [C.POINTER(vp), C.c_int, C.POINTER(NisqaConfig)]
    lib.nisqa_create.restype = C.c_int
    lib.nisqa_destroy.argtypes = [vp]
    lib.nisqa_destroy.restype = None
    lib.nisqa_last_error.argtypes = [vp]
    lib.nisqa_last_error.restype = C.c_char_p
    lib.nisqa_load_weights.argtypes = [vp, C.POINTER(NisqaTensor), C.c_int]
    lib.nisqa_load_weights.restype = C.c_int
    lib.nisqa_predict_pcm.argtypes = [vp, C.c_int, C.POINTER(vp), i64p, i32p, C.c_int, f32p, i32p, i32p]
    lib.nisqa_predict_pcm.restype = C.c_int
    lib.nisqa_submit_pcm.argtypes = [vp, C.c_int, C.POINTER(vp), i64p, i32p, C.c_int, f32p, i32p, i32p, i64p]
    lib.nisqa_submit_pcm.restype = C.c_int
    lib.nisqa_wav_probe.argtypes = [C.c_char_p, C.c_int32, i32p, i64p, i32p, i32p]
    lib.nisqa_wav_probe.restype = C.c_int
    lib.nisqa_wav_decode.argtypes = [C.c_char_p, C.c_int32, C.c_int32, vp, C.c_int64]
    lib.nisqa_wav_decode.restype = C.c_int64
    cpp = C.POINTER(C.c_char_p)
    lib.nisqa_wav_probe_batch.argtypes = [C.c_int, cpp, C.c_int32, C.c_int, i32p, i64p, i32p, i32p]
    lib.nisqa_wav_probe_batch.restype = C.c_int
    lib.nisqa_wav_decode_batch.argtypes = [C.c_int, cpp, C.c_int32, C.c_int32, vp, i64p, i64p, C.c_int, i32p]
    lib.nisqa_wav_decode_batch.restype = C.c_int
    lib.nisqa_resample_set_filter.argtypes = [C.POINTER(C.c_double), C.c_int64, C.c_int32]
    lib.nisqa_resample_set_filter.restype = C.c_int
    lib.nisqa_resample_out_len.argtypes = [C.c_int64, C.c_int32, C.c_int32]
    lib.nisqa_resample_out_len.restype = C.c_int64
    lib.nisqa_resample_f32.argtypes = [f32p, C.c_int64, C.c_int32, C.c_int32, f32p, C.c_int64]
    lib.nisqa_resample_f32.restype = C.c_int64
    lib.nisqa_resample_device.argtypes = [vp, vp, C.c_int64, C.c_int, C.c_int32, C.c_int32, f32p, C.c_int64]
    lib.nisqa_resample_device.restype = C.c_int
    lib.nisqa_predict_pcm_resampled.argtypes = [vp, C.c_int, C.POINTER(vp), i64p, i32p, C.c_int, C.c_int32, f32p, i32p, i32p]
    lib.nisqa_predict_pcm_resampled.restype = C.c_int
    lib.nisqa_set_gather_target.argtypes = [vp, vp, C.c_int]
    lib.nisqa_set_gather_target.restype = C.c_int
    lib.nisqa_join.argtypes = [vp]
    lib.nisqa_join.restype = C.c_int
    lib.nisqa_wait.argtypes = [vp, C.c_int64]
    lib.nisqa_wait.restype = C.c_int
    lib.nisqa_drain.argtypes = [vp]
    lib.nisqa_drain.restype = C.c_int
    lib.nisqa_predict_pcm_device.argtypes = [vp, C.c_int, vp, i64p, i64p, i32p, C.c_int, vp, i32p, i32p, C.c_int]
    lib.nisqa_predict_pcm_device.restype = C.c_int
    dbp = C.POINTER(NisqaDeviceBatch)
    lib.nisqa_predict_device_batch.argtypes = [vp, vp, dbp, dbp, C.c_int32, vp, i32p, i32p]
    lib.nisqa_predict_device_batch.restype = C.c_int
    lib.nisqa_predict_device_batch_segments.argtypes = [vp, vp, dbp, dbp, C.c_int32, vp, C.POINTER(NisqaSegmentOut), i32p, i32p]
    lib.nisqa_predict_device_batch_segments.restype = C.c_int
    lib.nisqa_embedding_width.argtypes = [vp, i32p]
    lib.nisqa_embedding_width.restype = C.c_int
    lib.nisqa_predict_device_batch_embeddings.argtypes = [vp, vp, dbp, dbp, C.c_int32, vp, C.POINTER(NisqaEmbeddingOut),
                                                          i32p, i32p]
    lib.nisqa_predict_device_batch_embeddings.restype = C.c_int
    lib.nisqa_predict_device_windows.argtypes = [vp, vp, dbp, C.c_int32, C.c_int64, C.c_int32, vp, C.c_int64, i32p, i32p]
    lib.nisqa_predict_device_windows.restype = C.c_int
    lib.nisqa_window_counts.argtypes = [C.POINTER(NisqaConfig), C.c_int64, C.c_int32, C.c_int64, C.c_int32, i64p, i32p, i32p,
                                        C.c_int64]
    lib.nisqa_window_counts.restype = C.c_int
    lib.nisqa_predict_device_window_pairs.argtypes = [vp, vp, dbp, dbp, C.c_int32, C.c_int64, C.c_int32, C.c_int32, vp,
                                                      C.c_int64, i32p, i32p, i32p, i32p]
    lib.nisqa_predict_device_window_pairs.restype = C.c_int
    lib.nisqa_predict_device_batch_alignment.argtypes = [vp, vp, dbp, dbp, C.c_int32, vp, C.POINTER(NisqaAlignmentOut),
                                                         i32p, i32p]
    lib.nisqa_predict_device_batch_alignment.restype = C.c_int
    lib.nisqa_predict_device_batch_shared_ref.argtypes = [vp, vp, dbp, dbp, i32p, C.c_int32, vp, C.POINTER(NisqaSegmentOut),
                                                          C.POINTER(NisqaEmbeddingOut), C.POINTER(NisqaAlignmentOut),
                                                          i32p, i32p, i32p, i32p]
    lib.nisqa_predict_device_batch_shared_ref.restype = C.c_int
    lib.nisqa_submit_pcm_pairs.argtypes = [vp, C.c_int, C.POINTER(vp), i64p, i32p, C.c_int, C.POINTER(vp), i64p, i32p, i32p,
                                           C.c_int, f32p, i32p, i32p, i32p, i32p, i64p]
    lib.nisqa_submit_pcm_pairs.restype = C.c_int
    lib.nisqa_predict_device_window_pairs_alignment.argtypes = [vp, vp, dbp, dbp, C.c_int32, C.c_int64, C.c_int32, C.c_int32,
                                                                vp, C.c_int64, C.POINTER(NisqaAlignmentOut), i32p, i32p,
                                                                i32p, i32p]
    lib.nisqa_predict_device_window_pairs_alignment.restype = C.c_int
    lib.nisqa_window_pair_counts.argtypes = [C.POINTER(NisqaConfig), C.c_int64, C.c_int64, C.c_int32, C.c_int64, C.c_int32,
                                             C.c_int32, i64p, i32p, i32p, i32p, i32p, C.c_int64]
    lib.nisqa_window_pair_counts.restype = C.c_int
    u8p = C.POINTER(C.c_uint8)
    lib.nisqa_feed_create.argtypes = [vp, C.POINTER(vp), C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_int64]
    lib.nisqa_feed_create.restype = C.c_int
    lib.nisqa_feed_rows.argtypes = [C.POINTER(NisqaConfig), C.c_int32, C.c_int64, C.c_int32, C.c_int32, i64p, i64p, u8p,
                                    i64p, i32p, i64p, i32p, i32p, C.c_int64]
    lib.nisqa_feed_rows.restype = C.c_int
    lib.nisqa_feed_push.argtypes = [vp, vp, dbp, u8p, vp, C.c_int64, i32p, i64p, i32p, i32p]
    lib.nisqa_feed_push.restype = C.c_int
    lib.nisqa_feed_device_bytes.argtypes = [vp]
    lib.nisqa_feed_device_bytes.restype = C.c_int64
    lib.nisqa_feed_destroy.argtypes = [vp]
    lib.nisqa_feed_destroy.restype = None
    lib.nisqa_feed_pair_create.argtypes = [vp, C.POINTER(vp), C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_int32,
                                           C.c_int64, C.c_int64]
    lib.nisqa_feed_pair_create.restype = C.c_int
    lib.nisqa_feed_pair_rows.argtypes = [C.POINTER(NisqaConfig), C.c_int32, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                         i64p, i64p, i64p, i64p, u8p, i64p, i32p, i64p, i32p, i32p, i32p, i32p, C.c_int64]
    lib.nisqa_feed_pair_rows.restype = C.c_int
    lib.nisqa_feed_pair_push.argtypes = [vp, vp, dbp, dbp, u8p, vp, C.c_int64, i32p, i64p, i32p, i32p, i32p, i32p]
    lib.nisqa_feed_pair_push.restype = C.c_int
    lib.nisqa_stage_dump.argtypes = [vp, C.c_int, f32p, C.c_int64]
    lib.nisqa_stage_dump.restype = C.c_int64
    lib.nisqa_segment_counts.argtypes = [C.POINTER(NisqaConfig), C.c_int64, C.c_int32, i32p, i32p, i32p]
    lib.nisqa_segment_counts.restype = C.c_int
    lib.nisqa_mel_filterbank.argtypes = [vp, C.c_int32, f32p, C.c_int64]
    lib.nisqa_mel_filterbank.restype = C.c_int
    lib.nisqa_gather_nccl.argtypes = [vp, vp, vp, C.c_int, vp]
    lib.nisqa_gather_nccl.restype = C.c_int
    lib.nisqa_nccl_unique_id.argtypes = [vp, vp]
    lib.nisqa_nccl_unique_id.restype = C.c_int
    lib.nisqa_nccl_init.argtypes = [vp, C.c_int, C.c_int, vp]
    lib.nisqa_nccl_init.restype = C.c_int
    lib.nisqa_kernel_launches.argtypes = [vp]
    lib.nisqa_kernel_launches.restype = C.c_int64
    lib.nisqa_stream.argtypes = [vp]
    lib.nisqa_stream.restype = vp
    lib.nisqa_set_profiling.argtypes = [vp, C.c_int]
    lib.nisqa_set_profiling.restype = C.c_int
    lib.nisqa_set_option.argtypes = [vp, C.c_char_p, C.c_int]
    lib.nisqa_set_option.restype = C.c_int
    lib.nisqa_set_cnn_pools.argtypes = [vp, i32p]
    lib.nisqa_set_cnn_pools.restype = C.c_int
    lib.nisqa_group_ms.argtypes = [vp, C.c_char_p]
    lib.nisqa_group_ms.restype = C.c_double
    if path is None:
        _lib = lib
    return lib


def config_from_args(args, max_chunk_segments=0):
    """Checkpoint ``args`` (reference model:941-942) -> nisqa_config.  Refuses anything the
    kernels do not implement (no fallback)."""
    cnn, td, pool = args.get("cnn_model"), args.get("td"), args.get("pool")
    if args.get("model") not in ("NISQA", "NISQA_DIM", "NISQA_DE"):
        raise NotImplementedError("Model not available in the engine: %r" % args.get("model"))
    de = args.get("model") == "NISQA_DE"
    pool_mode = {"avg": POOL_AVG, "max": POOL_MAX, "last_step": POOL_LAST_STEP, "last_step_bi": POOL_LAST_STEP_BI}.get(pool)
    if pool == "att":
        if args.get("pool_att_h") == 128:
            pool_mode = POOL_ATT_FF
        elif args.get("pool_att_h") in (None, 0):
            pool_mode = POOL_ATT
        else:
            raise NotImplementedError("pool_att_h=%r is not implemented by the engine (128 or None)" % args.get("pool_att_h"))
    if pool_mode is None:
        raise NotImplementedError("Pool option not available in the engine: %r" % pool)
    cnn_kind, cnn_fc, pools = CNN_CONV, 0, None
    td2 = args.get("td_2") or "skip"
    if td2 not in ("skip", "self_att", "lstm"):
        raise NotImplementedError("td_2=%r is not implemented by the engine (skip, self_att or lstm)" % (args.get("td_2"),))
    if de and td2 != "self_att":
        # (NISQA_DE fuses two self-attention outputs into a self-attention td_2, lib:404-424)
        raise NotImplementedError("NISQA_DE with td_2=%r: the engine runs NISQA_DE with td_2='self_att'" % (args.get("td_2"),))
    if cnn in ("adapt", None, "skip", "dff") and td == "self_att":
        # AdaptCNN, or a framewise model without convolutions (lib:504-583), in front of the self-attention stack
        arch = ARCH_ADAPT_SA_ATTFF
        cnn_kind, cnn_fc, pools = _framewise(args)
    elif (cnn, td) == ("standard", "self_att"):
        # StandardCNN (lib:811-836) in front of the self-attention stack; fc_out's width comes from the weights
        arch = ARCH_ADAPT_SA_ATTFF
        cnn_kind, cnn_fc, pools = _framewise(args)
    elif (cnn, td) == ("standard", "lstm"):
        # any LSTM width, depth and direction behind StandardCNN (lib:811-836, 925-943), every pooling module
        arch = ARCH_STD_LSTM_LASTBI
        _check_standard_cnn(args)
    elif cnn in ("adapt", None, "skip", "dff", "standard") and td in (None, "skip"):
        # no time-dependency model (TimeDependency._skip, lib:839-895): td_2, or the pooling module, reads the framewise rows
        if de:
            raise NotImplementedError("NISQA_DE with td=%r: the engine runs NISQA_DE with td='self_att'" % (td,))
        if td2 == "lstm" and cnn != "standard":
            raise NotImplementedError("td_2='lstm' behind td=%r and cnn_model=%r: the engine runs an LSTM td_2 behind no td "
                                      "for cnn_model='standard' only" % (td, cnn))
        arch = ARCH_SKIP
        cnn_kind, cnn_fc, pools = _framewise(args)
    else:
        raise NotImplementedError(
            "architecture cnn=%r td=%r pool=%r is not implemented by the engine" % (cnn, td, pool))
    if td2 == "lstm":
        arch = {ARCH_STD_LSTM_LASTBI: ARCH_LSTM_LSTM, ARCH_SKIP: ARCH_SKIP_LSTM}.get(arch, ARCH_SA_LSTM)
    # fan_out of each stage (lib:839-895): the pooling module reads the last one's rows
    td_lstm = arch in (ARCH_STD_LSTM_LASTBI, ARCH_LSTM_LSTM)
    skip = arch in (ARCH_SKIP, ARCH_SKIP_LSTM)
    fan1 = _check_lstm(args, "td_lstm") if td_lstm else None
    if skip:
        fan1 = int(args.get("cnn_fc_out_h") or 768) if cnn == "standard" else (
            cnn_fc or (pools[2][0] * int(args["cnn_c_out_3"]) if cnn == "adapt"
                       else int(args.get("ms_n_mels") or 0) * int(args.get("ms_seg_length") or 0)))
    fan2 = _check_lstm(args, "td_2_lstm") if td2 == "lstm" else None
    if pool_mode == POOL_LAST_STEP_BI:
        key = "td_2_lstm" if td2 == "lstm" else "td_lstm" if td2 == "skip" and td_lstm else None
        if key is None:
            raise NotImplementedError("pool='last_step_bi' behind td=%r, td_2=%r: PoolLastStepBi needs a bidirectional LSTM as the "
                                      "last time-dependency stage" % (td, args.get("td_2")))
        if not args.get(key + "_bidirectional"):
            raise NotImplementedError("pool='last_step_bi' with %s_bidirectional=%r: PoolLastStepBi needs a bidirectional LSTM"
                                      % (key, args.get(key + "_bidirectional")))
    if de:
        # double-ended model (reference lib:272-424, config/train_nisqa_double_ended.yaml): any framewise model + a
        # self-attention td, or StandardCNN + an LSTM td, on both signals; alignment and fusion at td's fan_out; td_2 =
        # self-attention
        if arch not in (ARCH_ADAPT_SA_ATTFF, ARCH_STD_LSTM_LASTBI):
            raise NotImplementedError("NISQA_DE is implemented for cnn_model='adapt', td='self_att'")
        if args.get("de_align") not in DE_ALIGN:
            raise NotImplementedError("de_align=%r is not implemented by the engine (dot, cosine, distance, luong, bahd)" % (args.get("de_align"),))
        if args.get("de_align_apply") not in DE_APPLY or args.get("de_fuse") not in DE_FUSE:
            raise NotImplementedError("de_align_apply / de_fuse option not available: %r / %r" % (args.get("de_align_apply"), args.get("de_fuse")))
        if args.get("de_fuse_dim") and int(args["de_fuse_dim"]) % 64 != 0:
            raise NotImplementedError("de_fuse_dim=%r: the engine needs a multiple of 64" % (args.get("de_fuse_dim"),))
    n_mels, seg_len = _check_mel_shape(args, td_lstm or cnn_kind == CNN_STANDARD)
    sa = td2w = (0, 0)
    if not td_lstm and not skip:
        sa = _sa_widths(args, "td_sa", de)
        fan1 = sa[0]
    if td2 == "self_att":
        td2w = _sa_widths(args, "td_2_sa", de)
        fan2 = td2w[0]
    if args["model"] == "NISQA_DIM" and fan2 is not None and fan2 != fan1:
        # NISQA_DIM builds its pooling heads for td's fan_out (lib:247-253): td_2 must keep it
        if td2 == "self_att" and not td_lstm and not skip:
            raise NotImplementedError("NISQA_DIM with td_2_sa_d_model=%d != td_sa_d_model=%d: the reference model cannot "
                                      "run it" % (fan2, fan1))
        raise NotImplementedError("NISQA_DIM with td_2 fan_out %d (%s) != td fan_out %d (%s): the reference model cannot run it" % (
            fan2, _fan_out_args(args, "td_2"), fan1, _fan_out_args(args, "td")))
    # ms_sr != None: the ingest converts every clip to that rate (nisqa_b200/resample.py) before the engine sees it
    cfg = NisqaConfig()
    cfg.abi_version = ABI_VERSION
    cfg.arch = arch
    cfg.n_out = 5 if args["model"] == "NISQA_DIM" else 1
    cfg.n_fft, cfg.n_mels, cfg.seg_len = 4096, n_mels, seg_len
    cfg.seg_hop = int(args["ms_seg_hop_length"])
    cfg.max_segments = int(args["ms_max_segments"]) if args.get("ms_max_segments") else 0
    cfg.hop_s, cfg.win_s = float(args["ms_hop_length"]), float(args["ms_win_length"])
    cfg.fmax = float(args["ms_fmax"])
    cfg.sa_layers = 0 if td_lstm or skip else int(args["td_sa_num_layers"])
    # NISQA_MAX_CHUNK: experiment knob (segments per internal pass) for A/B runs of the pass size
    cfg.max_chunk_segments = int(max_chunk_segments) or int(os.environ.get("NISQA_MAX_CHUNK", "0"))
    cfg.pool = pool_mode
    cfg.pos_enc = 1 if (not td_lstm and not skip and args.get("td_sa_pos_enc")) else 0
    cfg.cnn_kind, cfg.cnn_fc = cnn_kind, cnn_fc
    cfg.sa_d_model, cfg.sa_ff = sa
    cfg.td2_d_model, cfg.td2_ff = td2w
    if td2 == "self_att":
        cfg.td2_layers = int(args["td_2_sa_num_layers"])
        cfg.td2_pos_enc = 1 if args.get("td_2_sa_pos_enc") else 0
    if de:
        cfg.double_ended = 1
        cfg.de_fuse_dim = int(args.get("de_fuse_dim") or 0)
        cfg.de_align, cfg.de_align_apply, cfg.de_fuse = DE_ALIGN[args["de_align"]], DE_APPLY[args["de_align_apply"]], DE_FUSE[args["de_fuse"]]
    if pools is not None and pools != SHIPPED_POOLS:
        # (nisqa_config has no room for them: Engine applies them with nisqa_set_cnn_pools before the weights load)
        cfg.cnn_pools = pools
    return cfg


def _check_mel_shape(args, standard):
    """(n_mels, seg_len) of the checkpoint's Mel-spectrogram segments; refuses what the kernels do not implement, naming
    the value"""
    n_fft, n_mels, seg_len = args.get("ms_n_fft"), args.get("ms_n_mels"), args.get("ms_seg_length")
    if n_fft != 4096:
        raise NotImplementedError("ms_n_fft=%r: the engine's front end runs n_fft 4096 (four 1024-point FFTs)" % (n_fft,))
    if n_mels not in N_MELS or int(n_mels) != n_mels:
        raise NotImplementedError("ms_n_mels=%r: the engine runs %s Mel bands" % (n_mels, ", ".join(map(str, N_MELS))))
    if seg_len is None or int(seg_len) != seg_len or not SEG_LEN_MIN <= seg_len <= SEG_LEN_MAX:
        raise NotImplementedError("ms_seg_length=%r: the engine runs segments of %d to %d frames" % (seg_len, SEG_LEN_MIN, SEG_LEN_MAX))
    if seg_len % 2 == 0:
        raise NotImplementedError("ms_seg_length=%r: the reference's segment_specs refuses even segment lengths "
                                  "(seg_length must be odd)" % (seg_len,))
    if standard and (n_mels, seg_len) != (48, 15):
        raise NotImplementedError("ms_n_mels=%r, ms_seg_length=%r with cnn_model='standard': the reference's StandardCNN "
                                  "hard-codes output_height = 6, output_width = 2 (48 x 15 segments); use cnn_model='adapt'"
                                  % (n_mels, seg_len))
    return int(n_mels), int(seg_len)


def _fan_out_args(args, stage):
    """the args that set a time-dependency stage's fan_out, for refusals"""
    if args.get(stage) == "lstm":
        return "%s_lstm_h=%r, %s_lstm_bidirectional=%r" % (stage, args.get(stage + "_lstm_h"), stage,
                                                           args.get(stage + "_lstm_bidirectional"))
    if args.get(stage) in (None, "skip"):
        return "%s=%r: the framewise fan_out of cnn_model=%r, cnn_fc_out_h=%r" % (
            stage, args.get(stage), args.get("cnn_model"), args.get("cnn_fc_out_h"))
    return "%s_sa_d_model=%r" % (stage, args.get(stage + "_sa_d_model"))


def device_batch(data_ptr, sample_fmt, n_samples, n_channels, channel, length, clip_stride, channel_stride, sample_rate):
    """-> (NisqaDeviceBatch, its host n_samples array): one argument of Engine.predict_device_batch (element strides)"""
    ns = np.ascontiguousarray(n_samples, dtype=np.int64)
    b = NisqaDeviceBatch(data=data_ptr, sample_fmt=sample_fmt, n_clips=len(ns), n_channels=n_channels, channel=channel,
                         length=length, clip_stride=clip_stride, channel_stride=channel_stride,
                         n_samples=ns.ctypes.data_as(C.POINTER(C.c_int64)), sample_rate=sample_rate)
    return b, ns


def load_checkpoint(model_path, overrides=None):
    """-> (args, state_dict) of a checkpoint file, its ``args`` updated with ``overrides`` (the caller's dict takes
    precedence, reference model:941-942)."""
    import torch
    checkpoint = torch.load(model_path, map_location="cpu", weights_only=False)
    checkpoint["args"].update(overrides or {})
    return checkpoint["args"], checkpoint["model_state_dict"]


def engine_from_checkpoint(args, state_dict, device=0):
    """An Engine on ``device`` running the checkpoint: nisqa_config from its args, then its weights (strict: the engine
    names what is missing)."""
    cfg = config_from_args(args, max_chunk_segments=args.get("b200_max_chunk_segments", 0))
    eng = Engine(cfg, device=device)
    eng.load_state_dict(state_dict)
    return eng


def clip_status_error(status, where, n_samples, sample_rate, n_seg, hop_length, seg_length, max_length):
    """The reference's ValueError for a clip whose status is not CLIP_OK (lib:2259-2263 "Sample too short",
    lib:2276-2277 "n_wins > max_length"), else None.  ``where`` names the clip: a file path, or an argument and index."""
    if status == CLIP_TOO_SHORT:
        hop = int(sample_rate * hop_length)
        width = 1 + n_samples // hop if hop > 0 else 0
        return ValueError(
            "Sample too short. Only {} windows available but seg_length={}. "
            "Consider zero padding the audio sample. File: {}".format(width, seg_length, where))
    if status == CLIP_TOO_LONG:
        return ValueError(
            "n_wins {} > max_length {} --- {}. Increase max window length ms_max_segments!".format(n_seg, max_length, where))
    return None


def segment_counts(cfg, n_samples, sample_rate):
    """(n_frames, n_segments, status) - pure host arithmetic inside the library."""
    lib = load_library()
    a, b, c = C.c_int32(), C.c_int32(), C.c_int32()
    rc = lib.nisqa_segment_counts(C.byref(cfg), int(n_samples), int(sample_rate), C.byref(a), C.byref(b), C.byref(c))
    if rc != 0:
        raise EngineError("nisqa_segment_counts failed (%d)" % rc)
    return a.value, b.value, c.value


def window_counts(cfg, n_samples, sample_rate, window, hop_frames):
    """(n_segments int32[K], status int32[K]) of the K windows of a recording of ``n_samples`` samples at the model rate
    ``sample_rate``: ``window`` samples, a hop of ``hop_frames`` mel frames (nisqa_window_counts, host arithmetic)"""
    lib = load_library()
    k = C.c_int64()
    args = (C.byref(cfg), int(n_samples), int(sample_rate), int(window), int(hop_frames), C.byref(k))
    rc = lib.nisqa_window_counts(*args, None, None, 0)
    if rc != 0:
        raise EngineError("nisqa_window_counts failed (%d): window %d, hop_frames %d at %d Hz" % (rc, window, hop_frames,
                                                                                                  sample_rate))
    nseg, status = np.empty(k.value, np.int32), np.empty(k.value, np.int32)
    lib.nisqa_window_counts(*args, nseg.ctypes.data_as(C.POINTER(C.c_int32)), status.ctypes.data_as(C.POINTER(C.c_int32)),
                            k.value)
    return nseg, status


def window_pair_counts(cfg, n_samples, ref_n_samples, sample_rate, window, hop_frames, margin_frames):
    """(n_segments, status, ref_n_segments, ref_status), int32[K] each, of the K window pairs of a degraded recording of
    ``n_samples`` samples and its reference of ``ref_n_samples`` at the model rate ``sample_rate``: the windows of
    :func:`window_counts` and reference windows ``margin_frames`` mel frames wider on either side
    (nisqa_window_pair_counts, host arithmetic)"""
    lib = load_library()
    k = C.c_int64()
    args = (C.byref(cfg), int(n_samples), int(ref_n_samples), int(sample_rate), int(window), int(hop_frames),
            int(margin_frames), C.byref(k))
    rc = lib.nisqa_window_pair_counts(*args, None, None, None, None, 0)
    if rc != 0:
        raise EngineError("nisqa_window_pair_counts failed (%d): window %d, hop_frames %d, margin_frames %d at %d Hz"
                          % (rc, window, hop_frames, margin_frames, sample_rate))
    out = [np.empty(k.value, np.int32) for _ in range(4)]
    lib.nisqa_window_pair_counts(*args, *[_ptr(a, C.c_int32) for a in out], k.value)
    return tuple(out)


def _ptr(a, ct):
    return a.ctypes.data_as(C.POINTER(ct))


def feed_rows(cfg, sample_rate, window, hop_frames, held, n_samples, end=None):
    """(feed int32[N], index int64[N], n_segments int32[N], status int32[N]) of the windows a push of ``n_samples`` samples
    (and ``end`` flags) to feeds that hold ``held`` samples emits, in feed then window order (nisqa_feed_rows, host
    arithmetic)"""
    lib = load_library()
    held = np.ascontiguousarray(held, dtype=np.int64)
    ns = np.ascontiguousarray(n_samples, dtype=np.int64)
    e = None if end is None else np.ascontiguousarray(end, dtype=np.uint8)
    n = C.c_int64()
    args = (C.byref(cfg), int(sample_rate), int(window), int(hop_frames), len(held), _ptr(held, C.c_int64),
            _ptr(ns, C.c_int64), None if e is None else _ptr(e, C.c_uint8), C.byref(n))
    rc = lib.nisqa_feed_rows(*args, None, None, None, None, 0)
    if rc != 0:
        raise EngineError("nisqa_feed_rows failed (%d): window %d, hop_frames %d at %d Hz" % (rc, window, hop_frames,
                                                                                              sample_rate))
    feed, index = np.empty(n.value, np.int32), np.empty(n.value, np.int64)
    nseg, status = np.empty(n.value, np.int32), np.empty(n.value, np.int32)
    lib.nisqa_feed_rows(*args, _ptr(feed, C.c_int32), _ptr(index, C.c_int64), _ptr(nseg, C.c_int32),
                        _ptr(status, C.c_int32), n.value)
    return feed, index, nseg, status


def feed_pair_rows(cfg, sample_rate, window, hop_frames, margin_frames, held, ref_held, n_samples, ref_n_samples,
                   end=None):
    """(feed int32[N], index int64[N], n_segments, status, ref_n_segments, ref_status int32[N]) of the window pairs a push
    of ``n_samples`` degraded and ``ref_n_samples`` reference samples (and ``end`` flags) to pair feeds that hold
    ``held`` / ``ref_held`` samples emits, in feed then pair order (nisqa_feed_pair_rows, host arithmetic)"""
    lib = load_library()
    arrs = [np.ascontiguousarray(a, dtype=np.int64) for a in (held, ref_held, n_samples, ref_n_samples)]
    e = None if end is None else np.ascontiguousarray(end, dtype=np.uint8)
    n = C.c_int64()
    args = (C.byref(cfg), int(sample_rate), int(window), int(hop_frames), int(margin_frames), len(arrs[0]),
            *[_ptr(a, C.c_int64) for a in arrs], None if e is None else _ptr(e, C.c_uint8), C.byref(n))
    rc = lib.nisqa_feed_pair_rows(*args, None, None, None, None, None, None, 0)
    if rc != 0:
        raise EngineError("nisqa_feed_pair_rows failed (%d): window %d, hop_frames %d, margin_frames %d at %d Hz"
                          % (rc, window, hop_frames, margin_frames, sample_rate))
    feed, index = np.empty(n.value, np.int32), np.empty(n.value, np.int64)
    out = [np.empty(n.value, np.int32) for _ in range(4)]
    lib.nisqa_feed_pair_rows(*args, _ptr(feed, C.c_int32), _ptr(index, C.c_int64), *[_ptr(a, C.c_int32) for a in out],
                             n.value)
    return (feed, index) + tuple(out)


class Engine(object):
    """One engine per GPU (rank)."""

    def __init__(self, cfg, device=0):
        self.lib = load_library()
        self.cfg = cfg
        self.n_out = cfg.n_out
        self.h = C.c_void_p()
        rc = self.lib.nisqa_create(C.byref(self.h), int(device), C.byref(cfg))
        if rc != 0:
            msg = self._err()
            if self.h:
                self.lib.nisqa_destroy(self.h)
                self.h = C.c_void_p()
            raise EngineError("nisqa_create failed (%d): %s" % (rc, msg))
        self.device = int(device)
        self._feeds = set()                 # nisqa_feed handles, destroyed before the engine
        pools = getattr(cfg, "cnn_pools", None)
        if pools is not None:
            self.set_cnn_pools(pools)

    def _err(self):
        m = self.lib.nisqa_last_error(self.h)
        return m.decode() if m else ""

    def _check(self, rc, what):
        if rc != 0:
            raise EngineError("%s failed (%d): %s" % (what, rc, self._err()))

    def drain(self):
        """Abandon the submissions in flight (their buffers may be freed afterwards)."""
        if getattr(self, "h", None):
            self.lib.nisqa_drain(self.h)

    def close(self):
        if getattr(self, "h", None):
            for f in list(getattr(self, "_feeds", ())):
                self.feed_destroy(f)
            self.lib.nisqa_drain(self.h)
            self.lib.nisqa_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, state_dict):
        """state_dict: name -> torch.Tensor | ndarray, straight from the checkpoint."""
        keep, arr = [], (NisqaTensor * len(state_dict))()
        n = 0
        for name, t in state_dict.items():
            a = t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)
            if a.dtype != np.float32 or a.ndim > 4:
                continue                          # num_batches_tracked (int64) is not consumed
            a = np.ascontiguousarray(a)
            nm = name.encode()
            keep.append((a, nm))
            arr[n].name = nm
            arr[n].data = a.ctypes.data_as(C.POINTER(C.c_float))
            arr[n].ndim = a.ndim
            for d in range(a.ndim):
                arr[n].dims[d] = a.shape[d]
            n += 1
        self._check(self.lib.nisqa_load_weights(self.h, arr, n), "nisqa_load_weights")

    # ------------------------------------------------------------------ predict
    def predict_pcm(self, clips, sample_rates):
        """clips: list of 1-D contiguous int16 (all) or float32 (all) host arrays.
        Returns (scores [n, n_out] float32, n_segments int32[n], status int32[n])."""
        n = len(clips)
        if n == 0:
            return (np.zeros((0, self.n_out), np.float32), np.zeros(0, np.int32), np.zeros(0, np.int32))
        dt = clips[0].dtype
        if any(c.dtype != dt for c in clips):
            clips = [c if c.dtype == np.float32 else c.astype(np.float32) / np.float32(32768.0) for c in clips]
            dt = np.dtype(np.float32)
        if dt == np.int16:
            fmt = FMT_S16
        elif dt == np.float32:
            fmt = FMT_F32
        else:
            raise ValueError("clips must be int16 or float32")
        clips = [np.ascontiguousarray(c) for c in clips]
        ptrs = (C.c_void_p * n)(*[c.ctypes.data for c in clips])
        ns = np.array([c.shape[0] for c in clips], dtype=np.int64)
        sr = np.ascontiguousarray(sample_rates, dtype=np.int32)
        scores = np.empty((n, self.n_out), dtype=np.float32)
        nseg = np.empty(n, dtype=np.int32)
        status = np.empty(n, dtype=np.int32)
        rc = self.lib.nisqa_predict_pcm(
            self.h, n, ptrs, ns.ctypes.data_as(C.POINTER(C.c_int64)),
            sr.ctypes.data_as(C.POINTER(C.c_int32)), fmt,
            scores.ctypes.data_as(C.POINTER(C.c_float)), nseg.ctypes.data_as(C.POINTER(C.c_int32)),
            status.ctypes.data_as(C.POINTER(C.c_int32)))
        self._check(rc, "nisqa_predict_pcm")
        return scores, nseg, status

    def resample_device(self, x, sr_orig, sr_new):
        """One int16 / float32 clip converted on the device (csrc/resample_gpu.cu) -> float32 at sr_new."""
        from . import resample as _rs
        n_out = _rs.out_len(x.shape[0], sr_orig, sr_new)              # (also sets the interpolation table once)
        x = np.ascontiguousarray(x)
        fmt = FMT_S16 if x.dtype == np.int16 else FMT_F32
        if fmt == FMT_F32 and x.dtype != np.float32:
            raise ValueError("clips must be int16 or float32")
        y = np.empty(max(n_out, 1), dtype=np.float32)
        got = self.lib.nisqa_resample_device(self.h, x.ctypes.data, x.shape[0], fmt, int(sr_orig), int(sr_new),
                                             y.ctypes.data_as(C.POINTER(C.c_float)), y.shape[0])
        if got < 0:
            self._check(got, "nisqa_resample_device")
        return y[:got]

    def predict_pcm_resampled(self, clips, sample_rates, target_sr):
        """predict_pcm for checkpoints with ``ms_sr``: clips at their own rates are converted to ``target_sr`` on the
        device and scored there.  Synchronous.  Returns (scores, n_segments, status)."""
        from . import resample as _rs
        _rs.out_len(1, 1, 1)                                          # the interpolation table is set once
        n = len(clips)
        if n == 0:
            return (np.zeros((0, self.n_out), np.float32), np.zeros(0, np.int32), np.zeros(0, np.int32))
        dt = clips[0].dtype
        if any(c.dtype != dt for c in clips):
            clips = [c if c.dtype == np.float32 else c.astype(np.float32) / np.float32(32768.0) for c in clips]
            dt = np.dtype(np.float32)
        if dt not in (np.dtype(np.int16), np.dtype(np.float32)):
            raise ValueError("clips must be int16 or float32")
        clips = [np.ascontiguousarray(c) for c in clips]
        ptrs = (C.c_void_p * n)(*[c.ctypes.data for c in clips])
        ns = np.array([c.shape[0] for c in clips], dtype=np.int64)
        sr = np.ascontiguousarray(sample_rates, dtype=np.int32)
        scores = np.empty((n, self.n_out), dtype=np.float32)
        nseg = np.empty(n, dtype=np.int32)
        status = np.empty(n, dtype=np.int32)
        rc = self.lib.nisqa_predict_pcm_resampled(
            self.h, n, ptrs, ns.ctypes.data_as(C.POINTER(C.c_int64)), sr.ctypes.data_as(C.POINTER(C.c_int32)),
            FMT_S16 if dt == np.int16 else FMT_F32, int(target_sr), scores.ctypes.data_as(C.POINTER(C.c_float)),
            nseg.ctypes.data_as(C.POINTER(C.c_int32)), status.ctypes.data_as(C.POINTER(C.c_int32)))
        self._check(rc, "nisqa_predict_pcm_resampled")
        return scores, nseg, status

    def submit_pcm(self, clips, sample_rates):
        """Asynchronous predict_pcm: returns a handle; ``wait(handle)`` -> (scores, n_segments, status).
        Up to six submissions are in flight (H2D of the next batch overlaps this batch's kernels)."""
        n = len(clips)
        dt = clips[0].dtype if n else np.dtype(np.int16)
        if any(c.dtype != dt for c in clips):
            clips = [c if c.dtype == np.float32 else c.astype(np.float32) / np.float32(32768.0) for c in clips]
            dt = np.dtype(np.float32)
        if dt not in (np.dtype(np.int16), np.dtype(np.float32)):
            raise ValueError("clips must be int16 or float32")
        fmt = FMT_S16 if dt == np.int16 else FMT_F32
        clips = [np.ascontiguousarray(c) for c in clips]
        ptrs = (C.c_void_p * max(n, 1))(*[c.ctypes.data for c in clips])
        ns = np.array([c.shape[0] for c in clips], dtype=np.int64)
        sr = np.ascontiguousarray(sample_rates, dtype=np.int32)
        scores = np.empty((n, self.n_out), dtype=np.float32)
        nseg = np.empty(n, dtype=np.int32)
        status = np.empty(n, dtype=np.int32)
        ticket = C.c_int64(0)
        rc = self.lib.nisqa_submit_pcm(
            self.h, n, ptrs, ns.ctypes.data_as(C.POINTER(C.c_int64)), sr.ctypes.data_as(C.POINTER(C.c_int32)),
            fmt, scores.ctypes.data_as(C.POINTER(C.c_float)), nseg.ctypes.data_as(C.POINTER(C.c_int32)),
            status.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(ticket))
        self._check(rc, "nisqa_submit_pcm")
        return (ticket.value, scores, nseg, status, clips, ptrs, ns, sr)      # keeps the buffers alive

    def submit_pcm_pairs(self, clips, sample_rates, refs, ref_sample_rates, ref_index):
        """:meth:`submit_pcm` for NISQA_DE pairs whose references repeat: pair p is ``clips[p]`` and ``refs[ref_index[p]]``;
        each reference is uploaded and computed once per engine pass.  Returns a handle; ``wait(handle)`` -> (scores
        [n_pairs, n_out], n_segments [n_pairs], status [n_pairs]); ``handle[4]`` / ``handle[5]`` are the references'
        n_segments / status [n_refs]."""
        n, u = len(clips), len(refs)
        every = list(clips) + list(refs)
        if every and any(c.dtype != every[0].dtype for c in every):
            every = [c if c.dtype == np.float32 else c.astype(np.float32) / np.float32(32768.0) for c in every]
        dt = every[0].dtype if every else np.dtype(np.int16)
        if dt not in (np.dtype(np.int16), np.dtype(np.float32)):
            raise ValueError("clips must be int16 or float32")
        every = [np.ascontiguousarray(c) for c in every]
        ptrs = (C.c_void_p * max(n, 1))(*[c.ctypes.data for c in every[:n]])
        ref_ptrs = (C.c_void_p * max(u, 1))(*[c.ctypes.data for c in every[n:]])
        ns = np.array([c.shape[0] for c in every[:n]], dtype=np.int64)
        ref_ns = np.array([c.shape[0] for c in every[n:]], dtype=np.int64)
        sr = np.ascontiguousarray(sample_rates, dtype=np.int32)
        ref_sr = np.ascontiguousarray(ref_sample_rates, dtype=np.int32)
        idx = np.ascontiguousarray(ref_index, dtype=np.int32)
        scores = np.empty((n, self.n_out), dtype=np.float32)
        nseg, status = np.empty(n, dtype=np.int32), np.empty(n, dtype=np.int32)
        ref_nseg, ref_status = np.empty(u, dtype=np.int32), np.empty(u, dtype=np.int32)
        ticket = C.c_int64(0)
        p32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))      # noqa: E731
        rc = self.lib.nisqa_submit_pcm_pairs(
            self.h, n, ptrs, ns.ctypes.data_as(C.POINTER(C.c_int64)), p32(sr), u, ref_ptrs,
            ref_ns.ctypes.data_as(C.POINTER(C.c_int64)), p32(ref_sr), p32(idx), FMT_S16 if dt == np.int16 else FMT_F32,
            scores.ctypes.data_as(C.POINTER(C.c_float)), p32(nseg), p32(status), p32(ref_nseg), p32(ref_status),
            C.byref(ticket))
        self._check(rc, "nisqa_submit_pcm_pairs")
        return (ticket.value, scores, nseg, status, ref_nseg, ref_status, every, ptrs, ref_ptrs, ns, ref_ns, sr, ref_sr, idx)

    def wait(self, handle):
        if handle[0] is not None:             # (None: a synchronous call's results wrapped as a handle)
            self._check(self.lib.nisqa_wait(self.h, handle[0]), "nisqa_wait")
        return handle[1], handle[2], handle[3]

    def submit_pcm_ptrs(self, ptrs, n_samples, sample_rates, fmt, scores_out, nseg, status):
        """Raw-pointer asynchronous variant (bench e2e).  Returns the ticket."""
        ticket = C.c_int64(0)
        rc = self.lib.nisqa_submit_pcm(
            self.h, len(n_samples), ptrs, n_samples.ctypes.data_as(C.POINTER(C.c_int64)),
            sample_rates.ctypes.data_as(C.POINTER(C.c_int32)), fmt,
            scores_out.ctypes.data_as(C.POINTER(C.c_float)), nseg.ctypes.data_as(C.POINTER(C.c_int32)),
            status.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(ticket))
        self._check(rc, "nisqa_submit_pcm")
        return ticket.value

    def wait_ticket(self, ticket):
        self._check(self.lib.nisqa_wait(self.h, int(ticket)), "nisqa_wait")

    def predict_pcm_ptrs(self, ptrs, n_samples, sample_rates, fmt, scores_out):
        """Raw-pointer variant (bench e2e: pinned host buffers).  ptrs: ctypes array of void*."""
        n = len(n_samples)
        nseg = np.empty(n, dtype=np.int32)
        status = np.empty(n, dtype=np.int32)
        rc = self.lib.nisqa_predict_pcm(
            self.h, n, ptrs, n_samples.ctypes.data_as(C.POINTER(C.c_int64)),
            sample_rates.ctypes.data_as(C.POINTER(C.c_int32)), fmt,
            scores_out.ctypes.data_as(C.POINTER(C.c_float)),
            nseg.ctypes.data_as(C.POINTER(C.c_int32)), status.ctypes.data_as(C.POINTER(C.c_int32)))
        self._check(rc, "nisqa_predict_pcm")
        return nseg, status

    def predict_pcm_device(self, pcm_dev_ptr, offsets, n_samples, sample_rates, fmt, scores_dev_ptr, sync=True):
        """Packed PCM already in device memory (bench 'inputs resident in HBM' figure)."""
        n = len(n_samples)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        n_samples = np.ascontiguousarray(n_samples, dtype=np.int64)
        sr = np.ascontiguousarray(sample_rates, dtype=np.int32)
        nseg = np.empty(n, dtype=np.int32)
        status = np.empty(n, dtype=np.int32)
        rc = self.lib.nisqa_predict_pcm_device(
            self.h, n, C.c_void_p(pcm_dev_ptr), offsets.ctypes.data_as(C.POINTER(C.c_int64)),
            n_samples.ctypes.data_as(C.POINTER(C.c_int64)), sr.ctypes.data_as(C.POINTER(C.c_int32)),
            fmt, C.c_void_p(scores_dev_ptr), nseg.ctypes.data_as(C.POINTER(C.c_int32)),
            status.ctypes.data_as(C.POINTER(C.c_int32)), 1 if sync else 0)
        self._check(rc, "nisqa_predict_pcm_device")
        return nseg, status

    def predict_device_batch(self, stream, deg, scores_dev_ptr, ref=None, target_sr=0):
        """Clips already in device memory, ordered on the CUDA stream ``stream`` (a cudaStream_t as an int; 0: the
        legacy default stream): ``deg`` / ``ref`` are :func:`device_batch` tuples (``ref``: NISQA_DE only), ``target_sr``
        the checkpoint's ``ms_sr`` (0: none; every clip is converted to it on the device), the scores
        go to ``scores_dev_ptr`` ([rows, n_out] fp32 device memory; rows = n_clips, NISQA_DE 2 n_clips).  Returns
        (n_segments int32[rows], status int32[rows]), valid on return; the scores are valid in ``stream``'s order."""
        return self._device_batch(stream, deg, scores_dev_ptr, ref, target_sr, None)

    def predict_device_batch_segments(self, stream, deg, scores_dev_ptr, seg_scores_ptr, seg_weights_ptr, n_rows, ref=None,
                                      target_sr=0):
        """:meth:`predict_device_batch` that also writes every segment's score and pooling weight to the device arrays
        ``seg_scores_ptr`` / ``seg_weights_ptr`` ([n_rows, n_out] fp32 each; one row per segment of every OK clip in
        clip order, none for NISQA_DE's reference clips; include/nisqa_b200.h nisqa_segment_out).  Raises EngineError,
        with nothing enqueued, when ``n_rows`` is too small."""
        seg = NisqaSegmentOut(scores=seg_scores_ptr or None, weights=seg_weights_ptr or None, n_rows=int(n_rows))
        return self._device_batch(stream, deg, scores_dev_ptr, ref, target_sr, seg)

    def embedding_width(self):
        """The width of the embedding rows of the loaded checkpoint (nisqa_embedding_width)"""
        w = C.c_int32()
        self._check(self.lib.nisqa_embedding_width(self.h, C.byref(w)), "nisqa_embedding_width")
        return int(w.value)

    def predict_device_batch_embeddings(self, stream, deg, scores_dev_ptr, pooled_ptr, rows_ptr, n_rows, ref=None,
                                        target_sr=0):
        """:meth:`predict_device_batch` that also writes each pooling head's pooled vector to ``pooled_ptr`` ([rows,
        n_out, width] fp32 device memory, rows as the scores) and, unless ``rows_ptr`` is 0, every segment's row to
        ``rows_ptr`` ([n_rows, width] fp32; the row table of :meth:`predict_device_batch_segments`;
        include/nisqa_b200.h nisqa_embedding_out).  Raises EngineError, with nothing enqueued, when ``n_rows`` is too
        small."""
        emb = NisqaEmbeddingOut(pooled=pooled_ptr or None, rows=rows_ptr or None, n_rows=int(n_rows))
        return self._device_batch(stream, deg, scores_dev_ptr, ref, target_sr, emb)

    def predict_device_batch_alignment(self, stream, deg, ref, scores_dev_ptr, al, target_sr=0):
        """:meth:`predict_device_batch` of a NISQA_DE engine that also writes the alignment of every degraded segment to
        ``al``, a :class:`NisqaAlignmentOut` of device arrays (one row per segment of every OK degraded clip in clip
        order; include/nisqa_b200.h nisqa_alignment_out).  Raises EngineError, with nothing enqueued, for a refused call
        (a single-ended engine, a null array, a too-small ``al.n_rows``)."""
        return self._device_batch(stream, deg, scores_dev_ptr, ref, target_sr, al)

    def predict_device_batch_shared_ref(self, stream, deg, ref, ref_index, scores_dev_ptr, out=None, target_sr=0):
        """:meth:`predict_device_batch` of a NISQA_DE engine whose pairs share references: pair p is clip p of ``deg`` and
        clip ``ref_index[p]`` of ``ref`` (host ints); each reference is computed once per engine pass.  The scores go to
        ``scores_dev_ptr`` ([n_pairs, n_out], one row per pair); ``out``: None or a :class:`NisqaSegmentOut`,
        :class:`NisqaEmbeddingOut` (pooled [n_pairs, n_out, width]) or :class:`NisqaAlignmentOut`.  Returns (n_segments,
        status) int32[n_pairs] and (ref_n_segments, ref_status) int32[n_refs], valid on return."""
        if target_sr:
            from . import resample as _rs
            _rs.out_len(1, 1, 1)                                      # the interpolation table is set once
        n, u = deg[0].n_clips, ref[0].n_clips
        idx = None if ref_index is None else np.ascontiguousarray(ref_index, dtype=np.int32)
        nseg, status = np.empty(n, dtype=np.int32), np.empty(n, dtype=np.int32)
        ref_nseg, ref_status = np.empty(max(u, 0), dtype=np.int32), np.empty(max(u, 0), dtype=np.int32)
        outs = [None, None, None]
        for k, t in enumerate((NisqaSegmentOut, NisqaEmbeddingOut, NisqaAlignmentOut)):
            if isinstance(out, t):
                outs[k] = C.byref(out)
        p32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))      # noqa: E731
        self._check(self.lib.nisqa_predict_device_batch_shared_ref(
            self.h, C.c_void_p(stream or None), C.byref(deg[0]), C.byref(ref[0]),
            p32(idx) if idx is not None else None, int(target_sr or 0), C.c_void_p(scores_dev_ptr), *outs,
            p32(nseg), p32(status), p32(ref_nseg), p32(ref_status)), "nisqa_predict_device_batch_shared_ref")
        return nseg, status, ref_nseg, ref_status

    def predict_device_windows(self, stream, rec, scores_dev_ptr, n_rows, window, hop_frames, target_sr=0):
        """Windows of the recordings ``rec`` (a :func:`device_batch` tuple) ordered on ``stream``: ``window`` samples and a
        hop of ``hop_frames`` mel frames at the model rate (``target_sr``, else the batch's rate), the scores of every
        window to ``scores_dev_ptr`` ([n_rows, n_out] fp32 device memory, recording after recording).  Returns (n_segments,
        status) int32[windows], valid on return; raises EngineError, with nothing enqueued, for a refused call."""
        if target_sr:
            from . import resample as _rs
            _rs.out_len(1, 1, 1)                                      # the interpolation table is set once
        n = max(int(n_rows), 0)
        nseg, status = np.empty(n, dtype=np.int32), np.empty(n, dtype=np.int32)
        self._check(self.lib.nisqa_predict_device_windows(
            self.h, C.c_void_p(stream or None), C.byref(rec[0]), int(target_sr or 0), int(window), int(hop_frames),
            C.c_void_p(scores_dev_ptr), int(n_rows), nseg.ctypes.data_as(C.POINTER(C.c_int32)),
            status.ctypes.data_as(C.POINTER(C.c_int32))), "nisqa_predict_device_windows")
        return nseg, status

    def predict_device_window_pairs(self, stream, deg, ref, scores_dev_ptr, n_rows, window, hop_frames, margin_frames,
                                    target_sr=0):
        """Window pairs of the degraded recordings ``deg`` and their references ``ref`` (:func:`device_batch` tuples)
        ordered on ``stream``: the windows of :meth:`predict_device_windows` and reference windows ``margin_frames`` mel
        frames wider on either side; each pair's score to ``scores_dev_ptr`` ([n_rows, n_out] fp32 device memory, one row
        per pair, recording after recording).  Returns (n_segments, status, ref_n_segments, ref_status) int32[pairs],
        valid on return; raises EngineError, with nothing enqueued, for a refused call."""
        if target_sr:
            from . import resample as _rs
            _rs.out_len(1, 1, 1)                                      # the interpolation table is set once
        n = max(int(n_rows), 0)
        out = [np.empty(n, dtype=np.int32) for _ in range(4)]
        self._check(self.lib.nisqa_predict_device_window_pairs(
            self.h, C.c_void_p(stream or None), C.byref(deg[0]), C.byref(ref[0]), int(target_sr or 0), int(window),
            int(hop_frames), int(margin_frames), C.c_void_p(scores_dev_ptr), int(n_rows),
            *[_ptr(a, C.c_int32) for a in out]), "nisqa_predict_device_window_pairs")
        return tuple(out)

    def predict_device_window_pairs_alignment(self, stream, deg, ref, scores_dev_ptr, n_rows, window, hop_frames,
                                              margin_frames, al, target_sr=0):
        """:meth:`predict_device_window_pairs` that also writes the alignment of every segment of each pair's degraded
        window to ``al`` (:class:`NisqaAlignmentOut`; the pairs in order, include/nisqa_b200.h
        nisqa_predict_device_window_pairs_alignment).  Returns what :meth:`predict_device_window_pairs` returns."""
        if target_sr:
            from . import resample as _rs
            _rs.out_len(1, 1, 1)                                      # the interpolation table is set once
        n = max(int(n_rows), 0)
        out = [np.empty(n, dtype=np.int32) for _ in range(4)]
        self._check(self.lib.nisqa_predict_device_window_pairs_alignment(
            self.h, C.c_void_p(stream or None), C.byref(deg[0]), C.byref(ref[0]), int(target_sr or 0), int(window),
            int(hop_frames), int(margin_frames), C.c_void_p(scores_dev_ptr), int(n_rows), C.byref(al),
            *[_ptr(a, C.c_int32) for a in out]), "nisqa_predict_device_window_pairs_alignment")
        return tuple(out)

    def feed_create(self, n_feeds, sample_rate, window, hop_frames, max_push):
        """A feed object (nisqa_feed_create) -> its handle (an int)"""
        h = C.c_void_p()
        self._check(self.lib.nisqa_feed_create(self.h, C.byref(h), int(n_feeds), int(sample_rate), int(window),
                                               int(hop_frames), int(max_push)), "nisqa_feed_create")
        self._feeds.add(h.value)
        return h.value

    def feed_push(self, feed, stream, chunk, end, scores_dev_ptr, n_rows):
        """nisqa_feed_push of ``chunk`` (a :func:`device_batch` tuple, 0 samples allowed) and ``end`` (uint8[n_feeds] or
        None) ordered on ``stream``; the scores of the completed windows to ``scores_dev_ptr`` ([n_rows, n_out] fp32 device
        memory).  Returns (feed, index, n_segments, status) arrays of n_rows entries, the push's windows first (size
        n_rows with :func:`feed_rows`), valid on return; raises EngineError, with nothing enqueued, for a refused push."""
        n = max(int(n_rows), 0)
        fo, index = np.empty(n, np.int32), np.empty(n, np.int64)
        nseg, status = np.empty(n, np.int32), np.empty(n, np.int32)
        e = None if end is None else np.ascontiguousarray(end, dtype=np.uint8)
        self._check(self.lib.nisqa_feed_push(
            C.c_void_p(self._feed(feed)), C.c_void_p(stream or None), C.byref(chunk[0]),
            None if e is None else _ptr(e, C.c_uint8), C.c_void_p(scores_dev_ptr), int(n_rows), _ptr(fo, C.c_int32),
            _ptr(index, C.c_int64), _ptr(nseg, C.c_int32), _ptr(status, C.c_int32)), "nisqa_feed_push")
        return fo, index, nseg, status

    def feed_pair_create(self, n_feeds, sample_rate, window, hop_frames, margin_frames, max_push, max_skew):
        """A pair feed object (nisqa_feed_pair_create) -> its handle (an int)"""
        h = C.c_void_p()
        self._check(self.lib.nisqa_feed_pair_create(self.h, C.byref(h), int(n_feeds), int(sample_rate), int(window),
                                                    int(hop_frames), int(margin_frames), int(max_push), int(max_skew)),
                    "nisqa_feed_pair_create")
        self._feeds.add(h.value)
        return h.value

    def feed_pair_push(self, feed, stream, deg, ref, end, scores_dev_ptr, n_rows):
        """nisqa_feed_pair_push of ``deg`` and ``ref`` (:func:`device_batch` tuples, 0 samples allowed) and ``end``
        (uint8[n_feeds] or None) ordered on ``stream``; the scores of the completed pairs to ``scores_dev_ptr`` ([n_rows,
        n_out] fp32 device memory).  Returns (feed, index, n_segments, status, ref_n_segments, ref_status) arrays of
        n_rows entries (size n_rows with :func:`feed_pair_rows`), valid on return; raises EngineError, with nothing
        enqueued, for a refused push."""
        n = max(int(n_rows), 0)
        fo, index = np.empty(n, np.int32), np.empty(n, np.int64)
        out = [np.empty(n, np.int32) for _ in range(4)]
        e = None if end is None else np.ascontiguousarray(end, dtype=np.uint8)
        self._check(self.lib.nisqa_feed_pair_push(
            C.c_void_p(self._feed(feed)), C.c_void_p(stream or None), C.byref(deg[0]), C.byref(ref[0]),
            None if e is None else _ptr(e, C.c_uint8), C.c_void_p(scores_dev_ptr), int(n_rows), _ptr(fo, C.c_int32),
            _ptr(index, C.c_int64), *[_ptr(a, C.c_int32) for a in out]), "nisqa_feed_pair_push")
        return (fo, index) + tuple(out)

    def _feed(self, feed):
        if feed not in self._feeds:
            raise EngineError("the feed object is closed")
        return feed

    def feed_device_bytes(self, feed):
        return int(self.lib.nisqa_feed_device_bytes(C.c_void_p(self._feed(feed))))

    def feed_destroy(self, feed):
        if feed in self._feeds:
            self._feeds.discard(feed)
            self.lib.nisqa_feed_destroy(C.c_void_p(feed))

    def _device_batch(self, stream, deg, scores_dev_ptr, ref, target_sr, out):
        rows = deg[0].n_clips * (2 if ref is not None else 1)
        if target_sr:
            from . import resample as _rs
            _rs.out_len(1, 1, 1)                                      # the interpolation table is set once
        nseg = np.empty(rows, dtype=np.int32)
        status = np.empty(rows, dtype=np.int32)
        args = (self.h, C.c_void_p(stream or None), C.byref(deg[0]), C.byref(ref[0]) if ref is not None else None,
                int(target_sr or 0), C.c_void_p(scores_dev_ptr))
        outs = (nseg.ctypes.data_as(C.POINTER(C.c_int32)), status.ctypes.data_as(C.POINTER(C.c_int32)))
        if out is None:
            self._check(self.lib.nisqa_predict_device_batch(*args, *outs), "nisqa_predict_device_batch")
        elif isinstance(out, NisqaAlignmentOut):
            self._check(self.lib.nisqa_predict_device_batch_alignment(*args, C.byref(out), *outs),
                        "nisqa_predict_device_batch_alignment")
        elif isinstance(out, NisqaSegmentOut):
            self._check(self.lib.nisqa_predict_device_batch_segments(*args, C.byref(out), *outs),
                        "nisqa_predict_device_batch_segments")
        else:
            self._check(self.lib.nisqa_predict_device_batch_embeddings(*args, C.byref(out), *outs),
                        "nisqa_predict_device_batch_embeddings")
        return nseg, status

    # ------------------------------------------------------------------ introspection
    def stage_dump(self, stage):
        n = self.lib.nisqa_stage_dump(self.h, int(stage), None, 0)
        if n < 0:
            raise EngineError("nisqa_stage_dump failed (%d): %s" % (n, self._err()))
        out = np.empty(int(n), dtype=np.float32)
        if n:
            m = self.lib.nisqa_stage_dump(self.h, int(stage), out.ctypes.data_as(C.POINTER(C.c_float)), n)
            if m < 0:
                raise EngineError("nisqa_stage_dump failed (%d): %s" % (m, self._err()))
        return out

    def mel_filterbank(self, sample_rate):
        out = np.empty((self.cfg.n_mels, self.cfg.n_fft // 2 + 1), dtype=np.float32)
        self._check(self.lib.nisqa_mel_filterbank(self.h, int(sample_rate),
                                                  out.ctypes.data_as(C.POINTER(C.c_float)), out.size),
                    "nisqa_mel_filterbank")
        return out

    def kernel_launches(self):
        return int(self.lib.nisqa_kernel_launches(self.h))

    def stream(self):
        return self.lib.nisqa_stream(self.h)

    def join(self):
        self._check(self.lib.nisqa_join(self.h), "nisqa_join")

    def set_profiling(self, on):
        self._check(self.lib.nisqa_set_profiling(self.h, 1 if on else 0), "nisqa_set_profiling")

    def set_option(self, name, value):
        self._check(self.lib.nisqa_set_option(self.h, name.encode(), int(value)), "nisqa_set_option")

    def set_cnn_pools(self, pools):
        """AdaptCNN's cnn_pool_1/2/3 ((h1, w1), (h2, w2), (h3, w3)) for the next load_state_dict"""
        flat = (C.c_int32 * 6)(*[int(v) for p in pools for v in p])
        self._check(self.lib.nisqa_set_cnn_pools(self.h, flat), "nisqa_set_cnn_pools")

    def group_ms(self, group):
        return float(self.lib.nisqa_group_ms(self.h, group.encode()))

    # ------------------------------------------------------------------ multi-GPU exchange
    def nccl_unique_id(self):
        buf = (C.c_char * 128)()
        self._check(self.lib.nisqa_nccl_unique_id(self.h, buf), "nisqa_nccl_unique_id")
        return bytes(buf)

    def nccl_init(self, world, rank, uid):
        buf = (C.c_char * 128).from_buffer_copy(uid)
        self._check(self.lib.nisqa_nccl_init(self.h, int(world), int(rank), buf), "nisqa_nccl_init")

    def set_gather_target(self, global_dev_ptr, rows):
        self._check(self.lib.nisqa_set_gather_target(self.h, C.c_void_p(global_dev_ptr), int(rows)), "nisqa_set_gather_target")

    def gather_nccl(self, local_dev_ptr, max_rows, global_dev_ptr, comm=None):
        self._check(self.lib.nisqa_gather_nccl(self.h, C.c_void_p(comm), C.c_void_p(local_dev_ptr),
                                               int(max_rows), C.c_void_p(global_dev_ptr)),
                    "nisqa_gather_nccl")
